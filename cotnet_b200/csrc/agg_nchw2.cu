// LocalConv 3x3 on NCHW tensors (the reference contract), second-generation kernels (sm_90a).
//
// Same arithmetic as agg_fwd_nchw_fast / agg_bwd_nchw_fast (agg_zeropad.cu) -- one thread owns the K*K weights of its
// pixels in registers and loops over the C/wc channels sharing them -- but:
//   * each thread owns PXV (4 or 2) consecutive pixels of a row and moves them with one 16/8-byte access;
//     the 3x3 neighbourhood of the group is 3 x (1 vector + 2 edge scalars) loads instead of 9 scalars per pixel;
//   * one CTA row of the grid per (sample, weight-channel) plane: no 64-bit index decomposition per element;
//   * interior fast path without any predication, edge path with zero fill;
//   * bf16/fp16 are widened to fp32 for the FMA (exact products, fp32 accumulation).
// Requires W % PXV == 0 (56, 28 -> 4; 14 -> 2); other widths use the first-generation scalar kernels.
#include "common.cuh"
#include "agg.cuh"

namespace cotb200 {

// fp32 accumulator times storage-type element (used where one factor is already fp32)
template <typename T> __device__ __forceinline__ float mulacc(float a, T b, float c) { return fmaf(a, to_acc(b), c); }

// A row segment of PXV pixels plus its left / right neighbour: v[0] = w0-1, v[1..PXV] = w0..w0+PXV-1, v[PXV+1] = w0+PXV
template <typename T, int PXV, bool CHECK>
__device__ __forceinline__ void load_row(const T* __restrict__ rowp, int w0, int W, bool row_ok, T (&v)[PXV + 2]) {
  const T z = Elem<T>::from(0.f);
  if (CHECK && !row_ok) {
#pragma unroll
    for (int i = 0; i < PXV + 2; ++i) v[i] = z;
    return;
  }
  const Pack<T, PXV> c = ld_pack<T, PXV>(rowp + w0);
#pragma unroll
  for (int i = 0; i < PXV; ++i) v[i + 1] = c.v[i];
  v[0] = (!CHECK || w0 > 0) ? __ldg(rowp + w0 - 1) : z;
  v[PXV + 1] = (!CHECK || w0 + PXV < W) ? __ldg(rowp + w0 + PXV) : z;
}

// ------------------------------------------------------------------------------------------------ forward
template <typename T, int PXV, bool CHECK>
__device__ __forceinline__ void nchw2_fwd_body(const T* __restrict__ xp, const T* __restrict__ wp, T* __restrict__ yp, int H,
                                               int W, int HW, int h, int w0, int rep, long long cstride) {
  // weights of the PXV pixels: wt[t][i]
  Pack<T, PXV> wt[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wt[t] = ld_pack<T, PXV>(wp + (long long)t * HW + h * W + w0);
  if (CHECK) {   // padded taps contribute 0: zero the weights whose tap falls outside for this pixel
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int dh = t / 3 - 1, dw = t % 3 - 1;
#pragma unroll
      for (int i = 0; i < PXV; ++i)
        if (!((unsigned)(h + dh) < (unsigned)H && (unsigned)(w0 + i + dw) < (unsigned)W)) wt[t].v[i] = Elem<T>::from(0.f);
    }
  }
#pragma unroll 2
  for (int j = 0; j < rep; ++j) {
    float acc[PXV];
#pragma unroll
    for (int i = 0; i < PXV; ++i) acc[i] = 0.f;
#pragma unroll
    for (int dh = -1; dh <= 1; ++dh) {
      T v[PXV + 2];
      load_row<T, PXV, CHECK>(xp + (h + dh) * W, w0, W, (unsigned)(h + dh) < (unsigned)H, v);
#pragma unroll
      for (int dw = -1; dw <= 1; ++dw)
#pragma unroll
        for (int i = 0; i < PXV; ++i) acc[i] = mfma<T>(wt[(dh + 1) * 3 + dw + 1].v[i], v[i + 1 + dw], acc[i]);
    }
    Pack<T, PXV> o;
#pragma unroll
    for (int i = 0; i < PXV; ++i) o.v[i] = Elem<T>::from(acc[i]);
    st_pack<T, PXV>(yp + h * W + w0, o);
    xp += cstride; yp += cstride;
  }
}

template <typename T, int PXV>
__global__ void __launch_bounds__(256)
agg3_fwd_nchw2_kernel(const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, int C, int H, int W, int wc, int rep,
                      long long y_sn) {
  const int HW = H * W, WQ = W / PXV;
  const int item = blockIdx.x * 256 + threadIdx.x;
  if (item >= H * WQ) return;
  const int h = item / WQ, w0 = (item - h * WQ) * PXV;
  const int plane = blockIdx.y;                       // n * wc + gch
  const int n = plane / wc, gch = plane - n * wc;
  const T* xp = x + ((long long)n * C + gch) * HW;
  const T* wp = w + (long long)plane * 9 * HW;
  T* yp = y + n * y_sn + (long long)gch * HW;
  const long long cs = (long long)wc * HW;
  const bool interior = h >= 1 && h + 1 < H && w0 >= 1 && w0 + PXV < W;
  if (interior) nchw2_fwd_body<T, PXV, false>(xp, wp, yp, H, W, HW, h, w0, rep, cs);
  else nchw2_fwd_body<T, PXV, true>(xp, wp, yp, H, W, HW, h, w0, rep, cs);
}

// ------------------------------------------------------------------------------------------------ backward (fused dX + dW)
//   dW[t][i]   = sum_j x_j[p_i + off_t] * dY_j[p_i]
//   dX_j[p_i]  = sum_t w[t][p_i - off_t] * dY_j[p_i - off_t]
template <typename T, int PXV, bool DX, bool DW, bool CHECK>
__device__ __forceinline__ void nchw2_bwd_body(const T* __restrict__ dp, const T* __restrict__ xp, const T* __restrict__ wp,
                                               T* __restrict__ dxp, T* __restrict__ dwp, int H, int W, int HW, int h, int w0,
                                               int rep, long long cstride) {
  float gw[9][PXV];
  T ws[9][PXV];           // DX: w[t] sampled at p - off_t
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int i = 0; i < PXV; ++i) gw[t][i] = 0.f;
  if (DX) {
#pragma unroll
    for (int dh = -1; dh <= 1; ++dh)
#pragma unroll
      for (int dw = -1; dw <= 1; ++dw) {
        const int t = (dh + 1) * 3 + dw + 1;
        T v[PXV + 2];
        // row h - dh of weight plane t, columns w0-1 .. w0+PXV; we need columns (w0 + i - dw)
        load_row<T, PXV, CHECK>(wp + (long long)t * HW + (h - dh) * W, w0, W, (unsigned)(h - dh) < (unsigned)H, v);
#pragma unroll
        for (int i = 0; i < PXV; ++i) ws[t][i] = v[i + 1 - dw];
      }
  }
  for (int j = 0; j < rep; ++j) {
    T dy[3][PXV + 2];
#pragma unroll
    for (int dh = -1; dh <= 1; ++dh) {
      if (DX || dh == 0) load_row<T, PXV, CHECK>(dp + (h + dh) * W, w0, W, (unsigned)(h + dh) < (unsigned)H, dy[dh + 1]);
    }
    if (DW) {
#pragma unroll
      for (int dh = -1; dh <= 1; ++dh) {
        T xv[PXV + 2];
        load_row<T, PXV, CHECK>(xp + (h + dh) * W, w0, W, (unsigned)(h + dh) < (unsigned)H, xv);
#pragma unroll
        for (int dw = -1; dw <= 1; ++dw)
#pragma unroll
          for (int i = 0; i < PXV; ++i)
            gw[(dh + 1) * 3 + dw + 1][i] = mfma<T>(xv[i + 1 + dw], dy[1][i + 1], gw[(dh + 1) * 3 + dw + 1][i]);
      }
    }
    if (DX) {
      float acc[PXV];
#pragma unroll
      for (int i = 0; i < PXV; ++i) acc[i] = 0.f;
#pragma unroll
      for (int dh = -1; dh <= 1; ++dh)
#pragma unroll
        for (int dw = -1; dw <= 1; ++dw)
#pragma unroll
          for (int i = 0; i < PXV; ++i)      // output pixel (h - dh, w - dw) read (h, w) through tap (dh, dw)
            acc[i] = mfma<T>(ws[(dh + 1) * 3 + dw + 1][i], dy[1 - dh][i + 1 - dw], acc[i]);
      Pack<T, PXV> o;
#pragma unroll
      for (int i = 0; i < PXV; ++i) o.v[i] = Elem<T>::from(acc[i]);
      st_pack<T, PXV>(dxp + h * W + w0, o);
    }
    dp += cstride; xp += cstride; dxp += cstride;
  }
  if (DW) {
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      Pack<T, PXV> o;
#pragma unroll
      for (int i = 0; i < PXV; ++i) o.v[i] = Elem<T>::from(gw[t][i]);
      st_pack<T, PXV>(dwp + (long long)t * HW + h * W + w0, o);
    }
  }
}

// 16-bit types: 2 CTAs per SM (the fused dX+dW variant otherwise takes 130 registers -> one 8-warp CTA per SM).  fp32 keeps
// its 172 registers (capping it to 128 spills; the large fp32 planes go through agg_nchw_tma.cu).
template <typename T, int PXV, bool DX, bool DW>
__global__ void __launch_bounds__(256, (sizeof(T) == 2 ? 2 : 1))
agg3_bwd_nchw2_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ dx,
                      T* __restrict__ dw, int C, int H, int W, int wc, int rep, long long dy_sn) {
  const int HW = H * W, WQ = W / PXV;
  const int item = blockIdx.x * 256 + threadIdx.x;
  if (item >= H * WQ) return;
  const int h = item / WQ, w0 = (item - h * WQ) * PXV;
  const int plane = blockIdx.y;
  const int n = plane / wc, gch = plane - n * wc;
  const T* dp = dy + n * dy_sn + (long long)gch * HW;
  const T* xp = x + ((long long)n * C + gch) * HW;
  const T* wp = w + (long long)plane * 9 * HW;
  T* dxp = dx + ((long long)n * C + gch) * HW;
  T* dwp = dw + (long long)plane * 9 * HW;
  const long long cs = (long long)wc * HW;
  const bool interior = h >= 1 && h + 1 < H && w0 >= 1 && w0 + PXV < W;
  if (interior) nchw2_bwd_body<T, PXV, DX, DW, false>(dp, xp, wp, dxp, dwp, H, W, HW, h, w0, rep, cs);
  else nchw2_bwd_body<T, PXV, DX, DW, true>(dp, xp, wp, dxp, dwp, H, W, HW, h, w0, rep, cs);
}

// ------------------------------------------------------------------------------------------------ host
template <typename T>
static int nchw2_pxv(int W, int HW, const void* a, const void* b, const void* c, const void* d, const void* e) {
  if constexpr (std::is_same<T, double>::value) return 0;
  for (int pxv = 4; pxv >= 2; pxv >>= 1) {
    if (W % pxv) continue;
    const uintptr_t m = (uintptr_t)(pxv * sizeof(T)) - 1;
    auto ok = [&](const void* p) { return !p || ((uintptr_t)p & m) == 0; };
    if (ok(a) && ok(b) && ok(c) && ok(d) && ok(e)) return pxv;
  }
  return 0;
}

// returns 1 if handled
template <typename T>
int nchw2_fwd(int N, int C, int H, int W, int wc, long long y_sn, const T* x, const T* w, T* y, cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    const int pxv = nchw2_pxv<T>(W, H * W, x, w, y, nullptr, nullptr);
    if (!pxv || (long long)N * wc > 65535 || (y_sn * (long long)sizeof(T)) % (pxv * sizeof(T))) return 0;
    dim3 grid((H * (W / pxv) + 255) / 256, N * wc);
    COTB200_PROF_B("agg3_fwd_nchw2", ((double)N * H * W) * (2.0 * C + 9.0 * wc) * sizeof(T));
    if (pxv == 4) agg3_fwd_nchw2_kernel<T, 4><<<grid, 256, 0, st>>>(x, w, y, C, H, W, wc, C / wc, y_sn);
    else agg3_fwd_nchw2_kernel<T, 2><<<grid, 256, 0, st>>>(x, w, y, C, H, W, wc, C / wc, y_sn);
    *rc = check_launch("agg3_fwd_nchw2");
    return 1;
  }
}

template <typename T>
int nchw2_bwd(int N, int C, int H, int W, int wc, long long dy_sn, const T* dy, const T* x, const T* w, T* dx, T* dw,
              cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    const int pxv = nchw2_pxv<T>(W, H * W, dy, x, w, dx, dw);
    if (!pxv || (long long)N * wc > 65535 || (dy_sn * (long long)sizeof(T)) % (pxv * sizeof(T))) return 0;
    dim3 grid((H * (W / pxv) + 255) / 256, N * wc);
    const int rep = C / wc;
    COTB200_PROF_B(dx && dw ? "agg3_bwd_nchw2_dxdw" : (dx ? "agg3_bwd_nchw2_dx" : "agg3_bwd_nchw2_dw"), ((double)N * H * W) * ((dx && dw ? 3.0 : 2.0) * C + (dx && dw ? 18.0 : 9.0) * wc) * sizeof(T));
#define NCHW2_LAUNCH(P)                                                                                              \
  if (dx && dw) agg3_bwd_nchw2_kernel<T, P, true, true><<<grid, 256, 0, st>>>(dy, x, w, dx, dw, C, H, W, wc, rep, dy_sn); \
  else if (dx) agg3_bwd_nchw2_kernel<T, P, true, false><<<grid, 256, 0, st>>>(dy, x, w, dx, dw, C, H, W, wc, rep, dy_sn); \
  else agg3_bwd_nchw2_kernel<T, P, false, true><<<grid, 256, 0, st>>>(dy, x, w, dx, dw, C, H, W, wc, rep, dy_sn);
    if (pxv == 4) { NCHW2_LAUNCH(4) } else { NCHW2_LAUNCH(2) }
#undef NCHW2_LAUNCH
    *rc = check_launch("agg3_bwd_nchw2");
    return 1;
  }
}

#define COTB200_INST2(T)                                                                                             \
  template int nchw2_fwd<T>(int, int, int, int, int, long long, const T*, const T*, T*, cudaStream_t, int*);          \
  template int nchw2_bwd<T>(int, int, int, int, int, long long, const T*, const T*, const T*, T*, T*, cudaStream_t, int*);
COTB200_INST2(float) COTB200_INST2(double) COTB200_INST2(__nv_bfloat16) COTB200_INST2(__half)

}  // namespace cotb200
