// LocalConv 3x3 on NHWC tensors, second-generation kernels (sm_90a).
//
// First-generation kernels (agg_zeropad.cu) are instruction-issue bound: most issued instructions per output are address
// arithmetic, not FMAs.  These kernels remove that overhead:
//   * bf16/fp16 operands are widened to fp32 (exact) and accumulated with fp32 FMAs;
//   * a 2-D grid gives every CTA one image row, so pixel coordinates need no runtime div/mod, and all tap offsets
//     are 32-bit immediates added to one base pointer;
//   * forward / dX: each thread produces PX=2 horizontally adjacent pixels of one 16-byte channel packet and
//     re-uses the 3x4 neighbourhood it loads for both (L1 wavefronts per pixel 18 -> 15);
//   * dW: lanes run over channels (coalesced 128-byte lines), the reduction over the 8 channels that share a weight
//     is a butterfly transpose-reduce across lanes (each lane ends up owning the 16-byte packet of one tap).
// Weight layouts: COTB200_NHWC (g*9+t, the torch channels_last view) for forward; COTB200_NHWC_TAP (tap-major chunks
// of gc = 8 weight channels, the block-internal layout) for forward, dX and dW.
#include "common.cuh"
#include "agg.cuh"

namespace cotb200 {


template <typename T, int VEC> __device__ __forceinline__ Pack<T, VEC> zero_pack() {
  Pack<T, VEC> z;
#pragma unroll
  for (int i = 0; i < VEC; ++i) z.v[i] = Elem<T>::from(0.f);
  return z;
}

struct G2 {
  int N, C, H, W, wc, Cf, wcf, rep, gc;      // gc: TAP chunk width (>= VEC, multiple of VEC); 0 = plain NHWC order
  int x_sn, x_sp, w_sn, w_sp, y_sn, y_sp;    // element strides (fit 32 bits: checked on the host)
};

// offset (elements) of the weight packet of tap t for weight channels g0..g0+VEC-1 inside a pixel's weight row
template <int VEC>
__device__ __forceinline__ int wpk_off_tap(int g0, int t, int gc) { return ((g0 / gc) * 9 + t) * gc + g0 % gc; }

// ------------------------------------------------------------------------------------------------ forward / dX
// MODE 0: forward   y[p,c]  = sum_t w[p][g(c),t]      * x[p + off_t][c]
// MODE 1: dX        dx[p,c] = sum_t w[p - off_t][g,t] * dy[p - off_t][c]          (TAP layout only)
// `a` is the tensor gathered at neighbour pixels (x or dy), `w` the weights, `o` the output.
// CHECK=false is the interior fast path: every tap is in range, no predication at all.
template <typename T, int VEC, int PX, bool TAP, int MODE, bool CHECK>
__device__ __forceinline__ void agg3_nhwc2_body(const T* __restrict__ ab, const T* __restrict__ wb, T* __restrict__ ob,
                                                const G2& g, int h, int w0, int g0, int a_sp, int o_sp) {
  float acc[PX][VEC];
#pragma unroll
  for (int p = 0; p < PX; ++p)
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[p][i] = 0.f;
  if (MODE == 0) {
    Pack<T, VEC> wk[PX][9];
#pragma unroll
    for (int p = 0; p < PX; ++p) {
      const T* wr = wb + (h * g.W + w0 + p) * g.w_sp;
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int off = TAP ? wpk_off_tap<VEC>(g0, t, g.gc) : g0 * 9 + t * VEC;
        wk[p][t] = (!CHECK || w0 + p < g.W) ? ld_pack<T, VEC>(wr + off) : zero_pack<T, VEC>();
      }
    }
#pragma unroll
    for (int dh = -1; dh <= 1; ++dh) {
      const int hh = h + dh;
      if (CHECK && (unsigned)hh >= (unsigned)g.H) continue;
      Pack<T, VEC> xv[PX + 2];
#pragma unroll
      for (int cpos = 0; cpos < PX + 2; ++cpos) {
        const int ww = w0 - 1 + cpos;
        xv[cpos] = (!CHECK || (unsigned)ww < (unsigned)g.W) ? ld_pack<T, VEC>(ab + (hh * g.W + ww) * a_sp) : zero_pack<T, VEC>();
      }
#pragma unroll
      for (int p = 0; p < PX; ++p)
#pragma unroll
        for (int dw = -1; dw <= 1; ++dw) {
          const int t = (dh + 1) * 3 + (dw + 1);
#pragma unroll
          for (int i = 0; i < VEC; ++i) {
            // plain order: element (i,t) sits at flat i*9+t of the 9 packets; TAP order: packet t, lane i
            const T wv = TAP ? wk[p][t].v[i] : wk[p][(i * 9 + t) / VEC].v[(i * 9 + t) % VEC];
            acc[p][i] = mfma<T>(wv, xv[p + dw + 1].v[i], acc[p][i]);
          }
        }
    }
  } else {
    // dX: neighbour position (h - dh, w - dw) contributes through ITS tap (dh, dw).  TAP layout: one packet per tap.
#pragma unroll
    for (int dh = -1; dh <= 1; ++dh) {
      const int hh = h - dh;
      if (CHECK && (unsigned)hh >= (unsigned)g.H) continue;
#pragma unroll
      for (int cpos = 0; cpos < PX + 2; ++cpos) {
        const int ww = w0 - 1 + cpos;                       // neighbour column
        if (CHECK && (unsigned)ww >= (unsigned)g.W) continue;
        const Pack<T, VEC> gv = ld_pack<T, VEC>(ab + (hh * g.W + ww) * a_sp);
        const T* wr = wb + (hh * g.W + ww) * g.w_sp;
#pragma unroll
        for (int p = 0; p < PX; ++p) {
          const int dw = p - (cpos - 1);                    // output column minus neighbour column (compile time)
          if (dw < -1 || dw > 1) continue;
          const int t = (dh + 1) * 3 + (dw + 1);
          const Pack<T, VEC> wv = ld_pack<T, VEC>(wr + wpk_off_tap<VEC>(g0, t, g.gc));
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[p][i] = mfma<T>(wv.v[i], gv.v[i], acc[p][i]);
        }
      }
    }
  }
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    if (!CHECK || w0 + p < g.W) {
      Pack<T, VEC> r;
#pragma unroll
      for (int i = 0; i < VEC; ++i) r.v[i] = Elem<T>::from(acc[p][i]);
      st_pack<T, VEC>(ob + (h * g.W + w0 + p) * o_sp, r);
    }
  }
}

template <typename T, int VEC, int PX, bool TAP, int MODE>
__global__ void __launch_bounds__(256)
agg3_nhwc2_kernel(const T* __restrict__ a, const T* __restrict__ w, T* __restrict__ o, G2 g) {
  const int CQ = g.C / VEC;
  const int item = blockIdx.x * 256 + threadIdx.x;
  const int q = item % CQ, wp = item / CQ;
  const int w0 = wp * PX;
  if (w0 >= g.W) return;
  const int row = blockIdx.y;
  const int n = row / g.H, h = row - n * g.H;
  const int c0 = q * VEC;
  const int g0 = (c0 / g.Cf) * g.wcf + (c0 % g.Cf) % g.wcf;
  const T* ab = a + (long long)n * (MODE == 0 ? g.x_sn : g.y_sn) + c0;
  const T* wb = w + (long long)n * g.w_sn;
  T* ob = o + (long long)n * (MODE == 0 ? g.y_sn : g.x_sn) + c0;
  const int a_sp = MODE == 0 ? g.x_sp : g.y_sp;
  const int o_sp = MODE == 0 ? g.y_sp : g.x_sp;
  const bool interior = h >= 1 && h + 1 < g.H && w0 >= 1 && w0 + PX < g.W;
  if (interior) agg3_nhwc2_body<T, VEC, PX, TAP, MODE, false>(ab, wb, ob, g, h, w0, g0, a_sp, o_sp);
  else agg3_nhwc2_body<T, VEC, PX, TAP, MODE, true>(ab, wb, ob, g, h, w0, g0, a_sp, o_sp);
}

// ------------------------------------------------------------------------------------------------ dW (TAP layout)
// dW[p, (g0+i), t] = sum_j x[p + off_t][cb + j*wcf + i] * dY[p][cb + j*wcf + i],  8 sharers j (rep == 8).
// Warp lane = gvl + GQW * j + 8*GQW * pixel_slot;  GQW = min(wc/VEC, 4) weight packets per warp row.
template <typename T, int VEC, int GQW>
__global__ void __launch_bounds__(256)
agg3_dw_nhwc2_kernel(const T* __restrict__ dy, const T* __restrict__ x, T* __restrict__ dw, G2 g, int GQ) {
  constexpr int PXW = 32 / (8 * GQW);                 // pixels per warp
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gvl = lane % GQW, j = (lane / GQW) % 8, slot = lane / (8 * GQW);
  // work item of this warp: (pixel group, gv group)
  const int gvgroups = GQ / GQW;                      // warps needed per pixel group to cover all weight packets
  const int witem = (blockIdx.x * 8 + warp);
  const int gvg = witem % gvgroups, pg = witem / gvgroups;
  const int wq = pg * PXW + slot;
  const int row = blockIdx.y;
  const int n = row / g.H, h = row - n * g.H;
  const bool active = wq < g.W;
  const int gv = gvg * GQW + gvl;
  const int g0 = gv * VEC;
  const int cb = (g0 / g.wcf) * g.Cf + g0 % g.wcf + j * g.wcf;     // this lane's channel packet
  float part[9][VEC];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int i = 0; i < VEC; ++i) part[t][i] = 0.f;
  if (active) {
    const Pack<T, VEC> gvv = ld_pack<T, VEC>(dy + (long long)n * g.y_sn + (h * g.W + wq) * g.y_sp + cb);
    const T* xb = x + (long long)n * g.x_sn + cb;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int hh = h + t / 3 - 1, ww = wq + t % 3 - 1;
      if ((unsigned)hh < (unsigned)g.H && (unsigned)ww < (unsigned)g.W) {
        const Pack<T, VEC> xv = ld_pack<T, VEC>(xb + (hh * g.W + ww) * g.x_sp);
#pragma unroll
        for (int i = 0; i < VEC; ++i) part[t][i] = mfma<T>(xv.v[i], gvv.v[i], 0.f);
      }
    }
  }
  // butterfly transpose-reduce of taps 0..7 over the 8 j-lanes: afterwards lane j owns the sums of tap j
#pragma unroll
  for (int off = 4; off >= 1; off >>= 1) {
    const bool upper = (j & off) != 0;
#pragma unroll
    for (int t = 0; t < off; ++t)
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float send = upper ? part[t][i] : part[t + off][i];
        const float keep = upper ? part[t + off][i] : part[t][i];
        part[t][i] = keep + __shfl_xor_sync(0xffffffffu, send, off * GQW);
      }
  }
  // tap 8: plain xor-reduce, every lane gets the total; lane j == 0 stores it
#pragma unroll
  for (int off = 4; off >= 1; off >>= 1)
#pragma unroll
    for (int i = 0; i < VEC; ++i) part[8][i] += __shfl_xor_sync(0xffffffffu, part[8][i], off * GQW);
  if (active) {
    T* wr = dw + (long long)n * g.w_sn + (h * g.W + wq) * g.w_sp;
    Pack<T, VEC> r;
#pragma unroll
    for (int i = 0; i < VEC; ++i) r.v[i] = Elem<T>::from(part[0][i]);
    st_pack<T, VEC>(wr + wpk_off_tap<VEC>(g0, j, g.gc), r);           // lane j owns tap j
    if (j == 0) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) r.v[i] = Elem<T>::from(part[8][i]);
      st_pack<T, VEC>(wr + wpk_off_tap<VEC>(g0, 8, g.gc), r);
    }
  }
}

// ------------------------------------------------------------------------------------------------ host dispatch
template <typename T>
static bool nhwc2_ok(const Nhwc2Args& a, const void* p0, const void* p1, const void* p2, bool need_tap, G2& g) {
  constexpr int VEC = 16 / (int)sizeof(T);
  if (a.layout == COTB200_NCHW) return false;
  const bool tap = a.layout == COTB200_NHWC_TAP;
  if (need_tap && !tap) return false;
  const int Cf = a.C / a.fold, wcf = a.wc / a.fold;
  if (wcf % VEC || a.C % VEC) return false;
  if (tap && (a.gc < VEC || a.gc % VEC || a.wc % a.gc)) return false;
  auto okp = [&](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (!okp(p0) || !okp(p1) || !okp(p2)) return false;
  const long long lim = (1LL << 31) - 1;
  const long long strides[6] = {a.x_sn, a.x_sp, a.w_sn, a.w_sp, a.y_sn, a.y_sp};
  for (long long s : strides) if (s > lim || (s * (long long)sizeof(T)) % 16) return false;
  if ((long long)a.H * a.W * a.x_sp > lim || (long long)a.H * a.W * a.w_sp > lim || (long long)a.H * a.W * a.y_sp > lim) return false;
  if ((long long)a.N * a.H > 65535LL * 32768) return false;
  g.N = a.N; g.C = a.C; g.H = a.H; g.W = a.W; g.wc = a.wc; g.Cf = Cf; g.wcf = wcf; g.rep = a.C / a.wc; g.gc = tap ? a.gc : 0;
  g.x_sn = (int)a.x_sn; g.x_sp = (int)a.x_sp; g.w_sn = (int)a.w_sn; g.w_sp = (int)a.w_sp; g.y_sn = (int)a.y_sn; g.y_sp = (int)a.y_sp;
  return true;
}

// returns 1 if handled (rc in *rc), 0 if the caller should fall back to the first-generation kernels
template <typename T>
int nhwc2_fwd(const Nhwc2Args& a, const T* x, const T* w, T* y, cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    constexpr int VEC = 16 / (int)sizeof(T);
    G2 g;
    if (!nhwc2_ok<T>(a, x, w, y, false, g)) return 0;
    if ((long long)a.N * a.H > 2147483647LL) return 0;
    const bool tap = a.layout == COTB200_NHWC_TAP;
    const int CQ = a.C / VEC;
    const int px = (a.W % 2 == 0) ? 2 : 1;
    dim3 grid((((a.W + px - 1) / px) * CQ + 255) / 256, a.N * a.H);
    if (grid.y > 65535) {   // fold rows into x when the batch is huge
      return 0;
    }
    COTB200_PROF_B("agg3_fwd_nhwc2", ((double)a.N * a.H * a.W) * (2.0 * a.C + 9.0 * a.wc) * sizeof(T));
    if (px == 2) {
      if (tap) agg3_nhwc2_kernel<T, VEC, 2, true, 0><<<grid, 256, 0, st>>>(x, w, y, g);
      else agg3_nhwc2_kernel<T, VEC, 2, false, 0><<<grid, 256, 0, st>>>(x, w, y, g);
    } else {
      if (tap) agg3_nhwc2_kernel<T, VEC, 1, true, 0><<<grid, 256, 0, st>>>(x, w, y, g);
      else agg3_nhwc2_kernel<T, VEC, 1, false, 0><<<grid, 256, 0, st>>>(x, w, y, g);
    }
    *rc = check_launch("agg3_fwd_nhwc2");
    return 1;
  }
}

template <typename T>
int nhwc2_dx(const Nhwc2Args& a, const T* dy, const T* w, T* dx, cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    constexpr int VEC = 16 / (int)sizeof(T);
    G2 g;
    if (!nhwc2_ok<T>(a, dy, w, dx, true, g)) return 0;
    const int CQ = a.C / VEC;
    const int px = (a.W % 2 == 0) ? 2 : 1;
    dim3 grid((((a.W + px - 1) / px) * CQ + 255) / 256, a.N * a.H);
    if (grid.y > 65535) return 0;
    COTB200_PROF_B("agg3_dx_nhwc2", ((double)a.N * a.H * a.W) * (2.0 * a.C + 9.0 * a.wc) * sizeof(T));
    if (px == 2) agg3_nhwc2_kernel<T, VEC, 2, true, 1><<<grid, 256, 0, st>>>(dy, w, dx, g);
    else agg3_nhwc2_kernel<T, VEC, 1, true, 1><<<grid, 256, 0, st>>>(dy, w, dx, g);
    *rc = check_launch("agg3_dx_nhwc2");
    return 1;
  }
}

template <typename T>
int nhwc2_dw(const Nhwc2Args& a, const T* dy, const T* x, T* dw, cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    constexpr int VEC = 16 / (int)sizeof(T);
    G2 g;
    if (!nhwc2_ok<T>(a, dy, x, dw, true, g)) return 0;
    if (a.C / a.wc != 8) return 0;                       // the butterfly is written for 8 sharers (share_planes = 8)
    const int GQ = a.wc / VEC;                            // weight packets per pixel
    int gqw = GQ >= 4 ? 4 : GQ;
    if (GQ % gqw || (gqw != 1 && gqw != 2 && gqw != 4)) return 0;
    if (a.fold > 1 && (a.wc / a.fold) % (gqw * VEC)) return 0;
    const int pxw = 32 / (8 * gqw);
    const int witems = ((a.W + pxw - 1) / pxw) * (GQ / gqw);       // warps per image row
    dim3 grid((witems + 7) / 8, a.N * a.H);
    if (grid.y > 65535) return 0;
    COTB200_PROF_B("agg3_dw_nhwc2", ((double)a.N * a.H * a.W) * (2.0 * a.C + 9.0 * a.wc) * sizeof(T));
    if (gqw == 1) agg3_dw_nhwc2_kernel<T, VEC, 1><<<grid, 256, 0, st>>>(dy, x, dw, g, GQ);
    else if (gqw == 2) agg3_dw_nhwc2_kernel<T, VEC, 2><<<grid, 256, 0, st>>>(dy, x, dw, g, GQ);
    else agg3_dw_nhwc2_kernel<T, VEC, 4><<<grid, 256, 0, st>>>(dy, x, dw, g, GQ);
    *rc = check_launch("agg3_dw_nhwc2");
    return 1;
  }
}

#define COTB200_INST(T)                                                                             \
  template int nhwc2_fwd<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);          \
  template int nhwc2_dx<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);           \
  template int nhwc2_dw<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);
COTB200_INST(float) COTB200_INST(double) COTB200_INST(__nv_bfloat16) COTB200_INST(__half)

}  // namespace cotb200
