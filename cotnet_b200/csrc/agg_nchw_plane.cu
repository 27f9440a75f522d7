// LocalConv 3x3 / stride 1 / pad 1 backward on NCHW tensors whose planes are SMALL (100 <= H*W <= 256: the 14x14 stage of the
// reference models; cupy_layers/aggregation_zeropad.py:48-110).
//
// The other NCHW kernels tile a plane over the grid; on a 14x14 plane that leaves 98 threads of a 256-thread CTA with 8-byte
// accesses (the TMA ring cannot help: a 56-byte row is not a legal TMA stride) and the reference's own scalar kernel was faster
// in backward at [256,256,14,14] fp32.  Here a CTA owns whole
// (sample, weight-channel) items -- the rep = C/wc channel planes that share one set of 9 weight planes:
//   * all rep planes of x and/or dy are staged in shared memory as fp32 with a one-pixel ZERO halo (one load phase of
//     independent coalesced loads, one barrier), so the tap loops have no boundary predicates at all;
//   * thread = one pixel of one item; its 9 weights (at the pixel minus the tap offset) stay in registers across the rep
//     channels; dW is 9 register accumulators per thread, no reduction (one owner per (pixel, tap)).
// One pass over every tensor: (3C + 9wc) + (C + 9wc) elements per pixel (dy, x, w in; dx, dw out).
// The forward stays on the tiled kernels, which are faster there.
#include "common.cuh"
#include "agg.cuh"

namespace cotb200 {

template <typename T, int MODE>      // MODE 1: dX only; 2: dW only; 3: dX + dW
__global__ void __launch_bounds__(256)
agg3_plane_kernel(const T* __restrict__ a, const T* __restrict__ b, const T* __restrict__ w, T* __restrict__ o1, T* __restrict__ o2,
                  int C, int H, int W, int wc, int rep, int ipc, int items, long long a_sn, long long b_sn, long long w_sn,
                  long long o1_sn, long long o2_sn) {
  // a = dy, b = x, o1 = dx (MODE & 1), o2 = dw (MODE & 2)
  constexpr bool DX = (MODE & 1) != 0, DW = (MODE & 2) != 0;
  extern __shared__ float pl_sm[];
  const int HW = H * W, Wp = W + 2, PP = (H + 2) * Wp;
  float* as = pl_sm;                                  // [ipc][rep][PP]
  float* bs = pl_sm + (size_t)ipc * rep * PP;         // [ipc][rep][PP] (dW only)
  const int tid = threadIdx.x;
  const int nsm = ipc * rep * PP * (DW ? 2 : 1);
  __shared__ unsigned short s_hoff[256];              // pixel -> offset inside a haloed plane (the only division of the staging)
  for (int i = tid; i < nsm; i += 256) pl_sm[i] = 0.f;
  if (tid < HW) { const int ph = tid / W; s_hoff[tid] = (unsigned short)((ph + 1) * Wp + (tid - ph * W) + 1); }
  __syncthreads();
  const int item0 = blockIdx.x * ipc;
  // ---- stage the planes (fp32, haloed): warp w takes planes w, w + 8, ...; lanes walk the pixels of the plane (coalesced)
  {
    const int warp = tid >> 5, lane = tid & 31;
    const int nplanes = ipc * rep;
    for (int pl = warp; pl < nplanes; pl += 8) {
      const int il = pl / rep, j = pl - il * rep;
      const int item = item0 + il;
      if (item >= items) break;
      const int n = item / wc, g = item - n * wc;
      const T* ag = a + n * a_sn + (long long)(g + j * wc) * HW;
      const T* bg = DW ? b + n * b_sn + (long long)(g + j * wc) * HW : nullptr;
      float* ad = as + (size_t)pl * PP;
      float* bd = bs + (size_t)pl * PP;
      for (int p = lane; p < HW; p += 32) {
        const int so = s_hoff[p];
        ad[so] = (float)to_acc(__ldg(ag + p));
        if (DW) bd[so] = (float)to_acc(__ldg(bg + p));
      }
    }
  }
  // ---- this thread's pixel and its 9 weights (global loads in flight across the barrier)
  const int il = tid / HW, p = tid - il * HW;
  const int item = item0 + il;
  const bool active = il < ipc && item < items;
  const int n = active ? item / wc : 0, g = active ? item - n * wc : 0;
  const int ph = p / W, pw = p - ph * W;
  float wt[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wt[t] = 0.f;
  if (active && DX) {
    const T* wp = w + n * w_sn + (long long)g * 9 * HW;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int dh = t / 3 - 1, dw = t % 3 - 1;
      // weight of tap t at the output pixel q = p - off_t that read this input
      const int qh = ph - dh, qw = pw - dw;
      if ((unsigned)qh < (unsigned)H && (unsigned)qw < (unsigned)W) wt[t] = (float)to_acc(__ldg(wp + (long long)t * HW + qh * W + qw));
    }
  }
  __syncthreads();
  if (!active) return;
  const int ctr = (ph + 1) * Wp + pw + 1;
  float gw[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) gw[t] = 0.f;
  const float* ap = as + (size_t)il * rep * PP + ctr;
  const float* bp = bs + (size_t)il * rep * PP + ctr;
  for (int j = 0; j < rep; ++j, ap += PP, bp += PP) {
    const long long go = (long long)(g + j * wc) * HW + p;
    if (DX) {
      float acc = 0.f;
#pragma unroll
      for (int t = 0; t < 9; ++t) acc = fmaf(wt[t], ap[-(t / 3 - 1) * Wp - (t % 3 - 1)], acc);
      o1[n * o1_sn + go] = Elem<T>::from(acc);
    }
    if (DW) {
      const float d = ap[0];
#pragma unroll
      for (int t = 0; t < 9; ++t) gw[t] = fmaf(bp[(t / 3 - 1) * Wp + (t % 3 - 1)], d, gw[t]);
    }
  }
  if (DW) {
    T* dwp = o2 + n * o2_sn + (long long)g * 9 * HW + p;
#pragma unroll
    for (int t = 0; t < 9; ++t) dwp[(long long)t * HW] = Elem<T>::from(gw[t]);
  }
}

// mode 1 dX / 2 dW / 3 dX + dW; returns 1 when the call was taken (*rc = status), 0 when the geometry is not for this kernel
template <typename T>
int nchw_plane_launch(int mode, int N, int C, int H, int W, int wc, long long x_sn, long long y_sn, long long w_sn, const T* a, const T* b,
                      const T* w, T* o1, T* o2, cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    // planes of >= 100 pixels, where it beats the tiled kernels and the reference's own kernels
    const int HW = H * W;
    if (HW > 256 || HW < 100 || C % wc) return 0;
    const int rep = C / wc;
    int ipc = 256 / HW;
    const int PP = (H + 2) * (W + 2);
    const bool dwm = (mode & 2) != 0;
    while (ipc > 1 && (size_t)ipc * rep * PP * (dwm ? 2 : 1) * sizeof(float) > 96 * 1024) --ipc;
    const size_t smem = (size_t)ipc * rep * PP * (dwm ? 2 : 1) * sizeof(float);
    if (smem > 96 * 1024) return 0;
    const long long items_ll = (long long)N * wc;
    if (items_ll > 2000000000LL) return 0;
    const int items = (int)items_ll;
    const int grid = (items + ipc - 1) / ipc;
    const double px = (double)N * HW;
    cudaError_t e = cudaSuccess;
    static PerDevFlag cfg[4];
#define PL_GO(M, name, bytes)                                                                                                     \
    {                                                                                                                              \
      if (bool& c = cfg[M].get(); !c) { e = cudaFuncSetAttribute(agg3_plane_kernel<T, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024); c = (e == cudaSuccess); } \
      if (e == cudaSuccess) {                                                                                                      \
        COTB200_PROF_B(name, bytes);                                                                                               \
        agg3_plane_kernel<T, M><<<grid, 256, smem, st>>>(a, b, w, o1, o2, C, H, W, wc, rep, ipc, items, y_sn, x_sn, w_sn, x_sn, w_sn); \
      }                                                                                                                            \
    }
    if (mode == 1) PL_GO(1, "agg3_dx_plane", px * (2.0 * C + 9.0 * wc) * sizeof(T))
    else if (mode == 2) PL_GO(2, "agg3_dw_plane", px * (2.0 * C + 9.0 * wc) * sizeof(T))
    else PL_GO(3, "agg3_dxdw_plane", px * (3.0 * C + 9.0 * wc + C + 9.0 * wc) * sizeof(T))
#undef PL_GO
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(agg plane): %s", cudaGetErrorString(e)); *rc = (int)e; return 1; }
    *rc = check_launch("agg3_plane");
    return 1;
  }
}

#define COTB200_INST_PL(T) \
  template int nchw_plane_launch<T>(int, int, int, int, int, int, long long, long long, long long, const T*, const T*, const T*, T*, T*, cudaStream_t, int*);
COTB200_INST_PL(float) COTB200_INST_PL(double) COTB200_INST_PL(__nv_bfloat16) COTB200_INST_PL(__half)

}  // namespace cotb200
