// 3x3 / stride 2 / pad 1 pooling on NHWC tensors (sm_90a).
//
// The CoT bottleneck down-samples with nn.AvgPool2d(3, 2, padding=1) in front of the CoT layer of every stride-2 block
// (models/cotnet.py:199-202,237-238) and the trunk with nn.MaxPool2d(3, 2, 1) (models/resnet.py:555).  ATen's
// channels_last pooling kernels run far below the HBM bandwidth (and its avg_pool2d backward is wrong in this torch build); these are plain
// HBM-bound gathers: one thread per (output pixel, 16-byte channel packet), no atomics in backward (gather form).
#include "common.cuh"

namespace cotb200 {

template <typename T, int VEC>
__global__ void __launch_bounds__(256)
avgpool3s2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int H, int W, int Ho, int Wo, int CQ) {
  const int item = blockIdx.y * 256 + threadIdx.x;
  if (item >= Wo * CQ) return;
  const int q = item % CQ, wo = item / CQ;
  const int row = blockIdx.x, n = row / Ho, ho = row - n * Ho;
  const int C = CQ * VEC;
  const T* xb = x + ((long long)n * H * W) * C + q * VEC;
  float acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
    const int h = 2 * ho - 1 + kh;
    if ((unsigned)h >= (unsigned)H) continue;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int w = 2 * wo - 1 + kw;
      if ((unsigned)w >= (unsigned)W) continue;
      const Pack<T, VEC> v = ld_pack<T, VEC>(xb + (long long)(h * W + w) * C);
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] += to_acc(v.v[i]);
    }
  }
  Pack<T, VEC> o;
#pragma unroll
  for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(acc[i] * (1.f / 9.f));     // count_include_pad=True (module default)
  st_pack<T, VEC>(y + ((long long)(n * Ho + ho) * Wo + wo) * C + q * VEC, o);
}

template <typename T, int VEC>
__global__ void __launch_bounds__(256)
avgpool3s2_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, int H, int W, int Ho, int Wo, int CQ) {
  const int item = blockIdx.y * 256 + threadIdx.x;
  if (item >= W * CQ) return;
  const int q = item % CQ, w = item / CQ;
  const int row = blockIdx.x, n = row / H, h = row - n * H;
  const int C = CQ * VEC;
  const T* gb = dy + ((long long)n * Ho * Wo) * C + q * VEC;
  float acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
    const int hs = h + 1 - kh;
    if (hs < 0 || (hs & 1)) continue;
    const int ho = hs >> 1;
    if (ho >= Ho) continue;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int ws = w + 1 - kw;
      if (ws < 0 || (ws & 1)) continue;
      const int wo = ws >> 1;
      if (wo >= Wo) continue;
      const Pack<T, VEC> v = ld_pack<T, VEC>(gb + (long long)(ho * Wo + wo) * C);
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] += to_acc(v.v[i]);
    }
  }
  Pack<T, VEC> o;
#pragma unroll
  for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(acc[i] * (1.f / 9.f));
  st_pack<T, VEC>(dx + ((long long)(n * H + h) * W + w) * C + q * VEC, o);
}

// max pooling; idx[n,ho,wo,c] = tap (0..8) of the first maximal element in scan order (PyTorch's strict '>' rule)
template <typename T, int VEC>
__global__ void __launch_bounds__(256)
maxpool3s2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, unsigned char* __restrict__ idx, int H, int W, int Ho, int Wo,
                      int CQ) {
  const int item = blockIdx.y * 256 + threadIdx.x;
  if (item >= Wo * CQ) return;
  const int q = item % CQ, wo = item / CQ;
  const int row = blockIdx.x, n = row / Ho, ho = row - n * Ho;
  const int C = CQ * VEC;
  const T* xb = x + ((long long)n * H * W) * C + q * VEC;
  float best[VEC];
  unsigned char bi[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { best[i] = -INFINITY; bi[i] = 4; }
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
    const int h = 2 * ho - 1 + kh;
    if ((unsigned)h >= (unsigned)H) continue;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int w = 2 * wo - 1 + kw;
      if ((unsigned)w >= (unsigned)W) continue;
      const Pack<T, VEC> v = ld_pack<T, VEC>(xb + (long long)(h * W + w) * C);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float f = to_acc(v.v[i]);
        if (f > best[i] || f != f) { best[i] = f; bi[i] = (unsigned char)(kh * 3 + kw); }
      }
    }
  }
  Pack<T, VEC> o;
  Pack<unsigned char, VEC> oi;
#pragma unroll
  for (int i = 0; i < VEC; ++i) { o.v[i] = Elem<T>::from(best[i]); oi.v[i] = bi[i]; }
  const long long off = ((long long)(n * Ho + ho) * Wo + wo) * C + q * VEC;
  st_pack<T, VEC>(y + off, o);
#pragma unroll
  for (int i = 0; i < VEC; ++i) idx[off + i] = oi.v[i];
}

template <typename T, int VEC>
__global__ void __launch_bounds__(256)
maxpool3s2_bwd_kernel(const T* __restrict__ dy, const unsigned char* __restrict__ idx, T* __restrict__ dx, int H, int W, int Ho,
                      int Wo, int CQ) {
  const int item = blockIdx.y * 256 + threadIdx.x;
  if (item >= W * CQ) return;
  const int q = item % CQ, w = item / CQ;
  const int row = blockIdx.x, n = row / H, h = row - n * H;
  const int C = CQ * VEC;
  const long long gb = ((long long)n * Ho * Wo) * C + q * VEC;
  float acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
    const int hs = h + 1 - kh;
    if (hs < 0 || (hs & 1)) continue;
    const int ho = hs >> 1;
    if (ho >= Ho) continue;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int ws = w + 1 - kw;
      if (ws < 0 || (ws & 1)) continue;
      const int wo = ws >> 1;
      if (wo >= Wo) continue;
      const long long off = gb + (long long)(ho * Wo + wo) * C;
      const Pack<T, VEC> v = ld_pack<T, VEC>(dy + off);
#pragma unroll
      for (int i = 0; i < VEC; ++i)
        if (idx[off + i] == (unsigned char)(kh * 3 + kw)) acc[i] += to_acc(v.v[i]);
    }
  }
  Pack<T, VEC> o;
#pragma unroll
  for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(acc[i]);
  st_pack<T, VEC>(dx + ((long long)(n * H + h) * W + w) * C + q * VEC, o);
}

template <typename T>
static int pool_vec(int C, const void* a, const void* b) {
  for (int vec = 16 / (int)sizeof(T); vec >= 1; vec >>= 1) {
    if (C % vec) continue;
    const uintptr_t m = (uintptr_t)(vec * sizeof(T)) - 1;
    if (((uintptr_t)a & m) == 0 && ((uintptr_t)b & m) == 0) return vec;
  }
  return 1;
}

#define POOL_DISPATCH(vec, ...)                                                   \
  switch (vec) {                                                                   \
    case 8: if constexpr (sizeof(T) == 2) { constexpr int V = 8; __VA_ARGS__; } break; \
    case 4: { constexpr int V = 4; __VA_ARGS__; } break;                           \
    case 2: { constexpr int V = 2; __VA_ARGS__; } break;                           \
    default: { constexpr int V = 1; __VA_ARGS__; } break;                          \
  }

}  // namespace cotb200

using namespace cotb200;

// mode: 0 average (count_include_pad), 1 max.  idx: [N,Ho,Wo,C] uint8 (max only).
extern "C" int cotb200_pool3s2_fwd(int dtype, int mode, int N, int H, int W, int C, const void* x, void* y, void* idx, void* stream) {
  if (!x || !y || (mode == 1 && !idx)) { set_error("pool3s2_fwd: NULL pointer"); return COTB200_ENULL; }
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || (mode != 0 && mode != 1)) { set_error("pool3s2_fwd: bad arguments"); return COTB200_EINVAL; }
  if (dtype == COTB200_F64) { set_error("pool3s2: fp64 not supported"); return COTB200_EDTYPE; }
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  if ((long long)N * H > 2147483647LL || (long long)W * C > 65535LL * 256) { set_error("pool3s2: tensor too large for the launch grid"); return COTB200_ETOOBIG; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pool_vec<T>(C, x, y);
      const int CQ = C / vec;
      dim3 grid((unsigned)(N * Ho), (Wo * CQ + 255) / 256);   // rows on grid.x (2^31-1 limit), packets on grid.y
      COTB200_PROF_B(mode ? "maxpool3s2_fwd" : "avgpool3s2_fwd", ((double)N * C) * ((double)H * W + (double)Ho * Wo) * sizeof(T));
      POOL_DISPATCH(vec, {
        if (mode == 0) avgpool3s2_fwd_kernel<T, V><<<grid, 256, 0, st>>>((const T*)x, (T*)y, H, W, Ho, Wo, CQ);
        else maxpool3s2_fwd_kernel<T, V><<<grid, 256, 0, st>>>((const T*)x, (T*)y, (unsigned char*)idx, H, W, Ho, Wo, CQ);
      });
      return check_launch("pool3s2_fwd");
    }
  });
  return 0;
}

extern "C" int cotb200_pool3s2_bwd(int dtype, int mode, int N, int H, int W, int C, const void* dy, const void* idx, void* dx,
                                   void* stream) {
  if (!dy || !dx || (mode == 1 && !idx)) { set_error("pool3s2_bwd: NULL pointer"); return COTB200_ENULL; }
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || (mode != 0 && mode != 1)) { set_error("pool3s2_bwd: bad arguments"); return COTB200_EINVAL; }
  if (dtype == COTB200_F64) { set_error("pool3s2: fp64 not supported"); return COTB200_EDTYPE; }
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  if ((long long)N * H > 2147483647LL || (long long)W * C > 65535LL * 256) { set_error("pool3s2: tensor too large for the launch grid"); return COTB200_ETOOBIG; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pool_vec<T>(C, dy, dx);
      const int CQ = C / vec;
      dim3 grid((unsigned)(N * H), (W * CQ + 255) / 256);
      COTB200_PROF_B(mode ? "maxpool3s2_bwd" : "avgpool3s2_bwd", ((double)N * C) * ((double)H * W + (double)Ho * Wo) * sizeof(T));
      POOL_DISPATCH(vec, {
        if (mode == 0) avgpool3s2_bwd_kernel<T, V><<<grid, 256, 0, st>>>((const T*)dy, (T*)dx, H, W, Ho, Wo, CQ);
        else maxpool3s2_bwd_kernel<T, V><<<grid, 256, 0, st>>>((const T*)dy, (const unsigned char*)idx, (T*)dx, H, W, Ho, Wo, CQ);
      });
      return check_launch("pool3s2_bwd");
    }
  });
  return 0;
}
