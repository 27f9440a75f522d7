// out = src0 + src1 (+ src2 + src3) over row-pitched [rows, C] views (sm_90a).
//
// Inside the CoT block x feeds three consumers (key_embed conv, the concat, conv1x1) and k two (the concat and the
// radix-2 recombination): models/cotnet.py:80-84,97.  Autograd accumulates their gradients with a
// chain of pairwise adds, and the concat's gradients are channel slices (pitch 2C) that ATen adds with its
// non-vectorised strided kernel (dozens of launches per step).  This kernel does the whole
// accumulation in one pass of 16-byte packets: (n reads + 1 write) * C * rows * s bytes, HBM-bound.
#include "common.cuh"

namespace cotb200 {

struct SumSrc { const void* p[4]; long long ld[4]; };

template <typename T, int VEC, int NSRC>
__global__ void __launch_bounds__(256)
sum_rows_kernel(SumSrc s, T* __restrict__ out, long long ldo, long long rows, int CQ) {
  const long long total = rows * CQ;
  for (long long item = (long long)blockIdx.x * 256 + threadIdx.x; item < total; item += (long long)gridDim.x * 256) {
    const long long r = item / CQ;
    const int q = (int)(item - r * CQ);
    float acc[VEC];
    {
      const Pack<T, VEC> v = ld_pack<T, VEC>((const T*)s.p[0] + r * s.ld[0] + q * VEC);
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] = to_acc(v.v[i]);
    }
#pragma unroll
    for (int k = 1; k < NSRC; ++k) {
      const Pack<T, VEC> v = ld_pack<T, VEC>((const T*)s.p[k] + r * s.ld[k] + q * VEC);
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] += to_acc(v.v[i]);
    }
    Pack<T, VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(acc[i]);
    st_pack<T, VEC>(out + r * ldo + q * VEC, o);
  }
}

template <typename T, int VEC>
static void sum_rows_launch(int nsrc, const SumSrc& s, T* out, long long ldo, long long rows, int CQ, unsigned blocks, cudaStream_t st) {
  if (nsrc == 2) sum_rows_kernel<T, VEC, 2><<<blocks, 256, 0, st>>>(s, out, ldo, rows, CQ);
  else if (nsrc == 3) sum_rows_kernel<T, VEC, 3><<<blocks, 256, 0, st>>>(s, out, ldo, rows, CQ);
  else sum_rows_kernel<T, VEC, 4><<<blocks, 256, 0, st>>>(s, out, ldo, rows, CQ);
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_sum_rows(int dtype, long long rows, int C, const void* src0, long long ld0, const void* src1, long long ld1,
                                const void* src2, long long ld2, const void* src3, long long ld3, void* out, long long ldo,
                                void* stream) {
  if (!src0 || !src1 || !out) { set_error("sum_rows: NULL pointer"); return COTB200_ENULL; }
  if (!src2 && src3) { set_error("sum_rows: src3 given without src2"); return COTB200_EINVAL; }
  if (dtype == COTB200_F64) { set_error("sum_rows: fp64 not supported"); return COTB200_EDTYPE; }
  if (rows <= 0 || C <= 0) { set_error("sum_rows: non-positive dims"); return COTB200_EINVAL; }
  const int nsrc = src3 ? 4 : src2 ? 3 : 2;
  SumSrc s; s.p[0] = src0; s.p[1] = src1; s.p[2] = src2; s.p[3] = src3; s.ld[0] = ld0; s.ld[1] = ld1; s.ld[2] = ld2; s.ld[3] = ld3;
  for (int k = 0; k < nsrc; ++k) if (s.ld[k] < C) { set_error("sum_rows: pitch %lld < C %d", s.ld[k], C); return COTB200_EINVAL; }
  if (ldo < C) { set_error("sum_rows: output pitch %lld < C %d", ldo, C); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      int vec = 16 / (int)sizeof(T);
      auto fits = [&](int v) {
        if (C % v) return false;
        const uintptr_t m = (uintptr_t)(v * sizeof(T)) - 1;
        for (int k = 0; k < nsrc; ++k) if (((uintptr_t)s.p[k] & m) || (s.ld[k] % v)) return false;
        return !((uintptr_t)out & m) && !(ldo % v);
      };
      while (vec > 1 && !fits(vec)) vec >>= 1;
      const int CQ = C / vec;
      const long long total = rows * CQ;
      const int blocks = grid_stride_blocks(total, 256, 16);   // 2 waves of 8 CTAs per SM
      COTB200_PROF_B("sum_rows", (double)rows * C * (nsrc + 1) * sizeof(T));
      switch (vec) {
        case 8: if constexpr (sizeof(T) == 2) sum_rows_launch<T, 8>(nsrc, s, (T*)out, ldo, rows, CQ, blocks, st); break;
        case 4: sum_rows_launch<T, 4>(nsrc, s, (T*)out, ldo, rows, CQ, blocks, st); break;
        case 2: sum_rows_launch<T, 2>(nsrc, s, (T*)out, ldo, rows, CQ, blocks, st); break;
        default: sum_rows_launch<T, 1>(nsrc, s, (T*)out, ldo, rows, CQ, blocks, st); break;
      }
      return check_launch("sum_rows");
    }
  });
  return 0;
}
