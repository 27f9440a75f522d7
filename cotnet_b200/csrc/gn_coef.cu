// GroupNorm(9 taps) statistics from per-sample COLUMN sums (sm_90a).
//
// The logits GEMM (embed.3, models/cotnet.py:55) can emit, from its epilogue, the per-sample column sums of its raw
// accumulator: csum[b, j] = sum_px acc[b, px, j], csq[b, j] = sum_px acc^2 (cotb200_gemm_bf16_samplestats).  GroupNorm's
// group g of sample b (models/cotnet.py:56: the 9 tap channels of weight channel g over all H*W pixels) then needs no pass
// over the logits at all:
//     l = acc + bias_j           sum_g  = sum_t ( csum_j + HW * bias_j )
//                                sumsq_g = sum_t ( csq_j + 2 * bias_j * csum_j + HW * bias_j^2 ),      j = j(g, t)
// This kernel turns the column sums into mean[b, g], rstd[b, g] (the format cotb200_gn9_apply / _bwd take).
// Column order: reference order j = g*9 + t (gc == 0) or tap-major chunks (gc > 0), like everywhere else in the library.
#include "common.cuh"

namespace cotb200 {

__global__ void __launch_bounds__(128)
gn9_from_colsums_kernel(const float* __restrict__ csum, const float* __restrict__ csq, const float* __restrict__ bias, int B, int wc,
                        int gc, float hw, float eps, float* __restrict__ mean, float* __restrict__ rstd) {
  const int idx = blockIdx.x * 128 + threadIdx.x;
  if (idx >= B * wc) return;
  const int b = idx / wc, g = idx - b * wc;
  const int J = 9 * wc;
  float s = 0.f, q = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int j = gc > 0 ? ((g / gc) * 9 + t) * gc + g % gc : g * 9 + t;
    const float cs = csum[(long long)b * J + j], cq = csq[(long long)b * J + j];
    const float bj = bias ? __ldg(bias + j) : 0.f;
    s += fmaf(hw, bj, cs);
    q += cq + bj * fmaf(2.f, cs, hw * bj);
  }
  const float n = 9.f * hw;
  const float m = s / n;
  const float var = fmaxf(q / n - m * m, 0.f);
  mean[idx] = m;
  rstd[idx] = rsqrtf(var + eps);
}

// coef[b, j] = (rstd * gamma_j, beta_j - mean * rstd * gamma_j): one thread per (sample, group) writes its 9 columns
__global__ void __launch_bounds__(128)
gn9_coef_from_colsums_kernel(const float* __restrict__ csum, const float* __restrict__ csq, const float* __restrict__ bias,
                             const float* __restrict__ gamma, const float* __restrict__ beta, int B, int wc, int gc, float hw, float eps,
                             float2* __restrict__ coef) {
  const int idx = blockIdx.x * 128 + threadIdx.x;
  if (idx >= B * wc) return;
  const int b = idx / wc, g = idx - b * wc;
  const int J = 9 * wc;
  float s = 0.f, q = 0.f;
  int jj[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int j = gc > 0 ? ((g / gc) * 9 + t) * gc + g % gc : g * 9 + t;
    jj[t] = j;
    const float cs = csum[(long long)b * J + j], cq = csq[(long long)b * J + j];
    const float bj = bias ? __ldg(bias + j) : 0.f;
    s += fmaf(hw, bj, cs);
    q += cq + bj * fmaf(2.f, cs, hw * bj);
  }
  const float n = 9.f * hw;
  const float m = s / n;
  const float rs = rsqrtf(fmaxf(q / n - m * m, 0.f) + eps);
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float a = rs * __ldg(gamma + jj[t]);
    coef[(long long)b * J + jj[t]] = make_float2(a, fmaf(-m, a, __ldg(beta + jj[t])));
  }
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_gn9_coef_from_colsums(int B, int HW, int wc, int gc, const float* csum, const float* csq, const float* bias,
                                             const float* gamma, const float* beta, float eps, float* coef, void* stream) {
  if (!csum || !csq || !gamma || !beta || !coef) { set_error("gn9_coef_from_colsums: NULL pointer"); return COTB200_ENULL; }
  if (B <= 0 || HW <= 0 || wc <= 0 || gc < 0 || (gc > 0 && wc % gc)) { set_error("gn9_coef_from_colsums: bad dims"); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_PROF("gn9_coef_from_colsums");
  gn9_coef_from_colsums_kernel<<<(B * wc + 127) / 128, 128, 0, st>>>(csum, csq, bias, gamma, beta, B, wc, gc, (float)HW, eps, (float2*)coef);
  return check_launch("gn9_coef_from_colsums");
}

extern "C" int cotb200_gn9_from_colsums(int B, int HW, int wc, int gc, const float* csum, const float* csq, const float* bias,
                                        float eps, float* mean, float* rstd, void* stream) {
  if (!csum || !csq || !mean || !rstd) { set_error("gn9_from_colsums: NULL pointer"); return COTB200_ENULL; }
  if (B <= 0 || HW <= 0 || wc <= 0 || gc < 0 || (gc > 0 && wc % gc)) { set_error("gn9_from_colsums: bad dims"); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_PROF("gn9_from_colsums");
  gn9_from_colsums_kernel<<<(B * wc + 127) / 128, 128, 0, st>>>(csum, csq, bias, B, wc, gc, (float)HW, eps, mean, rstd);
  return check_launch("gn9_from_colsums");
}
