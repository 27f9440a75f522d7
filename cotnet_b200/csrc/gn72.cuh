// Launchers of the block-of-72 GroupNorm kernels (gn72.cu), called by the GroupNorm entry points in norm_tail.cu.
#pragma once
#include "common.cuh"

namespace cotb200 {

bool gn72_ok(int dtype, int wc, int gc, bool permuting, const void* p0, const void* p1, const void* p2);
template <typename T> int gn72_stats_launch(int B, int HW, int wc, const void* l, const float* lbias, float* gsum, float* gsq, cudaStream_t st);
template <typename T> int gn72_apply_launch(int B, int HW, int wc, const void* l, const float* lbias, const float* mean, const float* rstd,
                                            const float* gamma, const float* beta, void* out, cudaStream_t st);
template <typename T> int gn72_bwd_sums_launch(int B, int HW, int wc, const void* dg, const void* l, float* P, cudaStream_t st);
template <typename T> int gn72_bwd_apply_launch(int B, int HW, int wc, const void* dg, const void* l, const float* lbias, const float* mean,
                                                const float* rstd, const float* gamma, const float* s1, const float* s2, void* dl,
                                                cudaStream_t st);
int gn_bwd_finish_launch(int B, int HW, int wc, const float* P, int raw, const float* lbias, const float* mean, const float* rstd,
                         const float* gamma, float* s1, float* s2, float* dgamma, float* dbeta, float* dlbias, cudaStream_t st);

}  // namespace cotb200
