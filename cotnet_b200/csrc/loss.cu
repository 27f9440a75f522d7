// Soft-target cross entropy of the training recipe (sm_90a): SoftTargetCrossEntropy on mixup_target(labels, K, lam, smoothing)
// (loss/cross_entropy.py:29-36, datasets/mixup.py:17-27), which the reference selects whenever Mixup / CutMix is on (train.py:198-209).
//
// The [B, K] target is never formed.  Its rows sum to one, so per row b
//   loss_b = lse(z_b) - sum_c t_bc z_bc,   sum_c t_bc z_bc = off*sum_c z_bc + (on - off)*(lam*z_b[y_b] + (1-lam)*z_b[y_{B-1-b}])
// with off = smoothing/K, on = 1 - smoothing + off.  One CTA per row (two passes over the row, the second from L1/L2), then one
// CTA adds the B row losses in a fixed order: the loss is bit-identical from run to run.  lam = mix->target_lam is read from
// device memory so that a captured graph follows every step's Mixup / CutMix draw.
#include "common.cuh"

namespace cotb200 {

static constexpr int CE_THREADS = 256;

// fixed-order CTA reduction: warp shuffles in a fixed pattern, then warp 0 adds the 8 warp totals in order
template <class Op>
__device__ __forceinline__ float ce_block_reduce(float v, float* sm, Op op) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();                                   // sm may still be read by the previous reduction
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  float t = sm[0];
  for (int w = 1; w < CE_THREADS / 32; ++w) t = op(t, sm[w]);
  return t;
}

__device__ __forceinline__ float ce_lam(const cotb200_mix* mix) { return mix ? mix->target_lam : 1.f; }

template <typename T>
__global__ void __launch_bounds__(CE_THREADS)
soft_ce_rows_kernel(const T* __restrict__ z, long long ld, const long long* __restrict__ labels, const cotb200_mix* __restrict__ mix,
                    int B, int K, float off, float onoff, float* __restrict__ rows) {
  __shared__ float sm[CE_THREADS / 32];
  const int b = blockIdx.x;
  const T* zr = z + (long long)b * ld;
  float mx = -INFINITY, sz = 0.f;
  for (int c = threadIdx.x; c < K; c += CE_THREADS) { const float v = to_acc(zr[c]); mx = fmaxf(mx, v); sz += v; }
  mx = ce_block_reduce(mx, sm, [](float a, float b_) { return fmaxf(a, b_); });
  sz = ce_block_reduce(sz, sm, [](float a, float b_) { return a + b_; });
  float se = 0.f;
  for (int c = threadIdx.x; c < K; c += CE_THREADS) se += expf(to_acc(zr[c]) - mx);
  se = ce_block_reduce(se, sm, [](float a, float b_) { return a + b_; });
  if (threadIdx.x == 0) {
    const float lse = mx + logf(se);
    const float lam = ce_lam(mix);
    const long long y = labels[b];
    float own = __int_as_float(0x7fffffff), other = 0.f;
    if (y >= 0 && y < K) own = to_acc(zr[y]);
    if (mix) {
      const long long yp = labels[B - 1 - b];
      other = (yp >= 0 && yp < K) ? to_acc(zr[yp]) : __int_as_float(0x7fffffff);
    }
    const float dot = off * sz + onoff * (mix ? lam * own + (1.f - lam) * other : own);
    rows[b] = lse;
    rows[B + b] = lse - dot;
  }
}

__global__ void __launch_bounds__(CE_THREADS)
soft_ce_mean_kernel(const float* __restrict__ row_loss, int B, float* __restrict__ loss) {
  __shared__ float sm[CE_THREADS / 32];
  float s = 0.f;
  for (int b = threadIdx.x; b < B; b += CE_THREADS) s += row_loss[b];
  s = ce_block_reduce(s, sm, [](float a, float b_) { return a + b_; });
  if (threadIdx.x == 0) loss[0] = s / (float)B;
}

template <typename T>
__global__ void __launch_bounds__(CE_THREADS)
soft_ce_bwd_kernel(const T* __restrict__ z, long long ld, const long long* __restrict__ labels, const cotb200_mix* __restrict__ mix,
                   int B, int K, float off, float onoff, const float* __restrict__ rows, const float* __restrict__ dloss,
                   float* __restrict__ dz, long long ldz) {
  const int b = blockIdx.x;
  const T* zr = z + (long long)b * ld;
  float* dr = dz + (long long)b * ldz;
  const float lam = ce_lam(mix), g = __ldg(dloss) / (float)B, lse = rows[b];
  const long long y = labels[b], yp = mix ? labels[B - 1 - b] : y;
  const bool ok = y >= 0 && y < K && yp >= 0 && yp < K;
  const float w_own = onoff * (mix ? lam : 1.f), w_other = mix ? onoff * (1.f - lam) : 0.f;
  for (int c = threadIdx.x; c < K; c += CE_THREADS) {
    const float t = off + (c == y ? w_own : 0.f) + (c == yp ? w_other : 0.f);
    dr[c] = ok ? g * (expf(to_acc(zr[c]) - lse) - t) : __int_as_float(0x7fffffff);
  }
}

static int soft_ce_check(const char* what, int dtype, int B, int K, const void* logits, long long ld, const long long* labels,
                         const cotb200_mix* mix, float smoothing) {
  if (!logits || !labels) { set_error("%s: NULL pointer", what); return COTB200_ENULL; }
  if (B <= 0 || K <= 0 || ld < K) { set_error("%s: bad dims B=%d K=%d ld=%lld", what, B, K, ld); return COTB200_EINVAL; }
  if (mix && (B & 1)) { set_error("%s: batch size %d must be even when mixing", what, B); return COTB200_EINVAL; }
  if (!(smoothing >= 0.f && smoothing < 1.f)) { set_error("%s: smoothing %g outside [0, 1)", what, (double)smoothing); return COTB200_EINVAL; }
  if (dtype == COTB200_F64) { set_error("%s: fp64 not supported", what); return COTB200_EDTYPE; }
  return 0;
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_soft_ce(int dtype, int B, int K, const void* logits, long long ld, const long long* labels, const cotb200_mix* mix,
                               float smoothing, float* rows, float* loss, void* stream) {
  int rc = soft_ce_check("soft_ce", dtype, B, K, logits, ld, labels, mix, smoothing);
  if (rc) return rc;
  if (!rows || !loss) { set_error("soft_ce: NULL pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  const float off = smoothing / (float)K, onoff = 1.f - smoothing;       // on - off = 1 - smoothing
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("soft_ce", (double)B * K * sizeof(T));
      soft_ce_rows_kernel<T><<<B, CE_THREADS, 0, st>>>((const T*)logits, ld, labels, mix, B, K, off, onoff, rows);
      if ((rc = check_launch("soft_ce"))) return rc;
      soft_ce_mean_kernel<<<1, CE_THREADS, 0, st>>>(rows + B, B, loss);
      return check_launch("soft_ce_mean");
    }
  });
  return 0;
}

extern "C" int cotb200_soft_ce_bwd(int dtype, int B, int K, const void* logits, long long ld, const long long* labels,
                                   const cotb200_mix* mix, float smoothing, const float* rows, const float* dloss, float* dz,
                                   long long ldz, void* stream) {
  int rc = soft_ce_check("soft_ce_bwd", dtype, B, K, logits, ld, labels, mix, smoothing);
  if (rc) return rc;
  if (!rows || !dloss || !dz) { set_error("soft_ce_bwd: NULL pointer"); return COTB200_ENULL; }
  if (ldz < K) { set_error("soft_ce_bwd: ldz %lld < K %d", ldz, K); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const float off = smoothing / (float)K, onoff = 1.f - smoothing;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("soft_ce_bwd", (double)B * K * (sizeof(T) + 4));
      soft_ce_bwd_kernel<T><<<B, CE_THREADS, 0, st>>>((const T*)logits, ld, labels, mix, B, K, off, onoff, rows, dloss, dz, ldz);
      return check_launch("soft_ce_bwd");
    }
  });
  return 0;
}
