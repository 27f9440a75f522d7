// Soft-target cross entropy of the training recipe (sm_90a): SoftTargetCrossEntropy on mixup_target(labels, K, lam, smoothing)
// (loss/cross_entropy.py:29-36, datasets/mixup.py:17-27), which the reference selects whenever Mixup / CutMix is on (train.py:198-209).
//
// The [B, K] target is never formed.  Its rows sum to one, so per row b
//   loss_b = lse(z_b) - sum_c t_bc z_bc,   sum_c t_bc z_bc = off*sum_c z_bc + (on - off)*(lam*z_b[y_b] + (1-lam)*z_b[y_{B-1-b}])
// with off = smoothing/K, on = 1 - smoothing + off.  One CTA per row (two passes over the row, the second from L1/L2), then one
// CTA adds the B row losses in a fixed order: the loss is bit-identical from run to run.  lam = mix->target_lam is read from
// device memory so that a captured graph follows every step's Mixup / CutMix draw.  The per-sample modes read lam and the partner
// row y_{partner(b)} from a device table (cotb200_mix_row) instead, through the same kernels.
//
// JsdCrossEntropy (loss/jsd.py) of the augmentation splits: label-smoothed cross entropy on the clean split plus alpha/S times
// the KL divergence of every split's softmax from their clamped mixture.  One CTA per clean row handles its S rows; the row losses
// are added by the same fixed-order launch as the soft-target loss.
//
// Also the validation metric: top-k hit counts (utils/meters.py:12-19 accuracy(), evaler/evaler.py:37-57) accumulated as int64
// on the device, one warp per row, so that a captured eval graph needs no host synchronisation per batch.
#include <climits>

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

// whose label takes the rest of row b's soft target, and row b's own weight: the batch draw (partner B-1-b, one lam; no mixing
// without it) or the per-sample table (any partner, checked against the n_labels labels: -1 makes the row NaN)
struct CeBatchMix {
  const cotb200_mix* mix;
  int B;
  __device__ __forceinline__ bool on() const { return mix != nullptr; }
  __device__ __forceinline__ float lam(int) const { return mix ? mix->target_lam : 1.f; }
  __device__ __forceinline__ long long partner(int b) const { return B - 1 - b; }
};

struct CeRowMix {
  const cotb200_mix_row* rows;
  int n_labels;
  __device__ __forceinline__ bool on() const { return true; }
  __device__ __forceinline__ float lam(int b) const { return rows[b].target_lam; }
  __device__ __forceinline__ long long partner(int b) const {
    const int p = rows[b].partner;
    return (p >= 0 && p < n_labels) ? p : -1;
  }
};

// log-sum-exp and sum of one row, every thread of the CTA gets both
template <typename T>
__device__ __forceinline__ float ce_row_lse(const T* __restrict__ zr, int K, float* sm, float& sz) {
  float mx = -INFINITY;
  sz = 0.f;
  for (int c = threadIdx.x; c < K; c += CE_THREADS) { const float v = to_acc(zr[c]); mx = fmaxf(mx, v); sz += v; }
  mx = ce_block_reduce(mx, sm, [](float a, float b_) { return fmaxf(a, b_); });
  sz = ce_block_reduce(sz, sm, [](float a, float b_) { return a + b_; });
  float se = 0.f;
  for (int c = threadIdx.x; c < K; c += CE_THREADS) se += expf(to_acc(zr[c]) - mx);
  se = ce_block_reduce(se, sm, [](float a, float b_) { return a + b_; });
  return mx + logf(se);
}

template <typename T, class Mix>
__global__ void __launch_bounds__(CE_THREADS)
soft_ce_rows_kernel(const T* __restrict__ z, long long ld, const long long* __restrict__ labels, Mix mix, int B, int K, float off,
                    float onoff, float* __restrict__ rows) {
  __shared__ float sm[CE_THREADS / 32];
  const int b = blockIdx.x;
  const T* zr = z + (long long)b * ld;
  float sz;
  const float lse = ce_row_lse(zr, K, sm, sz);
  if (threadIdx.x == 0) {
    const float lam = mix.lam(b);
    const long long y = labels[b];
    float own = __int_as_float(0x7fffffff), other = 0.f;
    if (y >= 0 && y < K) own = to_acc(zr[y]);
    if (mix.on()) {
      const long long p = mix.partner(b), yp = p >= 0 ? labels[p] : -1;
      other = (yp >= 0 && yp < K) ? to_acc(zr[yp]) : __int_as_float(0x7fffffff);
    }
    const float dot = off * sz + onoff * (mix.on() ? lam * own + (1.f - lam) * other : own);
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

template <typename T, class Mix>
__global__ void __launch_bounds__(CE_THREADS)
soft_ce_bwd_kernel(const T* __restrict__ z, long long ld, const long long* __restrict__ labels, Mix mix, int B, int K, float off,
                   float onoff, const float* __restrict__ rows, const float* __restrict__ dloss, float* __restrict__ dz, long long ldz) {
  const int b = blockIdx.x;
  const T* zr = z + (long long)b * ld;
  float* dr = dz + (long long)b * ldz;
  const float lam = mix.lam(b), g = __ldg(dloss) / (float)B, lse = rows[b];
  const long long y = labels[b], p = mix.on() ? mix.partner(b) : b, yp = p >= 0 ? labels[p] : -1;
  const bool ok = y >= 0 && y < K && yp >= 0 && yp < K;
  const float w_own = onoff * (mix.on() ? lam : 1.f), w_other = mix.on() ? onoff * (1.f - lam) : 0.f;
  for (int c = threadIdx.x; c < K; c += CE_THREADS) {
    const float t = off + (c == y ? w_own : 0.f) + (c == yp ? w_other : 0.f);
    dr[c] = ok ? g * (expf(to_acc(zr[c]) - lse) - t) : __int_as_float(0x7fffffff);
  }
}

// ---------------------------------------------------------------- JSD + cross entropy of the augmentation splits
static constexpr int JSD_MAX_S = 8;

// class c of clean row b: p[s] = softmax(z_{b+sB})_c, lp[s] = its log (0 where p underflows to 0: the xlogy limit), the log of the
// clamped mixture, and whether the clamp passes (torch's clamp mask is inclusive)
template <typename T>
__device__ __forceinline__ float jsd_class(const T* __restrict__ z, long long ld, int b, int B, int S, int c, const float* lse,
                                           float* p, float* lp, bool& pass) {
  float msum = 0.f;
#pragma unroll
  for (int s = 0; s < JSD_MAX_S; ++s) {
    if (s < S) {
      const float d = to_acc(z[(long long)(b + s * B) * ld + c]) - lse[s];
      p[s] = expf(d);
      lp[s] = p[s] > 0.f ? d : 0.f;
      msum += p[s];
    }
  }
  const float m = msum / (float)S;
  pass = m >= 1e-7f && m <= 1.f;
  return logf(fminf(fmaxf(m, 1e-7f), 1.f));
}

template <typename T>
__global__ void __launch_bounds__(CE_THREADS)
jsd_ce_rows_kernel(const T* __restrict__ z, long long ld, const long long* __restrict__ labels, int S, int B, int K, float off,
                   float onoff, float alpha_s, float* __restrict__ rows) {
  __shared__ float sm[CE_THREADS / 32];
  const int b = blockIdx.x;
  float lse[JSD_MAX_S], sz0 = 0.f;
#pragma unroll
  for (int s = 0; s < JSD_MAX_S; ++s) {
    lse[s] = 0.f;
    if (s < S) {
      float sz;
      lse[s] = ce_row_lse(z + (long long)(b + s * B) * ld, K, sm, sz);
      if (s == 0) sz0 = sz;
      if (threadIdx.x == 0) rows[b + s * B] = lse[s];
    }
  }
  float kl = 0.f;
  for (int c = threadIdx.x; c < K; c += CE_THREADS) {
    float p[JSD_MAX_S], lp[JSD_MAX_S];
    bool pass;
    const float lm = jsd_class(z, ld, b, B, S, c, lse, p, lp, pass);
#pragma unroll
    for (int s = 0; s < JSD_MAX_S; ++s)
      if (s < S) kl += p[s] * lp[s] - p[s] * lm;
  }
  kl = ce_block_reduce(kl, sm, [](float a, float b_) { return a + b_; });
  if (threadIdx.x == 0) {
    const long long y = labels[b];
    const float own = (y >= 0 && y < K) ? to_acc(z[(long long)b * ld + y]) : __int_as_float(0x7fffffff);
    rows[(long long)S * B + b] = (lse[0] - (off * sz0 + onoff * own)) + alpha_s * kl;
  }
}

// dL/dp_sc = a (lp_sc - log m_c + [clamp binds]),  a = dloss * alpha / (S B); dz_sc = p_sc (dL/dp_sc - sum_c' p_sc' dL/dp_sc'),
// plus dloss / B (p_0c - t_c) on the clean split
template <typename T>
__global__ void __launch_bounds__(CE_THREADS)
jsd_ce_bwd_kernel(const T* __restrict__ z, long long ld, const long long* __restrict__ labels, int S, int B, int K, float off,
                  float onoff, float alpha_sb, const float* __restrict__ rows, const float* __restrict__ dloss,
                  float* __restrict__ dz, long long ldz) {
  __shared__ float sm[CE_THREADS / 32];
  const int b = blockIdx.x;
  const float dl = __ldg(dloss), g = dl / (float)B, a = dl * alpha_sb;
  const long long y = labels[b];
  const bool ok = y >= 0 && y < K;
  float lse[JSD_MAX_S], dot[JSD_MAX_S];
#pragma unroll
  for (int s = 0; s < JSD_MAX_S; ++s) {
    lse[s] = s < S ? rows[b + s * B] : 0.f;
    dot[s] = 0.f;
  }
  for (int c = threadIdx.x; c < K; c += CE_THREADS) {
    float p[JSD_MAX_S], lp[JSD_MAX_S];
    bool pass;
    const float lm = jsd_class(z, ld, b, B, S, c, lse, p, lp, pass);
#pragma unroll
    for (int s = 0; s < JSD_MAX_S; ++s)
      if (s < S) dot[s] += p[s] * (lp[s] - lm + (pass ? 0.f : 1.f));
  }
#pragma unroll
  for (int s = 0; s < JSD_MAX_S; ++s)
    if (s < S) dot[s] = ce_block_reduce(dot[s], sm, [](float u, float v) { return u + v; });
  for (int c = threadIdx.x; c < K; c += CE_THREADS) {
    float p[JSD_MAX_S], lp[JSD_MAX_S];
    bool pass;
    const float lm = jsd_class(z, ld, b, B, S, c, lse, p, lp, pass);
    const float t = off + (c == y ? onoff : 0.f);
#pragma unroll
    for (int s = 0; s < JSD_MAX_S; ++s) {
      if (s < S) {
        float d = a * p[s] * ((lp[s] - lm + (pass ? 0.f : 1.f)) - dot[s]);
        if (s == 0) d += g * (p[0] - t);
        dz[(long long)(b + s * B) * ldz + c] = ok ? d : __int_as_float(0x7fffffff);
      }
    }
  }
}

static int jsd_check(const char* what, int dtype, int S, int B, int K, const void* logits, long long ld, const long long* labels,
                     float smoothing, float alpha) {
  if (!logits || !labels) { set_error("%s: NULL pointer", what); return COTB200_ENULL; }
  if (S < 2 || S > JSD_MAX_S) { set_error("%s: %d splits (2..%d supported)", what, S, JSD_MAX_S); return COTB200_EINVAL; }
  if (B <= 0 || K <= 0 || ld < K || (long long)S * B > INT_MAX) {
    set_error("%s: bad dims S=%d B=%d K=%d ld=%lld", what, S, B, K, ld); return COTB200_EINVAL;
  }
  if (!(smoothing >= 0.f && smoothing < 1.f)) { set_error("%s: smoothing %g outside [0, 1)", what, (double)smoothing); return COTB200_EINVAL; }
  if (!(alpha >= 0.f && alpha < INFINITY)) { set_error("%s: alpha %g not finite and >= 0", what, (double)alpha); return COTB200_EINVAL; }
  if (dtype == COTB200_F64) { set_error("%s: fp64 not supported", what); return COTB200_EDTYPE; }
  return 0;
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

// ---------------------------------------------------------------- top-k hits
static constexpr int TK_THREADS = 256;               // 8 warps = 8 rows per CTA
static constexpr int TK_MAX_K = 4;

struct TopkKs { int k[TK_MAX_K]; };

// rank(b) = #{c : z_c > z_y} + #{c < y : z_c == z_y}; row b is a hit at k iff rank < k.  Without ties this is the position of
// the label in a descending sort, i.e. what output.topk(k) + eq counts; ties go to the lower class index.  A NaN label logit is
// a miss (no comparison with it holds, so it is tested explicitly); NaN competitors never outrank.  The row's warp streams its K
// logits once; per CTA the counters are added in shared memory, then one integer atomic per counter: exact in any order.
template <typename T>
__global__ void __launch_bounds__(TK_THREADS)
topk_hits_kernel(const T* __restrict__ z, long long ld, const long long* __restrict__ labels, const int* __restrict__ valid_dev,
                 int B, int K, int nk, TopkKs ks, unsigned long long* __restrict__ counts) {
  __shared__ unsigned sm[TK_THREADS / 32][TK_MAX_K + 2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * (TK_THREADS / 32) + warp;
  const int nvalid = valid_dev ? min(max(__ldg(valid_dev), 0), B) : B;
  unsigned hit[TK_MAX_K] = {}, counted = 0, bad = 0;
  if (b < nvalid) {
    counted = 1;
    const long long y = __ldg(labels + b);
    if (y < 0 || y >= K) {
      bad = 1;
    } else {
      const T* zr = z + (long long)b * ld;
      const int yi = (int)y;
      const float zy = to_acc(zr[yi]);
      if (zy == zy) {
        int r = 0;
#pragma unroll 4
        for (int c = lane; c < K; c += 32) {
          const float x = to_acc(zr[c]);
          r += (x > zy) | ((x == zy) & (c < yi));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
#pragma unroll
        for (int i = 0; i < TK_MAX_K; ++i) hit[i] = (i < nk && r < ks.k[i]) ? 1u : 0u;
      }
    }
  }
  if (lane == 0) {                                   // sm row: hits@k for the nk values of k, rows counted, bad labels
#pragma unroll
    for (int i = 0; i < TK_MAX_K; ++i) sm[warp][i] = hit[i];
    sm[warp][TK_MAX_K] = counted;
    sm[warp][TK_MAX_K + 1] = bad;
  }
  __syncthreads();
  if (threadIdx.x < nk + 2) {                        // counts[j] for j < nk from slot j, counts[nk], counts[nk + 1] from the last two
    const int j = threadIdx.x, slot = j < nk ? j : TK_MAX_K + (j - nk);
    unsigned s = 0;
#pragma unroll
    for (int w = 0; w < TK_THREADS / 32; ++w) s += sm[w][slot];
    if (s) atomicAdd(counts + j, (unsigned long long)s);
  }
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
      soft_ce_rows_kernel<T><<<B, CE_THREADS, 0, st>>>((const T*)logits, ld, labels, CeBatchMix{mix, B}, B, K, off, onoff, rows);
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
      soft_ce_bwd_kernel<T><<<B, CE_THREADS, 0, st>>>((const T*)logits, ld, labels, CeBatchMix{mix, B}, B, K, off, onoff, rows, dloss,
                                                       dz, ldz);
      return check_launch("soft_ce_bwd");
    }
  });
  return 0;
}

static int soft_ce_rows_check(const char* what, int dtype, int B, int K, const void* logits, long long ld, const long long* labels,
                              int n_labels, const cotb200_mix_row* mix_rows, float smoothing) {
  int rc = soft_ce_check(what, dtype, B, K, logits, ld, labels, nullptr, smoothing);
  if (rc) return rc;
  if (!mix_rows) { set_error("%s: NULL row table", what); return COTB200_ENULL; }
  if (n_labels < B || (n_labels & 1)) { set_error("%s: %d labels for %d rows (an even count >= B)", what, n_labels, B); return COTB200_EINVAL; }
  return 0;
}

extern "C" int cotb200_soft_ce_rows(int dtype, int B, int K, const void* logits, long long ld, const long long* labels, int n_labels,
                                    const cotb200_mix_row* mix_rows, float smoothing, float* rows, float* loss, void* stream) {
  int rc = soft_ce_rows_check("soft_ce_rows", dtype, B, K, logits, ld, labels, n_labels, mix_rows, smoothing);
  if (rc) return rc;
  if (!rows || !loss) { set_error("soft_ce_rows: NULL pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  const float off = smoothing / (float)K, onoff = 1.f - smoothing;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("soft_ce_rows", (double)B * K * sizeof(T));
      soft_ce_rows_kernel<T><<<B, CE_THREADS, 0, st>>>((const T*)logits, ld, labels, CeRowMix{mix_rows, n_labels}, B, K, off, onoff, rows);
      if ((rc = check_launch("soft_ce_rows"))) return rc;
      soft_ce_mean_kernel<<<1, CE_THREADS, 0, st>>>(rows + B, B, loss);
      return check_launch("soft_ce_rows_mean");
    }
  });
  return 0;
}

extern "C" int cotb200_soft_ce_rows_bwd(int dtype, int B, int K, const void* logits, long long ld, const long long* labels, int n_labels,
                                        const cotb200_mix_row* mix_rows, float smoothing, const float* rows, const float* dloss, float* dz,
                                        long long ldz, void* stream) {
  int rc = soft_ce_rows_check("soft_ce_rows_bwd", dtype, B, K, logits, ld, labels, n_labels, mix_rows, smoothing);
  if (rc) return rc;
  if (!rows || !dloss || !dz) { set_error("soft_ce_rows_bwd: NULL pointer"); return COTB200_ENULL; }
  if (ldz < K) { set_error("soft_ce_rows_bwd: ldz %lld < K %d", ldz, K); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const float off = smoothing / (float)K, onoff = 1.f - smoothing;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("soft_ce_rows_bwd", (double)B * K * (sizeof(T) + 4));
      soft_ce_bwd_kernel<T><<<B, CE_THREADS, 0, st>>>((const T*)logits, ld, labels, CeRowMix{mix_rows, n_labels}, B, K, off, onoff, rows,
                                                       dloss, dz, ldz);
      return check_launch("soft_ce_rows_bwd");
    }
  });
  return 0;
}

extern "C" int cotb200_jsd_ce(int dtype, int S, int B, int K, const void* logits, long long ld, const long long* labels,
                              float smoothing, float alpha, float* rows, float* loss, void* stream) {
  int rc = jsd_check("jsd_ce", dtype, S, B, K, logits, ld, labels, smoothing, alpha);
  if (rc) return rc;
  if (!rows || !loss) { set_error("jsd_ce: NULL pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  const float off = smoothing / (float)K, onoff = 1.f - smoothing;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("jsd_ce", 2.0 * S * B * K * sizeof(T));
      jsd_ce_rows_kernel<T><<<B, CE_THREADS, 0, st>>>((const T*)logits, ld, labels, S, B, K, off, onoff, alpha / (float)S, rows);
      if ((rc = check_launch("jsd_ce"))) return rc;
      soft_ce_mean_kernel<<<1, CE_THREADS, 0, st>>>(rows + (long long)S * B, B, loss);
      return check_launch("jsd_ce_mean");
    }
  });
  return 0;
}

extern "C" int cotb200_jsd_ce_bwd(int dtype, int S, int B, int K, const void* logits, long long ld, const long long* labels,
                                  float smoothing, float alpha, const float* rows, const float* dloss, float* dz, long long ldz,
                                  void* stream) {
  int rc = jsd_check("jsd_ce_bwd", dtype, S, B, K, logits, ld, labels, smoothing, alpha);
  if (rc) return rc;
  if (!rows || !dloss || !dz) { set_error("jsd_ce_bwd: NULL pointer"); return COTB200_ENULL; }
  if (ldz < K) { set_error("jsd_ce_bwd: ldz %lld < K %d", ldz, K); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const float off = smoothing / (float)K, onoff = 1.f - smoothing;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("jsd_ce_bwd", (double)S * B * K * (2 * sizeof(T) + 4));
      jsd_ce_bwd_kernel<T><<<B, CE_THREADS, 0, st>>>((const T*)logits, ld, labels, S, B, K, off, onoff, alpha / (float)(S * B), rows,
                                                     dloss, dz, ldz);
      return check_launch("jsd_ce_bwd");
    }
  });
  return 0;
}

extern "C" int cotb200_topk_hits(int dtype, int B, int K, const void* logits, long long ld, const long long* labels,
                                 const int* valid_dev, int nk, const int* ks, long long* counts_dev, void* stream) {
  if (!logits || !labels || !ks || !counts_dev) { set_error("topk_hits: NULL pointer"); return COTB200_ENULL; }
  if (B <= 0 || K <= 0 || ld < K) { set_error("topk_hits: bad dims B=%d K=%d ld=%lld", B, K, ld); return COTB200_EINVAL; }
  if (nk < 1 || nk > TK_MAX_K) { set_error("topk_hits: %d values of k (1..%d supported)", nk, TK_MAX_K); return COTB200_EINVAL; }
  TopkKs kk = {};
  for (int i = 0; i < nk; ++i) {
    if (ks[i] < 1 || ks[i] > K) { set_error("topk_hits: k=%d outside 1..K=%d", ks[i], K); return COTB200_EINVAL; }
    kk.k[i] = ks[i];
  }
  if (dtype == COTB200_F64) { set_error("topk_hits: fp64 not supported"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (B + TK_THREADS / 32 - 1) / (TK_THREADS / 32);
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("topk_hits", (double)B * K * sizeof(T));
      topk_hits_kernel<T><<<grid, TK_THREADS, 0, st>>>((const T*)logits, ld, labels, valid_dev, B, K, nk, kk,
                                                       reinterpret_cast<unsigned long long*>(counts_dev));
      return check_launch("topk_hits");
    }
  });
  return 0;
}
