// GroupNorm over the 9 taps of each weight channel, second generation: "blocks of 72" staged by bulk async copies (sm_90a).
//
// The logits l [B, HW, 9*wc] are in the reference channel order j = g*9 + t (models/cotnet.py:55-56), the normalised
// weights ghat (and their gradient) in the tap-major order the LocalConv kernels read: chunk of 8 weight channels, position
// of (g, t) = ((g/8)*9 + t)*8 + g%8 (COTB200_NHWC_TAP, gc = 8).  Both orders keep a chunk -- 8 groups x 9 taps = 72
// elements = 144 bytes in bf16 -- contiguous at the SAME offset: the permutation is an 8x9 -> 9x8 transpose inside each
// 144-byte block, and the whole tensor is a flat array of such blocks.
//
// The first-generation kernels (norm_tail.cu) did that transpose with stride-9 scalar gathers from global memory:
// 9 load instructions per 8 elements, far below the HBM roof.  Here
//   * a CTA moves its tile (256 consecutive blocks, 36 KB) with ONE cp.async.bulk global->shared (mbarrier complete_tx)
//     and writes its result with ONE cp.async.bulk shared->global: address generation leaves the SM's LSU entirely;
//   * apply / bwd_apply: thread = one block, 9 conflict-free 16-byte shared loads, the transpose is register renaming
//     (fully unrolled), per-(sample, column) coefficients come from a table in shared memory (broadcast reads);
//   * stats: thread = one block, 8 group sums by warp shuffles;
//   * bwd_sums: thread = one column, 16-bit shared loads, three fp32 FMAs per element (on the widened bf16
//     operands: sum dg, sum dg*l, sum l), per-(sample, column) partials -> a tiny finish kernel derives s1, s2, dgamma,
//     dbeta AND the bias gradient of the embed.3 convolution analytically (no extra pass over dl).
// Algorithmic bytes: stats J, apply 2J, bwd_sums 2J, bwd_apply 3J (x px x s) -- unchanged; the point is reaching them.
#include "common.cuh"
#include "tma.cuh"

namespace cotb200 {

struct GN72 {
  int B, HW, wc, nchunk, J;
  int bps;              // blocks of 72 per sample = HW * nchunk
  int tb;               // blocks per tile
  DetArena det;         // scratch + tickets of the per-sample reductions over the CTAs of a sample
};

template <typename T> struct G7 {
  static constexpr int NP = 72 * (int)sizeof(T) / 16;      // 16-byte packets per block: 9 (16-bit) / 18 (fp32)
  static constexpr int PV = 16 / (int)sizeof(T);           // elements per packet
  static constexpr int TB = sizeof(T) == 2 ? 256 : 128;    // blocks per tile
};

// read / write one block of 72 elements at shared address `sa` (144 / 288 bytes, 16-byte aligned)
template <typename T>
__device__ __forceinline__ void g7_ld_block(uint32_t sa, T (&v)[72]) {
#pragma unroll
  for (int p = 0; p < G7<T>::NP; ++p) {
    uint4 u;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "r"(sa + 16 * p));
    *reinterpret_cast<uint4*>(&v[p * G7<T>::PV]) = u;
  }
}
template <typename T>
__device__ __forceinline__ void g7_st_block(uint32_t sa, const T (&v)[72]) {
#pragma unroll
  for (int p = 0; p < G7<T>::NP; ++p) {
    const uint4 u = *reinterpret_cast<const uint4*>(&v[p * G7<T>::PV]);
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(sa + 16 * p), "r"(u.x), "r"(u.y), "r"(u.z), "r"(u.w) : "memory");
  }
}

// ------------------------------------------------------------------------------------------------ statistics
// gsum[b,g] += sum_{t,px} (l + lbias) ; gsq likewise.   grid (X, B): CTA (x, b) walks the tiles x, x+X, .. of sample b with a
// two-stage bulk-copy ring.  Thread = one block per tile; it keeps 72 per-COLUMN sums of the raw l and 8 per-group sums of
// l^2, both by fp32 FMAs on the widened 16-bit operands (9 LDS.128 per 144 bytes, no per-element
// bias loads); the bias enters analytically at the end:  sum (l+b) = S_j + n*b_j,  sum (l+b)^2 = Q_g + 2*sum_t b_j*S_j + n*b_j^2.
template <typename T>
__global__ void __launch_bounds__(G7<T>::TB)
gn72_stats_kernel(const T* __restrict__ l, const float* __restrict__ lbias, float* __restrict__ gsum, float* __restrict__ gsq, GN72 g) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar[2];
  __shared__ float s_acc[2 * 64];                 // [2][wc <= 64]
  constexpr int TB = G7<T>::TB;
  constexpr uint32_t TILE = TB * 72 * sizeof(T);
  const int tid = threadIdx.x, b = blockIdx.y;
  const int ntiles = (g.bps + TB - 1) / TB;
  const T* lb = l + (long long)b * g.bps * 72;
  auto issue = [&](int tile, int stage) {
    const int nblk = min(TB, g.bps - tile * TB);
    const uint32_t bytes = (uint32_t)nblk * 72u * sizeof(T);
    mbar_expect_tx(smem_u32(&bar[stage]), bytes);
    bulk_load(smem_u32(smem) + stage * TILE, lb + (long long)tile * TB * 72, bytes, smem_u32(&bar[stage]));
  };
  if (tid == 0) {
    mbar_init(smem_u32(&bar[0]), 1);
    mbar_init_fence();
    mbar_init(smem_u32(&bar[1]), 1);
    mbar_init_fence();
    if ((int)blockIdx.x < ntiles) issue(blockIdx.x, 0);
  }
  for (int i = tid; i < 2 * g.wc; i += TB) s_acc[i] = 0.f;
  __syncthreads();
  const int chunk = tid % g.nchunk;               // TB % nchunk == 0 -> blk % nchunk == tid % nchunk
  float S[72], Q[8];
#pragma unroll
  for (int j = 0; j < 72; ++j) S[j] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) Q[i] = 0.f;
  int npx = 0;                                    // blocks this thread accumulated
  const T one = one_of<T>();
  int it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const int stage = it & 1;
    if (tid == 0 && tile + (int)gridDim.x < ntiles) issue(tile + gridDim.x, stage ^ 1);   // stage^1 was drained before the last sync
    mbar_wait(smem_u32(&bar[stage]), (it >> 1) & 1);
    const int nblk = min(TB, g.bps - tile * TB);
    if (tid < nblk) {
      T v[72];
      g7_ld_block<T>(smem_u32(smem) + stage * TILE + tid * 72 * (int)sizeof(T), v);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          S[i * 9 + t] = mfma<T>(v[i * 9 + t], one, S[i * 9 + t]);
          Q[i] = mfma<T>(v[i * 9 + t], v[i * 9 + t], Q[i]);
        }
      ++npx;
    }
    __syncthreads();                              // everyone is done with `stage` before it is refilled two tiles later
  }
  // fold the bias in, then per-group sums
  float s[8], q[8];
  const float n = (float)npx;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float ss = 0.f, qq = Q[i];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float bj = lbias ? lbias[chunk * 72 + i * 9 + t] : 0.f;
      ss += S[i * 9 + t] + n * bj;
      qq += bj * (2.f * S[i * 9 + t] + n * bj);
    }
    s[i] = ss; q[i] = qq;
  }
  // lanes with equal lane % nchunk hold the same chunk: butterfly over the remaining lane bits
  for (int off = 16; off >= g.nchunk; off >>= 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i] += __shfl_xor_sync(0xffffffffu, s[i], off);
      q[i] += __shfl_xor_sync(0xffffffffu, q[i], off);
    }
  }
  // warps add their chunk totals in warp order (run-to-run identical sums), then the CTAs of the sample in CTA order
  for (int w = 0; w < TB / 32; ++w) {
    if (tid >> 5 == w && (tid & 31) < g.nchunk) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s_acc[chunk * 8 + i] += s[i];
        s_acc[g.wc + chunk * 8 + i] += q[i];
      }
    }
    __syncthreads();
  }
  float* scr = g.det.scr + b * det_floats(gridDim.x, 2 * g.wc);
  for (int i = tid; i < 2 * g.wc; i += TB) scr[(size_t)blockIdx.x * 2 * g.wc + i] = s_acc[i];
  det_finish(scr, 2 * g.wc, blockIdx.x, gridDim.x, g.det.tick + b * DET_TICKETS_PER_GROUP, tid, TB, [&](int k, float t) {
    if (k < g.wc) gsum[(long long)b * g.wc + k] += t; else gsq[(long long)b * g.wc + k - g.wc] += t;
  });
}

// ------------------------------------------------------------------------------------------------ apply
// ghat[tap pos] = (l[j] + lbias[j] - mean[b,g]) * rstd[b,g] * gamma[j] + beta[j];  in-place transpose of each block in
// shared memory, one bulk store.
template <typename T>
__global__ void __launch_bounds__(G7<T>::TB)
gn72_apply_kernel(const T* __restrict__ l, const float* __restrict__ lbias, const float* __restrict__ mean,
                  const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                  T* __restrict__ out, GN72 g) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  __shared__ float2 s_coef[576];                  // tap order inside each chunk: [chunk*72 + t*8 + i] = (a, c)
  constexpr int TB = G7<T>::TB;
  const int tid = threadIdx.x, b = blockIdx.y;
  const int blk0 = blockIdx.x * TB, nblk = min(TB, g.bps - blk0);
  const uint32_t bytes = (uint32_t)nblk * 72u * sizeof(T);
  const long long goff = ((long long)b * g.bps + blk0) * 72;
  if (tid == 0) {
    mbar_init(smem_u32(&bar), 1);
    mbar_init_fence();
    mbar_expect_tx(smem_u32(&bar), bytes);
    bulk_load(smem_u32(smem), l + goff, bytes, smem_u32(&bar));
  }
  for (int j = tid; j < g.J; j += TB) {           // j = reference index g*9 + t
    const int gi = j / 9, t = j - gi * 9;
    const float a = rstd[(long long)b * g.wc + gi] * gamma[j];
    const float c = beta[j] - (mean[(long long)b * g.wc + gi] - (lbias ? lbias[j] : 0.f)) * a;
    s_coef[(gi >> 3) * 72 + t * 8 + (gi & 7)] = make_float2(a, c);
  }
  __syncthreads();
  mbar_wait(smem_u32(&bar), 0);
  if (tid < nblk) {
    const uint32_t sa = smem_u32(smem) + tid * 72 * (int)sizeof(T);
    T v[72], o[72];
    g7_ld_block<T>(sa, v);
    const float2* cf = s_coef + (tid % g.nchunk) * 72;
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float2 ac = cf[t * 8 + i];
        o[t * 8 + i] = Elem<T>::from(fmaf(to_acc(v[i * 9 + t]), ac.x, ac.y));
      }
    g7_st_block<T>(sa, o);
    fence_proxy_async();
  }
  __syncthreads();
  if (tid == 0) bulk_store_and_wait(out + goff, smem_u32(smem), bytes);
}

// ------------------------------------------------------------------------------------------------ backward sums
// P[b][0][j] += sum_px dg ; P[b][1][j] += sum_px dg * l ; P[b][2][j] += sum_px l      (j = reference index, raw l)
// grid (ceil(HW / PR), B) with PR = TB / nchunk pixels per tile, 288 threads: thread = column (x row lane).
static constexpr int G7_SUM_THREADS = 288;
template <typename T>
__global__ void __launch_bounds__(G7_SUM_THREADS)
gn72_bwd_sums_kernel(const T* __restrict__ dg, const T* __restrict__ l, float* __restrict__ P, GN72 g) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  __shared__ float s_lane[3 * 576];                               // [3][RL][J] per-row-lane partials (J * RL <= 576)
  constexpr int TB = G7<T>::TB;
  const int tid = threadIdx.x, b = blockIdx.y;
  const int PR = TB / g.nchunk;                                   // pixels per tile
  const int px0 = blockIdx.x * PR, npx = min(PR, g.HW - px0);
  const uint32_t bytes = (uint32_t)npx * g.J * sizeof(T);
  const long long goff = ((long long)b * g.HW + px0) * g.J;
  const T* s_dg = reinterpret_cast<const T*>(smem);
  const T* s_l = reinterpret_cast<const T*>(smem + (size_t)TB * 72 * sizeof(T));
  if (tid == 0) {
    mbar_init(smem_u32(&bar), 1);
    mbar_init_fence();
    mbar_expect_tx(smem_u32(&bar), 2 * bytes);
    bulk_load(smem_u32(s_dg), dg + goff, bytes, smem_u32(&bar));
    bulk_load(smem_u32(s_l), l + goff, bytes, smem_u32(&bar));
  }
  __syncthreads();
  mbar_wait(smem_u32(&bar), 0);
  const int RL = G7_SUM_THREADS >= g.J ? G7_SUM_THREADS / g.J : 1;        // row lanes per column
  const int JR = g.J * RL;
  for (int c = tid; c < JR; c += G7_SUM_THREADS) {
    const int j = c % g.J, rl = c / g.J;
    const int gi = j / 9, t = j - gi * 9;
    const int pos = (gi >> 3) * 72 + t * 8 + (gi & 7);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    const T one = one_of<T>();
#pragma unroll 4
    for (int r = rl; r < npx; r += RL) {
      const T d = s_dg[r * g.J + pos], lv = s_l[r * g.J + j];
      a0 = mfma<T>(d, one, a0);
      a1 = mfma<T>(d, lv, a1);
      a2 = mfma<T>(lv, one, a2);
    }
    s_lane[c] = a0;
    s_lane[JR + c] = a1;
    s_lane[2 * JR + c] = a2;
  }
  __syncthreads();
  // the CTA's row: row-lane partials added in lane order (run-to-run identical), then across the CTAs of the sample
  float* Pb = P + (long long)b * 3 * g.J;
  float* scr = g.det.scr + b * det_floats(gridDim.x, 3 * g.J);
  for (int i = tid; i < 3 * g.J; i += G7_SUM_THREADS) {
    const int pl = i / g.J, j = i - pl * g.J;
    float v = 0.f;
    for (int rl = 0; rl < RL; ++rl) v += s_lane[pl * JR + rl * g.J + j];
    scr[(size_t)blockIdx.x * 3 * g.J + i] = v;
  }
  det_finish(scr, 3 * g.J, blockIdx.x, gridDim.x, g.det.tick + b * DET_TICKETS_PER_GROUP, tid, G7_SUM_THREADS, [&](int k, float t) { Pb[k] += t; });
}

// CTA = one group g, thread = sample b (strided): s1, s2 of (b, g) are written; the group's 9 columns of dgamma / dbeta /
// dlbias are reduced over the batch inside the CTA (no same-address atomics: one CTA owns its 27 outputs).
//   lhat_j = (l_j + lb_j - mean) * rstd:  sum dg*lhat = rstd*(P1 - m_j*P0),  sum lhat = rstd*(P2 - HW*m_j),  m_j = mean - lb_j
static constexpr int G7_FIN_THREADS = 256;
__global__ void __launch_bounds__(G7_FIN_THREADS)
gn_bwd_finish_kernel(const float* __restrict__ P, int raw, const float* __restrict__ lbias, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const float* __restrict__ gamma, float* __restrict__ s1,
                     float* __restrict__ s2, float* __restrict__ dgamma, float* __restrict__ dbeta,
                     float* __restrict__ dlbias, int B, int HW, int wc) {
  __shared__ float s_red[G7_FIN_THREADS / 32][27];
  const int gi = blockIdx.x, J = 9 * wc, tid = threadIdx.x;
  const float inv_n = 1.f / (9.f * (float)HW);
  float ga[9], lb[9], acc[27];
#pragma unroll
  for (int t = 0; t < 9; ++t) { ga[t] = gamma[gi * 9 + t]; lb[t] = lbias ? lbias[gi * 9 + t] : 0.f; }
#pragma unroll
  for (int i = 0; i < 27; ++i) acc[i] = 0.f;
  for (int b = tid; b < B; b += G7_FIN_THREADS) {
    const int idx = b * wc + gi;
    const float mn = mean[idx], rs = rstd[idx];
    const float* Pb = P + (long long)b * 3 * J + gi * 9;
    float D[9], DL[9], LH[9], a = 0.f, q = 0.f;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float m = mn - lb[t];
      D[t] = Pb[t];
      DL[t] = raw ? rs * (Pb[J + t] - m * D[t]) : Pb[J + t];           // raw: sums over l, else already over lhat
      LH[t] = raw ? rs * (Pb[2 * J + t] - (float)HW * m) : Pb[2 * J + t];
      a = fmaf(D[t], ga[t], a);
      q = fmaf(DL[t], ga[t], q);
    }
    s1[idx] = a;
    s2[idx] = q;
    const float k1 = a * inv_n, k2 = q * inv_n;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      acc[t] += D[t];
      acc[9 + t] += DL[t];
      acc[18 + t] += rs * (ga[t] * D[t] - (float)HW * k1 - k2 * LH[t]);
    }
  }
#pragma unroll
  for (int i = 0; i < 27; ++i) {
    float v = acc[i];
#pragma unroll
    for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if ((tid & 31) == 0) s_red[tid >> 5][i] = v;
  }
  __syncthreads();
  if (tid < 27) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < G7_FIN_THREADS / 32; ++w) v += s_red[w][tid];
    const int t = tid % 9, j = gi * 9 + t;
    if (tid < 9) dbeta[j] += v;
    else if (tid < 18) dgamma[j] += v;
    else if (dlbias) dlbias[j] += v;
  }
}

// ------------------------------------------------------------------------------------------------ backward apply
// dl[j] = rstd*(dg*gamma - k1 - lhat*k2) = dg*A_j + l*Bg + C_j   with A_j = rstd*gamma_j, Bg = -rstd^2*k2,
// C_j = -rstd*k1 + (mean - lb_j)*rstd^2*k2.   Thread = one block: dg read in tap order, l and dl in reference order.
template <typename T>
__global__ void __launch_bounds__(G7<T>::TB)
gn72_bwd_apply_kernel(const T* __restrict__ dg, const T* __restrict__ l, const float* __restrict__ lbias,
                      const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                      const float* __restrict__ s1, const float* __restrict__ s2, T* __restrict__ dl, GN72 g) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t bar;
  __shared__ float2 s_ac[576];                    // reference order: (A_j, C_j)
  __shared__ float s_bg[64];
  constexpr int TB = G7<T>::TB;
  const int tid = threadIdx.x, b = blockIdx.y;
  const int blk0 = blockIdx.x * TB, nblk = min(TB, g.bps - blk0);
  const uint32_t bytes = (uint32_t)nblk * 72u * sizeof(T);
  const long long goff = ((long long)b * g.bps + blk0) * 72;
  const uint32_t sa_dg = smem_u32(smem), sa_l = sa_dg + TB * 72 * (int)sizeof(T);
  if (tid == 0) {
    mbar_init(smem_u32(&bar), 1);
    mbar_init_fence();
    mbar_expect_tx(smem_u32(&bar), 2 * bytes);
    bulk_load(sa_dg, dg + goff, bytes, smem_u32(&bar));
    bulk_load(sa_l, l + goff, bytes, smem_u32(&bar));
  }
  const float inv_n = 1.f / (9.f * (float)g.HW);
  for (int j = tid; j < g.J; j += TB) {
    const int gi = j / 9;
    const float rs = rstd[(long long)b * g.wc + gi], mn = mean[(long long)b * g.wc + gi] - (lbias ? lbias[j] : 0.f);
    const float k1 = s1[(long long)b * g.wc + gi] * inv_n, k2 = s2[(long long)b * g.wc + gi] * inv_n;
    s_ac[j] = make_float2(rs * gamma[j], -rs * k1 + mn * rs * rs * k2);
    if (j == gi * 9) s_bg[gi] = -rs * rs * k2;
  }
  __syncthreads();
  mbar_wait(smem_u32(&bar), 0);
  if (tid < nblk) {
    const int chunk = tid % g.nchunk;
    T d[72], v[72], o[72];
    g7_ld_block<T>(sa_dg + tid * 72 * (int)sizeof(T), d);
    g7_ld_block<T>(sa_l + tid * 72 * (int)sizeof(T), v);
    const float2* ac = s_ac + chunk * 72;
    const float* bg = s_bg + chunk * 8;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float Bg = bg[i];
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const float2 c = ac[i * 9 + t];
        o[i * 9 + t] = Elem<T>::from(fmaf(to_acc(d[t * 8 + i]), c.x, fmaf(to_acc(v[i * 9 + t]), Bg, c.y)));
      }
    }
    g7_st_block<T>(sa_l + tid * 72 * (int)sizeof(T), o);
    fence_proxy_async();
  }
  __syncthreads();
  if (tid == 0) bulk_store_and_wait(dl + goff, sa_l, bytes);
}

// ------------------------------------------------------------------------------------------------ host side
// usable when the tensor is a flat array of 72-element blocks: wc in {8,16,32,64} = every CoTNet stage (gc == 8 for the
// permuting kernels), 16-byte aligned pointers, 16-bit or fp32 elements.
bool gn72_ok(int dtype, int wc, int gc, bool permuting, const void* p0, const void* p1, const void* p2) {
  if (dtype == COTB200_F64) return false;
  if (wc != 8 && wc != 16 && wc != 32 && wc != 64) return false;      // chunk count must divide the warp (shuffles) and the tile
  if (permuting && gc != 8) return false;
  return aligned16(p0) && (!p1 || aligned16(p1)) && (!p2 || aligned16(p2));
}

static GN72 make_gn72(int B, int HW, int wc, int tb) {
  GN72 g; g.B = B; g.HW = HW; g.wc = wc; g.nchunk = wc / 8; g.J = 9 * wc; g.bps = HW * g.nchunk; g.tb = tb;
  return g;
}

template <typename KFn>
static int g7_smem_attr(KFn fn, size_t smem) {
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
  }
  return 0;
}

template <typename T>
int gn72_stats_launch(int B, int HW, int wc, const void* l, const float* lbias, float* gsum, float* gsq, cudaStream_t st) {
  constexpr int TB = G7<T>::TB;
  GN72 g = make_gn72(B, HW, wc, TB);
  const size_t smem = (size_t)2 * TB * 72 * sizeof(T);
  int rc = g7_smem_attr(gn72_stats_kernel<T>, smem);
  if (rc) return rc;
  // walkers per sample: enough CTAs for ~4 per SM, never more than the sample has tiles
  const int ntiles = (g.bps + TB - 1) / TB;
  int X = (4 * num_sms() + B - 1) / B;
  if (X > ntiles) X = ntiles;
  if (X < 1) X = 1;
  DetScratch ds;
  if ((rc = ds.alloc(B * det_floats(X, 2 * wc), B, st))) return rc;
  g.det = ds.a;
  gn72_stats_kernel<T><<<dim3(X, B), TB, smem, st>>>((const T*)l, lbias, gsum, gsq, g);
  return check_launch("gn9_stats(gn72)");
}

template <typename T>
int gn72_apply_launch(int B, int HW, int wc, const void* l, const float* lbias, const float* mean, const float* rstd,
                      const float* gamma, const float* beta, void* out, cudaStream_t st) {
  constexpr int TB = G7<T>::TB;
  const GN72 g = make_gn72(B, HW, wc, TB);
  const size_t smem = (size_t)TB * 72 * sizeof(T);
  int rc = g7_smem_attr(gn72_apply_kernel<T>, smem);
  if (rc) return rc;
  gn72_apply_kernel<T><<<dim3((g.bps + TB - 1) / TB, B), TB, smem, st>>>((const T*)l, lbias, mean, rstd, gamma, beta, (T*)out, g);
  return check_launch("gn9_apply(gn72)");
}

template <typename T>
int gn72_bwd_sums_launch(int B, int HW, int wc, const void* dg, const void* l, float* P, cudaStream_t st) {
  constexpr int TB = G7<T>::TB;
  GN72 g = make_gn72(B, HW, wc, TB);
  const size_t smem = (size_t)2 * TB * 72 * sizeof(T);
  int rc = g7_smem_attr(gn72_bwd_sums_kernel<T>, smem);
  if (rc) return rc;
  const int PR = TB / g.nchunk;
  DetScratch ds;
  if ((rc = ds.alloc(B * det_floats((HW + PR - 1) / PR, 3 * g.J), B, st))) return rc;
  g.det = ds.a;
  gn72_bwd_sums_kernel<T><<<dim3((HW + PR - 1) / PR, B), G7_SUM_THREADS, smem, st>>>((const T*)dg, (const T*)l, P, g);
  return check_launch("gn9_bwd_sums(gn72)");
}

int gn_bwd_finish_launch(int B, int HW, int wc, const float* P, int raw, const float* lbias, const float* mean, const float* rstd,
                         const float* gamma, float* s1, float* s2, float* dgamma, float* dbeta, float* dlbias, cudaStream_t st) {
  gn_bwd_finish_kernel<<<wc, G7_FIN_THREADS, 0, st>>>(P, raw, lbias, mean, rstd, gamma, s1, s2, dgamma, dbeta, dlbias, B, HW, wc);
  return check_launch("gn9_bwd_finish");
}

template <typename T>
int gn72_bwd_apply_launch(int B, int HW, int wc, const void* dg, const void* l, const float* lbias, const float* mean,
                          const float* rstd, const float* gamma, const float* s1, const float* s2, void* dl, cudaStream_t st) {
  constexpr int TB = G7<T>::TB;
  const GN72 g = make_gn72(B, HW, wc, TB);
  const size_t smem = (size_t)2 * TB * 72 * sizeof(T);
  int rc = g7_smem_attr(gn72_bwd_apply_kernel<T>, smem);
  if (rc) return rc;
  gn72_bwd_apply_kernel<T><<<dim3((g.bps + TB - 1) / TB, B), TB, smem, st>>>((const T*)dg, (const T*)l, lbias, mean, rstd, gamma, s1, s2, (T*)dl, g);
  return check_launch("gn9_bwd_apply(gn72)");
}

#define G7_INST(T)                                                                                                         \
  template int gn72_stats_launch<T>(int, int, int, const void*, const float*, float*, float*, cudaStream_t);                \
  template int gn72_apply_launch<T>(int, int, int, const void*, const float*, const float*, const float*, const float*,     \
                                    const float*, void*, cudaStream_t);                                                    \
  template int gn72_bwd_sums_launch<T>(int, int, int, const void*, const void*, float*, cudaStream_t);                      \
  template int gn72_bwd_apply_launch<T>(int, int, int, const void*, const void*, const float*, const float*, const float*, \
                                        const float*, const float*, const float*, void*, cudaStream_t);
G7_INST(float)
G7_INST(__nv_bfloat16)
G7_INST(__half)

}  // namespace cotb200
