// Fused normalisation / split-attention kernels of the CoT block on NHWC tensors (sm_90a, HBM-bound).
//
// They replace long chains of eager element-wise / reduction launches of the reference block
// (/root/reference/models/cotnet.py:89-104 and the GroupNorm at :56), each a full HBM round trip:
//   * GroupNorm over the 9 taps of one weight channel (nn.GroupNorm(C/8, 9C/8), :56): stats, apply, backward
//   * the "tail":  y = SiLU(BN(u)) (:89-90);  p = mean_hw(y + k) (:92-98);  out = a0*y + a1*k (:101-104)
//     and its backward, including the BatchNorm batch-statistics reductions of training mode.
// All tensors are [B, HW, C] with the channel dimension contiguous (torch channels_last); math is fp32.
//
// One skeleton: a CTA owns (sample b, a chunk of rows); threads are (tx = 16-byte channel packet, ty = row lane), so a
// warp always touches whole 128-byte lines; per-column partial sums live in registers, are reduced across ty through
// shared memory and leave the CTA through one deterministic reduction per column (det_cols).
#include "common.cuh"

namespace cotb200 {

static constexpr int NT_THREADS = 256;

struct RowsGeo {
  int B, HW, C;          // rows per sample, channels
  int rows_per_cta;      // row chunk
  int cq;                // packets per row = C / VEC
  int ry;                // row lanes = NT_THREADS / cq_pad
  int cq_pad;            // power-of-two >= cq (thread x extent)
  int ld;                // row pitch in elements (== C unless the columns are processed in chunks)
  DetArena det;          // scratch + tickets of the closing column reductions (det_cols)
};

// fast sigmoid: ex2 + approximate reciprocal (2 ulp) instead of an IEEE division (~10 instructions) per element
__device__ __forceinline__ float sigmoidf_(float z) { return __fdividef(1.f, 1.f + __expf(-z)); }
// 16-bit tensors: sigmoid(z) = 0.5 + 0.5*tanh(z/2) with the hardware tanh (ONE MUFU op instead of ex2 + rcp; abs error
// ~2.5e-4, an order below the bf16 output ulp).  The SiLU kernels are MUFU-bound otherwise (2 x 10.7 elements/clk/SM at
// the HBM rate against 16 MUFU/clk/SM).  fp32 tensors keep the exact-ish form above.
template <typename T> __device__ __forceinline__ float sigmoid_t(float z) {
  if constexpr (sizeof(T) == 2) {
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * z));
    return fmaf(0.5f, t, 0.5f);
  } else {
    return sigmoidf_(z);
  }
}

// Reduce acc[NS][VEC] over the ty lanes of the CTA; result for column c lands in smem_out[s*C + c].
template <int NS, int VEC>
__device__ __forceinline__ void cta_col_reduce(float (&acc)[NS][VEC], float* sm, const RowsGeo& g, int tx, int ty, bool active) {
  // sm layout: [NS][ry][C]
  if (active) {
#pragma unroll
    for (int s = 0; s < NS; ++s)
#pragma unroll
      for (int i = 0; i < VEC; ++i) sm[(s * g.ry + ty) * g.C + tx * VEC + i] = acc[s][i];
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < NS * g.C; idx += NT_THREADS) {
    const int s = idx / g.C, c = idx - s * g.C;
    float t = 0.f;
    for (int y = 0; y < g.ry; ++y) t += sm[(s * g.ry + y) * g.C + c];
    sm[(s * g.ry) * g.C + c] = t;             // row 0 of each sum plane holds the CTA total
  }
  __syncthreads();
}

// The CTA's n partial values val(k) leave through det_finish (common.cuh): one group over the whole grid, or (per_sample) one
// group per sample b = blockIdx.y.  add(k, total) receives the run-to-run identical total of element k.
template <class V, class F>
__device__ __forceinline__ void det_cols(const RowsGeo& g, bool per_sample, int n, V val, F add) {
  const int nslots = per_sample ? gridDim.x : gridDim.x * gridDim.y;
  const int slot = per_sample ? blockIdx.x : blockIdx.y * gridDim.x + blockIdx.x;
  float* scr = g.det.scr + (per_sample ? blockIdx.y * det_floats(nslots, n) : 0);
  for (int k = threadIdx.x; k < n; k += NT_THREADS) scr[(size_t)slot * n + k] = val(k);
  det_finish(scr, n, slot, nslots, g.det.tick + (per_sample ? blockIdx.y : 0) * DET_TICKETS_PER_GROUP, threadIdx.x, NT_THREADS, add);
}
// the first `ns` CTA total planes of cta_col_reduce (sm[(s * ry) * C + c], s < ns) as val(k), k = s * C + c
#define NT_PLANES(sm, g) [&](int k) { const int s_ = k / (g).C; return (sm)[(s_ * (g).ry) * (g).C + (k - s_ * (g).C)]; }

// ------------------------------------------------------------------------------------------------ column statistics
// sum[c] += sum_rows x, sq[c] += sum_rows x^2       (BatchNorm batch statistics of u, models/cotnet.py:89)
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
col_stats_kernel(const T* __restrict__ x, float* __restrict__ sum, float* __restrict__ sq, RowsGeo g) {
  extern __shared__ float sm[];
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  const bool active = tx < g.cq && ty < g.ry;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float acc[2][VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  if (active) {
    const T* xp = x + ((long long)b * g.HW) * g.ld + tx * VEC;
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += g.ry) {
      const Pack<T, VEC> v = ld_pack<T, VEC>(xp + (long long)r * g.ld);
#pragma unroll
      for (int i = 0; i < VEC; ++i) { acc[0][i] = mfma<T>(v.v[i], one_of<T>(), acc[0][i]); acc[1][i] = mfma<T>(v.v[i], v.v[i], acc[1][i]); }
    }
  }
  cta_col_reduce<2, VEC>(acc, sm, g, tx, ty, active);
  det_cols(g, false, 2 * g.C, NT_PLANES(sm, g), [&](int k, float t) { if (k < g.C) sum[k] += t; else sq[k - g.C] += t; });
}

// ------------------------------------------------------------------------------------------------ tail forward
// psum[b,c] += sum_rows ( silu(u*scale+shift) + k )                      (models/cotnet.py:89-98)
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
tail_pool_kernel(const T* __restrict__ u, const T* __restrict__ k, const float* __restrict__ scale,
                 const float* __restrict__ shift, float* __restrict__ psum, RowsGeo g) {
  extern __shared__ float sm[];
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  const bool active = tx < g.cq && ty < g.ry;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float acc[1][VEC], sc[VEC], sh[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { acc[0][i] = 0.f; sc[i] = active ? scale[tx * VEC + i] : 0.f; sh[i] = active ? shift[tx * VEC + i] : 0.f; }
  if (active) {
    const long long base = ((long long)b * g.HW) * g.C + tx * VEC;
    #pragma unroll 2
    for (int r = r0 + ty; r < r1; r += g.ry) {
      const Pack<T, VEC> uv = ld_pack<T, VEC>(u + base + (long long)r * g.C);
      Pack<T, VEC> kv;
      if (k) kv = ld_pack<T, VEC>(k + base + (long long)r * g.C);      // k == NULL: SplitAttnConv2d (radix 1) pools y alone
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float z = fmaf(to_acc(uv.v[i]), sc[i], sh[i]);
        acc[0][i] += z * sigmoid_t<T>(z) + (k ? to_acc(kv.v[i]) : 0.f);
      }
    }
  }
  cta_col_reduce<1, VEC>(acc, sm, g, tx, ty, active);
  det_cols(g, true, g.C, NT_PLANES(sm, g), [&](int k, float t) { psum[(long long)b * g.C + k] += t; });
}

// out = a0 * silu(u*scale+shift) + a1 * k        a: [B, C, 2] fp32          (models/cotnet.py:101-104)
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
tail_combine_kernel(const T* __restrict__ u, const T* __restrict__ k, const float* __restrict__ scale,
                    const float* __restrict__ shift, const float* __restrict__ a, T* __restrict__ out, RowsGeo g) {
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  if (!(tx < g.cq && ty < g.ry)) return;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float sc[VEC], sh[VEC], a0[VEC], a1[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c = tx * VEC + i;
    sc[i] = scale[c]; sh[i] = shift[c];
    a0[i] = a[((long long)b * g.C + c) * 2]; a1[i] = a[((long long)b * g.C + c) * 2 + 1];
  }
  const long long base = ((long long)b * g.HW) * g.C + tx * VEC;
  #pragma unroll 2
  for (int r = r0 + ty; r < r1; r += g.ry) {
    const Pack<T, VEC> uv = ld_pack<T, VEC>(u + base + (long long)r * g.C);
    Pack<T, VEC> kv;
    if (k) kv = ld_pack<T, VEC>(k + base + (long long)r * g.C);
    Pack<T, VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float z = fmaf(to_acc(uv.v[i]), sc[i], sh[i]);
      o.v[i] = Elem<T>::from(k ? fmaf(a0[i], z * sigmoid_t<T>(z), a1[i] * to_acc(kv.v[i])) : a0[i] * (z * sigmoid_t<T>(z)));
    }
    st_pack<T, VEC>(out + base + (long long)r * g.C, o);
  }
}

// ------------------------------------------------------------------------------------------------ tail backward
// S[b,c,0] += sum_rows dout*y ; S[b,c,1] += sum_rows dout*k     (gradients of the radix-2 attention weights)
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
tail_bwd_sums_kernel(const T* __restrict__ dout, const T* __restrict__ u, const T* __restrict__ k,
                     const float* __restrict__ scale, const float* __restrict__ shift, float* __restrict__ S, RowsGeo g) {
  extern __shared__ float sm[];
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  const bool active = tx < g.cq && ty < g.ry;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float acc[2][VEC], sc[VEC], sh[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { acc[0][i] = acc[1][i] = 0.f; sc[i] = active ? scale[tx * VEC + i] : 0.f; sh[i] = active ? shift[tx * VEC + i] : 0.f; }
  if (active) {
    const long long base = ((long long)b * g.HW) * g.C + tx * VEC;
    #pragma unroll 2
    for (int r = r0 + ty; r < r1; r += g.ry) {
      const Pack<T, VEC> dv = ld_pack<T, VEC>(dout + base + (long long)r * g.C);
      const Pack<T, VEC> uv = ld_pack<T, VEC>(u + base + (long long)r * g.C);
      Pack<T, VEC> kv;
      if (k) kv = ld_pack<T, VEC>(k + base + (long long)r * g.C);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float z = fmaf(to_acc(uv.v[i]), sc[i], sh[i]);
        const float d = to_acc(dv.v[i]);
        acc[0][i] = fmaf(d, z * sigmoid_t<T>(z), acc[0][i]);
        if (k) acc[1][i] = fmaf(d, to_acc(kv.v[i]), acc[1][i]);
      }
    }
  }
  cta_col_reduce<2, VEC>(acc, sm, g, tx, ty, active);
  det_cols(g, true, 2 * g.C, NT_PLANES(sm, g), [&](int k, float t) {
    const int c = k < g.C ? k : k - g.C;
    S[((long long)b * g.C + c) * 2 + (k < g.C ? 0 : 1)] += t;
  });
}

// dz = (a0*dout + dpn) * silu'(z),  z = u*scale+shift  -- the gradient entering the BatchNorm.
// Accumulates sum_dz[c], sum_dzx[c] (x = normalised u) for the training-mode BatchNorm backward.
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
tail_bwd_dz_sums_kernel(const T* __restrict__ dout, const T* __restrict__ u, const float* __restrict__ scale,
                        const float* __restrict__ shift, const float* __restrict__ mu, const float* __restrict__ rstd,
                        const float* __restrict__ a, const float* __restrict__ dpn, float pscale, float* __restrict__ sum_dz,
                        float* __restrict__ sum_dzx, RowsGeo g) {
  extern __shared__ float sm[];
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  const bool active = tx < g.cq && ty < g.ry;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float acc[2][VEC], sc[VEC], sh[VEC], m[VEC], rs[VEC], a0[VEC], dp[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c = tx * VEC + i;
    acc[0][i] = acc[1][i] = 0.f;
    sc[i] = active ? scale[c] : 0.f; sh[i] = active ? shift[c] : 0.f; m[i] = active ? mu[c] : 0.f; rs[i] = active ? rstd[c] : 0.f;
    a0[i] = active ? a[((long long)b * g.C + c) * 2] : 0.f; dp[i] = active ? dpn[(long long)b * g.C + c] * pscale : 0.f;
  }
  if (active) {
    const long long base = ((long long)b * g.HW) * g.C + tx * VEC;
    #pragma unroll 2
    for (int r = r0 + ty; r < r1; r += g.ry) {
      const Pack<T, VEC> dv = ld_pack<T, VEC>(dout + base + (long long)r * g.C);
      const Pack<T, VEC> uv = ld_pack<T, VEC>(u + base + (long long)r * g.C);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float uf = to_acc(uv.v[i]);
        const float z = fmaf(uf, sc[i], sh[i]);
        const float s = sigmoid_t<T>(z);
        const float dz = fmaf(a0[i], to_acc(dv.v[i]), dp[i]) * (s * (1.f + z * (1.f - s)));
        acc[0][i] += dz;
        acc[1][i] = fmaf(dz, (uf - m[i]) * rs[i], acc[1][i]);
      }
    }
  }
  cta_col_reduce<2, VEC>(acc, sm, g, tx, ty, active);
  det_cols(g, false, 2 * g.C, NT_PLANES(sm, g), [&](int k, float t) { if (k < g.C) sum_dz[k] += t; else sum_dzx[k - g.C] += t; });
}

// du = scale * (dz - c1 - xhat*c2)   [c1 = sum_dz/n, c2 = sum_dzx/n in training; 0 in eval]
// dk = a1*dout + dpn
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
tail_bwd_apply_kernel(const T* __restrict__ dout, const T* __restrict__ u, const float* __restrict__ scale,
                      const float* __restrict__ shift, const float* __restrict__ mu, const float* __restrict__ rstd,
                      const float* __restrict__ a, const float* __restrict__ dpn, const float* __restrict__ c1,
                      const float* __restrict__ c2, float inv_n, float pscale, T* __restrict__ du, T* __restrict__ dk, RowsGeo g) {
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  if (!(tx < g.cq && ty < g.ry)) return;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float sc[VEC], sh[VEC], m[VEC], rs[VEC], a0[VEC], a1[VEC], dp[VEC], k1[VEC], k2[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c = tx * VEC + i;
    sc[i] = scale[c]; sh[i] = shift[c]; m[i] = mu[c]; rs[i] = rstd[c];
    a0[i] = a[((long long)b * g.C + c) * 2]; a1[i] = a[((long long)b * g.C + c) * 2 + 1]; dp[i] = dpn[(long long)b * g.C + c] * pscale;
    k1[i] = c1 ? c1[c] * inv_n : 0.f; k2[i] = c2 ? c2[c] * inv_n : 0.f;
  }
  const long long base = ((long long)b * g.HW) * g.C + tx * VEC;
  #pragma unroll 2
  for (int r = r0 + ty; r < r1; r += g.ry) {
    const Pack<T, VEC> dv = ld_pack<T, VEC>(dout + base + (long long)r * g.C);
    const Pack<T, VEC> uv = ld_pack<T, VEC>(u + base + (long long)r * g.C);
    Pack<T, VEC> o1, o2;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float uf = to_acc(uv.v[i]), d = to_acc(dv.v[i]);
      const float z = fmaf(uf, sc[i], sh[i]);
      const float s = sigmoid_t<T>(z);
      const float dz = fmaf(a0[i], d, dp[i]) * (s * (1.f + z * (1.f - s)));
      o1.v[i] = Elem<T>::from(sc[i] * (dz - k1[i] - (uf - m[i]) * rs[i] * k2[i]));
      o2.v[i] = Elem<T>::from(fmaf(a1[i], d, dp[i]));
    }
    st_pack<T, VEC>(du + base + (long long)r * g.C, o1);
    if (dk) st_pack<T, VEC>(dk + base + (long long)r * g.C, o2);
  }
}

// ------------------------------------------------------------------------------------------------ BatchNorm (+ReLU, +residual)
// Training / eval BatchNorm2d on NHWC tensors as 2 + 2 HBM passes (col_stats + apply; bwd sums + bwd apply), replacing
// ATen's channels_last batch-norm kernels (ncu: 4 kernels, ~0.65 TB/s on the stage-1 tensors).
//   ACT: 0 none, 1 ReLU.   y = act(x*scale + shift (+ res))                  (models/cotnet.py:45-46,53-54,61-62,:248-262)
// FIN: the BatchNorm bookkeeping of bn_finalize_kernel is done in the prologue instead of a separate launch -- every thread
// derives scale/shift of its own columns from the batch sums (4 loads + one rsqrt per column, nothing next to >= 64 rows of
// streaming), CTA (0,0) also publishes scale/shift/mean/rstd for the backward and updates the running statistics.
struct BnFin {
  const float* sum; const float* sq; const float* weight; const float* bias;
  float* running_mean; float* running_var;
  float n, eps, momentum; int update_running;
  float* scale; float* shift; float* mean; float* rstd;
};

// DS (stochastic depth, models/cotnet.py:256-257): y = act(ds[b]*(x*scale + shift) (+ res)), ds [B] per-sample scales in
// {0, 1/keep}; the kernels see the flattened rows, so the sample of row r is r / ds_hw.  DS == false compiles to the plain form.
template <typename T, int VEC, int ACT, bool RES, bool FIN, bool DS = false>
__global__ void __launch_bounds__(NT_THREADS)
bn_apply_kernel(const T* __restrict__ x, const T* __restrict__ res, const float* __restrict__ scale,
                const float* __restrict__ shift, T* __restrict__ y, RowsGeo g, BnFin f, const float* __restrict__ ds, int ds_hw) {
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  if (!(tx < g.cq && ty < g.ry)) return;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float sc[VEC], sh[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c = tx * VEC + i;
    if (FIN) {
      const float mean = f.sum[c] / f.n;
      const float var = fmaxf(f.sq[c] / f.n - mean * mean, 0.f);
      const float rstd = rsqrtf(var + f.eps);
      sc[i] = (f.weight ? f.weight[c] : 1.f) * rstd;
      sh[i] = (f.bias ? f.bias[c] : 0.f) - mean * sc[i];
      if (blockIdx.x == 0 && blockIdx.y == 0 && ty == 0) {
        f.scale[c] = sc[i]; f.shift[c] = sh[i]; f.mean[c] = mean; f.rstd[c] = rstd;
        if (f.update_running) {
          f.running_mean[c] = (1.f - f.momentum) * f.running_mean[c] + f.momentum * mean;
          f.running_var[c] = (1.f - f.momentum) * f.running_var[c] + f.momentum * var * (f.n / fmaxf(f.n - 1.f, 1.f));
        }
      }
    } else {
      sc[i] = scale[c]; sh[i] = shift[c];
    }
  }
  const long long base = ((long long)b * g.HW) * g.ld + tx * VEC;
  for (int r = r0 + ty; r < r1; r += g.ry) {
    const Pack<T, VEC> xv = ld_pack<T, VEC>(x + base + (long long)r * g.ld);
    Pack<T, VEC> rv;
    if (RES) rv = ld_pack<T, VEC>(res + base + (long long)r * g.ld);
    Pack<T, VEC> o;
    float s = 1.f;
    if (DS) s = __ldg(ds + r / ds_hw);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      float z = fmaf(to_acc(xv.v[i]), sc[i], sh[i]);
      if (DS) z *= s;
      if (RES) z += to_acc(rv.v[i]);
      if (ACT == 1) z = fmaxf(z, 0.f);
      o.v[i] = Elem<T>::from(z);
    }
    st_pack<T, VEC>(y + base + (long long)r * g.ld, o);
  }
}

// dz = dy * [y > 0] (ACT==1: mask read from y ; ACT==2: mask recomputed as x*scale+shift > 0, one HBM pass less) ;
// sum_dz[c] += dz ; sum_dzx[c] += dz * xhat.   DS: the BatchNorm output was scaled by ds[b], so its gradient is ds[b]*dz.
template <typename T, int VEC, int ACT, bool DS = false>
__global__ void __launch_bounds__(NT_THREADS)
bn_bwd_sums_kernel(const T* __restrict__ dy, const T* __restrict__ dy2, const T* __restrict__ x, const T* __restrict__ y, const float* __restrict__ scale,
                   const float* __restrict__ shift, const float* __restrict__ mu, const float* __restrict__ rstd,
                   float* __restrict__ sum_dz, float* __restrict__ sum_dzx, RowsGeo g, const float* __restrict__ ds, int ds_hw) {
  extern __shared__ float sm[];
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  const bool active = tx < g.cq && ty < g.ry;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float acc[2][VEC], m[VEC], rs[VEC], sc[VEC], sh[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    acc[0][i] = acc[1][i] = 0.f; m[i] = active ? mu[tx * VEC + i] : 0.f; rs[i] = active ? rstd[tx * VEC + i] : 0.f;
    sc[i] = (ACT == 2 && active) ? scale[tx * VEC + i] : 0.f; sh[i] = (ACT == 2 && active) ? shift[tx * VEC + i] : 0.f;
  }
  if (active) {
    const long long base = ((long long)b * g.HW) * g.ld + tx * VEC;
    for (int r = r0 + ty; r < r1; r += g.ry) {
      const Pack<T, VEC> dv = ld_pack<T, VEC>(dy + base + (long long)r * g.ld);
      const Pack<T, VEC> xv = ld_pack<T, VEC>(x + base + (long long)r * g.ld);
      Pack<T, VEC> yv, d2;
      if (ACT == 1) yv = ld_pack<T, VEC>(y + base + (long long)r * g.ld);
      if (dy2) d2 = ld_pack<T, VEC>(dy2 + base + (long long)r * g.ld);    // two-consumer output: dy = dy + dy2, summed here in fp32
      float s = 1.f;
      if (DS) s = __ldg(ds + r / ds_hw);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        float dz = to_acc(dv.v[i]);
        if (dy2) dz += to_acc(d2.v[i]);
        const float xf = to_acc(xv.v[i]);
        if (ACT == 1 && !(to_acc(yv.v[i]) > 0.f)) dz = 0.f;
        if (ACT == 2 && !((DS ? fmaf(xf, sc[i], sh[i]) * s : fmaf(xf, sc[i], sh[i])) > 0.f)) dz = 0.f;   // the forward's own fp32 z: identical mask, y not read
        if (DS) dz *= s;
        acc[0][i] += dz;
        acc[1][i] = fmaf(dz, (xf - m[i]) * rs[i], acc[1][i]);
      }
    }
  }
  cta_col_reduce<2, VEC>(acc, sm, g, tx, ty, active);
  det_cols(g, false, 2 * g.C, NT_PLANES(sm, g), [&](int k, float t) { if (k < g.C) sum_dz[k] += t; else sum_dzx[k - g.C] += t; });
}

// dx = scale * (dz - c1 - xhat*c2)   (c1 = c2 = 0 in eval mode);   dres = dz when RES
// DS: dx = scale * (ds[b]*dz - c1 - xhat*c2), dres = dz
template <typename T, int VEC, int ACT, bool RES, bool DS = false>
__global__ void __launch_bounds__(NT_THREADS)
bn_bwd_apply_kernel(const T* __restrict__ dy, const T* __restrict__ dy2, const T* __restrict__ x, const T* __restrict__ y, const float* __restrict__ scale,
                    const float* __restrict__ shift, const float* __restrict__ mu, const float* __restrict__ rstd,
                    const float* __restrict__ c1, const float* __restrict__ c2, float inv_n, T* __restrict__ dx,
                    T* __restrict__ dres, RowsGeo g, const float* __restrict__ ds, int ds_hw) {
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  if (!(tx < g.cq && ty < g.ry)) return;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float sc[VEC], sh[VEC], m[VEC], rs[VEC], k1[VEC], k2[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c = tx * VEC + i;
    sc[i] = scale[c]; sh[i] = ACT == 2 ? shift[c] : 0.f; m[i] = mu[c]; rs[i] = rstd[c];
    k1[i] = c1 ? c1[c] * inv_n : 0.f; k2[i] = c2 ? c2[c] * inv_n : 0.f;
  }
  const long long base = ((long long)b * g.HW) * g.ld + tx * VEC;
  for (int r = r0 + ty; r < r1; r += g.ry) {
    const Pack<T, VEC> dv = ld_pack<T, VEC>(dy + base + (long long)r * g.ld);
    const Pack<T, VEC> xv = ld_pack<T, VEC>(x + base + (long long)r * g.ld);
    Pack<T, VEC> yv, d2;
    if (ACT == 1) yv = ld_pack<T, VEC>(y + base + (long long)r * g.ld);
    if (dy2) d2 = ld_pack<T, VEC>(dy2 + base + (long long)r * g.ld);
    Pack<T, VEC> o, o2;
    float s = 1.f;
    if (DS) s = __ldg(ds + r / ds_hw);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      float dz = to_acc(dv.v[i]);
      if (dy2) dz += to_acc(d2.v[i]);
      const float xf = to_acc(xv.v[i]);
      if (ACT == 1 && !(to_acc(yv.v[i]) > 0.f)) dz = 0.f;
      if (ACT == 2 && !((DS ? fmaf(xf, sc[i], sh[i]) * s : fmaf(xf, sc[i], sh[i])) > 0.f)) dz = 0.f;
      o.v[i] = Elem<T>::from(sc[i] * ((DS ? dz * s : dz) - k1[i] - (xf - m[i]) * rs[i] * k2[i]));
      if (RES) o2.v[i] = Elem<T>::from(dz);
    }
    st_pack<T, VEC>(dx + base + (long long)r * g.ld, o);
    if (RES) st_pack<T, VEC>(dres + base + (long long)r * g.ld, o2);
  }
}

// One tiny launch instead of ~12 eager ops: batch mean / biased var from the column sums, scale/shift for the apply
// pass, mean/rstd for the backward pass, and the nn.BatchNorm2d running-buffer update (momentum, unbiased variance).
// use_batch == 0: eval mode, statistics come from the running buffers.
__global__ void bn_finalize_kernel(const float* __restrict__ sum, const float* __restrict__ sq, const float* __restrict__ weight,
                                   const float* __restrict__ bias, float* __restrict__ running_mean,
                                   float* __restrict__ running_var, float n, float eps, float momentum, int use_batch,
                                   int update_running, float* __restrict__ scale, float* __restrict__ shift,
                                   float* __restrict__ mean_out, float* __restrict__ rstd_out, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float mean, var;
  if (use_batch) {
    mean = sum[c] / n;
    var = fmaxf(sq[c] / n - mean * mean, 0.f);
    if (update_running) {
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * var * (n / fmaxf(n - 1.f, 1.f));
    }
  } else {
    mean = running_mean[c];
    var = running_var[c];
  }
  const float rstd = rsqrtf(var + eps);
  const float sc = (weight ? weight[c] : 1.f) * rstd;
  scale[c] = sc;
  shift[c] = (bias ? bias[c] : 0.f) - mean * sc;
  mean_out[c] = mean;
  rstd_out[c] = rstd;
}

// ------------------------------------------------------------------------------------------------ GroupNorm(9 taps)
// The logits l (and dl) are always in the reference channel order j = g*9 + t (they come out of / go into the
// embed.3 convolution).  The normalised weights ghat (and their gradient dg) are stored in the order the LocalConv
// kernels want: gc == 0 the same order; gc > 0 tap-major chunks of gc weight channels (COTB200_NHWC_TAP):
// position of (g, t) = ((g/gc)*9 + t)*gc + g%gc.
__device__ __forceinline__ int gn_pos(int j, int gc) {
  if (gc <= 0) return j;
  const int gi = j / 9, t = j - gi * 9;
  return ((gi / gc) * 9 + t) * gc + gi % gc;
}
__device__ __forceinline__ int gn_j_of_pos(int pos, int gc) {
  if (gc <= 0) return pos;
  const int chunk = pos / (9 * gc), rr = pos - chunk * 9 * gc;
  const int t = rr / gc, i = rr - t * gc;
  return (chunk * gc + i) * 9 + t;
}

// gsum[b,g] += sum over (9 taps x rows) of l ; gsq likewise
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
gn_stats_kernel(const T* __restrict__ l, const float* __restrict__ lbias, float* __restrict__ gsum, float* __restrict__ gsq,
                RowsGeo g, int wc) {
  extern __shared__ float sm[];
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  const bool active = tx < g.cq && ty < g.ry;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float acc[2][VEC], lb[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) { acc[0][i] = acc[1][i] = 0.f; lb[i] = (active && lbias) ? lbias[tx * VEC + i] : 0.f; }
  if (active) {
    const T* lp = l + ((long long)b * g.HW) * g.C + tx * VEC;
#pragma unroll 4
    for (int r = r0 + ty; r < r1; r += g.ry) {
      const Pack<T, VEC> v = ld_pack<T, VEC>(lp + (long long)r * g.C);
#pragma unroll
      for (int i = 0; i < VEC; ++i) { const float f = to_acc(v.v[i]) + lb[i]; acc[0][i] += f; acc[1][i] = fmaf(f, f, acc[1][i]); }
    }
  }
  cta_col_reduce<2, VEC>(acc, sm, g, tx, ty, active);
  det_cols(g, true, 2 * wc, [&](int k) {                        // fold the 9 tap columns of each group
    const int pl = k < wc ? 0 : 1, gi = k - pl * wc;
    float s = 0.f;
    for (int t = 0; t < 9; ++t) s += sm[pl * g.ry * g.C + gi * 9 + t];
    return s;
  }, [&](int k, float t) { if (k < wc) gsum[(long long)b * wc + k] += t; else gsq[(long long)b * wc + k - wc] += t; });
}

// ghat[pos(j)] = (l[j] - mean[b,g]) * rstd[b,g] * gamma[j] + beta[j].  Thread = one OUTPUT packet (coalesced 16-byte
// store); the VEC inputs are gathered (stride 9 inside the pixel's 18*wc-byte row, L1 hits).
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
gn_apply_kernel(const T* __restrict__ l, const float* __restrict__ lbias, const float* __restrict__ mean, const float* __restrict__ rstd,
                const float* __restrict__ gamma, const float* __restrict__ beta, T* __restrict__ out, RowsGeo g, int wc, int gc) {
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  if (!(tx < g.cq && ty < g.ry)) return;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float A[VEC], Bc[VEC];
  int jin[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int j = gn_j_of_pos(tx * VEC + i, gc), gi = j / 9;
    jin[i] = j;
    const float rs = rstd[(long long)b * wc + gi], mn = mean[(long long)b * wc + gi];
    A[i] = rs * gamma[j];
    Bc[i] = beta[j] - (mn - (lbias ? lbias[j] : 0.f)) * A[i];
  }
  const long long base = ((long long)b * g.HW) * g.C;
  for (int r = r0 + ty; r < r1; r += g.ry) {
    const T* lr = l + base + (long long)r * g.C;
    Pack<T, VEC> o;
    if (gc <= 0) {
      const Pack<T, VEC> v = ld_pack<T, VEC>(lr + tx * VEC);
#pragma unroll
      for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(fmaf(to_acc(v.v[i]), A[i], Bc[i]));
    } else {
#pragma unroll
      for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(fmaf(Elem<T>::ld(lr + jin[i]), A[i], Bc[i]));
    }
    st_pack<T, VEC>(out + base + (long long)r * g.C + tx * VEC, o);
  }
}

// backward sums, per (sample, column j) partials:  P[b][0][j] += sum dg ; P[b][1][j] += sum dg*lhat ; P[b][2][j] += sum lhat
// (lhat = (l + lbias - mean)*rstd).  gn_bwd_finish_kernel (gn72.cu) turns them into s1, s2, dgamma, dbeta and the bias
// gradient.  Thread = one packet of l in the reference order; dg gathered from its storage order.
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
gn_bwd_sums_kernel(const T* __restrict__ dg, const T* __restrict__ l, const float* __restrict__ lbias, const float* __restrict__ mean,
                   const float* __restrict__ rstd, float* __restrict__ P, RowsGeo g, int wc, int gc) {
  extern __shared__ float sm[];
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  const bool active = tx < g.cq && ty < g.ry;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  float acc[3][VEC], mn[VEC], rs[VEC];    // acc[0] = sum dg ; acc[1] = sum dg*lhat ; acc[2] = sum lhat   (per column j)
  int pos[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    acc[0][i] = acc[1][i] = acc[2][i] = 0.f;
    const int j = tx * VEC + i, gi = active ? j / 9 : 0;
    pos[i] = active ? gn_pos(j, gc) : 0;
    mn[i] = active ? mean[(long long)b * wc + gi] - (lbias ? lbias[j] : 0.f) : 0.f;     // (l + bias - mean) = l - mn
    rs[i] = active ? rstd[(long long)b * wc + gi] : 0.f;
  }
  if (active) {
    const long long base = ((long long)b * g.HW) * g.C;
    for (int r = r0 + ty; r < r1; r += g.ry) {
      const T* dr = dg + base + (long long)r * g.C;
      const Pack<T, VEC> lv = ld_pack<T, VEC>(l + base + (long long)r * g.C + tx * VEC);
      Pack<T, VEC> dv;
      if (gc <= 0) dv = ld_pack<T, VEC>(dr + tx * VEC);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float d = gc <= 0 ? to_acc(dv.v[i]) : (float)Elem<T>::ld(dr + pos[i]);
        const float lh = (to_acc(lv.v[i]) - mn[i]) * rs[i];
        acc[0][i] += d;
        acc[1][i] = fmaf(d, lh, acc[1][i]);
        acc[2][i] += lh;
      }
    }
  }
  cta_col_reduce<3, VEC>(acc, sm, g, tx, ty, active);
  float* Pb = P + (long long)b * 3 * g.C;
  det_cols(g, true, 3 * g.C, NT_PLANES(sm, g), [&](int k, float t) { Pb[k] += t; });
}

// dl = rstd * ( dg*gamma - s1/n - lhat * s2/n ),  n = 9*HW
template <typename T, int VEC>
__global__ void __launch_bounds__(NT_THREADS)
gn_bwd_apply_kernel(const T* __restrict__ dg, const T* __restrict__ l, const float* __restrict__ lbias,
                    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                    const float* __restrict__ s1, const float* __restrict__ s2, T* __restrict__ dl, RowsGeo g, int wc, int gc) {
  const int tx = threadIdx.x % g.cq_pad, ty = threadIdx.x / g.cq_pad;
  if (!(tx < g.cq && ty < g.ry)) return;
  const int b = blockIdx.y, r0 = blockIdx.x * g.rows_per_cta, r1 = min(g.HW, r0 + g.rows_per_cta);
  const float inv_n = 1.f / (9.f * (float)g.HW);
  float mn[VEC], rs[VEC], ga[VEC], k1[VEC], k2[VEC];
  int pos[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int j = tx * VEC + i, gi = j / 9;
    pos[i] = gn_pos(j, gc);
    mn[i] = mean[(long long)b * wc + gi] - (lbias ? lbias[j] : 0.f); rs[i] = rstd[(long long)b * wc + gi]; ga[i] = gamma[j];
    k1[i] = s1[(long long)b * wc + gi] * inv_n; k2[i] = s2[(long long)b * wc + gi] * inv_n;
  }
  const long long base = ((long long)b * g.HW) * g.C;
  for (int r = r0 + ty; r < r1; r += g.ry) {
    const T* dr = dg + base + (long long)r * g.C;
    const Pack<T, VEC> lv = ld_pack<T, VEC>(l + base + (long long)r * g.C + tx * VEC);
    Pack<T, VEC> dv;
    if (gc <= 0) dv = ld_pack<T, VEC>(dr + tx * VEC);
    Pack<T, VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float d = gc <= 0 ? to_acc(dv.v[i]) : (float)Elem<T>::ld(dr + pos[i]);
      const float lh = (to_acc(lv.v[i]) - mn[i]) * rs[i];
      o.v[i] = Elem<T>::from(rs[i] * (d * ga[i] - k1[i] - lh * k2[i]));
    }
    st_pack<T, VEC>(dl + base + (long long)r * g.C + tx * VEC, o);
  }
}

// ------------------------------------------------------------------------------------------------ host
template <typename T>
static int pick_vec(int C, const void* p0, const void* p1 = nullptr, const void* p2 = nullptr, const void* p3 = nullptr) {
  for (int vec = 16 / (int)sizeof(T); vec >= 1; vec >>= 1) {
    if (C % vec) continue;
    const uintptr_t m = (uintptr_t)(vec * sizeof(T)) - 1;
    auto ok = [&](const void* p) { return !p || ((uintptr_t)p & m) == 0; };
    if (ok(p0) && ok(p1) && ok(p2) && ok(p3)) return vec;
  }
  return 1;
}

static int make_geo(RowsGeo& g, int B, int HW, int C, int vec, int nsums, size_t* smem) {
  if (B <= 0 || HW <= 0 || C <= 0) { set_error("norm/tail kernel: non-positive dims"); return COTB200_EINVAL; }
  g.B = B; g.HW = HW; g.C = C; g.cq = C / vec; g.ld = C;
  g.cq_pad = 1;
  while (g.cq_pad < g.cq) g.cq_pad <<= 1;
  if (g.cq_pad > NT_THREADS) { set_error("norm/tail kernel: %d channels exceed the %d-packet row limit", C, NT_THREADS); return COTB200_EINVAL; }
  g.ry = NT_THREADS / g.cq_pad;
  // rows per CTA: the CTA count along the rows is a whole multiple k of the SM count (k = 6 .. 1: no partial last wave) with at
  // least `min_rows` rows each, so that the closing column reductions (vector reds, one per four columns per CTA) stay amortised.
  // Short, wide tensors (the 7x7 stage: 12 544 rows x 512..2048 channels) used to get 196 CTAs of 64 rows -- 1.3 waves of ONE
  // 256-thread CTA per SM, latency-bound at ~0.25 of the roof; they now get 3-4 CTAs per SM.
  int min_rows = g.ry * 2;
  if (min_rows < 24) min_rows = 24;
  const int sms = num_sms();
  int rows = HW;
  for (int k = 6; k >= 1; --k) {
    const long long ctas = (long long)sms * k;
    const int per_b = (int)((ctas + B - 1) / B);           // row chunks per sample
    const int r = (HW + per_b - 1) / per_b;
    rows = r;
    if (r >= min_rows) break;
  }
  if (rows < min_rows) rows = min_rows;
  if (rows > HW) rows = HW;
  g.rows_per_cta = rows;
  *smem = (size_t)nsums * g.ry * C * sizeof(float);
  if (*smem > 96 * 1024) { set_error("norm/tail kernel: shared memory %zu too large", *smem); return COTB200_EINVAL; }
  return 0;
}

// Stream-ordered scratch of the closing reduction of a reducing row kernel (det_cols) with geometry g and `nsums` planes of
// g.C values: one group over the whole grid or one per sample, whichever the kernel uses.
static int det_geo(DetScratch& ds, RowsGeo& g, int nsums, cudaStream_t st) {
  const int gx = (g.HW + g.rows_per_cta - 1) / g.rows_per_cta, n = nsums * g.C;
  const size_t per_sample = (size_t)g.B * det_floats(gx, n), whole = det_floats(gx * g.B, n);
  const int rc = ds.alloc(per_sample > whole ? per_sample : whole, g.B, st);
  g.det = ds.a;
  return rc;
}

// Wide tensors (more than 256 packets per row, e.g. the 2048-channel bn3 of layer4 in fp32) are processed in equal
// column chunks: returns the chunk width (a multiple of vec that divides C) or C itself.
static int col_chunk(int C, int vec) {
  if (C / vec <= NT_THREADS) return C;
  for (int nz = 2; nz <= 64; ++nz)
    if (C % nz == 0 && (C / nz) % vec == 0 && (C / nz) / vec <= NT_THREADS) return C / nz;
  return 0;
}

#define NT_DISPATCH_VEC(vec, ...)                                  \
  switch (vec) {                                                   \
    case 8: if constexpr (sizeof(T) == 2) { constexpr int V = 8; __VA_ARGS__; } break; \
    case 4: { constexpr int V = 4; __VA_ARGS__; } break;           \
    case 2: { constexpr int V = 2; __VA_ARGS__; } break;           \
    default: { constexpr int V = 1; __VA_ARGS__; } break;          \
  }

template <typename KFn>
static int ensure_smem(KFn fn, size_t smem) {
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
  }
  return 0;
}

// block-of-72 kernels (gn72.cu)
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

using namespace cotb200;

#define NT_GRID dim3((g.HW + g.rows_per_cta - 1) / g.rows_per_cta, g.B)

extern "C" int cotb200_col_stats(int dtype, int B, int HW, int C, const void* x, float* sum, float* sq, void* stream) {
  if (!x || !sum || !sq) { set_error("col_stats: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("col_stats: fp64 not supported"); return COTB200_EDTYPE; }
  { const long long rows = (long long)B * HW; if (rows > 2147483647LL) { set_error("cotb200_col_stats: too many rows"); return COTB200_ETOOBIG; }
    HW = (int)rows; B = 1; }      // per-channel statistics: flatten [B, HW] -> rows
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pick_vec<T>(C, x);
      const int cw = col_chunk(C, vec);
      if (!cw) { set_error("col_stats: cannot tile %d channels", C); return COTB200_EINVAL; }
      for (int c0 = 0; c0 < C; c0 += cw) {
        RowsGeo g; size_t smem;
        int rc = make_geo(g, B, HW, cw, vec, 2, &smem);
        if (rc) return rc;
        DetScratch ds;                                   // stream-ordered scratch of the closing reduction
        if ((rc = det_geo(ds, g, 2, st))) return rc;
        g.ld = C;
        COTB200_PROF_B("col_stats", (double)B * HW * cw * sizeof(T));
        NT_DISPATCH_VEC(vec, { if ((rc = ensure_smem(col_stats_kernel<T, V>, smem))) return rc;
                               col_stats_kernel<T, V><<<NT_GRID, NT_THREADS, smem, st>>>((const T*)x + c0, sum + c0, sq + c0, g); });
        if ((rc = check_launch("col_stats"))) return rc;
      }
      return 0;
    }
  });
  return 0;
}

extern "C" int cotb200_tail_pool(int dtype, int B, int HW, int C, const void* u, const void* k, const float* scale,
                                 const float* shift, float* psum, void* stream) {
  if (!u || !scale || !shift || !psum) { set_error("tail_pool: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("tail_pool: fp64 not supported"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pick_vec<T>(C, u, k);
      RowsGeo g; size_t smem;
      int rc = make_geo(g, B, HW, C, vec, 1, &smem);
      if (rc) return rc;
      DetScratch ds;                                   // stream-ordered scratch of the closing reduction
      if ((rc = det_geo(ds, g, 1, st))) return rc;
      COTB200_PROF_B("tail_pool", (double)B * HW * C * 2 * sizeof(T));
      NT_DISPATCH_VEC(vec, { if ((rc = ensure_smem(tail_pool_kernel<T, V>, smem))) return rc;
                             tail_pool_kernel<T, V><<<NT_GRID, NT_THREADS, smem, st>>>((const T*)u, (const T*)k, scale, shift, psum, g); });
      return check_launch("tail_pool");
    }
  });
  return 0;
}

extern "C" int cotb200_tail_combine(int dtype, int B, int HW, int C, const void* u, const void* k, const float* scale,
                                    const float* shift, const float* a, void* out, void* stream) {
  if (!u || !scale || !shift || !a || !out) { set_error("tail_combine: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("tail_combine: fp64 not supported"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pick_vec<T>(C, u, k, out);
      RowsGeo g; size_t smem;
      int rc = make_geo(g, B, HW, C, vec, 1, &smem);
      if (rc) return rc;
      COTB200_PROF_B("tail_combine", (double)B * HW * C * 3 * sizeof(T));
      NT_DISPATCH_VEC(vec, { tail_combine_kernel<T, V><<<NT_GRID, NT_THREADS, 0, st>>>((const T*)u, (const T*)k, scale, shift, a, (T*)out, g); });
      return check_launch("tail_combine");
    }
  });
  return 0;
}

extern "C" int cotb200_tail_bwd_sums(int dtype, int B, int HW, int C, const void* dout, const void* u, const void* k,
                                     const float* scale, const float* shift, float* S, void* stream) {
  if (!dout || !u || !scale || !shift || !S) { set_error("tail_bwd_sums: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("tail_bwd_sums: fp64 not supported"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pick_vec<T>(C, dout, u, k);
      RowsGeo g; size_t smem;
      int rc = make_geo(g, B, HW, C, vec, 2, &smem);
      if (rc) return rc;
      DetScratch ds;                                   // stream-ordered scratch of the closing reduction
      if ((rc = det_geo(ds, g, 2, st))) return rc;
      COTB200_PROF_B("tail_bwd_sums", (double)B * HW * C * 3 * sizeof(T));
      NT_DISPATCH_VEC(vec, { if ((rc = ensure_smem(tail_bwd_sums_kernel<T, V>, smem))) return rc;
                             tail_bwd_sums_kernel<T, V><<<NT_GRID, NT_THREADS, smem, st>>>((const T*)dout, (const T*)u, (const T*)k, scale, shift, S, g); });
      return check_launch("tail_bwd_sums");
    }
  });
  return 0;
}

extern "C" int cotb200_tail_bwd_dz_sums(int dtype, int B, int HW, int C, const void* dout, const void* u, const float* scale,
                                        const float* shift, const float* mu, const float* rstd, const float* a,
                                        const float* dpn, float pscale, float* sum_dz, float* sum_dzx, void* stream) {
  if (!dout || !u || !scale || !shift || !mu || !rstd || !a || !dpn || !sum_dz || !sum_dzx) { set_error("tail_bwd_dz_sums: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("tail_bwd_dz_sums: fp64 not supported"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pick_vec<T>(C, dout, u);
      RowsGeo g; size_t smem;
      int rc = make_geo(g, B, HW, C, vec, 2, &smem);
      if (rc) return rc;
      DetScratch ds;                                   // stream-ordered scratch of the closing reduction
      if ((rc = det_geo(ds, g, 2, st))) return rc;
      COTB200_PROF_B("tail_bwd_dz_sums", (double)B * HW * C * 2 * sizeof(T));
      NT_DISPATCH_VEC(vec, { if ((rc = ensure_smem(tail_bwd_dz_sums_kernel<T, V>, smem))) return rc;
                             tail_bwd_dz_sums_kernel<T, V><<<NT_GRID, NT_THREADS, smem, st>>>((const T*)dout, (const T*)u, scale, shift, mu, rstd, a, dpn, pscale, sum_dz, sum_dzx, g); });
      return check_launch("tail_bwd_dz_sums");
    }
  });
  return 0;
}

extern "C" int cotb200_tail_bwd_apply(int dtype, int B, int HW, int C, const void* dout, const void* u, const float* scale,
                                      const float* shift, const float* mu, const float* rstd, const float* a,
                                      const float* dpn, const float* c1, const float* c2, float inv_n, float pscale, void* du, void* dk,
                                      void* stream) {
  if (!dout || !u || !scale || !shift || !mu || !rstd || !a || !dpn || !du) { set_error("tail_bwd_apply: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("tail_bwd_apply: fp64 not supported"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pick_vec<T>(C, dout, u, du, dk);
      RowsGeo g; size_t smem;
      int rc = make_geo(g, B, HW, C, vec, 1, &smem);
      if (rc) return rc;
      COTB200_PROF_B("tail_bwd_apply", (double)B * HW * C * 4 * sizeof(T));
      NT_DISPATCH_VEC(vec, { tail_bwd_apply_kernel<T, V><<<NT_GRID, NT_THREADS, 0, st>>>((const T*)dout, (const T*)u, scale, shift, mu, rstd, a, dpn, c1, c2, inv_n, pscale, (T*)du, (T*)dk, g); });
      return check_launch("tail_bwd_apply");
    }
  });
  return 0;
}

extern "C" int cotb200_gn9_stats(int dtype, int B, int HW, int wc, int gc, const void* l, const float* lbias, float* gsum,
                                 float* gsq, void* stream) {
  if (!l || !gsum || !gsq) { set_error("gn9_stats: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("gn9_stats: fp64 not supported"); return COTB200_EDTYPE; }
  if (gc > 0 && wc % gc) { set_error("gn9: gc %d does not divide wc %d", gc, wc); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const int J = 9 * wc;
  const bool fast = gn72_ok(dtype, wc, gc, false, l, nullptr, nullptr);
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("gn9_stats", (double)B * HW * J * sizeof(T));
      if (fast) return gn72_stats_launch<T>(B, HW, wc, l, lbias, gsum, gsq, st);
      const int vec = pick_vec<T>(J, l);
      RowsGeo g; size_t smem;
      int rc = make_geo(g, B, HW, J, vec, 2, &smem);
      if (rc) return rc;
      DetScratch ds;                                   // stream-ordered scratch of the closing reduction
      if ((rc = det_geo(ds, g, 2, st))) return rc;
      NT_DISPATCH_VEC(vec, { if ((rc = ensure_smem(gn_stats_kernel<T, V>, smem))) return rc;
                             gn_stats_kernel<T, V><<<NT_GRID, NT_THREADS, smem, st>>>((const T*)l, lbias, gsum, gsq, g, wc); });
      return check_launch("gn9_stats");
    }
  });
  return 0;
}

extern "C" int cotb200_gn9_apply(int dtype, int B, int HW, int wc, int gc, const void* l, const float* lbias, const float* mean,
                                 const float* rstd, const float* gamma, const float* beta, void* out, void* stream) {
  if (!l || !mean || !rstd || !gamma || !beta || !out) { set_error("gn9_apply: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("gn9_apply: fp64 not supported"); return COTB200_EDTYPE; }
  if (gc > 0 && wc % gc) { set_error("gn9: gc %d does not divide wc %d", gc, wc); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const int J = 9 * wc;
  const bool fast = gn72_ok(dtype, wc, gc, true, l, out, nullptr);
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("gn9_apply", (double)B * HW * J * 2 * sizeof(T));
      if (fast) return gn72_apply_launch<T>(B, HW, wc, l, lbias, mean, rstd, gamma, beta, out, st);
      const int vec = pick_vec<T>(J, l, out);
      RowsGeo g; size_t smem;
      int rc = make_geo(g, B, HW, J, vec, 1, &smem);
      if (rc) return rc;
      NT_DISPATCH_VEC(vec, { gn_apply_kernel<T, V><<<NT_GRID, NT_THREADS, 0, st>>>((const T*)l, lbias, mean, rstd, gamma, beta, (T*)out, g, wc, gc); });
      return check_launch("gn9_apply");
    }
  });
  return 0;
}

extern "C" int cotb200_gn9_bwd_sums(int dtype, int B, int HW, int wc, int gc, const void* dg, const void* l, const float* lbias,
                                    const float* mean, const float* rstd, const float* gamma, float* work, float* s1,
                                    float* s2, float* dgamma, float* dbeta, float* dlbias, void* stream) {
  if (!dg || !l || !mean || !rstd || !gamma || !work || !s1 || !s2 || !dgamma || !dbeta) { set_error("gn9_bwd_sums: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("gn9_bwd_sums: fp64 not supported"); return COTB200_EDTYPE; }
  if (gc > 0 && wc % gc) { set_error("gn9: gc %d does not divide wc %d", gc, wc); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const int J = 9 * wc;
  const bool fast = gn72_ok(dtype, wc, gc, true, dg, l, nullptr);
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      int rc;
      {
        COTB200_PROF_B("gn9_bwd_sums", (double)B * HW * J * 2 * sizeof(T));
        if (fast) {
          if ((rc = gn72_bwd_sums_launch<T>(B, HW, wc, dg, l, work, st))) return rc;
        } else {
          const int vec = pick_vec<T>(J, dg, l);
          RowsGeo g; size_t smem;
          if ((rc = make_geo(g, B, HW, J, vec, 3, &smem))) return rc;
          DetScratch ds;                                   // stream-ordered scratch of the closing reduction
          if ((rc = det_geo(ds, g, 3, st))) return rc;
          NT_DISPATCH_VEC(vec, { if ((rc = ensure_smem(gn_bwd_sums_kernel<T, V>, smem))) return rc;
                                 gn_bwd_sums_kernel<T, V><<<NT_GRID, NT_THREADS, smem, st>>>((const T*)dg, (const T*)l, lbias, mean, rstd, work, g, wc, gc); });
          if ((rc = check_launch("gn9_bwd_sums"))) return rc;
        }
      }
      COTB200_PROF_B("gn9_bwd_finish", 0.0);
      return gn_bwd_finish_launch(B, HW, wc, work, fast ? 1 : 0, lbias, mean, rstd, gamma, s1, s2, dgamma, dbeta, dlbias, st);
    }
  });
  return 0;
}

extern "C" int cotb200_gn9_bwd_apply(int dtype, int B, int HW, int wc, int gc, const void* dg, const void* l, const float* lbias,
                                     const float* mean, const float* rstd, const float* gamma, const float* s1,
                                     const float* s2, void* dl, void* stream) {
  if (!dg || !l || !mean || !rstd || !gamma || !s1 || !s2 || !dl) { set_error("gn9_bwd_apply: NULL pointer"); return COTB200_ENULL; }
  if (dtype == COTB200_F64) { set_error("gn9_bwd_apply: fp64 not supported"); return COTB200_EDTYPE; }
  if (gc > 0 && wc % gc) { set_error("gn9: gc %d does not divide wc %d", gc, wc); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const int J = 9 * wc;
  const bool fast = gn72_ok(dtype, wc, gc, true, dg, l, dl);
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("gn9_bwd_apply", (double)B * HW * J * 3 * sizeof(T));
      if (fast) return gn72_bwd_apply_launch<T>(B, HW, wc, dg, l, lbias, mean, rstd, gamma, s1, s2, dl, st);
      const int vec = pick_vec<T>(J, dg, l, dl);
      RowsGeo g; size_t smem;
      int rc = make_geo(g, B, HW, J, vec, 1, &smem);
      if (rc) return rc;
      NT_DISPATCH_VEC(vec, { gn_bwd_apply_kernel<T, V><<<NT_GRID, NT_THREADS, 0, st>>>((const T*)dg, (const T*)l, lbias, mean, rstd, gamma, s1, s2, (T*)dl, g, wc, gc); });
      return check_launch("gn9_bwd_apply");
    }
  });
  return 0;
}

#define BN_APPLY_LAUNCH(ACT, RES, FIN)                                                                                   \
  do { if (sscale) bn_apply_kernel<T, V, ACT, RES, FIN, true><<<NT_GRID, NT_THREADS, 0, st>>>(xp, rp, scp, shp, yp, g, f, sscale, ds_hw); \
       else bn_apply_kernel<T, V, ACT, RES, FIN><<<NT_GRID, NT_THREADS, 0, st>>>(xp, rp, scp, shp, yp, g, f, nullptr, 1); } while (0)
static int bn_apply_impl(const char* what, int dtype, int B, int HW, int C, const void* x, const void* res, const float* scale,
                         const float* shift, int relu, void* y, const BnFin* fin, const float* sscale, void* stream) {
  if (dtype == COTB200_F64) { set_error("%s: fp64 not supported", what); return COTB200_EDTYPE; }
  const int ds_hw = HW;           // rows per sample: the sample of flattened row r is r / ds_hw
  { const long long rows = (long long)B * HW; if (rows > 2147483647LL) { set_error("%s: too many rows", what); return COTB200_ETOOBIG; }
    HW = (int)rows; B = 1; }      // per-channel affine: flatten [B, HW] -> rows
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pick_vec<T>(C, x, res, y);
      const int cw = col_chunk(C, vec);
      if (!cw) { set_error("%s: cannot tile %d channels", what, C); return COTB200_EINVAL; }
      for (int c0 = 0; c0 < C; c0 += cw) {
        RowsGeo g; size_t smem;
        int rc = make_geo(g, B, HW, cw, vec, 1, &smem);
        if (rc) return rc;
        g.ld = C;
        const T* xp = (const T*)x + c0; const T* rp = res ? (const T*)res + c0 : nullptr; T* yp = (T*)y + c0;
        BnFin f{};
        if (fin) {
          f = *fin;
          f.sum += c0; f.sq += c0; if (f.weight) f.weight += c0; if (f.bias) f.bias += c0;
          if (f.running_mean) f.running_mean += c0; if (f.running_var) f.running_var += c0;
          f.scale += c0; f.shift += c0; f.mean += c0; f.rstd += c0;
        }
        const float* scp = scale ? scale + c0 : nullptr; const float* shp = shift ? shift + c0 : nullptr;
        COTB200_PROF_B(fin ? "bn_apply_batch" : "bn_apply", (double)B * HW * cw * (2 + (res ? 1 : 0)) * sizeof(T));
        NT_DISPATCH_VEC(vec, {
          if (fin) {
            if (relu) { if (res) BN_APPLY_LAUNCH(1, true, true); else BN_APPLY_LAUNCH(1, false, true); }
            else { if (res) BN_APPLY_LAUNCH(0, true, true); else BN_APPLY_LAUNCH(0, false, true); }
          } else {
            if (relu) { if (res) BN_APPLY_LAUNCH(1, true, false); else BN_APPLY_LAUNCH(1, false, false); }
            else { if (res) BN_APPLY_LAUNCH(0, true, false); else BN_APPLY_LAUNCH(0, false, false); }
          }
        });
        if ((rc = check_launch(what))) return rc;
      }
      return 0;
    }
  });
  return 0;
}

extern "C" int cotb200_bn_apply(int dtype, int B, int HW, int C, const void* x, const void* res, const float* scale,
                                const float* shift, int relu, void* y, void* stream) {
  if (!x || !scale || !shift || !y) { set_error("bn_apply: NULL pointer"); return COTB200_ENULL; }
  return bn_apply_impl("bn_apply", dtype, B, HW, C, x, res, scale, shift, relu, y, nullptr, nullptr, stream);
}

extern "C" int cotb200_bn_apply_ds(int dtype, int B, int HW, int C, const void* x, const void* res, const float* scale,
                                   const float* shift, int relu, void* y, const float* sample_scale, void* stream) {
  if (!x || !scale || !shift || !y) { set_error("bn_apply_ds: NULL pointer"); return COTB200_ENULL; }
  return bn_apply_impl("bn_apply_ds", dtype, B, HW, C, x, res, scale, shift, relu, y, nullptr, sample_scale, stream);
}

extern "C" int cotb200_bn_apply_batch(int dtype, int B, int HW, int C, const void* x, const void* res, const float* sum,
                                      const float* sq, const float* weight, const float* bias, float* running_mean,
                                      float* running_var, float n, float eps, float momentum, int update_running, int relu,
                                      void* y, float* scale, float* shift, float* mean, float* rstd, void* stream) {
  if (!x || !y || !sum || !sq || !scale || !shift || !mean || !rstd) { set_error("bn_apply_batch: NULL pointer"); return COTB200_ENULL; }
  if (update_running && (!running_mean || !running_var)) { set_error("bn_apply_batch: running buffers missing"); return COTB200_ENULL; }
  BnFin f{sum, sq, weight, bias, running_mean, running_var, n, eps, momentum, update_running, scale, shift, mean, rstd};
  return bn_apply_impl("bn_apply_batch", dtype, B, HW, C, x, res, nullptr, nullptr, relu, y, &f, nullptr, stream);
}

extern "C" int cotb200_bn_apply_batch_ds(int dtype, int B, int HW, int C, const void* x, const void* res, const float* sum,
                                         const float* sq, const float* weight, const float* bias, float* running_mean,
                                         float* running_var, float n, float eps, float momentum, int update_running, int relu,
                                         void* y, float* scale, float* shift, float* mean, float* rstd, const float* sample_scale,
                                         void* stream) {
  if (!x || !y || !sum || !sq || !scale || !shift || !mean || !rstd) { set_error("bn_apply_batch_ds: NULL pointer"); return COTB200_ENULL; }
  if (update_running && (!running_mean || !running_var)) { set_error("bn_apply_batch_ds: running buffers missing"); return COTB200_ENULL; }
  BnFin f{sum, sq, weight, bias, running_mean, running_var, n, eps, momentum, update_running, scale, shift, mean, rstd};
  return bn_apply_impl("bn_apply_batch_ds", dtype, B, HW, C, x, res, nullptr, nullptr, relu, y, &f, sample_scale, stream);
}

#define BN_BWD_SUMS_LAUNCH(ACT, DS, YP)                                                                               \
  do { if ((rc = ensure_smem(bn_bwd_sums_kernel<T, V, ACT, DS>, smem))) return rc;                                    \
       bn_bwd_sums_kernel<T, V, ACT, DS><<<NT_GRID, NT_THREADS, smem, st>>>(dp, d2p, xp, YP, scp, shp, mu + c0, rstd + c0,  \
                                                                             sum_dz + c0, sum_dzx + c0, g, sscale, ds_hw); } while (0)
static int bn_bwd_sums_impl(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                            const float* scale, const float* shift, const float* mu, const float* rstd, int relu,
                            float* sum_dz, float* sum_dzx, const float* sscale, void* stream) {
  if (!dy || !x || !mu || !rstd || !sum_dz || !sum_dzx || (relu == 1 && !y) || (relu == 2 && (!scale || !shift))) {
    set_error("bn_bwd_sums: NULL pointer"); return COTB200_ENULL; }
  if (relu < 0 || relu > 2) { set_error("bn_bwd_sums: relu must be 0, 1 or 2"); return COTB200_EINVAL; }
  if (dtype == COTB200_F64) { set_error("bn_bwd_sums: fp64 not supported"); return COTB200_EDTYPE; }
  const int ds_hw = HW;           // rows per sample (drop-path scales)
  { const long long rows = (long long)B * HW; if (rows > 2147483647LL) { set_error("cotb200_bn_bwd_sums: too many rows"); return COTB200_ETOOBIG; }
    HW = (int)rows; B = 1; }      // per-channel statistics: flatten [B, HW] -> rows
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = pick_vec<T>(C, dy, x, relu == 1 ? y : nullptr, dy2);
      const int cw = col_chunk(C, vec);
      if (!cw) { set_error("bn_bwd_sums: cannot tile %d channels", C); return COTB200_EINVAL; }
      for (int c0 = 0; c0 < C; c0 += cw) {
        RowsGeo g; size_t smem;
        int rc = make_geo(g, B, HW, cw, vec, 2, &smem);
        if (rc) return rc;
        DetScratch ds;                                   // stream-ordered scratch of the closing reduction
        if ((rc = det_geo(ds, g, 2, st))) return rc;
        g.ld = C;
        const T* dp = (const T*)dy + c0; const T* xp = (const T*)x + c0; const T* yp = y ? (const T*)y + c0 : nullptr;
        const T* d2p = dy2 ? (const T*)dy2 + c0 : nullptr;
        COTB200_PROF_B("bn_bwd_sums", (double)B * HW * cw * (2 + (relu == 1 ? 1 : 0) + (dy2 ? 1 : 0)) * sizeof(T));
        const float* scp = scale ? scale + c0 : nullptr; const float* shp = shift ? shift + c0 : nullptr;
        NT_DISPATCH_VEC(vec, {
          if (sscale) {
            if (relu == 1) BN_BWD_SUMS_LAUNCH(1, true, yp); else if (relu == 2) BN_BWD_SUMS_LAUNCH(2, true, nullptr); else BN_BWD_SUMS_LAUNCH(0, true, nullptr);
          } else {
            if (relu == 1) BN_BWD_SUMS_LAUNCH(1, false, yp); else if (relu == 2) BN_BWD_SUMS_LAUNCH(2, false, nullptr); else BN_BWD_SUMS_LAUNCH(0, false, nullptr);
          }
        });
        if ((rc = check_launch("bn_bwd_sums"))) return rc;
      }
      return 0;
    }
  });
  return 0;
}

#define BN_BWD_APPLY_LAUNCH(ACT, RES, YP, DRP)                                                                         \
  do { if (sscale) bn_bwd_apply_kernel<T, V, ACT, RES, true><<<NT_GRID, NT_THREADS, 0, st>>>(dp, d2p, xp, YP, scale + c0, shp, mu + c0, \
                                                               rstd + c0, k1, k2, inv_n, dxp, DRP, g, sscale, ds_hw);      \
       else bn_bwd_apply_kernel<T, V, ACT, RES><<<NT_GRID, NT_THREADS, 0, st>>>(dp, d2p, xp, YP, scale + c0, shp, mu + c0,  \
                                                               rstd + c0, k1, k2, inv_n, dxp, DRP, g, nullptr, 1); } while (0)
static int bn_bwd_apply_impl(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                             const float* scale, const float* shift, const float* mu, const float* rstd,
                             const float* c1, const float* c2, float inv_n, int relu, void* dx, void* dres, const float* sscale,
                             void* stream) {
  if (!dy || !x || !scale || !mu || !rstd || !dx || (relu == 1 && !y) || (relu == 2 && !shift)) {
    set_error("bn_bwd_apply: NULL pointer"); return COTB200_ENULL; }
  if (relu < 0 || relu > 2) { set_error("bn_bwd_apply: relu must be 0, 1 or 2"); return COTB200_EINVAL; }
  if (dtype == COTB200_F64) { set_error("bn_bwd_apply: fp64 not supported"); return COTB200_EDTYPE; }
  const int ds_hw = HW;           // rows per sample (drop-path scales)
  { const long long rows = (long long)B * HW; if (rows > 2147483647LL) { set_error("cotb200_bn_bwd_apply: too many rows"); return COTB200_ETOOBIG; }
    HW = (int)rows; B = 1; }      // per-channel statistics: flatten [B, HW] -> rows
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      int vec = pick_vec<T>(C, dy, x, relu == 1 ? y : nullptr, dx);
      if (dres && ((uintptr_t)dres & (vec * sizeof(T) - 1))) vec = 1;
      if (dy2 && ((uintptr_t)dy2 & (vec * sizeof(T) - 1))) vec = 1;
      const int cw = col_chunk(C, vec);
      if (!cw) { set_error("bn_bwd_apply: cannot tile %d channels", C); return COTB200_EINVAL; }
      for (int c0 = 0; c0 < C; c0 += cw) {
        RowsGeo g; size_t smem;
        int rc = make_geo(g, B, HW, cw, vec, 1, &smem);
        if (rc) return rc;
        g.ld = C;
        const T* dp = (const T*)dy + c0; const T* xp = (const T*)x + c0; const T* yp = y ? (const T*)y + c0 : nullptr;
        T* dxp = (T*)dx + c0; T* drp = dres ? (T*)dres + c0 : nullptr;
        const T* d2p = dy2 ? (const T*)dy2 + c0 : nullptr;
        const float* k1 = c1 ? c1 + c0 : nullptr; const float* k2 = c2 ? c2 + c0 : nullptr;
        COTB200_PROF_B("bn_bwd_apply", (double)B * HW * cw * (3 + (relu == 1 ? 1 : 0) + (dres ? 1 : 0) + (dy2 ? 1 : 0)) * sizeof(T));
        const float* shp = shift ? shift + c0 : nullptr;
        NT_DISPATCH_VEC(vec, {
          if (relu == 1) { if (dres) BN_BWD_APPLY_LAUNCH(1, true, yp, drp); else BN_BWD_APPLY_LAUNCH(1, false, yp, nullptr); }
          else if (relu == 2) { if (dres) BN_BWD_APPLY_LAUNCH(2, true, nullptr, drp); else BN_BWD_APPLY_LAUNCH(2, false, nullptr, nullptr); }
          else { if (dres) BN_BWD_APPLY_LAUNCH(0, true, nullptr, drp); else BN_BWD_APPLY_LAUNCH(0, false, nullptr, nullptr); }
        });
        if ((rc = check_launch("bn_bwd_apply"))) return rc;
      }
      return 0;
    }
  });
  return 0;
}

extern "C" int cotb200_bn_finalize(int C, const float* sum, const float* sq, const float* weight, const float* bias,
                                   float* running_mean, float* running_var, float n, float eps, float momentum, int use_batch,
                                   int update_running, float* scale, float* shift, float* mean, float* rstd, void* stream) {
  if (!scale || !shift || !mean || !rstd || (use_batch && (!sum || !sq)) || ((!use_batch || update_running) && (!running_mean || !running_var))) {
    set_error("bn_finalize: NULL pointer"); return COTB200_ENULL;
  }
  if (C <= 0) { set_error("bn_finalize: C <= 0"); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_PROF("bn_finalize");
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(sum, sq, weight, bias, running_mean, running_var, n, eps, momentum, use_batch,
                                                     update_running, scale, shift, mean, rstd, C);
  return check_launch("bn_finalize");
}


// ---- public entry points of the BatchNorm backward: one incoming gradient, or two that are summed on the fly (fp32)
extern "C" int cotb200_bn_bwd_sums(int dtype, int B, int HW, int C, const void* dy, const void* x, const void* y,
                                   const float* scale, const float* shift, const float* mu, const float* rstd, int relu,
                                   float* sum_dz, float* sum_dzx, void* stream) {
  return bn_bwd_sums_impl(dtype, B, HW, C, dy, nullptr, x, y, scale, shift, mu, rstd, relu, sum_dz, sum_dzx, nullptr, stream);
}
extern "C" int cotb200_bn_bwd_sums2(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                                    const float* scale, const float* shift, const float* mu, const float* rstd, int relu,
                                    float* sum_dz, float* sum_dzx, void* stream) {
  return bn_bwd_sums_impl(dtype, B, HW, C, dy, dy2, x, y, scale, shift, mu, rstd, relu, sum_dz, sum_dzx, nullptr, stream);
}
extern "C" int cotb200_bn_bwd_sums_ds(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                                      const float* scale, const float* shift, const float* mu, const float* rstd, int relu,
                                      float* sum_dz, float* sum_dzx, const float* sample_scale, void* stream) {
  return bn_bwd_sums_impl(dtype, B, HW, C, dy, dy2, x, y, scale, shift, mu, rstd, relu, sum_dz, sum_dzx, sample_scale, stream);
}
extern "C" int cotb200_bn_bwd_apply(int dtype, int B, int HW, int C, const void* dy, const void* x, const void* y,
                                    const float* scale, const float* shift, const float* mu, const float* rstd,
                                    const float* c1, const float* c2, float inv_n, int relu, void* dx, void* dres, void* stream) {
  return bn_bwd_apply_impl(dtype, B, HW, C, dy, nullptr, x, y, scale, shift, mu, rstd, c1, c2, inv_n, relu, dx, dres, nullptr, stream);
}
extern "C" int cotb200_bn_bwd_apply2(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                                     const float* scale, const float* shift, const float* mu, const float* rstd,
                                     const float* c1, const float* c2, float inv_n, int relu, void* dx, void* dres, void* stream) {
  return bn_bwd_apply_impl(dtype, B, HW, C, dy, dy2, x, y, scale, shift, mu, rstd, c1, c2, inv_n, relu, dx, dres, nullptr, stream);
}
extern "C" int cotb200_bn_bwd_apply_ds(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                                       const float* scale, const float* shift, const float* mu, const float* rstd,
                                       const float* c1, const float* c2, float inv_n, int relu, void* dx, void* dres,
                                       const float* sample_scale, void* stream) {
  return bn_bwd_apply_impl(dtype, B, HW, C, dy, dy2, x, y, scale, shift, mu, rstd, c1, c2, inv_n, relu, dx, dres, sample_scale, stream);
}
