// The optimizer pass of the training step (train.py:274 -> optim/optim_factory.py:create_optimizer), sm_90a.
//
// One streaming pass per flat range for every update rule the library runs: read G*grad_scale, clip it (clip.cu makes the
// factors), apply the rule, the Lookahead synchronisation when this step has one, the EMA of the final weights
// (train.py:276-277) and the bf16 shadow.  The walkers -- a grid-stride float4 loop for no clip / norm / value, one warp per
// segment for AGC -- are templated on the rule.
//
//   cotb200_opt_prepare        one thread: advance the step counter t and compute what depends only on t and lr (fp64); plain
//                              SGD / momentum without Lookahead needs none of it and runs on the state as initialised
//   cotb200_opt_step           the pass, any rule, any clip mode (cotb200_clip, nullable)
//   cotb200_lookahead_sync     Lookahead.sync_lookahead (train.py:295-296): S += alpha (P - S); P = S; the bf16 shadow
//
// Everything depending on the step lives in device memory (hyper, cotb200_opt_state): a captured CUDA graph follows the LR
// schedule and the bias corrections, and a replay computes exactly what an eager step computes.
#include <cmath>

#include "common.cuh"

namespace cotb200 {

// The factory's defaults (create_optimizer passes only lr, momentum, weight_decay and eps)
static constexpr double OPT_B1 = 0.9, OPT_B2 = 0.999;        // Adam / AdamW / Nadam / RAdam betas
static constexpr double OPT_RHO = 0.9;                       // Adadelta rho
static constexpr double OPT_ALPHA = 0.9;                     // RMSprop / RMSpropTF alpha (optim_factory.py)
static constexpr double OPT_SCHEDULE_DECAY = 4e-3;           // Nadam

__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

template <bool NESTEROV>
__device__ __forceinline__ void sgd_elem(float& p, float& m, float gc, float lr, float mu, float wd) {
  const float g = fmaf(wd, p, gc);                // gc: the clipped grad*gscale
  m = fmaf(mu, m, g);
  const float st = NESTEROV ? fmaf(mu, m, g) : m;
  p = fmaf(-lr, st, p);
}

template <int MODE>
__device__ __forceinline__ float clip_uniform(float g, float f, float c) {
  if constexpr (MODE == COTB200_CLIP_NORM) return g * f;
  else if constexpr (MODE == COTB200_CLIP_VALUE) return clamp_nan(g, -c, c);
  else return g;
}

__host__ __device__ constexpr bool rule_has_v(int r) { return r != COTB200_OPT_SGD && r != COTB200_OPT_MOMENTUM; }
__host__ __device__ constexpr bool rule_m_optional(int r) { return r == COTB200_OPT_RMSPROP || r == COTB200_OPT_RMSPROPTF; }

template <typename TG>
struct OptArgs {
  float* P; float* M; float* V; float* S; float* E;        // M: NULL for RMSprop(TF) without momentum; V, S: NULL when unused
  const TG* G;
  __nv_bfloat16* Pb;
  const float* hyper;                                      // {lr, momentum, weight_decay, ema_decay, grad_scale}
  const cotb200_opt_state* state;
  float eps, la;
};

// Per-thread constants of one pass.
struct Coef {
  float lr, mu, wd, dec, gs, eps, la;
  float c0, c1, c2;                                        // cotb200_opt_state.c of this step
  float wdf;                                               // AdamW: 1 - lr*wd (a factor); RAdam: -wd*lr (an addend's factor)
  int sync;
  bool mom;
};

template <int RULE, typename TG>
__device__ __forceinline__ Coef load_coef(const OptArgs<TG>& a) {
  Coef k;
  k.lr = __ldg(a.hyper); k.mu = __ldg(a.hyper + 1); k.wd = __ldg(a.hyper + 2); k.dec = __ldg(a.hyper + 3); k.gs = __ldg(a.hyper + 4);
  k.eps = a.eps; k.la = a.la;
  k.c0 = k.c1 = k.c2 = 0.f; k.sync = 0;
  if (a.state) {
    k.c0 = __ldg(&a.state->c[0]); k.c1 = __ldg(&a.state->c[1]); k.c2 = __ldg(&a.state->c[2]);
    k.sync = __ldg(&a.state->sync);
  }
  // The reference forms these in Python floats from its (double) lr and weight_decay and hands them to a float tensor op
  if (RULE == COTB200_OPT_ADAMW) k.wdf = (float)(1.0 - (double)k.lr * (double)k.wd);          // p.mul_(1 - lr*wd)   (adamw.py:72)
  else if (RULE == COTB200_OPT_RADAM) k.wdf = (float)(-(double)k.wd * (double)k.lr);          // p.add_(-wd*lr, p)  (radam.py:71)
  else k.wdf = 0.f;
  k.mom = a.M != nullptr;
  return k;
}

// One element: p, m (first moment / momentum / acc_delta), v (second moment / square_avg) and the clipped averaged gradient g.
template <int RULE>
__device__ __forceinline__ void rule_elem(float& p, float& m, float& v, float g, const Coef& k) {
  constexpr float B1 = (float)OPT_B1, OB1 = (float)(1.0 - OPT_B1), B2 = (float)OPT_B2, OB2 = (float)(1.0 - OPT_B2);
  if constexpr (RULE == COTB200_OPT_SGD || RULE == COTB200_OPT_MOMENTUM) {
    sgd_elem<RULE == COTB200_OPT_SGD>(p, m, g, k.lr, k.mu, k.wd);
  } else if constexpr (RULE == COTB200_OPT_ADAM || RULE == COTB200_OPT_ADAMW) {
    // torch.optim.Adam: L2 decay in the gradient.  AdamW (adamw.py:72-117): decoupled p *= 1 - lr*wd first.
    if (RULE == COTB200_OPT_ADAM) g = fmaf(k.wd, p, g);
    else p = p * k.wdf;
    m = fmaf(B1, m, OB1 * g);
    v = fmaf(B2, v, OB2 * (g * g));
    const float denom = sqrtf(v) / k.c0 + k.eps;              // c0 = sqrt(1 - b2^t)
    p = fmaf(k.c1, m / denom, p);                             // c1 = -lr / (1 - b1^t)
  } else if constexpr (RULE == COTB200_OPT_NADAM) {
    g = fmaf(k.wd, p, g);                                     // nadam.py:61-88
    m = fmaf(B1, m, OB1 * g);
    v = fmaf(B2, v, OB2 * (g * g));
    const float denom = sqrtf(v / k.c0) + k.eps;              // c0 = 1 - b2^t
    p = fmaf(k.c1, g / denom, p);                             // c1 = -lr (1 - mc_t) / (1 - m_schedule_new)
    p = fmaf(k.c2, m / denom, p);                             // c2 = -lr mc_t+1 / (1 - m_schedule_next)
  } else if constexpr (RULE == COTB200_OPT_RADAM) {
    v = fmaf(B2, v, OB2 * (g * g));                           // radam.py:40-84: the moments see the raw gradient
    m = fmaf(B1, m, OB1 * g);
    p = fmaf(k.wdf, p, p);
    if (k.c1 != 0.f) p = fmaf(k.c0, m / (sqrtf(v) + k.eps), p);   // N_sma >= 5 (c1 = 1); c0 = -step_size
    else p = fmaf(k.c0, m, p);
  } else if constexpr (RULE == COTB200_OPT_ADADELTA) {
    constexpr float R = (float)OPT_RHO, OR = (float)(1.0 - OPT_RHO);
    g = fmaf(k.wd, p, g);                                     // torch.optim.Adadelta; m = acc_delta, v = square_avg
    v = fmaf(R, v, OR * (g * g));
    const float delta = sqrtf(m + k.eps) / sqrtf(v + k.eps) * g;
    m = fmaf(R, m, OR * (delta * delta));
    p = fmaf(-k.lr, delta, p);
  } else if constexpr (RULE == COTB200_OPT_RMSPROP) {
    constexpr float A = (float)OPT_ALPHA, OA = (float)(1.0 - OPT_ALPHA);
    g = fmaf(k.wd, p, g);                                     // torch.optim.RMSprop: square_avg from 0, eps outside the sqrt
    v = fmaf(A, v, OA * (g * g));
    const float q = g / (sqrtf(v) + k.eps);
    if (k.mom) { m = fmaf(k.mu, m, q); p = fmaf(-k.lr, m, p); }
    else p = fmaf(-k.lr, q, p);
  } else if constexpr (RULE == COTB200_OPT_RMSPROPTF) {
    constexpr float OA = (float)(1.0 - OPT_ALPHA);
    g = fmaf(k.wd, p, g);                                     // rmsprop_tf.py:97-136: square_avg from 1, eps inside the sqrt
    v = fmaf(OA, g * g - v, v);
    const float q = g / sqrtf(v + k.eps);
    if (k.mom) { m = fmaf(k.mu, m, k.lr * q); p = p - m; }   // lr_in_momentum: the buffer holds lr*g/avg
    else p = fmaf(-k.lr, q, p);
  }
}

// Lookahead.update_slow (lookahead.py:31-38) when this step syncs: sync 1 creates the slow weights from the fast ones (the
// reference's first sync, which leaves P as it is), sync 2 is S += alpha (P - S); P = S.
__device__ __forceinline__ void sync_elem(float& p, float& s, const Coef& k) {
  if (k.sync == 1) s = p;
  else { s = fmaf(k.la, p - s, s); p = s; }
}

// The whole element pipeline on one float4 (vec) or one element (one); `clip` maps G*grad_scale to the clipped g'.
template <typename TG, int RULE>
struct Pass {
  OptArgs<TG> a;
  Coef k;

  template <typename Clip>
  __device__ __forceinline__ void vec(long long i, Clip clip) const {
    constexpr bool HV = rule_has_v(RULE);
    const float4 p = reinterpret_cast<const float4*>(a.P)[i];
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f), v = m, s = m;
    if (k.mom) m = reinterpret_cast<const float4*>(a.M)[i];
    if (HV) v = reinterpret_cast<const float4*>(a.V)[i];
    if (k.sync == 2) s = reinterpret_cast<const float4*>(a.S)[i];
    const Pack<TG, 4> gp = ld_pack<TG, 4>(a.G + i * 4);
    float pv[4] = {p.x, p.y, p.z, p.w}, mv[4] = {m.x, m.y, m.z, m.w}, vv[4] = {v.x, v.y, v.z, v.w}, sv[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      rule_elem<RULE>(pv[e], mv[e], vv[e], clip((float)to_acc(gp.v[e]) * k.gs), k);
      if (k.sync) sync_elem(pv[e], sv[e], k);
    }
    reinterpret_cast<float4*>(a.P)[i] = make_float4(pv[0], pv[1], pv[2], pv[3]);
    if (k.mom) reinterpret_cast<float4*>(a.M)[i] = make_float4(mv[0], mv[1], mv[2], mv[3]);
    if (HV) reinterpret_cast<float4*>(a.V)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    if (k.sync) reinterpret_cast<float4*>(a.S)[i] = make_float4(sv[0], sv[1], sv[2], sv[3]);
    if (a.E) {
      float4 e = reinterpret_cast<float4*>(a.E)[i];
      e.x = fmaf(k.dec, e.x, (1.f - k.dec) * pv[0]); e.y = fmaf(k.dec, e.y, (1.f - k.dec) * pv[1]);
      e.z = fmaf(k.dec, e.z, (1.f - k.dec) * pv[2]); e.w = fmaf(k.dec, e.w, (1.f - k.dec) * pv[3]);
      reinterpret_cast<float4*>(a.E)[i] = e;
    }
    if (a.Pb) {
      Pack<__nv_bfloat16, 4> o;
#pragma unroll
      for (int e = 0; e < 4; ++e) o.v[e] = __float2bfloat16_rn(pv[e]);
      st_pack<__nv_bfloat16, 4>(a.Pb + i * 4, o);
    }
  }

  template <typename Clip>
  __device__ __forceinline__ void one(long long j, Clip clip) const {
    constexpr bool HV = rule_has_v(RULE);
    float p = a.P[j], m = k.mom ? a.M[j] : 0.f, v = HV ? a.V[j] : 0.f, s = k.sync == 2 ? a.S[j] : 0.f;
    rule_elem<RULE>(p, m, v, clip((float)to_acc(a.G[j]) * k.gs), k);
    if (k.sync) { sync_elem(p, s, k); a.S[j] = s; }
    a.P[j] = p;
    if (k.mom) a.M[j] = m;
    if (HV) a.V[j] = v;
    if (a.E) a.E[j] = fmaf(k.dec, a.E[j], (1.f - k.dec) * p);
    if (a.Pb) a.Pb[j] = __float2bfloat16_rn(p);
  }
};

// No clip / NORM / VALUE: one factor or bound for the whole range -- the grid-stride float4 loop.
template <typename TG, int RULE, int MODE>
__global__ void __launch_bounds__(256)
opt_uniform_kernel(OptArgs<TG> a, long long n4, const float* __restrict__ fdev, float c) {
  const Pass<TG, RULE> ps{a, load_coef<RULE>(a)};
  const float f = MODE == COTB200_CLIP_NORM ? __ldg(fdev) : 1.f;
  const auto clip = [f, c](float g) { return clip_uniform<MODE>(g, f, c); };
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) ps.vec(i, clip);
}

// AGC: one warp per segment of the host's table, so the factor is uniform inside a warp.  Segments start and end anywhere (the
// stem's 147-element rows put unit boundaries inside a float4): the elements before the first and after the last 16-byte
// boundary of the segment are updated one by one, the rest as float4.  Two warps may write different elements of one float4;
// no byte is written twice.
template <typename TG, int RULE>
__global__ void __launch_bounds__(256)
opt_agc_kernel(OptArgs<TG> a, const cotb200_clip_seg* __restrict__ segs, int n_segs, const float* __restrict__ factor) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= n_segs) return;
  const Pass<TG, RULE> ps{a, load_coef<RULE>(a)};
  const cotb200_clip_seg s = segs[w];
  const float f = s.unit >= 0 ? __ldg(factor + s.unit) : 1.f;
  const auto clip = [f](float g) { return g * f; };
  const long long lo = s.offset, hi = s.offset + s.numel;
  const long long a4 = (lo + 3) >> 2, b4 = hi >> 2;                   // float4 indices [a4, b4) lie inside [lo, hi)
  if (a4 >= b4) {                                                      // no whole float4 inside
    for (long long j = lo + lane; j < hi; j += 32) ps.one(j, clip);
    return;
  }
  if (lo + lane < a4 * 4) ps.one(lo + lane, clip);
  if (b4 * 4 + lane < hi) ps.one(b4 * 4 + lane, clip);
  for (long long i = a4 + lane; i < b4; i += 32) ps.vec(i, clip);
}

// ------------------------------------------------------------------------------------------------ per-step scalars
// The reference computes these per parameter in Python floats (double) from its int step and its lr; here once per step, in
// fp64, rounded to fp32 where the reference hands the value to a float tensor op.  Explicit _rn products: no FMA contraction.
__global__ void opt_prepare_kernel(int rule, int la_k, int advance, cotb200_opt_state* __restrict__ s, const float* __restrict__ hyper) {
  bool sync;
  if (advance) {
    const double t = s->t + 1.0, lr = (double)hyper[0];
    s->t = t;
    s->c[0] = s->c[1] = s->c[2] = s->c[3] = 0.f;
    if (rule == COTB200_OPT_ADAM || rule == COTB200_OPT_ADAMW) {
      const double bc1 = 1.0 - pow(OPT_B1, t), bc2 = 1.0 - pow(OPT_B2, t);
      s->c[0] = (float)sqrt(bc2);
      s->c[1] = (float)(-(lr / bc1));
    } else if (rule == COTB200_OPT_NADAM) {
      const double mc = __dmul_rn(OPT_B1, 1.0 - __dmul_rn(0.5, pow(0.96, __dmul_rn(t, OPT_SCHEDULE_DECAY))));
      const double mc1 = __dmul_rn(OPT_B1, 1.0 - __dmul_rn(0.5, pow(0.96, __dmul_rn(t + 1.0, OPT_SCHEDULE_DECAY))));
      const double ms_new = __dmul_rn(s->m_schedule, mc), ms_next = __dmul_rn(ms_new, mc1);
      s->m_schedule = ms_new;
      s->c[0] = (float)(1.0 - pow(OPT_B2, t));
      s->c[1] = (float)(__dmul_rn(-lr, 1.0 - mc) / (1.0 - ms_new));
      s->c[2] = (float)(__dmul_rn(-lr, mc1) / (1.0 - ms_next));
    } else if (rule == COTB200_OPT_RADAM) {
      const double b2t = pow(OPT_B2, t);
      const double n_max = 2.0 / (1.0 - OPT_B2) - 1.0;
      const double n_sma = n_max - __dmul_rn(__dmul_rn(2.0, t), b2t) / (1.0 - b2t);
      double step;
      if (n_sma >= 5.0) {
        double r = __dmul_rn(1.0 - b2t, n_sma - 4.0) / (n_max - 4.0);
        r = __dmul_rn(r, n_sma - 2.0) / n_sma;
        r = __dmul_rn(r, n_max) / (n_max - 2.0);
        step = __dmul_rn(lr, sqrt(r)) / (1.0 - pow(OPT_B1, t));
      } else {
        step = lr / (1.0 - pow(OPT_B1, t));
      }
      s->c[0] = (float)(-step);
      s->c[1] = n_sma >= 5.0 ? 1.f : 0.f;
    }
    sync = la_k > 0 && ((long long)t) % la_k == 0;
  } else {
    sync = la_k > 0;                                                   // sync_lookahead(): now, without a step
  }
  s->sync = sync ? (s->slow_init ? 2 : 1) : 0;
  if (sync) s->slow_init = 1;
}

__global__ void __launch_bounds__(256)
lookahead_sync_kernel(float* __restrict__ P, float* __restrict__ S, __nv_bfloat16* __restrict__ Pb, const cotb200_opt_state* __restrict__ st,
                      float la, long long n4) {
  const int sync = __ldg(&st->sync);
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    float4 p = reinterpret_cast<float4*>(P)[i];
    if (sync == 1) {
      reinterpret_cast<float4*>(S)[i] = p;
    } else {
      float4 s = reinterpret_cast<float4*>(S)[i];
      s.x = fmaf(la, p.x - s.x, s.x); s.y = fmaf(la, p.y - s.y, s.y); s.z = fmaf(la, p.z - s.z, s.z); s.w = fmaf(la, p.w - s.w, s.w);
      reinterpret_cast<float4*>(S)[i] = s;
      reinterpret_cast<float4*>(P)[i] = p = s;
    }
    if (Pb) {
      Pack<__nv_bfloat16, 4> o;
      o.v[0] = __float2bfloat16_rn(p.x); o.v[1] = __float2bfloat16_rn(p.y); o.v[2] = __float2bfloat16_rn(p.z); o.v[3] = __float2bfloat16_rn(p.w);
      st_pack<__nv_bfloat16, 4>(Pb + i * 4, o);
    }
  }
}

static bool rule_known(int r) { return r >= COTB200_OPT_SGD && r <= COTB200_OPT_RMSPROPTF; }

// Validation of a clip descriptor (NULL: no clip); 0 or an error code with the message set.
static int check_clip(const char* who, const cotb200_clip* clip) {
  if (!clip) return 0;
  const int mode = clip->mode;
  if (mode != COTB200_CLIP_NORM && mode != COTB200_CLIP_VALUE && mode != COTB200_CLIP_AGC) {
    set_error("%s: unknown clip mode %d", who, mode); return COTB200_EINVAL;
  }
  if (mode != COTB200_CLIP_VALUE && !clip->factor) { set_error("%s: the clip has no factor pointer", who); return COTB200_ENULL; }
  if (mode == COTB200_CLIP_AGC && !clip->segs) { set_error("%s: agc needs the segment table", who); return COTB200_ENULL; }
  if (mode == COTB200_CLIP_AGC && clip->n_segs <= 0) { set_error("%s: agc needs segments", who); return COTB200_EINVAL; }
  if (mode == COTB200_CLIP_VALUE && !(clip->value > 0.f)) { set_error("%s: clip value must be > 0", who); return COTB200_EINVAL; }
  return 0;
}

template <typename TG, int RULE>
static void launch_pass(const OptArgs<TG>& a, long long n4, const cotb200_clip* clip, cudaStream_t st) {
  const int mode = clip ? clip->mode : 0;
  if (mode == COTB200_CLIP_AGC) {
    opt_agc_kernel<TG, RULE><<<(unsigned)((clip->n_segs + 7) / 8), 256, 0, st>>>(a, clip->segs, clip->n_segs, clip->factor);
    return;
  }
  const int grid = grid_stride_blocks(n4, 256, 16);
  if (mode == COTB200_CLIP_NORM) opt_uniform_kernel<TG, RULE, COTB200_CLIP_NORM><<<grid, 256, 0, st>>>(a, n4, clip->factor, 0.f);
  else if (mode == COTB200_CLIP_VALUE) opt_uniform_kernel<TG, RULE, COTB200_CLIP_VALUE><<<grid, 256, 0, st>>>(a, n4, nullptr, clip->value);
  else opt_uniform_kernel<TG, RULE, 0><<<grid, 256, 0, st>>>(a, n4, nullptr, 0.f);
}

template <typename TG>
static void launch_rule(int rule, const OptArgs<TG>& a, long long n4, const cotb200_clip* clip, cudaStream_t st) {
  switch (rule) {
    case COTB200_OPT_SGD: launch_pass<TG, COTB200_OPT_SGD>(a, n4, clip, st); break;
    case COTB200_OPT_MOMENTUM: launch_pass<TG, COTB200_OPT_MOMENTUM>(a, n4, clip, st); break;
    case COTB200_OPT_ADAM: launch_pass<TG, COTB200_OPT_ADAM>(a, n4, clip, st); break;
    case COTB200_OPT_ADAMW: launch_pass<TG, COTB200_OPT_ADAMW>(a, n4, clip, st); break;
    case COTB200_OPT_NADAM: launch_pass<TG, COTB200_OPT_NADAM>(a, n4, clip, st); break;
    case COTB200_OPT_RADAM: launch_pass<TG, COTB200_OPT_RADAM>(a, n4, clip, st); break;
    case COTB200_OPT_ADADELTA: launch_pass<TG, COTB200_OPT_ADADELTA>(a, n4, clip, st); break;
    case COTB200_OPT_RMSPROP: launch_pass<TG, COTB200_OPT_RMSPROP>(a, n4, clip, st); break;
    default: launch_pass<TG, COTB200_OPT_RMSPROPTF>(a, n4, clip, st); break;
  }
}

template <typename TG>
static OptArgs<TG> make_args(float* P, float* M, float* V, float* S, float* E, const void* G, void* Pb, const float* hyper,
                             const cotb200_opt_state* state, float eps, float la) {
  return OptArgs<TG>{P, M, V, S, E, (const TG*)G, (__nv_bfloat16*)Pb, hyper, state, eps, la};
}

// Argument checks of the pass over a flat range (after those of the descriptor).
static int check_pass(const char* who, long long n, const float* P, const float* M, const float* V, const float* S, int g_dtype,
                      const void* G, const float* E, const void* Pb) {
  if (n <= 0 || (n & 3)) { set_error("%s: n=%lld must be a positive multiple of 4 (pad the flat range)", who, n); return COTB200_EINVAL; }
  if (!aligned16(P) || (M && !aligned16(M)) || (V && !aligned16(V)) || (S && !aligned16(S)) || (E && !aligned16(E)) ||
      (reinterpret_cast<uintptr_t>(G) & (g_dtype == COTB200_F32 ? 15 : 7)) || (Pb && (reinterpret_cast<uintptr_t>(Pb) & 7))) {
    set_error("%s: flat buffers must be 16-byte aligned", who); return COTB200_EALIGN;
  }
  if (g_dtype != COTB200_F32 && g_dtype != COTB200_BF16) { set_error("%s: gradient dtype must be fp32 or bf16", who); return COTB200_EDTYPE; }
  return 0;
}

static double pass_bytes(long long n, bool m, bool v, int sync_bytes, int g_dtype, const float* E, const void* Pb) {
  return (double)n * (8.0 + (m ? 8.0 : 0.0) + (v ? 8.0 : 0.0) + sync_bytes + (g_dtype == COTB200_F32 ? 4.0 : 2.0) + (E ? 8.0 : 0.0) +
                      (Pb ? 2.0 : 0.0));
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_opt_prepare(const cotb200_opt* opt, const float* hyper_dev, int advance, void* stream) {
  if (!opt || !opt->state || !hyper_dev) { set_error("opt_prepare: NULL pointer"); return COTB200_ENULL; }
  if (!rule_known(opt->rule)) { set_error("opt_prepare: unknown rule %d", opt->rule); return COTB200_EINVAL; }
  if (opt->lookahead_k < 0) { set_error("opt_prepare: lookahead_k=%d must be >= 0", opt->lookahead_k); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_PROF("opt_prepare");
  opt_prepare_kernel<<<1, 1, 0, st>>>(opt->rule, opt->lookahead_k, advance ? 1 : 0, opt->state, hyper_dev);
  return check_launch("opt_prepare");
}

extern "C" int cotb200_opt_step(long long n, float* P, int g_dtype, const void* G, float* E, void* Pb, const float* hyper_dev,
                                const cotb200_opt* opt, const cotb200_clip* clip, void* stream) {
  if (!P || !G || !hyper_dev || !opt || !opt->state) { set_error("opt_step: NULL pointer"); return COTB200_ENULL; }
  const int rule = opt->rule;
  if (!rule_known(rule)) { set_error("opt_step: unknown rule %d", rule); return COTB200_EINVAL; }
  if (!opt->M && !rule_m_optional(rule)) { set_error("opt_step: rule %d needs the state buffer M", rule); return COTB200_ENULL; }
  if (!opt->V && rule_has_v(rule)) { set_error("opt_step: rule %d needs the state buffer V", rule); return COTB200_ENULL; }
  if (opt->lookahead_k < 0 || !(opt->lookahead_alpha >= 0.f && opt->lookahead_alpha <= 1.f)) {
    set_error("opt_step: lookahead_k=%d must be >= 0 and lookahead_alpha in [0, 1]", opt->lookahead_k); return COTB200_EINVAL;
  }
  if (opt->lookahead_k > 0 && !opt->S) { set_error("opt_step: Lookahead needs the slow-weight buffer S"); return COTB200_ENULL; }
  if (!(opt->eps >= 0.f)) { set_error("opt_step: eps must be >= 0"); return COTB200_EINVAL; }
  if (int rc = check_clip("opt_step", clip)) return rc;
  float* S = opt->lookahead_k > 0 ? opt->S : nullptr;
  float* V = rule_has_v(rule) ? opt->V : nullptr;
  if (int rc = check_pass("opt_step", n, P, opt->M, V, S, g_dtype, G, E, Pb)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  // algorithmic bytes of a step without a Lookahead sync (a sync adds 8 per element, 4 for the first)
  double bytes = pass_bytes(n, opt->M != nullptr, V != nullptr, 0, g_dtype, E, Pb) + 40.0;
  if (clip) bytes += clip->mode == COTB200_CLIP_AGC ? (double)clip->n_segs * (16.0 + 4.0) : (clip->mode == COTB200_CLIP_NORM ? 4.0 : 0.0);
  COTB200_PROF_B("opt_step", bytes);
  if (g_dtype == COTB200_F32)
    launch_rule<float>(rule, make_args<float>(P, opt->M, V, S, E, G, Pb, hyper_dev, opt->state, opt->eps, opt->lookahead_alpha), n / 4, clip, st);
  else
    launch_rule<__nv_bfloat16>(rule, make_args<__nv_bfloat16>(P, opt->M, V, S, E, G, Pb, hyper_dev, opt->state, opt->eps, opt->lookahead_alpha),
                               n / 4, clip, st);
  return check_launch("opt_step");
}

extern "C" int cotb200_lookahead_sync(long long n, float* P, void* Pb, const cotb200_opt* opt, void* stream) {
  if (!P || !opt || !opt->state || !opt->S) { set_error("lookahead_sync: NULL pointer"); return COTB200_ENULL; }
  if (n <= 0 || (n & 3)) { set_error("lookahead_sync: n=%lld must be a positive multiple of 4", n); return COTB200_EINVAL; }
  if (!(opt->lookahead_alpha >= 0.f && opt->lookahead_alpha <= 1.f)) { set_error("lookahead_sync: alpha must be in [0, 1]"); return COTB200_EINVAL; }
  if (!aligned16(P) || !aligned16(opt->S) || (Pb && (reinterpret_cast<uintptr_t>(Pb) & 7))) {
    set_error("lookahead_sync: flat buffers must be 16-byte aligned"); return COTB200_EALIGN;
  }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_PROF_B("lookahead_sync", (double)n * (16.0 + (Pb ? 2.0 : 0.0)));
  lookahead_sync_kernel<<<grid_stride_blocks(n / 4, 256, 16), 256, 0, st>>>(P, opt->S, (__nv_bfloat16*)Pb, opt->state, opt->lookahead_alpha, n / 4);
  return check_launch("lookahead_sync");
}
