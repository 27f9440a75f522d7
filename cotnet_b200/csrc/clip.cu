// Gradient clipping of the training step (train.py:270-273 -> utils/clip_grad.py:dispatch_clip_grad), sm_90a.
//
// The step's gradients exist only in the flat buckets (optim.cu), between the all-reduce and the optimizer pass.  The clip is
// folded into that pass: the optimizer reads g' = G*grad_scale, clips it in fp32 and uses it in place of G*grad_scale, so the
// bucket is never rewritten (and never rounded to bf16 after the clip).
//
//   cotb200_grad_norm          NORM: N = ||g'|| over both buckets, one launch, deterministic (det_finish); f = min(1, c/(N+1e-6))
//   cotb200_unit_norms         AGC: ||P_u||, ||g'_u|| and the factor of every unit, one warp per unit
//
// The update pass that applies the factors, cotb200_opt_step, is in opt.cu.  With a factor of 1 or a clamp that does not bind, g'
// goes into the update unchanged: the same arithmetic, bit for bit, as the pass without a clip.
#include "common.cuh"

namespace cotb200 {

static constexpr int CLIP_SEG_MAX = 4096;        // elements per AGC segment (one warp): 32 float4 per lane at most

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------ grad_norm
// Blocks [0, b0) stride over range 0, blocks [b0, grid) over range 1; one partial per block, added by det_finish in block order.
template <typename TG0>
__global__ void __launch_bounds__(256)
grad_norm_kernel(const TG0* __restrict__ G0, const float* __restrict__ gs0, long long n04, const float* __restrict__ G1,
                 const float* __restrict__ gs1, long long n14, int b0, float max_norm, DetArena det, float* __restrict__ out) {
  __shared__ float red[8];
  float acc = 0.f;
  if ((int)blockIdx.x < b0) {
    const float gs = __ldg(gs0);
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n04; i += (long long)b0 * 256) {
      const Pack<TG0, 4> g = ld_pack<TG0, 4>(G0 + i * 4);
#pragma unroll
      for (int k = 0; k < 4; ++k) { const float v = (float)to_acc(g.v[k]) * gs; acc = fmaf(v, v, acc); }
    }
  } else {
    const float gs = __ldg(gs1);
    const int nb = gridDim.x - b0;
    for (long long i = (long long)(blockIdx.x - b0) * 256 + threadIdx.x; i < n14; i += (long long)nb * 256) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(G1) + i);
      const float v[4] = {g.x * gs, g.y * gs, g.z * gs, g.w * gs};
#pragma unroll
      for (int k = 0; k < 4; ++k) acc = fmaf(v[k], v[k], acc);
    }
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w];
    det.scr[blockIdx.x] = s;
  }
  det_finish(det.scr, 1, blockIdx.x, gridDim.x, det.tick, threadIdx.x, 256, [&](int, float total) {
    const float N = sqrtf(total);
    // clip_grad_norm_: clip_coef = max_norm / (total_norm + 1e-6) is torch's scalar / tensor, i.e. reciprocal() * max_norm;
    // clamp(clip_coef, max=1.0) keeps a NaN
    const float q = (1.f / (N + 1e-6f)) * max_norm;
    out[0] = N;
    out[1] = q > 1.f ? 1.f : q;
  });
}

// ------------------------------------------------------------------------------------------------ unit_norms
// adaptive_clip_grad (utils/clip_grad.py:12-24): max_norm = unitwise_norm(p).clamp_(min=1e-3).mul_(c); grad_norm = unitwise_norm(g);
// new = where(grad_norm < max_norm, g, g * (max_norm / grad_norm.clamp(min=1e-6))).  One warp per unit, lane-strided sums added
// by a fixed butterfly: the same factors at every run.
template <typename TG0>
__global__ void __launch_bounds__(256)
unit_norms_kernel(const cotb200_clip_unit* __restrict__ units, int n_units, const float* __restrict__ P0, const TG0* __restrict__ G0,
                  const float* __restrict__ gs0, const float* __restrict__ P1, const float* __restrict__ G1, const float* __restrict__ gs1,
                  float c, float* __restrict__ factor, float* __restrict__ norms) {
  const int u = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (u >= n_units) return;
  const cotb200_clip_unit un = units[u];
  float sp = 0.f, sg = 0.f;
  if (un.range == 0) {
    const float gs = __ldg(gs0);
    const float* p = P0 + un.offset;
    const TG0* g = G0 + un.offset;
    for (int i = lane; i < un.numel; i += 32) {
      const float pv = __ldg(p + i), gv = (float)to_acc(g[i]) * gs;
      sp = fmaf(pv, pv, sp); sg = fmaf(gv, gv, sg);
    }
  } else {
    const float gs = __ldg(gs1);
    const float* p = P1 + un.offset;
    const float* g = G1 + un.offset;
    for (int i = lane; i < un.numel; i += 32) {
      const float pv = __ldg(p + i), gv = __ldg(g + i) * gs;
      sp = fmaf(pv, pv, sp); sg = fmaf(gv, gv, sg);
    }
  }
  sp = warp_sum(sp);
  sg = warp_sum(sg);
  if (lane) return;
  const float pn = sqrtf(sp), gn = sqrtf(sg);
  const float m = (pn < 1e-3f ? 1e-3f : pn) * c;                       // clamp_(min=eps) keeps a NaN
  const float r = m / (gn < 1e-6f ? 1e-6f : gn);
  factor[u] = gn < m ? 1.f : r;                                        // a NaN norm fails `<`: the unit becomes NaN, as in torch
  if (norms) { norms[2 * u] = pn; norms[2 * u + 1] = gn; }
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_clip_seg_max(void) { return CLIP_SEG_MAX; }

extern "C" int cotb200_grad_norm(long long n0, int g0_dtype, const void* G0, const float* gs0, long long n1, const float* G1,
                                 const float* gs1, float max_norm, float* out, void* stream) {
  if (!out || !G0 || !gs0 || (n1 > 0 && (!G1 || !gs1))) { set_error("grad_norm: NULL pointer"); return COTB200_ENULL; }
  if (n0 <= 0 || (n0 & 3) || n1 < 0 || (n1 & 3)) {
    set_error("grad_norm: n0=%lld must be positive and n1=%lld non-negative, both multiples of 4", n0, n1); return COTB200_EINVAL;
  }
  if (g0_dtype != COTB200_F32 && g0_dtype != COTB200_BF16) { set_error("grad_norm: range 0 must be fp32 or bf16"); return COTB200_EDTYPE; }
  if ((reinterpret_cast<uintptr_t>(G0) & (g0_dtype == COTB200_F32 ? 15 : 7)) || (n1 > 0 && !aligned16(G1))) {
    set_error("grad_norm: flat buffers must be 16-byte aligned"); return COTB200_EALIGN;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const long long n04 = n0 / 4, n14 = n1 / 4;
  const int b0 = grid_stride_blocks(n04, 256, 4), b1 = n14 ? grid_stride_blocks(n14, 256, 1) : 0;
  DetScratch ds;
  if (int rc = ds.alloc(det_floats(b0 + b1, 1), 1, st)) return rc;
  COTB200_PROF_B("grad_norm", (double)n0 * (g0_dtype == COTB200_F32 ? 4.0 : 2.0) + (double)n1 * 4.0 + 8.0);
  if (g0_dtype == COTB200_F32)
    grad_norm_kernel<float><<<b0 + b1, 256, 0, st>>>((const float*)G0, gs0, n04, G1, gs1, n14, b0, max_norm, ds.a, out);
  else
    grad_norm_kernel<__nv_bfloat16><<<b0 + b1, 256, 0, st>>>((const __nv_bfloat16*)G0, gs0, n04, G1, gs1, n14, b0, max_norm, ds.a, out);
  return check_launch("grad_norm");
}

extern "C" int cotb200_unit_norms(int n_units, const cotb200_clip_unit* units_dev, long long unit_elems, const float* P0, int g0_dtype,
                                  const void* G0, const float* gs0, const float* P1, const float* G1, const float* gs1, float clip_factor,
                                  float* factor, float* norms, void* stream) {
  if (!units_dev || !P0 || !G0 || !gs0 || !factor) { set_error("unit_norms: NULL pointer"); return COTB200_ENULL; }
  if ((P1 != nullptr) != (G1 != nullptr) || (P1 != nullptr) != (gs1 != nullptr)) {
    set_error("unit_norms: range 1 needs all of P1, G1, gs1 or none"); return COTB200_ENULL;
  }
  if (n_units <= 0 || unit_elems < 0) { set_error("unit_norms: n_units=%d must be positive", n_units); return COTB200_EINVAL; }
  if (g0_dtype != COTB200_F32 && g0_dtype != COTB200_BF16) { set_error("unit_norms: range 0 must be fp32 or bf16"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = (unsigned)((n_units + 7) / 8);
  COTB200_PROF_B("unit_norms", (double)unit_elems * (8.0 + (g0_dtype == COTB200_F32 ? 0.0 : -2.0)) + (double)n_units * (16.0 + 4.0));
  if (g0_dtype == COTB200_F32)
    unit_norms_kernel<float><<<grid, 256, 0, st>>>(units_dev, n_units, P0, (const float*)G0, gs0, P1, G1, gs1, clip_factor, factor, norms);
  else
    unit_norms_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(units_dev, n_units, P0, (const __nv_bfloat16*)G0, gs0, P1, G1, gs1, clip_factor,
                                                           factor, norms);
  return check_launch("unit_norms");
}
