// LocalConv 3x3 forward on NHWC tensors, third generation: persistent CTAs fed by a TMA pipeline (sm_90a).
//
// The register-resident second-generation kernels are LATENCY bound: ~105 registers -> 2 CTAs/SM, 8 resident warps, every
// warp stalled on global loads.
// This kernel decouples the memory stream from the math:
//   * warp 0 is a TMA producer: per tile it issues cp.async.bulk.tensor loads of the input band WITH its halo
//     (4-D box {128 B of channels, W+2, TH+2, 1} fetched at (c0, -1, h0-1, n): out-of-bounds coordinates are
//     zero-filled by the TMA unit == the operator's zero padding) and of the weight band, into a multi-stage
//     shared-memory ring guarded by mbarriers (complete_tx);
//   * the other warps consume: one thread per (pixel, 16-byte channel packet), operands read from shared memory
//     with conflict-free 16-byte accesses (input rows are 128B-swizzled by TMA; the 8 lanes sharing a weight packet
//     broadcast), bf16/fp16 widened into fp32 FMAs, result stored straight to global, coalesced;
//   * CTAs are persistent (grid = resident CTAs), tiles = (sample, band of TH image rows) taken round-robin.
// Weight layout: COTB200_NHWC_TAP (tap-major chunks of gc weight channels) -- the block-internal layout.
#include <cuda.h>
#include <cstdlib>
#include "common.cuh"
#include "tma.cuh"

namespace cotb200 {


static constexpr int AT_MAX_STAGES = 4;

struct AggTmaP {
  int N, C, H, W, wc, Cf, wcf, gc, J;
  int TH;                 // image rows per tile
  int slabs;              // 128-byte channel slabs per pixel = C * sizeof(T) / 128
  int jboxes, jbox;       // weight row split into jboxes TMA boxes of jbox elements (<= 256)
  int stages;
  int slab_bytes;         // (TH+2)*(W+2)*128 rounded up to 1024
  int x_bytes_tx;         // bytes TMA reports for the input boxes of one stage
  int w_stage_bytes;      // TH*W*J*sizeof(T) rounded up to 128
  int w_bytes_tx;
  int stage_bytes;
  int bands;              // ceil(H / TH)
  int total_tiles;
  long long y_sn;         // output batch stride (elements)
  int y_sp;               // output pixel stride (elements)
  int mode;               // 0 forward, 1 dX (weights fetched WITH halo), 2 dW (second operand = dY band, output = dW)
  int whalo;              // 1: weight tile is (TH+2) x (W+2) rows
  int wrows;              // rows of the weight tile = (TH + 2*whalo) * (W + 2*whalo)
  int b_slab_bytes;       // dW: bytes of one 128-byte-wide dY slab [TH][W] rounded to 1024
  int GQ;                 // dW: weight packets per pixel
};

// explicit 16-byte shared-memory load from a 32-bit shared address (a generic LD would pay address translation)
template <typename T, int VEC>
__device__ __forceinline__ Pack<T, VEC> lds_pack(uint32_t saddr) {
  uint4 u;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "r"(saddr));
  Pack<T, VEC> r;
  *reinterpret_cast<uint4*>(&r) = u;
  return r;
}

template <typename T>
__device__ __forceinline__ void at_producer(const CUtensorMap& mapX, const CUtensorMap& mapW, const AggTmaP& p, uint8_t* smem,
                                            uint64_t* s_full, uint64_t* s_empty, int lane) {
    if (lane == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
        const int s = it % p.stages;
        const uint32_t ph = (it / p.stages) & 1;
        mbar_wait(smem_u32(&s_empty[s]), ph ^ 1);
        const int n = tile / p.bands, h0 = (tile - n * p.bands) * p.TH;
        const uint32_t full = smem_u32(&s_full[s]);
        const uint32_t base = smem_u32(smem + (size_t)s * p.stage_bytes);
        mbar_expect_tx(full, (uint32_t)(p.x_bytes_tx + p.w_bytes_tx));
        for (int sl = 0; sl < p.slabs; ++sl)      // input band + halo; OOB (w = -1 / W, h = -1 / H) zero-filled
          tma_load_4d(base + sl * p.slab_bytes, &mapX, full, sl * (128 / (int)sizeof(T)), -1, h0 - 1, n);
        const uint32_t wbase = base + p.slabs * p.slab_bytes;
        if (p.mode == 2) {        // dW: second operand = dY band (no halo), one box per 128-byte channel slab
          for (int sl = 0; sl < p.slabs; ++sl)
            tma_load_4d(wbase + sl * p.b_slab_bytes, &mapW, full, sl * (128 / (int)sizeof(T)), 0, h0, n);
        } else {                  // weights: [rows][J]; dX needs them at the neighbour pixels -> haloed band
          // one 5-D box {jbox, jboxes, W(+2), TH(+2), 1}: the J = jboxes*jbox weights of a pixel land contiguously
          tma_load_5d(wbase, &mapW, full, 0, 0, -p.whalo, h0 - p.whalo, n);
        }
      }
    }
}

template <typename T, int MODE>
__global__ void __launch_bounds__(1024, 1)
agg3_fwd_tma_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapW, T* __restrict__ y,
                    const AggTmaP p) {
  constexpr int VEC = 16 / (int)sizeof(T);
  extern __shared__ __align__(1024) uint8_t at_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t s_full[AT_MAX_STAGES], s_empty[AT_MAX_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ncw = (blockDim.x >> 5) - 1;               // consumer warps
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapX) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
    for (int s = 0; s < p.stages; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), ncw); }
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == 0) {
    at_producer<T>(mapX, mapW, p, smem, s_full, s_empty, lane);
  } else {
    // ===================== consumers: thread = (pixel of the band, 16-byte channel packet) =====================
    // The tile geometry is the same for every tile, so all index arithmetic (div/mod by runtime sizes) is done ONCE per
    // thread here; inside the tile loop an item costs 9 x (2 LDS.128 + 8 FMA) plus a handful of address adds.
    const int ct = threadIdx.x - 32, nct = ncw * 32;
    const int CQ = p.C / VEC;
    const int items = p.TH * p.W * CQ;
    const int Wp = p.W + 2;
    constexpr int MAXI = 2;                 // items per thread (host guarantees items <= MAXI * consumers)
    int i_hl[MAXI], i_rc[MAXI], i_xb[MAXI], i_ch[MAXI], i_wb[MAXI], i_ob[MAXI];
#pragma unroll
    for (int k = 0; k < MAXI; ++k) {
      const int item = ct + k * nct;
      i_hl[k] = -1;
      if (item < items) {
        const int q = item % CQ, px = item / CQ;
        const int hl = px / p.W, wl = px - hl * p.W;
        const int c0 = q * VEC;
        const int g0 = (c0 / p.Cf) * p.wcf + (c0 % p.Cf) % p.wcf;
        const int cb = c0 * (int)sizeof(T);
        const int e0 = (g0 / p.gc) * 9 * p.gc + g0 % p.gc;
        i_hl[k] = hl;
        i_rc[k] = (hl + 1) * Wp + wl + 1;                     // centre row of the haloed band
        i_xb[k] = (cb >> 7) * p.slab_bytes;
        i_ch[k] = (cb >> 4) & 7;
        i_wb[k] = (MODE == 0 ? (px * p.J + e0) : e0) * (int)sizeof(T);
        i_ob[k] = (hl * p.W + wl) * p.y_sp + c0;
      }
    }
    const uint32_t smem_base = smem_u32(smem);
    const int wtap = p.gc * (int)sizeof(T);                    // bytes between the packets of consecutive taps
    const int wrow = p.J * (int)sizeof(T);                     // bytes of one pixel's weight row
    int it = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
      const int s = it % p.stages;
      const uint32_t ph = (it / p.stages) & 1;
      mbar_wait(smem_u32(&s_full[s]), ph);
      const int n = tile / p.bands, h0 = (tile - n * p.bands) * p.TH;
      const uint32_t xs = smem_base + (uint32_t)(s * p.stage_bytes);
      const uint32_t ws = xs + (uint32_t)(p.slabs * p.slab_bytes);
      T* yt = y + n * p.y_sn + (long long)h0 * p.W * p.y_sp;
#pragma unroll
      for (int k = 0; k < MAXI; ++k) {
        if (i_hl[k] < 0 || h0 + i_hl[k] >= p.H) continue;
        const uint32_t xb = xs + (uint32_t)i_xb[k];
        const uint32_t wb = ws + (uint32_t)i_wb[k];
        float acc[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          // forward: neighbour (h+dh, w+dw) with the centre pixel's weights;  dX: neighbour (h-dh, w-dw) AND its weights
          const int dr = (t / 3 - 1) * Wp + (t % 3 - 1);
          const int r = MODE == 0 ? i_rc[k] + dr : i_rc[k] - dr;
          const Pack<T, VEC> wv = lds_pack<T, VEC>(wb + t * wtap + (MODE == 0 ? 0 : r * wrow));
          const Pack<T, VEC> xv = lds_pack<T, VEC>(xb + r * 128 + ((i_ch[k] ^ (r & 7)) << 4));
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] = mfma<T>(wv.v[i], xv.v[i], acc[i]);
        }
        Pack<T, VEC> o;
#pragma unroll
        for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(acc[i]);
        st_pack<T, VEC>(yt + i_ob[k], o);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&s_empty[s]));   // this warp is done reading the stage
    }
  }
}

// dW[p, (g0+i), t] = sum_{sharers j} x[p + off_t][cb_j + i] * dY[p][cb_j + i]          (TAP layout output)
// Thread = (pixel, weight packet) and loops over the `rep` sharers itself: 72 fp32 accumulators in registers, no
// cross-lane reduction at all.  Lanes are consecutive pixels; their 16-byte reads hit different 128-byte rows, which the
// TMA 128B swizzle spreads over all banks (chunk ^ row%8), so the all-sharers mapping that was L1-bound on global
// memory (first generation) is conflict-free here.
template <typename T>
__global__ void __launch_bounds__(512, 1)
agg3_dw_tma_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapG, T* __restrict__ dw,
                   const AggTmaP p) {
  constexpr int VEC = 16 / (int)sizeof(T);
  extern __shared__ __align__(1024) uint8_t at_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t s_full[AT_MAX_STAGES], s_empty[AT_MAX_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ncw = (blockDim.x >> 5) - 1;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapX) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapG) : "memory");
    for (int s = 0; s < p.stages; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), ncw); }
    mbar_init_fence();
  }
  __syncthreads();
  if (warp == 0) {
    at_producer<T>(mapX, mapG, p, smem, s_full, s_empty, lane);
  } else {
    const int ct = threadIdx.x - 32, nct = ncw * 32;
    const int items = p.TH * p.W * p.GQ;
    const int Wp = p.W + 2;
    const int rep = p.Cf / p.wcf;                      // sharers per weight channel
    const uint32_t smem_base = smem_u32(smem);
    int it = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
      const int s = it % p.stages;
      const uint32_t ph = (it / p.stages) & 1;
      mbar_wait(smem_u32(&s_full[s]), ph);
      const int n = tile / p.bands, h0 = (tile - n * p.bands) * p.TH;
      const uint32_t xs = smem_base + (uint32_t)(s * p.stage_bytes);
      const uint32_t gs = xs + (uint32_t)(p.slabs * p.slab_bytes);
      for (int item = ct; item < items; item += nct) {
        const int px = item % (p.TH * p.W), gv = item / (p.TH * p.W);      // lanes = consecutive pixels
        const int hl = px / p.W, wl = px - hl * p.W;
        if (h0 + hl >= p.H) continue;
        const int g0 = gv * VEC;
        const int cb0 = ((g0 / p.wcf) * p.Cf + g0 % p.wcf) * (int)sizeof(T);   // byte offset of sharer 0's packet
        const int cstep = p.wcf * (int)sizeof(T);
        const int rc = (hl + 1) * Wp + wl + 1;
        float acc[9][VEC];
#pragma unroll
        for (int t = 0; t < 9; ++t)
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[t][i] = 0.f;
        for (int j = 0; j < rep; ++j) {
          const int cb = cb0 + j * cstep;
          const int slab = cb >> 7, chunk = (cb >> 4) & 7;
          const Pack<T, VEC> gvv = lds_pack<T, VEC>(gs + (uint32_t)(slab * p.b_slab_bytes + px * 128 + ((chunk ^ (px & 7)) << 4)));
          const uint32_t xb = xs + (uint32_t)(slab * p.slab_bytes);
#pragma unroll
          for (int t = 0; t < 9; ++t) {
            const int r = rc + (t / 3 - 1) * Wp + (t % 3 - 1);
            const Pack<T, VEC> xv = lds_pack<T, VEC>(xb + (uint32_t)(r * 128 + ((chunk ^ (r & 7)) << 4)));
#pragma unroll
            for (int i = 0; i < VEC; ++i) acc[t][i] = mfma<T>(xv.v[i], gvv.v[i], acc[t][i]);
          }
        }
        T* wr = dw + n * p.y_sn + (long long)((h0 + hl) * p.W + wl) * p.y_sp + (g0 / p.gc) * 9 * p.gc + g0 % p.gc;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          Pack<T, VEC> o;
#pragma unroll
          for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(acc[t][i]);
          st_pack<T, VEC>(wr + t * p.gc, o);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&s_empty[s]));
    }
  }
}


// ------------------------------------------------------------------------------------------------ fused inference kernel
// out = SiLU(bn(LocalConv(v, GroupNorm(l))))  and  psum[n, c] += sum_px (out + k)     (models/cotnet.py:85-98, eval mode)
//   * prologue: the weight tile arrives as the RAW logits l (tap-major); the consumer warps turn it into the normalised
//     weights in place, w = l * a[n, j] + c[n, j] (a, c per sample and logit column: GroupNorm statistics + affine, from
//     cotb200_gn9_from_colsums) -- once per weight element instead of once per use (8 channels share a weight), and the
//     normalised weights never exist in HBM;
//   * main loop: as agg3_fwd_tma_kernel;
//   * epilogue: eval-mode BatchNorm (scale/shift) + SiLU on the accumulators, the result is stored, and (out + k) is pooled per
//     channel: registers -> warp shuffle over the lanes that own the same channel packet -> shared memory -> one global atomic
//     per (tile, channel).  The separate GroupNorm-apply and pooling passes of the block disappear.
struct AggEvalP {
  const float2* coef;        // [N, J] (a, c)
  const float* scale;        // [C] eval BatchNorm folded
  const float* shift;
  const void* k;             // [N, H, W, C] like the output
  float* psum;               // [N, C]
};

template <typename T>
__global__ void __launch_bounds__(1024, 1)
agg3_eval_tma_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapW, T* __restrict__ y,
                     const AggTmaP p, const AggEvalP q) {
  constexpr int VEC = 16 / (int)sizeof(T);
  extern __shared__ __align__(1024) uint8_t at_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t s_full[AT_MAX_STAGES], s_empty[AT_MAX_STAGES];
  __shared__ __align__(16) float2 s_coef[576];
  __shared__ __align__(16) float s_ss[2][512];
  __shared__ float s_pool[2][512];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ncw = (blockDim.x >> 5) - 1;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapX) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
    for (int s = 0; s < p.stages; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), ncw); }
    mbar_init_fence();
  }
  for (int i = threadIdx.x; i < p.C; i += blockDim.x) {
    s_ss[0][i] = q.scale[i]; s_ss[1][i] = q.shift[i];
    s_pool[0][i] = 0.f; s_pool[1][i] = 0.f;
  }
  __syncthreads();
  if (warp == 0) {
    at_producer<T>(mapX, mapW, p, smem, s_full, s_empty, lane);
  } else {
    const int ct = threadIdx.x - 32, nct = ncw * 32;
    const int CQ = p.C / VEC;
    const int items = p.TH * p.W * CQ;
    const int Wp = p.W + 2;
    constexpr int MAXI = 2;
    int i_hl[MAXI], i_rc[MAXI], i_xb[MAXI], i_ch[MAXI], i_wb[MAXI], i_ob[MAXI], i_c0[MAXI];
#pragma unroll
    for (int kk = 0; kk < MAXI; ++kk) {
      const int item = ct + kk * nct;
      i_hl[kk] = -1; i_c0[kk] = 0;
      if (item < items) {
        const int qq = item % CQ, px = item / CQ;
        const int hl = px / p.W, wl = px - hl * p.W;
        const int c0 = qq * VEC;
        const int g0 = (c0 / p.Cf) * p.wcf + (c0 % p.Cf) % p.wcf;
        const int cb = c0 * (int)sizeof(T);
        const int e0 = (g0 / p.gc) * 9 * p.gc + g0 % p.gc;
        i_hl[kk] = hl;
        i_rc[kk] = (hl + 1) * Wp + wl + 1;
        i_xb[kk] = (cb >> 7) * p.slab_bytes;
        i_ch[kk] = (cb >> 4) & 7;
        i_wb[kk] = (px * p.J + e0) * (int)sizeof(T);
        i_ob[kk] = (hl * p.W + wl) * p.y_sp + c0;
        i_c0[kk] = c0;
      }
    }
    // all items of a thread share the channel packet when the consumer count is a multiple of CQ (host guarantees it)
    const uint32_t smem_base = smem_u32(smem);
    const int wtap = p.gc * (int)sizeof(T);
    const int JP = p.J / VEC;                                  // 16-byte packets per weight row
    const int npk = p.TH * p.W * JP;
    const T* kg = reinterpret_cast<const T*>(q.k);
    int it = 0, last_n = -1;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
      const int s = it % p.stages;
      const uint32_t ph = (it / p.stages) & 1;
      const int n = tile / p.bands, h0 = (tile - n * p.bands) * p.TH;
      const int par = it & 1;
      if (n != last_n) {                                        // (a, c) of this sample -> shared memory
        asm volatile("bar.sync 2, %0;" ::"r"(nct) : "memory");  // nobody still reads the previous sample's table
        // stored element-major, [VEC][JP]: the prologue's lanes walk jp, so lane-consecutive float2 reads are conflict-free
        for (int j = ct; j < p.J; j += nct) s_coef[(j % VEC) * JP + j / VEC] = __ldg(q.coef + (long long)n * p.J + j);
        last_n = n;
      }
      // k of this thread's pixels: issued now, consumed in the epilogue -- the global-load latency hides behind the TMA wait,
      // the prologue and the tap loop (loading it at the point of use exposes its latency per item)
      const T* kt = kg + n * p.y_sn + (long long)h0 * p.W * p.y_sp;
      Pack<T, VEC> kpre[MAXI];
#pragma unroll
      for (int kk = 0; kk < MAXI; ++kk)
        if (i_hl[kk] >= 0 && h0 + i_hl[kk] < p.H) kpre[kk] = ld_pack<T, VEC>(kt + i_ob[kk]);
      mbar_wait(smem_u32(&s_full[s]), ph);
      const uint32_t xs = smem_base + (uint32_t)(s * p.stage_bytes);
      const uint32_t ws = xs + (uint32_t)(p.slabs * p.slab_bytes);
      asm volatile("bar.sync 2, %0;" ::"r"(nct) : "memory");    // table visible; every warp has seen the stage arrive
      // ---- prologue: GroupNorm affine on the weight tile, in place
      for (int pk = ct; pk < npk; pk += nct) {
        const int row = pk / JP, jp = pk - row * JP;
        const uint32_t addr = ws + (uint32_t)((row * p.J + jp * VEC) * (int)sizeof(T));
        Pack<T, VEC> lv = lds_pack<T, VEC>(addr);
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float2 ac = s_coef[i * JP + jp];
          lv.v[i] = Elem<T>::from(fmaf(to_acc(lv.v[i]), ac.x, ac.y));
        }
        const uint4 u = *reinterpret_cast<const uint4*>(&lv);
        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(u.x), "r"(u.y), "r"(u.z), "r"(u.w) : "memory");
      }
      asm volatile("bar.sync 2, %0;" ::"r"(nct) : "memory");
      T* yt = y + n * p.y_sn + (long long)h0 * p.W * p.y_sp;
      float pacc[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) pacc[i] = 0.f;
#pragma unroll
      for (int kk = 0; kk < MAXI; ++kk) {
        if (i_hl[kk] < 0 || h0 + i_hl[kk] >= p.H) continue;
        const uint32_t xb = xs + (uint32_t)i_xb[kk];
        const uint32_t wb = ws + (uint32_t)i_wb[kk];
        float acc[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const int r = i_rc[kk] + (t / 3 - 1) * Wp + (t % 3 - 1);
          const Pack<T, VEC> wv = lds_pack<T, VEC>(wb + t * wtap);
          const Pack<T, VEC> xv = lds_pack<T, VEC>(xb + r * 128 + ((i_ch[kk] ^ (r & 7)) << 4));
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] = mfma<T>(wv.v[i], xv.v[i], acc[i]);
        }
        const Pack<T, VEC> kv = kpre[kk];
        Pack<T, VEC> o;
        float bsc[VEC], bsh[VEC];                               // folded BatchNorm of the channel packet: 128-bit shared loads
#pragma unroll
        for (int i = 0; i < VEC; i += 4) {
          *reinterpret_cast<float4*>(&bsc[i]) = *reinterpret_cast<const float4*>(&s_ss[0][i_c0[kk] + i]);
          *reinterpret_cast<float4*>(&bsh[i]) = *reinterpret_cast<const float4*>(&s_ss[1][i_c0[kk] + i]);
        }
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float z = fmaf(acc[i], bsc[i], bsh[i]);
          float sg;
          if constexpr (sizeof(T) == 2) { float th; asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(0.5f * z)); sg = fmaf(0.5f, th, 0.5f); }
          else sg = __fdividef(1.f, 1.f + __expf(-z));
          o.v[i] = Elem<T>::from(z * sg);
          pacc[i] += to_acc(o.v[i]) + to_acc(kv.v[i]);          // pool what is stored (bf16-rounded), like a separate pass would
        }
        st_pack<T, VEC>(yt + i_ob[kk], o);
      }
      // the tile was WRITTEN by the generic proxy (prologue); order those writes before the TMA refill of the stage
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&s_empty[s]));        // this warp is done with the stage
      // ---- pooled (out + k): lanes owning the same channel packet are CQ apart
      for (int off = CQ; off < 32; off <<= 1)
#pragma unroll
        for (int i = 0; i < VEC; ++i) pacc[i] += __shfl_xor_sync(0xffffffffu, pacc[i], off);
      if (lane < CQ || CQ >= 32) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) atomicAdd(&s_pool[par][i_c0[0] + i], pacc[i]);
      }
      asm volatile("bar.sync 2, %0;" ::"r"(nct) : "memory");
      for (int c = ct; c < p.C; c += nct) {
        atomicAdd(q.psum + (long long)n * p.C + c, s_pool[par][c]);
        s_pool[par][c] = 0.f;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*AtEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static AtEncodeFn at_encode_fn() {
  static AtEncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (AtEncodeFn)p;
  }
  return fn;
}

template <typename T> static CUtensorMapDataType at_dtype();
template <> CUtensorMapDataType at_dtype<float>() { return CU_TENSOR_MAP_DATA_TYPE_FLOAT32; }
template <> CUtensorMapDataType at_dtype<__nv_bfloat16>() { return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; }
template <> CUtensorMapDataType at_dtype<__half>() { return CU_TENSOR_MAP_DATA_TYPE_FLOAT16; }

// NHWC tensor [N,H,W,Cdim] with pixel pitch sp / batch pitch sn (elements); box {b0, b1, b2, 1}
template <typename T>
static bool at_make_map(CUtensorMap* m, const void* base, int N, int H, int W, int Cdim, long long sp, long long sn, int b0, int b1,
                        int b2, bool swizzle) {
  AtEncodeFn enc = at_encode_fn();
  if (!enc) return false;
  cuuint64_t dims[4] = {(cuuint64_t)Cdim, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)sp * sizeof(T), (cuuint64_t)sp * sizeof(T) * W, (cuuint64_t)sn * sizeof(T)};
  cuuint32_t box[4] = {(cuuint32_t)b0, (cuuint32_t)b1, (cuuint32_t)b2, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  return enc(m, at_dtype<T>(), 4, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// weights [N,H,W,J] as 5-D {jbox, jboxes, W, H, N}; box {jbox, jboxes, bw, bh, 1} -> smem [bh][bw][J]
template <typename T>
static bool at_make_map_w(CUtensorMap* m, const void* base, int N, int H, int W, int jbox, int jboxes, long long sp, long long sn,
                          int bw, int bh) {
  AtEncodeFn enc = at_encode_fn();
  if (!enc) return false;
  cuuint64_t dims[5] = {(cuuint64_t)jbox, (cuuint64_t)jboxes, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[4] = {(cuuint64_t)jbox * sizeof(T), (cuuint64_t)sp * sizeof(T), (cuuint64_t)sp * sizeof(T) * W,
                           (cuuint64_t)sn * sizeof(T)};
  cuuint32_t box[5] = {(cuuint32_t)jbox, (cuuint32_t)jboxes, (cuuint32_t)bw, (cuuint32_t)bh, 1};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  return enc(m, at_dtype<T>(), 5, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct Nhwc2Args {
  int N, C, H, W, wc, fold, layout, gc, dtype;
  long long x_sn, x_sp, w_sn, w_sp, y_sn, y_sp;
};

// mode 0: a = x, b = w, out = y      mode 1: a = dy, b = w, out = dx      mode 2: a = x, b = dy, out = dw
// returns 1 if handled (rc in *rc), 0 if the caller should use the register-resident kernels
struct AtLaunch { AggTmaP p; CUtensorMap ma, mb; int threads, smem, grid; };

// geometry, tensor maps and launch shape shared by the forward / dX / dW kernels and the fused inference kernel;
// returns false when the TMA path cannot take the call
template <typename T>
static bool at_setup(int mode, const Nhwc2Args& a, const T* A, const T* Bp, const T* out, AtLaunch& L) {
  if constexpr (std::is_same<T, double>::value) { return false; } else {
    constexpr int VEC = 16 / (int)sizeof(T);
    static int disabled = -1;
    if (disabled < 0) { const char* e = getenv("COTB200_AGG_TMA"); disabled = (e && e[0] == '0') ? 1 : 0; }
    if (disabled) return false;
    if (a.layout != COTB200_NHWC_TAP) return false;
    const int Cf = a.C / a.fold, wcf = a.wc / a.fold;
    if ((a.C * (int)sizeof(T)) % 128 || wcf % VEC || a.gc < VEC || a.gc % VEC || a.wc % a.gc) return false;
    if (((uintptr_t)A | (uintptr_t)Bp | (uintptr_t)out) & 15) return false;
    const long long strides[6] = {a.x_sn, a.x_sp, a.w_sn, a.w_sp, a.y_sn, a.y_sp};
    for (long long sv : strides) if ((sv * (long long)sizeof(T)) % 16) return false;
    if (a.W + 2 > 256) return false;
    AggTmaP& p = L.p;
    p = AggTmaP{};
    p.N = a.N; p.C = a.C; p.H = a.H; p.W = a.W; p.wc = a.wc; p.Cf = Cf; p.wcf = wcf; p.gc = a.gc; p.J = 9 * a.wc;
    p.mode = mode; p.whalo = mode == 1 ? 1 : 0;
    p.slabs = a.C * (int)sizeof(T) / 128;
    p.jboxes = (p.J + 255) / 256;
    while (p.J % p.jboxes) ++p.jboxes;
    p.jbox = p.J / p.jboxes;
    if ((p.jbox * (int)sizeof(T)) % 16) return false;
    p.GQ = a.wc / VEC;

    // output strides: y (fwd), dx (dX: same layout as x), dw (dW: same layout as w)
    const long long o_sn = mode == 0 ? a.y_sn : (mode == 1 ? a.x_sn : a.w_sn);
    const long long o_sp = mode == 0 ? a.y_sp : (mode == 1 ? a.x_sp : a.w_sp);
    if (o_sp > 2147483647LL) return false;
    p.y_sn = o_sn; p.y_sp = (int)o_sp;
    // tile height: stage <= 72 KB, stop growing once a tile has ~900 work items
    const int CQ = a.C / VEC;
    int best_th = 0;
    for (int th = 1; th <= a.H && th <= 254; ++th) {
      const long long xb = (long long)p.slabs * ((((long long)(th + 2) * (a.W + 2) * 128) + 1023) / 1024 * 1024);
      long long bb;
      if (mode == 2) bb = (long long)p.slabs * ((((long long)th * a.W * 128) + 1023) / 1024 * 1024);
      else bb = ((long long)(th + 2 * p.whalo) * (a.W + 2 * p.whalo) * p.J * sizeof(T) + 1023) / 1024 * 1024;
      if (xb + bb > 72 * 1024) break;
      if (mode != 2 && (long long)th * a.W * CQ > 2 * 896) break;      // at most 2 work items per consumer thread
      best_th = th;
      if ((long long)th * a.W * CQ >= 896) break;
    }
    if (!best_th) return false;
    p.TH = best_th;
    p.wrows = (p.TH + 2 * p.whalo) * (a.W + 2 * p.whalo);
    p.slab_bytes = (int)((((long long)(p.TH + 2) * (a.W + 2) * 128) + 1023) / 1024 * 1024);
    p.x_bytes_tx = p.slabs * (p.TH + 2) * (a.W + 2) * 128;
    if (mode == 2) {
      p.b_slab_bytes = (int)((((long long)p.TH * a.W * 128) + 1023) / 1024 * 1024);
      p.w_bytes_tx = p.slabs * p.TH * a.W * 128;
      p.w_stage_bytes = p.slabs * p.b_slab_bytes;
    } else {
      p.w_bytes_tx = p.wrows * p.J * (int)sizeof(T);
      p.w_stage_bytes = (p.w_bytes_tx + 1023) / 1024 * 1024;
    }
    p.stage_bytes = p.slabs * p.slab_bytes + p.w_stage_bytes;
    p.stages = (int)((200 * 1024) / p.stage_bytes);
    if (p.stages > AT_MAX_STAGES) p.stages = AT_MAX_STAGES;
    if (p.stages < 2) return false;
    p.bands = (a.H + p.TH - 1) / p.TH;
    p.total_tiles = a.N * p.bands;
    CUtensorMap& ma = L.ma;
    CUtensorMap& mb = L.mb;
    const long long a_sp = mode == 1 ? a.y_sp : a.x_sp, a_sn = mode == 1 ? a.y_sn : a.x_sn;
    if (!at_make_map<T>(&ma, A, a.N, a.H, a.W, a.C, a_sp, a_sn, 128 / (int)sizeof(T), a.W + 2, p.TH + 2, true)) return false;
    if (mode == 2) {
      if (!at_make_map<T>(&mb, Bp, a.N, a.H, a.W, a.C, a.y_sp, a.y_sn, 128 / (int)sizeof(T), a.W, p.TH, true)) return false;
    } else {
      if (!at_make_map_w<T>(&mb, Bp, a.N, a.H, a.W, p.jbox, p.jboxes, a.w_sp, a.w_sn, a.W + 2 * p.whalo, p.TH + 2 * p.whalo)) return false;
    }
    int work_warps;
    if (mode == 2) work_warps = (p.TH * a.W * p.GQ + 31) / 32;
    else work_warps = (p.TH * a.W * CQ + 31) / 32;
    int cw = work_warps > 28 ? 28 : (work_warps < 4 ? 4 : work_warps);
    if (mode != 2 && (long long)p.TH * a.W * CQ > 2LL * cw * 32) return false;
    if (mode == 2 && cw > 15) cw = 15;                 // 72 accumulators per thread: 512 threads x <= 128 registers
    L.threads = (cw + 1) * 32;
    L.smem = p.stages * p.stage_bytes + 1024;
    L.grid = num_sms();
    if (L.grid > p.total_tiles) L.grid = p.total_tiles;
    return true;
  }
}

template <typename T>
static int agg_tma_launch(int mode, const Nhwc2Args& a, const T* A, const T* Bp, T* out, cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    AtLaunch L;
    if (!at_setup<T>(mode, a, A, Bp, out, L)) return 0;
    const AggTmaP& p = L.p;
    const CUtensorMap& ma = L.ma;
    const CUtensorMap& mb = L.mb;
    const int threads = L.threads, smem = L.smem, grid = L.grid;
    cudaError_t e = cudaSuccess;
    static PerDevFlag cfgd[3];
#define AT_CFG(idx, fn) if (bool& cfgf = cfgd[idx].get(); !cfgf) { e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024); cfgf = (e == cudaSuccess); }
    if (mode == 0) {
      AT_CFG(0, (agg3_fwd_tma_kernel<T, 0>));
      if (e == cudaSuccess) { COTB200_PROF_B("agg3_fwd_tma", ((double)a.N * a.H * a.W) * (2.0 * a.C + 9.0 * a.wc) * sizeof(T)); agg3_fwd_tma_kernel<T, 0><<<grid, threads, smem, st>>>(ma, mb, out, p); }
    } else if (mode == 1) {
      AT_CFG(1, (agg3_fwd_tma_kernel<T, 1>));
      if (e == cudaSuccess) { COTB200_PROF_B("agg3_dx_tma", ((double)a.N * a.H * a.W) * (2.0 * a.C + 9.0 * a.wc) * sizeof(T)); agg3_fwd_tma_kernel<T, 1><<<grid, threads, smem, st>>>(ma, mb, out, p); }
    } else {
      AT_CFG(2, (agg3_dw_tma_kernel<T>));
      if (e == cudaSuccess) { COTB200_PROF_B("agg3_dw_tma", ((double)a.N * a.H * a.W) * (2.0 * a.C + 9.0 * a.wc) * sizeof(T)); agg3_dw_tma_kernel<T><<<grid, threads, smem, st>>>(ma, mb, out, p); }
    }
#undef AT_CFG
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(agg tma): %s", cudaGetErrorString(e)); *rc = (int)e; return 1; }
    *rc = check_launch("agg3_tma");
    return 1;
  }
}

// fused inference forward; returns 1 if handled
template <typename T>
int agg_tma_eval(const Nhwc2Args& a, const T* v, const T* l, T* y, const float* coef, const float* scale, const float* shift, const T* k,
                 float* psum, cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    constexpr int VEC = 16 / (int)sizeof(T);
    AtLaunch L;
    if (!at_setup<T>(0, a, v, l, y, L)) return 0;
    const int CQ = a.C / VEC;
    if (a.C > 512 || L.p.J > 576 || (CQ & (CQ - 1))) return 0;          // static tables; power-of-two packet count for the shuffles
    // every item of a thread must own the same channel packet: (consumer threads) % CQ == 0
    int cw = L.threads / 32 - 1;
    while (cw > 0 && (cw * 32) % CQ) --cw;
    if (cw <= 0 || (long long)L.p.TH * a.W * CQ > 2LL * cw * 32) return 0;
    const int threads = (cw + 1) * 32;
    static PerDevFlag cfgd;
    if (bool& cfgf = cfgd.get(); !cfgf) {
      cudaError_t e = cudaFuncSetAttribute(agg3_eval_tma_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 204 * 1024);
      if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(agg eval): %s", cudaGetErrorString(e)); *rc = (int)e; return 1; }
      cfgf = true;
    }
    if (L.smem > 204 * 1024) return 0;
    AggEvalP q{reinterpret_cast<const float2*>(coef), scale, shift, k, psum};
    COTB200_PROF_B("agg3_eval_tma", ((double)a.N * a.H * a.W) * (3.0 * a.C + 9.0 * a.wc) * sizeof(T));
    agg3_eval_tma_kernel<T><<<L.grid, threads, L.smem, st>>>(L.ma, L.mb, y, L.p, q);
    *rc = check_launch("agg3_eval_tma");
    return 1;
  }
}

template <typename T> int agg_tma_fwd(const Nhwc2Args& a, const T* x, const T* w, T* y, cudaStream_t st, int* rc) {
  return agg_tma_launch<T>(0, a, x, w, y, st, rc);
}
template <typename T> int agg_tma_dx(const Nhwc2Args& a, const T* dy, const T* w, T* dx, cudaStream_t st, int* rc) {
  return agg_tma_launch<T>(1, a, dy, w, dx, st, rc);
}
template <typename T> int agg_tma_dw(const Nhwc2Args& a, const T* dy, const T* x, T* dw, cudaStream_t st, int* rc) {
  return agg_tma_launch<T>(2, a, x, dy, dw, st, rc);
}

#define COTB200_INST3(T)                                                                              \
  template int agg_tma_eval<T>(const Nhwc2Args&, const T*, const T*, T*, const float*, const float*, const float*, const T*, float*, cudaStream_t, int*); \
  template int agg_tma_fwd<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);          \
  template int agg_tma_dx<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);           \
  template int agg_tma_dw<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);
COTB200_INST3(float) COTB200_INST3(double) COTB200_INST3(__nv_bfloat16) COTB200_INST3(__half)

}  // namespace cotb200
