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

// geometry, tensor maps and launch shape of the forward / dX / dW kernels;
// returns false when the TMA path cannot take the call
template <typename T>
static bool at_setup(int mode, const Nhwc2Args& a, const T* A, const T* Bp, const T* out, AtLaunch& L) {
  if constexpr (std::is_same<T, double>::value) { return false; } else {
    constexpr int VEC = 16 / (int)sizeof(T);
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
  template int agg_tma_fwd<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);          \
  template int agg_tma_dx<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);           \
  template int agg_tma_dw<T>(const Nhwc2Args&, const T*, const T*, T*, cudaStream_t, int*);
COTB200_INST3(float) COTB200_INST3(double) COTB200_INST3(__nv_bfloat16) COTB200_INST3(__half)

}  // namespace cotb200
