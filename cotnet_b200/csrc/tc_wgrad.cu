// Weight gradient of the 1x1 convolutions on the Hopper tensor cores (wgmma, sm_90a):
//
//     OUT[R, Cc] += A[M, R]^T * [B1 | B2][M, Cc]            (contraction over the M pixels)
//
// A = dY (gradient of the convolution output, NHWC rows = pixels), B = the convolution input(s); OUT = dW in fp32.
// Replaces cuDNN's wgrad / the cuBLAS `dY^T X` of the autograd functions for  embed.0 / embed.3 / conv1x1.0 of the CoT layer
// (models/cotnet.py:52,55,60) and conv1 / conv3 / downsample of the enclosing bottleneck (:228-264).
//
// Both operands are "MN-major" for the MMA (the contraction index -- pixels -- is the SLOW index of the row-major pixel
// matrices), so the TMA tiles are used exactly as they land: a box {64 channels, 64 pixels} with the 128-byte swizzle IS
// the canonical MN-major SWIZZLE_128B wgmma layout (64 MN elements contiguous, 8 K rows per 1024-byte atom).  No transpose
// anywhere: wgmma with both transpose flags set (tc_wgmma.cuh).
//
// Split-K over pixels: CTA (tile_r, tile_c, split) accumulates a [128 x BC] fp32 tile of dW in registers over its pixel range
// (4-stage TMA ring) and stores it as that split's partial; wgrad_reduce_kernel adds the partials to OUT in split order.  Algorithmic bytes: (R + Cc) * M * 2 (each operand
// read once) + the dW tile traffic; HBM-bound for every layer of the network.
//   warps 0-7: two consumer warpgroups (warpgroup g: rows 64g .. 64g + 63 of the tile = A box g)   warp 8: TMA producer
#include <cuda.h>
#include <cstdlib>
#include "common.cuh"
#include "tma.cuh"
#include "tc_wgmma.cuh"

namespace cotb200 {

static constexpr int WG_BR = 128;          // rows of OUT per CTA (two warpgroups x 64)
static constexpr int WG_PX = 64;           // pixels per pipeline stage (4 MMAs of K = 16)
static constexpr int WG_STAGES = 4;
static constexpr int WG_THREADS = 288;     // two consumer warpgroups + one producer warp
static constexpr int WG_BOX_BYTES = 64 * WG_PX * 2;    // one {64 ch, 64 px} bf16 box = 8 KB

struct WgParams {
  int M, R, Cc, C1;          // pixels; rows of OUT (channels of A); columns (channels of B1|B2); channels of B1
  int bc;                    // column tile (multiple of 64, <= 256)
  int tiles_r, tiles_c, splits;
  int kb_total;              // ceil(M / 64)
  int transpose;             // 0: OUT[r * ldo + c]   1: OUT[c * ldo + r]
  int lbo, sbo;              // wgmma descriptor offsets (bytes) -- see wgmma_desc_mn_sw128()
  int px;                    // pixels per pipeline stage (multiple of 16): 64, or one output row of the stem convolution
  int stages;                // ring depth (<= WG_STAGES)
  int stem_ho;               // > 0: B = the stem's window matrices (4-D map, csrc/tc_gemm.cu stem mode); pixel block kb = (sample kb / stem_ho,
                             //      output row kb % stem_ho), column block j = s2d row tap a
  long long ldo;
  float* out;
  float* part;               // [splits][R][Cc] fp32 partial tiles of the split-K reduction (wgrad_reduce_kernel adds them in split order)
};

__global__ void __launch_bounds__(WG_THREADS, 1)
tc_wgrad_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB1,
                const __grid_constant__ CUtensorMap mapB2, const WgParams p) {
  extern __shared__ __align__(1024) uint8_t wg_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wg_smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t s_full[WG_STAGES], s_empty[WG_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nbb = p.bc / 64;                                   // B boxes per stage
  const int box_bytes = 128 * p.px;                            // one {64 ch, px pixels} bf16 box
  const int a_bytes = 2 * box_bytes;
  const int stage_bytes = a_bytes + nbb * box_bytes;
  // tile decode
  int t = blockIdx.x;
  const int split = t % p.splits; t /= p.splits;
  const int tc = t % p.tiles_c, tr = t / p.tiles_c;
  const int r0 = tr * WG_BR, c0 = tc * p.bc;
  const int per = (p.kb_total + p.splits - 1) / p.splits;
  const int kb_lo = split * per, kb_hi = min(p.kb_total, kb_lo + per);
  const int nkb = kb_hi - kb_lo;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB1) : "memory");
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), 2); }
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % p.stages;
        const uint32_t ph = (i / p.stages) & 1;
        mbar_wait(smem_u32(&s_empty[s]), ph ^ 1);
        const uint32_t full = smem_u32(&s_full[s]);
        const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes), sb = sa + a_bytes;
        const int px = (kb_lo + i) * p.px;
        mbar_expect_tx(full, (uint32_t)stage_bytes);            // TMA counts whole boxes (zero-filled parts included)
        tma_load_2d(sa, &mapA, full, r0, px);                    // out-of-range channels / pixels are zero-filled: they add 0
        tma_load_2d(sa + box_bytes, &mapA, full, r0 + 64, px);
        if (p.stem_ho > 0) {
          const int b = (kb_lo + i) / p.stem_ho, oh = (kb_lo + i) - b * p.stem_ho;
          for (int j = 0; j < nbb; ++j)                          // tap a = c0 / 64 + j: the windows of s2d row oh - 2 + a
            tma_load_4d(sb + j * box_bytes, &mapB1, full, 0, 0, oh - 2 + c0 / 64 + j, b);
        } else {
          for (int j = 0; j < nbb; ++j) {
            const int c = c0 + j * 64;
            if (c < p.C1) tma_load_2d(sb + j * box_bytes, &mapB1, full, c, px);
            else tma_load_2d(sb + j * box_bytes, &mapB2, full, c - p.C1, px);
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma over the pixel range, then registers -> global reductions =====================
  const int wg = warp >> 2, wl = warp & 3;
  float acc[4][32];
  if (nkb <= 0) {                                              // an empty split still stores its (zero) partial
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[c][i] = 0.f;
  }
  int prev_s = 0;
  for (int i = 0; i < nkb; ++i) {
    const int s = i % p.stages;
    const uint32_t ph = (i / p.stages) & 1;
    mbar_wait(smem_u32(&s_full[s]), ph);
    const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes), sb = sa + a_bytes;
    // A: this warpgroup's 64 rows are box wg; B: 64-column chunk c is box c.  8-pixel K groups are 1024 B apart (SBO),
    // 16 pixels = two 1024-byte atoms: start address += 2048 B per K step
    const uint64_t da = wgmma_desc_mn_sw128(sa + (uint32_t)(wg * box_bytes), p.lbo, p.sbo);
    const uint64_t db = wgmma_desc_mn_sw128(sb, p.lbo, p.sbo);
    wgmma_fence();
    for (int k = 0; k < p.px / 16; ++k) {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < nbb)
          wgmma_m64n64k16<1, 1>(acc[c], da + (uint64_t)(k * (2048 >> 4)), db + (uint64_t)((c * box_bytes) >> 4) + (uint64_t)(k * (2048 >> 4)),
                                (i | k) != 0);
    }
    wgmma_commit();
    if (i > 0) {                                                 // the previous stage's MMAs have retired: hand it back
      wgmma_wait<1>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(smem_u32(&s_empty[prev_s]));
    }
    prev_s = s;
  }
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < 4; ++c) if (c < nbb) wgmma_fence_acc(acc[c]);
  float* part = p.part + (size_t)split * p.R * p.Cc;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c >= nbb) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + wg * 64 + wl * 16 + (lane >> 2) + 8 * h;
      if (r >= p.R) continue;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int cb = c0 + c * 64 + j * 8 + 2 * (lane & 3);
        float* o = part + (size_t)r * p.Cc + cb;
        if (cb + 1 < p.Cc) *reinterpret_cast<float2*>(o) = make_float2(acc[c][4 * j + 2 * h], acc[c][4 * j + 2 * h + 1]);
        else if (cb < p.Cc) *o = acc[c][4 * j + 2 * h];
      }
    }
  }
}

// OUT += the sum of the split-K partial tiles, added in split order (run-to-run identical; float atomics would add them in the
// order the CTAs finish)
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ part, int splits, int R, int Cc, float* __restrict__ out, long long ldo, int transpose) {
  const long long n = (long long)R * Cc;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float t = 0.f;
    for (int s = 0; s < splits; ++s) t += __ldg(part + (size_t)s * n + i);
    const int r = (int)(i / Cc), c = (int)(i - (long long)r * Cc);
    float* o = transpose ? out + (long long)c * ldo + r : out + (long long)r * ldo + c;
    *o += t;
  }
}

static int wgrad_launch(const CUtensorMap& ma, const CUtensorMap& mb1, const CUtensorMap& mb2, WgParams p, int grid, int smem,
                        cudaStream_t st, const char* what, double alg_bytes) {
  DetScratch ds;                                               // the partials, stream-ordered (common.cuh)
  int rc = ds.alloc((size_t)p.splits * p.R * p.Cc, 0, st);
  if (rc) return rc;
  p.part = ds.a.scr;
  static PerDevFlag configured_d;
  if (bool& configured = configured_d.get(); !configured) {
    cudaError_t e = cudaFuncSetAttribute(tc_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
    configured = true;
  }
  {
    COTB200_PROF_B(what, alg_bytes);
    tc_wgrad_kernel<<<grid, WG_THREADS, smem, st>>>(ma, mb1, mb2, p);
    if ((rc = check_launch(what))) return rc;
  }
  const long long n = (long long)p.R * p.Cc;
  const int rgrid = (int)((n + 255) / 256 < 4LL * num_sms() ? (n + 255) / 256 : 4LL * num_sms());
  COTB200_PROF_B("wgrad_reduce", 4.0 * (double)n * (p.splits + 2));
  wgrad_reduce_kernel<<<rgrid, 256, 0, st>>>(p.part, p.splits, p.R, p.Cc, p.out, p.ldo, p.transpose);
  return check_launch("wgrad_reduce");
}

// bf16 pixel matrix [rows = pixels, cols = channels] with pitch ld: box {64 channels, 64 pixels}, 128B swizzle, zero OOB fill
static int wg_make_map(CUtensorMap* m, const void* base, long long pixels, long long channels, long long ld) {
  TcEncodeTiledFn enc = tc_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return COTB200_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || ((ld * 2) & 15)) { set_error("wgrad: TMA operand not 16-byte aligned (ld=%lld)", ld); return COTB200_EALIGN; }
  cuuint64_t dims[2] = {(cuuint64_t)channels, (cuuint64_t)pixels};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)WG_PX};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(wgrad) failed: %d", (int)r); return COTB200_EINVAL; }
  return 0;
}

}  // namespace cotb200

using namespace cotb200;

// OUT (fp32, += : the caller zeroes it) [R, C1+C2] (transpose = 0) or [C1+C2, R] (transpose = 1), row pitch ldo
//   = A[M, R]^T [B1[M, C1] | B2[M, C2]]     -- see include/cotb200.h
extern "C" int cotb200_wgrad_bf16(int M, int R, const void* A, long long lda, int C1, const void* B1, long long ldb1, int C2,
                                  const void* B2, long long ldb2, float* out, long long ldo, int transpose, void* stream) {
  if (M <= 0 || R <= 0 || C1 <= 0 || C2 < 0) { set_error("wgrad_bf16: bad dims M=%d R=%d C1=%d C2=%d", M, R, C1, C2); return COTB200_EINVAL; }
  if (!A || !B1 || !out || (C2 > 0 && !B2)) { set_error("wgrad_bf16: NULL operand"); return COTB200_ENULL; }
  if ((R & 7) || (C1 & 7) || (C2 & 7)) { set_error("wgrad_bf16: channel counts must be multiples of 8"); return COTB200_EALIGN; }
  if (C2 > 0 && (C1 & 63)) { set_error("wgrad_bf16: with two B operands C1 must be a multiple of 64"); return COTB200_EALIGN; }
  const int Cc = C1 + C2;
  if (!transpose && ((ldo & 3) || (reinterpret_cast<uintptr_t>(out) & 15))) { set_error("wgrad_bf16: OUT must be 16-byte aligned with ldo % 4 == 0"); return COTB200_EALIGN; }
  cudaStream_t st = (cudaStream_t)stream;
  WgParams p{};
  p.M = M; p.R = R; p.Cc = Cc; p.C1 = C1; p.transpose = transpose; p.ldo = ldo; p.out = out;
  const int cc64 = (Cc + 63) / 64 * 64;
  p.tiles_c = (cc64 + 255) / 256;
  p.bc = ((cc64 / 64 + p.tiles_c - 1) / p.tiles_c) * 64;       // balanced column tiles, multiples of 64, <= 256
  p.tiles_r = (R + WG_BR - 1) / WG_BR;
  p.kb_total = (M + WG_PX - 1) / WG_PX;
  const int tiles = p.tiles_r * p.tiles_c;
  int splits = (num_sms() + tiles - 1) / tiles;                // ~one CTA per SM
  const int max_splits = (p.kb_total + 3) / 4;                 // at least 4 pipeline stages (256 pixels) per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  const int per = (p.kb_total + splits - 1) / splits;
  splits = (p.kb_total + per - 1) / per;                       // no empty splits
  p.splits = splits;
  // MN blocks of 64 channels are one box (8 KB) apart = LBO; 8-pixel K groups are 1024 B apart = SBO.
  p.lbo = WG_BOX_BYTES; p.sbo = 1024;
  p.px = WG_PX; p.stages = WG_STAGES; p.stem_ho = 0;
  CUtensorMap ma, mb1, mb2;
  int rc;
  if ((rc = wg_make_map(&ma, A, M, R, lda))) return rc;
  if ((rc = wg_make_map(&mb1, B1, M, C1, ldb1))) return rc;
  if (C2 > 0) { if ((rc = wg_make_map(&mb2, B2, M, C2, ldb2))) return rc; } else mb2 = mb1;
  const int smem = WG_STAGES * (2 * WG_BOX_BYTES + (p.bc / 64) * WG_BOX_BYTES) + 1024;
  return wgrad_launch(ma, mb1, mb2, p, tiles * splits, smem, st, "tc_wgrad", 2.0 * (double)M * (R + Cc) + 4.0 * (double)R * Cc);
}


// Weight gradient of the stem convolution (cotb200_stem7x7s2_bf16), in the packed layout of its weight:
//   dWm[n, a*64 + j] += sum over output pixels (b, oh, ow) of  dY[(b, oh, ow), n] * P-window[b, oh - 2 + a, ow][j]
// P = the space-to-depth scratch image the forward call filled (B, H/2, W/2 + 4, 16).  One pipeline stage = one output row:
// the dY rows of that output row as the A operand, the four tap windows (overlapping-window TMA map) as four B boxes.
extern "C" int cotb200_stem7x7s2_wgrad_bf16(int B, int H, int W, const void* dY, long long ldy, int N, const void* scratch, float* dWm,
                                            void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || N <= 0) { set_error("stem7x7s2_wgrad: bad dims"); return COTB200_EINVAL; }
  if (!dY || !scratch || !dWm) { set_error("stem7x7s2_wgrad: NULL operand"); return COTB200_ENULL; }
  const int Hh = H / 2, Wh = W / 2;
  if ((H & 1) || (W & 1) || (Wh & 15) || Wh > 128 || (N & 7) || N > 128 || (reinterpret_cast<uintptr_t>(dWm) & 15)) {
    set_error("stem7x7s2_wgrad: geometry not supported (W/2 = %d must be a multiple of 16, <= 128; N = %d <= 128)", Wh, N);
    return COTB200_EUNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  WgParams p{};
  p.M = B * Hh * Wh; p.R = N; p.Cc = 256; p.C1 = 256; p.transpose = 0; p.ldo = 256; p.out = dWm;
  p.bc = 256; p.tiles_c = 1; p.tiles_r = 1;
  p.px = Wh; p.stem_ho = Hh;
  p.kb_total = B * Hh;
  int splits = num_sms();
  if (splits > p.kb_total) splits = p.kb_total;
  const int per = (p.kb_total + splits - 1) / splits;
  p.splits = (p.kb_total + per - 1) / per;
  const int box_bytes = 128 * p.px;
  p.lbo = box_bytes; p.sbo = 1024;
  const int stage_bytes = 6 * box_bytes;
  p.stages = (216 * 1024) / stage_bytes;
  if (p.stages > WG_STAGES) p.stages = WG_STAGES;
  if (p.stages < 2) { set_error("stem7x7s2_wgrad: row of %d pixels does not fit two pipeline stages", Wh); return COTB200_EUNSUPPORTED; }
  CUtensorMap ma, mb;
  TcEncodeTiledFn enc = tc_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return COTB200_EINVAL; }
  {
    if ((reinterpret_cast<uintptr_t>(dY) & 15) || ((ldy * 2) & 15)) { set_error("stem7x7s2_wgrad: dY not 16-byte aligned"); return COTB200_EALIGN; }
    cuuint64_t dims[2] = {(cuuint64_t)N, (cuuint64_t)p.M};
    cuuint64_t strides[1] = {(cuuint64_t)ldy * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)p.px};
    cuuint32_t es[2] = {1, 1};
    if (enc(&ma, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(dY), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(stem wgrad dY) failed"); return COTB200_EINVAL;
    }
  }
  {
    const long long Wp = Wh + 4;
    cuuint64_t dims[4] = {64, (cuuint64_t)(Wh + 1), (cuuint64_t)Hh, (cuuint64_t)B};
    cuuint64_t strides[3] = {32, (cuuint64_t)Wp * 32, (cuuint64_t)Wp * 32 * Hh};
    cuuint32_t box[4] = {64, (cuuint32_t)p.px, 1, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    if (enc(&mb, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(scratch), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(stem wgrad windows) failed"); return COTB200_EUNSUPPORTED;
    }
  }
  const int smem = p.stages * stage_bytes + 1024;
  return wgrad_launch(ma, mb, mb, p, p.splits, smem, st, "tc_stem_wgrad",
                      2.0 * (double)p.M * N + (double)B * Hh * (Wh + 4) * 32 + 4.0 * N * 256);
}
