// wgmma / TMA GEMM family for the dense contractions of the CoT block (sm_90a).
//
//   plain mode : D[M,N] = epi( A1[M,K1] * B1[N,K1]^T  (+ A2[M,K2] * B2[N,K2]^T) )
//                1x1 convolutions on NHWC activations (rows = pixels).  The optional second operand pair is the
//                concat-free form of  embed.0( cat[x, k] )  (models/cotnet.py:81,52).
//   conv mode  : 3x3 / pad 1 / stride 1 grouped convolution as an im2col-FREE implicit GEMM: for each tap the A
//                tile is a 4-D TMA box {64 ch, W, hbox, bbox} of the NHWC input fetched at the tap's (dh,dw) offset;
//                TMA's out-of-bounds zero fill IS the zero padding (key_embed.0, models/cotnet.py:44).
//   stem mode  : 7x7 / stride 2 / pad 3 convolution of a 3-channel image (models/resnet.py:552) as a 4-tap implicit GEMM over
//                the space-to-depth copy of the input made by stem_s2d_kernel: P[b, i, 2 + j, (di,dj,c)] =
//                x[b, 2i+di, 2j+dj, c], 16 channels per cell.  An output pixel's receptive field is 4 s2d rows x 4 cells x 16
//                channels; one TMA box {64 elements, tile width, 1, 1} of a tensor map whose pixel stride (32 B) is SMALLER than
//                its inner extent (128 B) fetches the overlapping 4-cell windows of a whole output row segment straight into the
//                K-major A tile -- im2col done by the TMA address generator.
//   epilogue   : per-column scale/shift (folded BatchNorm or bias), optional ReLU, bf16 store; optional per-column
//                sum / sum-of-squares of the stored bf16 values (training-mode BatchNorm statistics), summed
//                per CTA in tile order and over the CTAs in CTA order (det_finish): identical from run to run.
//
// Structure (one CTA per 128-row x BN-col tile at a time, 288 threads):
//   warps 0-7: two consumer warpgroups; warpgroup g issues the wgmma (m64n64k16, bf16 -> fp32 in registers) of rows
//              64g .. 64g + 63 of the tile and runs the epilogue of those rows
//   warp 8   : TMA producer  (cp.async.bulk.tensor -> 128B-swizzled smem stages, mbarrier complete_tx)
// All mbarrier waits are bounded (trap instead of hanging the GPU).
#include <cuda.h>
#include "common.cuh"
#include "tma.cuh"
#include "tc_wgmma.cuh"

namespace cotb200 {

static constexpr int TC_BM = 128;      // rows of a tile: two warpgroups x 64
static constexpr int TC_BK = 64;       // 64 bf16 = 128 B = one swizzle atom
static constexpr int TC_STAGES = 6;
static constexpr int TC_THREADS = 288; // two consumer warpgroups + one producer warp
static constexpr int TC_CONSUMERS = 256;
static constexpr int TC_PRODUCER_WARP = 8;

struct TcParams {
  int M, N;                 // valid rows (pixels) / output channels
  int rows_per_tile;        // D rows per CTA (128 plain; rows of the pixel box in conv mode)
  int bn;                   // N tile (multiple of 64, <= 256)
  int mode;                 // 0 plain, 1 conv3x3, 2 stem (row-window conv)
  int kb1, kb2;             // plain: 64-wide k-blocks of operand pair 1 / 2
  int H, W, B, hbox, bbox;  // conv geometry
  int kc;                   // conv: 64-channel chunks per tap (= bn / 64)
  int wtiles;               // stem: tiles per output row (tile width = rows_per_tile)
  int relu;
  int m_tiles;              // number of row tiles (persistent CTAs loop over m_tiles * n_tiles)
  int stages;               // smem ring depth actually used (<= TC_STAGES): short K loops take less smem -> more CTAs/SM
  long long ldd;            // D row pitch (elements)
  __nv_bfloat16* D;
  const float* scale;       // [N] or null (=1)
  const float* shift;       // [N] or null (=0)
  float* col_sum;           // [N] or null
  float* col_sqsum;         // [N] or null
  int rows_per_sample;      // > 0: col_sum / col_sqsum are PER SAMPLE, [M / rows_per_sample, N] (GroupNorm statistics of the logits)
  DetArena det;             // column statistics: per-CTA totals leave through det_finish (common.cuh)
};

// Writes one 64-column chunk of a warpgroup's accumulators (rows row0 .. row0 + 63 of the staging image) as bf16 after
// scale / shift / ReLU into a 128B-swizzled [rows][128 B] slab.  sc / sh point at the chunk's 64 column constants.
__device__ __forceinline__ void stage_chunk_bf16(const float (&acc)[32], uint32_t buf, int row0, const float* sc, const float* sh,
                                                 int relu) {
  const int lane = threadIdx.x & 31, wl = (threadIdx.x >> 5) & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + wl * 16 + (lane >> 2) + 8 * h;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int col = i * 8 + 2 * (lane & 3);
      float lo = fmaf(acc[4 * i + 2 * h], sc[col], sh[col]);
      float hi = fmaf(acc[4 * i + 2 * h + 1], sc[col + 1], sh[col + 1]);
      if (relu) { lo = fmaxf(lo, 0.f); hi = fmaxf(hi, 0.f); }
      __nv_bfloat162 h2 = __floats2bfloat162_rn(lo, hi);
      const uint32_t dst = buf + (uint32_t)(row * 128 + ((i ^ (row & 7)) << 4) + (lane & 3) * 4);
      asm volatile("st.shared.u32 [%0], %1;" ::"r"(dst), "r"(*reinterpret_cast<uint32_t*>(&h2)) : "memory");
    }
  }
}

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------- kernel
// Persistent: every CTA loops over output tiles.  The TMA producer runs ahead through a shared-memory ring (full/empty
// mbarriers, continuous across tiles), so the operands of tile i+1 arrive while the consumer warpgroups run the epilogue of
// tile i.  (One CTA per tile pays the fixed per-CTA cost -- barrier init, a cold TMA round trip -- on every tile, which
// dominates tiles with 1-2 k-blocks.)
__device__ __forceinline__ void tc_tile_origin(const TcParams& p, int tile_m, int& b0, int& h0, int& w0, long long& m0, int& rows_valid) {
  b0 = 0; h0 = 0; w0 = 0;
  if (p.mode == 0) {
    m0 = (long long)tile_m * TC_BM;
    rows_valid = (int)min((long long)TC_BM, (long long)p.M - m0);
  } else if (p.mode == 2) {                       // stem: tile = (sample, output row, segment of the row); H, W = OUTPUT dims
    const int per_b = p.H * p.wtiles;
    b0 = tile_m / per_b;
    const int rem = tile_m - b0 * per_b;
    h0 = rem / p.wtiles; w0 = (rem - h0 * p.wtiles) * p.rows_per_tile;
    m0 = ((long long)b0 * p.H + h0) * p.W + w0;
    rows_valid = p.rows_per_tile;
  } else if (p.bbox == 1) {
    const int tps = (p.H + p.hbox - 1) / p.hbox;
    b0 = tile_m / tps; h0 = (tile_m % tps) * p.hbox;
    m0 = ((long long)b0 * p.H + h0) * p.W;
    rows_valid = min(p.hbox, p.H - h0) * p.W;
  } else {
    b0 = tile_m * p.bbox;
    m0 = (long long)b0 * p.H * p.W;
    rows_valid = min(p.bbox, p.B - b0) * p.H * p.W;
  }
}

// MAXCH = most 64-column chunks of an N tile (accumulator registers per thread = 32 * MAXCH); MINB = CTAs per SM
template <int MAXCH, int MINB>
__global__ void __launch_bounds__(TC_THREADS, MINB)
tc_gemm_kernel(const __grid_constant__ CUtensorMap mapA1, const __grid_constant__ CUtensorMap mapB1,
               const __grid_constant__ CUtensorMap mapA2, const __grid_constant__ CUtensorMap mapB2,
               const __grid_constant__ CUtensorMap mapD, const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int a_bytes = TC_BM * TC_BK * 2;             // 16 KB
  const int b_bytes = p.bn * TC_BK * 2;
  const int stage_bytes = a_bytes + ((b_bytes + 1023) & ~1023);
  uint8_t* out_tile = smem + (size_t)p.stages * stage_bytes;      // two [128 rows][128 B] slabs, 128B-swizzled
  __shared__ __align__(8) uint64_t s_full[TC_STAGES], s_empty[TC_STAGES];
  // per row-group partials of the tile's column statistics: [4][256] floats each, in DYNAMIC shared memory behind the two slab
  // buffers and only when statistics are requested (static tables would cost every launch its second resident CTA)
  float (*s_sum)[256] = reinterpret_cast<float (*)[256]>(out_tile + 2 * TC_BM * 128);
  float (*s_sq)[256] = s_sum + 4;
  float* s_tot = &s_sq[4][0];                        // [2][N]: the CTA's column sums / sums of squares over all its tiles
  __shared__ __align__(16) float s_scale[256], s_shift[256];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = p.mode == 1 ? 9 * p.kc : p.kb1 + p.kb2;
  const int n_tiles = (p.N + p.bn - 1) / p.bn;
  const int total_tiles = p.m_tiles * n_tiles;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA1) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB1) : "memory");
    for (int s = 0; s < TC_STAGES; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), 2); }
    mbar_init_fence();
  }
  if (p.col_sum != nullptr && p.rows_per_sample == 0) {
    for (int i = threadIdx.x; i < 4 * 256; i += TC_THREADS) { (&s_sum[0][0])[i] = 0.f; (&s_sq[0][0])[i] = 0.f; }
    for (int i = threadIdx.x; i < 2 * p.N; i += TC_THREADS) s_tot[i] = 0.f;
  }
  __syncthreads();

  if (warp == TC_PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int kbc = 0;                                      // k-block counter, continuous across tiles
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int tile_m = tile / n_tiles, n0 = (tile % n_tiles) * p.bn;      // N tiles of one row tile are neighbours: its A tile stays in L2
        int b0, h0, w0, rows_valid; long long m0;
        tc_tile_origin(p, tile_m, b0, h0, w0, m0, rows_valid);
        for (int kb = 0; kb < nkb; ++kb, ++kbc) {
          const int s = kbc % p.stages;
          const uint32_t ph = (kbc / p.stages) & 1;
          mbar_wait(smem_u32(&s_empty[s]), ph ^ 1);
          const uint32_t full = smem_u32(&s_full[s]);
          const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes), sb = sa + a_bytes;
          // TMA counts the whole box (zero-filled elements included): conv boxes hold rows_per_tile <= 128 rows
          mbar_expect_tx(full, (uint32_t)(p.rows_per_tile * TC_BK * 2 + b_bytes));
          if (p.mode == 0) {
            if (kb < p.kb1) {
              tma_load_2d(sa, &mapA1, full, kb * TC_BK, (int)m0);
              tma_load_2d(sb, &mapB1, full, kb * TC_BK, n0);
            } else {
              tma_load_2d(sa, &mapA2, full, (kb - p.kb1) * TC_BK, (int)m0);
              tma_load_2d(sb, &mapB2, full, (kb - p.kb1) * TC_BK, n0);
            }
          } else if (p.mode == 2) {
            // A: the 4-cell windows of output pixels w0 .. w0 + tile width of s2d row h0 - 2 + kb (rows outside the image: zero fill)
            tma_load_4d(sa, &mapA1, full, 0, w0, h0 - 2 + kb, b0);
            tma_load_2d(sb, &mapB1, full, kb * TC_BK, n0);
          } else {
            const int tap = kb / p.kc, cc = kb % p.kc;
            const int dh = tap / 3 - 1, dw = tap % 3 - 1;
            // A: 4-D box {64 ch, W, hbox, bbox}; negative / overflowing coordinates are zero-filled == zero padding
            tma_load_4d(sa, &mapA1, full, n0 + cc * TC_BK, dw, h0 + dh, b0);
            tma_load_2d(sb, &mapB1, full, kb * TC_BK, n0);
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma main loop + epilogue (rows 64 wg .. 64 wg + 63 of each tile) =====================
  // Epilogue: registers -> (scale/shift/ReLU, bf16) -> 128B-swizzled smem SLAB of 64 columns x 128 rows -> one TMA store per
  // slab.  Two slab buffers alternate, so the store of slab i overlaps the conversion of slab i+1 and the staging area is 32 KB
  // whatever the N tile.  BatchNorm statistics are taken from the staged bf16 slab (what the normalisation will read back), one
  // column pair per thread of the first warpgroup.
  const int wg = warp >> 2;
  const int et = threadIdx.x;                          // 0..255 among the consumer threads
  const bool stats = p.col_sum != nullptr;
  const uint32_t out_base = smem_u32(out_tile);
  const int nch = p.bn / 64;
  int kbc = 0, last_n0 = -1;
  uint32_t slab_ctr = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int tile_m = tile / n_tiles, n0 = (tile % n_tiles) * p.bn;
    int b0, h0, w0, rows_valid; long long m0;
    tc_tile_origin(p, tile_m, b0, h0, w0, m0, rows_valid);
    if (n0 != last_n0) {                               // per-column epilogue constants of this N tile -> smem
      for (int j = et; j < p.bn; j += TC_CONSUMERS) {
        const bool in = n0 + j < p.N;
        s_scale[j] = (p.scale && in) ? __ldg(p.scale + n0 + j) : 1.f;
        s_shift[j] = (p.shift && in) ? __ldg(p.shift + n0 + j) : 0.f;
      }
      last_n0 = n0;
    }
    float acc[MAXCH][32];
    int prev_s = 0;
    for (int kb = 0; kb < nkb; ++kb, ++kbc) {
      const int s = kbc % p.stages;
      const uint32_t ph = (kbc / p.stages) & 1;
      mbar_wait(smem_u32(&s_full[s]), ph);
      const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes) + (uint32_t)wg * (64u * 128u), sb = smem_u32(smem + (size_t)s * stage_bytes) + a_bytes;
      const uint64_t da = wgmma_desc_sw128(sa), db = wgmma_desc_sw128(sb);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) {
        // advance 16 bf16 = 32 B inside the 128 B swizzle atom: start-address field += 2; N chunks are 64 rows = 8 KB apart
#pragma unroll
        for (int c = 0; c < MAXCH; ++c)
          if (c < nch) wgmma_m64n64k16<0, 0>(acc[c], da + 2 * k, db + (uint64_t)(c * 512) + 2 * k, (kb | k) != 0);
      }
      wgmma_commit();
      if (kb > 0) {                                    // the MMAs of the previous stage have retired: hand it back to the producer
        wgmma_wait<1>();
        if ((et & 127) == 0) mbar_arrive(smem_u32(&s_empty[prev_s]));
      }
      prev_s = s;
    }
    wgmma_wait<0>();
    if ((et & 127) == 0) mbar_arrive(smem_u32(&s_empty[prev_s]));
#pragma unroll
    for (int c = 0; c < MAXCH; ++c) if (c < nch) wgmma_fence_acc(acc[c]);

#pragma unroll
    for (int sl = 0; sl < MAXCH; ++sl) {
      if (sl >= nch) break;
      const uint32_t buf = out_base + (slab_ctr & 1u) * (uint32_t)(TC_BM * 128);
      ++slab_ctr;
      // the store that read this buffer two slabs ago must have finished READING it (at most the latest group may be pending)
      if (et == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      consumer_bar();
      stage_chunk_bf16(acc[sl], buf, wg * 64, &s_scale[sl * 64], &s_shift[sl * 64], p.relu);
      // make the generic-proxy smem writes visible to the async proxy, then one thread issues the bulk tensor store
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      consumer_bar();
      if (et == 0) {
        if (n0 + sl * 64 < p.N)
          asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                       ::"l"(&mapD), "r"(buf), "r"(n0 + sl * 64), "r"((int)m0) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
      if (stats && p.rows_per_sample > 0 && et < 128) {
        // PER-SAMPLE column sums of the staged slab (GroupNorm over the 9 taps x H x W of one sample, models/cotnet.py:56): a row
        // group of 32 rows touches at most two samples (rows_per_sample >= 32 is checked on the host); two partial sets per
        // thread, straight to the [sample, column] tables
        const int tp = et & 31, rg = et >> 5;
        if (sl * 64 + 2 * tp < p.bn && n0 + sl * 64 + 2 * tp < p.N) {
          const long long row0 = m0 + rg * 32;
          const int s_lo = (int)(row0 / p.rows_per_sample);
          const int rb = (int)min((long long)32, (long long)(s_lo + 1) * p.rows_per_sample - row0);   // rows [0, rb) belong to sample s_lo
          const int nrow = min(32, min(rows_valid, (int)min((long long)TC_BM, p.M - m0)) - rg * 32);
          const __nv_bfloat16 one = one_of<__nv_bfloat16>();
          float sa[2] = {0.f, 0.f}, qa[2] = {0.f, 0.f}, sb[2] = {0.f, 0.f}, qb[2] = {0.f, 0.f};
          uint32_t w2[32];
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {
            const int row = rg * 32 + rr;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w2[rr]) : "r"(buf + (uint32_t)(row * 128 + (((tp >> 2) ^ (row & 7)) << 4) + (tp & 3) * 4)));
          }
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {
            if (rr < nrow) {
              const __nv_bfloat16 lo = __ushort_as_bfloat16((unsigned short)(w2[rr] & 0xFFFFu)), hi = __ushort_as_bfloat16((unsigned short)(w2[rr] >> 16));
              const int h = rr < rb ? 0 : 1;
              if (h == 0) { sa[0] = mfma<__nv_bfloat16>(lo, one, sa[0]); qa[0] = mfma<__nv_bfloat16>(lo, lo, qa[0]);
                            sb[0] = mfma<__nv_bfloat16>(hi, one, sb[0]); qb[0] = mfma<__nv_bfloat16>(hi, hi, qb[0]); }
              else        { sa[1] = mfma<__nv_bfloat16>(lo, one, sa[1]); qa[1] = mfma<__nv_bfloat16>(lo, lo, qa[1]);
                            sb[1] = mfma<__nv_bfloat16>(hi, one, sb[1]); qb[1] = mfma<__nv_bfloat16>(hi, hi, qb[1]); }
            }
          }
          const int col = n0 + sl * 64 + 2 * tp;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if ((h == 0 && nrow > 0) || (h == 1 && nrow > rb)) {
              const long long srow = (long long)(s_lo + h) * p.N + col;
              atomicAdd(p.col_sum + srow, sa[h]); atomicAdd(p.col_sqsum + srow, qa[h]);
              if (col + 1 < p.N) { atomicAdd(p.col_sum + srow + 1, sb[h]); atomicAdd(p.col_sqsum + srow + 1, qb[h]); }
            }
          }
        }
      }
      if (stats && p.rows_per_sample == 0 && et < 128) {
        // column sums of the staged slab: thread = (column pair tp, row group rg of 32 rows); a warp reads one whole 128-byte
        // row per step (conflict-free under the swizzle)
        const int tp = et & 31, rg = et >> 5;
        if (sl * 64 + 2 * tp < p.bn) {
          float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
          const __nv_bfloat16 one = one_of<__nv_bfloat16>();
          const int nrow = min(32, min(rows_valid, (int)min((long long)TC_BM, p.M - m0)) - rg * 32);      // valid rows of this row group
          uint32_t w2[32];
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {               // all loads first (independent), then the arithmetic
            const int row = rg * 32 + rr;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w2[rr]) : "r"(buf + (uint32_t)(row * 128 + (((tp >> 2) ^ (row & 7)) << 4) + (tp & 3) * 4)));
          }
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {
            if (rr < nrow) {
              const __nv_bfloat16 lo = __ushort_as_bfloat16((unsigned short)(w2[rr] & 0xFFFFu)), hi = __ushort_as_bfloat16((unsigned short)(w2[rr] >> 16));
              s0 = mfma<__nv_bfloat16>(lo, one, s0); q0 = mfma<__nv_bfloat16>(lo, lo, q0);
              s1 = mfma<__nv_bfloat16>(hi, one, s1); q1 = mfma<__nv_bfloat16>(hi, hi, q1);
            }
          }
          // one owner per (row group, column): plain stores, no atomics; every column of the tile is written once per tile
          s_sum[rg][sl * 64 + 2 * tp] = s0; s_sq[rg][sl * 64 + 2 * tp] = q0;
          s_sum[rg][sl * 64 + 2 * tp + 1] = s1; s_sq[rg][sl * 64 + 2 * tp + 1] = q1;
        }
      }
    }
    if (stats && p.rows_per_sample == 0) {
      consumer_bar();                                  // every thread's shared-memory partials are in
      for (int j = et; j < p.bn; j += TC_CONSUMERS) {  // one owner per column: the CTA's totals add up in tile order
        if (n0 + j < p.N) {
          s_tot[n0 + j] += (s_sum[0][j] + s_sum[1][j]) + (s_sum[2][j] + s_sum[3][j]);
          s_tot[p.N + n0 + j] += (s_sq[0][j] + s_sq[1][j]) + (s_sq[2][j] + s_sq[3][j]);
        }
      }
    }
  }
  if (et == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");     // all stores complete before the CTA exits
  if (stats && p.rows_per_sample == 0) {
    consumer_bar();
    const int n = 2 * p.N;
    for (int i = et; i < n; i += TC_CONSUMERS) p.det.scr[(size_t)blockIdx.x * n + i] = s_tot[i];
    det_finish<true>(p.det.scr, n, blockIdx.x, gridDim.x, p.det.tick, et, TC_CONSUMERS, [&](int k, float t) {
      if (k < p.N) p.col_sum[k] += t; else p.col_sqsum[k - p.N] += t;
    });
  }
}

// ---------------------------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D bf16 row-major [rows, cols] with pitch ld (elements); box {64, box_rows}, 128B swizzle, zero OOB fill
static int make_map_2d(CUtensorMap* m, const void* base, long long rows, long long cols, long long ld, int box_rows) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return COTB200_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || ((ld * 2) & 15)) { set_error("TMA operand not 16-byte aligned (ld=%lld)", ld); return COTB200_EALIGN; }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(2d) failed: %d", (int)r); return COTB200_EINVAL; }
  return 0;
}

// 4-D NHWC bf16 activation [B,H,W,C] (pixel pitch ldc); box {64, W, hbox, bbox}
static int make_map_nhwc(CUtensorMap* m, const void* base, int B, int H, int W, int C, long long ldc, int hbox, int bbox) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return COTB200_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || ((ldc * 2) & 15)) { set_error("TMA operand not 16-byte aligned"); return COTB200_EALIGN; }
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)ldc * 2, (cuuint64_t)ldc * 2 * W, (cuuint64_t)ldc * 2 * W * H};
  cuuint32_t box[4] = {(cuuint32_t)TC_BK, (cuuint32_t)W, (cuuint32_t)hbox, (cuuint32_t)bbox};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(4d) failed: %d", (int)r); return COTB200_EINVAL; }
  return 0;
}

static int tc_launch(const CUtensorMap& a1, const CUtensorMap& b1, const CUtensorMap& a2, const CUtensorMap& b2,
                     TcParams p, int m_tiles, cudaStream_t st, const char* what, double alg_bytes) {
  // output tile staged in smem for the TMA store: one 128-row x 128-byte slab per 64 output columns
  CUtensorMap dmap;
  int rcd = make_map_2d(&dmap, p.D, p.M, p.N, p.ldd, p.rows_per_tile);
  if (rcd) return rcd;
  // two slab buffers (+ statistics partials of a tile and the CTA's column totals)
  const int out_bytes = 2 * TC_BM * 128 + ((p.col_sum && p.rows_per_sample == 0) ? 2 * 4 * 256 * 4 + 2 * p.N * 4 : 0);
  const int a_bytes = TC_BM * TC_BK * 2, b_bytes = p.bn * TC_BK * 2;
  const int stage_bytes = a_bytes + ((b_bytes + 1023) & ~1023);
  p.m_tiles = m_tiles;
  // two CTAs per SM (two epilogue teams, two producers) when N tiles of <= 128 columns keep the accumulators of a consumer thread
  // at <= 64 registers and at least 2 stages fit next to each other; else one CTA with as many stages as the ring supports
  int per_sm = 2;
  p.stages = (104 * 1024 - out_bytes) / stage_bytes;
  if (p.stages < 2 || p.bn > 128) {
    per_sm = 1;
    p.stages = (200 * 1024 - out_bytes) / stage_bytes;
  }
  if (p.stages > TC_STAGES) p.stages = TC_STAGES;
  if (p.stages < 2) p.stages = 2;
  const int smem = p.stages * stage_bytes + out_bytes + 1024;
  static PerDevFlag configured_d;
  if (bool& configured = configured_d.get(); !configured) {
    cudaError_t e = cudaFuncSetAttribute(tc_gemm_kernel<2, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_gemm_kernel<4, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 204 * 1024);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
    configured = true;
  }
  const int total = m_tiles * ((p.N + p.bn - 1) / p.bn);
  int grid = per_sm * num_sms();                          // resident CTAs only: a second wave would start from a cold pipeline
  if (grid > total) grid = total;
  DetScratch ds;
  if (p.col_sum && p.rows_per_sample == 0) {
    if (p.N > 4096) { set_error("%s: N=%d too wide for the statistics epilogue", what, p.N); return COTB200_EUNSUPPORTED; }
    int rcs = ds.alloc(det_floats(grid, 2 * p.N), 1, st);
    if (rcs) return rcs;
    p.det = ds.a;
  }
  COTB200_PROF_B(what, alg_bytes);
  if (per_sm == 2) tc_gemm_kernel<2, 2><<<grid, TC_THREADS, smem, st>>>(a1, b1, a2, b2, dmap, p);
  else tc_gemm_kernel<4, 1><<<grid, TC_THREADS, smem, st>>>(a1, b1, a2, b2, dmap, p);
  return check_launch(what);
}

static int pick_bn_wide(int N);
static int pick_bn(int N, int K = 1 << 30) {
  // short contractions (K <= 128) with a wide output are epilogue-bound: the operands of a 256-column tile arrive in a fraction
  // of the time its epilogue takes.  Two CTAs per SM with 128-column tiles run two epilogues side by side (the re-read A tile is
  // small and comes from L2).
  if (K <= 128 && N > 128) {
    const int parts = (N + 127) / 128;
    const int bn = (((N + parts - 1) / parts) + 63) & ~63;
    return bn > 128 ? 128 : bn;
  }
  return pick_bn_wide(N);
}
static int pick_bn_wide(int N) {
  // bn is a multiple of 64 (whole n64 wgmma chunks; every 64-column store slab lies inside its own tile), <= 256: rows of B
  // beyond N are zero-filled by the TMA and columns of D beyond N are clipped by the TMA store.
  const int parts = (N + 255) / 256;
  const int bn = (((N + parts - 1) / parts) + 63) & ~63;
  return bn > 256 ? 256 : bn;
}

// ---------------------------------------------------------------------------------------------- 3x3 conv, haloed-tile kernel
// conv mode of tc_gemm_kernel fetches one pixel box PER TAP: every input pixel travels L2 -> shared memory nine times and the
// kernel is L2-bound.  Here a CTA loads ONE haloed tile {64 ch, W+2, R+2} of the NHWC input per work item (TMA out-of-bounds
// fill = zero padding on all four sides) and the nine taps are nine wgmma A-descriptors INTO THAT TILE: with the output pixels
// enumerated in padded coordinates q = r*(W+2) + c, the A rows of tap (dh, dw) are the smem rows q + (dh+1)*(W+2) + (dw+1) -- a
// contiguous row range, i.e. the same K-major SW128 descriptor with a start address moved by a whole number of 128-byte rows (the
// 128B swizzle is a function of the absolute shared memory address, which is how TMA wrote the tile).  Outputs with c >= W are
// garbage columns that are never stored.
//   * weights of the CTA's 64 output channels (9 taps x 64 x 64, 72 KB) stay resident in shared memory: CTAs are bound to one
//     N tile, work items of that N tile are strided over the CTAs bound to it;
//   * accumulators: MB <= 2 M-blocks of 128 padded pixels x 64 columns; warpgroup g owns rows 64g .. 64g + 63 of each M-block;
//   * epilogue: registers -> scale/shift/ReLU -> bf16 -> compacted (garbage columns dropped) 128B-swizzled image of the R x W
//     output pixels -> ONE TMA store; BatchNorm column statistics from the staged image, accumulated in registers over ALL work
//     items of the CTA (its N tile never changes) and leaving through one deterministic reduction (det_finish).
// Geometry: bn = 64 (kc = 1), R | H, R*(W+2) <= 256.  Everything else stays on conv mode of tc_gemm_kernel.
struct HcParams {
  int B, H, W, C, R, MB, Wp, n_tiles, bands, items;   // items = B * bands work items per N tile
  int a_stage_bytes, stages, box_bytes, relu;
  const float* scale; const float* shift; float* col_sum; float* col_sqsum;
  DetArena det;
};

static constexpr int HC_WBYTES = 9 * 64 * 128;          // resident weights of one N tile

__global__ void __launch_bounds__(TC_THREADS, 1)
tc_conv3x3_halo_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapW,
                       const __grid_constant__ CUtensorMap mapD, const HcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* w_s = smem;                                               // [9][64 rows][128 B] SW128
  uint8_t* a_s = smem + HC_WBYTES;                                    // stages x haloed tile
  uint8_t* o_s = a_s + (size_t)p.stages * p.a_stage_bytes;           // [R*W rows][128 B] SW128 compacted output image
  __shared__ __align__(8) uint64_t s_full[4], s_empty[4], s_wfull;
  __shared__ __align__(16) float s_scale[64], s_shift[64];
  __shared__ float s_part[2][4][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = blockIdx.x % p.n_tiles, n0 = nt * 64;
  const int first = blockIdx.x / p.n_tiles, step = gridDim.x / p.n_tiles;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapX) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
    for (int s = 0; s < 4; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), 2); }
    mbar_init(smem_u32(&s_wfull), 1);
    mbar_init_fence();
  }
  if (threadIdx.x < 64) {
    s_scale[threadIdx.x] = p.scale ? __ldg(p.scale + n0 + threadIdx.x) : 1.f;
    s_shift[threadIdx.x] = p.shift ? __ldg(p.shift + n0 + threadIdx.x) : 0.f;
  }
  __syncthreads();

  if (warp == TC_PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      const uint32_t wf = smem_u32(&s_wfull);
      mbar_expect_tx(wf, HC_WBYTES);
      for (int t = 0; t < 9; ++t) tma_load_2d(smem_u32(w_s + t * 8192), &mapW, wf, t * 64, n0);
      int it = 0;
      for (int m = first; m < p.items; m += step, ++it) {
        const int s = it % p.stages;
        const uint32_t ph = (it / p.stages) & 1;
        const int b = m / p.bands, h0 = (m - b * p.bands) * p.R;
        mbar_wait(smem_u32(&s_empty[s]), ph ^ 1);
        const uint32_t full = smem_u32(&s_full[s]);
        mbar_expect_tx(full, (uint32_t)p.box_bytes);
        tma_load_4d(smem_u32(a_s + (size_t)s * p.a_stage_bytes), &mapX, full, n0, -1, h0 - 1, b);
      }
    }
    return;
  }

  // ===================== consumers: nine-tap wgmma + epilogue =====================
  const int wg = warp >> 2, wl = warp & 3;
  const int et = threadIdx.x;
  const bool stats = p.col_sum != nullptr;
  const uint32_t ob = smem_u32(o_s);
  const uint32_t wb = smem_u32(w_s);
  const int RW = p.R * p.W;
  const int tp = et & 31, rg = (et >> 5) & 3;
  float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;                     // statistics of columns 2tp, 2tp+1 over rows rg, rg+4, ... (et < 128)
  mbar_wait(smem_u32(&s_wfull), 0);
  int it = 0;
  for (int m = first; m < p.items; m += step, ++it) {
    const int s = it % p.stages;
    const uint32_t ph = (it / p.stages) & 1;
    const int b = m / p.bands, h0 = (m - b * p.bands) * p.R;
    mbar_wait(smem_u32(&s_full[s]), ph);
    const uint32_t ab = smem_u32(a_s + (size_t)s * p.a_stage_bytes);
    float acc[2][32];
    wgmma_fence();
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
      if (mb < p.MB) {
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const int row = mb * 128 + wg * 64 + (t / 3) * p.Wp + (t % 3);  // first smem row of this tap's A operand
          const uint64_t da = wgmma_desc_sw128(ab + (uint32_t)row * 128u);
          const uint64_t db = wgmma_desc_sw128(wb + (uint32_t)t * 8192u);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64n64k16<0, 0>(acc[mb], da + 2 * k, db + 2 * k, (t | k) != 0);
        }
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    if ((et & 127) == 0) mbar_arrive(smem_u32(&s_empty[s]));      // haloed tile consumed
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) if (mb < p.MB) wgmma_fence_acc(acc[mb]);
    // the previous item's store must have finished READING the staging image
    if (et == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    consumer_bar();
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
      if (mb < p.MB) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int q = mb * 128 + wg * 64 + wl * 16 + (lane >> 2) + 8 * h;   // padded output pixel
          const int ro = q / p.Wp, co = q - ro * p.Wp;
          if (ro < p.R && co < p.W) {
            const int prow = ro * p.W + co;                            // row of the compacted image
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int col = i * 8 + 2 * (lane & 3);
              float lo = fmaf(acc[mb][4 * i + 2 * h], s_scale[col], s_shift[col]);
              float hi = fmaf(acc[mb][4 * i + 2 * h + 1], s_scale[col + 1], s_shift[col + 1]);
              if (p.relu) { lo = fmaxf(lo, 0.f); hi = fmaxf(hi, 0.f); }
              __nv_bfloat162 h2 = __floats2bfloat162_rn(lo, hi);
              const uint32_t dst = ob + (uint32_t)(prow * 128 + ((i ^ (prow & 7)) << 4) + (lane & 3) * 4);
              asm volatile("st.shared.u32 [%0], %1;" ::"r"(dst), "r"(*reinterpret_cast<uint32_t*>(&h2)) : "memory");
            }
          }
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    consumer_bar();
    if (et == 0) {
      const int m0 = (b * p.H + h0) * p.W;
      asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                   ::"l"(&mapD), "r"(ob), "r"(n0), "r"(m0) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    if (stats && et < 128) {
      const __nv_bfloat16 one = one_of<__nv_bfloat16>();
      for (int r0 = rg; r0 < RW; r0 += 32) {                       // 8 rows per batch: loads first, then the arithmetic
        uint32_t w2[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int row = r0 + 4 * u;
          w2[u] = 0u;
          if (row < RW) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w2[u]) : "r"(ob + (uint32_t)(row * 128 + (((tp >> 2) ^ (row & 7)) << 4) + (tp & 3) * 4)));
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const __nv_bfloat16 lo = __ushort_as_bfloat16((unsigned short)(w2[u] & 0xFFFFu)), hi = __ushort_as_bfloat16((unsigned short)(w2[u] >> 16));
          s0 = mfma<__nv_bfloat16>(lo, one, s0); q0 = mfma<__nv_bfloat16>(lo, lo, q0);
          s1 = mfma<__nv_bfloat16>(hi, one, s1); q1 = mfma<__nv_bfloat16>(hi, hi, q1);
        }
      }
    }
  }
  if (et == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  if (stats) {
    if (et < 128) {
      s_part[0][rg][2 * tp] = s0; s_part[0][rg][2 * tp + 1] = s1;
      s_part[1][rg][2 * tp] = q0; s_part[1][rg][2 * tp + 1] = q1;
    }
    consumer_bar();
    // the CTA's row of the deterministic reduction: its 64 columns' totals, zeros for the other N tiles
    const int n = 2 * p.C;
    for (int i = et; i < n; i += TC_CONSUMERS) {
      const int pl = i < p.C ? 0 : 1, c = i - pl * p.C;
      float v = 0.f;
      if (c >= n0 && c < n0 + 64) v = (s_part[pl][0][c - n0] + s_part[pl][1][c - n0]) + (s_part[pl][2][c - n0] + s_part[pl][3][c - n0]);
      p.det.scr[(size_t)blockIdx.x * n + i] = v;
    }
    det_finish<true>(p.det.scr, n, blockIdx.x, gridDim.x, p.det.tick, et, TC_CONSUMERS, [&](int k, float t) {
      if (k < p.C) p.col_sum[k] += t; else p.col_sqsum[k - p.C] += t;
    });
  }
}

// returns 1 when the haloed-tile kernel took the convolution (*rc = status), 0 when conv mode of tc_gemm_kernel should run
static int conv3x3_halo_launch(int B, int H, int W, int C, const void* X, long long ldx, const void* Wp, int bn, void* D, long long ldd,
                               const float* scale, const float* shift, int relu, float* col_sum, float* col_sqsum, cudaStream_t st, int* rc) {
  static int mode = -2;                       // COTB200_CONV_HALO: 0 = off, 1 (default) = on
  if (mode == -2) { const char* e = getenv("COTB200_CONV_HALO"); mode = e ? atoi(e) : 1; }
  if (mode <= 0 || bn != 64 || C % 64 || W + 2 > 256 || ldx != C || ldd != C) return 0;
  const int Wpad = W + 2;
  static int maxpx = -1;                      // COTB200_HALO_MAXPX: padded output pixels per work item (128 -> one M block, more ring stages)
  if (maxpx < 0) { const char* e = getenv("COTB200_HALO_MAXPX"); maxpx = e ? atoi(e) : 256; if (maxpx < 128) maxpx = 128; if (maxpx > 256) maxpx = 256; }
  int R = 0;
  for (int r = 1; r <= H; ++r) if (H % r == 0 && r * Wpad <= maxpx && r * W <= 256) R = r;
  if (R == 0) return 0;
  HcParams p{};
  p.B = B; p.H = H; p.W = W; p.C = C; p.R = R; p.Wp = Wpad; p.MB = (R * Wpad + 127) / 128;
  p.n_tiles = C / 64; p.bands = H / R; p.items = B * p.bands;
  if (p.n_tiles > num_sms()) return 0;
  const int a_rows = max((R + 2) * Wpad, p.MB * 128 + 2 * Wpad + 2);
  p.a_stage_bytes = (a_rows * 128 + 1023) & ~1023;
  p.box_bytes = (R + 2) * Wpad * 128;
  const int out_bytes = (R * W * 128 + 1023) & ~1023;
  p.stages = (220 * 1024 - HC_WBYTES - out_bytes) / p.a_stage_bytes;
  if (p.stages > 4) p.stages = 4;
  if (p.stages < 2) return 0;
  p.relu = relu;
  p.scale = scale; p.shift = shift; p.col_sum = col_sum; p.col_sqsum = col_sqsum;
  CUtensorMap mx, mw, md;
  EncodeTiledFn enc = encode_fn();
  if (!enc) return 0;
  {
    if ((reinterpret_cast<uintptr_t>(X) & 15) || (reinterpret_cast<uintptr_t>(D) & 15)) return 0;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)C * 2 * W, (cuuint64_t)C * 2 * W * H};
    cuuint32_t box[4] = {64, (cuuint32_t)Wpad, (cuuint32_t)(R + 2), 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    if (enc(&mx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(X), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) return 0;
  }
  if (make_map_2d(&mw, Wp, C, 9LL * 64, 9LL * 64, 64)) return 0;
  if (make_map_2d(&md, D, (long long)B * H * W, C, ldd, R * W)) return 0;
  const int smem = HC_WBYTES + p.stages * p.a_stage_bytes + out_bytes + 1024;
  static PerDevFlag configured_d;
  if (bool& configured = configured_d.get(); !configured) {
    cudaError_t e = cudaFuncSetAttribute(tc_conv3x3_halo_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(conv halo): %s", cudaGetErrorString(e)); *rc = (int)e; return 1; }
    configured = true;
  }
  int grid = (num_sms() / p.n_tiles) * p.n_tiles;
  if (grid > p.items * p.n_tiles) grid = p.items * p.n_tiles;
  DetScratch ds;
  if (col_sum) {
    if ((*rc = ds.alloc(det_floats(grid, 2 * C), 1, st))) return 1;
    p.det = ds.a;
  }
  COTB200_PROF_B("tc_conv3x3_halo", 2.0 * (2.0 * (double)B * H * W * C + 9.0 * (double)C * 64));
  tc_conv3x3_halo_kernel<<<grid, TC_THREADS, smem, st>>>(mx, mw, md, p);
  *rc = check_launch("tc_conv3x3_halo");
  return 1;
}

}  // namespace cotb200

using namespace cotb200;

// D[M,N] = epi(A1 B1^T + A2 B2^T), all bf16 row-major; see include/cotb200.h
extern "C" int cotb200_gemm_bf16(int M, int N, int K1, const void* A1, long long lda1, const void* B1, long long ldb1,
                                 int K2, const void* A2, long long lda2, const void* B2, long long ldb2, void* D,
                                 long long ldd, const float* scale, const float* shift, int relu, float* col_sum,
                                 float* col_sqsum, void* stream) {
  if (M <= 0 || N <= 0 || K1 <= 0 || K2 < 0) { set_error("gemm_bf16: bad dims M=%d N=%d K1=%d K2=%d", M, N, K1, K2); return COTB200_EINVAL; }
  if (!A1 || !B1 || !D || (K2 > 0 && (!A2 || !B2))) { set_error("gemm_bf16: NULL operand"); return COTB200_ENULL; }
  if ((N & 7) || (K1 & 7) || (K2 & 7) || (ldd & 7)) { set_error("gemm_bf16: N, K, ldd must be multiples of 8"); return COTB200_EALIGN; }
  if ((col_sum == nullptr) != (col_sqsum == nullptr)) { set_error("gemm_bf16: col_sum and col_sqsum go together"); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  TcParams p{};
  p.M = M; p.N = N; p.rows_per_tile = TC_BM; p.bn = pick_bn(N, K1 + K2); p.mode = 0;
  p.kb1 = (K1 + TC_BK - 1) / TC_BK; p.kb2 = (K2 + TC_BK - 1) / TC_BK;
  p.relu = relu; p.ldd = ldd; p.D = (__nv_bfloat16*)D; p.scale = scale; p.shift = shift; p.col_sum = col_sum; p.col_sqsum = col_sqsum;
  CUtensorMap a1, b1, a2, b2;
  int rc;
  if ((rc = make_map_2d(&a1, A1, M, K1, lda1, TC_BM))) return rc;
  if ((rc = make_map_2d(&b1, B1, N, K1, ldb1, p.bn))) return rc;
  if (K2 > 0) {
    if ((rc = make_map_2d(&a2, A2, M, K2, lda2, TC_BM))) return rc;
    if ((rc = make_map_2d(&b2, B2, N, K2, ldb2, p.bn))) return rc;
  } else { a2 = a1; b2 = b1; }
  return tc_launch(a1, b1, a2, b2, p, (M + TC_BM - 1) / TC_BM, st, "tc_gemm_1x1",
                   2.0 * ((double)M * (K1 + K2 + N) + (double)N * (K1 + K2)));
}

// Same GEMM; col_sum / col_sqsum are accumulated PER SAMPLE of rows_per_sample consecutive rows: [M / rows_per_sample, N].
extern "C" int cotb200_gemm_bf16_samplestats(int M, int N, int K1, const void* A1, long long lda1, const void* B1, long long ldb1, void* D,
                                             long long ldd, const float* scale, const float* shift, int relu, int rows_per_sample,
                                             float* samp_sum, float* samp_sqsum, void* stream) {
  if (M <= 0 || N <= 0 || K1 <= 0) { set_error("gemm_bf16_samplestats: bad dims"); return COTB200_EINVAL; }
  if (!A1 || !B1 || !D || !samp_sum || !samp_sqsum) { set_error("gemm_bf16_samplestats: NULL operand"); return COTB200_ENULL; }
  if ((N & 7) || (K1 & 7) || (ldd & 7)) { set_error("gemm_bf16_samplestats: N, K, ldd must be multiples of 8"); return COTB200_EALIGN; }
  if (rows_per_sample < 32 || M % rows_per_sample) { set_error("gemm_bf16_samplestats: rows_per_sample=%d must be >= 32 and divide M=%d", rows_per_sample, M); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  TcParams p{};
  p.M = M; p.N = N; p.rows_per_tile = TC_BM; p.bn = pick_bn(N); p.mode = 0;
  p.kb1 = (K1 + TC_BK - 1) / TC_BK; p.kb2 = 0;
  p.relu = relu; p.ldd = ldd; p.D = (__nv_bfloat16*)D; p.scale = scale; p.shift = shift; p.col_sum = samp_sum; p.col_sqsum = samp_sqsum;
  p.rows_per_sample = rows_per_sample;
  CUtensorMap a1, b1;
  int rc;
  if ((rc = make_map_2d(&a1, A1, M, K1, lda1, TC_BM))) return rc;
  if ((rc = make_map_2d(&b1, B1, N, K1, ldb1, p.bn))) return rc;
  return tc_launch(a1, b1, a1, b1, p, (M + TC_BM - 1) / TC_BM, st, "tc_gemm_1x1", 2.0 * ((double)M * (K1 + N) + (double)N * K1));
}

// 3x3 / pad 1 / stride 1 convolution, NHWC bf16, with dense-per-N-tile prepared weights
//   Wp [C_out, 9 * bn] bf16 row-major: Wp[n, (tap*kc + cc)*64 + ci] = weight of output channel n for input channel
//   (n0(n) + cc*64 + ci) at tap (0 where that input channel is outside n's group); bn = N tile in {64,128,192,256}.
extern "C" int cotb200_conv3x3_bf16(int B, int H, int W, int C, const void* X, long long ldx, const void* Wp, int bn, void* D,
                                    long long ldd, const float* scale, const float* shift, int relu, float* col_sum,
                                    float* col_sqsum, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0) { set_error("conv3x3_bf16: bad dims"); return COTB200_EINVAL; }
  if (!X || !Wp || !D) { set_error("conv3x3_bf16: NULL operand"); return COTB200_ENULL; }
  if (bn % 64 || bn > 256 || C % bn) { set_error("conv3x3_bf16: N tile %d must be a multiple of 64 dividing C=%d", bn, C); return COTB200_EINVAL; }
  if (W > 128) { set_error("conv3x3_bf16: W=%d > 128 not supported by the pixel-box tiling", W); return COTB200_EINVAL; }
  if ((col_sum == nullptr) != (col_sqsum == nullptr)) { set_error("conv3x3_bf16: col_sum and col_sqsum go together"); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  {
    int hrc = 0;
    if (conv3x3_halo_launch(B, H, W, C, X, ldx, Wp, bn, D, ldd, scale, shift, relu, col_sum, col_sqsum, st, &hrc)) return hrc;
  }
  TcParams p{};
  p.M = B * H * W; p.N = C; p.bn = bn; p.mode = 1; p.kc = bn / 64;
  p.H = H; p.W = W; p.B = B;
  int m_tiles;
  if (H * W <= TC_BM / 2) {                      // several whole samples per tile (7x7: 2 samples = 98 rows)
    p.bbox = TC_BM / (H * W); p.hbox = H;
    m_tiles = (B + p.bbox - 1) / p.bbox;
  } else {                                       // a band of whole rows of one sample
    p.bbox = 1;
    int hb = TC_BM / W; if (hb > H) hb = H; if (hb < 1) hb = 1;
    while (H % hb) --hb;                         // bands tile the sample exactly
    p.hbox = hb;
    m_tiles = B * (H / hb);
  }
  p.rows_per_tile = p.bbox * p.hbox * W;
  p.relu = relu; p.ldd = ldd; p.D = (__nv_bfloat16*)D; p.scale = scale; p.shift = shift; p.col_sum = col_sum; p.col_sqsum = col_sqsum;
  CUtensorMap a1, b1;
  int rc;
  if ((rc = make_map_nhwc(&a1, X, B, H, W, C, ldx, p.hbox, p.bbox))) return rc;
  if ((rc = make_map_2d(&b1, Wp, C, 9LL * bn, 9LL * bn, bn))) return rc;
  return tc_launch(a1, b1, a1, b1, p, m_tiles, st, "tc_conv3x3", 2.0 * (2.0 * (double)B * H * W * C + 9.0 * (double)C * bn));
}

// ---------------------------------------------------------------------------------------------- stem: 7x7 / s2 / p3, 3 -> N
namespace cotb200 {

// Space-to-depth copy of the 3-channel NHWC image for the stem GEMM:
//   P[b, i, jp, (di*2+dj)*3 + c] = x[b, 2i+di, 2(jp-2)+dj, c]   for 2 <= jp < Wh+2, zero for the two pad cells either side and for
//   channels 12..15.  One thread per cell: three 4-byte loads per image row (the 6 bf16 of two neighbouring pixels are contiguous
//   and 4-byte aligned because W is even), two 16-byte stores.
__global__ void __launch_bounds__(256)
stem_s2d_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ P, int B, int H, int W) {
  const int Hh = H >> 1, Wh = W >> 1, Wp = Wh + 4;
  const long long total = (long long)B * Hh * Wp;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int jp = (int)(idx % Wp);
    const long long bi = idx / Wp;
    const int i = (int)(bi % Hh), b = (int)(bi / Hh);
    uint32_t o[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    const int j = jp - 2;
    if (j >= 0 && j < Wh) {
      const uint32_t* r0 = reinterpret_cast<const uint32_t*>(x + (((long long)b * H + 2 * i) * W + 2 * j) * 3);
      const uint32_t* r1 = reinterpret_cast<const uint32_t*>(x + (((long long)b * H + 2 * i + 1) * W + 2 * j) * 3);
      o[0] = __ldg(r0); o[1] = __ldg(r0 + 1); o[2] = __ldg(r0 + 2);
      o[3] = __ldg(r1); o[4] = __ldg(r1 + 1); o[5] = __ldg(r1 + 2);
    }
    uint4* dst = reinterpret_cast<uint4*>(P + idx * 16);
    dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
    dst[1] = make_uint4(o[4], o[5], 0u, 0u);
  }
}

// s2d image [B, Hh, Wh+4, 16] seen as the matrix of overlapping 4-cell windows: {64 elements (window), Wh+1 window starts (32 B
// apart), Hh rows, B}; box {64, tw, 1, 1}.  Rows outside [0, Hh) are zero-filled by the TMA = the vertical padding.
static int make_map_stem(CUtensorMap* m, const void* base, int B, int Hh, int Wh, int tw) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return COTB200_EINVAL; }
  const long long Wp = Wh + 4;
  cuuint64_t dims[4] = {64, (cuuint64_t)(Wh + 1), (cuuint64_t)Hh, (cuuint64_t)B};
  cuuint64_t strides[3] = {32, (cuuint64_t)Wp * 32, (cuuint64_t)Wp * 32 * Hh};
  cuuint32_t box[4] = {64, (cuuint32_t)tw, 1, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(stem windows) failed: %d", (int)r); return COTB200_EUNSUPPORTED; }
  return 0;
}

}  // namespace cotb200

extern "C" long long cotb200_stem7x7s2_scratch_bytes(int B, int H, int W) {
  return (long long)B * (H / 2) * (W / 2 + 4) * 16 * 2;
}

// 7x7 / stride 2 / pad 3 convolution of a 3-channel NHWC bf16 image, see include/cotb200.h
extern "C" int cotb200_stem7x7s2_bf16(int B, int H, int W, const void* X, const void* Wm, int N, void* D, long long ldd,
                                      const float* scale, const float* shift, int relu, float* col_sum, float* col_sqsum,
                                      void* scratch, void* stream) {
  if (B <= 0 || H <= 0 || W <= 0 || N <= 0) { set_error("stem7x7s2_bf16: bad dims"); return COTB200_EINVAL; }
  if (!X || !Wm || !D || !scratch) { set_error("stem7x7s2_bf16: NULL operand"); return COTB200_ENULL; }
  if ((H & 1) || (W & 1)) { set_error("stem7x7s2_bf16: H=%d, W=%d must be even", H, W); return COTB200_EUNSUPPORTED; }
  if ((N & 7) || N > 256 || (ldd & 7)) { set_error("stem7x7s2_bf16: N=%d must be a multiple of 8, <= 256", N); return COTB200_EUNSUPPORTED; }
  if ((col_sum == nullptr) != (col_sqsum == nullptr)) { set_error("stem7x7s2_bf16: col_sum and col_sqsum go together"); return COTB200_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(X) & 3) || (reinterpret_cast<uintptr_t>(scratch) & 15)) { set_error("stem7x7s2_bf16: misaligned operand"); return COTB200_EALIGN; }
  const int Hh = H / 2, Wh = W / 2;
  int wtiles = (Wh + TC_BM - 1) / TC_BM;
  while (Wh % wtiles) ++wtiles;                    // equal segments of an output row
  const int tw = Wh / wtiles;
  if (tw < 8) { set_error("stem7x7s2_bf16: W=%d not supported by the row tiling", W); return COTB200_EUNSUPPORTED; }
  cudaStream_t st = (cudaStream_t)stream;
  CUtensorMap a1, b1;
  int rc;
  if ((rc = make_map_stem(&a1, scratch, B, Hh, Wh, tw))) return rc;
  TcParams p{};
  p.M = B * Hh * Wh; p.N = N; p.bn = pick_bn_wide(N); p.mode = 2; p.kb1 = 4; p.kb2 = 0;
  p.H = Hh; p.W = Wh; p.B = B; p.wtiles = wtiles; p.rows_per_tile = tw;
  p.relu = relu; p.ldd = ldd; p.D = (__nv_bfloat16*)D; p.scale = scale; p.shift = shift; p.col_sum = col_sum; p.col_sqsum = col_sqsum;
  if ((rc = make_map_2d(&b1, Wm, N, 256, 256, p.bn))) return rc;
  {
    const long long cells = (long long)B * Hh * (Wh + 4);
    long long g = (cells + 255) / 256;
    const int grid = (int)(g < (long long)num_sms() * 16 ? g : (long long)num_sms() * 16);
    COTB200_PROF_B("stem_s2d", (double)B * H * W * 3 * 2 + (double)cells * 32);
    stem_s2d_kernel<<<grid, 256, 0, st>>>((const __nv_bfloat16*)X, (__nv_bfloat16*)scratch, B, H, W);
    if ((rc = check_launch("stem_s2d"))) return rc;
  }
  return tc_launch(a1, b1, a1, b1, p, B * Hh * wtiles, st, "tc_stem7x7",
                   (double)B * Hh * (Wh + 4) * 32 + 2.0 * (double)p.M * N + 2.0 * N * 256);
}
