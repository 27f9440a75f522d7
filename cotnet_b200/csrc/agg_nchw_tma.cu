// LocalConv 3x3 on NCHW tensors (the reference contract, fp32 first): persistent CTAs fed by a TMA pipeline (sm_90a).
//
// The register-resident NCHW kernels (agg_nchw2.cu) stay well below the HBM roof forward and near the speed of the
// reference's own kernels backward: 80-170 registers, one or two 8-warp CTAs
// per SM, every warp waiting on global loads, and each halo row costs one vector + two scalar global loads.
// Same cure as for the NHWC kernels (agg_tma.cu): one producer warp streams tiles into a shared-memory ring with
// cp.async.bulk.tensor, the compute warps never touch global memory for their operands.
//   tile      = (sample n, weight channel g, band of TH image rows);   channels of g: c = g + j*wc, j < rep (= C / wc)
//   planes    = x / dY / dX seen as the 5-D tensor {W, H, wc, rep, N}: ONE box {BW, TH+2, 1, rep, 1} fetched at
//               (-PXV, h0-1, g, 0, n) brings the band of all `rep` channels with its halo; out-of-bounds coordinates are
//               zero-filled by the TMA unit == the operator's zero padding.  The left halo is 16 bytes wide (4 fp32 / 8 bf16
//               pixels, not 1): a TMA box must start 16-byte aligned in global memory (a -8-byte start faults as "illegal
//               instruction"), and the centre vector of every thread then stays vector-aligned in shared memory.
//   weights   = {W, H, 9, wc, N}: box {BW', TH(+2), 9, 1, 1}.
//   compute   : thread = (row, PXV pixels, channel subset); 9 weight vectors in registers, per channel 3 x (1 vector +
//               2 scalar) shared loads and 9*PXV FMAs; results stored straight to global memory (PXV-wide, coalesced).
// Modes: 0 forward, 1 dX (weights AND dY fetched with halo), 2 dW (x with halo, dY plain; 9 planes of sums per tile).
// Requirements: K=3, stride 1, pad 1, heads 1, dense NCHW, W % PXV == 0, W*sizeof(T) % 16 == 0 (TMA global strides):
// fp32 W in {56, 28, ..}, 16-bit W = 56; everything else stays on agg_nchw2.cu / the generic kernels.
#include <cuda.h>
#include "common.cuh"
#include "tma.cuh"

namespace cotb200 {

static constexpr int NT_MAX_STAGES = 4;
static constexpr int NT_COMPUTE_THREADS = 384;
static constexpr int NT_THREADS_TOTAL = NT_COMPUTE_THREADS + 32;

struct NchwTmaP {
  int N, C, H, W, wc, rep;
  int TH, bands, total_tiles, stages;
  int halo;               // columns of left halo in the tiles: max(PXV, 16/sizeof(T)) -- the box must START 16-byte aligned in global memory
  int BWa;                // row pitch (elements) of haloed tiles: round_up(W + 2*halo, 16/sizeof(T))
  int BWb;                // row pitch of plain tiles: round_up(W, 16/sizeof(T))
  int a_bytes, b_bytes;   // per-stage bytes of operand A / B (each rounded up to 128)
  int a_tx, b_tx;         // bytes the TMA reports per stage
  int stage_bytes;
  int mode;               // 0 fwd: A = x (halo), B = w (plain) ; 1 dX: A = dY (halo), B = w (halo) ; 2 dW: A = x (halo), B = dY (plain)
  int nsplit;             // channel subsets per (row, quad)
  long long out_sn;       // batch stride of the output tensor (elements)
};

// PXV consecutive elements at `p` (PXV*sizeof(T)-aligned) plus the element before and after: v[0], v[1..PXV], v[PXV+1]
template <typename T, int PXV>
__device__ __forceinline__ void nt_ld_seg(const T* p, T (&v)[PXV + 2]) {
  const Pack<T, PXV> c = *reinterpret_cast<const Pack<T, PXV>*>(p);
#pragma unroll
  for (int i = 0; i < PXV; ++i) v[i + 1] = c.v[i];
  v[0] = p[-1];
  v[PXV + 1] = p[PXV];
}

template <typename T, int PXV, int MODE>
__global__ void __launch_bounds__(NT_THREADS_TOTAL, 1)
agg3_nchw_tma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, T* __restrict__ out,
                     const NchwTmaP p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ uint64_t s_full[NT_MAX_STAGES], s_empty[NT_MAX_STAGES];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int CW = NT_COMPUTE_THREADS / 32;
  if (tid == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), CW); }
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == CW) {                                       // ---------------- producer
    if (lane == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
        const int s = it % p.stages;
        mbar_wait(smem_u32(&s_empty[s]), ((it / p.stages) & 1) ^ 1);
        const int band = tile % p.bands, ng = tile / p.bands;
        const int g = ng % p.wc, n = ng / p.wc, h0 = band * p.TH;
        const uint32_t full = smem_u32(&s_full[s]);
        const uint32_t base = smem_u32(smem + (size_t)s * p.stage_bytes);
        mbar_expect_tx(full, (uint32_t)(p.a_tx + p.b_tx));
        tma_load_5d(base, &mapA, full, -p.halo, h0 - 1, g, 0, n);                        // haloed planes of the rep channels
        if (MODE == 0) tma_load_5d(base + p.a_bytes, &mapB, full, 0, h0, 0, g, n);      // weights, plain band
        else if (MODE == 1) tma_load_5d(base + p.a_bytes, &mapB, full, -p.halo, h0 - 1, 0, g, n);   // weights with halo
        else tma_load_5d(base + p.a_bytes, &mapB, full, 0, h0, g, 0, n);               // dY planes, plain band
      }
    }
    return;
  }

  // ---------------- consumers
  const int HW = p.H * p.W, nq = p.W / PXV;
  const int items = p.TH * nq * p.nsplit;
  const int rowsA = p.TH + 2;
  int it = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
    const int s = it % p.stages;
    mbar_wait(smem_u32(&s_full[s]), (it / p.stages) & 1);
    const int band = tile % p.bands, ng = tile / p.bands;
    const int g = ng % p.wc, n = ng / p.wc, h0 = band * p.TH;
    const T* sA = reinterpret_cast<const T*>(smem + (size_t)s * p.stage_bytes);
    const T* sB = reinterpret_cast<const T*>(smem + (size_t)s * p.stage_bytes + p.a_bytes);
    for (int item = tid; item < items; item += NT_COMPUTE_THREADS) {
      const int js = item % p.nsplit, rq = item / p.nsplit;
      const int q = rq % nq, r = rq / nq;
      const int h = h0 + r, w0 = q * PXV;
      if (h >= p.H) continue;
      if (MODE == 0) {
        // y_j[p] = sum_t w_t[p] * x_j[p + off_t]
        Pack<T, PXV> wt[9];
#pragma unroll
        for (int t = 0; t < 9; ++t) wt[t] = *reinterpret_cast<const Pack<T, PXV>*>(sB + (t * p.TH + r) * p.BWb + w0);
        T* yb = out + (long long)n * p.out_sn + (long long)g * HW + (long long)h * p.W + w0;
        for (int j = js; j < p.rep; j += p.nsplit) {
          const T* xb = sA + (j * rowsA + r + 1) * p.BWa + w0 + p.halo;               // centre row, centre vector
          float acc[PXV];
#pragma unroll
          for (int i = 0; i < PXV; ++i) acc[i] = 0.f;
#pragma unroll
          for (int dh = -1; dh <= 1; ++dh) {
            T v[PXV + 2];
            nt_ld_seg<T, PXV>(xb + dh * p.BWa, v);
#pragma unroll
            for (int dw = -1; dw <= 1; ++dw)
#pragma unroll
              for (int i = 0; i < PXV; ++i) acc[i] = mfma<T>(wt[(dh + 1) * 3 + dw + 1].v[i], v[i + 1 + dw], acc[i]);
          }
          Pack<T, PXV> o;
#pragma unroll
          for (int i = 0; i < PXV; ++i) o.v[i] = Elem<T>::from(acc[i]);
          st_pack<T, PXV>(yb + (long long)j * p.wc * HW, o);
        }
      } else if (MODE == 1) {
        // dx_j[p] = sum_t w_t[p - off_t] * dy_j[p - off_t]      (zero outside: both tiles are zero-filled there)
        T ws[9][PXV];
#pragma unroll
        for (int dh = -1; dh <= 1; ++dh)
#pragma unroll
          for (int dw = -1; dw <= 1; ++dw) {
            const int t = (dh + 1) * 3 + dw + 1;
            T v[PXV + 2];
            nt_ld_seg<T, PXV>(sB + (t * rowsA + r + 1 - dh) * p.BWa + w0 + p.halo, v);
#pragma unroll
            for (int i = 0; i < PXV; ++i) ws[t][i] = v[i + 1 - dw];
          }
        T* xb = out + (long long)n * p.out_sn + (long long)g * HW + (long long)h * p.W + w0;
        for (int j = js; j < p.rep; j += p.nsplit) {
          const T* db = sA + (j * rowsA + r + 1) * p.BWa + w0 + p.halo;
          float acc[PXV];
#pragma unroll
          for (int i = 0; i < PXV; ++i) acc[i] = 0.f;
#pragma unroll
          for (int dh = -1; dh <= 1; ++dh) {
            T v[PXV + 2];
            nt_ld_seg<T, PXV>(db - dh * p.BWa, v);                                   // row h - dh
#pragma unroll
            for (int dw = -1; dw <= 1; ++dw)
#pragma unroll
              for (int i = 0; i < PXV; ++i) acc[i] = mfma<T>(ws[(dh + 1) * 3 + dw + 1][i], v[i + 1 - dw], acc[i]);
          }
          Pack<T, PXV> o;
#pragma unroll
          for (int i = 0; i < PXV; ++i) o.v[i] = Elem<T>::from(acc[i]);
          st_pack<T, PXV>(xb + (long long)j * p.wc * HW, o);
        }
      } else {
        // dw_t[p] = sum_j x_j[p + off_t] * dy_j[p]              (nsplit == 1: one thread owns all channels of its pixels)
        float gw[9][PXV];
#pragma unroll
        for (int t = 0; t < 9; ++t)
#pragma unroll
          for (int i = 0; i < PXV; ++i) gw[t][i] = 0.f;
        for (int j = 0; j < p.rep; ++j) {
          const Pack<T, PXV> d = *reinterpret_cast<const Pack<T, PXV>*>(sB + (j * p.TH + r) * p.BWb + w0);
          const T* xb = sA + (j * rowsA + r + 1) * p.BWa + w0 + p.halo;
#pragma unroll
          for (int dh = -1; dh <= 1; ++dh) {
            T v[PXV + 2];
            nt_ld_seg<T, PXV>(xb + dh * p.BWa, v);
#pragma unroll
            for (int dw = -1; dw <= 1; ++dw)
#pragma unroll
              for (int i = 0; i < PXV; ++i)
                gw[(dh + 1) * 3 + dw + 1][i] = mfma<T>(v[i + 1 + dw], d.v[i], gw[(dh + 1) * 3 + dw + 1][i]);
          }
        }
        T* wb = out + ((long long)n * p.wc + g) * 9 * HW + (long long)h * p.W + w0;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          Pack<T, PXV> o;
#pragma unroll
          for (int i = 0; i < PXV; ++i) o.v[i] = Elem<T>::from(gw[t][i]);
          st_pack<T, PXV>(wb + (long long)t * HW, o);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&s_empty[s]));
  }
}

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*NtEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static NtEncodeFn nt_encode_fn() {
  static NtEncodeFn fn = nullptr;
  if (!fn) {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult r;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &r) == cudaSuccess && r == cudaDriverEntryPointSuccess)
      fn = (NtEncodeFn)q;
  }
  return fn;
}
template <typename T> static CUtensorMapDataType nt_dtype();
template <> CUtensorMapDataType nt_dtype<float>() { return CU_TENSOR_MAP_DATA_TYPE_FLOAT32; }
template <> CUtensorMapDataType nt_dtype<__nv_bfloat16>() { return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; }
template <> CUtensorMapDataType nt_dtype<__half>() { return CU_TENSOR_MAP_DATA_TYPE_FLOAT16; }

// generic 5-D map over a dense tensor: dims d[0..4] (d[0] innermost, unit stride), strides st[0..3] in ELEMENTS for d[1..4]
template <typename T>
static bool nt_make_map(CUtensorMap* m, const void* base, const long long (&d)[5], const long long (&st)[4], const int (&box)[5]) {
  NtEncodeFn enc = nt_encode_fn();
  if (!enc) return false;
  cuuint64_t dims[5], strides[4];
  cuuint32_t b[5], es[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < 5; ++i) { dims[i] = (cuuint64_t)d[i]; b[i] = (cuuint32_t)box[i]; }
  for (int i = 0; i < 4; ++i) strides[i] = (cuuint64_t)st[i] * sizeof(T);
  return enc(m, nt_dtype<T>(), 5, const_cast<void*>(base), dims, strides, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static inline int nt_round_up(int a, int b) { return (a + b - 1) / b * b; }

// mode 0: A = x, B = w, out = y ; mode 1: A = dy, B = w, out = dx ; mode 2: A = x, B = dy, out = dw.
// planes_sn: batch stride (elements) of the A tensor ; b_sn: of the B tensor when it is a plane tensor ; out_sn: of `out`.
// returns 1 if handled (*rc = status), 0 if the caller should use another kernel.
template <typename T>
int nchw_tma_launch(int mode, int N, int C, int H, int W, int wc, long long a_sn, long long b_sn, long long out_sn, const T* A,
                    const T* Bp, T* out, cudaStream_t st, int* rc) {
  if constexpr (std::is_same<T, double>::value) { return 0; } else {
    if (C % wc) return 0;
    const int rep = C / wc, es = (int)sizeof(T), al = 16 / es;
    int pxv = 0;
    if (W % 4 == 0) pxv = 4; else if (W % 2 == 0 && es == 4) pxv = 2;
    if (!pxv || rep > 16 || rep < 1) return 0;
    if (((long long)W * es) % 16 || ((long long)H * W * es) % 16) return 0;                 // TMA global strides: multiples of 16 B
    if ((a_sn * es) % 16 || (b_sn * es) % 16 || (out_sn * es) % (pxv * es)) return 0;
    if (!aligned16(A) || !aligned16(Bp) || !aligned16(out)) return 0;
    if (W + 2 * (pxv > al ? pxv : al) > 256 || H < 1 || N < 1) return 0;
    NchwTmaP p;
    p.N = N; p.C = C; p.H = H; p.W = W; p.wc = wc; p.rep = rep; p.mode = mode; p.out_sn = out_sn;
    p.halo = pxv > al ? pxv : al;
    p.BWa = nt_round_up(W + 2 * p.halo, al);
    p.BWb = nt_round_up(W, al);
    p.nsplit = mode == 2 ? 1 : (rep % 2 == 0 ? 2 : 1);
    const int nq = W / pxv;
    // rows per tile: enough (row, quad, split) items to occupy the compute threads, stage <= ~60 KB
    const int budget = 200 * 1024;
    int best_th = 0, best_stages = 0;
    for (int th = 1; th <= H && th <= 32; ++th) {
      const long long a_bytes = nt_round_up((int)((long long)rep * (th + 2) * p.BWa * es), 128);
      const long long b_bytes = nt_round_up((int)(mode == 0 ? (long long)9 * th * p.BWb * es
                                                  : mode == 1 ? (long long)9 * (th + 2) * p.BWa * es
                                                              : (long long)rep * th * p.BWb * es), 128);
      const long long stage = a_bytes + b_bytes;
      if (stage * 2 > budget) break;
      best_th = th;
      best_stages = (int)(budget / stage);
      if (th * nq * p.nsplit >= NT_COMPUTE_THREADS) break;
    }
    if (!best_th) return 0;
    p.TH = best_th;
    p.stages = best_stages > NT_MAX_STAGES ? NT_MAX_STAGES : best_stages;
    if (p.stages < 2) return 0;
    p.bands = (H + p.TH - 1) / p.TH;
    p.total_tiles = N * wc * p.bands;
    const int rowsA = p.TH + 2;
    p.a_tx = rep * rowsA * p.BWa * es;
    p.a_bytes = nt_round_up(p.a_tx, 128);
    p.b_tx = (mode == 0 ? 9 * p.TH * p.BWb : mode == 1 ? 9 * rowsA * p.BWa : rep * p.TH * p.BWb) * es;
    p.b_bytes = nt_round_up(p.b_tx, 128);
    p.stage_bytes = nt_round_up(p.a_bytes + p.b_bytes, 128);
    const size_t smem = (size_t)p.stages * p.stage_bytes + 1024;

    const long long HW = (long long)H * W;
    CUtensorMap ma, mb;
    {   // planes {W, H, wc, rep, N}
      const long long d[5] = {W, H, wc, rep, N};
      const long long s4[4] = {W, HW, (long long)wc * HW, a_sn};
      const int box[5] = {p.BWa, rowsA, 1, rep, 1};
      if (!nt_make_map<T>(&ma, A, d, s4, box)) return 0;
    }
    if (mode == 2) {
      const long long d[5] = {W, H, wc, rep, N};
      const long long s4[4] = {W, HW, (long long)wc * HW, b_sn};
      const int box[5] = {p.BWb, p.TH, 1, rep, 1};
      if (!nt_make_map<T>(&mb, Bp, d, s4, box)) return 0;
    } else {   // weights {W, H, 9, wc, N}
      const long long d[5] = {W, H, 9, wc, N};
      const long long s4[4] = {W, HW, 9 * HW, (long long)wc * 9 * HW};
      const int box0[5] = {p.BWb, p.TH, 9, 1, 1};
      const int box1[5] = {p.BWa, rowsA, 9, 1, 1};
      if (!(mode == 0 ? nt_make_map<T>(&mb, Bp, d, s4, box0) : nt_make_map<T>(&mb, Bp, d, s4, box1))) return 0;
    }
    int grid = num_sms();
    if (grid > p.total_tiles) grid = p.total_tiles;
    const double bytes = ((double)N * HW) * (2.0 * C + 9.0 * wc) * sizeof(T);
    COTB200_PROF_B(mode == 0 ? "agg3_fwd_nchw_tma" : mode == 1 ? "agg3_dx_nchw_tma" : "agg3_dw_nchw_tma", bytes);
#define NT_GO(P, M)                                                                                                   \
  {                                                                                                                   \
    static PerDevFlag cfgd; bool& cfg = cfgd.get();                                                                   \
    if (!cfg) {                                                                                                       \
      cudaError_t e = cudaFuncSetAttribute(agg3_nchw_tma_kernel<T, P, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                           220 * 1024);                                                               \
      if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); *rc = (int)e; return 1; } \
      cfg = true;                                                                                                     \
    }                                                                                                                 \
    agg3_nchw_tma_kernel<T, P, M><<<grid, NT_THREADS_TOTAL, smem, st>>>(ma, mb, out, p);                              \
  }
    if (pxv == 4) { if (mode == 0) NT_GO(4, 0) else if (mode == 1) NT_GO(4, 1) else NT_GO(4, 2) }
    else { if (mode == 0) NT_GO(2, 0) else if (mode == 1) NT_GO(2, 1) else NT_GO(2, 2) }
#undef NT_GO
    *rc = check_launch("agg3_nchw_tma");
    return 1;
  }
}

#define COTB200_INST_NT(T)                                                                                             \
  template int nchw_tma_launch<T>(int, int, int, int, int, int, long long, long long, long long, const T*, const T*, T*, \
                                  cudaStream_t, int*);
COTB200_INST_NT(float) COTB200_INST_NT(double) COTB200_INST_NT(__nv_bfloat16) COTB200_INST_NT(__half)

}  // namespace cotb200
