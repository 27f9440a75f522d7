// Train-step plumbing of the data-parallel CoT path (SURVEY.md section 8f rank 3/4), sm_90a.
//
// The reference's step (train.py:264-293) is, per parameter tensor: DDP bucket copy, optim.SGD(nesterov) update
// (optim/optim_factory.py:54-56), ModelEmaV2 lerp over the whole state_dict (utils/model_ema.py:45-53), and -- under AMP --
// a weight cast per convolution per step; the input pipeline normalises uint8 batches with three eager ops
// (datasets/loader.py:86-90).  ~500 parameter tensors make that ~2000 tiny launches.  Here the replica keeps
//   P  fp32 master weights, M momentum, E EMA   -- flat buffers, one element order
//   G  the step's gradients, gathered into ONE flat bucket (the unit of the NCCL all-reduce)
//   Pb the bf16 copy of the >=2-D weights the convolutions actually read
// and the whole parameter update is ONE pass (cotb200_opt_step, opt.cu):  read G, P, M, E  ->  write P, M, E, Pb.
//
//   cotb200_multi_gather   gradients (any mix of fp32 / bf16 tensors) -> flat bucket (fp32 or bf16), optional scale
//   cotb200_multi_gather_acc   the same added to an fp32 accumulator, optionally emitted into the bucket: the gradient sum over
//                          the micro-batches of a step with virtual ranks
//   cotb200_multi_lerp     EMA of the buffers (BatchNorm running statistics, integer counters) by pointer table
//   cotb200_u8_to_nhwc     uint8 NCHW batch -> (x - mean)/std in bf16/fp16/fp32 channels_last
//   cotb200_u8_mix_rows_to_nhwc   the same after Mixup / CutMix, one table row per output sample
//
// All HBM-bound streaming kernels: 16-byte accesses, grid = a few waves of 132 SMs, no atomics.
#include "common.cuh"

namespace cotb200 {

// ------------------------------------------------------------------------------------------------ multi_gather
// One table row per source tensor: (pointer, first element in the bucket, elements, dtype).  The block -> row map is a
// second table built by the host (rows are cut into chunks of GATHER_CHUNK elements) so no thread searches.
static constexpr int GATHER_CHUNK = 8192;       // elements per block: 32 KB of fp32

// Modes of the gather (cotb200_multi_gather / cotb200_multi_gather_acc).  The two accumulating modes add in fp32 with
// __fmul_rn / __fadd_rn (no FMA contraction), so a sum over micro-batches is bit-exact against torch fp32 adds in the same order.
enum GatherMode {
  GATHER_STORE = 0,   // dst[i] = TD(g * scale)
  GATHER_ACC = 1,     // acc[i] = acc[i] + g * scale          (dst is acc, TD = float)
  GATHER_EMIT = 2,    // dst[i] = TD(acc[i] + g * scale)      (dst may be acc itself when TD = float)
};

template <int MODE, typename TD>
__device__ __forceinline__ TD gather_elem(float g, float a, float scale) {
  if constexpr (MODE == GATHER_STORE) return Elem<TD>::from(g * scale);
  else return Elem<TD>::from(__fadd_rn(a, __fmul_rn(g, scale)));
}

template <int MODE, typename TS, typename TD>
__device__ __forceinline__ void gather_chunk(const TS* __restrict__ src, const float* acc, TD* dst, long long n, float scale) {
  // n <= GATHER_CHUNK elements; src/dst/acc each aligned to at least their element size.  Vector path when all are aligned to
  // the packet.  acc and dst may alias (GATHER_ACC, and GATHER_EMIT into an fp32 bucket): each element is read and then written
  // by the same thread, so they carry no __restrict__.
  constexpr int VS = 16 / (int)sizeof(TS), VD = 16 / (int)sizeof(TD), VA = MODE == GATHER_STORE ? 16 : 4;
  constexpr int V0 = VS < VD ? VS : VD;
  constexpr int V = V0 < VA ? V0 : VA;           // elements per thread step (4 for any fp32 side, 8 for a bf16 -> bf16 store)
  const bool vec = ((reinterpret_cast<uintptr_t>(src) % (V * sizeof(TS))) == 0) && ((reinterpret_cast<uintptr_t>(dst) % (V * sizeof(TD))) == 0) &&
                   (MODE == GATHER_STORE || (reinterpret_cast<uintptr_t>(acc) % (V * sizeof(float))) == 0);
  long long i0 = 0;
  if (vec) {
    const long long nv = n / V;
    for (long long i = threadIdx.x; i < nv; i += blockDim.x) {
      const Pack<TS, V> s = ld_pack<TS, V>(src + i * V);
      Pack<float, V> a;
      if constexpr (MODE != GATHER_STORE) a = *reinterpret_cast<const Pack<float, V>*>(acc + i * V);
      Pack<TD, V> d;
#pragma unroll
      for (int k = 0; k < V; ++k) d.v[k] = gather_elem<MODE, TD>((float)to_acc(s.v[k]), MODE == GATHER_STORE ? 0.f : a.v[k], scale);
      st_pack<TD, V>(dst + i * V, d);
    }
    i0 = nv * V;
  }
  for (long long i = i0 + threadIdx.x; i < n; i += blockDim.x)
    dst[i] = gather_elem<MODE, TD>((float)to_acc(src[i]), MODE == GATHER_STORE ? 0.f : acc[i], scale);
}

// A segment without a source (a parameter that got no gradient in this micro-batch) contributes zero: nothing to add, and the
// emit pass converts the accumulator alone.
template <typename TD>
__device__ __forceinline__ void emit_only(const float* acc, TD* dst, long long n) {
  for (long long i = threadIdx.x; i < n; i += blockDim.x) dst[i] = Elem<TD>::from(acc[i]);
}

template <int MODE, typename TD>
__global__ void __launch_bounds__(256)
multi_gather_kernel(const cotb200_seg* __restrict__ segs, const int2* __restrict__ blocks, const float* acc, TD* dst, float scale) {
  const int2 b = blocks[blockIdx.x];              // (row, chunk index inside the row)
  const cotb200_seg s = segs[b.x];
  const long long off = (long long)b.y * GATHER_CHUNK;
  long long n = s.numel - off;
  if (n > GATHER_CHUNK) n = GATHER_CHUNK;
  TD* d = dst + s.offset + off;
  const float* a = MODE == GATHER_STORE ? nullptr : acc + s.offset + off;
  if (MODE != GATHER_STORE && s.ptr == nullptr) {
    if (MODE == GATHER_EMIT) emit_only<TD>(a, d, n);
    return;
  }
  if (s.dtype == COTB200_F32) gather_chunk<MODE, float, TD>((const float*)s.ptr + off, a, d, n, scale);
  else if (s.dtype == COTB200_BF16) gather_chunk<MODE, __nv_bfloat16, TD>((const __nv_bfloat16*)s.ptr + off, a, d, n, scale);
  else gather_chunk<MODE, __half, TD>((const __half*)s.ptr + off, a, d, n, scale);
}

// ------------------------------------------------------------------------------------------------ multi_lerp
// e = decay*e + (1-decay)*m per buffer; integer buffers follow the reference's arithmetic literally:
// float(decay*e + (1-decay)*m) truncated back by copy_ (utils/model_ema.py:50,53).
__global__ void __launch_bounds__(256)
multi_lerp_kernel(const cotb200_seg2* __restrict__ segs, const float* __restrict__ hyper) {
  const cotb200_seg2 s = segs[blockIdx.x];
  const float dec = __ldg(hyper + 3);
  if (s.dtype == COTB200_F32) {
    float* e = (float*)s.dst; const float* m = (const float*)s.src;
    for (long long i = threadIdx.x; i < s.numel; i += 256) e[i] = fmaf(dec, e[i], (1.f - dec) * m[i]);
  } else {                                        // dtype 100: int64
    long long* e = (long long*)s.dst; const long long* m = (const long long*)s.src;
    for (long long i = threadIdx.x; i < s.numel; i += 256) e[i] = (long long)(dec * (float)e[i] + (1.f - dec) * (float)m[i]);
  }
}

// ------------------------------------------------------------------------------------------------ u8 -> NHWC
// x[n,c,h,w] uint8 (NCHW, what the loader's collate produces, datasets/loader.py:24-47) ->
// y[n,h,w,c] = (x - mean[c]) / std[c]  in T (channels_last memory of a [N,3,H,W] tensor).  4 pixels per thread:
// three 4-byte loads (one per plane, coalesced along w), one 4*3*sizeof(T)-byte contiguous store.
template <typename T>
__global__ void __launch_bounds__(256)
u8_to_nhwc3_kernel(const unsigned char* __restrict__ x, T* __restrict__ y, long long npix4, long long HW, float m0, float m1, float m2,
                   float d0, float d1, float d2) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < npix4; i += (long long)gridDim.x * 256) {
    const long long pix = i * 4;                 // HW % 4 == 0: the 4 pixels lie in one image
    const long long n = pix / HW, hw = pix - n * HW;
    const unsigned char* xb = x + n * 3 * HW + hw;
    const uchar4 a = *reinterpret_cast<const uchar4*>(xb), b = *reinterpret_cast<const uchar4*>(xb + HW),
                 c = *reinterpret_cast<const uchar4*>(xb + 2 * HW);
    // true division, like the reference's .sub_(mean).div_(std): bit-identical fp32 values before the storage rounding
    const float v[12] = {(a.x - m0) / d0, (b.x - m1) / d1, (c.x - m2) / d2, (a.y - m0) / d0, (b.y - m1) / d1, (c.y - m2) / d2,
                         (a.z - m0) / d0, (b.z - m1) / d1, (c.z - m2) / d2, (a.w - m0) / d0, (b.w - m1) / d1, (c.w - m2) / d2};
    T* o = y + pix * 3;
    if constexpr (sizeof(T) == 2) {              // 24 bytes: three 8-byte stores (pix*6 bytes is 8-byte aligned)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        Pack<T, 4> p;
#pragma unroll
        for (int e = 0; e < 4; ++e) p.v[e] = Elem<T>::from(v[k * 4 + e]);
        st_pack<T, 4>(o + k * 4, p);
      }
    } else {                                     // 48 bytes: three 16-byte stores
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        Pack<T, 4> p;
#pragma unroll
        for (int e = 0; e < 4; ++e) p.v[e] = Elem<T>::from(v[k * 4 + e]);
        st_pack<T, 4>(o + k * 4, p);
      }
    }
  }
}

// generic fallback (C != 3 or HW % 4 != 0): one thread per output element
template <typename T>
__global__ void __launch_bounds__(256)
u8_to_nhwc_generic_kernel(const unsigned char* __restrict__ x, T* __restrict__ y, long long total, int C, long long HW,
                          const float* __restrict__ mean, const float* __restrict__ stdv) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C);
    const long long pix = i / C, n = pix / HW, hw = pix - n * HW;
    y[i] = Elem<T>::from(((float)x[(n * C + c) * HW + hw] - __ldg(mean + c)) / __ldg(stdv + c));
  }
}

// ------------------------------------------------------------------------------------------------ u8 mix -> NHWC
// FastCollateMixup (datasets/mixup.py:223-299) on the uint8 batch, fused into the normalisation: the value of output row n at
// (c, h, w) given its own byte a and the byte p of its partner row.  Mixup is numpy's fp32 arithmetic
// (x.astype(float32)*lam + p.astype(float32)*(1-lam), then np.rint): two roundings of the products, one of the sum, no FMA.
__device__ __forceinline__ float mix_px(unsigned a, unsigned p, const cotb200_mix_row& m, int h, int w) {
  if (m.mode == 0) return (float)a;
  if (m.mode == 1) return rintf(__fadd_rn(__fmul_rn((float)a, m.lam), __fmul_rn((float)p, m.one_minus_lam)));
  if (m.mode == 2) return (h >= m.y0 && h < m.y1 && w >= m.x0 && w < m.x1) ? (float)p : (float)a;
  return __int_as_float(0x7fffffff);             // unknown mode: NaN, never a silently unmixed batch
}

// the 4 pixels hw..hw+3 of one image (HW % 4 == 0): own planes at xb, the partner's at xq -> 12 values stored contiguously at o
template <typename T>
__device__ __forceinline__ void mix4_to_nhwc3(const unsigned char* __restrict__ xb, const unsigned char* __restrict__ xq, long long HW,
                                              long long hw, int W, const cotb200_mix_row& m, const float (&mean)[3],
                                              const float (&sd)[3], T* __restrict__ o) {
  float v[12];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const uchar4 a = *reinterpret_cast<const uchar4*>(xb + k * HW), p = *reinterpret_cast<const uchar4*>(xq + k * HW);
    const unsigned av[4] = {a.x, a.y, a.z, a.w}, pv[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int h = (int)((hw + e) / W), w = (int)((hw + e) - (long long)h * W);
      v[e * 3 + k] = (mix_px(av[e], pv[e], m, h, w) - mean[k]) / sd[k];    // true division, like u8_to_nhwc3_kernel
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    Pack<T, 4> q;
#pragma unroll
    for (int e = 0; e < 4; ++e) q.v[e] = Elem<T>::from(v[k * 4 + e]);
    st_pack<T, 4>(o + k * 4, q);
  }
}

// row n of the table; a partner outside the N_in input rows (a device copy that differs from the validated host copy) becomes
// an unknown mode mixed with row n itself: NaN output, no read outside the batch
__device__ __forceinline__ cotb200_mix_row mix_row(const cotb200_mix_row* __restrict__ rows, long long n, int N_in) {
  cotb200_mix_row r = rows[n];
  if (r.partner < 0 || r.partner >= N_in) { r.mode = -1; r.partner = (int)n; }
  return r;
}

template <typename T>
__global__ void __launch_bounds__(256)
u8_mix_rows_to_nhwc3_kernel(const unsigned char* __restrict__ x, T* __restrict__ y, long long npix4, long long HW, int W, int N_in,
                            const cotb200_mix_row* __restrict__ rows, float m0, float m1, float m2, float d0, float d1, float d2) {
  const float mean[3] = {m0, m1, m2}, sd[3] = {d0, d1, d2};
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < npix4; i += (long long)gridDim.x * 256) {
    const long long pix = i * 4;
    const long long n = pix / HW, hw = pix - n * HW;
    const cotb200_mix_row r = mix_row(rows, n, N_in);
    mix4_to_nhwc3(x + n * 3 * HW + hw, x + (long long)r.partner * 3 * HW + hw, HW, hw, W, r, mean, sd, y + pix * 3);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
u8_mix_rows_to_nhwc_generic_kernel(const unsigned char* __restrict__ x, T* __restrict__ y, long long total, int C, long long HW, int W,
                                   int N_in, const cotb200_mix_row* __restrict__ rows, const float* __restrict__ mean,
                                   const float* __restrict__ stdv) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C);
    const long long pix = i / C, n = pix / HW, hw = pix - n * HW;
    const int h = (int)(hw / W), w = (int)(hw - (long long)h * W);
    const cotb200_mix_row r = mix_row(rows, n, N_in);
    const float v = mix_px(x[(n * C + c) * HW + hw], x[((long long)r.partner * C + c) * HW + hw], r, h, w);
    y[i] = Elem<T>::from((v - __ldg(mean + c)) / __ldg(stdv + c));
  }
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_multi_gather(const cotb200_seg* segs_dev, const int* blocks_dev, int n_blocks, int dst_dtype, void* dst,
                                    float scale, void* stream) {
  if (!segs_dev || !blocks_dev || !dst) { set_error("multi_gather: NULL pointer"); return COTB200_ENULL; }
  if (n_blocks <= 0) { set_error("multi_gather: no blocks"); return COTB200_EINVAL; }
  if (dst_dtype != COTB200_F32 && dst_dtype != COTB200_BF16) { set_error("multi_gather: bucket dtype must be fp32 or bf16"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_PROF("multi_gather");
  if (dst_dtype == COTB200_F32)
    multi_gather_kernel<GATHER_STORE, float><<<n_blocks, 256, 0, st>>>(segs_dev, (const int2*)blocks_dev, nullptr, (float*)dst, scale);
  else
    multi_gather_kernel<GATHER_STORE, __nv_bfloat16><<<n_blocks, 256, 0, st>>>(segs_dev, (const int2*)blocks_dev, nullptr,
                                                                               (__nv_bfloat16*)dst, scale);
  return check_launch("multi_gather");
}

extern "C" int cotb200_gather_chunk(void) { return GATHER_CHUNK; }

extern "C" int cotb200_multi_gather_acc(const cotb200_seg* segs_dev, const int* blocks_dev, int n_blocks, float* acc, int dst_dtype,
                                        void* dst, float scale, void* stream) {
  if (!segs_dev || !blocks_dev || !acc) { set_error("multi_gather_acc: NULL pointer"); return COTB200_ENULL; }
  if (n_blocks <= 0) { set_error("multi_gather_acc: no blocks"); return COTB200_EINVAL; }
  if (!aligned16(acc)) { set_error("multi_gather_acc: accumulator not 16-byte aligned"); return COTB200_EALIGN; }
  if (dst && dst_dtype != COTB200_F32 && dst_dtype != COTB200_BF16) {
    set_error("multi_gather_acc: bucket dtype must be fp32 or bf16"); return COTB200_EDTYPE;
  }
  if (dst == (void*)acc && dst_dtype != COTB200_F32) { set_error("multi_gather_acc: only an fp32 bucket can be its own accumulator"); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const int2* blocks = (const int2*)blocks_dev;
  if (!dst) {
    COTB200_PROF("multi_gather_acc");
    multi_gather_kernel<GATHER_ACC, float><<<n_blocks, 256, 0, st>>>(segs_dev, blocks, acc, acc, scale);
    return check_launch("multi_gather_acc");
  }
  COTB200_PROF("multi_gather_emit");
  if (dst_dtype == COTB200_F32) multi_gather_kernel<GATHER_EMIT, float><<<n_blocks, 256, 0, st>>>(segs_dev, blocks, acc, (float*)dst, scale);
  else multi_gather_kernel<GATHER_EMIT, __nv_bfloat16><<<n_blocks, 256, 0, st>>>(segs_dev, blocks, acc, (__nv_bfloat16*)dst, scale);
  return check_launch("multi_gather_emit");
}

extern "C" int cotb200_multi_lerp(const cotb200_seg2* segs_dev, int n_segs, const float* hyper_dev, void* stream) {
  if (!segs_dev || !hyper_dev) { set_error("multi_lerp: NULL pointer"); return COTB200_ENULL; }
  if (n_segs <= 0) { set_error("multi_lerp: no segments"); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_PROF("multi_lerp");
  multi_lerp_kernel<<<n_segs, 256, 0, st>>>(segs_dev, hyper_dev);
  return check_launch("multi_lerp");
}

extern "C" int cotb200_u8_to_nhwc(int dtype, int N, int C, int H, int W, const void* x_u8, void* y, const float* mean_host,
                                  const float* std_host, const float* mean_dev, const float* std_dev, void* stream) {
  if (!x_u8 || !y) { set_error("u8_to_nhwc: NULL pointer"); return COTB200_ENULL; }
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("u8_to_nhwc: non-positive dims"); return COTB200_EINVAL; }
  if (dtype == COTB200_F64) { set_error("u8_to_nhwc: fp64 not supported"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long HW = (long long)H * W;
  const bool fast = C == 3 && (HW % 4) == 0 && mean_host && std_host && (reinterpret_cast<uintptr_t>(x_u8) & 3) == 0 && aligned16(y);
  if (!fast && (!mean_dev || !std_dev)) { set_error("u8_to_nhwc: generic path needs device mean / std arrays"); return COTB200_ENULL; }
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("u8_to_nhwc", (double)N * C * HW * (1.0 + sizeof(T)));
      if (fast) {
        const long long npix4 = (long long)N * HW / 4;
        u8_to_nhwc3_kernel<T><<<grid_stride_blocks(npix4, 256, 16), 256, 0, st>>>((const unsigned char*)x_u8, (T*)y, npix4, HW, mean_host[0], mean_host[1],
                                                                   mean_host[2], std_host[0], std_host[1], std_host[2]);
      } else {
        const long long total = (long long)N * C * HW;
        u8_to_nhwc_generic_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const unsigned char*)x_u8, (T*)y, total, C, HW, mean_dev, std_dev);
      }
      return check_launch("u8_to_nhwc");
    }
  });
  return 0;
}

extern "C" int cotb200_u8_mix_rows_to_nhwc(int dtype, int N_in, int N_out, int C, int H, int W, const void* x_u8, void* y,
                                           const float* mean_host, const float* std_host, const float* mean_dev, const float* std_dev,
                                           const cotb200_mix_row* rows_host, const cotb200_mix_row* rows_dev, void* stream) {
  if (!x_u8 || !y || !rows_host || !rows_dev) { set_error("u8_mix_rows_to_nhwc: NULL pointer"); return COTB200_ENULL; }
  if (N_in <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("u8_mix_rows_to_nhwc: non-positive dims"); return COTB200_EINVAL; }
  if (N_in & 1) { set_error("u8_mix_rows_to_nhwc: batch size %d must be even", N_in); return COTB200_EINVAL; }
  if (N_out <= 0 || N_out > N_in) { set_error("u8_mix_rows_to_nhwc: %d output rows from %d input rows", N_out, N_in); return COTB200_EINVAL; }
  for (int n = 0; n < N_out; ++n) {
    const cotb200_mix_row& r = rows_host[n];
    if (r.mode < 0 || r.mode > 2) { set_error("u8_mix_rows_to_nhwc: row %d: unknown mode %d (0 none, 1 mixup, 2 cutmix)", n, r.mode); return COTB200_EINVAL; }
    if (r.partner < 0 || r.partner >= N_in) { set_error("u8_mix_rows_to_nhwc: row %d: partner %d outside [0, %d)", n, r.partner, N_in); return COTB200_EINVAL; }
    if (r.mode == 2 && !(0 <= r.y0 && r.y0 <= r.y1 && r.y1 <= H && 0 <= r.x0 && r.x0 <= r.x1 && r.x1 <= W)) {
      set_error("u8_mix_rows_to_nhwc: row %d: CutMix box (%d, %d, %d, %d) outside the %dx%d image", n, r.y0, r.y1, r.x0, r.x1, H, W);
      return COTB200_EINVAL;
    }
  }
  if (dtype == COTB200_F64) { set_error("u8_mix_rows_to_nhwc: fp64 not supported"); return COTB200_EDTYPE; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long HW = (long long)H * W;
  const bool fast = C == 3 && (HW % 4) == 0 && mean_host && std_host && (reinterpret_cast<uintptr_t>(x_u8) & 3) == 0 && aligned16(y);
  if (!fast && (!mean_dev || !std_dev)) { set_error("u8_mix_rows_to_nhwc: generic path needs device mean / std arrays"); return COTB200_ENULL; }
  COTB200_DISPATCH_DTYPE(dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      COTB200_PROF_B("u8_mix_rows_to_nhwc", (double)N_out * C * HW * (2.0 + sizeof(T)));
      if (fast) {
        const long long npix4 = (long long)N_out * HW / 4;
        u8_mix_rows_to_nhwc3_kernel<T><<<grid_stride_blocks(npix4, 256, 16), 256, 0, st>>>((const unsigned char*)x_u8, (T*)y, npix4, HW, W, N_in, rows_dev,
                                                                            mean_host[0], mean_host[1], mean_host[2], std_host[0],
                                                                            std_host[1], std_host[2]);
      } else {
        const long long total = (long long)N_out * C * HW;
        u8_mix_rows_to_nhwc_generic_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const unsigned char*)x_u8, (T*)y, total, C, HW, W, N_in,
                                                                                   rows_dev, mean_dev, std_dev);
      }
      return check_launch("u8_mix_rows_to_nhwc");
    }
  });
  return 0;
}

// ------------------------------------------------------------------------------------------------ SE MLP of the CoT tail (eval)
// a[b, c, 0:2] = softmax_r( W3[2c+r, :] . relu(s1 * (W0 . p[b] + b0) + t1) + b3[2c+r] ),  p[b] = psum[b] * inv_hw
// (models/cotnet.py:69-77,92-101 with the BatchNorm of `se` folded: s1 = gamma * rstd, t1 = beta - mean * s1).
// The eager form is ~10 launches of GEMV-sized ops per CoT layer.  Two tiny GEMMs [B, C] x [C, A] and [B, A] x [A, 2C]: the only
// thing that matters is memory-level parallelism, so each is one launch of (16 samples x 32 outputs) tiles whose operands are
// staged in shared memory with independent 16-byte loads (one latency round per 256-wide K chunk) -- one CTA per 2 samples
// walking whole weight rows with dependent loads is latency-bound.
// fp32 throughout.
namespace cotb200 {
static constexpr int SE_TS = 16;     // samples per tile
static constexpr int SE_TJ = 32;     // outputs per tile (16 pairs)
static constexpr int SE_KC = 256;    // K chunk staged per round
static constexpr int SE_LD = SE_KC + 1;

// EPI 0: out[s, j] = relu(s1[j] * (acc + b[j]) + t1[j])            (fc1 + folded BatchNorm + ReLU), in = psum * in_scale
// EPI 1: out[s, c, 0:2] = softmax(acc[2c] + b[2c], acc[2c+1] + b[2c+1])   (fc2 + radix-2 softmax)
template <int EPI>
__global__ void __launch_bounds__(256)
se_fc_kernel(const float* __restrict__ in, float in_scale, const float* __restrict__ Wt, const float* __restrict__ b,
             const float* __restrict__ s1, const float* __restrict__ t1, float* __restrict__ out, int B, int K, int J) {
  extern __shared__ float se_sm[];                 // in tile [SE_TS][SE_LD] | W tile [SE_TJ][SE_LD]
  float* is = se_sm;
  float* ws = se_sm + SE_TS * SE_LD;
  const int s0 = blockIdx.x * SE_TS, j0 = blockIdx.y * SE_TJ;
  const int t = threadIdx.x;
  const int s = t >> 4, pp = t & 15;               // sample of the tile, output pair
  float acc0 = 0.f, acc1 = 0.f;
  for (int k0 = 0; k0 < K; k0 += SE_KC) {
    const int kc = min(SE_KC, K - k0);
    if (k0) __syncthreads();
    // stage: rows of kc floats; 16-byte global loads when the row start allows (K % 4 == 0: always for C % 8 == 0)
    const bool v4 = (K & 3) == 0 && (kc & 3) == 0;
    if (v4) {
      const int q = kc >> 2;
      for (int i = t; i < (SE_TS + SE_TJ) * q; i += 256) {
        const int r = i / q, c4 = (i - r * q) << 2;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        float* dst;
        if (r < SE_TS) {
          if (s0 + r < B) v = __ldg(reinterpret_cast<const float4*>(in + (long long)(s0 + r) * K + k0 + c4));
          v.x *= in_scale; v.y *= in_scale; v.z *= in_scale; v.w *= in_scale;
          dst = is + r * SE_LD + c4;
        } else {
          const int jr = r - SE_TS;
          if (j0 + jr < J) v = __ldg(reinterpret_cast<const float4*>(Wt + (long long)(j0 + jr) * K + k0 + c4));
          dst = ws + jr * SE_LD + c4;
        }
        dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
      }
    } else {
      for (int i = t; i < (SE_TS + SE_TJ) * kc; i += 256) {
        const int r = i / kc, c = i - r * kc;
        if (r < SE_TS) is[r * SE_LD + c] = s0 + r < B ? __ldg(in + (long long)(s0 + r) * K + k0 + c) * in_scale : 0.f;
        else ws[(r - SE_TS) * SE_LD + c] = j0 + r - SE_TS < J ? __ldg(Wt + (long long)(j0 + r - SE_TS) * K + k0 + c) : 0.f;
      }
    }
    __syncthreads();
    const float* ip = is + s * SE_LD;
    const float* w0 = ws + (2 * pp) * SE_LD;
    const float* w1 = w0 + SE_LD;
#pragma unroll 8
    for (int k = 0; k < kc; ++k) {
      const float a = ip[k];
      acc0 = fmaf(a, w0[k], acc0);
      acc1 = fmaf(a, w1[k], acc1);
    }
  }
  const int j = j0 + 2 * pp;
  if (s0 + s >= B || j >= J) return;
  if (EPI == 0) {
    out[(long long)(s0 + s) * J + j] = fmaxf(fmaf(acc0 + (b ? __ldg(b + j) : 0.f), __ldg(s1 + j), __ldg(t1 + j)), 0.f);
    if (j + 1 < J) out[(long long)(s0 + s) * J + j + 1] = fmaxf(fmaf(acc1 + (b ? __ldg(b + j + 1) : 0.f), __ldg(s1 + j + 1), __ldg(t1 + j + 1)), 0.f);
  } else {
    const float u = acc0 + (b ? __ldg(b + j) : 0.f), v = acc1 + (b ? __ldg(b + j + 1) : 0.f);
    const float m = fmaxf(u, v), eu = __expf(u - m), ev = __expf(v - m), inv = 1.f / (eu + ev);
    out[(long long)(s0 + s) * J + j] = eu * inv;             // [B, C, 2] with J = 2C: (c, r) at 2c + r
    out[(long long)(s0 + s) * J + j + 1] = ev * inv;
  }
}
}  // namespace cotb200

extern "C" long long cotb200_se_eval_scratch_bytes(int B, int A) { return (long long)B * A * 4; }

extern "C" int cotb200_se_eval(int B, int C, int A, const float* psum, float inv_hw, const float* W0, const float* b0,
                               const float* s1, const float* t1, const float* W3, const float* b3, float* a, float* z_scratch,
                               void* stream) {
  if (!psum || !W0 || !s1 || !t1 || !W3 || !a || !z_scratch) { set_error("se_eval: NULL pointer"); return COTB200_ENULL; }
  if (B <= 0 || C <= 0 || A <= 0) { set_error("se_eval: non-positive dims"); return COTB200_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const int smem = (SE_TS + SE_TJ) * SE_LD * (int)sizeof(float);      // 49.3 KB
  static PerDevFlag cfgd;
  if (bool& cfg = cfgd.get(); !cfg) {
    cudaError_t e = cudaFuncSetAttribute(se_fc_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(se_fc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
    cfg = true;
  }
  COTB200_PROF("se_eval");
  dim3 g1((B + SE_TS - 1) / SE_TS, (A + SE_TJ - 1) / SE_TJ), g2((B + SE_TS - 1) / SE_TS, (2 * C + SE_TJ - 1) / SE_TJ);
  se_fc_kernel<0><<<g1, 256, smem, st>>>(psum, inv_hw, W0, b0, s1, t1, z_scratch, B, C, A);
  int rc = check_launch("se_eval fc1");
  if (rc) return rc;
  se_fc_kernel<1><<<g2, 256, smem, st>>>(z_scratch, 1.f, W3, b3, nullptr, nullptr, a, B, A, 2 * C);
  return check_launch("se_eval fc2");
}
