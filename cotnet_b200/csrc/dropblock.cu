// DropBlock (models/layers/drop.py:drop_block_fast_2d) on NHWC tensors (sm_90a).
//
// The mask of one site is drawn, max-pooled and counted on the device, so a captured training step draws a new mask at every
// replay.  The random stream is the library's own (include/cotb200.h, "DropBlock"): Philox4x32-10 keyed by two words read from
// device memory, counter (q mod 2^32, q >> 32, site, 0) with q = e >> 2 of the element's logical NCHW index e.
//
//   cotb200_dropblock_mask     one CTA per (sample, group of 8*NG channels): the CTA's elements are one contiguous range of
//                              NCHW indices, so each Philox call feeds four of them.  Seeds land as bits in shared memory
//                              (byte per pixel and 8 channels), a separable clipped OR pools them, the keep bits go out in
//                              the [B*H*W, C/8] layout of the fused BatchNorm's 1-bit ReLU masks and the CTA adds its kept
//                              count to one int32 with an integer atomic (exact, order-free).
//   cotb200_dropblock_apply    y = x * M * s, s = fp32(numel) * (1 / (fp32(count) + 1e-7)) rounded to the activation dtype.
//   cotb200_dropblock_res_relu out = relu(res + ds[b] * (z * M * s)), fp32 math and one rounding, and its 1-bit ReLU mask.
#include "common.cuh"

namespace cotb200 {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const unsigned lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const unsigned lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

__device__ __forceinline__ float dropblock_scale(const int* count, long long numel) {
  return __fmul_rn((float)numel, __frcp_rn(__fadd_rn(__int2float_rn(__ldg(count)), 1e-7f)));
}

template <typename T>
__device__ __forceinline__ float dropblock_scale_as(const int* count, long long numel) {
  return to_acc(Elem<T>::from(dropblock_scale(count, numel)));
}

constexpr int DB_THREADS = 256;
// The mask kernel's shared memory is all dynamic (no static __shared__), so this is its whole footprint: the per-warp kept
// counts, then 2*nb bytes of planes; at most the 48 KB a kernel may use without opting in to more.
constexpr int DB_KEPT_BYTES = DB_THREADS / 32 * (int)sizeof(int);
constexpr int DB_SMEM_MAX = 48 * 1024;
__host__ __device__ constexpr long long db_mask_smem(long long nb) { return DB_KEPT_BYTES + 2 * nb; }

// smem: the per-warp kept counts, the seeds [HW][NG] bytes (bit j of byte (p, g) = channel c0 + 8g + j), then the row-pooled
// copy.  nb = NG*HW rounded up to 4.
__global__ void __launch_bounds__(DB_THREADS)
dropblock_mask_kernel(int C, int H, int W, int NG, int cbs, float gamma, unsigned site, const long long* __restrict__ key,
                      unsigned char* __restrict__ mask, int* __restrict__ count, int nb) {
  extern __shared__ __align__(16) unsigned char db_smem[];
  int* s_kept = reinterpret_cast<int*>(db_smem);
  unsigned char* seed = db_smem + DB_KEPT_BYTES;
  unsigned char* rowp = seed + nb;
  const int HW = H * W, b = blockIdx.y, g0 = blockIdx.x * NG, C8 = C / 8;
  for (int i = threadIdx.x; i < nb / 4; i += DB_THREADS) reinterpret_cast<unsigned*>(seed)[i] = 0u;
  __syncthreads();
  const uint2 k = make_uint2((unsigned)__ldg(key), (unsigned)__ldg(key + 1));
  const long long e0 = ((long long)b * C + 8LL * g0) * HW, e1 = e0 + 8LL * NG * HW;
  for (long long q = (e0 >> 2) + threadIdx.x; q <= ((e1 - 1) >> 2); q += DB_THREADS) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)q, (unsigned)(q >> 32), site, 0u), k);
    const unsigned rl[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      const long long e = 4 * q + l;
      if (e < e0 || e >= e1) continue;
      if (!(__uint2float_rn(rl[l] >> 8) * 5.9604644775390625e-8f < gamma)) continue;
      const int off = (int)(e - e0), ch = off / HW, p = off - ch * HW;
      const int bi = p * NG + (ch >> 3);
      atomicOr(reinterpret_cast<unsigned*>(seed) + (bi >> 2), (1u << (ch & 7)) << ((bi & 3) * 8));
    }
  }
  __syncthreads();
  const int pad = cbs / 2;
  for (int i = threadIdx.x; i < NG * HW; i += DB_THREADS) {      // OR along the row, window clipped to the image
    const int g = i % NG, p = i / NG, h = p / W, w = p - h * W;
    unsigned v = 0;
    for (int ww = max(0, w - pad); ww <= min(W - 1, w + pad); ++ww) v |= seed[(h * W + ww) * NG + g];
    rowp[i] = (unsigned char)v;
  }
  __syncthreads();
  int kept = 0;
  const long long row0 = (long long)b * HW;
  for (int i = threadIdx.x; i < NG * HW; i += DB_THREADS) {      // then along the column; keep = NOT dropped
    const int g = i % NG, p = i / NG, h = p / W, w = p - h * W;
    unsigned v = 0;
    for (int hh = max(0, h - pad); hh <= min(H - 1, h + pad); ++hh) v |= rowp[(hh * W + w) * NG + g];
    const unsigned keep = ~v & 0xFFu;
    mask[(row0 + p) * C8 + g0 + g] = (unsigned char)keep;
    kept += __popc(keep);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
  if ((threadIdx.x & 31) == 0) s_kept[threadIdx.x >> 5] = kept;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
#pragma unroll
    for (int i = 0; i < DB_THREADS / 32; ++i) t += s_kept[i];
    atomicAdd(count, t);
  }
}

// One thread per packet of 8 channels of one pixel: packet i covers elements [8i, 8i + 8) of the NHWC tensor and is bit-for-bit
// byte i of a [B*H*W, C/8] mask (C % 8 == 0).  16-bit types move a packet with one 16-byte access, fp32 with two.
template <typename T>
__device__ __forceinline__ void ld8(const T* __restrict__ p, float (&f)[8]) {
  constexpr int VEC = 16 / sizeof(T);
#pragma unroll
  for (int h = 0; h < 8 / VEC; ++h) {
    const Pack<T, VEC> v = ld_pack<T, VEC>(p + h * VEC);
#pragma unroll
    for (int j = 0; j < VEC; ++j) f[h * VEC + j] = to_acc(v.v[j]);
  }
}

template <typename T>
__device__ __forceinline__ void st8(T* __restrict__ p, const float (&f)[8]) {
  constexpr int VEC = 16 / sizeof(T);
#pragma unroll
  for (int h = 0; h < 8 / VEC; ++h) {
    Pack<T, VEC> v;
#pragma unroll
    for (int j = 0; j < VEC; ++j) v.v[j] = Elem<T>::from(f[h * VEC + j]);
    st_pack<T, VEC>(p + h * VEC, v);
  }
}

template <typename T>
__global__ void __launch_bounds__(DB_THREADS)
dropblock_apply_kernel(const T* __restrict__ x, const unsigned char* __restrict__ m, const int* __restrict__ count,
                       long long numel, T* __restrict__ y, long long npk) {
  const float s = dropblock_scale_as<T>(count, numel);
  for (long long i = blockIdx.x * (long long)DB_THREADS + threadIdx.x; i < npk; i += (long long)gridDim.x * DB_THREADS) {
    float v[8];
    ld8<T>(x + i * 8, v);
    const unsigned bits = __ldg(m + i);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = __fmul_rn(__fmul_rn(v[j], (float)(bits >> j & 1u)), s);   // (x * M) * s, as torch: -0 stays -0
    st8<T>(y + i * 8, v);
  }
}

template <typename T, bool DS>
__global__ void __launch_bounds__(DB_THREADS)
dropblock_res_relu_kernel(const T* __restrict__ z, const T* __restrict__ res, const unsigned char* __restrict__ m,
                          const int* __restrict__ count, long long numel, const float* __restrict__ ds, long long sample_elems,
                          T* __restrict__ y, unsigned char* __restrict__ rmask, long long npk) {
  const float s = dropblock_scale_as<T>(count, numel);
  for (long long i = blockIdx.x * (long long)DB_THREADS + threadIdx.x; i < npk; i += (long long)gridDim.x * DB_THREADS) {
    float v[8], r[8];
    ld8<T>(z + i * 8, v);
    ld8<T>(res + i * 8, r);
    const unsigned bits = __ldg(m + i);
    const float d = DS ? __ldg(ds + i * 8 / sample_elems) : 1.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float a = (bits >> j & 1u) ? __fmul_rn(v[j], s) : 0.f;
      v[j] = fmaxf(DS ? __fmaf_rn(a, d, r[j]) : __fadd_rn(a, r[j]), 0.f);
    }
    st8<T>(y + i * 8, v);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = to_acc(Elem<T>::from(v[j]));
    unsigned rb = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) rb |= (o[j] > 0.f ? 1u : 0u) << j;
    rmask[i] = (unsigned char)rb;
  }
}

// dres = dy * [out > 0], dz = dres * ds[b] * M * s
template <typename T, bool DS>
__global__ void __launch_bounds__(DB_THREADS)
dropblock_res_relu_bwd_kernel(const T* __restrict__ dy, const unsigned char* __restrict__ rmask, const unsigned char* __restrict__ m,
                              const int* __restrict__ count, long long numel, const float* __restrict__ ds, long long sample_elems,
                              T* __restrict__ dres, T* __restrict__ dz, long long npk) {
  const float s = dropblock_scale_as<T>(count, numel);
  for (long long i = blockIdx.x * (long long)DB_THREADS + threadIdx.x; i < npk; i += (long long)gridDim.x * DB_THREADS) {
    float g[8], o[8];
    ld8<T>(dy + i * 8, g);
    const unsigned bits = __ldg(m + i), rb = __ldg(rmask + i);
    const float d = DS ? __ldg(ds + i * 8 / sample_elems) : 1.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      g[j] = (rb >> j & 1u) ? g[j] : 0.f;
      const float a = (bits >> j & 1u) ? __fmul_rn(g[j], s) : 0.f;
      o[j] = DS ? __fmul_rn(a, d) : a;
    }
    if (dres) st8<T>(dres + i * 8, g);
    st8<T>(dz + i * 8, o);
  }
}

// shared checks of the elementwise entry points: B*HW*C elements of a 16-bit or fp32 NHWC tensor, C % 8 == 0
static int db_rows_check(const char* what, int dtype, int B, int HW, int C) {
  if (B <= 0 || HW <= 0 || C <= 0 || C % 8) { set_error("%s: bad geometry B=%d HW=%d C=%d (C %% 8 == 0)", what, B, HW, C); return COTB200_EINVAL; }
  if (dtype != COTB200_F32 && dtype != COTB200_BF16 && dtype != COTB200_F16) { set_error("%s: dtype %d not supported", what, dtype); return COTB200_EDTYPE; }
  if ((long long)B * HW * C > 2147483647LL) { set_error("%s: more than 2^31 - 1 elements", what); return COTB200_ETOOBIG; }
  return 0;
}

// the three activation dtypes (fp64 is rejected by db_rows_check before this)
#define DB_DISPATCH(dtype, ...)                                                  \
  switch (dtype) {                                                               \
    case COTB200_F32:  { using T = float;         __VA_ARGS__; } break;          \
    case COTB200_BF16: { using T = __nv_bfloat16; __VA_ARGS__; } break;          \
    default:           { using T = __half;        __VA_ARGS__; } break;          \
  }

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_dropblock_mask(int B, int C, int H, int W, int cbs, float gamma, int site, const long long* key,
                                      void* mask, int* count, void* stream) {
  if (!key || !mask || !count) { set_error("dropblock_mask: NULL pointer"); return COTB200_ENULL; }
  if (((uintptr_t)count & 3) || ((uintptr_t)key & 7)) { set_error("dropblock_mask: count must be 4-byte and key 8-byte aligned"); return COTB200_EALIGN; }
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || C % 8 || site < 0) {
    set_error("dropblock_mask: bad geometry B=%d C=%d H=%d W=%d site=%d (C %% 8 == 0)", B, C, H, W, site); return COTB200_EINVAL; }
  if (cbs < 1 || !(cbs & 1) || cbs > H || cbs > W) {
    set_error("dropblock_mask: block size %d must be odd and fit the %dx%d plane", cbs, H, W); return COTB200_EINVAL; }
  if (gamma != gamma) { set_error("dropblock_mask: gamma is NaN"); return COTB200_EINVAL; }   // < 0: no seeds, >= 1: all (as the reference)
  if ((long long)B * C * H * W > 2147483647LL) { set_error("dropblock_mask: more than 2^31 - 1 elements"); return COTB200_ETOOBIG; }
  const int C8 = C / 8, HW = H * W;
  int NG = 16;
  const uintptr_t m0 = (uintptr_t)mask, c0 = (uintptr_t)count;
  if (c0 + sizeof(int) > m0 && c0 < m0 + (uintptr_t)B * HW * C8) { set_error("dropblock_mask: count lies inside the mask"); return COTB200_EINVAL; }
  while (NG > 1 && (C8 % NG || db_mask_smem(((long long)NG * HW + 3) & ~3LL) > DB_SMEM_MAX)) NG >>= 1;
  const long long nb = ((long long)NG * HW + 3) & ~3LL;
  if (db_mask_smem(nb) > DB_SMEM_MAX) {        // NG == 1: planes above (DB_SMEM_MAX - DB_KEPT_BYTES) / 2 = 24560 pixels
    set_error("dropblock_mask: a %dx%d plane exceeds the kernel's shared memory", H, W); return COTB200_EUNSUPPORTED; }
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid((unsigned)(C8 / NG), (unsigned)B);
  COTB200_PROF_B("dropblock_mask", (double)B * HW * C8);
  dropblock_mask_kernel<<<grid, DB_THREADS, (size_t)db_mask_smem(nb), st>>>(C, H, W, NG, cbs, gamma, (unsigned)site, key, (unsigned char*)mask, count, (int)nb);
  return check_launch("dropblock_mask");
}

extern "C" int cotb200_dropblock_apply(int dtype, int B, int HW, int C, const void* x, const void* mask, const int* count, void* y,
                                       void* stream) {
  if (!x || !mask || !count || !y) { set_error("dropblock_apply: NULL pointer"); return COTB200_ENULL; }
  if (int rc = db_rows_check("dropblock_apply", dtype, B, HW, C)) return rc;
  if (!aligned16(x) || !aligned16(y)) { set_error("dropblock_apply: x and y must be 16-byte aligned"); return COTB200_EALIGN; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * HW * C;
  DB_DISPATCH(dtype, {
    {
      const long long npk = n / 8;
      COTB200_PROF_B("dropblock_apply", (double)n * (2 * sizeof(T)) + n / 8.0);
      dropblock_apply_kernel<T><<<grid_stride_blocks(npk, DB_THREADS, 16), DB_THREADS, 0, st>>>((const T*)x, (const unsigned char*)mask, count, n, (T*)y, npk);
      return check_launch("dropblock_apply");
    }
  });
  return 0;
}

extern "C" int cotb200_dropblock_res_relu(int dtype, int B, int HW, int C, const void* z, const void* res, const void* mask,
                                          const int* count, const float* ds, void* y, void* relu_mask, void* stream) {
  if (!z || !res || !mask || !count || !y || !relu_mask) { set_error("dropblock_res_relu: NULL pointer"); return COTB200_ENULL; }
  if (int rc = db_rows_check("dropblock_res_relu", dtype, B, HW, C)) return rc;
  if (!aligned16(z) || !aligned16(res) || !aligned16(y)) { set_error("dropblock_res_relu: z, res and y must be 16-byte aligned"); return COTB200_EALIGN; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * HW * C, per = (long long)HW * C;
  DB_DISPATCH(dtype, {
    {
      const long long npk = n / 8;
      COTB200_PROF_B("dropblock_res_relu", (double)n * (3 * sizeof(T)) + n / 4.0);
      if (ds) dropblock_res_relu_kernel<T, true><<<grid_stride_blocks(npk, DB_THREADS, 16), DB_THREADS, 0, st>>>(
          (const T*)z, (const T*)res, (const unsigned char*)mask, count, n, ds, per, (T*)y, (unsigned char*)relu_mask, npk);
      else dropblock_res_relu_kernel<T, false><<<grid_stride_blocks(npk, DB_THREADS, 16), DB_THREADS, 0, st>>>(
          (const T*)z, (const T*)res, (const unsigned char*)mask, count, n, ds, per, (T*)y, (unsigned char*)relu_mask, npk);
      return check_launch("dropblock_res_relu");
    }
  });
  return 0;
}

extern "C" int cotb200_dropblock_res_relu_bwd(int dtype, int B, int HW, int C, const void* dy, const void* relu_mask, const void* mask,
                                              const int* count, const float* ds, void* dres, void* dz, void* stream) {
  if (!dy || !relu_mask || !mask || !count || !dz) { set_error("dropblock_res_relu_bwd: NULL pointer"); return COTB200_ENULL; }
  if (int rc = db_rows_check("dropblock_res_relu_bwd", dtype, B, HW, C)) return rc;
  if (!aligned16(dy) || !aligned16(dz) || (dres && !aligned16(dres))) {
    set_error("dropblock_res_relu_bwd: dy, dres and dz must be 16-byte aligned"); return COTB200_EALIGN; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * HW * C, per = (long long)HW * C;
  DB_DISPATCH(dtype, {
    {
      const long long npk = n / 8;
      COTB200_PROF_B("dropblock_res_relu_bwd", (double)n * ((dres ? 3 : 2) * sizeof(T)) + n / 4.0);
      if (ds) dropblock_res_relu_bwd_kernel<T, true><<<grid_stride_blocks(npk, DB_THREADS, 16), DB_THREADS, 0, st>>>(
          (const T*)dy, (const unsigned char*)relu_mask, (const unsigned char*)mask, count, n, ds, per, (T*)dres, (T*)dz, npk);
      else dropblock_res_relu_bwd_kernel<T, false><<<grid_stride_blocks(npk, DB_THREADS, 16), DB_THREADS, 0, st>>>(
          (const T*)dy, (const unsigned char*)relu_mask, (const unsigned char*)mask, count, n, ds, per, (T*)dres, (T*)dz, npk);
      return check_launch("dropblock_res_relu_bwd");
    }
  });
  return 0;
}
