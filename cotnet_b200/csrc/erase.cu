// Random erasing of the normalised batch (sm_90a): the reference's RandomErasing (datasets/random_erasing.py), which loops over
// the images in Python and launches a fill per box, as one launch over the boxes the host drew.  Only erased pixels are touched.
//
// Each CTA row (blockIdx.x) is one box; blockIdx.y splits its pixels.  Every pixel is written by exactly one box: a box skips
// the pixels that a later box of the same sample covers, which is what the reference's sequential writes leave there, so the
// result does not depend on which CTA runs first.  The random values are a function of (seed, sample, box, channel, y, x)
// alone (counter-based Philox4x32-10), not of the grid.
#include <curand_kernel.h>

#include "common.cuh"

namespace cotb200 {

static constexpr int ERASE_THREADS = 256;
static constexpr int ERASE_SPLIT = 8;            // CTAs per box

// four N(0,1) values of channels 4*grp .. 4*grp + 3 at counter position pix of box k of sample n
__device__ __forceinline__ float4 erase_normal4(unsigned long long seed, unsigned pix, int n, int k, int grp) {
  const uint4 r = curand_Philox4x32_10(make_uint4(pix, (unsigned)n, (unsigned)k, (unsigned)grp),
                                       make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  const float2 a = _curand_box_muller(r.x, r.y), b = _curand_box_muller(r.z, r.w);
  return make_float4(a.x, a.y, b.x, b.y);
}

template <typename T>
__global__ void __launch_bounds__(ERASE_THREADS)
erase_kernel(const cotb200_erase* __restrict__ hdr, int C, int H, int W, T* __restrict__ y) {
  __shared__ int4 later[COTB200_ERASE_MAX_COUNT];   // top, left, bottom, right of the sample's later boxes
  const cotb200_erase hd = *hdr;
  const cotb200_erase_box* boxes = reinterpret_cast<const cotb200_erase_box*>(hdr + 1);
  const cotb200_erase_box b = boxes[blockIdx.x];
  const int t = threadIdx.x, j = blockIdx.x + 1 + t;
  bool mine = false;
  if (t < COTB200_ERASE_MAX_COUNT && j < hd.n_boxes) {
    const cotb200_erase_box o = boxes[j];
    mine = o.n == b.n;                               // a sample's boxes are consecutive: the later ones are a prefix
    if (mine) later[t] = make_int4(o.top, o.left, o.top + o.h, o.left + o.w);
  }
  const int n_later = __syncthreads_count(mine);
  T* img = y + (long long)b.n * H * W * C;
  const int area = b.h * b.w;
  for (int e = blockIdx.y * blockDim.x + t; e < area; e += gridDim.y * blockDim.x) {
    const int yy = b.top + e / b.w, xx = b.left + e % b.w;
    bool covered = false;
    for (int q = 0; q < n_later; ++q) {
      const int4 o = later[q];
      covered = covered || (yy >= o.x && yy < o.z && xx >= o.y && xx < o.w);
    }
    if (covered) continue;
    T* px = img + ((long long)yy * W + xx) * C;
    for (int g = 0; g < C; g += 4) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (hd.mode) v = erase_normal4(hd.seed, hd.mode == 2 ? (unsigned)(yy * W + xx) : 0xffffffffu, b.n, b.k, g >> 2);
      const float vv[4] = {v.x, v.y, v.z, v.w};
      for (int q = 0; q < 4 && g + q < C; ++q) px[g + q] = Elem<T>::from(vv[q]);
    }
  }
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_aug_erase(int dtype, int N, int C, int H, int W, void* y, const cotb200_erase* erase_host,
                                 const cotb200_erase* erase_dev, void* stream) {
  if (!erase_host) { set_error("aug_erase: erase_host is NULL"); return COTB200_ENULL; }
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("aug_erase: non-positive dims"); return COTB200_EINVAL; }
  if (dtype != COTB200_F32 && dtype != COTB200_BF16 && dtype != COTB200_F16) {
    set_error("aug_erase: dtype %d is not fp32, bf16 or fp16", dtype); return COTB200_EDTYPE;
  }
  const cotb200_erase& hd = *erase_host;
  if (hd.mode < 0 || hd.mode > 2) { set_error("aug_erase: unknown mode %d (0 const, 1 rand, 2 pixel)", hd.mode); return COTB200_EINVAL; }
  if (hd.n_boxes < 0 || (long long)hd.n_boxes > (long long)N * COTB200_ERASE_MAX_COUNT) {
    set_error("aug_erase: %d boxes for %d samples", hd.n_boxes, N); return COTB200_EINVAL;
  }
  const cotb200_erase_box* boxes = reinterpret_cast<const cotb200_erase_box*>(erase_host + 1);
  long long area = 0;
  for (int i = 0; i < hd.n_boxes; ++i) {
    const cotb200_erase_box& b = boxes[i];
    const int prev = i ? boxes[i - 1].n : -1, next_k = i && prev == b.n ? boxes[i - 1].k + 1 : 0;
    if (b.n < 0 || b.n >= N || b.n < prev || b.k != next_k) {
      set_error("aug_erase: box %d (sample %d, index %d) out of order or outside the batch of %d", i, b.n, b.k, N); return COTB200_EINVAL;
    }
    if (b.k >= COTB200_ERASE_MAX_COUNT) {
      set_error("aug_erase: sample %d has more than %d boxes", b.n, COTB200_ERASE_MAX_COUNT); return COTB200_EINVAL;
    }
    if (b.top < 0 || b.left < 0 || b.h < 1 || b.w < 1 || b.h > H - b.top || b.w > W - b.left) {
      set_error("aug_erase: box %d (%d, %d, %d, %d) outside the %dx%d image", i, b.top, b.left, b.h, b.w, H, W); return COTB200_EINVAL;
    }
    area += (long long)b.h * b.w;
  }
  if (!hd.n_boxes) return 0;
  if (!y || !erase_dev) { set_error("aug_erase: NULL pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(hd.n_boxes, ERASE_SPLIT);
  COTB200_PROF_B("aug_erase", (double)area * C * (dtype == COTB200_F32 ? 4.0 : 2.0));
  if (dtype == COTB200_F32) erase_kernel<float><<<grid, ERASE_THREADS, 0, st>>>(erase_dev, C, H, W, (float*)y);
  else if (dtype == COTB200_BF16) erase_kernel<__nv_bfloat16><<<grid, ERASE_THREADS, 0, st>>>(erase_dev, C, H, W, (__nv_bfloat16*)y);
  else erase_kernel<__half><<<grid, ERASE_THREADS, 0, st>>>(erase_dev, C, H, W, (__half*)y);
  return check_launch("aug_erase");
}
