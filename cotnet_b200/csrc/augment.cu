// Image augmentation of the reference's input pipeline (sm_90a), byte-equal to its PIL transforms given the same draws:
// RandomResizedCrop + RandomHorizontalFlip + RandAugment (datasets/transforms_factory.py:44-129) and the eval
// Resize + CenterCrop (:132-166), on a ragged batch of decoded uint8 HWC images.
//
// Resize-crop is Pillow's two-pass resample (Resample.c): per output index, weights from the filter at
// support * max(scale, 1) around center = (i + 0.5) * scale, normalised in double and rounded to 22-bit fixed point, then
// (2^21 + sum w * x) >> 22 clipped to uint8; the horizontal pass runs first and its uint8 rows are the vertical pass's input.
// A pass whose size does not change has the weights {0, 2^22, 0, ...}: running it is byte-identical to Pillow skipping it.
// Pillow's weights depend only on the output index, so only the rows and columns of the output window are computed (the eval
// center crop, a flip mirrors the window's columns).  All double arithmetic goes through __d*_rn so that nothing is
// contracted to FMA (Pillow's C is compiled without it); the fp32 arithmetic of Image.blend and the SMOOTH filter likewise.
//
// RandAugment runs one CTA per image with the S x S x 3 image in shared memory (150,528 B at S = 224): histograms, the L mean
// and the LUTs are built there and the image is written to HBM once.  Ops that read neighbours (Sharpness, the affine ops)
// read the previous state from the output buffer in global memory and write shared memory.
//
// ColorJitter (+ RandomVerticalFlip), the reference's colour transform when RandAugment is off, runs the same way: one CTA per
// image in shared memory, between resize-crop and RandAugment, sharing RandAugment's enhance blends.
//
// Both have a second kernel for images up to 512 x 512 that do not fit one CTA's shared memory: one thread-block cluster of up
// to 4 CTAs per image, each holding a band of rows, with the same per-pixel arithmetic (the *_cluster entry points).
#include <cooperative_groups.h>

#include "common.cuh"

namespace cotb200 {

static constexpr int AUG_THREADS = 256;
static constexpr int AUG_HGRID = 8;           // CTAs per image of the horizontal pass
static constexpr int AUG_VROWS = 8;           // output rows per CTA of the vertical pass
static constexpr int RA_THREADS = 1024;
static constexpr int RA_MAX_S = 256;
static constexpr int AUG_MAX_SMEM = 200 * 1024;
static constexpr int PREC = 22;

enum { OP_AUTOCONTRAST = 0, OP_EQUALIZE, OP_INVERT, OP_ROTATE, OP_POSTERIZE, OP_SOLARIZE, OP_SOLARIZEADD, OP_COLOR,
       OP_CONTRAST, OP_BRIGHTNESS, OP_SHARPNESS, OP_SHEARX, OP_SHEARY, OP_TRANSLATEX, OP_TRANSLATEY, OP_CUTOUT, OP_COUNT };

__host__ __device__ inline bool is_affine(int op) { return op == OP_ROTATE || (op >= OP_SHEARX && op <= OP_TRANSLATEY); }

// ---------------------------------------------------------------- Pillow resample weights (precompute_coeffs + normalize_coeffs_8bpc)
struct Axis { double scale, sup, ss; int ksize, in; };

__host__ __device__ inline int axis_ksize(int in, int out, int filt) {
  double scale = (double)in / (double)out;            // one IEEE division: identical on host and device
  double fs = scale < 1.0 ? 1.0 : scale;
  return (int)ceil((filt ? 2.0 : 1.0) * fs) * 2 + 1;
}

__device__ __forceinline__ Axis make_axis(int in, int out, int filt) {
  Axis a;
  a.in = in;
  a.scale = __ddiv_rn((double)in, (double)out);
  const double fs = a.scale < 1.0 ? 1.0 : a.scale;
  a.sup = __dmul_rn(filt ? 2.0 : 1.0, fs);
  a.ksize = (int)ceil(a.sup) * 2 + 1;
  a.ss = __ddiv_rn(1.0, fs);
  return a;
}

__device__ __forceinline__ double filter_fn(double x, int filt) {
  if (x < 0.0) x = -x;
  if (!filt) return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
  if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);   // a = -0.5
  if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
  return 0.0;
}

__device__ __forceinline__ void axis_bounds(const Axis& a, int idx, double& center, int& xmin, int& xmax) {
  center = __dmul_rn(__dadd_rn((double)idx, 0.5), a.scale);
  xmin = (int)__dadd_rn(__dsub_rn(center, a.sup), 0.5);
  if (xmin < 0) xmin = 0;
  xmax = (int)__dadd_rn(__dadd_rn(center, a.sup), 0.5);
  if (xmax > a.in) xmax = a.in;
  xmax -= xmin;
}

// weights of output index idx into k[0..ksize) (zero past xmax); returns xmin
__device__ int axis_weights(const Axis& a, int filt, int idx, int* k) {
  double center;
  int xmin, xmax;
  axis_bounds(a, idx, center, xmin, xmax);
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x) ww = __dadd_rn(ww, filter_fn(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), a.ss), filt));
  for (int x = 0; x < a.ksize; ++x) {
    double w = 0.0;
    if (x < xmax) {
      w = filter_fn(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), a.ss), filt);
      if (ww != 0.0) w = __ddiv_rn(w, ww);
    }
    const double s = __dmul_rn(w, (double)(1 << PREC));
    k[x] = w < 0 ? (int)__dadd_rn(-0.5, s) : (int)__dadd_rn(0.5, s);
  }
  return xmin;
}

__device__ __forceinline__ unsigned char clip8(int acc) {
  acc >>= PREC;
  return (unsigned char)(acc < 0 ? 0 : acc > 255 ? 255 : acc);
}

// crop rows [r0, r1) that the vertical pass reads for the output window rows [oi, oi + S)
__device__ __forceinline__ void needed_rows(const cotb200_aug_sample& p, int S, int& r0, int& r1) {
  const Axis av = make_axis(p.ch, p.rh, p.filter);
  double c;
  int xmin, xmax;
  axis_bounds(av, p.oi, c, xmin, xmax);
  r0 = xmin;
  axis_bounds(av, p.oi + S - 1, c, xmin, xmax);
  r1 = xmin + xmax;
}

// ---------------------------------------------------------------- pass 1: horizontal, source rows -> tmp [3][ch][S]
__global__ void __launch_bounds__(AUG_THREADS)
aug_hpass_kernel(const unsigned char* __restrict__ src, const cotb200_aug_sample* __restrict__ params, int S, int kmax,
                 unsigned char* __restrict__ tmp) {
  extern __shared__ int sm_h[];                       // [S] xmin, then [S][kmax] weights
  const cotb200_aug_sample p = params[blockIdx.x];
  const Axis ah = make_axis(p.cw, p.rw, p.filter);
  int* xmin = sm_h;
  int* k = sm_h + S;
  for (int x = threadIdx.x; x < S; x += blockDim.x) {
    const int col = p.oj + (p.flip ? S - 1 - x : x);
    xmin[x] = axis_weights(ah, p.filter, col, k + x * kmax);
  }
  __syncthreads();
  int r0, r1;
  needed_rows(p, S, r0, r1);
  const unsigned char* img = src + p.offset;
  unsigned char* t = tmp + p.tmp_offset;
  const long long plane = (long long)p.ch * S;
  const int nr = r1 - r0;
  for (int e = blockIdx.y * blockDim.x + threadIdx.x; e < nr * S; e += gridDim.y * blockDim.x) {
    const int r = r0 + e / S, x = e % S;
    const unsigned char* row = img + ((long long)(p.ci + r) * p.w + p.cj + xmin[x]) * 3;
    const int* kx = k + x * kmax;
    int a0 = 1 << (PREC - 1), a1 = a0, a2 = a0;
    for (int q = 0; q < ah.ksize; ++q) {
      const int w = kx[q];
      if (w) { a0 += row[3 * q] * w; a1 += row[3 * q + 1] * w; a2 += row[3 * q + 2] * w; }
    }
    const long long o = (long long)r * S + x;
    t[o] = clip8(a0);
    t[plane + o] = clip8(a1);
    t[2 * plane + o] = clip8(a2);
  }
}

// ---------------------------------------------------------------- pass 2: vertical, tmp -> out [3][S][S]
__global__ void __launch_bounds__(AUG_THREADS)
aug_vpass_kernel(const unsigned char* __restrict__ tmp, const cotb200_aug_sample* __restrict__ params, int S, int kmax,
                 unsigned char* __restrict__ out) {
  extern __shared__ int sm_v[];                       // [AUG_VROWS] ymin, then [AUG_VROWS][kmax] weights
  const cotb200_aug_sample p = params[blockIdx.x];
  const Axis av = make_axis(p.ch, p.rh, p.filter);
  const int y0 = blockIdx.y * AUG_VROWS;
  const int ny = min(AUG_VROWS, S - y0);
  int* ymin = sm_v;
  int* k = sm_v + AUG_VROWS;
  if (threadIdx.x < ny) ymin[threadIdx.x] = axis_weights(av, p.filter, p.oi + y0 + threadIdx.x, k + threadIdx.x * kmax);
  __syncthreads();
  const unsigned char* t = tmp + p.tmp_offset;
  const long long plane = (long long)p.ch * S;
  unsigned char* o = out + (long long)blockIdx.x * 3 * S * S;
  for (int e = threadIdx.x; e < ny * S; e += blockDim.x) {
    const int yy = e / S, x = e % S;
    const int* ky = k + yy * kmax;
    const unsigned char* col = t + (long long)ymin[yy] * S + x;
    int a0 = 1 << (PREC - 1), a1 = a0, a2 = a0;
    for (int q = 0; q < av.ksize; ++q) {
      const int w = ky[q];
      if (w) {
        const long long i = (long long)q * S;
        a0 += col[i] * w; a1 += col[plane + i] * w; a2 += col[2 * plane + i] * w;
      }
    }
    const long long d = (long long)(y0 + yy) * S + x;
    o[d] = clip8(a0);
    o[(long long)S * S + d] = clip8(a1);
    o[2LL * S * S + d] = clip8(a2);
  }
}

// ---------------------------------------------------------------- RandAugment
__device__ __forceinline__ unsigned char blend_px(int a, int b, float alpha) {          // Image.blend(a, b, alpha), Blend.c
  const float t = __fadd_rn((float)a, __fmul_rn(alpha, (float)(b - a)));
  return t <= 0.f ? 0 : t >= 255.f ? 255 : (unsigned char)t;
}

__device__ __forceinline__ int l_of(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

// Geometry.c: BICUBIC(v, v1, v2, v3, v4, d) with a = -1; first stage on uint8 (the p's in int), second on doubles
__device__ __forceinline__ double cubic_i(int v1, int v2, int v3, int v4, double d) {
  const int p2 = -v1 + v3, p3 = 2 * (v1 - v2) + v3 - v4, p4 = -v1 + v2 - v3 + v4;
  return __dadd_rn((double)v2, __dmul_rn(d, __dadd_rn((double)p2, __dmul_rn(d, __dadd_rn((double)p3, __dmul_rn(d, (double)p4))))));
}
__device__ __forceinline__ double cubic_d(double v1, double v2, double v3, double v4, double d) {
  const double p2 = __dadd_rn(-v1, v3);
  const double p3 = __dsub_rn(__dadd_rn(__dmul_rn(2.0, __dsub_rn(v1, v2)), v3), v4);
  const double p4 = __dadd_rn(__dsub_rn(__dadd_rn(-v1, v2), v3), v4);
  return __dadd_rn(v2, __dmul_rn(d, __dadd_rn(p2, __dmul_rn(d, __dadd_rn(p3, __dmul_rn(d, p4))))));
}

// img.transform(size, AFFINE, m, filter, fillcolor) of one output pixel from the S x S planar image g
__device__ unsigned char affine_px(const unsigned char* g, int S, int c, const cotb200_aug_op& op, int x, int y, int fill) {
  const double xo = (double)x + 0.5, yo = (double)y + 0.5;
  double xin = __dadd_rn(__dadd_rn(__dmul_rn(op.m[0], xo), __dmul_rn(op.m[1], yo)), op.m[2]);
  double yin = __dadd_rn(__dadd_rn(__dmul_rn(op.m[3], xo), __dmul_rn(op.m[4], yo)), op.m[5]);
  if (!(xin >= 0.0 && xin < (double)S && yin >= 0.0 && yin < (double)S)) return (unsigned char)fill;
  xin = __dsub_rn(xin, 0.5);
  yin = __dsub_rn(yin, 0.5);
  int xi = (int)floor(xin), yi = (int)floor(yin);
  const double dx = __dsub_rn(xin, (double)xi), dy = __dsub_rn(yin, (double)yi);
  const unsigned char* pl = g + (long long)c * S * S;
  auto px = [&](int row, int col) -> int { return pl[(long long)row * S + col]; };
  auto xc = [&](int v) { return v < 0 ? 0 : v < S ? v : S - 1; };
  if (op.filter) {
    xi -= 1;
    yi -= 1;
    const int x0 = xc(xi), x1 = xc(xi + 1), x2 = xc(xi + 2), x3 = xc(xi + 3);
    double v[4];
    for (int q = 0; q < 4; ++q) {
      const int row = yi + q;
      if (q == 0 || (row >= 0 && row < S)) {
        const int rr = xc(row);
        v[q] = cubic_i(px(rr, x0), px(rr, x1), px(rr, x2), px(rr, x3), dx);
      } else {
        v[q] = v[q - 1];
      }
    }
    const double r = cubic_d(v[0], v[1], v[2], v[3], dy);
    return r <= 0.0 ? 0 : r >= 255.0 ? 255 : (unsigned char)r;
  }
  const int x0 = xc(xi), x1 = xc(xi + 1);
  const int r0 = xc(yi);
  const double v1 = __dadd_rn((double)px(r0, x0), __dmul_rn((double)(px(r0, x1) - px(r0, x0)), dx));
  double v2 = v1;
  if (yi + 1 >= 0 && yi + 1 < S) v2 = __dadd_rn((double)px(yi + 1, x0), __dmul_rn((double)(px(yi + 1, x1) - px(yi + 1, x0)), dx));
  const double r = __dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy));
  return r <= 0.0 ? 0 : r >= 255.0 ? 255 : (unsigned char)r;
}

// ImageFilter.SMOOTH of one interior pixel (Filter.c 3x3: rows y+1, y, y-1 in that order, fp32, rounded +0.5)
__device__ __forceinline__ int smooth_px(const unsigned char* pl, int S, int x, int y) {
  const float k1 = 1.f / 13.f, k5 = 5.f / 13.f;
  float ss = 0.f;
  for (int dy = 1; dy >= -1; --dy) {
    const unsigned char* r = pl + (long long)(y + dy) * S + x;
    const float kc = dy == 0 ? k5 : k1;
    ss = __fadd_rn(ss, __fadd_rn(__fadd_rn(__fmul_rn((float)r[-1], k1), __fmul_rn((float)r[0], kc)), __fmul_rn((float)r[1], k1)));
  }
  return ss <= 0.f ? 0 : ss >= 255.f ? 255 : (int)__fadd_rn(ss, 0.5f);
}

// The enhance blends work on n pixels of a planar image img [3][plane] in shared memory (the whole image, or one CTA's band of
// rows in the cluster kernels).  Every thread of the CTA calls these.
// Sum of L over the n pixels into the shared word *lsum; ends with the CTA synchronised.
__device__ void l_sum(const unsigned char* img, int plane, int n, unsigned long long* lsum) {
  if (threadIdx.x == 0) *lsum = 0;
  __syncthreads();
  unsigned long long part = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) part += l_of(img[i], img[plane + i], img[2 * plane + i]);
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(lsum, part);
  __syncthreads();
}

// int(mean(L) + 0.5) of an image of n_pix pixels whose L values sum to `sum` (ImageEnhance.Contrast's degenerate)
__device__ __forceinline__ int contrast_mean(unsigned long long sum, int n_pix) {
  return (int)__dadd_rn(__ddiv_rn((double)sum, (double)n_pix), 0.5);
}

// ImageEnhance.Color / Contrast / Brightness (op OP_COLOR, OP_CONTRAST, OP_BRIGHTNESS) in place: Image.blend(degenerate, img,
// factor) with the degenerate L (Color), `mean` (Contrast) or 0 (Brightness).  Ends with the CTA synchronised.
__device__ void enhance_apply(unsigned char* img, int plane, int n, int op, float factor, int mean) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int r = img[i], gg = img[plane + i], b = img[2 * plane + i];
    const int d = op == OP_COLOR ? l_of(r, gg, b) : op == OP_CONTRAST ? mean : 0;
    img[i] = blend_px(d, r, factor);
    img[plane + i] = blend_px(d, gg, factor);
    img[2 * plane + i] = blend_px(d, b, factor);
  }
  __syncthreads();
}

// The enhance blend of the whole image img [3][n_pix] held by one CTA; lsum is a shared scratch word.
__device__ void enhance_blend(unsigned char* img, int n_pix, int op, float factor, unsigned long long* lsum) {
  int mean = 0;
  if (op == OP_CONTRAST) {
    l_sum(img, n_pix, n_pix, lsum);
    mean = contrast_mean(*lsum, n_pix);
  } else {
    __syncthreads();
  }
  enhance_apply(img, n_pix, n_pix, op, factor, mean);
}

// ImageOps.autocontrast / equalize of one channel: the LUT from its histogram h (one thread per channel)
__device__ void hist_lut(int op, const int* h, unsigned char* lut) {
  if (op == OP_AUTOCONTRAST) {
    int lo = 0, hi = 255;
    while (lo < 255 && !h[lo]) ++lo;
    while (hi > 0 && !h[hi]) --hi;
    if (hi <= lo) {
      for (int i = 0; i < 256; ++i) lut[i] = (unsigned char)i;
    } else {
      const double scale = __ddiv_rn(255.0, (double)(hi - lo));
      const double offset = __dmul_rn((double)(-lo), scale);
      for (int i = 0; i < 256; ++i) {
        const int v = (int)__dadd_rn(__dmul_rn((double)i, scale), offset);
        lut[i] = (unsigned char)(v < 0 ? 0 : v > 255 ? 255 : v);
      }
    }
  } else {
    long long tot = 0, last = 0;
    int nz = 0;
    for (int i = 0; i < 256; ++i) if (h[i]) { tot += h[i]; last = h[i]; ++nz; }
    const long long step = nz <= 1 ? 0 : (tot - last) / 255;
    if (!step) {
      for (int i = 0; i < 256; ++i) lut[i] = (unsigned char)i;
    } else {
      long long nn = step / 2;
      for (int i = 0; i < 256; ++i) {
        const long long v = nn / step;
        lut[i] = (unsigned char)(v > 255 ? 255 : v);
        nn += h[i];
      }
    }
  }
}

// Invert / Posterize / Solarize / SolarizeAdd of the value v (every other op: v unchanged)
__device__ __forceinline__ int point_lut(const cotb200_aug_op& op, int v) {
  if (op.op == OP_INVERT) return 255 - v;
  if (op.op == OP_POSTERIZE) return op.v[0] >= 8 ? v : v & (~((1 << (8 - op.v[0])) - 1) & 255);
  if (op.op == OP_SOLARIZE) return v < op.v[0] ? v : 255 - v;
  if (op.op == OP_SOLARIZEADD) return v < 128 ? min(255, v + op.v[0]) : v;
  return v;
}

__global__ void __launch_bounds__(RA_THREADS)
aug_randaug_kernel(const cotb200_aug_sample* __restrict__ params, int S, unsigned char* out) {
  extern __shared__ unsigned char sm_img[];          // [3][S][S]
  __shared__ int hist[3][256];
  __shared__ unsigned char lut[3][256];
  __shared__ unsigned long long lsum;
  const cotb200_aug_sample& p = params[blockIdx.x];
  const int n_pix = S * S, n_all = 3 * n_pix;
  unsigned char* g = out + (long long)blockIdx.x * n_all;   // plain loads: g is rewritten by this CTA between ops
  bool loaded = false, g_current = true;
  const int fill[3] = {124, 116, 104};                // the reference's img_mean fill
  for (int s = 0; s < COTB200_AUG_MAX_OPS; ++s) {
    const cotb200_aug_op op = p.ops[s];
    if (op.op < 0) continue;
    if (op.op == OP_SHARPNESS || is_affine(op.op)) {  // neighbours: read the previous state from global memory
      if (!g_current) {
        for (int i = threadIdx.x; i < n_all; i += blockDim.x) g[i] = sm_img[i];
        __syncthreads();
      }
      for (int i = threadIdx.x; i < n_all; i += blockDim.x) {
        const int c = i / n_pix, y = (i % n_pix) / S, x = i % S;
        if (op.op == OP_SHARPNESS) {
          const unsigned char* pl = g + (long long)c * n_pix;
          const int v = pl[y * S + x];
          const int d = (x == 0 || y == 0 || x == S - 1 || y == S - 1) ? v : smooth_px(pl, S, x, y);
          sm_img[i] = blend_px(d, v, op.factor);
        } else {
          sm_img[i] = affine_px(g, S, c, op, x, y, fill[c]);
        }
      }
      __syncthreads();
      loaded = true;
      g_current = false;
      continue;
    }
    if (!loaded) {
      for (int i = threadIdx.x; i < n_all; i += blockDim.x) sm_img[i] = g[i];
      loaded = true;
    }
    if (op.op == OP_CUTOUT) {
      __syncthreads();
      const int x0 = max(op.v[0], 0), y0 = max(op.v[1], 0), x1 = min(op.v[2], S - 1), y1 = min(op.v[3], S - 1);
      const int bw = x1 - x0 + 1, bh = y1 - y0 + 1;
      if (bw > 0 && bh > 0)
        for (int i = threadIdx.x; i < 3 * bw * bh; i += blockDim.x) {
          const int c = i / (bw * bh), y = y0 + (i % (bw * bh)) / bw, x = x0 + i % bw;
          sm_img[c * n_pix + y * S + x] = (unsigned char)fill[c];
        }
      __syncthreads();
      g_current = false;
      continue;
    }
    if (op.op >= OP_COLOR && op.op <= OP_BRIGHTNESS) {
      enhance_blend(sm_img, n_pix, op.op, op.factor, &lsum);
      g_current = false;
      continue;
    }
    // LUT ops
    if (op.op == OP_AUTOCONTRAST || op.op == OP_EQUALIZE) {
      for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) (&hist[0][0])[i] = 0;
      __syncthreads();
      for (int i = threadIdx.x; i < n_all; i += blockDim.x) atomicAdd(&hist[i / n_pix][sm_img[i]], 1);
      __syncthreads();
      if (threadIdx.x < 3) hist_lut(op.op, hist[threadIdx.x], lut[threadIdx.x]);   // per channel
    } else {
      for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) lut[i >> 8][i & 255] = (unsigned char)point_lut(op, i & 255);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_all; i += blockDim.x) sm_img[i] = lut[i / n_pix][sm_img[i]];
    __syncthreads();
    g_current = false;
  }
  if (!g_current)
    for (int i = threadIdx.x; i < n_all; i += blockDim.x) g[i] = sm_img[i];
}

// ---------------------------------------------------------------- ColorJitter + vertical flip
// torchvision ColorJitter on PIL images: brightness / contrast / saturation are ImageEnhance.Brightness / Contrast / Color
// (enhance_blend), hue is adjust_hue: Pillow's RGB -> HSV, h += uint8(int32(hue_factor * 255)) (mod 256), Pillow's HSV -> RGB.
// The two conversions follow Pillow's C arithmetic: float where it declares float, double where its expressions promote, C
// round() (half away from zero) and truncating casts; every operation is an explicit _rn intrinsic so that nothing contracts.
enum { JIT_BRIGHTNESS = 0, JIT_CONTRAST, JIT_SATURATION, JIT_HUE, JIT_COUNT };

__device__ __forceinline__ int clip255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

__device__ __forceinline__ void rgb_to_hsv_px(int r, int g, int b, int& h, int& s, int& v) {
  const int maxc = max(r, max(g, b)), minc = min(r, min(g, b));
  v = maxc;
  if (maxc == minc) { h = 0; s = 0; return; }
  const float cr = (float)(maxc - minc);
  const float sf = __fdiv_rn(cr, (float)maxc);
  const float rc = __fdiv_rn((float)(maxc - r), cr), gc = __fdiv_rn((float)(maxc - g), cr), bc = __fdiv_rn((float)(maxc - b), cr);
  float hf;
  if (r == maxc) hf = __fsub_rn(bc, gc);
  else if (g == maxc) hf = (float)__dsub_rn(__dadd_rn(2.0, (double)rc), (double)bc);
  else hf = (float)__dsub_rn(__dadd_rn(4.0, (double)gc), (double)rc);
  hf = (float)fmod(__dadd_rn(__ddiv_rn((double)hf, 6.0), 1.0), 1.0);
  h = clip255((int)__dmul_rn((double)hf, 255.0));
  s = clip255((int)__dmul_rn((double)sf, 255.0));
}

__device__ __forceinline__ void hsv_to_rgb_px(int h, int s, int v, int& r, int& g, int& b) {
  if (s == 0) { r = g = b = v; return; }
  const double hh = __ddiv_rn(__dmul_rn((double)h, 6.0), 255.0);
  const int i = (int)floor(hh);
  const float f = (float)__dsub_rn(hh, (double)(float)i);
  const float fs = (float)__ddiv_rn((double)s, 255.0);
  const double vf = (double)v;
  const int p = clip255((int)round(__dmul_rn(vf, __dsub_rn(1.0, (double)fs))));
  const int q = clip255((int)round(__dmul_rn(vf, __dsub_rn(1.0, (double)__fmul_rn(fs, f)))));
  const int t = clip255((int)round(__dmul_rn(vf, __dsub_rn(1.0, __dmul_rn((double)fs, __dsub_rn(1.0, (double)f))))));
  switch (i % 6) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// np.int32(hue_factor * 255).astype(np.uint8)
__device__ __forceinline__ int hue_shift(double hue) { return (int)(unsigned char)(int)__dmul_rn(hue, 255.0); }

// adjust_hue of pixel i of the planar image img [3][plane], in place
__device__ __forceinline__ void hue_px(unsigned char* img, int plane, int i, int shift) {
  int h, s, v, r, gg, b;
  rgb_to_hsv_px(img[i], img[plane + i], img[2 * plane + i], h, s, v);
  hsv_to_rgb_px((h + shift) & 255, s, v, r, gg, b);
  img[i] = (unsigned char)r;
  img[plane + i] = (unsigned char)gg;
  img[2 * plane + i] = (unsigned char)b;
}

__device__ __forceinline__ bool jitter_any(const cotb200_aug_jitter& p) {
  bool any = p.vflip != 0;
  for (int k = 0; k < JIT_COUNT; ++k) any = any || p.order[k] >= 0;
  return any;
}

__device__ __forceinline__ int jitter_enhance_op(int op) {
  return op == JIT_BRIGHTNESS ? OP_BRIGHTNESS : op == JIT_CONTRAST ? OP_CONTRAST : OP_COLOR;
}

__global__ void __launch_bounds__(RA_THREADS)
aug_jitter_kernel(const cotb200_aug_jitter* __restrict__ params, int S, unsigned char* out) {
  extern __shared__ unsigned char sm_img[];          // [3][S][S]
  __shared__ unsigned long long lsum;
  const cotb200_aug_jitter p = params[blockIdx.x];
  if (!jitter_any(p)) return;                        // the image stays as resize-crop wrote it
  const int n_pix = S * S, n_all = 3 * n_pix;
  unsigned char* g = out + (long long)blockIdx.x * n_all;
  for (int i = threadIdx.x; i < n_all; i += blockDim.x) {
    const int c = i / n_pix, y = (i % n_pix) / S, x = i % S;
    sm_img[i] = g[p.vflip ? c * n_pix + (S - 1 - y) * S + x : i];   // RandomVerticalFlip: a row mirror of the S x S image
  }
  __syncthreads();
  for (int k = 0; k < JIT_COUNT; ++k) {
    const int op = p.order[k];
    if (op < 0) continue;
    if (op == JIT_HUE) {
      const int shift = hue_shift(p.hue);
      for (int i = threadIdx.x; i < n_pix; i += blockDim.x) hue_px(sm_img, n_pix, i, shift);
      __syncthreads();
    } else {
      enhance_blend(sm_img, n_pix, jitter_enhance_op(op), p.factor[op], &lsum);
    }
  }
  for (int i = threadIdx.x; i < n_all; i += blockDim.x) g[i] = sm_img[i];
}

// ---------------------------------------------------------------- the same two transforms on thread-block clusters (S <= 512)
// An S x S x 3 image above 261 rows does not fit the 200 KB budget of one CTA, so one cluster of cs CTAs holds it: CTA r keeps
// rows [r R, min(S, (r + 1) R)) of all three planes (R = ceil(S / cs)) in its shared memory.  The whole-image quantities
// (AutoContrast's and Equalize's histograms, Contrast's L sum) are integer sums: each CTA builds its band's partial, and after a
// cluster barrier every CTA adds the cs partials in rank order through distributed shared memory, so every CTA holds the exact
// total the one-CTA kernel computes and builds the same LUT or mean.  A cluster barrier follows every such read, before the
// partial is rebuilt and before any CTA exits, since a CTA's shared memory must outlive its neighbours' reads of it.
// Ops that read neighbouring rows (Sharpness, the affine ops) read the previous state of the whole image from `out` in global
// memory, as the one-CTA kernel does; every CTA writes its band there first, and a cluster barrier orders those writes before
// the other CTAs' reads.
namespace cg = cooperative_groups;

// barrier.cluster.arrive.release + barrier.cluster.wait.acquire (PTX ISA, "Parallel Synchronization and Communication
// Instructions: barrier.cluster", and the memory consistency model's release and acquire patterns): every memory access a
// thread of the cluster made before its arrive, to shared, distributed shared or global memory, happens before every access a
// thread of the cluster makes after its wait.  It also synchronises the threads of each CTA, as __syncthreads does.
__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

struct Band {
  int img, rank, cs, y0, plane;      // the image of this cluster, this CTA's rank, its first row and its rows * S
};

__device__ __forceinline__ Band band_of(int S, int R) {
  cg::cluster_group cl = cg::this_cluster();
  Band b;
  b.cs = (int)cl.num_blocks();
  b.rank = (int)cl.block_rank();
  b.img = blockIdx.x / b.cs;
  b.y0 = min(S, b.rank * R);
  b.plane = (min(S, b.y0 + R) - b.y0) * S;
  return b;
}

// The whole image's sum of the cs CTAs' partials *part, in rank order (a cluster barrier must precede it).
__device__ __forceinline__ unsigned long long cluster_sum(unsigned long long* part, int cs) {
  cg::cluster_group cl = cg::this_cluster();
  unsigned long long t = 0;
  for (int r = 0; r < cs; ++r) t += *cl.map_shared_rank(part, r);
  return t;
}

// enhance_blend on a band: Contrast's mean comes from the cluster's L sum
__device__ void enhance_blend_band(unsigned char* img, const Band& b, int n_pix, int op, float factor, unsigned long long* lsum) {
  int mean = 0;
  if (op == OP_CONTRAST) {
    l_sum(img, b.plane, b.plane, lsum);
    cluster_barrier();
    const unsigned long long tot = cluster_sum(lsum, b.cs);
    cluster_barrier();
    mean = contrast_mean(tot, n_pix);
  } else {
    __syncthreads();
  }
  enhance_apply(img, b.plane, b.plane, op, factor, mean);
}

__global__ void __launch_bounds__(RA_THREADS)
aug_randaug_cluster_kernel(const cotb200_aug_sample* __restrict__ params, int S, int R, unsigned char* out) {
  extern __shared__ unsigned char sm_img[];          // [3][rows of the band][S]
  __shared__ int hist[3][256];                       // this band's histograms
  __shared__ int htot[3][256];                       // the image's
  __shared__ unsigned char lut[3][256];
  __shared__ unsigned long long lsum;
  const Band b = band_of(S, R);
  const cotb200_aug_sample& p = params[b.img];
  const int n_pix = S * S, n_band = 3 * b.plane;
  unsigned char* g = out + (long long)b.img * 3 * n_pix;
  auto gi = [&](int i) { return (i / b.plane) * n_pix + b.y0 * S + i % b.plane; };   // band index -> image index
  bool loaded = false, g_current = true;
  const int fill[3] = {124, 116, 104};
  for (int s = 0; s < COTB200_AUG_MAX_OPS; ++s) {
    const cotb200_aug_op op = p.ops[s];
    if (op.op < 0) continue;
    if (op.op == OP_SHARPNESS || is_affine(op.op)) {
      if (!g_current) {
        for (int i = threadIdx.x; i < n_band; i += blockDim.x) g[gi(i)] = sm_img[i];
        cluster_barrier();                           // every band is in `out` before any CTA reads its neighbours' rows
      }
      for (int i = threadIdx.x; i < n_band; i += blockDim.x) {
        const int c = i / b.plane, y = b.y0 + (i % b.plane) / S, x = i % S;
        if (op.op == OP_SHARPNESS) {
          const unsigned char* pl = g + (long long)c * n_pix;
          const int v = pl[y * S + x];
          const int d = (x == 0 || y == 0 || x == S - 1 || y == S - 1) ? v : smooth_px(pl, S, x, y);
          sm_img[i] = blend_px(d, v, op.factor);
        } else {
          sm_img[i] = affine_px(g, S, c, op, x, y, fill[c]);
        }
      }
      cluster_barrier();                             // every CTA has read `out` before any CTA writes its band there again
      loaded = true;
      g_current = false;
      continue;
    }
    if (!loaded) {
      for (int i = threadIdx.x; i < n_band; i += blockDim.x) sm_img[i] = g[gi(i)];
      loaded = true;
    }
    if (op.op == OP_CUTOUT) {                        // the box clipped to the band
      __syncthreads();
      const int x0 = max(op.v[0], 0), y0 = max(op.v[1], b.y0), x1 = min(op.v[2], S - 1);
      const int y1 = min(op.v[3], b.y0 + b.plane / S - 1);
      const int bw = x1 - x0 + 1, bh = y1 - y0 + 1;
      if (bw > 0 && bh > 0)
        for (int i = threadIdx.x; i < 3 * bw * bh; i += blockDim.x) {
          const int c = i / (bw * bh), y = y0 + (i % (bw * bh)) / bw, x = x0 + i % bw;
          sm_img[c * b.plane + (y - b.y0) * S + x] = (unsigned char)fill[c];
        }
      __syncthreads();
      g_current = false;
      continue;
    }
    if (op.op >= OP_COLOR && op.op <= OP_BRIGHTNESS) {
      enhance_blend_band(sm_img, b, n_pix, op.op, op.factor, &lsum);
      g_current = false;
      continue;
    }
    if (op.op == OP_AUTOCONTRAST || op.op == OP_EQUALIZE) {
      for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) (&hist[0][0])[i] = 0;
      __syncthreads();
      for (int i = threadIdx.x; i < n_band; i += blockDim.x) atomicAdd(&hist[i / b.plane][sm_img[i]], 1);
      cluster_barrier();
      cg::cluster_group cl = cg::this_cluster();
      for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) {
        int t = 0;
        for (int r = 0; r < b.cs; ++r) t += cl.map_shared_rank(&hist[0][0], r)[i];
        (&htot[0][0])[i] = t;
      }
      cluster_barrier();
      if (threadIdx.x < 3) hist_lut(op.op, htot[threadIdx.x], lut[threadIdx.x]);
    } else {
      for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) lut[i >> 8][i & 255] = (unsigned char)point_lut(op, i & 255);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_band; i += blockDim.x) sm_img[i] = lut[i / b.plane][sm_img[i]];
    __syncthreads();
    g_current = false;
  }
  if (!g_current)
    for (int i = threadIdx.x; i < n_band; i += blockDim.x) g[gi(i)] = sm_img[i];
}

__global__ void __launch_bounds__(RA_THREADS)
aug_jitter_cluster_kernel(const cotb200_aug_jitter* __restrict__ params, int S, int R, unsigned char* out) {
  extern __shared__ unsigned char sm_img[];          // [3][rows of the band][S]
  __shared__ unsigned long long lsum;
  const Band b = band_of(S, R);
  const cotb200_aug_jitter p = params[b.img];
  if (!jitter_any(p)) return;                        // the whole cluster returns: the image stays as resize-crop wrote it
  const int n_pix = S * S, n_band = 3 * b.plane;
  unsigned char* g = out + (long long)b.img * 3 * n_pix;
  for (int i = threadIdx.x; i < n_band; i += blockDim.x) {
    const int c = i / b.plane, y = b.y0 + (i % b.plane) / S, x = i % S;
    sm_img[i] = g[c * n_pix + (p.vflip ? S - 1 - y : y) * S + x];   // the vertical flip reads the mirrored rows
  }
  if (p.vflip) cluster_barrier();                    // every CTA has read its mirrored rows before any CTA writes its band
  __syncthreads();
  for (int k = 0; k < JIT_COUNT; ++k) {
    const int op = p.order[k];
    if (op < 0) continue;
    if (op == JIT_HUE) {
      const int shift = hue_shift(p.hue);
      for (int i = threadIdx.x; i < b.plane; i += blockDim.x) hue_px(sm_img, b.plane, i, shift);
      __syncthreads();
    } else {
      enhance_blend_band(sm_img, b, n_pix, jitter_enhance_op(op), p.factor[op], &lsum);
    }
  }
  for (int i = threadIdx.x; i < n_band; i += blockDim.x) g[(i / b.plane) * n_pix + b.y0 * S + i % b.plane] = sm_img[i];
}

// ---------------------------------------------------------------- host: argument checks shared by both kernel families
static int check_samples(const char* what, int N, int S, const cotb200_aug_sample* h) {
  if (!h) { set_error("%s: params_host is NULL", what); return COTB200_ENULL; }
  if (N <= 0 || S <= 0) { set_error("%s: bad dims N=%d S=%d", what, N, S); return COTB200_EINVAL; }
  return 0;
}

// cotb200_aug_randaug's arguments, for images of at most max_s rows held in the shared memory of `where`
static int check_randaug(const char* what, int N, int S, int max_s, const char* where, const cotb200_aug_sample* params_host,
                         const cotb200_aug_sample* params_dev, const unsigned char* out) {
  int rc = check_samples(what, N, S, params_host);
  if (rc) return rc;
  if (!params_dev || !out) { set_error("%s: NULL pointer", what); return COTB200_ENULL; }
  if (S > max_s) { set_error("%s: S=%d above %d (the image is held in %s)", what, S, max_s, where); return COTB200_EUNSUPPORTED; }
  for (int n = 0; n < N; ++n)
    for (int s = 0; s < COTB200_AUG_MAX_OPS; ++s) {
      const cotb200_aug_op& op = params_host[n].ops[s];
      bool ok = op.op >= -1 && op.op < OP_COUNT;
      if (ok && is_affine(op.op)) {
        ok = op.filter == 0 || op.filter == 1;
        for (int i = 0; i < 6; ++i) ok = ok && isfinite(op.m[i]);
      }
      if (ok && op.op == OP_POSTERIZE) ok = op.v[0] >= 0;
      if (ok && op.op >= OP_COLOR && op.op <= OP_SHARPNESS) ok = isfinite(op.factor);
      if (!ok) { set_error("%s: sample %d op %d: unknown op id %d or bad argument", what, n, s, op.op); return COTB200_EINVAL; }
    }
  return 0;
}

// cotb200_aug_color_jitter's arguments, likewise
static int check_jitter(const char* what, int N, int S, int max_s, const char* where, const cotb200_aug_jitter* params_host,
                        const cotb200_aug_jitter* params_dev, const unsigned char* out) {
  if (!params_host) { set_error("%s: params_host is NULL", what); return COTB200_ENULL; }
  if (N <= 0 || S <= 0) { set_error("%s: bad dims N=%d S=%d", what, N, S); return COTB200_EINVAL; }
  if (!params_dev || !out) { set_error("%s: NULL pointer", what); return COTB200_ENULL; }
  if (S > max_s) { set_error("%s: S=%d above %d (the image is held in %s)", what, S, max_s, where); return COTB200_EUNSUPPORTED; }
  for (int n = 0; n < N; ++n) {
    const cotb200_aug_jitter& p = params_host[n];
    if (p.vflip != 0 && p.vflip != 1) { set_error("%s: sample %d: vflip %d not 0 or 1", what, n, p.vflip); return COTB200_EINVAL; }
    bool seen[JIT_COUNT] = {};
    for (int k = 0; k < JIT_COUNT; ++k) {
      const int op = p.order[k];
      if (op == -1) continue;
      if (op < -1 || op >= JIT_COUNT || seen[op]) {
        set_error("%s: sample %d: order[%d] = %d is unknown or repeated", what, n, k, op); return COTB200_EINVAL;
      }
      seen[op] = true;
      if (op == JIT_HUE ? !(p.hue >= -0.5 && p.hue <= 0.5) : !(isfinite(p.factor[op]) && p.factor[op] >= 0.f)) {
        set_error("%s: sample %d: factor of op %d out of range", what, n, op); return COTB200_EINVAL;
      }
    }
  }
  return 0;
}

static const char* const ONE_CTA = "shared memory";
static const char* const CLUSTER = "the shared memory of a cluster of at most 4 CTAs";

// The cluster size of an S x S image: the smallest cs in 1..4 whose band of ceil(S / cs) rows fits AUG_MAX_SMEM (0: none does)
static int cluster_size(int S) {
  for (int cs = 1; cs <= 4; ++cs)
    if (3LL * ((S + cs - 1) / cs) * S <= AUG_MAX_SMEM) return cs;
  return 0;
}

// One cluster of cluster_size(S) CTAs per image.  The occupancy query is memoised per kernel, device and cluster size.
template <typename P>
static int launch_cluster(const char* what, void (*kernel)(const P*, int, int, unsigned char*), int N, int S, const P* params_dev,
                          unsigned char* out, cudaStream_t st) {
  static int fits[64][5] = {};                       // 0 unknown, 1 fits, -1 does not
  const int cs = cluster_size(S), R = (S + cs - 1) / cs;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.gridDim = dim3(N * cs);
  cfg.blockDim = dim3(RA_THREADS);
  cfg.dynamicSmemBytes = (size_t)3 * R * S;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int& f = fits[cur_dev_slot()][cs];
  if (!f) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AUG_MAX_SMEM);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
    int clusters = 0;
    e = cudaOccupancyMaxActiveClusters(&clusters, kernel, &cfg);
    if (e != cudaSuccess) { set_error("%s: cudaOccupancyMaxActiveClusters: %s", what, cudaGetErrorString(e)); return (int)e; }
    f = clusters > 0 ? 1 : -1;
  }
  if (f < 0) {
    set_error("%s: the device cannot run a cluster of %d CTAs with %d B of shared memory each (S=%d)", what, cs,
              (int)cfg.dynamicSmemBytes, S);
    return COTB200_EUNSUPPORTED;
  }
  COTB200_PROF_B(what, 6.0 * N * S * S);
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, params_dev, S, R, out);
  if (e != cudaSuccess) { set_error("%s: %s", what, cudaGetErrorString(e)); return (int)e; }
  return check_launch(what);
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_aug_resize_crop(int N, int S, const unsigned char* src, long long src_bytes, const cotb200_aug_sample* params_host,
                                       const cotb200_aug_sample* params_dev, unsigned char* tmp, long long tmp_bytes,
                                       unsigned char* out, void* stream) {
  int rc = check_samples("aug_resize_crop", N, S, params_host);
  if (rc) return rc;
  if (!src || !params_dev || !tmp || !out) { set_error("aug_resize_crop: NULL pointer"); return COTB200_ENULL; }
  int kmax = 1;
  double nbytes = 0;
  for (int n = 0; n < N; ++n) {
    const cotb200_aug_sample& p = params_host[n];
    if (p.h < 1 || p.w < 1) { set_error("aug_resize_crop: sample %d: image %dx%d smaller than 1x1", n, p.h, p.w); return COTB200_EINVAL; }
    if (p.offset < 0 || p.offset > src_bytes || (src_bytes - p.offset) / 3 / p.w < p.h) {
      set_error("aug_resize_crop: sample %d: %dx%d image at offset %lld past the %lld-byte buffer", n, p.h, p.w, p.offset, src_bytes);
      return COTB200_EINVAL;
    }
    if (p.ci < 0 || p.cj < 0 || p.ch < 1 || p.cw < 1 || p.ch > p.h - p.ci || p.cw > p.w - p.cj) {
      set_error("aug_resize_crop: sample %d: crop (%d, %d, %d, %d) outside the %dx%d image", n, p.ci, p.cj, p.ch, p.cw, p.h, p.w);
      return COTB200_EINVAL;
    }
    if (p.oi < 0 || p.oj < 0 || p.rh < S || p.rw < S || p.oi > p.rh - S || p.oj > p.rw - S) {
      set_error("aug_resize_crop: sample %d: window (%d, %d) of size %d outside the %dx%d resize", n, p.oi, p.oj, S, p.rh, p.rw);
      return COTB200_EINVAL;
    }
    if ((p.filter != 0 && p.filter != 1) || (p.flip != 0 && p.flip != 1)) {
      set_error("aug_resize_crop: sample %d: filter %d / flip %d not 0 or 1", n, p.filter, p.flip); return COTB200_EINVAL;
    }
    if (p.tmp_offset < 0 || p.tmp_offset > tmp_bytes || (tmp_bytes - p.tmp_offset) / 3 / S < p.ch) {
      set_error("aug_resize_crop: sample %d: scratch range at %lld past the %lld-byte buffer", n, p.tmp_offset, tmp_bytes);
      return COTB200_EINVAL;
    }
    kmax = max(kmax, max(axis_ksize(p.cw, p.rw, p.filter), axis_ksize(p.ch, p.rh, p.filter)));
    nbytes += 3.0 * p.ch * p.cw;
  }
  const size_t smem_h = (size_t)S * (kmax + 1) * sizeof(int), smem_v = (size_t)AUG_VROWS * (kmax + 1) * sizeof(int);
  if (smem_h > (size_t)AUG_MAX_SMEM) {
    set_error("aug_resize_crop: %d filter taps at S=%d exceed the kernel's shared memory", kmax, S); return COTB200_EUNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaFuncSetAttribute(aug_hpass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AUG_MAX_SMEM);
  if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
  {
    COTB200_PROF_B("aug_hpass", nbytes + 3.0 * N * S * S);
    aug_hpass_kernel<<<dim3(N, AUG_HGRID), AUG_THREADS, smem_h, st>>>(src, params_dev, S, kmax, tmp);
    if ((rc = check_launch("aug_hpass"))) return rc;
  }
  COTB200_PROF_B("aug_vpass", 6.0 * N * S * S);
  aug_vpass_kernel<<<dim3(N, (S + AUG_VROWS - 1) / AUG_VROWS), AUG_THREADS, smem_v, st>>>(tmp, params_dev, S, kmax, out);
  return check_launch("aug_vpass");
}

extern "C" int cotb200_aug_randaug(int N, int S, const cotb200_aug_sample* params_host, const cotb200_aug_sample* params_dev,
                                   unsigned char* out, void* stream) {
  int rc = check_randaug("aug_randaug", N, S, RA_MAX_S, ONE_CTA, params_host, params_dev, out);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int smem = 3 * S * S;
  cudaError_t e = cudaFuncSetAttribute(aug_randaug_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 3 * RA_MAX_S * RA_MAX_S);
  if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
  COTB200_PROF_B("aug_randaug", 6.0 * N * S * S);
  aug_randaug_kernel<<<N, RA_THREADS, smem, st>>>(params_dev, S, out);
  return check_launch("aug_randaug");
}

extern "C" int cotb200_aug_color_jitter(int N, int S, const cotb200_aug_jitter* params_host, const cotb200_aug_jitter* params_dev,
                                  unsigned char* out, void* stream) {
  const int rc = check_jitter("aug_color_jitter", N, S, RA_MAX_S, ONE_CTA, params_host, params_dev, out);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaFuncSetAttribute(aug_jitter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 3 * RA_MAX_S * RA_MAX_S);
  if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return (int)e; }
  COTB200_PROF_B("aug_jitter", 6.0 * N * S * S);
  aug_jitter_kernel<<<N, RA_THREADS, 3 * S * S, st>>>(params_dev, S, out);
  return check_launch("aug_jitter");
}

extern "C" int cotb200_aug_randaug_cluster(int N, int S, const cotb200_aug_sample* params_host, const cotb200_aug_sample* params_dev,
                                           unsigned char* out, void* stream) {
  const int rc = check_randaug("aug_randaug_cluster", N, S, COTB200_AUG_CLUSTER_MAX_S, CLUSTER, params_host, params_dev, out);
  if (rc) return rc;
  return launch_cluster("aug_randaug_cluster", aug_randaug_cluster_kernel, N, S, params_dev, out, (cudaStream_t)stream);
}

extern "C" int cotb200_aug_color_jitter_cluster(int N, int S, const cotb200_aug_jitter* params_host, const cotb200_aug_jitter* params_dev,
                                                unsigned char* out, void* stream) {
  const int rc = check_jitter("aug_color_jitter_cluster", N, S, COTB200_AUG_CLUSTER_MAX_S, CLUSTER, params_host, params_dev, out);
  if (rc) return rc;
  return launch_cluster("aug_jitter_cluster", aug_jitter_cluster_kernel, N, S, params_dev, out, (cudaStream_t)stream);
}
