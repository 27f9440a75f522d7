// The remaining LocalConv variants of the reference's cupy_layers package (SURVEY.md section 8f rank 4), sm_90a:
//
//   aggregation_refpad            reflect padding          /root/reference/cupy_layers/aggregation_refpad.py:21-127
//   aggregation_zeropad_dilate    per-weight-channel dilation, 3x3, stride 1   .../aggregation_zeropad_dilate.py:20-146
//
// No registered model of the reference constructs them (lr_net / san_lowrank / botnet import them); they are runtime-
// dimension, any-dtype (fp32/fp64/bf16/fp16) kernels on the reference's NCHW contract so the whole package imports and
// runs without CuPy.  One thread per output element, 64-bit indexing, grid-stride; fp32 (fp64) accumulation.
//
// Differences from the reference's formulation that do NOT change results:
//   * refpad dX: the reference computes the gradient on the PADDED grid [H+2p, W+2p] and then folds the four borders back
//     with torch flips/adds (aggregation_refpad.py:188-199); here every input pixel gathers directly from the (at most
//     3 x 3) padded positions that reflect onto it -- one kernel, no temporary, no in-place adds.
#include "common.cuh"

namespace cotb200 {

struct VGeo {
  int N, C, H, W, heads, wc, KH, KW, SH, SW, PH, PW, DH, DW, HO, WO, K2, rep;
};

__device__ __forceinline__ int reflect_idx(int i, int n) {
  if (i < 0) i = -i;                       // aggregation_refpad.py:42-45
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// ------------------------------------------------------------------------------------------------ refpad
template <typename T>
__global__ void refpad_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, VGeo g, long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int wo = r % g.WO; r /= g.WO;
    const int ho = r % g.HO; r /= g.HO;
    const int c = r % g.C; r /= g.C;
    const int head = r % g.heads;
    const int n = r / g.heads;
    const long long plane = (long long)g.HO * g.WO;
    const T* wp = w + (((long long)(n * g.heads + head) * g.wc + c % g.wc) * g.K2) * plane + (long long)ho * g.WO + wo;
    const T* xp = x + ((long long)(n * g.C + c) * g.H) * g.W;
    Acc acc = 0;
    for (int kh = 0; kh < g.KH; ++kh) {
      const int hi = reflect_idx(-g.PH + ho * g.SH + kh * g.DH, g.H);
      for (int kw = 0; kw < g.KW; ++kw) {
        const int wi = reflect_idx(-g.PW + wo * g.SW + kw * g.DW, g.W);
        acc += to_acc(wp[(long long)(kh * g.KW + kw) * plane]) * to_acc(xp[(long long)hi * g.W + wi]);
      }
    }
    y[idx] = Elem<T>::from(acc);
  }
}

// padded coordinates (un-shifted: -P .. H-1+P) that reflect onto i; returns the count (1..3)
__device__ __forceinline__ int reflect_sources(int i, int n, int pad, int (&src)[3]) {
  int k = 0;
  src[k++] = i;
  if (i >= 1 && i <= pad) src[k++] = -i;                              // top / left border
  if (i <= n - 2 && i >= n - 1 - pad) src[k++] = 2 * (n - 1) - i;     // bottom / right border
  return k;
}

template <typename T>
__global__ void refpad_dx_kernel(const T* __restrict__ dy, const T* __restrict__ w, T* __restrict__ dx, VGeo g, long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int wq = r % g.W; r /= g.W;
    const int h = r % g.H; r /= g.H;
    const int c = r % g.C;
    const int n = r / g.C;
    const long long plane = (long long)g.HO * g.WO;
    int hsrc[3], wsrc[3];
    const int nh = reflect_sources(h, g.H, g.PH, hsrc), nw = reflect_sources(wq, g.W, g.PW, wsrc);
    Acc acc = 0;
    for (int head = 0; head < g.heads; ++head) {
      const T* wp = w + (((long long)(n * g.heads + head) * g.wc + c % g.wc) * g.K2) * plane;
      const T* dp = dy + ((long long)(n * g.heads + head) * g.C + c) * plane;
      for (int a = 0; a < nh; ++a) {
        for (int kh = 0; kh < g.KH; ++kh) {
          const int hs = hsrc[a] + g.PH - kh * g.DH;           // aggregation_refpad.py:73-79 on the padded grid
          if (hs < 0 || hs % g.SH) continue;
          const int ho = hs / g.SH;
          if (ho >= g.HO) continue;
          for (int b = 0; b < nw; ++b) {
            for (int kw = 0; kw < g.KW; ++kw) {
              const int ws = wsrc[b] + g.PW - kw * g.DW;
              if (ws < 0 || ws % g.SW) continue;
              const int wo = ws / g.SW;
              if (wo >= g.WO) continue;
              const long long o = (long long)ho * g.WO + wo;
              acc += to_acc(wp[(long long)(kh * g.KW + kw) * plane + o]) * to_acc(dp[o]);
            }
          }
        }
      }
    }
    dx[idx] = Elem<T>::from(acc);
  }
}

template <typename T>
__global__ void refpad_dw_kernel(const T* __restrict__ dy, const T* __restrict__ x, T* __restrict__ dw, VGeo g, long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int wo = r % g.WO; r /= g.WO;
    const int ho = r % g.HO; r /= g.HO;
    const int tap = r % g.K2; r /= g.K2;
    const int gch = r % g.wc; r /= g.wc;
    const int head = r % g.heads;
    const int n = r / g.heads;
    const int kh = tap / g.KW, kw = tap % g.KW;
    const int hi = reflect_idx(-g.PH + ho * g.SH + kh * g.DH, g.H);
    const int wi = reflect_idx(-g.PW + wo * g.SW + kw * g.DW, g.W);
    const long long plane = (long long)g.HO * g.WO;
    Acc acc = 0;
    for (int cc = gch; cc < g.C; cc += g.wc)
      acc += to_acc(x[((long long)(n * g.C + cc) * g.H + hi) * g.W + wi]) *
             to_acc(dy[((long long)(n * g.heads + head) * g.C + cc) * plane + (long long)ho * g.WO + wo]);
    dw[idx] = Elem<T>::from(acc);
  }
}

// ------------------------------------------------------------------------------------------------ dilate (3x3, stride 1, pad = dilation)
template <typename T>
__global__ void dilate_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w, const T* __restrict__ dil, T* __restrict__ y,
                                  VGeo g, long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int wq = r % g.W; r /= g.W;
    const int h = r % g.H; r /= g.H;
    const int c = r % g.C; r /= g.C;
    const int head = r % g.heads;
    const int n = r / g.heads;
    const int d = (int)to_acc(dil[c % g.wc]);              // aggregation_zeropad_dilate.py:31-35
    const long long plane = (long long)g.H * g.W;
    const T* wp = w + (((long long)(n * g.heads + head) * g.wc + c % g.wc) * 9) * plane + (long long)h * g.W + wq;
    const T* xp = x + ((long long)(n * g.C + c)) * plane;
    Acc acc = 0;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = h + (kh - 1) * d;
      if (hi < 0 || hi >= g.H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = wq + (kw - 1) * d;
        if (wi < 0 || wi >= g.W) continue;
        acc += to_acc(wp[(long long)(kh * 3 + kw) * plane]) * to_acc(xp[(long long)hi * g.W + wi]);
      }
    }
    y[idx] = Elem<T>::from(acc);
  }
}

template <typename T>
__global__ void dilate_dx_kernel(const T* __restrict__ dy, const T* __restrict__ w, const T* __restrict__ dil, T* __restrict__ dx,
                                 VGeo g, long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int wq = r % g.W; r /= g.W;
    const int h = r % g.H; r /= g.H;
    const int c = r % g.C;
    const int n = r / g.C;
    const int d = (int)to_acc(dil[c % g.wc]);
    const long long plane = (long long)g.H * g.W;
    Acc acc = 0;
    for (int head = 0; head < g.heads; ++head) {
      const T* wp = w + (((long long)(n * g.heads + head) * g.wc + c % g.wc) * 9) * plane;
      const T* dp = dy + ((long long)(n * g.heads + head) * g.C + c) * plane;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int ho = h + d - kh * d;                       // :83-88 with stride 1
        if (ho < 0 || ho >= g.H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int wo = wq + d - kw * d;
          if (wo < 0 || wo >= g.W) continue;
          const long long o = (long long)ho * g.W + wo;
          acc += to_acc(wp[(long long)(kh * 3 + kw) * plane + o]) * to_acc(dp[o]);
        }
      }
    }
    dx[idx] = Elem<T>::from(acc);
  }
}

template <typename T>
__global__ void dilate_dw_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ dil, T* __restrict__ dw,
                                 VGeo g, long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int wq = r % g.W; r /= g.W;
    const int h = r % g.H; r /= g.H;
    const int tap = r % 9; r /= 9;
    const int gch = r % g.wc; r /= g.wc;
    const int head = r % g.heads;
    const int n = r / g.heads;
    const int d = (int)to_acc(dil[gch]);
    const int hi = h + (tap / 3 - 1) * d, wi = wq + (tap % 3 - 1) * d;
    const long long plane = (long long)g.H * g.W;
    Acc acc = 0;
    if (hi >= 0 && hi < g.H && wi >= 0 && wi < g.W) {
      for (int cc = gch; cc < g.C; cc += g.wc)
        acc += to_acc(x[(long long)(n * g.C + cc) * plane + (long long)hi * g.W + wi]) *
               to_acc(dy[((long long)(n * g.heads + head) * g.C + cc) * plane + (long long)h * g.W + wq]);
    }
    dw[idx] = Elem<T>::from(acc);
  }
}

// Register-resident forwards (the common small-footprint cases): one thread per (n, head, weight channel, output pixel) keeps
// the K*K weights and the K*K input offsets in registers and walks the C / wc input channels that share them, so a weight is
// read once instead of C / wc times and the index arithmetic is paid once per pixel (32-bit throughout; host checks the sizes).
template <typename T, int K>
__global__ void __launch_bounds__(256)
refpad_fwd_fast(const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, VGeo g, int total) {
  using Acc = typename Elem<T>::Acc;
  constexpr int K2 = K * K;
  const int plane = g.HO * g.WO, iplane = g.H * g.W;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int p = idx % plane;
    int r = idx / plane;
    const int gch = r % g.wc; r /= g.wc;
    const int head = r % g.heads;
    const int n = r / g.heads;
    const int ho = p / g.WO, wo = p - ho * g.WO;
    Acc wt[K2];
    int off[K2];
    const T* wp = w + ((long long)((n * g.heads + head) * g.wc + gch) * K2) * plane + p;
#pragma unroll
    for (int kh = 0; kh < K; ++kh) {
      const int hi = reflect_idx(-g.PH + ho * g.SH + kh * g.DH, g.H);
#pragma unroll
      for (int kw = 0; kw < K; ++kw) {
        const int wi = reflect_idx(-g.PW + wo * g.SW + kw * g.DW, g.W);
        wt[kh * K + kw] = to_acc(wp[(long long)(kh * K + kw) * plane]);
        off[kh * K + kw] = hi * g.W + wi;
      }
    }
    const T* xp = x + (long long)(n * g.C + gch) * iplane;
    T* yp = y + (long long)((n * g.heads + head) * g.C + gch) * plane + p;
    for (int rr = 0; rr < g.rep; ++rr) {
      Acc acc = 0;
#pragma unroll
      for (int t = 0; t < K2; ++t) acc += wt[t] * to_acc(xp[off[t]]);
      *yp = Elem<T>::from(acc);
      xp += (long long)g.wc * iplane;
      yp += (long long)g.wc * plane;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
dilate_fwd_fast(const T* __restrict__ x, const T* __restrict__ w, const T* __restrict__ dil, T* __restrict__ y, VGeo g, int total) {
  using Acc = typename Elem<T>::Acc;
  const int plane = g.H * g.W;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int p = idx % plane;
    int r = idx / plane;
    const int gch = r % g.wc; r /= g.wc;
    const int head = r % g.heads;
    const int n = r / g.heads;
    const int h = p / g.W, wq = p - h * g.W;
    const int d = (int)to_acc(dil[gch]);
    Acc wt[9];
    int off[9];
    const T* wp = w + ((long long)((n * g.heads + head) * g.wc + gch) * 9) * plane + p;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int hi = h + (t / 3 - 1) * d, wi = wq + (t % 3 - 1) * d;
      const bool ok = hi >= 0 && hi < g.H && wi >= 0 && wi < g.W;
      wt[t] = ok ? to_acc(wp[(long long)t * plane]) : Acc(0);
      off[t] = ok ? hi * g.W + wi : -1;                            // an out-of-range tap is skipped (never multiplied)
    }
    const T* xp = x + (long long)(n * g.C + gch) * plane;
    T* yp = y + (long long)((n * g.heads + head) * g.C + gch) * plane + p;
    for (int rr = 0; rr < g.rep; ++rr) {
      Acc acc = 0;
#pragma unroll
      for (int t = 0; t < 9; ++t) if (off[t] >= 0) acc += wt[t] * to_acc(xp[off[t]]);
      *yp = Elem<T>::from(acc);
      xp += (long long)g.wc * plane;
      yp += (long long)g.wc * plane;
    }
  }
}

static int vresolve(const cotb200_agg_desc* d, VGeo& g, const char* what, bool dilate) {
  if (!d) { set_error("%s: desc is NULL", what); return COTB200_ENULL; }
  if (d->layout != COTB200_NCHW) { set_error("%s supports the NCHW layout only (the reference contract)", what); return COTB200_ELAYOUT; }
  if (d->n <= 0 || d->c <= 0 || d->h <= 0 || d->w <= 0 || d->heads <= 0 || d->wc <= 0 || d->kh <= 0 || d->kw <= 0 || d->ho <= 0 || d->wo <= 0) {
    set_error("%s: non-positive dimension in desc", what); return COTB200_EINVAL;
  }
  if (d->c % d->wc) { set_error("%s: input channels %d not divisible by weight channels %d", what, d->c, d->wc); return COTB200_EINVAL; }
  g.N = d->n; g.C = d->c; g.H = d->h; g.W = d->w; g.heads = d->heads; g.wc = d->wc; g.KH = d->kh; g.KW = d->kw;
  g.K2 = d->kh * d->kw; g.rep = d->c / d->wc;
  if (dilate) {
    if (d->kh != 3 || d->kw != 3) { set_error("%s: kernel size must be 3 (aggregation_zeropad_dilate.py:255)", what); return COTB200_EINVAL; }
    if (d->ho != d->h || d->wo != d->w) { set_error("%s: output size must equal input size", what); return COTB200_EINVAL; }
    g.SH = g.SW = 1; g.PH = g.PW = g.DH = g.DW = 0; g.HO = d->h; g.WO = d->w;
    return 0;
  }
  if (d->sh <= 0 || d->sw <= 0 || d->dh <= 0 || d->dw <= 0 || d->ph < 0 || d->pw < 0) { set_error("%s: bad stride / dilation / padding", what); return COTB200_EINVAL; }
  if (d->ph >= d->h || d->pw >= d->w) { set_error("%s: reflect padding must be smaller than the input (pad %d,%d vs %dx%d)", what, d->ph, d->pw, d->h, d->w); return COTB200_EINVAL; }
  const int span_h = d->h + 2 * d->ph - (d->dh * (d->kh - 1) + 1), span_w = d->w + 2 * d->pw - (d->dw * (d->kw - 1) + 1);
  // a window larger than the padded input has no output position; the division below truncates towards zero, so it would
  // yield a size of 1, or two negative sizes whose product matches the weight plane, and the taps would reflect off the planes
  if (span_h < 0 || span_w < 0) { set_error("%s: kernel window larger than the padded input %dx%d", what, d->h + 2 * d->ph, d->w + 2 * d->pw); return COTB200_EINVAL; }
  const int ho = span_h / d->sh + 1, wo = span_w / d->sw + 1;
  if (ho * wo != d->ho * d->wo) { set_error("%s: output size %dx%d does not match weight spatial size %dx%d", what, ho, wo, d->ho, d->wo); return COTB200_EINVAL; }
  g.SH = d->sh; g.SW = d->sw; g.PH = d->ph; g.PW = d->pw; g.DH = d->dh; g.DW = d->dw; g.HO = ho; g.WO = wo;
  return 0;
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_agg_refpad_fwd(const cotb200_agg_desc* d, const void* x, const void* w, void* y, void* stream) {
  VGeo g;
  int rc = vresolve(d, g, "agg_refpad_fwd", false);
  if (rc) return rc;
  if (!x || !w || !y) { set_error("agg_refpad_fwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)g.N * g.heads * g.C * g.HO * g.WO;
  COTB200_DISPATCH_DTYPE(d->dtype, {
    COTB200_PROF_B("agg_refpad_fwd", ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * (g.wc * g.K2 + g.C) * g.HO * g.WO) * sizeof(T));
    const long long items = total / g.rep;
    const bool small = total < (1LL << 31) && (long long)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO < (1LL << 31) && g.H * g.W < (1 << 24);
    if (small && g.KH == g.KW && (g.KH == 3 || g.KH == 5 || g.KH == 7)) {
      if (g.KH == 3) refpad_fwd_fast<T, 3><<<grid_stride_blocks(items, 256, 16), 256, 0, st>>>((const T*)x, (const T*)w, (T*)y, g, (int)items);
      else if (g.KH == 5) refpad_fwd_fast<T, 5><<<grid_stride_blocks(items, 256, 16), 256, 0, st>>>((const T*)x, (const T*)w, (T*)y, g, (int)items);
      else refpad_fwd_fast<T, 7><<<grid_stride_blocks(items, 256, 16), 256, 0, st>>>((const T*)x, (const T*)w, (T*)y, g, (int)items);
    } else {
      refpad_fwd_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)x, (const T*)w, (T*)y, g, total);
    }
    return check_launch("agg_refpad_fwd");
  });
  return 0;
}

extern "C" int cotb200_agg_refpad_bwd(const cotb200_agg_desc* d, const void* dy, const void* x, const void* w, void* dx, void* dw,
                                      void* stream) {
  VGeo g;
  int rc = vresolve(d, g, "agg_refpad_bwd", false);
  if (rc) return rc;
  if (!dy || (dx && !w) || (dw && !x)) { set_error("agg_refpad_bwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(d->dtype, {
    if (dx) {
      const long long total = (long long)g.N * g.C * g.H * g.W;
      COTB200_PROF("agg_refpad_dx");
      refpad_dx_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)w, (T*)dx, g, total);
      rc = check_launch("agg_refpad_dx");
      if (rc) return rc;
    }
    if (dw) {
      const long long total = (long long)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO;
      COTB200_PROF("agg_refpad_dw");
      refpad_dw_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)x, (T*)dw, g, total);
      rc = check_launch("agg_refpad_dw");
    }
    return rc;
  });
  return 0;
}

extern "C" int cotb200_agg_zeropad_dilate_fwd(const cotb200_agg_desc* d, const void* x, const void* w, const void* dilation, void* y,
                                              void* stream) {
  VGeo g;
  int rc = vresolve(d, g, "agg_zeropad_dilate_fwd", true);
  if (rc) return rc;
  if (!x || !w || !dilation || !y) { set_error("agg_zeropad_dilate_fwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)g.N * g.heads * g.C * g.H * g.W;
  COTB200_DISPATCH_DTYPE(d->dtype, {
    COTB200_PROF_B("agg_dilate_fwd", ((double)g.N * g.H * g.W) * ((double)g.C + g.heads * (g.wc * 9.0 + g.C)) * sizeof(T));
    if (total < (1LL << 31) && (long long)g.N * g.heads * g.wc * 9 * g.H * g.W < (1LL << 31))
      dilate_fwd_fast<T><<<grid_stride_blocks(total / g.rep, 256, 16), 256, 0, st>>>((const T*)x, (const T*)w, (const T*)dilation, (T*)y, g, (int)(total / g.rep));
    else
      dilate_fwd_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)x, (const T*)w, (const T*)dilation, (T*)y, g, total);
    return check_launch("agg_zeropad_dilate_fwd");
  });
  return 0;
}

extern "C" int cotb200_agg_zeropad_dilate_bwd(const cotb200_agg_desc* d, const void* dy, const void* x, const void* w,
                                              const void* dilation, void* dx, void* dw, void* stream) {
  VGeo g;
  int rc = vresolve(d, g, "agg_zeropad_dilate_bwd", true);
  if (rc) return rc;
  if (!dy || !dilation || (dx && !w) || (dw && !x)) { set_error("agg_zeropad_dilate_bwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(d->dtype, {
    if (dx) {
      const long long total = (long long)g.N * g.C * g.H * g.W;
      COTB200_PROF("agg_dilate_dx");
      dilate_dx_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)w, (const T*)dilation, (T*)dx, g, total);
      rc = check_launch("agg_dilate_dx");
      if (rc) return rc;
    }
    if (dw) {
      const long long total = (long long)g.N * g.heads * g.wc * 9 * g.H * g.W;
      COTB200_PROF("agg_dilate_dw");
      dilate_dw_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)x, (const T*)dilation, (T*)dw, g, total);
      rc = check_launch("agg_dilate_dw");
    }
    return rc;
  });
  return 0;
}
