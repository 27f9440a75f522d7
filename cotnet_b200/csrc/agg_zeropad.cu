// LocalConv ("aggregation_zeropad") kernels for sm_90a.
//
// Replaces the reference's NVRTC string kernels
//   aggregation_zeropad_forward_kernel          /root/reference/cupy_layers/aggregation_zeropad.py:20-46
//   aggregation_zeropad_input_backward_kernel   :48-79
//   aggregation_zeropad_weight_backward_kernel  :81-110
//   aggregation_zeropad_mix_*                   /root/reference/cupy_layers/aggregation_zeropad_mix.py:20-207
// with runtime-dimension kernels.  The operator is HBM-bound (1.4 FLOP/B fp32): the design goal is to move
// each byte of x / w / y exactly once:
//   * NCHW fast path (k in {3,5}, stride 1, "same" padding, heads 1): one thread owns one pixel of one weight
//     channel, keeps its K*K weights in registers and loops over the C/wc input channels that share them, so a
//     weight element is read from HBM once (the reference re-reads it from 8 distant thread blocks);
//     neighbouring threads' taps overlap in L1.
//   * NHWC fast path: one thread owns a 16-byte channel packet of one pixel; packets of a pixel are
//     contiguous so every warp-wide access is a run of full 128-byte lines.
//   * generic path: any kernel size / stride / dilation / heads / dtype (incl. fp64), 64-bit indexing.
// Accumulation is fp32 (fp64 for double).  Zero padding == skipped taps, exactly like the reference.
#include "common.cuh"
#include "agg.cuh"

namespace cotb200 {

struct Geo {
  int N, C, H, W, heads, wc, KH, KW, SH, SW, PH, PW, DH, DW, HO, WO, K2, rep;
  int layout, gc;
  int fold, Cf, wcf;                           // CoXt fold: channel c -> weight channel (c/Cf)*wcf + (c%Cf)%wcf
  long long x_sn, x_sc, x_sh, x_sw;            // input strides (elements)
  long long w_sn, w_shead, w_sh, w_sw;         // weight strides; (g,tap) offset via w_gt()
  long long y_sn, y_sc, y_sh, y_sw;            // output strides
};

__device__ __forceinline__ int wch_of(const Geo& g, int c) { return (c / g.Cf) * g.wcf + (c % g.Cf) % g.wcf; }

__device__ __forceinline__ long long w_gt(const Geo& g, int gch, int tap) {
  if (g.layout == COTB200_NCHW) return (long long)(gch * g.K2 + tap) * g.HO * g.WO;
  if (g.layout == COTB200_NHWC) return (long long)gch * g.K2 + tap;
  return (long long)((gch / g.gc) * g.K2 + tap) * g.gc + (gch % g.gc);
}

// ------------------------------------------------------------------------------------------------ generic
template <typename T>
__global__ void agg_fwd_generic(const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, Geo g,
                                long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int n, head, c, ho, wo;
    long long r = idx;
    if (g.layout == COTB200_NCHW) {
      wo = r % g.WO; r /= g.WO; ho = r % g.HO; r /= g.HO; c = r % g.C; r /= g.C; head = r % g.heads; n = r / g.heads;
    } else {
      c = r % g.C; r /= g.C; head = r % g.heads; r /= g.heads; wo = r % g.WO; r /= g.WO; ho = r % g.HO; n = r / g.HO;
    }
    const int gch = wch_of(g, c);
    const T* wp = w + n * g.w_sn + head * g.w_shead + ho * g.w_sh + wo * g.w_sw;
    const T* xp = x + n * g.x_sn + c * g.x_sc;
    Acc acc = 0;
    for (int kh = 0; kh < g.KH; ++kh) {
      const int hi = -g.PH + ho * g.SH + kh * g.DH;
      if (hi < 0 || hi >= g.H) continue;
      for (int kw = 0; kw < g.KW; ++kw) {
        const int wi = -g.PW + wo * g.SW + kw * g.DW;
        if (wi < 0 || wi >= g.W) continue;
        acc += to_acc(wp[w_gt(g, gch, kh * g.KW + kw)]) * to_acc(xp[hi * g.x_sh + wi * g.x_sw]);
      }
    }
    y[n * g.y_sn + (long long)(head * g.C + c) * g.y_sc + ho * g.y_sh + wo * g.y_sw] = Elem<T>::from(acc);
  }
}

// dX[n,c,h,w] = sum_head sum_taps w[n,head,c%wc,tap,ho,wo] * dY[n,head*C+c,ho,wo],  ho = (h + p - kh*d)/s when divisible
template <typename T, bool ACCUM>
__global__ void agg_dx_generic(const T* __restrict__ dy, const T* __restrict__ w, T* __restrict__ dx, Geo g,
                               long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int n, c, h, wq;
    long long r = idx;
    if (g.layout == COTB200_NCHW) {
      wq = r % g.W; r /= g.W; h = r % g.H; r /= g.H; c = r % g.C; n = r / g.C;
    } else {
      c = r % g.C; r /= g.C; wq = r % g.W; r /= g.W; h = r % g.H; n = r / g.H;
    }
    const int gch = wch_of(g, c);
    Acc acc = 0;
    for (int head = 0; head < g.heads; ++head) {
      const T* wp = w + n * g.w_sn + head * g.w_shead;
      const T* dp = dy + n * g.y_sn + (long long)(head * g.C + c) * g.y_sc;
      for (int kh = 0; kh < g.KH; ++kh) {
        const int hs = h + g.PH - kh * g.DH;
        if (hs < 0 || hs % g.SH) continue;
        const int ho = hs / g.SH;
        if (ho >= g.HO) continue;
        for (int kw = 0; kw < g.KW; ++kw) {
          const int ws = wq + g.PW - kw * g.DW;
          if (ws < 0 || ws % g.SW) continue;
          const int wo = ws / g.SW;
          if (wo >= g.WO) continue;
          acc += to_acc(wp[ho * g.w_sh + wo * g.w_sw + w_gt(g, gch, kh * g.KW + kw)]) *
                 to_acc(dp[ho * g.y_sh + wo * g.y_sw]);
        }
      }
    }
    T* o = dx + n * g.x_sn + c * g.x_sc + h * g.x_sh + wq * g.x_sw;
    if (ACCUM) acc += to_acc(*o);
    *o = Elem<T>::from(acc);
  }
}

// Mix op: dX = dX(kernel 1) + dX(kernel 2) accumulated in fp32 in ONE pass (a second accumulate-in-place launch would
// round the first half to the storage type first -- visible in bf16).
template <typename T>
__global__ void agg_dx_generic2(const T* __restrict__ dy1, const T* __restrict__ w1, Geo g1, const T* __restrict__ dy2,
                                const T* __restrict__ w2, Geo g2, T* __restrict__ dx, long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    const int wq = r % g1.W; r /= g1.W;
    const int h = r % g1.H; r /= g1.H;
    const int c = r % g1.C;
    const int n = r / g1.C;
    Acc acc = 0;
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      const Geo& g = pass ? g2 : g1;
      const T* dy = pass ? dy2 : dy1;
      const T* w = pass ? w2 : w1;
      const int gch = wch_of(g, c);
      for (int head = 0; head < g.heads; ++head) {
        const T* wp = w + n * g.w_sn + head * g.w_shead;
        const T* dp = dy + n * g.y_sn + (long long)(head * g.C + c) * g.y_sc;
        for (int kh = 0; kh < g.KH; ++kh) {
          const int hs = h + g.PH - kh * g.DH;
          if (hs < 0 || hs % g.SH) continue;
          const int ho = hs / g.SH;
          if (ho >= g.HO) continue;
          for (int kw = 0; kw < g.KW; ++kw) {
            const int ws = wq + g.PW - kw * g.DW;
            if (ws < 0 || ws % g.SW) continue;
            const int wo = ws / g.SW;
            if (wo >= g.WO) continue;
            acc += to_acc(wp[ho * g.w_sh + wo * g.w_sw + w_gt(g, gch, kh * g.KW + kw)]) *
                   to_acc(dp[ho * g.y_sh + wo * g.y_sw]);
          }
        }
      }
    }
    dx[n * g1.x_sn + c * g1.x_sc + h * g1.x_sh + wq * g1.x_sw] = Elem<T>::from(acc);
  }
}

// dW[n,head,gch,tap,ho,wo] = sum_{cc = gch (mod wc)} x[n,cc,hi,wi] * dY[n,head*C+cc,ho,wo]   (0 for padded taps)
template <typename T>
__global__ void agg_dw_generic(const T* __restrict__ dy, const T* __restrict__ x, T* __restrict__ dw, Geo g,
                               long long total) {
  using Acc = typename Elem<T>::Acc;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int n, head, gch, tap, ho, wo;
    long long r = idx;
    if (g.layout == COTB200_NCHW) {
      wo = r % g.WO; r /= g.WO; ho = r % g.HO; r /= g.HO; tap = r % g.K2; r /= g.K2; gch = r % g.wc; r /= g.wc;
      head = r % g.heads; n = r / g.heads;
    } else {
      int jdx = r % (g.wc * g.K2); r /= (g.wc * g.K2);
      head = r % g.heads; r /= g.heads; wo = r % g.WO; r /= g.WO; ho = r % g.HO; n = r / g.HO;
      if (g.layout == COTB200_NHWC) { gch = jdx / g.K2; tap = jdx % g.K2; }
      else { int chunk = jdx / (g.K2 * g.gc), rr = jdx % (g.K2 * g.gc); tap = rr / g.gc; gch = chunk * g.gc + rr % g.gc; }
    }
    const int kh = tap / g.KW, kw = tap % g.KW;
    const int hi = -g.PH + ho * g.SH + kh * g.DH;
    const int wi = -g.PW + wo * g.SW + kw * g.DW;
    Acc acc = 0;
    if (hi >= 0 && hi < g.H && wi >= 0 && wi < g.W) {
      const int cbase = (gch / g.wcf) * g.Cf + gch % g.wcf;
      for (int j = 0; j < g.rep; ++j) {
        const int cc = cbase + j * g.wcf;
        acc += to_acc(x[n * g.x_sn + cc * g.x_sc + hi * g.x_sh + wi * g.x_sw]) *
               to_acc(dy[n * g.y_sn + (long long)(head * g.C + cc) * g.y_sc + ho * g.y_sh + wo * g.y_sw]);
      }
    }
    dw[n * g.w_sn + head * g.w_shead + ho * g.w_sh + wo * g.w_sw + w_gt(g, gch, tap)] = Elem<T>::from(acc);
  }
}

// ------------------------------------------------------------------------------------------------ NCHW fast
// Thread = (n, gch, pixel).  K*K weights live in registers; loop over the rep = C/wc sharers.
// Planes are [H*W] contiguous; y batch stride (y_sn) is a parameter so the mix op can write channel halves.
template <typename T, int K>
__global__ void __launch_bounds__(256)
agg_fwd_nchw_fast(const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, int N, int C, int H, int W,
                  int wc, int rep, long long y_sn, long long w_sn, int total) {
  constexpr int R = K / 2, K2 = K * K;
  const int HW = H * W;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int p = idx % HW;
    const int gch = (idx / HW) % wc;
    const int n = idx / (HW * wc);
    const int h = p / W, wq = p - h * W;
    float wt[K2];
    const T* wp = w + n * w_sn + ((long long)gch * K2) * HW + p;
#pragma unroll
    for (int t = 0; t < K2; ++t) {
      const int dh = t / K - R, dw = t % K - R;
      const bool ok = (unsigned)(h + dh) < (unsigned)H && (unsigned)(wq + dw) < (unsigned)W;
      wt[t] = ok ? Elem<T>::ld(wp + (long long)t * HW) : 0.f;   // padded taps contribute 0
    }
    const T* xp = x + ((long long)n * C + gch) * HW + p;
    T* yp = y + n * y_sn + (long long)gch * HW + p;
#pragma unroll 2
    for (int j = 0; j < rep; ++j) {
      float acc = 0.f;
#pragma unroll
      for (int t = 0; t < K2; ++t) {
        const int dh = t / K - R, dw = t % K - R;
        const bool ok = (unsigned)(h + dh) < (unsigned)H && (unsigned)(wq + dw) < (unsigned)W;
        const float xv = ok ? Elem<T>::ld(xp + dh * W + dw) : 0.f;
        acc = fmaf(wt[t], xv, acc);
      }
      *yp = Elem<T>::from(acc);
      xp += (long long)wc * HW;
      yp += (long long)wc * HW;
    }
  }
}

// Mix forward, fused: one pass over x produces both the 3x3 and the 5x5 aggregation (x read once).
template <typename T>
__global__ void __launch_bounds__(256)
agg_mix_fwd_nchw_fast(const T* __restrict__ x, const T* __restrict__ w1, const T* __restrict__ w2,
                      T* __restrict__ y, int N, int C, int H, int W, int wc, int rep, int total) {
  const int HW = H * W;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int p = idx % HW;
    const int gch = (idx / HW) % wc;
    const int n = idx / (HW * wc);
    const int h = p / W, wq = p - h * W;
    float a[9], b[25];
    const T* w1p = w1 + ((long long)(n * wc + gch) * 9) * HW + p;
    const T* w2p = w2 + ((long long)(n * wc + gch) * 25) * HW + p;
#pragma unroll
    for (int t = 0; t < 25; ++t) {
      const int dh = t / 5 - 2, dw = t % 5 - 2;
      const bool ok = (unsigned)(h + dh) < (unsigned)H && (unsigned)(wq + dw) < (unsigned)W;
      b[t] = ok ? Elem<T>::ld(w2p + (long long)t * HW) : 0.f;
      if (dh >= -1 && dh <= 1 && dw >= -1 && dw <= 1) {
        const int t3 = (dh + 1) * 3 + (dw + 1);
        a[t3] = ok ? Elem<T>::ld(w1p + (long long)t3 * HW) : 0.f;
      }
    }
    const T* xp = x + ((long long)n * C + gch) * HW + p;
    T* y1 = y + ((long long)n * 2 * C + gch) * HW + p;          // channel (0*heads+0)*C + c
    T* y2 = y1 + (long long)C * HW;                              // channel (1*heads+0)*C + c
    for (int j = 0; j < rep; ++j) {
      float acc1 = 0.f, acc2 = 0.f;
#pragma unroll
      for (int t = 0; t < 25; ++t) {
        const int dh = t / 5 - 2, dw = t % 5 - 2;
        const bool ok = (unsigned)(h + dh) < (unsigned)H && (unsigned)(wq + dw) < (unsigned)W;
        const float xv = ok ? Elem<T>::ld(xp + dh * W + dw) : 0.f;
        acc2 = fmaf(b[t], xv, acc2);
        if (dh >= -1 && dh <= 1 && dw >= -1 && dw <= 1) acc1 = fmaf(a[(dh + 1) * 3 + (dw + 1)], xv, acc1);
      }
      *y1 = Elem<T>::from(acc1);
      *y2 = Elem<T>::from(acc2);
      xp += (long long)wc * HW; y1 += (long long)wc * HW; y2 += (long long)wc * HW;
    }
  }
}

// Fused backward: dW (registers, summed over the sharers) and dX (per sharer) in one pass over dY.
//   dW[n,g,t,p]   = sum_j x[n,c_j,p+off_t] * dY[n,c_j,p]
//   dX[n,c_j,p]   = sum_t w[n,g,t,p-off_t] * dY[n,c_j,p-off_t]
// ACC_DX: dX += (used by the mix op's second kernel).
template <typename T, int K, bool DX, bool DW, bool ACC_DX>
__global__ void __launch_bounds__(256)
agg_bwd_nchw_fast(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ dx,
                  T* __restrict__ dw, int N, int C, int H, int W, int wc, int rep, long long dy_sn, long long w_sn, int total) {
  constexpr int R = K / 2, K2 = K * K;
  const int HW = H * W;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int p = idx % HW;
    const int gch = (idx / HW) % wc;
    const int n = idx / (HW * wc);
    const int h = p / W, wq = p - h * W;
    float ws[K2];   // DX: w at the shifted (output) positions p - off_t
    float gw[K2];   // DW accumulators
    const T* wp = w + n * w_sn + ((long long)gch * K2) * HW + p;
#pragma unroll
    for (int t = 0; t < K2; ++t) {
      const int dh = t / K - R, dw_ = t % K - R;
      gw[t] = 0.f;
      if (DX) {
        const bool ok = (unsigned)(h - dh) < (unsigned)H && (unsigned)(wq - dw_) < (unsigned)W;
        ws[t] = ok ? Elem<T>::ld(wp + (long long)t * HW - (dh * W + dw_)) : 0.f;
      }
    }
    const T* xp = x + ((long long)n * C + gch) * HW + p;
    const T* dp = dy + n * dy_sn + (long long)gch * HW + p;
    T* dxp = dx + ((long long)n * C + gch) * HW + p;
#pragma unroll 2
    for (int j = 0; j < rep; ++j) {
      if (DW) {
        const float g0 = Elem<T>::ld(dp);
#pragma unroll
        for (int t = 0; t < K2; ++t) {
          const int dh = t / K - R, dw_ = t % K - R;
          const bool ok = (unsigned)(h + dh) < (unsigned)H && (unsigned)(wq + dw_) < (unsigned)W;
          const float xv = ok ? Elem<T>::ld(xp + dh * W + dw_) : 0.f;
          gw[t] = fmaf(xv, g0, gw[t]);
        }
      }
      if (DX) {
        float acc = 0.f;
#pragma unroll
        for (int t = 0; t < K2; ++t) {
          const int dh = t / K - R, dw_ = t % K - R;
          const bool ok = (unsigned)(h - dh) < (unsigned)H && (unsigned)(wq - dw_) < (unsigned)W;
          const float gv = ok ? Elem<T>::ld(dp - (dh * W + dw_)) : 0.f;
          acc = fmaf(ws[t], gv, acc);
        }
        if (ACC_DX) acc += to_acc(*dxp);
        *dxp = Elem<T>::from(acc);
      }
      xp += (long long)wc * HW; dp += (long long)wc * HW; dxp += (long long)wc * HW;
    }
    if (DW) {
      T* dwp = dw + n * w_sn + ((long long)gch * K2) * HW + p;
#pragma unroll
      for (int t = 0; t < K2; ++t) dwp[(long long)t * HW] = Elem<T>::from(gw[t]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ NHWC fast (3x3)
// Thread = (pixel, VEC-channel packet).  wc % VEC == 0 so a packet maps to VEC consecutive weight channels.
// TAP=false: weights [.., g*9 + t]   (torch channels_last view of the reference layout)
// TAP=true : weights [.., (g/VEC)*9*VEC + t*VEC + g%VEC]   (block-internal, gc == VEC)
template <typename T, int VEC, bool TAP>
__device__ __forceinline__ float wsel(const Pack<T, VEC>* wp, int i, int t) {
  if (TAP) return to_acc(wp[t].v[i]);
  const int f = i * 9 + t;
  return to_acc(wp[f / VEC].v[f % VEC]);
}

template <typename T, int VEC, bool TAP>
__global__ void __launch_bounds__(256)
agg3_fwd_nhwc_fast(const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, int N, int C, int H, int W,
                   int Cf, int wcf, long long x_sn, long long x_sp, long long w_sn, long long w_sp, long long y_sn,
                   long long y_sp, int total) {
  const int CQ = C / VEC;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int q = idx % CQ;
    int pix = idx / CQ;
    const int wq = pix % W; pix /= W;
    const int h = pix % H;
    const int n = pix / H;
    const int c0 = q * VEC;
    const int g0 = (c0 / Cf) * wcf + (c0 % Cf) % wcf;   // CoXt fold aware (Cf = C, wcf = wc when fold == 1)
    const T* wb = w + n * w_sn + (long long)(h * W + wq) * w_sp + (long long)g0 * 9;
    Pack<T, VEC> wp[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) wp[t] = ld_pack<T, VEC>(wb + t * VEC);
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
    const T* xb = x + n * x_sn + c0;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int hh = h + t / 3 - 1, ww = wq + t % 3 - 1;
      if ((unsigned)hh < (unsigned)H && (unsigned)ww < (unsigned)W) {
        const Pack<T, VEC> xv = ld_pack<T, VEC>(xb + (long long)(hh * W + ww) * x_sp);
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] = fmaf(wsel<T, VEC, TAP>(wp, i, t), to_acc(xv.v[i]), acc[i]);
      }
    }
    Pack<T, VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(acc[i]);
    st_pack<T, VEC>(y + n * y_sn + (long long)(h * W + wq) * y_sp + c0, o);
  }
}

// dX[p, c0+i] = sum_t w[p - off_t][(g0+i), t] * dY[p - off_t][c0+i]
template <typename T, int VEC, bool TAP>
__global__ void __launch_bounds__(256)
agg3_dx_nhwc_fast(const T* __restrict__ dy, const T* __restrict__ w, T* __restrict__ dx, int N, int C, int H, int W,
                  int Cf, int wcf, long long x_sn, long long x_sp, long long w_sn, long long w_sp, long long y_sn,
                  long long y_sp, int total) {
  const int CQ = C / VEC;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int q = idx % CQ;
    int pix = idx / CQ;
    const int wq = pix % W; pix /= W;
    const int h = pix % H;
    const int n = pix / H;
    const int c0 = q * VEC;
    const int g0 = (c0 / Cf) * wcf + (c0 % Cf) % wcf;   // CoXt fold aware (Cf = C, wcf = wc when fold == 1)
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int hh = h - (t / 3 - 1), ww = wq - (t % 3 - 1);   // the output pixel whose tap t reads (h, wq)
      if ((unsigned)hh < (unsigned)H && (unsigned)ww < (unsigned)W) {
        const long long po = (long long)(hh * W + ww);
        const Pack<T, VEC> gv = ld_pack<T, VEC>(dy + n * y_sn + po * y_sp + c0);
        const T* wb = w + n * w_sn + po * w_sp + (long long)g0 * 9;
        if (TAP) {
          const Pack<T, VEC> wv = ld_pack<T, VEC>(wb + t * VEC);
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] = fmaf(to_acc(wv.v[i]), to_acc(gv.v[i]), acc[i]);
        } else {
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] = fmaf(Elem<T>::ld(wb + i * 9 + t), to_acc(gv.v[i]), acc[i]);
        }
      }
    }
    Pack<T, VEC> o;
#pragma unroll
    for (int i = 0; i < VEC; ++i) o.v[i] = Elem<T>::from(acc[i]);
    st_pack<T, VEC>(dx + n * x_sn + (long long)(h * W + wq) * x_sp + c0, o);
  }
}

// dW[p, (g0+i), t] = sum_j x[p + off_t][j*wc + g0 + i] * dY[p][j*wc + g0 + i].   Thread = (pixel, weight packet).
template <typename T, int VEC, bool TAP>
__global__ void __launch_bounds__(256)
agg3_dw_nhwc_fast(const T* __restrict__ dy, const T* __restrict__ x, T* __restrict__ dw, int N, int C, int H, int W,
                  int wc, int Cf, int wcf, int rep, long long x_sn, long long x_sp, long long w_sn, long long w_sp, long long y_sn,
                  long long y_sp, int total) {
  const int GQ = wc / VEC;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int gq = idx % GQ;
    int pix = idx / GQ;
    const int wq = pix % W; pix /= W;
    const int h = pix % H;
    const int n = pix / H;
    const int g0 = gq * VEC;
    float acc[9][VEC];
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[t][i] = 0.f;
    const int cb = (g0 / wcf) * Cf + g0 % wcf;             // first channel using weight channel g0
    const T* dp = dy + n * y_sn + (long long)(h * W + wq) * y_sp + cb;
    const T* xb = x + n * x_sn + cb;
    for (int j = 0; j < rep; ++j) {
      const Pack<T, VEC> gv = ld_pack<T, VEC>(dp + j * wcf);
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int hh = h + t / 3 - 1, ww = wq + t % 3 - 1;
        if ((unsigned)hh < (unsigned)H && (unsigned)ww < (unsigned)W) {
          const Pack<T, VEC> xv = ld_pack<T, VEC>(xb + (long long)(hh * W + ww) * x_sp + j * wcf);
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[t][i] = fmaf(to_acc(xv.v[i]), to_acc(gv.v[i]), acc[t][i]);
        }
      }
    }
    T* wb = dw + n * w_sn + (long long)(h * W + wq) * w_sp + (long long)g0 * 9;
    Pack<T, VEC> o[9];
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        if (TAP) o[t].v[i] = Elem<T>::from(acc[t][i]);
        else { const int f = i * 9 + t; o[f / VEC].v[f % VEC] = Elem<T>::from(acc[t][i]); }
      }
#pragma unroll
    for (int t = 0; t < 9; ++t) st_pack<T, VEC>(wb + t * VEC, o[t]);
  }
}

// ------------------------------------------------------------------------------------------------ host
static int resolve(const cotb200_agg_desc* d, Geo& g) {
  if (!d) { set_error("desc is NULL"); return COTB200_ENULL; }
  if (d->n <= 0 || d->c <= 0 || d->h <= 0 || d->w <= 0 || d->heads <= 0 || d->wc <= 0 || d->kh <= 0 || d->kw <= 0 ||
      d->sh <= 0 || d->sw <= 0 || d->dh <= 0 || d->dw <= 0 || d->ph < 0 || d->pw < 0 || d->ho <= 0 || d->wo <= 0) {
    set_error("non-positive dimension in desc"); return COTB200_EINVAL;
  }
  if (d->c % d->wc) { set_error("input channels %d not divisible by weight channels %d", d->c, d->wc); return COTB200_EINVAL; }
  // aggregation_zeropad.py:119-122
  const int span_h = d->h + 2 * d->ph - (d->dh * (d->kh - 1) + 1), span_w = d->w + 2 * d->pw - (d->dw * (d->kw - 1) + 1);
  // a window larger than the padded input has no output position (the division below truncates towards zero: it would
  // yield a size of 1, or two negative sizes whose product matches the weight plane)
  if (span_h < 0 || span_w < 0) { set_error("kernel window larger than the padded input %dx%d", d->h + 2 * d->ph, d->w + 2 * d->pw); return COTB200_EINVAL; }
  const int ho = span_h / d->sh + 1, wo = span_w / d->sw + 1;
  if (ho * wo != d->ho * d->wo) {
    set_error("output size %dx%d does not match weight spatial size %dx%d", ho, wo, d->ho, d->wo); return COTB200_EINVAL;
  }
  g.N = d->n; g.C = d->c; g.H = d->h; g.W = d->w; g.heads = d->heads; g.wc = d->wc; g.KH = d->kh; g.KW = d->kw;
  g.SH = d->sh; g.SW = d->sw; g.PH = d->ph; g.PW = d->pw; g.DH = d->dh; g.DW = d->dw; g.HO = ho; g.WO = wo;
  g.K2 = d->kh * d->kw; g.rep = d->c / d->wc; g.layout = d->layout; g.gc = d->gc > 0 ? d->gc : 1;
  g.fold = d->fold > 0 ? d->fold : 1;
  if (d->c % g.fold || d->wc % g.fold || (d->c / g.fold) % (d->wc / g.fold)) {
    set_error("fold %d does not divide c=%d / wc=%d", g.fold, d->c, d->wc); return COTB200_EINVAL;
  }
  g.Cf = d->c / g.fold; g.wcf = d->wc / g.fold;
  const long long J = (long long)d->heads * d->wc * g.K2;
  if (d->layout == COTB200_NCHW) {
    g.x_sw = 1; g.x_sh = g.W; g.x_sc = (long long)g.H * g.W; g.x_sn = g.x_sc * g.C;
    g.w_sw = 1; g.w_sh = g.WO; g.w_shead = (long long)g.wc * g.K2 * g.HO * g.WO; g.w_sn = g.w_shead * g.heads;
    g.y_sw = 1; g.y_sh = g.WO; g.y_sc = (long long)g.HO * g.WO; g.y_sn = g.y_sc * g.C * g.heads;
  } else if (d->layout == COTB200_NHWC || d->layout == COTB200_NHWC_TAP) {
    if (d->layout == COTB200_NHWC_TAP && (g.wc % g.gc)) { set_error("gc %d does not divide wc %d", g.gc, g.wc); return COTB200_EINVAL; }
    g.x_sc = 1; g.x_sw = d->x_sp ? d->x_sp : g.C; g.x_sh = g.x_sw * g.W; g.x_sn = d->x_sn ? d->x_sn : g.x_sh * g.H;
    g.w_sw = d->w_sp ? d->w_sp : J; g.w_sh = g.w_sw * g.WO; g.w_sn = d->w_sn ? d->w_sn : g.w_sh * g.HO;
    g.w_shead = (long long)g.wc * g.K2;
    g.y_sc = 1; g.y_sw = d->y_sp ? d->y_sp : (long long)g.C * g.heads; g.y_sh = g.y_sw * g.WO;
    g.y_sn = d->y_sn ? d->y_sn : g.y_sh * g.HO;
  } else { set_error("unknown layout %d", d->layout); return COTB200_ELAYOUT; }
  return 0;
}

static bool is_same3(const Geo& g, int K) {
  return g.KH == K && g.KW == K && g.SH == 1 && g.SW == 1 && g.DH == 1 && g.DW == 1 && g.PH == K / 2 && g.PW == K / 2 &&
         g.heads == 1;
}
static bool nofold(const Geo& g) { return g.fold == 1; }
static bool fits32(const Geo& g) {
  const long long a = (long long)g.N * g.C * g.heads * g.HO * g.WO, b = (long long)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO,
                  c = (long long)g.N * g.C * g.H * g.W;
  return a < (1LL << 31) && b < (1LL << 31) && c < (1LL << 31);
}

// largest packet width (elements) usable by the NHWC fast path for this call, 0 if none
template <typename T>
static int nhwc_vec(const Geo& g, const void* a, const void* b, const void* c) {
  if (!is_same3(g, 3) || !fits32(g)) return 0;
  for (int vec = 16 / (int)sizeof(T); vec >= 1; vec >>= 1) {
    if (g.layout == COTB200_NHWC_TAP && vec != g.gc) continue;
    const int bytes = vec * (int)sizeof(T);
    if (bytes < 4 && vec != 1) continue;
    if (g.wcf % vec) continue;
    auto okp = [&](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) % bytes) == 0; };
    auto oks = [&](long long s) { return (s * (long long)sizeof(T)) % bytes == 0; };
    if (!okp(a) || !okp(b) || !okp(c)) continue;
    if (!oks(g.x_sw) || !oks(g.x_sn) || !oks(g.w_sw) || !oks(g.w_sn) || !oks(g.y_sw) || !oks(g.y_sn)) continue;
    if (vec == 1 && g.layout == COTB200_NHWC_TAP && g.gc != 1) continue;
    return vec;
  }
  return 0;
}

static Nhwc2Args nhwc2_args(const Geo& g) {
  Nhwc2Args a;
  a.N = g.N; a.C = g.C; a.H = g.H; a.W = g.W; a.wc = g.wc; a.fold = g.fold; a.layout = g.layout; a.gc = g.gc; a.dtype = 0;
  a.x_sn = g.x_sn; a.x_sp = g.x_sw; a.w_sn = g.w_sn; a.w_sp = g.w_sw; a.y_sn = g.y_sn; a.y_sp = g.y_sw;
  return a;
}

template <typename T>
static int fwd_impl(const Geo& g, const T* x, const T* w, T* y, cudaStream_t st) {
  if (g.layout != COTB200_NCHW && is_same3(g, 3)) {
    int rc2 = 0;
    if (agg_tma_fwd<T>(nhwc2_args(g), x, w, y, st, &rc2)) return rc2;     // persistent TMA-pipelined kernel (TAP layout)
    if (nhwc2_fwd<T>(nhwc2_args(g), x, w, y, st, &rc2)) return rc2;
  }
  if (g.layout == COTB200_NCHW && nofold(g) && fits32(g) && is_same3(g, 3) && g.w_sn == (long long)g.wc * 9 * g.H * g.W) {
    int rc2 = 0;
    if (g.x_sn == (long long)g.C * g.H * g.W &&
        nchw_tma_launch<T>(0, g.N, g.C, g.H, g.W, g.wc, g.x_sn, 0, g.y_sn, x, w, y, st, &rc2)) return rc2;
    if (nchw2_fwd<T>(g.N, g.C, g.H, g.W, g.wc, g.y_sn, x, w, y, st, &rc2)) return rc2;
  }
  if (g.layout == COTB200_NCHW && nofold(g) && fits32(g) && (is_same3(g, 3) || is_same3(g, 5))) {
    if constexpr (!std::is_same<T, double>::value) {
      const int total = g.N * g.wc * g.H * g.W;
      const int grid = grid_stride_blocks(total, 256, 8);
      COTB200_PROF_B(g.KH == 3 ? "agg_fwd_nchw_k3" : "agg_fwd_nchw_k5", ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO + (double)g.N * g.heads * g.C * g.HO * g.WO) * sizeof(T));
      if (g.KH == 3) agg_fwd_nchw_fast<T, 3><<<grid, 256, 0, st>>>(x, w, y, g.N, g.C, g.H, g.W, g.wc, g.rep, g.y_sn, g.w_sn, total);
      else agg_fwd_nchw_fast<T, 5><<<grid, 256, 0, st>>>(x, w, y, g.N, g.C, g.H, g.W, g.wc, g.rep, g.y_sn, g.w_sn, total);
      return check_launch("agg_fwd_nchw_fast");
    }
  }
  if (g.layout != COTB200_NCHW) {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = nhwc_vec<T>(g, x, w, y);
      if (vec) {
        const int total = g.N * g.H * g.W * (g.C / vec);
        const int grid = grid_stride_blocks(total, 256, 8);
        const bool tap = g.layout == COTB200_NHWC_TAP;
        COTB200_PROF_B("agg3_fwd_nhwc", ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO + (double)g.N * g.heads * g.C * g.HO * g.WO) * sizeof(T));
#define COTB200_LAUNCH_FWD(V)                                                                                     \
  if (vec == V) {                                                                                                 \
    if (tap) agg3_fwd_nhwc_fast<T, V, true><<<grid, 256, 0, st>>>(x, w, y, g.N, g.C, g.H, g.W, g.Cf, g.wcf, g.x_sn, \
                                                                   g.x_sw, g.w_sn, g.w_sw, g.y_sn, g.y_sw, total); \
    else agg3_fwd_nhwc_fast<T, V, false><<<grid, 256, 0, st>>>(x, w, y, g.N, g.C, g.H, g.W, g.Cf, g.wcf, g.x_sn, g.x_sw, \
                                                                g.w_sn, g.w_sw, g.y_sn, g.y_sw, total);            \
    return check_launch("agg3_fwd_nhwc_fast");                                                                    \
  }
        if constexpr (sizeof(T) == 2) { COTB200_LAUNCH_FWD(8) }
        COTB200_LAUNCH_FWD(4) COTB200_LAUNCH_FWD(2) COTB200_LAUNCH_FWD(1)
#undef COTB200_LAUNCH_FWD
      }
    }
  }
  const long long total = (long long)g.N * g.heads * g.C * g.HO * g.WO;
  COTB200_PROF_B("agg_fwd_generic", ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO + (double)g.N * g.heads * g.C * g.HO * g.WO) * sizeof(T));
  agg_fwd_generic<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>(x, w, y, g, total);
  return check_launch("agg_fwd_generic");
}

template <typename T>
static int bwd_impl(const Geo& g, const T* dy, const T* x, const T* w, T* dx, T* dw, bool acc_dx, cudaStream_t st) {
  if (!dx && !dw) return 0;
  if (g.layout == COTB200_NCHW && nofold(g) && fits32(g) && is_same3(g, 3) && !acc_dx && g.w_sn == (long long)g.wc * 9 * g.H * g.W) {
    int rc2 = 0;
    if (g.H * g.W <= 256 && nchw_plane_launch<T>(dx && dw ? 3 : (dx ? 1 : 2), g.N, g.C, g.H, g.W, g.wc, g.x_sn, g.y_sn, g.w_sn, dy, x, w,
                                                 dx, dw, st, &rc2)) return rc2;
    if (g.x_sn == (long long)g.C * g.H * g.W && g.w_sn == (long long)g.wc * 9 * g.H * g.W) {
      // TMA-pipelined kernels, one per gradient; if only one of the two is eligible the register kernel does the other
      int done_dx = !dx, done_dw = !dw;
      if (dx && nchw_tma_launch<T>(1, g.N, g.C, g.H, g.W, g.wc, g.y_sn, 0, g.x_sn, dy, w, dx, st, &rc2)) { if (rc2) return rc2; done_dx = 1; }
      if (dw && nchw_tma_launch<T>(2, g.N, g.C, g.H, g.W, g.wc, g.x_sn, g.y_sn, g.w_sn, x, dy, dw, st, &rc2)) { if (rc2) return rc2; done_dw = 1; }
      if (done_dx && done_dw) return 0;
      if (nchw2_bwd<T>(g.N, g.C, g.H, g.W, g.wc, g.y_sn, dy, x, w, done_dx ? nullptr : dx, done_dw ? nullptr : dw, st, &rc2)) return rc2;
      if (done_dx) dx = nullptr;
      if (done_dw) dw = nullptr;
    } else if (nchw2_bwd<T>(g.N, g.C, g.H, g.W, g.wc, g.y_sn, dy, x, w, dx, dw, st, &rc2)) return rc2;
  }
  if (g.layout == COTB200_NCHW && nofold(g) && fits32(g) && (is_same3(g, 3) || is_same3(g, 5))) {
    if constexpr (!std::is_same<T, double>::value) {
      const int total = g.N * g.wc * g.H * g.W;
      const int grid = grid_stride_blocks(total, 256, 8);
      COTB200_PROF_B(dx && dw ? "agg_bwd_nchw_dxdw" : (dx ? "agg_bwd_nchw_dx" : "agg_bwd_nchw_dw"), (dx && dw ? 1.0 : 0.0) * ((double)g.N * g.C * g.H * g.W + (double)g.N * g.wc * g.K2 * g.HO * g.WO) * sizeof(T) + ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO + (double)g.N * g.heads * g.C * g.HO * g.WO) * sizeof(T));
#define COTB200_LAUNCH_BWD(K, DX, DW, ACC)                                                                          \
  agg_bwd_nchw_fast<T, K, DX, DW, ACC><<<grid, 256, 0, st>>>(dy, x, w, dx, dw, g.N, g.C, g.H, g.W, g.wc, g.rep,      \
                                                            g.y_sn, g.w_sn, total)
      if (g.KH == 3) {
        if (dx && dw) { if (acc_dx) COTB200_LAUNCH_BWD(3, true, true, true); else COTB200_LAUNCH_BWD(3, true, true, false); }
        else if (dx) { if (acc_dx) COTB200_LAUNCH_BWD(3, true, false, true); else COTB200_LAUNCH_BWD(3, true, false, false); }
        else COTB200_LAUNCH_BWD(3, false, true, false);
      } else {
        if (dx && dw) { if (acc_dx) COTB200_LAUNCH_BWD(5, true, true, true); else COTB200_LAUNCH_BWD(5, true, true, false); }
        else if (dx) { if (acc_dx) COTB200_LAUNCH_BWD(5, true, false, true); else COTB200_LAUNCH_BWD(5, true, false, false); }
        else COTB200_LAUNCH_BWD(5, false, true, false);
      }
#undef COTB200_LAUNCH_BWD
      return check_launch("agg_bwd_nchw_fast");
    }
  }
  if (g.layout == COTB200_NHWC_TAP && !acc_dx && is_same3(g, 3)) {
    // second-generation kernels; whatever they do not take falls through to the first-generation ones below
    int rc2 = 0;
    if (dx && agg_tma_dx<T>(nhwc2_args(g), dy, w, dx, st, &rc2)) { if (rc2) return rc2; dx = nullptr; }
    if (dw && agg_tma_dw<T>(nhwc2_args(g), dy, x, dw, st, &rc2)) { if (rc2) return rc2; dw = nullptr; }
    if (dx && nhwc2_dx<T>(nhwc2_args(g), dy, w, dx, st, &rc2)) { if (rc2) return rc2; dx = nullptr; }
    if (dw && nhwc2_dw<T>(nhwc2_args(g), dy, x, dw, st, &rc2)) { if (rc2) return rc2; dw = nullptr; }
    if (!dx && !dw) return 0;
  }
  if (g.layout != COTB200_NCHW && !acc_dx) {
    if constexpr (!std::is_same<T, double>::value) {
      const int vec = nhwc_vec<T>(g, dy, x, w);
      auto okp = [&](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) % (vec * sizeof(T))) == 0; };
      if (vec && okp(dx) && okp(dw)) {
        const bool tap = g.layout == COTB200_NHWC_TAP;
        int rc = 0;
#define COTB200_LAUNCH_BWD(V)                                                                                        \
  if (vec == V) {                                                                                                    \
    if (dx) {                                                                                                        \
      const int total = g.N * g.H * g.W * (g.C / V);                                                                 \
      const int grid = grid_stride_blocks(total, 256, 8);                                                            \
      COTB200_PROF_B("agg3_dx_nhwc", ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO + (double)g.N * g.heads * g.C * g.HO * g.WO) * sizeof(T));                                                                                 \
      if (tap) agg3_dx_nhwc_fast<T, V, true><<<grid, 256, 0, st>>>(dy, w, dx, g.N, g.C, g.H, g.W, g.Cf, g.wcf, g.x_sn, \
                                                                    g.x_sw, g.w_sn, g.w_sw, g.y_sn, g.y_sw, total);  \
      else agg3_dx_nhwc_fast<T, V, false><<<grid, 256, 0, st>>>(dy, w, dx, g.N, g.C, g.H, g.W, g.Cf, g.wcf, g.x_sn, g.x_sw, \
                                                                 g.w_sn, g.w_sw, g.y_sn, g.y_sw, total);             \
      rc = check_launch("agg3_dx_nhwc_fast");                                                                        \
      if (rc) return rc;                                                                                             \
    }                                                                                                                \
    if (dw) {                                                                                                        \
      const int total = g.N * g.H * g.W * (g.wc / V);                                                                \
      const int grid = grid_stride_blocks(total, 256, 8);                                                            \
      COTB200_PROF_B("agg3_dw_nhwc", ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO + (double)g.N * g.heads * g.C * g.HO * g.WO) * sizeof(T));                                                                                 \
      if (tap) agg3_dw_nhwc_fast<T, V, true><<<grid, 256, 0, st>>>(dy, x, dw, g.N, g.C, g.H, g.W, g.wc, g.Cf, g.wcf, g.rep, \
                                                                    g.x_sn, g.x_sw, g.w_sn, g.w_sw, g.y_sn, g.y_sw,  \
                                                                    total);                                          \
      else agg3_dw_nhwc_fast<T, V, false><<<grid, 256, 0, st>>>(dy, x, dw, g.N, g.C, g.H, g.W, g.wc, g.Cf, g.wcf, g.rep, g.x_sn, \
                                                                 g.x_sw, g.w_sn, g.w_sw, g.y_sn, g.y_sw, total);     \
      rc = check_launch("agg3_dw_nhwc_fast");                                                                        \
    }                                                                                                                \
    return rc;                                                                                                       \
  }
        if constexpr (sizeof(T) == 2) { COTB200_LAUNCH_BWD(8) }
        COTB200_LAUNCH_BWD(4) COTB200_LAUNCH_BWD(2) COTB200_LAUNCH_BWD(1)
#undef COTB200_LAUNCH_BWD
      }
    }
  }
  int rc = 0;
  if (dx) {
    const long long total = (long long)g.N * g.C * g.H * g.W;
    COTB200_PROF_B("agg_dx_generic", ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO + (double)g.N * g.heads * g.C * g.HO * g.WO) * sizeof(T));
    if (acc_dx) agg_dx_generic<T, true><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>(dy, w, dx, g, total);
    else agg_dx_generic<T, false><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>(dy, w, dx, g, total);
    rc = check_launch("agg_dx_generic");
    if (rc) return rc;
  }
  if (dw) {
    const long long total = (long long)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO;
    COTB200_PROF_B("agg_dw_generic", ((double)g.N * g.C * g.H * g.W + (double)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO + (double)g.N * g.heads * g.C * g.HO * g.WO) * sizeof(T));
    agg_dw_generic<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>(dy, x, dw, g, total);
    rc = check_launch("agg_dw_generic");
  }
  return rc;
}

}  // namespace cotb200

using namespace cotb200;

extern "C" int cotb200_agg_zeropad_fwd(const cotb200_agg_desc* d, const void* x, const void* w, void* y, void* stream) {
  Geo g;
  int rc = resolve(d, g);
  if (rc) return rc;
  if (!x || !w || !y) { set_error("agg_zeropad_fwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(d->dtype, return fwd_impl<T>(g, (const T*)x, (const T*)w, (T*)y, st));
  return 0;
}

extern "C" int cotb200_agg_zeropad_bwd(const cotb200_agg_desc* d, const void* dy, const void* x, const void* w, void* dx,
                                       void* dw, void* stream) {
  Geo g;
  int rc = resolve(d, g);
  if (rc) return rc;
  if (!dy || (dx && !w) || (dw && !x)) { set_error("agg_zeropad_bwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  COTB200_DISPATCH_DTYPE(d->dtype, return bwd_impl<T>(g, (const T*)dy, (const T*)x, (const T*)w, (T*)dx, (T*)dw, false, st));
  return 0;
}

// ---- mix: y = cat_c[ agg(x,w1;k1,p1), agg(x,w2;k2,p2) ]  (aggregation_zeropad_mix.py:20-74), NCHW only
static int resolve_mix(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w, Geo& g1, Geo& g2) {
  if (!d) { set_error("desc is NULL"); return COTB200_ENULL; }
  if (d->layout != COTB200_NCHW) { set_error("agg_zeropad_mix supports the NCHW layout only"); return COTB200_ELAYOUT; }
  int rc = resolve(d, g1);
  if (rc) return rc;
  cotb200_agg_desc d2 = *d;
  d2.kh = k2h; d2.kw = k2w; d2.ph = p2h; d2.pw = p2w;
  rc = resolve(&d2, g2);
  if (rc) return rc;
  // both halves live in one [n, 2*heads*c, ho, wo] tensor (aggregation_zeropad_mix.py:26-31,:220)
  g1.y_sn *= 2; g2.y_sn *= 2;
  return 0;
}

extern "C" int cotb200_agg_zeropad_mix_fwd(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w, const void* x,
                                           const void* w1, const void* w2, void* y, void* stream) {
  Geo g1, g2;
  int rc = resolve_mix(d, k2h, k2w, p2h, p2w, g1, g2);
  if (rc) return rc;
  if (!x || !w1 || !w2 || !y) { set_error("agg_zeropad_mix_fwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long half = (long long)g1.heads * g1.C * g1.HO * g1.WO;
  COTB200_DISPATCH_DTYPE(d->dtype, {
    if constexpr (!std::is_same<T, double>::value) {
      if (is_same3(g1, 3) && is_same3(g2, 5) && fits32(g2) && 2 * half * g1.N < (1LL << 31)) {
        const int total = g1.N * g1.wc * g1.H * g1.W;
        COTB200_PROF("agg_mix_fwd_nchw");
        agg_mix_fwd_nchw_fast<T><<<grid_stride_blocks(total, 256, 8), 256, 0, st>>>((const T*)x, (const T*)w1, (const T*)w2, (T*)y, g1.N,
                                                                                   g1.C, g1.H, g1.W, g1.wc, g1.rep, total);
        return check_launch("agg_mix_fwd_nchw_fast");
      }
    }
    rc = fwd_impl<T>(g1, (const T*)x, (const T*)w1, (T*)y, st);
    if (rc) return rc;
    return fwd_impl<T>(g2, (const T*)x, (const T*)w2, (T*)y + half, st);
  });
  return 0;
}

extern "C" int cotb200_agg_zeropad_mix_bwd(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w, const void* dy,
                                           const void* x, const void* w1, const void* w2, void* dx, void* dw1, void* dw2,
                                           void* stream) {
  Geo g1, g2;
  int rc = resolve_mix(d, k2h, k2w, p2h, p2w, g1, g2);
  if (rc) return rc;
  if (!dy || (dx && (!w1 || !w2)) || ((dw1 || dw2) && !x)) { set_error("agg_zeropad_mix_bwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long half = (long long)g1.heads * g1.C * g1.HO * g1.WO;
  COTB200_DISPATCH_DTYPE(d->dtype, {
    if (sizeof(T) >= 4 && is_same3(g1, 3) && is_same3(g2, 5) && fits32(g2)) {
      // fp32 / fp64 storage: the second kernel can accumulate into dX exactly, so both halves run on the register-resident
      // fused dX + dW kernels (the generic path below is kept for 16-bit storage, where dX must be summed before rounding)
      rc = bwd_impl<T>(g1, (const T*)dy, (const T*)x, (const T*)w1, (T*)dx, (T*)dw1, false, st);
      if (rc) return rc;
      return bwd_impl<T>(g2, (const T*)dy + half, (const T*)x, (const T*)w2, (T*)dx, (T*)dw2, dx != nullptr, st);
    }
    if (dx) {   // both halves of dX in one fp32-accumulating pass
      const long long total = (long long)g1.N * g1.C * g1.H * g1.W;
      COTB200_PROF("agg_mix_dx");
      agg_dx_generic2<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)w1, g1, (const T*)dy + half,
                                                                            (const T*)w2, g2, (T*)dx, total);
      rc = check_launch("agg_mix_dx");
      if (rc) return rc;
    }
    rc = bwd_impl<T>(g1, (const T*)dy, (const T*)x, (const T*)w1, (T*)nullptr, (T*)dw1, false, st);
    if (rc) return rc;
    return bwd_impl<T>(g2, (const T*)dy + half, (const T*)x, (const T*)w2, (T*)nullptr, (T*)dw2, false, st);
  });
  return 0;
}

// ---- mix_merge: the mix op with BOTH weight sets packed in one tensor w [n, heads*wc*(k1^2 + k2^2), ho, wo]
// (cupy_layers/aggregation_zeropad_mix_merge.py:20-179; the first heads*wc*k1^2 channels are w1 viewed [heads, wc, k1^2],
// the rest w2).  Same arithmetic as cotb200_agg_zeropad_mix_*; only the batch stride of the weights differs, so the
// stride-aware generic kernels run it on the packed tensor in place (no split / cat copies).
static void merge_strides(Geo& g1, Geo& g2, long long& off2) {
  const long long plane = (long long)g1.HO * g1.WO;
  const long long tot = (long long)g1.heads * g1.wc * (g1.K2 + g2.K2) * plane;
  off2 = (long long)g1.heads * g1.wc * g1.K2 * plane;
  g1.w_sn = tot; g2.w_sn = tot;
}

extern "C" int cotb200_agg_zeropad_mix_merge_fwd(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w, const void* x,
                                                 const void* w, void* y, void* stream) {
  Geo g1, g2;
  int rc = resolve_mix(d, k2h, k2w, p2h, p2w, g1, g2);
  if (rc) return rc;
  if (!x || !w || !y) { set_error("agg_zeropad_mix_merge_fwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  long long off2;
  merge_strides(g1, g2, off2);
  const long long half = (long long)g1.heads * g1.C * g1.HO * g1.WO;
  const long long total = (long long)g1.N * half;
  (void)total;
  COTB200_DISPATCH_DTYPE(d->dtype, {
    rc = fwd_impl<T>(g1, (const T*)x, (const T*)w, (T*)y, st);                  // register-resident kernels when 3x3 / 5x5 same-pad, heads 1
    if (rc) return rc;
    return fwd_impl<T>(g2, (const T*)x, (const T*)w + off2, (T*)y + half, st);
  });
  return 0;
}

extern "C" int cotb200_agg_zeropad_mix_merge_bwd(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w, const void* dy,
                                                 const void* x, const void* w, void* dx, void* dw, void* stream) {
  Geo g1, g2;
  int rc = resolve_mix(d, k2h, k2w, p2h, p2w, g1, g2);
  if (rc) return rc;
  if (!dy || (dx && !w) || (dw && !x)) { set_error("agg_zeropad_mix_merge_bwd: NULL tensor pointer"); return COTB200_ENULL; }
  cudaStream_t st = (cudaStream_t)stream;
  long long off2;
  merge_strides(g1, g2, off2);
  const long long half = (long long)g1.heads * g1.C * g1.HO * g1.WO;
  COTB200_DISPATCH_DTYPE(d->dtype, {
    if (sizeof(T) >= 4 && is_same3(g1, 3) && is_same3(g2, 5) && fits32(g2)) {
      rc = bwd_impl<T>(g1, (const T*)dy, (const T*)x, (const T*)w, (T*)dx, (T*)dw, false, st);
      if (rc) return rc;
      return bwd_impl<T>(g2, (const T*)dy + half, (const T*)x, (const T*)w + off2, (T*)dx, dw ? (T*)dw + off2 : (T*)nullptr, dx != nullptr, st);
    }
    if (dx) {
      const long long total = (long long)g1.N * g1.C * g1.H * g1.W;
      COTB200_PROF("agg_mix_merge_dx");
      agg_dx_generic2<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)w, g1, (const T*)dy + half,
                                                                            (const T*)w + off2, g2, (T*)dx, total);
      rc = check_launch("agg_mix_merge_dx");
      if (rc) return rc;
    }
    if (dw) {
      COTB200_PROF("agg_mix_merge_dw");
      const long long t1 = (long long)g1.N * g1.heads * g1.wc * g1.K2 * g1.HO * g1.WO;
      agg_dw_generic<T><<<grid_stride_blocks(t1, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)x, (T*)dw, g1, t1);
      rc = check_launch("agg_mix_merge_dw");
      if (rc) return rc;
      const long long t2 = (long long)g2.N * g2.heads * g2.wc * g2.K2 * g2.HO * g2.WO;
      agg_dw_generic<T><<<grid_stride_blocks(t2, 256, 16), 256, 0, st>>>((const T*)dy + half, (const T*)x, (T*)dw + off2, g2, t2);
      rc = check_launch("agg_mix_merge_dw");
    }
    return rc;
  });
  return 0;
}
