// Host interface between the LocalConv dispatch (agg_zeropad.cu) and the kernel files it calls.  Every launcher returns 1 when
// it took the call (status in *rc) and 0 when the geometry, layout or alignment is not for its kernel, so the dispatch tries
// the next one.
#pragma once
#include "common.cuh"

namespace cotb200 {

// an NHWC call: element strides per sample (_sn) and per pixel (_sp) of x, w and y
struct Nhwc2Args {
  int N, C, H, W, wc, fold, layout, gc, dtype;
  long long x_sn, x_sp, w_sn, w_sp, y_sn, y_sp;
};

// second-generation NHWC kernels (agg_nhwc2.cu)
template <typename T> int nhwc2_fwd(const Nhwc2Args& a, const T* x, const T* w, T* y, cudaStream_t st, int* rc);
template <typename T> int nhwc2_dx(const Nhwc2Args& a, const T* dy, const T* w, T* dx, cudaStream_t st, int* rc);
template <typename T> int nhwc2_dw(const Nhwc2Args& a, const T* dy, const T* x, T* dw, cudaStream_t st, int* rc);
// TMA-pipelined NHWC kernels (agg_tma.cu)
template <typename T> int agg_tma_fwd(const Nhwc2Args& a, const T* x, const T* w, T* y, cudaStream_t st, int* rc);
template <typename T> int agg_tma_dx(const Nhwc2Args& a, const T* dy, const T* w, T* dx, cudaStream_t st, int* rc);
template <typename T> int agg_tma_dw(const Nhwc2Args& a, const T* dy, const T* x, T* dw, cudaStream_t st, int* rc);
// TMA-pipelined NCHW kernels (agg_nchw_tma.cu): mode 0 fwd / 1 dX / 2 dW
template <typename T> int nchw_tma_launch(int mode, int N, int C, int H, int W, int wc, long long a_sn, long long b_sn, long long out_sn,
                                          const T* A, const T* Bp, T* out, cudaStream_t st, int* rc);
// small-plane NCHW backward kernels (agg_nchw_plane.cu): mode 1 dX / 2 dW / 3 dX + dW
template <typename T> int nchw_plane_launch(int mode, int N, int C, int H, int W, int wc, long long x_sn, long long y_sn, long long w_sn,
                                            const T* a, const T* b, const T* w, T* o1, T* o2, cudaStream_t st, int* rc);
// second-generation NCHW kernels (agg_nchw2.cu)
template <typename T> int nchw2_fwd(int N, int C, int H, int W, int wc, long long y_sn, const T* x, const T* w, T* y, cudaStream_t st,
                                    int* rc);
template <typename T> int nchw2_bwd(int N, int C, int H, int W, int wc, long long dy_sn, const T* dy, const T* x, const T* w, T* dx,
                                    T* dw, cudaStream_t st, int* rc);

}  // namespace cotb200
