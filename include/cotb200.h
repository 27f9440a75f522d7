/*
 * cotb200.h -- C ABI of libcotb200.so: the H100-native (sm_90a) kernels of the CoT-block hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  The reference has no C ABI: its "FFI" is CuPy --
 *   load_kernel(name, code, **literals) -> cupy.cuda.compile_with_cache(code).get_function(name)
 *                                                       (cupy_layers/utils.py:14-18)
 *   f(block=(1024,1,1), grid=(GET_BLOCKS(n),1,1), args=[ptr,...], stream=Stream(ptr=current_stream))
 *                                                       (cupy_layers/aggregation_zeropad.py:130-143)
 * with every dimension baked into the NVRTC source.  Each entry point below names the reference launch it
 * replaces; dimensions are runtime arguments (no per-shape JIT), pointers are raw device pointers, the
 * stream is a cudaStream_t passed as void*.  No torch types, no hidden synchronisation: every call is asynchronous on
 * the given stream and safe under CUDA-graph capture.
 *
 * Reductions over many CTAs (the statistics and backward sums below, the GEMM / convolution statistics epilogues, the split
 * weight gradients) are deterministic: partial sums are added in a fixed order, so the same inputs give bit-identical results
 * from run to run.  Those calls take their scratch stream-ordered: cudaMallocAsync + cudaMemsetAsync before the launch and
 * cudaFreeAsync after it, all on the given stream (from the device's default memory pool; inside a graph capture they become
 * the graph's own allocation, memset and free nodes).  Calls on different streams therefore never share scratch.
 *
 * Return value: 0 on success; >0 = cudaError_t from the launch; <0 = COTB200_E* argument error.
 * cotb200_last_error() returns a thread-local, human-readable description of the last failure.
 */
#ifndef COTB200_H_
#define COTB200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define COTB200_VERSION 100

/* element types (the reference supports only float/double: cupy_layers/utils.py:8-12) */
enum { COTB200_F32 = 0, COTB200_F64 = 1, COTB200_BF16 = 2, COTB200_F16 = 3 };

/* memory layouts of activations / weights
 *   NCHW  : x [N,C,H,W], w [N,heads,wc,kh*kw,Ho,Wo], y [N,heads*C,Ho,Wo]   -- the reference contract
 *           (cupy_layers/aggregation_zeropad.py:37-38)
 *   NHWC  : x [N,H,W,C], w [N,Ho,Wo,heads,wc,kh*kw], y [N,Ho,Wo,heads*C]   -- torch channels_last
 *   NHWC_TAP : as NHWC but weight channels are stored tap-major inside chunks of `gc` weight channels:
 *           index of (head, g, tap) = head*wc*K2 + ((g/gc)*K2 + tap)*gc + g%gc.  This is the layout the fused
 *           CoT block uses internally (the logits GEMM emits it for free by permuting its weight rows). */
enum { COTB200_NCHW = 0, COTB200_NHWC = 1, COTB200_NHWC_TAP = 2 };

enum {
  COTB200_EINVAL = -1,      /* inconsistent / unsupported dimensions */
  COTB200_EDTYPE = -2,      /* unknown dtype */
  COTB200_ELAYOUT = -3,     /* unknown layout */
  COTB200_EALIGN = -4,      /* pointer / stride alignment required by the selected kernel not met */
  COTB200_ENULL = -5,       /* required pointer is NULL */
  COTB200_ETOOBIG = -6,     /* tensor exceeds the 2^31-element index range of the fast kernels */
  COTB200_EUNSUPPORTED = -7 /* a fused fast path cannot take this geometry: the caller uses the separate kernels */
};

/* Geometry of one LocalConv call.  Mirrors the literals substituted into the reference kernels
 * (cupy_layers/aggregation_zeropad.py:131-139). */
typedef struct cotb200_agg_desc {
  int n, c, h, w;            /* input  [n, c, h, w] */
  int heads, wc;             /* weight heads, weight channels; c % wc == 0; input channel ch uses weight channel ch % wc */
  int kh, kw;                /* kernel size */
  int sh, sw, ph, pw, dh, dw;/* stride, zero padding, dilation */
  int ho, wo;                /* output spatial size = weight spatial size */
  int dtype;                 /* COTB200_F32 ... */
  int layout;                /* COTB200_NCHW / NHWC / NHWC_TAP */
  int gc;                    /* NHWC_TAP only: weight-channel chunk width (divides wc); ignored otherwise */
  int fold;                  /* CoXt channel fold (models/cotnet.py:157-162): 0/1 = none; F>1: channel c uses weight
                              * channel (c/(C/F))*(wc/F) + (c%(C/F))%(wc/F), i.e. the F channel groups own disjoint
                              * wc/F-wide weight ranges -- the un-folded form of the reference's view(B*F, ...) trick */
  /* NHWC layouts only: element strides of the batch and pixel dimensions (channel stride is 1).
   * 0 selects the dense default.  They let the CoXt "fold the two channel halves into the batch"
   * view (models/cotnet.py:157-162) run without a copy. */
  long long x_sn, x_sp;
  long long w_sn, w_sp;
  long long y_sn, y_sp;
} cotb200_agg_desc;

int cotb200_version(void);
const char* cotb200_last_error(void);
/* number of kernels launched by this library in this process (the bench's gpu_launches counter) */
long long cotb200_launch_count(void);

/* Per-kernel device timing for the bench's roofline line: when enabled every launch of this library is
 * bracketed by CUDA events on its stream; cotb200_prof_report writes "<kernel> <launches> <total_ms> <algorithmic bytes>" lines
 * (returns the length needed).  Off by default; do not enable during CUDA-graph capture. */
void cotb200_prof_enable(int on);
int cotb200_prof_report(char* buf, int len);

/* Replaces aggregation_zeropad_forward_kernel (cupy_layers/aggregation_zeropad.py:20-46, launch :130-143).
 * y[n, head*C + c, ho, wo] = sum_{kh,kw} w[n, head, c % wc, kh*KW+kw, ho, wo] * x[n, c, ho*s-p+kh*d, wo*s-p+kw*d] */
int cotb200_agg_zeropad_fwd(const cotb200_agg_desc* d, const void* x, const void* w, void* y, void* stream);

/* Replaces aggregation_zeropad_input_backward_kernel (:48-79) and ..._weight_backward_kernel (:81-110),
 * launches :168-185.  dx and/or dw may be NULL (ctx.needs_input_grad, :168,:177); when both are wanted
 * and the fast path applies they are produced by ONE fused kernel that reads dy once. */
int cotb200_agg_zeropad_bwd(const cotb200_agg_desc* d, const void* dy, const void* x, const void* w,
                            void* dx, void* dw, void* stream);

/* Replaces aggregation_zeropad_mix_forward_kernel (cupy_layers/aggregation_zeropad_mix.py:20-74).
 * d describes the FIRST kernel (kh,kw,ph,pw = kernel_size1/padding1); the second kernel is (k2h,k2w,p2h,p2w).
 * y = cat_channels[ agg(x, w1; k1,p1), agg(x, w2; k2,p2) ]  -> [n, 2*heads*c, ho, wo].  NCHW layout only. */
int cotb200_agg_zeropad_mix_fwd(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w,
                                const void* x, const void* w1, const void* w2, void* y, void* stream);

/* Replaces aggregation_zeropad_mix_{input,weight}_backward_kernel (aggregation_zeropad_mix.py:76-207).
 * dx, or dw1 and dw2 together, may be NULL. */
int cotb200_agg_zeropad_mix_bwd(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w,
                                const void* dy, const void* x, const void* w1, const void* w2,
                                void* dx, void* dw1, void* dw2, void* stream);

/* ---- the remaining LocalConv variants of cupy_layers (SURVEY.md section 8f rank 4); NCHW (reference contract), any dtype ----
 * Reflect padding instead of zero padding (cupy_layers/aggregation_refpad.py:21-127; launches :153-160,:183-207).
 * Padding must be smaller than the input (one reflection), like nn.ReflectionPad2d.  dX is gathered directly on the
 * un-padded grid (the reference computes it on the padded grid and folds the borders with torch ops, :188-199). */
int cotb200_agg_refpad_fwd(const cotb200_agg_desc* d, const void* x, const void* w, void* y, void* stream);
int cotb200_agg_refpad_bwd(const cotb200_agg_desc* d, const void* dy, const void* x, const void* w,
                           void* dx, void* dw, void* stream);
/* Per-weight-channel dilation (cupy_layers/aggregation_zeropad_dilate.py:20-146): 3x3, stride 1, output size = input size,
 * weight channel g uses dilation = padding = (int)dilation[g]; `dilation` is a device array of wc elements of the SAME
 * dtype as x (the reference passes a tensor of the input dtype, :23,:33).  d->kh = d->kw = 3; d->{s,p,d}* are ignored. */
int cotb200_agg_zeropad_dilate_fwd(const cotb200_agg_desc* d, const void* x, const void* w, const void* dilation,
                                   void* y, void* stream);
int cotb200_agg_zeropad_dilate_bwd(const cotb200_agg_desc* d, const void* dy, const void* x, const void* w,
                                   const void* dilation, void* dx, void* dw, void* stream);
/* The mix op with both weight sets packed in ONE tensor w [n, heads*wc*(k1^2+k2^2), ho, wo]
 * (cupy_layers/aggregation_zeropad_mix_merge.py:20-179): first heads*wc*k1^2 channels = w1 [heads, wc, k1^2], then w2.
 * dw has the same packed layout.  Runs on the packed tensor in place (no split / cat). */
int cotb200_agg_zeropad_mix_merge_fwd(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w,
                                      const void* x, const void* w, void* y, void* stream);
int cotb200_agg_zeropad_mix_merge_bwd(const cotb200_agg_desc* d, int k2h, int k2w, int p2h, int p2w,
                                      const void* dy, const void* x, const void* w, void* dx, void* dw, void* stream);

/* ---- fused normalisation / split-attention kernels on NHWC tensors [B, HW, C] (channel contiguous), fp32 math ----
 * They replace chains of eager launches of the reference block (models/cotnet.py:56 and :89-104).
 * dtype: COTB200_F32 / BF16 / F16.  All float* arguments are fp32 device arrays; sums are ACCUMULATED (+=), in a fixed
 * order (see the top of this file), so the caller zeroes them. */

/* sum[c] += sum_rows x, sq[c] += sum_rows x^2 : BatchNorm batch statistics (nn.BatchNorm2d training mode, :65,:89) */
int cotb200_col_stats(int dtype, int B, int HW, int C, const void* x, float* sum, float* sq, void* stream);
/* psum[b,c] += sum_rows( silu(u*scale+shift) + k ) : bn + SiLU (:89-90) and the pooled descriptor of :92-98.
 * In all tail kernels k (and dk) may be NULL: then they compute the SplitAttnConv2d (radix 1) chain of the SE-CoTNetD
 * blocks -- bn0 -> SiLU -> global pool ... x * sigmoid(attn) (models/layers/split_attn.py:68-86) -- with a[b,c,0] the gate. */
int cotb200_tail_pool(int dtype, int B, int HW, int C, const void* u, const void* k, const float* scale,
                      const float* shift, float* psum, void* stream);
/* out = a[b,c,0]*silu(u*scale+shift) + a[b,c,1]*k : the radix-2 recombination (:101-104); a is [B,C,2] fp32 */
int cotb200_tail_combine(int dtype, int B, int HW, int C, const void* u, const void* k, const float* scale,
                         const float* shift, const float* a, void* out, void* stream);
/* S[b,c,0] += sum_rows dout*y, S[b,c,1] += sum_rows dout*k : gradient of the attention weights */
int cotb200_tail_bwd_sums(int dtype, int B, int HW, int C, const void* dout, const void* u, const void* k,
                          const float* scale, const float* shift, float* S, void* stream);
/* dz = (a0*dout + dpn)*silu'(z); sum_dz[c] += sum dz, sum_dzx[c] += sum dz*xhat (BatchNorm backward reductions) */
int cotb200_tail_bwd_dz_sums(int dtype, int B, int HW, int C, const void* dout, const void* u, const float* scale,
                             const float* shift, const float* mu, const float* rstd, const float* a, const float* dpn,
                             float pscale, float* sum_dz, float* sum_dzx, void* stream);
/* du = scale*(dz - c1*inv_n - xhat*c2*inv_n) (c1,c2 = the raw sums above, NULL in eval mode), dk = a1*dout + dpn*pscale.
 * dpn is the gradient w.r.t. the pooled descriptor [B,C]; pscale = 1/HW turns it into the per-pixel term. */
int cotb200_tail_bwd_apply(int dtype, int B, int HW, int C, const void* dout, const void* u, const float* scale,
                           const float* shift, const float* mu, const float* rstd, const float* a, const float* dpn,
                           const float* c1, const float* c2, float inv_n, float pscale, void* du, void* dk, void* stream);
/* The SE MLP of the split attention in EVAL mode (models/cotnet.py:69-77,92-101), two tiled launches (fc1, fc2 + softmax):
 *   a[b,c,0:2] = softmax_r( W3[2c+r,:] . relu(s1*(W0 . (psum[b]*inv_hw) + b0) + t1) + b3[2c+r] )
 * with the BatchNorm of `se` folded into s1 / t1.  psum [B,C] is what cotb200_tail_pool accumulates; a [B,C,2] is what
 * cotb200_tail_combine takes.  All fp32; W0 [A,C], W3 [2C,A] row-major; b0 / b3 may be NULL; z_scratch: B*A floats
 * (cotb200_se_eval_scratch_bytes) for the hidden activations between the two launches. */
long long cotb200_se_eval_scratch_bytes(int B, int A);
int cotb200_se_eval(int B, int C, int A, const float* psum, float inv_hw, const float* W0, const float* b0,
                    const float* s1, const float* t1, const float* W3, const float* b3, float* a, float* z_scratch,
                    void* stream);
/* BatchNorm2d (+ReLU) (+residual add) on NHWC tensors: y = act(x*scale + shift (+ res)).  With cotb200_col_stats this
 * replaces nn.BatchNorm2d / nn.ReLU pairs of the block (models/cotnet.py:45-46,53-54,61-62) and of the enclosing
 * bottleneck (models/cotnet.py:231-235,:249-262) in 2 forward + 2 backward HBM passes.  relu: 0/1; res may be NULL. */
int cotb200_bn_apply(int dtype, int B, int HW, int C, const void* x, const void* res, const float* scale,
                     const float* shift, int relu, void* y, void* stream);
/* Training-mode variant: the bookkeeping of cotb200_bn_finalize folded into the apply kernel's prologue (one launch less per
 * BatchNorm): scale/shift are derived from the batch sums of cotb200_col_stats (n rows), scale/shift/mean/rstd [C] are
 * written for the backward, the running statistics updated when update_running (momentum, unbiased variance). */
int cotb200_bn_apply_batch(int dtype, int B, int HW, int C, const void* x, const void* res, const float* sum, const float* sq,
                           const float* weight, const float* bias, float* running_mean, float* running_var, float n,
                           float eps, float momentum, int update_running, int relu, void* y, float* scale, float* shift,
                           float* mean, float* rstd, void* stream);
/* dz = dy*mask ; sum_dz[c] += sum dz ; sum_dzx[c] += sum dz*xhat.
 * relu: 0 = no activation; 1 = ReLU, mask = [y > 0] read from the forward output y; 2 = ReLU, mask recomputed as
 * [x*scale + shift > 0] from the forward's own fp32 scale/shift (identical mask, y is NOT read: one HBM pass less; only for
 * BatchNorms without a residual input).  y may be NULL unless relu == 1; scale/shift may be NULL unless relu == 2. */
int cotb200_bn_bwd_sums(int dtype, int B, int HW, int C, const void* dy, const void* x, const void* y, const float* scale,
                        const float* shift, const float* mu, const float* rstd, int relu, float* sum_dz, float* sum_dzx,
                        void* stream);
/* Two-consumer form: the BatchNorm output fed TWO consumers (the next block's conv1 and its shortcut, models/cotnet.py:228-262) and
 * autograd would first add their gradients (one more kernel, three HBM passes); here dy := dy + dy2 is formed in fp32 inside the
 * backward kernels (dy2 may be NULL = the one-gradient form). */
int cotb200_bn_bwd_sums2(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                         const float* scale, const float* shift, const float* mu, const float* rstd, int relu, float* sum_dz,
                         float* sum_dzx, void* stream);
int cotb200_bn_bwd_apply2(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                          const float* scale, const float* shift, const float* mu, const float* rstd, const float* c1,
                          const float* c2, float inv_n, int relu, void* dx, void* dres, void* stream);
/* dx = scale*(dz - c1*inv_n - xhat*c2*inv_n) (c1,c2 = the raw sums of cotb200_bn_bwd_sums, NULL in eval mode) ;
 * dres = dz when dres != NULL (gradient of the residual) */
int cotb200_bn_bwd_apply(int dtype, int B, int HW, int C, const void* dy, const void* x, const void* y, const float* scale,
                         const float* shift, const float* mu, const float* rstd, const float* c1, const float* c2,
                         float inv_n, int relu, void* dx, void* dres, void* stream);
/* Stochastic depth (DropPath after bn3, models/cotnet.py:256-257) inside the same kernels.  sample_scale: device fp32 [B] = s_b,
 * 0 for a dropped sample and 1/keep for a kept one (NULL = all 1: then each call is its plain form above, bit for bit).
 *   forward:  y = act(s_b*(x*scale + shift) (+ res))
 *   backward: g = dy*mask (dy := dy + dy2 when dy2 != NULL); dres = g; the BatchNorm output gradient is s_b*g, so
 *             sum_dz += sum s_b*g, sum_dzx += sum s_b*g*xhat and dx = scale*(s_b*g - c1*inv_n - xhat*c2*inv_n).
 * The batch statistics (cotb200_col_stats, the GEMM epilogue) still cover every sample, dropped or not. */
int cotb200_bn_apply_ds(int dtype, int B, int HW, int C, const void* x, const void* res, const float* scale,
                        const float* shift, int relu, void* y, const float* sample_scale, void* stream);
int cotb200_bn_apply_batch_ds(int dtype, int B, int HW, int C, const void* x, const void* res, const float* sum, const float* sq,
                              const float* weight, const float* bias, float* running_mean, float* running_var, float n,
                              float eps, float momentum, int update_running, int relu, void* y, float* scale, float* shift,
                              float* mean, float* rstd, const float* sample_scale, void* stream);
int cotb200_bn_bwd_sums_ds(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                           const float* scale, const float* shift, const float* mu, const float* rstd, int relu, float* sum_dz,
                           float* sum_dzx, const float* sample_scale, void* stream);
int cotb200_bn_bwd_apply_ds(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x, const void* y,
                            const float* scale, const float* shift, const float* mu, const float* rstd, const float* c1,
                            const float* c2, float inv_n, int relu, void* dx, void* dres, const float* sample_scale,
                            void* stream);
/* 1-bit ReLU mask for BatchNorms with a residual input (relu code 3).  With a residual the mask cannot be recomputed from x
 * (code 2), and reading y back costs two full passes of the widest tensors of the bottleneck.  The training-mode apply writes,
 * next to y, mask [B*HW, C/8] bytes: bit c%8 of byte c/8 of a row = [y > 0] of the STORED y (so the mask equals relu code 1's
 * bit for bit); the backward kernels read the mask instead of y (C/8 bytes per row instead of C elements).  Needs C % 8 == 0.
 * Otherwise these are cotb200_bn_apply_batch_ds (relu = 1, res required), cotb200_bn_bwd_sums_ds and cotb200_bn_bwd_apply_ds:
 * dy2 and sample_scale may be NULL. */
int cotb200_bn_apply_batch_mask(int dtype, int B, int HW, int C, const void* x, const void* res, const float* sum, const float* sq,
                                const float* weight, const float* bias, float* running_mean, float* running_var, float n,
                                float eps, float momentum, int update_running, void* y, float* scale, float* shift,
                                float* mean, float* rstd, const float* sample_scale, unsigned char* mask, void* stream);
int cotb200_bn_bwd_sums_mask(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x,
                             const unsigned char* mask, const float* mu, const float* rstd, float* sum_dz, float* sum_dzx,
                             const float* sample_scale, void* stream);
int cotb200_bn_bwd_apply_mask(int dtype, int B, int HW, int C, const void* dy, const void* dy2, const void* x,
                              const unsigned char* mask, const float* scale, const float* mu, const float* rstd, const float* c1,
                              const float* c2, float inv_n, void* dx, void* dres, const float* sample_scale, void* stream);
/* One launch for the BatchNorm bookkeeping: from the column sums of cotb200_col_stats (or a GEMM epilogue) compute
 * scale = gamma*rstd, shift = beta - mean*scale, mean, rstd, and update running_mean / running_var like nn.BatchNorm2d
 * (momentum, unbiased variance).  use_batch = 0: eval mode, statistics read from the running buffers. */
int cotb200_bn_finalize(int C, const float* sum, const float* sq, const float* weight, const float* bias,
                        float* running_mean, float* running_var, float n, float eps, float momentum, int use_batch,
                        int update_running, float* scale, float* shift, float* mean, float* rstd, void* stream);

/* GroupNorm(num_groups = wc, channels = 9*wc) of the attention logits (models/cotnet.py:56): group g = the 9 taps of
 * weight channel g.  The logits l / dl are always in the reference channel order j = g*9 + t; `gc` is the storage order
 * of the normalised weights (and of their gradient dg): 0 = same order, > 0 = tap-major chunks (COTB200_NHWC_TAP), so
 * the permutation the LocalConv kernels want costs nothing extra.  (cotb200_gn9_stats ignores gc.)
 * lbias (NULL or [9*wc] fp32, reference order): the bias of the embed.3 convolution (models/cotnet.py:55) added to l on
 * load, so the convolution can run bias-free; cotb200_gn9_bwd_sums then also returns its gradient
 * dlbias[j] += sum_{b,px} dl (NULL = not wanted), derived analytically from the column sums -- no extra pass over dl.
 * cotb200_gn9_bwd_sums: work = [B, 3, 9*wc] fp32 zeros (per-sample column partials); s1, s2 [B, wc] are written;
 * dgamma, dbeta (and dlbias) [9*wc] are accumulated into (zero them first).
 * Fast path ("blocks of 72", csrc/gn72.cu): wc in {8,16,32,64}, gc == 8, 16-byte aligned tensors -- tiles moved by
 * cp.async.bulk, the tap permutation done in registers.  Everything else runs the generic kernels. */
int cotb200_gn9_stats(int dtype, int B, int HW, int wc, int gc, const void* l, const float* lbias, float* gsum, float* gsq,
                      void* stream);
int cotb200_gn9_apply(int dtype, int B, int HW, int wc, int gc, const void* l, const float* lbias, const float* mean,
                      const float* rstd, const float* gamma, const float* beta, void* out, void* stream);
int cotb200_gn9_bwd_sums(int dtype, int B, int HW, int wc, int gc, const void* dg, const void* l, const float* lbias,
                         const float* mean, const float* rstd, const float* gamma, float* work, float* s1, float* s2,
                         float* dgamma, float* dbeta, float* dlbias, void* stream);
int cotb200_gn9_bwd_apply(int dtype, int B, int HW, int wc, int gc, const void* dg, const void* l, const float* lbias,
                          const float* mean, const float* rstd, const float* gamma, const float* s1, const float* s2,
                          void* dl, void* stream);

/* out[r, 0:C] = sum_i src_i[r, 0:C] over up to four row-pitched sources (ld_i elements; src2/src3 may be NULL).
 * Gradient accumulation of a tensor with several consumers inside the block -- x feeds key_embed, the concat and
 * conv1x1 (models/cotnet.py:80-84), k feeds the concat and the recombination (:81,:97) -- in ONE pass, including the
 * channel-sliced (pitch 2C) gradients of the concat, instead of autograd's chain of pairwise strided adds. */
int cotb200_sum_rows(int dtype, long long rows, int C, const void* src0, long long ld0, const void* src1, long long ld1,
                     const void* src2, long long ld2, const void* src3, long long ld3, void* out, long long ldo,
                     void* stream);

/* 3x3 / stride 2 / pad 1 pooling on NHWC tensors x [N,H,W,C] -> y [N,Ho,Wo,C], Ho = (H-1)/2+1.
 * mode 0: average with count_include_pad (nn.AvgPool2d(3, 2, padding=1), the `avd` of models/cotnet.py:199-202,237-238);
 * mode 1: max (nn.MaxPool2d(3, 2, 1) of the trunk, models/resnet.py:555); idx [N,Ho,Wo,C] uint8 = winning tap, consumed
 * by the backward (first maximum in scan order, like ATen).  Backward is a gather: no atomics. */
int cotb200_pool3s2_fwd(int dtype, int mode, int N, int H, int W, int C, const void* x, void* y, void* idx, void* stream);
int cotb200_pool3s2_bwd(int dtype, int mode, int N, int H, int W, int C, const void* dy, const void* idx, void* dx,
                        void* stream);

/* ---- dense contractions of the block on the Hopper tensor cores (wgmma, register accumulators, TMA operands) ----
 * bf16 operands, fp32 accumulation, bf16 output.  Row-major everywhere; "ld*" are row pitches in elements.
 *
 * cotb200_gemm_bf16:  D[M,N] = epi( A1[M,K1] B1[N,K1]^T + A2[M,K2] B2[N,K2]^T )      (K2 == 0: single product)
 *   Replaces the 1x1 nn.Conv2d launches of the block (cuDNN in the reference): embed.0 on cat[x,k] without the
 *   concat (models/cotnet.py:52,81), embed.3 (:55), conv1x1.0 (:60) -- rows are NHWC pixels.
 *   epi(acc)[m,n] = relu?( acc*scale[n] + shift[n] )  (scale/shift NULL = 1/0: folded eval-mode BatchNorm or bias);
 *   col_sum/col_sqsum (both or neither): += sum_m D[m,n], sum_m D[m,n]^2 of the STORED bf16 output (with scale/shift NULL
 *   and relu 0 that is the raw product: the training-mode BatchNorm batch statistics of the convolution output,
 *   models/cotnet.py:45,53,61 -- taken from the staged output tile, exactly the values the normalisation reads back).
 *   Requirements: N, K1, K2, ldd multiples of 8; operands 16-byte aligned. */
int cotb200_gemm_bf16(int M, int N, int K1, const void* A1, long long lda1, const void* B1, long long ldb1,
                      int K2, const void* A2, long long lda2, const void* B2, long long ldb2,
                      void* D, long long ldd, const float* scale, const float* shift, int relu,
                      float* col_sum, float* col_sqsum, void* stream);

/* cotb200_conv3x3_bf16: 3x3 / stride 1 / zero-pad 1 grouped convolution on an NHWC bf16 tensor X[B,H,W,C] (pixel pitch
 *   ldx) as an im2col-free implicit GEMM; replaces key_embed.0 = nn.Conv2d(dim, dim, 3, padding=1, groups=4)
 *   (models/cotnet.py:44) and, with transposed/flipped weights, its data gradient.
 *   Wp [C, 9*bn] is the weight prepared per N tile of bn output channels (bn in {64,128,192,256}, bn | C, every
 *   group inside one tile): Wp[n, (tap*(bn/64) + cc)*64 + ci] multiplies input channel (n/bn)*bn + cc*64 + ci at tap
 *   (tap = 3*kh + kw), zero for channels outside n's group.  Same epilogue as cotb200_gemm_bf16. */
int cotb200_conv3x3_bf16(int B, int H, int W, int C, const void* X, long long ldx, const void* Wp, int bn,
                         void* D, long long ldd, const float* scale, const float* shift, int relu,
                         float* col_sum, float* col_sqsum, void* stream);

/* cotb200_stem7x7s2_bf16: the stem convolution conv1 = nn.Conv2d(3, N, 7, stride=2, padding=3, bias=False)
 *   (models/resnet.py:552, called at :601; cuDNN in the reference) on an NHWC bf16 image X[B,H,W,3] (dense, H and W even) as a
 *   4-tap implicit wgmma GEMM: a space-to-depth copy of the image (scratch, cotb200_stem7x7s2_scratch_bytes bytes, 16-byte
 *   aligned) turns the 7x7/s2 window into 4 rows x 4 cells x 16 channels, and one TMA box per row fetches the overlapping
 *   windows of a whole output-row segment as the K-major A tile (K = 4 x 64).  D[B*(H/2)*(W/2), N] bf16 (row pitch ldd).
 *   Wm [N, 256] bf16: Wm[n, a*64 + a2*16 + (di*2+dj)*3 + c] = weight[n, c, 2a+di-1, 2a2+dj-1] (0 where an index is -1 and
 *   for the 4 pad channels).  Same epilogue as cotb200_gemm_bf16 (scale/shift/ReLU, optional BatchNorm column statistics).
 *   Returns COTB200_EUNSUPPORTED when the geometry / driver cannot take it (the caller then keeps its cuDNN convolution). */
long long cotb200_stem7x7s2_scratch_bytes(int B, int H, int W);
int cotb200_stem7x7s2_bf16(int B, int H, int W, const void* X, const void* Wm, int N, void* D, long long ldd,
                           const float* scale, const float* shift, int relu, float* col_sum, float* col_sqsum,
                           void* scratch, void* stream);

/* cotb200_stem7x7s2_wgrad_bf16: weight gradient of that convolution in the packed layout of Wm (cuDNN wgrad in the reference's
 *   autograd graph):  dWm[n, a*64 + j] += sum_px dY[px, n] * window_a(px)[j], fp32 [N, 256], ZEROED by the caller.  dY [B*(H/2)*(W/2), N]
 *   bf16 (row pitch ldy); scratch = the space-to-depth image cotb200_stem7x7s2_bf16 filled for the same X.  One pipeline stage of
 *   the MN-major wgmma wgrad kernel = one output row (W/2 pixels, a multiple of 16, <= 128).  COTB200_EUNSUPPORTED otherwise. */
int cotb200_stem7x7s2_wgrad_bf16(int B, int H, int W, const void* dY, long long ldy, int N, const void* scratch, float* dWm,
                                 void* stream);

/* cotb200_wgrad_bf16: weight gradient of a 1x1 convolution,  OUT += A[M,R]^T [B1[M,C1] | B2[M,C2]]  (contraction over the M
 *   pixels; A = dY, B = the convolution input(s); bf16 operands, fp32 accumulation, fp32 OUT).  Replaces cuDNN's wgrad
 *   for embed.0 / embed.3 / conv1x1.0 (models/cotnet.py:52,55,60) and the bottleneck's 1x1 convolutions (:228-264).
 *   Both operands are consumed MN-major straight from their NHWC tiles (no transposes).  Split over pixel ranges across the
 *   SMs; the partial tiles are added to OUT in split order by a second kernel, so the caller ZEROES OUT first.
 *   transpose = 0: OUT[r*ldo + c] (r < R, c < C1+C2); transpose = 1: OUT[c*ldo + r].
 *   Requirements: R, C1, C2 multiples of 8 (C1 a multiple of 64 when C2 > 0); operands 16-byte aligned. */
int cotb200_wgrad_bf16(int M, int R, const void* A, long long lda, int C1, const void* B1, long long ldb1,
                       int C2, const void* B2, long long ldb2, float* out, long long ldo, int transpose, void* stream);

/* ---- train-step plumbing (SURVEY.md section 8f rank 3): what the reference does per parameter tensor -- DDP bucket copy,
 * optim.SGD(nesterov=True) (optim/optim_factory.py:54-56), ModelEmaV2.update over the state_dict (utils/model_ema.py:45-53),
 * one AMP weight cast per convolution -- as ONE pass over flat buffers; and the loader's uint8 normalisation
 * (datasets/loader.py:86-90) as one kernel.  Tables (cotb200_seg*) live in DEVICE memory and are built by the caller. */
typedef struct cotb200_seg {          /* one source tensor of a gather */
  const void* ptr;                    /* device pointer of the tensor (dense, `numel` elements in memory order) */
  long long offset;                   /* first element of its slot in the flat bucket */
  long long numel;
  int dtype;                          /* COTB200_F32 / BF16 / F16 */
  int pad_;
} cotb200_seg;
typedef struct cotb200_seg2 {         /* one (destination, source) pair of a multi-tensor lerp */
  void* dst;
  const void* src;
  long long numel;
  int dtype;                          /* COTB200_F32, or 100 = int64 */
  int pad_;
} cotb200_seg2;
/* Elements per gather block: the caller cuts every source into ceil(numel / chunk) blocks and passes the block table
 * blocks[2*i] = segment index, blocks[2*i+1] = chunk index inside the segment. */
int cotb200_gather_chunk(void);
/* dst[seg.offset + i] = (dst type)(src_seg[i] * scale) for every segment: the gradients of a step (any mix of fp32 / bf16
 * tensors) into ONE flat fp32 or bf16 bucket = the unit of the NCCL all-reduce (replaces DDP's bucket copies, train.py:113-115). */
int cotb200_multi_gather(const cotb200_seg* segs_dev, const int* blocks_dev, int n_blocks, int dst_dtype, void* dst,
                         float scale, void* stream);
/* Over a flat range of n (multiple of 4) elements: torch.optim.SGD update with momentum (nesterov flag), weight decay,
 * then EMA  E = decay*E + (1-decay)*P  (E NULL: none) and the bf16 copy Pb of the new weights (NULL: none).
 * G is fp32 or bf16 (g_dtype).  hyper_dev = device fp32[5] {lr, momentum, weight_decay, ema_decay, grad_scale}: device
 * resident so that a captured CUDA graph follows the learning-rate schedule. */
int cotb200_sgd_ema_step(long long n, float* P, float* M, int g_dtype, const void* G, float* E, void* Pb,
                         const float* hyper_dev, int nesterov, void* stream);
/* dst = decay*dst + (1-decay)*src per segment (fp32; int64 with the reference's float round trip): ModelEmaV2 over the
 * BUFFERS of the state_dict (BatchNorm running statistics / counters), one launch. decay = hyper_dev[3]. */
int cotb200_multi_lerp(const cotb200_seg2* segs_dev, int n_segs, const float* hyper_dev, void* stream);

/* ---- gradient clipping on the flat buckets (train.py:270-273 -> utils/clip_grad.py:dispatch_clip_grad) ----
 * g' = G[i] * grad_scale is the averaged gradient the optimizer reads; the clip acts on g' in fp32 inside the optimizer pass
 * and never writes the bucket.  Modes (torch semantics, NaN propagated as torch.clamp does):
 *   NORM  (clip_grad_norm_, norm 2):  g' * f,  f = min(1, c / (N + 1e-6)),  N = ||g'|| over every element of both buckets
 *   VALUE (clip_grad_value_):          clamp(g', -c, c)
 *   AGC   (adaptive_clip_grad):        per unit u (a row along dim 0 of a >=2-D parameter, or a whole 1-D parameter):
 *                                      m = max(||P_u||, 1e-3) * c,  n = ||g'_u||;  g'_u unchanged if n < m, else
 *                                      g'_u * (m / max(n, 1e-6)).  P_u: the fp32 master weights before the update. */
enum { COTB200_CLIP_NORM = 1, COTB200_CLIP_VALUE = 2, COTB200_CLIP_AGC = 3 };
typedef struct cotb200_clip_unit {    /* AGC: one unit, `numel` consecutive elements of flat range `range` (0 or 1) */
  long long offset;
  int numel;
  int range;
} cotb200_clip_unit;
typedef struct cotb200_clip_seg {     /* AGC: one piece of the optimizer's flat range, handled by one warp */
  long long offset;
  int numel;                          /* 1 .. cotb200_clip_seg_max() */
  int unit;                           /* index into the factors; -1: factor 1 (slot padding, parameters left out) */
} cotb200_clip_seg;
typedef struct cotb200_clip {         /* the clip of one cotb200_sgd_ema_step_clip call */
  int mode;                           /* COTB200_CLIP_* */
  float value;                        /* VALUE: c (> 0) */
  const float* factor;                /* NORM: device pointer to f (out[1] of cotb200_grad_norm); AGC: device per-unit factors */
  const cotb200_clip_seg* segs;       /* AGC: device table of segments tiling [0, n) in order */
  int n_segs;
  int pad_;
} cotb200_clip;
/* Largest cotb200_clip_seg.numel: the caller cuts longer pieces. */
int cotb200_clip_seg_max(void);
/* out[0] = N = sqrt(sum over both ranges of (G*gs)^2), out[1] = f = min(1, max_norm / (N + 1e-6)) (fp32, device).  Range 0:
 * n0 elements of fp32 or bf16 (g0_dtype), range 1: n1 fp32 elements (n1 = 0: none); each scaled by its device scalar gs0 / gs1.
 * n0, n1 multiples of 4.  Deterministic: the partial sums are added in a fixed order. */
int cotb200_grad_norm(long long n0, int g0_dtype, const void* G0, const float* gs0, long long n1, const float* G1, const float* gs1,
                      float max_norm, float* out, void* stream);
/* AGC factors: factor[u] = 1 when ||g'_u|| < m_u, else m_u / max(||g'_u||, 1e-6), for every unit of the device table (one warp
 * per unit, a fixed summation order).  Range 0 = (P0, G0 of g0_dtype, gs0), range 1 = (P1, G1 fp32, gs1; all NULL if no unit
 * lies there).  norms: NULL, or device fp32 [n_units][2] receiving (||P_u||, ||g'_u||).  unit_elems = the sum of the units'
 * numel (the launch's algorithmic bytes). */
int cotb200_unit_norms(int n_units, const cotb200_clip_unit* units_dev, long long unit_elems, const float* P0, int g0_dtype,
                       const void* G0, const float* gs0, const float* P1, const float* G1, const float* gs1, float clip_factor,
                       float* factor, float* norms, void* stream);
/* cotb200_sgd_ema_step with the clip applied to g' = G*grad_scale on the way in: the update reads the clipped g' in place of
 * G*grad_scale.  A factor of 1 or a clamp that does not bind gives bit-for-bit the result of cotb200_sgd_ema_step. */
int cotb200_sgd_ema_step_clip(long long n, float* P, float* M, int g_dtype, const void* G, float* E, void* Pb,
                              const float* hyper_dev, int nesterov, const cotb200_clip* clip, void* stream);

/* ---- the update rules of create_optimizer (optim/optim_factory.py) on the flat buckets ----
 * One pass per flat range: g' = G*grad_scale, the clip (cotb200_clip, NULL: none), the rule, the Lookahead synchronisation when
 * this step has one, E = decay*E + (1-decay)*P of the final weights, and the bf16 copy Pb.  hyper_dev is the fp32[5] of
 * cotb200_sgd_ema_step ({lr, momentum, weight_decay, ema_decay, grad_scale}); betas, rho and alpha are the factory's defaults:
 *   SGD / MOMENTUM  torch.optim.SGD, nesterov / not                     M = momentum_buffer
 *   ADAM            torch.optim.Adam (L2 decay), betas (0.9, 0.999)     M = exp_avg, V = exp_avg_sq
 *   ADAMW           optim/adamw.py: P *= 1 - lr*wd, then Adam           M, V as ADAM
 *   NADAM           optim/nadam.py (L2 decay, schedule_decay 4e-3)      M, V as ADAM; m_schedule in the state (fp64)
 *   RADAM           optim/radam.py RAdam: P += -wd*lr*P; rectified update once N_sma >= 5, else P -= step_size*M
 *   ADADELTA        torch.optim.Adadelta, rho 0.9                       M = acc_delta, V = square_avg
 *   RMSPROP         torch.optim.RMSprop, alpha 0.9                      V = square_avg (from 0), M = momentum_buffer or NULL
 *   RMSPROPTF       optim/rmsprop_tf.py, alpha 0.9, lr in momentum      V = square_avg (the caller fills it with 1), M or NULL
 * Lookahead (optim/lookahead.py) wraps any of them: every lookahead_k-th update, S += alpha (P - S); P = S, where the first
 * synchronisation creates S from P (P unchanged). */
enum {
  COTB200_OPT_SGD = 1, COTB200_OPT_MOMENTUM = 2, COTB200_OPT_ADAM = 3, COTB200_OPT_ADAMW = 4, COTB200_OPT_NADAM = 5,
  COTB200_OPT_RADAM = 6, COTB200_OPT_ADADELTA = 7, COTB200_OPT_RMSPROP = 8, COTB200_OPT_RMSPROPTF = 9
};
typedef struct cotb200_opt_state {    /* device; the caller initialises t = 0, m_schedule = 1, the rest 0 */
  double t;                           /* updates done (every cotb200_opt_prepare with advance) */
  double m_schedule;                  /* NADAM: the product of the momentum caches */
  float c[4];                         /* this step's coefficients of the rule (cotb200_opt_prepare) */
  int sync;                           /* this step's Lookahead action: 0 none, 1 create S = P, 2 S += alpha (P - S); P = S */
  int slow_init;                      /* S holds the slow weights */
} cotb200_opt_state;
typedef struct cotb200_opt {          /* the optimizer of one flat range */
  int rule;                           /* COTB200_OPT_* */
  float eps;                          /* solver.opt_eps */
  int lookahead_k;                    /* 0: no Lookahead */
  float lookahead_alpha;
  float* M;                           /* fp32 state buffers of the range, 16-byte aligned (see the table above) */
  float* V;
  float* S;                           /* Lookahead's slow weights */
  cotb200_opt_state* state;           /* device, shared by the ranges of one optimizer */
} cotb200_opt;
/* Once per step before the passes: t += 1 (advance != 0) and everything that depends only on t and lr = hyper_dev[0], in fp64
 * (bias corrections, Nadam's momentum caches and m_schedule, RAdam's N_sma and step size, the Lookahead flag).  advance = 0:
 * only the flag, set to synchronise now (TrainStep.sync_lookahead).  One thread. */
int cotb200_opt_prepare(const cotb200_opt* opt, const float* hyper_dev, int advance, void* stream);
/* The pass over a flat range of n (multiple of 4) elements.  G fp32 or bf16 (g_dtype); E, Pb NULL: none; clip NULL: none. */
int cotb200_opt_step(long long n, float* P, int g_dtype, const void* G, float* E, void* Pb, const float* hyper_dev,
                     const cotb200_opt* opt, const cotb200_clip* clip, void* stream);
/* The Lookahead synchronisation prepared by cotb200_opt_prepare(advance = 0), and the bf16 copy Pb (NULL: none). */
int cotb200_lookahead_sync(long long n, float* P, void* Pb, const cotb200_opt* opt, void* stream);
/* y[n,h,w,c] = (x_u8[n,c,h,w] - mean[c]) / std[c]: uint8 NCHW batch -> normalised channels_last tensor of `dtype`
 * (PrefetchLoader, datasets/loader.py:66-67,86-90, + the channels_last / bf16 conversion of the AMP forward) in one
 * pass.  C == 3 with H*W % 4 == 0 takes mean_host/std_host (host arrays of 3); anything else needs the device arrays. */
int cotb200_u8_to_nhwc(int dtype, int N, int C, int H, int W, const void* x_u8, void* y, const float* mean_host,
                       const float* std_host, const float* mean_dev, const float* std_dev, void* stream);

/* ---- the training recipe of the reference configs: batch Mixup / CutMix and the soft-target loss ----
 * Per-step parameters of FastCollateMixup in batch mode (datasets/mixup.py:143-159,282-299, correct_lam).  The struct lives
 * in DEVICE memory and is read by the kernels, never passed by value, so a captured CUDA graph follows every step's draw.
 *   mode 0: no mixing (lam = 1); 1: mixup; 2: CutMix with the box rows [y0, y1) x columns [x0, x1).
 *   lam, one_minus_lam: the blend weights, each rounded to fp32 from the float64 draw (numpy's weak-scalar rule).
 *   target_lam: the weight of the sample's own label in the soft target (the box-corrected lam for CutMix). */
typedef struct cotb200_mix {
  int mode;
  float lam, one_minus_lam, target_lam;
  int y0, y1, x0, x1;
} cotb200_mix;
/* cotb200_u8_to_nhwc of the mixed batch: sample n is mixed with its partner N-1-n before the normalisation.  mode 1:
 * rint(x_n*lam + x_p*(1-lam)) in fp32 without FMA contraction (ties to even, np.rint); mode 2: x_p's pixels inside the box;
 * mode 0: bit-equal to cotb200_u8_to_nhwc.  N must be even when mix != NULL; mix == NULL means mode 0. */
int cotb200_u8_mix_to_nhwc(int dtype, int N, int C, int H, int W, const void* x_u8, void* y, const float* mean_host,
                           const float* std_host, const float* mean_dev, const float* std_dev, const cotb200_mix* mix,
                           void* stream);
/* Soft-target cross entropy of SoftTargetCrossEntropy(mixup_target(labels, K, lam, smoothing)) (loss/cross_entropy.py:29-36,
 * datasets/mixup.py:17-27) without materialising the target: per row b, with off = smoothing/K, on = 1 - smoothing + off,
 *   loss_b = lse(z_b) - off*sum_c z_bc - (on - off)*(lam*z_b[y_b] + (1-lam)*z_b[y_{B-1-b}]),  lam = mix->target_lam.
 * mix == NULL: lam = 1 (LabelSmoothingCrossEntropy; with smoothing 0 plain cross entropy).  logits: fp32 / bf16 / fp16
 * [B, K] with row pitch ld; labels int64 [B].  rows: fp32 [2, B] written: rows[b] = lse(z_b) (the backward reads it),
 * rows[B + b] = loss_b.  loss: fp32 [1] written with the batch mean, the rows added in a fixed order.  A label outside
 * [0, K) makes its row (and the mean) NaN; it is never read out of bounds.  An odd B with mix != NULL is rejected. */
int cotb200_soft_ce(int dtype, int B, int K, const void* logits, long long ld, const long long* labels, const cotb200_mix* mix,
                    float smoothing, float* rows, float* loss, void* stream);
/* dz[b, c] = dloss[0]/B * (softmax(z_b)_c - t_bc), fp32 [B, K] with row pitch ldz; dloss is read from device memory. */
int cotb200_soft_ce_bwd(int dtype, int B, int K, const void* logits, long long ld, const long long* labels,
                        const cotb200_mix* mix, float smoothing, const float* rows, const float* dloss, float* dz,
                        long long ldz, void* stream);
/* JsdCrossEntropy(num_splits=S, alpha, smoothing) (loss/jsd.py) of the augmentation splits.  logits: fp32 / bf16 / fp16
 * [S*B, K] with row pitch ld, split-major (row b + s*B is view s of sample b, view 0 the clean one); labels int64, only the
 * first B read.  Per clean row b, with p_sc = softmax(z_{b+sB})_c and m_c = clamp((sum_{s=0..S-1} p_sc) / S, 1e-7, 1):
 *   loss_b = ce_b + alpha/S * sum_s sum_c (xlogy(p_sc, p_sc) - p_sc log m_c),
 * ce_b the cotb200_soft_ce row of z_b without mixing (LabelSmoothingCrossEntropy; plain cross entropy at smoothing 0).  rows:
 * fp32 [S*B + B] written: rows[b + s*B] = lse(z_{b+sB}) (the backward reads them), rows[S*B + b] = loss_b.  loss: fp32 [1],
 * the mean of the B row losses added in a fixed order.  2 <= S <= 8, 0 <= smoothing < 1, alpha finite and >= 0.  A label
 * outside [0, K) makes its row (and the mean) NaN; it is never read out of bounds.
 * Where p_sc underflows to exactly 0 the term is taken at its xlogy limit, 0 in the loss and in the gradient; the reference's
 * autograd returns NaN there (0 * log 0 in the derivative of xlogy). */
int cotb200_jsd_ce(int dtype, int S, int B, int K, const void* logits, long long ld, const long long* labels,
                   float smoothing, float alpha, float* rows, float* loss, void* stream);
/* dz = dloss[0] * d(mean_b loss_b)/dz, fp32 [S*B, K] with row pitch ldz: per split the softmax Jacobian applied to
 * alpha/(S*B) * (log p_sc - log m_c + [the clamp binds at c]) (torch's clamp passes the gradient on the closed interval
 * [1e-7, 1]), plus the cross-entropy gradient on split 0.  dloss is read from device memory; an invalid label makes all S rows
 * of its sample NaN. */
int cotb200_jsd_ce_bwd(int dtype, int S, int B, int K, const void* logits, long long ld, const long long* labels,
                       float smoothing, float alpha, const float* rows, const float* dloss, float* dz, long long ldz, void* stream);

/* ---- validation metric ----
 * Top-k hit counts of utils/meters.py:12-19 (accuracy(): output.topk(maxk) then eq), accumulated on the device so that a
 * captured eval graph needs no host synchronisation per batch.  logits: fp32 / bf16 / fp16 [B, K] with row pitch ld; labels
 * int64 [B].  Rank rule: rank(b) = #{c : z_c > z_y} + #{c < y : z_c == z_y}; row b is a hit at k iff rank(b) < k.  On rows
 * without ties this equals accuracy(); on tied rows the lower class index wins (torch's topk order there is unspecified).  A
 * NaN label logit is a miss; NaN competitors never outrank.  Only rows b < *valid_dev count (valid_dev: device int, clamped to
 * [0, B]; NULL = all B rows), so a captured graph takes a short last batch.  ks: HOST array of nk (1..4) values, each in 1..K.
 * counts_dev: int64 [nk + 2], ACCUMULATED (+=): hits at each k, rows counted, rows whose label is outside [0, K) (a miss).
 * Integer sums: exact and independent of order. */
int cotb200_topk_hits(int dtype, int B, int K, const void* logits, long long ld, const long long* labels, const int* valid_dev,
                      int nk, const int* ks, long long* counts_dev, void* stream);

/* ---- image augmentation of the reference's input pipeline, byte-equal to its PIL transforms ----
 * RandomResizedCrop + horizontal flip + RandAugment (datasets/transforms_factory.py:44-129, datasets/rand_augment.py) and the
 * eval Resize + CenterCrop (:132-166) on a ragged batch of decoded HWC uint8 RGB images.  Every value the host draws lives in
 * DEVICE memory (an array of cotb200_aug_sample); the host copy of the same array is only validated, so that nothing is
 * ever read out of bounds.  Output: uint8 NCHW [N, 3, S, S], the batch fast_collate builds.
 * One RandAugment op.  op: -1 none, else the index in the reference's _RAND_TRANSFORMS: 0 AutoContrast, 1 Equalize, 2 Invert,
 * 3 Rotate, 4 Posterize, 5 Solarize, 6 SolarizeAdd, 7 Color, 8 Contrast, 9 Brightness, 10 Sharpness, 11 ShearX, 12 ShearY,
 * 13 TranslateX, 14 TranslateY, 15 Cutout. */
#define COTB200_AUG_MAX_OPS 2
typedef struct cotb200_aug_op {
  int op;
  int filter;          /* affine ops (3, 11..14): 0 bilinear, 1 bicubic */
  int v[4];            /* Posterize bits, Solarize threshold, SolarizeAdd addend in v[0]; Cutout box x0, y0, x1, y1 (ends inclusive) */
  float factor;        /* enhance ops (7..10): the Image.blend factor, rounded to fp32 as Pillow does */
  int pad_;
  double m[6];         /* affine ops: Image.transform's inverse matrix (x_in = m0 x + m1 y + m2, y_in = m3 x + m4 y + m5) */
} cotb200_aug_op;
/* One image: the crop (ci, cj, ch, cw) of the h x w source at byte `offset` is resized to rh x rw with `filter` (0 bilinear,
 * 1 bicubic; Pillow's two-pass resample, horizontal first, 22-bit fixed-point weights); the output is the window rows
 * [oi, oi + S) x columns [oj, oj + S) of that, mirrored left-right when flip.  tmp_offset: this image's 3*S*ch bytes of the
 * scratch buffer (horizontal-pass rows).  Then ops[0], ops[1] in order. */
typedef struct cotb200_aug_sample {
  long long offset;
  int h, w;
  int ci, cj, ch, cw;
  int rh, rw;
  int oi, oj;
  int filter, flip;
  long long tmp_offset;
  cotb200_aug_op ops[COTB200_AUG_MAX_OPS];
} cotb200_aug_sample;
/* Resize-crop (+ flip) of N images into out [N, 3, S, S].  src: src_bytes of concatenated HWC images; tmp: tmp_bytes of scratch.
 * params_host / params_dev: the same N samples on the host (validated) and on the device (read by the kernels).  Rejected with
 * COTB200_EINVAL: an image smaller than 1 x 1, an offset or scratch range past its buffer, a crop or window outside its image, a
 * bad filter; COTB200_EUNSUPPORTED: a downscale whose filter taps exceed the kernel's shared memory. */
int cotb200_aug_resize_crop(int N, int S, const unsigned char* src, long long src_bytes, const cotb200_aug_sample* params_host,
                            const cotb200_aug_sample* params_dev, unsigned char* tmp, long long tmp_bytes, unsigned char* out,
                            void* stream);
/* RandAugment ops of each sample applied in place to out [N, 3, S, S] (one CTA per image, the image held in shared memory).
 * An unknown op id or a bad argument is rejected with COTB200_EINVAL; S above 256 with COTB200_EUNSUPPORTED. */
int cotb200_aug_randaug(int N, int S, const cotb200_aug_sample* params_host, const cotb200_aug_sample* params_dev,
                        unsigned char* out, void* stream);
/* ColorJitter + RandomVerticalFlip of one image (transforms_factory.py:75-76,100-109, torchvision ColorJitter on PIL images).
 * vflip: 0/1, a row mirror of the S x S output, applied first.  order: the ops in application order (torchvision's randperm),
 * -1 entries skipped, each op at most once: 0 brightness (ImageEnhance.Brightness), 1 contrast (ImageEnhance.Contrast),
 * 2 saturation (ImageEnhance.Color), 3 hue (adjust_hue).  factor[op]: the Image.blend factor of ops 0..2 (>= 0, rounded to
 * fp32 as Pillow does); hue: adjust_hue's hue_factor in [-0.5, 0.5], shifting H by uint8(int32(hue * 255)) mod 256 between
 * Pillow's RGB -> HSV and HSV -> RGB conversions. */
typedef struct cotb200_aug_jitter {
  int vflip;
  int order[4];
  float factor[3];
  double hue;
} cotb200_aug_jitter;
/* ColorJitter (+ vflip) of each sample applied in place to out [N, 3, S, S], after cotb200_aug_resize_crop and before
 * cotb200_aug_randaug (one CTA per image, the image held in shared memory; a sample with nothing to do is not touched).
 * params_host / params_dev: the same N structs on the host (validated) and on the device (read by the kernel).  Rejected with
 * COTB200_EINVAL: a vflip other than 0/1, an unknown or repeated op, a factor below 0 or not finite, a hue outside
 * [-0.5, 0.5]; S above 256 with COTB200_EUNSUPPORTED. */
int cotb200_aug_color_jitter(int N, int S, const cotb200_aug_jitter* params_host, const cotb200_aug_jitter* params_dev,
                       unsigned char* out, void* stream);
/* Random erasing of the normalised batch (datasets/random_erasing.py, applied by PrefetchLoader after the normalisation,
 * datasets/loader.py:90-91).  The host draws the boxes; one buffer holds a cotb200_erase header followed directly by its n_boxes
 * cotb200_erase_box entries, grouped by sample n in increasing order, each sample's boxes in draw order with k = 0, 1, ...
 * (k < COTB200_ERASE_MAX_COUNT).  A box covers rows [top, top + h) x columns [left, left + w) of sample n; where boxes of a
 * sample overlap, the later one wins.  mode 0 ('const'): 0; 1 ('rand'): one N(0,1) value per (sample, box, channel); 2
 * ('pixel'): one N(0,1) value per element.  The values come from Philox4x32-10 with key = seed and counter = (y * W + x, or
 * 0xffffffff in mode 1, n, k, c / 4), Box-Muller-transformed, so they depend on the draw and the seed alone. */
#define COTB200_ERASE_MAX_COUNT 32
typedef struct cotb200_erase {
  int mode;
  int n_boxes;
  unsigned long long seed;
} cotb200_erase;
typedef struct cotb200_erase_box {
  int n, k;
  int top, left, h, w;
} cotb200_erase_box;
/* Erases the boxes in place in y, a channels_last [N, C, H, W] tensor of dtype fp32 / bf16 / fp16 (the output of
 * cotb200_u8_to_nhwc / cotb200_u8_mix_to_nhwc); written values are rounded to the dtype (round to nearest even).  erase_host /
 * erase_dev: the same buffer on the host (validated) and on the device (read by the kernel).  Only the erased pixels are
 * touched; n_boxes = 0 launches nothing.  Rejected with COTB200_EINVAL: a bad mode, a box outside its image or the batch, boxes
 * out of order, a sample with more than COTB200_ERASE_MAX_COUNT boxes; COTB200_EDTYPE: another dtype. */
int cotb200_aug_erase(int dtype, int N, int C, int H, int W, void* y, const cotb200_erase* erase_host,
                      const cotb200_erase* erase_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* COTB200_H_ */
