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

/* Fused inference step of the CoT block (models/cotnet.py:85-98 in eval mode), one kernel on the TMA ring:
 *   w = l * a[n,j] + c[n,j]          GroupNorm of the logits as a per-(sample, column) affine (coef = [N, 9*wc, 2] fp32, tap-major
 *                                    column order, from cotb200_gn9_from_colsums) applied to the weight tile in shared memory
 *   u = LocalConv(v, w)              3x3 / stride 1 / zero pad 1
 *   y = SiLU(u * bn_scale + bn_shift)      eval-mode BatchNorm folded, y stored
 *   psum[n, c] += sum_px (y + k)     the pooled descriptor of the split attention (caller zeroes psum)
 * d: NHWC_TAP layout, l in tap-major column order with chunk width d->gc.  Returns COTB200_EUNSUPPORTED when the geometry does
 * not fit the kernel. */
int cotb200_cot_agg_eval(const cotb200_agg_desc* d, const void* v, const void* l, const float* coef, const float* bn_scale,
                         const float* bn_shift, const void* k, void* y, float* psum, void* stream);

/* out = a[b,c,0]*y + a[b,c,1]*k on NHWC tensors [B, HW, C]: the radix-2 recombination (models/cotnet.py:101-104) when
 * y = SiLU(bn(.)) was already stored by cotb200_cot_agg_eval.  a [B,C,2] fp32. */
int cotb200_mix2(int dtype, int B, int HW, int C, const void* y, const void* k, const float* a, void* out, void* stream);

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

/* cotb200_gemm_bf16_samplestats: the single-product GEMM above whose statistics epilogue accumulates PER SAMPLE:
 *   samp_sum / samp_sqsum [M / rows_per_sample, N] += column sums / sums of squares of the STORED output (scale / shift
 *   applied, bf16-rounded) over the rows_per_sample consecutive rows (= H*W pixels) of each sample.  With
 *   cotb200_gn9_from_colsums (bias = NULL: it is already in the stored logits) this gives the GroupNorm statistics of the
 *   attention logits (models/cotnet.py:55-56) without a pass over them.  rows_per_sample >= 32, M % it == 0. */
int cotb200_gemm_bf16_samplestats(int M, int N, int K1, const void* A1, long long lda1, const void* B1, long long ldb1,
                                  void* D, long long ldd, const float* scale, const float* shift, int relu,
                                  int rows_per_sample, float* samp_sum, float* samp_sqsum, void* stream);
/* mean[b,g], rstd[b,g] of GroupNorm(wc groups of 9 taps) from per-sample column sums csum / csq [B, 9*wc] of the logits.
 * bias [9*wc]: a bias that is NOT yet contained in the summed values is accounted for analytically (NULL when the sums were
 * taken over the final logits); column order given by gc like cotb200_gn9_apply. */
int cotb200_gn9_from_colsums(int B, int HW, int wc, int gc, const float* csum, const float* csq, const float* bias,
                             float eps, float* mean, float* rstd, void* stream);
/* Same statistics, returned as the per-(sample, column) affine of the normalisation: coef[b, j] = (rstd*gamma_j,
 * beta_j - mean*rstd*gamma_j) with gamma / beta [9*wc] in the SAME column order as csum (what cotb200_cot_agg_eval takes). */
int cotb200_gn9_coef_from_colsums(int B, int HW, int wc, int gc, const float* csum, const float* csq, const float* bias,
                                  const float* gamma, const float* beta, float eps, float* coef, void* stream);

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

#ifdef __cplusplus
}
#endif
#endif /* COTB200_H_ */
