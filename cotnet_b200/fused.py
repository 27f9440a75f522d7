"""Autograd functions over the fused normalisation / split-attention kernels (csrc/norm_tail.cu).

They turn the reference block's long eager chains into a few HBM passes while keeping autograd semantics:

  GroupNorm9Fn   nn.GroupNorm(C/8, 9C/8) on the attention logits          /root/reference/models/cotnet.py:56
                 (under autocast the eager op runs in fp32 and writes 4-byte logits; here: 2 reads + 1 write)
  CotTailFn      bn -> SiLU -> (y + k) pooled -> se -> softmax(radix 2) -> a0*y + a1*k        :89-104
                 fwd: [stats] + pool + combine = 3 passes; bwd: sums + dz-sums + apply = 3 passes;
                 the tiny SE MLP on [B, C] stays PyTorch and is differentiated by autograd inside the function.

All tensors are channels_last (NHWC memory); math is fp32; outputs keep the input dtype.
"""
import torch
from torch.autograd import Function

from . import _lib


class _ZeroArena:
    """Pre-zeroed fp32 scratch for the kernels' accumulators (column sums, pooled sums, ...).  Every fused function needs a
    few KB of zeros per call; as torch.zeros that is ~370 fill launches per CoTNet-50 step.  A trainer that calls
    `fused.step_begin()` once per step gets them as slices of one buffer that is cleared by ONE memset of the part the
    previous step used.  Without step_begin() (or when the arena is exhausted) this is plain torch.zeros."""
    SIZE = 8 << 20                     # floats (32 MB)

    def __init__(self):
        self.buf = {}                  # device -> [buffer, used]
        self.active = False
        self.escape_ok = False         # a trainer that consumes every gradient before the next step_begin() may set this (see _zeros_esc)

    def begin(self, device):
        ent = self.buf.get(device)
        if ent is None:
            ent = [torch.zeros(self.SIZE, dtype=torch.float32, device=device), 0]
            self.buf[device] = ent
        elif ent[1]:
            ent[0][:ent[1]].zero_()
        ent[1] = 0
        self.active = True

    def take(self, n, device):
        ent = self.buf.get(device) if self.active else None
        if ent is None:
            return None
        n4 = (n + 3) & ~3              # keep 16-byte alignment of every slice
        if ent[1] + n4 > self.SIZE:
            return None
        out = ent[0][ent[1]:ent[1] + n]
        ent[1] += n4
        return out


_ARENA = _ZeroArena()


def step_begin(device=None):
    """Call once at the start of every training step (before the forward): recycles the accumulator scratch."""
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    _ARENA.begin(torch.device(device))


def step_arena_off():
    _ARENA.active = False


def _zeros(shape, device):
    n = 1
    for d in shape:
        n *= int(d)
    t = _ARENA.take(n, torch.device(device)) if n else None
    if t is None:
        return torch.zeros(*shape, dtype=torch.float32, device=device)
    return t.view(*shape)


def _zeros_esc(shape, device):
    """Zeros that ESCAPE the autograd function as gradients (BatchNorm d-gamma / d-beta sums).  Plain torch.zeros in general -- a
    gradient must survive until its owner reads it -- but a trainer that gathers every gradient inside the step (TrainStep: one gather
    launch into the flat bucket before the next step_begin()) may take them from the pre-zeroed arena too: ~140 fill launches per
    CoTNet-50 step less."""
    return _zeros(shape, device) if _ARENA.escape_ok else torch.zeros(*shape, dtype=torch.float32, device=device)


def arena_escape_ok(on=True):
    _ARENA.escape_ok = bool(on)


#: BatchNorm `num_batches_tracked += 1` bookkeeping: one tiny kernel per BatchNorm per step (~106 in CoTNet-50).  A trainer may defer
#: them (defer_bn_counters) and bump all counters with ONE multi-tensor add per step (flush_bn_counters).
_DEFERRED_COUNTERS = None


def defer_bn_counters(on=True):
    global _DEFERRED_COUNTERS
    _DEFERRED_COUNTERS = [] if on else None


def flush_bn_counters():
    if _DEFERRED_COUNTERS:
        with torch.no_grad():
            torch._foreach_add_(_DEFERRED_COUNTERS, 1)
        _DEFERRED_COUNTERS.clear()


def _bump_counter(bn):
    """num_batches_tracked += 1 now, or on the trainer's flush; returns True when the caller may rely on the NEW value immediately."""
    if _DEFERRED_COUNTERS is not None and bn.momentum is not None:
        _DEFERRED_COUNTERS.append(bn.num_batches_tracked)
        return False
    with torch.no_grad():
        bn.num_batches_tracked += 1
    return True


def _is_cl(t):
    return t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last)


def supported(t):
    return t.is_cuda and t.dtype in (torch.float32, torch.bfloat16, torch.float16) and _is_cl(t) and not t.is_contiguous()


def _f32(t):
    return t.detach().float().contiguous()


def _bn_running(bn, use_batch):
    """Bookkeeping shared by the two finalize routes: bumps num_batches_tracked, returns (update, momentum, rm, rv, copy_back)."""
    update = bool(use_batch and bn.running_mean is not None and bn.track_running_stats)
    mom = 0.0
    rm = rv = None
    if update:
        _bump_counter(bn)
        mom = bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked)
    if update or not use_batch:
        rm, rv = bn.running_mean, bn.running_var
        if rm.dtype != torch.float32:
            rm, rv = rm.float(), rv.float()
    return update, mom, rm, rv


def _bn_running_writeback(bn, update, rm, rv):
    if update and rm is not bn.running_mean:
        with torch.no_grad():
            bn.running_mean.copy_(rm)
            bn.running_var.copy_(rv)


def _bn_prepare(bn, weight, bias, C, n, sums, device, st):
    """[4, C] fp32 = (scale, shift, mean, rstd) in ONE launch (cotb200_bn_finalize).  `sums` = [2, C] column sums of the
    batch (training mode) or None (eval: running statistics).  Training updates the module's running buffers exactly like
    nn.BatchNorm2d (momentum, unbiased variance, num_batches_tracked)."""
    lib = _lib.load()
    out = torch.empty(4, C, dtype=torch.float32, device=device)
    use_batch = sums is not None
    update, mom, rm, rv = _bn_running(bn, use_batch)
    w32 = None if weight is None else weight.detach().float().contiguous()
    b32 = None if bias is None else bias.detach().float().contiguous()
    _lib.check(lib.cotb200_bn_finalize(C, _lib.ptr(sums[0]) if use_batch else None, _lib.ptr(sums[1]) if use_batch else None,
                                       _lib.ptr(w32), _lib.ptr(b32), _lib.ptr(rm), _lib.ptr(rv), float(n), float(bn.eps),
                                       float(mom), 1 if use_batch else 0, 1 if update else 0, out[0].data_ptr(),
                                       out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), st), "bn_finalize")
    _bn_running_writeback(bn, update, rm, rv)
    return out


def _bn_batch_stats(x, bn, weight, bias, lib, st, dt):
    """Statistics pass (training) + finalize -> ([4,C] scale/shift/mean/rstd, used_batch_stats)."""
    B, C, H, W = x.shape
    if bn.training or bn.running_mean is None:
        sums = _zeros((2, C,), x.device)
        _lib.check(lib.cotb200_col_stats(dt, B, H * W, C, x.data_ptr(), sums[0].data_ptr(), sums[1].data_ptr(), st), "col_stats")
        return _bn_prepare(bn, weight, bias, C, float(B * H * W), sums, x.device, st), True
    return _bn_prepare(bn, weight, bias, C, float(B * H * W), None, x.device, st), False


def _bn_apply_batch(x, res, sums, bn, weight, bias, relu, y, lib, st, dt, ds=None):
    """Training-mode BatchNorm tail shared by BNActFn and the wgmma functions: ONE kernel finalises the batch statistics
    (sums = [2, C] column sums over the B*H*W rows of x), updates the running buffers and applies scale/shift(+res)(+ReLU).
    ds: None or the [B] fp32 per-sample drop-path scales applied to the BatchNorm output before the residual add.
    Returns ss = [4, C] (scale, shift, mean, rstd) for the backward."""
    B, C, H, W = x.shape
    ss = torch.empty(4, C, dtype=torch.float32, device=x.device)
    update, mom, rm, rv = _bn_running(bn, True)
    w32 = None if weight is None else weight.detach().float().contiguous()
    b32 = None if bias is None else bias.detach().float().contiguous()
    args = (dt, B, H * W, C, x.data_ptr(), _lib.ptr(res), sums[0].data_ptr(), sums[1].data_ptr(), _lib.ptr(w32), _lib.ptr(b32),
            _lib.ptr(rm), _lib.ptr(rv), float(B * H * W), float(bn.eps), float(mom), 1 if update else 0, 1 if relu else 0,
            y.data_ptr(), ss[0].data_ptr(), ss[1].data_ptr(), ss[2].data_ptr(), ss[3].data_ptr())
    if ds is None:
        _lib.check(lib.cotb200_bn_apply_batch(*args, st), "bn_apply_batch")
    else:
        _lib.check(lib.cotb200_bn_apply_batch_ds(*args, ds.data_ptr(), st), "bn_apply_batch_ds")
    _bn_running_writeback(bn, update, rm, rv)
    return ss


def _drop_scale(ds, x):
    """The per-sample drop-path scales as the kernels take them: fp32 [B], contiguous, on x's device (None stays None)."""
    if ds is None:
        return None
    ds = ds.detach()
    assert ds.dim() == 1 and ds.shape[0] == x.shape[0] and ds.device == x.device, "drop_scale must be [B] on the input's device"
    return ds.float().contiguous()


def _bn_bwd(lib, dt, B, HW, C, dy, dy2, x, y, scale, shift, mean, rstd, rcode, sums, batch, inv_n, dx, dres, ds, st):
    """BatchNorm backward (sums + apply) of the plain / two-gradient form, or of the drop-path form when ds is given."""
    if sums is not None:
        args = (dt, B, HW, C, dy.data_ptr(), _lib.ptr(dy2), x.data_ptr(), _lib.ptr(y), _lib.ptr(scale), _lib.ptr(shift),
                mean.data_ptr(), rstd.data_ptr(), rcode, sums[0].data_ptr(), sums[1].data_ptr())
        if ds is None:
            _lib.check(lib.cotb200_bn_bwd_sums2(*args, st), "bn_bwd_sums")
        else:
            _lib.check(lib.cotb200_bn_bwd_sums_ds(*args, ds.data_ptr(), st), "bn_bwd_sums_ds")
    args = (dt, B, HW, C, dy.data_ptr(), _lib.ptr(dy2), x.data_ptr(), _lib.ptr(y), scale.data_ptr(), _lib.ptr(shift),
            mean.data_ptr(), rstd.data_ptr(), _lib.ptr(sums[0]) if batch else None, _lib.ptr(sums[1]) if batch else None,
            inv_n, rcode, dx.data_ptr(), _lib.ptr(dres))
    if ds is None:
        _lib.check(lib.cotb200_bn_bwd_apply2(*args, st), "bn_bwd_apply")
    else:
        _lib.check(lib.cotb200_bn_bwd_apply_ds(*args, ds.data_ptr(), st), "bn_bwd_apply_ds")


class BNActFn(Function):
    """y = act(BatchNorm2d(x) (+ res)) on channels_last tensors: col_stats + bn_finalize + bn_apply forward,
    bn_bwd_sums + bn_bwd_apply backward.  Replaces the nn.BatchNorm2d / nn.ReLU (/ residual add) modules of
    models/cotnet.py:45-46,53-54,61-62 and :231-235,:249-262 -- ATen's channels_last batch-norm kernels are the largest
    single cost of the eager step.  drop_scale: None or [B] per-sample stochastic-depth scales (models/cotnet.py:256-257),
    y = act(drop_scale[b]*BatchNorm2d(x) (+ res)) in the same kernels."""

    @staticmethod
    def forward(ctx, x, weight, bias, res, bn, relu, fork=False, drop_scale=None):
        assert _is_cl(x) and (res is None or (_is_cl(res) and res.dtype == x.dtype and res.shape == x.shape))
        ctx.set_materialize_grads(False)
        B, C, H, W = x.shape
        lib, st, dt = _lib.load(), _lib.stream_ptr(x), _lib.dtype_code(x)
        x = x.detach()
        ds = _drop_scale(drop_scale, x)
        y = torch.empty_like(x, memory_format=torch.channels_last)
        batch = bool(bn.training or bn.running_mean is None)
        if batch:       # training: column sums, then ONE kernel that finalises the statistics in its prologue and applies them
            sums = _zeros((2, C,), x.device)
            _lib.check(lib.cotb200_col_stats(dt, B, H * W, C, x.data_ptr(), sums[0].data_ptr(), sums[1].data_ptr(), st), "col_stats")
            ss = _bn_apply_batch(x, res, sums, bn, weight, bias, relu, y, lib, st, dt, ds)   # [4,C]: scale, shift, mean, rstd
        else:
            ss = _bn_prepare(bn, weight, bias, C, float(B * H * W), None, x.device, st)
            args = (dt, B, H * W, C, x.data_ptr(), _lib.ptr(res), ss[0].data_ptr(), ss[1].data_ptr(), 1 if relu else 0, y.data_ptr())
            if ds is None:
                _lib.check(lib.cotb200_bn_apply(*args, st), "bn_apply")
            else:
                _lib.check(lib.cotb200_bn_apply_ds(*args, ds.data_ptr(), st), "bn_apply_ds")
        # ReLU mask in the backward: with a residual it must come from y; without one it is recomputed from x and the
        # forward's own scale/shift (relu code 2) and y is neither saved nor read
        ctx.save_for_backward(x, y if (relu and res is not None) else None, ss, ds)
        ctx.cfg = (relu, batch, res is not None, weight.dtype, bias.dtype)
        if fork:            # two aliases of ONE tensor: each consumer's gradient reaches backward() separately (see _two_grads)
            return y, y.detach()
        return y

    @staticmethod
    def backward(ctx, *grads):
        x, y, ss, ds = ctx.saved_tensors
        relu, batch, has_res, wdt, bdt = ctx.cfg
        B, C, H, W = x.shape
        lib, st, dt = _lib.load(), _lib.stream_ptr(x), _lib.dtype_code(x)
        dy, dy2 = _two_grads(grads)
        if dy is None:
            return (None,) * 8
        rcode = 0 if not relu else (1 if y is not None else 2)
        sums = None
        if batch or ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            sums = _zeros_esc((2, C,), x.device)       # escapes as dgamma/dbeta
        dx = torch.empty_like(x, memory_format=torch.channels_last)
        dres = torch.empty_like(x, memory_format=torch.channels_last) if (has_res and ctx.needs_input_grad[3]) else None
        _bn_bwd(lib, dt, B, H * W, C, dy, dy2, x, y, ss[0], ss[1], ss[2], ss[3], rcode, sums, batch, 1.0 / float(B * H * W), dx, dres,
                ds, st)
        dgamma = sums[1].to(wdt) if ctx.needs_input_grad[1] else None
        dbeta = sums[0].to(bdt) if ctx.needs_input_grad[2] else None
        return dx, dgamma, dbeta, dres, None, None, None, None


def _two_grads(grads):
    """Incoming gradients of a (possibly forked) output: (dy, dy2) as channels_last tensors, dy2 None when there is one gradient.
    A forked BatchNorm output feeds two consumers -- the next bottleneck's conv1 and its shortcut (models/cotnet.py:228-262) -- and
    autograd would add their gradients with a separate kernel (read 2 + write 1 of the block-sized tensor);
    handing both to the BatchNorm backward kernels, which sum them in fp32 while they stream dy anyway, costs one extra read each."""
    g = [t.contiguous(memory_format=torch.channels_last) for t in grads if t is not None]
    if not g:
        return None, None
    if len(g) == 1:
        return g[0], None
    return g[0], g[1]


def bn_act(x, bn: torch.nn.BatchNorm2d, relu=False, res=None, fork=False, drop_scale=None):
    """Fused BatchNorm2d (+ residual add) (+ ReLU) with the module's parameters / buffers / train-eval semantics.
    fork=True returns two aliases of the output (see _two_grads); drop_scale: per-sample stochastic-depth scales [B] or None."""
    return BNActFn.apply(x, bn.weight, bn.bias, res, bn, relu, fork, drop_scale)


class GroupNorm9Fn(Function):
    """l [B, 9*wc, H, W] channels_last -> GroupNorm with wc groups of 9 consecutive channels (gc=0) or tap-major
    chunks (gc>0); gamma/beta [9*wc].  `lbias` (None or [9*wc]): bias of the producing embed.3 convolution, added to l
    inside the kernels (the convolution then runs bias-free and its bias gradient comes out of gn9_bwd_apply)."""

    @staticmethod
    def forward(ctx, l, gamma, beta, eps, gc=0, lbias=None):
        assert _is_cl(l)
        B, J, H, W = l.shape
        wc, HW = J // 9, H * W
        lib, st, dt = _lib.load(), _lib.stream_ptr(l), _lib.dtype_code(l)
        l = l.detach()
        lb32 = None if lbias is None else _f32(lbias)
        stats = _zeros((2, B, wc,), l.device)
        _lib.check(lib.cotb200_gn9_stats(dt, B, HW, wc, gc, l.data_ptr(), _lib.ptr(lb32), stats[0].data_ptr(),
                                         stats[1].data_ptr(), st), "gn9_stats")
        fin = torch.empty(4, B * wc, dtype=torch.float32, device=l.device)      # (rstd, -mean*rstd, mean, rstd)
        _lib.check(lib.cotb200_bn_finalize(B * wc, stats[0].data_ptr(), stats[1].data_ptr(), None, None, None, None, 9.0 * HW,
                                           float(eps), 0.0, 1, 0, fin[0].data_ptr(), fin[1].data_ptr(), fin[2].data_ptr(),
                                           fin[3].data_ptr(), st), "bn_finalize")
        mean, rstd = fin[2], fin[3]
        g32, b32 = _f32(gamma), _f32(beta)
        out = torch.empty_like(l, memory_format=torch.channels_last)
        _lib.check(lib.cotb200_gn9_apply(dt, B, HW, wc, gc, l.data_ptr(), _lib.ptr(lb32), mean.data_ptr(), rstd.data_ptr(),
                                         g32.data_ptr(), b32.data_ptr(), out.data_ptr(), st), "gn9_apply")
        ctx.save_for_backward(l, mean, rstd, g32, lb32)
        ctx.gc = gc
        ctx.param_dtype = (gamma.dtype, beta.dtype, None if lbias is None else lbias.dtype)
        return out

    @staticmethod
    def backward(ctx, dg):
        l, mean, rstd, g32, lb32 = ctx.saved_tensors
        B, J, H, W = l.shape
        wc, HW = J // 9, H * W
        dg = dg.contiguous(memory_format=torch.channels_last)
        lib, st, dt = _lib.load(), _lib.stream_ptr(l), _lib.dtype_code(l)
        sums = torch.empty(2, B, wc, dtype=torch.float32, device=l.device)      # s1, s2 (written)
        dgb = _zeros_esc((3, J,), l.device)            # dgamma, dbeta, dlbias (escape)
        work = _zeros((3 * B * J,), l.device)                                     # per-sample column partials
        want_db = lb32 is not None and ctx.needs_input_grad[5]
        _lib.check(lib.cotb200_gn9_bwd_sums(dt, B, HW, wc, ctx.gc, dg.data_ptr(), l.data_ptr(), _lib.ptr(lb32), mean.data_ptr(),
                                            rstd.data_ptr(), g32.data_ptr(), work.data_ptr(), sums[0].data_ptr(),
                                            sums[1].data_ptr(), dgb[0].data_ptr(), dgb[1].data_ptr(),
                                            dgb[2].data_ptr() if want_db else None, st), "gn9_bwd_sums")
        dl = None
        if ctx.needs_input_grad[0]:
            dl = torch.empty_like(l, memory_format=torch.channels_last)
            _lib.check(lib.cotb200_gn9_bwd_apply(dt, B, HW, wc, ctx.gc, dg.data_ptr(), l.data_ptr(), _lib.ptr(lb32),
                                                 mean.data_ptr(), rstd.data_ptr(), g32.data_ptr(), sums[0].data_ptr(),
                                                 sums[1].data_ptr(), dl.data_ptr(), st), "gn9_bwd_apply")
        return (dl, dgb[0].to(ctx.param_dtype[0]), dgb[1].to(ctx.param_dtype[1]), None, None,
                dgb[2].to(ctx.param_dtype[2]) if want_db else None)


def _row_view(t):
    """(pitch in elements) of a [B, C, H, W] tensor whose memory is NHWC rows with a constant pixel pitch >= C (a
    channels_last tensor or a channel slice of one), else None."""
    if t.dim() != 4:
        return None
    B, C, H, W = t.shape
    sb, sc, sh, sw = t.stride()
    if C > 1 and sc != 1:
        return None
    ld = sw if W > 1 else (sh if H > 1 else (sb if B > 1 else C))
    if ld < C or (W > 1 and H > 1 and sh != W * ld) or (B > 1 and H * W > 1 and sb != H * W * ld):
        return None
    return ld


class FanOutFn(Function):
    """x -> n aliases of x whose gradients are accumulated by ONE kernel (cotb200_sum_rows) instead of autograd's chain
    of pairwise adds; the concat's channel-sliced gradients (pitch 2C) are read in place."""

    @staticmethod
    def forward(ctx, x, n):
        ctx.n = n
        return tuple(x.view_as(x) for _ in range(n))

    @staticmethod
    def backward(ctx, *grads):
        gs = [g for g in grads if g is not None]
        if not gs:
            return None, None
        if len(gs) == 1:
            return gs[0], None
        srcs = []
        for g in gs:
            ld = _row_view(g) if g.is_cuda else None
            if ld is None:
                g = g.contiguous(memory_format=torch.channels_last)
                ld = g.shape[1]
            srcs.append((g, ld))
        B, C, H, W = gs[0].shape
        lib, st, dt = _lib.load(), _lib.stream_ptr(gs[0]), _lib.dtype_code(gs[0])
        out = torch.empty((B, C, H, W), dtype=gs[0].dtype, device=gs[0].device, memory_format=torch.channels_last)
        while len(srcs) > 1:
            grp, srcs = srcs[:4], srcs[4:]
            args = []
            for i in range(4):
                args += [grp[i][0].data_ptr(), grp[i][1]] if i < len(grp) else [None, 0]
            _lib.check(lib.cotb200_sum_rows(dt, B * H * W, C, *args, out.data_ptr(), C, st), "sum_rows")
            srcs = [(out, C)] + srcs
        return out, None


def fan_out(x, n):
    """n aliases of x for n consumers; see FanOutFn.  Falls through (returns x n times) when no gradient is needed."""
    if not (torch.is_grad_enabled() and x.requires_grad):
        return (x,) * n
    return FanOutFn.apply(x, n)


class CotTailFn(Function):
    """(u, k) -> out of models/cotnet.py:89-104.  `bn` is the nn.BatchNorm2d(dim) module (its buffers are updated in
    training mode exactly like the module would); `attn_fn` maps the pooled mean [B, C] (fp32, requires grad) to the
    mixing weights a [B, C, 2] -- the radix-2 softmax of the `se` MLP for the CoT layer.  With k = None the same kernels
    compute SplitAttnConv2d's radix-1 chain (models/layers/split_attn.py:68-86): bn0 -> SiLU -> pool -> MLP -> sigmoid
    gate, a[..., 0] = the gate."""

    @staticmethod
    def forward(ctx, u, k, bn_weight, bn_bias, bn, attn_fn, *mlp_params):
        assert _is_cl(u) and (k is None or (_is_cl(k) and u.dtype == k.dtype and u.shape == k.shape))
        B, C, H, W = u.shape
        HW, n = H * W, float(B * H * W)
        lib, st, dt = _lib.load(), _lib.stream_ptr(u), _lib.dtype_code(u)
        u, k = u.detach(), (None if k is None else k.detach())
        ss, training = _bn_batch_stats(u, bn, bn_weight, bn_bias, lib, st, dt)     # [4,C]: scale, shift, mean, rstd
        scale, shift, mean, rstd = ss[0], ss[1], ss[2], ss[3]
        psum = _zeros((B, C,), u.device)
        _lib.check(lib.cotb200_tail_pool(dt, B, HW, C, u.data_ptr(), _lib.ptr(k), scale.data_ptr(), shift.data_ptr(),
                                         psum.data_ptr(), st), "tail_pool")
        # the SE MLP on [B, C] (3 tiny GEMV-sized ops) stays PyTorch; its graph is kept for backward
        # ... in fp32 whatever the storage dtype: se.1 normalises over the batch, which amplifies bf16 rounding of the
        # pooled descriptor by an order of magnitude (the fp32 math costs nothing at [B, C])
        with torch.enable_grad(), torch.autocast("cuda", enabled=False):
            p_leaf = (psum / HW).requires_grad_(True)
            a = attn_fn(p_leaf)
        a_c = a.detach().contiguous()
        out = torch.empty_like(u, memory_format=torch.channels_last)
        _lib.check(lib.cotb200_tail_combine(dt, B, HW, C, u.data_ptr(), _lib.ptr(k), scale.data_ptr(), shift.data_ptr(),
                                            a_c.data_ptr(), out.data_ptr(), st), "tail_combine")
        ctx.save_for_backward(u, k, scale, shift, mean, rstd, a_c)
        ctx.graph = (p_leaf, a, [p for p in mlp_params])
        ctx.training = training
        ctx.bn_dtypes = (bn_weight.dtype, bn_bias.dtype)
        return out

    @staticmethod
    def backward(ctx, dout):
        u, k, scale, shift, mean, rstd, a_c = ctx.saved_tensors
        p_leaf, a, mlp_params = ctx.graph
        B, C, H, W = u.shape
        HW, n = H * W, float(B * H * W)
        lib, st, dt = _lib.load(), _lib.stream_ptr(u), _lib.dtype_code(u)
        dout = dout.contiguous(memory_format=torch.channels_last)
        S = _zeros((B, C, 2,), u.device)
        _lib.check(lib.cotb200_tail_bwd_sums(dt, B, HW, C, dout.data_ptr(), u.data_ptr(), _lib.ptr(k), scale.data_ptr(),
                                             shift.data_ptr(), S.data_ptr(), st), "tail_bwd_sums")
        grads = torch.autograd.grad(a, [p_leaf] + mlp_params, grad_outputs=S, allow_unused=True)
        dpn = grads[0].contiguous()                      # d/d(pooled mean); the kernels apply the 1/HW (pscale)
        mlp_grads = [None if g is None else g for g in grads[1:]]
        sums = _zeros_esc((2, C,), u.device)          # escapes as dgamma/dbeta
        need_param = ctx.needs_input_grad[2] or ctx.needs_input_grad[3]
        if ctx.training or need_param:
            _lib.check(lib.cotb200_tail_bwd_dz_sums(dt, B, HW, C, dout.data_ptr(), u.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                                                    mean.data_ptr(), rstd.data_ptr(), a_c.data_ptr(), dpn.data_ptr(), 1.0 / HW,
                                                    sums[0].data_ptr(), sums[1].data_ptr(), st), "tail_bwd_dz_sums")
        c1 = c2 = None
        if ctx.training:
            c1, c2 = sums[0], sums[1]
        du = torch.empty_like(u, memory_format=torch.channels_last)
        dk = torch.empty_like(u, memory_format=torch.channels_last) if (k is not None and ctx.needs_input_grad[1]) else None
        _lib.check(lib.cotb200_tail_bwd_apply(dt, B, HW, C, dout.data_ptr(), u.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                                              mean.data_ptr(), rstd.data_ptr(), a_c.data_ptr(), dpn.data_ptr(), _lib.ptr(c1),
                                              _lib.ptr(c2), 1.0 / n, 1.0 / HW, du.data_ptr(), _lib.ptr(dk), st), "tail_bwd_apply")
        dgamma = sums[1].to(ctx.bn_dtypes[0]) if ctx.needs_input_grad[2] else None
        dbeta = sums[0].to(ctx.bn_dtypes[1]) if ctx.needs_input_grad[3] else None
        ctx.graph = None
        return (du, dk, dgamma, dbeta, None, None) + tuple(mlp_grads)


class AggTapFn(Function):
    """LocalConv 3x3 (stride 1, zero pad 1) on channels_last tensors with the weights in the block-internal tap-major
    order (COTB200_NHWC_TAP, chunk width gc) -- or the reference order when gc == 0.  v [B,C,H,W], w [B,9*wc,H,W]."""

    @staticmethod
    def forward(ctx, v, w, fold, gc):
        assert _is_cl(v) and _is_cl(w) and v.dtype == w.dtype
        v, w = v.detach(), w.detach()
        out = torch.empty_like(v, memory_format=torch.channels_last)
        dsc = AggTapFn._desc(v, w, fold, gc)
        _lib.check(_lib.load().cotb200_agg_zeropad_fwd(dsc, v.data_ptr(), w.data_ptr(), out.data_ptr(), _lib.stream_ptr(v)),
                   "agg_zeropad_fwd")
        ctx.save_for_backward(v, w)
        ctx.cfg = (fold, gc)
        return out

    @staticmethod
    def _desc(v, w, fold, gc):
        B, C, H, W = v.shape
        d = _lib.AggDesc()
        d.n, d.c, d.h, d.w = B, C, H, W
        d.heads, d.wc = 1, w.shape[1] // 9
        d.kh = d.kw = 3
        d.sh = d.sw = d.ph = d.pw = d.dh = d.dw = 1
        d.ho, d.wo = H, W
        d.dtype = _lib.dtype_code(v)
        d.layout = _lib.NHWC_TAP if gc > 0 else _lib.NHWC
        d.gc, d.fold = gc, fold
        return d

    @staticmethod
    def backward(ctx, dy):
        v, w = ctx.saved_tensors
        fold, gc = ctx.cfg
        dy = dy.contiguous(memory_format=torch.channels_last)
        dv = torch.empty_like(v, memory_format=torch.channels_last) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(w, memory_format=torch.channels_last) if ctx.needs_input_grad[1] else None
        if dv is not None or dw is not None:
            dsc = AggTapFn._desc(v, w, fold, gc)
            _lib.check(_lib.load().cotb200_agg_zeropad_bwd(dsc, dy.data_ptr(), v.data_ptr(), w.data_ptr(), _lib.ptr(dv),
                                                           _lib.ptr(dw), _lib.stream_ptr(v)), "agg_zeropad_bwd")
        return dv, dw, None, None


class Pool3x3S2Fn(Function):
    """nn.AvgPool2d(3, 2, padding=1) (mode 0, count_include_pad) / nn.MaxPool2d(3, 2, 1) (mode 1) on channels_last."""

    @staticmethod
    def forward(ctx, x, mode):
        assert _is_cl(x)
        B, C, H, W = x.shape
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        x = x.detach()
        y = torch.empty((B, C, Ho, Wo), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        idx = torch.empty((B, Ho, Wo, C), dtype=torch.uint8, device=x.device) if mode == 1 else None
        _lib.check(_lib.load().cotb200_pool3s2_fwd(_lib.dtype_code(x), mode, B, H, W, C, x.data_ptr(), y.data_ptr(), _lib.ptr(idx),
                                                   _lib.stream_ptr(x)), "pool3s2_fwd")
        ctx.save_for_backward(idx)
        ctx.cfg = (mode, B, C, H, W, x.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        mode, B, C, H, W, dtype = ctx.cfg
        dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty((B, C, H, W), dtype=dtype, device=dy.device, memory_format=torch.channels_last)
        _lib.check(_lib.load().cotb200_pool3s2_bwd(_lib.dtype_code(dy), mode, B, H, W, C, dy.data_ptr(), _lib.ptr(idx), dx.data_ptr(),
                                                   _lib.stream_ptr(dy)), "pool3s2_bwd")
        return dx, None


def avg_pool3x3s2(x):
    return Pool3x3S2Fn.apply(x, 0)


def max_pool3x3s2(x):
    return Pool3x3S2Fn.apply(x, 1)


def tap_chunk(wc, fold=1):
    """Chunk width of the tap-major weight order the fast kernels use, 0 when wc does not allow it."""
    return 8 if (wc // fold) % 8 == 0 else 0


def _mlp_fp32(c0, b1, c3, p, act):
    """conv1x1 -> BatchNorm2d -> act -> conv1x1 on p [B, C] in fp32 (models/cotnet.py:69-77 with ReLU;
    models/layers/split_attn.py:51-55,76-80 with SiLU), using (and updating) the modules' parameters / buffers;
    differentiable w.r.t. p and the parameters.  The BatchNorm is ONE fused ATen kernel each way (F.batch_norm on private
    copies of the running buffers -- autograd saves those copies, so updating the module's own buffers afterwards cannot
    invalidate the graph); the whole MLP is ~10 launches forward, ~10 backward."""
    F = torch.nn.functional
    z = F.linear(p, c0.weight.float().flatten(1), None if c0.bias is None else c0.bias.float())
    w1, bb1 = b1.weight.float(), b1.bias.float()
    if b1.training or b1.running_mean is None:
        track = b1.running_mean is not None and b1.track_running_stats
        rm = rv = None
        mom = 0.0
        if track:
            _bump_counter(b1)
            with torch.no_grad():
                mom = b1.momentum if b1.momentum is not None else 1.0 / float(b1.num_batches_tracked)
                rm, rv = b1.running_mean.float().clone(), b1.running_var.float().clone()
        z = F.batch_norm(z, rm, rv, w1, bb1, True, mom, b1.eps)
        if track:
            with torch.no_grad():
                b1.running_mean.copy_(rm)
                b1.running_var.copy_(rv)
    else:
        z = F.batch_norm(z, b1.running_mean.float(), b1.running_var.float(), w1, bb1, False, 0.0, b1.eps)
    z = act(z)
    return F.linear(z, c3.weight.float().flatten(1), None if c3.bias is None else c3.bias.float())


def _se_fp32(se, p):
    return _mlp_fp32(se[0], se[1], se[3], p, torch.relu)


def group_norm9(l, gn: torch.nn.GroupNorm, gc=0, lbias=None):
    return GroupNorm9Fn.apply(l, gn.weight, gn.bias, gn.eps, gc, lbias)


def _se_eval_params(se):
    """fp32 weights of the `se` MLP with its BatchNorm folded (eval mode), cached until a parameter / buffer changes."""
    key = tuple(t._version for t in list(se.parameters()) + list(se.buffers())) + (str(next(se.parameters()).device),)
    cache = getattr(se, "_cotb200_eval_cache", None)
    if cache is not None and cache[0] == key:
        return cache[1]
    c0, b1, c3 = se[0], se[1], se[3]
    with torch.no_grad():
        rstd = torch.rsqrt(b1.running_var.float() + b1.eps)
        s1 = (b1.weight.float() * rstd).contiguous()
        t1 = (b1.bias.float() - b1.running_mean.float() * s1).contiguous()
        prm = (c0.weight.detach().float().flatten(1).contiguous(), None if c0.bias is None else c0.bias.detach().float().contiguous(), s1, t1,
               c3.weight.detach().float().flatten(1).contiguous(), None if c3.bias is None else c3.bias.detach().float().contiguous())
    se._cotb200_eval_cache = (key, prm)
    return prm


def _cot_tail_eval(u, k, bn, se):
    """Inference form of models/cotnet.py:89-104 in three launches: pool (bn + SiLU + (y + k) summed over the pixels), the
    whole SE MLP + radix-2 softmax (cotb200_se_eval), recombination."""
    B, C, H, W = u.shape
    lib, st, dt = _lib.load(), _lib.stream_ptr(u), _lib.dtype_code(u)
    ss = _bn_prepare(bn, bn.weight, bn.bias, C, float(B * H * W), None, u.device, st)
    psum = torch.zeros(B, C, dtype=torch.float32, device=u.device)
    _lib.check(lib.cotb200_tail_pool(dt, B, H * W, C, u.data_ptr(), k.data_ptr(), ss[0].data_ptr(), ss[1].data_ptr(), psum.data_ptr(), st),
               "tail_pool")
    w0, b0, s1, t1, w3, b3 = _se_eval_params(se)
    a = torch.empty(B, C, 2, dtype=torch.float32, device=u.device)
    zs = torch.empty(B, w0.shape[0], dtype=torch.float32, device=u.device)
    _lib.check(lib.cotb200_se_eval(B, C, w0.shape[0], psum.data_ptr(), 1.0 / (H * W), w0.data_ptr(), _lib.ptr(b0), s1.data_ptr(),
                                   t1.data_ptr(), w3.data_ptr(), _lib.ptr(b3), a.data_ptr(), zs.data_ptr(), st), "se_eval")
    out = torch.empty_like(u, memory_format=torch.channels_last)
    _lib.check(lib.cotb200_tail_combine(dt, B, H * W, C, u.data_ptr(), k.data_ptr(), ss[0].data_ptr(), ss[1].data_ptr(), a.data_ptr(),
                                        out.data_ptr(), st), "tail_combine")
    return out


def group_norm9_from_colsums(l, gn: torch.nn.GroupNorm, gc, csum, csq, lbias_in_stats):
    """Inference GroupNorm(9 taps) whose statistics come from the logits GEMM's epilogue (per-sample column sums of the raw
    accumulator, cotb200_gemm_bf16_samplestats): one tiny kernel turns them into mean / rstd, then the apply kernel.  `l` already
    contains the embed.3 bias and so do the sums (they are taken from the stored logits): `lbias_in_stats` is None unless the
    sums come from somewhere that has not seen the bias."""
    B, J, H, W = l.shape
    wc = J // 9
    lib, st, dt = _lib.load(), _lib.stream_ptr(l), _lib.dtype_code(l)
    mr = torch.empty(2, B * wc, dtype=torch.float32, device=l.device)
    _lib.check(lib.cotb200_gn9_from_colsums(B, H * W, wc, 0, csum.data_ptr(), csq.data_ptr(), _lib.ptr(lbias_in_stats), float(gn.eps),
                                            mr[0].data_ptr(), mr[1].data_ptr(), st), "gn9_from_colsums")
    g32, b32 = _f32(gn.weight), _f32(gn.bias)
    out = torch.empty_like(l, memory_format=torch.channels_last)
    _lib.check(lib.cotb200_gn9_apply(dt, B, H * W, wc, gc, l.data_ptr(), None, mr[0].data_ptr(), mr[1].data_ptr(), g32.data_ptr(),
                                     b32.data_ptr(), out.data_ptr(), st), "gn9_apply")
    return out


def cot_eval_tail_fused(v, l2d, csum, csq, lbias_p, gamma_p, beta_p, eps, gc, bn_ss, k, se):
    """Inference tail of the CoT block from the logits GEMM on: coefficient kernel (GroupNorm statistics -> per-(sample, column)
    affine), the fused LocalConv kernel (GroupNorm affine + aggregation + bn + SiLU + pooled (y + k)), the SE kernel, and the
    recombination -- 4 launches for models/cotnet.py:85-104.  v, k: channels_last [B,C,H,W]; l2d: [B*H*W, 9C/8] tap-major logits
    (bias included) with per-sample column sums csum / csq of the pre-bias accumulator.  Returns None when the fused kernel cannot
    take the geometry (the caller then uses the separate kernels)."""
    B, C, H, W = v.shape
    wc = C // 8
    lib, st, dt = _lib.load(), _lib.stream_ptr(v), _lib.dtype_code(v)
    coef = torch.empty(B, 9 * wc, 2, dtype=torch.float32, device=v.device)
    _lib.check(lib.cotb200_gn9_coef_from_colsums(B, H * W, wc, gc, csum.data_ptr(), csq.data_ptr(), _lib.ptr(lbias_p), gamma_p.data_ptr(),
                                                 beta_p.data_ptr(), float(eps), coef.data_ptr(), st), "gn9_coef_from_colsums")
    d = _lib.AggDesc()
    d.n, d.c, d.h, d.w = B, C, H, W
    d.heads, d.wc = 1, wc
    d.kh = d.kw = 3
    d.sh = d.sw = d.ph = d.pw = d.dh = d.dw = 1
    d.ho, d.wo = H, W
    d.dtype, d.layout, d.gc, d.fold = dt, _lib.NHWC_TAP, gc, 1
    y = torch.empty_like(v, memory_format=torch.channels_last)
    psum = torch.zeros(B, C, dtype=torch.float32, device=v.device)
    rc = lib.cotb200_cot_agg_eval(d, v.data_ptr(), l2d.data_ptr(), coef.data_ptr(), bn_ss[0].data_ptr(), bn_ss[1].data_ptr(), k.data_ptr(),
                                  y.data_ptr(), psum.data_ptr(), st)
    if rc == -7:                                   # COTB200_EUNSUPPORTED
        return None
    _lib.check(rc, "cot_agg_eval")
    w0, b0, s1, t1, w3, b3 = _se_eval_params(se)
    a = torch.empty(B, C, 2, dtype=torch.float32, device=v.device)
    zs = torch.empty(B, w0.shape[0], dtype=torch.float32, device=v.device)
    _lib.check(lib.cotb200_se_eval(B, C, w0.shape[0], psum.data_ptr(), 1.0 / (H * W), w0.data_ptr(), _lib.ptr(b0), s1.data_ptr(),
                                   t1.data_ptr(), w3.data_ptr(), _lib.ptr(b3), a.data_ptr(), zs.data_ptr(), st), "se_eval")
    out = torch.empty_like(v, memory_format=torch.channels_last)
    _lib.check(lib.cotb200_mix2(dt, B, H * W, C, y.data_ptr(), k.data_ptr(), a.data_ptr(), out.data_ptr(), st), "mix2")
    return out


def cot_tail(u, k, bn: torch.nn.BatchNorm2d, se: torch.nn.Module):
    if (not torch.is_grad_enabled() and not bn.training and not se[1].training and k is not None and se[1].running_mean is not None
            and bn.running_mean is not None and isinstance(se[2], torch.nn.ReLU)):
        return _cot_tail_eval(u.detach(), k.detach(), bn, se)
    params = [p for p in se.parameters()]
    B, C = u.shape[0], u.shape[1]
    return CotTailFn.apply(u, k, bn.weight, bn.bias, bn, lambda p: torch.softmax(_se_fp32(se, p).view(B, C, 2), dim=2), *params)


def split_attn_tail(u, bn0: torch.nn.BatchNorm2d, fc1, bn1, fc2):
    """SplitAttnConv2d (radix 1) after its convolution (models/layers/split_attn.py:68-86): bn0 -> SiLU -> global average
    pool -> fc1 -> bn1 -> SiLU -> fc2 -> sigmoid -> rescale, on the CoT tail kernels with k absent: 3 HBM passes forward
    (statistics, pool, gate) and 3 backward instead of ~12 eager ones."""
    params = list(fc1.parameters()) + list(bn1.parameters()) + list(fc2.parameters())
    F = torch.nn.functional

    def gate(p):
        g = torch.sigmoid(_mlp_fp32(fc1, bn1, fc2, p, F.silu))
        return torch.stack([g, torch.zeros_like(g)], dim=2)
    return CotTailFn.apply(u, None, bn0.weight, bn0.bias, bn0, gate, *params)


# ====================================================================================================================
# Dense parts of the block on the wgmma kernels, with autograd.
#   forward      : tc GEMM / implicit-GEMM conv; training-mode BatchNorm statistics come out of the GEMM epilogue
#   data gradient: the same tc kernels (transposed weights; the 3x3 conv with flipped taps)
#   weight grad  : 1x1: the MN-major wgmma kernel (tc_wgrad.cu); the grouped 3x3 still goes through cuDNN
# ====================================================================================================================
from . import tc as _tc  # noqa: E402
import os as _os  # noqa: E402


def _rows2d(t):
    """[B,C,H,W] channels_last -> [B*H*W, C] view."""
    B, C, H, W = t.shape
    return t.permute(0, 2, 3, 1).reshape(B * H * W, C)


def _bn_from_sums(sums, n, bn, weight, bias):
    """(scale, shift, mean, rstd) from epilogue column sums; updates the running buffers like nn.BatchNorm2d."""
    ss = _bn_prepare(bn, weight, bias, sums.shape[1], n, sums, sums.device, torch.cuda.current_stream(sums.device).cuda_stream)
    return ss[0], ss[1], ss[2], ss[3]


def _bn_eval_fold(bn, weight, bias):
    ss = _bn_prepare(bn, weight, bias, weight.shape[0], 1.0, None, weight.device,
                     torch.cuda.current_stream(weight.device).cuda_stream)
    return ss[0], ss[1], ss[2], ss[3]


class TcConv1x1Fn(Function):
    """y = act(BN(conv1x1([a1 ; a2]))) or conv1x1 + bias, on channels_last bf16 activations.

    a1 [B,K1,H,W], a2 [B,K2,H,W] or None (the concat-free embed.0 of models/cotnet.py:81,52), weight [N, K1+K2, 1, 1].
    bn = nn.BatchNorm2d or None (then `cbias` is the conv bias or None)."""

    @staticmethod
    def forward(ctx, a1, a2, weight, cbias, bn_w, bn_b, bn, relu, res=None, drop_scale=None):
        return TcConv1x1Fn._fwd(ctx, False, a1, a2, weight, cbias, bn_w, bn_b, bn, relu, res, drop_scale)

    @staticmethod
    def backward(ctx, *grads):
        return TcConv1x1Fn._bwd(ctx, grads)

    @staticmethod
    def _fwd(ctx, fork, a1, a2, weight, cbias, bn_w, bn_b, bn, relu, res, drop_scale=None):
        assert _is_cl(a1) and a1.dtype == torch.bfloat16 and (a2 is None or (_is_cl(a2) and a2.dtype == a1.dtype))
        if fork:
            ctx.set_materialize_grads(False)
        assert res is None or (bn is not None and _is_cl(res) and res.dtype == a1.dtype)
        assert drop_scale is None or bn is not None
        B, K1, H, W = a1.shape
        K2 = 0 if a2 is None else a2.shape[1]
        N = weight.shape[0]
        M = B * H * W
        lib, st, dt = _lib.load(), _lib.stream_ptr(a1), _lib.dtype_code(a1)
        a1, a2 = a1.detach(), (None if a2 is None else a2.detach())
        ds = _drop_scale(drop_scale, a1)
        wb = weight.detach().reshape(N, K1 + K2).to(torch.bfloat16).contiguous()
        b1, b2 = wb[:, :K1], (wb[:, K1:] if K2 else None)
        out = torch.empty((B, N, H, W), dtype=torch.bfloat16, device=a1.device, memory_format=torch.channels_last)
        out2d = _rows2d(out)
        pre = scale = mean = rstd = None
        batch = False
        if bn is None:
            _tc.gemm_bf16(a1, b1, a2, b2, shift=None if cbias is None else cbias.detach().float().contiguous(), relu=relu, out=out2d)
        elif bn.training or bn.running_mean is None:
            batch = True
            sums = _zeros((2, N,), a1.device)
            pre = torch.empty_like(out, memory_format=torch.channels_last)
            _tc.gemm_bf16(a1, b1, a2, b2, stats=(sums[0], sums[1]), out=_rows2d(pre))
            ss = _bn_apply_batch(pre, None if res is None else res.detach(), sums, bn, bn_w, bn_b, relu, out, lib, st, dt, ds)
            scale, shift, mean, rstd = ss[0], ss[1], ss[2], ss[3]
        else:
            scale, shift, mean, rstd = _bn_eval_fold(bn, bn_w, bn_b)
            if res is None and ds is None:
                _tc.gemm_bf16(a1, b1, a2, b2, scale=scale, shift=shift, relu=relu, out=out2d)
            else:       # eval mode with a residual: raw GEMM, then the fused scale/shift + residual + ReLU kernel
                pre = torch.empty_like(out, memory_format=torch.channels_last)
                _tc.gemm_bf16(a1, b1, a2, b2, out=_rows2d(pre))
                args = (dt, B, H * W, N, pre.data_ptr(), _lib.ptr(res), scale.data_ptr(), shift.data_ptr(), 1 if relu else 0,
                        out.data_ptr())
                if ds is None:
                    _lib.check(lib.cotb200_bn_apply(*args, st), "bn_apply")
                else:
                    _lib.check(lib.cotb200_bn_apply_ds(*args, ds.data_ptr(), st), "bn_apply_ds")
        need_bwd = any(ctx.needs_input_grad)
        if need_bwd and bn is not None and pre is None:      # eval-mode module under grad: BN backward needs the raw conv output
            pre = torch.empty_like(out, memory_format=torch.channels_last)
            _tc.gemm_bf16(a1, b1, a2, b2, out=_rows2d(pre))
        ctx.save_for_backward(a1, a2, wb, pre, out if relu else None, scale, mean, rstd, ds)
        ctx.cfg = (relu, batch, bn is not None, cbias is not None, weight.dtype, weight.shape,
                   None if bn_w is None else bn_w.dtype, None if cbias is None else cbias.dtype, K1, K2, res is not None)
        if fork:
            assert bn is not None, "fork needs the BatchNorm form (the sum of the two gradients happens in its backward kernels)"
            return out, out.detach()
        return out

    @staticmethod
    def _bwd(ctx, grads):
        a1, a2, wb, pre, y, scale, mean, rstd, ds = ctx.saved_tensors
        relu, batch, has_bn, has_bias, wdt, wshape, bndt, cbdt, K1, K2, has_res = ctx.cfg
        dy, dy2 = _two_grads(grads)
        if dy is None:
            return (None,) * 10
        B, N, H, W = dy.shape
        M = B * H * W
        lib, st, dt = _lib.load(), _lib.stream_ptr(dy), _lib.BF16
        dgamma = dbeta = dcb = dres = None
        if has_bn:
            sums = _zeros_esc((2, N,), dy.device)      # escapes as dgamma/dbeta
            if has_res and ctx.needs_input_grad[8]:
                dres = torch.empty_like(dy, memory_format=torch.channels_last)
            dpre = torch.empty_like(dy, memory_format=torch.channels_last)
            _bn_bwd(lib, dt, B, H * W, N, dy, dy2, pre, y, scale, None, mean, rstd, 1 if relu else 0, sums, batch, 1.0 / M, dpre, dres,
                    ds, st)
            dgamma, dbeta = sums[1].to(bndt), sums[0].to(bndt)
        else:
            dpre = dy if not relu else dy * (y > 0)
            if has_bias:
                dcb = _rows2d(dpre).float().sum(0).to(cbdt)
        d2 = _rows2d(dpre)
        da1 = da2 = None
        wt = wb.t().contiguous()                                  # [K1+K2, N]: B operand of the data-gradient GEMM
        if ctx.needs_input_grad[0]:
            da1 = torch.empty_like(a1, memory_format=torch.channels_last)
            _tc.gemm_bf16(dpre, wt[:K1], out=_rows2d(da1))
        if a2 is not None and ctx.needs_input_grad[1]:
            da2 = torch.empty_like(a2, memory_format=torch.channels_last)
            _tc.gemm_bf16(dpre, wt[K1:], out=_rows2d(da2))
        dw = None
        if ctx.needs_input_grad[2]:
            # weight gradient dW = dpre^T [a1 | a2] on the MN-major wgmma kernel (csrc/tc_wgrad.cu): the NHWC tiles are
            # consumed as they land, fp32 accumulation, one launch for both operand pairs
            if N * (K1 + K2) >= 1024 * 1024 or (N * (K1 + K2) >= 256 * 1024 and M >= 40000):
                # large, compute-shaped weight gradients (bottleneck convolutions of stages 3-4): the library kernel is faster
                # ; everything byte-heavy stays on the MN-major wgmma kernel
                parts = [torch.mm(d2.t(), _rows2d(a1))]
                if a2 is not None:
                    parts.append(torch.mm(d2.t(), _rows2d(a2)))
                dw = (parts[0] if a2 is None else torch.cat(parts, 1)).reshape(wshape).to(wdt)
            else:
                acc = _zeros((N, K1 + K2,), dy.device)
                _tc.wgrad_bf16(dpre, a1, a2, out=acc)
                dw = acc.reshape(wshape).to(wdt)
        return da1, da2, dw, dcb, dgamma, dbeta, None, None, dres, None


class TcConv1x1ForkFn(Function):
    """TcConv1x1Fn whose output comes as TWO aliases (one per consumer); their gradients are summed inside the BatchNorm backward
    kernels (_two_grads) instead of by an autograd add kernel."""

    @staticmethod
    def forward(ctx, a1, a2, weight, cbias, bn_w, bn_b, bn, relu, res=None, drop_scale=None):
        return TcConv1x1Fn._fwd(ctx, True, a1, a2, weight, cbias, bn_w, bn_b, bn, relu, res, drop_scale)

    @staticmethod
    def backward(ctx, *grads):
        return TcConv1x1Fn._bwd(ctx, grads)


class TcConv3x3Fn(Function):
    """k = ReLU(BN(conv3x3 grouped(x))) -- key_embed of models/cotnet.py:43-47 -- on channels_last bf16."""

    @staticmethod
    def forward(ctx, x, weight, bn_w, bn_b, bn, groups, relu):
        assert _is_cl(x) and x.dtype == torch.bfloat16
        B, C, H, W = x.shape
        M = B * H * W
        lib, st, dt = _lib.load(), _lib.stream_ptr(x), _lib.BF16
        x = x.detach()
        wp, bnt = _tc.prepare_conv3x3_weight(weight, groups)
        out = torch.empty_like(x, memory_format=torch.channels_last)
        pre = None
        batch = bn.training or bn.running_mean is None
        if batch:
            sums = _zeros((2, C,), x.device)
            pre = torch.empty_like(x, memory_format=torch.channels_last)
            _tc.conv3x3_bf16(x, wp, bnt, stats=(sums[0], sums[1]), out=pre)
            ss = _bn_apply_batch(pre, None, sums, bn, bn_w, bn_b, relu, out, lib, st, dt)
            scale, shift, mean, rstd = ss[0], ss[1], ss[2], ss[3]
        else:
            scale, shift, mean, rstd = _bn_eval_fold(bn, bn_w, bn_b)
            _tc.conv3x3_bf16(x, wp, bnt, scale=scale, shift=shift, relu=relu, out=out)
            if any(ctx.needs_input_grad):
                pre = _tc.conv3x3_bf16(x, wp, bnt)
        ctx.save_for_backward(x, weight.detach(), pre, out if relu else None, scale, mean, rstd)
        ctx.cfg = (relu, batch, groups, bn_w.dtype)
        return out

    @staticmethod
    def backward(ctx, dy):
        x, weight, pre, y, scale, mean, rstd = ctx.saved_tensors
        relu, batch, groups, bndt = ctx.cfg
        B, C, H, W = x.shape
        M = B * H * W
        lib, st, dt = _lib.load(), _lib.stream_ptr(x), _lib.BF16
        dy = dy.contiguous(memory_format=torch.channels_last)
        sums = _zeros_esc((2, C,), x.device)          # escapes as dgamma/dbeta
        _lib.check(lib.cotb200_bn_bwd_sums(dt, B, H * W, C, dy.data_ptr(), pre.data_ptr(), _lib.ptr(y), scale.data_ptr(),
                                           None, mean.data_ptr(), rstd.data_ptr(), 1 if relu else 0, sums[0].data_ptr(),
                                           sums[1].data_ptr(), st),
                   "bn_bwd_sums")
        dpre = torch.empty_like(dy, memory_format=torch.channels_last)
        _lib.check(lib.cotb200_bn_bwd_apply(dt, B, H * W, C, dy.data_ptr(), pre.data_ptr(), _lib.ptr(y), scale.data_ptr(),
                                            None, mean.data_ptr(), rstd.data_ptr(), _lib.ptr(sums[0]) if batch else None,
                                            _lib.ptr(sums[1]) if batch else None, 1.0 / M, 1 if relu else 0,
                                            dpre.data_ptr(), None, st), "bn_bwd_apply")
        dx = dw = None
        if ctx.needs_input_grad[0]:
            wpt, bnt = _tc.prepare_conv3x3_weight(weight, groups, transpose_for_dgrad=True)
            dx = _tc.conv3x3_bf16(dpre, wpt, bnt)
        if ctx.needs_input_grad[1]:
            # weight gradient: cuDNN grouped wgrad through torch (DESIGN.md section 6)
            dw = torch.nn.grad.conv2d_weight(x, weight.shape, dpre, stride=1, padding=1, dilation=1, groups=groups).to(weight.dtype)
        return dx, dw, sums[1].to(bndt), sums[0].to(bndt), None, None, None


class StemConvBNFn(Function):
    """act1(bn1(conv1(x))) of the trunk (models/resnet.py:552-554,601-603): 7x7 / stride 2 / pad 3, 3 -> N channels, on the 4-tap
    wgmma implicit GEMM (cotb200_stem7x7s2_bf16) with the BatchNorm statistics in its epilogue.  x: channels_last bf16.
    Backward: fused BatchNorm backward kernels; the weight gradient of the 3-channel convolution stays on cuDNN (the image
    needs no gradient)."""

    @staticmethod
    def forward(ctx, x, weight, bn_w, bn_b, bn, relu):
        B, _, H, W = x.shape
        N = weight.shape[0]
        lib, st, dt = _lib.load(), _lib.stream_ptr(x), _lib.BF16
        xd = x.detach()
        wm = _tc.prepare_stem_weight(weight)
        out = torch.empty((B, N, H // 2, W // 2), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
        pre = scale = mean = rstd = scratch = None
        batch = bn.training or bn.running_mean is None
        if batch:
            sums = _zeros((2, N,), x.device)
            pre = torch.empty_like(out, memory_format=torch.channels_last)
            r = _tc.stem7x7s2_bf16(xd, wm, stats=(sums[0], sums[1]), out=pre, return_scratch=True)
            if r is None:
                raise RuntimeError("cotb200 stem7x7s2: geometry not supported")
            scratch = r[1]
            ss = _bn_apply_batch(pre, None, sums, bn, bn_w, bn_b, relu, out, lib, st, dt)
            scale, shift, mean, rstd = ss[0], ss[1], ss[2], ss[3]
        else:
            scale, shift, mean, rstd = _bn_eval_fold(bn, bn_w, bn_b)
            if _tc.stem7x7s2_bf16(xd, wm, scale=scale, shift=shift, relu=relu, out=out) is None:
                raise RuntimeError("cotb200 stem7x7s2: geometry not supported")
            if any(ctx.needs_input_grad):
                pre = _tc.stem7x7s2_bf16(xd, wm)
        ctx.save_for_backward(xd, weight.detach(), pre, out if relu else None, scale, mean, rstd, scratch)
        ctx.cfg = (relu, batch, bn_w.dtype)
        return out

    @staticmethod
    def backward(ctx, dy):
        x, weight, pre, y, scale, mean, rstd, scratch = ctx.saved_tensors
        relu, batch, bndt = ctx.cfg
        B, N, Ho, Wo = dy.shape
        M = B * Ho * Wo
        lib, st, dt = _lib.load(), _lib.stream_ptr(dy), _lib.BF16
        dy = dy.contiguous(memory_format=torch.channels_last)
        sums = _zeros_esc((2, N,), dy.device)          # escapes as dgamma/dbeta
        _lib.check(lib.cotb200_bn_bwd_sums(dt, B, Ho * Wo, N, dy.data_ptr(), pre.data_ptr(), _lib.ptr(y), scale.data_ptr(),
                                           None, mean.data_ptr(), rstd.data_ptr(), 1 if relu else 0, sums[0].data_ptr(),
                                           sums[1].data_ptr(), st), "bn_bwd_sums")
        dpre = torch.empty_like(dy, memory_format=torch.channels_last)
        _lib.check(lib.cotb200_bn_bwd_apply(dt, B, Ho * Wo, N, dy.data_ptr(), pre.data_ptr(), _lib.ptr(y), scale.data_ptr(),
                                            None, mean.data_ptr(), rstd.data_ptr(), _lib.ptr(sums[0]) if batch else None,
                                            _lib.ptr(sums[1]) if batch else None, 1.0 / M, 1 if relu else 0,
                                            dpre.data_ptr(), None, st), "bn_bwd_apply")
        dx = dw = None
        wq = weight.to(dpre.dtype)
        if ctx.needs_input_grad[0]:
            dx = torch.nn.grad.conv2d_input(x.shape, wq, dpre, stride=2, padding=3)
        if ctx.needs_input_grad[1]:
            # weight gradient on the MN-major wgmma wgrad kernel over the space-to-depth image of the forward (one stage = one
            # output row, the four row taps as four B boxes); geometries it does not take: cuDNN
            if scratch is not None and stem_wgrad_tc:
                dw = _tc.stem7x7s2_wgrad(dpre, scratch, x.shape, N)
            if dw is None:
                dw = torch.nn.grad.conv2d_weight(x, weight.shape, dpre, stride=2, padding=3)
            dw = dw.to(weight.dtype)
        return dx, dw, sums[1].to(bndt), sums[0].to(bndt), None, None


#: the trunk's 7x7 stem convolution on the wgmma implicit GEMM (0 = cuDNN, the round-1 path)
stem_tc = _os.environ.get("COTB200_STEM_TC", "1") != "0"
stem_wgrad_tc = _os.environ.get("COTB200_STEM_WGRAD_TC", "1") != "0"


def stem_conv_bn(x, conv, bn, relu=True):
    """act(bn(conv(x))) for the 7x7/s2 stem.  wgmma path for channels_last bf16 3-channel images of even size (and an image
    row of at most 256 output pixels per tile segment); anything else: cuDNN + the fused BatchNorm kernels."""
    w = conv.weight
    if (stem_tc and x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.shape[1] == 3 and tuple(w.shape[1:]) == (3, 7, 7)
            and conv.stride == (2, 2) and conv.padding == (3, 3) and conv.dilation == (1, 1) and conv.bias is None
            and x.shape[2] % 2 == 0 and x.shape[3] % 2 == 0 and w.shape[0] % 8 == 0 and w.shape[0] <= 256
            and x.is_contiguous(memory_format=torch.channels_last)):
        return StemConvBNFn.apply(x, w, bn.weight, bn.bias, bn, relu)
    return bn_act(conv(x).contiguous(memory_format=torch.channels_last), bn, relu=relu)


#: which 1x1 convolutions of the ENCLOSING bottleneck (conv1 / conv3 / stride-1 downsample) run on the wgmma kernels in
#: training: "tc_all1x1" = all of them (forward with the BatchNorm statistics in the epilogue, data and weight gradients),
#: anything else = cuDNN + the fused BatchNorm kernels.  Same environment variable as CotLayer.train_conv_backend.
trunk_conv_backend = _os.environ.get("COTB200_TRAIN_CONV", "tc_all1x1+k").replace("+k", "")


#: the bottleneck convolutions of stages 3-4 (weights of 256K .. 1M elements, 12.5K-50K pixels) are compute-shaped
#: (K = 1024 / 2048) and stay on cuDNN; the wgmma path takes the byte-heavy stages 1-2
TC_TRUNK_MAX_WEIGHT = int(_os.environ.get("COTB200_TC_TRUNK_MAX_WEIGHT", str(128 * 1024)))


TC_MIN_PIXELS = int(_os.environ.get("COTB200_TC_MIN_PIXELS", "100000"))


def conv1x1_bn(x, conv, bn, relu, res=None, fork=False, drop_scale=None):
    """act(BN(conv1x1(x)) (+ res)) for the bottleneck's 1x1 convolutions (models/cotnet.py:229-235,249-262): on the wgmma
    GEMMs when the backend says so and the geometry allows (bf16 channels_last, stride 1, dense, no bias), else cuDNN + the
    fused BatchNorm kernels.  drop_scale: None or [B] stochastic-depth scales, act(drop_scale[b]*BN(conv1x1(x)) + res)
    (models/cotnet.py:256-262)."""
    w = conv.weight
    if (trunk_conv_backend == "tc_all1x1" and x.dtype == torch.bfloat16 and supported(x) and conv.kernel_size == (1, 1)
            and conv.stride == (1, 1) and conv.groups == 1 and conv.bias is None and w.shape[0] % 8 == 0 and w.shape[1] % 8 == 0
            and w.shape[0] * w.shape[1] <= TC_TRUNK_MAX_WEIGHT and x.shape[0] * x.shape[2] * x.shape[3] >= TC_MIN_PIXELS
            and (torch.is_grad_enabled() or not bn.training)):
        if drop_scale is None:
            return (TcConv1x1ForkFn if fork else TcConv1x1Fn).apply(x, None, w, None, bn.weight, bn.bias, bn, relu, res)
        return (TcConv1x1ForkFn if fork else TcConv1x1Fn).apply(x, None, w, None, bn.weight, bn.bias, bn, relu, res, drop_scale)
    return bn_act(conv(x).contiguous(memory_format=torch.channels_last), bn, relu=relu, res=res, fork=fork, drop_scale=drop_scale)


def tc_supported(x, dim):
    return (x.is_cuda and x.dtype == torch.bfloat16 and _is_cl(x) and not x.is_contiguous() and dim % 64 == 0
            and _tc.conv_tile(dim, 4) is not None and x.shape[3] <= 128)
