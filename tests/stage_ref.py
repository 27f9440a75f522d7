"""Stage-by-stage references of the bf16 training step: a recorder of the autograd functions in cotnet_b200/fused.py and
cotnet_b200/dropblock.py, fp64 restatements of each stage from the inputs that stage actually received, error bounds derived
from the fp32 accumulation chains, and a Python mirror of the dispatch predicates that pick the wgmma functions.

Comparing each stage with fp64 of its own recorded inputs keeps bf16 rounding from cascading through batch-statistics BatchNorms,
so the bounds are as tight as the kernel tests': 1/2 bf16 ulp of the stored value plus the fp32 error of the stage.

Rounding model.  u = 2^-24.  A sequential fp32 sum of n terms (chain length n) is within gamma(n) * sum|terms| of the exact sum,
gamma(n) = n*u / (1 - n*u), when every add rounds to nearest.  Tensor-core accumulation aligns a k-group's products and truncates,
so the wgmma and cuDNN convolution chains use gamma_tc(n), the same bound with 2u per add.  Every order of summation of n terms has a chain of at most n, so n = number of terms is a valid
bound wherever a kernel's order is not pinned here; the wgmma weight gradients pin theirs (wgrad_chain) because a bound over all
M pixels would let a bf16-rounded weight gradient (relative error 2^-9) pass.
"""
import os

import torch

U32 = 2.0 ** -24
#: abs error of the 16-bit tensors' sigmoid, 0.5 + 0.5*tanh.approx(z/2) (csrc/norm_tail.cu sigmoid_t): tanh.approx.f32 is within
#: 2^-10.99 absolute, halved by the 0.5 factor, plus the fma; 2^-11 bounds it
SIGMOID_ERR_16 = 2.0 ** -11
#: fp32 tensors: __fdividef(1, 1 + __expf(-z)): a few ulp of 1
SIGMOID_ERR_32 = 2.0 ** -20
#: __expf(x) is within (2 + floor(|1.173 * x|)) ulp of e^x: CUDA C++ Programming Guide (12.x), appendix "Mathematical Functions",
#: table "Single-Precision Floating-Point Intrinsic Functions".  Results below the normal range are flushed to zero (ex2.approx.ftz).
EXPF_ULP_BASE, EXPF_ULP_SLOPE = 2.0, 1.173
#: rsqrtf (torch.rsqrt of an fp32 CUDA tensor) is within 2 ulp: the same guide, table "Single-Precision Mathematical Functions"
RSQRTF_ULP = 2.0

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ rounding and bounds
def round_mant(x, bits):
    """Round-to-nearest-even of fp64 values to `bits` significand bits (8 = bfloat16, 24 = float32); normal range only."""
    x = x.double()
    m, e = torch.frexp(x)                                 # x = m * 2^e, 0.5 <= |m| < 1
    r = torch.round(torch.ldexp(m, torch.full_like(e, bits)))      # torch.round: half to even; exact in fp64 for bits <= 52
    return torch.ldexp(r, e - bits)


def bf16(x):
    return round_mant(x, 8)


def f32(x):
    return round_mant(x, 24)


def ulp(x, bits):
    """unit in the last place at |x| for a `bits`-bit significand (fp64 tensor; zero maps to the smallest normal's ulp)"""
    e = torch.frexp(x.double().abs().clamp_min(2.0 ** -126))[1]
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - bits)


def gamma(n):
    """Higham's gamma_n for fp32: the relative bound of an n-term sequential sum, in units of sum|terms|"""
    nu = n * U32
    assert nu < 1.0
    return nu / (1.0 - nu)


def gamma_tc(n):
    """gamma_n with 2u per add: the tensor-core accumulations (wgmma GEMMs, convolutions, weight gradients) align the products of a
    k-group to the largest exponent and truncate, so one add may cost up to one fp32 ulp instead of half of one"""
    nu = 2 * n * U32
    assert nu < 1.0
    return nu / (1.0 - nu)


def gamma_bf16(n):
    """gamma_n for bf16 adds (u = 2^-8): autograd sums the gradients of a tensor with several consumers in its dtype"""
    nu = n * 2.0 ** -8
    assert nu < 1.0
    return nu / (1.0 - nu)


def store_bound(exact, err, dtype):
    """|stored - exact| bound of a value computed in fp32 within `err` of `exact` and stored as `dtype` (round to nearest)"""
    if dtype == torch.float32:
        return err + 0.5 * ulp(exact.abs() + err, 24)
    if dtype == torch.bfloat16:
        return err + 0.5 * ulp(exact.abs() + err, 8)
    raise ValueError(dtype)


def epilogue_ref(acc, scale, shift, relu):
    """The wgmma epilogue on an exact fp64 accumulator: fmaf(acc, scale, shift) (one fp32 rounding; scale None = 1, shift None =
    0), ReLU, then the bf16 store.  Exact whenever acc * scale + shift is exact in fp64 (small-integer acc, fp32 scale / shift)."""
    z = acc.double()
    if scale is not None:
        z = z * scale.double()
    if shift is not None:
        z = z + shift.double()
    z = f32(z)
    return bf16(z.clamp_min(0.0) if relu else z)


def expf_rel_err(x):
    """relative error bound of __expf at fp64 arguments x (EXPF_ULP_*; an ulp of a normal fp32 result is at most 2^-23 of it)"""
    return (EXPF_ULP_BASE + torch.floor(EXPF_ULP_SLOPE * x.abs())) * 2.0 ** -23


def softmax2_fast_ref(z, e):
    """cotb200_se_eval's radix-2 softmax on logits z [..., 2] (fp64, each within e of the fp32 logits the kernel holds):
    m = max(u, v), eu = __expf(u - m), ev = __expf(v - m), a = e_r * (1 / (eu + ev)).  Returns (softmax(z), bound).

    Relative errors d0, d1 of eu, ev move a_r by a_r * a_(1-r) * (d0 + d1) to first order.  Each d_r is __expf's own error plus
    that of its argument: u - m rounds once (not exact when u and m differ in sign or scale), an absolute u|u - m| that moves the
    exponential by the same relative amount.  The sum, the IEEE division and the product round three times (3u of a_r); a flushed
    __expf result (an argument below -87) leaves a_r < 2^-125.  A logit error moves a_r by at most (e_u + e_v) / 4 (the softmax's
    derivative, a0 * a1 <= 1/4), which also bounds the shift of the arguments."""
    a = torch.softmax(z.double(), -1)
    es = e.double().sum(-1, keepdim=True)
    d = z.double() - z.double().max(-1, keepdim=True)[0]
    arg = d.abs() + es
    dexp = (expf_rel_err(arg) + U32 * arg).sum(-1, keepdim=True)
    ap = a + 0.25 * es
    return a, 0.25 * es + ap * (ap.flip(-1) * dexp + 3 * U32) * 1.01 + 2.0 ** -125


def fold_bound(bn):
    """fp64 eval-mode BatchNorm fold of the module's running statistics and a bound of each fp32 result, for the three forms the
    library uses (CotLayer._tc_params and fused._se_eval_params: torch ops; _bn_eval_fold: bn_finalize):
      rstd  = rsqrt(fl(var + eps)): RSQRTF_ULP ulp (an ulp is at most 2u of the result), plus u/2 from the add and u/2 from eps as fp32
      scale = fl(gamma * rstd): one more u
      shift = fl(beta - fl(mean * scale)) (or one fma): |mean * scale| * (rel(scale) + u) + u |shift|
    First order, with a 1% margin for the products of the small relative errors.  Returns dict of values and absolute bounds."""
    rv, rm = bn.running_var.detach().double(), bn.running_mean.detach().double()
    g = bn.weight.detach().double() if bn.weight is not None else torch.ones_like(rv)
    b = bn.bias.detach().double() if bn.bias is not None else torch.zeros_like(rv)
    rstd = 1.0 / torch.sqrt(rv + bn.eps)
    rel_r = 2 * RSQRTF_ULP * U32 + U32
    rel_s = rel_r + U32
    scale = g * rstd
    shift = b - rm * scale
    return dict(rstd=rstd, rstd_err=1.01 * rel_r * rstd, scale=scale, scale_err=1.01 * rel_s * scale.abs(), shift=shift,
                shift_err=1.01 * ((rel_s + U32) * (rm * scale).abs() + U32 * shift.abs()))


def within(got, exact, bound, what):
    """assert |got - exact| <= bound elementwise; returns the fraction of elements that differ from the correctly rounded exact
    value (for a bf16 `got`: the one-ulp differences)"""
    g = got.detach().double()
    exact = exact.double().to(g.device)
    bound = torch.as_tensor(bound, dtype=torch.float64, device=g.device).expand_as(exact)
    err = (g - exact).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError("%s: %d of %d beyond the bound, e.g. got %r want %r bound %r (max err/bound %.3g)" % (
            what, int(bad.sum()), g.numel(), g.flatten()[i].item(), exact.flatten()[i].item(), bound.flatten()[i].item(),
            (err / bound.clamp_min(1e-300)).max().item()))
    if got.dtype == torch.bfloat16:
        return float((g != bf16(exact)).double().mean()) if g.numel() else 0.0
    return 0.0


def equal(got, want, what):
    if not torch.equal(got, want):
        d = (got.double() - want.double()).abs()
        raise AssertionError("%s: %d of %d elements differ (max %g), dtypes %s/%s" % (
            what, int((d != 0).sum()), got.numel(), d.max().item(), got.dtype, want.dtype))


# ------------------------------------------------------------------------------------------------ dispatch mirror
#: The source lines the predicates below restate (tests/test_stage_grads_cpu.py pins them: editing one fails a CPU test).
SOURCE_ANCHORS = {
    "cotnet_b200/fused.py": [
        "if N * (K1 + K2) >= 1024 * 1024 or (N * (K1 + K2) >= 256 * 1024 and M >= 40000):",
        "and conv.stride == (1, 1) and conv.groups == 1 and conv.bias is None and w.shape[0] % 8 == 0 and w.shape[1] % 8 == 0",
        "and w.shape[0] * w.shape[1] <= TC_TRUNK_MAX_WEIGHT and x.shape[0] * x.shape[2] * x.shape[3] >= TC_MIN_PIXELS",
        "return (x.is_cuda and x.dtype == torch.bfloat16 and _is_cl(x) and not x.is_contiguous() and dim % 64 == 0",
        "and _tc.conv_tile(dim, 4) is not None and x.shape[3] <= 128)",
        "and x.shape[2] % 2 == 0 and x.shape[3] % 2 == 0 and w.shape[0] % 8 == 0 and w.shape[0] <= 256",
        "TC_MIN_PIXELS = 100000",
        "TC_KEY_MAX_DIM = 128",
        "TC_TRUNK_MAX_WEIGHT = 128 * 1024",
        "rcode = 0 if not relu else (3 if mask is not None else (2 if (BN_MASK and res is None and row) else 1))",
        "return 8 if (wc // fold) % 8 == 0 else 0",
        # the eval dispatch (eval_* generators below)
        "if (not torch.is_grad_enabled() and not bn.training and not se[1].training and k is not None and se[1].running_mean is not None",
        "and bn.running_mean is not None and isinstance(se[2], torch.nn.ReLU)):",
        "if not (torch.is_grad_enabled() and x.requires_grad):\n        return (x,) * n",
        "row = not epilogue or res is not None or ds is not None",
        "produce(out, scale=ss[0], shift=ss[1], relu=relu)",
        "and (torch.is_grad_enabled() or not bn.training)):",
        "r = _tc.stem7x7s2_bf16(xd, wm, stats=stats, out=dst, return_scratch=True, **epi)",
    ],
    "cotnet_b200/cot_layer.py": [
        "big = B * H * W >= fused.TC_MIN_PIXELS",
        "if big and self.dim <= fused.TC_KEY_MAX_DIM and tc_ok and self.key_embed[0].weight.dtype == x.dtype:",
        "if tc_ok and big:",
        "if x.dtype == torch.bfloat16 and C % 16 == 0 and k.dtype == x.dtype and w0.dtype == x.dtype:",
        "k = fused.bn_act(F.conv2d(xk, wkey, None, 1, self.kernel_size // 2).contiguous(memory_format=cl), self.key_embed[1], relu=True)",
        "v = fused.bn_act(F.conv2d(xv, _dense_from_grouped(cv[0].weight, G)).contiguous(memory_format=cl), cv[1], relu=False)",
        "gc = fused.tap_chunk(C // 8, self.dw_group)",
        "return (not self.training and not torch.is_grad_enabled() and x.dtype == torch.bfloat16 and self.kernel_size == 3",
        "and self.dim % 64 == 0 and tc.conv_tile(self.dim, 4) is not None and x.shape[3] <= 128)",
        "if self._tc_eval_ok(x):\n                return self._forward_tc_eval(x)\n            return self._forward_fused(x)",
        "if ks == 3 and fused.supported(x):\n            return self._forward_fused(x)",
        "w = fused.group_norm9(l.view(B, H, W, J).permute(0, 3, 1, 2), self.embed[4], gc)",
    ],
    "cotnet_b200/backbone.py": [
        "y = dropblock.drop_block(y, key, self.drop_block_sites[0], self.drop_block)",
        "if key is not None:\n            z = fused.conv1x1_bn(y.contiguous(memory_format=cl), self.conv3, self.bn3, relu=False)",
        "x = fused.max_pool3x3s2(fused.stem_conv_bn(x, self.conv1, self.bn1, relu=True))",
    ],
    "cotnet_b200/backbone_hybrid.py": [
        "if self.radix == 1 and self.cardinality == 1 and fused.supported(x) and drop_block is None:",
        "if drop_block is not None and fused.supported(x):",
        "if (width in conv_dim) or (width == c4_dim and block_idx not in c4_idx):",
        "if stride > 1 and avd:",
        "if self.avd is not None and self.avd_first:",
        "if self.avd is not None and not self.avd_first:",
        "return dict(radix=1, conv_dim={64, 128}, c4_dim=256, c4_idx=set(range(0, n_l3, 2)), **kw)",
        "stride = 2 if b == 0 else 1",
        "x = fused.bn_act(c[6](x).contiguous(memory_format=cl), self.bn1, relu=True)",
        # the stride-2 pool of conv2 (HYBRID: which trunk pools how, and where)
        "return nn.AvgPool2d(3, s, padding=1) if aa_layer is None else aa_layer(channels=width, stride=s)",
        "self.avd = pool(stride)\n                stride = 1",
        "if stride > 1:\n                self.avd = pool(stride)",
        "if isinstance(self.avd, nn.AvgPool2d) and self.avd.kernel_size == 3 and self.avd.stride == 2 and fused.supported(y):",
        "return F.pad(x, (1, 1, 1, 1), mode=\"reflect\")",
        "return F.conv2d(_ReflectPad1.apply(x), self._filt.to(x.dtype), stride=self.stride, groups=x.shape[1])",
        "c = torch.tensor([0.25, 0.5, 0.25])",
        "return CoTHybridNet([3, 4, 6, 3], stem_width=32, block_args=_args(6, avd=False, avd_first=True), **kw)",
        "return CoTHybridNet([3, 8, 36, 3], stem_width=64, aa_layer=BlurPool2d, block_args=_args(36, avd=True, avd_first=False), **kw)",
        "return se_cotnetd_152(**kw)",
    ],
    "cotnet_b200/tc.py": [
        "for bn in (64, 128, 192, 256):",
        "if C % bn == 0 and (bn % cg == 0):",
        "if a2 is not None and K1 % 64:",
    ],
    "cotnet_b200/csrc/tc_wgrad.cu": [
        "p.tiles_c = (cc64 + 255) / 256;",
        "p.tiles_r = (R + WG_BR - 1) / WG_BR;",
        "int splits = (num_sms() + tiles - 1) / tiles;",
        "const int max_splits = (p.kb_total + 3) / 4;",
        "const int per = (p.kb_total + splits - 1) / splits;",
        "splits = (p.kb_total + per - 1) / per;",
        "int splits = num_sms();",
        "if (splits > p.kb_total) splits = p.kb_total;",
        "for (int s = 0; s < splits; ++s) t += __ldg(part + (size_t)s * n + i);",
        "if ((H & 1) || (W & 1) || (Wh & 15) || Wh > 128 || (N & 7) || N > 128 || (reinterpret_cast<uintptr_t>(dWm) & 15)) {",
    ],
}

TC_MIN_PIXELS = 100000
TC_KEY_MAX_DIM = 128
TC_TRUNK_MAX_WEIGHT = 128 * 1024


def mm_wgrad(N, K, M):
    """TcConv1x1Fn takes its weight gradient from torch.mm (bf16 result) instead of the wgmma kernel (fp32)"""
    return N * K >= 1024 * 1024 or (N * K >= 256 * 1024 and M >= 40000)


def conv_tile(C, groups):
    cg = C // groups
    for bn in (64, 128, 192, 256):
        if C % bn == 0 and bn % cg == 0:
            return bn
    return None


def tc_supported(dim, W):
    """fused.tc_supported for a bf16 channels_last input of width W"""
    return dim % 64 == 0 and conv_tile(dim, 4) is not None and W <= 128


def conv1x1_tc(cin, cout, M, stride=1, min_pixels=TC_MIN_PIXELS):
    """fused.conv1x1_bn on a bf16 channels_last input with a bias-free dense 1x1 convolution, under grad"""
    return stride == 1 and cout % 8 == 0 and cin % 8 == 0 and cin * cout <= TC_TRUNK_MAX_WEIGHT and M >= min_pixels


def cot_dispatch(B, dim, H, W, min_pixels=TC_MIN_PIXELS):
    """CotLayer._forward_fused on bf16: (key conv on wgmma, embed.0 on wgmma, embed.3 and conv1x1 on wgmma)"""
    tc_ok = tc_supported(dim, W)
    big = B * H * W >= min_pixels
    return big and dim <= TC_KEY_MAX_DIM and tc_ok, tc_ok, tc_ok and big


def stem_tc(H, W, N):
    return H % 2 == 0 and W % 2 == 0 and N % 8 == 0 and N <= 256


def stem_wgrad_tc(H, W, N):
    """the stem's weight gradient runs on the wgmma kernel (else cuDNN, bf16 result)"""
    Wh = W // 2
    return H % 2 == 0 and W % 2 == 0 and Wh % 16 == 0 and Wh <= 128 and N % 8 == 0 and N <= 128


def _wgrad_launch_chain(M, R, Cc, sms):
    cc64 = (Cc + 63) // 64 * 64
    tiles_c = (cc64 + 255) // 256
    tiles_r = (R + 127) // 128
    kb = (M + 63) // 64
    tiles = tiles_r * tiles_c
    splits = max(1, min((sms + tiles - 1) // tiles, (kb + 3) // 4))
    per = (kb + splits - 1) // splits
    splits = (kb + per - 1) // per
    return per * 64 + splits + 1          # pixels of one split in the accumulator, the split-order reduction, the add to OUT


def wgrad_chain(M, N, K1, K2, sms):
    """Longest fp32 chain of one dW element of tc.wgrad_bf16 (csrc/tc_wgrad.cu): a split's pixels, then the partials in split order.
    Both orientations and the two-launch form are bounded (the larger chain is taken)."""
    cands = [_wgrad_launch_chain(M, N, K1 + K2, sms), _wgrad_launch_chain(M, K1 + K2, N, sms)]
    if K2:
        cands += [_wgrad_launch_chain(M, N, K1, sms), _wgrad_launch_chain(M, K1, N, sms),
                  _wgrad_launch_chain(M, N, K2, sms), _wgrad_launch_chain(M, K2, N, sms)]
    return max(cands)


def stem_wgrad_chain(B, Ho, Wo, sms):
    """tc_stem_wgrad: one pipeline stage = one output row (Wo pixels); splits = min(SMs, rows)"""
    kb = B * Ho
    splits = min(sms, kb)
    per = (kb + splits - 1) // splits
    splits = (kb + per - 1) // per
    return per * Wo + splits + 1


# ------------------------------------------------------------------------------------------------ the recorder
FUSED_FNS = ("BNActFn", "GroupNorm9Fn", "FanOutFn", "CotTailFn", "AggTapFn", "Pool3x3S2Fn", "TcConv1x1Fn", "TcConv3x3Fn",
             "StemConvBNFn")
DROPBLOCK_FNS = ("DropBlockFn", "DropBlockResReluFn")
TRAINER_FNS = ("SoftTargetCrossEntropyFn",)


def _snap(v):
    if isinstance(v, torch.Tensor):
        return v.detach().clone()
    if isinstance(v, (tuple, list)):
        return type(v)(_snap(t) for t in v)
    return v


class Call:
    """One autograd function application: args (the objects passed), inp (tensor snapshots), out, saved (ctx tensors at the end of
    the forward), gin (incoming gradients), gout (returned gradients), apply / bwd (captured _bn_apply_batch / _bn_bwd), extra."""

    def __init__(self, name, args):
        self.name = name
        self.args = args
        self.inp = tuple(_snap(a) for a in args)
        self.out = self.saved = self.gin = self.gout = None
        self.apply = self.bwd = None
        self.extra = {}

    def __repr__(self):
        return "Call(%s)" % self.name


class Recorder:
    """Swaps every fused autograd function for a subclass that calls the parent and records it; wraps _bn_apply_batch and _bn_bwd
    to capture `pre` / `dpre` and the BatchNorm statistics of the wgmma functions.  Changes no bit and no launch."""

    def __init__(self, monkeypatch, keep_outputs=False):
        from cotnet_b200 import dropblock, fused, trainer
        self.calls = []
        self._stack = []
        # keep_outputs: hold every recorded output, so that no later tensor reuses its storage (under no_grad nothing else holds
        # them, and the dataflow checks match producers by storage)
        self.kept = [] if keep_outputs else None
        for mod, names in ((fused, FUSED_FNS), (dropblock, DROPBLOCK_FNS), (trainer, TRAINER_FNS)):
            for n in names:
                monkeypatch.setattr(mod, n, self._subclass(getattr(mod, n)))
        apply0, bwd0 = fused._bn_apply_batch, fused._bn_bwd
        rec = self

        def bn_apply_batch(x, res, sums, bn, weight, bias, relu, y, lib, st, dt, ds=None, mask=None):
            cap = dict(x=_snap(x), res=_snap(res), sums=_snap(sums), weight=_snap(weight), bias=_snap(bias), relu=relu, ds=_snap(ds),
                       eps=bn.eps, rm0=_snap(bn.running_mean), rv0=_snap(bn.running_var), n=x.shape[0] * x.shape[2] * x.shape[3])
            ss = apply0(x, res, sums, bn, weight, bias, relu, y, lib, st, dt, ds, mask)
            cap.update(y=_snap(y), ss=_snap(ss), mask=_snap(mask), rm1=_snap(bn.running_mean), rv1=_snap(bn.running_var),
                       momentum=bn.momentum, nbt=None if bn.num_batches_tracked is None else int(bn.num_batches_tracked))
            rec._stack[-1].apply = cap
            return ss

        def bn_bwd(lib, dt, B, HW, C, dy, x, y, scale, shift, mean, rstd, rcode, sums, batch, inv_n, dx, dres, ds, st):
            cap = dict(dy=_snap(dy), x=_snap(x), y=_snap(y), scale=_snap(scale), shift=_snap(shift), mean=_snap(mean), rstd=_snap(rstd),
                       rcode=rcode, batch=batch, inv_n=inv_n, ds=_snap(ds), B=B, HW=HW, C=C)
            bwd0(lib, dt, B, HW, C, dy, x, y, scale, shift, mean, rstd, rcode, sums, batch, inv_n, dx, dres, ds, st)
            cap.update(sums=_snap(sums), dx=_snap(dx), dres=_snap(dres))
            rec._stack[-1].bwd = cap
        monkeypatch.setattr(fused, "_bn_apply_batch", bn_apply_batch)
        monkeypatch.setattr(fused, "_bn_bwd", bn_bwd)
        # where each DropBlock mask came from: the key, site and DropBlock the caller passed (the DropBlock calls carry them)
        self._masks = {}
        device_mask0 = dropblock.device_mask

        def device_mask(x, key, site, spec):
            mask, count = device_mask0(x, key, site, spec)
            rec._masks[mask.data_ptr()] = dict(key=_snap(key), site=site, spec=spec)
            return mask, count
        monkeypatch.setattr(dropblock, "device_mask", device_mask)

    def _subclass(self, cls):
        rec = self

        class Rec(cls):
            @staticmethod
            def forward(ctx, *args):
                call = Call(cls.__name__, args)
                rec.calls.append(call)
                rec._stack.append(call)
                try:
                    out = cls.forward(ctx, *args)
                finally:
                    rec._stack.pop()
                call.out = _snap(out)
                call.out_ptr = tuple(o.data_ptr() for o in (out if isinstance(out, tuple) else (out,)))
                if rec.kept is not None:
                    rec.kept.append(out)
                call.saved = _snap(tuple(getattr(ctx, "to_save", ()) or ()))
                if cls.__name__ == "CotTailFn":
                    call.extra["p"] = _snap(ctx.graph[0])
                    call.extra["training"] = ctx.training
                if cls.__name__ in DROPBLOCK_FNS:
                    call.extra.update(rec._masks[args[1 if cls.__name__ == "DropBlockFn" else 2].data_ptr()])
                ctx._stage_call = call
                return out

            @staticmethod
            def backward(ctx, *grads):
                call = ctx._stage_call
                call.gin = _snap(grads)
                rec._stack.append(call)
                grad0 = torch.autograd.grad
                if cls.__name__ == "CotTailFn":         # the MLP's backward inside: its incoming S and its fp32 results

                    def grad(outputs, inputs, grad_outputs=None, **kw):
                        res = grad0(outputs, inputs, grad_outputs=grad_outputs, **kw)
                        call.extra["S"], call.extra["mlp_grads"] = _snap(grad_outputs), _snap(res)
                        return res
                    torch.autograd.grad = grad
                try:
                    gout = cls.backward(ctx, *grads)
                finally:
                    torch.autograd.grad = grad0
                    rec._stack.pop()
                call.gout = _snap(gout)
                return gout

        Rec.__name__ = Rec.__qualname__ = cls.__name__
        return Rec

    def named(self, name):
        return [c for c in self.calls if c.name == name]


# ------------------------------------------------------------------------------------------------ fp64 restatements
def bn_stats_ref(x, n):
    """fp64 column sums (sum x, sum x^2) of a channels_last [B,C,H,W] tensor and their sum|terms| for the bound"""
    x = x.double()
    s0 = x.sum((0, 2, 3))
    s1 = (x * x).sum((0, 2, 3))
    return s0, s1, x.abs().sum((0, 2, 3))


def bn_apply_ref(x, scale, shift, relu, res=None, ds=None):
    """y = act(ds[b] * (x*scale + shift) (+ res)) in fp64 from the captured fp32 scale / shift; returns (y, fp32 error bound)"""
    x = x.double()
    sc, sh = scale.double().view(1, -1, 1, 1), shift.double().view(1, -1, 1, 1)
    z = x * sc + sh
    mag = (x * sc).abs() + sh.abs()
    if ds is not None:
        d = ds.double().view(-1, 1, 1, 1)
        z, mag = z * d, mag * d.abs()
    if res is not None:
        z = z + res.double()
        mag = mag + res.double().abs()
    return (torch.relu(z) if relu else z), 4 * U32 * mag


def bn_bwd_ref(dy, x, gate, scale, mean, rstd, sums_got, batch, ds=None):
    """BatchNorm backward of y = act(ds*(x*scale+shift) + res) in fp64, with the ReLU decision `gate` (bool, from the library's y)
    and the captured fp32 statistics.  Returns dict(dres, s0, s1, s_abs, dx, dx_err): dres = dy*gate (exact), s0 / s1 the dbeta /
    dgamma column sums with their sum|terms| bound inputs, dx from the captured fp32 sums `sums_got` (the stage's own inputs)."""
    dy = dy.double()
    g = dy * gate.double() if gate is not None else dy
    dz = g * (ds.double().view(-1, 1, 1, 1) if ds is not None else 1.0)
    m, r, sc = mean.double().view(1, -1, 1, 1), rstd.double().view(1, -1, 1, 1), scale.double().view(1, -1, 1, 1)
    x = x.double()
    xh = (x - m) * r
    xh_err = 4 * U32 * (x.abs() + m.abs()) * r                 # the kernels may form xhat as x*rstd - mean*rstd
    out = dict(dres=g, s0=dz.sum((0, 2, 3)), s1=(dz * xh).sum((0, 2, 3)), s0_abs=dz.abs().sum((0, 2, 3)),
               s1_abs=(dz.abs() * (xh.abs() + xh_err)).sum((0, 2, 3)) + (dz.abs() * xh_err).sum((0, 2, 3)))
    if batch:
        n = x.shape[0] * x.shape[2] * x.shape[3]
        c0, c1 = sums_got[0].double().view(1, -1, 1, 1) / n, sums_got[1].double().view(1, -1, 1, 1) / n
        out["dx"] = sc * (dz - c0 - xh * c1)
        out["dx_err"] = 8 * U32 * sc.abs() * (dz.abs() + c0.abs() + (xh.abs() + 1) * c1.abs()) + sc.abs() * c1.abs() * xh_err
    else:
        out["dx"] = sc * dz
        out["dx_err"] = 2 * U32 * (sc * dz).abs()
    return out


def gemm_ref(a_list, w_list):
    """sum_i a_i @ w_i^T over NHWC rows, fp64, and sum|terms| ; a_i [B,K,H,W] channels_last, w_i [N,K]"""
    acc = mag = None
    for a, w in zip(a_list, w_list):
        a2 = a.double().permute(0, 2, 3, 1).reshape(-1, a.shape[1])
        w2 = w.double()
        t, tm = a2 @ w2.t(), a2.abs() @ w2.abs().t()
        acc, mag = (t, tm) if acc is None else (acc + t, mag + tm)
    B, _, H, W = a_list[0].shape
    N = w_list[0].shape[0]
    shp = lambda t: t.view(B, H, W, N).permute(0, 3, 1, 2)        # noqa: E731
    return shp(acc), shp(mag)


def rows(t):
    return t.double().permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def gn9_ref(l, lb, gam, beta, mean, rstd, gc, eps):
    """GroupNorm9Fn forward in fp64 from the recorded logits and the captured fp32 statistics: (out in storage order, bound,
    xhat in reference order, fp64 mean / rstd of the logits and their bounds)"""
    B, J, H, W = l.shape
    wc = J // 9
    x = (l.double() + (0 if lb is None else lb.double().view(1, -1, 1, 1))).contiguous()
    xg = x.view(B, wc, 9 * H * W)
    n = 9 * H * W
    m64 = xg.mean(2)
    v64 = ((xg - m64.unsqueeze(2)) ** 2).mean(2)
    m, r = mean.double().view(B, wc, 1), rstd.double().view(B, wc, 1)
    xh = ((xg - m) * r).view(B, J, H, W)
    gm, bt = gam.double().view(1, -1, 1, 1), beta.double().view(1, -1, 1, 1)
    out = xh * gm + bt
    # the kernels (csrc/gn72.cu) apply fmaf(l, a, beta - (mean - lbias) * a) with a = rstd * gamma: the roundings scale with |l|,
    # |lbias| and |mean| separately, not with |l + lbias| (which cancels when lbias ~ -l)
    xa = l.double().abs() + (0 if lb is None else lb.double().abs().view(1, -1, 1, 1))
    err = 8 * U32 * ((xa.contiguous().view(B, wc, -1) + m.abs()) * r).view(B, J, H, W) * gm.abs() + 4 * U32 * bt.abs()
    # statistics: sums of n terms (gamma(n)); var = E[x^2] - mean^2 in fp32
    ax = x.abs().view(B, wc, -1)
    m_err = gamma(n + 1) * ax.mean(2) + 2 * U32 * (lb.double().abs().max() if lb is not None else 0) + U32 * m64.abs()
    e2 = (xg * xg).mean(2)
    v_err = gamma(n + 1) * e2 * 2 + 2 * m64.abs() * m_err + 4 * U32 * (e2 + m64 * m64)
    r64 = 1.0 / torch.sqrt(v64 + eps)
    r_err = 0.5 * r64 * v_err / (v64 + eps) * 1.01 + 4 * ulp(r64, 24)
    return to_storage(out, gc), to_storage(err, gc), xh, (m64, m_err, r64, r_err)


def to_storage(t, gc):
    """reference channel order (g*9+t) -> tap-major chunks of gc (COTB200_NHWC_TAP), [B, J, H, W]"""
    if gc == 0:
        return t
    B, J, H, W = t.shape
    wc = J // 9
    return t.reshape(B, wc // gc, gc, 9, H, W).permute(0, 1, 3, 2, 4, 5).reshape(B, J, H, W)


def from_storage(t, gc):
    if gc == 0:
        return t
    B, J, H, W = t.shape
    wc = J // 9
    return t.reshape(B, wc // gc, 9, gc, H, W).permute(0, 1, 3, 2, 4, 5).reshape(B, J, H, W)


def gn9_bwd_ref(dg_ref_order, xh, gam, rstd, n_group):
    """GroupNorm backward in fp64 (reference order): dl, its fp32 error, dgamma, dbeta, dlbias and their sum|terms|"""
    B, J, H, W = dg_ref_order.shape
    wc = J // 9
    dg = dg_ref_order.double().contiguous()
    gd = dg * gam.double().view(1, -1, 1, 1)
    g3, x3 = gd.reshape(B, wc, -1), xh.reshape(B, wc, -1)
    m1 = g3.mean(2, keepdim=True)
    m2 = (g3 * x3).mean(2, keepdim=True)
    r = rstd.double().view(B, wc, 1)
    dl = (r * (g3 - m1 - x3 * m2)).view(B, J, H, W)
    e_m1 = gamma(n_group + 1) * g3.abs().mean(2, keepdim=True)
    e_m2 = gamma(n_group + 1) * (g3 * x3).abs().mean(2, keepdim=True) * 2
    dl_err = (r * (8 * U32 * (g3.abs() + m1.abs() + (x3.abs() + 1) * m2.abs()) + e_m1 + x3.abs() * e_m2)).view(B, J, H, W)
    return dict(dl=dl, dl_err=dl_err, dgamma=(dg * xh).sum((0, 2, 3)), dbeta=dg.sum((0, 2, 3)), dlbias=dl.sum((0, 2, 3)),
                dgamma_abs=(dg.abs() * (xh.abs() + 1e-30)).sum((0, 2, 3)), dbeta_abs=dg.abs().sum((0, 2, 3)),
                dlbias_abs=dl.abs().sum((0, 2, 3)), dlbias_err=dl_err.sum((0, 2, 3)))


def _mlp_fwd(p, mods, kind, training, se_eval=False):
    """fp64 forward of the tail MLP with a first-order bound of each fp32 intermediate (dict of values and errors).
    se_eval: the inference kernel cotb200_se_eval instead of the fp32 PyTorch MLP (see mlp_ref)."""
    c0, b1, c3 = mods
    F = torch.nn.functional
    B, C = p.shape
    w0, bb0 = c0.weight.detach().double().flatten(1), (c0.bias.detach().double() if c0.bias is not None else 0.0)
    w3, bb3 = c3.weight.detach().double().flatten(1), (c3.bias.detach().double() if c3.bias is not None else 0.0)
    p = p.detach().double()
    z1 = p @ w0.t() + bb0
    # the kernel forms its operand psum * inv_hw in fp32: one more rounding in the chain
    e1 = gamma(w0.shape[1] + (2 if se_eval else 1)) * (p.abs() @ w0.abs().t() + (bb0.abs() if torch.is_tensor(bb0) else 0.0))
    g1, be1 = b1.weight.detach().double(), b1.bias.detach().double()
    if se_eval:
        # fmaf(fl(acc + b0), s1, t1) with the fold of fused._se_eval_params (fold_bound): the chain's error, u of the add, the
        # fold's errors of s1 (times |z1|) and t1, then u of the fma
        assert not training and kind == "cot"
        fb = fold_bound(b1)
        s1 = fb["scale"]
        z2 = z1 * s1 + fb["shift"]
        e2 = s1.abs() * (e1 + U32 * z1.abs()) + fb["scale_err"] * z1.abs() + fb["shift_err"] + U32 * z2.abs()
        h, eh = torch.relu(z2), e2
        z3 = h @ w3.t() + bb3
        e3 = eh @ w3.abs().t() + gamma(w3.shape[1] + 1) * (h.abs() @ w3.abs().t() + (bb3.abs() if torch.is_tensor(bb3) else 0.0))
        a, ea = softmax2_fast_ref(z3.view(B, C, 2), e3.view(B, C, 2))
        return dict(p=p, z1=z1, e1=e1, z2=z2, e2=e2, h=h, eh=eh, a=a, ea=ea)
    if training:
        mu = z1.mean(0, keepdim=True)
        sd = torch.sqrt(z1.var(0, unbiased=False, keepdim=True) + b1.eps)
        zh = (z1 - mu) / sd
        e_sd = 2 * e1.max(0, keepdim=True)[0] + 4 * U32 * sd       # any perturbation of the B values moves sd by at most its max
        e_h = (2 * e1.max(0, keepdim=True)[0] / sd) * (1 + zh.abs()) + 16 * U32 * (zh.abs() + 1)
    else:
        sd = torch.sqrt(b1.running_var.double() + b1.eps)
        zh = (z1 - b1.running_mean.double()) / sd
        e_sd = 4 * U32 * sd
        e_h = e1 / sd + 16 * U32 * (zh.abs() + 1)
    z2 = zh * g1 + be1
    e2 = e_h * g1.abs() + 4 * U32 * (z2.abs() + be1.abs())
    if kind == "cot":
        h, eh = torch.relu(z2), e2
    else:
        h, eh = F.silu(z2), 1.1 * e2 + 4 * U32 * z2.abs()
    z3 = h @ w3.t() + bb3
    e3 = eh @ w3.abs().t() + gamma(w3.shape[1] + 1) * (h.abs() @ w3.abs().t() + (bb3.abs() if torch.is_tensor(bb3) else 0.0))
    if kind == "cot":
        z3, e3 = z3.view(B, C, 2), e3.view(B, C, 2)
        a = torch.softmax(z3, 2)
        ea = (0.25 * (e3[..., :1] + e3[..., 1:]) + 8 * U32).expand_as(a)
    else:
        g = torch.sigmoid(z3)
        a = torch.stack([g, torch.zeros_like(g)], 2)
        ea = torch.stack([0.25 * e3 + 8 * U32, torch.zeros_like(e3)], 2)
    return dict(p=p, w0=w0, w3=w3, z1=z1, e1=e1, g1=g1, sd=sd, e_sd=e_sd, zh=zh, e_h=e_h, z2=z2, e2=e2, h=h, eh=eh, a=a, ea=ea)


def mlp_ref(p, mods, kind, training, se_eval=False):
    """the CoT `se` MLP (+ radix-2 softmax) or the split-attention gate MLP (+ sigmoid) in fp64 on the pooled mean p [B, C], and a
    first-order bound of the fp32 result.  mods: (conv0, bn, conv3).  The default bounds the fp32 PyTorch MLP (a correctly rounded
    exp); se_eval=True bounds cotb200_se_eval instead: the BatchNorm folded into the fc1 epilogue and the __expf softmax
    (softmax2_fast_ref), with p = psum * inv_hw as the kernel's fp32 operands give it."""
    f = _mlp_fwd(p, mods, kind, training, se_eval)
    return f["a"], f["ea"]


def mlp_bwd_ref(p, S, mods, kind, training):
    """The tail MLP's backward in fp64 for the incoming gradient S [B, C, 2] (d/da) at the pooled mean p: (dp, [dW0, db0, dgamma1,
    dbeta1, dW3, db3]) and a first-order bound of each, from the fp32 forward intermediates' bounds (_mlp_fwd) and the rounding of
    every backward op (gamma(n) for an n-term sum).  A ReLU whose input lies within its bound of zero may take either branch."""
    f = _mlp_fwd(p, mods, kind, training)
    U = U32
    B, C = f["p"].shape
    a, ea, S = f["a"], f["ea"], S.double()
    if kind == "cot":                       # softmax backward: a * (S - sum(a*S))
        aS = (a * S).sum(2, keepdim=True)
        dz3 = a * (S - aS)
        aSa = (a * S).abs().sum(2, keepdim=True)
        e_dz3 = ea * (S.abs() + aSa) + a.abs() * (ea * S.abs()).sum(2, keepdim=True) + 4 * U * a.abs() * (S.abs() + aSa)
        dz3, e_dz3 = dz3.reshape(B, 2 * C), e_dz3.reshape(B, 2 * C)
    else:                                   # sigmoid backward on the gate; the stacked zeros take no gradient
        g, eg, S0 = a[..., 0], ea[..., 0], S[..., 0]
        dz3 = S0 * g * (1 - g)
        e_dz3 = S0.abs() * eg * (1 + eg) + 4 * U * dz3.abs()
    h, eh, w3 = f["h"], f["eh"], f["w3"]
    dW3 = dz3.t() @ h
    e_dW3 = e_dz3.t() @ h.abs() + dz3.abs().t() @ eh + gamma(B + 1) * (dz3.abs().t() @ h.abs())
    db3, e_db3 = dz3.sum(0), e_dz3.sum(0) + gamma(B + 1) * dz3.abs().sum(0)
    dh = dz3 @ w3
    e_dh = e_dz3 @ w3.abs() + gamma(w3.shape[0] + 1) * (dz3.abs() @ w3.abs())
    z2, e2 = f["z2"], f["e2"]
    if kind == "cot":
        dz2 = dh * (z2 > 0)
        e_dz2 = e_dh * (z2 > 0) + dh.abs() * (z2.abs() <= e2)
    else:
        sg = torch.sigmoid(z2)
        dz2 = dh * sg * (1 + z2 * (1 - sg))
        e_dz2 = 1.1 * e_dh + 0.5 * dh.abs() * e2 + 4 * U * dz2.abs()
    zh, e_h, g1, sd, e_sd = f["zh"], f["e_h"], f["g1"], f["sd"], f["e_sd"]
    dg1 = (dz2 * zh).sum(0)
    e_dg1 = (e_dz2 * zh.abs() + dz2.abs() * e_h).sum(0) + gamma(B + 1) * (dz2 * zh).abs().sum(0)
    db1, e_db1 = dz2.sum(0), e_dz2.sum(0) + gamma(B + 1) * dz2.abs().sum(0)
    dzh = dz2 * g1
    e_dzh = e_dz2 * g1.abs() + U * dzh.abs()
    if training:
        m1, m2 = dzh.mean(0, keepdim=True), (dzh * zh).mean(0, keepdim=True)
        dz1 = (dzh - m1 - zh * m2) / sd
        e_dz1 = ((e_dzh + e_dzh.mean(0, keepdim=True) + zh.abs() * (e_dzh * zh.abs() + dzh.abs() * e_h).mean(0, keepdim=True)
                  + e_h * m2.abs() + gamma(B + 1) * (dzh.abs().mean(0, keepdim=True) + zh.abs() * (dzh * zh).abs().mean(0, keepdim=True)))
                 / sd + dz1.abs() * e_sd / sd + 8 * U * (dzh.abs() + m1.abs() + (zh * m2).abs()) / sd)
    else:
        dz1 = dzh / sd
        e_dz1 = e_dzh / sd + dz1.abs() * e_sd / sd + 4 * U * dz1.abs()
    pp, w0 = f["p"], f["w0"]
    dW0 = dz1.t() @ pp
    e_dW0 = e_dz1.t() @ pp.abs() + gamma(B + 1) * (dz1.abs().t() @ pp.abs())
    db0, e_db0 = dz1.sum(0), e_dz1.sum(0) + gamma(B + 1) * dz1.abs().sum(0)
    dp = dz1 @ w0
    e_dp = e_dz1 @ w0.abs() + gamma(w0.shape[0] + 1) * (dz1.abs() @ w0.abs())
    return (dp, e_dp), [(dW0, e_dW0), (db0, e_db0), (dg1, e_dg1), (db1, e_db1), (dW3, e_dW3), (db3, e_db3)]


def tail_bwd_ref(u, k, scale, shift, mean, rstd, a_c, dout, dpn, training, sig_err):
    """CotTailFn's backward in fp64 from the recorded u, k, fp32 scale / shift / mean / rstd, attention weights a_c, incoming dout
    and the MLP's fp32 d/dp (dpn).  Returns dict of S (the per-sample sums the MLP backward takes), dbeta / dgamma, du, dk, each
    with its bound.  Pooling p = mean(y + k) sends dpn / HW to every pixel of both y and k."""
    U = U32
    B, C, H, W = u.shape
    HW, M = H * W, B * H * W
    sc, sh = scale.double().view(1, -1, 1, 1), shift.double().view(1, -1, 1, 1)
    uu, do = u.double(), dout.double()
    z = uu * sc + sh
    ze = 4 * U * ((uu * sc).abs() + sh.abs())
    sg = torch.sigmoid(z)
    y = z * sg
    ye = z.abs() * sig_err + 1.1 * ze + 4 * U * y.abs()
    out = {}
    out["S0"] = (do * y).sum((2, 3))
    out["S0_err"] = (do.abs() * ye).sum((2, 3)) + gamma(HW + 1) * (do * y).abs().sum((2, 3))
    if k is not None:
        kk = k.double()
        out["S1"] = (do * kk).sum((2, 3))
        out["S1_err"] = gamma(HW + 1) * (do * kk).abs().sum((2, 3))
    a0, a1 = a_c[..., 0].double().view(B, C, 1, 1), a_c[..., 1].double().view(B, C, 1, 1)
    dpp = dpn.double().view(B, C, 1, 1) / HW
    dyt = do * a0 + dpp
    ds = sg * (1 + z * (1 - sg))                                    # silu'
    dz = dyt * ds
    e_dz = dyt.abs() * (sig_err * (1 + z.abs()) + 0.5 * ze + 8 * U * ds.abs()) + 4 * U * (do * a0).abs() + 4 * U * dpp.abs()
    m, r = mean.double().view(1, -1, 1, 1), rstd.double().view(1, -1, 1, 1)
    xh = (uu - m) * r
    xh_err = 4 * U * (uu.abs() + m.abs()) * r
    out["dbeta"] = dz.sum((0, 2, 3))
    out["dbeta_err"] = e_dz.sum((0, 2, 3)) + gamma(M + 1) * dz.abs().sum((0, 2, 3))
    out["dgamma"] = (dz * xh).sum((0, 2, 3))
    out["dgamma_err"] = (e_dz * (xh.abs() + xh_err) + dz.abs() * xh_err).sum((0, 2, 3)) + gamma(M + 1) * (dz * xh).abs().sum((0, 2, 3))
    if training:
        c0, c1 = out["dbeta"].view(1, -1, 1, 1) / M, out["dgamma"].view(1, -1, 1, 1) / M
        e0, e1 = out["dbeta_err"].view(1, -1, 1, 1) / M, out["dgamma_err"].view(1, -1, 1, 1) / M
        out["du"] = sc * (dz - c0 - xh * c1)
        out["du_err"] = sc.abs() * (e_dz + e0 + (xh.abs() + xh_err) * e1 + xh_err * c1.abs()
                                    + 8 * U * (dz.abs() + c0.abs() + (xh.abs() + 1) * c1.abs()))
    else:
        out["du"] = sc * dz
        out["du_err"] = sc.abs() * e_dz + 2 * U * (sc * dz).abs()
    if k is not None:
        out["dk"] = do * a1 + dpp
        out["dk_err"] = 4 * U * ((do * a1).abs() + dpp.abs())
    return out


def dense_from_grouped_adjoint(g, groups):
    """adjoint of cot_layer._dense_from_grouped: the gradient [N, K, ...] of the block-diagonal dense weight -> the gradient of
    the grouped weight [N, K/groups, ...], the diagonal blocks gathered (a gather: exact in any dtype)"""
    if groups == 1:
        return g
    N, K = g.shape[0], g.shape[1]
    ng, kg, rest = N // groups, K // groups, tuple(g.shape[2:])
    idx = torch.arange(groups, device=g.device)
    return g.reshape((groups, ng, groups, kg) + rest)[idx, :, idx].reshape((N, kg) + rest)


def coxt_embed0_adjoint(gx, gk, groups):
    """adjoint of cot_layer._coxt_embed0_dense: the gradients of the dense operand-pair weights (Wx, Wk) [N, C] -> the gradient
    of the grouped embed.0 weight [N, 2C/groups, 1, 1], whose input channels interleave x and k (x0, k0, x1, k1, ...)"""
    N, C = gx.shape[0], gx.shape[1]
    ng, ch = N // groups, C // groups
    idx = torch.arange(groups, device=gx.device)
    bx = gx.reshape(groups, ng, groups, ch)[idx, :, idx]
    bk = gk.reshape(groups, ng, groups, ch)[idx, :, idx]
    return torch.stack([bx, bk], 3).reshape(N, 2 * ch, 1, 1)


class DerivedRecorder:
    """Wraps cot_layer._dense_from_grouped / _coxt_embed0_dense, recording only: which parameter each dense weight came from.
    of[id(parameter)] = [dict(kind="grouped", groups, dense) | dict(kind="embed0", groups, wx, wk)]"""

    def __init__(self, monkeypatch):
        from cotnet_b200 import cot_layer
        self.of = {}
        dfg0, e00 = cot_layer._dense_from_grouped, cot_layer._coxt_embed0_dense

        def dense_from_grouped(w, groups):
            out = dfg0(w, groups)
            if groups != 1:
                self.of.setdefault(id(w), []).append(dict(kind="grouped", groups=groups, dense=out))
            return out

        def coxt_embed0_dense(w, groups):
            wx, wk = e00(w, groups)
            self.of.setdefault(id(w), []).append(dict(kind="embed0", groups=groups, wx=wx, wk=wk))
            return wx, wk
        monkeypatch.setattr(cot_layer, "_dense_from_grouped", dense_from_grouped)
        monkeypatch.setattr(cot_layer, "_coxt_embed0_dense", coxt_embed0_dense)


def tail_pool_ref(u, k, scale, shift, sig_err):
    """cotb200_tail_pool in fp64 from the recorded u, k and fp32 scale / shift: psum[b, c] = sum over the pixels of silu(u*scale +
    shift) + k, with its bound (the fma, the sigmoid's sig_err, any order of the HW-term sum); also y and its bound for the combine"""
    sc, sh = scale.double().view(1, -1, 1, 1), shift.double().view(1, -1, 1, 1)
    z = u.double() * sc + sh
    ze = 4 * U32 * ((u.double() * sc).abs() + sh.abs())
    y = torch.nn.functional.silu(z)
    ye = z.abs() * sig_err + 1.1 * ze + 4 * U32 * y.abs()
    t = y + k.double()
    HW = u.shape[2] * u.shape[3]
    return t.sum((2, 3)), ye.sum((2, 3)) + gamma(HW + 1) * t.abs().sum((2, 3)), y, ye


def tail_combine_ref(y, ye, k, a):
    """cotb200_tail_combine in fp64: out = a0 * y + a1 * k from the recorded a, and the fp32 bound (before the storage rounding)"""
    B, C = a.shape[0], a.shape[1]
    a0, a1 = a[..., 0].double().view(B, C, 1, 1), a[..., 1].double().view(B, C, 1, 1)
    o = a0 * y + a1 * k.double()
    return o, a0.abs() * ye + 4 * U32 * (o.abs() + (a1 * k.double()).abs())


def agg_ref(v, w, fold, gc):
    """AggTapFn forward in fp64: out[b,c,p] = sum_t v[b,c,p+off_t] * w[b, wch(c), t, p] with zero padding; and sum|terms|"""
    B, C, H, W = v.shape
    J = w.shape[1]
    wc = J // 9
    wr = from_storage(w.double(), gc).view(B, wc, 9, H, W)
    cf = C // fold
    wcf = wc // fold
    c = torch.arange(C, device=v.device)
    wch = (c // cf) * wcf + (c % cf) % wcf
    vu = torch.nn.functional.unfold(v.double(), 3, padding=1).view(B, C, 9, H, W)
    wt = wr[:, wch]
    return (vu * wt).sum(2), (vu.abs() * wt.abs()).sum(2)


# ------------------------------------------------------------------------------------------------ expected call lists
_STAGE1_CUDNN = ["BNActFn(relu)", "FanOutFn(3)", "BNActFn(relu)", "FanOutFn(2)", "TcConv1x1Fn(two,relu)", "BNActFn(plain)",
                 "GroupNorm9Fn(gc8+lbias)", "AggTapFn(fold1,gc8)", "CotTailFn(k)", "BNActFn(plain)", "BNActFn(relu+res)"]
_STAGE1_TC = ["TcConv1x1Fn(one,relu)", "FanOutFn(3)", "TcConv3x3Fn", "FanOutFn(2)", "TcConv1x1Fn(two,relu)", "TcConv1x1Fn(one,nobn)",
              "TcConv1x1Fn(one,bn)", "GroupNorm9Fn(gc8+lbias)", "AggTapFn(fold1,gc8)", "CotTailFn(k)", "TcConv1x1Fn(one,bn)",
              "TcConv1x1Fn(one,relu+res)"]
_STAGE4 = [c for c in _STAGE1_CUDNN[:9]] + ["BNActFn(relu+res)"]
#: Dataflow between recorded calls, "consumer.argument<-producer.output" (x: the block input).  Inputs that come out of a torch
#: convolution in the glue (cuDNN conv1 / key conv / embed.3 / conv1x1 / downsample / conv3) have no recorded producer.
_FLOW_STAGE1_CUDNN = ["1.0<-0.0", "3.0<-2.0", "4.0<-1.1", "4.1<-3.0", "7.0<-5.0", "7.1<-6.0", "8.0<-7.0", "8.1<-3.1", "10.3<-9.0"]
_FLOW_STAGE1_TC = ["0.0<-x", "1.0<-0.0", "2.0<-1.0", "3.0<-2.0", "4.0<-1.1", "4.1<-3.0", "5.0<-4.0", "6.0<-1.2", "7.0<-5.0", "8.0<-6.0",
                   "8.1<-7.0", "9.0<-8.0", "9.1<-3.1", "10.0<-x", "11.0<-9.0", "11.8<-10.0"]
#: CoT bottlenecks of cotnet50 (bf16 weights and activations, channels_last, training): geometry, the recorded forward calls and
#: their dataflow
BLOCK_CASES = {
    # the real bench dispatch at the default threshold: B*H*W = 100352 pixels, every 1x1 conv and the key conv on wgmma
    "stage1_b32": dict(model="cotnet50", block="layer1.0", B=32, cin=64, cout=256, H=56, stride=1, min_pixels=None, calls=_STAGE1_TC,
                       flow=_FLOW_STAGE1_TC),
    # 6272 pixels: only embed.0 on wgmma
    "stage1_b2": dict(model="cotnet50", block="layer1.0", B=2, cin=64, cout=256, H=56, stride=1, min_pixels=None, calls=_STAGE1_CUDNN,
                      flow=_FLOW_STAGE1_CUDNN),
    # the golden tests' threshold 0 at the same size
    "stage1_b2_all_wgmma": dict(model="cotnet50", block="layer1.0", B=2, cin=64, cout=256, H=56, stride=1, min_pixels=0,
                                calls=_STAGE1_TC, flow=_FLOW_STAGE1_TC),
    # the stride-2 first block of stage 2: avd average pool, stride-2 downsample on cuDNN
    "stage2_first_b2": dict(model="cotnet50", block="layer2.0", B=2, cin=256, cout=512, H=28, stride=2, min_pixels=None,
                            calls=["BNActFn(relu)", "Pool3x3S2Fn(avg)"] + _STAGE1_CUDNN[1:],
                            flow=["1.0<-0.0", "2.0<-1.0", "4.0<-3.0", "5.0<-2.1", "5.1<-4.0", "8.0<-6.0", "8.1<-7.0", "9.0<-8.0", "9.1<-4.1",
                                  "11.3<-10.0"]),
    # a stage-4 block: key conv (dim 512) and every trunk convolution on cuDNN, the residual is the block input
    "stage4_b2": dict(model="cotnet50", block="layer4.1", B=2, cin=2048, cout=2048, H=7, stride=1, min_pixels=None, calls=_STAGE4,
                      flow=_FLOW_STAGE1_CUDNN[:-1] + ["9.3<-x"]),
}


def tap_chunk(wc, fold=1):
    return 8 if (wc // fold) % 8 == 0 else 0


def cot_calls(B, dim, H, min_pixels=TC_MIN_PIXELS):
    """the forward calls of CotLayer._forward_fused on a bf16 channels_last input (bf16 weights)"""
    key_tc, e0_tc, rest_tc = cot_dispatch(B, dim, H, H, min_pixels)
    out = ["FanOutFn(3)", "TcConv3x3Fn" if key_tc else "BNActFn(relu)", "FanOutFn(2)",
           "TcConv1x1Fn(two,relu)" if e0_tc else "BNActFn(relu)"]
    out += ["TcConv1x1Fn(one,nobn)", "TcConv1x1Fn(one,bn)"] if rest_tc else ["BNActFn(plain)"]
    gc = tap_chunk(dim // 8)
    return out + ["GroupNorm9Fn(gc%d+lbias)" % gc, "AggTapFn(fold1,gc%d)" % gc, "CotTailFn(k)"]


def coxt_calls(dim):
    """the forward calls of CoXtLayer._forward_fused on bf16: the dense key conv on cuDNN, embed.0 on the wgmma GEMM when
    C % 16 == 0, embed.3 and conv1x1 on cuDNN, the fold-2 GroupNorm and LocalConv"""
    gc = tap_chunk(dim // 8, 2)
    return ["FanOutFn(3)", "BNActFn(relu)", "FanOutFn(2)", "TcConv1x1Fn(two,relu)" if dim % 16 == 0 else "BNActFn(relu)",
            "BNActFn(plain)", "GroupNorm9Fn(gc%d+lbias)" % gc, "AggTapFn(fold2,gc%d)" % gc, "CotTailFn(k)"]


def _tail_calls(B, width, cout, Ho, min_pixels, drop_block, ds):
    """conv3 + bn3 (+ DropBlock) (+ drop path) + residual + ReLU"""
    tc = conv1x1_tc(width, cout, B * Ho * Ho, 1, min_pixels)
    if drop_block:
        return ["TcConv1x1Fn(one,bn)" if tc else "BNActFn(plain)", "DropBlockResReluFn"]
    return ["TcConv1x1Fn(one,relu+res%s)" % ("+ds" if ds else "") if tc else "BNActFn(relu+res%s)" % ("+ds" if ds else "")]


def bottleneck_calls(B, cin, width, cout, H, stride, min_pixels=TC_MIN_PIXELS, coxt=False, drop_block=False, ds=False):
    """the forward calls of backbone.Bottleneck._forward_fused with a CotLayer (or a CoXtLayer), from the dispatch predicates
    above; drop_block: a DropBlock key reaches the block (sites bn1 and bn3); ds: a drop_scale reaches it"""
    M = B * H * H
    Ho = H // stride
    out = ["TcConv1x1Fn(one,relu)" if conv1x1_tc(cin, width, M, 1, min_pixels) else "BNActFn(relu)"]
    if drop_block:
        out.append("DropBlockFn")
    if stride > 1:
        out.append("Pool3x3S2Fn(avg)")
    out += coxt_calls(width) if coxt else cot_calls(B, width, Ho, min_pixels)
    if stride > 1 or cin != cout:
        out.append("TcConv1x1Fn(one,bn)" if conv1x1_tc(cin, cout, B * Ho * Ho, stride, min_pixels) else "BNActFn(plain)")
    return out + _tail_calls(B, width, cout, Ho, min_pixels, drop_block, ds)


#: The SE-CoTNetD trunks (backbone_hybrid.se_cotnetd_*): blocks per stage, deep-stem width, the pool of a stride-2 conv2 (the
#: 3x3/s2 average pool on Pool3x3S2Fn, or BlurPool2d: F.pad reflect + a depthwise [1,2,1]x[1,2,1]/16 torch convolution, so no
#: recorded call), avd (a split-attention conv2 runs at stride 1 and pools), avd_first (the pool before conv2, else after it),
#: c4_idx (the stage-3 blocks whose conv2 is a CoT layer: the even ones)
HYBRID = {
    "se_cotnetd_50": dict(layers=(3, 4, 6, 3), stem_width=32, blur=False, avd=False, avd_first=True, c4_idx=tuple(range(0, 6, 2))),
    "se_cotnetd_152": dict(layers=(3, 8, 36, 3), stem_width=64, blur=True, avd=True, avd_first=False,
                           c4_idx=tuple(range(0, 36, 2))),
}
#: the model name each trunk's block configuration is registered under (se_cotnetd_152_L is se_cotnetd_152 at 320)
HYBRID["se_cotnetd_152_L"] = HYBRID["se_cotnetd_152"]


def hybrid_split(width, block_idx, conv_dim=(64, 128), c4_dim=256, c4_idx=HYBRID["se_cotnetd_50"]["c4_idx"]):
    """backbone_hybrid.CoTBottleneck: conv2 is a SplitAttnConv2d (else the CoT layer); se_cotnetd_50's block arguments unless
    c4_idx says otherwise"""
    return width in conv_dim or (width == c4_dim and block_idx not in c4_idx)


def hybrid_block_calls(B, block_idx, cin, width, H, stride, min_pixels=TC_MIN_PIXELS, drop_block=False, ds=False,
                       model="se_cotnetd_50"):
    """the forward calls of backbone_hybrid.CoTBottleneck.forward on a bf16 channels_last input: a split-attention conv2 runs
    the cuDNN 3x3 convolution (stride 2 itself unless avd) and the fused gate tail, or with DropBlock bn0 on BNActFn, the
    DropBlock and the rest of the gate in torch; a CoT conv2 pools at stride 2, before it (avd_first) at the output size or
    after it at the input size; a BlurPool is torch glue; the avg_down downsample pools in torch before its 1x1 convolution"""
    cfg = HYBRID[model]
    cout = 4 * width
    Ho = conv_out(H, stride)
    split = hybrid_split(width, block_idx, c4_idx=cfg["c4_idx"])
    pool = stride > 1 and (cfg["avd"] if split else True)
    avd_first, pool_call = cfg["avd_first"], [] if cfg["blur"] else ["Pool3x3S2Fn(avg)"]
    out = ["TcConv1x1Fn(one,relu)" if conv1x1_tc(cin, width, B * H * H, 1, min_pixels) else "BNActFn(relu)"]
    if drop_block:
        out.append("DropBlockFn")
    if pool and avd_first:
        out += pool_call
    if split:
        out += ["BNActFn(plain)", "DropBlockFn"] if drop_block else ["CotTailFn(gate)"]
    else:
        out += cot_calls(B, width, Ho if pool and avd_first else H, min_pixels)
    if pool and not avd_first:
        out += pool_call
    if block_idx == 0:
        out.append("TcConv1x1Fn(one,bn)" if conv1x1_tc(cin, cout, B * Ho * Ho, 1, min_pixels) else "BNActFn(plain)")
    return out + _tail_calls(B, width, cout, Ho, min_pixels, drop_block, ds)


def stem_calls(model, H, W):
    """the stems: cotnet50's 7x7/s2 StemConvBNFn (wgmma for even sizes) + the max pool; the deep stem's three cuDNN 3x3
    convolutions, each followed by a BatchNorm + ReLU"""
    if model in HYBRID:
        return ["BNActFn(relu)"] * 3
    return ["StemConvBNFn" if stem_tc(H, W, 64) else "BNActFn(relu)", "Pool3x3S2Fn(max)"]


def case_calls(c):
    """the call list of a STEP_BLOCK_CASES entry, from the generators"""
    mp = TC_MIN_PIXELS if c.get("min_pixels") is None else c["min_pixels"]
    if c["kind"] == "stem":
        return stem_calls(c["model"], c["H"], c["W"])
    db, ds = bool(c.get("sites")), c.get("ds") is not None
    if c["model"] in HYBRID:
        return hybrid_block_calls(c["B"], int(c["block"].split(".")[1]), c["cin"], c["width"], c["H"], c["stride"], mp, db, ds,
                                  c["model"])
    return bottleneck_calls(c["B"], c["cin"], c["width"], c["cout"], c["H"], c["stride"], mp, c["model"] != "cotnet50", db, ds)


#: Blocks beyond the cotnet50 CoT bottlenecks: CoXt, SE-CoTNetD (split attention, avg_down, c4_idx), stochastic depth, DropBlock
#: and the two stems.  ds: the drop_scale handed to the block (1.25 = 1/keep at keep 0.8, exact in bf16); sites: the DropBlock
#: site numbers the block must use in its model (stages 1-2 have none; cotnet50's layer3.0 takes 0 and 1, se_cotnetd_50's
#: layer3.0 (CoT) 0 and 1, its layer3.1 (split attention: bn1, conv2.bn0, bn3) 2, 3 and 4).  flow: as BLOCK_CASES, plus "c<j>":
#: the input of the j-th torch convolution of the block (cuDNN glue: conv1 / downsample / conv3 off the wgmma path, the key conv,
#: embed.3, conv1x1, the split-attention 3x3 and its gate's fc1 / fc2) where it is a recorded call's output or x.
_DS = (0.0, 1.25)
_COXT = ["FanOutFn(3)", "BNActFn(relu)", "FanOutFn(2)", "TcConv1x1Fn(two,relu)", "BNActFn(plain)"]
_COT_E0 = ["FanOutFn(3)", "BNActFn(relu)", "FanOutFn(2)", "TcConv1x1Fn(two,relu)", "BNActFn(plain)", "GroupNorm9Fn(gc8+lbias)",
           "AggTapFn(fold1,gc8)", "CotTailFn(k)"]
STEP_BLOCK_CASES = {
    "coxt_stage1_b2": dict(model="cotnext50_2x48d", kind="block", block="layer1.0", B=2, cin=64, width=96, cout=256, H=56, stride=1,
        calls=["BNActFn(relu)"] + _COXT + ["GroupNorm9Fn(gc0+lbias)", "AggTapFn(fold2,gc0)", "CotTailFn(k)", "BNActFn(plain)", "BNActFn(relu+res)"],
        flow=['1.0<-0.0', '10.3<-9.0', '3.0<-2.0', '4.0<-1.2', '4.1<-3.1', '7.0<-5.0', '7.1<-6.0', '8.0<-7.0', '8.1<-3.1', 'c0<-x', 'c1<-1.2', 'c2<-4.0', 'c3<-1.2', 'c4<-x', 'c5<-8.0']),
    "coxt_stage1_b2_all_wgmma": dict(model="cotnext50_2x48d", kind="block", block="layer1.0", B=2, cin=64, width=96, cout=256, H=56,
                                     stride=1, min_pixels=0,
        calls=["TcConv1x1Fn(one,relu)"] + _COXT + ["GroupNorm9Fn(gc0+lbias)", "AggTapFn(fold2,gc0)", "CotTailFn(k)", "TcConv1x1Fn(one,bn)", "TcConv1x1Fn(one,relu+res)"],
        flow=['0.0<-x', '1.0<-0.0', '10.0<-8.0', '10.8<-9.0', '3.0<-2.0', '4.0<-1.2', '4.1<-3.1', '7.0<-5.0', '7.1<-6.0', '8.0<-7.0', '8.1<-3.1', '9.0<-x', 'c0<-1.2', 'c1<-4.0', 'c2<-1.2']),
    "coxt_stage2_first_b2": dict(model="cotnext50_2x48d", kind="block", block="layer2.0", B=2, cin=256, width=192, cout=512, H=28,
                                 stride=2,
        calls=["BNActFn(relu)", "Pool3x3S2Fn(avg)"] + _COXT + ["GroupNorm9Fn(gc0+lbias)", "AggTapFn(fold2,gc0)", "CotTailFn(k)", "BNActFn(plain)", "BNActFn(relu+res)"],
        flow=['1.0<-0.0', '11.3<-10.0', '2.0<-1.0', '4.0<-3.0', '5.0<-2.2', '5.1<-4.1', '8.0<-6.0', '8.1<-7.0', '9.0<-8.0', '9.1<-4.1', 'c0<-x', 'c1<-2.2', 'c2<-5.0', 'c3<-2.2', 'c4<-x', 'c5<-9.0']),
    "coxt_stage4_b2": dict(model="cotnext50_2x48d", kind="block", block="layer4.1", B=2, cin=2048, width=768, cout=2048, H=7, stride=1,
        calls=["BNActFn(relu)"] + _COXT + ["GroupNorm9Fn(gc8+lbias)", "AggTapFn(fold2,gc8)", "CotTailFn(k)", "BNActFn(relu+res)"],
        flow=['1.0<-0.0', '3.0<-2.0', '4.0<-1.2', '4.1<-3.1', '7.0<-5.0', '7.1<-6.0', '8.0<-7.0', '8.1<-3.1', '9.3<-x', 'c0<-x', 'c1<-1.2', 'c2<-4.0', 'c3<-1.2', 'c4<-8.0']),
    "hybrid_stage1_first_b2": dict(model="se_cotnetd_50", kind="block", block="layer1.0", B=2, cin=64, width=64, cout=256, H=56,
                                   stride=2,
        calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(plain)", "BNActFn(relu+res)"],
        flow=['3.3<-2.0', 'c0<-x', 'c1<-0.0', 'c3<-1.0']),
    "hybrid_stage3_cot_first_b2": dict(model="se_cotnetd_50", kind="block", block="layer3.0", B=2, cin=512, width=256, cout=1024, H=28,
                                       stride=2,
        calls=["BNActFn(relu)", "Pool3x3S2Fn(avg)"] + _COT_E0 + ["BNActFn(plain)", "BNActFn(relu+res)"],
        flow=['1.0<-0.0', '11.3<-10.0', '2.0<-1.0', '4.0<-3.0', '5.0<-2.2', '5.1<-4.1', '8.0<-6.0', '8.1<-7.0', '9.0<-8.0', '9.1<-4.1', 'c0<-x', 'c1<-2.2', 'c2<-5.0', 'c3<-2.2', 'c5<-9.0']),
    "hybrid_stage3_split_b2": dict(model="se_cotnetd_50", kind="block", block="layer3.1", B=2, cin=1024, width=256, cout=1024, H=14,
                                   stride=1,
        calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(relu+res)"],
        flow=['2.3<-x', 'c0<-x', 'c1<-0.0', 'c2<-1.0']),
    "hybrid_stage4_first_b2": dict(model="se_cotnetd_50", kind="block", block="layer4.0", B=2, cin=1024, width=512, cout=2048, H=14,
                                   stride=2,
        calls=["BNActFn(relu)", "Pool3x3S2Fn(avg)"] + _COT_E0 + ["BNActFn(plain)", "BNActFn(relu+res)"],
        flow=['1.0<-0.0', '11.3<-10.0', '2.0<-1.0', '4.0<-3.0', '5.0<-2.2', '5.1<-4.1', '8.0<-6.0', '8.1<-7.0', '9.0<-8.0', '9.1<-4.1', 'c0<-x', 'c1<-2.2', 'c2<-5.0', 'c3<-2.2', 'c5<-9.0']),
    "cotnet_stage2_drop_path_b2": dict(model="cotnet50", kind="block", block="layer2.1", B=2, cin=512, width=128, cout=512, H=28,
                                       stride=1, ds=_DS,
        calls=["BNActFn(relu)"] + _COT_E0 + ["BNActFn(relu+res+ds)"],
        flow=['1.0<-0.0', '3.0<-2.0', '4.0<-1.2', '4.1<-3.1', '7.0<-5.0', '7.1<-6.0', '8.0<-7.0', '8.1<-3.1', '9.3<-x', 'c0<-x', 'c1<-1.2', 'c2<-4.0', 'c3<-1.2', 'c4<-8.0']),
    "hybrid_stage2_drop_path_b2": dict(model="se_cotnetd_50", kind="block", block="layer2.1", B=2, cin=512, width=128, cout=512, H=28,
                                       stride=1, ds=_DS,
        calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(relu+res+ds)"],
        flow=['2.3<-x', 'c0<-x', 'c1<-0.0', 'c2<-1.0']),
    "cotnet_stage3_dropblock_b2": dict(model="cotnet50", kind="block", block="layer3.0", B=2, cin=512, width=256, cout=1024, H=28,
                                       stride=2, sites=(0, 1),
        calls=["BNActFn(relu)", "DropBlockFn", "Pool3x3S2Fn(avg)"] + _COT_E0 + ["BNActFn(plain)", "BNActFn(plain)", "DropBlockResReluFn"],
        flow=['1.0<-0.0', '10.0<-9.0', '10.1<-5.1', '13.0<-12.0', '13.1<-11.0', '2.0<-1.0', '3.0<-2.0', '5.0<-4.0', '6.0<-3.2', '6.1<-5.1', '9.0<-7.0', '9.1<-8.0', 'c0<-x', 'c1<-3.2', 'c2<-6.0', 'c3<-3.2', 'c4<-x', 'c5<-10.0']),
    "hybrid_stage3_split_dropblock_b4": dict(model="se_cotnetd_50", kind="block", block="layer3.1", B=4, cin=1024, width=256, cout=1024,
                                             H=14, stride=1, sites=(2, 3, 4), ds=(0.0, 1.25, 1.25, 1.25),
        calls=["BNActFn(relu)", "DropBlockFn", "BNActFn(plain)", "DropBlockFn", "BNActFn(plain)", "DropBlockResReluFn"],
        flow=['1.0<-0.0', '3.0<-2.0', '5.0<-4.0', '5.1<-x', 'c0<-x', 'c1<-1.0']),
    "cotnet_stem_wgmma_wgrad": dict(model="cotnet50", kind="stem", B=2, H=96, W=96,
        calls=["StemConvBNFn", "Pool3x3S2Fn(max)"],
        flow=['1.0<-0.0']),
    "cotnet_stem_cudnn_wgrad": dict(model="cotnet50", kind="stem", B=2, H=64, W=72,
        calls=["StemConvBNFn", "Pool3x3S2Fn(max)"],
        flow=['1.0<-0.0']),
    "hybrid_deep_stem": dict(model="se_cotnetd_50", kind="stem", B=2, H=64, W=64,
        calls=["BNActFn(relu)"] * 3,
        flow=['c1<-0.0', 'c2<-1.0']),
}
#: SE-CoTNetD-152 at its 320 (cot_l) and 256 (cot_s) configs: BlurPool after conv2 of every stride-2 block (avd, avd_first=False),
#: so a split-attention conv2 of a first block runs at stride 1 on the block's input size and a CoT layer of layer3.0 / layer4.0
#: before the pool.  min_pixels=0 where the bench's bs64 step is above TC_MIN_PIXELS (stages 1-2 and layer3.0 at 320: 102400
#: pixels), the default below it; layer3.0 at B=64 takes the real threshold.  ds: drop path at the config's rate 0.15.  In the
#: flows, "c<j><-pad(k.o)": torch convolution j (the BlurPool) reads the reflect padding of k.o; "<-c<j>": the BlurPool's output.
_DS152 = (0.0, 1.0 / 0.85)
_HYB152 = dict(model="se_cotnetd_152", kind="block")
_COT152_FIRST = ["BNActFn(relu)"] + _COT_E0 + ["BNActFn(plain)", "BNActFn(relu+res)"]
_FLOW152_FIRST = ['1.0<-0.0', '3.0<-2.0', '4.0<-1.2', '4.1<-3.1', '7.0<-5.0', '7.1<-6.0', '8.0<-7.0', '8.1<-3.1', '10.3<-9.0', 'c0<-x',
                  'c1<-1.2', 'c2<-4.0', 'c3<-1.2', 'c4<-pad(8.0)', 'c6<-c4']
_COT152 = ["BNActFn(relu)"] + _COT_E0
_FLOW152 = ['1.0<-0.0', '3.0<-2.0', '4.0<-1.2', '4.1<-3.1', '7.0<-5.0', '7.1<-6.0', '8.0<-7.0', '8.1<-3.1', '9.3<-x', 'c0<-x', 'c1<-1.2',
            'c2<-4.0', 'c3<-1.2', 'c4<-8.0']
#: layer3.0 with its CoT layer's embed.3 and conv1x1 on wgmma (embed.3: N = 288, three 128-wide tiles), conv1 too; the key conv
#: (dim 256 > TC_KEY_MAX_DIM), the downsample and conv3 (weights above TC_TRUNK_MAX_WEIGHT) on cuDNN
_L30_TC = ["TcConv1x1Fn(one,relu)", "FanOutFn(3)", "BNActFn(relu)", "FanOutFn(2)", "TcConv1x1Fn(two,relu)", "TcConv1x1Fn(one,nobn)",
           "TcConv1x1Fn(one,bn)", "GroupNorm9Fn(gc8+lbias)", "AggTapFn(fold1,gc8)", "CotTailFn(k)", "BNActFn(plain)", "BNActFn(relu+res)"]
_L30_TC_FLOW = ['0.0<-x', '1.0<-0.0', '3.0<-2.0', '4.0<-1.2', '4.1<-3.1', '5.0<-4.0', '6.0<-1.2', '7.0<-5.0', '8.0<-6.0', '8.1<-7.0',
                '9.0<-8.0', '9.1<-3.1', '11.3<-10.0', 'c0<-1.2', 'c1<-pad(9.0)', 'c3<-c1']
STEP_BLOCK_CASES.update({
    "hybrid152_320_layer1_first_b2": dict(_HYB152, block="layer1.0", B=2, cin=128, width=64, cout=256, H=160, stride=2, min_pixels=0,
        calls=["TcConv1x1Fn(one,relu)", "CotTailFn(gate)", "TcConv1x1Fn(one,bn)", "TcConv1x1Fn(one,relu+res)"],
        flow=['0.0<-x', '3.0<-c1', '3.8<-2.0', 'c0<-0.0', 'c1<-pad(1.0)']),
    "hybrid152_320_layer2_split_drop_path_b2": dict(_HYB152, block="layer2.3", B=2, cin=512, width=128, cout=512, H=40, stride=1,
                                                     min_pixels=0, ds=_DS152,
        calls=["TcConv1x1Fn(one,relu)", "CotTailFn(gate)", "TcConv1x1Fn(one,relu+res+ds)"],
        flow=['0.0<-x', '2.0<-1.0', '2.8<-x', 'c0<-0.0']),
    "hybrid152_320_layer3_cot_first_b2": dict(_HYB152, block="layer3.0", B=2, cin=512, width=256, cout=1024, H=40, stride=2,
                                               min_pixels=0, calls=_L30_TC, flow=_L30_TC_FLOW),
    "hybrid152_320_layer3_cot_first_b64": dict(_HYB152, block="layer3.0", B=64, cin=512, width=256, cout=1024, H=40, stride=2,
                                                calls=_L30_TC, flow=_L30_TC_FLOW),
    "hybrid152_320_layer3_split_b2": dict(_HYB152, block="layer3.17", B=2, cin=1024, width=256, cout=1024, H=20, stride=1,
        calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(relu+res)"],
        flow=['2.3<-x', 'c0<-x', 'c1<-0.0', 'c2<-1.0']),
    "hybrid152_320_layer3_cot_drop_path_b2": dict(_HYB152, block="layer3.2", B=2, cin=1024, width=256, cout=1024, H=20, stride=1,
                                                   ds=_DS152, calls=_COT152 + ["BNActFn(relu+res+ds)"], flow=_FLOW152),
    "hybrid152_320_layer4_first_b2": dict(_HYB152, block="layer4.0", B=2, cin=1024, width=512, cout=2048, H=20, stride=2,
                                           calls=_COT152_FIRST, flow=_FLOW152_FIRST),
    "hybrid152_320_layer4_b2": dict(_HYB152, block="layer4.1", B=2, cin=2048, width=512, cout=2048, H=10, stride=1,
                                     calls=_COT152 + ["BNActFn(relu+res)"], flow=_FLOW152),
    # 256: at bs64 layer3.0 sees 65536 pixels, below the threshold
    "hybrid152_256_layer3_cot_first_b2": dict(_HYB152, block="layer3.0", B=2, cin=512, width=256, cout=1024, H=32, stride=2,
                                               calls=_COT152_FIRST, flow=_FLOW152_FIRST),
    "hybrid152_256_layer3_cot_b2": dict(_HYB152, block="layer3.34", B=2, cin=1024, width=256, cout=1024, H=16, stride=1,
                                         calls=_COT152 + ["BNActFn(relu+res)"], flow=_FLOW152),
    "hybrid152_256_layer4_first_b2": dict(_HYB152, block="layer4.0", B=2, cin=1024, width=512, cout=2048, H=16, stride=2,
                                           calls=_COT152_FIRST, flow=_FLOW152_FIRST),
    "hybrid152_256_layer4_drop_path_b2": dict(_HYB152, block="layer4.2", B=2, cin=2048, width=512, cout=2048, H=8, stride=1,
                                               ds=_DS152, calls=_COT152 + ["BNActFn(relu+res+ds)"], flow=_FLOW152),
    "hybrid152_deep_stem_320": dict(model="se_cotnetd_152", kind="stem", B=2, H=320, W=320, calls=["BNActFn(relu)"] * 3,
                                    flow=['c1<-0.0', 'c2<-1.0']),
    "hybrid152_deep_stem_256": dict(model="se_cotnetd_152", kind="stem", B=2, H=256, W=256, calls=["BNActFn(relu)"] * 3,
                                    flow=['c1<-0.0', 'c2<-1.0']),
})


def conv_out(H, stride):
    """output size of every stride-2 stage of the trunks (7x7/s2 pad 3, 3x3/s2 pad 1 convolutions and pools, the avg_down 2x2/s2
    ceil-mode pool): (H - 1) // 2 + 1, which is H // 2 only for even H"""
    return H if stride == 1 else (H - 1) // 2 + 1


def model_blocks(model, H0, W0=None):
    """[(name, block index in its stage, cin, width, cout, H in, W in, stride)] of every bottleneck of cotnet50 / cotnext50_2x48d /
    the SE-CoTNetD trunks for an H0 x W0 image: cotnet's 7x7/s2 stem and max pool, stride 2 from stage 2 on; the deep stem's
    stride 2 (2 * stem_width channels out), stride 2 in every stage (backbone.CoTResNet, backbone_hybrid.CoTHybridNet).  A stride-2
    BlurPool (reflect pad 1, 3x3, stride 2) gives the same size as the 3x3/s2 average pool."""
    W0 = H0 if W0 is None else W0
    hybrid = model in HYBRID
    H, W = conv_out(H0, 2), conv_out(W0, 2)
    if not hybrid:
        H, W = conv_out(H, 2), conv_out(W, 2)
    cin = 2 * HYBRID[model]["stem_width"] if hybrid else 64
    layers = HYBRID[model]["layers"] if hybrid else (3, 4, 6, 3)
    out = []
    for si, (planes, n) in enumerate(zip((64, 128, 256, 512), layers)):
        width = planes * 48 // 64 * 2 if model == "cotnext50_2x48d" else planes
        for b in range(n):
            stride = 2 if b == 0 and (hybrid or si > 0) else 1
            out.append(("layer%d.%d" % (si + 1, b), b, cin, width, planes * 4, H, W, stride))
            cin, H, W = planes * 4, conv_out(H, stride), conv_out(W, stride)
    return out


def model_calls(model, B, H0, min_pixels=TC_MIN_PIXELS, drop_block=True):
    """the recorded calls of one TrainStep forward with drop path (every block but the first) and DropBlock (stages 3-4, unless
    drop_block is False) on, as [stem calls, [calls of each block], loss calls]"""
    blocks = []
    for i, (name, b, cin, width, cout, H, W, stride) in enumerate(model_blocks(model, H0)):
        db = drop_block and name.startswith(("layer3", "layer4"))
        if model in HYBRID:
            blocks.append(hybrid_block_calls(B, b, cin, width, H, stride, min_pixels, db, i > 0, model))
        else:
            blocks.append(bottleneck_calls(B, cin, width, cout, H, stride, min_pixels, model != "cotnet50", db, i > 0))
    return stem_calls(model, H0, H0), blocks, ["SoftTargetCrossEntropyFn"]


def model_sites(model):
    """the DropBlock site numbers of every block, counted here in forward order: stages 3-4 only; bn1 and bn3, and conv2.bn0
    between them in a split-attention block"""
    out, site = {}, 0
    for name, b, cin, width, cout, H, W, stride in model_blocks(model, 224):
        if not name.startswith(("layer3", "layer4")):
            continue
        n = 3 if model in HYBRID and hybrid_split(width, b, c4_idx=HYBRID[model]["c4_idx"]) else 2
        out[name] = tuple(range(site, site + n))
        site += n
    return out


# ------------------------------------------------------------------------------------------------ the eval dispatch
#: An eval forward runs as EvalStep._body runs it: model.eval(), no_grad, bf16 autocast (cache_enabled=False), step arena off, on a
#: bf16 channels_last image.  Besides the autograd functions above, the eval recorder of tests/test_eval_stages_gpu.py lists the
#: top-level wgmma calls of CotLayer._forward_tc_eval (conv3x3_bf16, gemm_bf16) and its tail (cot_tail_eval); the GEMMs that
#: TcConv1x1Fn makes inside itself are part of that call.  What differs from training:
#:   * a CotLayer takes _forward_tc_eval whenever _tc_eval_ok (dim, and W <= 128), whatever the pixel count; above W = 128 it
#:     takes _forward_fused under no_grad: no FanOutFn (fan_out falls through), cuDNN convolutions, and the eval tail;
#:   * cot_tail takes _cot_tail_eval (running statistics, cotb200_se_eval); the split-attention gate stays CotTailFn;
#:   * conv1x1_bn takes TcConv1x1Fn in eval at the same geometry rule as in training (weights of any dtype are cast to bf16);
#:   * CoXt's embed.0 is on the wgmma GEMM only with bf16 weights: fp32 weights under autocast go to cuDNN + BNActFn.
EVAL_LAYER_TC = ["conv3x3_bf16", "gemm_bf16", "gemm_bf16", "gemm_bf16"]


def eval_cot_calls(B, dim, H, W, bf16_weights, min_pixels=TC_MIN_PIXELS):
    """the recorded calls of a CotLayer's eval forward on a bf16 channels_last [B, dim, H, W] input; only W and dim decide between
    _forward_tc_eval and _forward_fused, the rest matter inside _forward_fused"""
    gc = tap_chunk(dim // 8)
    if tc_supported(dim, W):                         # CotLayer._tc_eval_ok: the same dim conditions and W <= 128
        return EVAL_LAYER_TC + ["GroupNorm9Fn(gc%d)" % gc, "AggTapFn(fold1,gc%d)" % gc, "cot_tail_eval"]
    key_tc, e0_tc, rest_tc = cot_dispatch(B, dim, H, W, min_pixels)
    out = ["TcConv3x3Fn" if key_tc and bf16_weights else "BNActFn(relu)", "TcConv1x1Fn(two,relu)" if e0_tc else "BNActFn(relu)"]
    out += ["TcConv1x1Fn(one,nobn)", "TcConv1x1Fn(one,bn)"] if rest_tc else ["BNActFn(plain)"]
    return out + ["GroupNorm9Fn(gc%d+lbias)" % gc, "AggTapFn(fold1,gc%d)" % gc, "cot_tail_eval"]


def eval_coxt_calls(dim, bf16_weights):
    """CoXtLayer's eval forward: _forward_fused under no_grad; embed.0 on the wgmma GEMM only when its dense weight is bf16"""
    gc = tap_chunk(dim // 8, 2)
    e0 = "TcConv1x1Fn(two,relu)" if bf16_weights and dim % 16 == 0 else "BNActFn(relu)"
    return ["BNActFn(relu)", e0, "BNActFn(plain)", "GroupNorm9Fn(gc%d+lbias)" % gc, "AggTapFn(fold2,gc%d)" % gc, "cot_tail_eval"]


def _eval_1x1(cin, cout, M, stride, min_pixels, label):
    return "TcConv1x1Fn(one,%s)" % label if conv1x1_tc(cin, cout, M, stride, min_pixels) else "BNActFn(%s)" % label.replace("bn", "plain")


def eval_bottleneck_calls(B, cin, width, cout, H, W, stride, bf16_weights, min_pixels=TC_MIN_PIXELS, coxt=False):
    """backbone.Bottleneck._forward_fused in eval: conv1 + bn1 + ReLU, the avd pool at stride 2, conv2, the downsample, conv3 + bn3 +
    residual + ReLU"""
    Ho, Wo = conv_out(H, stride), conv_out(W, stride)
    out = [_eval_1x1(cin, width, B * H * W, 1, min_pixels, "relu")]
    if stride > 1:
        out.append("Pool3x3S2Fn(avg)")
    out += eval_coxt_calls(width, bf16_weights) if coxt else eval_cot_calls(B, width, Ho, Wo, bf16_weights, min_pixels)
    if stride > 1 or cin != cout:
        out.append(_eval_1x1(cin, cout, B * Ho * Wo, stride, min_pixels, "bn"))
    return out + [_eval_1x1(width, cout, B * Ho * Wo, 1, min_pixels, "relu+res")]


def eval_hybrid_block_calls(B, block_idx, cin, width, H, W, stride, bf16_weights, min_pixels=TC_MIN_PIXELS, model="se_cotnetd_50"):
    """backbone_hybrid.CoTBottleneck.forward in eval: a split-attention conv2 is the cuDNN 3x3 (stride 2 itself unless avd) and the
    gate on CotTailFn with running statistics; a CoT conv2 pools at stride 2, before or after it as avd_first says (a BlurPool
    is torch glue); the avg_down downsample pools in torch"""
    cfg = HYBRID[model]
    cout = 4 * width
    Ho, Wo = conv_out(H, stride), conv_out(W, stride)
    split = hybrid_split(width, block_idx, c4_idx=cfg["c4_idx"])
    pool = stride > 1 and (cfg["avd"] if split else True)
    avd_first, pool_call = cfg["avd_first"], [] if cfg["blur"] else ["Pool3x3S2Fn(avg)"]
    out = [_eval_1x1(cin, width, B * H * W, 1, min_pixels, "relu")]
    if pool and avd_first:
        out += pool_call
    if split:
        out.append("CotTailFn(gate)")
    else:
        first = pool and avd_first
        out += eval_cot_calls(B, width, Ho if first else H, Wo if first else W, bf16_weights, min_pixels)
    if pool and not avd_first:
        out += pool_call
    if block_idx == 0:
        out.append(_eval_1x1(cin, cout, B * Ho * Wo, 1, min_pixels, "bn"))
    return out + [_eval_1x1(width, cout, B * Ho * Wo, 1, min_pixels, "relu+res")]


def eval_stem_calls(model, H, W):
    """the stems in eval: as in training (the wgmma stem folds the running statistics into its epilogue)"""
    return stem_calls(model, H, W)


def eval_model_calls(model, B, H0, W0, bf16_weights, min_pixels=TC_MIN_PIXELS):
    """the recorded calls of one eval forward of the whole network: (stem calls, [calls of each block]); the global pool and fc
    are torch ops"""
    blocks = []
    for name, b, cin, width, cout, H, W, stride in model_blocks(model, H0, W0):
        if model in HYBRID:
            blocks.append(eval_hybrid_block_calls(B, b, cin, width, H, W, stride, bf16_weights, min_pixels, model))
        else:
            blocks.append(eval_bottleneck_calls(B, cin, width, cout, H, W, stride, bf16_weights, min_pixels,
                                                model != "cotnet50"))
    return eval_stem_calls(model, H0, W0), blocks


def eval_case_calls(c):
    """the call list of an EVAL_BLOCK_CASES entry, from the generators"""
    mp = TC_MIN_PIXELS if c.get("min_pixels") is None else c["min_pixels"]
    if c["kind"] == "stem":
        return eval_stem_calls(c["model"], c["H"], c["W"])
    if c["model"] in HYBRID:
        return eval_hybrid_block_calls(c["B"], int(c["block"].split(".")[1]), c["cin"], c["width"], c["H"], c["W"], c["stride"],
                                       c["bf16"], mp, c["model"])
    return eval_bottleneck_calls(c["B"], c["cin"], c["width"], c["cout"], c["H"], c["W"], c["stride"], c["bf16"], mp,
                                 c["model"] != "cotnet50")


#: Eval blocks and stems.  calls: as the eval recorder labels them (BNActFn / TcConv1x1Fn / ... as in the training lists; the wgmma
#: CoT layer as EVAL_LAYER_TC + GroupNorm9Fn + AggTapFn + cot_tail_eval, whose output 3 is the layer output).  flow: as
#: STEP_BLOCK_CASES ("consumer.argument<-producer.output", "c<j>" the input of the j-th torch convolution), producers matched by
#: storage and by value in NHWC row order (a gemm_bf16 output [B*H*W, N] is the next stage's [B, N, H, W] input).
_EVAL_TC = EVAL_LAYER_TC + ["GroupNorm9Fn(gc8)", "AggTapFn(fold1,gc8)", "cot_tail_eval"]


def _tc_layer_flow(i, x):
    """the dataflow inside a wgmma CoT layer whose first call is number i and whose input is `x`"""
    return ["%d.0<-%s" % (i, x), "%d.0<-%s" % (i + 1, x), "%d.2<-%d.0" % (i + 1, i), "%d.0<-%d.0" % (i + 2, i + 1),
            "%d.0<-%s" % (i + 3, x), "%d.0<-%d.0" % (i + 4, i + 2), "%d.0<-%d.0" % (i + 5, i + 3), "%d.1<-%d.0" % (i + 5, i + 4),
            "%d.0<-%d.0" % (i + 6, i + 5), "%d.1<-%d.0" % (i + 6, i)]


EVAL_BLOCK_CASES = {
    # the bench's stage-1 dispatch: B*H*W = 100352, conv1, downsample and conv3 on wgmma (conv3: raw GEMM + bn_apply with the residual)
    "cot_stage1_b32": dict(model="cotnet50", kind="block", block="layer1.0", B=32, cin=64, width=64, cout=256, H=56, W=56, stride=1,
                           bf16=True, calls=["TcConv1x1Fn(one,relu)"] + _EVAL_TC + ["TcConv1x1Fn(one,bn)", "TcConv1x1Fn(one,relu+res)"],
                           flow=["0.0<-x"] + _tc_layer_flow(1, "0.0") + ["8.0<-x", "9.0<-7.3", "9.8<-8.0"]),
    # 6272 pixels: the trunk 1x1 convolutions on cuDNN, the CoT layer on wgmma all the same
    "cot_stage1_b2": dict(model="cotnet50", kind="block", block="layer1.0", B=2, cin=64, width=64, cout=256, H=56, W=56, stride=1,
                          bf16=True, calls=["BNActFn(relu)"] + _EVAL_TC + ["BNActFn(plain)", "BNActFn(relu+res)"],
                          flow=_tc_layer_flow(1, "0.0") + ["9.3<-8.0", "c0<-x", "c1<-x", "c2<-7.3"]),
    # stride 2: the avd average pool in front of the CoT layer, the stride-2 downsample on cuDNN
    "cot_stage2_first_b2": dict(model="cotnet50", kind="block", block="layer2.0", B=2, cin=256, width=128, cout=512, H=28, W=28,
                                stride=2, bf16=True,
                                calls=["BNActFn(relu)", "Pool3x3S2Fn(avg)"] + _EVAL_TC + ["BNActFn(plain)", "BNActFn(relu+res)"],
                                flow=["1.0<-0.0"] + _tc_layer_flow(2, "1.0") + ["10.3<-9.0", "c0<-x", "c1<-x", "c2<-8.3"]),
    # 7x7, dim 512: the conv-mode key convolution; the residual is the block input
    "cot_stage4_b2": dict(model="cotnet50", kind="block", block="layer4.1", B=2, cin=2048, width=512, cout=2048, H=7, W=7, stride=1,
                          bf16=True, calls=["BNActFn(relu)"] + _EVAL_TC + ["BNActFn(relu+res)"],
                          flow=_tc_layer_flow(1, "0.0") + ["8.3<-x", "c0<-x", "c1<-7.3"]),
    # W = 130 > 128: CotLayer._forward_fused under no_grad (no FanOutFn, cuDNN convolutions) and the eval tail
    "cot_stage1_wide_b1": dict(model="cotnet50", kind="block", block="layer1.0", B=1, cin=64, width=64, cout=256, H=130, W=130,
                               stride=1, bf16=True,
                               calls=["BNActFn(relu)", "BNActFn(relu)", "BNActFn(relu)", "BNActFn(plain)", "GroupNorm9Fn(gc8+lbias)",
                                      "AggTapFn(fold1,gc8)", "cot_tail_eval", "BNActFn(plain)", "BNActFn(relu+res)"],
                               flow=["5.0<-3.0", "5.1<-4.0", "6.0<-5.0", "6.1<-1.0", "8.3<-7.0", "c0<-x", "c1<-0.0", "c3<-2.0",
                                     "c4<-0.0", "c5<-x", "c6<-6.3"]),
    # CoXt, embed.0 on the wgmma GEMM (bf16 weights) or on cuDNN (fp32 weights under autocast)
    "coxt_stage1_b2_bf16w": dict(model="cotnext50_2x48d", kind="block", block="layer1.0", B=2, cin=64, width=96, cout=256, H=56, W=56,
                                 stride=1, bf16=True,
                                 calls=["BNActFn(relu)", "BNActFn(relu)", "TcConv1x1Fn(two,relu)", "BNActFn(plain)",
                                        "GroupNorm9Fn(gc0+lbias)", "AggTapFn(fold2,gc0)", "cot_tail_eval", "BNActFn(plain)",
                                        "BNActFn(relu+res)"],
                                 flow=["2.0<-0.0", "2.1<-1.0", "5.0<-3.0", "5.1<-4.0", "6.0<-5.0", "6.1<-1.0", "8.3<-7.0", "c0<-x",
                                       "c1<-0.0", "c2<-2.0", "c3<-0.0", "c4<-x", "c5<-6.3"]),
    "coxt_stage1_b2_fp32w": dict(model="cotnext50_2x48d", kind="block", block="layer1.0", B=2, cin=64, width=96, cout=256, H=56, W=56,
                                 stride=1, bf16=False,
                                 calls=["BNActFn(relu)", "BNActFn(relu)", "BNActFn(relu)", "BNActFn(plain)", "GroupNorm9Fn(gc0+lbias)",
                                        "AggTapFn(fold2,gc0)", "cot_tail_eval", "BNActFn(plain)", "BNActFn(relu+res)"],
                                 flow=["5.0<-3.0", "5.1<-4.0", "6.0<-5.0", "6.1<-1.0", "8.3<-7.0", "c0<-x", "c1<-0.0", "c3<-2.0",
                                       "c4<-0.0", "c5<-x", "c6<-6.3"]),
    "coxt_stage4_b2": dict(model="cotnext50_2x48d", kind="block", block="layer4.1", B=2, cin=2048, width=768, cout=2048, H=7, W=7,
                           stride=1, bf16=True,
                           calls=["BNActFn(relu)", "BNActFn(relu)", "TcConv1x1Fn(two,relu)", "BNActFn(plain)", "GroupNorm9Fn(gc8+lbias)",
                                  "AggTapFn(fold2,gc8)", "cot_tail_eval", "BNActFn(relu+res)"],
                           flow=["2.0<-0.0", "2.1<-1.0", "5.0<-3.0", "5.1<-4.0", "6.0<-5.0", "6.1<-1.0", "7.3<-x", "c0<-x", "c1<-0.0",
                                 "c2<-2.0", "c3<-0.0", "c4<-6.3"]),
    # SE-CoTNetD: split attention with the stride-2 cuDNN 3x3 and avg_down; the CoT layer of layer3.0 (c4_idx); split attention at
    # 14x14 and at a non-square 29x25 (the gate's H*W normaliser)
    "hybrid_stage1_first_b2": dict(model="se_cotnetd_50", kind="block", block="layer1.0", B=2, cin=64, width=64, cout=256, H=56, W=56,
                                   stride=2, bf16=True,
                                   calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(plain)", "BNActFn(relu+res)"],
                                   flow=["3.3<-2.0", "c0<-x", "c1<-0.0", "c3<-1.0"]),
    "hybrid_stage3_cot_first_b2": dict(model="se_cotnetd_50", kind="block", block="layer3.0", B=2, cin=512, width=256, cout=1024, H=28,
                                       W=28, stride=2, bf16=True,
                                       calls=["BNActFn(relu)", "Pool3x3S2Fn(avg)"] + _EVAL_TC + ["BNActFn(plain)", "BNActFn(relu+res)"],
                                       flow=["1.0<-0.0"] + _tc_layer_flow(2, "1.0") + ["10.3<-9.0", "c0<-x", "c2<-8.3"]),
    "hybrid_stage3_split_b2": dict(model="se_cotnetd_50", kind="block", block="layer3.1", B=2, cin=1024, width=256, cout=1024, H=14,
                                   W=14, stride=1, bf16=True, calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(relu+res)"],
                                   flow=["2.3<-x", "c0<-x", "c1<-0.0", "c2<-1.0"]),
    "hybrid_stage2_29x25_b2": dict(model="se_cotnetd_50", kind="block", block="layer2.1", B=2, cin=512, width=128, cout=512, H=29,
                                   W=25, stride=1, bf16=True, calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(relu+res)"],
                                   flow=["2.3<-x", "c0<-x", "c1<-0.0", "c2<-1.0"]),
    # stems: the wgmma 7x7/s2 stem at even sizes, cuDNN at odd ones, the deep stem on cuDNN
    "cotnet_stem_224": dict(model="cotnet50", kind="stem", B=2, H=224, W=224, bf16=True, calls=["StemConvBNFn", "Pool3x3S2Fn(max)"],
                            flow=["0.0<-x", "1.0<-0.0"]),
    "cotnet_stem_225": dict(model="cotnet50", kind="stem", B=2, H=225, W=225, bf16=True, calls=["BNActFn(relu)", "Pool3x3S2Fn(max)"],
                            flow=["1.0<-0.0", "c0<-x"]),
    "cotnet_stem_232x200": dict(model="cotnet50", kind="stem", B=2, H=232, W=200, bf16=False, calls=["StemConvBNFn", "Pool3x3S2Fn(max)"],
                                flow=["0.0<-x", "1.0<-0.0"]),
    "hybrid_deep_stem": dict(model="se_cotnetd_50", kind="stem", B=2, H=224, W=224, bf16=True, calls=["BNActFn(relu)"] * 3,
                             flow=["c0<-x", "c1<-0.0", "c2<-1.0"]),
}
#: SE-CoTNetD-152 at 320 and 256 (see STEP_BLOCK_CASES): the BlurPool after conv2, and the wgmma key convolution of every CoT layer
#: geometry the trunk has: dim 256 on the haloed kernel at 40x40 (R = 5), 20x20 (R = 10), 32x32 (R = 4) and 16x16 (R = 8), dim
#: 512 in conv mode at 20x20 (100-row bands), 10x10 (100-row tiles), 16x16 (128-row bands) and 8x8 (two samples per tile)
_EVAL152_FIRST = ["BNActFn(relu)"] + _EVAL_TC + ["BNActFn(plain)", "BNActFn(relu+res)"]
_EVAL152_FIRST_FLOW = _tc_layer_flow(1, "0.0") + ["9.3<-8.0", "c0<-x", "c1<-pad(7.3)", "c3<-c1"]
_EVAL152 = ["BNActFn(relu)"] + _EVAL_TC + ["BNActFn(relu+res)"]
_EVAL152_FLOW = _tc_layer_flow(1, "0.0") + ["8.3<-x", "c0<-x", "c1<-7.3"]
_EVAL152_SPLIT = dict(calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(relu+res)"], flow=["2.3<-x", "c0<-x", "c1<-0.0", "c2<-1.0"])
EVAL_BLOCK_CASES.update({
    "hybrid152_320_layer1_first_b2": dict(_HYB152, block="layer1.0", B=2, cin=128, width=64, cout=256, H=160, W=160, stride=2,
                                          bf16=True, calls=["BNActFn(relu)", "CotTailFn(gate)", "BNActFn(plain)", "BNActFn(relu+res)"],
                                          flow=["3.3<-2.0", "c0<-x", "c1<-0.0", "c2<-pad(1.0)", "c4<-c2"]),
    "hybrid152_320_layer2_split_b2": dict(_HYB152, block="layer2.5", B=2, cin=512, width=128, cout=512, H=40, W=40, stride=1, bf16=True,
                                          **_EVAL152_SPLIT),
    "hybrid152_320_layer3_cot_first_b2": dict(_HYB152, block="layer3.0", B=2, cin=512, width=256, cout=1024, H=40, W=40, stride=2,
                                              bf16=True, calls=_EVAL152_FIRST, flow=_EVAL152_FIRST_FLOW),
    "hybrid152_320_layer3_split_b2": dict(_HYB152, block="layer3.1", B=2, cin=1024, width=256, cout=1024, H=20, W=20, stride=1,
                                          bf16=True, **_EVAL152_SPLIT),
    "hybrid152_320_layer3_cot_b2": dict(_HYB152, block="layer3.2", B=2, cin=1024, width=256, cout=1024, H=20, W=20, stride=1,
                                        bf16=True, calls=_EVAL152, flow=_EVAL152_FLOW),
    "hybrid152_320_layer4_first_b2": dict(_HYB152, block="layer4.0", B=2, cin=1024, width=512, cout=2048, H=20, W=20, stride=2,
                                          bf16=True, calls=_EVAL152_FIRST, flow=_EVAL152_FIRST_FLOW),
    "hybrid152_320_layer4_b3": dict(_HYB152, block="layer4.1", B=3, cin=2048, width=512, cout=2048, H=10, W=10, stride=1, bf16=True,
                                    calls=_EVAL152, flow=_EVAL152_FLOW),
    "hybrid152_256_layer3_cot_first_b2": dict(_HYB152, block="layer3.0", B=2, cin=512, width=256, cout=1024, H=32, W=32, stride=2,
                                              bf16=True, calls=_EVAL152_FIRST, flow=_EVAL152_FIRST_FLOW),
    "hybrid152_256_layer3_cot_b2": dict(_HYB152, block="layer3.20", B=2, cin=1024, width=256, cout=1024, H=16, W=16, stride=1,
                                        bf16=True, calls=_EVAL152, flow=_EVAL152_FLOW),
    "hybrid152_256_layer4_first_b2": dict(_HYB152, block="layer4.0", B=2, cin=1024, width=512, cout=2048, H=16, W=16, stride=2,
                                          bf16=True, calls=_EVAL152_FIRST, flow=_EVAL152_FIRST_FLOW),
    # odd B: a half-empty last tile of the two-sample conv mode
    "hybrid152_256_layer4_b3": dict(_HYB152, block="layer4.2", B=3, cin=2048, width=512, cout=2048, H=8, W=8, stride=1, bf16=True,
                                    calls=_EVAL152, flow=_EVAL152_FLOW),
    "hybrid152_deep_stem_320": dict(model="se_cotnetd_152", kind="stem", B=2, H=320, W=320, bf16=True, calls=["BNActFn(relu)"] * 3,
                                    flow=["c0<-x", "c1<-0.0", "c2<-1.0"]),
    "hybrid152_deep_stem_256": dict(model="se_cotnetd_152", kind="stem", B=2, H=256, W=256, bf16=True, calls=["BNActFn(relu)"] * 3,
                                    flow=["c0<-x", "c1<-0.0", "c2<-1.0"]),
})
