"""The CoT layer's inference forward (CotLayer._forward_tc_eval + fused._cot_tail_eval), stage by stage and against what it caches.

test_cot_layer_eval_stage_by_stage records the forward (the wgmma calls, GroupNorm9Fn, AggTapFn and the eval tail's fold, pooled
sums, attention weights and output) without changing a bit or a launch, and checks every producer -> consumer edge bit for bit,
every stage against fp64 of its own inputs within the bounds of tests/stage_ref.py, and every BatchNorm fold against fp64 of the
module's running statistics (stage_ref.fold_bound).

_forward_tc_eval reads bf16 / BatchNorm-folded copies of its weights (CotLayer._tc_params) and of its `se` MLP
(fused._se_eval_params), keyed by the version counters of the module's parameters and buffers.  A copy that outlived a change
of the tensor it was made from would make validation score stale weights.  Every parameter and floating-point buffer of the
layer is changed in place in turn; the next eval forward must equal, bit for bit, that of a freshly built layer loaded with the
same state.  A raw write that does not bump the version (what the optimizer kernels and the EMA graph's .data rebinding do) must
leave a cached copy (a bf16 weight, a folded BatchNorm) in use until evaler.drop_weight_caches forgets it.  (fp32 tensors the
kernels take as they are, such as embed.3's bias or the `se` convolutions of an fp32 module, are not copied and need no drop.)"""
import pytest
import torch
import torch.nn.functional as F

import stage_ref as S
from cotnet_b200 import _lib, evaler, fused, tc
from cotnet_b200.cot_layer import CotLayer
from test_persistent_gpu import pack_conv3x3
from test_stage_grads_gpu import ONE_ULP, _w, check_agg, check_gn9

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _layer(dim, state=None, seed=0):
    m = CotLayer(dim, 3)
    if state is None:
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, t in m.state_dict().items():
                if t.dtype.is_floating_point:
                    t.copy_(torch.rand(t.shape, generator=g) + 0.5 if name.endswith("running_var") else
                            0.2 * torch.randn(t.shape, generator=g))
    else:
        m.load_state_dict(state)
    return m.to(DEV).eval()


def _x(dim, H, B=2, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, dim, H, H, generator=g))
    return x.to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _fwd(m, x):
    with torch.no_grad():
        assert m._tc_eval_ok(x)
        return m(x)


@pytest.mark.parametrize("dim,H", [(64, 14), (256, 7)])
def test_weight_caches_follow_in_place_changes(dim, H):
    m = _layer(dim)
    x = _x(dim, H)
    prev = _fwd(m, x)
    names = [n for n, t in m.state_dict().items() if t.dtype.is_floating_point]
    assert any(n.startswith("se.") for n in names) and any(n.startswith("key_embed.") for n in names)
    tensors = dict(m.named_parameters(), **dict(m.named_buffers()))
    for name in names:
        t = tensors[name]
        with torch.no_grad():
            t.mul_(1.25) if name.endswith("running_var") else t.add_(0.05 + 0.1 * t.abs())
        got = _fwd(m, x)
        want = _fwd(_layer(dim, m.state_dict()), x)
        assert torch.equal(got, want), "%s: the eval forward after an in-place change differs from a fresh layer's" % name
        assert not torch.equal(got, prev), "%s: the change did not reach the output" % name
        prev = got


@pytest.mark.parametrize("name", ["key_embed.0.weight", "key_embed.1.running_var", "embed.0.weight", "embed.1.weight", "embed.3.weight",
                                  "conv1x1.0.weight", "conv1x1.1.bias", "se.1.running_mean", "se.1.weight"])
def test_drop_weight_caches_after_raw_write(name):
    dim, H = 64, 14
    m = _layer(dim, seed=3)
    x = _x(dim, H)
    before = _fwd(m, x)
    t = dict(m.named_parameters(), **dict(m.named_buffers()))[name]
    v = t._version
    t.data.add_(0.3)                               # a write that bypasses the version counter
    assert t._version == v
    assert torch.equal(_fwd(m, x), before), "the cached copy should still be in use"
    evaler.drop_weight_caches(m)
    got = _fwd(m, x)
    assert torch.equal(got, _fwd(_layer(dim, m.state_dict()), x))
    assert not torch.equal(got, before)


# ================================================================================================ the eval forward, stage by stage
def _bf16_weights(m):
    """the layout TrainStep(weights="bf16") gives the model: convolution weights bf16, 1-D parameters and buffers fp32"""
    for p in m.parameters():
        if p.dim() >= 2:
            p.data = p.data.to(torch.bfloat16)
    return m


def _rows2(t):
    return S.rows(t) if t.dim() == 4 else t.double()


class _EvalRecorder:
    """S.Recorder (GroupNorm9Fn, AggTapFn, ...) plus the wgmma calls of _forward_tc_eval (tc.gemm_bf16, tc.conv3x3_bf16) and the eval
    tail's stages (fused._cot_tail_eval_stages), all into one ordered call list.  Only top-level wgmma calls are listed: the GEMM a
    recorded function (TcConv1x1Fn) makes inside itself is part of that call.  The eval BatchNorm fold of the wgmma functions
    (fused._bn_eval_fold) is captured into their call's extra["fold"].  Snapshots only: no bit and no launch changes."""

    def __init__(self, monkeypatch, keep_outputs=False):
        self.rec = S.Recorder(monkeypatch, keep_outputs)
        calls, stack, kept = self.rec.calls, self.rec._stack, self.rec.kept
        gemm0, conv0, tail0, fold0 = tc.gemm_bf16, tc.conv3x3_bf16, fused._cot_tail_eval_stages, fused._bn_eval_fold

        def done(c, o):
            c.out = S._snap(o)
            c.out_ptr = tuple(t.data_ptr() for t in (o if isinstance(o, tuple) else (o,)))
            if kept is not None:
                kept.append(o)

        def gemm_w(*a, **kw):
            if stack:
                return gemm0(*a, **kw)
            c = S.Call("gemm_bf16", (None,))
            calls.append(c)
            o = gemm0(*a, **kw)
            names = ("a1", "b1", "a2", "b2", "scale", "shift", "relu", "stats", "out")
            args = dict(zip(names, a), **kw)
            assert args.get("stats") is None
            c.args = tuple(args.get(n) for n in names[:7])
            c.inp = tuple(S._snap(v) for v in c.args)
            done(c, o)
            return o

        def conv_w(x, wp, bn, scale=None, shift=None, relu=False, stats=None, out=None):
            if stack:
                return conv0(x, wp, bn, scale=scale, shift=shift, relu=relu, stats=stats, out=out)
            assert stats is None
            c = S.Call("conv3x3_bf16", (x, wp, bn, scale, shift, relu))
            calls.append(c)
            o = conv0(x, wp, bn, scale=scale, shift=shift, relu=relu, out=out)
            done(c, o)
            return o

        def tail_w(u, k, bn, se):
            c = S.Call("cot_tail_eval", (u, k))
            c.extra.update(bn=bn, se=se)
            calls.append(c)
            r = tail0(u, k, bn, se)
            done(c, r)
            return r

        def fold_w(bn, weight, bias):
            r = fold0(bn, weight, bias)
            if stack:
                stack[-1].extra["fold"] = (bn,) + tuple(S._snap(t) for t in r)
            return r
        monkeypatch.setattr(tc, "gemm_bf16", gemm_w)
        monkeypatch.setattr(tc, "conv3x3_bf16", conv_w)
        monkeypatch.setattr(fused, "_cot_tail_eval_stages", tail_w)
        monkeypatch.setattr(fused, "_bn_eval_fold", fold_w)
        self.calls = calls


EVAL_LAYER_CALLS = ["conv3x3_bf16", "gemm_bf16", "gemm_bf16", "gemm_bf16", "GroupNorm9Fn", "AggTapFn", "cot_tail_eval"]


def _check_gemm(call, what, stage):
    a1, b1, a2, b2, scale, shift, relu = call.inp
    acc = _rows2(a1) @ b1.double().t()
    mag = _rows2(a1).abs() @ b1.double().abs().t()
    if a2 is not None:
        acc, mag = acc + _rows2(a2) @ b2.double().t(), mag + _rows2(a2).abs() @ b2.double().abs().t()
    err = S.gamma_tc(b1.shape[1] + (0 if b2 is None else b2.shape[1]) + 1) * mag
    sc = scale.double() if scale is not None else torch.ones_like(acc[0])
    sh = shift.double() if shift is not None else torch.zeros_like(acc[0])
    z = acc * sc + sh
    zerr = sc.abs() * err + 4 * S.U32 * ((acc * sc).abs() + sh.abs())
    if relu:
        z = z.clamp_min(0.0)
    _w(call.out, z, zerr, what, stage)


def _check_conv(call, weight, what):
    x, wp, bnt, scale, shift, relu = call.inp
    w64 = weight.to(torch.bfloat16)
    S.equal(wp, pack_conv3x3(w64, 4, bnt), what + " packed weight = the key weight in bf16")
    w64 = w64.double()
    acc = F.conv2d(x.double(), w64, padding=1, groups=4)
    mag = F.conv2d(x.double().abs(), w64.abs(), padding=1, groups=4)
    y, yerr = S.bn_apply_ref(acc, scale, shift, relu)
    _w(call.out, y, yerr + scale.double().abs().view(1, -1, 1, 1) * S.gamma_tc(9 * w64.shape[1] + 1) * mag, what, "eval_conv")


def _check_fold(got_scale, got_shift, bn, what):
    fb = S.fold_bound(bn)
    S.within(got_scale, fb["scale"], fb["scale_err"], what + " folded scale")
    S.within(got_shift, fb["shift"], fb["shift_err"], what + " folded shift")


@pytest.fixture(scope="module", autouse=True)
def _report_one_ulp():
    """after the module: per stage type, the fraction of bf16 outputs one ulp from the correctly rounded fp64 value"""
    ONE_ULP.clear()
    yield
    for k in sorted(ONE_ULP):
        one, far, n = ONE_ULP[k]
        print("\neval bf16 outputs one ulp off, %-10s %.2e (%d of %d; %d farther)" % (k, one / max(n, 1), one, n, far), end="")


@pytest.mark.parametrize("layout", ["fp32", "bf16w"])
@pytest.mark.parametrize("dim,H,B", [(64, 56, 2), (128, 28, 2), (256, 14, 4), (512, 7, 8)])
def test_cot_layer_eval_stage_by_stage(dim, H, B, layout, monkeypatch):
    """CotLayer._forward_tc_eval under no_grad, recorded: (a) the call list, (b) every producer -> consumer edge bit for bit, (c)
    every stage within 1/2 bf16 ulp plus its fp32 chain bound of fp64 of its own inputs, (d) every BatchNorm fold within its
    fold_bound of fp64 of the module's running statistics"""
    m = _layer(dim, seed=dim + B)
    if layout == "bf16w":
        _bf16_weights(m)
    x = _x(dim, H, B, seed=dim)
    lc = _lib.launch_count()
    plain = _fwd(m, x)
    n_launch = _lib.launch_count() - lc
    rec = _EvalRecorder(monkeypatch)
    lc = _lib.launch_count()
    out = _fwd(m, x)
    assert _lib.launch_count() - lc == n_launch, "the recorder changed the launches"
    S.equal(out, plain, "recorded forward == plain forward")
    check_eval_layer(rec.calls, m, x, out, "CotLayer(%d) eval %dx%d B=%d %s" % (dim, H, H, B, layout))


def check_eval_layer(calls, m, x, out, what):
    """CotLayer m's recorded _forward_tc_eval calls on input x with output out: (a) the call list, (b) every producer -> consumer
    edge bit for bit, (c) every stage within 1/2 bf16 ulp plus its fp32 chain bound of fp64 of its own inputs, (d) every BatchNorm
    fold within its fold_bound of fp64 of the module's running statistics"""
    assert [c.name for c in calls] == EVAL_LAYER_CALLS, [c.name for c in calls]
    B, dim, H, W = x.shape
    conv, e0, e3, v1, gn, agg, tail = calls
    J = 9 * dim // 8
    nhwc = lambda t, n: t.view(B, H, W, n).permute(0, 3, 1, 2)        # noqa: E731
    # (b) dataflow
    for c, i in ((conv, 0), (e0, 0), (v1, 0)):
        S.equal(c.inp[i], x, what + " %s input = x" % c.name)
    S.equal(e0.inp[2], conv.out, what + " embed.0's second operand = the key conv output")
    S.equal(tail.inp[1], conv.out, what + " the tail's k = the key conv output")
    S.equal(e3.inp[0], e0.out, what + " embed.3 input = embed.0 output")
    S.equal(gn.inp[0], nhwc(e3.out, J), what + " GroupNorm input = embed.3 output")
    assert gn.inp[5] is None, "embed.3's bias is in its GEMM epilogue, not in the GroupNorm"
    S.equal(agg.inp[0], nhwc(v1.out, dim), what + " LocalConv v = conv1x1 output")
    S.equal(agg.inp[1], gn.out, what + " LocalConv w = GroupNorm output")
    S.equal(tail.inp[0], agg.out, what + " tail u = LocalConv output")
    S.equal(tail.out[-1], out, what + " layer output = tail output")
    # the GEMM operands are the module's weights in bf16, embed.3's bias in fp32
    C = dim
    w_e0 = m.embed[0].weight.detach().view(C // 2, 2 * C).to(torch.bfloat16)
    S.equal(e0.inp[1], w_e0[:, :C], what + " embed.0 W_x")
    S.equal(e0.inp[3], w_e0[:, C:], what + " embed.0 W_k")
    S.equal(e3.inp[1], m.embed[3].weight.detach().view(J, C // 2).to(torch.bfloat16), what + " embed.3 weight")
    S.equal(e3.inp[5], m.embed[3].bias.detach().float(), what + " embed.3 bias (the shift-only epilogue)")
    assert e3.inp[4] is None and not e3.inp[6], "embed.3: shift only, no ReLU"
    S.equal(v1.inp[1], m.conv1x1[0].weight.detach().view(C, C).to(torch.bfloat16), what + " conv1x1 weight")
    assert conv.inp[5] and e0.inp[6] and not v1.inp[6]
    # (d) the folds: _tc_params (torch.rsqrt) and the tail's bn_finalize
    _check_fold(conv.inp[3], conv.inp[4], m.key_embed[1], what + " key_embed.1")
    _check_fold(e0.inp[4], e0.inp[5], m.embed[1], what + " embed.1")
    _check_fold(v1.inp[4], v1.inp[5], m.conv1x1[1], what + " conv1x1.1")
    # (c) every stage against fp64 of its own inputs
    _check_conv(conv, m.key_embed[0].weight.detach(), what + " key conv")
    _check_gemm(e0, what + " embed.0", "eval_gemm")
    _check_gemm(e3, what + " embed.3", "eval_gemm")
    _check_gemm(v1, what + " conv1x1", "eval_gemm")
    check_gn9(gn, what + " GroupNorm9Fn")
    check_agg(agg, what + " AggTapFn")
    check_tail_eval(tail, m.bn, m.se, what)


def check_tail_eval(tail, bn, se, what):
    """fused._cot_tail_eval_stages, recorded: the BatchNorm fold (bn_finalize of the running statistics), the pooled sums, the
    attention weights of cotb200_se_eval at p = psum * fl(1 / (H * W)) and the recombination, each against fp64 of its own inputs"""
    u, k = tail.inp
    H, W = u.shape[2], u.shape[3]
    ss, psum, a, tout = tail.out
    _check_fold(ss[0], ss[1], bn, what + " bn (tail)")
    fb = S.fold_bound(bn)
    S.within(ss[3], fb["rstd"], fb["rstd_err"], what + " bn (tail) rstd")
    ps, pe, y, ye = S.tail_pool_ref(u, k, ss[0], ss[1], S.SIGMOID_ERR_16)
    S.within(psum, ps, pe, what + " tail_pool psum")
    p = psum.double() * torch.tensor(1.0 / (H * W), dtype=torch.float32).double()
    ar, ea = S.mlp_ref(p, (se[0], se[1], se[3]), "cot", False, se_eval=True)
    S.within(a, ar, ea, what + " se_eval attention weights")
    o, oe = S.tail_combine_ref(y, ye, k, a)
    _w(tout, o, oe, what + " tail_combine", "eval_tail")
