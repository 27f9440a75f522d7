"""Every LocalConv kernel the dispatch can pick, through the C ABI, exactly, at the cases of tests/test_agg_geometry_cpu.py.

Each case describes its call with cotb200_agg_desc directly (layout, gc, fold, pitches, pointer offsets under the test's control) and
makes four calls: the forward and the backward with both gradients, with dX only and with dW only (the other pointer NULL).  Every
call runs inside the library's profiler and must launch exactly the multiset of kernels the Python mirror of the dispatch predicts.

Operands are small integers drawn per case so that every output is an integer the storage type holds (test_agg_geometry_cpu
.amplitude); the fp64 reference is the header's definition (agg_ref: weight channel with the CoXt fold, NHWC_TAP column order) with
autograd for the gradients, and whole outputs are compared exactly: a wrong tap, lane, fold mapping or pitch changes some element.
Operands of NHWC layouts live inside wider buffers when the descriptor has pitches; the padding of the inputs is NaN (a read of it
shows) and every output buffer is prefilled with NaN, whose bytes outside the described slice must survive the call.  The "float"
cases compare random operands with fp64 under a tolerance (the widen-and-round steps)."""
import pytest
import torch

from cotnet_b200 import _lib
from test_agg_geometry_cpu import (BWD_VARIANTS, CASES, MIX_K2, MIX_P2, NCHW, agg_ref, amplitude, mix_ref, predict,
                                   tensor_extent, weight_column)
from test_determinism_gpu import TOL

pytestmark = pytest.mark.gpu

TD = {"fp32": torch.float32, "fp64": torch.float64, "bf16": torch.bfloat16, "fp16": torch.float16}
BITS = {2: torch.int16, 4: torch.int32, 8: torch.int64}
REL = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11, "fp32": 0.0, "fp64": 0.0}


def _st():
    return torch.cuda.current_stream().cuda_stream


class Buf:
    """A tensor of the case carved out of a flat buffer: `view` is the described slice (shape / strides of tensor_extent) at
    element offset `off`; everything else in the buffer is padding."""

    def __init__(self, extent, off, dtype, fill):
        shape, strides, n = extent
        self.flat = torch.full((off + n,), fill, dtype=dtype, device="cuda")
        self.view = self.flat.as_strided(shape, strides, off)
        mask = torch.zeros(off + n, dtype=torch.bool, device="cuda")
        mask.as_strided(shape, strides, off).fill_(True)
        self.pad = ~mask
        self.before = self.flat.clone()

    def ptr(self):
        return self.view.data_ptr()

    def check_padding(self, what):
        es = self.flat.element_size()
        a, b = self.flat.view(BITS[es])[self.pad], self.before.view(BITS[es])[self.pad]
        if not torch.equal(a, b):
            bad = (a != b).nonzero()[:4].flatten().tolist()
            raise AssertionError("%s: %d padding elements written (first at padding positions %s)" % (what, int((a != b).sum()), bad))


def _eq(got, want, what):
    """got (storage dtype) == want (fp64) element for element; reports the first differing indices"""
    g = got.double()
    bad = ~(g == want)
    if bool(bad.any()):
        idx = bad.nonzero()[:4].tolist()
        raise AssertionError("%s: %d of %d elements differ, first %s: got %s want %s" % (
            what, int(bad.sum()), bad.numel(), idx, [g[tuple(i)].item() for i in idx], [want[tuple(i)].item() for i in idx]))


def _close(got, ref, absterms, what, dt):
    """|got - ref| <= rel * |ref| + TOL * sum|terms|: the storage rounding of the output plus fp32 accumulation"""
    err = (got.double() - ref).abs()
    lim = REL[dt] * ref.abs() + (1e-12 if dt == "fp64" else TOL) * absterms
    bad = ~(err <= lim)
    assert not bool(bad.any()), "%s: %d of %d elements off; worst err/limit %.3g" % (
        what, int(bad.sum()), bad.numel(), float((err / lim.clamp_min(1e-30)).max()))


def _desc(c):
    d, s = _lib.AggDesc(), c.desc
    for k, v in vars(s).items():
        setattr(d, k, v)
    d.dtype = _lib.dtype_code(torch.empty(0, dtype=TD[c.dt]))
    return d


# ------------------------------------------------------------------------------------------------ storage <-> canonical layouts
def canon_x(c, t):
    """[N,C,H,W] (x, dx) or [N,heads*C,Ho,Wo] (y, dy) of a storage view"""
    return t if c.desc.layout == NCHW else t.permute(0, 3, 1, 2)


def canon_w(c, t):
    """[N,heads,wc,K2,Ho,Wo] of a weight storage view"""
    d = c.desc
    if d.layout == NCHW:
        return t
    col = weight_column(d.heads, d.wc, d.kh * d.kw, d.layout, d.gc).to(t.device)
    return t[..., col].permute(0, 3, 4, 5, 1, 2)


def _draw(c, shape, g):
    if c.kind == "float":
        return torch.randn(shape, generator=g, device="cuda", dtype=torch.float64)
    a = amplitude(c)
    return torch.randint(-a, a + 1, shape, generator=g, device="cuda").double()


# ------------------------------------------------------------------------------------------------ one case
def _run(c, call, fn):
    """fn() under the profiler; the launched names and counts must equal the mirror's prediction"""
    want = dict(predict(c)[call].names())
    torch.cuda.synchronize()
    _lib.prof_enable(True)
    try:
        fn()
        got = {k: v[0] for k, v in _lib.prof_report().items()}
    finally:
        _lib.prof_enable(False)
    assert got == want, "%s %s: launched %s, the dispatch mirror predicts %s" % (c.name, call, got, want)


def _compare(c, what, got, ref, absref):
    if c.kind == "float":
        _close(got, ref, absref, what, c.dt)
    else:
        _eq(got, ref, what)


@pytest.mark.parametrize("c", [c for c in CASES if c.op == "agg"], ids=lambda c: c.name)
def test_agg_case(c):
    dtype, ext = TD[c.dt], tensor_extent(c)
    lib = _lib.load()
    d = _desc(c)
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, c.name)))
    inp = {k: Buf(ext[k], c.offs[k], dtype, float("nan")) for k in ("x", "w", "dy")}
    vals = {}
    for k in ("x", "w", "dy"):
        v = _draw(c, ext[k][0], g)
        inp[k].view.copy_(v)
        vals[k] = inp[k].view.double()          # the operands as stored
    x = canon_x(c, vals["x"]).requires_grad_(True)
    w = canon_w(c, vals["w"]).requires_grad_(True)
    dy = canon_x(c, vals["dy"])
    y_ref = agg_ref(x, w, c.desc)
    dx_ref, dw_ref = torch.autograd.grad(y_ref, (x, w), dy)
    ab = [None] * 3
    if c.kind == "float":
        xa, wa = x.detach().abs().requires_grad_(True), w.detach().abs().requires_grad_(True)
        ya = agg_ref(xa, wa, c.desc)
        ab = [ya.detach()] + list(torch.autograd.grad(ya, (xa, wa), dy.abs()))
    name = "%s (%s)" % (c.name, c.desc)

    y = Buf(ext["y"], c.offs["y"], dtype, float("nan"))
    _run(c, "fwd", lambda: _lib.check(lib.cotb200_agg_zeropad_fwd(d, inp["x"].ptr(), inp["w"].ptr(), y.ptr(), _st()), "agg fwd"))
    torch.cuda.synchronize()
    _compare(c, name + " y", canon_x(c, y.view), y_ref.detach(), ab[0])
    y.check_padding(name + " y")
    for call, want_dx, want_dw in BWD_VARIANTS:
        dx = Buf(ext["dx"], c.offs["dx"], dtype, float("nan")) if want_dx else None
        dw = Buf(ext["dw"], c.offs["dw"], dtype, float("nan")) if want_dw else None
        _run(c, call, lambda: _lib.check(lib.cotb200_agg_zeropad_bwd(
            d, inp["dy"].ptr(), inp["x"].ptr(), inp["w"].ptr(), dx.ptr() if dx else None, dw.ptr() if dw else None, _st()), "agg bwd"))
        torch.cuda.synchronize()
        if dx:
            _compare(c, "%s dX [%s]" % (name, call), canon_x(c, dx.view), dx_ref, ab[1])
            dx.check_padding("%s dX [%s]" % (name, call))
        if dw:
            _compare(c, "%s dW [%s]" % (name, call), canon_w(c, dw.view), dw_ref, ab[2])
            dw.check_padding("%s dW [%s]" % (name, call))


@pytest.mark.parametrize("c", [c for c in CASES if c.op == "mix"], ids=lambda c: c.name)
def test_mix_case(c):
    """the mix op (3x3 and 5x5 halves of one [n, 2*heads*c, ho, wo] output): its fused forward, agg_mix_dx for 16-bit storage, and
    the two halves through bwd_impl (the 5x5 half accumulating into dX) for fp32 / fp64"""
    dtype, ext = TD[c.dt], tensor_extent(c)
    lib = _lib.load()
    d = _desc(c)
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, c.name)))
    inp, vals = {}, {}
    for k in ("x", "w1", "w2", "dy"):
        inp[k] = Buf(ext[k], c.offs[k], dtype, float("nan"))
        inp[k].view.copy_(_draw(c, ext[k][0], g))
        vals[k] = inp[k].view.double()
    x, w1, w2 = (vals[k].clone().requires_grad_(True) for k in ("x", "w1", "w2"))
    y_ref = mix_ref(x, w1, w2, c.desc)
    refs = torch.autograd.grad(y_ref, (x, w1, w2), vals["dy"])
    ab = [None] * 4
    if c.kind == "float":
        xa, w1a, w2a = (t.detach().abs().requires_grad_(True) for t in (x, w1, w2))
        ya = mix_ref(xa, w1a, w2a, c.desc)
        ab = [ya.detach()] + list(torch.autograd.grad(ya, (xa, w1a, w2a), vals["dy"].abs()))
    name = "%s (%s)" % (c.name, c.desc)
    y = Buf(ext["y"], c.offs["y"], dtype, float("nan"))
    _run(c, "fwd", lambda: _lib.check(lib.cotb200_agg_zeropad_mix_fwd(d, MIX_K2, MIX_K2, MIX_P2, MIX_P2, inp["x"].ptr(), inp["w1"].ptr(),
                                                                      inp["w2"].ptr(), y.ptr(), _st()), "mix fwd"))
    torch.cuda.synchronize()
    _compare(c, name + " y", y.view, y_ref.detach(), ab[0])
    for call, want_dx, want_dw in BWD_VARIANTS:
        outs = {k: Buf(ext[k], c.offs[k], dtype, float("nan")) for k, on in (("dx", want_dx), ("dw1", want_dw), ("dw2", want_dw)) if on}
        p = lambda k: outs[k].ptr() if k in outs else None
        _run(c, call, lambda: _lib.check(lib.cotb200_agg_zeropad_mix_bwd(
            d, MIX_K2, MIX_K2, MIX_P2, MIX_P2, inp["dy"].ptr(), inp["x"].ptr(), inp["w1"].ptr(), inp["w2"].ptr(), p("dx"), p("dw1"),
            p("dw2"), _st()), "mix bwd"))
        torch.cuda.synchronize()
        for k, ref, a in zip(("dx", "dw1", "dw2"), refs, ab[1:]):
            if k in outs:
                _compare(c, "%s %s [%s]" % (name, k, call), outs[k].view, ref, a)
                outs[k].check_padding("%s %s [%s]" % (name, k, call))
