"""Every kernel the refpad, dilate and mix_merge dispatch can pick, through the C ABI, at the cases of
tests/test_variant_geometry_cpu.py, against the fp64 Unfold oracle (oracle/agg_ref.py).

Each case makes four calls: the forward and the backward with both gradients, with dX only and with dW only (the other pointer
NULL).  Every call runs inside the library's profiler and must open exactly the profiler records the Python mirror of the dispatch
predicts, and launch exactly as many kernels; before that, the case's predicted grid-stride passes are checked on this device's
own SM count.  Outputs are prefilled with NaN.

Integer cases draw operands from [-a, a] with a chosen from the case's largest number of products per sum (amplitude), so every
sum, every fp32 partial sum and the final rounding are exact: the outputs must equal the oracle rounded to the storage type, bit
for bit.  Float cases draw random operands and bound |got - ref| by the unit roundoff of the storage type times |ref| plus that of
the accumulator times the number of products times the sum of |terms| (the oracle on |operands|)."""
import pytest
import torch

from cotnet_b200 import _lib
from oracle import agg_ref
from test_variant_geometry_cpu import BWD_VARIANTS, SMS_H100, VCASES, amplitude, max_terms, predict, profile_names

pytestmark = pytest.mark.gpu

TD = {"fp32": torch.float32, "fp64": torch.float64, "bf16": torch.bfloat16, "fp16": torch.float16}
U_STORE = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11, "fp32": 2.0 ** -24, "fp64": 2.0 ** -53}
U_ACC = {"bf16": 2.0 ** -24, "fp16": 2.0 ** -24, "fp32": 2.0 ** -24, "fp64": 2.0 ** -53}
TINY = {"bf16": 2.0 ** -134, "fp16": 2.0 ** -25, "fp32": 2.0 ** -150, "fp64": 0.0}     # half the smallest subnormal


def _st():
    return torch.cuda.current_stream().cuda_stream


def _desc(c):
    d = _lib.AggDesc()
    for k, v in c.desc.fields().items():
        setattr(d, k, v)
    d.dtype = _lib.dtype_code(torch.empty(0, dtype=TD[c.dt]))
    return d


def _shapes(d):
    K2 = d.kh * d.kw
    if d.op == "merge":
        w = (d.n, d.heads * d.wc * (K2 + d.k2 * d.k2), d.ho, d.wo)
        y = (d.n, 2 * d.heads * d.c, d.ho, d.wo)
    else:
        w = (d.n, d.heads, d.wc, K2, d.ho, d.wo)
        y = (d.n, d.heads * d.c, d.ho, d.wo)
    return (d.n, d.c, d.h, d.w), w, y


def _apply(d, x, w, dil):
    """the fp64 Unfold oracle of one call"""
    if d.op == "refpad":
        return agg_ref.agg_refpad_unfold(x, w, (d.kh, d.kw), (d.sh, d.sw), (d.ph, d.pw), (d.dh, d.dw))
    if d.op == "dilate":
        return agg_ref.agg_dilate_unfold(x, w, dil)
    return agg_ref.agg_zeropad_mix_merge_unfold(x, w, d.heads, d.wc, d.kh, d.k2, d.sh, d.ph, d.p2, d.dh)


def oracle(d, x, w, dy):
    """(y, dX, dW) in fp64, sample by sample (each sample's outputs depend on that sample alone)"""
    ys, dxs, dws = [], [], []
    for n in range(d.n):
        xs, ws = x[n:n + 1].clone().requires_grad_(True), w[n:n + 1].clone().requires_grad_(True)
        y = _apply(d, xs, ws, d.dil)
        gx, gw = torch.autograd.grad(y, (xs, ws), dy[n:n + 1])
        ys.append(y.detach())
        dxs.append(gx)
        dws.append(gw)
    return torch.cat(ys), torch.cat(dxs), torch.cat(dws)


def _draw(c, shape, g):
    if c.kind == "float":
        return torch.randn(shape, generator=g, device="cuda", dtype=torch.float64).to(TD[c.dt])
    a = amplitude(c)
    return torch.randint(-a, a + 1, shape, generator=g, device="cuda").to(TD[c.dt])


def _check(c, what, got, ref, absterms):
    assert not bool(got.isnan().any()), "%s: %d elements never written" % (what, int(got.isnan().sum()))
    if c.kind == "int":
        want = ref.to(got.dtype)
        assert torch.equal(want.double(), ref), "%s: the oracle is not exact in %s" % (what, c.dt)
        if not torch.equal(got, want):
            bad = (got != want).nonzero()[:4].tolist()
            raise AssertionError("%s: %d of %d elements differ, first %s: got %s want %s" % (
                what, int((got != want).sum()), got.numel(), bad, [got[tuple(i)].item() for i in bad],
                [want[tuple(i)].item() for i in bad]))
        return
    err = (got.double() - ref).abs()
    lim = U_STORE[c.dt] * ref.abs() + (max_terms(c.desc) + 2) * U_ACC[c.dt] * absterms + TINY[c.dt]
    bad = ~(err <= lim)
    assert not bool(bad.any()), "%s: %d of %d elements off; worst err/limit %.3g" % (
        what, int(bad.sum()), bad.numel(), float((err / lim).max()))


def _run(c, call, fn):
    """fn() under the profiler: the records and the number of launches must be the mirror's"""
    launches = predict(c)[call]
    want = profile_names(launches)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    _lib.prof_enable(True)
    try:
        fn()
        got = {k: v[0] for k, v in _lib.prof_report().items()}
    finally:
        _lib.prof_enable(False)
    assert got == want, "%s %s: profiled %s, the dispatch mirror predicts %s" % (c.name, call, got, want)
    assert _lib.launch_count() - n0 == len(launches), "%s %s: %d launches, the mirror predicts %d" % (
        c.name, call, _lib.launch_count() - n0, len(launches))


@pytest.mark.parametrize("c", VCASES, ids=lambda c: c.name)
def test_variant_case(c):
    lib = _lib.load()
    d = c.desc
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    P = predict(c)
    for call, launches in P.items():
        for l in launches:
            print("%s %s: %s %s grid %d, %d grid-stride passes at %d SMs" % (
                c.name, call, l.kernel, "/".join(sorted(l.tags)), l.grid(sms), l.passes(sms), sms))
    if c.name.startswith("loop-") and sms <= max(SMS_H100):
        short = [l for l in P["fwd"] if l.passes(sms) < 2]
        assert not short, "%s: one grid-stride pass at %d SMs: %s" % (c.name, sms, short)

    dtype = TD[c.dt]
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, c.name)))
    xs, ws, ys = _shapes(d)
    x, w, dy = _draw(c, xs, g), _draw(c, ws, g), _draw(c, ys, g)
    dil_t = torch.tensor(d.dil, dtype=dtype, device="cuda") if d.op == "dilate" else None
    if dil_t is not None:
        assert dil_t.double().tolist() == [float(v) for v in d.dil]
    y_ref, dx_ref, dw_ref = oracle(d, x.double(), w.double(), dy.double())
    ab = (None, None, None)
    if c.kind == "float":
        ab = oracle(d, x.double().abs(), w.double().abs(), dy.double().abs())
    dsc = _desc(c)
    name = "%s (%s)" % (c.name, d)
    k2, p2 = d.k2, d.p2

    def fwd(out):
        if d.op == "refpad":
            return lib.cotb200_agg_refpad_fwd(dsc, x.data_ptr(), w.data_ptr(), out.data_ptr(), _st())
        if d.op == "dilate":
            return lib.cotb200_agg_zeropad_dilate_fwd(dsc, x.data_ptr(), w.data_ptr(), dil_t.data_ptr(), out.data_ptr(), _st())
        return lib.cotb200_agg_zeropad_mix_merge_fwd(dsc, k2, k2, p2, p2, x.data_ptr(), w.data_ptr(), out.data_ptr(), _st())

    def bwd(gx, gw):
        px, pw = _lib.ptr(gx), _lib.ptr(gw)
        if d.op == "refpad":
            return lib.cotb200_agg_refpad_bwd(dsc, dy.data_ptr(), x.data_ptr(), w.data_ptr(), px, pw, _st())
        if d.op == "dilate":
            return lib.cotb200_agg_zeropad_dilate_bwd(dsc, dy.data_ptr(), x.data_ptr(), w.data_ptr(), dil_t.data_ptr(), px, pw, _st())
        return lib.cotb200_agg_zeropad_mix_merge_bwd(dsc, k2, k2, p2, p2, dy.data_ptr(), x.data_ptr(), w.data_ptr(), px, pw, _st())

    y = torch.full(ys, float("nan"), dtype=dtype, device="cuda")
    _run(c, "fwd", lambda: _lib.check(fwd(y), "%s fwd" % d.op))
    torch.cuda.synchronize()
    _check(c, name + " y", y, y_ref, ab[0])
    for call, want_dx, want_dw in BWD_VARIANTS:
        gx = torch.full(xs, float("nan"), dtype=dtype, device="cuda") if want_dx else None
        gw = torch.full(ws, float("nan"), dtype=dtype, device="cuda") if want_dw else None
        _run(c, call, lambda: _lib.check(bwd(gx, gw), "%s bwd" % d.op))
        torch.cuda.synchronize()
        if gx is not None:
            _check(c, "%s dX [%s]" % (name, call), gx, dx_ref, ab[1])
        if gw is not None:
            _check(c, "%s dW [%s]" % (name, call), gw, dw_ref, ab[2])
