"""The remaining cupy_layers variants (SURVEY.md section 8f rank 4) -- aggregation_refpad, aggregation_zeropad_dilate,
aggregation_zeropad_mix_merge -- against (a) the REFERENCE'S OWN kernels (incl. the reference's host-side border fold for the
refpad input gradient), as their outputs stored at seeded positions in tests/golden/ref_kernels.npz (oracle/ref_golden.py), and (b) the CPU oracle's Unfold identities, which are the
right-hand sides of the reference's self-tests (aggregation_refpad.py:223-251, aggregation_zeropad_dilate.py:258-306,
aggregation_zeropad_mix_merge.py:332-366).  Gates: fp64 1e-9 (the reference's own), fp32 1e-3, bf16 1e-2."""
import pytest
import torch

from oracle import agg_ref, ref_golden
from oracle.ref_golden import sampled

pytestmark = pytest.mark.gpu

TOL = {"double": 1e-9, "float": 1e-3}
_RK = {}


def rk():
    if "k" not in _RK:
        _RK["k"] = ref_golden.GoldenRef()
    return _RK["k"]


def _close(a, b, tol, what):
    err = (a.double() - b.double()).abs()
    assert bool((err <= tol + tol * b.double().abs()).all()), "%s: max err %.3e" % (what, err.max().item())


@pytest.mark.parametrize("tag,dtype", [("refpad_selftest", "double"), ("refpad_selftest", "float"), ("refpad_k3", "double"),
                                       ("refpad_k3", "float"), ("refpad_s2_b8", "float")])
def test_refpad_matches_reference_kernels(tag, dtype):
    import cotnet_b200
    e, x, w, dy = rk().make_variant_inputs(tag, dtype, "refpad")
    _close(sampled(x), rk().ref("refpad", tag, dtype, 0, "x"), 0, "inputs")
    y_ref, dx_ref, dw_ref = [rk().ref("refpad", tag, dtype, 0, n) for n in ("y", "dx", "dw")]
    xo, wo = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = cotnet_b200.aggregation_refpad(xo, wo, e["k"], 1, e["pad"], 1)
    dx, dw = torch.autograd.grad(y, (xo, wo), dy)
    tol = TOL[dtype]
    _close(sampled(y), y_ref, tol, "forward")
    _close(sampled(dx), dx_ref, tol, "dX")
    _close(sampled(dw), dw_ref, tol, "dW")


@pytest.mark.parametrize("tag,dtype", [("dilate_selftest", "double"), ("dilate_selftest", "float"), ("dilate_s2_b8", "float")])
def test_dilate_matches_reference_kernels(tag, dtype):
    import cotnet_b200
    e, x, w, dil, dy = rk().make_variant_inputs(tag, dtype, "dilate")
    _close(sampled(x), rk().ref("dilate", tag, dtype, 0, "x"), 0, "inputs")
    y_ref, dx_ref, dw_ref = [rk().ref("dilate", tag, dtype, 0, n) for n in ("y", "dx", "dw")]
    xo, wo = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = cotnet_b200.aggregation_zeropad_dilate(xo, wo, dil, 3, 1)
    dx, dw = torch.autograd.grad(y, (xo, wo), dy)
    tol = TOL[dtype]
    _close(sampled(y), y_ref, tol, "forward")
    _close(sampled(dx), dx_ref, tol, "dX")
    _close(sampled(dw), dw_ref, tol, "dW")


@pytest.mark.parametrize("tag,dtype", [("merge_selftest", "double"), ("merge_selftest", "float"), ("merge_s1_b8", "float")])
def test_mix_merge_matches_reference_kernels(tag, dtype):
    import cotnet_b200
    e, x, w, dy = rk().make_variant_inputs(tag, dtype, "merge")
    _close(sampled(x), rk().ref("merge", tag, dtype, 0, "x"), 0, "inputs")
    y_ref, dx_ref, dw_ref = [rk().ref("merge", tag, dtype, 0, n) for n in ("y", "dx", "dw")]
    xo, wo = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = cotnet_b200.aggregation_zeropad_mix_merge(xo, wo, e["heads"], e["wc"], 3, 5, 1, 1, 2, 1)
    dx, dw = torch.autograd.grad(y, (xo, wo), dy)
    tol = TOL[dtype]
    _close(sampled(y), y_ref, tol, "forward")
    _close(sampled(dx), dx_ref, tol, "dX")
    _close(sampled(dw), dw_ref, tol, "dW")


# ---------------------------------------------------------------- vs the CPU oracle (runs also where oracle/_ref is absent)
def _rand(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=torch.float64).to(dtype)


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-9), (torch.float32, 1e-3), (torch.bfloat16, 1e-2)])
@pytest.mark.parametrize("k,pad,stride,dil,H,W", [(5, 2, 1, 1, 9, 9), (3, 1, 1, 1, 7, 5), (3, 2, 1, 2, 8, 8), (3, 1, 2, 1, 9, 8)])
def test_refpad_vs_oracle(dtype, tol, k, pad, stride, dil, H, W):
    import cotnet_b200
    n, c, wc, heads = 2, 8, 4, 2
    Ho, Wo = agg_ref.out_size(H, W, k, stride, pad, dil)
    x, w = _rand((n, c, H, W), dtype, 1), _rand((n, heads, wc, k * k, Ho, Wo), dtype, 2)
    dy = _rand((n, heads * c, Ho, Wo), dtype, 3)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yr = agg_ref.agg_refpad_unfold(xr, wr, k, stride, pad, dil)
    dxr, dwr = torch.autograd.grad(yr, (xr, wr), dy.double())
    xo, wo = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    y = cotnet_b200.aggregation_refpad(xo, wo, k, stride, pad, dil)
    dx, dw = torch.autograd.grad(y, (xo, wo), dy.cuda())
    scale = 1.0 if dtype != torch.bfloat16 else 4.0          # sums of k*k (x heads x reflected duplicates) O(1) products
    _close(y.cpu(), yr.detach(), tol * scale, "forward")
    _close(dx.cpu(), dxr, tol * scale, "dX")
    _close(dw.cpu(), dwr, tol * scale, "dW")


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-9), (torch.float32, 1e-3), (torch.bfloat16, 1e-2)])
def test_dilate_vs_oracle(dtype, tol):
    import cotnet_b200
    n, c, wc, heads, H, W = 2, 8, 4, 2, 7, 7
    dil = [1, 1, 2, 4]
    x, w = _rand((n, c, H, W), dtype, 4), _rand((n, heads, wc, 9, H, W), dtype, 5)
    dy = _rand((n, heads * c, H, W), dtype, 6)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yr = agg_ref.agg_dilate_unfold(xr, wr, dil)
    dxr, dwr = torch.autograd.grad(yr, (xr, wr), dy.double())
    xo, wo = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    y = cotnet_b200.aggregation_zeropad_dilate(xo, wo, torch.tensor(dil, dtype=dtype, device="cuda"), 3, 1)
    dx, dw = torch.autograd.grad(y, (xo, wo), dy.cuda())
    scale = 1.0 if dtype != torch.bfloat16 else 4.0
    _close(y.cpu(), yr.detach(), tol * scale, "forward")
    _close(dx.cpu(), dxr, tol * scale, "dX")
    _close(dw.cpu(), dwr, tol * scale, "dW")


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-9), (torch.float32, 1e-3), (torch.bfloat16, 1e-2)])
def test_mix_merge_vs_oracle(dtype, tol):
    import cotnet_b200
    n, c, wc, heads, H, W = 2, 8, 4, 2, 6, 6
    x, w = _rand((n, c, H, W), dtype, 7), _rand((n, heads * wc * 34, H, W), dtype, 8)
    dy = _rand((n, 2 * heads * c, H, W), dtype, 9)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yr = agg_ref.agg_zeropad_mix_merge_unfold(xr, wr, heads, wc, 3, 5, 1, 1, 2, 1)
    dxr, dwr = torch.autograd.grad(yr, (xr, wr), dy.double())
    xo, wo = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    y = cotnet_b200.aggregation_zeropad_mix_merge(xo, wo, heads, wc, 3, 5, 1, 1, 2, 1)
    dx, dw = torch.autograd.grad(y, (xo, wo), dy.cuda())
    scale = 1.0 if dtype != torch.bfloat16 else 8.0          # dX sums 34 x heads products
    _close(y.cpu(), yr.detach(), tol * scale, "forward")
    _close(dx.cpu(), dxr, tol * scale, "dX")
    _close(dw.cpu(), dwr, tol * scale, "dW")


def test_variants_gradcheck_fp64():
    """The reference's self-tests end with torch.autograd.gradcheck (refpad :251, dilate :306)."""
    import cotnet_b200
    from functools import partial
    x = torch.randn(1, 4, 5, 5, dtype=torch.float64, device="cuda", requires_grad=True)
    w = torch.randn(1, 1, 2, 9, 5, 5, dtype=torch.float64, device="cuda", requires_grad=True)
    assert torch.autograd.gradcheck(partial(cotnet_b200.aggregation_refpad, kernel_size=3, stride=1, padding=1, dilation=1), (x, w))
    dil = torch.tensor([1, 2], dtype=torch.float64, device="cuda")
    assert torch.autograd.gradcheck(lambda a, b: cotnet_b200.aggregation_zeropad_dilate(a, b, dil, 3, 1), (x, w))
    wm = torch.randn(1, 2 * 34, 5, 5, dtype=torch.float64, device="cuda", requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, b: cotnet_b200.aggregation_zeropad_mix_merge(a, b, 1, 2, 3, 5, 1, 1, 2, 1), (x, wm))


def test_variant_argument_errors():
    import cotnet_b200
    x = torch.randn(1, 4, 3, 3, device="cuda")
    w = torch.randn(1, 1, 2, 9, 3, 3, device="cuda")
    with pytest.raises(RuntimeError, match="reflect padding"):
        cotnet_b200.aggregation_refpad(x, torch.randn(1, 1, 2, 49, 3, 3, device="cuda"), 7, 1, 3, 1)     # pad 3 >= H 3
    with pytest.raises(AssertionError):
        cotnet_b200.aggregation_zeropad_dilate(x, w, torch.ones(3, device="cuda"), 3, 1)                  # dilation.shape[0] != wc
    with pytest.raises(AssertionError):
        cotnet_b200.aggregation_zeropad_mix_merge(x, torch.randn(1, 10, 3, 3, device="cuda"), 1, 2)      # packed channel count
