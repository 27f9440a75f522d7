"""Parity of libcotb200 against the REFERENCE'S OWN GPU kernels on identical inputs.

The reference's kernel sources (cupy_layers/aggregation_zeropad.py:20-110, aggregation_zeropad_mix.py:20-207), compiled by
oracle/build_ref_kernels.py exactly as its `load_kernel` would at first use and launched like :140-143, were run on these
seeded inputs by oracle/ref_golden.py; tests/golden/ref_kernels.npz holds their outputs at 1024 seeded positions per array,
and the tests compare ours at the same positions.  This is the bar BASELINE.json
states: "outputs must match the reference CuPy aggregation_zeropad path on identical inputs within 1e-3 (fp32) /
1e-2 (bf16)"; fp64 keeps the reference self-test gate 1e-9.  Also cross-checks the CPU oracle against the same kernels.
"""
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
    """a: our full output; b: the reference's values at the stored positions"""
    a = sampled(a)
    err = (a - b.double()).abs()
    assert bool((err <= tol + tol * b.double().abs()).all()), "%s: max err %.3e" % (what, err.max().item())


AGG_CASES = [("cfg1", "float"), ("cfg1", "double"), ("selftest_k5", "double"), ("selftest_k1", "double"), ("ragged", "float"),
             ("ragged", "double"), ("s1_b8", "float"), ("s1_b256", "float"), ("s2_b256", "float"), ("s3_b256", "float"),
             ("s4_b256", "float")]


@pytest.mark.parametrize("tag,dtype", AGG_CASES)
def test_agg_matches_reference_kernels(tag, dtype):
    import cotnet_b200
    e, x, w, dy = rk().make_inputs(tag, dtype)
    y_ref, dx_ref, dw_ref = [rk().ref("agg", tag, dtype, 0, n) for n in ("y", "dx", "dw")]
    _close(x, rk().ref("agg", tag, dtype, 0, "x"), 0, "inputs")
    xo, wo = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = cotnet_b200.aggregation_zeropad(xo, wo, e["k"], 1, e["pad"], 1)
    dx, dw = torch.autograd.grad(y, (xo, wo), dy)
    tol = TOL[dtype]
    _close(y, y_ref, tol, "forward")
    _close(dx, dx_ref, tol, "dX")
    _close(dw, dw_ref, tol, "dW")
    assert y.shape == (e["N"], e["heads"] * e["C"], e["Ho"], e["Wo"]) and y.dtype == x.dtype and y.is_contiguous()


@pytest.mark.parametrize("tag", ["s1_b8", "s2_b256", "s4_b256", "cfg1"])
def test_agg_bf16_channels_last_vs_reference_kernels(tag):
    """The production layout (bf16, channels_last) against the reference's fp32 NCHW kernels fed the same bf16-representable
    values: 1e-2."""
    import cotnet_b200
    e, x, w, dy = rk().make_inputs(tag, "float", seed=3)
    x, w, dy = [t.to(torch.bfloat16).float() for t in (x, w, dy)]
    _close(x, rk().ref("agg_bf16", tag, "float", 3, "x"), 0, "inputs")
    y_ref, dx_ref, dw_ref = [rk().ref("agg_bf16", tag, "float", 3, n) for n in ("y", "dx", "dw")]
    xo = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wo = w.to(torch.bfloat16).permute(0, 4, 5, 1, 2, 3).contiguous().permute(0, 3, 4, 5, 1, 2).requires_grad_(True)
    y = cotnet_b200.aggregation_zeropad(xo, wo, 3, 1, 1, 1)
    dx, dw = torch.autograd.grad(y, (xo, wo), dy.to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
    _close(y, y_ref, 1e-2, "forward")
    _close(dx, dx_ref, 1e-2, "dX")
    # dW sums 8 products of O(1) values: judge relative to the typical magnitude like the other bf16 tests
    err = (sampled(dw) - dw_ref).abs()
    assert bool((err <= 2e-2 + 1e-2 * dw_ref.double().abs()).all()), "dW: max err %.3e" % err.max().item()


@pytest.mark.parametrize("tag,dtype", [("mix_selftest", "double"), ("mix_selftest", "float"), ("mix_s1_b32", "float")])
def test_mix_matches_reference_kernels(tag, dtype):
    import cotnet_b200
    e, x, w1, w2, dy = rk().make_inputs(tag, dtype, op="mix")
    _close(x, rk().ref("mix", tag, dtype, 0, "x"), 0, "inputs")
    y_ref, dx_ref, dw1_ref, dw2_ref = [rk().ref("mix", tag, dtype, 0, n) for n in ("y", "dx", "dw1", "dw2")]
    xo, w1o, w2o = [t.clone().requires_grad_(True) for t in (x, w1, w2)]
    y = cotnet_b200.aggregation_zeropad_mix(xo, w1o, w2o, 3, 5, 1, 1, 2, 1)
    dx, dw1, dw2 = torch.autograd.grad(y, (xo, w1o, w2o), dy)
    tol = TOL[dtype]
    _close(y, y_ref, tol, "forward")
    _close(dw1, dw1_ref, tol, "dW1")
    _close(dw2, dw2_ref, tol, "dW2")
    # heads == 1 (the only in-tree use): the reference's input gradient, which visits head 0 only
    # (aggregation_zeropad_mix.py:88), is the full gradient
    _close(dx, dx_ref, tol, "dX")


@pytest.mark.parametrize("tag,dtype", [("cfg1", "double"), ("selftest_k5", "double"), ("ragged", "double")])
def test_cpu_oracle_matches_reference_kernels(tag, dtype):
    """Pins oracle/agg_ref.py (the CPU restatement every other parity test trusts) to the reference's real kernels."""
    e, x, w, dy = rk().make_inputs(tag, dtype, seed=5)
    _close(x, rk().ref("agg", tag, dtype, 5, "x"), 0, "inputs")
    y_ref, dx_ref, dw_ref = [rk().ref("agg", tag, dtype, 5, n) for n in ("y", "dx", "dw")]
    xc, wc = x.cpu().requires_grad_(True), w.cpu().requires_grad_(True)
    yo = agg_ref.agg_zeropad_unfold(xc, wc, e["k"], 1, e["pad"], 1)
    dxo, dwo = torch.autograd.grad(yo, (xc, wc), dy.cpu())
    for a, b, n in ((yo, y_ref, "forward"), (dxo, dx_ref, "dX"), (dwo, dw_ref, "dW")):
        _close(a, b, 1e-9, "oracle " + n)
