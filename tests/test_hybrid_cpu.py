"""SE-CoTNetD trunks (cotnet_b200/backbone_hybrid.py) against the reference's model code -- CPU, host logic only.

The LocalConv op has no CPU implementation in the product (the reference bounces CPU tensors through the GPU too), so for
these structure / wiring tests the operator mirror is pointed at the oracle's Unfold identity, exactly like
oracle/ref_import.py does for the reference modules.  What is pinned here: state-dict layout (strict loads of reference
checkpoints), parameter counts of README.md:45-51, the block-type schedule (SplitAttn vs CoT layer), and bit-level
agreement of the forward pass with the reference's unmodified se_cotnetd_50 (golden logits; live model when the reference
tree is present)."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import agg_ref, make_golden, ref_import

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture()
def cpu_op(monkeypatch):
    az = importlib.import_module("cotnet_b200.aggregation_zeropad")
    monkeypatch.setattr(az, "aggregation_zeropad",
                        lambda i, w, kernel_size=3, stride=1, padding=0, dilation=1:
                        agg_ref.agg_zeropad_unfold(i, w, kernel_size, stride, padding, dilation))
    yield


def test_param_counts_and_block_schedule():
    from cotnet_b200 import backbone_hybrid as bh
    from cotnet_b200.cot_layer import CoTLayer
    want = {"se_cotnetd_50": 23.1, "se_cotnetd_101": 40.9, "se_cotnetd_152": 55.8}          # README.md:45-51 (M parameters)
    for name, mp in want.items():
        m = bh.MODELS[name]()
        n = sum(p.numel() for p in m.parameters()) / 1e6
        assert abs(n - mp) < 0.06, (name, n)
        # layer1/2: split attention only; layer3: CoT layer in the even blocks; layer4: CoT layer everywhere (:138-156)
        assert all(isinstance(b.conv2, bh.SplitAttnConv2d) for b in list(m.layer1) + list(m.layer2))
        assert [isinstance(b.conv2, CoTLayer) for b in m.layer3] == [i % 2 == 0 for i in range(len(m.layer3))]
        assert all(isinstance(b.conv2, CoTLayer) for b in m.layer4)
    m152 = bh.se_cotnetd_152()
    assert isinstance(m152.layer2[0].avd, bh.BlurPool2d) and not m152.layer2[0].avd_first


def test_golden_logits_se_cotnetd_50(cpu_op):
    """Mirror + seeded parameters == the reference's se_cotnetd_50 on the same parameters (fixture made by
    oracle/make_golden.py from the reference's own code)."""
    from cotnet_b200 import backbone_hybrid as bh
    g = np.load(os.path.join(GOLDEN, "se_cotnetd50_eval_logits.npz"))
    m = make_golden.hybrid_seeded_state(bh.se_cotnetd_50(), int(g["seed"])).eval()
    assert sum(p.numel() for p in m.parameters()) == int(g["n_params"])
    with torch.no_grad():
        y = m(torch.from_numpy(g["x"]))
    err = (y - torch.from_numpy(g["logits"])).abs().max().item()
    assert err <= 1e-5, err


def test_stored_reference_state_dict_and_train_step(cpu_op):
    """The state-dict layout of SE-CoTNetD-50/101/152 and one fp64 training step of SE-CoTNetD-50 (output, every parameter
    gradient, running statistics) against the reference's model code, as stored in tests/golden/se_cotnetd50_train_fp64.npz
    (oracle/make_golden.py); test_live_reference_state_dict_and_forward checks the same live where a reference checkout exists."""
    import json
    from cotnet_b200 import backbone_hybrid as bh
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "se_cotnetd50_train_fp64.npz"))
    for name in ("se_cotnetd_50", "se_cotnetd_101", "se_cotnetd_152"):
        want = json.loads(bytes(g["layout/" + name]).decode())
        assert [[k, list(v.shape)] for k, v in bh.MODELS[name]().state_dict().items()] == want, name
    m = make_golden.hybrid_seeded_state(bh.se_cotnetd_50(zero_init_last_bn=False), make_golden.HYBRID_TRAIN_SEED).double()
    y, grads, run = make_golden.hybrid_train_record(m)
    assert np.abs(y - g["y"]).max() <= 1e-10 * max(1.0, np.abs(g["y"]).max())
    scale = np.abs(g["grads"]).max(axis=0)
    assert (np.abs(grads - g["grads"]) <= 1e-9 * scale + 1e-300).all()
    assert np.allclose(run, g["running"], rtol=1e-12, atol=1e-12)


@pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")
def test_live_reference_state_dict_and_forward(cpu_op):
    from cotnet_b200 import backbone_hybrid as bh
    ns = ref_import.load()
    for name in ("se_cotnetd_50", "se_cotnetd_101", "se_cotnetd_152"):
        ref, m = getattr(ns.hybrid, name)(), bh.MODELS[name]()
        a, b = ref.state_dict(), m.state_dict()
        assert list(a.keys()) == list(b.keys()), name                                       # same names, same order
        assert all(a[k].shape == b[k].shape for k in a), name
    ref = ns.hybrid.se_cotnetd_50(zero_init_last_bn=False).double()
    m = bh.se_cotnetd_50(zero_init_last_bn=False).double()
    m.load_state_dict(ref.state_dict(), strict=True)
    x = torch.randn(2, 3, 64, 64, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
    cot = torch.randn(2, 1000, dtype=torch.float64, generator=torch.Generator().manual_seed(6))
    ref.train(); m.train()
    yr, ym = ref(x), m(x)
    assert (yr - ym).abs().max().item() <= 1e-12
    gr = torch.autograd.grad((yr * cot).sum(), list(ref.parameters()))
    gm = torch.autograd.grad((ym * cot).sum(), list(m.parameters()))
    scale = max(t.abs().max().item() for t in gr)
    assert max((a_ - b_).abs().max().item() for a_, b_ in zip(gr, gm)) <= 1e-10 * scale
    for (k, v), (_, w) in zip(ref.state_dict().items(), m.state_dict().items()):           # running statistics moved alike
        if k.endswith("running_mean") or k.endswith("running_var"):
            assert torch.allclose(v, w, atol=1e-12), k
