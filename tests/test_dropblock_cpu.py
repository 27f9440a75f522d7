"""DropBlock without a GPU: the host restatement of the library's stream, mask, count and scale against the reference's own
drop_block_fast_2d (tests/golden/dropblock.npz, tools/make_dropblock_golden.py), the models' DropBlock sites against the
reference modules', the unfused fp64 training step of both trunks against the reference's, the geometry errors and the C-ABI
argument checks."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, backbone, backbone_hybrid, dropblock
from oracle import agg_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "dropblock.npz"))
MODELS = dict(backbone.MODELS, **backbone_hybrid.MODELS)


@pytest.fixture()
def cpu_op(monkeypatch):
    """The LocalConv op has no CPU implementation: point it at the oracle's Unfold identity (as tests/test_hybrid_cpu.py does)."""
    az = importlib.import_module("cotnet_b200.aggregation_zeropad")
    monkeypatch.setattr(az, "aggregation_zeropad",
                        lambda i, w, kernel_size=3, stride=1, padding=0, dilation=1:
                        agg_ref.agg_zeropad_unfold(i, w, kernel_size, stride, padding, dilation))
    yield


def _geo(i):
    B, C, H, W, bs, gs, rate, site, k0, k1 = GOLDEN["geo_params"][i]
    return (int(B), int(C), int(H), int(W)), dropblock.DropBlock(rate, int(bs), gs), int(site), (int(k0), int(k1))


GEOS = range(len(GOLDEN["geo_params"]))


def test_philox_known_answer():
    """Philox4x32-10 at counter 0, key 0 (the Random123 known-answer vector)."""
    r = dropblock.philox4x32_10(np.zeros(1, dtype=np.uint64), 0, 0, 0)
    assert [int(v[0]) for v in r] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


@pytest.mark.parametrize("i", GEOS)
def test_host_mask_count_and_scale_equal_reference(i):
    shape, spec, site, key = _geo(i)
    keep, count, scale = dropblock.host_mask(shape, site, key, spec)
    assert np.array_equal(keep, GOLDEN["geo%d_keep" % i])
    assert count == int(GOLDEN["geo%d_count" % i])
    assert np.float32(scale).view(np.int32) == np.float32(GOLDEN["geo%d_scale" % i]).view(np.int32)


def test_geometries_cover_the_edge_counts():
    counts = {int(GOLDEN["geo%d_count" % i]) for i in GEOS}
    assert 0 in counts and 1 in counts
    sizes = {int(p) for p in GOLDEN["geo_params"][:, 4]}
    assert sizes == {1, 3, 5}


@pytest.mark.parametrize("i", GEOS)
def test_unfused_forward_and_backward_equal_reference_bits(i):
    shape, spec, site, key = _geo(i)
    x = torch.from_numpy(GOLDEN["geo%d_x" % i]).requires_grad_(True)
    y = dropblock.drop_block(x, torch.tensor(key, dtype=torch.int64), site, spec)
    y.backward(torch.from_numpy(GOLDEN["geo%d_dy" % i]))
    assert np.array_equal(y.detach().numpy().view(np.int32), GOLDEN["geo%d_y" % i].view(np.int32))
    assert np.array_equal(x.grad.numpy().view(np.int32), GOLDEN["geo%d_dx" % i].view(np.int32))


def _site_shapes(model, res):
    """(block_size, gamma_scale, C, H, W) of each DropBlock call of a training forward at res x res, batch 2."""
    calls = []
    orig = dropblock.drop_block

    def rec(x, key, site, spec):
        assert site == len(calls)
        calls.append((spec.block_size, spec.gamma_scale) + tuple(x.shape[1:]))
        return x
    model.fixed_drop_block_key = torch.tensor([1, 2])
    dropblock.drop_block = rec
    try:
        with torch.no_grad():
            model(torch.randn(2, 3, res, res))
    finally:
        dropblock.drop_block = orig
    return calls


@pytest.mark.parametrize("name", sorted(MODELS))
def test_site_table_equals_reference(name, monkeypatch):
    from cotnet_b200 import cot_layer
    for cls in (cot_layer.CotLayer, cot_layer.CoXtLayer, cot_layer.CoTLayer):       # shape-preserving; only the shapes matter here
        monkeypatch.setattr(cls, "forward", lambda self, x: x)
    torch.manual_seed(0)
    m = MODELS[name](num_classes=10, drop_block_rate=0.1).train()
    for res in (128, 224, 320):
        got = np.array(_site_shapes(m, res), dtype=np.float64)
        assert np.array_equal(got, GOLDEN["sites_%s_%d" % (name, res)]), (name, res)
    assert m.n_drop_block_sites == len(GOLDEN["sites_%s_128" % name]) == len(m.drop_block_table())


@pytest.mark.parametrize("fn", [backbone.cotnet50, backbone_hybrid.se_cotnetd_50])
def test_state_dict_unchanged_by_drop_block(fn):
    torch.manual_seed(0)
    a = fn(num_classes=10)
    torch.manual_seed(0)
    b = fn(num_classes=10, drop_block_rate=0.2)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    assert a.n_drop_block_sites == 0 and b.n_drop_block_sites > 0


@pytest.mark.parametrize("name", ["cotnet50", "se_cotnetd_50"])
def test_unfused_fp64_step_matches_reference(name, cpu_op):
    """One fp64 training step of the unfused path (CPU) with drop_block_rate 0.1 and the fixture's key against the reference's
    step with the same uniforms (tools/make_dropblock_golden.py:_step)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_dropblock_golden import step_input
    from oracle import make_golden
    pre = "step_%s_" % name
    seed = int(GOLDEN["step_seed"])
    torch.manual_seed(0)
    m = make_golden.hybrid_seeded_state(MODELS[name](drop_block_rate=float(GOLDEN["step_rate"])), seed)
    with torch.no_grad():
        for t in m.state_dict().values():
            if t.dtype.is_floating_point:
                t.copy_(t.bfloat16().float())
    m = m.double().train()
    m.fixed_drop_block_key = torch.from_numpy(GOLDEN["key"])
    assert m.n_drop_block_sites == int(GOLDEN[pre + "sites"])
    x, y = step_input()
    logp = torch.log_softmax(m(x.double()), dim=-1)
    s = float(GOLDEN["step_smoothing"])
    loss = (-(1 - s) * logp.gather(1, y.view(-1, 1)).squeeze(1) - s * logp.mean(-1)).mean()
    loss.backward()
    assert abs(loss.item() - float(GOLDEN[pre + "loss"])) <= 1e-9 * abs(float(GOLDEN[pre + "loss"]))
    names = [n for n, _ in m.named_parameters()]
    assert names == list(GOLDEN[pre + "names"])
    for i, (n, q) in enumerate(m.named_parameters()):
        gn, gp = q.grad.norm().item(), (q.grad * make_golden.proj_vector(n, q.shape, seed)).sum().item()
        assert abs(gn - GOLDEN[pre + "gnorm"][i]) <= 1e-7 * GOLDEN[pre + "gnorm"][i] + 1e-12, n
        assert abs(gp - GOLDEN[pre + "gproj"][i]) <= 1e-7 * GOLDEN[pre + "gnorm"][i] + 1e-12, n


def test_geometry_errors(cpu_op):
    st3, st4 = dropblock.stage_drop_blocks(0.1)[2:]
    with pytest.raises(ValueError, match="site 7.*even"):
        st3.geometry(4, 4, 7)                              # cbs 4: the reference's pooled mask is 5x5
    with pytest.raises(ValueError, match="even"):
        st4.geometry(2, 9, 0)
    with pytest.raises(ValueError, match="site 3.*no valid"):
        st3.geometry(3, 4, 3)                              # (W - 5 + 1) == 0
    assert st3.geometry(3, 5, 0)[0] == 3 and st4.geometry(1, 1, 0)[0] == 1
    assert dropblock.stage_drop_blocks(0.)[2:] == [None, None]
    m = backbone.cotnet50(num_classes=10, drop_block_rate=0.1).train()
    with pytest.raises(ValueError, match="DropBlock site"):
        m(torch.randn(2, 3, 64, 64))
    m.eval()
    with torch.no_grad():
        m(torch.randn(2, 3, 64, 64))                       # eval mode: no DropBlock


def test_dropblock_argument_errors():
    """The DropBlock entry points reject bad arguments with the documented codes before any CUDA call."""
    lib = _lib.load()
    P, Q = 16, 18         # any non-NULL "pointer" (P 16-byte aligned, Q not): these calls must fail in validation
    EINVAL, EDTYPE, EALIGN, ENULL, ETOOBIG, EUNSUP = -1, -2, -4, -5, -6, -7
    K = 1 << 40          # the count "pointer" of the mask calls: aligned and far from the mask
    assert lib.cotb200_dropblock_mask(2, 16, 7, 7, 3, 0.1, 0, None, P, K, None) == ENULL
    assert lib.cotb200_dropblock_mask(2, 16, 7, 7, 3, 0.1, 0, P, P, None, None) == ENULL
    assert lib.cotb200_dropblock_mask(2, 16, 7, 7, 3, 0.1, 0, P, P, K + 2, None) == EALIGN    # count not 4-byte aligned
    assert lib.cotb200_dropblock_mask(2, 16, 7, 7, 3, 0.1, 0, P + 4, P, K, None) == EALIGN    # key not 8-byte aligned
    assert lib.cotb200_dropblock_mask(2, 16, 7, 7, 3, 0.1, 0, P, K, K + 192, None) == EINVAL  # count inside the 196-byte mask
    assert lib.cotb200_dropblock_mask(2, 12, 7, 7, 3, 0.1, 0, P, P, K, None) == EINVAL       # C % 8
    assert lib.cotb200_dropblock_mask(2, 16, 7, 7, 4, 0.1, 0, P, P, K, None) == EINVAL       # even block
    assert lib.cotb200_dropblock_mask(2, 16, 2, 7, 3, 0.1, 0, P, P, K, None) == EINVAL       # block larger than the plane
    assert lib.cotb200_dropblock_mask(2, 16, 7, 7, 3, float("nan"), 0, P, P, K, None) == EINVAL   # gamma NaN
    assert lib.cotb200_dropblock_mask(2, 16, 7, 7, 3, 0.1, -1, P, P, K, None) == EINVAL      # site
    assert lib.cotb200_dropblock_mask(4096, 4096, 400, 400, 3, 0.1, 0, P, P, K, None) == ETOOBIG
    # shared memory: 32 bytes of per-warp counts + 2 bytes per pixel and 8 channels must fit 48 KB, so one 8-channel group takes
    # planes up to 24560 pixels; 24561 .. 24576 (the planes where the counts tipped the kernel over 48 KB) and beyond are refused
    for H, W in ((1, 24561), (96, 256), (200, 200)):
        assert lib.cotb200_dropblock_mask(1, 8, H, W, 1, 0.1, 0, P, P, K, None) == EUNSUP, (H, W)
    assert lib.cotb200_dropblock_apply(_lib.BF16, 2, 49, 16, P, None, P, P, None) == ENULL
    assert lib.cotb200_dropblock_apply(_lib.F64, 2, 49, 16, P, P, P, P, None) == EDTYPE
    assert lib.cotb200_dropblock_apply(_lib.BF16, 2, 49, 12, P, P, P, P, None) == EINVAL
    assert lib.cotb200_dropblock_apply(_lib.BF16, 2, 49, 16, Q, P, P, P, None) == EALIGN
    assert lib.cotb200_dropblock_res_relu(_lib.BF16, 2, 49, 16, P, P, P, P, None, P, None, None) == ENULL
    assert lib.cotb200_dropblock_res_relu(_lib.F32, 0, 49, 16, P, P, P, P, None, P, P, None) == EINVAL
    assert lib.cotb200_dropblock_res_relu(_lib.BF16, 2, 49, 16, P, Q, P, P, None, P, P, None) == EALIGN
    assert lib.cotb200_dropblock_res_relu_bwd(_lib.BF16, 2, 49, 16, P, P, P, P, None, None, None, None) == ENULL
    assert lib.cotb200_dropblock_res_relu_bwd(_lib.F16, 2, 49, 16, P, P, P, P, None, Q, P, None) == EALIGN
    assert lib.cotb200_dropblock_res_relu_bwd(9, 2, 49, 16, P, P, P, P, None, None, P, None) == EDTYPE
    assert lib.cotb200_last_error()
