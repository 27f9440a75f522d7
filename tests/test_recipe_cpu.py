"""The training recipe's host logic on CPU: MixupCutmix draws against the reference's own FastCollateMixup draws
(tests/golden/recipe.npz, tools/make_recipe_golden.py), the per-block stochastic-depth rates against the reference's modules,
unchanged state dicts, and the argument checks of the new C entry points (no kernel is launched)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, backbone, backbone_hybrid, trainer
import mix_ref
from mix_ref import batch_row

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recipe.npz"))


def mix_batch(seed):
    """The seeded uint8 batch of the mixed-batch fixture (tools/make_recipe_golden.py:mix_batch)."""
    rng = np.random.RandomState(1000 + seed)
    x = rng.randint(0, 256, size=(4, 3, 16, 20)).astype(np.uint8)
    return x, rng.randint(0, 1000, size=4).astype(np.int64)


@pytest.mark.parametrize("key,prob", [("draws_p1", 1.0), ("draws_p05", 0.5)])
def test_batch_tables_equal_reference_draws(key, prob):
    """lam (box-corrected for CutMix), the CutMix switch and the box of every seed, exactly, on every row of the table."""
    want = GOLDEN[key]
    modes = set()
    for seed, (lam, use_cutmix, yl, yh, xl, xh) in enumerate(want):
        mc = trainer.MixupCutmix(0.8, 1.0, prob=prob, switch_prob=0.5, label_smoothing=0.1, num_classes=1000, seed=seed, device=None)
        p = mc.draw(8, 128, 128)
        r = batch_row(p, 8)
        assert p.lam == lam and r.target_lam == float(np.float32(lam)), (seed, p.lam, lam)
        assert r.mode == (0 if lam == 1. else (2 if use_cutmix else 1)), seed
        if r.mode == 2:
            assert (r.y0, r.y1, r.x0, r.x1) == (yl, yh, xl, xh), seed
        if r.mode == 1:
            assert r.lam == float(np.float32(lam)) and r.one_minus_lam == float(np.float32(1 - lam))
        modes.add(r.mode)
    assert modes == ({1, 2} if prob == 1.0 else {0, 1, 2})


def test_batch_tables_reproduce_the_golden_batches():
    """The draws that made the stored mixed batches (4 x 3 x 16 x 20), and the numpy arithmetic of the reference on them."""
    for kind, mode in (("mixup", 1), ("cutmix", 2)):
        seed = int(GOLDEN[kind + "_seed"])
        x, labels = mix_batch(seed)
        p = trainer.MixupCutmix(seed=seed, device=None).draw(*x.shape[:1], *x.shape[2:])
        r = batch_row(p, x.shape[0])
        assert r.mode == mode
        xp = x[::-1]
        if mode == 1:
            want = np.rint(x.astype(np.float32) * np.float32(r.lam) + xp.astype(np.float32) * np.float32(r.one_minus_lam))
        else:
            y0, y1, x0, x1 = r.y0, r.y1, r.x0, r.x1
            want = x.copy()
            want[:, :, y0:y1, x0:x1] = xp[:, :, y0:y1, x0:x1]
        assert np.array_equal(want.astype(np.uint8), GOLDEN[kind + "_out"])
        assert np.array_equal(mix_ref.mixed_batch(x, p.host), GOLDEN[kind + "_out"])
        eye = np.eye(1000)
        t = 1e-4 + 0.9 * (p.lam * eye[labels] + (1 - p.lam) * eye[labels[::-1]])     # mixup_target, smoothing 0.1
        assert np.abs(t - GOLDEN[kind + "_target"]).max() < 1e-6


def test_mixup_disabled_table_and_odd_batch():
    mc = trainer.MixupCutmix(seed=0, device=None)
    mc.enabled = False
    state = mc.rng.get_state()[2]
    p = mc.draw(4, 8, 8)
    r = batch_row(p, 4)
    assert r.mode == 0 and r.target_lam == 1.0 and p.lam == 1.0 and mc.rng.get_state()[2] == state
    with pytest.raises(ValueError):
        mc.draw(5, 8, 8)
    with pytest.raises(ValueError):
        trainer.MixupCutmix(0., 0., device=None)


def test_batch_table_validation():
    """A batch-shaped table with an unknown mode, for an odd batch, or with a CutMix box outside the image is rejected: by
    MixRows.check or by cotb200_u8_mix_rows_to_nhwc's host validation, before any launch."""
    lib = _lib.load()
    P, EINVAL = 16, -1
    f3 = (ctypes.c_float * 3)(1, 1, 1)

    def u8(t, N):
        return lib.cotb200_u8_mix_rows_to_nhwc(_lib.BF16, N, t.n_out, 3, 8, 8, P, P, f3, f3, None, None, t.host, P, None)
    t = trainer.MixupCutmix(0.8, 0.0, device=None).draw(4, 8, 8)
    rows = np.frombuffer(t.host, dtype=np.dtype(_lib.MixRow))
    assert (rows["mode"] == 1).all()
    rows["mode"] = 3
    assert u8(t, 4) == EINVAL and b"unknown mode" in lib.cotb200_last_error()
    rows["mode"] = 1
    with pytest.raises(ValueError, match="drawn for 4"):
        t.check(5, 8, 8)
    odd = trainer.MixRows((_lib.MixRow * 5).from_buffer_copy(bytes(t.host) + bytes(t.host[0])), 5)
    assert u8(odd, 5) == EINVAL and b"must be even" in lib.cotb200_last_error()
    rows["mode"], rows["y0"], rows["y1"], rows["x0"], rows["x1"] = 2, 2, 9, 0, 4
    assert u8(t, 4) == EINVAL and b"box" in lib.cotb200_last_error()


@pytest.mark.parametrize("name,fn,rate", [("cotnet50", backbone.cotnet50, 0.1), ("cotnet101", backbone.cotnet101, 0.1),
                                          ("se_cotnetd_152", backbone_hybrid.se_cotnetd_152, 0.15)])
def test_drop_path_rates_equal_reference(name, fn, rate):
    m = fn(drop_path_rate=rate, num_classes=10)
    assert m.drop_path_rates() == list(GOLDEN["rates_" + name])


@pytest.mark.parametrize("fn", [backbone.cotnet50, backbone.cotnext50_2x48d, backbone_hybrid.se_cotnetd_50])
def test_state_dict_unchanged_by_the_rates(fn):
    torch.manual_seed(0)
    a = fn(num_classes=10).state_dict()
    torch.manual_seed(0)
    m = fn(num_classes=10, drop_rate=0.25, drop_path_rate=0.1)
    b = m.state_dict()
    assert list(a) == list(b)
    assert all(a[k].shape == b[k].shape and torch.equal(a[k], b[k]) for k in a)
    m.load_state_dict(a, strict=True)


def test_drop_path_bn_argument_errors():
    """The BatchNorm entry points with drop-path scales: rejected before any launch, like without them."""
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EDTYPE = -5, -1, -2
    assert lib.cotb200_bn_apply(_lib.BF16, 2, 4, 8, None, None, P, P, 1, P, P, None) == ENULL
    assert lib.cotb200_bn_apply_batch(_lib.BF16, 2, 4, 8, P, None, P, P, None, None, None, None, 8.0, 1e-5, 0.1, 1, 1, P, P, P,
                                      P, P, P, None, None) == ENULL
    assert lib.cotb200_bn_apply_batch(_lib.BF16, 2, 4, 8, P, P, P, P, None, None, None, None, 8.0, 1e-5, 0.1, 0, 0, P, P, P,
                                      P, P, P, P, None) == EINVAL
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 2, 4, 8, P, P, None, None, P, P, P, P, 1, P, P, P, None) == ENULL
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 2, 4, 8, P, P, P, None, P, P, P, P, 3, P, P, P, None) == ENULL
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 2, 4, 8, P, P, P, P, P, P, P, P, 2, P, P, P, None) == EINVAL
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 2, 4, 8, P, P, P, None, P, P, P, P, 4, P, P, P, None) == EINVAL
    assert lib.cotb200_bn_bwd_apply(_lib.F64, 2, 4, 8, P, P, P, None, P, P, P, P, None, None, 0.1, 1, P, None, P, None) == EDTYPE


def test_soft_ce_argument_errors():
    """NULL operands, an odd label count with mixing, bad dimensions / smoothing, fp64: rejected before any launch."""
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EDTYPE = -5, -1, -2
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, None, 10, P, 4, None, 0.1, P, P, None) == ENULL
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, P, 10, P, 4, None, 0.1, None, P, None) == ENULL
    assert lib.cotb200_soft_ce(_lib.BF16, 3, 10, P, 10, P, 3, P, 0.1, P, P, None) == EINVAL         # odd n_labels with a table
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, P, 10, P, 3, None, 0.1, P, P, None) == EINVAL      # n_labels < B without one
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, P, 8, P, 4, None, 0.1, P, P, None) == EINVAL       # ld < K
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, P, 10, P, 4, None, 1.0, P, P, None) == EINVAL      # smoothing outside [0, 1)
    assert lib.cotb200_soft_ce(_lib.F64, 4, 10, P, 10, P, 4, None, 0.1, P, P, None) == EDTYPE
    assert lib.cotb200_soft_ce_bwd(_lib.F32, 4, 10, P, 10, P, 4, None, 0.1, P, None, P, 10, None) == ENULL
    assert lib.cotb200_soft_ce_bwd(_lib.F32, 4, 10, P, 10, P, 4, None, 0.1, P, P, P, 5, None) == EINVAL
    assert lib.cotb200_soft_ce_bwd(_lib.F32, 3, 10, P, 10, P, 3, P, 0.1, P, P, P, 10, None) == EINVAL
    assert lib.cotb200_last_error()


def test_recipe_step_fixture_inputs_regenerate_from_the_batch_table():
    """The inputs of the recipe training-step fixture
    (tests/test_recipe_gpu.py::test_recipe_step_with_batch_table_matches_reference_golden):
    the uint8 batch from its seed, the reference collate's draw from MixupCutmix, the mixed batch's checksum, the DropPath
    masks the reference drew at the per-block rates of the trunk."""
    from oracle import make_golden
    B, R = int(GOLDEN["step_B"]), int(GOLDEN["step_res"])
    x, y = make_golden.train_batch(int(GOLDEN["step_seed"]), B, R)
    u8 = (x * 45.0 + 120.0).round().clamp(0, 255).to(torch.uint8).numpy()
    assert int(u8.astype(np.int64).sum()) == int(GOLDEN["step_u8_sum"]) and np.array_equal(y.numpy(), GOLDEN["step_labels"])
    p = trainer.MixupCutmix(seed=int(GOLDEN["step_mix_seed"]), device=None).draw(B, R, R)
    r = batch_row(p, B)
    assert r.mode == 1 and p.lam == float(GOLDEN["step_lam"]) and r.target_lam == float(np.float32(GOLDEN["step_lam"]))
    mixed = np.rint(u8.astype(np.float32) * np.float32(r.lam) + u8[::-1].astype(np.float32) * np.float32(r.one_minus_lam))
    assert int(mixed.astype(np.int64).sum()) == int(GOLDEN["step_mixed_sum"])
    rates = backbone.cotnet50(num_classes=10, drop_path_rate=float(GOLDEN["step_rate"])).drop_path_rates()
    assert np.allclose(1.0 - np.array(rates), GOLDEN["step_keep"], rtol=0, atol=1e-15)
    masks = GOLDEN["step_masks"]
    assert masks.shape == (len(rates), B) and masks[0].all() and 0 < masks.sum() < masks.size
