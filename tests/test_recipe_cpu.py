"""The training recipe's host logic on CPU: MixupCutmix draws against the reference's own FastCollateMixup draws
(tests/golden/recipe.npz, tools/make_recipe_golden.py), the per-block stochastic-depth rates against the reference's modules,
unchanged state dicts, and the argument checks of the new C entry points (no kernel is launched)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, backbone, backbone_hybrid, trainer

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recipe.npz"))


def mix_batch(seed):
    """The seeded uint8 batch of the mixed-batch fixture (tools/make_recipe_golden.py:mix_batch)."""
    rng = np.random.RandomState(1000 + seed)
    x = rng.randint(0, 256, size=(4, 3, 16, 20)).astype(np.uint8)
    return x, rng.randint(0, 1000, size=4).astype(np.int64)


@pytest.mark.parametrize("key,prob", [("draws_p1", 1.0), ("draws_p05", 0.5)])
def test_mixup_cutmix_draws_equal_reference(key, prob):
    """lam (box-corrected for CutMix), the CutMix switch and the box of every seed, exactly."""
    want = GOLDEN[key]
    modes = set()
    for seed, (lam, use_cutmix, yl, yh, xl, xh) in enumerate(want):
        mc = trainer.MixupCutmix(0.8, 1.0, prob=prob, switch_prob=0.5, label_smoothing=0.1, num_classes=1000, seed=seed, device=None)
        p = mc.draw(8, 128, 128)
        assert p.target_lam == lam, (seed, p.target_lam, lam)
        assert p.mode == (0 if lam == 1. else (2 if use_cutmix else 1)), seed
        if p.mode == 2:
            assert p.box == (yl, yh, xl, xh), seed
        if p.mode == 1:
            assert p.host.lam == float(np.float32(lam)) and p.host.one_minus_lam == float(np.float32(1 - lam))
        modes.add(p.mode)
    assert modes == ({1, 2} if prob == 1.0 else {0, 1, 2})


def test_mixup_cutmix_batch_draws_reproduce_the_golden_batches():
    """The draws that made the stored mixed batches (4 x 3 x 16 x 20), and the numpy arithmetic of the reference on them."""
    for kind, mode in (("mixup", 1), ("cutmix", 2)):
        seed = int(GOLDEN[kind + "_seed"])
        x, labels = mix_batch(seed)
        p = trainer.MixupCutmix(seed=seed, device=None).draw(*x.shape[:1], *x.shape[2:])
        assert p.mode == mode
        xp = x[::-1]
        if mode == 1:
            want = np.rint(x.astype(np.float32) * np.float32(p.host.lam) + xp.astype(np.float32) * np.float32(p.host.one_minus_lam))
        else:
            y0, y1, x0, x1 = p.box
            want = x.copy()
            want[:, :, y0:y1, x0:x1] = xp[:, :, y0:y1, x0:x1]
        assert np.array_equal(want.astype(np.uint8), GOLDEN[kind + "_out"])
        eye = np.eye(1000)
        t = 1e-4 + 0.9 * (p.target_lam * eye[labels] + (1 - p.target_lam) * eye[labels[::-1]])     # mixup_target, smoothing 0.1
        assert np.abs(t - GOLDEN[kind + "_target"]).max() < 1e-6


def test_mixup_disabled_and_odd_batch():
    mc = trainer.MixupCutmix(seed=0, device=None)
    mc.enabled = False
    state = mc.rng.get_state()[2]
    p = mc.draw(4, 8, 8)
    assert p.mode == 0 and p.target_lam == 1.0 and mc.rng.get_state()[2] == state
    with pytest.raises(ValueError):
        mc.draw(5, 8, 8)
    with pytest.raises(ValueError):
        trainer.MixupCutmix(0., 0., device=None)


def test_mix_params_validation():
    m = _lib.Mix()
    m.mode = 3
    with pytest.raises(ValueError, match="mode"):
        trainer.MixParams(m).check(4, 8, 8)
    m.mode = 1
    with pytest.raises(ValueError, match="even"):
        trainer.MixParams(m).check(5, 8, 8)
    m.mode, m.y0, m.y1, m.x0, m.x1 = 2, 2, 9, 0, 4
    with pytest.raises(ValueError, match="box"):
        trainer.MixParams(m).check(4, 8, 8)
    assert ctypes.sizeof(_lib.Mix) == 32


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


def test_new_entry_point_argument_errors():
    """NULL operands, an odd batch with mixing, bad dimensions / smoothing, fp64: rejected before any launch."""
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EDTYPE = -5, -1, -2
    # the mixing input kernel
    f3 = (ctypes.c_float * 3)(1, 1, 1)
    assert lib.cotb200_u8_mix_to_nhwc(_lib.BF16, 4, 3, 8, 8, None, P, f3, f3, None, None, P, None) == ENULL
    assert lib.cotb200_u8_mix_to_nhwc(_lib.BF16, 5, 3, 8, 8, P, P, f3, f3, None, None, P, None) == EINVAL
    assert lib.cotb200_u8_mix_to_nhwc(_lib.BF16, 0, 3, 8, 8, P, P, f3, f3, None, None, None, None) == EINVAL
    # the loss
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, None, 10, P, None, 0.1, P, P, None) == ENULL
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, P, 10, P, None, 0.1, None, P, None) == ENULL
    assert lib.cotb200_soft_ce(_lib.BF16, 3, 10, P, 10, P, P, 0.1, P, P, None) == EINVAL           # odd B with mixing
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, P, 8, P, None, 0.1, P, P, None) == EINVAL          # ld < K
    assert lib.cotb200_soft_ce(_lib.BF16, 4, 10, P, 10, P, None, 1.0, P, P, None) == EINVAL         # smoothing outside [0, 1)
    assert lib.cotb200_soft_ce(_lib.F64, 4, 10, P, 10, P, None, 0.1, P, P, None) == EDTYPE
    assert lib.cotb200_soft_ce_bwd(_lib.F32, 4, 10, P, 10, P, None, 0.1, P, None, P, 10, None) == ENULL
    assert lib.cotb200_soft_ce_bwd(_lib.F32, 4, 10, P, 10, P, None, 0.1, P, P, P, 5, None) == EINVAL
    assert lib.cotb200_soft_ce_bwd(_lib.F32, 3, 10, P, 10, P, P, 0.1, P, P, P, 10, None) == EINVAL
    assert lib.cotb200_last_error()


def test_recipe_step_fixture_inputs_regenerate():
    """The inputs of the recipe training-step fixture (tests/test_recipe_gpu.py::test_recipe_step_matches_reference_golden):
    the uint8 batch from its seed, the reference collate's draw from MixupCutmix, the mixed batch's checksum, the DropPath
    masks the reference drew at the per-block rates of the trunk."""
    from oracle import make_golden
    B, R = int(GOLDEN["step_B"]), int(GOLDEN["step_res"])
    x, y = make_golden.train_batch(int(GOLDEN["step_seed"]), B, R)
    u8 = (x * 45.0 + 120.0).round().clamp(0, 255).to(torch.uint8).numpy()
    assert int(u8.astype(np.int64).sum()) == int(GOLDEN["step_u8_sum"]) and np.array_equal(y.numpy(), GOLDEN["step_labels"])
    p = trainer.MixupCutmix(seed=int(GOLDEN["step_mix_seed"]), device=None).draw(B, R, R)
    assert p.mode == 1 and p.target_lam == float(GOLDEN["step_lam"])
    mixed = np.rint(u8.astype(np.float32) * np.float32(p.host.lam) + u8[::-1].astype(np.float32) * np.float32(p.host.one_minus_lam))
    assert int(mixed.astype(np.int64).sum()) == int(GOLDEN["step_mixed_sum"])
    rates = backbone.cotnet50(num_classes=10, drop_path_rate=float(GOLDEN["step_rate"])).drop_path_rates()
    assert np.allclose(1.0 - np.array(rates), GOLDEN["step_keep"], rtol=0, atol=1e-15)
    masks = GOLDEN["step_masks"]
    assert masks.shape == (len(rates), B) and masks[0].all() and 0 < masks.sum() < masks.size
