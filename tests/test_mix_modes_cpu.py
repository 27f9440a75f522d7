"""Per-sample Mixup / CutMix ('elem', 'pair', 'half') and min-max CutMix boxes on CPU: MixupCutmix's draws against the reference's
own FastCollateMixup draws (tests/golden/mix_modes.npz, tools/make_mix_modes_golden.py), the row tables applied by the numpy
restatement (mix_ref.py) against the reference's mixed uint8 batches and soft targets, and the argument checks of the new C
entry points (no kernel is launched)."""
import ctypes
import os

import numpy as np
import pytest

import mix_ref
from cotnet_b200 import _lib, trainer

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mix_modes.npz"))
MODES = ("elem", "pair", "half")
ALPHAS = {"both": (0.8, 1.0, None), "mixup": (0.8, 0.0, None), "cutmix": (0.0, 1.0, None), "minmax": (0.8, 1.0, [0.2, 0.8])}
SEEDS, DRAW_B, DRAW_H, DRAW_W = 16, 8, 32, 48
NUM_CLASSES = 100


def mixed_batch(seed, shape):
    """tools/make_mix_modes_golden.py:mixed_batch"""
    rng = np.random.RandomState(2000 + seed)
    x = rng.randint(0, 256, size=shape).astype(np.uint8)
    return x, rng.randint(0, NUM_CLASSES, size=shape[0]).astype(np.int64)


def mixer(mode, aset, prob=1.0, seed=0, device=None):
    mixup, cutmix, minmax = ALPHAS[aset]
    return trainer.MixupCutmix(mixup, cutmix, prob=prob, switch_prob=0.5, label_smoothing=0.1, num_classes=NUM_CLASSES, seed=seed,
                               device=device, mode=mode, cutmix_minmax=minmax)


@pytest.mark.parametrize("prob", [1.0, 0.5])
@pytest.mark.parametrize("aset", list(ALPHAS))
@pytest.mark.parametrize("mode", MODES)
def test_row_draws_equal_reference(mode, aset, prob):
    """Every element's switch, fp32 lam, fp32 blend weights, box and box-corrected fp32 target lam, for 16 seeds, exactly; and
    the rows the table puts them in (pair: row B-1-i repeats row i's draw with the partners swapped)."""
    key = "%s_%s_%s_" % (mode, aset, "p10" if prob == 1.0 else "p05")
    lam0, cut, lam, box = (GOLDEN[key + k] for k in ("lam0", "cut", "lam", "box"))
    seen = set()
    for seed in range(SEEDS):
        t = mixer(mode, aset, prob, seed).draw(DRAW_B, DRAW_H, DRAW_W)
        n = DRAW_B if mode == "elem" else DRAW_B // 2
        assert isinstance(t, trainer.MixRows) and t.n_in == DRAW_B and t.n_out == (DRAW_B // 2 if mode == "half" else DRAW_B)
        for i in range(n):
            r, j = t.host[i], DRAW_B - 1 - i
            mode_i = 0 if lam0[seed, i] == 1. else (2 if cut[seed, i] else 1)
            assert (r.mode, r.partner) == (mode_i, j), (seed, i)
            assert np.float32(r.target_lam) == lam[seed, i], (seed, i, r.target_lam, lam[seed, i])
            if mode_i == 1:
                assert np.float32(r.lam) == lam0[seed, i] and np.float32(r.one_minus_lam) == np.float32(1) - lam0[seed, i]
            if mode_i == 2:
                assert (r.y0, r.y1, r.x0, r.x1) == tuple(box[seed, i]), (seed, i)
            if mode == "pair":
                q = t.host[j]
                assert q.partner == i and bytes(q)[8:] == bytes(r)[8:] and q.mode == r.mode
            seen.add(mode_i)
    assert seen == {0, 1, 2} - ({1} if aset == "cutmix" else set()) - ({2} if aset == "mixup" else set()) - \
        ({0} if prob == 1.0 else set())


@pytest.mark.parametrize("prob", [1.0, 0.5])
def test_batch_minmax_draws_equal_reference(prob):
    """Batch mode with cutmix_minmax: the reference's lam (always box-corrected), switch and min-max box, exactly."""
    want = GOLDEN["batch_minmax_%s" % ("p10" if prob == 1.0 else "p05")]
    modes = set()
    for seed, (lam, use_cutmix, yl, yh, xl, xh) in enumerate(want):
        p = trainer.MixupCutmix(0.8, 1.0, prob=prob, seed=seed, device=None, cutmix_minmax=[0.2, 0.8]).draw(8, 128, 128)
        assert isinstance(p, trainer.MixParams) and p.target_lam == lam, (seed, p.target_lam, lam)
        assert p.mode == (0 if lam == 1. else (2 if use_cutmix else 1)), seed
        if p.mode == 2:
            assert p.box == (yl, yh, xl, xh), seed
        modes.add(p.mode)
    assert modes == ({1, 2} if prob == 1.0 else {0, 1, 2})


def test_minmax_forces_cutmix_alpha_and_empty_list_is_off():
    assert trainer.MixupCutmix(0.8, 0.0, device=None, cutmix_minmax=[0.2, 0.8]).cutmix_alpha == 1.0
    mc = trainer.MixupCutmix(0.8, 0.0, device=None, cutmix_minmax=[])
    assert mc.cutmix_minmax is None and mc.cutmix_alpha == 0.0
    with pytest.raises(ValueError, match="mode"):
        trainer.MixupCutmix(device=None, mode="pairs")
    with pytest.raises(ValueError, match="two ratios"):
        trainer.MixupCutmix(device=None, cutmix_minmax=[0.2])


@pytest.mark.parametrize("mode", ("batch",) + MODES)
def test_disabled_draws_consume_no_random_numbers(mode):
    mc = trainer.MixupCutmix(seed=3, device=None, mode=mode, cutmix_minmax=[0.2, 0.8])
    mc.enabled = False
    state = mc.rng.get_state()[1].copy(), mc.rng.get_state()[2]
    t = mc.draw(8, 16, 16)
    assert np.array_equal(mc.rng.get_state()[1], state[0]) and mc.rng.get_state()[2] == state[1]
    if mode == "batch":
        assert t.mode == 0 and t.target_lam == 1.0
    else:
        assert all(r.mode == 0 and r.target_lam == 1.0 for r in t.host)


@pytest.mark.parametrize("case", ["%s_%s" % (m, a) for m in MODES for a in ALPHAS] + ["%s_both_generic" % m for m in MODES])
def test_row_tables_reproduce_the_reference_batches(case):
    """The table drawn with the fixture's seed, applied by the numpy restatement to the seeded uint8 batch, gives the reference's
    mixed bytes exactly, and its soft targets to 1e-6."""
    mode, aset = case.split("_")[:2]
    out, target, seed = GOLDEN["out_" + case], GOLDEN["target_" + case], int(GOLDEN["seed_" + case])
    x, labels = mixed_batch(seed, (out.shape[0] * (2 if mode == "half" else 1),) + out.shape[1:])
    t =mixer(mode, aset, 1.0, seed).draw(x.shape[0], x.shape[2], x.shape[3])
    assert np.array_equal(mix_ref.mixed_batch(x, t.host), out)
    assert np.abs(mix_ref.soft_targets(labels, t.host, NUM_CLASSES, 0.1) - target).max() < 1e-6
    assert {r.mode for r in t.host} >= ({1} if aset != "cutmix" else set()) | ({2} if aset != "mixup" else set())


def test_mix_row_struct():
    assert ctypes.sizeof(_lib.MixRow) == 36


def test_row_entry_point_argument_errors():
    """NULL operands, odd N, N_out > N_in, a partner or box out of range, a bad mode, n_labels < B: rejected before any launch."""
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EDTYPE = -5, -1, -2
    f3 = (ctypes.c_float * 3)(1, 1, 1)

    def table(n, **kw):
        rows = (_lib.MixRow * n)()
        for i in range(n):
            rows[i].mode, rows[i].partner, rows[i].lam, rows[i].one_minus_lam, rows[i].target_lam = 1, n - 1 - i, 0.5, 0.5, 0.5
        for k, v in kw.items():
            setattr(rows[0], k, v)
        return rows

    def u8(N_in, N_out, rows, x=P, dev=P, dtype=_lib.BF16):
        return lib.cotb200_u8_mix_rows_to_nhwc(dtype, N_in, N_out, 3, 8, 8, x, P, f3, f3, None, None, rows, dev, None)
    assert u8(4, 4, table(4), x=None) == ENULL
    assert u8(4, 4, None) == ENULL
    assert u8(4, 4, table(4), dev=None) == ENULL
    assert u8(5, 5, table(5)) == EINVAL                                    # odd N
    assert u8(4, 6, table(6)) == EINVAL                                    # N_out > N_in
    assert u8(4, 0, table(1)) == EINVAL
    assert u8(4, 4, table(4, partner=4)) == EINVAL
    assert u8(4, 4, table(4, partner=-1)) == EINVAL
    assert u8(4, 4, table(4, mode=3)) == EINVAL
    assert u8(4, 4, table(4, mode=-1)) == EINVAL
    assert u8(4, 4, table(4, mode=2, y0=2, y1=9, x0=0, x1=4)) == EINVAL   # box past H = 8
    assert u8(4, 4, table(4, mode=2, y0=3, y1=2, x0=0, x1=4)) == EINVAL
    assert u8(4, 4, table(4, mode=2, y0=0, y1=8, x0=-1, x1=4)) == EINVAL
    assert u8(4, 4, table(4), dtype=_lib.F64) == EDTYPE
    assert u8(4, 2, table(2), dtype=_lib.F64) == EDTYPE                    # 'half': the rows pass, only the dtype is refused
    # the loss
    assert lib.cotb200_soft_ce_rows(_lib.BF16, 4, 10, None, 10, P, 4, P, 0.1, P, P, None) == ENULL
    assert lib.cotb200_soft_ce_rows(_lib.BF16, 4, 10, P, 10, P, 4, None, 0.1, P, P, None) == ENULL
    assert lib.cotb200_soft_ce_rows(_lib.BF16, 4, 10, P, 10, P, 4, P, 0.1, None, P, None) == ENULL
    assert lib.cotb200_soft_ce_rows(_lib.BF16, 4, 10, P, 10, P, 3, P, 0.1, P, P, None) == EINVAL        # n_labels < B
    assert lib.cotb200_soft_ce_rows(_lib.BF16, 3, 10, P, 10, P, 5, P, 0.1, P, P, None) == EINVAL        # odd n_labels
    assert lib.cotb200_soft_ce_rows(_lib.BF16, 4, 10, P, 8, P, 4, P, 0.1, P, P, None) == EINVAL         # ld < K
    assert lib.cotb200_soft_ce_rows(_lib.BF16, 4, 10, P, 10, P, 4, P, 1.0, P, P, None) == EINVAL        # smoothing
    assert lib.cotb200_soft_ce_rows(_lib.F64, 4, 10, P, 10, P, 8, P, 0.1, P, P, None) == EDTYPE
    assert lib.cotb200_soft_ce_rows_bwd(_lib.F32, 4, 10, P, 10, P, 4, None, 0.1, P, P, P, 10, None) == ENULL
    assert lib.cotb200_soft_ce_rows_bwd(_lib.F32, 4, 10, P, 10, P, 4, P, 0.1, P, None, P, 10, None) == ENULL
    assert lib.cotb200_soft_ce_rows_bwd(_lib.F32, 4, 10, P, 10, P, 4, P, 0.1, P, P, P, 5, None) == EINVAL
    assert lib.cotb200_soft_ce_rows_bwd(_lib.F32, 4, 10, P, 10, P, 2, P, 0.1, P, P, P, 10, None) == EINVAL
    assert lib.cotb200_last_error()


def test_row_table_batch_size_and_step_kinds():
    t = trainer.MixupCutmix(seed=0, device=None, mode="half").draw(8, 16, 16)
    assert t.shape == ("rows", 4, 8)
    with pytest.raises(ValueError, match="drawn for 8"):
        t.check(6, 16, 16)
    assert trainer.MixupCutmix(seed=0, device=None).draw(8, 16, 16).shape == ("batch",)
