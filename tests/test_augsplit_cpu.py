"""CPU checks of the augmentation splits and the JSD loss: TrainAugment(num_splits=S) draws what the reference's AugMixDataset
draws (tests/golden/augsplit.npz), num_splits 0 and 1 pack exactly the structs they packed before, the fp64 restatement
tests/jsd_ref.py equals the reference's JsdCrossEntropy, and bad arguments are refused before any launch."""
import hashlib
import math
import os
import random

import numpy as np
import pytest
import torch

from cotnet_b200 import augment, trainer
import jsd_ref
from oracle import aug_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augsplit.npz")
#: tools/make_augsplit_golden.py CASES
CASES = {"s2_rand_v0": (2, "rand-m15-mstd0.5-n2", 0.), "s2_cj_v5": (2, None, 0.5), "s3_rand_v5": (3, "rand-m15-mstd0.5-n2", 0.5),
         "s3_cj_v0": (3, None, 0.), "s2_rand_v5": (2, "rand-m15-mstd0.5-n2", 0.5), "s2_cj_v0": (2, None, 0.),
         "s3_rand_v0": (3, "rand-m15-mstd0.5-n2", 0.), "s3_cj_v5": (3, None, 0.5)}
SIZE = 112


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _tf(case, **kw):
    S, aa, vflip = CASES[case]
    return augment.TrainAugment(size=SIZE, auto_augment=aa, color_jitter=0.4, vflip=vflip, num_splits=S, **kw)


@pytest.mark.parametrize("case", sorted(CASES))
def test_split_draws_equal_reference(gold, case):
    S, aa, vflip = CASES[case]
    tf = _tf(case)
    seed = int(gold["d_%s_seed" % case][0])
    rnd, nrnd, tgen = random.Random(seed), np.random.RandomState(seed), torch.Generator().manual_seed(seed)
    sizes = [tuple(int(v) for v in hw) for hw in gold["d_sizes"]]
    draws = tf.draw(sizes, rnd, nrnd, tgen)
    assert (rnd.random(), nrnd.random_sample(), float(torch.rand(1, generator=tgen))) == tuple(gold["d_%s_next" % case])
    for n, p in enumerate(draws):
        assert (p["i"], p["j"], p["h"], p["w"]) == tuple(gold["d_%s_crop" % case][n]), n
        assert int(p["flip"]) == gold["d_%s_flip" % case][n] and int(p.get("vflip", 0)) == gold["d_%s_vflip" % case][n], n
        assert p["ops"] == [] and "jitter" not in p and len(p["views"]) == S - 1          # the clean view: no colour op
        for v, view in enumerate(p["views"]):
            k = n * (S - 1) + v                                                        # the reference's call order
            if aa:
                applied = [o for o in view["ops"] if o is not None]
                assert [o["id"] for o in applied] + [-1] * (2 - len(applied)) == list(gold["d_%s_ids" % case][k]), (n, v)
                assert [float(o["arg"]) for o in applied] == list(gold["d_%s_args" % case][k][:len(applied)]), (n, v)
            else:
                want_f = gold["d_%s_factors" % case][k]
                f = view["jitter"]["factors"]
                assert [x is None for x in f] == [math.isnan(x) for x in want_f], (n, v)
                assert [x for x in f if x is not None] == [x for x in want_f if not math.isnan(x)], (n, v)
                perm = [int(x) for x in gold["d_%s_perm" % case][k]]
                assert view["jitter"]["order"] == [x for x in perm if not math.isnan(want_f[x])], (n, v)
    imgs = [np.zeros((H, W, 3), np.uint8) for H, W in sizes]
    labels = [int(v) for v in np.random.RandomState(1).randint(0, 1000, len(sizes))]
    b = tf.collate_draws(imgs, labels, draws)
    assert b.labels.tolist() == gold["d_%s_labels" % case].tolist()
    B = len(sizes)
    rec = b.params.numpy().view(augment.SAMPLE_DTYPE)
    assert len(rec) == S * B and b.data.numel() == sum(3 * H * W for H, W in sizes)          # every image shipped once
    assert (rec["ops"]["op"][:B] == -1).all()
    views = rec[B:]
    assert (views["h"] == 0).all() and (views["ch"] == 0).all()                               # the view structs carry ops only
    if aa:
        assert (views["ops"]["op"] >= 0).any()
    if tf.has_jitter_kernel:
        jrec = b.jitter.numpy().view(augment.JITTER_DTYPE)
        assert len(jrec) == S * B
        assert (jrec["vflip"][:B] == gold["d_%s_vflip" % case]).all() and (jrec["vflip"][B:] == 0).all()
        assert (jrec["order"][:B] == -1).all()
        if not aa:
            assert (jrec["order"][B:] >= 0).any()
    else:
        assert b.jitter is None


def test_split_draws_cover_ops_and_jitter(gold):
    ids = np.concatenate([gold["d_%s_ids" % c] for c in CASES if CASES[c][1]])
    assert (ids == -1).any() and len(set(ids[ids >= 0].tolist())) >= 8
    assert gold["d_s3_cj_v5_vflip"].any() and not gold["d_s3_cj_v5_vflip"].all()


#: sha256 (first 32 hex digits) of the params, jitter and label bytes that TrainAugment.collate packed before num_splits existed,
#: for the configurations of _digest
DIGESTS = ("db8a4925abffbba80ee283d78828d70e", "b9938fdd23f5860036465ec8c001fdc3", "3d00d55de0671691cf6f5bb85d732602",
           "b27db2b12f3c832108e61276005d9ad2")


@pytest.mark.parametrize("num_splits", [None, 0, 1])
def test_no_splits_packs_the_same_bytes(num_splits):
    cfgs = [dict(), dict(auto_augment=None, color_jitter=(0.4, 0.4, 0.4, 0.1), vflip=0.5), dict(vflip=0.5, interpolation="random"),
            dict(auto_augment=None, color_jitter=None)]
    for kw, want in zip(cfgs, DIGESTS):
        tf = augment.TrainAugment(**kw, **({} if num_splits is None else {"num_splits": num_splits}))
        r = np.random.RandomState(0)
        batch = [(np.zeros((int(r.randint(40, 300)), int(r.randint(40, 300)), 3), np.uint8), i) for i in range(16)]
        random.seed(11)
        np.random.seed(11)
        torch.manual_seed(11)
        b = tf.collate(batch)
        blob = b.params.numpy().tobytes() + (b"" if b.jitter is None else b.jitter.numpy().tobytes()) + b.labels.numpy().tobytes()
        assert hashlib.sha256(blob).hexdigest()[:32] == want, kw


@pytest.mark.parametrize("name", ["r3", "r2", "clamp", "underflow"])
def test_jsd_restatement_equals_reference(gold, name):
    S, smoothing = gold["jsd_%s_meta" % name]
    loss, dz = jsd_ref.jsd_ce(gold["jsd_%s_z" % name], gold["jsd_%s_y" % name], int(S), float(smoothing))
    want = gold["jsd_%s_grad" % name]
    assert abs(loss - gold["jsd_%s_loss" % name][0]) <= 1e-13 * abs(loss)
    fin = np.isfinite(want)
    assert np.abs(dz - want)[fin].max() <= 1e-13
    assert np.isfinite(dz).all()
    if name == "underflow":
        assert (~fin).any()                      # the reference's gradient is NaN where a probability is exactly 0
    if name == "clamp":                          # the mixture meets both clamp bounds
        z = gold["jsd_clamp_z"]
        p = np.exp(z - z.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        m = p.reshape(int(S), -1, z.shape[1]).mean(0)
        assert (m == 1.0).any() and (m < jsd_ref.CLAMP_LO).any()


def test_argument_errors():
    model = torch.nn.Linear(4, 3)
    for bad in (1, -1, 2.5):
        with pytest.raises(ValueError):
            trainer.TrainStep(model, jsd_splits=bad)
    z, y = torch.zeros(6, 5), torch.zeros(3, dtype=torch.int64)
    for S in (1, 0, 4):
        with pytest.raises(ValueError):
            trainer.jsd_cross_entropy(z, y, S)
    with pytest.raises(ValueError):
        trainer.jsd_cross_entropy(z, y[:1], 3)
    for bad in (-1, 1.5):
        with pytest.raises(ValueError):
            augment.TrainAugment(num_splits=bad)
    assert augment.TrainAugment(num_splits=1).num_splits == 0


def test_jsd_entry_points_reject_bad_arguments():
    """Validation happens before any CUDA call: the pointers below are never dereferenced."""
    from cotnet_b200 import _lib
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EDTYPE = -5, -1, -2

    def fwd(dtype=_lib.F32, S=3, B=4, K=10, z=P, ld=10, y=P, sm=0.1, alpha=12.0, rows=P, loss=P):
        return lib.cotb200_jsd_ce(dtype, S, B, K, z, ld, y, sm, alpha, rows, loss, None)

    def bwd(dtype=_lib.F32, S=3, B=4, K=10, z=P, ld=10, y=P, sm=0.1, alpha=12.0, rows=P, dl=P, dz=P, ldz=10):
        return lib.cotb200_jsd_ce_bwd(dtype, S, B, K, z, ld, y, sm, alpha, rows, dl, dz, ldz, None)

    for f in (fwd, bwd):
        assert f(z=None) == ENULL and f(y=None) == ENULL and f(rows=None) == ENULL
        for kw in (dict(S=1), dict(S=0), dict(S=9), dict(B=0), dict(K=0), dict(ld=9), dict(S=8, B=1 << 28), dict(sm=-0.1),
                   dict(sm=1.0), dict(sm=math.nan), dict(alpha=-1.0), dict(alpha=math.inf), dict(alpha=math.nan)):
            assert f(**kw) == EINVAL, (f.__name__, kw)
        assert f(dtype=_lib.F64) == EDTYPE
    assert fwd(loss=None) == ENULL
    assert bwd(dl=None) == ENULL and bwd(dz=None) == ENULL
    assert bwd(ldz=9) == EINVAL
