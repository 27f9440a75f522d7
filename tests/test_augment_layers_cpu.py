"""CPU checks of RandAugment with any number of layers and with the weighted op choice ('w0'): the parsed weights are the
reference's bit for bit, TrainAugment.draw leaves the generators where the reference's transform leaves them
(tests/golden/augment_layers.npz), oracle/aug_ref.py gives the reference's bytes, the structs are pass-major with n <= 2
packing exactly the bytes it packed before, and configs the reference refuses or this library cannot honour raise."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch

from cotnet_b200 import augment
from oracle import aug_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment_layers.npz")
#: tools/make_augment_layers_golden.py CONFIGS
CONFIGS = ("rand-m9-n3-mstd0.5", "rand-m15-n5-mstd0.5", "rand-mstd1-w0", "rand-m15-n4-mstd0.5-w0")


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _gens(seed):
    return random.Random(seed), np.random.RandomState(seed), torch.Generator().manual_seed(seed)


def _next(rnd, nrnd, tgen):
    return rnd.random(), nrnd.random_sample(), float(torch.rand(1, generator=tgen))


def _cases(gold, prefix):
    k = 0
    while "%s_%d" % (prefix, k) in gold:
        yield "%s_%d" % (prefix, k)
        k += 1


def _applied(p):
    return [o for o in p["ops"] if o is not None]


def test_fixture_configs():
    assert tuple(aug_ref.load_golden(GOLD)["configs"]) == CONFIGS


def test_choice_weights_equal_reference_bitwise(gold):
    want = gold["weights_0"]
    assert want.dtype == np.float64 and want.shape == (16,)
    for got in (augment.choice_weights(0), augment.TrainAugment(auto_augment="rand-mstd1-w0").choice_weights):
        assert got.dtype == np.float64
        np.testing.assert_array_equal(got.view(np.int64), want.view(np.int64))
    assert augment.TrainAugment().choice_weights is None
    assert np.count_nonzero(want) == 14


@pytest.mark.parametrize("c", range(len(CONFIGS)))
def test_draws_and_generator_states_equal_reference(gold, c):
    """DRAW_SEEDS images per config: the applied ops' ids and arguments and the three generators' next values after each."""
    tf = augment.TrainAugment(auto_augment=CONFIGS[c])
    ids, args, nxt = gold["d_%d_ids" % c], gold["d_%d_args" % c], gold["d_%d_next" % c]
    seed0 = int(gold["d_%d_seed0" % c][0])
    assert tf.num_layers == ids.shape[1]
    for s, (H, W) in enumerate(gold["d_sizes"]):
        gens = _gens(seed0 + s)
        p = tf.draw_one(int(H), int(W), *gens)
        assert len(p["ops"]) == tf.num_layers
        applied = _applied(p)
        assert [o["id"] for o in applied] + [-1] * (tf.num_layers - len(applied)) == ids[s].tolist(), s
        assert [float(o["arg"]) for o in applied] == args[s][:len(applied)].tolist(), s
        assert _next(*gens) == tuple(nxt[s]), s
        if tf.choice_weights is not None:                 # without replacement
            chosen = [o["id"] for o in applied]
            assert len(set(chosen)) == len(chosen) and not {2, 4} & set(chosen)   # Invert, Posterize: weight 0
    n_applied = (ids >= 0).sum(1)
    assert n_applied.min() < tf.num_layers and n_applied.max() == tf.num_layers


@pytest.mark.parametrize("c", range(len(CONFIGS)))
@pytest.mark.parametrize("S", [224, 320])
def test_oracle_equals_reference_fixture(gold, c, S):
    """oracle/aug_ref.train_sample applies every drawn op in order; the generators end where the reference's do."""
    tf = augment.TrainAugment(size=S, auto_augment=CONFIGS[c])
    keys = list(_cases(gold, "train_%d_%d" % (c, S)))
    assert len(keys) >= 2
    for key in keys:
        H, W, seed, iseed = (int(v) for v in gold[key + "_size"])
        gens = _gens(seed)
        p = tf.draw_one(H, W, *gens)
        assert _next(*gens) == tuple(gold[key + "_next"]), key
        np.testing.assert_array_equal(aug_ref.train_sample(aug_ref.source_image(iseed, H, W), p, S), gold[key], err_msg=key)


@pytest.mark.parametrize("S", [224, 320])
def test_split_draws_and_oracle_equal_reference(gold, S):
    seed, B, size = (int(v) for v in gold["split_%d_meta" % S])
    src = gold["split_%d_src" % S]
    tf = augment.TrainAugment(size=S, auto_augment="rand-m9-n3-mstd0.5", num_splits=3)
    gens = _gens(seed)
    draws = tf.draw([(int(H), int(W)) for H, W, _ in src], *gens)
    assert _next(*gens) == tuple(gold["split_%d_next" % S])
    want = gold["split_%d" % S].reshape(3 * B, 3, S, S)
    for n, ((H, W, iseed), p) in enumerate(zip(src, draws)):
        img = aug_ref.source_image(int(iseed), int(H), int(W))
        assert p["ops"] == [] and all(len(v["ops"]) == 3 for v in p["views"])
        for k, d in enumerate([p] + [dict(p, ops=v["ops"]) for v in p["views"]]):
            np.testing.assert_array_equal(aug_ref.train_sample(img, d, S), want[k * B + n], err_msg="view %d image %d" % (k, n))


@pytest.mark.parametrize("interp", ["bicubic", "random"])
@pytest.mark.parametrize("S", [224, 320])
def test_noaug_oracle_equals_reference(gold, interp, S):
    """transforms_noaug_train is EvalTransform(size, crop_pct=1.0): Resize(size) + CenterCrop(size), 'random' bilinear."""
    ev = augment.EvalTransform(S, crop_pct=1.0, interpolation=interp)
    assert ev.filter == (augment.BICUBIC if interp == "bicubic" else augment.BILINEAR)
    keys = list(_cases(gold, "noaug_%s_%d" % (interp, S)))
    assert len(keys) >= 2
    for key in keys:
        H, W, iseed = (int(v) for v in gold[key + "_size"])
        got = aug_ref.eval_transform(aug_ref.source_image(iseed, H, W), S, 1.0, ev.filter).transpose(2, 0, 1)
        np.testing.assert_array_equal(got, gold[key], err_msg=key)


def _collate(tf, n_img=7, seed=3):
    r = np.random.RandomState(seed)
    imgs = [np.zeros((int(r.randint(40, 300)), int(r.randint(40, 300)), 3), np.uint8) for _ in range(n_img)]
    draws = tf.draw([a.shape[:2] for a in imgs], *_gens(seed))
    return imgs, draws, tf.collate_draws(imgs, list(range(n_img)), draws)


@pytest.mark.parametrize("aa", ["rand-m9-n3-mstd0.5", "rand-m15-n4-mstd0.5-w0", "rand-m15-n5-mstd0.5", "rand-n14-w0"])
@pytest.mark.parametrize("num_splits", [0, 3])
def test_structs_are_pass_major(aa, num_splits):
    tf = augment.TrainAugment(auto_augment=aa, num_splits=num_splits)
    n = tf.num_layers
    assert tf.passes == (n + 1) // 2
    imgs, draws, b = _collate(tf)
    B, S = len(imgs), max(1, num_splits)
    rows = list(draws) + [p["views"][v] for v in range(S - 1) for p in draws]
    rec = b.params.numpy().view(augment.SAMPLE_DTYPE)
    assert len(rec) == tf.passes * S * B
    assert len(b.labels) == S * B
    pass0 = tf.pack([a.shape[:2] for a in imgs], draws)
    if num_splits:
        pass0 = np.concatenate([pass0, tf.pack_views(draws)])
    assert rec[:S * B].tobytes() == pass0.tobytes()
    ref = np.zeros(1, augment.SAMPLE_DTYPE)
    for k in range(1, tf.passes):
        blk = rec[k * S * B:(k + 1) * S * B]
        assert blk.tobytes() == tf.pack_pass(draws, k).tobytes()
        rest = blk.copy()
        rest["ops"] = ref["ops"][0]
        assert not rest.view(np.uint8).any()                      # nothing but the ops is set
        for r, p in zip(blk, rows):
            ops = p["ops"][2 * k:2 * k + 2]
            for s in range(2):
                want = np.zeros(1, augment.SAMPLE_DTYPE)
                augment.pack_op(want["ops"][0][s], ops[s] if s < len(ops) else None)
                assert r["ops"][s].tobytes() == want["ops"][0][s].tobytes()
    last = rec[(tf.passes - 1) * S * B:]["ops"]["op"]
    if n % 2:                                                     # an odd n leaves the last pass's second slot empty
        assert (last[:, 1] == -1).all()
    for k in range(tf.passes if num_splits else 0):               # the clean view has no op in any pass
        assert (rec["ops"]["op"][k * S * B:k * S * B + B] == -1).all()
    assert (rec["ops"]["op"] >= 0).sum() == sum(len(_applied(p)) for p in rows)


def test_run_refuses_a_partial_pass():
    tf = augment.TrainAugment(auto_augment="rand-m9-n3-mstd0.5")
    _, _, b = _collate(tf)
    cut = augment.AugBatch(b.data, b.params[:-augment.SAMPLE_DTYPE.itemsize], b.labels)
    for batch, passes in ((cut, 2), (b, 3), (b, 0), (b, 1.5)):
        with pytest.raises(ValueError):
            augment.run(batch, 224, "cuda:0", passes=passes)


#: sha256 (first 32 hex digits) of the params, jitter and label bytes that TrainAugment.collate packed for these configs before
#: more than two layers were supported
N_LE_2 = (("rand-m9-n1-mstd0.5", {}, "2206cbaa5c712e187842dc30530aa1b8"),
          ("rand-m9-n2", {}, "b95ffe49334eede1ae2ce816628bcbe7"),
          ("rand-m15-mstd0.5-n2", {"size": 320}, "f9e873d84c37fd136c25bf3641d49532"),
          ("rand-m9-n1-mstd1", {"num_splits": 3}, "445536bc376a3c029ce49fe09258caf0"),
          ("rand-m15-mstd0.5-n2", {"num_splits": 2, "vflip": 0.5}, "0183d48fc9ec22610bf5d7f833c75bd5"),
          ("rand-m7-n0", {}, "c7485f0dd6d9c8a0e57dc7b6b23fa33e"))


@pytest.mark.parametrize("aa,kw,want", N_LE_2)
def test_up_to_two_layers_pack_the_same_bytes(aa, kw, want):
    tf = augment.TrainAugment(auto_augment=aa, **kw)
    assert tf.passes == 1
    r = np.random.RandomState(0)
    batch = [(np.zeros((int(r.randint(40, 300)), int(r.randint(40, 300)), 3), np.uint8), i) for i in range(16)]
    random.seed(12)
    np.random.seed(12)
    torch.manual_seed(12)
    b = tf.collate(batch)
    blob = b.params.numpy().tobytes() + (b"" if b.jitter is None else b.jitter.numpy().tobytes()) + b.labels.numpy().tobytes()
    assert hashlib.sha256(blob).hexdigest()[:32] == want


def test_parsing():
    tf = augment.TrainAugment(auto_augment="rand-m9-n3-mstd0.5")
    assert (tf.magnitude, tf.num_layers, tf.mstd, tf.choice_weights) == (9, 3, 0.5, None)
    tf = augment.TrainAugment(auto_augment="rand-mstd1-w0")
    assert (tf.magnitude, tf.num_layers, tf.mstd, tf.passes) == (10, 2, 1.0, 1) and tf.choice_weights is not None
    tf = augment.TrainAugment(auto_augment="rand-m15-n4-mstd0.5-w0-inc1")
    assert (tf.magnitude, tf.num_layers, tf.mstd, tf.passes) == (15, 4, 0.5, 2)
    assert augment.TrainAugment(auto_augment="rand-n14-w0").num_layers == 14
    assert augment.TrainAugment(auto_augment="rand-n40").passes == 20
    assert augment.TrainAugment(auto_augment="rand-n0").passes == 1


@pytest.mark.parametrize("aa", ["rand-m9-w1", "rand-w2-n2", "rand-n15-w0", "rand-w0-n16", "rand-n-1", "rand-m9-x3",
                                "rand-m9-n3-foo1", "augmix-m5", "v0", "original-mstd0.5"])
def test_bad_configs_raise(aa):
    with pytest.raises(ValueError):
        augment.TrainAugment(auto_augment=aa)


def test_weighted_choice_without_replacement_draws_fourteen_distinct_ops():
    tf = augment.TrainAugment(auto_augment="rand-m9-n14-w0")
    for s in range(20):
        p = tf.draw_one(300, 400, *_gens(s))
        assert len(p["ops"]) == 14
        chosen = [o["id"] for o in _applied(p)]
        assert len(set(chosen)) == len(chosen) and not {2, 4} & set(chosen)
