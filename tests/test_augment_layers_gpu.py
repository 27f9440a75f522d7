"""RandAugment with more than two layers and with the weighted op choice on the GPU, byte for byte: TrainAugment's output
against the reference's PIL outputs in tests/golden/augment_layers.npz at 224 (one CTA per image) and 320 (thread-block
clusters), with and without augmentation splits, and against oracle/aug_ref.py on random draws; ceil(n / 2) RandAugment
launches per batch, and exactly the launches of before for n <= 2; and the no_aug transform (EvalTransform(crop_pct=1.0))."""
import os
import random

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, augment
from oracle import aug_ref

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment_layers.npz")
#: tools/make_augment_layers_golden.py CONFIGS
CONFIGS = ("rand-m9-n3-mstd0.5", "rand-m15-n5-mstd0.5", "rand-mstd1-w0", "rand-m15-n4-mstd0.5-w0")


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _gens(seed):
    return random.Random(seed), np.random.RandomState(seed), torch.Generator().manual_seed(seed)


def _cases(gold, prefix):
    k = 0
    while "%s_%d" % (prefix, k) in gold:
        yield "%s_%d" % (prefix, k)
        k += 1


def _augment(tf, imgs, draws):
    x, _ = tf(tf.collate_draws(imgs, list(range(len(imgs))), draws))
    torch.cuda.synchronize()
    return x.cpu().numpy()


def _launches(fn):
    torch.cuda.synchronize()
    _lib.prof_enable(True)
    try:
        fn()
        torch.cuda.synchronize()
        rep = _lib.prof_report()
    finally:
        _lib.prof_enable(False)
    return {k: v[0] for k, v in rep.items()}


@pytest.mark.parametrize("c", range(len(CONFIGS)))
@pytest.mark.parametrize("S", [224, 320])
def test_train_equals_reference_fixture(gold, c, S):
    tf = augment.TrainAugment(size=S, auto_augment=CONFIGS[c])
    keys = list(_cases(gold, "train_%d_%d" % (c, S)))
    sz = [tuple(int(v) for v in gold[k + "_size"]) for k in keys]
    imgs = [aug_ref.source_image(iseed, H, W) for H, W, _, iseed in sz]
    draws = [tf.draw_one(H, W, *_gens(seed)) for H, W, seed, _ in sz]
    got = _augment(tf, imgs, draws)
    assert len(keys) >= 2
    for n, k in enumerate(keys):
        np.testing.assert_array_equal(got[n], gold[k], err_msg=k)


@pytest.mark.parametrize("S", [224, 320])
def test_three_splits_equal_reference_fixture(gold, S):
    seed, B, _ = (int(v) for v in gold["split_%d_meta" % S])
    src = [tuple(int(v) for v in r) for r in gold["split_%d_src" % S]]
    tf = augment.TrainAugment(size=S, auto_augment="rand-m9-n3-mstd0.5", num_splits=3)
    imgs = [aug_ref.source_image(iseed, H, W) for H, W, iseed in src]
    draws = tf.draw([(H, W) for H, W, _ in src], *_gens(seed))
    got = _augment(tf, imgs, draws)
    np.testing.assert_array_equal(got, gold["split_%d" % S].reshape(3 * B, 3, S, S))


@pytest.mark.parametrize("interp", ["bicubic", "random"])
@pytest.mark.parametrize("S", [224, 320])
def test_noaug_equals_reference_fixture(gold, interp, S):
    ev = augment.EvalTransform(S, crop_pct=1.0, interpolation=interp)
    keys = list(_cases(gold, "noaug_%s_%d" % (interp, S)))
    imgs = [aug_ref.source_image(iseed, H, W) for H, W, iseed in (tuple(int(v) for v in gold[k + "_size"]) for k in keys)]
    x, _ = ev(ev.collate([(a, 0) for a in imgs]))
    got = x.cpu().numpy()
    assert len(keys) >= 2
    for n, k in enumerate(keys):
        np.testing.assert_array_equal(got[n], gold[k], err_msg=k)


def _sizes(r, n):
    return [(int(r.randint(150, 600)), int(r.randint(150, 600))) for _ in range(n)]


@pytest.mark.parametrize("aa", ["rand-m15-n3-mstd0.5", "rand-m9-n4-mstd1-w0", "rand-m12-n7-mstd0.5", "rand-n14-w0"])
@pytest.mark.parametrize("S", [224, 320])
def test_random_draws_equal_oracle(aa, S):
    """Every drawn op of every image applied in sequence, with and without splits."""
    r = np.random.RandomState(S + len(aa))
    for num_splits in (0, 3):
        tf = augment.TrainAugment(size=S, auto_augment=aa, interpolation="random", num_splits=num_splits)
        sizes = _sizes(r, 12)
        imgs = [aug_ref.source_image(7 * S + n, H, W) for n, (H, W) in enumerate(sizes)]
        draws = tf.draw(sizes, *_gens(S + 31 * num_splits))
        got = _augment(tf, imgs, draws)
        B = len(imgs)
        for n, p in enumerate(draws):
            views = [p] + [dict(p, ops=v["ops"]) for v in p.get("views", [])]
            for k, d in enumerate(views):
                np.testing.assert_array_equal(got[k * B + n], aug_ref.train_sample(imgs[n], d, S),
                                              err_msg="%s splits %d view %d image %d" % (aa, num_splits, k, n))


@pytest.mark.parametrize("S", [224, 320])
def test_randaug_launches_per_layer_count(S):
    """ceil(n / 2) RandAugment launches on the one-CTA (224) or cluster (320) kernel, one resize-crop pair; n <= 2 launches
    what it launched before: one of each."""
    r = np.random.RandomState(5)
    sizes = _sizes(r, 16)
    imgs = [aug_ref.source_image(n, H, W) for n, (H, W) in enumerate(sizes)]
    kernel = "aug_randaug_cluster" if S > 256 else "aug_randaug"
    for aa in ("rand-m9-n1", "rand-m15-mstd0.5-n2", "rand-mstd1-w0", "rand-m9-n3-mstd0.5", "rand-m15-n4-mstd0.5-w0",
               "rand-m15-n5-mstd0.5", "rand-m9-n8"):
        for num_splits in (0, 3):
            tf = augment.TrainAugment(size=S, auto_augment=aa, num_splits=num_splits)
            batch = tf.collate_draws(imgs, list(range(len(imgs))), tf.draw(sizes, *_gens(11)))
            got = _launches(lambda: tf(batch))
            assert got == {"aug_hpass": 1, "aug_vpass": 1, kernel: -(-tf.num_layers // 2)}, (aa, num_splits)
