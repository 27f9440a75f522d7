"""The augmentation kernels (cotb200_aug_resize_crop, cotb200_aug_randaug) byte for byte: against the reference's PIL outputs
in tests/golden/augment.npz and against oracle/aug_ref.py on random draws over ImageNet-like sizes."""
import os
import random

import numpy as np
import pytest
import torch

from cotnet_b200 import augment
from oracle import aug_ref

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment.npz")


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _batch(imgs, rec):
    data = torch.from_numpy(np.concatenate([np.ascontiguousarray(a).reshape(-1) for a in imgs]))
    return augment.AugBatch(data, torch.from_numpy(rec.view(np.uint8).copy()), torch.zeros(len(imgs), dtype=torch.int64))


def _train(tf, imgs, draws):
    rec = tf.pack([a.shape[:2] for a in imgs], draws)
    out = augment.run(_batch(imgs, rec), tf.size)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _draw(tf, s, H, W):
    return tf.draw_one(H, W, random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


def test_train_equals_reference_fixture(gold):
    tf = augment.TrainAugment()
    imgs, draws, want = [], [], []
    k = 0
    while "train_%d" % k in gold:
        H, W, seed, iseed = (int(v) for v in gold["train_%d_size" % k])
        imgs.append(aug_ref.source_image(iseed, H, W))
        draws.append(_draw(tf, seed, H, W))
        want.append(gold["train_%d" % k])
        k += 1
    got = _train(tf, imgs, draws)                    # one ragged batch of mixed sizes
    for n in range(k):
        np.testing.assert_array_equal(got[n], want[n], err_msg="train image %d" % n)


def test_ops_equal_reference_fixture(gold):
    src = gold["op_src"]
    S = src.shape[0]
    cases = gold["op_cases"]
    tf = augment.TrainAugment(size=S)
    draws = [dict(i=0, j=0, h=S, w=S, filter=1, flip=False, ops=[aug_ref.fixture_op(c, S)]) for c in cases]
    got = _train(tf, [src] * len(cases), draws)      # an unchanged size: the resize is the identity
    for n, c in enumerate(cases):
        np.testing.assert_array_equal(got[n], gold["op_%d" % int(c[2])].transpose(2, 0, 1), err_msg="op case %s" % (c,))


def test_eval_equals_reference_fixture(gold):
    ev = augment.EvalTransform()
    imgs, want = [], []
    k = 0
    while "eval_%d" % k in gold:
        H, W, iseed = (int(v) for v in gold["eval_%d_size" % k])
        imgs.append(aug_ref.source_image(iseed, H, W))
        want.append(gold["eval_%d" % k])
        k += 1
    out = augment.run(_batch(imgs, ev.pack([a.shape[:2] for a in imgs])), 224, randaug=False).cpu().numpy()
    for n in range(k):
        np.testing.assert_array_equal(out[n], want[n], err_msg="eval image %d" % n)


def _sizes(r, n):
    """ImageNet-like: mostly 4:3 / 3:4 around 500 x 375, some small, some large, some extreme."""
    out = []
    for _ in range(n):
        u = r.rand()
        if u < 0.6:
            H, W = (375, 500) if r.rand() < 0.7 else (500, 375)
            H, W = H + int(r.randint(-60, 61)), W + int(r.randint(-60, 61))
        elif u < 0.8:
            H, W = (int(v) for v in r.randint(40, 260, 2))
        elif u < 0.95:
            H, W = (int(v) for v in r.randint(600, 1400, 2))
        else:
            H, W = (int(r.randint(20, 60)), int(r.randint(400, 800)))
        out.append((H, W))
    return out


@pytest.mark.parametrize("interp", ["bicubic", "random"])
def test_train_equals_oracle_random_sweep(interp):
    r = np.random.RandomState(11 if interp == "bicubic" else 12)
    tf = augment.TrainAugment(interpolation=interp)
    for b in range(5):
        sizes = _sizes(r, 50)
        imgs = [aug_ref.source_image(1000 * b + n, H, W) for n, (H, W) in enumerate(sizes)]
        draws = [_draw(tf, 7919 * b + n, H, W) for n, (H, W) in enumerate(sizes)]
        got = _train(tf, imgs, draws)
        for n in range(len(imgs)):
            want = aug_ref.train_sample(imgs[n], draws[n])
            np.testing.assert_array_equal(got[n], want, err_msg="batch %d image %d %s draw %s" % (b, n, sizes[n], draws[n]))


def test_every_op_at_224_equals_oracle():
    r = np.random.RandomState(5)
    tf = augment.TrainAugment()
    base = aug_ref.source_image(77, 300, 400)
    draws, ops = [], []
    for i in range(16):
        for _ in range(3):
            for sign in (1, -1):
                rnd = random.Random(int(r.randint(1 << 30)))
                d = None
                while d is None:                    # draw until op i is applied
                    d = tf._op(i, rnd, np.random.RandomState(int(r.randint(1 << 30))))
                ops.append(d)
                draws.append(dict(i=10, j=20, h=280, w=370, filter=1, flip=bool(sign < 0), ops=[d, ops[len(ops) // 2]]))
    got = _train(tf, [base] * len(draws), draws)
    for n, d in enumerate(draws):
        np.testing.assert_array_equal(got[n], aug_ref.train_sample(base, d), err_msg="draw %s" % (d,))


@pytest.mark.parametrize("n", [1, 3])
def test_small_and_odd_batches_and_repeats(n):
    tf = augment.TrainAugment()
    r = np.random.RandomState(n)
    sizes = _sizes(r, n)
    imgs = [aug_ref.source_image(n + k, H, W) for k, (H, W) in enumerate(sizes)]
    draws = [_draw(tf, 31 * n + k, H, W) for k, (H, W) in enumerate(sizes)]
    a = _train(tf, imgs, draws)
    b = _train(tf, imgs, draws)
    np.testing.assert_array_equal(a, b)
    for k in range(n):
        np.testing.assert_array_equal(a[k], aug_ref.train_sample(imgs[k], draws[k]))


def test_collate_and_call_end_to_end():
    tf = augment.TrainAugment()
    r = np.random.RandomState(9)
    items = [(aug_ref.source_image(k, H, W), k) for k, (H, W) in enumerate(_sizes(r, 8))]
    random.seed(4)
    np.random.seed(4)
    torch.manual_seed(4)
    batch = tf.collate(items)
    x, y = tf(batch)
    random.seed(4)
    np.random.seed(4)
    torch.manual_seed(4)
    draws = tf.draw([a.shape[:2] for a, _ in items], random, np.random, torch.default_generator)
    torch.cuda.synchronize()
    assert x.shape == (8, 3, 224, 224) and x.dtype == torch.uint8
    assert y.tolist() == list(range(8))
    for k, (a, _) in enumerate(items):
        np.testing.assert_array_equal(x[k].cpu().numpy(), aug_ref.train_sample(a, draws[k]))
    # the batch feeds the existing normalisation / mix path unchanged
    from cotnet_b200.trainer import MixupCutmix, normalize_u8
    mix = MixupCutmix(seed=0).draw(8, 224, 224)
    z = normalize_u8(x, (0.485 * 255, 0.456 * 255, 0.406 * 255), (0.229 * 255, 0.224 * 255, 0.225 * 255), mix=mix)
    assert z.shape == (8, 3, 224, 224) and torch.isfinite(z.float()).all()
