"""The augmentation above 256 x 256 on the thread-block-cluster kernels (cotb200_aug_randaug_cluster,
cotb200_aug_color_jitter_cluster), byte for byte: against the reference's PIL outputs at 288 and 320 in
tests/golden/augment_large.npz, against oracle/aug_ref.py and tests/jitter_ref.py for every op and jitter order at the four
cluster sizes (S = 257, 320, 384, 512: 1, 2, 3 and 4 CTAs) and on random draws, and against the one-CTA kernels at 224 and 256."""
import itertools
import os
import random

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, augment
from cotnet_b200.trainer import normalize_u8
import jitter_ref
from oracle import aug_ref

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "augment_large.npz")
OPS_GOLD = os.path.join(HERE, "golden", "augment.npz")
CLUSTER = {257: 1, 320: 2, 384: 3, 512: 4}             # S -> CTAs per cluster (the band budget of include/cotb200.h)
MEAN = tuple(x * 255 for x in (0.485, 0.456, 0.406))
STD = tuple(x * 255 for x in (0.229, 0.224, 0.225))


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _draw(tf, s, H, W):
    return tf.draw_one(H, W, random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


def _batch(tf, imgs, draws):
    sizes = [a.shape[:2] for a in imgs]
    data = torch.from_numpy(np.concatenate([np.ascontiguousarray(a).reshape(-1) for a in imgs]))
    jit = None
    if tf.has_jitter_kernel:
        jit = torch.from_numpy(tf.pack_jitter(draws).view(np.uint8).copy())
    return augment.AugBatch(data, torch.from_numpy(tf.pack(sizes, draws).view(np.uint8).copy()),
                            torch.zeros(len(imgs), dtype=torch.int64), jit)


def _run(tf, imgs, draws, cluster=None):
    out = augment.run(_batch(tf, imgs, draws), tf.size, randaug=tf.num_layers > 0, cluster=cluster)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _cases(gold, prefix):
    k = 0
    while "%s_%d" % (prefix, k) in gold:
        yield [int(v) for v in gold["%s_%d_size" % (prefix, k)]], gold["%s_%d" % (prefix, k)]
        k += 1


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


# ---------------------------------------------------------------- the reference's PIL outputs
@pytest.mark.parametrize("S", [288, 320])
def test_train_equals_reference_fixture(gold, S):
    tf = augment.TrainAugment(size=S)
    cases = list(_cases(gold, "train_%d" % S))
    imgs = [aug_ref.source_image(iseed, H, W) for (H, W, _, iseed), _ in cases]
    draws = [_draw(tf, seed, H, W) for (H, W, seed, _), _ in cases]
    got = _run(tf, imgs, draws)
    assert len(cases) >= 4
    for n, (_, want) in enumerate(cases):
        np.testing.assert_array_equal(got[n], want, err_msg="train %d image %d" % (S, n))


def test_jitter_equals_reference_fixture(gold):
    tf = augment.TrainAugment(size=320, auto_augment=None, color_jitter=0.4, vflip=0.5)
    cases = list(_cases(gold, "jout_320"))
    imgs = [aug_ref.source_image(iseed, H, W) for (H, W, _, iseed), _ in cases]
    draws = [_draw(tf, seed, H, W) for (H, W, seed, _), _ in cases]
    got = _run(tf, imgs, draws)
    assert len(cases) >= 4
    for n, (_, want) in enumerate(cases):
        np.testing.assert_array_equal(got[n], want, err_msg="jitter image %d" % n)


@pytest.mark.parametrize("S", [288, 320])
def test_eval_equals_reference_fixture(gold, S):
    ev = augment.EvalTransform(size=S, crop_pct=float(gold["eval_%d_crop_pct" % S]))
    cases = list(_cases(gold, "eval_%d" % S))
    imgs = [aug_ref.source_image(iseed, H, W) for (H, W, iseed), _ in cases]
    data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs]))
    rec = ev.pack([a.shape[:2] for a in imgs])
    batch = augment.AugBatch(data, torch.from_numpy(rec.view(np.uint8).copy()), torch.zeros(len(imgs), dtype=torch.int64))
    x, _ = ev(batch)
    got = x.cpu().numpy()
    for n, (_, want) in enumerate(cases):
        np.testing.assert_array_equal(got[n], want, err_msg="eval %d image %d" % (S, n))


# ---------------------------------------------------------------- every op and jitter order at every cluster size
def _band_ops(S):
    """Ops placed on the band boundaries of S: Cutout boxes across each boundary (and the image's edges), translations by a
    few rows that pull a neighbouring band's rows in, and a shear whose rows next to a boundary read across it."""
    cs = CLUSTER[S]
    R = -(-S // cs)
    ops = []
    for r in range(cs + 1):
        y = r * R
        for x0, h in ((3, 1), (S // 3, 6), (S - 20, 40)):
            ops.append({"id": 15, "box": (x0, y - h, min(S, x0 + 30), min(S, y + h))})
        for t in (-2.5, 1.0, 3.0):
            ops.append({"id": 14, "matrix": (1, 0, 0, 0, 1, t), "filter": 1})
    ops.append({"id": 12, "matrix": (1, 0, 0, 0.3, 1, 0), "filter": 0})
    ops.append({"id": 10, "factor": 1.9})
    return ops


@pytest.mark.parametrize("S", sorted(CLUSTER))
def test_every_op_equals_oracle_at_every_cluster_size(S):
    """Each op of the fixture's cases (16 ops, three magnitudes, both signs) alone, the band-boundary ops alone, and pairs of
    them (a neighbour op after a shared-memory op and the other way round) on an S x S image (the resize is the identity)."""
    cases = aug_ref.load_golden(OPS_GOLD)["op_cases"]
    single = [aug_ref.fixture_op(c, S) for c in cases] + _band_ops(S)
    r = np.random.RandomState(S)
    pairs = [[single[int(a)], single[int(b)]] for a, b in r.randint(0, len(single), (48, 2))]
    tf = augment.TrainAugment(size=S)
    src = aug_ref.source_image(S, S, S)
    draws = [dict(i=0, j=0, h=S, w=S, filter=1, flip=False, ops=[op, None]) for op in single]
    draws += [dict(i=0, j=0, h=S, w=S, filter=1, flip=False, ops=p) for p in pairs]
    for lo in range(0, len(draws), 64):
        part = draws[lo:lo + 64]
        got = _run(tf, [src] * len(part), part)
        for n, d in enumerate(part):
            np.testing.assert_array_equal(got[n], aug_ref.train_sample(src, d, S), err_msg="S=%d ops %s" % (S, d["ops"]))


@pytest.mark.parametrize("S", sorted(CLUSTER))
def test_jitter_orders_and_vflip_equal_oracle_at_every_cluster_size(S):
    """All 24 op orders and subsets of them, hue of both signs incl. +-0.5, vflip on and off."""
    r = np.random.RandomState(S)
    tf = augment.TrainAugment(size=S, auto_augment=None, color_jitter=(0.4, 0.4, 0.4, 0.5), vflip=0.5)
    hues = [0.5, -0.5, 0.1, -0.1, 0.003, -0.003, 0.0, 0.25]
    imgs, draws = [], []
    for n, perm in enumerate(list(itertools.permutations(range(4))) * 2):
        H, W = (int(v) for v in r.randint(200, 700, 2))
        p = _draw(tf, S * 1000 + n, H, W)
        f = [float(v) for v in r.uniform(0.0, 2.0, 3)] + [hues[n % len(hues)]]
        p["jitter"] = dict(order=list(perm) if n < 24 else [k for k in perm if r.rand() < 0.6], factors=f)
        p["vflip"] = bool(n % 3 == 0)
        imgs.append(aug_ref.source_image(S * 100 + n, H, W))
        draws.append(p)
    got = _run(tf, imgs, draws)
    for n in range(len(imgs)):
        np.testing.assert_array_equal(got[n], jitter_ref.train_sample_jitter(imgs[n], draws[n], S), err_msg="draw %s" % (draws[n],))


# ---------------------------------------------------------------- random draws at 288 and 320
@pytest.mark.parametrize("S", [288, 320])
def test_train_random_draws_equal_oracle(S):
    r = np.random.RandomState(S)
    for interp in ("bicubic", "random"):
        tf = augment.TrainAugment(size=S, interpolation=interp, vflip=0.5 if interp == "random" else 0.)
        sizes = _sizes(r, 60)
        imgs = [aug_ref.source_image(3 * S + n, H, W) for n, (H, W) in enumerate(sizes)]
        draws = [_draw(tf, 7919 * S + 101 * len(interp) + n, H, W) for n, (H, W) in enumerate(sizes)]
        got = _run(tf, imgs, draws)
        for n in range(len(imgs)):
            want = jitter_ref.train_sample_jitter(imgs[n], draws[n], S)
            np.testing.assert_array_equal(got[n], want, err_msg="%s image %d %s draw %s" % (interp, n, sizes[n], draws[n]))


def test_jitter_random_draws_equal_oracle_at_320():
    r = np.random.RandomState(1)
    tf = augment.TrainAugment(size=320, auto_augment=None, color_jitter=(0.4, 0.4, 0.4, 0.1), vflip=0.5)
    sizes = _sizes(r, 100)
    imgs = [aug_ref.source_image(40 + n, H, W) for n, (H, W) in enumerate(sizes)]
    draws = [_draw(tf, 500 + n, H, W) for n, (H, W) in enumerate(sizes)]
    got = _run(tf, imgs, draws)
    for n in range(len(imgs)):
        np.testing.assert_array_equal(got[n], jitter_ref.train_sample_jitter(imgs[n], draws[n], 320), err_msg="draw %s" % (draws[n],))


@pytest.mark.parametrize("aa", ["rand-m15-mstd0.5-n2", None])
def test_three_splits_and_random_erasing_at_320(aa):
    S, B = 320, 12
    tf = augment.TrainAugment(size=S, auto_augment=aa, color_jitter=0.4, vflip=0.5, num_splits=3)
    r = np.random.RandomState(3)
    sizes = _sizes(r, B)
    imgs = [aug_ref.source_image(80 + n, H, W) for n, (H, W) in enumerate(sizes)]
    draws = tf.draw(sizes, random.Random(5), np.random.RandomState(5), torch.Generator().manual_seed(5))
    x, y = tf(tf.collate_draws(imgs, list(range(B)), draws))
    torch.cuda.synchronize()
    assert x.shape == (3 * B, 3, S, S) and y.tolist() == list(range(B)) * 3
    got = x.cpu().numpy()
    for n, p in enumerate(draws):
        views = [dict(p, ops=[])] + [dict(p, ops=v.get("ops", []), jitter=v.get("jitter")) for v in p["views"]]
        for k, d in enumerate(views):
            np.testing.assert_array_equal(got[k * B + n], jitter_ref.train_sample_jitter(imgs[n], d, S), err_msg="view %d image %d" % (k, n))
    z = normalize_u8(x, MEAN, STD, dtype=torch.float32)
    er = augment.RandomErasing(1.0, "const", 3, num_splits=3, seed=4)
    boxes = er.draw(3 * B, S, S, random.Random(9))
    before = z.clone()
    er.apply(z, augment.EraseParams(er.pack(boxes, 1), z.device))
    torch.cuda.synchronize()
    own = jitter_ref.erase_owner(3 * B, S, S, boxes)
    hit = np.broadcast_to((own >= 0)[:, None], z.shape)
    a, b = z.cpu().numpy(), before.cpu().numpy()
    assert hit[:B].sum() == 0 and hit.sum() > 0
    np.testing.assert_array_equal(a[~hit].view(np.int32), b[~hit].view(np.int32))
    assert (a[hit] == 0).all()


# ---------------------------------------------------------------- the cluster kernels against the one-CTA kernels
@pytest.mark.parametrize("S", [224, 256])
def test_cluster_kernels_equal_one_cta_kernels(S):
    r = np.random.RandomState(S + 1)
    for tf in (augment.TrainAugment(size=S, vflip=0.5, interpolation="random"),
               augment.TrainAugment(size=S, auto_augment=None, color_jitter=(0.4, 0.4, 0.4, 0.5), vflip=0.5)):
        for b in range(2):
            sizes = _sizes(r, 110)
            imgs = [aug_ref.source_image(1000 * b + n, H, W) for n, (H, W) in enumerate(sizes)]
            draws = [_draw(tf, 31 * S + 1000 * b + n, H, W) for n, (H, W) in enumerate(sizes)]
            one = _run(tf, imgs, draws, cluster=False)
            cl = _run(tf, imgs, draws, cluster=True)
            np.testing.assert_array_equal(cl, one)


def test_two_runs_give_identical_bytes():
    r = np.random.RandomState(2)
    for tf in (augment.TrainAugment(size=320), augment.TrainAugment(size=512, auto_augment=None, color_jitter=(0.4, 0.4, 0.4, 0.1),
                                                                      vflip=0.5)):
        sizes = _sizes(r, 24)
        imgs = [aug_ref.source_image(n, H, W) for n, (H, W) in enumerate(sizes)]
        draws = [_draw(tf, 60 + n, H, W) for n, (H, W) in enumerate(sizes)]
        np.testing.assert_array_equal(_run(tf, imgs, draws), _run(tf, imgs, draws))


def test_profiler_records_show_the_dispatch():
    r = np.random.RandomState(8)
    items = [(aug_ref.source_image(k, int(H), int(W)), k) for k, (H, W) in enumerate(r.randint(100, 600, (8, 2)))]
    seen = {}
    for S in (224, 320):
        for kw in (dict(), dict(auto_augment=None, color_jitter=0.4)):
            tf = augment.TrainAugment(size=S, **kw)
            batch = tf.collate_draws([a for a, _ in items], list(range(8)),
                                     tf.draw([a.shape[:2] for a, _ in items], random.Random(S), np.random.RandomState(S),
                                             torch.Generator().manual_seed(S)))
            torch.cuda.synchronize()
            _lib.prof_enable(True)
            try:
                tf(batch)
                torch.cuda.synchronize()
                rep = _lib.prof_report()
            finally:
                _lib.prof_enable(False)
            seen[S, "jitter" if kw else "randaug"] = sorted(rep)
    assert seen[224, "randaug"] == ["aug_hpass", "aug_randaug", "aug_vpass"]
    assert seen[224, "jitter"] == ["aug_hpass", "aug_jitter", "aug_vpass"]
    assert seen[320, "randaug"] == ["aug_hpass", "aug_randaug_cluster", "aug_vpass"]
    assert seen[320, "jitter"] == ["aug_hpass", "aug_jitter_cluster", "aug_vpass"]
