"""The ColorJitter / vertical-flip kernel (cotb200_aug_color_jitter) byte for byte against the reference's PIL outputs in
tests/golden/augment_jitter.npz and tests/jitter_ref.py, and the random-erasing kernel (cotb200_aug_erase) against the fixture's
'const' batches and the properties of its 'rand' / 'pixel' values."""
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

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment_jitter.npz")
CONFIGS = (0.4, (0.4, 0.4, 0.4, 0.1))
MEAN = tuple(x * 255 for x in (0.485, 0.456, 0.406))
STD = tuple(x * 255 for x in (0.229, 0.224, 0.225))


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _draw(tf, s, H, W):
    return tf.draw_one(H, W, random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


def _train(tf, imgs, draws):
    sizes = [a.shape[:2] for a in imgs]
    data = torch.from_numpy(np.concatenate([np.ascontiguousarray(a).reshape(-1) for a in imgs]))
    rec, jrec = tf.pack(sizes, draws), tf.pack_jitter(draws)
    batch = augment.AugBatch(data, torch.from_numpy(rec.view(np.uint8).copy()), torch.zeros(len(imgs), dtype=torch.int64),
                             torch.from_numpy(jrec.view(np.uint8).copy()))
    out = augment.run(batch, tf.size, randaug=tf.num_layers > 0)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _fixture_case(gold, prefix, tf):
    imgs, draws, want = [], [], []
    k = 0
    while "%s_%d" % (prefix, k) in gold:
        H, W, seed, iseed = (int(v) for v in gold["%s_%d_size" % (prefix, k)])
        imgs.append(aug_ref.source_image(iseed, H, W))
        draws.append(_draw(tf, seed, H, W))
        want.append(gold["%s_%d" % (prefix, k)])
        k += 1
    assert k >= 4
    return imgs, draws, want


@pytest.mark.parametrize("c", [0, 1])
def test_jitter_equals_reference_fixture(gold, c):
    tf = augment.TrainAugment(auto_augment=None, color_jitter=CONFIGS[c], vflip=0.5)
    imgs, draws, want = _fixture_case(gold, "jout_%d" % c, tf)
    got = _train(tf, imgs, draws)
    for n in range(len(imgs)):
        np.testing.assert_array_equal(got[n], want[n], err_msg="image %d" % n)


def test_vflip_randaug_equals_reference_fixture(gold):
    tf = augment.TrainAugment(vflip=0.5, color_jitter=0.4)
    imgs, draws, want = _fixture_case(gold, "jra", tf)
    got = _train(tf, imgs, draws)
    for n in range(len(imgs)):
        np.testing.assert_array_equal(got[n], want[n], err_msg="image %d" % n)


@pytest.mark.parametrize("S", [224, 256, 97])
def test_jitter_random_sweep_equals_oracle(S):
    """All 24 op orders, subsets of them, hue of both signs incl. +-0.5 (wrap-around), vflip on and off, mixed image sizes."""
    r = np.random.RandomState(S)
    tf = augment.TrainAugment(size=S, auto_augment=None, color_jitter=(0.4, 0.4, 0.4, 0.5), vflip=0.5)
    hues = [0.5, -0.5, 0.1, -0.1, 0.003, -0.003, 0.0, 0.25]
    imgs, draws = [], []
    for n, perm in enumerate(list(itertools.permutations(range(4))) * 2):
        H, W = (int(v) for v in r.randint(40, 600, 2))
        img = aug_ref.source_image(S * 100 + n, H, W)
        p = _draw(tf, S * 1000 + n, H, W)
        f = [float(v) for v in r.uniform(0.0, 2.0, 3)] + [hues[n % len(hues)]]
        order = list(perm) if n < 24 else [k for k in perm if r.rand() < 0.6]
        p["jitter"] = dict(order=order, factors=f)
        p["vflip"] = bool(n % 3 == 0)
        imgs.append(img)
        draws.append(p)
    got = _train(tf, imgs, draws)
    for n in range(len(imgs)):
        np.testing.assert_array_equal(got[n], jitter_ref.train_sample_jitter(imgs[n], draws[n], S), err_msg="draw %s" % (draws[n],))


def test_vflip_with_randaug_random_draws_equal_oracle():
    tf = augment.TrainAugment(vflip=0.5)
    r = np.random.RandomState(3)
    sizes = [(int(a), int(b)) for a, b in r.randint(60, 700, (24, 2))]
    imgs = [aug_ref.source_image(50 + n, H, W) for n, (H, W) in enumerate(sizes)]
    draws = [_draw(tf, 900 + n, H, W) for n, (H, W) in enumerate(sizes)]
    assert any(d["vflip"] for d in draws) and not all(d["vflip"] for d in draws)
    got = _train(tf, imgs, draws)
    for n in range(len(imgs)):
        np.testing.assert_array_equal(got[n], jitter_ref.train_sample_jitter(imgs[n], draws[n]), err_msg="draw %s" % (draws[n],))


def test_hue_kernel_equals_oracle_on_every_colour():
    a = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8)          # [2^24, 3]
    planar = torch.from_numpy(img.reshape(256, 256 * 256, 3).transpose(0, 2, 1).copy()).cuda()  # 256 images of 256 x 256
    lib = _lib.load()
    for hue in (0.1, -0.1, 0.5, -0.5, 0.37):
        rec = np.zeros(256, augment.JITTER_DTYPE)
        rec["order"] = -1
        rec["order"][:, 0] = 3
        rec["hue"] = hue
        out = planar.clone()
        dev = torch.from_numpy(rec.view(np.uint8).copy()).cuda()
        _lib.check(lib.cotb200_aug_color_jitter(256, 256, rec.ctypes.data, dev.data_ptr(), out.data_ptr(), _lib.stream_ptr(out)),
                   "aug_color_jitter")
        got = out.cpu().numpy().transpose(0, 2, 1).reshape(-1, 3)
        want = jitter_ref.adjust_hue(img.reshape(4096, 4096, 3), hue).reshape(-1, 3)
        bad = np.any(got != want, -1)
        assert not bad.any(), (hue, img[bad][:4], got[bad][:4], want[bad][:4])


def test_default_train_augment_launches_as_before():
    r = np.random.RandomState(9)
    items = [(aug_ref.source_image(k, int(H), int(W)), k) for k, (H, W) in enumerate(r.randint(100, 500, (8, 2)))]
    counts = {}
    for name, tf in (("default", augment.TrainAugment()), ("aa_with_cj", augment.TrainAugment(color_jitter=0.4)),
                     ("jitter", augment.TrainAugment(auto_augment=None, color_jitter=0.4))):
        random.seed(4)
        np.random.seed(4)
        torch.manual_seed(4)
        batch = tf.collate(items)
        assert (batch.jitter is None) == (name != "jitter")
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        tf(batch)
        torch.cuda.synchronize()
        counts[name] = _lib.launch_count() - n0
    assert counts == {"default": 3, "aa_with_cj": 3, "jitter": 3}       # hpass, vpass + randaug or color_jitter


def test_collate_and_call_with_jitter_end_to_end():
    tf = augment.TrainAugment(auto_augment=None, color_jitter=(0.4, 0.4, 0.4, 0.1), vflip=0.5)
    r = np.random.RandomState(2)
    items = [(aug_ref.source_image(k, int(H), int(W)), k) for k, (H, W) in enumerate(r.randint(100, 500, (8, 2)))]
    random.seed(5)
    np.random.seed(5)
    torch.manual_seed(5)
    x, y = tf(tf.collate(items))
    random.seed(5)
    np.random.seed(5)
    torch.manual_seed(5)
    draws = tf.draw([a.shape[:2] for a, _ in items], random, np.random, torch.default_generator)
    torch.cuda.synchronize()
    for k, (a, _) in enumerate(items):
        np.testing.assert_array_equal(x[k].cpu().numpy(), jitter_ref.train_sample_jitter(a, draws[k]))


# ---------------------------------------------------------------- random erasing
def _case(gold, name):
    p, mode, count, splits, B, H, W, seed = gold["er_case_%s" % name]
    er = augment.RandomErasing(p, ("const", "rand", "pixel")[int(mode)], int(count), int(splits))
    return er, int(B), int(H), int(W), int(seed)


def _erase(er, x, boxes, seed=0):
    er.apply(x, augment.EraseParams(er.pack(boxes, seed), x.device))
    torch.cuda.synchronize()
    return x


def _bits(t):
    return t.cpu().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).numpy()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", ["c1", "c3s"])
def test_erase_const_equals_reference_fixture(gold, name, dtype):
    er, B, H, W, seed = _case(gold, name)
    u8 = torch.from_numpy(gold["er_u8"]).cuda()
    x = normalize_u8(u8, MEAN, STD, dtype=dtype)
    _erase(er, x, er.draw(B, H, W, random.Random(seed)))
    want = torch.from_numpy(gold["er_const_%s" % name]).to(dtype)
    np.testing.assert_array_equal(_bits(x), _bits(want))


def test_erase_with_mix_keeps_the_mixed_batch_outside_the_boxes():
    from cotnet_b200.trainer import MixupCutmix
    u8 = torch.randint(0, 256, (8, 3, 64, 64), dtype=torch.uint8).cuda()
    mix = MixupCutmix(seed=1).draw(8, 64, 64)
    base = normalize_u8(u8, MEAN, STD, mix=mix)
    er = augment.RandomErasing(1.0, "pixel", 3, seed=2)
    boxes = er.draw(8, 64, 64)
    x = _erase(er, base.clone(), boxes)
    own = jitter_ref.erase_owner(8, 64, 64, boxes)
    keep = np.broadcast_to((own < 0)[:, None], x.shape)
    assert (own >= 0).any() and keep.any()
    np.testing.assert_array_equal(_bits(x)[keep], _bits(base)[keep])


def _random_batch(B, H, W, dtype=torch.float32):
    g = torch.Generator().manual_seed(B * H)
    return normalize_u8(torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g).cuda(), MEAN, STD, dtype=dtype)


@pytest.mark.parametrize("name", ["r3", "p1", "p3s"])
def test_erase_rand_pixel_outside_boxes_and_per_box_values(gold, name):
    er, B, H, W, seed = _case(gold, name)
    base = _random_batch(B, H, W)
    boxes = er.draw(B, H, W, random.Random(seed))
    x = _erase(er, base.clone(), boxes, seed=11).cpu().numpy()
    own = jitter_ref.erase_owner(B, H, W, boxes)
    keep = np.broadcast_to((own < 0)[:, None], x.shape)
    np.testing.assert_array_equal(x[keep].view(np.int32), base.cpu().numpy()[keep].view(np.int32))
    assert (own >= 0).sum() > 1000
    for n in range(B):
        for k in range(int(own[n].max()) + 1):
            m = own[n] == k
            if not m.any():
                continue
            for c in range(3):
                v = x[n, c][m]
                assert np.isfinite(v).all()
                if er.mode == "rand":
                    assert (v == v[0]).all(), (n, k, c)                      # one value per (sample, box, channel)
                elif m.sum() > 16:
                    assert len(np.unique(v)) > m.sum() // 2, (n, k, c)        # a value per element


@pytest.mark.parametrize("mode", ["rand", "pixel"])
def test_erase_later_box_wins(mode):
    er = augment.RandomErasing(1.0, mode, 3)
    b0, b1, b0_far = (10, 10, 100, 100), (60, 60, 100, 100), (0, 150, 20, 20)
    base = _random_batch(2, 224, 224)
    a = _erase(er, base.clone(), [[b0, b1], []], seed=3).cpu().numpy()
    only0 = _erase(er, base.clone(), [[b0], []], seed=3).cpu().numpy()              # b0 is box 0 in both
    only1 = _erase(er, base.clone(), [[b0_far, b1], []], seed=3).cpu().numpy()      # b1 is box 1 in both
    own = jitter_ref.erase_owner(2, 224, 224, [[b0, b1], []])
    m1 = np.broadcast_to((own == 1)[:, None], a.shape)
    m0 = np.broadcast_to((own == 0)[:, None], a.shape)
    np.testing.assert_array_equal(a[m1], only1[m1])
    np.testing.assert_array_equal(a[m0], only0[m0])
    overlap = np.zeros_like(m1)
    overlap[0, :, 60:110, 60:110] = True
    assert not np.array_equal(a[overlap], only0[overlap])


def test_erase_pixel_values_are_standard_normal():
    from scipy import stats
    er = augment.RandomErasing(1.0, "pixel", 1)
    x = _erase(er, _random_batch(8, 224, 224), [[(0, 0, 224, 224)]] * 8, seed=12345).cpu().numpy().ravel()
    assert x.size >= 10 ** 6
    assert abs(x.mean()) < 0.01 and abs(x.std() - 1) < 0.01
    assert stats.kstest(x, "norm").pvalue > 1e-4


@pytest.mark.parametrize("mode", ["rand", "pixel"])
def test_erase_seed_determines_the_values(mode):
    er = augment.RandomErasing(1.0, mode, 2)
    boxes = er.draw(16, 224, 224, random.Random(1))
    base = _random_batch(16, 224, 224)
    a = _bits(_erase(er, base.clone(), boxes, seed=77))
    b = _bits(_erase(er, base.clone(), boxes, seed=77))
    c = _bits(_erase(er, base.clone(), boxes, seed=78))
    np.testing.assert_array_equal(a, b)
    own = jitter_ref.erase_owner(16, 224, 224, boxes)
    m = np.broadcast_to((own >= 0)[:, None], a.shape)
    assert (a[m] != c[m]).mean() > 0.99


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_erase_16bit_values_are_the_fp32_values_rounded(dtype):
    er = augment.RandomErasing(1.0, "pixel", 3)
    boxes = er.draw(8, 224, 224, random.Random(2))
    own = jitter_ref.erase_owner(8, 224, 224, boxes)
    m = np.broadcast_to((own >= 0)[:, None], (8, 3, 224, 224))
    f = _erase(er, _random_batch(8, 224, 224), boxes, seed=5)
    h = _erase(er, _random_batch(8, 224, 224, dtype), boxes, seed=5)
    np.testing.assert_array_equal(_bits(h)[m], _bits(f.to(dtype))[m])


def test_random_erasing_call_end_to_end():
    er = augment.RandomErasing(0.5, "rand", 3, num_splits=2, seed=9)
    base = _random_batch(32, 224, 224, torch.bfloat16)
    x = er(base.clone())
    torch.cuda.synchronize()
    boxes = augment.RandomErasing(0.5, "rand", 3, num_splits=2, seed=9).draw(32, 224, 224)
    assert all(not b for b in boxes[:16]) and any(boxes[16:])
    own = jitter_ref.erase_owner(32, 224, 224, boxes)
    xb, bb = _bits(x), _bits(base)
    keep = np.broadcast_to((own < 0)[:, None], xb.shape)
    np.testing.assert_array_equal(xb[keep], bb[keep])
    assert (xb[~keep] != bb[~keep]).mean() > 0.9
