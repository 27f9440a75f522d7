"""CPU checks of ColorJitter, the vertical flip and random erasing: the draws equal the reference's (tests/golden/augment_jitter.npz),
the numpy restatement tests/jitter_ref.py equals the fixture's PIL outputs and Pillow's HSV conversions over every colour, and
the C entry points reject malformed structs before any launch."""
import math
import os
import random

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, augment
import jitter_ref
from oracle import aug_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment_jitter.npz")
CONFIGS = (0.4, (0.4, 0.4, 0.4, 0.1))


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _tf(c):
    return augment.TrainAugment(auto_augment=None, color_jitter=CONFIGS[c], vflip=0.5)


def _draw(tf, s, H, W):
    return tf.draw_one(H, W, random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


@pytest.mark.parametrize("c", [0, 1])
def test_jitter_draws_equal_reference(gold, c):
    tf = _tf(c)
    for s, (H, W) in enumerate(gold["jd_sizes"]):
        rnd, nrnd, tgen = random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s)
        p = tf.draw_one(int(H), int(W), rnd, nrnd, tgen)
        assert (p["i"], p["j"], p["h"], p["w"]) == tuple(gold["jd_crop_%d" % c][s]), s
        assert int(p["flip"]) == gold["jd_flip_%d" % c][s] and int(p["vflip"]) == gold["jd_vflip_%d" % c][s], s
        want_f = gold["jd_factors_%d" % c][s]
        assert [f is None for f in p["jitter"]["factors"]] == [math.isnan(v) for v in want_f], s
        assert [f for f in p["jitter"]["factors"] if f is not None] == [v for v in want_f if not math.isnan(v)], s
        perm = [int(k) for k in gold["jd_perm_%d" % c][s]]
        assert p["jitter"]["order"] == [k for k in perm if not math.isnan(want_f[k])], s
        assert (rnd.random(), nrnd.random_sample(), float(torch.rand(1, generator=tgen))) == tuple(gold["jd_next_%d" % c][s]), s


def test_jitter_draws_cover_both_flips_and_hue_signs(gold):
    f = gold["jd_factors_1"]
    assert (f[:, 3] > 0).any() and (f[:, 3] < 0).any()
    assert gold["jd_vflip_1"].any() and not gold["jd_vflip_1"].all()
    assert np.isnan(gold["jd_factors_0"][:, 3]).all()


def test_auto_augment_ignores_color_jitter():
    a = augment.TrainAugment(vflip=0.5)
    b = augment.TrainAugment(vflip=0.5, color_jitter=0.4)
    assert b.jitter is None
    for s in range(40):
        da, db = _draw(a, s, 300 + s, 400 - s), _draw(b, s, 300 + s, 400 - s)
        assert da == db
    # and with the defaults, the draws and the packed structs are exactly those of TrainAugment()
    c, d = augment.TrainAugment(), augment.TrainAugment(color_jitter=0.4)
    for s in range(40):
        dc, dd = _draw(c, s, 375, 500), _draw(d, s, 375, 500)
        assert dc == dd and "vflip" not in dc and "jitter" not in dc
    assert not c.has_jitter_kernel and not d.has_jitter_kernel


def test_jitter_ranges():
    assert augment.jitter_ranges(0.4) == [(0.6, 1.4), (0.6, 1.4), (0.6, 1.4), None]
    assert augment.jitter_ranges((0.4, 0.0, 1.5, 0.1)) == [(0.6, 1.4), None, (0.0, 2.5), (-0.1, 0.1)]
    assert augment.jitter_ranges(0.0) == [None] * 4
    with pytest.raises(ValueError):
        augment.jitter_ranges((0.4, 0.4))
    with pytest.raises(ValueError):
        augment.jitter_ranges((0.4, 0.4, 0.4, 0.6))
    with pytest.raises(ValueError):
        augment.jitter_ranges(-0.1)


def test_jitter_off_still_draws_the_permutation():
    tf = augment.TrainAugment(auto_augment=None, color_jitter=0.0)
    g = torch.Generator().manual_seed(3)
    p = tf.draw_one(300, 300, random.Random(3), np.random.RandomState(3), g)
    assert p["jitter"]["order"] == [] and p["jitter"]["factors"] == [None] * 4
    ref = torch.Generator().manual_seed(3)
    torch.rand(1, generator=ref)                     # hflip
    torch.randperm(4, generator=ref)
    assert float(torch.rand(1, generator=g)) == float(torch.rand(1, generator=ref))


def test_pack_jitter_layout():
    tf = _tf(1)
    draws = [_draw(tf, s, 200, 300) for s in range(6)]
    rec = tf.pack_jitter(draws)
    assert rec.dtype.itemsize == 40
    for n, p in enumerate(draws):
        assert rec["vflip"][n] == int(p["vflip"])
        assert list(rec["order"][n]) == p["jitter"]["order"] + [-1] * (4 - len(p["jitter"]["order"]))
        assert rec["hue"][n] == p["jitter"]["factors"][3]
        assert list(rec["factor"][n]) == [np.float32(f) for f in p["jitter"]["factors"][:3]]


# ---------------------------------------------------------------- jitter_ref against the fixture and Pillow
@pytest.mark.parametrize("c", [0, 1])
def test_jitter_ref_jitter_equals_fixture(gold, c):
    tf = _tf(c)
    k = 0
    while "jout_%d_%d" % (c, k) in gold:
        H, W, seed, iseed = (int(v) for v in gold["jout_%d_%d_size" % (c, k)])
        got = jitter_ref.train_sample_jitter(aug_ref.source_image(iseed, H, W), _draw(tf, seed, H, W))
        np.testing.assert_array_equal(got, gold["jout_%d_%d" % (c, k)], err_msg="image %d" % k)
        k += 1
    assert k >= 4


def test_jitter_ref_vflip_randaug_equals_fixture(gold):
    tf = augment.TrainAugment(vflip=0.5, color_jitter=0.4)
    k = 0
    while "jra_%d" % k in gold:
        H, W, seed, iseed = (int(v) for v in gold["jra_%d_size" % k])
        got = jitter_ref.train_sample_jitter(aug_ref.source_image(iseed, H, W), _draw(tf, seed, H, W))
        np.testing.assert_array_equal(got, gold["jra_%d" % k], err_msg="image %d" % k)
        k += 1
    assert k >= 4


def _all_colours():
    a = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


def test_rgb_to_hsv_equals_pil_on_every_colour():
    Image = pytest.importorskip("PIL.Image")
    img = _all_colours()
    np.testing.assert_array_equal(jitter_ref.rgb_to_hsv(img), np.asarray(Image.fromarray(img).convert("HSV")))


def test_hsv_to_rgb_equals_pil_on_every_triple():
    Image = pytest.importorskip("PIL.Image")
    img = _all_colours()
    want = np.asarray(Image.frombytes("HSV", (4096, 4096), img.tobytes()).convert("RGB"))
    np.testing.assert_array_equal(jitter_ref.hsv_to_rgb(img), want)


def test_hue_shift_truncates_then_wraps():
    assert [jitter_ref.hue_shift(h) for h in (0.1, -0.1, 0.5, -0.5, 0.0, -0.001)] == [25, 231, 127, 129, 0, 0]


@pytest.mark.parametrize("seed", range(2))
def test_jitter_ref_jitter_ops_equal_pil(seed):
    Image = pytest.importorskip("PIL.Image")
    from PIL import ImageEnhance
    r = np.random.RandomState(seed)
    a = r.randint(0, 256, size=(int(r.randint(3, 120)), int(r.randint(3, 120)), 3)).astype(np.uint8)
    p = Image.fromarray(a)
    np.testing.assert_array_equal(jitter_ref.vflip(a), np.asarray(p.transpose(Image.FLIP_TOP_BOTTOM)))
    for order in ([0, 1, 2, 3], [3, 2, 1, 0], [1, 3], [2]):
        f = [float(v) for v in r.uniform(0.6, 1.4, 3)] + [float(r.uniform(-0.5, 0.5))]
        q = p
        for op in order:
            q = (ImageEnhance.Brightness(q).enhance(f[0]) if op == 0 else ImageEnhance.Contrast(q).enhance(f[1]) if op == 1
                 else ImageEnhance.Color(q).enhance(f[2]) if op == 2 else _pil_adjust_hue(q, f[3]))
        np.testing.assert_array_equal(jitter_ref.color_jitter(a, order, f), np.asarray(q), err_msg=str((order, f)))


def _pil_adjust_hue(img, hue_factor):                  # torchvision's adjust_hue for PIL images, restated with Pillow calls
    from PIL import Image
    h, s, v = img.convert("HSV").split()
    nh = np.array(h, dtype=np.uint8)
    nh += np.int32(hue_factor * 255).astype(np.uint8)
    return Image.merge("HSV", (Image.fromarray(nh, "L"), s, v)).convert("RGB")


# ---------------------------------------------------------------- RandomErasing draws against the fixture
def _erase_case(gold, name):
    p, mode, count, splits, B, H, W, seed = gold["er_case_%s" % name]
    er = augment.RandomErasing(p, ("const", "rand", "pixel")[int(mode)], int(count), int(splits))
    return er, int(B), int(H), int(W), int(seed)


def test_erase_draws_equal_reference(gold):
    names = [k[len("er_case_"):] for k in gold if k.startswith("er_case_")]
    assert len(names) >= 5
    for name in names:
        er, B, H, W, seed = _erase_case(gold, name)
        rnd = random.Random(seed)
        boxes = er.draw(B, H, W, rnd)
        table = [(n, k, t, l, h, w) for n, bs in enumerate(boxes) for k, (t, l, h, w) in enumerate(bs)]
        assert table == [tuple(int(v) for v in row) for row in gold["er_boxes_%s" % name]], name
        start = B // er.num_splits if er.num_splits > 1 else 0
        hit = gold["er_hit_%s" % name]
        assert (hit[:start] == -1).all() and (hit[start:] >= 0).all(), name
        for n in range(start, B):                      # an erased image may still place no box (10 failed attempts)
            assert bool(boxes[n]) <= bool(hit[n]), (name, n)
        assert rnd.random() == gold["er_next_%s" % name][0], name
    assert any(len(gold["er_boxes_%s" % n]) > 20 for n in names)


def test_erase_const_oracle_equals_fixture(gold):
    mean = np.array([x * 255 for x in (0.485, 0.456, 0.406)], np.float32).reshape(1, 3, 1, 1)
    std = np.array([x * 255 for x in (0.229, 0.224, 0.225)], np.float32).reshape(1, 3, 1, 1)
    x = (gold["er_u8"].astype(np.float32) - mean) / std
    for name in ("c1", "c3s"):
        er, B, H, W, seed = _erase_case(gold, name)
        got = jitter_ref.erase_const(x, er.draw(B, H, W, random.Random(seed)))
        np.testing.assert_array_equal(got, gold["er_const_%s" % name])
        assert (got == 0).any()


def test_erase_pack_layout():
    er = augment.RandomErasing(1.0, "pixel", 3)
    boxes = [[(1, 2, 3, 4), (0, 0, 0, 5)], [], [(5, 6, 7, 8)]]
    buf = er.pack(boxes, 0x1234_5678_9abc_def0)
    hdr = buf[:16].view(augment.ERASE_DTYPE)[0]
    assert (hdr["mode"], hdr["n_boxes"], int(hdr["seed"])) == (2, 2, 0x1234_5678_9abc_def0)
    assert buf[16:].view(augment.ERASE_BOX_DTYPE).tolist() == [(0, 0, 1, 2, 3, 4), (2, 0, 5, 6, 7, 8)]


# ---------------------------------------------------------------- C-ABI argument errors (no kernel is launched)
FAKE = 1 << 20                                          # never dereferenced: validation fails first


def _jrec(**kw):
    r = np.zeros(1, augment.JITTER_DTYPE)
    r["order"] = [0, 1, 2, 3]
    r["factor"] = [1.1, 0.9, 1.2]
    r["hue"] = 0.1
    for k, v in kw.items():
        r[k][0] = v
    return r


def _jitter(rec, S=8, N=1):
    return _lib.load().cotb200_aug_color_jitter(N, S, rec.ctypes.data, FAKE, FAKE, None)


def test_capi_color_jitter_rejects_bad_structs():
    E = -1
    for bad in (dict(order=[0, 1, 2, 4]), dict(order=[0, -2, 1, 2]), dict(order=[0, 1, 1, 2]), dict(order=[3, -1, -1, 3]),
                dict(factor=[-0.1, 1, 1]), dict(factor=[1, float("nan"), 1]), dict(factor=[1, 1, float("inf")]),
                dict(hue=0.5000001), dict(hue=-0.6), dict(hue=float("nan")), dict(vflip=2), dict(vflip=-1)):
        assert _jitter(_jrec(**bad)) == E, bad
    assert _jitter(_jrec(), N=0) == E
    assert _jitter(_jrec(), S=0) == E
    assert _jitter(_jrec(), S=257) == -7
    assert _lib.load().cotb200_aug_color_jitter(1, 8, None, FAKE, FAKE, None) == -5
    assert _lib.load().cotb200_aug_color_jitter(1, 8, _jrec().ctypes.data, None, FAKE, None) == -5


def _ebuf(boxes, mode=0):
    hdr = np.zeros(1, augment.ERASE_DTYPE)
    hdr["mode"], hdr["n_boxes"], hdr["seed"] = mode, len(boxes), 1
    return np.concatenate([hdr.view(np.uint8), np.array(boxes, augment.ERASE_BOX_DTYPE).view(np.uint8)])


def _erase(buf, N=2, C=3, H=16, W=20, dtype=_lib.F32):
    return _lib.load().cotb200_aug_erase(dtype, N, C, H, W, FAKE, buf.ctypes.data, FAKE, None)


def test_capi_erase_rejects_bad_tables():
    E = -1
    ok = [(0, 0, 1, 2, 3, 4), (0, 1, 0, 0, 16, 20), (1, 0, 15, 19, 1, 1)]
    for b in ([(0, 0, -1, 0, 2, 2)], [(0, 0, 0, -1, 2, 2)], [(0, 0, 15, 0, 2, 2)], [(0, 0, 0, 19, 2, 2)],
              [(0, 0, 0, 0, 0, 2)], [(0, 0, 0, 0, 2, 0)], [(0, 0, 0, 0, 17, 1)], [(0, 0, 0, 0, 1, 21)],
              [(2, 0, 0, 0, 1, 1)], [(-1, 0, 0, 0, 1, 1)],                       # outside the batch
              [(1, 0, 0, 0, 1, 1), (0, 0, 0, 0, 1, 1)],                          # samples out of order
              [(0, 1, 0, 0, 1, 1)], [(0, 0, 0, 0, 1, 1), (0, 2, 0, 0, 1, 1)]):  # box indices not 0, 1, ...
        assert _erase(_ebuf(b)) == E, b
    for mode in (-1, 3):
        assert _erase(_ebuf(ok, mode)) == E, mode
    too_many = [(0, k, 0, 0, 1, 1) for k in range(augment.ERASE_MAX_COUNT + 1)]
    assert _erase(_ebuf(too_many), N=2) == E
    assert _erase(_ebuf(ok), dtype=_lib.F64) == -2
    assert _erase(_ebuf(ok), N=0) == E
    assert _lib.load().cotb200_aug_erase(_lib.F32, 2, 3, 16, 20, FAKE, None, FAKE, None) == -5
    assert _lib.load().cotb200_aug_erase(_lib.F32, 2, 3, 16, 20, None, _ebuf(ok).ctypes.data, FAKE, None) == -5
    assert _erase(_ebuf([])) == 0                      # nothing to erase: nothing launched, nothing dereferenced


def test_random_erasing_arguments():
    with pytest.raises(ValueError):
        augment.RandomErasing(0.5, "noise")
    with pytest.raises(ValueError):
        augment.RandomErasing(0.5, max_count=augment.ERASE_MAX_COUNT + 1)
    assert augment.RandomErasing(0.5, "").mode == "const"
