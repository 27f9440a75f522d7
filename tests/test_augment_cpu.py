"""CPU checks of the GPU augmentation's host side and oracle: the draws equal the reference's (fixture), oracle/aug_ref.py
equals Pillow op by op and equals the fixture's PIL outputs, and the C entry points reject bad arguments before any launch."""
import os
import random

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, augment
from oracle import aug_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment.npz")


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _draw(tf, s, H, W):
    return tf.draw_one(H, W, random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


def test_draws_equal_reference(gold):
    tf = augment.TrainAugment()
    for s, (H, W) in enumerate(gold["draws_sizes"]):
        rnd, nrnd, tgen = random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s)
        p = tf.draw_one(int(H), int(W), rnd, nrnd, tgen)
        assert (p["i"], p["j"], p["h"], p["w"]) == tuple(gold["draws_crop"][s]), s
        assert int(p["flip"]) == gold["draws_flip"][s], s
        applied = [o for o in p["ops"] if o is not None]
        ids = [o["id"] for o in applied] + [-1] * (2 - len(applied))
        assert ids == list(gold["draws_ids"][s]), s
        for k, o in enumerate(applied):
            assert float(o["arg"]) == gold["draws_args"][s][k], (s, k)
        # every generator consumed exactly what the reference consumed
        assert (rnd.random(), nrnd.random_sample(), float(torch.rand(1, generator=tgen))) == tuple(gold["draws_next"][s]), s


def test_draws_cover_the_fallback_and_every_op(gold):
    tf = augment.TrainAugment()
    ids = set()
    fallback = 0
    for s, (H, W) in enumerate(gold["draws_sizes"]):
        p = _draw(tf, s, int(H), int(W))
        ids |= {o["id"] for o in p["ops"] if o is not None}
        fallback += (p["h"], p["w"]) in ((H, int(round(H * 4 / 3))), (int(round(W / (4 / 3))), W))
    assert fallback > 0
    assert len(ids) >= 14


def test_pack_layout():
    tf = augment.TrainAugment()
    sizes = [(300, 200), (50, 70)]
    rec = tf.pack(sizes, tf.draw(sizes, random.Random(3), np.random.RandomState(3), torch.Generator().manual_seed(3)))
    assert rec.dtype.itemsize == 224
    assert list(rec["offset"]) == [0, 300 * 200 * 3]
    assert list(rec["tmp_offset"]) == [0, 3 * 224 * rec["ch"][0]]


# ---------------------------------------------------------------- aug_ref against the fixture (the reference's PIL outputs)
def test_aug_ref_train_equals_fixture(gold):
    tf = augment.TrainAugment()
    k = 0
    while "train_%d" % k in gold:
        H, W, seed, iseed = (int(v) for v in gold["train_%d_size" % k])
        p = _draw(tf, seed, H, W)
        got = aug_ref.train_sample(aug_ref.source_image(iseed, H, W), p)
        np.testing.assert_array_equal(got, gold["train_%d" % k], err_msg="train image %d" % k)
        k += 1
    assert k >= 4


def test_aug_ref_ops_equal_fixture(gold):
    src = gold["op_src"]
    cases = gold["op_cases"]
    assert len(cases) >= 16 * 3
    for case in cases:
        got = aug_ref.apply_op(src, aug_ref.fixture_op(case, src.shape[0]))
        np.testing.assert_array_equal(got, gold["op_%d" % int(case[2])], err_msg="op case %s" % (case,))


def test_aug_ref_eval_equals_fixture(gold):
    k = 0
    while "eval_%d" % k in gold:
        H, W, iseed = (int(v) for v in gold["eval_%d_size" % k])
        got = aug_ref.eval_transform(aug_ref.source_image(iseed, H, W)).transpose(2, 0, 1)
        np.testing.assert_array_equal(got, gold["eval_%d" % k])
        k += 1
    assert k >= 2


def test_eval_geometry_matches_oracle():
    for H, W in ((500, 375), (375, 500), (256, 256), (1, 900), (900, 3)):
        assert augment.eval_geometry(H, W) == aug_ref.eval_geometry(H, W)
    for deg in (45.0, -45.0, 13.25, 0.0):
        assert augment.rotate_matrix(deg, 224, 224) == aug_ref.rotate_matrix(deg, 224, 224)


# ---------------------------------------------------------------- aug_ref against Pillow on random images
def _img(r, h, w):
    yy, xx = np.mgrid[0:h, 0:w]
    a = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 200 // max(h - 1, 1)) + 20, ((xx + yy) * 3) % 256], -1)
    return np.clip(a + r.randint(-25, 26, size=a.shape), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("seed", range(4))
def test_aug_ref_equals_pil(seed):
    Image = pytest.importorskip("PIL.Image")
    from PIL import ImageDraw, ImageEnhance, ImageOps
    r = np.random.RandomState(seed)
    h, w = (int(v) for v in r.randint(3, 300, 2))
    a = _img(r, h, w)
    p = Image.fromarray(a)
    eq = np.testing.assert_array_equal
    for f, pf in ((0, Image.BILINEAR), (1, Image.BICUBIC)):
        for rh, rw in ((int(r.randint(1, 400)), int(r.randint(1, 400))), (h, int(r.randint(1, 40))), (1, 1)):
            eq(aug_ref.resize_window(a, rh, rw, f), np.asarray(p.resize((rw, rh), pf)))
    eq(aug_ref.apply_op(a, {"id": 0}), np.asarray(ImageOps.autocontrast(p)))
    eq(aug_ref.apply_op(a, {"id": 1}), np.asarray(ImageOps.equalize(p)))
    eq(aug_ref.apply_op(a, {"id": 2}), np.asarray(ImageOps.invert(p)))
    for b in (0, 1, 4, 6):
        eq(aug_ref.apply_op(a, {"id": 4, "iarg": b}), np.asarray(ImageOps.posterize(p, b)))
    for t in (0, 100, 256, 384):
        eq(aug_ref.apply_op(a, {"id": 5, "iarg": t}), np.asarray(ImageOps.solarize(p, t)))
    for add in (0, 55, 110, 165):
        lut = [min(255, i + add) if i < 128 else i for i in range(256)]
        eq(aug_ref.apply_op(a, {"id": 6, "iarg": add}), np.asarray(p.point(lut * 3)))
    for f in (0.1, 0.55, 1.0, 1.9, 2.8, 2.95):
        eq(aug_ref.apply_op(a, {"id": 7, "factor": f}), np.asarray(ImageEnhance.Color(p).enhance(f)))
        eq(aug_ref.apply_op(a, {"id": 8, "factor": f}), np.asarray(ImageEnhance.Contrast(p).enhance(f)))
        eq(aug_ref.apply_op(a, {"id": 9, "factor": f}), np.asarray(ImageEnhance.Brightness(p).enhance(f)))
        eq(aug_ref.apply_op(a, {"id": 10, "factor": f}), np.asarray(ImageEnhance.Sharpness(p).enhance(f)))
    fill = aug_ref.FILL
    for f, pf in ((0, Image.BILINEAR), (1, Image.BICUBIC)):
        for deg in (45.0, -45.0, 13.7, -0.3):
            eq(aug_ref.affine(a, aug_ref.rotate_matrix(deg, w, h), f), np.asarray(p.rotate(deg, resample=pf, fillcolor=fill)))
        for m in ((1, 0.45, 0, 0, 1, 0), (1, 0, 0, -0.3, 1, 0), (1, 0, -150.0, 0, 1, 0), (1, 0, 0, 0, 1, 37.5)):
            eq(aug_ref.affine(a, m, f), np.asarray(p.transform(p.size, Image.AFFINE, m, resample=pf, fillcolor=fill)))
    for box in ((0, 0, 0, 0), (w - 5, h - 5, w, h), (3, 2, 3 + 80, 2 + 80)):
        q = p.copy()
        ImageDraw.Draw(q).rectangle(box, fill)
        eq(aug_ref.cutout(a, *box), np.asarray(q))


# ---------------------------------------------------------------- C-ABI argument errors (no kernel is launched)
def _rec(**kw):
    r = np.zeros(1, augment.SAMPLE_DTYPE)
    base = dict(offset=0, h=10, w=10, ci=0, cj=0, ch=10, cw=10, rh=8, rw=8, oi=0, oj=0, filter=1, flip=0, tmp_offset=0)
    base.update(kw)
    for k, v in base.items():
        r[0][k] = v
    r["ops"]["op"] = -1
    return r


def _resize(rec, src_bytes=300, tmp_bytes=3 * 8 * 10, S=8, N=1):
    lib = _lib.load()
    fake = 1 << 20                                           # never dereferenced: validation fails first
    return lib.cotb200_aug_resize_crop(N, S, fake, src_bytes, rec.ctypes.data, fake, fake, tmp_bytes, fake, None)


def test_capi_resize_rejects_bad_samples():
    E = -1
    assert _resize(_rec(h=0)) == E
    assert _resize(_rec(w=0)) == E
    assert _resize(_rec(offset=1)) == E                      # 10x10x3 bytes at offset 1 run past 300 bytes
    assert _resize(_rec(offset=-3)) == E
    assert _resize(_rec(ci=1)) == E                          # crop past the image
    assert _resize(_rec(cw=11)) == E
    assert _resize(_rec(oi=1)) == E                          # window past the resize
    assert _resize(_rec(rw=7)) == E
    assert _resize(_rec(filter=2)) == E
    assert _resize(_rec(flip=3)) == E
    assert _resize(_rec(), tmp_bytes=3 * 8 * 10 - 1) == E    # scratch too small
    assert _resize(_rec(), S=0) == E
    assert _resize(_rec(), N=0) == E
    lib = _lib.load()
    assert lib.cotb200_aug_resize_crop(1, 8, None, 300, _rec().ctypes.data, 1, 1, 240, 1, None) == -5
    assert lib.cotb200_aug_resize_crop(1, 8, 1, 300, None, 1, 1, 240, 1, None) == -5


def test_capi_resize_rejects_huge_downscale():
    r = _rec(h=1, w=100000, ch=1, cw=100000, rh=8, rw=8)
    assert _resize(r, src_bytes=300000) == -7


def test_capi_randaug_rejects_bad_ops():
    lib = _lib.load()
    fake = 1 << 20
    for op, extra in ((16, {}), (-2, {}), (3, {"filter": 2}), (4, {"v": [-1, 0, 0, 0]}), (7, {"factor": float("nan")}),
                      (11, {"m": [float("inf"), 0, 0, 0, 1, 0]})):
        r = _rec()
        r["ops"]["op"][0, 1] = op
        for k, v in extra.items():
            r["ops"][k][0, 1] = v
        assert lib.cotb200_aug_randaug(1, 8, r.ctypes.data, fake, fake, None) == -1, (op, extra)
    assert lib.cotb200_aug_randaug(1, 257, _rec().ctypes.data, fake, fake, None) == -7
    assert lib.cotb200_aug_randaug(1, 8, None, fake, fake, None) == -5
