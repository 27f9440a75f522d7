"""Numpy restatement of the reference's vertical flip, ColorJitter (torchvision on PIL images) and random-erasing masks, byte-equal
to Pillow.  TEST INFRASTRUCTURE: it builds on oracle/aug_ref.py (resize-crop, the enhance blends) and is pinned to Pillow and
to tests/golden/augment_jitter.npz by tests/test_augment_jitter_cpu.py, so that the kernels can be checked on any draws.

Images are uint8 arrays [H, W, 3].
"""
import numpy as np

from oracle.aug_ref import OP_ID, apply_op, resized_crop


def vflip(img):
    """RandomVerticalFlip of the resized image: a row mirror."""
    return np.ascontiguousarray(img[::-1])


def rgb_to_hsv(img):
    """img.convert('HSV') (Pillow Convert.c rgb2hsv): float32 where Pillow declares float, float64 where its expressions
    promote (2.0 + rc - bc, h / 6.0 + 1.0, h * 255.0), truncating casts."""
    f32, f64 = np.float32, np.float64
    x = img.astype(np.int32)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    maxc = np.maximum(r, np.maximum(g, b))
    minc = np.minimum(r, np.minimum(g, b))
    grey = maxc == minc
    cr = np.where(grey, 1, maxc - minc).astype(f32)
    s = cr / np.where(maxc == 0, 1, maxc).astype(f32)
    rc, gc, bc = ((maxc - c).astype(f32) / cr for c in (r, g, b))
    h = np.where(r == maxc, bc - gc,
                 np.where(g == maxc, ((2.0 + rc.astype(f64)) - bc.astype(f64)).astype(f32),
                          ((4.0 + gc.astype(f64)) - rc.astype(f64)).astype(f32)))
    h = np.fmod(h.astype(f64) / 6.0 + 1.0, 1.0).astype(f32)
    uh = np.where(grey, 0, np.clip(np.trunc(h.astype(f64) * 255.0), 0, 255)).astype(np.uint8)
    us = np.where(grey, 0, np.clip(np.trunc(s.astype(f64) * 255.0), 0, 255)).astype(np.uint8)
    return np.stack([uh, us, maxc.astype(np.uint8)], -1)


def _c_round(x):
    return np.where(x >= 0, np.floor(x + 0.5), np.ceil(x - 0.5))     # C round(): halves away from zero


def hsv_to_rgb(hsv):
    """Image.merge('HSV', ...).convert('RGB') (Pillow Convert.c hsv2rgb): i = floor(h * 6.0 / 255.0), f and fs rounded to
    float32, p / q / t in float64 with C round(); s = 0 gives (v, v, v)."""
    f32, f64 = np.float32, np.float64
    h, s, v = (hsv[..., k].astype(np.int32) for k in range(3))
    hh = h.astype(f64) * 6.0 / 255.0
    i = np.floor(hh).astype(np.int32)
    f = (hh - i.astype(f32).astype(f64)).astype(f32)
    fs = (s.astype(f64) / 255.0).astype(f32)
    vf = v.astype(f64)
    p = _c_round(vf * (1.0 - fs.astype(f64)))
    q = _c_round(vf * (1.0 - (fs * f).astype(f64)))
    t = _c_round(vf * (1.0 - fs.astype(f64) * (1.0 - f.astype(f64))))
    up, uq, ut = (np.clip(a, 0, 255).astype(np.uint8) for a in (p, q, t))
    vv = v.astype(np.uint8)
    sel = ((vv, ut, up), (uq, vv, up), (up, vv, ut), (up, uq, vv), (ut, up, vv), (vv, up, uq))
    k = i % 6
    out = np.empty(hsv.shape, np.uint8)
    for c in range(3):
        out[..., c] = np.where(s == 0, vv, np.select([k == j for j in range(6)], [sel[j][c] for j in range(6)]))
    return out


def hue_shift(hue_factor):
    """adjust_hue's shift of the H channel: np.int32(hue_factor * 255).astype(np.uint8) (truncation, then mod 256)."""
    return int(np.int32(hue_factor * 255).astype(np.uint8))


def adjust_hue(img, hue_factor):
    """torchvision F.adjust_hue on a PIL RGB image: RGB -> HSV, H += hue_shift (uint8 wrap-around), HSV -> RGB."""
    hsv = rgb_to_hsv(img)
    hsv[..., 0] += np.uint8(hue_shift(hue_factor))
    return hsv_to_rgb(hsv)


#: ColorJitter op ids (torchvision's fn_idx) -> the RandAugment enhance op that computes the same blend
JITTER_ENHANCE = {0: OP_ID["Brightness"], 1: OP_ID["Contrast"], 2: OP_ID["Color"]}


def color_jitter(img, order, factors):
    """ColorJitter.forward on a PIL RGB image given its draws: the ops of `order` (0 brightness, 1 contrast, 2 saturation,
    3 hue) with factors[op]."""
    for op in order:
        img = adjust_hue(img, factors[3]) if op == 3 else apply_op(img, {"id": JITTER_ENHANCE[op], "factor": factors[op]})
    return img


def train_sample_jitter(img, p, size=224):
    """train_sample with a vertical flip (p['vflip']) after the horizontal one and, when p has 'jitter' (order, factors),
    ColorJitter; then p's RandAugment ops.  CHW uint8."""
    out = resized_crop(img, p["i"], p["j"], p["h"], p["w"], size, p["filter"], p["flip"])
    if p.get("vflip"):
        out = vflip(out)
    if p.get("jitter"):
        out = color_jitter(out, p["jitter"]["order"], p["jitter"]["factors"])
    for op in p["ops"]:
        if op is not None:
            out = apply_op(out, op)
    return np.ascontiguousarray(out.transpose(2, 0, 1))


def erase_owner(B, H, W, boxes):
    """int [B, H, W]: the index (within its image) of the box that last wrote each pixel, -1 where none did.  boxes: B lists
    of (top, left, h, w) in draw order, as RandomErasing writes them one after the other."""
    own = np.full((B, H, W), -1, np.int64)
    for n, bs in enumerate(boxes):
        for k, (t, l, h, w) in enumerate([b for b in bs if b[2] > 0 and b[3] > 0]):
            own[n, t:t + h, l:l + w] = k
    return own


def erase_const(x, boxes):
    """RandomErasing in mode 'const' of the normalised batch x [B, C, H, W]: zeros in every box."""
    out = np.array(x, copy=True)
    own = erase_owner(out.shape[0], out.shape[2], out.shape[3], boxes)
    out[np.broadcast_to((own >= 0)[:, None], out.shape)] = 0
    return out
