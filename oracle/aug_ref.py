"""Numpy restatement of the reference's PIL image augmentation, byte-equal to Pillow.

The reference builds every training batch with PIL in DataLoader workers (datasets/transforms_factory.py:44-129):
RandomResizedCropAndInterpolation (datasets/transforms.py:58-145, i.e. torchvision F.resized_crop = PIL crop + resize),
RandomHorizontalFlip, RandAugment (datasets/rand_augment.py) and ToNumpy; validation is Resize(short side) + CenterCrop
(:132-166).  This module restates each step on uint8 HWC numpy arrays with Pillow's own arithmetic (integer fixed point
where Pillow uses it, float32 / float64 in Pillow's operation order where it does not; numpy never contracts to FMA), so
that the CUDA kernels of cotnet_b200/csrc/augment.cu can be checked on any number of random draws without Pillow.

Images are uint8 arrays [H, W, 3].  Op ids are the positions in OPS (the reference's _RAND_TRANSFORMS order).
"""
import math

import numpy as np

BILINEAR, BICUBIC = 0, 1
OPS = ("AutoContrast", "Equalize", "Invert", "Rotate", "Posterize", "Solarize", "SolarizeAdd", "Color", "Contrast",
       "Brightness", "Sharpness", "ShearX", "ShearY", "TranslateX", "TranslateY", "Cutout")
OP_ID = {n: i for i, n in enumerate(OPS)}
AFFINE_OPS = (OP_ID["Rotate"], OP_ID["ShearX"], OP_ID["ShearY"], OP_ID["TranslateX"], OP_ID["TranslateY"])
ENHANCE_OPS = (OP_ID["Color"], OP_ID["Contrast"], OP_ID["Brightness"], OP_ID["Sharpness"])
FILL = (124, 116, 104)
PRECISION_BITS = 22          # Pillow Resample.c: 32 - 8 - 2


# ---------------------------------------------------------------------------------------------------------------------
# resample (Pillow Resample.c): two passes, horizontal first, each with 22-bit fixed-point weights
# ---------------------------------------------------------------------------------------------------------------------
def _filter(x, filt):
    x = np.abs(x)
    if filt == BILINEAR:
        return np.where(x < 1.0, 1.0 - x, 0.0)
    a = -0.5
    return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1,
                    np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))


def support(filt):
    return 1.0 if filt == BILINEAR else 2.0


def coeffs(in_size, out_size, filt, idx):
    """precompute_coeffs + normalize_coeffs_8bpc for the output indices `idx` (box (0, in_size)).
    Returns (xmin [n], int64 weights [n, ksize]; zero past each row's xmax)."""
    idx = np.asarray(idx, dtype=np.int64)
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    sup = support(filt) * filterscale
    ksize = int(math.ceil(sup)) * 2 + 1
    center = (idx + 0.5) * scale
    ss = 1.0 / filterscale
    xmin = np.maximum(np.trunc(center - sup + 0.5), 0).astype(np.int64)
    xmax = np.minimum(np.trunc(center + sup + 0.5), in_size).astype(np.int64) - xmin
    w = np.zeros((len(idx), ksize))
    ww = np.zeros(len(idx))
    for x in range(ksize):                                 # sequential sum, as the C loop
        live = x < xmax
        wx = np.where(live, _filter(((x + xmin).astype(np.float64) - center + 0.5) * ss, filt), 0.0)
        w[:, x] = wx
        ww = ww + wx
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    one = float(1 << PRECISION_BITS)
    k = np.where(w < 0, np.trunc(-0.5 + w * one), np.trunc(0.5 + w * one)).astype(np.int64)
    return xmin, k


def _apply(src, xmin, k, axis):
    """One pass: out[..., i, ...] = clip8(2^21 + sum_x src[xmin_i + x] * k[i, x]) >> 22 along `axis` (0 rows, 1 cols)."""
    n, ksize = k.shape
    L = src.shape[axis]
    acc = np.full((n,) + (src.shape[1 - axis], 3), 1 << (PRECISION_BITS - 1), dtype=np.int64)
    s = np.moveaxis(src, axis, 0).astype(np.int64)
    for x in range(ksize):
        pos = np.minimum(xmin + x, L - 1)                  # weights past xmax are zero
        acc += s[pos] * k[:, x][:, None, None]
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize_window(img, rh, rw, filt, rows=None, cols=None):
    """PIL img.resize((rw, rh), filt), restricted to the output rows / columns listed (default: all).
    A pass whose size does not change is skipped, as Pillow does."""
    h, w = img.shape[:2]
    rows = np.arange(rh) if rows is None else np.asarray(rows)
    cols = np.arange(rw) if cols is None else np.asarray(cols)
    if rw != w:
        xmin, k = coeffs(w, rw, filt, cols)
        img = _apply(img, xmin, k, 1)
    else:
        img = img[:, cols]
    if rh != h:
        ymin, k = coeffs(h, rh, filt, rows)
        img = _apply(img, ymin, k, 0)
    else:
        img = img[rows]
    return np.ascontiguousarray(img)


def resized_crop(img, i, j, h, w, size, filt, flip=False):
    """F.resized_crop(img, i, j, h, w, (size, size), filt), then RandomHorizontalFlip when flip."""
    out = resize_window(img[i:i + h, j:j + w], size, size, filt)
    return np.ascontiguousarray(out[:, ::-1]) if flip else out


def eval_geometry(H, W, size=224, crop_pct=0.875):
    """Resize(floor(size / crop_pct)) + CenterCrop(size) (torchvision): (resized h, resized w, top, left)."""
    short = int(math.floor(size / crop_pct))
    if W <= H:
        rw, rh = short, int(short * H / W)
    else:
        rh, rw = short, int(short * W / H)
    return rh, rw, int(round((rh - size) / 2.0)), int(round((rw - size) / 2.0))


def eval_transform(img, size=224, crop_pct=0.875, filt=BICUBIC):
    H, W = img.shape[:2]
    rh, rw, top, left = eval_geometry(H, W, size, crop_pct)
    return resize_window(img, rh, rw, filt, np.arange(top, top + size), np.arange(left, left + size))


# ---------------------------------------------------------------------------------------------------------------------
# RandAugment ops
# ---------------------------------------------------------------------------------------------------------------------
def _lut(img, luts):
    return np.stack([np.clip(luts[c], 0, 255).astype(np.uint8)[img[..., c]] for c in range(3)], -1)


def _hist(img, c):
    return np.bincount(img[..., c].ravel(), minlength=256).astype(np.int64)


def autocontrast_lut(h):
    nz = np.nonzero(h)[0]
    lo, hi = (int(nz[0]), int(nz[-1])) if len(nz) else (255, 0)   # empty: the Python loops end at 255 / 0
    if hi <= lo:
        return np.arange(256)
    scale = 255.0 / (hi - lo)
    offset = -lo * scale
    return np.clip(np.trunc(np.arange(256) * scale + offset), 0, 255).astype(np.int64)


def equalize_lut(h):
    histo = h[h > 0]
    if len(histo) <= 1:
        return np.arange(256)
    step = (int(histo.sum()) - int(histo[-1])) // 255
    if not step:
        return np.arange(256)
    n = step // 2 + np.concatenate([[0], np.cumsum(h)[:-1]])
    return n // step


def to_l(img):
    """RGB -> L (Pillow Convert.c rgb2l)."""
    x = img.astype(np.int64)
    return ((x[..., 0] * 19595 + x[..., 1] * 38470 + x[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def blend(a, b, factor):
    """Image.blend(a, b, factor) (Pillow Blend.c): float32 arithmetic, truncation, clipping when extrapolating."""
    alpha = np.float32(factor)
    a32 = a.astype(np.int32)
    t = a32.astype(np.float32) + alpha * (b.astype(np.int32) - a32).astype(np.float32)
    return np.clip(np.trunc(t), 0, 255).astype(np.uint8)


def smooth(img):
    """ImageFilter.SMOOTH (3x3, weights 1 1 1 / 1 5 1 / 1 1 1, scale 13): border pixels are copied."""
    out = img.copy()
    if img.shape[0] < 3 or img.shape[1] < 3:
        return out
    k = np.float32(1.0) / np.float32(13.0)
    k5 = np.float32(5.0) / np.float32(13.0)
    f = img.astype(np.float32)
    ss = np.float32(0.0)
    for dy in (1, 0, -1):
        r = f[1 + dy:f.shape[0] - 1 + dy]
        kc = k5 if dy == 0 else k
        row = r[:, :-2] * k + r[:, 1:-1] * kc + r[:, 2:] * k
        ss = ss + row
    out[1:-1, 1:-1] = np.where(ss <= 0, 0, np.where(ss >= 255, 255, np.trunc(ss + np.float32(0.5)))).astype(np.uint8)
    return out


def rotate_matrix(degrees, w, h):
    """Image.rotate's inverse affine matrix (centre (w/2, h/2), no translation)."""
    angle = degrees % 360.0
    cx, cy = w / 2, h / 2
    angle = -math.radians(angle)
    m = [round(math.cos(angle), 15), round(math.sin(angle), 15), 0.0,
         round(-math.sin(angle), 15), round(math.cos(angle), 15), 0.0]
    a, b, c, d, e, f = m
    m[2], m[5] = a * -cx + b * -cy + c, d * -cx + e * -cy + f
    m[2] += cx
    m[5] += cy
    return m


def affine(img, m, filt, fill=FILL):
    """img.transform(img.size, AFFINE, m, filt, fillcolor=fill) (Pillow Geometry.c, generic transform)."""
    H, W = img.shape[:2]
    yo, xo = np.meshgrid(np.arange(H, dtype=np.float64) + 0.5, np.arange(W, dtype=np.float64) + 0.5, indexing="ij")
    xin = m[0] * xo + m[1] * yo + m[2]
    yin = m[3] * xo + m[4] * yo + m[5]
    ok = (xin >= 0.0) & (xin < W) & (yin >= 0.0) & (yin < H)
    xin = np.where(ok, xin, 0.5) - 0.5
    yin = np.where(ok, yin, 0.5) - 0.5
    x = np.floor(xin).astype(np.int64)
    y = np.floor(yin).astype(np.int64)
    dx = xin - x
    dy = yin - y
    src = img.astype(np.int64)
    out = np.empty_like(img)
    if filt == BICUBIC:
        x -= 1
        y -= 1
        xs = [np.clip(x + t, 0, W - 1) for t in range(4)]

        def cubic(v1, v2, v3, v4, d):
            p1 = v2
            p2 = -v1 + v3
            p3 = 2 * (v1 - v2) + v3 - v4
            p4 = -v1 + v2 - v3 + v4
            return p1 + d * (p2 + d * (p3 + d * p4))

        for c in range(3):
            vs = []
            for t in range(4):
                yy = y + t
                row = np.clip(yy, 0, H - 1)
                v = cubic(*[src[row, xs[q], c] for q in range(4)], dx)
                if t > 0:
                    v = np.where((yy >= 0) & (yy < H), v, vs[-1])
                vs.append(v)
            v = cubic(*vs, dy)
            out[..., c] = np.where(v <= 0.0, 0, np.where(v >= 255.0, 255, np.trunc(np.clip(v, 0, 255)))).astype(np.uint8)
    else:
        x0, x1 = np.clip(x, 0, W - 1), np.clip(x + 1, 0, W - 1)
        for c in range(3):
            r0 = np.clip(y, 0, H - 1)
            v1 = src[r0, x0, c] + (src[r0, x1, c] - src[r0, x0, c]) * dx
            y1 = y + 1
            r1 = np.clip(y1, 0, H - 1)
            v2 = np.where((y1 >= 0) & (y1 < H), src[r1, x0, c] + (src[r1, x1, c] - src[r1, x0, c]) * dx, v1)
            v = v1 + (v2 - v1) * dy
            out[..., c] = np.trunc(np.clip(v, 0, 255)).astype(np.uint8)
    for c in range(3):
        out[..., c] = np.where(ok, out[..., c], fill[c])
    return out


def cutout(img, x0, y0, x1, y1, fill=FILL):
    """ImageDraw.rectangle((x0, y0, x1, y1), fill): both ends inclusive, clipped to the image."""
    out = img.copy()
    out[max(y0, 0):y1 + 1, max(x0, 0):x1 + 1] = fill
    return out


def apply_op(img, op):
    """One drawn op: a dict with 'id' and the arguments the draw resolved (see cotnet_b200.augment.TrainAugment)."""
    i = op["id"]
    name = OPS[i]
    if name == "AutoContrast":
        return _lut(img, [autocontrast_lut(_hist(img, c)) for c in range(3)])
    if name == "Equalize":
        return _lut(img, [equalize_lut(_hist(img, c)) for c in range(3)])
    if name == "Invert":
        return 255 - img
    if name == "Posterize":
        bits = op["iarg"]
        if bits >= 8:
            return img.copy()
        return img & np.uint8(~(2 ** (8 - bits) - 1) & 255)
    if name == "Solarize":
        t = op["iarg"]
        return np.where(img < t, img, 255 - img).astype(np.uint8)
    if name == "SolarizeAdd":
        a = op["iarg"]
        return np.where(img < 128, np.minimum(255, img.astype(np.int64) + a), img).astype(np.uint8)
    if name == "Color":
        return blend(np.repeat(to_l(img)[..., None], 3, -1), img, op["factor"])
    if name == "Contrast":
        lv = to_l(img).astype(np.int64)
        mean = int(float(lv.sum()) / lv.size + 0.5)
        return blend(np.full_like(img, mean), img, op["factor"])
    if name == "Brightness":
        return blend(np.zeros_like(img), img, op["factor"])
    if name == "Sharpness":
        return blend(smooth(img), img, op["factor"])
    if i in AFFINE_OPS:
        return affine(img, op["matrix"], op["filter"])
    if name == "Cutout":
        return cutout(img, *op["box"])
    raise ValueError("unknown op id %r" % (i,))


def source_image(seed, h, w):
    """Smooth synthetic RGB content from a seed: gradients, a wave, a disc and a darkened bar (no noise, so that the fixture
    built on it compresses)."""
    r = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    a, b, c = r.uniform(0.2, 1.0, 3)
    img = np.stack([255 * a * xx / max(w - 1, 1), 255 * b * yy / max(h - 1, 1), 128 + 100 * c * np.sin((xx + yy) / 23.0)], -1)
    cy, cx, rad = r.uniform(0, h), r.uniform(0, w), r.uniform(0.1, 0.4) * min(h, w)
    img[(yy - cy) ** 2 + (xx - cx) ** 2 < rad ** 2] = r.uniform(0, 255, 3)
    y0 = r.randint(0, h)
    img[y0:y0 + max(h // 10, 1), :, :] *= 0.4
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def load_golden(path):
    """tests/golden/augment.npz as a dict, images decoded: every uint8 3-D array is stored as its differences along axis -2
    (mod 256, the first row against 0), which deflate packs several times smaller than the smooth images themselves."""
    g = np.load(path)
    return {k: np.cumsum(g[k], axis=-2, dtype=np.uint8) if g[k].dtype == np.uint8 and g[k].ndim == 3 else g[k] for k in g.files}


def encode_golden(a):
    """The inverse of load_golden's decoding for one array."""
    a = np.asarray(a)
    return np.diff(a, axis=-2, prepend=np.zeros_like(a[..., :1, :])) if a.dtype == np.uint8 and a.ndim == 3 else a


def fixture_op(case, S):
    """The op dict of a tests/golden/augment.npz op case (id, level argument, case index; Cutout's position drawn from
    np.random.seed(case index)) on an S x S image."""
    i, arg, idx = int(case[0]), float(case[1]), int(case[2])
    op = {"id": i}
    if i == 3:
        op.update(matrix=rotate_matrix(arg, S, S), filter=1)
    elif i in (11, 12):
        op.update(matrix=(1, arg, 0, 0, 1, 0) if i == 11 else (1, 0, 0, arg, 1, 0), filter=1)
    elif i in (13, 14):
        op.update(matrix=(1, 0, arg, 0, 1, 0) if i == 13 else (1, 0, 0, 0, 1, arg), filter=1)
    elif i in (4, 5, 6):
        op["iarg"] = int(arg)
    elif i in (7, 8, 9, 10):
        op["factor"] = arg
    elif i == 15:
        px = int(arg)
        r = np.random.RandomState(idx)
        x0, y0 = r.uniform(S), r.uniform(S)
        x0, y0 = int(max(0, x0 - px)), int(max(0, y0 - px))
        op["box"] = (x0, y0, min(S, x0 + 2 * px), min(S, y0 + 2 * px))
    return op


def train_sample(img, p, size=224):
    """The whole train transform of one image from its drawn parameters (cotnet_b200.augment.TrainAugment.draw),
    returned as CHW uint8 (ToNumpy)."""
    out = resized_crop(img, p["i"], p["j"], p["h"], p["w"], size, p["filter"], p["flip"])
    for op in p["ops"]:
        if op is not None:
            out = apply_op(out, op)
    return np.ascontiguousarray(out.transpose(2, 0, 1))
