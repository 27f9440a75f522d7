"""The reference's image augmentation on the GPU, byte-equal to its PIL pipeline given the same random draws.

DataLoader workers still decode (JPEG -> RGB uint8 HWC, the reference dataset's ``.convert('RGB')``).  From there:

* ``TrainAugment``: RandomResizedCrop(scale, ratio, interpolation) + RandomHorizontalFlip(0.5) + RandAugment
  (``rand-m15-mstd0.5-n2`` and every config rand_augment_transform parses: any magnitude, std and number of layers, and the
  weighted op choice ``w0``; datasets/transforms_factory.py:44-129).  Two ops per sample go in one RandAugment launch, so
  ``n`` layers take ceil(n / 2) launches in sequence on the same images.  ``draw`` consumes a
  ``random.Random``, an ``np.random.RandomState`` and a torch CPU ``Generator`` in the reference's call order, so a seeded draw
  equals what the reference's transforms draw from the global generators; ``collate`` does that inside DataLoader workers
  and packs the batch into one ragged buffer; ``__call__`` runs the kernels (cotb200_aug_resize_crop, cotb200_aug_randaug)
  and returns the uint8 NCHW batch that fast_collate builds, ready for ``normalize_u8(mix=MixupCutmix.draw(...))``.
  Above 256 x 256 (the 288 and 320 data configs) RandAugment and ColorJitter run on their thread-block-cluster kernels
  (cotb200_aug_randaug_cluster, cotb200_aug_color_jitter_cluster), up to 512 x 512.
  With ``vflip`` a RandomVerticalFlip follows the horizontal one; without ``auto_augment``, ``color_jitter`` gives torchvision's
  ColorJitter (:100-109), both in one more kernel (cotb200_aug_color_jitter) between resize-crop and RandAugment.
  With ``num_splits`` S >= 2 it is the reference's AugMixDataset over the separated transform (datasets/dataset.py:181-215,
  transforms_factory.py:44-129): a clean view (crop, flips) and S - 1 views that each add their own RandAugment or ColorJitter
  draw to the same crop, in fast_collate's split-major order, for the JSD loss (trainer.jsd_cross_entropy).
* ``EvalTransform``: Resize(floor(size / crop_pct)) + CenterCrop(size) (:132-166) on the same resize kernel; with
  crop_pct=1.0 also the train transform of augmentation.no_aug (transforms_noaug_train, :17-41).
* ``RandomErasing``: the reference's random erasing of the normalised batch (datasets/random_erasing.py, applied by
  PrefetchLoader, datasets/loader.py:72-91), boxes drawn on the host in its order and erased by one kernel (cotb200_aug_erase).

oracle/aug_ref.py restates every step in numpy; tests/golden/augment.npz holds the reference's own outputs.
"""
import ctypes
import math
import numbers
import random
import re
from collections import namedtuple

import numpy as np
import torch

from . import _lib

BILINEAR, BICUBIC = 0, 1
#: op ids: the positions in the reference's _RAND_TRANSFORMS (the `op` of struct cotb200_aug_op)
OPS = ("AutoContrast", "Equalize", "Invert", "Rotate", "Posterize", "Solarize", "SolarizeAdd", "Color", "Contrast",
       "Brightness", "Sharpness", "ShearX", "ShearY", "TranslateX", "TranslateY", "Cutout")
AFFINE_OPS = (3, 11, 12, 13, 14)
MAX_LEVEL = 10.          # rand_augment.py _MAX_LEVEL (level -> argument scale)
MAG_CLIP = 15            # AugmentOp.MAX_LEVEL (magnitude clip)
ONE_CTA_MAX_S = 256      # the largest output size of cotb200_aug_randaug / cotb200_aug_color_jitter (one CTA per image)
CLUSTER_MAX_S = 512      # COTB200_AUG_CLUSTER_MAX_S, the *_cluster entry points' (one thread-block cluster per image)

_OP_DTYPE = np.dtype([("op", "<i4"), ("filter", "<i4"), ("v", "<i4", (4,)), ("factor", "<f4"), ("pad_", "<i4"),
                      ("m", "<f8", (6,))], align=True)
#: struct cotb200_aug_sample (include/cotb200.h)
SAMPLE_DTYPE = np.dtype([("offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("ci", "<i4"), ("cj", "<i4"), ("ch", "<i4"),
                         ("cw", "<i4"), ("rh", "<i4"), ("rw", "<i4"), ("oi", "<i4"), ("oj", "<i4"), ("filter", "<i4"),
                         ("flip", "<i4"), ("tmp_offset", "<i8"), ("ops", _OP_DTYPE, (2,))], align=True)
assert _OP_DTYPE.itemsize == 80 and SAMPLE_DTYPE.itemsize == 224

_INTERP = {"bilinear": BILINEAR, "bicubic": BICUBIC}

#: struct cotb200_aug_jitter (include/cotb200.h): vertical flip, ColorJitter op order (0 brightness, 1 contrast, 2 saturation,
#: 3 hue, -1 none), the three blend factors and the hue factor
JITTER_DTYPE = np.dtype([("vflip", "<i4"), ("order", "<i4", (4,)), ("factor", "<f4", (3,)), ("hue", "<f8")], align=True)
#: struct cotb200_erase, then struct cotb200_erase_box (include/cotb200.h)
ERASE_DTYPE = np.dtype([("mode", "<i4"), ("n_boxes", "<i4"), ("seed", "<u8")])
ERASE_BOX_DTYPE = np.dtype([("n", "<i4"), ("k", "<i4"), ("top", "<i4"), ("left", "<i4"), ("h", "<i4"), ("w", "<i4")])
ERASE_MAX_COUNT = 32     # COTB200_ERASE_MAX_COUNT
assert JITTER_DTYPE.itemsize == 40 and ERASE_DTYPE.itemsize == 16 and ERASE_BOX_DTYPE.itemsize == 24

#: what a worker's collate hands to the main process: concatenated HWC images, the drawn parameter structs, the labels, and
#: the JITTER_DTYPE structs when the transform has a vertical flip or ColorJitter (None otherwise)
AugBatch = namedtuple("AugBatch", "data params labels jitter", defaults=(None,))


#: rand_augment.py _RAND_CHOICE_WEIGHTS_0, in OPS order: the op-choice weights of the 'w0' section
_CHOICE_WEIGHTS_0 = (0.025, .005, 0, 0.2, 0, .005, .005, .025, .005, .005, 0.025, 0.2, 0.2, 0.1, 0.1, 0.1)


def choice_weights(weight_idx):
    """_select_rand_weights(weight_idx) (rand_augment.py:312-318): the weights over OPS divided by their np.sum, float64, bit for
    bit (numpy's choice compares their cumulative sum against its uniforms, so any other rounding can pick another op)."""
    if weight_idx != 0:
        raise ValueError("RandAugment weight index must be 0 (the reference's only weight set), got %d" % weight_idx)
    probs = list(_CHOICE_WEIGHTS_0)
    return np.asarray(probs, np.float64) / np.sum(probs)


def _parse_rand(config_str):
    """rand_augment_transform's config string -> (magnitude, num_layers, magnitude_std, choice weights or None)."""
    parts = config_str.split("-")
    if parts[0] != "rand":
        raise ValueError("only RandAugment ('rand-...') is supported, got %r" % config_str)
    mag, n, mstd, weights = 10, 2, 0., None
    for c in parts[1:]:
        cs = re.split(r"(\d.*)", c)
        if len(cs) < 2:
            continue
        key, val = cs[:2]
        if key == "mstd":
            mstd = float(val)
        elif key == "m":
            mag = int(val)
        elif key == "n":
            n = int(val)
        elif key == "w":
            weights = choice_weights(int(val))
        elif key == "inc":
            pass
        else:
            raise ValueError("RandAugment section %r is not supported" % c)
    if n < 0:
        raise ValueError("RandAugment layer count must be >= 0, got %d" % n)
    # without replacement, numpy's choice needs n ops of non-zero weight; the reference finds out on its first image
    if weights is not None and n > np.count_nonzero(weights):
        raise ValueError("RandAugment with weights picks %d distinct ops, but only %d have a non-zero weight"
                         % (n, np.count_nonzero(weights)))
    return mag, n, mstd, weights


def _check_input(value, name, center=1., bound=(0., float("inf")), clip_first_on_zero=True):
    """torchvision ColorJitter._check_input: a number v -> [center - v, center + v] (the lower end clipped at 0 for the blend
    factors), a pair -> itself; None when the range is the identity."""
    if isinstance(value, numbers.Number):
        if value < 0:
            raise ValueError("color_jitter: %s %r must be non-negative" % (name, value))
        value = [center - float(value), center + float(value)]
        if clip_first_on_zero:
            value[0] = max(value[0], 0.0)
    elif isinstance(value, (tuple, list)) and len(value) == 2:
        value = [float(value[0]), float(value[1])]
    else:
        raise TypeError("color_jitter: %s must be a number or a pair, got %r" % (name, value))
    if not bound[0] <= value[0] <= value[1] <= bound[1]:
        raise ValueError("color_jitter: %s range %s outside %s" % (name, value, bound))
    return None if value[0] == value[1] == center else tuple(value)


def jitter_ranges(color_jitter):
    """transforms_factory.py:100-109 + ColorJitter(*color_jitter): a scalar c -> brightness, contrast, saturation c and no
    hue; a 3- or 4-sequence -> per channel.  Returns the four (lo, hi) factor ranges, None for a channel that is off."""
    if isinstance(color_jitter, (list, tuple)):
        if len(color_jitter) not in (3, 4):
            raise ValueError("color_jitter: expected a scalar or 3 or 4 values, got %r" % (color_jitter,))
    else:
        color_jitter = (float(color_jitter),) * 3
    b, c, s = (_check_input(v, n) for v, n in zip(color_jitter[:3], ("brightness", "contrast", "saturation")))
    h = _check_input(color_jitter[3] if len(color_jitter) == 4 else 0, "hue", center=0., bound=(-0.5, 0.5),
                     clip_first_on_zero=False)
    return [b, c, s, h]


def rotate_matrix(degrees, w, h):
    """The inverse affine matrix Image.rotate(degrees) builds for a w x h image (centre (w/2, h/2), no translation)."""
    cx, cy = w / 2, h / 2
    angle = -math.radians(degrees % 360.0)
    m = [round(math.cos(angle), 15), round(math.sin(angle), 15), 0.0,
         round(-math.sin(angle), 15), round(math.cos(angle), 15), 0.0]
    a, b, c, d, e, f = m
    m[2], m[5] = a * -cx + b * -cy + c, d * -cx + e * -cy + f
    m[2] += cx
    m[5] += cy
    return m


def eval_geometry(H, W, size=224, crop_pct=0.875):
    """torchvision Resize(floor(size / crop_pct)) + CenterCrop(size) of an H x W image: (resized h, resized w, top, left)."""
    short = int(math.floor(size / crop_pct))
    if W <= H:
        rw, rh = short, int(short * H / W)
    else:
        rh, rw = short, int(short * W / H)
    return rh, rw, int(round((rh - size) / 2.0)), int(round((rw - size) / 2.0))


def rrc_params(H, W, scale, ratio, rnd):
    """RandomResizedCropAndInterpolation.get_params (datasets/transforms.py:89-130) -> (i, j, h, w)."""
    area = W * H
    for _ in range(10):
        target_area = rnd.uniform(*scale) * area
        log_ratio = (math.log(ratio[0]), math.log(ratio[1]))
        aspect_ratio = math.exp(rnd.uniform(*log_ratio))
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if w <= W and h <= H:
            i = rnd.randint(0, H - h)
            j = rnd.randint(0, W - w)
            return i, j, h, w
    in_ratio = W / H
    if in_ratio < min(ratio):
        w = W
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = H
        w = int(round(h * max(ratio)))
    else:
        w = W
        h = H
    return (H - h) // 2, (W - w) // 2, h, w


class TrainAugment:
    """The reference's training transform (transforms_imagenet_train with use_prefetcher=True) on the GPU."""

    def __init__(self, size=224, scale=(0.08, 1.0), ratio=(3. / 4., 4. / 3.), interpolation="bicubic", hflip=0.5,
                 auto_augment="rand-m15-mstd0.5-n2", translate_const=100, cutout_const=40, vflip=0., color_jitter=None,
                 num_splits=0):
        """num_splits: augmentation.aug_splits of the reference (0 and 1: one view per image).
        auto_augment: a rand_augment_transform config string ('rand-m9-n3-mstd0.5', 'rand-mstd1-w0', ...) or None.  One
        difference: 'w0' with n above the 14 ops of non-zero weight raises ValueError here, where the reference's numpy
        choice raises on the first image."""
        if int(num_splits) != num_splits or num_splits < 0:
            raise ValueError("num_splits must be 0 or a positive integer, got %r" % (num_splits,))
        self.num_splits = int(num_splits) if num_splits >= 2 else 0
        if interpolation != "random" and interpolation not in _INTERP:
            raise ValueError("interpolation must be 'bilinear', 'bicubic' or 'random', got %r" % (interpolation,))
        self.size = int(size)
        self.scale, self.ratio = tuple(scale), tuple(ratio)
        self.interpolation = interpolation
        self.hflip = hflip
        self.vflip = float(vflip)
        parsed = _parse_rand(auto_augment) if auto_augment else (0, 0, 0., None)
        self.magnitude, self.num_layers, self.mstd, self.choice_weights = parsed
        self.translate_const, self.cutout_const = translate_const, cutout_const
        # ColorJitter is the reference's colour transform only when RandAugment is off (transforms_factory.py:79-109)
        self.jitter = None if auto_augment or color_jitter is None else jitter_ranges(color_jitter)

    def _filter(self, rnd):
        if self.interpolation == "random":
            return rnd.choice((BILINEAR, BICUBIC))
        return _INTERP[self.interpolation]

    def _op(self, i, rnd, nrnd):
        """AugmentOp.__call__ of op i (rand_augment.py:287-296): the draws and the resolved argument, or None (not applied)."""
        if rnd.random() > rnd.uniform(0.2, 0.8):
            return None
        mag = self.magnitude
        if self.mstd > 0:
            mag = rnd.gauss(mag, self.mstd)
        mag = min(MAG_CLIP, max(0, mag))
        name, S = OPS[i], self.size
        op = {"id": i, "arg": 0.0}

        def negate(v):
            return -v if rnd.random() > 0.5 else v

        if name == "Rotate":
            deg = negate((mag / MAX_LEVEL) * 30.)
            op.update(arg=deg, matrix=rotate_matrix(deg, S, S), filter=self._filter(rnd))
        elif name in ("ShearX", "ShearY"):
            f = negate((mag / MAX_LEVEL) * 0.3)
            op.update(arg=f, matrix=(1, f, 0, 0, 1, 0) if name == "ShearX" else (1, 0, 0, f, 1, 0), filter=self._filter(rnd))
        elif name in ("TranslateX", "TranslateY"):
            t = negate((mag / MAX_LEVEL) * float(self.translate_const))
            op.update(arg=t, matrix=(1, 0, t, 0, 1, 0) if name == "TranslateX" else (1, 0, 0, 0, 1, t), filter=self._filter(rnd))
        elif name == "Posterize":
            op["arg"] = op["iarg"] = int((mag / MAX_LEVEL) * 4)
        elif name == "Solarize":
            op["arg"] = op["iarg"] = int((mag / MAX_LEVEL) * 256)
        elif name == "SolarizeAdd":
            op["arg"] = op["iarg"] = int((mag / MAX_LEVEL) * 110)
        elif name in ("Color", "Contrast", "Brightness", "Sharpness"):
            op["arg"] = op["factor"] = (mag / MAX_LEVEL) * 1.8 + 0.1
        elif name == "Cutout":
            op["arg"] = px = int((mag / MAX_LEVEL) * self.cutout_const)
            x0 = nrnd.uniform(S)            # numpy reads uniform(w) as low = w, high = 1.0; kept as the reference does
            y0 = nrnd.uniform(S)
            x0 = int(max(0, x0 - px))
            y0 = int(max(0, y0 - px))
            op["box"] = (x0, y0, min(S, x0 + 2 * px), min(S, y0 + 2 * px))
        return op

    def _secondary(self, rnd, nrnd, tgen):
        """The colour part's draws: RandAugment's ops, or ColorJitter's."""
        p = dict(ops=[])
        if self.num_layers:                             # RandAugment.__call__: without replacement when weighted
            w = self.choice_weights
            for k in nrnd.choice(len(OPS), self.num_layers, replace=w is None, p=w):
                p["ops"].append(self._op(int(k), rnd, nrnd))
        elif self.jitter is not None:                   # ColorJitter.get_params + forward (torchvision)
            perm = torch.randperm(4, generator=tgen).tolist()
            f = [None if r is None else float(torch.empty(1).uniform_(r[0], r[1], generator=tgen)) for r in self.jitter]
            p["jitter"] = dict(order=[k for k in perm if f[k] is not None], factors=f)
        return p

    def draw_one(self, H, W, rnd, nrnd, tgen):
        """The draws of one H x W image as a dict (the form oracle/aug_ref.train_sample takes).  With num_splits S >= 2 the dict
        holds the clean view's draws (no ops) and, under "views", the S - 1 augmented views' colour draws, drawn after the
        clean view's as AugMixDataset.__getitem__ runs them."""
        i, j, h, w = rrc_params(H, W, self.scale, self.ratio, rnd)
        p = dict(i=i, j=j, h=h, w=w, filter=self._filter(rnd), flip=False)
        if self.hflip > 0:
            p["flip"] = bool(torch.rand(1, generator=tgen) < self.hflip)
        if self.vflip > 0:
            p["vflip"] = bool(torch.rand(1, generator=tgen) < self.vflip)
        if self.num_splits:
            p["ops"] = []
            p["views"] = [self._secondary(rnd, nrnd, tgen) for _ in range(self.num_splits - 1)]
        else:
            p.update(self._secondary(rnd, nrnd, tgen))
        return p

    def draw(self, sizes, py_random, np_random, torch_gen):
        """Per-sample parameters of images of `sizes` [(H, W), ...], drawn image by image in the reference's order:
        crop, filter (interpolation 'random' only), flip, vertical flip (vflip > 0 only), the op choice (num_layers ops, with
        replacement, or without it by the choice weights of a 'w0' config), then per op apply / magnitude / sign (/ filter) and
        Cutout's two positions; or, with ColorJitter, randperm(4) and one uniform per enabled factor in brightness, contrast,
        saturation, hue order.  Returns the list of dicts; ``pack`` and ``pack_jitter`` turn it into the device structs;
        ``pack_views`` the augmented views' ones when num_splits >= 2, ``pack_pass`` those of ops 2k and 2k + 1 when
        num_layers > 2."""
        return [self.draw_one(int(H), int(W), py_random, np_random, torch_gen) for H, W in sizes]

    def pack(self, sizes, draws):
        """numpy SAMPLE_DTYPE [N] of the draws (offsets of consecutive images of `sizes` in one buffer, scratch offsets)."""
        S = self.size
        rec = np.zeros(len(draws), SAMPLE_DTYPE)
        off = tmp = 0
        for n, ((H, W), p) in enumerate(zip(sizes, draws)):
            r = rec[n]
            r["offset"], r["h"], r["w"] = off, H, W
            r["ci"], r["cj"], r["ch"], r["cw"] = p["i"], p["j"], p["h"], p["w"]
            r["rh"] = r["rw"] = S
            r["filter"], r["flip"], r["tmp_offset"] = p["filter"], int(p["flip"]), tmp
            off += 3 * H * W
            tmp += 3 * S * p["h"]
            for s in range(2):
                pack_op(r["ops"][s], p["ops"][s] if s < len(p["ops"]) else None)
        return rec

    def pack_views(self, draws):
        """numpy SAMPLE_DTYPE [(S-1) * N] of the augmented views' RandAugment ops, split-major (view v of sample n at
        v * N + n); the other fields stay 0, as cotb200_aug_randaug reads only the ops."""
        views = [p["views"][v] for v in range(self.num_splits - 1) for p in draws]
        return _pack_ops(views, 0)

    @property
    def passes(self):
        """RandAugment launches per batch: ceil(num_layers / 2), as a launch applies COTB200_AUG_MAX_OPS = 2 ops per sample
        (at least 1: pass 0 also carries the resize-crop structs)."""
        return max(1, -(-self.num_layers // 2))

    def pack_pass(self, draws, k):
        """numpy SAMPLE_DTYPE of pass k >= 1: ops 2k and 2k + 1 of every row of pass 0 (the N samples, then with num_splits S
        the (S-1) * N views split-major); only the ops are set, as cotb200_aug_randaug reads nothing else."""
        rows = list(draws) + [p["views"][v] for v in range(self.num_splits - 1) for p in draws]
        return _pack_ops(rows, k)

    @property
    def has_jitter_kernel(self):
        """Whether the transform needs cotb200_aug_color_jitter (a vertical flip or ColorJitter)."""
        return self.vflip > 0 or self.jitter is not None

    @staticmethod
    def pack_jitter(draws):
        """numpy JITTER_DTYPE [N] of the draws' vertical flips and ColorJitter ops."""
        rec = np.zeros(len(draws), JITTER_DTYPE)
        rec["order"] = -1
        for n, p in enumerate(draws):
            rec["vflip"][n] = int(p.get("vflip", False))
            j = p.get("jitter")
            if j is None:
                continue
            rec["order"][n, :len(j["order"])] = j["order"]
            for k in range(3):
                if j["factors"][k] is not None:
                    rec["factor"][n, k] = j["factors"][k]
            if j["factors"][3] is not None:
                rec["hue"][n] = j["factors"][3]
        return rec

    def collate(self, batch):
        """DataLoader collate_fn (runs in the workers): [(HWC uint8 array, label), ...] -> AugBatch of CPU tensors, drawing
        from the worker's global `random`, `np.random` and torch generators as the reference's transforms do.  With the
        DataLoader's pin_memory=True the main process receives it pinned."""
        import random
        imgs = [np.ascontiguousarray(b[0], dtype=np.uint8) for b in batch]
        for a in imgs:
            if a.ndim != 3 or a.shape[2] != 3:
                raise ValueError("expected HWC RGB uint8 images, got shape %s" % (a.shape,))
        sizes = [a.shape[:2] for a in imgs]
        draws = self.draw(sizes, random, np.random, torch.default_generator)
        return self.collate_draws(imgs, [int(b[1]) for b in batch], draws)

    def collate_draws(self, imgs, labels, draws):
        """AugBatch of HWC uint8 `imgs` with their labels and draws.  With num_splits S >= 2 each image is shipped once; the
        structs are the B clean samples then the (S-1) * B views (pack_views), the jitter structs and the labels cover all S * B
        rows in fast_collate's order (labels repeated per split).  With more than two RandAugment layers the structs hold
        `passes` such blocks, pass k carrying ops 2k and 2k + 1 (pack_pass)."""
        sizes = [a.shape[:2] for a in imgs]
        rec = self.pack(sizes, draws)
        jit = [draws]
        if self.num_splits:
            rec = np.concatenate([rec, self.pack_views(draws)])
            jit += [[p["views"][k] for p in draws] for k in range(self.num_splits - 1)]
        if self.passes > 1:                             # pass-major: then the ops 2k, 2k + 1 of the same rows
            rec = np.concatenate([rec] + [self.pack_pass(draws, k) for k in range(1, self.passes)])
        data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs]))
        jitter = None
        if self.has_jitter_kernel:
            jitter = torch.from_numpy(np.concatenate([self.pack_jitter(d) for d in jit]).view(np.uint8).copy())
        lab = torch.tensor(labels, dtype=torch.int64)
        return AugBatch(data, torch.from_numpy(rec.view(np.uint8).copy()), lab.repeat(max(1, self.num_splits)), jitter)

    def __call__(self, batch, device=None):
        """AugBatch -> (uint8 [N, 3, S, S] on `device`, labels on `device`), on the current stream."""
        out = run(batch, self.size, device, randaug=self.num_layers > 0, num_splits=self.num_splits, passes=self.passes)
        return out, batch.labels.to(out.device, non_blocking=True)


def _pack_ops(rows, k):
    """SAMPLE_DTYPE [len(rows)] with only the ops set: ops 2k and 2k + 1 of each row's draws (op -1 past its list)."""
    rec = np.zeros(len(rows), SAMPLE_DTYPE)
    for r, p in zip(rec, rows):
        ops = p.get("ops", [])[2 * k:2 * k + 2]
        for s in range(2):
            pack_op(r["ops"][s], ops[s] if s < len(ops) else None)
    return rec


def pack_op(dst, op):
    dst["op"] = -1
    if op is None:
        return
    i = op["id"]
    dst["op"] = i
    if i in AFFINE_OPS:
        dst["m"] = op["matrix"]
        dst["filter"] = op["filter"]
    elif "iarg" in op:
        dst["v"][0] = op["iarg"]
    elif "factor" in op:
        dst["factor"] = op["factor"]
    elif "box" in op:
        dst["v"] = op["box"]


class EvalTransform:
    """transforms_imagenet_eval (use_prefetcher=True): Resize(floor(size / crop_pct), interpolation) + CenterCrop(size).
    Interpolation 'random' is bilinear here, as the reference's _pil_interp makes it.  With crop_pct=1.0 this is also the
    reference's train transform under augmentation.no_aug (transforms_noaug_train: Resize(size) + CenterCrop(size))."""

    def __init__(self, size=224, crop_pct=0.875, interpolation="bicubic"):
        self.size, self.crop_pct = int(size), crop_pct
        self.filter = BILINEAR if interpolation == "random" else _INTERP[interpolation]

    def pack(self, sizes):
        S = self.size
        rec = np.zeros(len(sizes), SAMPLE_DTYPE)
        off = tmp = 0
        for n, (H, W) in enumerate(sizes):
            rh, rw, top, left = eval_geometry(H, W, S, self.crop_pct)
            r = rec[n]
            r["offset"], r["h"], r["w"], r["ch"], r["cw"] = off, H, W, H, W
            r["rh"], r["rw"], r["oi"], r["oj"], r["filter"], r["tmp_offset"] = rh, rw, top, left, self.filter, tmp
            r["ops"]["op"] = -1
            off += 3 * H * W
            tmp += 3 * S * H
        return rec

    def collate(self, batch):
        imgs = [np.ascontiguousarray(b[0], dtype=np.uint8) for b in batch]
        rec = self.pack([a.shape[:2] for a in imgs])
        data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs]))
        return AugBatch(data, torch.from_numpy(rec.view(np.uint8).copy()),
                        torch.tensor([int(b[1]) for b in batch], dtype=torch.int64))

    def __call__(self, batch, device=None):
        out = run(batch, self.size, device, randaug=False)
        return out, batch.labels.to(out.device, non_blocking=True)


def uses_cluster_kernels(S):
    """Whether run() takes the thread-block-cluster kernels at output size S: above ONE_CTA_MAX_S, where one CTA's shared
    memory cannot hold the image."""
    return S > ONE_CTA_MAX_S


def run(batch, S, device=None, randaug=True, num_splits=0, cluster=None, passes=1):
    """The kernels on an AugBatch: H2D copies of the ragged buffer and the structs, resize-crop (+ flip), vertical flip and
    ColorJitter when the batch carries them, then RandAugment in place.  Returns uint8 [N, 3, S, S] on `device` (default: the
    current CUDA device).  With num_splits >= 2 (TrainAugment(num_splits=...)'s batch of B images) the clean views are
    resized, cropped and flipped into out[:B] and copied into each of the num_splits - 1 blocks after it, where the views'
    ColorJitter or RandAugment run in place: N = num_splits * B.
    The structs are `passes` blocks of N (TrainAugment.passes, pass-major): pass 0 drives every kernel, and each pass k
    launches RandAugment once more on the same rows, applying its ops after those of pass k - 1.
    ColorJitter and RandAugment run one CTA per image up to S = ONE_CTA_MAX_S and one thread-block cluster per image above
    it, up to CLUSTER_MAX_S, with the same bytes; `cluster` True / False forces one kind (None: by size)."""
    cluster = uses_cluster_kernels(S) if cluster is None else bool(cluster)
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    rec = batch.params.numpy().view(SAMPLE_DTYPE)
    if int(passes) != passes or passes < 1 or len(rec) % passes:
        raise ValueError("AugBatch: %d sample structs are not %r passes" % (len(rec), passes))
    N = len(rec) // passes
    splits = num_splits if num_splits >= 2 else 1
    if N % splits:
        raise ValueError("AugBatch: %d sample structs are not %d splits" % (N, splits))
    B = N // splits
    data = batch.data.to(device, non_blocking=True)
    params = batch.params.to(device, non_blocking=True)
    tmp_bytes = int((3 * S * rec["ch"][:B].astype(np.int64)).sum())
    tmp = torch.empty(max(tmp_bytes, 1), dtype=torch.uint8, device=device)
    out = torch.empty(N, 3, S, S, dtype=torch.uint8, device=device)
    lib = _lib.load()
    st = _lib.stream_ptr(out)
    host = rec.ctypes.data_as(ctypes.c_void_p)
    _lib.check(lib.cotb200_aug_resize_crop(B, S, data.data_ptr(), data.numel(), host, params.data_ptr(), tmp.data_ptr(),
                                           tmp.numel(), out.data_ptr(), st), "aug_resize_crop")
    jrec = jdev = None
    if batch.jitter is not None:
        jrec = batch.jitter.numpy().view(JITTER_DTYPE)
        if len(jrec) != N:
            raise ValueError("AugBatch: %d jitter structs for %d samples" % (len(jrec), N))
        if jrec["vflip"].any() or (jrec["order"] >= 0).any():
            jdev = batch.jitter.to(device, non_blocking=True)

    def jitter(lo, hi):
        if jdev is not None and (jrec["vflip"][lo:hi].any() or (jrec["order"][lo:hi] >= 0).any()):
            fn = lib.cotb200_aug_color_jitter_cluster if cluster else lib.cotb200_aug_color_jitter
            _lib.check(fn(hi - lo, S, jrec[lo:].ctypes.data_as(ctypes.c_void_p), jdev.data_ptr() + lo * JITTER_DTYPE.itemsize,
                          out[lo].data_ptr(), st), "aug_color_jitter")

    def randaug_(lo, hi, base):                     # rows lo..hi of out, their structs at base + lo
        if randaug and (rec["ops"]["op"][base + lo:base + hi] >= 0).any():
            fn = lib.cotb200_aug_randaug_cluster if cluster else lib.cotb200_aug_randaug
            _lib.check(fn(hi - lo, S, rec[base + lo:].ctypes.data_as(ctypes.c_void_p),
                          params.data_ptr() + (base + lo) * SAMPLE_DTYPE.itemsize, out[lo].data_ptr(), st), "aug_randaug")
    jitter(0, B)
    if splits > 1:                                  # the augmented views start from the clean view, vertical flip included
        for k in range(1, splits):
            out[k * B:(k + 1) * B].copy_(out[:B])
        jitter(B, N)
    for k in range(passes):                         # in order on one stream: pass k works on pass k - 1's output
        randaug_(B if splits > 1 else 0, N, k * N)
    return out


# ---------------------------------------------------------------------------------------------------- random erasing
class EraseParams:
    """One batch's erase table (struct cotb200_erase + its boxes): `host` the uint8 buffer and its device copy (_lib.DeviceCopy,
    issued on the stream current at creation), which consumers take through on_stream()."""

    def __init__(self, host, device):
        self.host = host
        self._copy = _lib.DeviceCopy(host, device)

    @property
    def header(self):
        return self.host[:ERASE_DTYPE.itemsize].view(ERASE_DTYPE)[0]

    @property
    def boxes(self):
        return self.host[ERASE_DTYPE.itemsize:].view(ERASE_BOX_DTYPE)

    def on_stream(self, device):
        return self._copy.on_stream(device, "erase")


class RandomErasing:
    """The reference's RandomErasing (datasets/random_erasing.py) on the normalised channels_last batch that normalize_u8
    returns, as PrefetchLoader applies it after the normalisation (datasets/loader.py:72-91): per image (from B // num_splits
    when num_splits > 1) with `probability`, 1..max_count boxes of area 0.02..1/3 of the image (divided by the count) and
    aspect 0.3..1/0.3, filled with 0 ('const'), one N(0,1) value per channel ('rand') or per element ('pixel').  The boxes are
    drawn on the host from a ``random.Random`` in the reference's order (``draw``); the normal values come from the kernel's
    counter-based generator keyed by a per-call seed, and are rounded to the batch's dtype.  ``resplit`` of the reference's
    loader is num_splits=2 (loader.py:158-161)."""
    MODES = {"const": 0, "rand": 1, "pixel": 2}

    def __init__(self, probability=0.5, mode="const", max_count=1, num_splits=0, seed=0):
        mode = (mode or "const").lower()
        if mode not in self.MODES:
            raise ValueError("RandomErasing: mode must be 'const', 'rand' or 'pixel', got %r" % (mode,))
        max_count = int(max_count or 1)
        if not 1 <= max_count <= ERASE_MAX_COUNT:
            raise ValueError("RandomErasing: max_count %d outside 1..%d" % (max_count, ERASE_MAX_COUNT))
        self.probability, self.mode = float(probability), mode
        self.min_area, self.max_area = 0.02, 1 / 3
        self.log_aspect_ratio = (math.log(0.3), math.log(1 / 0.3))
        self.min_count, self.max_count = 1, max_count
        self.num_splits = int(num_splits)
        self.rnd = random.Random(seed)
        self._seeds = np.random.default_rng(seed)

    def _erase(self, H, W, rnd):                                    # RandomErasing._erase, the draws only
        if rnd.random() > self.probability:
            return []
        area = H * W
        count = self.min_count if self.min_count == self.max_count else rnd.randint(self.min_count, self.max_count)
        boxes = []
        for _ in range(count):
            for _ in range(10):
                target_area = rnd.uniform(self.min_area, self.max_area) * area / count
                aspect_ratio = math.exp(rnd.uniform(*self.log_aspect_ratio))
                h = int(round(math.sqrt(target_area * aspect_ratio)))
                w = int(round(math.sqrt(target_area / aspect_ratio)))
                if w < W and h < H:
                    top = rnd.randint(0, H - h)
                    left = rnd.randint(0, W - w)
                    boxes.append((top, left, h, w))
                    break
        return boxes

    def draw(self, B, H, W, rnd=None):
        """The boxes of a batch of B images of H x W, drawn in the reference's order from `rnd` (default: this object's own
        random.Random(seed)): a list of B lists of (top, left, h, w), each in draw order."""
        rnd = self.rnd if rnd is None else rnd
        start = B // self.num_splits if self.num_splits > 1 else 0
        return [self._erase(H, W, rnd) if i >= start else [] for i in range(B)]

    def pack(self, boxes, seed):
        """uint8 numpy buffer: the ERASE_DTYPE header and the ERASE_BOX_DTYPE table of `boxes` (empty boxes dropped)."""
        rows = [(n, k, t, l, h, w) for n, bs in enumerate(boxes)
                for k, (t, l, h, w) in enumerate([b for b in bs if b[2] > 0 and b[3] > 0])]
        hdr = np.zeros(1, ERASE_DTYPE)
        hdr["mode"], hdr["n_boxes"], hdr["seed"] = self.MODES[self.mode], len(rows), seed
        return np.concatenate([hdr.view(np.uint8), np.array(rows, ERASE_BOX_DTYPE).view(np.uint8)])

    def params(self, B, H, W, device):
        """The next batch's draws as EraseParams on `device` (the copy issued on the current stream)."""
        seed = int(self._seeds.integers(0, 1 << 64, dtype=np.uint64))
        return EraseParams(self.pack(self.draw(B, H, W), seed), device)

    def apply(self, x, params):
        """Erases the boxes of `params` in x (CUDA [B, C, H, W], channels_last, fp32 / bf16 / fp16) in place on the current
        stream; returns x."""
        _lib.require_cuda(x, "RandomErasing")
        if x.dim() != 4 or not x.is_contiguous(memory_format=torch.channels_last):
            raise ValueError("RandomErasing: expected a channels_last [B, C, H, W] batch (normalize_u8's output)")
        if x.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            raise TypeError("RandomErasing: dtype %s is not fp32, bf16 or fp16" % x.dtype)
        B, C, H, W = x.shape
        host = params.host
        if params.header["n_boxes"] == 0:
            return x
        _lib.check(_lib.load().cotb200_aug_erase(_lib.dtype_code(x), B, C, H, W, x.data_ptr(), host.ctypes.data,
                                                 params.on_stream(x.device).data_ptr(), _lib.stream_ptr(x)), "aug_erase")
        return x

    def __call__(self, x):
        """Draws the next batch's boxes and erases them in x in place (the reference's random_erasing(next_input))."""
        return self.apply(x, self.params(x.shape[0], x.shape[2], x.shape[3], x.device))
