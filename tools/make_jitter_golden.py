"""Build tests/golden/augment_jitter.npz from the reference's own transforms_imagenet_train (ColorJitter, RandomVerticalFlip)
and RandomErasing, run with Pillow and torch on the CPU.  Needs the reference checkout (oracle/ref_import.py provides the import
shims) and Pillow.

    python tools/make_jitter_golden.py [out.npz]

Holds, for cfg 0 (color_jitter=0.4) and cfg 1 (color_jitter=(0.4, 0.4, 0.4, 0.1)), both with vflip=0.5, no auto_augment:
  jd_*         per seed: crop box, horizontal / vertical flip, ColorJitter's permutation and factors (NaN: off) and the next
               value of each generator afterwards (random, np.random, torch);
  jout_*       full train-pipeline outputs (uint8 CHW) with their (H, W, seed, image seed);
  jra_*        vflip=0.5 with auto_augment='rand-m15-mstd0.5-n2' (ColorJitter is then not applied);
  er_*         RandomErasing: the uint8 batch `er_u8`, the 'const' erased fp32 batches PrefetchLoader's normalisation + erasing
               produce (er_const_*), and for every case the boxes (image, k, top, left, h, w) and which images were erased
               (1 erased, 0 skipped, -1 before batch_start), plus random.random() afterwards.
Source images are oracle.aug_ref.source_image(seed, H, W), not stored; uint8 images are stored as row differences
(oracle.aug_ref.encode_golden); read the file with oracle.aug_ref.load_golden.
"""
import math
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402
from oracle.aug_ref import encode_golden, source_image  # noqa: E402

DRAW_SEEDS = 100
OUT_SIZES = ((500, 375), (375, 500), (150, 180), (333, 333), (256, 310), (200, 900))
CONFIGS = (0.4, (0.4, 0.4, 0.4, 0.1))
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
#: erase cases: name -> (probability, mode, max_count, num_splits, B, H, W, store the erased batch)
ERASE_CASES = {"c1": (0.5, "const", 1, 0, 8, 32, 48, True), "c3s": (0.7, "const", 3, 2, 8, 32, 48, True),
               "r3": (0.25, "rand", 3, 0, 64, 224, 224, False), "p1": (0.25, "pixel", 1, 0, 64, 224, 224, False),
               "p3s": (0.6, "pixel", 3, 2, 64, 224, 224, False)}


def draw_size(seed):
    r = np.random.RandomState(20_000 + seed)
    return int(r.randint(64, 640)), int(r.randint(64, 640))


def seed_all(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def main(path):
    if not ref_import.available():
        raise SystemExit("reference checkout not found")
    ref_import._install_shims()
    sys.path.insert(0, ref_import.REF)
    from PIL import Image
    from torchvision import transforms
    import datasets.random_erasing as rer
    import datasets.transforms as rt
    from datasets.transforms_factory import transforms_imagenet_train

    rec = {}
    orig_get_params = rt.RandomResizedCropAndInterpolation.get_params
    orig_cj_params = transforms.ColorJitter.get_params

    def get_params(img, scale, ratio):
        p = orig_get_params(img, scale, ratio)
        rec["crop"] = p
        return p

    def cj_params(*a):
        p = orig_cj_params(*a)
        rec["cj"] = p
        return p

    rt.RandomResizedCropAndInterpolation.get_params = staticmethod(get_params)
    transforms.ColorJitter.get_params = staticmethod(cj_params)

    def recording(t, key):                                       # a flip returns its input object when it does not flip
        def f(img):
            out = t(img)
            rec[key] = out is not img
            return out
        return f

    def build(**kw):
        tf = transforms_imagenet_train(224, interpolation="bicubic", use_prefetcher=True, vflip=0.5, **kw)
        tf.transforms[1] = recording(tf.transforms[1], "flip")
        tf.transforms[2] = recording(tf.transforms[2], "vflip")
        return tf

    g = {}
    g["jd_sizes"] = np.array([draw_size(s) for s in range(DRAW_SEEDS)], np.int32)
    for c, cj in enumerate(CONFIGS):
        tf = build(auto_augment=None, color_jitter=cj)
        crops, flips, vflips, perms, factors, nxt = [], [], [], [], [], []
        for s in range(DRAW_SEEDS):
            H, W = (int(v) for v in g["jd_sizes"][s])
            img = Image.fromarray(source_image(s, H, W)) if s < 8 else Image.new("RGB", (W, H), (90, 120, 150))
            seed_all(s)
            tf(img)
            crops.append(rec["crop"])
            flips.append(rec["flip"])
            vflips.append(rec["vflip"])
            perm, *f = rec["cj"]
            perms.append([int(v) for v in perm])
            factors.append([math.nan if v is None else v for v in f])
            nxt.append((random.random(), np.random.random_sample(), float(torch.rand(1))))
        g["jd_crop_%d" % c] = np.array(crops, np.int32)
        g["jd_flip_%d" % c] = np.array(flips, np.int32)
        g["jd_vflip_%d" % c] = np.array(vflips, np.int32)
        g["jd_perm_%d" % c] = np.array(perms, np.int32)
        g["jd_factors_%d" % c] = np.array(factors, np.float64)
        g["jd_next_%d" % c] = np.array(nxt, np.float64)
        for k, (H, W) in enumerate(OUT_SIZES):
            seed, iseed = 3000 + 100 * c + k, 300 + k
            seed_all(seed)
            g["jout_%d_%d" % (c, k)] = np.asarray(tf(Image.fromarray(source_image(iseed, H, W))), np.uint8)
            g["jout_%d_%d_size" % (c, k)] = np.array([H, W, seed, iseed], np.int32)
    tf = build(auto_augment="rand-m15-mstd0.5-n2", color_jitter=0.4)
    for k, (H, W) in enumerate(OUT_SIZES):
        seed, iseed = 4000 + k, 400 + k
        seed_all(seed)
        g["jra_%d" % k] = np.asarray(tf(Image.fromarray(source_image(iseed, H, W))), np.uint8)
        g["jra_%d_size" % k] = np.array([H, W, seed, iseed], np.int32)

    # ---- random erasing: the draws seen through the module's `random` and `_get_pixels`
    class Recorder:
        def __init__(self):
            self.log = []

        def random(self):
            v = random.random()
            self.log.append(("random", v))
            return v

        def randint(self, a, b):
            v = random.randint(a, b)
            self.log.append(("randint", v))
            return v

        def uniform(self, a, b):
            return random.uniform(a, b)

    recorder = Recorder()
    rer.random = recorder
    orig_get_pixels = rer._get_pixels
    boxes = []

    def get_pixels(per_pixel, rand_color, patch_size, dtype=torch.float32, device="cuda"):
        top, left = recorder.log[-2][1], recorder.log[-1][1]
        boxes.append((rec["image"], top, left, int(patch_size[1]), int(patch_size[2])))
        return orig_get_pixels(per_pixel, rand_color, patch_size, dtype=dtype, device=device)

    rer._get_pixels = get_pixels
    orig_erase = rer.RandomErasing._erase

    def erase(self, img, chan, img_h, img_w, dtype):
        rec["image"] += 1
        n0 = len(recorder.log)
        orig_erase(self, img, chan, img_h, img_w, dtype)
        rec["hit"][rec["image"]] = int(recorder.log[n0][1] <= self.probability)

    rer.RandomErasing._erase = erase
    u8 = np.stack([source_image(500 + n, 32, 48).transpose(2, 0, 1) for n in range(8)])
    g["er_u8"] = u8
    mean = torch.tensor([x * 255 for x in MEAN]).view(1, 3, 1, 1)
    std = torch.tensor([x * 255 for x in STD]).view(1, 3, 1, 1)
    for ci, (name, (p, mode, count, splits, B, H, W, store)) in enumerate(ERASE_CASES.items()):
        re_ = rer.RandomErasing(probability=p, mode=mode, max_count=count, num_splits=splits, device="cpu")
        x = torch.from_numpy(u8).float().sub_(mean).div_(std) if store else torch.zeros(B, 3, H, W)
        batch_start = B // splits if splits > 1 else 0
        rec["image"] = batch_start - 1
        rec["hit"] = [-1] * B
        boxes.clear()
        random.seed(7000 + ci)
        torch.manual_seed(7000 + ci)
        out = re_(x)
        table, k_of = [], {}
        for n, t, l, h, w in boxes:
            k_of[n] = k_of.get(n, -1) + 1
            table.append((n, k_of[n], t, l, h, w))
        g["er_boxes_%s" % name] = np.array(table, np.int32).reshape(-1, 6)
        g["er_hit_%s" % name] = np.array(rec["hit"], np.int32)
        g["er_next_%s" % name] = np.array([random.random()], np.float64)
        g["er_case_%s" % name] = np.array([p, ("const", "rand", "pixel").index(mode), count, splits, B, H, W, 7000 + ci], np.float64)
        if store:
            g["er_const_%s" % name] = out.numpy().astype(np.float32)
    np.savez_compressed(path, **{k: encode_golden(v) for k, v in g.items()})
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "augment_jitter.npz"))
