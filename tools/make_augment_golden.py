"""Build tests/golden/augment.npz from the reference's own transforms (datasets/transforms_factory.py, datasets/rand_augment.py)
run with Pillow.  Needs the reference checkout (oracle/ref_import.py provides the import shims) and Pillow.

    python tools/make_augment_golden.py [out.npz]

Holds:
  draws_*   what the reference's train transform drew for 200 seeds on varied image sizes (crop box, flip, op ids, whether each
            op ran, its resolved argument) plus the next value of each generator afterwards (so a draw that consumes more or
            less than the reference is caught);
  train_*   full train-pipeline outputs (uint8 CHW) for portrait, landscape, smaller-than-224 and central-crop-fallback sources;
  op_*      each of the 16 RandAugment ops at three magnitudes (and both signs) on a 64 x 64 image, incl. rotate +-45 deg (magnitude 15);
  eval_*    eval transform outputs (Resize(256) + CenterCrop(224), bicubic).
Source images are smooth synthetic content generated from a seed (oracle.aug_ref.source_image), not stored.  Images are
stored as row differences (oracle.aug_ref.encode_golden); read the file with oracle.aug_ref.load_golden.
"""
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402
from oracle.aug_ref import encode_golden, source_image  # noqa: E402

OPS = ("AutoContrast", "Equalize", "Invert", "Rotate", "Posterize", "Solarize", "SolarizeAdd", "Color", "Contrast",
       "Brightness", "Sharpness", "ShearX", "ShearY", "TranslateX", "TranslateY", "Cutout")
DRAW_SEEDS = 200
TRAIN_SIZES = ((500, 375), (375, 500), (150, 180), (200, 900), (333, 333), (256, 310))
EVAL_SIZES = ((500, 375), (375, 500), (224, 224))


def draw_size(seed):
    r = np.random.RandomState(10_000 + seed)
    if seed % 10 == 9:                       # extreme aspect ratios: the central-crop fallback
        return (int(r.randint(16, 60)), int(r.randint(300, 600))) if seed % 20 == 9 else (int(r.randint(300, 600)), int(r.randint(16, 60)))
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
    import datasets.rand_augment as ra
    import datasets.transforms as rt
    from datasets.transforms_factory import transforms_imagenet_eval, transforms_imagenet_train

    rec = {}
    orig_get_params = rt.RandomResizedCropAndInterpolation.get_params
    orig_ops = dict(ra.NAME_TO_OP)

    def get_params(img, scale, ratio):
        p = orig_get_params(img, scale, ratio)
        rec["crop"] = p
        return p

    rt.RandomResizedCropAndInterpolation.get_params = staticmethod(get_params)

    def wrap(name):
        f = orig_ops[name]

        def g(img, *args, **kw):
            out = f(img, *args, **kw)
            rec["ops"].append((OPS.index(name), args[0] if args else 0.0))
            return out
        return g

    for name in OPS:
        ra.NAME_TO_OP[name] = wrap(name)
    # AugmentOp looks its function up at construction, so the transform is built after the wrapping
    tf = transforms_imagenet_train(224, auto_augment="rand-m15-mstd0.5-n2", interpolation="bicubic", use_prefetcher=True)
    flip = tf.transforms[1]                                  # RandomHorizontalFlip returns its input object when not flipping

    def flip_rec(img):
        out = flip(img)
        rec["flip"] = out is not img
        return out

    tf.transforms[1] = flip_rec
    g = {}
    # ---- draws
    crops, flips, ids, args, sizes, nxt = [], [], [], [], [], []
    for s in range(DRAW_SEEDS):
        H, W = draw_size(s)
        img = Image.fromarray(source_image(s, H, W)) if s < 8 else Image.new("RGB", (W, H), (90, 120, 150))
        seed_all(s)
        rec["ops"] = []
        tf(img)
        crops.append(rec["crop"])
        flips.append(rec["flip"])
        applied = rec["ops"]
        sizes.append((H, W))
        nxt.append((random.random(), np.random.random_sample(), float(torch.rand(1))))
        ids.append([o[0] for o in applied] + [-1] * (2 - len(applied)))
        args.append([float(o[1]) for o in applied] + [0.0] * (2 - len(applied)))
    g["draws_sizes"] = np.array(sizes, np.int32)
    g["draws_crop"] = np.array(crops, np.int32)
    g["draws_flip"] = np.array(flips, np.int32)
    g["draws_ids"] = np.array(ids, np.int32)
    g["draws_args"] = np.array(args, np.float64)
    g["draws_next"] = np.array(nxt, np.float64)
    # ---- full train outputs
    for k, (H, W) in enumerate(TRAIN_SIZES):
        seed_all(1000 + k)
        rec["ops"] = []
        out = tf(Image.fromarray(source_image(100 + k, H, W)))
        g["train_%d" % k] = np.asarray(out, np.uint8)
        g["train_%d_size" % k] = np.array([H, W, 1000 + k, 100 + k], np.int32)
    # ---- single ops on a 64 x 64 image
    src = Image.fromarray(source_image(7, 64, 64))
    kw = dict(fillcolor=(124, 116, 104), resample=Image.BICUBIC)
    cases = []
    for name in OPS:
        for mag in (0.0, 7.5, 15.0):
            lf = ra.LEVEL_TO_ARG[name]
            for sign in ((0.9, 0.1) if name in ("Rotate", "ShearX", "ShearY", "TranslateX", "TranslateY") else (0.9,)):
                random.seed(0)
                np.random.seed(0)
                saved = random.random
                random.random = (lambda v=sign: v)
                try:
                    level = lf(mag, {"translate_const": 100, "cutout_const": 40}) if lf else ()
                finally:
                    random.random = saved
                np.random.seed(len(cases))
                out = orig_ops[name](src, *level, **dict(kw))
                cases.append((OPS.index(name), float(level[0]) if level else 0.0, len(cases)))
                g["op_%d" % (len(cases) - 1)] = np.asarray(out, np.uint8)
    g["op_src"] = np.asarray(src, np.uint8)
    g["op_cases"] = np.array(cases, np.float64)
    # ---- eval
    etf = transforms_imagenet_eval(224, interpolation="bicubic", use_prefetcher=True)
    for k, (H, W) in enumerate(EVAL_SIZES):
        g["eval_%d" % k] = np.asarray(etf(Image.fromarray(source_image(200 + k, H, W))), np.uint8)
        g["eval_%d_size" % k] = np.array([H, W, 200 + k], np.int32)
    np.savez_compressed(path, **{k: encode_golden(v) for k, v in g.items()})
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "augment.npz"))
