"""Build tests/golden/augment_large.npz: the reference's own transforms (datasets/transforms_factory.py) run with Pillow at the
288 x 288 and 320 x 320 data configs (models/cotnet_hybrid.py cot_m and cot_l), whose images do not fit one CTA's shared memory
and go through the thread-block-cluster augmentation kernels.  Needs the reference checkout (oracle/ref_import.py provides the
import shims) and Pillow.

    python tools/make_augment_large_golden.py [out.npz]

Holds:
  train_<S>_<k>   RandomResizedCrop + horizontal flip + rand-m15-mstd0.5-n2, bicubic, at S = 288 and 320 (uint8 CHW), with
                  train_<S>_<k>_size = (H, W, seed, image seed);
  jout_320_<k>    ColorJitter 0.4 + vertical flip 0.5 without auto_augment, at 320, likewise;
  eval_<S>_<k>    Resize(floor(S / crop_pct)) + CenterCrop(S), bicubic, at 320 / crop_pct 0.909 and 288 / 0.9, with
                  eval_<S>_<k>_size = (H, W, image seed) and eval_<S>_crop_pct.
Source images are oracle.aug_ref.source_image(seed, H, W), not stored; uint8 images are stored as row differences
(oracle.aug_ref.encode_golden); read the file with oracle.aug_ref.load_golden.
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

#: ImageNet-like sources: landscape and portrait 4:3, square, a small one (upscaled) and a wide one
SIZES = ((375, 500), (500, 375), (333, 333), (180, 240), (300, 900))
TRAIN = {288: 4, 320: 5}
JITTER = {320: 5}
EVAL = {320: 0.909, 288: 0.9}


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
    from datasets.transforms_factory import transforms_imagenet_eval, transforms_imagenet_train

    g = {}
    for S, n in TRAIN.items():
        tf = transforms_imagenet_train(S, auto_augment="rand-m15-mstd0.5-n2", interpolation="bicubic", use_prefetcher=True)
        for k in range(n):
            H, W = SIZES[k]
            seed, iseed = 5000 + 10 * S + k, 500 + k
            seed_all(seed)
            g["train_%d_%d" % (S, k)] = np.asarray(tf(Image.fromarray(source_image(iseed, H, W))), np.uint8)
            g["train_%d_%d_size" % (S, k)] = np.array([H, W, seed, iseed], np.int32)
    for S, n in JITTER.items():
        tf = transforms_imagenet_train(S, auto_augment=None, color_jitter=0.4, vflip=0.5, interpolation="bicubic",
                                       use_prefetcher=True)
        for k in range(n):
            H, W = SIZES[k]
            seed, iseed = 6000 + 10 * S + k, 600 + k
            seed_all(seed)
            g["jout_%d_%d" % (S, k)] = np.asarray(tf(Image.fromarray(source_image(iseed, H, W))), np.uint8)
            g["jout_%d_%d_size" % (S, k)] = np.array([H, W, seed, iseed], np.int32)
    for S, crop_pct in EVAL.items():
        tf = transforms_imagenet_eval(S, crop_pct=crop_pct, interpolation="bicubic", use_prefetcher=True)
        g["eval_%d_crop_pct" % S] = np.array(crop_pct, np.float64)
        for k in range(3):
            H, W = SIZES[k]
            iseed = 700 + 10 * k + S
            g["eval_%d_%d" % (S, k)] = np.asarray(tf(Image.fromarray(source_image(iseed, H, W))), np.uint8)
            g["eval_%d_%d_size" % (S, k)] = np.array([H, W, iseed], np.int32)
    np.savez_compressed(path, **{k: encode_golden(v) for k, v in g.items()})
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "augment_large.npz"))
