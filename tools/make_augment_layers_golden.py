"""Build tests/golden/augment_layers.npz: the reference's own transforms (datasets/transforms_factory.py,
datasets/rand_augment.py) run with Pillow on RandAugment configs with more than two layers and with the weighted op choice
('w0'), and its no_aug train transform.  Needs the reference checkout (oracle/ref_import.py provides the import shims) and
Pillow.

    python tools/make_augment_layers_golden.py [out.npz]

Holds (c the index into `configs`):
  configs             the RandAugment config strings (CONFIGS);
  weights_0           _select_rand_weights(0), the reference's choice weights of 'w0' (float64);
  d_<c>_*             what transforms_imagenet_train(224, auto_augment=configs[c]) drew for DRAW_SEEDS seeds on the sizes
                      d_sizes (uniform images): the applied ops' ids and level arguments (-1 / 0 padded to the layer count) and
                      the next value of each generator afterwards (random, np.random, torch);
  train_<c>_<S>_<k>   its uint8 CHW output at S = 224 and 320, with _size = (H, W, seed, image seed) and _next the generators'
                      next values after the image;
  split_<S>           AugMixDataset(num_splits=3) over transforms_imagenet_train(S, 'rand-m9-n3-mstd0.5', separate=True),
                      collated by fast_collate: uint8 [3*B, 3, S, S] stored as [3*B*3, S, S], with split_<S>_meta = (seed, B, S),
                      split_<S>_src = (H, W, image seed) per image and split_<S>_next;
  noaug_<interp>_<S>_<k>  transforms_noaug_train(S, interpolation) for 'bicubic' and 'random', with _size = (H, W, image seed).
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

CONFIGS = ("rand-m9-n3-mstd0.5", "rand-m15-n5-mstd0.5", "rand-mstd1-w0", "rand-m15-n4-mstd0.5-w0")
DRAW_SEEDS = 60
#: ImageNet-like sources: landscape and portrait 4:3, square, small (upscaled), wide
SIZES = ((375, 500), (500, 375), (333, 333), (180, 240), (300, 900))
TRAIN_N = 2
SPLIT_SIZES = ((375, 500), (240, 180))
NOAUG_N = 2


def draw_size(seed):
    r = np.random.RandomState(20_000 + seed)
    return int(r.randint(64, 640)), int(r.randint(64, 640))


def seed_all(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def next_values():
    return random.random(), np.random.random_sample(), float(torch.rand(1))


def main(path):
    if not ref_import.available():
        raise SystemExit("reference checkout not found")
    ref_import._install_shims()
    sys.path.insert(0, ref_import.REF)
    from PIL import Image
    import datasets.rand_augment as ra
    from datasets.dataset import AugMixDataset
    from datasets.loader import fast_collate
    from datasets.transforms_factory import transforms_imagenet_train, transforms_noaug_train

    names = list(ra._RAND_TRANSFORMS)
    orig_ops = dict(ra.NAME_TO_OP)
    rec = {"ops": []}

    def wrap(name):
        f = orig_ops[name]

        def g(img, *args, **kw):
            rec["ops"].append((names.index(name), args[0] if args else 0.0))
            return f(img, *args, **kw)
        return g

    for name in names:                   # AugmentOp looks its function up at construction: wrap before building
        ra.NAME_TO_OP[name] = wrap(name)

    def train_tf(S, aa, **kw):
        return transforms_imagenet_train(S, auto_augment=aa, interpolation="bicubic", use_prefetcher=True, **kw)

    g = {"configs": np.array(CONFIGS), "weights_0": np.asarray(ra._select_rand_weights(0), np.float64)}
    g["d_sizes"] = np.array([draw_size(s) for s in range(DRAW_SEEDS)], np.int32)
    for c, aa in enumerate(CONFIGS):
        n = ra.rand_augment_transform(aa, {}).num_layers
        tf = train_tf(224, aa)
        ids, args, nxt = [], [], []
        for s, (H, W) in enumerate(g["d_sizes"]):
            img = Image.new("RGB", (int(W), int(H)), (90, 120, 150))
            seed_all(40_000 + 100 * c + s)
            rec["ops"] = []
            tf(img)
            nxt.append(next_values())
            ids.append([o[0] for o in rec["ops"]] + [-1] * (n - len(rec["ops"])))
            args.append([float(o[1]) for o in rec["ops"]] + [0.0] * (n - len(rec["ops"])))
        g["d_%d_ids" % c] = np.array(ids, np.int32).reshape(DRAW_SEEDS, n)
        g["d_%d_args" % c] = np.array(args, np.float64).reshape(DRAW_SEEDS, n)
        g["d_%d_next" % c] = np.array(nxt, np.float64)
        g["d_%d_seed0" % c] = np.array([40_000 + 100 * c], np.int64)
        for S in (224, 320):
            tf = train_tf(S, aa)
            for k in range(TRAIN_N):
                H, W = SIZES[(c + k) % len(SIZES)]
                seed, iseed = 50_000 + 1000 * c + 10 * S + k, 900 + 10 * c + k
                seed_all(seed)
                key = "train_%d_%d_%d" % (c, S, k)
                g[key] = np.asarray(tf(Image.fromarray(source_image(iseed, H, W))), np.uint8)
                g[key + "_size"] = np.array([H, W, seed, iseed], np.int32)
                g[key + "_next"] = np.array(next_values(), np.float64)

    class Images:
        def __init__(self, imgs):
            self.imgs, self.transform = imgs, None

        def __getitem__(self, i):
            return self.transform(self.imgs[i]), i

        def __len__(self):
            return len(self.imgs)

    for S in (224, 320):
        primary, secondary, final = train_tf(S, "rand-m9-n3-mstd0.5", separate=True)
        src = [(H, W, 960 + k) for k, (H, W) in enumerate(SPLIT_SIZES)]
        ds = AugMixDataset(Images([Image.fromarray(source_image(i, H, W)) for H, W, i in src]), num_splits=3)
        ds.transform = (primary, secondary, final)
        seed = 70_000 + S
        seed_all(seed)
        x, _ = fast_collate([ds[i] for i in range(len(ds))])
        g["split_%d" % S] = x.numpy().reshape(-1, S, S)
        g["split_%d_meta" % S] = np.array([seed, len(src), S], np.int64)
        g["split_%d_src" % S] = np.array(src, np.int32)
        g["split_%d_next" % S] = np.array(next_values(), np.float64)

    for interp in ("bicubic", "random"):
        for S in (224, 320):
            tf = transforms_noaug_train(S, interpolation=interp, use_prefetcher=True)
            for k in range(NOAUG_N):
                H, W = SIZES[(2 * k + (S == 320)) % len(SIZES)]
                iseed = 980 + 10 * k + S
                key = "noaug_%s_%d_%d" % (interp, S, k)
                g[key] = np.asarray(tf(Image.fromarray(source_image(iseed, H, W))), np.uint8)
                g[key + "_size"] = np.array([H, W, iseed], np.int32)
    np.savez_compressed(path, **{k: encode_golden(v) for k, v in g.items()})
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "augment_layers.npz"))
