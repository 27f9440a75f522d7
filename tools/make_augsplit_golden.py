"""Build tests/golden/augsplit.npz from the reference's own augmentation splits and JSD loss, run with Pillow and torch on the
CPU: transforms_imagenet_train(separate=True) inside AugMixDataset(num_splits=S), collated by fast_collate, and
JsdCrossEntropy.  Needs the reference checkout (oracle/ref_import.py provides the import shims) and Pillow.

    python tools/make_augsplit_golden.py [out.npz]

Cases (CASES): S = 2 and 3, 'rand-m15-mstd0.5-n2' or color_jitter=0.4 without auto_augment, vflip 0 or 0.5, bicubic.  Per case:
  d_<case>_*   a batch of DRAW_N images of the sizes `d_sizes` (source_image(seed, H, W)) after seed_all(seed): per image the
               crop box, horizontal and vertical flip; per augmented view (image-major, view-minor) the applied RandAugment ops
               (id, level argument; -1 padded) or ColorJitter's permutation and factors (NaN: off); the next value of each
               generator afterwards (random, np.random, torch) and fast_collate's labels;
  o_<case>     fast_collate's uint8 batch [S*B, 3, SIZE, SIZE] of OUT_SIZES at SIZE, stored as [S*B*3, SIZE, SIZE], with
               o_<case>_meta = (seed, B, SIZE) and o_<case>_src = (H, W, image seed) per image;
  jsd_<name>   JsdCrossEntropy(num_splits=S, smoothing) on fp64 logits: _z the logits, _y the labels, _loss, _grad (autograd;
               NaN where the reference's gradient is), _meta = (S, smoothing).
uint8 images are stored as row differences (oracle.aug_ref.encode_golden); read the file with oracle.aug_ref.load_golden.
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

SIZE = 112
DRAW_N = 12
OUT_SIZES = ((300, 220), (180, 260))
#: name -> (num_splits, auto_augment, vflip)
CASES = {"s2_rand_v0": (2, "rand-m15-mstd0.5-n2", 0.), "s2_cj_v5": (2, None, 0.5), "s3_rand_v5": (3, "rand-m15-mstd0.5-n2", 0.5),
         "s3_cj_v0": (3, None, 0.), "s2_rand_v5": (2, "rand-m15-mstd0.5-n2", 0.5), "s2_cj_v0": (2, None, 0.),
         "s3_rand_v0": (3, "rand-m15-mstd0.5-n2", 0.), "s3_cj_v5": (3, None, 0.5)}


def draw_size(seed):
    r = np.random.RandomState(30_000 + seed)
    return int(r.randint(64, 400)), int(r.randint(64, 400))


def seed_all(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def jsd_cases():
    """name -> (S, smoothing, logits [S*B, K] fp64, labels [B])."""
    r = np.random.RandomState(5)
    out = {"r3": (3, 0.1, r.randn(3 * 4, 10) * 3, r.randint(0, 10, 4)),
           "r2": (2, 0.0, r.randn(2 * 5, 7) * 2, r.randint(0, 7, 5))}
    # clamp: sample 0 is one-hot-like in every split (its mixture is exactly 1 at class 0 and below 1e-7 elsewhere); sample 1
    # puts one split's mass elsewhere; sample 2 is ordinary
    z = r.randn(3 * 3, 6)
    for s in range(3):
        z[s * 3] = [40, 0, 0, 0, 0, 0]
        z[1 + s * 3] = [0, 0, 30, 0, 0, 0] if s == 1 else [30, 0, 0, 0, 0, 0]
    out["clamp"] = (3, 0.1, z, np.array([0, 2, 4]))
    # underflow: split 1 of sample 0 has a probability that is exactly 0 in fp64 (the reference's gradient is NaN there)
    z = r.randn(3 * 2, 5)
    z[2, 3] = -800.0
    out["underflow"] = (3, 0.1, z, np.array([1, 3]))
    return out


def main(path):
    if not ref_import.available():
        raise SystemExit("reference checkout not found")
    ref_import._install_shims()
    sys.path.insert(0, ref_import.REF)
    from PIL import Image
    from torchvision import transforms
    import datasets.rand_augment as ra
    import datasets.transforms as rt
    from datasets.dataset import AugMixDataset
    from datasets.loader import fast_collate
    from datasets.transforms_factory import transforms_imagenet_train
    from loss.jsd import JsdCrossEntropy

    rec = {}
    orig_get_params = rt.RandomResizedCropAndInterpolation.get_params
    orig_cj_params = transforms.ColorJitter.get_params
    orig_ops = dict(ra.NAME_TO_OP)
    ops_names = list(ra._RAND_TRANSFORMS)

    def get_params(img, scale, ratio):
        p = orig_get_params(img, scale, ratio)
        rec["crop"].append(p)
        return p

    def cj_params(*a):
        p = orig_cj_params(*a)
        rec["views"][-1].append(p)
        return p

    def wrap(name):
        f = orig_ops[name]

        def g(img, *args, **kw):
            rec["views"][-1].append((ops_names.index(name), args[0] if args else 0.0))
            return f(img, *args, **kw)
        return g

    rt.RandomResizedCropAndInterpolation.get_params = staticmethod(get_params)
    transforms.ColorJitter.get_params = staticmethod(cj_params)
    for name in ops_names:
        ra.NAME_TO_OP[name] = wrap(name)

    def recording(t, key):                                       # a flip returns its input object when it does not flip
        def f(img):
            out = t(img)
            rec[key].append(out is not img)
            return out
        return f

    class Images:
        def __init__(self, imgs, labels):
            self.imgs, self.labels, self.transform = imgs, labels, None

        def __getitem__(self, i):
            return self.transform(self.imgs[i]), self.labels[i]

        def __len__(self):
            return len(self.imgs)

    def build(S, aa, vflip, imgs, labels):
        primary, secondary, final = transforms_imagenet_train(SIZE, interpolation="bicubic", use_prefetcher=True, vflip=vflip,
                                                              auto_augment=aa, color_jitter=0.4, separate=True)
        primary.transforms[1] = recording(primary.transforms[1], "flip")
        if vflip > 0:
            primary.transforms[2] = recording(primary.transforms[2], "vflip")

        def sec(img):
            rec["views"].append([])
            return secondary(img)
        ds = AugMixDataset(Images(imgs, labels), num_splits=S)
        ds.transform = (primary, sec, final)
        return ds

    def run(ds, seed):
        for k in ("crop", "flip", "vflip", "views"):
            rec[k] = []
        seed_all(seed)
        x, y = fast_collate([ds[i] for i in range(len(ds))])
        return x.numpy(), y.numpy()

    g = {"d_sizes": np.array([draw_size(s) for s in range(DRAW_N)], np.int32)}
    d_imgs = [Image.fromarray(source_image(600 + s, int(H), int(W))) for s, (H, W) in enumerate(g["d_sizes"])]
    d_labels = [int(v) for v in np.random.RandomState(1).randint(0, 1000, DRAW_N)]
    o_imgs = [Image.fromarray(source_image(700 + k, H, W)) for k, (H, W) in enumerate(OUT_SIZES)]
    for ci, (name, (S, aa, vflip)) in enumerate(CASES.items()):
        seed = 8000 + ci
        _, y = run(build(S, aa, vflip, d_imgs, d_labels), seed)
        nxt = (random.random(), np.random.random_sample(), float(torch.rand(1)))
        g["d_%s_seed" % name] = np.array([seed], np.int64)
        g["d_%s_crop" % name] = np.array(rec["crop"], np.int32)
        g["d_%s_flip" % name] = np.array(rec["flip"], np.int32)
        g["d_%s_vflip" % name] = np.array(rec["vflip"] or [0] * DRAW_N, np.int32)
        assert len(rec["views"]) == DRAW_N * (S - 1)
        if aa:
            g["d_%s_ids" % name] = np.array([[o[0] for o in v] + [-1] * (2 - len(v)) for v in rec["views"]], np.int32)
            g["d_%s_args" % name] = np.array([[float(o[1]) for o in v] + [0.0] * (2 - len(v)) for v in rec["views"]], np.float64)
        else:
            g["d_%s_perm" % name] = np.array([[int(k) for k in v[0][0]] for v in rec["views"]], np.int32)
            g["d_%s_factors" % name] = np.array([[math.nan if f is None else f for f in v[0][1:]] for v in rec["views"]], np.float64)
        g["d_%s_next" % name] = np.array(nxt, np.float64)
        g["d_%s_labels" % name] = y.astype(np.int64)
        x, _ = run(build(S, aa, vflip, o_imgs, [3, 5]), seed + 100)
        g["o_%s" % name] = x.reshape(-1, SIZE, SIZE)
        g["o_%s_meta" % name] = np.array([seed + 100, len(o_imgs), SIZE], np.int64)
    g["o_src"] = np.array([(H, W, 700 + k) for k, (H, W) in enumerate(OUT_SIZES)], np.int32)

    for name, (S, smoothing, z, y) in jsd_cases().items():
        zt = torch.from_numpy(z).requires_grad_(True)
        loss = JsdCrossEntropy(num_splits=S, smoothing=smoothing)(zt, torch.from_numpy(y).long())
        loss.backward()
        g["jsd_%s_z" % name], g["jsd_%s_y" % name] = z, y.astype(np.int64)
        g["jsd_%s_loss" % name] = np.array([loss.item()], np.float64)
        g["jsd_%s_grad" % name] = zt.grad.numpy()
        g["jsd_%s_meta" % name] = np.array([S, smoothing], np.float64)
    assert np.isfinite(g["jsd_underflow_loss"]).all() and np.isnan(g["jsd_underflow_grad"]).any()
    np.savez_compressed(path, **{k: encode_golden(v) for k, v in g.items()})
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "augsplit.npz"))
