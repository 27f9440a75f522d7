"""GPU time of the augmentation kernels per batch, against Pillow on one CPU core.  Prints one JSON line per measurement with
the GPU name and power limit beside the numbers.

    python tools/bench_augment.py [--batch 256] [--iters 20] [--cpu-images 64]

* train / eval: cotb200_aug_resize_crop (+ cotb200_aug_randaug for train) on a ragged batch with a fixed ImageNet-like size mix
  (seeded), timed with CUDA events after warm-up; the host-to-device copy of the pinned ragged buffer and structs is timed
  separately (bytes listed).
* cpu: the same crop / resize / flip / RandAugment draws applied with Pillow (the operations the reference's transforms call),
  single process, ms per image.  This is not the reference's own transform object, which is not part of this repository.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cotnet_b200 import augment  # noqa: E402
from oracle import aug_ref  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def sizes(r, n):
    out = []
    for _ in range(n):
        u = r.rand()
        if u < 0.7:
            H, W = (375, 500) if r.rand() < 0.7 else (500, 375)
            out.append((H + int(r.randint(-40, 41)), W + int(r.randint(-40, 41))))
        elif u < 0.9:
            out.append(tuple(int(v) for v in r.randint(200, 400, 2)))
        else:
            out.append(tuple(int(v) for v in r.randint(600, 1000, 2)))
    return out


def pil_ms_per_image(imgs, draws, S=224):
    from PIL import Image, ImageEnhance, ImageOps
    pil = [Image.fromarray(a) for a in imgs]
    t0 = time.perf_counter()
    for p, d in zip(pil, draws):
        im = p.crop((d["j"], d["i"], d["j"] + d["w"], d["i"] + d["h"])).resize((S, S), Image.BICUBIC)
        if d["flip"]:
            im = im.transpose(Image.FLIP_LEFT_RIGHT)
        for op in d["ops"]:
            if op is None:
                continue
            i = op["id"]
            if i in augment.AFFINE_OPS:
                im = im.transform(im.size, Image.AFFINE, tuple(op["matrix"]), resample=Image.BICUBIC, fillcolor=aug_ref.FILL)
            elif i == 0:
                im = ImageOps.autocontrast(im)
            elif i == 1:
                im = ImageOps.equalize(im)
            elif i in (2, 4, 5, 6):
                im = im.point(list(range(256)) * 3)
            elif i in (7, 8, 9, 10):
                im = (ImageEnhance.Color, ImageEnhance.Contrast, ImageEnhance.Brightness, ImageEnhance.Sharpness)[i - 7](im).enhance(op["factor"])
        np.asarray(im)
    return (time.perf_counter() - t0) * 1e3 / len(pil)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu-images", type=int, default=64)
    a = ap.parse_args()
    name, power = gpu_info()
    r = np.random.RandomState(0)
    sz = sizes(r, a.batch)
    imgs = [aug_ref.source_image(k, H, W) for k, (H, W) in enumerate(sz)]
    tf, ev = augment.TrainAugment(), augment.EvalTransform()
    draws = tf.draw(sz, random.Random(0), np.random.RandomState(0), torch.Generator().manual_seed(0))
    data = torch.from_numpy(np.concatenate([x.reshape(-1) for x in imgs])).pin_memory()
    labels = torch.zeros(a.batch, dtype=torch.int64)
    batches = {"train": augment.AugBatch(data, torch.from_numpy(tf.pack(sz, draws).view(np.uint8).copy()).pin_memory(), labels),
               "eval": augment.AugBatch(data, torch.from_numpy(ev.pack(sz).view(np.uint8).copy()).pin_memory(), labels)}
    dev = torch.device("cuda", 0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    # host -> device copy of the ragged buffer
    for _ in range(3):
        data.to(dev, non_blocking=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(a.iters):
        data.to(dev, non_blocking=True)
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps(dict(what="h2d", batch=a.batch, bytes=int(data.numel()), ms=e0.elapsed_time(e1) / a.iters, gpu=name,
                          power_limit=power)), flush=True)
    for kind, b in batches.items():
        dd = augment.AugBatch(b.data.to(dev), b.params, b.labels)          # device-resident source: kernels only
        for _ in range(3):
            augment.run(dd, 224, dev, randaug=kind == "train")
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.iters):
            augment.run(dd, 224, dev, randaug=kind == "train")
        e1.record()
        torch.cuda.synchronize()
        print(json.dumps(dict(what=kind, batch=a.batch, gpu_ms_per_batch=e0.elapsed_time(e1) / a.iters,
                              src_bytes=int(data.numel()), gpu=name, power_limit=power)), flush=True)
    try:
        n = min(a.cpu_images, a.batch)
        print(json.dumps(dict(what="cpu_pil_train", images=n, ms_per_image=pil_ms_per_image(imgs[:n], draws[:n]),
                              note="one process, Pillow calls of the same draws")), flush=True)
    except ImportError:
        print(json.dumps(dict(what="cpu_pil_train", note="Pillow not installed: not measured")), flush=True)


if __name__ == "__main__":
    main()
