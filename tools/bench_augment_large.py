"""GPU TrainAugment throughput above 256 x 256: the thread-block-cluster kernels at 288 and 320 against the one-CTA kernels at
224, on the same draws over the same ImageNet-like source sizes.  Prints one JSON line per case with the GPU name and power
limit read in the same run.

    python tools/bench_augment_large.py [--batch 64] [--iters 30]

Cases (the draws of TrainAugment(size=S), default rand-m15-mstd0.5-n2; and ColorJitter 0.4 + vflip 0.5 without RandAugment):
  224      one CTA per image (cotb200_aug_randaug / cotb200_aug_color_jitter);
  224c     the cluster kernels forced at 224 (one CTA per cluster there), for comparison with the line above;
  288, 320 the cluster kernels (2 CTAs per image).
Each line gives the whole augment.run() per batch (the source already on the device: resize-crop + colour kernel) as
images/s, timed with CUDA events after warm-up, and the colour kernel's own time per batch from the library's profiler,
taken in a separate pass.
"""
import argparse
import json
import os
import random
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cotnet_b200 import _lib, augment  # noqa: E402
from oracle import aug_ref  # noqa: E402
from tools.bench_augment import gpu_info, sizes  # noqa: E402

CASES = (("224", 224, False), ("224c", 224, True), ("288", 288, True), ("320", 320, True))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_augment_large: no CUDA device")
    name, power = gpu_info()
    dev = torch.device("cuda", 0)
    r = np.random.RandomState(0)
    sz = sizes(r, a.batch)
    imgs = [aug_ref.source_image(k, H, W) for k, (H, W) in enumerate(sz)]
    data = torch.from_numpy(np.concatenate([x.reshape(-1) for x in imgs])).to(dev)
    labels = torch.zeros(a.batch, dtype=torch.int64)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for transform in ("randaug", "jitter"):
        for case, S, cluster in CASES:
            kw = {} if transform == "randaug" else dict(auto_augment=None, color_jitter=0.4, vflip=0.5)
            tf = augment.TrainAugment(size=S, **kw)
            draws = tf.draw(sz, random.Random(0), np.random.RandomState(0), torch.Generator().manual_seed(0))
            jit = torch.from_numpy(tf.pack_jitter(draws).view(np.uint8).copy()) if tf.has_jitter_kernel else None
            b = augment.AugBatch(data, torch.from_numpy(tf.pack(sz, draws).view(np.uint8).copy()), labels, jit)

            def step():
                augment.run(b, S, dev, randaug=tf.num_layers > 0, cluster=cluster)
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.iters):
                step()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.iters
            _lib.prof_enable(True)
            try:
                for _ in range(a.iters):
                    step()
                torch.cuda.synchronize()
                rep = _lib.prof_report()
            finally:
                _lib.prof_enable(False)
            kern = {k: v[1] / a.iters for k, v in rep.items()}
            colour = {k: round(v, 4) for k, v in kern.items() if k not in ("aug_hpass", "aug_vpass")}
            print(json.dumps(dict(transform=transform, case=case, S=S, cluster=cluster, batch=a.batch, ms_per_batch=round(ms, 4),
                                  images_per_s=round(a.batch / ms * 1e3, 1), colour_kernel_ms=colour,
                                  resize_ms=round(kern.get("aug_hpass", 0.0) + kern.get("aug_vpass", 0.0), 4), gpu=name,
                                  power_limit=power)), flush=True)


if __name__ == "__main__":
    main()
