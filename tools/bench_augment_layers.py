"""GPU time of TrainAugment per batch against its number of RandAugment layers: n = 2, 3 and 4 (one, two and two RandAugment
launches) at 224 (one CTA per image) and 320 (thread-block clusters), for batches of 64 and 256 images.  Prints one JSON line
per case with the GPU name and power limit read in the same run.

    python tools/bench_augment_layers.py [--iters 20] [--rounds 3]

Each case is TrainAugment(size=S, auto_augment='rand-m15-mstd0.5-n<n>') on the same ImageNet-like source sizes, with the
source already on the device: augment.run() as TrainAugment calls it (struct copy, resize-crop, the RandAugment passes).
The cases alternate: each round times every case once (CUDA events over `iters` batches after warm-up), and a line gives the
median and the range of the rounds.  The RandAugment kernels' own time per batch comes from the library's profiler, in a
separate pass after the timed rounds.
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

LAYERS = (2, 3, 4)
SIZES = (224, 320)
BATCHES = (64, 256)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_augment_layers: no CUDA device")
    name, power = gpu_info()
    dev = torch.device("cuda", 0)
    r = np.random.RandomState(0)
    sz = sizes(r, max(BATCHES))
    imgs = [aug_ref.source_image(k, H, W) for k, (H, W) in enumerate(sz)]
    cases = []
    for B in BATCHES:
        data = torch.from_numpy(np.concatenate([x.reshape(-1) for x in imgs[:B]])).to(dev)
        for S in SIZES:
            for n in LAYERS:
                tf = augment.TrainAugment(size=S, auto_augment="rand-m15-mstd0.5-n%d" % n)
                draws = tf.draw(sz[:B], random.Random(0), np.random.RandomState(0), torch.Generator().manual_seed(0))
                b = tf.collate_draws(imgs[:B], [0] * B, draws)._replace(data=data)      # the source stays on the device

                def step(b=b, S=S, tf=tf):
                    augment.run(b, S, dev, randaug=True, passes=tf.passes)
                cases.append(dict(batch=B, S=S, layers=n, passes=tf.passes, step=step, ms=[]))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for c in cases:
        for _ in range(3):
            c["step"]()
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for c in cases:
            e0.record()
            for _ in range(a.iters):
                c["step"]()
            e1.record()
            torch.cuda.synchronize()
            c["ms"].append(e0.elapsed_time(e1) / a.iters)
    for c in cases:
        _lib.prof_enable(True)
        try:
            for _ in range(a.iters):
                c["step"]()
            torch.cuda.synchronize()
            rep = _lib.prof_report()
        finally:
            _lib.prof_enable(False)
        kern = {k: v for k, v in rep.items() if k.startswith("aug_randaug")}
        ms = sorted(c["ms"])
        print(json.dumps(dict(batch=c["batch"], S=c["S"], layers=c["layers"], randaug_launches=c["passes"],
                              ms_per_batch=round(float(np.median(ms)), 4), ms_range=[round(ms[0], 4), round(ms[-1], 4)],
                              images_per_s=round(c["batch"] / float(np.median(ms)) * 1e3, 1),
                              randaug_kernel_ms={k: round(v[1] / a.iters, 4) for k, v in kern.items()},
                              launches_per_batch={k: v[0] // a.iters for k, v in kern.items()}, gpu=name,
                              power_limit=power)), flush=True)


if __name__ == "__main__":
    main()
