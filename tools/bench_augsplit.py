"""GPU cost of the augmentation splits and of the JSD loss beside what they replace.  Prints one JSON line per measurement with
the GPU name and power limit beside the numbers.

    python tools/bench_augsplit.py [--batch 64] [--splits 3] [--model cotnet50] [--steps 20] [--rounds 3] [--iters 50]

* augment: the GPU part of TrainAugment (H2D copies, resize-crop, flips, the split copies, RandAugment) on `batch` images of
  ImageNet-like sizes with rand-m15-mstd0.5-n2, with num_splits=splits, against num_splits=0 on `batch` and on splits * batch
  images; CUDA events around `iters` calls after warm-up.
* loss: cotb200_jsd_ce + cotb200_jsd_ce_bwd (trainer.jsd_cross_entropy, forward and backward) on [splits * batch, 1000] bf16
  logits, against the same loss written as torch ops (loss/jsd.py's formula) on the same GPU.
* step: the TrainStep graph step (bench.py's workload: bf16 weights, autocast, channels_last, cuDNN deterministic) with
  jsd_splits=splits on splits * batch images, against label smoothing 0.1 on the same total batch, alternated over `rounds`.
"""
import argparse
import json
import os
import random
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cotnet_b200 import augment, backbone, trainer  # noqa: E402
from tools.bench_augment import gpu_info  # noqa: E402
from tools.bench_jitter_erase import timed  # noqa: E402


def torch_jsd(out, y, S, smoothing=0.1, alpha=12.0):
    B = out.shape[0] // S
    splits = torch.split(out.float(), B)
    lp = F.log_softmax(splits[0], dim=-1)
    ce = ((1 - smoothing) * -lp.gather(1, y[:B, None])[:, 0] + smoothing * -lp.mean(-1)).mean()
    probs = [F.softmax(z, dim=1) for z in splits]
    logm = torch.clamp(torch.stack(probs).mean(0), 1e-7, 1).log()
    return ce + alpha * sum(F.kl_div(logm, p, reduction="batchmean") for p in probs) / S


def bench_augment(a, name, power):
    r = np.random.RandomState(0)
    imgs = [r.randint(0, 256, (int(r.randint(300, 500)), int(r.randint(300, 500)), 3)).astype(np.uint8)
            for _ in range(a.batch * a.splits)]
    for splits, n in ((a.splits, a.batch), (0, a.batch), (0, a.batch * a.splits)):
        tf = augment.TrainAugment(num_splits=splits)
        sizes = [im.shape[:2] for im in imgs[:n]]
        draws = tf.draw(sizes, random.Random(1), np.random.RandomState(1), torch.Generator().manual_seed(1))
        b = tf.collate_draws(imgs[:n], list(range(n)), draws)
        b = augment.AugBatch(*(t.pin_memory() if t is not None else None for t in b))
        ms = timed(lambda: tf(b), a.iters)
        print(json.dumps(dict(bench="augment", num_splits=splits, images=n, rows=n * max(1, splits), gpu_ms_per_batch=ms, gpu=name,
                              power_limit=power)), flush=True)


def bench_loss(a, name, power):
    N, S = a.batch * a.splits, a.splits
    g = torch.Generator(device="cuda").manual_seed(0)
    z = (torch.randn(N, 1000, generator=g, device="cuda") * 3).to(torch.bfloat16).requires_grad_(True)
    y = torch.randint(0, 1000, (a.batch,), generator=g, device="cuda").repeat(S)

    def lib():
        trainer.jsd_cross_entropy(z, y, S, 0.1).backward()

    def ops():
        torch_jsd(z, y, S).backward()
    for kind, fn in (("cotb200_jsd_ce", lib), ("torch_ops", ops)):
        ms = timed(fn, a.iters)
        print(json.dumps(dict(bench="loss", impl=kind, shape=[N, 1000], dtype="bf16", gpu_ms_fwd_bwd=ms, gpu=name, power_limit=power)),
              flush=True)


def one_step(a, x, lab, jsd):
    torch.manual_seed(1234)
    model = backbone.MODELS[a.model](zero_init_last_bn=False).cuda().to(memory_format=torch.channels_last).train()
    ts = trainer.TrainStep(model, lr=0.05, momentum=0.9, weight_decay=1e-4, ema_decay=0.9999, weights="bf16", label_smoothing=0.1,
                           jsd_splits=a.splits if jsd else 0)
    info = ts.capture(x, lab, warmup=3)
    for _ in range(3):
        ts.step()
    ms = timed(ts.step, a.steps, warmup=0)
    del ts, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms, info["libcotb200_kernels_per_replay"]


def bench_step(a, name, power):
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    N = a.batch * a.splits
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(N, 3, 224, 224, generator=gen).to(torch.bfloat16).cuda().contiguous(memory_format=torch.channels_last)
    lab = torch.randint(0, 1000, (a.batch,), generator=gen).repeat(a.splits).cuda()
    times, launches = {"jsd": [], "label_smoothing": []}, {}
    for _ in range(a.rounds):
        for k in times:
            ms, n = one_step(a, x, lab, k == "jsd")
            times[k].append(ms)
            launches[k] = n
    print(json.dumps(dict(bench="step", model=a.model, batch=N, splits=a.splits, graph_ms_per_step=times,
                          best_ms_per_step={k: min(v) for k, v in times.items()}, libcotb200_kernels_per_replay=launches, gpu=name,
                          power_limit=power)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--splits", type=int, default=3)
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_augsplit.py: no CUDA device")
    name, power = gpu_info()
    bench_augment(a, name, power)
    bench_loss(a, name, power)
    bench_step(a, name, power)


if __name__ == "__main__":
    main()
