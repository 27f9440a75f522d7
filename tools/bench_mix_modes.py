"""Cost of per-sample Mixup / CutMix (MixupCutmix mode 'elem') against batch mixing.  Prints one JSON line.

    python tools/bench_mix_modes.py [--model cotnet50] [--batch 256] [--res 224] [--launches 200] [--steps 20] [--rounds 3]

* kernel: normalize_u8 of a uint8 3 x res^2 batch to bf16 with a batch draw (cotb200_u8_mix_to_nhwc) and with an 'elem' row table
  (cotb200_u8_mix_rows_to_nhwc), CUDA events over --launches launches, the two alternating in 5 rounds; bytes/s from the bytes
  the kernel must move (two uint8 reads and one bf16 write per element; the row reads are not counted).
* graph: the TrainStep graph step time (bench.py's workload: bf16 weights, autocast, channels_last, cuDNN deterministic, label
  smoothing 0.1) with a new batch draw and with a new 'elem' table every step, in alternating rounds; each round captures its
  own step and frees it before the next.
* draw: host time of MixupCutmix.draw() per batch for each mode (device copy issued, not waited for).
* the GPU name and power limit next to the numbers.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cotnet_b200 import backbone, trainer  # noqa: E402
from tools.bench_recipe import MEAN, STD, gpu_info, timed  # noqa: E402


def kernel_times(a, u8):
    B, R = u8.shape[0], u8.shape[2]
    draws = {"batch": trainer.MixupCutmix(seed=0).draw(B, R, R), "elem": trainer.MixupCutmix(seed=0, mode="elem").draw(B, R, R)}
    times = {k: [] for k in draws}
    for k, d in draws.items():
        for _ in range(5):
            trainer.normalize_u8(u8, MEAN, STD, torch.bfloat16, mix=d)
    for _ in range(5):
        for k, d in draws.items():
            times[k].append(timed(lambda: trainer.normalize_u8(u8, MEAN, STD, torch.bfloat16, mix=d), a.launches))
    nbytes = u8.numel() * (2 + 2)
    return {k: {"ms": v, "best_ms": min(v), "gb_per_s": nbytes / (min(v) / 1e3) / 1e9} for k, v in times.items()}


def graph_round(a, mode, u8, lab):
    torch.manual_seed(1234)
    model = backbone.MODELS[a.model](zero_init_last_bn=False).cuda().to(memory_format=torch.channels_last).train()
    ts = trainer.TrainStep(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=0.9999, weights="bf16",
                           label_smoothing=0.1)
    B, R = u8.shape[0], u8.shape[2]
    mc = trainer.MixupCutmix(seed=0, mode=mode)
    mix = mc.draw(B, R, R)
    ts.capture(trainer.normalize_u8(u8, MEAN, STD, torch.bfloat16, mix=mix), lab, warmup=3, mix=mix)
    x, lab_s = ts.static_inputs
    mixes = [mc.draw(B, R, R) for _ in range(a.steps)]
    it = iter(range(10 ** 9))

    def step():
        ts.step(x, lab_s, mix=mixes[next(it) % a.steps])
    for _ in range(3):
        step()
    ms = timed(step, a.steps)
    del ts, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms


def draw_times(a):
    out = {}
    for mode in trainer.MIX_MODES:
        mc = trainer.MixupCutmix(seed=0, mode=mode)
        for _ in range(5):
            mc.draw(a.batch, a.res, a.res)
        t0 = time.perf_counter()
        for _ in range(100):
            mc.draw(a.batch, a.res, a.res)
        out[mode] = (time.perf_counter() - t0) * 1e3 / 100
    torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mix_modes.py: no CUDA device")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    gen = torch.Generator().manual_seed(1234)
    u8 = torch.randint(0, 256, (a.batch, 3, a.res, a.res), generator=gen, dtype=torch.uint8).cuda()
    lab = torch.randint(0, 1000, (a.batch,), generator=gen, dtype=torch.int64).cuda()
    kern = kernel_times(a, u8)
    graph = {"batch": [], "elem": []}
    for _ in range(a.rounds):
        for mode in graph:
            graph[mode].append(graph_round(a, mode, u8, lab))
    name, limit = gpu_info()
    print(json.dumps({"model": a.model, "batch": a.batch, "res": a.res, "gpu": name, "power_limit": limit,
                      "normalize_u8_bf16": kern, "graph_ms_per_step": graph,
                      "graph_elem_minus_batch_ms": min(graph["elem"]) - min(graph["batch"]),
                      "draw_ms_per_batch": draw_times(a)}))


if __name__ == "__main__":
    main()
