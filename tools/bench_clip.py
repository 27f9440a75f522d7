"""Cost of gradient clipping on the library's one-graph training step (bench.py's workload: CoTNet-50, bf16 weights, autocast,
channels_last, cuDNN deterministic).  Prints one JSON line.

    python tools/bench_clip.py [--model cotnet50] [--batch 256] [--res 224] [--steps 20] [--rounds 3] [--clip 1.0]

* graph: the TrainStep graph step time with clipping off and in each mode (norm / value / agc, solver.clip_grad = --clip; agc
  uses 0.01, the reference's default clip factor), the modes alternating within each round in one process.  Each measurement
  captures its own step and frees it before the next.
* kernels: per mode, the library's kernels of the optimizer pass (cotb200_prof_enable: CUDA events around each launch, eager,
  outside the timed graph window): ms per launch and GB/s of algorithmic bytes.
* the GPU name and power limit next to the numbers.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_recipe import gpu_info, timed  # noqa: E402
from cotnet_b200 import _lib, backbone, trainer  # noqa: E402

MODES = (None, "norm", "value", "agc")
KERNELS = ("opt_step", "grad_norm", "unit_norms", "multi_lerp")


def one_round(a, mode, x, lab, profile):
    dev = torch.device("cuda")
    torch.manual_seed(1234)
    model = backbone.MODELS[a.model](zero_init_last_bn=False).to(dev).to(memory_format=torch.channels_last).train()
    clip = dict(clip_grad=(0.01 if mode == "agc" else a.clip), clip_mode=mode) if mode else {}
    ts = trainer.TrainStep(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=0.9999, weights="bf16", **clip)
    ts.capture(x, lab, warmup=3)
    for _ in range(3):
        ts.step()
    ms = timed(ts.step, a.steps)
    kern = None
    if profile:
        torch.cuda.synchronize()
        _lib.prof_enable(True)
        for _ in range(a.steps):
            ts.optimizer_step()
        rep = _lib.prof_report()
        _lib.prof_enable(False)
        kern = {k: {"launches_per_step": v[0] / a.steps, "ms_per_step": v[1] / a.steps,
                    "GB_per_s": (v[2] / 1e9) / (v[1] / 1e3) if v[1] > 0 else None}
                for k, v in rep.items() if k in KERNELS}
    norm = None if ts.grad_norm is None else float(ts.grad_norm.item())
    del ts, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms, kern, norm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--clip", type=float, default=1.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip.py: no CUDA device")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(a.batch, 3, a.res, a.res, generator=gen).to(torch.bfloat16).cuda().contiguous(memory_format=torch.channels_last)
    lab = torch.randint(0, 1000, (a.batch,), generator=gen).cuda()
    times = {str(m): [] for m in MODES}
    kernels, norms = {}, {}
    for r in range(a.rounds):
        for mode in MODES:
            ms, kern, norm = one_round(a, mode, x, lab, profile=(r == a.rounds - 1))
            times[str(mode)].append(ms)
            if kern is not None:
                kernels[str(mode)] = kern
            if norm is not None:
                norms[str(mode)] = norm
    name, limit = gpu_info()
    best = {k: min(v) for k, v in times.items()}
    print(json.dumps({"model": a.model, "batch": a.batch, "res": a.res, "gpu": name, "power_limit": limit, "clip": a.clip,
                      "agc_clip": 0.01, "graph_ms_per_step": times, "best_ms_per_step": best,
                      "overhead_pct": {k: 100.0 * (v - best["None"]) / best["None"] for k, v in best.items() if k != "None"},
                      "optimizer_kernels": kernels, "grad_norm_last_step": norms}))


if __name__ == "__main__":
    main()
