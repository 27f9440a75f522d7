"""Cost of virtual ranks on the library's one-graph training step (bench.py's workload: CoTNet-50, bf16 weights and bucket, autocast,
channels_last, cuDNN deterministic).  Prints one JSON line.

    python tools/bench_virtual_ranks.py [--model cotnet50] [--res 224] [--steps 10] [--rounds 2]

* graph: the captured step of bench.py's bs256 and of TrainStep(virtual_ranks=K) over micro-batches of 80 (K = 8 is the
  CoTNet-50 recipe's eight ranks of 80, K = 4 half of it), the configurations alternating within each round in one process.
  Each measurement builds and captures its own step and frees it before the next.  Per configuration: ms per step, images per
  second and torch.cuda.max_memory_allocated.
* kernels: the accumulate and emit passes of cotb200_multi_gather_acc in eager steps of the K = 8 configuration
  (cotb200_prof_enable: CUDA events around each launch, outside the timed graph window): ms per launch and GB/s of the bytes the
  pass must move (gradient read + fp32 accumulator read + accumulator or bucket write, from the parameter shapes).
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

CONFIGS = ((1, 256), (8, 80), (4, 80))          # (virtual ranks, images per rank)


def _byte_model(ts):
    """Bytes one accumulate pass and one emit pass must move (bf16 gradients of the big bucket, fp32 of the small one)."""
    big = sum(p.numel() for _, p, _ in ts.plan["big"])
    small = sum(p.numel() for _, p, _ in ts.plan["small"])
    gb = 2 if ts.weights_bf16 else 4
    bucket = ts.G_big.element_size()
    acc = big * (gb + 4 + 4) + small * (4 + 4 + 4)
    emit = big * (gb + 4 + bucket) + small * (4 + 4 + 4)
    return acc, emit


def one_round(a, K, B, profile):
    dev = torch.device("cuda")
    torch.manual_seed(1234)
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(K * B, 3, a.res, a.res, generator=gen).to(torch.bfloat16).to(dev).contiguous(memory_format=torch.channels_last)
    lab = torch.randint(0, 1000, (K * B,), generator=gen).to(dev)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    model = backbone.MODELS[a.model](zero_init_last_bn=False).to(dev).to(memory_format=torch.channels_last).train()
    ts = trainer.TrainStep(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=0.9999, weights="bf16",
                           virtual_ranks=K)
    info = ts.capture(x, lab, warmup=3)
    for _ in range(3):
        ts.step()
    ms = timed(ts.step, a.steps)
    mem = torch.cuda.max_memory_allocated()
    kern = None
    if profile and K > 2:
        torch.cuda.synchronize()
        _lib.prof_enable(True)
        n = 2
        for _ in range(n):
            ts.step_eager(x, lab)
        rep = _lib.prof_report()
        _lib.prof_enable(False)
        acc_b, emit_b = _byte_model(ts)
        kern = {}
        for name, per_step_bytes in (("multi_gather_acc", acc_b * (K - 2)), ("multi_gather_emit", emit_b)):
            cnt, tot_ms, _ = rep.get(name, (0, 0.0, 0.0))
            kern[name] = {"launches_per_step": cnt / n, "ms_per_step": tot_ms / n, "bytes_per_step": per_step_bytes,
                          "GB_per_s": (per_step_bytes / 1e9) / (tot_ms / n / 1e3) if tot_ms > 0 else None}
    kpr = info["libcotb200_kernels_per_replay"]
    del ts, model, x, lab
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms, mem, kern, kpr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_virtual_ranks.py: no CUDA device")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    times = {"%dx%d" % c: [] for c in CONFIGS}
    mem, kpr, kernels = {}, {}, None
    for r in range(a.rounds):
        for K, B in CONFIGS:
            key = "%dx%d" % (K, B)
            ms, m, kern, n = one_round(a, K, B, profile=(r == a.rounds - 1))
            times[key].append(ms)
            mem[key] = max(mem.get(key, 0), m)
            kpr[key] = n
            if kern is not None and K == 8:
                kernels = kern
    name, limit = gpu_info()
    out = {}
    for K, B in CONFIGS:
        key = "%dx%d" % (K, B)
        best = min(times[key])
        out[key] = {"virtual_ranks": K, "images_per_rank": B, "ms_per_step": times[key], "best_ms_per_step": best,
                    "images_per_s": 1e3 * K * B / best, "max_memory_allocated_GB": mem[key] / 1e9,
                    "libcotb200_kernels_per_replay": kpr[key]}
    print(json.dumps({"model": a.model, "res": a.res, "steps": a.steps, "rounds": a.rounds, "gpu": name, "power_limit": limit,
                      "configs": out, "gather_acc_kernels_8x80": kernels}))


if __name__ == "__main__":
    main()
