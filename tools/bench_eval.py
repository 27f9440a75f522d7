"""Validation throughput (images/s) of the library's eval graph against the reference-style eager loop.  Prints one JSON line
per (model, batch) and the GPU name and power limit beside the numbers.

    python tools/bench_eval.py [--models cotnet50,se_cotnetd_50] [--batches 128,256] [--res 224] [--steps 20] [--rounds 3]

* graph: EvalStep's live graph (eval-mode forward under bf16 autocast, channels_last, top-1/top-5 counted on the device by
  cotb200_topk_hits), one replay per batch, no host synchronisation until the end of the window.
* eager: what evaler/evaler.py:37-57 does per batch -- model.eval(), no_grad, autocast, utils/meters.py accuracy()
  (output.topk(5) + eq), then torch.cuda.synchronize().  The forward itself runs on the same library kernels; only the loop
  around it differs.
The two are timed in alternating rounds in one process (CUDA events around `steps` batches after warm-up); the median round
is reported.  Inputs are seeded normalised batches that already sit on the device (decoding and the transform are not timed).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cotnet_b200 import backbone, backbone_hybrid, evaler  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(), "unknown"


def timed(fn, steps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def accuracy(output, target, topk=(1,)):
    """utils/meters.py:12-19."""
    _, pred = output.topk(max(topk), 1, True, True)
    pred = pred.t()
    correct = pred.eq(target.reshape(1, -1).expand_as(pred))
    return [correct[:k].reshape(-1).float().sum(0) * 1.0 for k in topk]


def bench(name, batch, a):
    dev = torch.device("cuda")
    ctor = backbone.MODELS.get(name) or backbone_hybrid.MODELS[name]
    torch.manual_seed(1234)
    model = ctor(zero_init_last_bn=False).to(dev).to(memory_format=torch.channels_last).eval()
    gen = torch.Generator(device=dev).manual_seed(7)
    xs = [torch.randn(batch, 3, a.res, a.res, device=dev, generator=gen).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
          for _ in range(2)]
    ys = [torch.randint(0, 1000, (batch,), device=dev, generator=gen) for _ in range(2)]
    ev = evaler.EvalStep(model, batch, a.res, topk=(1, 5))
    ev.capture()
    acc = [torch.zeros((), device=dev), torch.zeros((), device=dev)]

    def graph_step(i):
        ev.run(xs[i & 1], ys[i & 1])

    def eager_step(i):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(xs[i & 1])
        t1, t5 = accuracy(out, ys[i & 1], topk=(1, 5))
        acc[0] += t1
        acc[1] += t5
        torch.cuda.synchronize()

    for _ in range(a.warmup):
        graph_step(0)
        eager_step(0)
    g_ms, e_ms = [], []
    for _ in range(a.rounds):
        g_ms.append(timed(graph_step, a.steps))
        e_ms.append(timed(eager_step, a.steps))
    # reported, not asserted: the hits of one batch by both loops (they agree unless a label logit is tied)
    r = ev.result()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        out = model(xs[0])
    same = [int(v) for v in accuracy(out, ys[0], topk=(1, 5))]
    ev.run(xs[0], ys[0])
    r1 = ev.result()
    gm, em = statistics.median(g_ms), statistics.median(e_ms)
    res = {"model": name, "batch": batch, "res": a.res, "amp": "bf16", "steps": a.steps, "rounds": a.rounds,
           "graph_ms_per_batch": g_ms, "eager_ms_per_batch": e_ms,
           "graph_images_per_s": batch / (gm / 1e3), "eager_images_per_s": batch / (em / 1e3), "speedup": em / gm,
           "graph_n_counted": r["n"], "hits_graph_vs_eager": [[round(r1["top1"] * batch / 100), round(r1["top5"] * batch / 100)], same]}
    del ev, model, xs
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="cotnet50,se_cotnetd_50")
    ap.add_argument("--batches", default="128,256")
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py: no CUDA device")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    name, limit = gpu_info()
    for m in a.models.split(","):
        for b in a.batches.split(","):
            res = bench(m, int(b), a)
            res.update(gpu=name, power_limit=limit)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
