"""Cost of the reference training recipe on the library's one-graph training step (bench.py's workload: CoTNet-50, bf16
weights, autocast, channels_last, cuDNN deterministic).  Prints one JSON line.

    python tools/bench_recipe.py [--model cotnet50] [--batch 256] [--res 224] [--steps 20] [--rounds 2]

* graph: the TrainStep graph step time with the recipe OFF (bench.py's step) and ON -- drop_path_rate 0.1, drop_rate 0.25,
  Mixup 0.8 / CutMix 1.0 batch mixing with a new draw every step, label smoothing 0.1 (the reference configs) -- measured in
  alternating rounds in one process.  Each round captures its own step and frees it before the next.
* e2e: the recipe step with the input path of every step: pinned uint8 batch -> H2D -> normalize_u8(mix=) -> step -> loss read back.
* the GPU name and power limit next to the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cotnet_b200 import backbone, trainer  # noqa: E402

MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


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
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def one_round(a, recipe, host_u8, host_lab, e2e):
    dev = torch.device("cuda")
    torch.manual_seed(1234)
    kw = dict(drop_rate=0.25, drop_path_rate=0.1) if recipe else {}
    model = backbone.MODELS[a.model](zero_init_last_bn=False, **kw).to(dev).to(memory_format=torch.channels_last).train()
    ts = trainer.TrainStep(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=0.9999, weights="bf16",
                           label_smoothing=0.1 if recipe else 0.)
    mc = trainer.MixupCutmix(0.8, 1.0, prob=1.0, switch_prob=0.5, label_smoothing=0.1, seed=0) if recipe else None
    B, R = host_u8.shape[0], host_u8.shape[2]

    def batch():
        u8, lab = host_u8.to(dev, non_blocking=True), host_lab.to(dev, non_blocking=True)
        mix = mc.draw(B, R, R) if recipe else None
        return trainer.normalize_u8(u8, MEAN, STD, torch.bfloat16, mix=mix), lab, mix

    x, lab, mix = batch()
    ts.capture(x, lab, warmup=3, mix=mix)
    x, lab = ts.static_inputs
    mixes = [mc.draw(B, R, R) for _ in range(a.steps)] if recipe else None
    it = iter(range(10 ** 9))

    def step():
        ts.step(x, lab, mix=mixes[next(it) % a.steps] if recipe else None)
    for _ in range(3):
        step()
    ms = timed(step, a.steps)
    ms_e2e = None
    if e2e:
        def e2e_step():
            xb, lb, mb = batch()
            return float(ts.step(xb, lb, mix=mb).item())
        for _ in range(2):
            e2e_step()
        ms_e2e = timed(e2e_step, a.steps)
    del ts, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms, ms_e2e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_recipe.py: no CUDA device")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    gen = torch.Generator().manual_seed(1234)
    host_u8 = torch.randint(0, 256, (a.batch, 3, a.res, a.res), generator=gen, dtype=torch.uint8).pin_memory()
    host_lab = torch.randint(0, 1000, (a.batch,), generator=gen, dtype=torch.int64).pin_memory()
    off, on, e2e = [], [], []
    for r in range(a.rounds):
        off.append(one_round(a, False, host_u8, host_lab, False)[0])
        ms, ms_e = one_round(a, True, host_u8, host_lab, r == a.rounds - 1)
        on.append(ms)
        if ms_e is not None:
            e2e.append(ms_e)
    name, limit = gpu_info()
    best_off, best_on = min(off), min(on)
    print(json.dumps({"model": a.model, "batch": a.batch, "res": a.res, "gpu": name, "power_limit": limit,
                      "graph_ms_per_step_recipe_off": off, "graph_ms_per_step_recipe_on": on,
                      "recipe_overhead_pct": 100.0 * (best_on - best_off) / best_off,
                      "images_per_s_off": a.batch / (best_off / 1e3), "images_per_s_on": a.batch / (best_on / 1e3),
                      "e2e_ms_per_step_recipe_on": e2e, "e2e_images_per_s_recipe_on": a.batch / (min(e2e) / 1e3) if e2e else None}))


if __name__ == "__main__":
    main()
