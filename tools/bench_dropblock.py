"""Cost of DropBlock on the library's one-graph training step (bench.py's workload: CoTNet-50, bf16 weights, autocast,
channels_last, cuDNN deterministic) and of its kernels.  Prints one JSON line.

    python tools/bench_dropblock.py [--model cotnet50] [--batch 256] [--res 224] [--steps 20] [--rounds 3] [--rate 0.1]

* graph: the TrainStep graph step time at drop_block_rate 0 (bench.py's step) and at --rate, in alternating rounds in one
  process; each round captures its own step and frees it before the next.
* kernels: cotb200_dropblock_mask and cotb200_dropblock_apply timed with CUDA events at every DropBlock site of the model at this
  batch and resolution (bf16), with GB/s from the byte model below.
* the GPU name and power limit, read in the same run, next to the numbers.

Byte model (what each kernel must move, per site of n = B*C*H*W elements): the mask kernel writes the n/8-byte keep mask (and
reads nothing but the key); apply reads x and the mask and writes y: 2*n*2 + n/8 bytes in bf16.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_recipe import MEAN, STD, gpu_info, timed  # noqa: E402
from cotnet_b200 import backbone, backbone_hybrid, dropblock, trainer  # noqa: E402

MODELS = dict(backbone.MODELS, **backbone_hybrid.MODELS)


def one_round(a, rate, host_u8, host_lab):
    dev = torch.device("cuda")
    torch.manual_seed(1234)
    model = MODELS[a.model](zero_init_last_bn=False, drop_block_rate=rate).to(dev).to(memory_format=torch.channels_last).train()
    ts = trainer.TrainStep(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=0.9999, weights="bf16")
    x = trainer.normalize_u8(host_u8.to(dev), MEAN, STD, torch.bfloat16)
    ts.capture(x, host_lab.to(dev), warmup=3)
    x, lab = ts.static_inputs

    def step():
        ts.step(x, lab)
    for _ in range(3):
        step()
    ms = timed(step, a.steps)
    del ts, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms


def site_shapes(a):
    """(C, H, W, DropBlock) of every site of the model at a.res, from one training forward at batch 2 with the sites recorded."""
    calls = []
    orig = dropblock.drop_block

    def rec(x, key, site, spec):
        calls.append((x.shape[1], x.shape[2], x.shape[3], spec))
        return orig(x, key, site, spec)
    orig_tail = dropblock.drop_block_res_relu

    def rec_tail(z, res, key, site, spec, drop_scale=None):
        calls.append((z.shape[1], z.shape[2], z.shape[3], spec))
        return orig_tail(z, res, key, site, spec, drop_scale)
    dropblock.drop_block, dropblock.drop_block_res_relu = rec, rec_tail
    try:
        m = MODELS[a.model](drop_block_rate=a.rate).cuda().to(memory_format=torch.channels_last).train()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            m(torch.randn(2, 3, a.res, a.res, device="cuda").contiguous(memory_format=torch.channels_last))
    finally:
        dropblock.drop_block, dropblock.drop_block_res_relu = orig, orig_tail
    del m
    return calls


def kernel_times(a):
    key = torch.tensor([1, 2], dtype=torch.int64, device="cuda")
    mask_ms = apply_ms = mask_bytes = apply_bytes = 0.0
    for site, (C, H, W, spec) in enumerate(site_shapes(a)):
        x = torch.randn(a.batch, C, H, W, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        n = x.numel()
        m, cnt = dropblock.device_mask(x, key, site, spec)
        mask_ms += timed(lambda: dropblock.device_mask(x, key, site, spec), a.steps)
        apply_ms += timed(lambda: dropblock.DropBlockFn.apply(x, m, cnt), a.steps)
        mask_bytes += n / 8
        apply_bytes += 2 * n * x.element_size() + n / 8
    return dict(sites=site + 1, mask_ms=mask_ms, mask_gbps=mask_bytes / mask_ms / 1e6, apply_ms=apply_ms,
                apply_gbps=apply_bytes / apply_ms / 1e6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rate", type=float, default=0.1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dropblock.py: no CUDA device")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    gen = torch.Generator().manual_seed(1234)
    host_u8 = torch.randint(0, 256, (a.batch, 3, a.res, a.res), generator=gen, dtype=torch.uint8).pin_memory()
    host_lab = torch.randint(0, 1000, (a.batch,), generator=gen, dtype=torch.int64).pin_memory()
    off, on = [], []
    for _ in range(a.rounds):
        off.append(one_round(a, 0., host_u8, host_lab))
        on.append(one_round(a, a.rate, host_u8, host_lab))
    kern = kernel_times(a)
    name, limit = gpu_info()
    best_off, best_on = min(off), min(on)
    print(json.dumps({"model": a.model, "batch": a.batch, "res": a.res, "rate": a.rate, "gpu": name, "power_limit": limit,
                      "graph_ms_per_step_rate0": off, "graph_ms_per_step_rate": on,
                      "dropblock_overhead_ms": best_on - best_off, "dropblock_overhead_pct": 100.0 * (best_on - best_off) / best_off,
                      "kernels_per_step_bf16": kern}))


if __name__ == "__main__":
    main()
