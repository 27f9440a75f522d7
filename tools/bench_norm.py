#!/usr/bin/env python
"""Per-shape timing of the row-streaming kernels (BatchNorm / GroupNorm / tail / sum_rows) at every (pixels, channels)
shape the CoTNet-50 bs256 step launches them with.

    python tools/bench_norm.py [--batch 256] [--iters 20] [--json out.json]

CUDA-event timing, inputs rotated through > 126 MB so every launch streams from HBM; GB/s of ALGORITHMIC bytes
(the same per-launch byte counts the library's profiling records use) and the fraction of the measured HBM peak."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from cotnet_b200 import _lib  # noqa: E402

# (H=W, C) of every BatchNorm input of cotnet50 at 224^2 (stem, conv1/conv3/downsample, CoT-internal k/e/v/u)
SHAPES = [(112, 64), (56, 64), (56, 32), (56, 256), (56, 128), (28, 128), (28, 64), (28, 512), (28, 256), (14, 256), (14, 128),
          (14, 1024), (14, 512), (7, 512), (7, 256), (7, 2048)]


def peak():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 6650.0


def timeit(fn, nsets, iters):
    for i in range(3):
        fn(i % nsets)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i % nsets)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3     # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--shapes", default=None, help="comma list of HWxC, e.g. 56x256,7x2048 (default: all)")
    a = ap.parse_args()
    shapes = SHAPES if not a.shapes else [tuple(int(v) for v in s.split("x")) for s in a.shapes.split(",")]
    lib = _lib.load()
    dev = torch.device("cuda")
    pk = peak()
    st = torch.cuda.current_stream().cuda_stream
    B = a.batch
    out = []
    for HW, C in shapes:
        rows = B * HW * HW
        es = 2
        nbytes = rows * C * es
        nsets = max(2, int(400e6 // (3 * nbytes)) + 1)
        xs = [torch.randn(rows, C, device=dev).to(torch.bfloat16) for _ in range(nsets)]
        ys = [torch.relu(torch.randn(rows, C, device=dev)).to(torch.bfloat16) for _ in range(nsets)]
        ds = [torch.randn(rows, C, device=dev).to(torch.bfloat16) for _ in range(nsets)]
        o1 = torch.empty(rows, C, device=dev, dtype=torch.bfloat16)
        o2 = torch.empty(rows, C, device=dev, dtype=torch.bfloat16)
        f = torch.zeros(8, C, device=dev)
        f[3] = 1.0
        dt = 2
        rec = {"HW": HW, "C": C, "MB": nbytes / 1e6}

        def run(name, passes, fn):
            us = timeit(fn, nsets, a.iters)
            gbs = passes * nbytes / us / 1e3
            rec[name + "_us"] = round(us, 2)
            rec[name + "_frac"] = round(gbs / pk, 3)

        run("col_stats", 1, lambda i: _lib.check(lib.cotb200_col_stats(dt, 1, rows, C, xs[i].data_ptr(), f[0].data_ptr(), f[1].data_ptr(), st), "cs"))
        run("bn_apply", 2, lambda i: _lib.check(lib.cotb200_bn_apply(dt, 1, rows, C, xs[i].data_ptr(), None, f[3].data_ptr(), f[2].data_ptr(), 1, o1.data_ptr(), None, st), "ba"))
        run("bn_apply_res", 3, lambda i: _lib.check(lib.cotb200_bn_apply(dt, 1, rows, C, xs[i].data_ptr(), ds[i].data_ptr(), f[3].data_ptr(), f[2].data_ptr(), 1, o1.data_ptr(), None, st), "bar"))
        run("bn_bwd_sums", 3, lambda i: _lib.check(lib.cotb200_bn_bwd_sums(dt, 1, rows, C, ds[i].data_ptr(), xs[i].data_ptr(), ys[i].data_ptr(), None, f[3].data_ptr(), f[2].data_ptr(), f[2].data_ptr(), f[3].data_ptr(), 1, f[4].data_ptr(), f[5].data_ptr(), None, st), "bs"))
        run("bn_bwd_sums_xmask", 2, lambda i: _lib.check(lib.cotb200_bn_bwd_sums(dt, 1, rows, C, ds[i].data_ptr(), xs[i].data_ptr(), None, None, f[3].data_ptr(), f[2].data_ptr(), f[2].data_ptr(), f[3].data_ptr(), 2, f[4].data_ptr(), f[5].data_ptr(), None, st), "bsx"))
        run("bn_bwd_apply", 4, lambda i: _lib.check(lib.cotb200_bn_bwd_apply(dt, 1, rows, C, ds[i].data_ptr(), xs[i].data_ptr(), ys[i].data_ptr(), None, f[3].data_ptr(), f[2].data_ptr(), f[2].data_ptr(), f[3].data_ptr(), f[4].data_ptr(), f[5].data_ptr(), 1.0 / rows, 1, o1.data_ptr(), None, None, st), "bb"))
        run("bn_bwd_apply_xmask", 3, lambda i: _lib.check(lib.cotb200_bn_bwd_apply(dt, 1, rows, C, ds[i].data_ptr(), xs[i].data_ptr(), None, None, f[3].data_ptr(), f[2].data_ptr(), f[2].data_ptr(), f[3].data_ptr(), f[4].data_ptr(), f[5].data_ptr(), 1.0 / rows, 2, o1.data_ptr(), None, None, st), "bbx"))
        run("bn_bwd_apply_res", 5, lambda i: _lib.check(lib.cotb200_bn_bwd_apply(dt, 1, rows, C, ds[i].data_ptr(), xs[i].data_ptr(), ys[i].data_ptr(), None, f[3].data_ptr(), f[2].data_ptr(), f[2].data_ptr(), f[3].data_ptr(), f[4].data_ptr(), f[5].data_ptr(), 1.0 / rows, 1, o1.data_ptr(), o2.data_ptr(), None, st), "bbr"))
        run("sum_rows3", 4, lambda i: _lib.check(lib.cotb200_sum_rows(dt, rows, C, xs[i].data_ptr(), C, ys[i].data_ptr(), C, ds[i].data_ptr(), C, None, 0, o1.data_ptr(), C, st), "sr"))
        out.append(rec)
        print(json.dumps(rec), flush=True)
        del xs, ys, ds
    if a.json:
        json.dump(out, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
