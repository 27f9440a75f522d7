#!/usr/bin/env python
"""CoT-block microbenchmark (BASELINE.json metric "CoT-block us"): one CotLayer per CoTNet-50 stage shape, bs256, bf16.

    python tools/bench_block.py [--batch 256] [--iters 10] [--json out.json] [--train]

Arms (same module weights, same inputs, CUDA-event timing, >= 3 warm-ups, inputs rotated through > 126 MB):
  eager      the reference's own eager graph (models/cotnet.py:79-104: cat / GroupNorm / bn / SiLU / cat-sum-mean / softmax ...)
             with only the LocalConv op on our kernel -- what "drop in the op only" gives; stands in for the GPU
             reference block (the CuPy op itself cannot run here: SURVEY.md D5)
  fused      this repo, cuDNN convolutions + fused BatchNorm / GroupNorm / tail kernels (training-capable path)
  tc         this repo, eval mode: every convolution on the wgmma kernels, BatchNorms folded (no cuDNN/cuBLAS)
Roofline (SURVEY 8d): max(FLOPs / bf16 peak, 2*C*px*2 bytes / HBM peak) for the fully fused block."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from cotnet_b200 import _lib  # noqa: E402
from cotnet_b200.cot_layer import CotLayer  # noqa: E402

STAGES = [(64, 56), (128, 28), (256, 14), (512, 7)]


def eager_forward(m, x):
    """The reference forward, op by op (models/cotnet.py:79-104), LocalConv on our op kernel."""
    k = m.key_embed(x)
    qk = torch.cat([x, k], dim=1)
    b, c, hh, ww = qk.size()
    w = m.embed(qk)
    w = w.view(b, 1, -1, 9, hh, ww)
    v = m.conv1x1(x)
    y = m.local_conv(v, w)
    y = m.act(m.bn(y))
    B, C, H, W = y.shape
    y5 = y.view(B, C, 1, H, W)
    k5 = k.view(B, C, 1, H, W)
    t = torch.cat([y5, k5], dim=2)
    gap = t.sum(dim=2).mean((2, 3), keepdim=True)
    attn = F.softmax(m.se(gap).view(B, C, 2), dim=2)
    return (t * attn.reshape(B, C, 2, 1, 1)).sum(dim=2).contiguous()


def peaks():
    try:
        d = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return float(d["hbm_gbs"]), float(d["bf16_tflops"])
    except Exception:
        return 6650.0, 1590.0


def timeit(fn, xs, iters):
    for i in range(3):
        fn(xs[i % len(xs)])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(xs[i % len(xs)])
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--train", action="store_true", help="also time training-mode forward+backward (eager vs fused)")
    a = ap.parse_args()
    _lib.load()
    torch.backends.cudnn.benchmark = True
    hbm, tf = peaks()
    rows = []
    B = a.batch
    for C, H in STAGES:
        m = CotLayer(C, 3).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, torch.nn.BatchNorm2d):
                    mod.running_mean.normal_(0, 0.2); mod.running_var.uniform_(0.5, 1.5)
                    mod.weight.uniform_(0.5, 1.5); mod.bias.normal_(0, 0.2)
        px = B * H * H
        nset = max(2, int(300e6 // (px * C * 2)) + 1)
        xs = [torch.relu(torch.randn(B, C, H, H, device="cuda")).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
              for _ in range(nset)]
        flops = (9.625 * C * C + 18 * C) * px
        roof_us = max(flops / (tf * 1e12), 2 * C * px * 2 / (hbm * 1e9)) * 1e6
        row = {"C": C, "HW": H, "B": B, "roofline_us": roof_us, "flops": flops, "min_bytes": 2 * C * px * 2}
        m.eval()
        with torch.no_grad():
            ref = eager_forward(m, xs[0])
            out_tc = m(xs[0])
            row["tc_vs_eager_maxabs"] = float((out_tc.float() - ref.float()).abs().max())
            row["eager_eval_us"] = timeit(lambda x: eager_forward(m, x), xs, a.iters)
            row["tc_eval_us"] = timeit(lambda x: m(x), xs, a.iters)
            # the same forward replayed from a CUDA graph: removes the ~0.5 ms of Python/launch overhead of ~25 small launches
            try:
                xg = xs[0].clone()
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    for _ in range(3):
                        m(xg)
                torch.cuda.current_stream().wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    yg = m(xg)
                row["tc_eval_graph_us"] = timeit(lambda x: graph.replay(), xs, a.iters)
                row["graph_vs_eager_maxabs"] = float((yg.float() - m(xg).float()).abs().max())
            except Exception as e:      # noqa: BLE001
                row["tc_eval_graph_error"] = repr(e)[:200]
        with torch.enable_grad():     # grad mode on -> the cuDNN-conv fused path is taken even in eval
            row["fused_eval_us"] = timeit(lambda x: m(x), xs, a.iters)
        row["tc_frac_of_roofline"] = roof_us / min(row["tc_eval_us"], row.get("tc_eval_graph_us", 1e30))
        if a.train:
            m.train()

            def fb(fn):
                def run(x):
                    x = x.detach().requires_grad_(True)
                    fn(x).float().sum().backward()
                return run
            row["eager_train_fwdbwd_us"] = timeit(fb(lambda x: eager_forward(m, x)), xs, a.iters)
            row["fused_train_fwdbwd_us"] = timeit(fb(lambda x: m(x)), xs, a.iters)
            m.train_conv_backend = "tc"
            row["tc_train_fwdbwd_us"] = timeit(fb(lambda x: m(x)), xs, a.iters)
            m.train_conv_backend = "cudnn"
        rows.append(row)
        print(json.dumps(row), flush=True)
        del xs, m
        torch.cuda.empty_cache()
    if a.json:
        json.dump({"hbm_gbs": hbm, "bf16_tflops": tf, "rows": rows}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
