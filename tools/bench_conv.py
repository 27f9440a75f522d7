#!/usr/bin/env python
"""conv1x1 -> BatchNorm(batch stats) -> ReLU, forward + backward, at every 1x1-conv shape of the CoTNet-50 bs256 step:
cuDNN conv + fused BN kernels against the wgmma GEMM with the statistics epilogue (TcConv1x1Fn).  In training, the
geometry thresholds fused.TC_MIN_PIXELS and fused.TC_TRUNK_MAX_WEIGHT pick between the two per shape."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from cotnet_b200 import fused  # noqa: E402

# (name, HW, K, N): CoT-internal (embed.0 2C->C/2, embed.3 C/2->9C/8 [no BN], conv1x1 C->C) and bottleneck convs
SHAPES = [("s1.e0", 56, 128, 32), ("s1.v", 56, 64, 64), ("s1.conv1", 56, 256, 64), ("s1.conv3", 56, 64, 256),
          ("s2.e0", 28, 256, 64), ("s2.v", 28, 128, 128), ("s2.conv1", 28, 512, 128), ("s2.conv3", 28, 128, 512),
          ("s3.e0", 14, 512, 128), ("s3.v", 14, 256, 256), ("s3.conv1", 14, 1024, 256), ("s3.conv3", 14, 256, 1024),
          ("s4.e0", 7, 1024, 256), ("s4.v", 7, 512, 512), ("s4.conv1", 7, 2048, 512), ("s4.conv3", 7, 512, 2048)]


def timeit(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda")
    rows = []
    for name, HW, K, N in SHAPES:
        x = torch.randn(a.batch, K, HW, HW, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        conv = nn.Conv2d(K, N, 1, bias=False).to(dev)
        bn = nn.BatchNorm2d(N).to(dev).train()
        cot = torch.randn(a.batch, N, HW, HW, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        wb = conv.weight.detach().to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)

        def cudnn_fb():
            y = fused.bn_act(F.conv2d(x, wb).contiguous(memory_format=torch.channels_last), bn, relu=True)
            return torch.autograd.grad(y, (x, wb, bn.weight, bn.bias), cot)

        def tc_fb():
            y = fused.TcConv1x1Fn.apply(x, None, conv.weight, None, bn.weight, bn.bias, bn, True, None)
            return torch.autograd.grad(y, (x, conv.weight, bn.weight, bn.bias), cot)

        def cudnn_f():
            with torch.no_grad():
                return fused.bn_act(F.conv2d(x, wb).contiguous(memory_format=torch.channels_last), bn, relu=True)

        def tc_f():
            with torch.no_grad():
                return fused.TcConv1x1Fn.apply(x, None, conv.weight, None, bn.weight, bn.bias, bn, True, None)

        # raw pieces: our kernels vs the library kernels cuDNN picks for the same contraction (bytes = operands once + result once)
        from cotnet_b200 import tc
        M = a.batch * HW * HW
        wk = conv.weight.detach().reshape(N, K).to(torch.bfloat16).contiguous()
        wkt = wk.t().contiguous()
        cs, cq = torch.zeros(N, device=dev), torch.zeros(N, device=dev)
        outb = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        dxb = torch.empty(M, K, device=dev, dtype=torch.bfloat16)
        dwf = torch.zeros(N, K, device=dev)
        x2, c2 = x.detach().permute(0, 2, 3, 1).reshape(M, K), cot.permute(0, 2, 3, 1).reshape(M, N)
        xd = x.detach()
        raw = {
            "tc_fwd_stats_us": timeit(lambda: tc.gemm_bf16(x2, wk, stats=(cs, cq), out=outb), a.iters),
            "tc_dgrad_us": timeit(lambda: tc.gemm_bf16(c2, wkt, out=dxb), a.iters),
            "tc_wgrad_us": timeit(lambda: tc.wgrad_bf16(c2, x2, out=dwf), a.iters),
            "cudnn_fprop_us": timeit(lambda: F.conv2d(xd, wb.detach()), a.iters),
            "cudnn_dgrad_us": timeit(lambda: torch.nn.grad.conv2d_input(xd.shape, wb.detach(), cot), a.iters),
            "cudnn_wgrad_us": timeit(lambda: torch.nn.grad.conv2d_weight(xd, wb.shape, cot), a.iters),
        }
        by = 2.0 * M * (K + N) + 2.0 * N * K
        raw["roof_us_at_6485GBps"] = round(by / 6485.2e3, 1)
        raw = {k_: round(v_, 1) for k_, v_ in raw.items()}
        rec = {"name": name, "HW": HW, "K": K, "N": N, "raw": raw,
               "cudnn_fwd_us": round(timeit(cudnn_f, a.iters), 1), "tc_fwd_us": round(timeit(tc_f, a.iters), 1),
               "cudnn_fwdbwd_us": round(timeit(cudnn_fb, a.iters), 1), "tc_fwdbwd_us": round(timeit(tc_fb, a.iters), 1)}
        rec["tc_over_cudnn_fwdbwd"] = round(rec["tc_fwdbwd_us"] / rec["cudnn_fwdbwd_us"], 3)
        rows.append(rec)
        print(json.dumps(rec), flush=True)
    if a.json:
        json.dump(rows, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
