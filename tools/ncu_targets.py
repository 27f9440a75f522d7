#!/usr/bin/env python
"""The launches worth an `ncu --set full` capture, warmed up first and bracketed by cudaProfilerStart/Stop:

    ncu --set full --clock-control none --import-source on --profile-from-start off -o gpurun_out/targets \
        python tools/ncu_targets.py [--what eval,gemm,train]

  eval  : one eval-mode CotLayer forward (wgmma path, 8 launches) at the stage-1 and stage-3 shapes of CoTNet-50 bs256
  gemm  : the 1x1-convolution GEMMs of the training step with the BatchNorm-statistics epilogue, and their data-gradient GEMMs
  train : one training-mode CotLayer forward + backward at the stage-1 shape (LocalConv dX / dW, GroupNorm, tail kernels)
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from cotnet_b200 import _lib, tc  # noqa: E402
from cotnet_b200.cot_layer import CotLayer  # noqa: E402


def layer(C):
    m = CotLayer(C, 3).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.2); mod.running_var.uniform_(0.5, 1.5)
                mod.weight.uniform_(0.5, 1.5); mod.bias.normal_(0, 0.2)
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="eval,gemm")
    ap.add_argument("--batch", type=int, default=256)
    a = ap.parse_args()
    what = a.what.split(",")
    _lib.load()
    torch.backends.cudnn.benchmark = True
    B = a.batch
    jobs = []
    if "eval" in what:
        for C, H in ((64, 56), (256, 14)):
            m = layer(C).eval()
            x = torch.relu(torch.randn(B, C, H, H, device="cuda")).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

            def run(m=m, x=x):
                with torch.no_grad():
                    m(x)
            jobs.append(run)
    if "gemm" in what:
        for HW, K, N in ((56, 64, 64), (56, 64, 256), (56, 256, 64), (28, 128, 512), (14, 256, 256)):
            M = B * HW * HW
            x2 = torch.randn(M, K, device="cuda").to(torch.bfloat16)
            wk = torch.randn(N, K, device="cuda").to(torch.bfloat16)
            cs, cq = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
            out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            dy = torch.randn(M, N, device="cuda").to(torch.bfloat16)
            dx = torch.empty(M, K, device="cuda", dtype=torch.bfloat16)
            wt = wk.t().contiguous()
            dw = torch.zeros(N, K, device="cuda")

            def run(x2=x2, wk=wk, cs=cs, cq=cq, out=out, dy=dy, dx=dx, wt=wt, dw=dw):
                tc.gemm_bf16(x2, wk, stats=(cs, cq), out=out)      # forward with the statistics epilogue
                tc.gemm_bf16(x2, wk, out=out)                       # the same GEMM, plain epilogue
                tc.gemm_bf16(dy, wt, out=dx)                        # data gradient
                tc.wgrad_bf16(dy, x2, out=dw)                       # weight gradient
            jobs.append(run)
    if "train" in what:
        m = layer(64).train()
        x = torch.relu(torch.randn(B, 64, 56, 56, device="cuda")).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

        def run(m=m, x=x):
            xx = x.detach().requires_grad_(True)
            m(xx).float().sum().backward()
        jobs.append(run)
    for j in jobs:
        for _ in range(2):
            j()
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    for j in jobs:
        j()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()


if __name__ == "__main__":
    main()
