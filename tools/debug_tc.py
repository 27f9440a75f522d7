#!/usr/bin/env python
"""Debug helper: per-gradient errors of the wgmma-backed autograd functions vs eager fp32."""
import copy
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from cotnet_b200 import fused, tc  # noqa: E402


def cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def report(names, got, want):
    for n, a, b in zip(names, got, want):
        e = (a.float() - b.float()).abs().max().item()
        print("   %-10s err %.4e  scale %.3e  shape %s" % (n, e, b.abs().max().item(), tuple(b.shape)))


def conv1x1(two, training):
    g = torch.Generator(device="cuda").manual_seed(3)
    B, K1, K2, N, H = 8, 64, (64 if two else 0), 32, 14
    conv = nn.Conv2d(K1 + K2, N, 1, bias=False).cuda()
    bn = nn.BatchNorm2d(N).cuda()
    with torch.no_grad():
        conv.weight.copy_(conv.weight.bfloat16().float())
        bn.weight.uniform_(0.5, 1.5, generator=g); bn.bias.normal_(0, 0.3, generator=g)
        bn.running_mean.normal_(0, 0.3, generator=g); bn.running_var.uniform_(0.5, 2, generator=g)
    conv_r, bn_r = copy.deepcopy(conv), copy.deepcopy(bn)
    bn.train(training); bn_r.train(training)
    a1 = cl(torch.randn(B, K1, H, H, generator=g, device="cuda").bfloat16()).requires_grad_(True)
    a2 = cl(torch.randn(B, K2, H, H, generator=g, device="cuda").bfloat16()).requires_grad_(True) if two else None
    cot = cl(torch.randn(B, N, H, H, generator=g, device="cuda").bfloat16())
    y = fused.TcConv1x1Fn.apply(a1, a2, conv.weight, None, bn.weight, bn.bias, bn, True, None)
    ins = [a1, conv.weight, bn.weight, bn.bias] + ([a2] if two else [])
    grads = torch.autograd.grad(y, ins, cot)
    a1r = a1.detach().float().requires_grad_(True)
    a2r = a2.detach().float().requires_grad_(True) if two else None
    xin = torch.cat([a1r, a2r], 1) if two else a1r
    pre_r = conv_r(xin)
    yr = torch.relu(bn_r(pre_r))
    grads_r = torch.autograd.grad(yr, [a1r, conv_r.weight, bn_r.weight, bn_r.bias] + ([a2r] if two else []), cot.float())
    print("conv1x1 two=%s training=%s" % (two, training))
    report(["y"], [y], [yr])
    report(["da1", "dW", "dgamma", "dbeta"] + (["da2"] if two else []), grads, grads_r)
    # direct GEMM checks of the data-gradient shapes
    M = B * H * H
    d = torch.randn(M, N, generator=g, device="cuda").bfloat16()
    wt = torch.randn(K1 + K2, N, generator=g, device="cuda").bfloat16()
    o1 = tc.gemm_bf16(d, wt[:K1])
    report(["gemm[:K1]"], [o1], [d.float() @ wt[:K1].float().t()])
    if two:
        o2 = tc.gemm_bf16(d, wt[K1:])
        report(["gemm[K1:]"], [o2], [d.float() @ wt[K1:].float().t()])
        o3 = torch.empty(M, K2, device="cuda", dtype=torch.bfloat16)
        tc.gemm_bf16(d, wt[K1:], out=o3)
        report(["gemm out="], [o3], [d.float() @ wt[K1:].float().t()])


def conv3x3(training):
    g = torch.Generator(device="cuda").manual_seed(4)
    B, C, H = 6, 128, 14
    conv = nn.Conv2d(C, C, 3, padding=1, groups=4, bias=False).cuda()
    bn = nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        conv.weight.copy_(conv.weight.bfloat16().float())
        bn.weight.uniform_(0.5, 1.5, generator=g); bn.bias.normal_(0, 0.3, generator=g)
        bn.running_mean.normal_(0, 0.3, generator=g); bn.running_var.uniform_(0.5, 2, generator=g)
    conv_r, bn_r = copy.deepcopy(conv), copy.deepcopy(bn)
    bn.train(training); bn_r.train(training)
    x = cl(torch.randn(B, C, H, H, generator=g, device="cuda").bfloat16()).requires_grad_(True)
    cot = cl(torch.randn(B, C, H, H, generator=g, device="cuda").bfloat16())
    y = fused.TcConv3x3Fn.apply(x, conv.weight, bn.weight, bn.bias, bn, 4, True)
    grads = torch.autograd.grad(y, [x, conv.weight, bn.weight, bn.bias], cot)
    xr = x.detach().float().requires_grad_(True)
    yr = torch.relu(bn_r(conv_r(xr)))
    grads_r = torch.autograd.grad(yr, [xr, conv_r.weight, bn_r.weight, bn_r.bias], cot.float())
    print("conv3x3 training=%s" % training)
    report(["y"], [y], [yr])
    report(["dx", "dW", "dgamma", "dbeta"], grads, grads_r)
    if training:
        print("   running_mean err %.3e var err %.3e" % ((bn.running_mean - bn_r.running_mean).abs().max().item(),
                                                          (bn.running_var - bn_r.running_var).abs().max().item()))


if __name__ == "__main__":
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for two in (False, True):
        for tr in (False, True):
            conv1x1(two, tr)
    for tr in (False, True):
        conv3x3(tr)
