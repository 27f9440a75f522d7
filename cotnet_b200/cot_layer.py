"""CoT block host modules with the reference's module / state-dict contract.

    CotLayer(dim, kernel_size)    /root/reference/models/cotnet.py:36-104
    CoXtLayer(dim, kernel_size)   /root/reference/models/cotnet.py:106-178
    CoTLayer = CotLayer           /root/reference/models/cotnet_hybrid.py:48-116 (same arithmetic)

Sub-module names (hence checkpoint keys) are the reference's: key_embed.{0,1}, embed.{0,1,3,4}, conv1x1.{0,1},
local_conv, bn, se.{0,1,3} (SURVEY.md section 8b), so reference checkpoints load with strict=True and
``utils/flops_counter.py`` still finds a ``LocalConvolution`` child.

Forward maths is SURVEY.md Appendix A.  Differences from the reference's eager graph that do NOT change results:
  * no ``torch.cat([x, k])`` / ``cat(dim=2)`` / ``sum(dim=2)`` temporaries for the radix-2 tail: the pooled
    descriptor is mean(y + k) and the output is a0*y + a1*k directly;
  * the memory format of the input is preserved (NCHW in -> NCHW-contiguous out as the reference's
    ``.contiguous()`` gives; channels_last in -> channels_last out, no transposes), and the LocalConv runs on
    the H100 kernels (NHWC kernels for channels_last tensors).
"""
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import fused, tc
from .aggregation_zeropad import AggregationZeropad, LocalConvolution


def _radix2_tail(y, k, se):
    """models/cotnet.py:92-104 without the [B,C,2,H,W] temporaries."""
    B, C = y.shape[0], y.shape[1]
    gap = (y + k).mean((2, 3), keepdim=True)
    a = se(gap).view(B, C, 2)
    a = F.softmax(a, dim=2).to(y.dtype)
    return y * a[:, :, 0].reshape(B, C, 1, 1) + k * a[:, :, 1].reshape(B, C, 1, 1)


def _keep_format(out, like):
    if like.dim() == 4 and not like.is_contiguous() and like.is_contiguous(memory_format=torch.channels_last):
        return out.contiguous(memory_format=torch.channels_last)
    return out.contiguous()


def _dense_from_grouped(w, groups):
    """[N, K/groups, kh, kw] weight of a grouped convolution -> the block-diagonal dense weight [N, K, kh, kw] of the same
    convolution (exact zeros outside the blocks).  Differentiable (one index_put; its backward is one gather): the gradient of
    the grouped parameter is the blocks of the dense weight gradient."""
    if groups == 1:
        return w
    N, kg = w.shape[0], w.shape[1]
    ng, rest = N // groups, tuple(w.shape[2:])
    dense = w.new_zeros((groups, ng, groups, kg) + rest)
    idx = torch.arange(groups, device=w.device)
    dense[idx, :, idx] = w.reshape((groups, ng, kg) + rest)             # (idx, :, idx) -> [groups, ng, kg, ...]
    return dense.reshape((N, groups * kg) + rest)


def _coxt_embed0_dense(w, groups):
    """embed.0 of CoXtLayer (models/cotnet.py:122-123) consumes qk = [x0, k0, x1, k1, ...] (:153-154) with `groups` groups:
    group g sees the interleave of x[g*Ch:(g+1)*Ch] and k[g*Ch:(g+1)*Ch], Ch = C/groups.  Returns (Wx, Wk), dense [N, C]
    weights with  embed.0(qk) == x @ Wx^T + k @ Wk^T  -- the operand pairs of the concat-free GEMM."""
    N, kg = w.shape[0], w.shape[1]                 # kg = 2C / groups
    ng, ch = N // groups, kg // 2
    w2 = w.reshape(groups, ng, ch, 2)
    idx = torch.arange(groups, device=w.device)
    wx = w.new_zeros((groups, ng, groups, ch))
    wk = w.new_zeros((groups, ng, groups, ch))
    wx[idx, :, idx] = w2[..., 0]
    wk[idx, :, idx] = w2[..., 1]
    return wx.reshape(N, groups * ch), wk.reshape(N, groups * ch)


class CotLayer(nn.Module):
    def __init__(self, dim, kernel_size):
        super(CotLayer, self).__init__()
        self.dim = dim
        self.kernel_size = kernel_size
        ks2 = kernel_size * kernel_size
        share_planes, factor = 8, 2
        self.key_embed = nn.Sequential(
            nn.Conv2d(dim, dim, kernel_size, stride=1, padding=kernel_size // 2, groups=4, bias=False),
            nn.BatchNorm2d(dim),
            nn.ReLU(inplace=True))
        self.embed = nn.Sequential(
            nn.Conv2d(2 * dim, dim // factor, 1, bias=False),
            nn.BatchNorm2d(dim // factor),
            nn.ReLU(inplace=True),
            nn.Conv2d(dim // factor, ks2 * dim // share_planes, kernel_size=1),
            nn.GroupNorm(num_groups=dim // share_planes, num_channels=ks2 * dim // share_planes))
        self.conv1x1 = nn.Sequential(
            nn.Conv2d(dim, dim, kernel_size=1, stride=1, padding=0, dilation=1, bias=False),
            nn.BatchNorm2d(dim))
        self.local_conv = LocalConvolution(dim, dim, kernel_size=kernel_size, stride=1,
                                           padding=(kernel_size - 1) // 2, dilation=1)
        self.bn = nn.BatchNorm2d(dim)
        self.act = nn.SiLU(inplace=True)          # get_act_layer('swish'), models/layers/create_act.py:12,80-81
        self.radix = 2
        attn_chs = max(dim * self.radix // 4, 32)
        self.se = nn.Sequential(
            nn.Conv2d(dim, attn_chs, 1),
            nn.BatchNorm2d(attn_chs),
            nn.ReLU(inplace=True),
            nn.Conv2d(attn_chs, self.radix * dim, 1))

    def _forward_fused(self, x):
        """channels_last fast path: GroupNorm, bn+SiLU+pool and the radix-2 recombination are fused kernels."""
        B, C, H, W = x.shape
        ks2 = self.kernel_size * self.kernel_size
        cl = torch.channels_last
        # x has three consumers and k two: their gradients (two of them channel slices of the concat's) are summed by
        # one kernel each (fused.fan_out) instead of autograd's pairwise strided adds
        xk, xc, xv = fused.fan_out(x, 3)
        be = self.train_conv_backend
        if B * H * W < self.tc_min_pixels and be not in ("cudnn", "tc_e0"):
            be = "tc_e0"           # small problems: only the concat-free embed.0 GEMM stays on wgmma (fixed per-launch costs dominate)
        if (be.endswith("+k") and self.dim <= self.tc_key_max_dim and fused.tc_supported(x, self.dim)
                and self.key_embed[0].weight.dtype == x.dtype):
            # key_embed on the haloed-tile wgmma convolution: forward with the BatchNorm statistics in the epilogue, data gradient by
            # the same kernel (flipped / transposed weights); the grouped weight gradient stays on cuDNN
            ke = self.key_embed
            k = fused.TcConv3x3Fn.apply(xk, ke[0].weight, ke[1].weight, ke[1].bias, ke[1], ke[0].groups, True)
            be = be[:-2]
        else:
            be = be[:-2] if be.endswith("+k") else be
            k = fused.bn_act(self.key_embed[0](xk).contiguous(memory_format=cl), self.key_embed[1], relu=True)
        kc, kt = fused.fan_out(k, 2)
        hybrid = (be in ("tc_e0", "tc_1x1", "tc_e0e3", "tc_all1x1") and fused.tc_supported(x, self.dim)
                  and k.dtype == x.dtype)
        if hybrid:      # embed.0 as ONE wgmma GEMM over the operand pairs (x, W_x), (k, W_k): no concat, statistics in the epilogue
            em = self.embed
            e = fused.TcConv1x1Fn.apply(xc, kc, em[0].weight, None, em[1].weight, em[1].bias, em[1], True, None)
        else:
            e = fused.bn_act(self.embed[0](torch.cat([xc, kc], dim=1)).contiguous(memory_format=cl), self.embed[1], relu=True)
        # embed.3 runs bias-free; its bias is added (and differentiated) inside the GroupNorm kernels
        if hybrid and be in ("tc_e0e3", "tc_all1x1"):
            l = fused.TcConv1x1Fn.apply(e, None, self.embed[3].weight, None, None, None, None, False, None)
        else:
            l = F.conv2d(e, self.embed[3].weight, None)
        if hybrid and be in ("tc_1x1", "tc_all1x1"):
            cv = self.conv1x1
            v = fused.TcConv1x1Fn.apply(xv, None, cv[0].weight, None, cv[1].weight, cv[1].bias, cv[1], False, None)
        else:
            v = fused.bn_act(self.conv1x1[0](xv).contiguous(memory_format=cl), self.conv1x1[1], relu=False)
        if l.dtype != v.dtype:
            l = l.to(v.dtype)
        l = l.contiguous(memory_format=torch.channels_last)
        gc = fused.tap_chunk(C // 8)                                       # tap-major weight order for the fast kernels
        w = fused.group_norm9(l, self.embed[4], gc, self.embed[3].bias)    # fp32 statistics, storage dtype out
        u = fused.AggTapFn.apply(v.contiguous(memory_format=torch.channels_last), w, 1, gc)
        return fused.cot_tail(u, kt.contiguous(memory_format=torch.channels_last), self.bn, self.se)

    # ---- inference path: every convolution of the block on the wgmma kernels, BatchNorms folded into epilogues ----
    def _tc_eval_ok(self, x):
        return (not self.training and not torch.is_grad_enabled() and x.dtype == torch.bfloat16 and self.kernel_size == 3
                and self.dim % 64 == 0 and tc.conv_tile(self.dim, 4) is not None and x.shape[3] <= 128)

    def _tc_params(self, device):
        """bf16 GEMM operands + folded BatchNorm scale/shift, cached until a parameter / buffer changes."""
        key = (str(device),) + tuple(t._version for t in list(self.parameters()) + list(self.buffers()))
        cache = getattr(self, "_tc_cache", None)
        if cache is not None and cache["key"] == key:
            return cache
        C = self.dim

        def fold(bn):
            rstd = torch.rsqrt(bn.running_var.float() + bn.eps)
            scale = bn.weight.float() * rstd
            return scale.contiguous(), (bn.bias.float() - bn.running_mean.float() * scale).contiguous()

        with torch.no_grad():
            wk, bnk = tc.prepare_conv3x3_weight(self.key_embed[0].weight, 4)
            we1 = self.embed[0].weight.detach().view(C // 2, 2 * C).to(torch.bfloat16)
            cache = {
                "key": key, "wk": wk, "bnk": bnk, "k_ss": fold(self.key_embed[1]),
                "bn_ss": fold(self.bn),
                "we1x": we1[:, :C].contiguous(), "we1k": we1[:, C:].contiguous(), "e_ss": fold(self.embed[1]),
                "we2": self.embed[3].weight.detach().view(-1, C // 2).to(torch.bfloat16).contiguous(),
                "be2": self.embed[3].bias.detach().float().contiguous(),
                "wv": self.conv1x1[0].weight.detach().view(C, C).to(torch.bfloat16).contiguous(),
                "v_ss": fold(self.conv1x1[1]),
            }
        self._tc_cache = cache
        return cache

    def _forward_tc_eval(self, x):
        """models/cotnet.py:79-104 in eval mode with NO cuDNN/cuBLAS call: 3x3 grouped key conv = implicit GEMM over TMA
        pixel boxes, the three 1x1 convs = wgmma GEMMs on the NHWC pixel matrix (embed.0 consumes x and k as two
        operand pairs, no concat), every BatchNorm / bias / ReLU is a GEMM epilogue."""
        B, C, H, W = x.shape
        p = self._tc_params(x.device)
        k = tc.conv3x3_bf16(x, p["wk"], p["bnk"], scale=p["k_ss"][0], shift=p["k_ss"][1], relu=True)
        e = tc.gemm_bf16(x, p["we1x"], k, p["we1k"], scale=p["e_ss"][0], shift=p["e_ss"][1], relu=True)
        gc = fused.tap_chunk(C // 8)
        l = tc.gemm_bf16(e, p["we2"], shift=p["be2"])
        v = tc.gemm_bf16(x, p["wv"], scale=p["v_ss"][0], shift=p["v_ss"][1])
        J = l.shape[1]
        w = fused.group_norm9(l.view(B, H, W, J).permute(0, 3, 1, 2), self.embed[4], gc)
        u = fused.AggTapFn.apply(v.view(B, H, W, C).permute(0, 3, 1, 2), w, 1, gc)
        return fused.cot_tail(u, k, self.bn, self.se)

    def _forward_tc_train(self, x):
        """Autograd-capable path with every convolution of the block on the wgmma kernels (forward + data gradients;
        BatchNorm batch statistics from the GEMM epilogues; no torch.cat, no separate statistics pass)."""
        B, C, H, W = x.shape
        ke, em, cv = self.key_embed, self.embed, self.conv1x1
        k = fused.TcConv3x3Fn.apply(x, ke[0].weight, ke[1].weight, ke[1].bias, ke[1], 4, True)
        e = fused.TcConv1x1Fn.apply(x, k, em[0].weight, None, em[1].weight, em[1].bias, em[1], True, None)
        l = fused.TcConv1x1Fn.apply(e, None, em[3].weight, em[3].bias, None, None, None, False, None)
        v = fused.TcConv1x1Fn.apply(x, None, cv[0].weight, None, cv[1].weight, cv[1].bias, cv[1], False, None)
        gc = fused.tap_chunk(C // 8)
        w = fused.group_norm9(l, em[4], gc)
        u = fused.AggTapFn.apply(v, w, 1, gc)
        return fused.cot_tail(u, k, self.bn, self.se)

    #: Training-mode convolution backend of the block (COTB200_TRAIN_CONV):
    #:   "cudnn"      cuDNN convolutions + the fused normalisation kernels
    #:   "tc_e0"      embed.0 (the 2C -> C/2 conv on [x ; k]) as ONE concat-free two-operand-pair wgmma GEMM: forward with the
    #:                BatchNorm statistics in the epilogue, data and weight gradients on the wgmma kernels
    #:   "tc_1x1" / "tc_e0e3" / "tc_all1x1"   + conv1x1 / + embed.3 / + both (all three 1x1 convolutions of the block; with
    #:                "tc_all1x1" the enclosing bottleneck's conv1 / conv3 / downsample of stages 1-2 as well, fused.conv1x1_bn)
    #:   "...+k"      key_embed (grouped 3x3) on the haloed-tile wgmma convolution for dim <= tc_key_max_dim
    #:   "tc"         the older all-wgmma autograd path (TcConv3x3Fn + TcConv1x1Fn for everything, per-tap conv at 7x7)
    #: Inference (no_grad, eval) always takes the wgmma path when the shape allows.
    #: "tc_all1x1+k" is the default (bf16 channels_last, dim % 64 == 0; anything else uses cuDNN for that convolution): it puts the
    #: most of the step on this library.  tools/bench_conv.py and bench.py compare the backends (COTB200_TRAIN_CONV).
    train_conv_backend = os.environ.get("COTB200_TRAIN_CONV", "tc_all1x1+k")
    #: "+k" suffix of the backend: key_embed on the haloed-tile wgmma convolution for dim <= this (stages 1-2;
    #: at 14x14 / 7x7 cuDNN's grouped kernels are used)
    tc_key_max_dim = int(os.environ.get("COTB200_TC_KEY_MAX_DIM", "128"))
    #: pixels (B*H*W) below which the backend degrades to "tc_e0": on the 14x14 / 7x7 stages the fixed per-launch costs of the
    #: all-wgmma path outweigh its byte savings
    tc_min_pixels = int(os.environ.get("COTB200_TC_MIN_PIXELS", "100000"))

    def forward(self, x):
        B, C, H, W = x.shape
        if self.kernel_size == 3 and fused.supported(x):
            if self._tc_eval_ok(x):
                return self._forward_tc_eval(x)
            if self.train_conv_backend == "tc" and fused.tc_supported(x, self.dim):
                return self._forward_tc_train(x)
            return self._forward_fused(x)
        k = self.key_embed(x)                                              # static context
        w = self.embed(torch.cat([x, k], dim=1))                           # logits, GroupNorm'ed, NOT softmaxed
        v = self.conv1x1(x)
        # cast BEFORE the 6-D view: .to() on the 4-D tensor keeps channels_last, so the view below is the NHWC weight
        # layout the kernels take without a copy
        w = w.to(v.dtype).view(B, 1, C // 8, self.kernel_size * self.kernel_size, H, W)
        y = self.local_conv(v, w)                                          # H100 LocalConv kernel
        y = self.act(self.bn(y))
        return _keep_format(_radix2_tail(y, k, self.se), x)


class CoXtLayer(nn.Module):
    def __init__(self, dim, kernel_size):
        super(CoXtLayer, self).__init__()
        self.dim = dim
        self.kernel_size = kernel_size
        ks2 = kernel_size * kernel_size
        self.dw_group = 2
        share_planes, factor = 8, 2
        self.key_embed = nn.Sequential(
            nn.Conv2d(dim, dim, kernel_size, stride=1, padding=kernel_size // 2, groups=8, bias=False),
            nn.BatchNorm2d(dim),
            nn.ReLU(inplace=True))
        self.embed = nn.Sequential(
            nn.Conv2d(2 * dim, dim // factor, 1, groups=self.dw_group, bias=False),
            nn.BatchNorm2d(dim // factor),
            nn.ReLU(inplace=True),
            nn.Conv2d(dim // factor, ks2 * dim // share_planes, kernel_size=1, groups=self.dw_group),
            nn.GroupNorm(num_groups=dim // share_planes, num_channels=ks2 * dim // share_planes))
        self.conv1x1 = nn.Sequential(
            nn.Conv2d(dim, dim, kernel_size=1, stride=1, padding=0, dilation=1, groups=self.dw_group, bias=False),
            nn.BatchNorm2d(dim))
        self.local_conv = LocalConvolution(dim, dim, kernel_size=kernel_size, stride=1,
                                           padding=(kernel_size - 1) // 2, dilation=1)
        self.bn = nn.BatchNorm2d(dim)
        self.act = nn.SiLU(inplace=True)
        self.radix = 2
        attn_chs = max(dim * self.radix // 4, 32)
        self.se = nn.Sequential(
            nn.Conv2d(dim, attn_chs, 1),
            nn.BatchNorm2d(attn_chs),
            nn.ReLU(inplace=True),
            nn.Conv2d(attn_chs, self.radix * dim, 1))

    def _forward_fused(self, x):
        """channels_last fast path.  The grouped convolutions (groups 8 / 2 / 2 / 2, :113-133) run as DENSE convolutions with
        block-diagonal weights built from the grouped parameters (differentiable scatter, exact zeros elsewhere -- the same
        arithmetic): cuDNN's grouped NHWC kernels for 12..96-channel groups spend much of their time in layout transforms
        (tensorTransformGeneric in a torch.profiler trace), the extra dense FLOPs are free on an
        HBM-bound block, and the dense form puts embed.0 on the concat-free two-pair wgmma GEMM like the CoT layer (the
        channel interleave of qk, :153-154, becomes a column permutation of the weight)."""
        B, C, H, W = x.shape
        cl = torch.channels_last
        G = self.dw_group
        xk, xc, xv = fused.fan_out(x, 3)
        wkey = _dense_from_grouped(self.key_embed[0].weight, self.key_embed[0].groups)
        k = fused.bn_act(F.conv2d(xk, wkey, None, 1, self.kernel_size // 2).contiguous(memory_format=cl), self.key_embed[1], relu=True)
        kc, kt = fused.fan_out(k, 2)
        wx, wk = _coxt_embed0_dense(self.embed[0].weight, G)
        w0 = torch.cat([wx, wk], 1).reshape(C // 2, 2 * C, 1, 1)
        be = self.train_conv_backend.replace("+k", "")      # the grouped key conv of CoXt (groups 8, dense block-diagonal) stays on cuDNN
        use_tc = be != "cudnn" and x.dtype == torch.bfloat16 and C % 16 == 0 and k.dtype == x.dtype and w0.dtype == x.dtype
        em, cv = self.embed, self.conv1x1
        if use_tc:
            e = fused.TcConv1x1Fn.apply(xc, kc, w0, None, em[1].weight, em[1].bias, em[1], True, None)
        else:
            e = fused.bn_act(F.conv2d(torch.cat([xc, kc], dim=1), w0).contiguous(memory_format=cl), em[1], relu=True)
        w3 = _dense_from_grouped(em[3].weight, G)
        if use_tc and be in ("tc_e0e3", "tc_all1x1", "tc") and w3.shape[0] % 8 == 0:
            l = fused.TcConv1x1Fn.apply(e, None, w3, None, None, None, None, False, None)
        else:
            l = F.conv2d(e, w3, None)
        wv = _dense_from_grouped(cv[0].weight, G)
        if use_tc and be in ("tc_1x1", "tc_all1x1", "tc"):
            v = fused.TcConv1x1Fn.apply(xv, None, wv, None, cv[1].weight, cv[1].bias, cv[1], False, None)
        else:
            v = fused.bn_act(F.conv2d(xv, wv).contiguous(memory_format=cl), cv[1], relu=False)
        if l.dtype != v.dtype:
            l = l.to(v.dtype)
        gc = fused.tap_chunk(C // 8, self.dw_group)
        w = fused.group_norm9(l.contiguous(memory_format=torch.channels_last), self.embed[4], gc, self.embed[3].bias)
        u = fused.AggTapFn.apply(v.contiguous(memory_format=torch.channels_last), w, self.dw_group, gc)
        return fused.cot_tail(u, kt.contiguous(memory_format=torch.channels_last), self.bn, self.se)

    #: CoXt: the dense block-diagonal form of its grouped 1x1 convolutions doubles their FLOPs, so only embed.0 (the concat-free
    #: two-pair GEMM) runs on the wgmma kernels by default
    train_conv_backend = os.environ.get("COTB200_TRAIN_CONV_COXT", "tc_e0")

    def forward(self, x):
        B, C, H, W = x.shape
        ks = self.kernel_size
        if ks == 3 and fused.supported(x):
            return self._forward_fused(x)
        k = self.key_embed(x)
        qk = torch.stack([x, k], dim=2).reshape(B, 2 * C, H, W)            # interleaved x0,k0,x1,k1,.. (:153-154)
        if not x.is_contiguous() and x.is_contiguous(memory_format=torch.channels_last):
            qk = qk.contiguous(memory_format=torch.channels_last)
        v = self.conv1x1(x)
        w = self.embed(qk).to(v.dtype)
        # The reference folds the two channel halves into the batch: view(2B, C/2, H, W) with weights
        # view(2B, 1, C/16, 9, H, W) (:157-162).  Same arithmetic un-folded: channel c of half f uses weight channel
        # f*(C/16) + (c % (C/2)) % (C/16) -- the kernels' `fold` argument -- so channels_last tensors need no copy.
        if v.is_contiguous() and w.is_contiguous():
            # NCHW: the reference's batch fold is a free view and keeps the register-resident fast kernel
            G = self.dw_group
            y = AggregationZeropad.apply(v.view(B * G, C // G, H, W), w.view(B * G, 1, -1, ks * ks, H, W),
                                         ks, 1, (ks - 1) // 2, 1).view(B, C, H, W)
        else:
            w = w.view(B, 1, C // 8, ks * ks, H, W)
            y = AggregationZeropad.apply(v, w, ks, 1, (ks - 1) // 2, 1, self.dw_group)
        y = self.act(self.bn(y))
        return _keep_format(_radix2_tail(y, k, self.se), x)


CoTLayer = CotLayer   # models/cotnet_hybrid.py:48-116 is the same block under another name
