"""GPU tests of the wgmma/TMA GEMM and implicit-GEMM 3x3 conv against fp32 torch math on the same
bf16-representable operands (tolerance: bf16 output rounding, atol=rtol=1e-2)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _tc():
    from cotnet_b200 import tc
    return tc


def _close(got, want, tol=1e-2):
    got, want = got.float(), want.float()
    err = (got - want).abs()
    lim = tol + tol * want.abs()
    assert bool((err <= lim).all()), "max err %.4e at |ref| %.3e" % (err.max().item(), want.abs().max().item())


@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (1000, 32, 128), (3136, 72, 32), (777, 144, 64), (4096, 256, 512),
                                   (513, 288, 128), (2048, 576, 256), (300, 512, 1024), (128, 16, 8)])
def test_gemm_plain(M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g, device="cuda").bfloat16()
    b = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).bfloat16()
    d = _tc().gemm_bf16(a, b)
    _close(d, a.float() @ b.float().t())


def test_gemm_two_pairs_epilogue_and_stats():
    g = torch.Generator(device="cuda").manual_seed(5)
    M, N, K1, K2 = 3000, 64, 128, 128
    a1 = torch.randn(M, K1, generator=g, device="cuda").bfloat16()
    a2 = torch.randn(M, K2, generator=g, device="cuda").bfloat16()
    b = (torch.randn(N, K1 + K2, generator=g, device="cuda") / 16).bfloat16()
    b1, b2 = b[:, :K1], b[:, K1:]                       # column slices of one weight: concat-free embed.0
    scale = torch.rand(N, generator=g, device="cuda") + 0.5
    shift = torch.randn(N, generator=g, device="cuda")
    cs = torch.zeros(N, device="cuda")
    cq = torch.zeros(N, device="cuda")
    d = _tc().gemm_bf16(a1, b1, a2, b2, scale=scale, shift=shift, relu=True, stats=(cs, cq))
    acc = torch.cat([a1, a2], 1).float() @ b.float().t()
    _close(d, torch.relu(acc * scale + shift))
    # the statistics are those of the STORED tensor (what a following normalisation reads back)
    assert torch.allclose(cs, d.float().sum(0), atol=1e-2, rtol=1e-4)
    assert torch.allclose(cq, (d.float() * d.float()).sum(0), atol=1e-2, rtol=1e-4)
    # training-mode use: raw product, no epilogue transform -> BatchNorm batch statistics of the convolution output
    cs.zero_(); cq.zero_()
    d2 = _tc().gemm_bf16(a1, b1, a2, b2, stats=(cs, cq))
    _close(d2, acc)
    assert torch.allclose(cs, d2.float().sum(0), atol=1e-2, rtol=1e-4) and torch.allclose(cs, acc.sum(0), atol=0.5, rtol=5e-3)
    assert torch.allclose(cq, (d2.float() * d2.float()).sum(0), atol=1e-2, rtol=1e-4) and torch.allclose(cq, (acc * acc).sum(0), atol=1.0, rtol=5e-3)


def test_gemm_channels_last_rows():
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(3, 64, 14, 14, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    w = (torch.randn(64, 64, generator=g, device="cuda") / 8).bfloat16()
    d = _tc().gemm_bf16(x, w)
    want = F.conv2d(x.float(), w.float()[:, :, None, None])
    _close(d.view(3, 14, 14, 64).permute(0, 3, 1, 2), want)


@pytest.mark.parametrize("C,groups,H,B", [(64, 4, 56, 2), (128, 4, 28, 3), (256, 4, 14, 3), (512, 4, 7, 5), (64, 4, 8, 2),
                                          (64, 1, 10, 2), (128, 4, 40, 2), (64, 4, 80, 1), (192, 1, 12, 2)])
def test_conv3x3(C, groups, H, B):
    tc = _tc()
    g = torch.Generator(device="cuda").manual_seed(C + H)
    x = torch.randn(B, C, H, H, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    w = (torch.randn(C, C // groups, 3, 3, generator=g, device="cuda") / (3 * (C // groups) ** 0.5)).bfloat16()
    wp, bn = tc.prepare_conv3x3_weight(w, groups)
    cs = torch.zeros(C, device="cuda")
    cq = torch.zeros(C, device="cuda")
    d = tc.conv3x3_bf16(x, wp, bn, stats=(cs, cq))
    want = F.conv2d(x.float(), w.float(), None, 1, 1, 1, groups)
    _close(d, want)
    assert torch.allclose(cs, d.float().sum((0, 2, 3)), atol=1e-2, rtol=1e-4) and torch.allclose(cs, want.sum((0, 2, 3)), atol=5e-1, rtol=5e-3)
    # data gradient as the same kernel with transposed / flipped weights
    wpt, bnt = tc.prepare_conv3x3_weight(w, groups, transpose_for_dgrad=True)
    gy = torch.randn(B, C, H, H, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    dx = tc.conv3x3_bf16(gy, wpt, bnt)
    want_dx = torch.nn.grad.conv2d_input(x.shape, w.float(), gy.float(), 1, 1, 1, groups)
    _close(dx, want_dx)


@pytest.mark.parametrize("M,N,K1,K2", [(3136, 64, 256, 0), (3136, 256, 64, 0), (1000, 32, 64, 64), (12544, 72, 32, 0), (200, 128, 128, 0),
                                       (6272, 512, 2048, 0), (6272, 2048, 512, 0), (4096, 64, 64, 64), (70, 16, 24, 0), (3136, 48, 96, 96)])
def test_wgrad(M, N, K1, K2):
    """dW = dY^T [A1 | A2] on the MN-major wgmma kernel (TMA tiles consumed as they land) vs fp32 matmul."""
    tc = _tc()
    g = torch.Generator(device="cuda").manual_seed(M + N)
    dy = torch.randn(M, N, generator=g, device="cuda").bfloat16()
    a1 = torch.randn(M, K1, generator=g, device="cuda").bfloat16()
    a2 = torch.randn(M, K2, generator=g, device="cuda").bfloat16() if K2 else None
    want = dy.float().t() @ (torch.cat([a1, a2], 1) if K2 else a1).float()
    got = tc.wgrad_bf16(dy, a1, a2)
    rel = ((got - want).norm() / want.norm()).item()
    assert rel <= 2e-3, rel               # fp32 accumulation of exact bf16 products: only the summation order differs


def test_wgrad_channels_last_views_and_accumulate():
    tc = _tc()
    g = torch.Generator(device="cuda").manual_seed(9)
    dy = torch.randn(4, 96, 14, 14, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    x = torch.randn(4, 192, 14, 14, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    want = torch.einsum("bnhw,bkhw->nk", dy.float(), x.float())
    out = torch.ones(96, 192, device="cuda")
    tc.wgrad_bf16(dy, x, out=out)                                         # the kernel ADDS into `out`
    assert ((out - 1.0 - want).norm() / want.norm()).item() <= 2e-3


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _rel_l2(a, b, tol=3e-2):
    """Gradients through bf16 conv -> BN(batch stats) -> ReLU: the ReLU mask is taken from the bf16-ROUNDED pre-activation
    (as in any bf16 pipeline), so a handful of near-zero elements flip and dominate a max-abs comparison; the Frobenius
    error stays at the bf16 level."""
    a, b = a.float(), b.float()
    rel = ((a - b).norm() / b.norm().clamp_min(1e-6)).item()
    assert rel <= tol, "relative L2 error %.3e" % rel


@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("two", [False, True])
def test_tc_conv1x1_fn_autograd(training, two):
    """TcConv1x1Fn (wgmma forward + data gradient, BN statistics from the epilogue) vs eager conv+BN+ReLU in fp32."""
    import copy
    import torch.nn as nn
    from cotnet_b200 import fused
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
    a1 = _cl(torch.randn(B, K1, H, H, generator=g, device="cuda").bfloat16()).requires_grad_(True)
    a2 = _cl(torch.randn(B, K2, H, H, generator=g, device="cuda").bfloat16()).requires_grad_(True) if two else None
    cot = _cl(torch.randn(B, N, H, H, generator=g, device="cuda").bfloat16())
    y = fused.TcConv1x1Fn.apply(a1, a2, conv.weight, None, bn.weight, bn.bias, bn, True, None)
    ins = [a1, conv.weight, bn.weight, bn.bias] + ([a2] if two else [])
    grads = torch.autograd.grad(y, ins, cot)
    a1r = a1.detach().float().requires_grad_(True)
    a2r = a2.detach().float().requires_grad_(True) if two else None
    xin = torch.cat([a1r, a2r], 1) if two else a1r
    yr = torch.relu(bn_r(conv_r(xin)))
    grads_r = torch.autograd.grad(yr, [a1r, conv_r.weight, bn_r.weight, bn_r.bias] + ([a2r] if two else []), cot.float())
    _close(y, yr, 3e-2)
    for a, b in zip(grads, grads_r):
        _rel_l2(a, b)
    if training:
        assert torch.allclose(bn.running_mean, bn_r.running_mean, atol=2e-2)


@pytest.mark.parametrize("training", [False, True])
def test_tc_conv1x1_fn_residual(training):
    """The bottleneck's conv3 -> bn3 -> (+ residual) -> ReLU (models/cotnet.py:249-262) as one TcConv1x1Fn: forward,
    data / weight / residual gradients vs eager fp32."""
    import copy
    import torch.nn as nn
    from cotnet_b200 import fused
    g = torch.Generator(device="cuda").manual_seed(5)
    B, K, N, H = 8, 64, 256, 14
    conv = nn.Conv2d(K, N, 1, bias=False).cuda()
    bn = nn.BatchNorm2d(N).cuda()
    with torch.no_grad():
        conv.weight.copy_(conv.weight.bfloat16().float())
        bn.weight.uniform_(0.5, 1.5, generator=g); bn.bias.normal_(0, 0.3, generator=g)
        bn.running_mean.normal_(0, 0.3, generator=g); bn.running_var.uniform_(0.5, 2, generator=g)
    conv_r, bn_r = copy.deepcopy(conv), copy.deepcopy(bn)
    bn.train(training); bn_r.train(training)
    x = _cl(torch.randn(B, K, H, H, generator=g, device="cuda").bfloat16()).requires_grad_(True)
    res = _cl(torch.randn(B, N, H, H, generator=g, device="cuda").bfloat16()).requires_grad_(True)
    cot = _cl(torch.randn(B, N, H, H, generator=g, device="cuda").bfloat16())
    y = fused.TcConv1x1Fn.apply(x, None, conv.weight, None, bn.weight, bn.bias, bn, True, res)
    grads = torch.autograd.grad(y, [x, conv.weight, bn.weight, bn.bias, res], cot)
    xr, rr = x.detach().float().requires_grad_(True), res.detach().float().requires_grad_(True)
    yr = torch.relu(bn_r(conv_r(xr)) + rr)
    grads_r = torch.autograd.grad(yr, [xr, conv_r.weight, bn_r.weight, bn_r.bias, rr], cot.float())
    _close(y, yr, 3e-2)
    for a, b in zip(grads, grads_r):
        _rel_l2(a, b)


@pytest.mark.parametrize("training", [False, True])
def test_tc_conv3x3_fn_autograd(training):
    import copy
    import torch.nn as nn
    from cotnet_b200 import fused
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
    x = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").bfloat16()).requires_grad_(True)
    cot = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").bfloat16())
    y = fused.TcConv3x3Fn.apply(x, conv.weight, bn.weight, bn.bias, bn, 4, True)
    grads = torch.autograd.grad(y, [x, conv.weight, bn.weight, bn.bias], cot)
    xr = x.detach().float().requires_grad_(True)
    yr = torch.relu(bn_r(conv_r(xr)))
    grads_r = torch.autograd.grad(yr, [xr, conv_r.weight, bn_r.weight, bn_r.bias], cot.float())
    _close(y, yr, 3e-2)
    for a, b in zip(grads, grads_r):
        _rel_l2(a, b)


@pytest.mark.parametrize("B,H,W,N", [(2, 224, 224, 64), (3, 64, 96, 64), (1, 32, 480, 32)])
def test_stem7x7s2_vs_conv2d(B, H, W, N):
    """conv1 of the trunk (models/resnet.py:552) on the 4-tap wgmma implicit GEMM against fp32 torch math on the same bf16 operands;
    raw output + BatchNorm column statistics, and the eval epilogue (folded scale / shift + ReLU)."""
    g = torch.Generator(device="cuda").manual_seed(B + H + W)
    x = torch.randn(B, 3, H, W, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    w = (torch.randn(N, 3, 7, 7, generator=g, device="cuda") / 12).bfloat16()
    want = F.conv2d(x.float(), w.float(), None, 2, 3)
    tc = _tc()
    wm = tc.prepare_stem_weight(w)
    cs, cq = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    d = tc.stem7x7s2_bf16(x, wm, stats=(cs, cq))
    assert d is not None, "stem geometry refused"
    assert d.shape == want.shape and d.is_contiguous(memory_format=torch.channels_last)
    _close(d, want)
    assert torch.allclose(cs, d.float().sum((0, 2, 3)), atol=2e-2, rtol=1e-4)
    assert torch.allclose(cq, (d.float() ** 2).sum((0, 2, 3)), atol=2e-2, rtol=1e-4)
    scale = torch.rand(N, generator=g, device="cuda") + 0.5
    shift = torch.randn(N, generator=g, device="cuda")
    d2 = tc.stem7x7s2_bf16(x, wm, scale=scale, shift=shift, relu=True)
    _close(d2, torch.relu(want * scale[None, :, None, None] + shift[None, :, None, None]))


def test_stem_conv_bn_autograd_vs_cudnn_path():
    """fused.stem_conv_bn (wgmma stem + statistics epilogue + fused BatchNorm) against the cuDNN convolution + the same fused
    BatchNorm kernels: outputs, BatchNorm buffers and parameter gradients."""
    import copy
    from cotnet_b200 import fused
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(4, 3, 96, 128, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    conv = torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False).cuda().to(torch.bfloat16)
    bn = torch.nn.BatchNorm2d(64).cuda().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(0, 0.2)
    conv2, bn2 = copy.deepcopy(conv), copy.deepcopy(bn)
    cot = torch.randn(4, 64, 48, 64, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    y1 = fused.stem_conv_bn(x, conv, bn, relu=True)
    y2 = fused.bn_act(conv2(x).contiguous(memory_format=torch.channels_last), bn2, relu=True)
    _close(y1, y2, 2e-2)
    assert torch.allclose(bn.running_mean, bn2.running_mean, atol=1e-3) and torch.allclose(bn.running_var, bn2.running_var, atol=1e-3, rtol=1e-2)
    g1 = torch.autograd.grad(y1, (conv.weight, bn.weight, bn.bias), cot)
    g2 = torch.autograd.grad(y2, (conv2.weight, bn2.weight, bn2.bias), cot)
    for a, b in zip(g1, g2):
        rel = ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-6)).item()
        assert rel <= 3e-2, rel
    # eval mode: BatchNorm folded into the GEMM epilogue
    bn.eval(); bn2.eval()
    with torch.no_grad():
        _close(fused.stem_conv_bn(x, conv, bn, relu=True), fused.bn_act(conv2(x).contiguous(memory_format=torch.channels_last), bn2, relu=True), 2e-2)


@pytest.mark.parametrize("B,H,W,N", [(2, 224, 224, 64), (3, 64, 96, 64), (5, 32, 160, 32)])
def test_stem7x7s2_wgrad_vs_conv2d_weight(B, H, W, N):
    """Weight gradient of the stem convolution on the MN-major wgmma kernel (one stage = one output row over the space-to-depth
    image) against fp32 torch math on the same bf16 operands."""
    g = torch.Generator(device="cuda").manual_seed(B + H)
    x = torch.randn(B, 3, H, W, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    w = (torch.randn(N, 3, 7, 7, generator=g, device="cuda") / 12).bfloat16()
    dy = torch.randn(B, N, H // 2, W // 2, generator=g, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    tc = _tc()
    out, scratch = tc.stem7x7s2_bf16(x, tc.prepare_stem_weight(w), return_scratch=True)
    got = tc.stem7x7s2_wgrad(dy, scratch, x.shape, N)
    assert got is not None, "stem wgrad geometry refused"
    want = torch.nn.grad.conv2d_weight(x.float(), w.shape, dy.float(), stride=2, padding=3)
    rel = ((got - want).norm() / want.norm()).item()
    assert got.shape == want.shape and rel <= 2e-3, rel
