"""GPU tests of the fused normalisation / tail autograd functions against eager PyTorch on the same inputs."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_tf32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _to_tap(t, gc):
    """reference channel order (g*9+t) -> tap-major chunks of gc, on a [B, J, H, W] tensor"""
    if gc == 0:
        return t
    B, J, H, W = t.shape
    wc = J // 9
    return t.view(B, wc // gc, gc, 9, H, W).permute(0, 1, 3, 2, 4, 5).reshape(B, J, H, W)


def _from_tap(t, gc):
    if gc == 0:
        return t
    B, J, H, W = t.shape
    wc = J // 9
    return t.view(B, wc // gc, 9, gc, H, W).permute(0, 1, 3, 2, 4, 5).reshape(B, J, H, W)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("C,wc,H,fold,gc", [(64, 8, 56, 1, 8), (128, 16, 28, 1, 8), (256, 32, 14, 1, 8), (512, 64, 7, 1, 8),
                                           (384, 48, 7, 2, 8), (64, 8, 9, 1, 0), (96, 12, 10, 2, 0), (192, 24, 14, 2, 0)])
def test_agg_tap(dtype, C, wc, H, fold, gc):
    """AggTapFn (block-internal weight order, second-generation kernels) vs the oracle, fwd + dX + dW."""
    from cotnet_b200 import fused
    from oracle import agg_ref
    g = torch.Generator().manual_seed(C + H + gc)
    B = 3
    x64 = torch.randn(B, C, H, H, generator=g, dtype=torch.float64).to(dtype).double()
    w64 = torch.randn(B, 9 * wc, H, H, generator=g, dtype=torch.float64).to(dtype).double()
    c64 = torch.randn(B, C, H, H, generator=g, dtype=torch.float64).to(dtype).double()
    x = _cl(x64.to(dtype).cuda()).requires_grad_(True)
    w = _cl(_to_tap(w64, gc).to(dtype).cuda()).requires_grad_(True)
    y = fused.AggTapFn.apply(x, w, fold, gc)
    gx, gw = torch.autograd.grad(y, (x, w), _cl(c64.to(dtype).cuda()))
    xr, wr = x64.clone().requires_grad_(True), w64.clone().requires_grad_(True)
    # un-folded semantics == the reference's view(B*fold, C/fold, ...) trick (models/cotnet.py:157-162)
    yr = agg_ref.agg_zeropad_unfold(xr.view(B * fold, C // fold, H, H), wr.view(B * fold, 1, wc // fold, 9, H, H), 3, 1, 1, 1)
    yr = yr.view(B, C, H, H)
    gxr, gwr = torch.autograd.grad(yr, (xr, wr), c64)
    tol = 1e-3 if dtype == torch.float32 else 1e-2
    for a, b, name in ((y, yr, "y"), (gx, gxr, "dX"), (_from_tap(gw, gc), gwr, "dW")):
        err = (a.double().cpu() - b).abs()
        assert bool((err <= tol + tol * b.abs()).all()), "%s max err %.3e" % (name, err.max().item())


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-4), (torch.bfloat16, 3e-2)])
@pytest.mark.parametrize("gc", [0, 8])
@pytest.mark.parametrize("wc,H", [(8, 14), (16, 9), (12, 7), (64, 7), (8, 56), (32, 14), (24, 5)])
@pytest.mark.parametrize("with_lbias", [False, True])
def test_groupnorm9(dtype, tol, wc, H, gc, with_lbias):
    if gc and wc % gc:
        pytest.skip("chunk does not divide wc")
    from cotnet_b200 import fused
    g = torch.Generator(device="cuda").manual_seed(wc + H)
    B, J = 5, 9 * wc
    gn = nn.GroupNorm(wc, J).cuda()
    with torch.no_grad():
        gn.weight.uniform_(0.5, 1.5, generator=g)
        gn.bias.normal_(0, 0.3, generator=g)
    l = _cl((torch.randn(B, J, H, H, generator=g, device="cuda") * 2 + 0.5).to(dtype)).requires_grad_(True)
    cot = _cl(torch.randn(B, J, H, H, generator=g, device="cuda").to(dtype))
    # lbias = the embed.3 convolution bias folded into the kernels: GroupNorm(l + bias), gradient from gn9_bwd_apply
    lbias = (torch.randn(J, generator=g, device="cuda") * 0.7).requires_grad_(True) if with_lbias else None
    out_t = fused.group_norm9(l, gn, gc, lbias)
    wanted = (l, gn.weight, gn.bias) + ((lbias,) if with_lbias else ())
    got = torch.autograd.grad(out_t, wanted, _cl(_to_tap(cot, gc)))
    out = _from_tap(out_t, gc)
    lr = l.detach().double().requires_grad_(True)
    br = lbias.detach().double().requires_grad_(True) if with_lbias else None
    gnr = nn.GroupNorm(wc, J).cuda().double()
    gnr.load_state_dict(gn.state_dict())
    ref = gnr(lr + br.view(1, J, 1, 1)) if with_lbias else gnr(lr)
    refs = torch.autograd.grad(ref, (lr, gnr.weight, gnr.bias) + ((br,) if with_lbias else ()), cot.double())
    for a, b, name in zip((out,) + tuple(got), (ref,) + tuple(refs), ("out", "dl", "dgamma", "dbeta", "dlbias")):
        err = (a.double() - b).abs().max().item()
        scale = max(1.0, b.abs().max().item())
        assert err <= tol * scale, "%s err %.3e scale %.3e" % (name, err, scale)
    assert out_t.is_contiguous(memory_format=torch.channels_last) and out_t.dtype == dtype


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C,H", [(64, 14), (24, 9), (3, 5)])
def test_fan_out_sums_gradients(dtype, C, H):
    """fused.fan_out: one cotb200_sum_rows launch accumulates the gradients of all consumers, reading the channel
    slices of a concat gradient (pitch 2C) in place; must equal autograd's own accumulation."""
    from cotnet_b200 import fused
    g = torch.Generator(device="cuda").manual_seed(C * H)
    B = 3
    x = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype)).requires_grad_(True)
    wgt = [torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype) for _ in range(2)]
    wcat = _cl(torch.randn(B, 2 * C, H, H, generator=g, device="cuda").to(dtype))

    def graph(a, b, c):
        # consumer 1: elementwise; consumer 2: first half of a concat (sliced, pitch-2C gradient); consumer 3: NCHW product
        cat = torch.cat([b, torch.zeros_like(b)], dim=1) * wcat
        return (a * _cl(wgt[0])).sum() + cat.sum() + (c * wgt[1]).sum()

    a, b, c = fused.fan_out(x, 3)
    (gx,) = torch.autograd.grad(graph(a, b, c), x)
    xr = x.detach().double().requires_grad_(True)
    ref = (xr * wgt[0].double()).sum() + (xr * wcat[:, :C].double()).sum() + (xr * wgt[1].double()).sum()
    (gr,) = torch.autograd.grad(ref, xr)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    err = (gx.double() - gr).abs()
    assert bool((err <= tol + tol * gr.abs()).all()), "max err %.3e" % err.max().item()
    assert gx.is_contiguous(memory_format=torch.channels_last) or C == 1
    # no-grad: pass-through
    with torch.no_grad():
        assert all(t is x for t in fused.fan_out(x, 2))


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 5e-4), (torch.bfloat16, 4e-2)])
@pytest.mark.parametrize("C,H", [(64, 14), (128, 7), (48, 9), (512, 7)])
@pytest.mark.parametrize("training", [False, True])
def test_cot_tail(dtype, tol, C, H, training):
    from cotnet_b200 import fused
    g = torch.Generator(device="cuda").manual_seed(C + H)
    B, A = 16, max(C // 2, 32)
    # the SE convolutions are initialised from a seed of this test, not from whatever the global generator holds after the tests
    # that ran before: in training mode the gradient of se[0].bias is zero in exact arithmetic (a batch-statistics BatchNorm
    # follows), so what is compared for it is rounding noise, and its size depends on these weights
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(C + H)
        bn = nn.BatchNorm2d(C).cuda()
        se = nn.Sequential(nn.Conv2d(C, A, 1), nn.BatchNorm2d(A), nn.ReLU(inplace=True), nn.Conv2d(A, 2 * C, 1)).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5, generator=g); bn.bias.normal_(0, 0.3, generator=g)
        bn.running_mean.normal_(0, 0.3, generator=g); bn.running_var.uniform_(0.5, 2, generator=g)
        se[1].running_mean.normal_(0, 0.1, generator=g); se[1].running_var.uniform_(0.5, 2, generator=g)
    import copy
    bn_r, se_r = copy.deepcopy(bn).double(), copy.deepcopy(se).double()
    for m in (bn, se, bn_r, se_r):
        m.train(training)
    u = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype)).requires_grad_(True)
    k = _cl(torch.relu(torch.randn(B, C, H, H, generator=g, device="cuda")).to(dtype)).requires_grad_(True)
    cot = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype))
    out = fused.cot_tail(u, k, bn, se)
    params = [bn.weight, bn.bias] + list(se.parameters())
    grads = torch.autograd.grad(out, [u, k] + params, cot)
    # eager reference in fp64 (models/cotnet.py:89-104)
    ur, kr = u.detach().double().requires_grad_(True), k.detach().double().requires_grad_(True)
    y = F.silu(bn_r(ur))
    gap = (y + kr).mean((2, 3), keepdim=True)
    a = torch.softmax(se_r(gap).view(B, C, 2), 2)
    ref = y * a[:, :, 0].reshape(B, C, 1, 1) + kr * a[:, :, 1].reshape(B, C, 1, 1)
    params_r = [bn_r.weight, bn_r.bias] + list(se_r.parameters())
    grads_r = torch.autograd.grad(ref, [ur, kr] + params_r, cot.double())
    err = (out.double() - ref).abs().max().item()
    assert err <= tol * max(1.0, ref.abs().max().item()), "out err %.3e" % err
    for i, (a_, b_) in enumerate(zip(grads, grads_r)):
        e = (a_.double() - b_).abs().max().item()
        s = max(1.0, b_.abs().max().item())
        assert e <= 4 * tol * s, "grad %d err %.3e scale %.3e" % (i, e, s)
    if training:
        assert torch.allclose(bn.running_mean.double(), bn_r.running_mean, atol=1e-2 if dtype != torch.float32 else 1e-5)
        assert torch.allclose(bn.running_var.double(), bn_r.running_var, atol=1e-2 if dtype != torch.float32 else 1e-4)
        assert int(bn.num_batches_tracked) == 1


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-4), (torch.bfloat16, 3e-2)])
@pytest.mark.parametrize("C,H", [(64, 14), (256, 7), (96, 9), (2048, 7)])
@pytest.mark.parametrize("relu,res", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("training", [False, True])
def test_bn_act(dtype, tol, C, H, relu, res, training):
    """Fused BatchNorm2d (+residual) (+ReLU) vs eager fp64 modules: output, dX, dres, dgamma, dbeta, running buffers."""
    import copy
    from cotnet_b200 import fused
    g = torch.Generator(device="cuda").manual_seed(C + H)
    B = 8
    bn = nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5, generator=g); bn.bias.normal_(0, 0.3, generator=g)
        bn.running_mean.normal_(0, 0.3, generator=g); bn.running_var.uniform_(0.5, 2, generator=g)
    bn_r = copy.deepcopy(bn).double()
    bn.train(training); bn_r.train(training)
    x = _cl((torch.randn(B, C, H, H, generator=g, device="cuda") * 1.5 + 0.3).to(dtype)).requires_grad_(True)
    r = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype)).requires_grad_(True) if res else None
    cot = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype))
    y = fused.bn_act(x, bn, relu=relu, res=r)
    ins = [x, bn.weight, bn.bias] + ([r] if res else [])
    grads = torch.autograd.grad(y, ins, cot)
    xr = x.detach().double().requires_grad_(True)
    rr = r.detach().double().requires_grad_(True) if res else None
    z = bn_r(xr)
    if res:
        z = z + rr
    yr = torch.relu(z) if relu else z
    grads_r = torch.autograd.grad(yr, [xr, bn_r.weight, bn_r.bias] + ([rr] if res else []), cot.double())
    assert (y.double() - yr).abs().max().item() <= tol * max(1.0, yr.abs().max().item())
    for i, (a, b) in enumerate(zip(grads, grads_r)):
        e = (a.double() - b).abs().max().item()
        assert e <= 4 * tol * max(1.0, b.abs().max().item()), "grad %d err %.3e" % (i, e)
    if training:
        assert torch.allclose(bn.running_mean.double(), bn_r.running_mean, atol=2e-2 if dtype != torch.float32 else 1e-5)
        assert torch.allclose(bn.running_var.double(), bn_r.running_var, atol=2e-2 if dtype != torch.float32 else 1e-4)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C,H,W", [(64, 56, 56), (128, 28, 28), (64, 112, 112), (24, 9, 7), (256, 14, 14)])
@pytest.mark.parametrize("mode", [0, 1])
def test_pool3x3s2(dtype, C, H, W, mode):
    """Fused NHWC pooling vs nn.AvgPool2d(3,2,1) / nn.MaxPool2d(3,2,1): forward and backward (ties included: ReLU'd input)."""
    from cotnet_b200 import fused
    g = torch.Generator(device="cuda").manual_seed(C + H)
    B = 3
    x = _cl(torch.relu(torch.randn(B, C, H, W, generator=g, device="cuda")).to(dtype)).requires_grad_(True)
    y = fused.avg_pool3x3s2(x) if mode == 0 else fused.max_pool3x3s2(x)
    ref_mod = nn.AvgPool2d(3, 2, padding=1) if mode == 0 else nn.MaxPool2d(3, 2, 1)
    # NCHW-contiguous reference on purpose: ATen's channels_last avg_pool2d BACKWARD kernel of this torch build
    # (avg_pool2d_backward_out_cuda_frame_nhwc) disagrees with its own NCHW and CPU implementations by O(1)
    # (tools/debug_pool.py); the NCHW path is the semantic definition.
    xr = x.detach().float().contiguous().requires_grad_(True)
    yr = ref_mod(xr)
    cot = _cl(torch.randn(yr.shape, generator=g, device="cuda").to(dtype))
    (gx,) = torch.autograd.grad(y, x, cot)
    (gxr,) = torch.autograd.grad(yr, xr, cot.float().contiguous())
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert y.shape == yr.shape and y.is_contiguous(memory_format=torch.channels_last)
    assert (y.float() - yr).abs().max().item() <= tol * max(1.0, yr.abs().max().item())
    assert (gx.float() - gxr).abs().max().item() <= tol * max(1.0, gxr.abs().max().item())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C,H,B", [(64, 14, 5), (512, 7, 17), (96, 8, 3)])
def test_cot_tail_eval_kernel_path(dtype, C, H, B):
    """Inference tail (tail_pool -> cotb200_se_eval -> tail_combine, no autograd) against the autograd-capable path (PyTorch
    SE MLP) and against the plain formula of models/cotnet.py:89-104."""
    import torch.nn as nn
    from cotnet_b200 import fused
    g = torch.Generator(device="cuda").manual_seed(C + B)
    A = max(C // 2, 32)
    bn = nn.BatchNorm2d(C).cuda()
    se = nn.Sequential(nn.Conv2d(C, A, 1), nn.BatchNorm2d(A), nn.ReLU(inplace=True), nn.Conv2d(A, 2 * C, 1)).cuda()
    with torch.no_grad():
        for m in (bn, se[1]):
            m.weight.uniform_(0.5, 1.5, generator=g); m.bias.normal_(0, 0.3, generator=g)
            m.running_mean.normal_(0, 0.3, generator=g); m.running_var.uniform_(0.5, 2.0, generator=g)
    bn.eval(); se.eval()
    u = torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
    k = torch.relu(torch.randn(B, C, H, H, generator=g, device="cuda")).to(dtype).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        got = fused.cot_tail(u, k, bn, se)                       # kernel path (grad disabled, eval)
        y = torch.nn.functional.silu(bn(u.float()))
        gap = (y + k.float()).mean((2, 3), keepdim=True)
        a = torch.softmax(se(gap).view(B, C, 2), dim=2)
        want = y * a[:, :, 0].reshape(B, C, 1, 1) + k.float() * a[:, :, 1].reshape(B, C, 1, 1)
    with torch.enable_grad():
        ref2 = fused.cot_tail(u.clone().requires_grad_(True), k, bn, se)     # autograd path (PyTorch MLP)
    tol = 1e-4 if dtype == torch.float32 else 1.5e-2
    assert torch.allclose(got.float(), want, atol=tol, rtol=tol), (got.float() - want).abs().max().item()
    assert torch.allclose(got.float(), ref2.float(), atol=tol, rtol=tol)


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-4), (torch.bfloat16, 2e-2)])
@pytest.mark.parametrize("path", ["bn_act", "tc_conv1x1"])
def test_forked_output_sums_the_two_gradients_in_the_bn_backward(dtype, tol, path, monkeypatch):
    """fork=True: the output comes as two aliases; the gradients of their two consumers are summed inside the BatchNorm backward
    kernels (cotb200_bn_bwd_{sums,apply}2) -- same parameter / input / residual gradients as the un-forked op behind an autograd add."""
    import copy
    from cotnet_b200 import fused
    if path == "tc_conv1x1" and dtype != torch.bfloat16:
        pytest.skip("the wgmma path is bf16 only")
    g = torch.Generator(device="cuda").manual_seed(17)
    B, K, N, H = 6, 64, 128, 14
    x = torch.randn(B, K if path == "tc_conv1x1" else N, H, H, generator=g, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
    r = torch.randn(B, N, H, H, generator=g, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
    c1 = torch.randn(B, N, H, H, generator=g, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
    c2 = torch.randn(B, N, H, H, generator=g, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
    bn = torch.nn.BatchNorm2d(N).cuda().train()
    conv = torch.nn.Conv2d(K, N, 1, bias=False).cuda().to(dtype)
    if path == "tc_conv1x1":
        monkeypatch.setattr(fused, "trunk_conv_backend", "tc_all1x1")
        monkeypatch.setattr(fused, "TC_MIN_PIXELS", 0)
    res = []
    for fork in (False, True):
        bn_, conv_ = copy.deepcopy(bn), copy.deepcopy(conv)
        xx, rr = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
        if path == "bn_act":
            out = fused.bn_act(xx, bn_, relu=True, res=rr, fork=fork)
        else:
            out = fused.conv1x1_bn(xx, conv_, bn_, relu=True, res=rr, fork=fork)
        ya, yb = out if fork else (out, out)
        assert (not fork) or (ya.data_ptr() == yb.data_ptr() and ya is not yb)
        ((ya.float() * c1.float()).sum() + (yb.float() * c2.float()).sum()).backward()
        res.append([xx.grad.float(), rr.grad.float(), bn_.weight.grad.float(), bn_.bias.grad.float()] +
                   ([conv_.weight.grad.float()] if path != "bn_act" else []))
    for a, b in zip(*res):
        rel = ((a - b).norm() / b.norm().clamp_min(1e-6)).item()
        assert rel <= tol, rel
