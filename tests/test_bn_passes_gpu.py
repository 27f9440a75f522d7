"""The BatchNorm backward without reading the forward output back: the 1-bit ReLU mask of residual BatchNorms (relu code 3) and
the mask recomputed from the pre-activation on the wgmma convolutions (relu code 2).  Both must reproduce the y-reading path
(relu code 1) bit for bit: kernels, autograd functions, and three graph-replayed training steps of cotnet50."""
import copy

import pytest
import torch

from cotnet_b200 import _lib, backbone, fused, trainer

pytestmark = pytest.mark.gpu


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _p(t):
    return _lib.ptr(t)


# ------------------------------------------------------------------------------------------------ mask kernels (C ABI)
def _inputs(dtype, B, HW, C, seed):
    """x, res, dy, dy2 [B*HW, C] with exact zeros and values next to zero in x, res and the residual sum, so that the stored
    y has exact zeros, tiny positives and tiny negatives clamped to zero."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = B * HW
    x = torch.randn(n, C, generator=g, device="cuda")
    x[::5] = 0.0
    x[1::7, ::3] = 1e-30
    res = torch.randn(n, C, generator=g, device="cuda")
    res[2::5] = 0.0
    res[3::11, 1::4] = -1e-30
    res[4::13, 2::4] = 1e-38
    dy = torch.randn(n, C, generator=g, device="cuda")
    dy2 = torch.randn(n, C, generator=g, device="cuda")
    return [t.to(dtype).contiguous() for t in (x, res, dy, dy2)]


def _forward(lib, dt, B, HW, C, x, res, ds, mask):
    """col_stats + training-mode apply (relu, residual): (y, [4, C] scale/shift/mean/rstd, running mean/var)."""
    st = torch.cuda.current_stream().cuda_stream
    sums = torch.zeros(2, C, device="cuda")
    _lib.check(lib.cotb200_col_stats(dt, B, HW, C, _p(x), _p(sums[0]), _p(sums[1]), st), "col_stats")
    w = torch.linspace(0.5, 1.5, C, device="cuda")
    b = torch.linspace(-0.3, 0.3, C, device="cuda")
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    ss = torch.empty(4, C, device="cuda")
    y = torch.empty_like(x)
    args = (dt, B, HW, C, _p(x), _p(res), _p(sums[0]), _p(sums[1]), _p(w), _p(b), _p(rm), _p(rv), float(B * HW), 1e-5, 0.1, 1)
    outs = (_p(y), _p(ss[0]), _p(ss[1]), _p(ss[2]), _p(ss[3]))
    if mask is not None:
        _lib.check(lib.cotb200_bn_apply_batch_mask(*args, *outs, _p(ds), _p(mask), st), "bn_apply_batch_mask")
    elif ds is not None:
        _lib.check(lib.cotb200_bn_apply_batch_ds(*args, 1, *outs, _p(ds), st), "bn_apply_batch_ds")
    else:
        _lib.check(lib.cotb200_bn_apply_batch(*args, 1, *outs, st), "bn_apply_batch")
    return y, ss, rm, rv


def _backward(lib, dt, B, HW, C, dy, dy2, x, y_or_mask, ss, ds, rcode):
    st = torch.cuda.current_stream().cuda_stream
    sums = torch.zeros(2, C, device="cuda")
    dx, dres = torch.empty_like(x), torch.empty_like(x)
    scale, mean, rstd = ss[0], ss[2], ss[3]
    inv_n = 1.0 / (B * HW)
    if rcode == 3:
        _lib.check(lib.cotb200_bn_bwd_sums_mask(dt, B, HW, C, _p(dy), _p(dy2), _p(x), _p(y_or_mask), _p(mean), _p(rstd), _p(sums[0]),
                                                _p(sums[1]), _p(ds), st), "bn_bwd_sums_mask")
        _lib.check(lib.cotb200_bn_bwd_apply_mask(dt, B, HW, C, _p(dy), _p(dy2), _p(x), _p(y_or_mask), _p(scale), _p(mean), _p(rstd),
                                                 _p(sums[0]), _p(sums[1]), inv_n, _p(dx), _p(dres), _p(ds), st), "bn_bwd_apply_mask")
    else:
        _lib.check(lib.cotb200_bn_bwd_sums_ds(dt, B, HW, C, _p(dy), _p(dy2), _p(x), _p(y_or_mask), _p(scale), None, _p(mean), _p(rstd),
                                              1, _p(sums[0]), _p(sums[1]), _p(ds), st), "bn_bwd_sums_ds")
        _lib.check(lib.cotb200_bn_bwd_apply_ds(dt, B, HW, C, _p(dy), _p(dy2), _p(x), _p(y_or_mask), _p(scale), None, _p(mean), _p(rstd),
                                               _p(sums[0]), _p(sums[1]), inv_n, 1, _p(dx), _p(dres), _p(ds), st), "bn_bwd_apply_ds")
    return sums, dx, dres


def _unpack(mask, C):
    bits = torch.arange(8, device=mask.device, dtype=torch.uint8)
    return ((mask.unsqueeze(-1) >> bits) & 1).reshape(mask.shape[0], -1)[:, :C].bool()


@pytest.mark.parametrize("ds_on", [False, True])
@pytest.mark.parametrize("two", [False, True])
@pytest.mark.parametrize("C", [64, 2048, 200])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_mask_kernels_equal_y_path(dtype, C, two, ds_on):
    """Forward: the mask form writes the same y, statistics and running buffers as the plain form, and its mask is [y > 0].
    Backward: sums, dx and dres from the mask (code 3) equal those from y (code 1) bit for bit, with and without a second incoming
    gradient and drop-path scales.  C = 2048 in fp32 runs in column chunks; C = 200 is not a multiple of 64 (fp32: two threads
    share each mask byte)."""
    lib = _lib.load()
    dt = _lib.dtype_code(torch.empty(0, dtype=dtype))
    B, HW = 3, 37
    x, res, dy, dy2 = _inputs(dtype, B, HW, C, seed=C + (1 if two else 0))
    dy2 = dy2 if two else None
    ds = torch.tensor([2.0, 0.0, 1.25], device="cuda") if ds_on else None
    y1, ss1, rm1, rv1 = _forward(lib, dt, B, HW, C, x, res, ds, None)
    mask = torch.full((B * HW, C // 8), 0xA5, dtype=torch.uint8, device="cuda")     # garbage: every byte must be written
    y3, ss3, rm3, rv3 = _forward(lib, dt, B, HW, C, x, res, ds, mask)
    assert torch.equal(y1, y3) and torch.equal(ss1, ss3) and torch.equal(rm1, rm3) and torch.equal(rv1, rv3)
    m = _unpack(mask, C)
    assert torch.equal(m, y1.float() > 0)
    assert (y1 == 0).any() and m.any() and (~m).any()
    got = _backward(lib, dt, B, HW, C, dy, dy2, x, mask, ss3, ds, 3)
    want = _backward(lib, dt, B, HW, C, dy, dy2, x, y1, ss1, ds, 1)
    for a, b, name in zip(got, want, ("sums", "dx", "dres")):
        assert torch.equal(a, b), name


def test_mask_entry_points_reject_bad_channels():
    lib = _lib.load()
    x = torch.zeros(4, 12, device="cuda", dtype=torch.bfloat16)
    m = torch.zeros(4, 2, dtype=torch.uint8, device="cuda")
    f = torch.zeros(12, device="cuda")
    rc = lib.cotb200_bn_bwd_sums_mask(_lib.BF16, 1, 4, 12, _p(x), None, _p(x), _p(m), _p(f), _p(f), _p(f), _p(f), None, None)
    assert rc == -1                      # COTB200_EINVAL: C % 8 != 0
    rc = lib.cotb200_bn_bwd_apply_mask(_lib.BF16, 1, 4, 8, _p(x), None, _p(x), None, _p(f), _p(f), _p(f), None, None, 0.25,
                                       _p(x), None, None, None)
    assert rc == -5                      # COTB200_ENULL: no mask


# ------------------------------------------------------------------------------------------------ autograd functions
def _bn(C, g):
    bn = torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5, generator=g)
        bn.bias.normal_(0, 0.3, generator=g)
    return bn


def _run_both(monkeypatch, fn):
    """fn() -> list of tensors, once with BN_MASK on and once off (fresh module copies inside fn); both must be equal bitwise."""
    monkeypatch.setattr(fused, "BN_MASK", True)
    a = fn()
    monkeypatch.setattr(fused, "BN_MASK", False)
    b = fn()
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), "output %d differs" % i


@pytest.mark.parametrize("res", [False, True])
def test_tc_conv1x1_mask_paths(monkeypatch, res):
    """TcConv1x1Fn with ReLU: code 2 (no residual) or the 1-bit mask (residual) against code 1."""
    g = torch.Generator(device="cuda").manual_seed(11)
    B, K, N, H = 4, 64, 256, 14
    conv = torch.nn.Conv2d(K, N, 1, bias=False).cuda()
    bn0 = _bn(N, g)
    x0 = _cl(torch.randn(B, K, H, H, generator=g, device="cuda").bfloat16())
    r0 = _cl(torch.randn(B, N, H, H, generator=g, device="cuda").bfloat16())
    cot = _cl(torch.randn(B, N, H, H, generator=g, device="cuda").bfloat16())

    def run():
        bn = copy.deepcopy(bn0)
        x = x0.clone().requires_grad_(True)
        r = r0.clone().requires_grad_(True) if res else None
        y = fused.TcConv1x1Fn.apply(x, None, conv.weight, None, bn.weight, bn.bias, bn, True, r)
        ins = [x, conv.weight, bn.weight, bn.bias] + ([r] if res else [])
        return [y] + list(torch.autograd.grad(y, ins, cot)) + [bn.running_mean, bn.running_var]
    _run_both(monkeypatch, run)


def test_tc_conv3x3_code2(monkeypatch):
    g = torch.Generator(device="cuda").manual_seed(12)
    B, C, H = 4, 128, 14
    conv = torch.nn.Conv2d(C, C, 3, padding=1, groups=4, bias=False).cuda()
    bn0 = _bn(C, g)
    x0 = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").bfloat16())
    cot = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").bfloat16())

    def run():
        bn = copy.deepcopy(bn0)
        x = x0.clone().requires_grad_(True)
        y = fused.TcConv3x3Fn.apply(x, conv.weight, bn.weight, bn.bias, bn, 4, True)
        return [y] + list(torch.autograd.grad(y, [x, conv.weight, bn.weight, bn.bias], cot))
    _run_both(monkeypatch, run)


def test_stem_code2(monkeypatch):
    g = torch.Generator(device="cuda").manual_seed(13)
    B, H, N = 2, 64, 64
    conv = torch.nn.Conv2d(3, N, 7, stride=2, padding=3, bias=False).cuda()
    bn0 = _bn(N, g)
    x0 = _cl(torch.randn(B, 3, H, H, generator=g, device="cuda").bfloat16())
    cot = _cl(torch.randn(B, N, H // 2, H // 2, generator=g, device="cuda").bfloat16())

    def run():
        bn = copy.deepcopy(bn0)
        y = fused.StemConvBNFn.apply(x0, conv.weight, bn.weight, bn.bias, bn, True)
        return [y] + list(torch.autograd.grad(y, [conv.weight, bn.weight, bn.bias], cot))
    _run_both(monkeypatch, run)


# ------------------------------------------------------------------------------------------------ model level
def _train_state(m0, x, y):
    ts = trainer.TrainStep(copy.deepcopy(m0), lr=0.002, momentum=0.9, weight_decay=1e-3, nesterov=True, ema_decay=0.99,
                           amp_dtype=torch.bfloat16, weights="bf16")
    info = ts.capture(x, y, warmup=2)
    assert info["cuda_graph"]
    losses = [ts.step(x, y).clone() for _ in range(3)]
    torch.cuda.synchronize()
    st = {"loss": torch.stack([l_.detach().float().reshape(()) for l_ in losses])}
    for kind, d in (("master", ts.master_state()), ("grad", ts.grads()), ("ema", ts.ema_state())):
        for n, t in d.items():
            st["%s:%s" % (kind, n)] = t.detach().clone()
    for n in ("M_big", "M_small"):
        st["momentum:" + n] = getattr(ts, n).clone()
    for n, b in ts.model.named_buffers():
        st["buffer:" + n] = b.detach().clone()
    return st


def test_cotnet50_steps_equal_with_and_without_masks(monkeypatch):
    """Three graph-replayed training steps of cotnet50 (batch 4, 128x128, the stage 1-2 bottleneck convolutions on the wgmma
    path) give bitwise-equal loss, gradients, master weights, momentum, EMA and BatchNorm buffers with the masks on and off."""
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(fused, "TC_MIN_PIXELS", 0)
    torch.manual_seed(21)
    m0 = backbone.cotnet50(zero_init_last_bn=False).cuda().to(memory_format=torch.channels_last).train()
    g0 = torch.Generator().manual_seed(22)
    x = torch.randn(4, 3, 128, 128, generator=g0).cuda().to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (4,), generator=g0).cuda()
    monkeypatch.setattr(fused, "BN_MASK", True)
    on = _train_state(m0, x, y)
    monkeypatch.setattr(fused, "BN_MASK", False)
    off = _train_state(m0, x, y)
    assert on.keys() == off.keys()
    differ = [k for k in on if not torch.equal(on[k], off[k])]
    assert not differ, differ[:5]
