"""DropBlock on the GPU: the mask kernel against the host restatement of the stream (tests/golden/dropblock.npz geometries and
one site of >= 2^24 elements), the apply and residual-tail kernels against torch / fp64 compositions, the blocks' fused paths
against their fp64 unfused paths with the same key, the bench-path training step against the reference's fp64 step, and the
captured step's replays."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, backbone, backbone_hybrid, dropblock, fused, trainer
from cotnet_b200.backbone_hybrid import CoTBottleneck

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "dropblock.npz"))
CL = torch.channels_last
MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


def _geo(i):
    B, C, H, W, bs, gs, rate, site, k0, k1 = GOLDEN["geo_params"][i]
    return (int(B), int(C), int(H), int(W)), dropblock.DropBlock(rate, int(bs), gs), int(site), (int(k0), int(k1))


def _bits_to_nchw(mask, shape):
    """[B*H*W, C/8] uint8 -> bool [B, C, H, W] (bit c%8 of byte c/8)."""
    B, C, H, W = shape
    bits = (mask.cpu().numpy()[:, :, None] >> np.arange(8, dtype=np.uint8)) & 1
    return bits.reshape(B, H, W, C).transpose(0, 3, 1, 2).astype(bool)


def _device_mask(shape, site, key, spec, dtype=torch.bfloat16):
    x = torch.zeros(shape, dtype=dtype, device="cuda").contiguous(memory_format=CL)
    return dropblock.device_mask(x, torch.tensor(key, dtype=torch.int64, device="cuda"), site, spec)


LARGE = ((64, 1024, 16, 16), dropblock.DropBlock(0.1, 5, 0.25), 11, (987654321, 123456789))      # 2^24 elements
# planes at the mask kernel's 48 KB shared-memory budget: layer3 block 0's bn1 site of CoTNet-50 at 256x384 and 384x512 inputs
# (16 and 8 channel groups would need 48 KB + the per-warp counts; the call takes 8 and 4), and the largest single-group plane
EXTRA = {"l3_256x384": ((2, 256, 32, 48), dropblock.DropBlock(0.1, 5, 0.25), 4, (11, 12)),
         "l3_384x512": ((1, 256, 48, 64), dropblock.DropBlock(0.1, 5, 0.25), 5, (13, 14)),
         "plane_24560": ((1, 8, 1, 24560), dropblock.DropBlock(0.1, 1, 1.0), 6, (15, 16))}


@pytest.mark.parametrize("i", list(range(len(GOLDEN["geo_params"]))) + ["large"] + sorted(EXTRA))
def test_mask_bits_count_and_scale_equal_host(i):
    shape, spec, site, key = LARGE if i == "large" else (EXTRA[i] if i in EXTRA else _geo(i))
    keep, count, scale = dropblock.host_mask(shape, site, key, spec)
    mask, cnt = _device_mask(shape, site, key, spec)
    assert np.array_equal(_bits_to_nchw(mask, shape), keep)
    assert int(cnt.item()) == count
    if isinstance(i, int):
        assert count == int(GOLDEN["geo%d_count" % i])
    ones = torch.ones(shape, dtype=torch.float32, device="cuda").contiguous(memory_format=CL)
    y = dropblock.DropBlockFn.apply(ones, mask, cnt)
    s = np.float32(scale)
    assert np.array_equal(y.cpu().numpy().view(np.int32), (keep * s).astype(np.float32).view(np.int32))
    if count and i == "large":      # torch's own fp32 sum of a >= 2^24-element mask is rounded: within 1 ulp of it
        m = torch.from_numpy(keep).cuda().float()
        st = (m.numel() / m.sum().add(1e-7)).item()
        assert abs(np.float32(st).view(np.int32) - s.view(np.int32)) <= 1


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("i", [0, 1, 5, 9, 14, 15])
def test_apply_forward_backward_equal_torch(dtype, i):
    shape, spec, site, key = _geo(i)
    mask, cnt = _device_mask(shape, site, key, spec)
    keep, count, scale = dropblock.host_mask(shape, site, key, spec)
    g = torch.Generator(device="cuda").manual_seed(i)
    x = torch.randn(shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=CL).requires_grad_(True)
    dy = torch.randn(shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=CL)
    y = dropblock.DropBlockFn.apply(x, mask, cnt)
    y.backward(dy)
    xr = x.detach().clone().requires_grad_(True)
    m = torch.from_numpy(keep).cuda().to(dtype)
    yr = xr * m * torch.tensor(float(scale), dtype=torch.float32, device="cuda").to(dtype)        # the reference's composition
    yr.backward(dy)
    iv = torch.int16 if dtype == torch.bfloat16 else torch.int32
    assert torch.equal(y.detach().contiguous().view(iv), yr.detach().contiguous().view(iv))
    assert torch.equal(x.grad.contiguous().view(iv), xr.grad.contiguous().view(iv))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("with_ds", [False, True])
def test_residual_tail_matches_fp64(dtype, with_ds):
    shape, spec, site, key = (8, 64, 14, 14), dropblock.DropBlock(0.1, 5, 0.25), 3, (5, 6)
    g = torch.Generator(device="cuda").manual_seed(7)
    z = torch.randn(shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=CL).requires_grad_(True)
    res = torch.randn(shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=CL).requires_grad_(True)
    dy = torch.randn(shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=CL)
    ds = torch.tensor([0., 1.25, 1.25, 0., 1.25, 1.25, 1.25, 1.25], device="cuda") if with_ds else None
    keydev = torch.tensor(key, device="cuda")
    mask, cnt = dropblock.device_mask(z, keydev, site, spec)
    y = dropblock.DropBlockResReluFn.apply(z, res, mask, cnt, ds)
    y.backward(dy)
    keep, count, scale = dropblock.host_mask(shape, site, key, spec)
    s = float(torch.tensor(float(scale)).to(dtype))
    zr, rr = z.detach().double().requires_grad_(True), res.detach().double().requires_grad_(True)
    a = zr * torch.from_numpy(keep).cuda().double() * s
    if with_ds:
        a = a * ds.double().view(-1, 1, 1, 1)
    yr = torch.relu(a + rr)
    yr.backward(dy.double())
    tol = 1e-2 if dtype == torch.bfloat16 else 1e-6
    for got, want in ((y, yr), (z.grad, zr.grad), (res.grad, rr.grad)):
        assert torch.allclose(got.double(), want.detach(), rtol=tol, atol=tol)
    # the 1-bit ReLU mask the forward keeps for its backward equals (out > 0)
    ctx_mask = torch.empty_like(mask)
    B, C, H, W = shape
    yy = torch.empty_like(z, memory_format=CL)
    _lib.check(_lib.load().cotb200_dropblock_res_relu(_lib.dtype_code(z), B, H * W, C, z.data_ptr(), res.data_ptr(), mask.data_ptr(),
                                                      cnt.data_ptr(), _lib.ptr(ds), yy.data_ptr(), ctx_mask.data_ptr(),
                                                      _lib.stream_ptr(z)), "dropblock_res_relu")
    assert torch.equal(yy, y.detach())
    assert np.array_equal(_bits_to_nchw(ctx_mask, shape), (y.detach() > 0).cpu().numpy())


def _block_cases():
    from cotnet_b200.backbone import Bottleneck
    torch.manual_seed(0)
    yield "cotnet", Bottleneck(256, 64, 1, None), (4, 256, 14, 14)
    yield "cotnext", Bottleneck(256, 64, 1, None, cardinality=2, base_width=48), (4, 256, 14, 14)
    yield "cot_bottleneck", CoTBottleneck(0, 256, 64, 1, None), (4, 256, 14, 14)
    yield "split_attn", CoTBottleneck(1, 256, 64, 1, None, conv_dim={64}), (4, 256, 14, 14)


def _block_errors(blk, ref, shape, key):
    """Relative errors (output, input gradient) of the fused bf16 block against its fp64 unfused copy, drop path on."""
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(shape, device="cuda", generator=g)
    dy = torch.randn(shape, device="cuda", generator=g)
    ds = torch.tensor([1.25, 0., 1.25, 1.25], device="cuda")
    xf = x.to(torch.bfloat16).contiguous(memory_format=CL).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = blk(xf, drop_scale=ds, drop_block_key=key)
    y.float().backward(dy)
    xr = xf.detach().double().contiguous().requires_grad_(True)
    yr = ref(xr, drop_scale=ds.double(), drop_block_key=key)
    yr.backward(dy.double())

    def rel(a, b):
        return ((a.double() - b).norm() / b.norm()).item()
    return rel(y.detach(), yr.detach()), rel(xf.grad, xr.grad), yr.detach()


@pytest.mark.parametrize("case", ["cotnet", "cotnext", "cot_bottleneck", "split_attn"])
def test_block_fused_matches_fp64_unfused(case):
    """The fused block with DropBlock (the same key, so the same masks) against its fp64 unfused path: the output within 3 %,
    and the input gradient within 1.5x (+1 %) of the same block's error without DropBlock."""
    name, blk, shape = [c for c in _block_cases() if c[0] == case][0]
    with torch.no_grad():
        for m in blk.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
    key = torch.tensor([31, 41], dtype=torch.int64, device="cuda")
    errs = {}
    for spec in (None, dropblock.DropBlock(0.3, 5, 0.25)):
        blk.set_drop_block(spec, 4)
        ref = copy.deepcopy(blk).cuda().double().train()
        fb = copy.deepcopy(blk).cuda().to(memory_format=CL).train()
        errs[spec is not None] = _block_errors(fb, ref, shape, key)
    assert (case == "split_attn") == (len(blk.drop_block_sites) == 3)
    (ey, edx, yr), (ey0, edx0, yr0) = errs[True], errs[False]
    assert ((yr - yr0).norm() / yr0.norm()).item() > 0.1           # the masks drop something
    assert ey < 3e-2, (ey, edx, ey0, edx0)
    assert edx <= 1.5 * edx0 + 1e-2, (ey, edx, ey0, edx0)


# ------------------------------------------------------------------------------------------------ the step vs the reference
def _step_errors(name, monkeypatch):
    from oracle import make_golden
    from test_trainer_gpu import _grad_errors
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_dropblock_golden import step_input
    pre = "step_%s_" % name
    g = {"names": GOLDEN[pre + "names"], "seed": GOLDEN["step_seed"], "gnorm": GOLDEN[pre + "gnorm"], "gproj": GOLDEN[pre + "gproj"]}
    seed, smooth = int(GOLDEN["step_seed"]), float(GOLDEN["step_smoothing"])
    x, y = step_input()
    x, y = x.cuda(), y.cuda()
    fn = backbone.cotnet50 if name == "cotnet50" else backbone_hybrid.se_cotnetd_50
    m = make_golden.hybrid_seeded_state(fn(zero_init_last_bn=False, drop_block_rate=float(GOLDEN["step_rate"])), seed)
    with torch.no_grad():
        for t in m.state_dict().values():
            if t.dtype.is_floating_point:
                t.copy_(t.bfloat16().float())
    key = torch.from_numpy(GOLDEN["key"]).cuda()
    lref = float(GOLDEN[pre + "loss"])
    mp_ = copy.deepcopy(m).cuda().train()          # plain eager AMP arm: NCHW, the modules' unfused branch
    mp_.fixed_drop_block_key = key
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logp = torch.log_softmax(mp_(x.float().contiguous()).float(), dim=-1)
    loss_plain = (-(1 - smooth) * logp.gather(1, y.view(-1, 1)).squeeze(1) - smooth * logp.mean(-1)).mean()
    loss_plain.backward()
    errs_plain = _grad_errors({n: q.grad for n, q in mp_.named_parameters()}, g)
    del mp_
    monkeypatch.setattr(fused, "TC_MIN_PIXELS", 0)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    m = m.cuda().to(memory_format=CL).train()
    m.fixed_drop_block_key = key
    ts = trainer.TrainStep(m, lr=0.0, momentum=0.9, weight_decay=1e-4, nesterov=True, weights="bf16", label_smoothing=smooth)
    xc = x.contiguous(memory_format=CL)
    info = ts.capture(xc, y, warmup=2)
    loss = ts.step(xc, y).item()
    errs = _grad_errors(ts.grads(), g)
    assert info["cuda_graph"]
    return loss, lref, loss_plain.item(), errs, errs_plain


@pytest.mark.parametrize("name", ["cotnet50", "se_cotnetd_50"])
def test_step_matches_reference_golden(name, monkeypatch):
    """The bench path (bf16 weights, autocast, channels_last, one captured graph) with drop_block_rate 0.1 and the fixture's key
    against the reference's fp64 step with the same uniforms; gates of test_recipe_gpu.test_recipe_step_matches_reference_golden."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    loss, lref, lplain, errs, errs_plain = _step_errors(name, monkeypatch)
    assert abs(loss - lref) <= 1e-2 * lref, (loss, lref)
    assert errs["median_norm"] <= 2.5 * errs_plain["median_norm"] + 1e-2, (errs, errs_plain)
    assert errs["median_proj"] <= 2.5 * errs_plain["median_proj"] + 1e-2, (errs, errs_plain)
    print(name, "dropblock step: loss", loss, "ref", lref, "plain", lplain, "bench path", errs, "plain AMP", errs_plain)


# ------------------------------------------------------------------------------------------------ the captured step
def _model(**kw):
    torch.manual_seed(0)
    return backbone.CoTResNet([1, 1, 2, 2], num_classes=100, **kw).cuda().to(memory_format=CL)


def _batch(seed, B=8, res=96):
    g0 = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (B, 3, res, res), generator=g0, dtype=torch.uint8).cuda()
    return trainer.normalize_u8(x, MEAN, STD), torch.randint(0, 100, (B,), generator=g0).cuda()


def test_graph_replays_draw_new_masks_and_seeded_runs_repeat(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    runs = []
    for _ in range(2):
        m = _model(drop_block_rate=0.2)
        keys = []
        orig = m._drop_block_key

        def rec(x):
            k = orig(x)
            keys.append(k)
            return k
        m._drop_block_key = rec
        ts = trainer.TrainStep(m, lr=0.01, label_smoothing=0.1)
        x, lab = _batch(1)
        torch.manual_seed(9)
        ts.capture(x, lab, warmup=1)
        gk = keys[-1]
        seen, losses = [], []
        for step in range(4):
            x, lab = _batch(2 + step)
            losses.append(ts.step(x, lab).item())
            seen.append(tuple(gk.tolist()))
        torch.cuda.synchronize()
        assert len(set(seen)) == 4
        runs.append((losses, seen, {k: v.clone() for k, v in ts.master_state().items()}))
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1]
    assert all(torch.equal(runs[0][2][k], runs[1][2][k]) for k in runs[0][2])


def test_rate_zero_is_bit_identical_and_launches_nothing(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    calls = []
    orig = dropblock.device_mask
    monkeypatch.setattr(dropblock, "device_mask", lambda *a: calls.append(1) or orig(*a))
    out = []
    for kw in ({}, {"drop_block_rate": 0.}):
        ts = trainer.TrainStep(_model(**kw), lr=0.01)
        x, lab = _batch(1)
        ts.capture(x, lab, warmup=1)
        losses = [ts.step(*_batch(2 + s)).item() for s in range(2)]
        out.append((losses, {k: v.clone() for k, v in ts.master_state().items()}))
    assert out[0][0] == out[1][0] and all(torch.equal(out[0][1][k], out[1][1][k]) for k in out[0][1])
    assert not calls
    ts = trainer.TrainStep(_model(drop_block_rate=0.1), lr=0.01)
    ts.step_eager(*_batch(1))
    assert calls                                   # and with a rate the kernels do run


def test_trunk_trains_at_planes_of_the_shared_memory_budget():
    """A 256x384 input puts layer3 block 0's bn1 site at a 32x48 plane with 256 channels (see EXTRA): the step runs and drops."""
    m = backbone.CoTResNet([1, 1, 1, 1], num_classes=10, drop_block_rate=0.1).cuda().to(memory_format=CL).train()
    m.fixed_drop_block_key = torch.tensor([7, 8])
    x = torch.randn(2, 3, 256, 384, device="cuda").contiguous(memory_format=CL)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = m(x)
    out.float().sum().backward()
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and all(torch.isfinite(q.grad).all() for q in m.parameters() if q.grad is not None)


def test_eval_outputs_do_not_depend_on_the_rate():
    x, _ = _batch(4)
    for fn in (lambda **kw: _model(**kw),
               lambda **kw: backbone_hybrid.CoTHybridNet([1, 1, 2, 1], num_classes=10, stem_width=32,
                                                         block_args=backbone_hybrid._args(2), **kw).cuda().to(memory_format=CL)):
        torch.manual_seed(0)
        a = fn().eval()
        torch.manual_seed(0)
        b = fn(drop_block_rate=0.3).eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            assert torch.equal(a(x), b(x))
