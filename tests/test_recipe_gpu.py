"""The training recipe on the GPU: the Mixup / CutMix input kernel against the reference's own mixed batches
(tests/golden/recipe.npz), stochastic depth inside the fused BatchNorm kernels against an fp64 torch composition, the
soft-target cross entropy against fp64 SoftTargetCrossEntropy(mixup_target(...)), and the recipe under CUDA-graph replay."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from cotnet_b200 import _lib, backbone, fused, trainer

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recipe.npz"))
MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _mix_batch(seed):
    """tools/make_recipe_golden.py:mix_batch"""
    rng = np.random.RandomState(1000 + seed)
    x = rng.randint(0, 256, size=(4, 3, 16, 20)).astype(np.uint8)
    return x, rng.randint(0, 1000, size=4).astype(np.int64)


def _mix(B, mode, lam=1.0, box=(0, 0, 0, 0)):
    """A batch draw as MixupCutmix makes it: B rows, partner B-1-n, the same mode, fp32 weights and box on every row."""
    rows = (_lib.MixRow * B)()
    for n, r in enumerate(rows):
        r.mode, r.partner, r.lam, r.one_minus_lam, r.target_lam = mode, B - 1 - n, float(np.float32(lam)), float(np.float32(1 - lam)), lam
        r.y0, r.y1, r.x0, r.x1 = box
    return trainer.MixRows(rows, B, "cuda", lam)


# ------------------------------------------------------------------------------------------------ Mixup / CutMix input kernel
@pytest.mark.parametrize("kind", ["mixup", "cutmix"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_batch_table_equals_reference_mixed_batch(kind, dtype):
    """C = 3 fast path: normalize_u8(x, mix=draw) == normalize_u8(the reference's mixed uint8 batch), bit for bit."""
    seed = int(GOLDEN[kind + "_seed"])
    x, _ = _mix_batch(seed)
    p = trainer.MixupCutmix(seed=seed).draw(4, 16, 20)
    assert p.host[0].mode == (1 if kind == "mixup" else 2)
    xd = torch.from_numpy(x).cuda()
    got = trainer.normalize_u8(xd, MEAN, STD, dtype, mix=p)
    want = trainer.normalize_u8(torch.from_numpy(GOLDEN[kind + "_out"]).cuda(), MEAN, STD, dtype)
    assert torch.equal(got, want)
    assert torch.equal(trainer.normalize_u8(xd, MEAN, STD, dtype, mix=_mix(4, 0)), trainer.normalize_u8(xd, MEAN, STD, dtype))


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("shape", [(4, 3, 15, 19), (2, 5, 8, 8)])
def test_batch_table_generic_path(mode, shape):
    """Generic path (C != 3 or H*W % 4 != 0) against the reference's numpy arithmetic (datasets/mixup.py:291-298)."""
    N, C, H, W = shape
    x = np.random.RandomState(7).randint(0, 256, size=shape).astype(np.uint8)
    lam, box = 0.37 if mode == 1 else 0.8, (3, H - 2, 2, W - 5)
    p = _mix(N, mode, lam, box)
    if mode == 1:
        want = np.rint(x.astype(np.float32) * np.float32(lam) + x[::-1].astype(np.float32) * np.float32(1 - lam)).astype(np.uint8)
    elif mode == 2:
        want = x.copy()
        want[:, :, box[0]:box[1], box[2]:box[3]] = x[::-1][:, :, box[0]:box[1], box[2]:box[3]]
    else:
        want = x
    mean, std = (MEAN + [100.0, 50.0])[:C], (STD + [60.0, 70.0])[:C]
    got = trainer.normalize_u8(torch.from_numpy(x).cuda(), mean, std, torch.float32, mix=p)
    assert torch.equal(got, trainer.normalize_u8(torch.from_numpy(np.ascontiguousarray(want)).cuda(), mean, std, torch.float32))


# ------------------------------------------------------------------------------------------------ stochastic depth in BatchNorm
def _scales(B, keep=0.8):
    s = torch.tensor([0.0 if b % 3 == 1 else 1.0 / np.float32(keep) for b in range(B)], dtype=torch.float32, device="cuda")
    assert (s == 0).any() and (s > 1).any()
    return s


def _ds_case(dtype, C, H, seed, tc=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B = 8
    bn = nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5, generator=g); bn.bias.normal_(0, 0.3, generator=g)
    if tc:
        K = 64
        a = _cl(torch.randn(B, K, H, H, generator=g, device="cuda").to(dtype)).requires_grad_(True)
        w = (torch.randn(C, K, 1, 1, generator=g, device="cuda") * 0.1).to(dtype).requires_grad_(True)
    else:
        a = _cl((torch.randn(B, C, H, H, generator=g, device="cuda") * 1.5 + 0.3).to(dtype)).requires_grad_(True)
        w = None
    r = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype)).requires_grad_(True)
    cot = _cl(torch.randn(B, C, H, H, generator=g, device="cuda").to(dtype))
    return bn, a, w, r, cot


def _run(bn, a, w, r, cot, ds):
    if w is None:
        y = fused.bn_act(a, bn, relu=True, res=r, drop_scale=ds)
        ins = [a, bn.weight, bn.bias, r]
    else:
        y = fused.TcConv1x1Fn.apply(a, None, w, None, bn.weight, bn.bias, bn, True, r, ds)
        ins = [a, w, bn.weight, bn.bias, r]
    return [y] + list(torch.autograd.grad(y, ins, cot))


@pytest.mark.parametrize("path,dtype,tol,C,H", [("bn_act", torch.float32, 2e-4, 64, 14), ("bn_act", torch.bfloat16, 3e-2, 256, 7),
                                                 ("bn_act", torch.float32, 2e-4, 2048, 7), ("tc", torch.bfloat16, 3e-2, 256, 14)])
def test_drop_path_batchnorm(path, dtype, tol, C, H):
    """relu(s_b * BN(x) + res) with s containing 0 and 1/keep: forward and every gradient against fp64 torch; an all-ones
    scale is bit-identical to the plain path; repeats are bit-identical."""
    tc = path == "tc"
    bn, a, w, r, cot = _ds_case(dtype, C, H, C + H, tc)
    bn_ref = copy.deepcopy(bn).double()
    s = _scales(a.shape[0])
    out = _run(copy.deepcopy(bn), a, w, r, cot, s)
    assert all(torch.equal(u, v) for u, v in zip(out, _run(copy.deepcopy(bn), a, w, r, cot, s)))
    ones = torch.ones_like(s)
    plain, unit = _run(copy.deepcopy(bn), a, w, r, cot, None), _run(copy.deepcopy(bn), a, w, r, cot, ones)
    assert all(torch.equal(u, v) for u, v in zip(plain, unit))
    ad = a.detach().double().requires_grad_(True)
    wd = None if w is None else w.detach().double().requires_grad_(True)
    rd = r.detach().double().requires_grad_(True)
    pre = ad if wd is None else torch.nn.functional.conv2d(ad, wd)
    yd = torch.relu(bn_ref(pre) * s.double().view(-1, 1, 1, 1) + rd)
    ins = [ad, bn_ref.weight, bn_ref.bias, rd] if wd is None else [ad, wd, bn_ref.weight, bn_ref.bias, rd]
    want = [yd] + list(torch.autograd.grad(yd, ins, cot.double()))
    if not tc:
        for i, (u, v) in enumerate(zip(out, want)):
            e = (u.double() - v).abs().max().item()
            lim = (1 if i == 0 else 4) * tol * max(1.0, v.abs().max().item())
            assert e <= lim, "output %d err %.3e > %.3e" % (i, e, lim)
        return
    # wgmma path: the GEMM output feeding the BatchNorm is stored in bf16, and the BatchNorm backward amplifies that rounding in a
    # few elements; judge by norm error, and against the plain path's own error at s = 1
    bn_ref1 = copy.deepcopy(bn).double()
    yd1 = torch.relu(bn_ref1(torch.nn.functional.conv2d(ad, wd)) + rd)
    want1 = [yd1] + list(torch.autograd.grad(yd1, [ad, wd, bn_ref1.weight, bn_ref1.bias, rd], cot.double()))

    def rel(u, v):
        return ((u.double() - v).norm() / v.norm().clamp_min(1e-12)).item()
    for i, (u, v, p, v1) in enumerate(zip(out, want, plain, want1)):
        e, e1 = rel(u, v), rel(p, v1)
        assert e <= tol and e <= 2 * e1 + 1e-3, "output %d norm err %.3e (plain path %.3e)" % (i, e, e1)


# ------------------------------------------------------------------------------------------------ soft-target cross entropy
def _soft_ce_ref(z, labels, lam, smoothing):
    K = z.shape[1]
    off = smoothing / K
    on = 1.0 - smoothing + off
    y1 = torch.full_like(z, off).scatter_(1, labels.view(-1, 1), on)                     # datasets/mixup.py:17-27
    y2 = torch.full_like(z, off).scatter_(1, labels.flip(0).view(-1, 1), on)
    t = y1 * lam + y2 * (1.0 - lam)
    return torch.sum(-t * torch.log_softmax(z, dim=-1), dim=-1).mean()                  # loss/cross_entropy.py:34-36


@pytest.mark.parametrize("K", [10, 1000, 1001])
@pytest.mark.parametrize("B", [2, 256])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("lam", [1.0, 0.37])
def test_soft_ce_batch_table_matches_fp64(K, B, dtype, lam):
    g = torch.Generator(device="cuda").manual_seed(K + B)
    z = (torch.randn(B, K, generator=g, device="cuda") * 3).to(dtype).requires_grad_(True)
    labels = torch.randint(0, K, (B,), generator=g, device="cuda")
    for smoothing, mix in ((0.1, _mix(B, 1, lam)), (0.1, None), (0.0, None)):
        lam_eff = lam if mix is not None else 1.0
        loss = trainer.soft_target_cross_entropy(z, labels, mix, smoothing)
        (gz,) = torch.autograd.grad(loss * 1.7, [z])
        zd = z.detach().double().requires_grad_(True)
        want = _soft_ce_ref(zd, labels, lam_eff, smoothing)
        (gd,) = torch.autograd.grad(want * 1.7, [zd])
        assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item()), (loss.item(), want.item())
        assert gz.dtype == dtype
        err = (gz.double() - gd).abs().max().item()
        assert err <= (1e-6 if dtype == torch.float32 else 0.5 ** 8 * gd.abs().max().item() + 1e-6), err
        if smoothing == 0.0:
            ce = torch.nn.functional.cross_entropy(zd, labels)
            assert abs(loss.item() - ce.item()) <= 1e-5 * abs(ce.item())
        again = trainer.soft_target_cross_entropy(z, labels, mix, smoothing)
        assert torch.equal(loss, again)


def test_soft_ce_table_fp32_gradients_before_the_cast():
    """The kernel's own fp32 gradient (what the bf16 logits receive before the storage cast) against fp64: <= 1e-6 abs."""
    B, K = 256, 1000
    g = torch.Generator(device="cuda").manual_seed(3)
    z = (torch.randn(B, K, generator=g, device="cuda") * 3).to(torch.bfloat16)
    labels = torch.randint(0, K, (B,), generator=g, device="cuda")
    mix = _mix(B, 1, 0.37)
    lib, st = _lib.load(), torch.cuda.current_stream().cuda_stream
    rows = torch.empty(2, B, device="cuda")
    loss = torch.empty((), device="cuda")
    _lib.check(lib.cotb200_soft_ce(_lib.BF16, B, K, z.data_ptr(), K, labels.data_ptr(), B, mix.dev.data_ptr(), 0.1,
                                   rows.data_ptr(), loss.data_ptr(), st), "soft_ce")
    one = torch.ones((), device="cuda")
    dz = torch.empty(B, K, device="cuda")
    _lib.check(lib.cotb200_soft_ce_bwd(_lib.BF16, B, K, z.data_ptr(), K, labels.data_ptr(), B, mix.dev.data_ptr(), 0.1,
                                       rows.data_ptr(), one.data_ptr(), dz.data_ptr(), K, st), "soft_ce_bwd")
    zd = z.double().requires_grad_(True)
    (gd,) = torch.autograd.grad(_soft_ce_ref(zd, labels, 0.37, 0.1), [zd])
    assert (dz.double() - gd).abs().max().item() <= 1e-6


def test_soft_ce_invalid_label_with_or_without_table_is_nan():
    z = torch.randn(4, 10, device="cuda")
    labels = torch.tensor([1, 2, 10, 3], device="cuda")
    assert torch.isnan(trainer.soft_target_cross_entropy(z, labels, None, 0.1))
    labels[2] = -1
    assert torch.isnan(trainer.soft_target_cross_entropy(z, labels, _mix(4, 1, 0.5), 0.1))


# ------------------------------------------------------------------------------------------------ the recipe in a training step
def _model(**kw):
    torch.manual_seed(0)
    return backbone.CoTResNet([1, 1, 1, 1], num_classes=100, **kw).cuda().to(memory_format=torch.channels_last)


def _batch(seed, B=8, res=96):
    g0 = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (B, 3, res, res), generator=g0, dtype=torch.uint8).cuda()
    return x, torch.randint(0, 100, (B,), generator=g0).cuda()


def test_graph_replays_follow_each_steps_batch_table_and_draw_new_masks(monkeypatch):
    """Over 4 replays of one captured step the drop-path scales change; and with fixed masks and lr 0 the replayed loss equals,
    bit for bit, the eager step's loss for each step's target_lam, so the graph reads every step's mixing parameters."""
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    m = _model(drop_path_rate=0.5)
    seen = []
    orig = m._drop_path_scales

    def rec(x):
        s = orig(x)
        seen.append(s)
        return s
    m._drop_path_scales = rec
    ts = trainer.TrainStep(m, lr=0.0, momentum=0.0, weight_decay=0.0, label_smoothing=0.1)
    xu, lab = _batch(1)
    x = trainer.normalize_u8(xu, MEAN, STD)
    ts.capture(x, lab, warmup=1, mix=_mix(8, 1, 0.5))
    graph_scales = seen[-1]
    masks = []
    for lam in (0.2, 0.4, 0.6, 0.8):
        ts.step(x, lab, mix=_mix(8, 1, lam))
        masks.append(graph_scales.clone())
    assert len({tuple(t.flatten().tolist()) for t in masks}) == 4
    tsg, tse = [trainer.TrainStep(_model(drop_path_rate=0.5), lr=0.0, momentum=0.0, weight_decay=0.0, label_smoothing=0.1)
                for _ in range(2)]
    for t in (tsg, tse):
        t.model.fixed_drop_path_scales = torch.tensor([1.0, 0.0, 1.5, 2.0], device="cuda").repeat_interleave(2).view(1, 8).repeat(4, 1)
    tsg.capture(x, lab, warmup=1, mix=_mix(8, 1, 0.5))
    tse.step_eager(x, lab, _mix(8, 1, 0.5))
    lams = (0.1, 0.3, 0.9, 0.3)
    lg = [tsg.step(x, lab, mix=_mix(8, 1, lam)).item() for lam in lams]
    le = [tse.step_eager(x, lab, _mix(8, 1, lam)).item() for lam in lams]
    assert lg == le and len(set(lg)) == 3, (lg, le)


def test_identically_seeded_recipe_steps_are_bit_identical(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    runs = []
    for _ in range(2):
        m = _model(drop_path_rate=0.1, drop_rate=0.25)
        ts = trainer.TrainStep(m, lr=0.01, label_smoothing=0.1)
        mc = trainer.MixupCutmix(seed=5)
        xu, lab = _batch(2)
        torch.manual_seed(9)
        p = mc.draw(8, 96, 96)
        ts.capture(trainer.normalize_u8(xu, MEAN, STD, mix=p), lab, warmup=1, mix=p)
        losses = []
        for step in range(3):
            xu, lab = _batch(3 + step)
            p = mc.draw(8, 96, 96)
            losses.append(ts.step(trainer.normalize_u8(xu, MEAN, STD, mix=p), lab, mix=p).item())
        torch.cuda.synchronize()
        runs.append((losses, {k: v.clone() for k, v in ts.master_state().items()}))
    assert runs[0][0] == runs[1][0]
    assert all(torch.equal(runs[0][1][k], runs[1][1][k]) for k in runs[0][1])


def test_eval_mode_ignores_the_rates():
    xu, _ = _batch(4)
    x = trainer.normalize_u8(xu, MEAN, STD)
    a, b = _model().eval(), _model(drop_rate=0.25, drop_path_rate=0.2).eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        assert torch.equal(a(x), b(x))


# ------------------------------------------------------------------------------------------------ the recipe step vs the reference
def _step_batch(g):
    """tools/make_recipe_golden.py:step_batch -- the uint8 batch of the training-step fixture, checked against its checksum."""
    from oracle import make_golden
    x, y = make_golden.train_batch(int(g["step_seed"]), int(g["step_B"]), int(g["step_res"]))
    u8 = (x * 45.0 + 120.0).round().clamp(0, 255).to(torch.uint8)
    assert int(u8.long().sum()) == int(g["step_u8_sum"]) and np.array_equal(y.numpy(), g["step_labels"])
    return u8, y


def test_recipe_step_with_batch_table_matches_reference_golden(monkeypatch):
    """The bench.py path (bf16 weights, autocast, channels_last, the whole step replayed from one CUDA graph, gradients from the
    flat bucket) with the recipe -- drop_path_rate 0.1 with the reference's own DropPath masks injected, the batch mixed by
    normalize_u8(mix=) from MixupCutmix's draw, the soft-target loss with smoothing 0.1 -- against one step of the reference's
    cotnet50 in fp64 (tests/golden/recipe.npz step_*).  Gates of test_trainer_gpu.test_bench_path_matches_reference_golden: the
    loss within 1 %, the gradient errors (_grad_errors) within 2.5x those of the plain eager AMP graph of the same modules."""
    from oracle import make_golden
    from test_trainer_gpu import _grad_errors
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)         # as the golden train-step tests: no TF32
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    B, R, seed = int(GOLDEN["step_B"]), int(GOLDEN["step_res"]), int(GOLDEN["step_seed"])
    g = {"names": GOLDEN["step_names"], "seed": GOLDEN["step_seed"], "gnorm": GOLDEN["step_gnorm"], "gproj": GOLDEN["step_gproj"]}
    u8, y = _step_batch(GOLDEN)
    y = y.cuda()
    # the draw of the reference's collate, and its mixed batch
    p = trainer.MixupCutmix(seed=int(GOLDEN["step_mix_seed"])).draw(B, R, R)
    assert p.host[0].mode == 1 and p.lam == float(GOLDEN["step_lam"])
    un = u8.numpy()
    mixed = np.rint(un.astype(np.float32) * np.float32(p.host[0].lam) + un[::-1].astype(np.float32) * np.float32(p.host[0].one_minus_lam))
    assert int(mixed.astype(np.int64).sum()) == int(GOLDEN["step_mixed_sum"])
    xc = trainer.normalize_u8(u8.cuda(), MEAN, STD, torch.bfloat16, mix=p)
    assert torch.equal(xc, trainer.normalize_u8(torch.from_numpy(mixed.astype(np.uint8)).cuda(), MEAN, STD, torch.bfloat16))
    scales = torch.from_numpy(GOLDEN["step_masks"] / GOLDEN["step_keep"][:, None]).float().cuda()
    assert (scales == 0).any()

    m = make_golden.hybrid_seeded_state(backbone.cotnet50(zero_init_last_bn=False, drop_path_rate=float(GOLDEN["step_rate"])), seed)
    with torch.no_grad():
        for t in m.state_dict().values():
            if t.dtype.is_floating_point:
                t.copy_(t.bfloat16().float())
    assert m.drop_path_rates() == list(GOLDEN["rates_cotnet50"])
    lref = float(GOLDEN["step_loss"])
    # (a) plain eager AMP arm: NCHW tensors take the modules' un-fused PyTorch branch, the loss is torch's soft-target CE
    mp_ = copy.deepcopy(m).cuda().train()
    mp_.fixed_drop_path_scales = scales
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss_plain = _soft_ce_ref(mp_(xc.float().contiguous()).float(), y, p.lam, 0.1)
    loss_plain.backward()
    errs_plain = _grad_errors({n: q.grad for n, q in mp_.named_parameters()}, g)
    del mp_
    # (b) the bench path, every layer on the path the bs256 bench takes in stages 1-2 (see test_bench_path_matches_reference_golden)
    monkeypatch.setattr(fused, "TC_MIN_PIXELS", 0)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    m = m.cuda().to(memory_format=torch.channels_last).train()
    m.fixed_drop_path_scales = scales
    ts = trainer.TrainStep(m, lr=0.0, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=0.9999, weights="bf16",
                           label_smoothing=0.1)
    info = ts.capture(xc, y, warmup=2, mix=p)
    loss = ts.step(xc, y, mix=p).item()
    errs = _grad_errors(ts.grads(), g)
    loss_eager = ts.step_eager(xc, y, p).item()
    errs_eager = _grad_errors(ts.grads(), g)
    assert info["cuda_graph"]
    assert abs(loss - lref) <= 1e-2 * lref and abs(loss_eager - lref) <= 1e-2 * lref, (loss, loss_eager, lref)
    for e_ in (errs, errs_eager):
        assert e_["median_norm"] <= 2.5 * errs_plain["median_norm"] + 1e-2, (e_, errs_plain)
        assert e_["median_proj"] <= 2.5 * errs_plain["median_proj"] + 1e-2, (e_, errs_plain)
    print("recipe step: loss", loss, "ref", lref, "plain", loss_plain.item(), "bench path", errs, "plain AMP", errs_plain)
