"""CPU checks of tests/stage_ref.py: the fp64 stage restatements against torch fp64 autograd of the modules, the rounding helper
against torch's casts, the bound helpers on crafted cases, and the dispatch mirror pinned to the source lines it restates."""
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import stage_ref as S


# ------------------------------------------------------------------------------------------------ rounding and bounds
def test_bf16_rounding_matches_torch_casts_with_ties():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(100000, generator=g) * torch.exp2(torch.randint(-30, 30, (100000,), generator=g).float())
    # exact ties: bf16 values plus half their ulp, with even and odd last significand bits
    b = torch.randn(4096, generator=g).to(torch.bfloat16).float()
    b = b[b != 0]
    ties = b + torch.sign(b) * S.ulp(b.double(), 8).float() * 0.5
    near = ties.double() + S.ulp(ties.double(), 24) * torch.where(torch.rand(ties.shape, generator=g) < 0.5, -1.0, 1.0)
    for v in (x, ties, near.float()):
        want = v.to(torch.bfloat16).double()
        assert torch.equal(S.bf16(v.double()), want)
    assert bool((ties.to(torch.bfloat16).double() != b.double()).any()) and bool((ties.to(torch.bfloat16).double() == b.double()).any())
    d = torch.randn(10000, generator=g, dtype=torch.float64)
    assert torch.equal(S.f32(d), d.float().double())


def test_ulp_and_gamma():
    assert S.ulp(torch.tensor([1.0], dtype=torch.float64), 8).item() == 2.0 ** -7
    assert S.ulp(torch.tensor([1.5], dtype=torch.float64), 24).item() == 2.0 ** -23
    assert S.ulp(torch.tensor([-0.75], dtype=torch.float64), 8).item() == 2.0 ** -8
    assert S.gamma(1) == pytest.approx(2.0 ** -24, rel=1e-6)
    assert S.gamma(2 ** 20) == pytest.approx(2 ** -4 / (1 - 2 ** -4))
    with pytest.raises(AssertionError):
        S.gamma(2 ** 24)


def test_sum_bound_holds_and_catches_bf16_rounding():
    """gamma(n) * sum|t| bounds an fp32 sequential sum; at the chain lengths of the wgmma weight gradients (a few hundred) a
    bf16-rounded result of the same sum exceeds it"""
    g = torch.Generator().manual_seed(1)
    for n in (16, 300):
        t = torch.randn(n, 64, generator=g, dtype=torch.float64)
        exact = t.sum(0)
        acc = torch.zeros(64, dtype=torch.float32)
        for i in range(n):
            acc = acc + t[i].float()
        bound = S.gamma(n) * t.abs().sum(0)
        S.within(acc, exact, bound, "sequential fp32 sum")
        with pytest.raises(AssertionError):
            S.within(acc.to(torch.bfloat16).float(), exact, bound, "bf16-rounded sum")


def test_store_bound():
    e = torch.tensor([1.0 + 2.0 ** -8], dtype=torch.float64)           # a bf16 tie: rounds to 1 (even), half an ulp away
    S.within(torch.tensor([1.0], dtype=torch.bfloat16), e, S.store_bound(e, 0.0, torch.bfloat16), "tie")
    with pytest.raises(AssertionError):
        S.within(torch.tensor([1.0 + 2.0 ** -7], dtype=torch.bfloat16), torch.tensor([1.0], dtype=torch.float64),
                 S.store_bound(torch.tensor([1.0], dtype=torch.float64), 0.0, torch.bfloat16), "one ulp")


# ------------------------------------------------------------------------------------------------ fp64 restatements
@pytest.mark.parametrize("cfg", ["plain", "relu", "relu_res_ds", "eval_relu"])
def test_bn_restatement_matches_autograd(cfg):
    g = torch.Generator().manual_seed(2)
    B, C, H = 3, 16, 5
    x = torch.randn(B, C, H, H, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    b = torch.randn(C, generator=g, dtype=torch.float64)
    w.requires_grad_(True)
    b.requires_grad_(True)
    rm, rv = torch.randn(C, generator=g, dtype=torch.float64), torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    train = not cfg.startswith("eval")
    res = torch.randn(B, C, H, H, generator=g, dtype=torch.float64, requires_grad=True) if "res" in cfg else None
    ds = torch.tensor([2.0, 0.0, 0.5], dtype=torch.float64) if "ds" in cfg else None
    relu = "relu" in cfg
    z = F.batch_norm(x, rm.clone(), rv.clone(), w, b, train, 0.1, 1e-5)
    if ds is not None:
        z = z * ds.view(-1, 1, 1, 1)
    if res is not None:
        z = z + res
    y = torch.relu(z) if relu else z
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    n = B * H * H
    if train:
        mean, var = x.detach().mean((0, 2, 3)), x.detach().var((0, 2, 3), unbiased=False)
    else:
        mean, var = rm, rv
    rstd = 1 / torch.sqrt(var + 1e-5)
    scale, shift = w.detach() * rstd, b.detach() - mean * w.detach() * rstd
    yr, _ = S.bn_apply_ref(x.detach(), scale, shift, relu, None if res is None else res.detach(), ds)
    assert torch.allclose(yr, y.detach(), rtol=0, atol=1e-12)
    gate = (y.detach() > 0) if relu else None
    sums = None
    r = S.bn_bwd_ref(dy, x.detach(), gate, scale, mean, rstd, None, False, ds)
    sums = torch.stack([r["s0"], r["s1"]])
    r = S.bn_bwd_ref(dy, x.detach(), gate, scale, mean, rstd, sums, train, ds)
    assert torch.allclose(r["dx"], x.grad, rtol=0, atol=1e-12)
    assert torch.allclose(r["s0"], b.grad, rtol=0, atol=1e-12) and torch.allclose(r["s1"], w.grad, rtol=0, atol=1e-12)
    if res is not None:
        assert torch.allclose(r["dres"], res.grad, rtol=0, atol=1e-12)


@pytest.mark.parametrize("gc", [0, 8])
def test_gn9_restatement_matches_autograd(gc):
    g = torch.Generator().manual_seed(3)
    B, wc, H = 2, 16, 4
    J = 9 * wc
    gn = nn.GroupNorm(wc, J).double()
    with torch.no_grad():
        gn.weight.uniform_(0.5, 1.5, generator=g)
        gn.bias.normal_(generator=g)
    l = torch.randn(B, J, H, H, generator=g, dtype=torch.float64, requires_grad=True)
    lb = torch.randn(J, generator=g, dtype=torch.float64, requires_grad=True)
    out = gn(l + lb.view(1, -1, 1, 1))
    dg = torch.randn(out.shape, generator=g, dtype=torch.float64)
    out.backward(dg)
    x = (l + lb.view(1, -1, 1, 1)).detach().view(B, wc, -1)
    mean, rstd = x.mean(2), 1 / torch.sqrt(x.var(2, unbiased=False) + gn.eps)
    o, _, xh, (m64, _, r64, _) = S.gn9_ref(l.detach(), lb.detach(), gn.weight.detach(), gn.bias.detach(), mean, rstd, gc, gn.eps)
    assert torch.allclose(S.from_storage(o, gc), out.detach(), rtol=0, atol=1e-12)
    assert torch.allclose(m64, mean, atol=1e-12) and torch.allclose(r64, rstd, atol=1e-12)
    assert torch.equal(S.from_storage(S.to_storage(o, gc), gc), o)
    r = S.gn9_bwd_ref(dg, xh, gn.weight.detach(), rstd, 9 * H * H)
    assert torch.allclose(r["dl"], l.grad, rtol=0, atol=1e-12)
    assert torch.allclose(r["dlbias"], lb.grad, rtol=0, atol=1e-12)
    assert torch.allclose(r["dgamma"], gn.weight.grad, rtol=0, atol=1e-12)
    assert torch.allclose(r["dbeta"], gn.bias.grad, rtol=0, atol=1e-12)


def test_gn9_tap_major_order_matches_header():
    """index of (g, tap) in tap-major chunks of gc = ((g/gc)*9 + tap)*gc + g%gc (include/cotb200.h)"""
    B, wc, gc = 1, 16, 8
    ref = torch.arange(9 * wc, dtype=torch.float64).view(1, -1, 1, 1)           # value = reference index g*9 + tap
    st = S.to_storage(ref, gc).flatten()
    for gch in range(wc):
        for t in range(9):
            assert st[((gch // gc) * 9 + t) * gc + gch % gc].item() == gch * 9 + t


@pytest.mark.parametrize("kind,train", [("cot", True), ("cot", False), ("split", True), ("split", False)])
def test_mlp_restatement_matches_modules(kind, train):
    g = torch.Generator().manual_seed(4)
    B, C, A = 4, 32, 16
    c0 = nn.Conv2d(C, A, 1).double()
    b1 = nn.BatchNorm2d(A).double()
    c3 = nn.Conv2d(A, 2 * C if kind == "cot" else C, 1).double()
    with torch.no_grad():
        b1.running_mean.normal_(generator=g)
        b1.running_var.uniform_(0.5, 1.5, generator=g)
        b1.weight.uniform_(0.5, 1.5, generator=g)
    b1.train(train)
    p = torch.randn(B, C, generator=g, dtype=torch.float64)
    z = c3((torch.relu if kind == "cot" else F.silu)(b1(c0(p.view(B, C, 1, 1))))).view(B, -1)
    want = torch.softmax(z.view(B, C, 2), 2) if kind == "cot" else torch.sigmoid(z)
    b1.eval()        # the restatement reads batch statistics from `training`, not from the module's mode
    a, ea = S.mlp_ref(p, (c0, b1, c3), kind, train)
    got = a if kind == "cot" else a[..., 0]
    assert torch.allclose(got, want, rtol=0, atol=1e-12)
    assert bool((ea[..., 0] > 0).all())


@pytest.mark.parametrize("fold,gc", [(1, 0), (1, 8), (2, 0)])
def test_agg_restatement_matches_loop(fold, gc):
    """out[b,c,h,w] = sum over taps of v[b,c,h+i-1,w+j-1] * w[b, weight channel of c, tap, h, w], the CoXt fold of the header"""
    g = torch.Generator().manual_seed(5)
    B, C, H = 1, 16 * fold if gc == 0 else 64, 4
    wc = C // 8
    v = torch.randn(B, C, H, H, generator=g, dtype=torch.float64)
    wr = torch.randn(B, 9 * wc, H, H, generator=g, dtype=torch.float64)     # reference order
    got, _ = S.agg_ref(v, S.to_storage(wr, gc), fold, gc)
    vp = F.pad(v, (1, 1, 1, 1))
    cf, wcf = C // fold, wc // fold
    for c in range(C):
        gch = (c // cf) * wcf + (c % cf) % wcf
        want = sum(vp[:, c, i:i + H, j:j + H] * wr[:, gch * 9 + i * 3 + j] for i in range(3) for j in range(3))
        assert torch.allclose(got[:, c], want, rtol=0, atol=1e-12)


def test_agg_restatement_matches_oracle():
    from oracle import agg_ref
    g = torch.Generator().manual_seed(6)
    B, C, H = 2, 16, 5
    wc = C // 8
    v = torch.randn(B, C, H, H, generator=g, dtype=torch.float64)
    w = torch.randn(B, 1, wc, 9, H, H, generator=g, dtype=torch.float64)
    want = agg_ref.agg_zeropad_unfold(v, w, 3, 1, 1, 1)
    got, _ = S.agg_ref(v, w.view(B, 9 * wc, H, H), 1, 0)
    assert torch.allclose(got, want, rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------ dispatch mirror
def test_mirror_source_anchors():
    """the source lines the dispatch mirror restates are still there, verbatim"""
    for rel, snippets in S.SOURCE_ANCHORS.items():
        with open(os.path.join(S.REPO, rel)) as f:
            src = f.read()
        for s in snippets:
            assert s in src, "%s no longer contains: %s" % (rel, s)


def test_mirror_constants_match_the_library():
    from cotnet_b200 import fused, tc
    assert (fused.TC_MIN_PIXELS, fused.TC_KEY_MAX_DIM, fused.TC_TRUNK_MAX_WEIGHT) == (S.TC_MIN_PIXELS, S.TC_KEY_MAX_DIM,
                                                                                         S.TC_TRUNK_MAX_WEIGHT)
    for C in (64, 96, 128, 192, 256, 384, 512, 768):
        for groups in (2, 4, 8):
            assert tc.conv_tile(C, groups) == S.conv_tile(C, groups)


@pytest.mark.parametrize("geo", sorted(S.BLOCK_CASES))
def test_block_call_lists_follow_the_mirror(geo):
    c = S.BLOCK_CASES[geo]
    width = c["cout"] // 4
    mp = S.TC_MIN_PIXELS if c["min_pixels"] is None else c["min_pixels"]
    assert S.bottleneck_calls(c["B"], c["cin"], width, c["cout"], c["H"], c["stride"], mp) == c["calls"]


def test_weight_gradient_branches():
    """torch.mm for the stage 3-4 bottleneck convolutions at bs256, the wgmma kernel for every CoT-layer and stage 1-2 shape"""
    assert S.mm_wgrad(2048, 512, 12544) and S.mm_wgrad(1024, 256, 50176) and S.mm_wgrad(256, 1024, 50176)
    assert not S.mm_wgrad(256, 1024, 12544 // 4) and not S.mm_wgrad(256, 64, 802816) and not S.mm_wgrad(64, 128, 802816)
    assert S.stem_wgrad_tc(96, 96, 64) and not S.stem_wgrad_tc(64, 72, 64) and S.stem_wgrad_tc(224, 224, 64)


def test_wgrad_chain():
    """crafted: one tile, 132 SMs, 6272 pixels -> 98 blocks, 25 splits of 4 blocks: 256 pixels + 25 partials + the add to OUT"""
    assert S._wgrad_launch_chain(6272, 64, 128, 132) == 4 * 64 + 25 + 1
    # many tiles leave one split: the whole pixel range in one accumulator
    assert S._wgrad_launch_chain(1000, 2048, 4096, 132) == 16 * 64 + 1 + 1
    assert S.wgrad_chain(6272, 48, 96, 96, 132) >= S._wgrad_launch_chain(6272, 48, 96, 132)
    assert S.stem_wgrad_chain(2, 48, 48, 132) == 48 + 96 + 1


@pytest.mark.parametrize("kind,train", [("cot", True), ("cot", False), ("split", True), ("split", False)])
def test_tail_backward_restatement_matches_autograd(kind, train):
    """tail_bwd_ref and mlp_bwd_ref (with the rounding bounds unused) against fp64 autograd of the tail: bn -> SiLU -> pooled mean of
    (y + k) -> MLP -> radix-2 softmax / sigmoid gate -> a0*y + a1*k; the CoT form is also the reference tail of oracle/cot_ref"""
    from oracle import cot_ref
    g = torch.Generator().manual_seed(7)
    B, C, H, A = 4, 16, 5, 32
    c0, b1 = nn.Conv2d(C, A, 1).double(), nn.BatchNorm2d(A).double()
    c3 = nn.Conv2d(A, 2 * C if kind == "cot" else C, 1).double()
    bn = nn.BatchNorm2d(C).double()
    with torch.no_grad():
        for m in (b1, bn):
            m.weight.uniform_(0.5, 1.5, generator=g)
            m.bias.normal_(generator=g)
            m.running_mean.normal_(generator=g)
            m.running_var.uniform_(0.5, 1.5, generator=g)
    u = torch.randn(B, C, H, H, generator=g, dtype=torch.float64, requires_grad=True)
    k = torch.relu(torch.randn(B, C, H, H, generator=g, dtype=torch.float64)).requires_grad_(True) if kind == "cot" else None
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    z = F.batch_norm(u, rm.clone(), rv.clone(), bn.weight, bn.bias, train, 0.1, bn.eps)
    y = F.silu(z)
    p = (y + (0 if k is None else k)).mean((2, 3))
    p.retain_grad()
    zz = c3((torch.relu if kind == "cot" else F.silu)(F.batch_norm(c0(p.view(B, C, 1, 1)), b1.running_mean.clone(),
                                                                    b1.running_var.clone(), b1.weight, b1.bias, train, 0.1, b1.eps)))
    zz = zz.view(B, -1)
    a = torch.softmax(zz.view(B, C, 2), 2) if kind == "cot" else torch.stack([torch.sigmoid(zz), torch.zeros_like(zz)], 2)
    a.retain_grad()
    out = a[..., 0].reshape(B, C, 1, 1) * y + (0 if k is None else a[..., 1].reshape(B, C, 1, 1) * k)
    if kind == "cot":
        sd = {"bn.weight": bn.weight, "bn.bias": bn.bias, "bn.running_mean": rm.clone(), "bn.running_var": rv.clone(),
              "se.0.weight": c0.weight, "se.0.bias": c0.bias, "se.1.weight": b1.weight, "se.1.bias": b1.bias,
              "se.1.running_mean": b1.running_mean.clone(), "se.1.running_var": b1.running_var.clone(),
              "se.3.weight": c3.weight, "se.3.bias": c3.bias}
        want = cot_ref._radix_tail(F.silu(cot_ref._bn(u, sd, "bn", train)), k, sd, train)
        assert torch.allclose(out, want, rtol=0, atol=1e-12)
    dout = torch.randn(out.shape, generator=g, dtype=torch.float64)
    out.backward(dout)
    if train:
        mean, var = u.detach().mean((0, 2, 3)), u.detach().var((0, 2, 3), unbiased=False)
    else:
        mean, var = rm, rv
    rstd = 1 / torch.sqrt(var + bn.eps)
    scale = bn.weight.detach() * rstd
    shift = bn.bias.detach() - mean * scale
    r = S.tail_bwd_ref(u.detach(), None if k is None else k.detach(), scale, shift, mean, rstd, a.detach(), dout, p.grad, train, 0.0)
    Sg = a.grad
    assert torch.allclose(r["S0"], Sg[..., 0], rtol=0, atol=1e-12)
    if k is not None:
        assert torch.allclose(r["S1"], Sg[..., 1], rtol=0, atol=1e-12)
    a_mod, _ = S.mlp_ref(p.detach(), (c0, b1, c3), kind, train)
    assert torch.allclose(a_mod, a.detach(), rtol=0, atol=1e-12)
    (dp, e_dp), prm = S.mlp_bwd_ref(p.detach(), Sg, (c0, b1, c3), kind, train)
    assert torch.allclose(dp, p.grad, rtol=0, atol=1e-12) and bool((e_dp > 0).all())
    for (ref, err), prm_t in zip(prm, (c0.weight, c0.bias, b1.weight, b1.bias, c3.weight, c3.bias)):
        assert torch.allclose(ref.reshape(prm_t.shape), prm_t.grad, rtol=0, atol=1e-12)
        assert bool((err[ref.reshape(err.shape) != 0] > 0).all())
    assert torch.allclose(r["du"], u.grad, rtol=0, atol=1e-12)
    assert torch.allclose(r["dgamma"], bn.weight.grad, rtol=0, atol=1e-12)
    assert torch.allclose(r["dbeta"], bn.bias.grad, rtol=0, atol=1e-12)
    if k is not None:
        assert torch.allclose(r["dk"], k.grad, rtol=0, atol=1e-12)


@pytest.mark.parametrize("geo", sorted(S.STEP_BLOCK_CASES))
def test_step_block_call_lists_follow_the_mirror(geo):
    """CoXt, SE-CoTNetD, drop-path, DropBlock and stem cases: the pinned list is what the generators derive"""
    c = S.STEP_BLOCK_CASES[geo]
    assert S.case_calls(c) == c["calls"]


def test_step_block_cases_match_the_models():
    """each case's geometry is its block's in the model: input / width / output channels, stride, conv2 kind, DropBlock sites"""
    from cotnet_b200 import backbone, backbone_hybrid
    from cotnet_b200.backbone_hybrid import SplitAttnConv2d
    from cotnet_b200.cot_layer import CoXtLayer
    models = {"cotnet50": backbone.cotnet50(drop_block_rate=0.1), "cotnext50_2x48d": backbone.cotnext50_2x48d(drop_block_rate=0.1),
              "se_cotnetd_50": backbone_hybrid.se_cotnetd_50(drop_block_rate=0.1), "se_cotnetd_152": backbone_hybrid.se_cotnetd_152()}
    for geo, c in S.STEP_BLOCK_CASES.items():
        if c["kind"] != "block":
            continue
        m = models[c["model"]]
        stage, i = c["block"].split(".")
        blk = getattr(m, stage)[int(i)]
        assert (blk.conv1.in_channels, blk.conv1.out_channels, blk.conv3.out_channels) == (c["cin"], c["width"], c["cout"]), geo
        if c["model"] in S.HYBRID:
            assert isinstance(blk.conv2, SplitAttnConv2d) == S.hybrid_split(c["width"], int(i), c4_idx=S.HYBRID[c["model"]]["c4_idx"]), geo
            assert (2 if int(i) == 0 else 1) == c["stride"]
        else:
            assert isinstance(blk.conv2, CoXtLayer) == (c["model"] != "cotnet50") and blk.stride == c["stride"], geo
        if "sites" in c:
            assert blk.drop_block_sites == c["sites"], geo
        if c["model"] == "se_cotnetd_152":          # the input size the block sees in the named config
            res = 320 if "_320_" in geo else 256
            (H,) = [h for n, _, _, _, _, h, _, _ in S.model_blocks(c["model"], res) if n == c["block"]]
            assert H == c["H"], geo
    # every hybrid block's conv2 kind and pool follow the mirror
    for name in ("se_cotnetd_50", "se_cotnetd_152"):
        _check_hybrid_blocks(name, models[name])


def _check_hybrid_blocks(name, m):
    """conv2 kind (c4_idx), the pool of a stride-2 conv2 (BlurPool2d or the 3x3/s2 average pool; present on a split-attention
    conv2 only with avd), avd_first and the deep stem's width: what stage_ref.HYBRID says of the trunk"""
    from cotnet_b200.backbone_hybrid import BlurPool2d, SplitAttnConv2d
    cfg = S.HYBRID[name]
    assert m.conv1[0].out_channels == cfg["stem_width"] and m.bn1.num_features == 2 * cfg["stem_width"], name
    assert tuple(len(getattr(m, "layer%d" % (s + 1))) for s in range(4)) == cfg["layers"], name
    for stage in ("layer1", "layer2", "layer3", "layer4"):
        for i, blk in enumerate(getattr(m, stage)):
            split = S.hybrid_split(blk.conv1.out_channels, i, c4_idx=cfg["c4_idx"])
            assert isinstance(blk.conv2, SplitAttnConv2d) == split, (name, stage, i)
            pooled = i == 0 and (cfg["avd"] if split else True)
            assert (blk.avd is not None) == pooled and blk.avd_first == cfg["avd_first"], (name, stage, i)
            if pooled:
                assert isinstance(blk.avd, BlurPool2d) == cfg["blur"], (name, stage, i)
                assert isinstance(blk.avd, BlurPool2d) or (blk.avd.kernel_size, blk.avd.stride, blk.avd.padding) == (3, 2, 1)
            if split:
                assert blk.conv2.conv.stride == ((1, 1) if pooled or i else (2, 2)), (name, stage, i)


def test_hybrid152_call_lists():
    """se_cotnetd_152 at 320 and 256 through the training mirror: no recorded pool anywhere (every stride-2 conv2 is followed by a
    BlurPool); the bench's bs64 step at 320 puts layer3.0's embed.3 and conv1x1 on wgmma (102400 pixels), at 256 it does not
    (65536); one more pixel of threshold moves layer3.0 back; the CoT layers are the even stage-3 blocks and stage 4"""
    for res, tc in ((320, True), (256, False)):
        stem, blocks, _ = S.model_calls("se_cotnetd_152", 64, res, drop_block=False)
        assert len(blocks) == 50 and stem == ["BNActFn(relu)"] * 3
        flat = sum(blocks, [])
        assert not any(c.startswith("Pool3x3S2Fn") for c in flat), res
        assert flat.count("CotTailFn(k)") == 18 + 3 and flat.count("CotTailFn(gate)") == 3 + 8 + 18, res
        l30 = blocks[3 + 8]
        assert ("TcConv1x1Fn(one,nobn)" in l30 and "TcConv1x1Fn(one,bn)" in l30) == tc, (res, l30)
        assert all("TcConv1x1Fn(one,nobn)" not in b for b in blocks[3 + 8 + 1:]), res
    l30 = S.model_calls("se_cotnetd_152", 64, 320, 102401, drop_block=False)[1][11]
    assert "TcConv1x1Fn(one,nobn)" not in l30 and l30[0] == "BNActFn(relu)"
    l30 = S.model_calls("se_cotnetd_152", 64, 320, 102400, drop_block=False)[1][11]
    assert "TcConv1x1Fn(one,nobn)" in l30 and l30[0] == "TcConv1x1Fn(one,relu)"
    # the CoT layers of layer3.0 / layer4.0 run before the pool: at the stage's input size
    mb = {n: (H, s) for n, _, _, _, _, H, _, s in S.model_blocks("se_cotnetd_152", 320)}
    assert mb["layer1.0"] == (160, 2) and mb["layer3.0"] == (40, 2) and mb["layer4.0"] == (20, 2) and mb["layer4.1"] == (10, 1)


@pytest.mark.parametrize("groups,shape", [(2, (48, 96, 1, 1)), (8, (96, 12, 3, 3)), (2, (96, 48, 1, 1))])
def test_dense_from_grouped_adjoint_matches_autograd(groups, shape):
    """the gather of the diagonal blocks is the gradient autograd gives the grouped weight through _dense_from_grouped, bit for
    bit (in bf16 too); the dense weight's convolution equals the grouped convolution"""
    from cotnet_b200.cot_layer import _dense_from_grouped
    g = torch.Generator().manual_seed(groups + shape[1])
    for dtype in (torch.float64, torch.bfloat16):
        w = torch.randn(shape, generator=g).to(dtype).requires_grad_(True)
        dense = _dense_from_grouped(w, groups)
        gd = torch.randn(dense.shape, generator=g).to(dtype)
        dense.backward(gd)
        got = S.dense_from_grouped_adjoint(gd, groups)
        assert got.dtype == dtype and torch.equal(got, w.grad)
    x = torch.randn(2, shape[1] * groups, 5, 5, generator=g, dtype=torch.float64)
    w = torch.randn(shape, generator=g, dtype=torch.float64)
    p = shape[2] // 2
    assert torch.allclose(F.conv2d(x, _dense_from_grouped(w, groups), padding=p), F.conv2d(x, w, padding=p, groups=groups),
                          rtol=0, atol=1e-12)


@pytest.mark.parametrize("C", [96, 192, 768])
def test_coxt_embed0_adjoint_matches_autograd(C):
    """the de-interleave of (dWx, dWk) is the gradient autograd gives embed.0's grouped weight through _coxt_embed0_dense and
    the cat of the concat-free GEMM, bit for bit; and x @ Wx^T + k @ Wk^T is the grouped convolution of the interleave of x, k"""
    from cotnet_b200.cot_layer import _coxt_embed0_dense
    G = 2
    g = torch.Generator().manual_seed(C)
    for dtype in (torch.float64, torch.bfloat16):
        w = torch.randn(C // 2, 2 * C // G, 1, 1, generator=g).to(dtype).requires_grad_(True)
        wx, wk = _coxt_embed0_dense(w, G)
        w0 = torch.cat([wx, wk], 1).reshape(C // 2, 2 * C, 1, 1)          # as CoXtLayer._forward_fused hands it to the GEMM
        gd = torch.randn(w0.shape, generator=g).to(dtype)
        w0.backward(gd)
        g2 = gd.reshape(C // 2, 2 * C)
        got = S.coxt_embed0_adjoint(g2[:, :C], g2[:, C:], G)
        assert got.dtype == dtype and torch.equal(got, w.grad)
    x = torch.randn(2, C, 3, 3, generator=g, dtype=torch.float64)
    k = torch.randn(2, C, 3, 3, generator=g, dtype=torch.float64)
    w = torch.randn(C // 2, 2 * C // G, 1, 1, generator=g, dtype=torch.float64)
    wx, wk = _coxt_embed0_dense(w, G)
    qk = torch.stack([x, k], 2).reshape(2, 2 * C, 3, 3)                    # models/cotnet.py:153-154
    want = F.conv2d(qk, w, groups=G)
    got = torch.einsum("bchw,nc->bnhw", x, wx) + torch.einsum("bchw,nc->bnhw", k, wk)
    assert torch.allclose(got, want, rtol=0, atol=1e-12)


@pytest.mark.parametrize("H,W", [(2, 2), (3, 5), (8, 7), (40, 40)])
def test_blurpool_reflect_padding_matches_torch(H, W):
    """BlurPool2d's padding: the values of F.pad(mode="reflect") and, bit for bit in fp64, the gradient autograd gives through it"""
    from cotnet_b200.backbone_hybrid import _ReflectPad1
    g = torch.Generator().manual_seed(H * 100 + W)
    x = torch.randn(2, 3, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    dy = torch.randn(2, 3, H + 2, W + 2, generator=g, dtype=torch.float64)
    want = F.pad(x, (1, 1, 1, 1), mode="reflect")
    got = _ReflectPad1.apply(x)
    assert torch.equal(got, want)
    (gw,) = torch.autograd.grad(want, x, dy)
    (gg,) = torch.autograd.grad(got, x, dy)
    assert torch.allclose(gg, gw, rtol=0, atol=1e-12)
