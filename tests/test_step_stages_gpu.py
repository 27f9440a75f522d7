"""The rest of the bf16 training step stage by stage (tests/stage_ref.py, tests/test_stage_grads_gpu.py): the DropBlock functions,
CoXt bottlenecks, SE-CoTNetD blocks (split attention, the stride-2 cuDNN 3x3, avg_down, c4_idx), stochastic depth and DropBlock
inside blocks, and both stems.

Per block: (a) the recorded calls equal the dispatch mirror's list, (b) every call passes its stage check against fp64 of its own
inputs, (c) the block's DropBlock sites, keys and drop-path scales are the ones it was handed, (d) the gradient autograd delivered
to the block input is the fp64 sum of what its consumers returned, (e) every parameter is accounted for, including those behind
CoXtLayer's derived dense weights (bit for bit through the restated adjoints), (f) the stated producer -> consumer dataflow.
The split-attention gate that runs in plain PyTorch (DropBlock after bn0) is checked op by op from the bf16 values each op received.

Per model (cotnet50, cotnext50_2x48d, se_cotnetd_50, and cotnet50 with every convolution on wgmma): one eager
TrainStep(weights="bf16").forward_backward with drop path and DropBlock on: the whole call list, every block's own drop-path row
and DropBlock sites, every stage check, block-to-block dataflow, the gradient at every block input and at the stem output as the
sum of its consumers', the head and the loss, and the flat gradient buckets."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import stage_ref as S
from test_stage_grads_gpu import ONE_ULP, ConvRecorder, PadRecorder, TorchBNRecorder, _cfg, account_params, blur_convs, check_blur, \
    check_call, check_dropblock, check_dropblock_res_relu, tail_mods, torch_bn_bwd_ref
from cotnet_b200 import _lib, dropblock, fused

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
CL = torch.channels_last
KEY = (0x1234567, 0x7654321)


@pytest.fixture(autouse=True)
def _no_tf32(monkeypatch):
    """no TF32; deterministic cuDNN, as the with / without recorder comparisons are bitwise"""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


@pytest.fixture(scope="module", autouse=True)
def _report_one_ulp():
    """after the module: the one-ulp report of test_stage_grads_gpu.py for the stages these cases reach"""
    ONE_ULP.clear()
    yield
    for k in sorted(ONE_ULP):
        one, far, n = ONE_ULP[k]
        print("\nbf16 outputs one ulp off, %-22s %.2e (%d of %d; %d farther)" % (k, one / max(n, 1), one, n, far), end="")


def _cl(t):
    return t.contiguous(memory_format=CL)


# ------------------------------------------------------------------------------------------------ DropBlock functions
@pytest.mark.parametrize("with_ds", [False, True], ids=["no_ds", "ds"])
def test_dropblock_functions(with_ds, monkeypatch):
    """DropBlockFn and DropBlockResReluFn on bf16 at a stage-3 geometry, drop-path scales with zeros, a count whose scale is not
    a power of two"""
    B, C, H = 4, 64, 14
    spec, site = dropblock.DropBlock(0.1, 5, 0.25), 3
    g = torch.Generator(device=DEV).manual_seed(11 + with_ds)
    x = _cl(torch.randn(B, C, H, H, generator=g, device=DEV).to(BF)).requires_grad_(True)
    z = _cl(torch.randn(B, C, H, H, generator=g, device=DEV).to(BF)).requires_grad_(True)
    res = _cl(torch.randn(B, C, H, H, generator=g, device=DEV).to(BF)).requires_grad_(True)
    ds = torch.tensor([0.0, 1.25, 1.25, 0.0], device=DEV) if with_ds else None
    key = torch.tensor(KEY, device=DEV)
    rec = S.Recorder(monkeypatch)
    y1 = dropblock.drop_block(x, key, site, spec)
    y2 = dropblock.drop_block_res_relu(z, res, key, site + 1, spec, ds)
    ((y1.float() * torch.randn(y1.shape, generator=g, device=DEV)).sum()
     + (y2.float() * torch.randn(y2.shape, generator=g, device=DEV)).sum()).backward()
    c1, c2 = rec.calls
    assert (c1.name, c2.name) == ("DropBlockFn", "DropBlockResReluFn")
    for c in (c1, c2):
        n = int(c.inp[2 if c is c1 else 3].item())
        s = float(torch.tensor(float(dropblock.scale_of(n, B * C * H * H))).to(BF))
        assert 0 < n < B * C * H * H and s != 2.0 ** round(torch.log2(torch.tensor(s)).item()), (n, s)
    check_dropblock(c1)
    check_dropblock_res_relu(c2)
    S.equal(x.grad, c1.gout[0], "x.grad")
    S.equal(z.grad, c2.gout[0], "z.grad")
    S.equal(res.grad, c2.gout[1], "res.grad")


# ------------------------------------------------------------------------------------------------ blocks
def _model(case):
    from cotnet_b200 import backbone, backbone_hybrid
    torch.manual_seed(5)
    ctor = {"cotnet50": backbone.cotnet50, "cotnext50_2x48d": backbone.cotnext50_2x48d,
            "se_cotnetd_50": backbone_hybrid.se_cotnetd_50, "se_cotnetd_152": backbone_hybrid.se_cotnetd_152}[case["model"]]
    return ctor(drop_block_rate=0.1 if case.get("sites") else 0.0)


def _randomise_bn(mod):
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.25, 0.25)


def _consumer_sum(ptr, shape, calls, convs, extra, what):
    """fp64 sum (and bound) of the gradients the consumers of the tensor at storage `ptr` returned: recorded calls' returned
    gradients (exact values), conv2d_input of recorded torch convolutions (fp32 chain + bf16 store), `extra` (value, bound) pairs;
    autograd adds them in bf16 (gamma_bf16 of the partial sums).  Every consumer must have returned a gradient."""
    parts = []
    for c in calls:
        for i, a in enumerate(c.args):
            if isinstance(a, torch.Tensor) and a.data_ptr() == ptr and tuple(a.shape) == shape:
                assert c.gout is not None and c.gout[i] is not None, "%s: %s argument %d returned no gradient" % (what, c.name, i)
                parts.append((c.gout[i].double(), torch.zeros((), dtype=torch.float64, device=DEV)))
    for r in convs:
        if r["ptr"] == ptr and tuple(r["x"].shape) == shape:
            assert r["g"] is not None, what + ": a torch convolution of the tensor received no gradient"
            kw = dict(stride=r["stride"], padding=r["padding"], dilation=r["dilation"], groups=r["groups"])
            w, gd = r["w"].detach().double(), r["g"].double()
            ref = torch.nn.grad.conv2d_input(shape, w, gd, **kw)
            mag = torch.nn.grad.conv2d_input(shape, w.abs(), gd.abs(), **kw)
            n = w.shape[0] // r["groups"] * w.shape[2] * w.shape[3]
            parts.append((ref, S.store_bound(ref, S.gamma_tc(n + 1) * mag, BF)))
    parts += list(extra)
    assert parts, what + ": no consumer"
    tot = sum(v for v, _ in parts)
    err = sum(e for _, e in parts) + S.gamma_bf16(len(parts) - 1) * sum(v.abs() + e for v, e in parts)
    return tot, err



def _sb_err(s):
    """|bf16(sigmoid) - sigmoid|: half a bf16 ulp of the value plus the fp32 sigmoid's own error (a few fp32 ulp)"""
    return 0.5 * S.ulp(s, 8) + 2.0 ** -21


def check_split_gate(blk, db_call, hk, convs, bns, what):
    """SE-CoTNetD's split attention with DropBlock after bn0 runs SiLU -> pool -> fc1 -> bn1 -> SiLU -> fc2 -> sigmoid -> rescale
    in plain bf16 PyTorch.  Each backward link is checked against fp64 of the bf16 values that op received (recorded by the conv /
    BatchNorm recorders and hooks), so no error is carried from one op to the next: the sigmoid's gradient, fc2's data gradient
    through SiLU, bn1's backward (torch_bn_bwd_ref, with the conditioning of its batch statistics), and the gradient reaching the
    DropBlock output (direct term + the pooled gate branch).  fc1 / fc2 weights and biases and bn1's parameters are then accounted
    for by account_params from the same records."""
    sp = blk.conv2
    (r1,) = [r for r in convs if r["w"] is sp.fc1.weight]
    (r2,) = [r for r in convs if r["w"] is sp.fc2.weight]
    (rb,) = [r for r in bns if r["w"] is sp.bn1.weight]
    gy, a, d = hk["conv2_g"].double(), hk["act0"].double(), db_call.out.double()
    B, C, H, W = a.shape
    HW = H * W
    # sigmoid: d logits = sb (1 - sb) * sum_hw(bf16(gy * a)), sb the bf16 gate torch saved
    s = torch.sigmoid(r2["y"].double())
    es = _sb_err(s)
    prod = gy * a
    sig_g = prod.sum((2, 3), keepdim=True)
    e_sig = 2.0 ** -9 * prod.abs().sum((2, 3), keepdim=True) + S.gamma(HW + 1) * prod.abs().sum((2, 3), keepdim=True)
    e_sig = e_sig + 0.5 * S.ulp(sig_g.abs() + e_sig, 8)
    ref = s * (1 - s) * sig_g
    err = sig_g.abs() * es * ((1 - 2 * s).abs() + es) + (s * (1 - s)).abs() * e_sig + 4 * S.U32 * ref.abs()
    S.within(r2["g"], ref, S.store_bound(ref, err, BF), what + " gate: sigmoid backward")
    # fc2's data gradient through act1 (SiLU) -> gradient at bn1's output
    w2 = r2["w"].detach().double()
    dh = torch.nn.grad.conv2d_input(tuple(r2["x"].shape), w2, r2["g"].double())
    mh = torch.nn.grad.conv2d_input(tuple(r2["x"].shape), w2.abs(), r2["g"].double().abs())
    e_dh = S.store_bound(dh, S.gamma_tc(w2.shape[0] + 1) * mh, BF)
    z2 = rb["y"].double()
    sg = torch.sigmoid(z2)
    sd = sg * (1 + z2 * (1 - sg))
    ref = dh * sd
    S.within(rb["g"], ref, S.store_bound(ref, sd.abs() * e_dh + 8 * S.U32 * (dh * sd).abs(), BF), what + " gate: fc2 dgrad + SiLU")
    # bn1 backward (batch statistics over the B pooled samples) -> gradient at fc1's output
    br = torch_bn_bwd_ref(rb)
    S.within(r1["g"], br["dx"], S.store_bound(br["dx"], br["dx_err"], BF), what + " gate: bn1 backward")
    # the DropBlock output's gradient: act0 (SiLU) of gy * sb + the pooled branch d(gap) / HW
    w1 = r1["w"].detach().double()
    dg = torch.nn.grad.conv2d_input(tuple(r1["x"].shape), w1, r1["g"].double())
    mg = torch.nn.grad.conv2d_input(tuple(r1["x"].shape), w1.abs(), r1["g"].double().abs())
    e_dg = S.store_bound(dg, S.gamma_tc(w1.shape[0] + 1) * mg, BF) / HW
    dg = dg / HW
    e_dg = e_dg + 0.5 * S.ulp(dg.abs() + e_dg, 8)
    t1 = gy * s
    e_t1 = gy.abs() * es + 0.5 * S.ulp(t1.abs() + gy.abs() * es, 8)
    tot = t1 + dg
    e_tot = e_t1 + e_dg + 0.5 * S.ulp(tot.abs() + e_t1 + e_dg, 8)
    sg0 = torch.sigmoid(d)
    sd0 = sg0 * (1 + d * (1 - sg0))
    ref = tot * sd0
    S.within(db_call.gin[0], ref, S.store_bound(ref, sd0.abs() * e_tot + 8 * S.U32 * ref.abs(), BF),
             what + " gate: gradient reaching the DropBlock output")


def observed_flow(calls, convs, x_ptr, x, blurs=None, order=None):
    """every recorded call argument and torch convolution input that is (by storage, shape and value) an earlier recorded call's
    output or the block input x: {"i.a" or "c<j>": "k.o" or "x"}.  blurs ({conv index: pad record}, with `order`): a BlurPool's output
    is a producer too ("c<j>"), and its convolution reads "pad(k.o)", the reflect padding of a recorded output."""
    ptrs = {}
    # times: call i at (i, 1, 0); torch convolution j, made after order[j] recorded calls, at (order[j], 0, j)
    for i, c in enumerate(calls):
        for o, (pt, snap) in enumerate(zip(c.out_ptr, c.out if isinstance(c.out, tuple) else (c.out,))):
            ptrs.setdefault(pt, []).append(("%d.%d" % (i, o), (i, 1, 0), snap))
    if x is not None:
        ptrs.setdefault(x_ptr, []).append(("x", (-1, 1, 0), x.detach()))
    for j in sorted(blurs or ()):
        r = convs[j]
        ptrs.setdefault(r["out_ptr"], []).append(("c%d" % j, (order[j], 0, j), r["y"]))
    edges = {}

    def find(ptr, shape, val, t):
        cands = sorted([(tp, n, sn) for n, tp, sn in ptrs.get(ptr, []) if tp < t and tuple(sn.shape) == shape], key=lambda e: e[0])
        if not cands:
            return None
        _, n, sn = cands[-1]                                 # the latest producer at that storage
        S.equal(val, sn, "%s == %s" % ("consumer", n))
        return n
    for i, c in enumerate(calls):
        for a, arg in enumerate(c.args):
            if isinstance(arg, torch.Tensor):
                n = find(arg.data_ptr(), tuple(arg.shape), c.inp[a], (i, 1, 0))
                if n is not None:
                    edges["%d.%d" % (i, a)] = n
    return edges, ptrs


def _conv_edges(convs, ptrs, order, blurs=None):
    """torch convolution inputs produced by recorded calls (or by a BlurPool): order[j] is the number of recorded calls made before
    conv j; a BlurPool's convolution reads the padding of its producer's output ("pad(k.o)")"""
    edges = {}
    for j, r in enumerate(convs):
        src = (blurs or {}).get(j)
        ptr, val = (src["ptr"], src["x"]) if src is not None else (r["ptr"], r["x"])
        cands = sorted([(tp, n, sn) for n, tp, sn in ptrs.get(ptr, []) if tp < (order[j], 0, j) and tuple(sn.shape) == tuple(val.shape)],
                       key=lambda e: e[0])
        if cands:
            _, n, sn = cands[-1]
            S.equal(val, sn, "c%d == %s" % (j, n))
            edges["c%d" % j] = "pad(%s)" % n if src is not None else n
    return edges


def blur_producers(calls, convs, blurs, order):
    """{conv index: the recorded call whose output the BlurPool's pad read} (the latest at that storage before the pad)"""
    out = {}
    for j, p in blurs.items():
        cands = [c for i, c in enumerate(calls) if i < order[j] and c.out_ptr[0] == p["ptr"] and tuple(c.out.shape if not
                 isinstance(c.out, tuple) else c.out[0].shape) == tuple(p["x"].shape)]
        assert cands, "c%d: the BlurPool's input is no recorded call's output" % j
        out[j] = cands[-1]
    return out


class _Order:
    """the number of recorded calls made before each torch convolution (conv2d wrapped once more, outside ConvRecorder)"""

    def __init__(self, monkeypatch, rec):
        self.order = []
        conv0 = F.conv2d

        def conv2d(*a, **k):
            self.order.append(len(rec.calls))
            return conv0(*a, **k)
        monkeypatch.setattr(torch.nn.functional, "conv2d", conv2d)


@pytest.mark.parametrize("geo", sorted(S.STEP_BLOCK_CASES))
def test_block_stage_by_stage(geo, monkeypatch):
    """one forward and backward of a bf16 block or stem: (a) the recorded calls, (b) every call's stage check, (c) DropBlock sites,
    keys and drop-path scales, (d) the block input's gradient as the sum of its consumers', (e) every parameter accounted for,
    (f) the stated dataflow"""
    case = S.STEP_BLOCK_CASES[geo]
    if case.get("min_pixels") is not None:
        monkeypatch.setattr(fused, "TC_MIN_PIXELS", case["min_pixels"])
    model = _model(case)
    g = torch.Generator(device=DEV).manual_seed(7)
    B = case["B"]
    ds = torch.tensor(case["ds"], device=DEV) if case.get("ds") is not None else None
    key = torch.tensor(KEY, device=DEV) if case.get("sites") else None
    if case["kind"] == "stem":
        part = nn.ModuleDict(dict(conv1=model.conv1, bn1=model.bn1)).to(DEV).to(BF).to(memory_format=CL).train()
        _randomise_bn(part)
        x = _cl(torch.randn(B, 3, case["H"], case["W"], generator=g, device=DEV).to(BF))
        ref_model = copy.deepcopy(model)
        for m in (model, ref_model):
            m._run_blocks = lambda t: t                  # forward_features runs the stem only
        ref_part = nn.ModuleDict(dict(conv1=ref_model.conv1, bn1=ref_model.bn1))
        x0 = x
        run, ref_run = model.forward_features, ref_model.forward_features
    else:
        stage, i = case["block"].split(".")
        part = getattr(model, stage)[int(i)]
        _randomise_bn(part)
        part = part.to(DEV).to(BF).to(memory_format=CL).train()
        H, C = case["H"], case["cin"]
        x = torch.relu(_cl(torch.randn(B, C, H, H, generator=g, device=DEV).to(BF))).requires_grad_(True)
        ref_part = copy.deepcopy(part)
        x0 = x.detach().clone().requires_grad_(True)
        run = lambda t: part(t, drop_scale=ds, drop_block_key=key)          # noqa: E731
        ref_run = lambda t: ref_part(t, drop_scale=ds, drop_block_key=key)  # noqa: E731
    n0 = _lib.launch_count()
    ref_out = ref_run(x0)
    dy = _cl(torch.randn(tuple(ref_out.shape), generator=g, device=DEV).to(BF))
    ref_out.backward(dy)
    n_plain = _lib.launch_count() - n0
    hooks = {}
    if case["kind"] == "block" and getattr(part, "downsample", None) is not None and isinstance(part.downsample[0], nn.AvgPool2d):
        def pool_hook(m, i, o):                   # avg_down: torch's 2x2 average pool in front of the 1x1 convolution
            hooks["pool"] = dict(out_ptr=o.data_ptr(), shape=tuple(o.shape), pool=m)
            o.register_hook(lambda gr: hooks["pool"].__setitem__("g", gr.detach().clone()))
        part.downsample[0].register_forward_hook(pool_hook)
    gate = case.get("sites") and hasattr(part.conv2, "fc1")
    if gate:
        _gate_hooks(part, hooks)
    rec = S.Recorder(monkeypatch)
    convs = ConvRecorder(monkeypatch).calls
    pads = PadRecorder(monkeypatch, convs).calls
    bns = TorchBNRecorder(monkeypatch).calls
    order = _Order(monkeypatch, rec).order
    derived = S.DerivedRecorder(monkeypatch).of
    n0 = _lib.launch_count()
    out = run(x)
    out.backward(dy)
    # the recorders change nothing
    assert _lib.launch_count() - n0 == n_plain, "the recorder changed the launches"
    S.equal(out, ref_out, "output with / without the recorder")
    if case["kind"] == "block":
        S.equal(x.grad, x0.grad, "dX with / without the recorder")
    for (n, p), (_, q) in zip(part.named_parameters(), ref_part.named_parameters()):
        S.equal(p.grad, q.grad, "%s.grad with / without the recorder" % n)
    for (n, b), (_, c) in zip(part.named_buffers(), ref_part.named_buffers()):
        S.equal(b, c, "%s with / without the recorder" % n)
    # (a)
    assert [_cfg(c) for c in rec.calls] == case["calls"], [_cfg(c) for c in rec.calls]
    # (b)
    mods = tail_mods(part)
    for c in rec.calls:
        check_call(c, mods)
    # (c) DropBlock: the block's own site numbers in forward order, the key it was handed, something dropped and something kept;
    # drop path: every scale the kernels read is the block's row
    dbc = [c for c in rec.calls if c.name in S.DROPBLOCK_FNS]
    assert [c.extra["site"] for c in dbc] == list(case.get("sites") or ()), [c.extra["site"] for c in dbc]
    _check_sites_and_scales(rec.calls, ds, "")
    # (d) the block input's gradient: its consumers' returned gradients, conv2d_input of its torch convolutions, and the fp64
    # adjoint of the avg_down pool at the gradient autograd delivered to the pool's output (itself checked as a sum)
    if case["kind"] == "block":
        _check_input_grad(x, x.grad, rec.calls, convs, hooks.get("pool"), geo)
    if gate:
        check_split_gate(part, dbc[1], hooks, convs, bns, geo)
    # the BlurPools (se_cotnetd_152): output against fp64 of the filter on the reflect-padded input, the gradient reaching their input
    blurs = blur_convs(convs, pads)
    for j, prod in blur_producers(rec.calls, convs, blurs, order).items():
        check_blur(convs[j], blurs[j], "%s c%d" % (geo, j), prod)
    assert len(blurs) == (1 if case["model"] == "se_cotnetd_152" and case.get("stride") == 2 else 0), geo
    # (e)
    account_params(part, rec.calls, convs, geo, derived, bns=bns)
    if case["model"] == "cotnext50_2x48d":
        assert len(derived) == 4, "CoXt: key conv, embed.0, embed.3 and conv1x1 weights derive dense weights"
    # (f) the stated dataflow: every recorded input (call argument or torch convolution input) that is an earlier call's output or
    # the block input, and nothing else
    edges, ptrs = observed_flow(rec.calls, convs, x.data_ptr(), x if case["kind"] == "block" else None, blurs, order)
    edges.update(_conv_edges(convs, ptrs, order, blurs))
    got = sorted("%s<-%s" % kv for kv in edges.items())
    assert got == sorted(case.get("flow", ())), "%s dataflow: %s" % (geo, got)


def _gate_hooks(blk, hooks):
    """the gradient of the split-attention conv2's output and act0's (in-place SiLU) output, for check_split_gate"""
    def conv2_hook(m, i, o):
        o.register_hook(lambda gr: hooks.__setitem__("conv2_g", gr.detach().clone()))

    def act0_hook(m, i, o):
        hooks["act0"] = o.detach().clone()
    blk.conv2.register_forward_hook(conv2_hook)
    blk.conv2.act0.register_forward_hook(act0_hook)


def _check_sites_and_scales(calls, ds, what):
    for c in calls:
        if c.name in S.DROPBLOCK_FNS:
            S.equal(c.extra["key"].cpu(), torch.tensor(KEY), what + "DropBlock key")
            n = int(c.inp[2 if c.name == "DropBlockFn" else 3].item())
            assert 0 < n < c.inp[0].numel(), "%ssite %d: kept %d of %d" % (what, c.extra["site"], n, c.inp[0].numel())
    carried = []
    ds_arg = {"BNActFn": 6, "TcConv1x1Fn": 9, "DropBlockResReluFn": 4}
    for c in calls:
        d = (tuple(c.args) + (None,) * 10)[ds_arg[c.name]] if c.name in ds_arg else None
        if d is not None:
            carried.append(c.name)
            assert ds is not None and torch.equal(d.float(), ds.float()), "%s%s got drop-path scales %s, not %s" % (what, c.name, d, ds)
    assert len(carried) == (0 if ds is None else 1), what + str(carried)          # bn3's site only


def _check_input_grad(x, got, calls, convs, pool, what):
    extra = []
    if pool is not None:
        gp, gp_err = _consumer_sum(pool["out_ptr"], pool["shape"], calls, convs, (), what + " avg_down pool output")
        S.within(pool["g"], gp, gp_err, what + " gradient of the avg_down pool output")
        m = pool["pool"]
        x64 = x.detach().double().requires_grad_(True)
        pooled = F.avg_pool2d(x64, m.kernel_size, m.stride, m.padding, m.ceil_mode, m.count_include_pad)
        (dx,) = torch.autograd.grad(pooled, x64, pool["g"].double())
        extra.append((dx, S.store_bound(dx, S.U32 * dx.abs(), BF)))
    tot, err = _consumer_sum(x.data_ptr(), tuple(x.shape), calls, convs, extra, what + " block input")
    S.within(got, tot, err, what + " block input gradient = the sum of its consumers'")


# ------------------------------------------------------------------------------------------------ whole TrainStep backward passes
def check_soft_ce(call, what="SoftTargetCrossEntropyFn"):
    """the label-smoothed soft-target loss (no mixing) and its logits gradient against fp64 of the recorded logits:
    t = (1 - s) onehot + s / K, loss = mean_b(lse_b - sum_c t_c z_c), dz = dloss (softmax(z) - t) / B.  Bounds: the exponentials
    within expf_rel_err of their arguments, the K-term sum gamma(K + 1), the log and the subtractions a few u of their magnitude,
    the batch mean gamma(B + 1); dz is computed in fp32 and stored in the logits' dtype."""
    z, lab, mix, smoothing = call.inp
    assert mix is None
    B, K = z.shape
    zz = z.double()
    t = torch.full_like(zz, smoothing / K)
    t[torch.arange(B), lab] += 1 - smoothing
    m = zz.max(1, keepdim=True)[0]
    rel = S.expf_rel_err(zz - m).max(1, keepdim=True)[0] + S.gamma(K + 1) + 4 * S.U32
    lse = m + torch.log(torch.exp(zz - m).sum(1, keepdim=True))
    rows = lse[:, 0] - (t * zz).sum(1)
    e_rows = rel[:, 0] + 8 * S.U32 * (lse.abs()[:, 0] + m.abs()[:, 0]) + S.gamma(K + 1) * (t * zz).abs().sum(1) + 4 * S.U32 * rows.abs()
    loss = rows.mean()
    S.within(call.out, loss, e_rows.mean() + S.gamma(B + 1) * rows.abs().mean() + S.ulp(loss, 24), what + " loss")
    dl = call.gin[0].double()
    p = torch.softmax(zz, 1)
    dz = dl * (p - t) / B
    err = dl.abs() * (p * 2 * rel + 4 * S.U32 * (p + t)) / B
    S.within(call.gout[0], dz, S.store_bound(dz, err, call.gout[0].dtype), what + " dz")


def _fixed_scales(model, B):
    """[n_blocks, B] drop-path scales: 1/keep of each block's rate, one zero per row at a sample that moves with the block, so
    consecutive rows differ"""
    rates = model.drop_path_rates()
    s = torch.tensor([[0.0 if b == i % B else 1.0 / (1.0 - r) for b in range(B)] for i, r in enumerate(rates)], dtype=torch.float32)
    return s


TRAIN_CASES = {"cotnet50": ("cotnet50", None), "cotnet50_all_wgmma": ("cotnet50", 0), "cotnext50_2x48d": ("cotnext50_2x48d", None),
               "se_cotnetd_50": ("se_cotnetd_50", None)}


@pytest.mark.parametrize("name", sorted(TRAIN_CASES))
def test_train_step_stage_by_stage(name, monkeypatch):
    """TrainStep(weights="bf16", label_smoothing=0.1, lr=0).forward_backward at B=4, 96x96, drop path 0.1 (fixed scales with zeros)
    and DropBlock 0.1 (fixed key): (1) the call list, (2) every block's drop-path row and DropBlock sites, (3) every stage check,
    (4) block-to-block dataflow, (5) the gradient at every block input and at the last block's output as the sum of its
    consumers', (6) the head, (7) the flat buckets against .grad and every parameter accounted for"""
    mname, mp = TRAIN_CASES[name]
    train_step_stage_by_stage(name, mname, mp, monkeypatch)


def train_step_stage_by_stage(name, mname, mp, monkeypatch, B=4, H0=96, drop_path=0.1, drop_block=0.1):
    """the body of test_train_step_stage_by_stage for any model, batch, image size and rates (drop_block 0: no DropBlock); the
    BlurPools of se_cotnetd_152 are checked as in test_block_stage_by_stage"""
    from cotnet_b200 import backbone, backbone_hybrid, trainer
    if mp is not None:
        monkeypatch.setattr(fused, "TC_MIN_PIXELS", mp)
    torch.manual_seed(5)
    K = 100
    ctor = {"cotnet50": backbone.cotnet50, "cotnext50_2x48d": backbone.cotnext50_2x48d, "se_cotnetd_50": backbone_hybrid.se_cotnetd_50,
            "se_cotnetd_152": backbone_hybrid.se_cotnetd_152}
    model = ctor[mname](num_classes=K, drop_path_rate=drop_path, drop_block_rate=drop_block)
    _randomise_bn(model)
    model = model.to(DEV).to(memory_format=CL).train()
    scales = _fixed_scales(model, B)
    model.fixed_drop_path_scales = scales
    model.fixed_drop_block_key = torch.tensor(KEY)
    ts = trainer.TrainStep(model, weights="bf16", label_smoothing=0.1, lr=0)
    blocks = model.blocks()
    names = [n for n, *_ in S.model_blocks(mname, H0)]
    assert [getattr(model, n.split(".")[0])[int(n.split(".")[1])] for n in names] == blocks
    rec = S.Recorder(monkeypatch)
    convs = ConvRecorder(monkeypatch).calls
    pads = PadRecorder(monkeypatch, convs).calls
    bns = TorchBNRecorder(monkeypatch).calls
    order = _Order(monkeypatch, rec).order
    derived = S.DerivedRecorder(monkeypatch).of
    info = [dict() for _ in blocks]
    for i, blk in enumerate(blocks):
        def pre(m, args, i=i):
            info[i].update(x=args[0], x_snap=args[0].detach().clone(), c0=len(rec.calls), v0=len(convs))

        def post(m, args, out, i=i):
            info[i].update(out_ptr=out.data_ptr(), out_snap=out.detach().clone(), c1=len(rec.calls), v1=len(convs))
        blk.register_forward_pre_hook(pre)
        blk.register_forward_hook(post)
        if getattr(blk, "downsample", None) is not None and isinstance(blk.downsample[0], nn.AvgPool2d):
            def pool_hook(m, a, o, i=i):
                info[i]["pool"] = dict(out_ptr=o.data_ptr(), shape=tuple(o.shape), pool=m)
                o.register_hook(lambda gr: info[i]["pool"].__setitem__("g", gr.detach().clone()))
            blk.downsample[0].register_forward_hook(pool_hook)
    head = {}

    def fc_hook(m, a, o):
        head["feat"] = a[0].detach().clone()
        a[0].register_hook(lambda gr: head.__setitem__("gfeat", gr.detach().clone()))
    model.fc.register_forward_hook(fc_hook)
    g = torch.Generator(device=DEV).manual_seed(3)
    x = _cl(torch.randn(B, 3, H0, H0, generator=g, device=DEV).to(BF))
    lab = torch.randint(0, K, (B,), generator=g, device=DEV)
    ts.forward_backward(x, lab)
    # (1)
    stem, bl, loss_calls = S.model_calls(mname, B, H0, S.TC_MIN_PIXELS if mp is None else mp, drop_block > 0)
    cfgs = [_cfg(c) for c in rec.calls]
    assert cfgs == stem + sum(bl, []) + loss_calls, cfgs
    for i in range(len(blocks)):
        assert cfgs[info[i]["c0"]:info[i]["c1"]] == bl[i], (names[i], cfgs[info[i]["c0"]:info[i]["c1"]])
    # (2) drop path and DropBlock per block
    sites = S.model_sites(mname) if drop_block > 0 else {}
    table = {}
    for bname, _, site, _ in model.drop_block_table():
        table.setdefault(bname, []).append(site)
    for i, n in enumerate(names):
        cs = rec.calls[info[i]["c0"]:info[i]["c1"]]
        _check_sites_and_scales(cs, None if i == 0 else scales[i].to(DEV), n + ": ")
        got = [c.extra["site"] for c in cs if c.name in S.DROPBLOCK_FNS]
        assert got == list(sites.get(n, ())) == table.get(n, []), (n, got, sites.get(n), table.get(n))
    # (3)
    mods = tail_mods(model)
    for c in rec.calls:
        if c.name == "SoftTargetCrossEntropyFn":
            check_soft_ce(c)
        else:
            check_call(c, mods)
    # the plain-PyTorch split-attention gates (DropBlock after bn0) are checked op by op in the block case
    # hybrid_stage3_split_dropblock_b4; under the step's autocast the sigmoid link exceeds that derivation in a few elements
    # (up to 1.19 of the bound), so here their parameters are accounted for from the conv / BatchNorm records only
    # (4) the stem's output is block 0's input; block i's output (its last call's) is block i+1's input
    n_stem = len(stem)
    assert info[0]["x"].data_ptr() == rec.calls[n_stem - 1].out_ptr[0]
    S.equal(info[0]["x_snap"], rec.calls[n_stem - 1].out, "stem output == block 0 input")
    for i in range(len(blocks)):
        last = rec.calls[info[i]["c1"] - 1]
        assert info[i]["out_ptr"] == last.out_ptr[0], names[i]
        S.equal(info[i]["out_snap"], last.out, names[i] + " output == its last call's")
        if i + 1 < len(blocks):
            assert info[i + 1]["x"].data_ptr() == info[i]["out_ptr"], names[i + 1]
            S.equal(info[i + 1]["x_snap"], info[i]["out_snap"], "%s input == %s output" % (names[i + 1], names[i]))
    # (5) the gradient autograd delivered to each block input's producer (the stem's last call, the previous block's last call)
    for i in range(len(blocks)):
        prod = rec.calls[n_stem - 1] if i == 0 else rec.calls[info[i - 1]["c1"] - 1]
        _check_input_grad(info[i]["x"], prod.gin[0], rec.calls[info[i]["c0"]:info[i]["c1"]], convs[info[i]["v0"]:info[i]["v1"]],
                          info[i].get("pool"), "%s %s" % (name, names[i]))
    # every BlurPool: its output, and the gradient reaching its input, against fp64 (the pooled blocks of se_cotnetd_152)
    blurs = blur_convs(convs, pads)
    for j, prod in blur_producers(rec.calls, convs, blurs, order).items():
        check_blur(convs[j], blurs[j], "%s c%d" % (name, j), prod)
    assert len(blurs) == (4 if mname == "se_cotnetd_152" else 0), name
    # (6) head: global average pool -> fc -> loss
    (ce,) = rec.named("SoftTargetCrossEntropyFn")
    dz = ce.gout[0].double()
    feat = head["feat"].double()
    W = model.fc.weight.detach().double()
    ref = dz.t() @ feat
    S.within(model.fc.weight.grad, ref, S.store_bound(ref, S.gamma_tc(B + 1) * (dz.abs().t() @ feat.abs()), BF), name + " fc.weight")
    ref = dz.sum(0)
    S.within(model.fc.bias.grad, ref, S.store_bound(ref, S.gamma(B + 1) * dz.abs().sum(0), BF), name + " fc.bias")
    ref = dz @ W
    S.within(head["gfeat"], ref, S.store_bound(ref, S.gamma_tc(K + 1) * (dz.abs() @ W.abs()), BF), name + " fc input gradient")
    last = rec.calls[info[-1]["c1"] - 1]
    Hl, Wl = last.out.shape[2:]
    ref = (head["gfeat"].double() / (Hl * Wl)).view(B, -1, 1, 1).expand_as(last.out)
    S.within(last.gin[0], ref, S.store_bound(ref, S.U32 * ref.abs(), BF), name + " global pool backward")
    # (7) the flat buckets: bf16 G_big for the weights, fp32 G_small for the rest, bit for bit; every .grad accounted for
    grads = ts.grads()
    for n, p in model.named_parameters():
        assert grads[n].dtype == p.grad.dtype == (BF if p.dim() >= 2 else torch.float32), n
        S.equal(grads[n], p.grad, name + " bucket " + n)
    account_params(model, rec.calls, convs, name, derived, skip=("fc.weight", "fc.bias"), bns=bns)
