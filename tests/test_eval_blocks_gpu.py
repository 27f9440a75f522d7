"""The bf16 eval forward of whole blocks, stems and networks stage by stage, as EvalStep runs it (model.eval(), no_grad, bf16 autocast
without its weight-cast cache, step arena off): CoT, CoXt and SE-CoTNetD bottlenecks, both stems, non-square resolutions.

Per block or stem (stage_ref.EVAL_BLOCK_CASES): (a) the recorded calls equal the eval dispatch mirror's list, (b) every call against
fp64 of its own inputs within the bounds of tests/stage_ref.py and every BatchNorm fold within fold_bound of the running statistics,
(c) every torch (cuDNN) convolution's output against fp64 of its recorded bf16 input and weight, (d) the stated dataflow with no
unlisted edge, (e) outputs and launch counts bit-identical with and without the recorders.

Per network (cotnet50, cotnext50_2x48d, se_cotnetd_50; bf16 and fp32 weights; 224 x 224 and 232 x 200; every trunk 1x1 on wgmma):
the whole call list against stage_ref.eval_model_calls, every stage, stem -> block -> block dataflow and each block's input shape,
the global average pool and fc, and a captured EvalStep on the same batch: logits bit-equal to the recorded eager ones and counts
equal to the rank rule of them.  And fp32 weights holding bf16 values give the bf16-weight layout's logits bit for bit."""
import contextlib
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import stage_ref as S
from cotnet_b200 import _lib, evaler, fused
from cotnet_b200.cot_layer import CotLayer
from test_eval_gpu import rank_rule_counts
from test_eval_stages_gpu import _EvalRecorder, _check_fold, check_eval_layer, check_tail_eval
from test_stage_grads_gpu import ONE_ULP, ConvRecorder, PadRecorder, _cfg, _w, blur_convs, check_blur, check_call, tail_mods
from test_step_stages_gpu import _Order

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
CL = torch.channels_last
_CONV2D = F.conv2d                      # the reference convolutions bypass the recorders
_TC_CALLS = ("conv3x3_bf16", "gemm_bf16", "cot_tail_eval")


@pytest.fixture(autouse=True)
def _deterministic(monkeypatch):
    """no TF32; deterministic cuDNN, as the with / without recorder comparisons are bitwise"""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


@pytest.fixture(scope="module", autouse=True)
def _report_one_ulp():
    """after the module: per stage type, the fraction of bf16 outputs one ulp from the correctly rounded fp64 value"""
    ONE_ULP.clear()
    yield
    for k in sorted(ONE_ULP):
        one, far, n = ONE_ULP[k]
        print("\neval bf16 outputs one ulp off, %-10s %.2e (%d of %d; %d farther)" % (k, one / max(n, 1), one, n, far), end="")


@contextlib.contextmanager
def _eval_body():
    """the conditions of EvalStep._body"""
    fused.step_arena_off()
    with torch.no_grad(), torch.autocast("cuda", dtype=BF, cache_enabled=False):
        yield


def _cl(t):
    return t.contiguous(memory_format=CL)


def _ctor(name):
    from cotnet_b200 import backbone, backbone_hybrid
    return {"cotnet50": backbone.cotnet50, "cotnext50_2x48d": backbone.cotnext50_2x48d, "se_cotnetd_50": backbone_hybrid.se_cotnetd_50,
            "se_cotnetd_152": backbone_hybrid.se_cotnetd_152, "se_cotnetd_152_L": backbone_hybrid.se_cotnetd_152_L}[name]


def _randomise(mod, seed):
    """BatchNorm affine parameters and running statistics away from their defaults"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5, generator=g)
                m.bias.uniform_(-0.25, 0.25, generator=g)
                m.running_mean.normal_(0, 0.2, generator=g)
                m.running_var.uniform_(0.6, 1.6, generator=g)
    return mod


def _layout(mod, bf16):
    """bf16: the layout TrainStep(weights="bf16") gives the model (convolution and fc weights bf16, the rest fp32)"""
    if bf16:
        for p in mod.parameters():
            if p.dim() >= 2:
                p.data = p.data.to(BF)
    return mod


def _label(c):
    return c.name if c.name in _TC_CALLS else _cfg(c)


# ------------------------------------------------------------------------------------------------ checks
def check_eval_calls(calls, model, what):
    """every recorded call of an eval forward of (part of) `model` against fp64 of its own inputs, and every BatchNorm fold"""
    mods = tail_mods(model)
    layers = {id(m._tc_cache["wk"]): m for m in model.modules() if isinstance(m, CotLayer) and getattr(m, "_tc_cache", None)}
    i = 0
    while i < len(calls):
        c = calls[i]
        w = "%s call %d %s" % (what, i, _label(c))
        if c.name == "conv3x3_bf16":              # a CotLayer's _forward_tc_eval: its seven calls
            grp = calls[i:i + 7]
            check_eval_layer(grp, layers[id(c.args[1])], c.inp[0], grp[6].out[3], w)
            i += 7
            continue
        assert c.name not in ("gemm_bf16",), w + ": a wgmma GEMM outside a CoT layer"
        if c.name == "cot_tail_eval":             # the eval tail after CotLayer._forward_fused
            check_tail_eval(c, c.extra["bn"], c.extra["se"], w)
        else:
            check_call(c, mods)
            if c.name == "BNActFn":
                assert c.apply is None, w + ": batch statistics in eval"
                _check_fold(c.saved[2][0], c.saved[2][1], c.args[4], w)
            elif c.name in ("TcConv1x1Fn", "StemConvBNFn") and "fold" in c.extra:
                bn, scale, shift = c.extra["fold"][:3]
                _check_fold(scale, shift, bn, w)
            elif c.name == "CotTailFn":
                assert not c.extra["training"], w
                _check_fold(c.saved[2], c.saved[3], c.args[4], w)
            assert c.name not in ("TcConv1x1Fn", "StemConvBNFn") or c.args[6 if c.name == "TcConv1x1Fn" else 4] is None \
                or "fold" in c.extra, w + ": no eval fold"
        i += 1


def check_torch_conv(r, what):
    """a cuDNN convolution under autocast: its output against fp64 of the recorded bf16 input and the weight (and bias) autocast cast
    to bf16; fp32 accumulation (gamma_tc of the terms per output) and the bf16 store"""
    x = r["x"]
    assert x.dtype == BF and r["y"].dtype == BF, what
    w = r["w"].detach().to(BF).double()
    b = None if r["b"] is None else r["b"].detach().to(BF).double()
    kw = dict(stride=r["stride"], padding=r["padding"], dilation=r["dilation"], groups=r["groups"])
    ref = _CONV2D(x.double(), w, b, **kw)
    mag = _CONV2D(x.double().abs(), w.abs(), None if b is None else b.abs(), **kw)
    n = w.shape[1] * w.shape[2] * w.shape[3] + (b is not None)
    _w(r["y"], ref, S.gamma_tc(n + 1) * mag, what + " cuDNN convolution output", "cudnn_conv")


def _rows_view(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]) if t.dim() == 4 else t


def eval_flow(calls, convs, order, x, blurs=None):
    """every recorded call argument and torch convolution input that is an earlier recorded output (or x), matched by storage and
    compared by value in NHWC row order: sorted "consumer<-producer" edges.  The recorder holds every output, so no storage is
    reused during the forward.  blurs ({conv index: pad record}): a BlurPool's output is a producer ("c<j>") and its convolution
    reads "pad(k.o)", the reflect padding of a recorded output."""
    prod = {}
    # times: call i at (i, 1, 0); torch convolution j, made after order[j] recorded calls, at (order[j], 0, j)
    for i, c in enumerate(calls):
        for o, (pt, snap) in enumerate(zip(c.out_ptr, c.out if isinstance(c.out, tuple) else (c.out,))):
            prod.setdefault(pt, []).append(("%d.%d" % (i, o), (i, 1, 0), snap))
    prod.setdefault(x.data_ptr(), []).append(("x", (-1, 1, 0), x.detach()))
    for j in sorted(blurs or ()):
        prod.setdefault(convs[j]["out_ptr"], []).append(("c%d" % j, (order[j], 0, j), convs[j]["y"]))

    def find(ptr, snap, t, what):
        cands = sorted([(tp, n, s) for n, tp, s in prod.get(ptr, []) if tp < t and _rows_view(s).shape == _rows_view(snap).shape],
                       key=lambda e: e[0])
        if not cands:
            return None
        _, n, s = cands[-1]
        S.equal(_rows_view(snap), _rows_view(s), "%s == %s" % (what, n))
        return n
    edges = {}
    for i, c in enumerate(calls):
        for a, arg in enumerate(c.args):
            if isinstance(arg, torch.Tensor):
                n = find(arg.data_ptr(), c.inp[a], (i, 1, 0), "%d.%d" % (i, a))
                if n is not None:
                    edges["%d.%d" % (i, a)] = n
    for j, r in enumerate(convs):
        src = (blurs or {}).get(j)
        n = find(src["ptr"] if src else r["ptr"], src["x"] if src else r["x"], (order[j], 0, j), "c%d" % j)
        if n is not None:
            edges["c%d" % j] = "pad(%s)" % n if src else n
    return sorted("%s<-%s" % kv for kv in edges.items())


# ------------------------------------------------------------------------------------------------ blocks and stems
@pytest.mark.parametrize("geo", sorted(S.EVAL_BLOCK_CASES))
def test_eval_block_stage_by_stage(geo, monkeypatch):
    """one eval forward of a bf16 block or stem: (a) the call list, (b) every call and fold, (c) every cuDNN convolution output,
    (d) the stated dataflow, (e) bit-identical with and without the recorders"""
    case = S.EVAL_BLOCK_CASES[geo]
    if case.get("min_pixels") is not None:
        monkeypatch.setattr(fused, "TC_MIN_PIXELS", case["min_pixels"])
    torch.manual_seed(5)
    model = _randomise(_ctor(case["model"])(), 3)
    g = torch.Generator(device=DEV).manual_seed(7)
    B, H, W = case["B"], case["H"], case["W"]
    if case["kind"] == "stem":
        part = nn.ModuleDict(dict(conv1=model.conv1, bn1=model.bn1))
        model._run_blocks = lambda t: t                   # forward_features runs the stem only
        run = model.forward_features
        x = _cl(torch.randn(B, 3, H, W, generator=g, device=DEV).to(BF))
    else:
        stage, i = case["block"].split(".")
        part = run = getattr(model, stage)[int(i)]
        x = torch.relu(_cl(torch.randn(B, case["cin"], H, W, generator=g, device=DEV).to(BF)))
    _layout(part.to(DEV).to(memory_format=CL), case["bf16"]).eval()
    with _eval_body():
        run(x)                                            # builds the eval weight caches
        n0 = _lib.launch_count()
        plain = run(x)
        n_plain = _lib.launch_count() - n0
    rec = _EvalRecorder(monkeypatch, keep_outputs=True)
    conv_rec = ConvRecorder(monkeypatch)
    pad_rec = PadRecorder(monkeypatch, conv_rec.calls)
    order_rec = _Order(monkeypatch, rec)
    with _eval_body():
        n0 = _lib.launch_count()
        out = run(x)
        n_rec = _lib.launch_count() - n0
    calls, convs, order = rec.calls, list(conv_rec.calls), list(order_rec.order)
    blurs = blur_convs(convs, pad_rec.calls)
    assert len(blurs) == (1 if case["model"] == "se_cotnetd_152" and case.get("stride") == 2 else 0), geo
    # (e)
    assert n_rec == n_plain, "the recorders changed the launches"
    S.equal(out, plain, geo + " output with / without the recorders")
    # (a)
    assert [_label(c) for c in calls] == case["calls"], [_label(c) for c in calls]
    # (b)
    check_eval_calls(calls, part, geo)
    # (c)
    for j, r in enumerate(convs):
        check_torch_conv(r, "%s c%d" % (geo, j))
    for j, p in blurs.items():
        check_blur(convs[j], p, "%s c%d" % (geo, j))
    # (d)
    got = eval_flow(calls, convs, order, x, blurs)
    assert got == sorted(case["flow"]), "%s dataflow: %s" % (geo, got)
    S.equal(out, calls[-1].out if not isinstance(calls[-1].out, tuple) else calls[-1].out[-1], geo + " output = the last call's")


# ------------------------------------------------------------------------------------------------ whole networks through EvalStep
NET_CASES = {
    "cotnet50_224_bf16w": ("cotnet50", (224, 224), True, None),
    "cotnet50_224_all_wgmma": ("cotnet50", (224, 224), True, 0),
    "cotnet50_232x200_fp32w": ("cotnet50", (232, 200), False, None),
    "cotnext50_224_bf16w": ("cotnext50_2x48d", (224, 224), True, None),
    "se_cotnetd50_224_bf16w": ("se_cotnetd_50", (224, 224), True, None),
}


def _net(mname, bf16, K=100):
    torch.manual_seed(5)
    model = _randomise(_ctor(mname)(num_classes=K, zero_init_last_bn=False), 3)
    return _layout(model.to(DEV).to(memory_format=CL), bf16).eval()


@pytest.mark.parametrize("name", sorted(NET_CASES))
def test_eval_network_stage_by_stage(name, monkeypatch):
    """one eager eval forward at B=2, recorded: (1) the whole call list and each block's, (2) every stage and cuDNN convolution,
    (3) stem -> block -> block dataflow and each block's input shape, (4) the global average pool and fc, (5) a captured EvalStep
    on the same batch gives the same logits bit for bit and the rank rule's counts of them"""
    mname, (H0, W0), bf16, mp = NET_CASES[name]
    eval_network_stage_by_stage(name, mname, H0, W0, bf16, mp, monkeypatch)


def eval_network_stage_by_stage(name, mname, H0, W0, bf16, mp, monkeypatch, B=2, bn3_gain=1.0):
    """the body of test_eval_network_stage_by_stage for any model, image size and batch; every BlurPool (se_cotnetd_152) against
    fp64 of its filter on the reflect-padded input.  bn3_gain scales each block's last BatchNorm weight: random running statistics
    do not normalise, so each residual branch multiplies the activations by a factor of order its bn3 gain, and over a deep trunk
    (50 blocks) they would leave fp32's range."""
    if mp is not None:
        monkeypatch.setattr(fused, "TC_MIN_PIXELS", mp)
    K, ks = 100, (1, 5)
    model = _net(mname, bf16, K)
    if bn3_gain != 1.0:
        with torch.no_grad():
            for blk in model.blocks():
                blk.bn3.weight.mul_(bn3_gain)
    g = torch.Generator(device=DEV).manual_seed(3)
    x = _cl(torch.randn(B, 3, H0, W0, generator=g, device=DEV).to(BF))
    lab = torch.randint(0, K, (B,), generator=g, device=DEV)
    # (5, first) the captured graph, before any recorder is in place
    ev = evaler.EvalStep(model, B, (H0, W0), topk=ks)
    ev.capture()
    glogits = ev.run(x, lab).clone()
    gcounts = ev.counts["live"].cpu().tolist()
    blocks = model.blocks()
    mb = S.model_blocks(mname, H0, W0)
    assert [getattr(model, n.split(".")[0])[int(n.split(".")[1])] for n, *_ in mb] == blocks
    rec = _EvalRecorder(monkeypatch, keep_outputs=True)
    conv_rec = ConvRecorder(monkeypatch)
    pad_rec = PadRecorder(monkeypatch, conv_rec.calls)
    info = [dict() for _ in blocks]
    hooks = []
    for i, blk in enumerate(blocks):
        def pre(m, args, i=i):
            info[i].update(x_ptr=args[0].data_ptr(), x_snap=args[0].detach().clone(), c0=len(rec.calls))

        def post(m, args, out, i=i):
            info[i].update(out_ptr=out.data_ptr(), out_snap=out.detach().clone(), c1=len(rec.calls))
        hooks += [blk.register_forward_pre_hook(pre), blk.register_forward_hook(post)]
    head = {}

    def fc_hook(m, a, o):
        head.update(feat=a[0].detach().clone(), logits=o.detach().clone())
    hooks.append(model.fc.register_forward_hook(fc_hook))
    with _eval_body():
        logits = model(x)
    for h in hooks:
        h.remove()
    calls, convs = rec.calls, list(conv_rec.calls)
    # (1)
    stem, bl = S.eval_model_calls(mname, B, H0, W0, bf16, S.TC_MIN_PIXELS if mp is None else mp)
    labels = [_label(c) for c in calls]
    assert labels == stem + sum(bl, []), labels
    for i in range(len(blocks)):
        assert labels[info[i]["c0"]:info[i]["c1"]] == bl[i], (mb[i][0], labels[info[i]["c0"]:info[i]["c1"]])
    # (2)
    check_eval_calls(calls, model, name)
    for j, r in enumerate(convs):
        check_torch_conv(r, "%s c%d" % (name, j))
    blurs = blur_convs(convs, pad_rec.calls)
    assert len(blurs) == (4 if mname.startswith("se_cotnetd_152") else 0), name
    for j, p in blurs.items():
        check_blur(convs[j], p, "%s c%d" % (name, j))
    # (3) the stem's output is block 0's input; block i's output (its last call's) is block i+1's input; input shapes
    n_stem = len(stem)
    assert info[0]["x_ptr"] == calls[n_stem - 1].out_ptr[0]
    S.equal(info[0]["x_snap"], calls[n_stem - 1].out, "stem output == block 0 input")
    for i, (bname, _, cin, _, cout, H, W, stride) in enumerate(mb):
        assert tuple(info[i]["x_snap"].shape) == (B, cin, H, W), (bname, tuple(info[i]["x_snap"].shape))
        assert tuple(info[i]["out_snap"].shape) == (B, cout, S.conv_out(H, stride), S.conv_out(W, stride)), bname
        last = calls[info[i]["c1"] - 1]
        assert info[i]["out_ptr"] == last.out_ptr[0], bname
        S.equal(info[i]["out_snap"], last.out, bname + " output == its last call's")
        if i + 1 < len(blocks):
            assert info[i + 1]["x_ptr"] == info[i]["out_ptr"], mb[i + 1][0]
    # (4) head: global average pool (fp32 accumulation, bf16 result) and fc under autocast (bf16 weight and bias)
    last = info[-1]["out_snap"].double()
    hw = last.shape[2] * last.shape[3]
    _w(head["feat"], last.mean((2, 3)), S.gamma(hw + 2) * last.abs().mean((2, 3)), name + " global average pool", "head_pool")
    f = head["feat"].to(BF).double()               # autocast runs fc on bf16 operands
    wf, bfc = model.fc.weight.detach().to(BF).double(), model.fc.bias.detach().to(BF).double()
    ref = f @ wf.t() + bfc
    _w(head["logits"], ref, S.gamma_tc(wf.shape[1] + 2) * (f.abs() @ wf.abs().t() + bfc.abs()), name + " fc", "head_fc")
    S.equal(logits, head["logits"], name + " logits = fc output")
    # (5)
    S.equal(glogits, logits, name + " captured EvalStep logits == the recorded eager logits")
    want = rank_rule_counts(logits.double().cpu().numpy(), lab.cpu().numpy(), ks)
    assert gcounts == want.tolist(), (gcounts, want.tolist())


@pytest.mark.parametrize("mname", ["cotnet50", "se_cotnetd_50"])
def test_fp32_weights_of_bf16_values_match_the_bf16_layout(mname):
    """every weight reaches its kernel as the same bf16 value in both layouts (CotLayer._tc_params, TcConv1x1Fn, prepare_stem_weight,
    autocast's conv / linear cast, .float() of the se and gate weights), so the logits are bit-identical"""
    m16 = _net(mname, True)
    m32 = copy.deepcopy(m16)
    for p in m32.parameters():
        p.data = p.data.float()
    assert all(p.dtype == torch.float32 for p in m32.parameters()) and any(p.dtype == BF for p in m16.parameters())
    g = torch.Generator(device=DEV).manual_seed(4)
    x = _cl(torch.randn(2, 3, 224, 224, generator=g, device=DEV).to(BF))
    with _eval_body():
        a, b = m32(x), m16(x)
    S.equal(a, b, mname + ": fp32 weights of bf16 values vs the bf16 layout")
