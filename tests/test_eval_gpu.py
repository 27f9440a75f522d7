"""Validation on the GPU: cotb200_topk_hits against torch's accuracy() and the rank rule, the live and EMA eval graphs of
EvalStep against eager eval-mode forwards, and the absence of side effects on training (cotnet_b200/evaler.py)."""
import copy

import numpy as np
import pytest
import torch

from cotnet_b200 import backbone, backbone_hybrid, evaler, trainer

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _deterministic(monkeypatch):
    """Graph and eager runs are compared bit for bit: cuDNN on deterministic, heuristically chosen algorithms (as in bench.py)."""
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)


def rank_rule_counts(z, y, ks, valid=None):
    """numpy statement of the rank rule (include/cotb200.h): [hits at each k, rows counted, bad labels]."""
    z = np.asarray(z, dtype=np.float64)
    B, K = z.shape
    n = B if valid is None else min(max(int(valid), 0), B)
    out = np.zeros(len(ks) + 2, dtype=np.int64)
    for b in range(n):
        out[len(ks)] += 1
        if not 0 <= y[b] < K:
            out[len(ks) + 1] += 1
            continue
        zy = z[b, y[b]]
        if np.isnan(zy):
            continue
        r = int(np.sum(z[b] > zy)) + int(np.sum(z[b, :y[b]] == zy))
        out[:len(ks)] += np.array([r < k for k in ks], dtype=np.int64)
    return out


def accuracy_hits(output, target, topk):
    """utils/meters.py:12-19 accuracy() per row: [len(topk), B] bool of output.topk(maxk) + eq."""
    _, pred = output.topk(max(topk), 1, True, True)
    correct = pred.t().eq(target.reshape(1, -1).expand_as(pred.t()))
    return torch.stack([correct[:k].any(0) for k in topk])


def _tie_free_logits(B, K, ld, dtype, gen):
    """[B, K] view (row pitch ld) of distinct values per row, exactly representable in bf16 (1.0 .. 512 in bf16 steps); the
    pitch padding holds +inf, which would win every comparison if it were read."""
    vals = torch.arange(0x3F80, 0x3F80 + 1152, dtype=torch.int16).view(torch.bfloat16).float()
    z = torch.empty(B, K)
    for b in range(B):
        z[b] = vals[torch.randperm(1152, generator=gen)[:K]]
    sign = torch.where(torch.rand(B, 1, generator=gen) < 0.5, -1.0, 1.0)
    full = torch.full((B, ld), float("inf"))
    full[:, :K] = z * sign
    return full.to(dtype).cuda()[:, :K]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("K", [10, 1000, 1001])
@pytest.mark.parametrize("B", [1, 128, 256])
@pytest.mark.parametrize("ks", [(1, 5), (1, 2, 3, 10)])
def test_topk_hits_equals_accuracy(dtype, K, B, ks):
    gen = torch.Generator().manual_seed(K * 1000 + B)
    z = _tie_free_logits(B, K, K + 7, dtype, gen)
    y = torch.randint(0, K, (B,), generator=gen).cuda()
    z[0, y[0]] = 1024.0                                                   # at least one hit ...
    if B > 1:
        z[1, y[1]] = -1024.0                                              # ... and one miss at every k
    hits = accuracy_hits(z, y, ks)
    want = [int(h.sum()) for h in hits]
    counts = torch.zeros(len(ks) + 2, dtype=torch.int64, device="cuda")
    evaler.topk_hits(z, y, counts, ks)
    assert counts.tolist() == want + [B, 0]
    assert rank_rule_counts(z.double().cpu().numpy(), y.cpu().numpy(), ks).tolist() == want + [B, 0]
    # a prefix of the rows (device-side count), accumulated onto the first call
    nv = max(1, B // 2 - 3)
    valid = torch.tensor([nv], dtype=torch.int32, device="cuda")
    evaler.topk_hits(z, y, counts, ks, valid)
    assert counts.tolist() == [w + int(h[:nv].sum()) for w, h in zip(want, hits)] + [B + nv, 0]
    # graph replay: the row count is read at replay time
    counts.zero_()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        evaler.topk_hits(z, y, counts, ks, valid)
    torch.cuda.current_stream().wait_stream(s)
    counts.zero_()
    with torch.cuda.graph(g):
        evaler.topk_hits(z, y, counts, ks, valid)
    valid.fill_(B)
    g.replay()
    valid.fill_(nv)
    g.replay()
    torch.cuda.synchronize()
    assert counts.tolist() == [w + int(h[:nv].sum()) for w, h in zip(want, hits)] + [B + nv, 0]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_topk_hits_rank_rule_ties_nan_bad_labels(dtype):
    gen = torch.Generator().manual_seed(5)
    B, K, ks = 256, 37, (1, 2, 5, 37)
    z = torch.randint(-2, 3, (B, K), generator=gen).float()             # five values: ties everywhere
    z[torch.rand(B, K, generator=gen) < 0.05] = float("nan")
    z[torch.rand(B, K, generator=gen) < 0.02] = float("inf")
    z[torch.rand(B, K, generator=gen) < 0.02] = -float("inf")
    y = torch.randint(0, K, (B,), generator=gen)
    y[::17] = -1
    y[5::23] = K
    y[7::29] = 1 << 40
    zc = z.to(dtype).cuda()
    counts = torch.zeros(len(ks) + 2, dtype=torch.int64, device="cuda")
    evaler.topk_hits(zc, y.cuda(), counts, ks)
    want = rank_rule_counts(zc.double().cpu().numpy(), y.numpy(), ks)
    assert counts.tolist() == want.tolist()
    assert want[-1] > 0 and 0 < want[0] < want[-2] - want[-1]
    evaler.topk_hits(zc, y.cuda(), counts, ks, torch.tensor([100], dtype=torch.int32, device="cuda"))
    assert counts.tolist() == (want + rank_rule_counts(zc.double().cpu().numpy(), y.numpy(), ks, 100)).tolist()


# ------------------------------------------------------------------------------------------------ the eval graphs
def _perturb_bn(m, seed):
    g0 = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.2, generator=g0)
                mod.running_var.uniform_(0.6, 1.6, generator=g0)
    return m


def _batch(B, res, K, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, res, res, generator=g).to(torch.bfloat16).cuda().contiguous(memory_format=torch.channels_last)
    return x, torch.randint(0, K, (B,), generator=g).cuda()


def _eager_logits(model, x):
    """Eager eval-mode forward.  The optimizer kernels write the weights without bumping their version counters, so the
    eval-mode weight caches are dropped first."""
    evaler.drop_weight_caches(model)
    modes = [(m, m.training) for m in model.modules()]
    model.eval()
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return model(x)
    finally:
        for m, t in modes:
            m.training = t


def _check_counts(counts, logits_rows, labels_rows, ks):
    """Kernel counts == the rank rule on every row; the rank rule == torch's accuracy() on every row whose label logit is untied."""
    z, y = logits_rows.double().cpu().numpy(), labels_rows.cpu().numpy()
    assert counts == rank_rule_counts(z, y, ks).tolist()
    hits = accuracy_hits(logits_rows.float(), labels_rows, ks).cpu().numpy()
    untied = [b for b in range(len(y)) if np.sum(z[b] == z[b, y[b]]) == 1]
    assert len(untied) >= len(y) // 2
    for b in untied:
        rr = rank_rule_counts(z[b:b + 1], y[b:b + 1], ks)[:len(ks)]
        assert rr.tolist() == hits[:, b].astype(np.int64).tolist(), b


@pytest.mark.parametrize("name,res", [("cotnet50", 96), ("se_cotnetd_50", 128)])
def test_live_graph_equals_eager_eval(name, res):
    ctor = backbone.MODELS.get(name) or backbone_hybrid.MODELS[name]
    torch.manual_seed(0)
    K, B, ks = 100, 8, (1, 5)
    m = _perturb_bn(ctor(num_classes=K, zero_init_last_bn=False), 1).cuda().to(memory_format=torch.channels_last)
    ev = evaler.EvalStep(m, B, res, topk=ks)
    info = ev.capture()
    assert info["graphs"] == ["live"] and info["K"] == K and info["libcotb200_launches"] > 0
    x1, y1 = _batch(B, res, K, 11)
    x2, y2 = _batch(5, res, K, 12)                                        # short last batch
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        l1 = ev.run(x1, y1).clone()
        l2 = ev.run(x2, y2).clone()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    static_x = ev.x.clone()
    r = ev.result()
    assert torch.equal(l1, _eager_logits(m, x1))
    assert torch.equal(l2, _eager_logits(m, static_x))                   # rows 5..7 of the short batch are the stale inputs
    c1 = rank_rule_counts(l1.double().cpu().numpy(), y1.cpu().numpy(), ks)
    c2 = rank_rule_counts(l2[:5].double().cpu().numpy(), y2.cpu().numpy(), ks)
    _check_counts(c1.tolist(), l1, y1, ks)
    _check_counts(c2.tolist(), l2[:5], y2, ks)
    tot = c1 + c2
    assert r["n"] == 13 and r["bad_labels"] == 0
    assert r["top1"] == 100.0 * tot[0] / 13 and r["top5"] == 100.0 * tot[1] / 13
    assert ev.result()["n"] == 0                                          # result() resets the counters


def _state(ts):
    t = [ts.P_big, ts.P_small, ts.M_big, ts.M_small, ts.E_big, ts.E_small, ts.Pb]
    return [x.clone() for x in t + list(ts.model.buffers()) + list(ts.ema_buffers)]


def test_ema_graph_rebinding_and_no_side_effects():
    """TrainStep graph steps, then both eval graphs, then more steps: the EMA graph equals an eager eval of a fresh model holding
    ts.ema_state() with the same bf16 weights, live and EMA logits differ, and training is bitwise unaffected (against the same
    steps without the evaluations)."""
    K, B, res, ks = 100, 8, 96, (1, 5)
    torch.manual_seed(0)
    mk = lambda: backbone.CoTResNet([1, 1, 1, 1], num_classes=K, zero_init_last_bn=False)   # noqa: E731
    ma = mk().cuda().to(memory_format=torch.channels_last).train()
    mb = copy.deepcopy(ma)
    kw = dict(lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=0.9, weights="bf16")
    ta, tb = trainer.TrainStep(ma, **kw), trainer.TrainStep(mb, **kw)
    batches = [_batch(B, res, K, 100 + i) for i in range(4)]
    ta.capture(*batches[0], warmup=2)
    tb.capture(*batches[0], warmup=2)
    for x, y in batches[:2]:
        ta.step(x, y)
        tb.step(x, y)
    ptrs = [p.data_ptr() for p in ma.parameters()] + [b.data_ptr() for b in ma.buffers()]
    ta.distribute_bn()                                                    # world 1: nothing to do
    ev = evaler.EvalStep(ma, B, res, train_step=ta, topk=ks)
    info = ev.capture()
    assert info["graphs"] == ["live", "ema"]
    assert [p.data_ptr() for p in ma.parameters()] + [b.data_ptr() for b in ma.buffers()] == ptrs
    assert all(m.training for m in ma.modules())                         # the training modes are restored
    xe, ye = _batch(B, res, K, 7)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        live = ev.run(xe, ye, which="live").clone()
        ema = ev.run(xe, ye, which="ema").clone()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert not torch.equal(live, ema)                                     # the EMA graph reads other weights
    assert torch.equal(live, _eager_logits(ma, xe))
    # a fresh model holding the EMA state, laid out by a TrainStep of its own (bf16 copies of the >=2-D weights)
    fresh = mk().cuda().to(memory_format=torch.channels_last)
    fresh.load_state_dict(ta.ema_state())
    trainer.TrainStep(fresh, weights="bf16")
    assert torch.equal(ema, _eager_logits(fresh, xe))
    rl, re_ = ev.result("live"), ev.result("ema")
    assert rl["n"] == re_["n"] == B
    _check_counts([round(rl["top1"] * B / 100), round(rl["top5"] * B / 100), B, 0], live, ye, ks)
    _check_counts([round(re_["top1"] * B / 100), round(re_["top5"] * B / 100), B, 0], ema, ye, ks)
    # training continues exactly as without the evaluations
    for x, y in batches[2:]:
        la = ta.step(x, y).clone()
        lb = tb.step(x, y).clone()
    assert torch.equal(la, lb)
    sa, sb = _state(ta), _state(tb)
    assert all(torch.equal(a, b) for a, b in zip(sa, sb)), [i for i, (a, b) in enumerate(zip(sa, sb)) if not torch.equal(a, b)]
    # and the eval graphs follow the new weights
    live2 = ev.run(xe, ye, which="live").clone()
    assert torch.equal(live2, _eager_logits(ma, xe)) and not torch.equal(live2, live)


def test_distribute_bn_world1_keeps_bits():
    m = _perturb_bn(backbone.CoTResNet([1, 1, 1, 1], num_classes=10), 3).cuda()
    ts = trainer.TrainStep(m, ema_decay=0.9)
    before = [b.clone() for b in list(m.buffers()) + list(ts.ema_buffers)]
    ts.distribute_bn(reduce=True)
    ts.distribute_bn(reduce=False)
    assert all(torch.equal(a, b) for a, b in zip(before, list(m.buffers()) + list(ts.ema_buffers)))
