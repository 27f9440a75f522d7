"""Gradient clipping on the H100 (train.py:270-273): the norm kernel against fp64, the clipped optimizer pass against the torch
restatement of utils/clip_grad.py (tests/clip_ref.py) followed by the SGD / EMA formulas in fp64, bit-identity with the plain
optimizer pass when the clip does not bind, NaN propagation, and TrainStep end to end (eager, captured, launch counts)."""
import copy

import numpy as np
import pytest
import torch

import clip_ref

pytestmark = pytest.mark.gpu

LR, MU, WD, DEC = 0.1, 0.9, 1e-2, 0.99


@pytest.fixture(autouse=True)
def _no_tf32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _st():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ 1. the norm
@pytest.mark.parametrize("gdt,n0", [(torch.bfloat16, 22_000_000), (torch.float32, 8_000_000), (torch.bfloat16, 8_000_000)])
def test_grad_norm_accuracy_and_repeatability(gdt, n0):
    from cotnet_b200 import _lib
    lib = _lib.load()
    gen = torch.Generator(device="cuda").manual_seed(7)
    G0 = (torch.randn(n0, device="cuda", generator=gen) * 1e-3).to(gdt)
    G1 = torch.randn(52_000, device="cuda", generator=gen) * 1e-2
    gs = torch.tensor([1.0 / 3.0, 0.25], device="cuda")
    out = torch.zeros(2, device="cuda")
    c = 1e-3

    def run():
        _lib.check(lib.cotb200_grad_norm(n0, _lib.dtype_code(G0), G0.data_ptr(), gs.data_ptr(), G1.numel(), G1.data_ptr(),
                                         gs.data_ptr() + 4, c, out.data_ptr(), _st()), "grad_norm")
        return out.clone()
    first = run()
    want = torch.sqrt(((G0.float() * gs[0]).double() ** 2).sum() + ((G1 * gs[1]).double() ** 2).sum()).item()
    assert abs(first[0].item() - want) <= 1e-5 * want, (first[0].item(), want)
    N = np.float32(first[0].item())
    assert first[1].item() == min(1.0, float((np.float32(1.0) / (N + np.float32(1e-6))) * np.float32(c)))   # torch's c / tensor
    for _ in range(3):
        assert torch.equal(run(), first)
    out.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        lib.cotb200_grad_norm(n0, _lib.dtype_code(G0), G0.data_ptr(), gs.data_ptr(), G1.numel(), G1.data_ptr(), gs.data_ptr() + 4, c,
                              out.data_ptr(), _st())
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first)


# ------------------------------------------------------------------------------------------------ flat buckets of the toy module
class _Flat:
    """clip_ref.Toy laid out by plan_flat: fp32 masters / momentum / EMA, a gradient bucket of `gdt` for the >= 2-D weights and
    an fp32 one for the rest, seeded with a spread of per-unit scales (so that AGC binds for some units only)."""

    def __init__(self, gdt, seed=0, gs=1.0 / 3.0):
        from cotnet_b200 import trainer
        self.model = clip_ref.Toy()
        self.plan = trainer.plan_flat(list(self.model.named_parameters()))
        g0 = torch.Generator().manual_seed(seed)
        self.gs = gs
        self.bufs = []                                       # per bucket: P, M, E, G (cpu, filled below), hyper
        for key, n, dt, wd in (("big", self.plan["n_big"], gdt, WD), ("small", self.plan["n_small"], torch.float32, 0.0)):
            P, M, E, G = (torch.zeros(n) for _ in range(4))
            for _, p, off in self.plan[key]:
                rows = p.shape[0] if p.dim() > 1 else 1
                shape = (rows,) + (1,) * (p.dim() - 1) if p.dim() > 1 else (1,)
                trainer._strided_view(P, p, off).copy_(torch.randn(p.shape, generator=g0) * torch.exp(torch.randn(shape, generator=g0)) * 0.1)
                trainer._strided_view(G, p, off).copy_(torch.randn(p.shape, generator=g0) * torch.exp(torch.randn(shape, generator=g0)) * 0.3)
                trainer._strided_view(M, p, off).copy_(torch.randn(p.shape, generator=g0) * 0.01)
            E = P + torch.randn(n, generator=g0) * 1e-3
            hyper = torch.tensor([LR, MU, wd, DEC, gs], device="cuda")
            self.bufs.append(dict(P=P.cuda(), M=M.cuda(), E=E.cuda(), G=G.to(dt).cuda(), hyper=hyper, n=n,
                                  Pb=torch.zeros(n, dtype=torch.bfloat16, device="cuda") if key == "big" else None))

    def clone(self):
        c = copy.copy(self)
        c.bufs = [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in b.items()} for b in self.bufs]
        return c

    def gbar(self):
        """The averaged gradients g' = G * gs in fp32 (what the kernels clip), per bucket."""
        return [b["G"].float() * b["hyper"][4] for b in self.bufs]

    def params(self, flats):
        """name-free per-parameter views (model.parameters() order) of two flat tensors [big, small]."""
        from cotnet_b200 import trainer
        where = {}
        for bi, key in enumerate(("big", "small")):
            for _, p, off in self.plan[key]:
                where[id(p)] = (bi, p, off)
        return [trainer._strided_view(flats[where[id(p)][0]], p, where[id(p)][2]) for p in self.model.parameters()]

    def scatter(self, grads, like):
        """Per-parameter tensors -> flat tensors shaped like `like` (padding keeps like's values)."""
        out = [t.clone() for t in like]
        for v, g in zip(self.params(out), grads):
            v.copy_(g)
        return out

    # the library's sequence for one step (what TrainStep.optimizer_step launches)
    def step(self, mode, c, plain=False):
        from cotnet_b200 import _lib, trainer
        lib = _lib.load()
        B = self.bufs
        if plain:
            for b in B:
                _lib.check(lib.cotb200_sgd_ema_step(b["n"], b["P"].data_ptr(), b["M"].data_ptr(), _lib.dtype_code(b["G"]), b["G"].data_ptr(),
                                                    b["E"].data_ptr(), _lib.ptr(b["Pb"]), b["hyper"].data_ptr(), 1, _st()), "sgd")
            return None
        code = trainer.CLIP_MODES[mode]
        descs = [_lib.Clip(mode=code, value=c), _lib.Clip(mode=code, value=c)]
        self.keep = []
        out = None
        if mode == "norm":
            out = torch.zeros(2, device="cuda")
            _lib.check(lib.cotb200_grad_norm(B[0]["n"], _lib.dtype_code(B[0]["G"]), B[0]["G"].data_ptr(), B[0]["hyper"].data_ptr() + 16,
                                             B[1]["n"], B[1]["G"].data_ptr(), B[1]["hyper"].data_ptr() + 16, c, out.data_ptr(), _st()),
                       "grad_norm")
            for d in descs:
                d.factor = out.data_ptr() + 4
        elif mode == "agc":
            units, _ = trainer.plan_clip_units(self.model, self.plan)
            utab = trainer._table(_lib.ClipUnit, [(off, ln, b) for b, off, ln in units], "cuda")
            fac = torch.zeros(len(units), device="cuda")
            out = torch.zeros(len(units), 2, device="cuda")
            _lib.check(lib.cotb200_unit_norms(len(units), utab.data_ptr(), sum(u[2] for u in units), B[0]["P"].data_ptr(),
                                              _lib.dtype_code(B[0]["G"]), B[0]["G"].data_ptr(), B[0]["hyper"].data_ptr() + 16,
                                              B[1]["P"].data_ptr(), B[1]["G"].data_ptr(), B[1]["hyper"].data_ptr() + 16, c,
                                              fac.data_ptr(), out.data_ptr(), _st()), "unit_norms")
            for bi in (0, 1):
                segs = trainer._clip_segments([(i, off, ln) for i, (b, off, ln) in enumerate(units) if b == bi], B[bi]["n"], 4096)
                st = trainer._table(_lib.ClipSeg, segs, "cuda")
                self.keep.append(st)
                descs[bi].factor, descs[bi].segs, descs[bi].n_segs = fac.data_ptr(), st.data_ptr(), len(segs)
            self.keep += [utab, fac]
            self.factors = fac
        for b, d in zip(B, descs):
            _lib.check(lib.cotb200_sgd_ema_step_clip(b["n"], b["P"].data_ptr(), b["M"].data_ptr(), _lib.dtype_code(b["G"]), b["G"].data_ptr(),
                                                     b["E"].data_ptr(), _lib.ptr(b["Pb"]), b["hyper"].data_ptr(), 1, d, _st()), "sgd_clip")
        torch.cuda.synchronize()
        return out


def _binding_value(f, mode):
    """A clip value (exact in fp32) that binds for about half of the units / elements / the norm, and the smallest distance of a
    unit's ratio to it (agc)."""
    gb = [t.double() for t in f.gbar()]
    if mode == "norm":
        return float(np.float32(0.5 * torch.sqrt(sum((t ** 2).sum() for t in gb)).item())), None
    if mode == "value":
        return float(np.float32(torch.cat(gb).abs().median().item())), None
    ps = f.params([b["P"].double() for b in f.bufs])
    gs = f.params(gb)
    kept = clip_ref.model_parameters(f.model, exclude_head=True)
    idx = [[id(q) for q in f.model.parameters()].index(id(p)) for p in kept]
    r = torch.cat([(clip_ref.unitwise_norm(gs[i]) / clip_ref.unitwise_norm(ps[i]).clamp(min=1e-3)).reshape(-1) for i in idx]).sort().values
    k = len(r) // 2
    c = float(np.float32((r[k - 1] + r[k]).item() / 2))
    return c, (r / c - 1).abs().min().item()


def _oracle(f, mode, c):
    """clip in fp64 on the fp32 g', then SGD-nesterov / EMA in fp64: [(P, M, E)] per bucket."""
    gb = [t.double() for t in f.gbar()]
    ps = f.params([b["P"].double() for b in f.bufs])
    clipped, _ = clip_ref.clip_model_grads(f.model, ps, f.params(gb), c, mode)
    gc = f.scatter(clipped, gb)                             # slot padding: g' = 0 stays 0 in every mode
    out = []
    for b, g in zip(f.bufs, gc):
        wd = b["hyper"][2].item()
        out.append(clip_ref.sgd_ema(b["P"].double(), b["M"].double(), b["E"].double(), g, LR, MU, wd, DEC))
    return out


# ------------------------------------------------------------------------------------------------ 2. clipped update vs the oracle
@pytest.mark.parametrize("mode", clip_ref.MODES)
@pytest.mark.parametrize("gdt", [torch.bfloat16, torch.float32])
def test_clipped_update_matches_oracle(mode, gdt):
    from cotnet_b200 import trainer
    f = _Flat(gdt, seed=1)
    c, margin = _binding_value(f, mode)
    if margin is not None:
        assert margin > 1e-4, margin
    want = _oracle(f, mode, c)
    before = f.clone()
    out = f.step(mode, c)
    if mode == "agc":
        fac = f.factors.cpu()
        assert 0.3 <= (fac < 1).float().mean().item() <= 0.7, fac
        units, _ = trainer.plan_clip_units(f.model, f.plan)
        assert 147 in {u[2] for u in units}
    if mode == "norm":
        gb = [t.double() for t in before.gbar()]
        N = torch.sqrt(sum((t ** 2).sum() for t in gb)).item()
        assert abs(out[0].item() - N) <= 1e-5 * N and out[1].item() < 1
    for b, (P, M, E) in zip(f.bufs, want):
        scale = P.abs().max().item()
        torch.testing.assert_close(b["P"].double(), P, rtol=1e-6, atol=1e-7 * scale)
        torch.testing.assert_close(b["M"].double(), M, rtol=1e-6, atol=1e-7 * M.abs().max().item())
        torch.testing.assert_close(b["E"].double(), E, rtol=1e-6, atol=1e-7 * scale)
        if b["Pb"] is not None:
            assert torch.equal(b["Pb"], b["P"].to(torch.bfloat16))
    # the clip changed the update: the plain pass gives another result
    before.step(mode, c, plain=True)
    assert not torch.equal(before.bufs[0]["P"], f.bufs[0]["P"])


# ------------------------------------------------------------------------------------------------ 3. a clip that does not bind
@pytest.mark.parametrize("mode", clip_ref.MODES)
@pytest.mark.parametrize("gdt", [torch.bfloat16, torch.float32])
def test_non_binding_clip_is_bit_identical(mode, gdt):
    a = _Flat(gdt, seed=2)
    b = a.clone()
    a.step(mode, 1e30)
    b.step(mode, 1e30, plain=True)
    torch.cuda.synchronize()
    for x, y in zip(a.bufs, b.bufs):
        for k in ("P", "M", "E", "Pb"):
            if x[k] is not None:
                assert torch.equal(x[k], y[k]), (mode, k)


# ------------------------------------------------------------------------------------------------ 4. NaN propagation
@pytest.mark.parametrize("mode", clip_ref.MODES)
def test_nan_propagation(mode):
    f = _Flat(torch.bfloat16, seed=3)
    name, p, off = f.plan["big"][1]                        # conv2.weight [16, 8, 1, 1]
    assert name == "conv2.weight"
    row = p.numel() // p.shape[0]
    bad = off + 3 * row + 5                                # unit 3 of conv2.weight
    f.bufs[0]["G"][bad] = float("nan")
    c, _ = _binding_value(_Flat(torch.bfloat16, seed=3), mode)
    f.step(mode, c)
    nan = [torch.isnan(b["P"]) for b in f.bufs]
    if mode == "norm":
        assert all(t.all() for t in nan)
    elif mode == "value":
        assert nan[0].nonzero().flatten().tolist() == [bad] and not nan[1].any()
    else:
        assert nan[0].nonzero().flatten().tolist() == list(range(off + 3 * row, off + 4 * row)) and not nan[1].any()


# ------------------------------------------------------------------------------------------------ 5. TrainStep against the oracle
def _small_model():
    from cotnet_b200 import backbone
    torch.manual_seed(0)
    m = backbone.CoTResNet([1, 1, 1, 1], zero_init_last_bn=False)
    g0 = torch.Generator().manual_seed(11)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.2, generator=g0)
                mod.running_var.uniform_(0.6, 1.6, generator=g0)
    return m.cuda().to(memory_format=torch.channels_last).eval()


def _batch(seed, dtype=torch.float32):
    g0 = torch.Generator().manual_seed(seed)
    x = torch.randn(8, 3, 64, 64, generator=g0).cuda().to(dtype).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (8,), generator=g0).cuda()
    return x, y


def _trainstep_binding_value(mode, x, y):
    """Gradients of the same model and batch from a step without clipping -> a clip value that binds (about half for agc)."""
    from cotnet_b200 import trainer
    m = _small_model()
    ts = trainer.TrainStep(m, lr=LR, momentum=MU, weight_decay=WD, nesterov=True, ema_decay=DEC, amp_dtype=None, weights="fp32")
    ts.forward_backward(x, y)
    grads, ms = ts.grads(), ts.master_state()
    names = [n for n, _ in m.named_parameters()]
    gb = [grads[n].double() for n in names]
    if mode == "norm":
        return float(np.float32(0.5 * torch.sqrt(sum((g ** 2).sum() for g in gb)).item()))
    if mode == "value":
        return float(np.float32(torch.cat([g.reshape(-1) for g in gb]).abs().median().item()))
    r = torch.cat([(clip_ref.unitwise_norm(g) / clip_ref.unitwise_norm(ms[n].double()).clamp(min=1e-3)).reshape(-1)
                   for n, g in zip(names[:-2], gb[:-2])]).sort().values
    k = len(r) // 2
    return float(np.float32((r[k - 1] + r[k]).item() / 2))


@pytest.mark.parametrize("mode", clip_ref.MODES)
def test_trainstep_step_matches_oracle(mode):
    from cotnet_b200 import trainer
    x, y = _batch(21)
    c = _trainstep_binding_value(mode, x, y)
    m = _small_model()
    ts = trainer.TrainStep(m, lr=LR, momentum=MU, weight_decay=WD, nesterov=True, ema_decay=DEC, amp_dtype=None, weights="fp32",
                           clip_grad=c, clip_mode=mode)
    assert (ts.grad_norm is not None) == (mode == "norm")
    ts.step_eager(x, y)                                    # a first step: momentum and EMA away from their initial values
    ts.forward_backward(x, y)
    names = [n for n, _ in m.named_parameters()]
    grads = {n: t.double().clone() for n, t in ts.grads().items()}
    master = {n: t.double().clone() for n, t in ts.master_state().items()}
    ema = {n: t.double().clone() for n, t in ts.ema_state().items()}
    flat_m = [ts.M_big.clone(), ts.M_small.clone()]
    mom = {}
    for bi, key in enumerate(("big", "small")):
        for n, p, off in ts.plan[key]:
            mom[n] = trainer._strided_view(flat_m[bi], p, off).double()
    ts.optimizer_step()
    torch.cuda.synchronize()
    ps = [master[n] for n in names]
    clipped, norm = clip_ref.clip_model_grads(m, ps, [grads[n] for n in names], c, mode)
    changed = sum(int(not torch.equal(g, grads[n])) for g, n in zip(clipped, names))
    assert changed > 0
    if mode == "norm":
        assert abs(ts.grad_norm.item() - norm.item()) <= 1e-5 * norm.item()
    small = {n for n, _, _ in ts.plan["small"]}
    after = ts.master_state()
    for n, g in zip(names, clipped):
        wd = 0.0 if n in small else WD
        P, _, E = clip_ref.sgd_ema(master[n], mom[n], ema[n], g, LR, MU, wd, DEC)
        torch.testing.assert_close(after[n].double(), P, rtol=1e-6, atol=1e-6 * P.abs().max().item(), msg=lambda s: n + ": " + s)
        torch.testing.assert_close(ts.ema_state()[n].double(), E, rtol=1e-6, atol=1e-6 * E.abs().max().item())


# ------------------------------------------------------------------------------------------------ 6./7. graph replay and launch counts
@pytest.mark.parametrize("mode", ["norm", "agc"])
def test_captured_step_equals_eager_with_clipping(mode, monkeypatch):
    from cotnet_b200 import trainer
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    x, y = _batch(6, torch.bfloat16)
    kw = dict(lr=0.002, momentum=0.9, weight_decay=1e-3, nesterov=True, ema_decay=0.99, amp_dtype=torch.bfloat16, weights="bf16",
              clip_grad=1e-3, clip_mode=mode)
    t1, t2 = trainer.TrainStep(_small_model(), **kw), trainer.TrainStep(_small_model(), **kw)
    info = t1.capture(x, y, warmup=2)
    assert info["cuda_graph"]
    for _ in range(2):
        t2.step_eager(x, y)
    la, na = [], []
    lb, nb = [], []
    for _ in range(2):
        la.append(t1.step(x, y).item())
        lb.append(t2.step_eager(x, y).item())
        if mode == "norm":
            na.append(t1.grad_norm.item())
            nb.append(t2.grad_norm.item())
    assert la == lb and na == nb, (la, lb, na, nb)
    if mode == "norm":
        assert na[0] > 1e-3                                 # the clip binds
    s1, s2 = t1.master_state(), t2.master_state()
    assert not [n for n in s1 if not torch.equal(s1[n], s2[n])]


def test_launch_count_grows_by_the_clip_launches_only():
    from cotnet_b200 import trainer
    x, y = _batch(8, torch.bfloat16)
    counts = {}
    for mode in (None, "norm", "value", "agc"):
        kw = dict(lr=0.002, weights="bf16", amp_dtype=torch.bfloat16)
        if mode:
            kw.update(clip_grad=1e-3, clip_mode=mode)
        ts = trainer.TrainStep(_small_model(), **kw)
        counts[mode] = ts.capture(x, y, warmup=1)["libcotb200_kernels_per_replay"]
    assert counts["norm"] == counts[None] + 1 and counts["value"] == counts[None] and counts["agc"] == counts[None] + 1, counts
