"""The update rules of create_optimizer on the H100: cotb200_opt_step against the fp64 restatement (tests/optim_ref.py) for every
rule, gradient dtype and clip mode; the reference's own 14-step sequences (tests/golden/optim.npz) replayed through the kernels;
TrainStep(opt=...) end to end; captured replays bit-identical to eager steps across set_lr and Lookahead synchronisations;
sync_lookahead(); and the launch count of the step."""
import ctypes
import os

import numpy as np
import pytest
import torch

import clip_ref
import optim_ref
from test_clip_gpu import DEC, LR, MU, WD, _binding_value, _Flat, _small_model, _batch, _st

pytestmark = pytest.mark.gpu

EPS = 1e-8
#: case -> (solver.opt, momentum, t before the tested step, Lookahead slow weights already created)
CASES = {
    "sgd": ("sgd", MU, 3, False), "momentum": ("momentum", MU, 3, False), "adam": ("adam", MU, 3, False),
    "adamw": ("adamw", MU, 3, False), "nadam": ("nadam", MU, 3, False), "radam": ("radam", MU, 9, False),
    "radam_early": ("radam", MU, 2, False), "adadelta": ("adadelta", MU, 3, False), "rmsprop": ("rmsprop", MU, 3, False),
    "rmsprop_m0": ("rmsprop", 0.0, 3, False), "rmsproptf": ("rmsproptf", MU, 3, False), "rmsproptf_m0": ("rmsproptf", 0.0, 3, False),
    "lookahead_adamw_first": ("lookahead_adamw", MU, 5, False), "lookahead_rmsproptf": ("lookahead_rmsproptf", MU, 11, True),
    "lookahead_sgd": ("lookahead_sgd", MU, 5, True), "lookahead_nadam_nosync": ("lookahead_nadam", MU, 6, True),
}


def _opt_for(name, momentum, bufs, state_dev):
    from cotnet_b200 import _lib, trainer
    base, rule, la = trainer.parse_opt(name)
    uses_m = not (base in ("rmsprop", "rmsproptf") and momentum == 0)
    return _lib.Opt(rule=rule, eps=EPS, lookahead_k=6 if la else 0, lookahead_alpha=0.5, M=bufs["M"].data_ptr() if uses_m else None,
                    V=bufs["V"].data_ptr(), S=bufs["S"].data_ptr(), state=state_dev.data_ptr()), uses_m


def _state_dev(t, m_schedule, slow_init):
    from cotnet_b200 import _lib
    st = _lib.OptState(t=float(t), m_schedule=m_schedule, slow_init=1 if slow_init else 0)
    return torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).cuda()


def _clip_descs(f, mode, c):
    """The clip factors of `mode` for the flat buckets of f (a _Flat), as TrainStep launches them; (descs, keep-alive)."""
    from cotnet_b200 import _lib, trainer
    lib, B = _lib.load(), f.bufs
    if mode == "none":
        return [None, None], []
    code = trainer.CLIP_MODES[mode]
    descs = [_lib.Clip(mode=code, value=c), _lib.Clip(mode=code, value=c)]
    keep = []
    if mode == "norm":
        out = torch.zeros(2, device="cuda")
        _lib.check(lib.cotb200_grad_norm(B[0]["n"], _lib.dtype_code(B[0]["G"]), B[0]["G"].data_ptr(), B[0]["hyper"].data_ptr() + 16,
                                         B[1]["n"], B[1]["G"].data_ptr(), B[1]["hyper"].data_ptr() + 16, c, out.data_ptr(), _st()), "grad_norm")
        for d in descs:
            d.factor = out.data_ptr() + 4
        keep.append(out)
    elif mode == "agc":
        units, _ = trainer.plan_clip_units(f.model, f.plan)
        utab = trainer._table(_lib.ClipUnit, [(off, ln, b) for b, off, ln in units], "cuda")
        fac = torch.zeros(len(units), device="cuda")
        _lib.check(lib.cotb200_unit_norms(len(units), utab.data_ptr(), sum(u[2] for u in units), B[0]["P"].data_ptr(),
                                          _lib.dtype_code(B[0]["G"]), B[0]["G"].data_ptr(), B[0]["hyper"].data_ptr() + 16,
                                          B[1]["P"].data_ptr(), B[1]["G"].data_ptr(), B[1]["hyper"].data_ptr() + 16, c,
                                          fac.data_ptr(), None, _st()), "unit_norms")
        for bi in (0, 1):
            segs = trainer._clip_segments([(i, off, ln) for i, (b, off, ln) in enumerate(units) if b == bi], B[bi]["n"], 4096)
            stab = trainer._table(_lib.ClipSeg, segs, "cuda")
            descs[bi].factor, descs[bi].segs, descs[bi].n_segs = fac.data_ptr(), stab.data_ptr(), len(segs)
            keep.append(stab)
        keep += [utab, fac]
    return descs, keep


def _f32(x):
    """A hyper-parameter as the kernels hold it.  The restatement takes these values: where a gradient cancels its weight-decay
    term and the square average is tiny (RMSprop's first steps), the update is sensitive enough to tell 0.01 from fp32(0.01)."""
    return float(np.float32(x))


def _rel_err(got, want):
    return ((got.double() - want).abs().max() / want.abs().max().clamp(min=1e-30)).item()


# ------------------------------------------------------------------------------------------------ 1. one pass vs the restatement
@pytest.mark.parametrize("mode", ["none", "norm", "value", "agc"])
@pytest.mark.parametrize("gdt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("case", sorted(CASES))
def test_pass_matches_restatement(case, gdt, mode):
    from cotnet_b200 import _lib
    lib = _lib.load()
    name, mom, t0, slow_init = CASES[case]
    base, la = optim_ref.split(name)
    f = _Flat(gdt, seed=5)
    g0 = torch.Generator().manual_seed(9)
    for b in f.bufs:                                          # moments of a run in progress; square averages positive
        b["V"] = (torch.rand(b["n"], generator=g0) * 0.2 + (0.5 if base == "rmsproptf" else 1e-3)).cuda() * 0.05
        b["S"] = (b["P"].cpu() + torch.randn(b["n"], generator=g0) * 0.01).cuda()
        if base == "adadelta":
            b["M"] = b["M"].abs() * 1e-2
    c = _binding_value(f, mode)[0] if mode != "none" else None
    ms0 = 0.7
    state = _state_dev(t0, ms0, slow_init)
    # the oracle, from the same fp32 state in fp64
    gb = [t.double() for t in f.gbar()]
    if mode != "none":
        ps = f.params([b["P"].double() for b in f.bufs])
        clipped, _ = clip_ref.clip_model_grads(f.model, ps, f.params(gb), c, mode)
        gb = f.scatter(clipped, gb)
    want = [b["P"].double().clone() for b in f.bufs]
    o = optim_ref.Optim(name, [(_f32(WD), [want[0]]), (0.0, [want[1]])], _f32(LR), _f32(mom), _f32(EPS))
    o.t, o.la_step = t0, t0
    for s, b in zip(o.state, f.bufs):
        for k in list(s):
            if k in ("momentum_buffer", "exp_avg", "acc_delta"):
                s[k] = b["M"].double().clone()
            elif k in ("exp_avg_sq", "square_avg"):
                s[k] = b["V"].double().clone()
            elif k == "m_schedule":
                s[k] = ms0
        if slow_init:
            s["slow_buffer"] = b["S"].double().clone()
    o.step(gb)
    E0 = [b["E"].double().clone() for b in f.bufs]
    # the kernels
    descs, keep = _clip_descs(f, mode, c)
    opts = [_opt_for(name, mom, b, state) for b in f.bufs]
    _lib.check(lib.cotb200_opt_prepare(ctypes.byref(opts[0][0]), f.bufs[0]["hyper"].data_ptr(), 1, _st()), "prepare")
    for b, (od, _), d in zip(f.bufs, opts, descs):
        _lib.check(lib.cotb200_opt_step(b["n"], b["P"].data_ptr(), _lib.dtype_code(b["G"]), b["G"].data_ptr(), b["E"].data_ptr(),
                                        _lib.ptr(b["Pb"]), b["hyper"].data_ptr(), ctypes.byref(od), None if d is None else ctypes.byref(d),
                                        _st()), "opt_step")
    torch.cuda.synchronize()
    assert state[:8].view(torch.float64).item() == t0 + 1
    worst = {}
    for bi, (b, s) in enumerate(zip(f.bufs, o.state)):
        checks = [("P", b["P"], want[bi]), ("E", b["E"], optim_ref.ema(E0[bi], want[bi], DEC))]
        for k, v in s.items():
            if not torch.is_tensor(v):
                continue
            buf = {"momentum_buffer": "M", "exp_avg": "M", "acc_delta": "M", "exp_avg_sq": "V", "square_avg": "V", "slow_buffer": "S"}[k]
            checks.append((k, b[buf], v))
        for k, got, ref in checks:
            err = _rel_err(got, ref)
            worst[(bi, k)] = err
            assert err <= 1e-6, (case, bi, k, err)
        if b["Pb"] is not None:
            assert torch.equal(b["Pb"], b["P"].to(torch.bfloat16))
    print(case, gdt, mode, "largest error / max|ref|: %.2e" % max(worst.values()))


def test_pass_ema_follows_the_synchronised_weights():
    """E = decay*E + (1 - decay)*P of the weights after the Lookahead synchronisation (train.py:274-277)."""
    from cotnet_b200 import _lib
    lib = _lib.load()
    f = _Flat(torch.float32, seed=6)
    for b in f.bufs:
        b["V"] = torch.full_like(b["P"], 1e-3)
        b["S"] = b["P"] + 0.05
    E0 = [b["E"].clone() for b in f.bufs]
    state = _state_dev(5, 1.0, True)                          # the next step is the 6th: a synchronisation
    opts = [_opt_for("lookahead_adam", MU, b, state)[0] for b in f.bufs]
    _lib.check(lib.cotb200_opt_prepare(ctypes.byref(opts[0]), f.bufs[0]["hyper"].data_ptr(), 1, _st()), "prepare")
    for b, od in zip(f.bufs, opts):
        _lib.check(lib.cotb200_opt_step(b["n"], b["P"].data_ptr(), _lib.F32, b["G"].data_ptr(), b["E"].data_ptr(), _lib.ptr(b["Pb"]),
                                        b["hyper"].data_ptr(), ctypes.byref(od), None, _st()), "opt_step")
    torch.cuda.synchronize()
    for b, e0 in zip(f.bufs, E0):
        assert torch.equal(b["P"], b["S"])
        want = e0.double() * DEC + (1 - DEC) * b["P"].double()
        assert _rel_err(b["E"], want) <= 1e-6


# ------------------------------------------------------------------------------------------------ 2. the reference's sequences
@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "optim.npz"))


def test_golden_sequences_through_the_kernels(golden):
    from cotnet_b200 import _lib
    lib = _lib.load()
    lr, lr2, lr2_step, wd = float(golden["lr"]), float(golden["lr2"]), int(golden["lr2_step"]), float(golden["weight_decay"])
    worst = 0.0
    for case, name, mom in zip(golden["cases"], golden["opts"], golden["momenta"]):
        case, name, mom = str(case), str(name), float(mom)
        base, _ = optim_ref.split(name)
        bufs = []
        for src, n, w in (("w0", 64, wd), ("b0", 8, 0.0)):
            P = torch.zeros(n, device="cuda")
            v0 = torch.from_numpy(golden[src]).reshape(-1)
            P[:v0.numel()] = v0.float().cuda()
            V = torch.full((n,), 1.0 if base == "rmsproptf" else 0.0, device="cuda")
            bufs.append(dict(P=P, M=torch.zeros(n, device="cuda"), V=V, S=torch.zeros(n, device="cuda"),
                             G=torch.zeros(n, device="cuda"), hyper=torch.tensor([lr, mom, w, 0.0, 1.0], device="cuda"), n=n, k=v0.numel()))
        state = _state_dev(0, 1.0, False)
        opts = [_opt_for(name, mom, b, state)[0] for b in bufs]
        for s in range(1, 15):
            for b, key in zip(bufs, ("gw_%d", "gb_%d")):
                b["G"][:b["k"]] = torch.from_numpy(golden[key % s]).reshape(-1).float().cuda()
                if s == lr2_step:
                    b["hyper"][0] = lr2
            _lib.check(lib.cotb200_opt_prepare(ctypes.byref(opts[0]), bufs[0]["hyper"].data_ptr(), 1, _st()), "prepare")
            for b, od in zip(bufs, opts):
                _lib.check(lib.cotb200_opt_step(b["n"], b["P"].data_ptr(), _lib.F32, b["G"].data_ptr(), None, None, b["hyper"].data_ptr(),
                                                ctypes.byref(od), None, _st()), "opt_step")
            for b, tag in zip(bufs, "wb"):
                want = torch.from_numpy(golden["%s/%s_%d" % (case, tag, s)]).reshape(-1)
                err = _rel_err(b["P"][:b["k"]].cpu(), want)
                worst = max(worst, err)
                assert err <= 1e-6, (case, s, tag, err)
                assert not b["P"][b["k"]:].any()                # slot padding stays 0
        keys = {"M": ("momentum_buffer", "exp_avg", "acc_delta"), "V": ("exp_avg_sq", "square_avg"), "S": ("slow_buffer",)}
        for b, tag in zip(bufs, "wb"):
            for buf, names in keys.items():
                for k in names:
                    gk = "%s/state_%s_%s" % (case, k, tag)
                    if gk in golden.files:
                        err = _rel_err(b[buf][:b["k"]].cpu(), torch.from_numpy(golden[gk]).reshape(-1).double())
                        worst = max(worst, err)
                        assert err <= 1e-6, (case, k, tag, err)
    print("golden sequences: largest error / max|ref| %.2e" % worst)


# ------------------------------------------------------------------------------------------------ 3. TrainStep end to end
@pytest.mark.parametrize("opt", ["adam", "adamw", "nadam", "radam", "adadelta", "rmsprop", "rmsproptf", "lookahead_sgd"])
def test_trainstep_step_matches_restatement(opt):
    from cotnet_b200 import trainer
    x, y = _batch(21)
    m = _small_model()
    ts = trainer.TrainStep(m, lr=LR * 0.1, momentum=MU, weight_decay=WD, ema_decay=DEC, amp_dtype=None, weights="fp32", opt=opt)
    ts.step_eager(x, y)
    ts.forward_backward(x, y)
    names = [n for n, _ in m.named_parameters()]
    grads = {n: t.double().clone() for n, t in ts.grads().items()}
    master = {n: t.double().clone() for n, t in ts.master_state().items()}
    ema = {n: t.double().clone() for n, t in ts.ema_state().items()}
    ostate = {n: {k: (v.double().clone() if v.dim() else v.item()) for k, v in d.items()} for n, d in ts.optimizer_state().items()}
    ts.optimizer_step()
    torch.cuda.synchronize()
    small = {n for n, _, _ in ts.plan["small"]}
    hyp = ts.hyper.tolist()                                   # lr, momentum, weight_decay as the step holds them (fp32)
    after, after_ema, after_state = ts.master_state(), ts.ema_state(), ts.optimizer_state()
    worst = 0.0
    for n in names:
        p = master[n].clone()
        o = optim_ref.Optim(opt, [(0.0 if n in small else hyp[2], [p])], hyp[0], hyp[1], _f32(EPS))
        o.t = o.la_step = int(ostate[n].get("step", 1))
        for k, v in ostate[n].items():
            if k in o.state[0] or k == "slow_buffer":
                o.state[0][k] = v.clone() if torch.is_tensor(v) else v
        o.step([grads[n]])
        for k, got, ref in [("P", after[n], p), ("E", after_ema[n], optim_ref.ema(ema[n], p, DEC))] + \
                [(k, after_state[n][k], v) for k, v in o.state[0].items() if torch.is_tensor(v) and k != "slow_buffer"]:
            d = (got.double() - ref).abs()
            err = (d.max() / ref.abs().max()).item()
            worst = max(worst, err)
            i = int(d.argmax())
            assert err <= 1e-6, "%s %s %s: error %.3g at %d: before %r grad %r state %r got %r want %r" % (
                opt, n, k, err, i, master[n].reshape(-1)[i].item(), grads[n].reshape(-1)[i].item(),
                {kk: (vv.reshape(-1)[i].item() if torch.is_tensor(vv) else vv) for kk, vv in ostate[n].items()},
                got.reshape(-1)[i].item(), ref.reshape(-1)[i].item())
        if "step" in after_state[n]:
            assert after_state[n]["step"].item() == 2
    print(opt, "largest error / max|ref| %.2e" % worst)


# ------------------------------------------------------------------------------------------------ 4. graph replay == eager
def test_captured_steps_equal_eager_steps(monkeypatch):
    from cotnet_b200 import trainer
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    x, y = _batch(6, torch.bfloat16)
    kw = dict(lr=0.002, momentum=0.9, weight_decay=1e-3, ema_decay=0.99, amp_dtype=torch.bfloat16, weights="bf16",
              opt="lookahead_adamw", clip_grad=1e-3, clip_mode="agc")
    t1, t2, t3 = (trainer.TrainStep(_small_model(), **kw) for _ in range(3))
    assert t1.capture(x, y, warmup=2)["cuda_graph"] and t3.capture(x, y, warmup=2)["cuda_graph"]
    for _ in range(2):
        t2.step_eager(x, y)
    losses = [[], [], []]
    for i in range(11):                                       # steps 3..13: synchronisations at 6 and 12, a new LR from step 8
        if i == 5:
            for t in (t1, t2, t3):
                t.set_lr(0.001)
        losses[0].append(t1.step(x, y).item())
        losses[1].append(t2.step_eager(x, y).item())
        losses[2].append(t3.step(x, y).item())
    assert losses[0] == losses[1] == losses[2], losses
    for other in (t2, t3):
        for get in ("master_state", "ema_state"):
            a, b = getattr(t1, get)(), getattr(other, get)()
            assert not [n for n in a if not torch.equal(a[n], b[n])], get
        oa, ob = t1.optimizer_state(), other.optimizer_state()
        assert not [(n, k) for n in oa for k in oa[n] if not torch.equal(oa[n][k], ob[n][k])]
        assert torch.equal(t1.Pb, other.Pb)
    st = t1.optimizer_state()
    assert all(d["step"].item() == 13 for d in st.values())
    assert torch.equal(t1.Pb, t1.P_big.to(torch.bfloat16))


# ------------------------------------------------------------------------------------------------ 5. sync_lookahead
def test_sync_lookahead():
    from cotnet_b200 import trainer
    x, y = _batch(4, torch.bfloat16)
    ts = trainer.TrainStep(_small_model(), lr=1e-3, ema_decay=0.99, amp_dtype=torch.bfloat16, weights="bf16", opt="lookahead_rmsproptf")
    for _ in range(2):
        ts.step_eager(x, y)
    P0, E0 = ts.P_big.clone(), ts.E_big.clone()
    ts.sync_lookahead()                                       # the first synchronisation: slow weights = fast weights
    torch.cuda.synchronize()
    assert torch.equal(ts.P_big, P0) and torch.equal(ts.S_big, P0) and torch.equal(ts.S_small, ts.P_small)
    ts.step_eager(x, y)
    P1, S1, Ps1, Ss1 = ts.P_big.clone(), ts.S_big.clone(), ts.P_small.clone(), ts.S_small.clone()
    assert not torch.equal(P1, S1)
    ts.Pb.zero_()
    E1 = ts.E_big.clone()
    ts.sync_lookahead()
    torch.cuda.synchronize()
    for P, S, p1, s1 in ((ts.P_big, ts.S_big, P1, S1), (ts.P_small, ts.S_small, Ps1, Ss1)):
        want = s1 + 0.5 * (p1 - s1)
        assert _rel_err(P, want.double()) <= 1e-6 and torch.equal(P, S)
    assert torch.equal(ts.Pb, ts.P_big.to(torch.bfloat16))   # the bf16 copy is refreshed
    assert torch.equal(ts.E_big, E1)                          # the EMA does not move
    assert all(d["step"].item() == 3 for d in ts.optimizer_state().values())
    assert not torch.equal(E0, E1)
    plain = trainer.TrainStep(_small_model(), opt="adamw")
    plain.sync_lookahead()                                    # no Lookahead: nothing to do


# ------------------------------------------------------------------------------------------------ 6. launches per replay
def test_launch_count_is_sgd_plus_prepare():
    from cotnet_b200 import trainer
    x, y = _batch(8, torch.bfloat16)
    counts = {}
    for opt, clip in (("sgd", None), ("adamw", None), ("lookahead_rmsproptf", None), ("nadam", None), ("sgd", "agc"),
                      ("radam", "agc"), ("lookahead_sgd", "norm"), ("sgd", "norm")):
        kw = dict(lr=0.002, weights="bf16", amp_dtype=torch.bfloat16, ema_decay=0.99, opt=opt)
        if clip:
            kw.update(clip_grad=1e-3, clip_mode=clip)
        ts = trainer.TrainStep(_small_model(), **kw)
        counts[(opt, clip)] = ts.capture(x, y, warmup=1)["libcotb200_kernels_per_replay"]
        del ts
    base = counts[("sgd", None)]
    assert counts[("adamw", None)] == counts[("lookahead_rmsproptf", None)] == counts[("nadam", None)] == base + 1, counts
    assert counts[("radam", "agc")] == counts[("sgd", "agc")] + 1, counts
    assert counts[("lookahead_sgd", "norm")] == counts[("sgd", "norm")] + 1, counts
