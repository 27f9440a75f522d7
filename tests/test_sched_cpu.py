"""CPU checks of the learning-rate schedules (cotnet_b200/sched.py): every case of the reference's own create_scheduler
(tests/golden/sched.npz, tools/make_sched_golden.py) reproduced exactly, the factory's mapping of the solver keys, and the set_lr
calls a TrainStep receives, through a recording stand-in."""
import functools
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from cotnet_b200 import sched

CONFIGS = ["CoTNeXt-101-350epoch", "CoTNeXt-50-350epoch", "CoTNet-101-350epoch", "CoTNet-50-350epoch", "SE-CoTNetD-101_350epoch",
           "SE-CoTNetD-152_350epoch", "SE-CoTNetD-50_350epoch"]
CASES = CONFIGS + ["tanh", "step", "plateau_max", "plateau_min", "plateau_none", "cosine_restarts", "cosine_cooldown",
                   "cosine_noise_pair", "cosine_noise_one", "cosine_no_warmup", "cosine_start_epoch", "unknown_sched",
                   "cosine_warmup_prefix", "tanh_warmup_prefix"]
#: cases recorded with the factory's cosine and tanh classes given warmup_prefix=True
WARMUP_PREFIX = ("cosine_warmup_prefix", "tanh_warmup_prefix")


class Recorder:
    """A TrainStep as the schedules see it: the device hyper-parameters (here on the host) and set_lr, which is recorded."""

    def __init__(self, lr):
        self.hyper = torch.tensor([lr, 0.9, 1e-4, 0.0, 1.0], dtype=torch.float32)
        self.calls = []

    def set_lr(self, lr):
        self.calls.append(lr)
        self.hyper[0:1].fill_(lr)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sched.npz"))


def _case(g, case, monkeypatch=None):
    if case in WARMUP_PREFIX:
        for name in ("CosineLRScheduler", "TanhLRScheduler"):
            monkeypatch.setattr(sched, name, functools.partial(getattr(sched, name), warmup_prefix=True))
    solver = json.loads(str(g[case + "/solver"]))
    return solver, float(g[case + "/seed"]), str(g[case + "/eval_metric"])


def _solver(**keys):
    """The CoTNet-50 config's solver section after pop_unused_value, with `keys` on top."""
    s = dict(sched="cosine", lr=0.25, lr_noise_pct=0.67, lr_noise_std=1.0, lr_cycle_mul=1.0, lr_cycle_limit=1, warmup_lr=0.0001,
             min_lr=1e-5, epochs=350, decay_epochs=30, warmup_epochs=5, cooldown_epochs=0, patience_epochs=10, decay_rate=0.1)
    s.update(keys)
    return s


def test_golden_covers_every_case(golden):
    assert sorted(str(c) for c in golden["cases"]) == sorted(CASES)
    for c in CONFIGS:
        solver, seed, metric = _case(golden, c)
        assert solver["sched"] == "cosine" and solver["warmup_epochs"] == 5 and seed == 1.0 and metric == "top1"
        assert "lr_noise" not in solver and "start_epoch" not in solver
    lr = golden["CoTNet-50-350epoch/lr"]
    assert golden["CoTNet-50-350epoch/lr_init"] == 1e-4 and abs(lr[0] - 0.05008) < 1e-12 and abs(lr[4] - 0.249874) < 1e-6


@pytest.mark.parametrize("case", CASES)
def test_schedule_matches_reference(golden, case, monkeypatch):
    solver, seed, metric = _case(golden, case, monkeypatch)
    ts = Recorder(solver["lr"])
    s, num_epochs = sched.create_scheduler(solver, ts, seed=seed, eval_metric=metric)
    assert num_epochs == int(golden[case + "/num_epochs"])
    assert (s is None) == bool(golden[case + "/sched_none"])
    want_lr = golden[case + "/lr"]
    assert len(want_lr) == num_epochs + 5
    lr = solver["lr"] if s is None else s.lr
    assert lr == float(golden[case + "/lr_init"])
    expected_calls = [lr] if lr != solver["lr"] else []
    for e, (m, want) in enumerate(zip(golden[case + "/metrics"], want_lr), 1):
        if s is not None:
            s.step(e, None if np.isnan(m) else float(m))
            got = s.lr
            assert float(ts.hyper[0]) == float(np.float32(got))
        else:
            got = solver["lr"]
        assert got == float(want), "%s epoch %d: %r, reference %r" % (case, e, got, float(want))
        if got != lr:
            expected_calls.append(got)
        lr = got
    assert ts.calls == expected_calls                     # one set_lr per change of the LR, in order, and none otherwise


@pytest.mark.parametrize("case", CASES)
def test_setup_applies_start_epoch(golden, case, monkeypatch):
    solver, seed, metric = _case(golden, case, monkeypatch)
    ts = Recorder(solver["lr"])
    s, start, num_epochs = sched.setup_scheduler(solver, ts, seed=seed, eval_metric=metric)
    assert start == int(golden[case + "/start_epoch"]) and num_epochs == int(golden[case + "/num_epochs"])
    assert (solver["lr"] if s is None else s.lr) == float(golden[case + "/lr_start"])
    if case == "cosine_start_epoch":
        assert start == 3 and s.lr == float(golden[case + "/lr"][2]) and len(ts.calls) == 2   # warmup_lr, then epoch 3's LR


def test_attribute_solver_equals_mapping(golden):
    solver, seed, _ = _case(golden, "cosine_noise_pair")
    a, b = Recorder(solver["lr"]), Recorder(solver["lr"])
    sa, na = sched.create_scheduler(solver, a, seed=seed)
    sb, nb = sched.create_scheduler(SimpleNamespace(**solver), b, seed=seed)
    assert na == nb
    for e in range(1, na + 1):
        sa.step(e)
        sb.step(e)
        assert sa.lr == sb.lr
    assert a.calls == b.calls


def test_unknown_sched_gives_no_scheduler():
    ts = Recorder(0.25)
    for name in ("multistep", "none", "", "Cosine"):
        assert sched.create_scheduler(_solver(sched=name, epochs=123), ts) == (None, 123)
        assert sched.setup_scheduler(_solver(sched=name, epochs=123, start_epoch=4), ts) == (None, 4, 123)
    assert ts.calls == []


@pytest.mark.parametrize("name,keys,want", [
    ("cosine", dict(epochs=10, lr_cycle_limit=1, cooldown_epochs=4), 14),
    ("cosine", dict(epochs=10, lr_cycle_limit=3, cooldown_epochs=4), 34),
    ("cosine", dict(epochs=10, lr_cycle_mul=2.0, lr_cycle_limit=3, cooldown_epochs=4), 74),     # 10 + 20 + 40
    ("cosine", dict(epochs=10, lr_cycle_mul=1.5, lr_cycle_limit=3, cooldown_epochs=0), 47),     # floor(10 + 15 + 22.5)
    ("cosine", dict(epochs=10, lr_cycle_limit=0, cooldown_epochs=2), 12),                      # no limit: one cycle counted
    ("tanh", dict(epochs=30, lr_cycle_limit=2, cooldown_epochs=5), 65),
    ("step", dict(epochs=30, cooldown_epochs=5), 30),
    ("plateau", dict(epochs=30, cooldown_epochs=5), 30),
])
def test_num_epochs(name, keys, want):
    s, n = sched.create_scheduler(_solver(sched=name, **keys), Recorder(0.25))
    assert n == want
    if name in ("cosine", "tanh"):
        assert n == s.get_cycle_length() + keys["cooldown_epochs"]


@pytest.mark.parametrize("lr_noise,want", [([0.3, 0.9], [6.0, 18.0]), ((0.3, 0.9), [6.0, 18.0]), ([0.5], 10.0), (0.5, 10.0),
                                           ([], None), (None, None)])
def test_lr_noise_forms(lr_noise, want):
    keys = dict(epochs=20) if lr_noise is None else dict(epochs=20, lr_noise=lr_noise)
    for name in sched.SCHEDS:
        s, _ = sched.create_scheduler(_solver(sched=name, **keys), Recorder(0.25))
        assert s.noise_range_t == want, name


def test_noise_window_and_std():
    """Noise on [lo, hi) for a pair and on t >= lo for a number; lr_noise_std does not change the draw (the reference's 'normal'
    noise is torch.randn at unit std, redrawn until it is inside lr_noise_pct)."""
    base = _solver(epochs=20, warmup_epochs=0, lr_cycle_limit=0)
    clean, _ = sched.create_scheduler(base, Recorder(0.25))
    runs = {}
    for key, lr_noise, std in (("pair", [0.3, 0.9], 1.0), ("pair_std", [0.3, 0.9], 0.25), ("one", [0.5], 1.0)):
        s, _ = sched.create_scheduler(dict(base, lr_noise=lr_noise, lr_noise_pct=0.4, lr_noise_std=std), Recorder(0.25))
        runs[key] = []
        for e in range(1, 31):
            s.step(e)
            clean.step(e)
            runs[key].append(s.lr / clean.lr - 1.0)
    assert runs["pair"] == runs["pair_std"]
    for key, lo, hi in (("pair", 6, 18), ("one", 10, 31)):
        for e, rel in enumerate(runs[key], 1):
            assert (abs(rel) > 0) == (lo <= e < hi), (key, e)
            assert abs(rel) < 0.4 + 1e-12
    assert runs["pair"][9:17] == runs["one"][9:17]        # the draw depends on seed + t only


def test_construction_lr_must_be_solver_lr():
    with pytest.raises(ValueError, match="solver.lr"):
        sched.create_scheduler(_solver(lr=0.25), Recorder(0.2))
    s, _ = sched.create_scheduler(_solver(lr=0.1), Recorder(0.1))          # fp32(0.1) held, 0.1 scheduled
    assert s.base_lr == 0.1


def test_construction_moves_to_warmup_lr_only_with_a_warmup():
    ts = Recorder(0.25)
    s, _ = sched.create_scheduler(_solver(), ts)
    assert ts.calls == [0.0001] and s.lr == 0.0001
    for name in sched.SCHEDS:
        ts = Recorder(0.25)
        s, _ = sched.create_scheduler(_solver(sched=name, warmup_epochs=0), ts)
        assert ts.calls == [] and s.lr == 0.25


def test_step_update_leaves_the_lr():
    ts = Recorder(0.25)
    s, _ = sched.create_scheduler(_solver(), ts)
    for n in range(100):
        s.step_update(n)
    assert ts.calls == [0.0001] and s.lr == 0.0001


def test_plateau_without_metric_keeps_its_counters():
    ts = Recorder(0.25)
    s, _ = sched.create_scheduler(_solver(sched="plateau", epochs=30, patience_epochs=1), ts)
    for e in range(1, 6):
        s.step(e)
    warm = s.lr                                            # the end of the warm-up
    for e in range(6, 20):
        s.step(e)
    assert s.lr == warm and s.num_bad_epochs == 0 and s.best == -float("inf")
    s.step(20, 1.0)
    s.step(21, 1.0)
    s.step(22, 1.0)                                        # two epochs without improvement > patience 1
    assert s.lr == warm * 0.1 and ts.calls[-1] == warm * 0.1 and len(ts.calls) == 7


def test_non_integral_noise_seed_is_refused():
    with pytest.raises(ValueError, match="seed"):
        sched.create_scheduler(_solver(lr_noise=[0.5]), Recorder(0.25), seed=1.5)
    sched.create_scheduler(_solver(), Recorder(0.25), seed=1.5)             # no noise: the seed is not used
