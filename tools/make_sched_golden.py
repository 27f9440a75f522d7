"""Generate tests/golden/sched.npz from the reference's OWN learning-rate schedules.  TEST INFRASTRUCTURE ONLY.

Run where the reference tree exists (oracle/ref_import.py finds it):   python tools/make_sched_golden.py

Every schedule is built by the reference's create_scheduler (scheduler/scheduler_factory.py) over an SGD optimizer with the two
parameter groups of optim_factory.add_weight_decay (a Linear layer: decayed weight, undecayed bias), both at solver.lr.  The
solver sections are the config's defaults (config/config.py) updated with the case's keys, after pop_unused_value.  Three
test-only shims, none of which touches the schedule arithmetic:
* PyYAML reads values such as ``1e-5`` as strings; they pass through ast.literal_eval, as yacs's merge_from_file decodes them.
* The installed torch no longer accepts ``ReduceLROnPlateau(verbose=)``; the keyword only switched on logging and is dropped.
* ``ReduceLROnPlateau.step(None)`` raises (float(None)); the library skips the plateau rule on a None metric (only the warm-up
  and the noise act), so the shim returns early on None to record that case through the reference's own warm-up, noise and
  restore_lr code.
``torch.Generator.manual_seed`` takes integers only, so the configs' seed 1.0 reaches the reference as the integer 1.

Stored per case c (``cases`` lists them): c/solver (the resolved solver section as JSON), c/seed, c/eval_metric, c/sched_none
(1 when the factory returns no scheduler), c/num_epochs, c/lr_init (the LR after construction), c/start_epoch and c/lr_start
(the LR after train.py's step(start_epoch), lr_init when there is none), c/metrics (the metric fed to step(e), NaN for None) and
c/lr (the LR after step(e) for e = 1 .. num_epochs + 5, one run from construction).  The WARMUP_PREFIX cases run the factory
with its cosine and tanh classes given warmup_prefix=True.
"""
import ast
import functools
import json
import os
import sys
import warnings
from types import SimpleNamespace

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sched.npz")
EXTRA_EPOCHS = 5
BASE = "CoTNet-50-350epoch"                        # the config the scaled-down cases start from

#: (case, solver keys set on top of BASE's, eval_metric, metrics)
#: metrics: None -> step(e) without a metric; "rise_flat" / "fall_flat" -> the plateau sequences of _metrics
CASES = [
    ("tanh", dict(sched="tanh", epochs=30, cooldown_epochs=5), "top1", None),
    ("step", dict(sched="step", epochs=100, decay_epochs=30, decay_rate=0.1), "top1", None),
    ("plateau_max", dict(sched="plateau", epochs=60, patience_epochs=5), "top1", "rise_flat"),
    ("plateau_min", dict(sched="plateau", epochs=60, patience_epochs=5), "loss", "fall_flat"),
    ("plateau_none", dict(sched="plateau", epochs=30, lr_noise=[0.2, 0.8], lr_noise_pct=0.5), "top1", None),
    ("cosine_restarts", dict(epochs=10, lr_cycle_mul=2.0, lr_cycle_limit=3, decay_rate=0.5), "top1", None),
    ("cosine_cooldown", dict(epochs=20, lr_cycle_limit=1, cooldown_epochs=10), "top1", None),
    ("cosine_noise_pair", dict(epochs=20, cooldown_epochs=3, lr_noise=[0.3, 0.9], lr_noise_pct=0.4, lr_noise_std=0.5),
     "top1", None),
    ("cosine_noise_one", dict(epochs=10, lr_cycle_mul=2.0, lr_cycle_limit=2, lr_noise=[0.5], lr_noise_pct=0.3,
                                    lr_noise_std=2.0), "top1", None),
    ("cosine_no_warmup", dict(epochs=20, warmup_epochs=0), "top1", None),
    ("cosine_start_epoch", dict(epochs=20, start_epoch=3), "top1", None),
    ("unknown_sched", dict(sched="multistep", epochs=20), "top1", None),
    ("cosine_warmup_prefix", dict(epochs=20, cooldown_epochs=3), "top1", None),
    ("tanh_warmup_prefix", dict(sched="tanh", epochs=20, cooldown_epochs=3), "top1", None),
]
#: cases whose cosine / tanh class is built with warmup_prefix=True (the factory leaves it False)
WARMUP_PREFIX = ("cosine_warmup_prefix", "tanh_warmup_prefix")


def _decode(v):
    if isinstance(v, str):
        try:
            return ast.literal_eval(v)
        except (ValueError, SyntaxError):
            return v
    return v


def _config(name):
    with open(os.path.join(ref_import.REF, "cot_experiments", name, "config.yaml")) as f:
        return yaml.safe_load(f)


def _solver(defaults, name, keys):
    """config defaults <- the yaml's solver section <- keys, then pop_unused_value's solver part."""
    solver = dict(defaults)
    solver.update({k: _decode(v) for k, v in _config(name)["solver"].items()})
    solver.update(keys)
    solver = {k: (list(v) if isinstance(v, tuple) else v) for k, v in solver.items()}
    if len(solver["lr_noise"]) == 0:
        solver.pop("lr_noise")
    if solver["start_epoch"] < 0:
        solver.pop("start_epoch")
    return solver


def _metrics(kind, n):
    e = np.arange(1, n + 1, dtype=np.float64)
    if kind is None:
        return np.full(n, np.nan)
    if kind == "rise_flat":                        # top-1 rising to epoch 20, then flat
        return np.where(e <= 20, 40.0 + 1.5 * e, 70.0)
    return np.where(e <= 15, 6.9 * 0.9 ** e, 6.9 * 0.9 ** 15)     # a loss falling to epoch 15, then flat


def _install_plateau_shim():
    base = torch.optim.lr_scheduler.ReduceLROnPlateau

    class Plateau(base):
        def __init__(self, *a, verbose=None, **k):
            super().__init__(*a, **k)

        def step(self, metrics, epoch=None):
            if metrics is None:
                return
            with warnings.catch_warnings():                      # plateau_lr.py passes the deprecated `epoch`
                warnings.simplefilter("ignore", UserWarning)
                super().step(metrics, epoch)

    torch.optim.lr_scheduler.ReduceLROnPlateau = Plateau


def run(create_scheduler, add_weight_decay, solver, seed, eval_metric, metrics_kind):
    cfg = SimpleNamespace(solver=_Solver(solver), seed=int(seed), eval=SimpleNamespace(eval_metric=eval_metric))
    model = torch.nn.Linear(4, 3)
    opt = torch.optim.SGD(add_weight_decay(model, solver["weight_decay"]), lr=solver["lr"], momentum=solver["momentum"],
                          nesterov=True)

    def lr_of():
        lrs = [g["lr"] for g in opt.param_groups]
        assert lrs[0] == lrs[1], lrs
        return float(lrs[0])

    sched, num_epochs = create_scheduler(cfg, opt)
    rec = {"sched_none": np.int64(sched is None), "num_epochs": np.int64(num_epochs), "lr_init": np.float64(lr_of())}
    start = solver.get("start_epoch", 0)
    if sched is not None and start > 0:
        sched.step(start)                          # train.py:setup_scheduler
    rec["start_epoch"], rec["lr_start"] = np.int64(start), np.float64(lr_of())
    n = num_epochs + EXTRA_EPOCHS
    metrics = _metrics(metrics_kind, n)
    lrs = []
    for e in range(1, n + 1):
        if sched is not None:
            m = None if np.isnan(metrics[e - 1]) else float(metrics[e - 1])
            sched.step(e, m)
        lrs.append(lr_of())
    rec["metrics"], rec["lr"] = metrics, np.array(lrs, dtype=np.float64)
    return rec


class _Solver(dict):
    """The solver section as the factory reads it: attributes and `in`."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


def main():
    ref_import.load()
    _install_plateau_shim()
    from config import config as ref_config                      # noqa: E402  (the reference package is on sys.path now)
    from optim.optim_factory import add_weight_decay              # noqa: E402
    from scheduler import scheduler_factory                      # noqa: E402
    defaults = dict(ref_config._C.solver)
    configs = sorted(d for d in os.listdir(os.path.join(ref_import.REF, "cot_experiments")))
    cases = [(c, c, {}, None, None) for c in configs] + [(c, BASE, k, m, mk) for c, k, m, mk in CASES]
    rec = {"cases": np.array([c for c, _, _, _, _ in cases])}
    for case, src, keys, eval_metric, metrics_kind in cases:
        y = _config(src)
        solver = _solver(defaults, src, keys)
        seed = float(_decode(y.get("seed", ref_config._C.seed)))
        eval_metric = eval_metric or y.get("eval", {}).get("eval_metric", "top1")
        saved = {k: getattr(scheduler_factory, k) for k in ("CosineLRScheduler", "TanhLRScheduler")}
        if case in WARMUP_PREFIX:
            for k, cls in saved.items():
                setattr(scheduler_factory, k, functools.partial(cls, warmup_prefix=True))
        try:
            r = run(scheduler_factory.create_scheduler, add_weight_decay, solver, seed, eval_metric, metrics_kind)
        finally:
            for k, cls in saved.items():
                setattr(scheduler_factory, k, cls)
        r.update(solver=np.array(json.dumps(solver, sort_keys=True)), seed=np.float64(seed), eval_metric=np.array(eval_metric))
        for k, v in r.items():
            rec["%s/%s" % (case, k)] = v
        print("%-28s num_epochs %4d  lr_init %.6g  lr[:6] %s" % (case, r["num_epochs"], r["lr_init"],
                                                                   " ".join("%.6g" % v for v in r["lr"][:6])))
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, "%d bytes" % os.path.getsize(OUT))


if __name__ == "__main__":
    main()
