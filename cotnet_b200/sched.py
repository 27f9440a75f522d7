"""The reference's learning-rate schedules (scheduler/scheduler_factory.py:create_scheduler and the cosine, tanh, step and plateau
classes it builds) with a TrainStep as their target instead of a torch.optim.Optimizer.

The factory builds epoch-indexed schedules only (t_in_epochs=True), and train.py calls ``step(epoch + 1, None)`` once after
every epoch (train.py:360-361), so the learning rate changes at most once per epoch.  It is computed here on the host in Python
doubles, in the reference's order of operations, and every change reaches the device through ``train_step.set_lr``: one fill of
``hyper[0]`` / ``hyper_small[0]``, which a captured step reads at every replay.  The device holds it in fp32, where the
reference's param_group keeps the double; ``lr`` is that double.

The reference's optimizer has the two parameter groups of add_weight_decay, both at solver.lr, so every per-group list of the
reference holds one value twice; here it is one value.
"""
import math
from collections.abc import Mapping

import numpy as np
import torch

SCHEDS = ("cosine", "tanh", "step", "plateau")


class Scheduler:
    """scheduler/scheduler.py:Scheduler.  `base_lr` is the optimizer's initial_lr: the LR the TrainStep was built with.
    step(epoch, metric) moves the LR to the schedule's value for `epoch`; step_update() never changes it (per-update schedules
    are not built by the factory).  `lr` is the value the reference's param_group['lr'] would hold."""

    def __init__(self, train_step, base_lr, noise_range_t=None, noise_pct=0.67, noise_std=1.0, noise_seed=None):
        self.train_step = train_step
        self.base_lr = base_lr
        self.lr = base_lr                                 # what the TrainStep holds already: no set_lr
        self.metric = None
        self.noise_range_t = noise_range_t
        self.noise_pct = noise_pct
        self.noise_std = noise_std                        # stored only: the reference's 'normal' noise draws at unit std
        self.noise_seed = noise_seed if noise_seed is not None else 42
        if noise_range_t is not None and float(self.noise_seed) != int(self.noise_seed):
            raise ValueError("lr noise: the seed must be a whole number (torch.Generator.manual_seed), got %r" % (self.noise_seed,))

    def _set(self, lr):
        """update_groups(lr), forwarded to the device only when the value changes."""
        if lr != self.lr:
            self.lr = lr
            self.train_step.set_lr(lr)

    def _start_warmup(self, lr_at_end):
        """A linear warm-up from warmup_lr_init, where the LR starts, to lr_at_end over warmup_t epochs."""
        if self.warmup_t:
            self.warmup_step = (lr_at_end - self.warmup_lr_init) / self.warmup_t
            self._set(self.warmup_lr_init)
        else:
            self.warmup_step = 1

    def get_epoch_values(self, epoch):
        return None

    def step(self, epoch, metric=None):
        self.metric = metric
        lr = self.get_epoch_values(epoch)
        if lr is not None:
            noise = self._noise(epoch)
            self._set(lr if noise is None else lr + lr * noise)

    def step_update(self, num_updates, metric=None):
        self.metric = metric

    def _noise(self, t):
        """The relative noise of epoch t, or None outside noise_range_t ([lo, hi) for a pair, t >= lo for a number).  A fresh
        generator seeded with noise_seed + t per epoch, torch.randn redrawn until |noise| < noise_pct (the reference's 'normal'
        noise, the only kind its schedules are built with).  The configs' seed is the float 1.0, which Generator.manual_seed
        refuses; the seed used is the whole number it names."""
        r = self.noise_range_t
        if r is None:
            return None
        if not (r[0] <= t < r[1] if isinstance(r, (list, tuple)) else t >= r):
            return None
        g = torch.Generator()
        g.manual_seed(int(self.noise_seed + t))
        while True:
            noise = torch.randn(1, generator=g).item()
            if abs(noise) < self.noise_pct:
                return noise


class _CyclicScheduler(Scheduler):
    """What cosine_lr.py and tanh_lr.py share: the warm-up, the warm-up prefix, the cycle index (log-floor when t_mul != 1),
    decay_rate ** i on lr_max and lr_min, the cycle limit and get_cycle_length()."""

    def __init__(self, train_step, base_lr, t_initial, t_mul=1., lr_min=0., decay_rate=1., warmup_t=0, warmup_lr_init=0,
                 warmup_prefix=False, cycle_limit=0, noise_range_t=None, noise_pct=0.67, noise_std=1.0, noise_seed=42):
        super().__init__(train_step, base_lr, noise_range_t=noise_range_t, noise_pct=noise_pct, noise_std=noise_std,
                         noise_seed=noise_seed)
        if not t_initial > 0 or not lr_min >= 0:
            raise ValueError("t_initial must be > 0 and lr_min >= 0, got %r and %r" % (t_initial, lr_min))
        self.t_initial = t_initial
        self.t_mul = t_mul
        self.lr_min = lr_min
        self.decay_rate = decay_rate
        self.cycle_limit = cycle_limit
        self.warmup_t = warmup_t
        self.warmup_lr_init = warmup_lr_init
        self.warmup_prefix = warmup_prefix

    def _get_lr(self, t):
        if t < self.warmup_t:
            return self.warmup_lr_init + t * self.warmup_step
        if self.warmup_prefix:
            t = t - self.warmup_t
        if self.t_mul != 1:
            i = math.floor(math.log(1 - t / self.t_initial * (1 - self.t_mul), self.t_mul))
            t_i = self.t_mul ** i * self.t_initial
            t_curr = t - (1 - self.t_mul ** i) / (1 - self.t_mul) * self.t_initial
        else:
            i = t // self.t_initial
            t_i = self.t_initial
            t_curr = t - (self.t_initial * i)
        if self.cycle_limit == 0 or (self.cycle_limit > 0 and i < self.cycle_limit):
            gamma = self.decay_rate ** i
            return self._curve(self.lr_min * gamma, self.base_lr * gamma, t_curr, t_i)
        return self._past_limit()

    def get_epoch_values(self, epoch):
        return self._get_lr(epoch)

    def get_cycle_length(self, cycles=0):
        if not cycles:
            cycles = self.cycle_limit
        cycles = max(1, cycles)
        if self.t_mul == 1.0:
            return self.t_initial * cycles
        return int(math.floor(-self.t_initial * (self.t_mul ** cycles - 1) / (1 - self.t_mul)))


class CosineLRScheduler(_CyclicScheduler):
    """scheduler/cosine_lr.py: cosine decay with restarts (SGDR).  Past the cycle limit the LR is lr_min, undecayed."""

    def __init__(self, train_step, base_lr, t_initial, **kw):
        super().__init__(train_step, base_lr, t_initial, **kw)
        self._start_warmup(self.base_lr)

    def _curve(self, lr_min, lr_max, t_curr, t_i):
        return lr_min + 0.5 * (lr_max - lr_min) * (1 + math.cos(math.pi * t_curr / t_i))

    def _past_limit(self):
        return self.lr_min


class TanhLRScheduler(_CyclicScheduler):
    """scheduler/tanh_lr.py: hyperbolic-tangent decay with restarts.  Without warmup_prefix the warm-up ends at the schedule's
    value for warmup_t; past the cycle limit the LR is lr_min * decay_rate ** cycle_limit."""

    def __init__(self, train_step, base_lr, t_initial, lb=-6., ub=4., **kw):
        super().__init__(train_step, base_lr, t_initial, **kw)
        if not lb < ub or not self.cycle_limit >= 0 or not self.warmup_t >= 0 or not self.warmup_lr_init >= 0:
            raise ValueError("tanh schedule: needs lb < ub and cycle_limit, warmup_t, warmup_lr_init >= 0")
        self.lb = lb
        self.ub = ub
        self._start_warmup(self.base_lr if self.warmup_prefix else self._get_lr(self.warmup_t))

    def _curve(self, lr_min, lr_max, t_curr, t_i):
        tr = t_curr / t_i
        return lr_min + 0.5 * (lr_max - lr_min) * (1 - math.tanh(self.lb * (1. - tr) + self.ub * tr))

    def _past_limit(self):
        return self.lr_min * (self.decay_rate ** self.cycle_limit)


class StepLRScheduler(Scheduler):
    """scheduler/step_lr.py: base_lr * decay_rate ** (t // decay_t) after the warm-up."""

    def __init__(self, train_step, base_lr, decay_t, decay_rate=1., warmup_t=0, warmup_lr_init=0, noise_range_t=None,
                 noise_pct=0.67, noise_std=1.0, noise_seed=42):
        super().__init__(train_step, base_lr, noise_range_t=noise_range_t, noise_pct=noise_pct, noise_std=noise_std,
                         noise_seed=noise_seed)
        self.decay_t = decay_t
        self.decay_rate = decay_rate
        self.warmup_t = warmup_t
        self.warmup_lr_init = warmup_lr_init
        self._start_warmup(base_lr)

    def get_epoch_values(self, epoch):
        if epoch < self.warmup_t:
            return self.warmup_lr_init + epoch * self.warmup_step
        return self.base_lr * (self.decay_rate ** (epoch // self.decay_t))


class PlateauLRScheduler(Scheduler):
    """scheduler/plateau_lr.py: torch's ReduceLROnPlateau (relative threshold, `patience_t`, `cooldown_t`, `lr_min`, its 1e-8
    eps) after a warm-up that runs up to and including epoch warmup_t, with noise on top.  The noise is applied to the LR the
    plateau rule left and undone (restore_lr) before the next step, so the rule never sees it.

    step(epoch, metric): `metric` is the evaluation metric (top-1 in 'max' mode, a loss in 'min' mode).  With metric=None, which is
    what train.py passes, only the warm-up and the noise act: the plateau rule is skipped and its counters do not move.  (The
    reference hands None on to ReduceLROnPlateau.step, whose float(None) raises after the warm-up.)"""

    def __init__(self, train_step, base_lr, decay_rate=0.1, patience_t=10, threshold=1e-4, cooldown_t=0, warmup_t=0,
                 warmup_lr_init=0, lr_min=0, mode="max", noise_range_t=None, noise_pct=0.67, noise_std=1.0, noise_seed=None):
        super().__init__(train_step, base_lr, noise_range_t=noise_range_t, noise_pct=noise_pct, noise_std=noise_std,
                         noise_seed=noise_seed)
        if decay_rate >= 1.0:
            raise ValueError("plateau schedule: decay_rate must be < 1.0, got %r" % (decay_rate,))
        if mode not in ("min", "max"):
            raise ValueError("plateau schedule: mode must be 'min' or 'max', got %r" % (mode,))
        self.factor = decay_rate
        self.patience = patience_t
        self.threshold = threshold
        self.cooldown = cooldown_t
        self.min_lr = lr_min
        self.mode = mode
        self.eps = 1e-8
        self.best = math.inf if mode == "min" else -math.inf
        self.num_bad_epochs = 0
        self.cooldown_counter = 0
        self.warmup_t = warmup_t
        self.warmup_lr_init = warmup_lr_init
        self._start_warmup(base_lr)
        self.restore_lr = None

    def _is_better(self, a):
        if self.mode == "min":
            return a < self.best * (1.0 - self.threshold)
        return a > self.best * (self.threshold + 1.0)

    def _plateau(self, current, lr):
        """ReduceLROnPlateau.step on the LR `lr`; returns the new LR."""
        if self._is_better(current):
            self.best = current
            self.num_bad_epochs = 0
        else:
            self.num_bad_epochs += 1
        if self.cooldown_counter > 0:
            self.cooldown_counter -= 1
            self.num_bad_epochs = 0
        if self.num_bad_epochs > self.patience:
            new_lr = max(lr * self.factor, self.min_lr)
            if lr - new_lr > self.eps:
                lr = new_lr
            self.cooldown_counter = self.cooldown
            self.num_bad_epochs = 0
        return lr

    def step(self, epoch, metric=None):
        if epoch <= self.warmup_t:
            self._set(self.warmup_lr_init + epoch * self.warmup_step)
            return
        lr = self.lr
        if self.restore_lr is not None:
            lr, self.restore_lr = self.restore_lr, None
        if metric is not None:
            lr = self._plateau(float(metric), lr)
        noise = self._noise(epoch)
        if noise is not None:
            self.restore_lr = lr
            lr = lr + lr * noise
        self._set(lr)


_MISSING = object()


def _get(solver, key, default=_MISSING):
    """solver[key] of a mapping (a yacs CfgNode is one) or solver.key of an attribute object."""
    if isinstance(solver, Mapping):
        value = solver.get(key, default)
    else:
        value = getattr(solver, key, default)
    if value is _MISSING:
        raise KeyError("solver.%s is missing" % key)
    return value


def _construction_lr(solver, train_step):
    """solver.lr, the initial_lr of the reference's optimizer; the TrainStep must have been built with it."""
    lr = _get(solver, "lr")
    held = float(train_step.hyper[0])
    if held != float(np.float32(lr)):
        raise ValueError("create_scheduler: the TrainStep holds lr %r, not solver.lr = %r; build it with lr=solver.lr" % (held, lr))
    return lr


def create_scheduler(solver, train_step, seed=1.0, eval_metric="top1"):
    """scheduler_factory.create_scheduler(cfg, optimizer) -> (scheduler, num_epochs).

    solver: the config's solver section, a mapping or an attribute object, after pop_unused_value (an absent or empty lr_noise
    means no noise).  seed: the config's seed (the noise seed); eval_metric: eval.eval_metric ('min' plateau mode when it contains
    'loss').  The TrainStep must have been built with lr=solver.lr, which is the schedule's base value; construction already moves
    the LR to warmup_lr when there is a warm-up.  cosine and tanh return num_epochs = get_cycle_length() + cooldown_epochs, step and
    plateau return solver.epochs, and any other sched gives (None, solver.epochs).  solver.start_epoch is not applied here:
    setup_scheduler does that."""
    num_epochs = _get(solver, "epochs")
    lr_noise = _get(solver, "lr_noise", None)
    if lr_noise is None or (isinstance(lr_noise, (list, tuple)) and len(lr_noise) == 0):
        noise_range = None
    elif isinstance(lr_noise, (list, tuple)):
        noise_range = [n * num_epochs for n in lr_noise]
        if len(noise_range) == 1:
            noise_range = noise_range[0]
    else:
        noise_range = lr_noise * num_epochs
    sched = _get(solver, "sched")
    if sched not in SCHEDS:
        return None, num_epochs
    base_lr = _construction_lr(solver, train_step)
    common = dict(warmup_lr_init=_get(solver, "warmup_lr"), warmup_t=_get(solver, "warmup_epochs"), noise_range_t=noise_range,
                  noise_pct=_get(solver, "lr_noise_pct"), noise_std=_get(solver, "lr_noise_std"), noise_seed=seed)
    if sched in ("cosine", "tanh"):
        cyclic = dict(t_mul=_get(solver, "lr_cycle_mul"), lr_min=_get(solver, "min_lr"), cycle_limit=_get(solver, "lr_cycle_limit"))
        if sched == "cosine":
            lr_scheduler = CosineLRScheduler(train_step, base_lr, num_epochs, decay_rate=_get(solver, "decay_rate"), **cyclic, **common)
        else:
            lr_scheduler = TanhLRScheduler(train_step, base_lr, num_epochs, **cyclic, **common)
        num_epochs = lr_scheduler.get_cycle_length() + _get(solver, "cooldown_epochs")
    elif sched == "step":
        lr_scheduler = StepLRScheduler(train_step, base_lr, _get(solver, "decay_epochs"), decay_rate=_get(solver, "decay_rate"),
                                       **common)
    else:
        lr_scheduler = PlateauLRScheduler(train_step, base_lr, decay_rate=_get(solver, "decay_rate"),
                                          patience_t=_get(solver, "patience_epochs"), lr_min=_get(solver, "min_lr"),
                                          mode="min" if "loss" in eval_metric else "max", cooldown_t=0, **common)
    return lr_scheduler, num_epochs


def setup_scheduler(solver, train_step, seed=1.0, eval_metric="top1"):
    """train.py:setup_scheduler without resuming -> (scheduler, start_epoch, num_epochs): create_scheduler, then, when
    solver.start_epoch is present and > 0, step(start_epoch) once.  A negative start_epoch is unset, as pop_unused_value reads
    it.  Train epochs range(start_epoch, num_epochs) and call scheduler.step(epoch + 1) after each."""
    lr_scheduler, num_epochs = create_scheduler(solver, train_step, seed, eval_metric)
    start_epoch = max(0, _get(solver, "start_epoch", 0))
    if lr_scheduler is not None and start_epoch > 0:
        lr_scheduler.step(start_epoch)
    return lr_scheduler, start_epoch, num_epochs
