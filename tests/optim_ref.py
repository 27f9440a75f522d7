"""Restatement in torch of the reference's update rules (optim/optim_factory.py:create_optimizer with lr, momentum, weight_decay,
opt_eps and the factory's defaults; optim/adamw.py, nadam.py, radam.py, rmsprop_tf.py, lookahead.py; torch.optim.SGD, Adam,
Adadelta, RMSprop) and of the EMA that follows the step, for the tests of the optimizer passes.  TEST INFRASTRUCTURE ONLY.

The dtype of the tensors handed in (fp32 or fp64) is the dtype of the element arithmetic; the per-step scalars are Python floats
as in the reference.  Pinned to the reference's own classes by tests/golden/optim.npz (tools/make_optim_golden.py).
"""
import math

import torch

RULES = ("sgd", "nesterov", "momentum", "adam", "adamw", "nadam", "radam", "adadelta", "rmsprop", "rmsproptf")
B1, B2 = 0.9, 0.999
LA_ALPHA, LA_K = 0.5, 6


def split(name):
    """create_optimizer's reading of solver.opt: (rule, lookahead)."""
    parts = name.lower().split("_")
    return parts[-1], len(parts) > 1 and parts[0] == "lookahead"


class Optim:
    """One optimizer over parameter groups [(weight_decay, [tensors])] (the factory's add_weight_decay groups); every tensor gets a
    gradient at every step.  step(grads) updates the tensors in place; state[i] is the reference's state of tensor i."""

    def __init__(self, name, groups, lr, momentum=0.9, eps=1e-8, nesterov=True, radam_fp32=False):
        """radam_fp32: compute RAdam in fp32 whatever the tensors' dtype, as the reference's class does (for its golden)."""
        self.rule, self.lookahead = split(name)
        self.radam_fp32 = radam_fp32
        assert self.rule in RULES, name
        self.groups = groups
        self.lr, self.momentum, self.eps = lr, momentum, eps
        self.nesterov = nesterov if self.rule == "sgd" else self.rule == "nesterov"
        self.t = 0
        self.la_step = 0
        self.state = []
        for _, ps in groups:
            for p in ps:
                s = {}
                if self.rule in ("sgd", "nesterov", "momentum"):
                    s["momentum_buffer"] = torch.zeros_like(p)
                elif self.rule in ("adam", "adamw", "nadam", "radam"):
                    s["exp_avg"], s["exp_avg_sq"] = torch.zeros_like(p), torch.zeros_like(p)
                    if self.rule == "nadam":
                        s["m_schedule"] = 1.0
                elif self.rule == "adadelta":
                    s["square_avg"], s["acc_delta"] = torch.zeros_like(p), torch.zeros_like(p)
                else:
                    s["square_avg"] = torch.ones_like(p) if self.rule == "rmsproptf" else torch.zeros_like(p)
                    if momentum > 0:
                        s["momentum_buffer"] = torch.zeros_like(p)
                self.state.append(s)

    def params(self):
        return [(wd, p) for wd, ps in self.groups for p in ps]

    def step(self, grads):
        self.t += 1
        for (wd, p), g, s in zip(self.params(), grads, self.state):
            s["step"] = self.t
            getattr(self, "_" + ("sgd" if self.rule in ("nesterov", "momentum") else self.rule))(p, g.to(p.dtype), s, wd)
        if self.lookahead:
            self.la_step += 1
            if self.la_step % LA_K == 0:
                self.sync_lookahead()

    def sync_lookahead(self):
        """Lookahead.update_slow (optim/lookahead.py:31-38): the first call creates the slow weights from the fast ones."""
        for (_, p), s in zip(self.params(), self.state):
            if "slow_buffer" not in s:
                s["slow_buffer"] = p.clone()
            slow = s["slow_buffer"]
            slow.add_(p - slow, alpha=LA_ALPHA)
            p.copy_(slow)

    # ---------------------------------------------------------------------------------------- the rules
    def _sgd(self, p, g, s, wd):                                  # torch.optim.SGD(momentum, dampening 0)
        mu = self.momentum
        d = g + wd * p
        buf = s["momentum_buffer"]
        buf.mul_(mu).add_(d)
        p.sub_(self.lr * (d + mu * buf if self.nesterov else buf))

    def _adam(self, p, g, s, wd):                                 # torch.optim.Adam, amsgrad off
        g = g + wd * p
        m, v = s["exp_avg"], s["exp_avg_sq"]
        m.mul_(B1).add_((1 - B1) * g)
        v.mul_(B2).add_((1 - B2) * g * g)
        bc1, bc2 = 1 - B1 ** self.t, 1 - B2 ** self.t
        denom = v.sqrt() / math.sqrt(bc2) + self.eps
        p.add_(-(self.lr / bc1) * m / denom)

    def _adamw(self, p, g, s, wd):                                # optim/adamw.py:55-117
        p.mul_(1 - self.lr * wd)
        m, v = s["exp_avg"], s["exp_avg_sq"]
        m.mul_(B1).add_((1 - B1) * g)
        v.mul_(B2).add_((1 - B2) * g * g)
        bc1, bc2 = 1 - B1 ** self.t, 1 - B2 ** self.t
        denom = v.sqrt() / math.sqrt(bc2) + self.eps
        p.add_(-(self.lr / bc1) * m / denom)

    def _nadam(self, p, g, s, wd):                                # optim/nadam.py:34-88, schedule_decay 4e-3
        t, sd = self.t, 4e-3
        g = g + wd * p
        mc = B1 * (1. - 0.5 * (0.96 ** (t * sd)))
        mc1 = B1 * (1. - 0.5 * (0.96 ** ((t + 1) * sd)))
        ms_new = s["m_schedule"] * mc
        ms_next = s["m_schedule"] * mc * mc1
        s["m_schedule"] = ms_new
        m, v = s["exp_avg"], s["exp_avg_sq"]
        m.mul_(B1).add_((1. - B1) * g)
        v.mul_(B2).add_((1. - B2) * g * g)
        denom = (v / (1. - B2 ** t)).sqrt() + self.eps
        p.add_(-self.lr * (1. - mc) / (1. - ms_new) * g / denom)
        p.add_(-self.lr * mc1 / (1. - ms_next) * m / denom)

    def _radam(self, p, g, s, wd):                                # optim/radam.py:20-87 (RAdam)
        if self.radam_fp32 and p.dtype != torch.float32:
            # the reference updates p.data.float() with fp32 moments and copies the result back (radam.py:32-44,86)
            p32 = p.float()
            for k in ("exp_avg", "exp_avg_sq"):
                s[k] = s[k].float()
            self._radam(p32, g.float(), s, wd)
            p.copy_(p32)
            return
        t = self.t
        m, v = s["exp_avg"], s["exp_avg_sq"]
        v.mul_(B2).addcmul_(g, g, value=1 - B2)
        m.mul_(B1).add_(g, alpha=1 - B1)
        b2t = B2 ** t
        n_max = 2 / (1 - B2) - 1
        n_sma = n_max - 2 * t * b2t / (1 - b2t)
        if n_sma >= 5:
            step = self.lr * math.sqrt((1 - b2t) * (n_sma - 4) / (n_max - 4) * (n_sma - 2) / n_sma * n_max / (n_max - 2)) / (1 - B1 ** t)
        else:
            step = self.lr / (1 - B1 ** t)
        if wd != 0:
            p.add_(p, alpha=-wd * self.lr)
        if n_sma >= 5:
            p.addcdiv_(m, v.sqrt().add_(self.eps), value=-step)
        else:
            p.add_(m, alpha=-step)

    def _adadelta(self, p, g, s, wd):                             # torch.optim.Adadelta, rho 0.9
        rho = 0.9
        g = g + wd * p
        sq, acc = s["square_avg"], s["acc_delta"]
        sq.mul_(rho).add_((1 - rho) * g * g)
        delta = (acc + self.eps).sqrt() / (sq + self.eps).sqrt() * g
        acc.mul_(rho).add_((1 - rho) * delta * delta)
        p.add_(-self.lr * delta)

    def _rmsprop(self, p, g, s, wd):                              # torch.optim.RMSprop, alpha 0.9
        a = 0.9
        g = g + wd * p
        sq = s["square_avg"]
        sq.mul_(a).add_((1 - a) * g * g)
        avg = sq.sqrt() + self.eps
        if "momentum_buffer" in s:
            buf = s["momentum_buffer"]
            buf.mul_(self.momentum).add_(g / avg)
            p.add_(-self.lr * buf)
        else:
            p.add_(-self.lr * g / avg)

    def _rmsproptf(self, p, g, s, wd):                            # optim/rmsprop_tf.py:71-136, lr_in_momentum
        a = 0.9
        g = g + wd * p
        sq = s["square_avg"]
        sq.add_((1. - a) * (g * g - sq))
        avg = (sq + self.eps).sqrt()
        if "momentum_buffer" in s:
            buf = s["momentum_buffer"]
            buf.mul_(self.momentum).add_(self.lr * g / avg)
            p.sub_(buf)
        else:
            p.add_(-self.lr * g / avg)


def ema(e, p, decay):
    """ModelEmaV2.update on one tensor (utils/model_ema.py:52-53)."""
    return decay * e + (1.0 - decay) * p
