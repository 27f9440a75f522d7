"""Generate tests/golden/optim.npz from the reference's OWN optimizers.  TEST INFRASTRUCTURE ONLY.

Run where the reference tree exists (oracle/ref_import.py finds it):   python tools/make_optim_golden.py

Every optimizer is built by the reference's create_optimizer (optim/optim_factory.py) from a solver config -- so adamw, nadam,
radam, rmsproptf and lookahead are the reference's classes, adam, adadelta and rmsprop torch.optim's, with the factory's
arguments -- over a module with one decayed 2-D weight `w` [6, 10] and one undecayed 1-D bias `b` [6] (add_weight_decay), in
fp64 on CPU.  14 steps of seeded gradients; the learning rate changes before step 8 (LR2_STEP).  Stored:
* w0, b0: the initial weights; gw_<s>, gb_<s> (s = 1..14): the gradients of step s;
* <case>/w_<s>, <case>/b_<s>: the weights after step s; <case>/state_<key>_<w|b>: the final optimizer state of each tensor
  (Lookahead's slow_buffer included), <case>/step: the final step count;
* cases, opts, momenta: the case names, their solver.opt and solver.momentum.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "optim.npz")
SEED = 31415
STEPS, LR, LR2, LR2_STEP, WD, EPS = 14, 0.01, 0.004, 8, 0.05, 1e-8
#: (case, solver.opt, solver.momentum)
CASES = [("sgd", "sgd", 0.9), ("momentum", "momentum", 0.9), ("adam", "adam", 0.9), ("adamw", "adamw", 0.9),
         ("nadam", "nadam", 0.9), ("radam", "radam", 0.9), ("adadelta", "adadelta", 0.9), ("rmsprop", "rmsprop", 0.9),
         ("rmsprop_m0", "rmsprop", 0.0), ("rmsproptf", "rmsproptf", 0.9), ("rmsproptf_m0", "rmsproptf", 0.0),
         ("lookahead_sgd", "lookahead_sgd", 0.9), ("lookahead_adamw", "lookahead_adamw", 0.9),
         ("lookahead_rmsproptf", "lookahead_rmsproptf", 0.9), ("lookahead_radam", "lookahead_radam", 0.9)]


class Mod(torch.nn.Module):
    def __init__(self, w, b):
        super().__init__()
        self.w = torch.nn.Parameter(w.clone())
        self.b = torch.nn.Parameter(b.clone())


def inputs(seed=SEED):
    g = torch.Generator().manual_seed(seed)
    w0 = torch.randn(6, 10, generator=g, dtype=torch.float64) * 0.5
    b0 = torch.randn(6, generator=g, dtype=torch.float64) * 0.5
    grads = []
    for s in range(STEPS):
        scale = torch.exp(torch.randn(6, 1, generator=g, dtype=torch.float64))       # a spread of row scales
        grads.append(((torch.randn(6, 10, generator=g, dtype=torch.float64) * scale * 0.1),
                      torch.randn(6, generator=g, dtype=torch.float64) * 0.1))
    return w0, b0, grads


def main():
    ref_import.load()
    from optim.optim_factory import create_optimizer                  # noqa: E402  (the reference package is on sys.path now)
    w0, b0, grads = inputs()
    rec = {"w0": w0.numpy(), "b0": b0.numpy(), "cases": np.array([c for c, _, _ in CASES]),
           "opts": np.array([o for _, o, _ in CASES]), "momenta": np.array([m for _, _, m in CASES]),
           "lr": np.float64(LR), "lr2": np.float64(LR2), "lr2_step": np.int64(LR2_STEP), "weight_decay": np.float64(WD),
           "eps": np.float64(EPS)}
    for s, (gw, gb) in enumerate(grads, 1):
        rec["gw_%d" % s], rec["gb_%d" % s] = gw.numpy(), gb.numpy()
    for case, opt, mom in CASES:
        m = Mod(w0, b0)
        cfg = types.SimpleNamespace(amp=False, solver=types.SimpleNamespace(opt=opt, lr=LR, momentum=mom, weight_decay=WD, opt_eps=EPS))
        o = create_optimizer(cfg, m)
        for s, (gw, gb) in enumerate(grads, 1):
            if s == LR2_STEP:
                for grp in o.param_groups:
                    grp["lr"] = LR2
            m.w.grad, m.b.grad = gw.clone(), gb.clone()
            o.step()
            rec["%s/w_%d" % (case, s)] = m.w.detach().numpy().copy()
            rec["%s/b_%d" % (case, s)] = m.b.detach().numpy().copy()
        states = [o.state[m.w], o.state[m.b]]
        if hasattr(o, "base_optimizer"):
            states = [{**o.base_optimizer.state[p], **o.state[p]} for p in (m.w, m.b)]
        for tag, st in zip("wb", states):
            for k, v in st.items():
                if torch.is_tensor(v) and v.numel() > 1:
                    rec["%s/state_%s_%s" % (case, k, tag)] = v.detach().numpy().copy()
                elif k in ("step", "m_schedule"):
                    rec["%s/%s_%s" % (case, k, tag)] = np.float64(float(v))
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, "%d bytes" % os.path.getsize(OUT))


if __name__ == "__main__":
    main()
