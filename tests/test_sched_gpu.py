"""A learning-rate schedule driving TrainStep on the H100: a scaled-down cosine config (warm-up, noise, cooldown) stepped between
epochs of captured replays.  After every epoch the device LR is fp32(sched.lr), one step per epoch matches the fp64 restatement of
the update rule (tests/optim_ref.py) at the scheduled LR, and a second TrainStep stepped eagerly through the same schedule is
bit-identical to the captured one."""
import numpy as np
import pytest
import torch

import optim_ref
from test_clip_gpu import DEC, MU, WD, _batch, _small_model
from test_optim_gpu import EPS, _f32

pytestmark = pytest.mark.gpu

REPLAYS = 3
#: the CoTNet-50 config's solver section scaled down: 3 warm-up epochs, a 6-epoch cosine, 2 cooldown epochs at min_lr, and noise
#: on epochs [3, 6)
SOLVER = dict(sched="cosine", lr_noise=[0.5, 1.0], lr_noise_pct=0.67, lr_noise_std=1.0, lr_cycle_mul=1.0, lr_cycle_limit=1,
              warmup_lr=1e-4, min_lr=1e-5, epochs=6, decay_epochs=30, warmup_epochs=3, cooldown_epochs=2, patience_epochs=10,
              decay_rate=0.1)
LRS = {"sgd": 0.1, "adamw": 2e-3, "lookahead_rmsproptf": 1e-3}


def _step_against_restatement(ts, x, y, lr, opt):
    """One eager step of `ts` split into forward_backward and optimizer_step, its fp32 masters and EMA checked against optim_ref
    from the state before the step at learning rate `lr`.  Returns (loss, largest error / max|ref|)."""
    loss = ts.forward_backward(x, y)
    names = [n for n, _ in ts.model.named_parameters()]
    grads = {n: t.double().clone() for n, t in ts.grads().items()}
    master = {n: t.double().clone() for n, t in ts.master_state().items()}
    ema = {n: t.double().clone() for n, t in ts.ema_state().items()}
    ostate = {n: {k: (v.double().clone() if v.dim() else v.item()) for k, v in d.items()} for n, d in ts.optimizer_state().items()}
    hyp = ts.hyper.tolist()
    assert hyp[0] == lr and ts.hyper_small[0].item() == lr
    ts.optimizer_step()
    torch.cuda.synchronize()
    small = {n for n, _, _ in ts.plan["small"]}
    after, after_ema = ts.master_state(), ts.ema_state()
    worst = 0.0
    for n in names:
        p = master[n].clone()
        o = optim_ref.Optim(opt, [(0.0 if n in small else hyp[2], [p])], lr, hyp[1], _f32(EPS))
        o.t = o.la_step = int(ostate[n].get("step", 1))
        for k, v in ostate[n].items():
            if k in o.state[0] or (k == "slow_buffer" and o.la_step >= optim_ref.LA_K):
                o.state[0][k] = v.clone() if torch.is_tensor(v) else v
        o.step([grads[n]])
        for k, got, ref in (("P", after[n], p), ("E", after_ema[n], optim_ref.ema(ema[n], p, DEC))):
            err = ((got.double() - ref).abs().max() / ref.abs().max()).item()
            worst = max(worst, err)
            assert err <= 1e-6, (opt, n, k, err)
    return loss, worst


@pytest.mark.parametrize("opt", sorted(LRS))
def test_schedule_drives_captured_steps(opt, monkeypatch):
    from cotnet_b200 import sched, trainer
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    solver = dict(SOLVER, lr=LRS[opt])
    kw = dict(lr=solver["lr"], momentum=MU, weight_decay=WD, ema_decay=DEC, amp_dtype=torch.bfloat16, weights="bf16", opt=opt)
    t1, t2 = trainer.TrainStep(_small_model(), **kw), trainer.TrainStep(_small_model(), **kw)
    s1, start, num_epochs = sched.setup_scheduler(solver, t1)
    s2, _, _ = sched.setup_scheduler(solver, t2)
    assert (start, num_epochs) == (0, 8) and s1.lr == s2.lr == solver["warmup_lr"]
    batches = [_batch(40 + i, torch.bfloat16) for i in range(REPLAYS)]
    assert t1.capture(*batches[0], warmup=1)["cuda_graph"]
    t2.step_eager(*batches[0])
    lrs, worst = [], 0.0
    for epoch in range(start, num_epochs):
        lrs.append(s1.lr)
        la, lb = [], []
        for r, (x, y) in enumerate(batches):
            la.append(t1.step(x, y).item())
            if r < REPLAYS - 1:
                lb.append(t2.step_eager(x, y).item())
            else:
                loss, err = _step_against_restatement(t2, x, y, _f32(s2.lr), opt)
                lb.append(loss.item())
                worst = max(worst, err)
        assert la == lb, (epoch, la, lb)
        s1.step(epoch + 1)
        s2.step(epoch + 1)
        torch.cuda.synchronize()
        for t, s in ((t1, s1), (t2, s2)):
            assert t.hyper[0].item() == t.hyper_small[0].item() == _f32(s.lr), (epoch, s.lr)
        for get in ("master_state", "ema_state"):
            a, b = getattr(t1, get)(), getattr(t2, get)()
            assert not [n for n in a if not torch.equal(a[n], b[n])], (epoch, get)
        oa, ob = t1.optimizer_state(), t2.optimizer_state()
        assert not [(n, k) for n in oa for k in oa[n] if not torch.equal(oa[n][k], ob[n][k])], epoch
        assert torch.equal(t1.Pb, t2.Pb)
    # warm-up 1e-4 .. , noisy cosine on epochs 3-5, min_lr for the cooldown epochs 6 and 7
    assert lrs[0] == solver["warmup_lr"] and lrs[6] == lrs[7] == solver["min_lr"] and len(set(lrs)) == 7, lrs
    print(opt, "LRs", ["%.4g" % v for v in lrs], "largest error / max|ref| %.2e" % worst)
