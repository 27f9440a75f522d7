"""Cost of the update rules (solver.opt) on the library's training step.  Prints one JSON line.

    python tools/bench_optim.py [--model cotnet50] [--batch 256] [--res 224] [--steps 20] [--rounds 3] [--iters 50]

* passes: each rule's optimizer pass over the big bucket at the model's real flat size (plan_flat), bf16 gradients, EMA and the
  bf16 shadow, timed with CUDA events over --iters back-to-back launches (the per-step prepare launch included for the rules that
  have one and for Lookahead, as TrainStep launches them); GB/s from the byte model per element: P r/w 8, G 2, E r/w 8, Pb 2,
  plus 8 per fp32 state buffer (M, V), plus 8 for a Lookahead synchronisation step (S r/w).  SGD = 28 B, the Adam family /
  RMSprop with momentum / Adadelta = 36 B.
* graph: the TrainStep graph step time (bench.py's workload: bf16 weights, autocast, channels_last, cuDNN deterministic) for
  sgd, adamw, rmsproptf and lookahead_sgd, alternating within each of --rounds rounds in one process.
* the GPU name and power limit next to the numbers.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_recipe import gpu_info, timed  # noqa: E402
from cotnet_b200 import _lib, backbone, trainer  # noqa: E402

PASS_RULES = ("sgd", "adam", "adamw", "nadam", "radam", "adadelta", "rmsprop", "rmsproptf")
GRAPH_OPTS = ("sgd", "adamw", "rmsproptf", "lookahead_sgd")


def bench_passes(a, n):
    lib, dev = _lib.load(), torch.device("cuda")
    st = torch.cuda.current_stream().cuda_stream
    f32 = dict(dtype=torch.float32, device=dev)
    P, M, V, S, E = (torch.rand(n, **f32) for _ in range(5))
    V += 0.1
    G = (torch.randn(n, device=dev) * 1e-3).to(torch.bfloat16)
    Pb = torch.empty(n, dtype=torch.bfloat16, device=dev)
    hyper = torch.tensor([1e-4, 0.9, 1e-4, 0.9999, 1.0], **f32)
    out = {}

    def record(name, fn, per_elem):
        for _ in range(3):
            fn()
        ms = timed(fn, a.iters)
        out[name] = {"ms": ms, "bytes_per_elem": per_elem, "GB_per_s": n * per_elem / 1e9 / (ms / 1e3)}

    for name in PASS_RULES + ("lookahead_adamw sync step",):
        base, rule, la = trainer.parse_opt(name.split(" ")[0])
        state = torch.frombuffer(bytearray(bytes(_lib.OptState(m_schedule=1.0, slow_init=1))), dtype=torch.uint8).to(dev)
        o = _lib.Opt(rule=rule, eps=1e-8, lookahead_k=1 if la else 0, lookahead_alpha=0.5, M=M.data_ptr(),
                     V=V.data_ptr() if base not in ("sgd",) else None, S=S.data_ptr(), state=state.data_ptr())

        def run(o=o, prepare=base not in ("sgd", "momentum") or la):
            if prepare:                                   # as TrainStep: plain SGD has no per-step scalar
                lib.cotb200_opt_prepare(ctypes.byref(o), hyper.data_ptr(), 1, st)
            lib.cotb200_opt_step(n, P.data_ptr(), _lib.BF16, G.data_ptr(), E.data_ptr(), Pb.data_ptr(), hyper.data_ptr(), ctypes.byref(o),
                                 None, st)
        per = 28 + (8 if base != "sgd" else 0) + (8 if la else 0)
        record(name + ("" if la else " (cotb200_opt_step)"), run, per)
        P.copy_(torch.rand(n, **f32))                     # keep the weights finite and away from the previous rule's fixed point
    return out


def one_round(a, opt, x, lab):
    torch.manual_seed(1234)
    model = backbone.MODELS[a.model](zero_init_last_bn=False).cuda().to(memory_format=torch.channels_last).train()
    ts = trainer.TrainStep(model, lr=0.05 if opt in ("sgd", "lookahead_sgd") else 1e-3, momentum=0.9, weight_decay=1e-4,
                           ema_decay=0.9999, weights="bf16", opt=opt)
    ts.capture(x, lab, warmup=3)
    for _ in range(3):
        ts.step()
    ms = timed(ts.step, a.steps)
    n_big = ts.plan["n_big"]
    del ts, model
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms, n_big


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim.py: no CUDA device")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    plan = trainer.plan_flat(list(backbone.MODELS[a.model](zero_init_last_bn=False).named_parameters()))
    passes = bench_passes(a, plan["n_big"])
    gen = torch.Generator().manual_seed(1234)
    x = torch.randn(a.batch, 3, a.res, a.res, generator=gen).to(torch.bfloat16).cuda().contiguous(memory_format=torch.channels_last)
    lab = torch.randint(0, 1000, (a.batch,), generator=gen).cuda()
    times = {o: [] for o in GRAPH_OPTS}
    for _ in range(a.rounds):
        for o in GRAPH_OPTS:
            times[o].append(one_round(a, o, x, lab)[0])
    name, limit = gpu_info()
    best = {k: min(v) for k, v in times.items()}
    print(json.dumps({"model": a.model, "batch": a.batch, "res": a.res, "gpu": name, "power_limit": limit, "n_big": plan["n_big"],
                      "n_small": plan["n_small"], "passes_big_bucket": passes, "graph_ms_per_step": times, "best_ms_per_step": best,
                      "overhead_pct": {k: 100.0 * (v - best["sgd"]) / best["sgd"] for k, v in best.items() if k != "sgd"}}))


if __name__ == "__main__":
    main()
