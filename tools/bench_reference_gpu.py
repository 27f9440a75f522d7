#!/usr/bin/env python
"""GPU REFERENCE ARM: the UNMODIFIED reference model (its eager module graph, its own NVRTC-style kernels for the LocalConv
op) timed on the same box as bench.py -- BASELINE.md section 4 rows 2-3, the honest "x over the reference on a H100".

    python tools/make_ref_snapshot.py                      # in the build container: baseline/_ref/ (git-ignored) <- reference packages
    python tools/bench_reference_gpu.py --model cotnet50 --batch 256 --amp bf16 [--steps 10] [--json out.json]

What runs: `models.cotnet.cotnet50()` etc. from baseline/_ref, NCHW like the reference trains, torch.optim.SGD(nesterov)
(optim/optim_factory.py:54-56), optional torch.autocast (the reference's `amp_autocast`, train.py:259).  Its LocalConv goes
through ITS `AggregationZeropad` Function and ITS kernel strings, compiled per shape exactly as `load_kernel` does, with
oracle/cupy_shim.py standing in for CuPy (nvcc instead of NVRTC, driver-API launch).  The reference op accepts only
fp32/fp64 tensors (cupy_layers/utils.py:8-12), so under autocast its inputs are cast to fp32 and the result back -- the
minimum a user has to do to run the reference under AMP.  None of libcotb200 is on this path.
"""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REFDIR = os.path.join(ROOT, "baseline", "_ref")

import torch  # noqa: E402


def load_reference():
    if not os.path.isdir(os.path.join(REFDIR, "cupy_layers")):
        raise SystemExit("bench_reference_gpu: baseline/_ref missing -- run tools/make_ref_snapshot.py where /root/reference exists")
    from oracle import cupy_shim
    cupy_shim.install()
    if "yacs" not in sys.modules:                        # config only (config/config.py:2), no arithmetic
        yacs, yc = types.ModuleType("yacs"), types.ModuleType("yacs.config")

        class CfgNode(dict):
            __getattr__ = dict.__getitem__
            __setattr__ = dict.__setitem__
        yc.CfgNode = CfgNode
        yacs.config = yc
        sys.modules["yacs"], sys.modules["yacs.config"] = yacs, yc
    sys.path.insert(0, REFDIR)
    import cupy_layers.aggregation_zeropad as agg
    import models.cotnet as mc
    import models.cotnet_hybrid as mh
    # AMP: the reference op takes fp32 / fp64 only
    inner = agg.aggregation_zeropad

    def amp_safe(input, weight, kernel_size=3, stride=1, padding=0, dilation=1):
        if input.dtype in (torch.float16, torch.bfloat16) or weight.dtype != input.dtype:
            return inner(input.float(), weight.float(), kernel_size, stride, padding, dilation).to(input.dtype)
        return inner(input, weight, kernel_size, stride, padding, dilation)
    agg.aggregation_zeropad = amp_safe
    return mc, mh


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--amp", default="bf16", choices=["fp32", "bf16"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--fwd-only", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    mc, mh = load_reference()
    ctor = getattr(mc, a.model, None) or getattr(mh, a.model)
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(1234)
    model = ctor().cuda().train()
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, nesterov=True, weight_decay=1e-4)
    x = torch.randn(a.batch, 3, a.res, a.res, device="cuda")
    y = torch.randint(0, 1000, (a.batch,), device="cuda")

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=a.amp == "bf16"):
            out = model(x)
            loss = torch.nn.functional.cross_entropy(out.float(), y)
        if not a.fwd_only:
            loss.backward()
            opt.step()
        return loss

    for _ in range(max(a.warmup, 3)):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    out = {"impl": "reference-gpu", "model": a.model, "batch": a.batch, "res": a.res, "amp": a.amp, "fwd_only": a.fwd_only,
           "ms_per_step": ms, "images_per_s": a.batch / (ms / 1e3), "loss": float(loss),
           "what": "unmodified reference model zoo + its own LocalConv kernels (compiled per shape by its load_kernel through "
                   "oracle/cupy_shim.py), eager, NCHW, torch SGD-nesterov; no libcotb200 code on this path",
           "gpu": torch.cuda.get_device_name(0), "max_mem_GB": torch.cuda.max_memory_allocated() / 1e9}
    print(json.dumps(out))
    if a.json:
        json.dump(out, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
