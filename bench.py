#!/usr/bin/env python
"""bench.py -- headline benchmark of the CoT-block hot path (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W]                (N>1: launched by torch.distributed.run)
    python bench.py --impl reference [--gpus N] [--steps K] [--warmup W]

Workload (config.workload): CoTNet-50, 224x224, batch 256 per GPU, fwd + bwd + SGD-nesterov step, bf16 autocast
over fp32 master weights, channels_last, synthetic ImageNet-shaped data -- BASELINE.json configs[1].
A "step" is one pass of that over one synthetic batch.  The CoT layers (16 per step) run on the sm_90a kernels
of libcotb200.so through the reference's operator API; the rest of the backbone is stock PyTorch (north_star:
"host code stays PyTorch").

One JSON line on stdout (rank 0):
  value          images/s, whole job, inputs already resident in HBM when the timed region starts
  e2e            same metric through the public API with HOST buffers: pinned uint8 batch -> device -> step -> loss
                 read back, every step inside the timed region
  roofline       the dominant libcotb200 kernel of the step: algorithmic bytes / CUDA-event time vs measured HBM peak
  cpu_baseline   the oracle's CPU restatement of the reference model timed on this box's host cores (bounded sample)
  clocks         nvidia-smi SM clocks / throttle reasons sampled during the timed region

--dump-outputs DIR writes, after the timed steps, what the last timed step left its caller as DIR/<name>.npy (float32):
the loss, and the fp32 master weights, momentum and EMA of the flat optimizer state (a fixed, seeded sample of
DUMP_SAMPLE positions of each).  Inputs and initial weights are seeded, so two builds can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

IMAGENET_MEAN = (0.485 * 255, 0.456 * 255, 0.406 * 255)
IMAGENET_STD = (0.229 * 255, 0.224 * 255, 0.225 * 255)


PRETTY = {"cotnet50": "CoTNet-50", "cotnext50_2x48d": "CoTNeXt-50", "cotnet101": "CoTNet-101",
          "cotnext101_2x48d": "CoTNeXt-101", "se_cotnetd_50": "SE-CoTNetD-50", "se_cotnetd_101": "SE-CoTNetD-101",
          "se_cotnetd_152": "SE-CoTNetD-152"}


def metric_name(model, res, batch, fwd_only=False):
    """ONE metric string for both arms (the driver divides lines whose `metric` matches exactly).  The CPU arm times a
    bounded sample of this workload and says so in its `config` / `cpu_baseline.sample`."""
    return "%s images/sec (%s, %d^2, bs%d/GPU)" % (PRETTY.get(model, model), "fwd" if fwd_only else "fwd+bwd", res, batch)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--model", default="cotnet50")
    ap.add_argument("--batch", type=int, default=256, help="images per GPU")
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--fwd-only", action="store_true", help="diagnostic: time the forward pass only (not the headline)")
    ap.add_argument("--graph", default="auto", choices=["auto", "on", "off"], help="replay the whole step from a CUDA graph")
    ap.add_argument("--weights", default="bf16", choices=["bf16", "fp32"],
                    help="bf16: >=2-D weights kept as a bf16 copy written by the optimizer kernel (fp32 master in the flat state); "
                         "fp32: parameters are the fp32 masters and autocast casts them every step")
    ap.add_argument("--bucket", default="auto", choices=["auto", "bf16", "fp32"], help="dtype of the all-reduced gradient bucket")
    ap.add_argument("--chunks", type=int, default=3, help="N>1: ranges of the gradient bucket all-reduced separately (overlap)")
    ap.add_argument("--no-overlap", action="store_true", help="N>1: one all-reduce after backward instead of chunked overlap")
    ap.add_argument("--no-nccl-capture", action="store_true", help="N>1: keep NCCL out of the CUDA graph (two graphs + eager collectives)")
    ap.add_argument("--no-ema", action="store_true", help="skip the EMA of the weights (the reference's configs enable it)")
    ap.add_argument("--no-cot-leg", action="store_true", help="skip the CoT-layers-only forward measurement")
    ap.add_argument("--exposed-comm", action="store_true", default=False,
                    help="N>1: also capture the step WITHOUT collectives and report the exposed communication time (a second graph "
                         "capture next to the NCCL-carrying one; off by default: the second capture can invalidate the first, after "
                         "which the ranks hang in the process-group teardown)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the outputs of the last timed step as DIR/<name>.npy")
    return ap.parse_args()


# ----------------------------------------------------------------------------------------------- clocks
class ClockSampler:
    """Samples nvidia-smi during the timed region (the 'clocks' entry of the JSON line)."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            f = [c.strip() for c in r.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx.append(float(f[1]))
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons)}


# ----------------------------------------------------------------------------------------------- algorithmic bytes
def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            d = json.load(open(p))
            return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
        except Exception:
            pass
    return 3350.0, "fallback (H100 SXM data sheet)"


# ----------------------------------------------------------------------------------------------- CPU baseline / reference arm
def usable_cores():
    """Host cores this process may actually run on: cpu_count capped by the affinity mask and the cgroup CPU quota
    (a container that sees 128 CPUs but is throttled to a fraction of them collapses with 128 OpenMP threads)."""
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:
        pass
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = min(n, max(1, int(float(quota) / float(period) + 0.5)))
    except Exception:
        pass
    return max(1, n)


def pick_cpu_threads(model, res):
    """Thread count for the CPU arm: the fastest of {all usable cores, 1/2, 1/4, 16} on one bs2 forward of the model
    (torchrun exports OMP_NUM_THREADS=1 and oversubscribed boxes get SLOWER with more threads, so neither the
    environment nor cpu_count can be trusted).  Returns (threads, {threads: seconds})."""
    top = usable_cores()
    cands = sorted({c for c in (top, top // 2, top // 4, 16) if 1 <= c <= top}, reverse=True)
    x = torch.randn(2, 3, res, res)
    timing = {}
    with torch.no_grad():
        for c in cands:
            torch.set_num_threads(c)
            model(x)                                   # thread-pool spin-up
            t0 = time.perf_counter()
            model(x)
            timing[c] = round(time.perf_counter() - t0, 3)
    best = min(timing, key=timing.get)
    torch.set_num_threads(best)
    return best, timing


CPU_THREADS = {"n": None, "timing": None}


def cpu_step_fn(model_name, res, sample_batch, seed=0):
    """One fwd+bwd+SGD step of the oracle's CPU restatement of the reference model (fp32, host threads chosen by
    pick_cpu_threads)."""
    from oracle import cot_model_ref
    torch.manual_seed(seed)
    m = cot_model_ref.build(model_name).train()
    CPU_THREADS["n"], CPU_THREADS["timing"] = pick_cpu_threads(m, res)
    opt = torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-4)
    x = torch.randn(sample_batch, 3, res, res)
    y = torch.randint(0, 1000, (sample_batch,))

    def step():
        opt.zero_grad(set_to_none=True)
        loss = torch.nn.functional.cross_entropy(m(x), y)
        loss.backward()
        opt.step()
        return float(loss.detach())
    return step


def run_cpu_baseline(model_name, res, sample_batch=8):
    step = cpu_step_fn(model_name, res, sample_batch)
    t0 = time.perf_counter()
    step()                                  # warm-up (allocator, thread pool)
    warm = time.perf_counter() - t0
    n = 1 if warm > 12 else 2
    t0 = time.perf_counter()
    for _ in range(n):
        step()
    dt = (time.perf_counter() - t0) / n
    return {"value": sample_batch / dt, "unit": "images/s", "cores": CPU_THREADS["n"], "kind": "port",
            "sample": "oracle CPU restatement of %s (fp32, Unfold LocalConv), fwd+bwd+SGD on %d images %dx%d, "
                      "1 warm-up + mean of %d; %d threads (host reports %d CPUs, %d usable; bs2-forward seconds per "
                      "thread count: %s)" % (model_name, sample_batch, res, res, n, CPU_THREADS["n"], os.cpu_count() or 1,
                                             usable_cores(), CPU_THREADS["timing"])}


def main_reference(a):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    sample = 8
    step = cpu_step_fn(a.model, a.res, sample)
    for _ in range(a.warmup):
        step()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        step()
    dt = time.perf_counter() - t0
    v = sample * a.steps / dt
    cb = {"value": v, "unit": "images/s", "cores": CPU_THREADS["n"], "kind": "port",
          "sample": "oracle CPU restatement of the reference %s (fp32), fwd+bwd+SGD, %d images %dx%d per step; %d threads "
                    "(host reports %d CPUs, %d usable; bs2-forward seconds per thread count: %s)"
                    % (a.model, sample, a.res, a.res, CPU_THREADS["n"], os.cpu_count() or 1, usable_cores(),
                       CPU_THREADS["timing"])}
    print(json.dumps({
        "impl": "reference", "metric": metric_name(a.model, a.res, a.batch), "value": v, "unit": "images/s",
        "n_gpus": a.gpus, "steps": a.steps, "warmup": a.warmup, "ms_per_step": 1e3 * dt / a.steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "%s %dx%d fwd+bwd+SGD on host CPU cores, %d images/step (bounded sample of the bs%d workload)"
                   % (a.model, a.res, a.res, sample, a.batch)},
        "cpu_baseline": cb,
        "e2e": {"value": v, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0}))
    return 0


# ----------------------------------------------------------------------------------------------- our arm
def _train_backend():
    from cotnet_b200.cot_layer import CotLayer
    return CotLayer.train_conv_backend


def build_model(name, **kw):
    from cotnet_b200 import backbone, backbone_hybrid
    ctor = backbone.MODELS.get(name) or backbone_hybrid.MODELS.get(name)
    if ctor is None:
        raise SystemExit("bench.py: unknown model %r (have: %s)" % (name, sorted(list(backbone.MODELS) + list(backbone_hybrid.MODELS))))
    return ctor(**kw)


def peaks_all():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        d = json.load(open(p))
        return float(d["hbm_gbs"]), float(d["bf16_tflops"]), float(d.get("bf16_tflops_sustained", d["bf16_tflops"])), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return 3350.0, 989.0, 989.0, "fallback (H100 SXM data sheet: dense BF16, HBM3)"


def cot_forward_leg(model, x, steps):
    """Eval-mode bf16 forward with CUDA events around every CoT layer: the north-star number "CoT layers forward as a
    fraction of the CoT-block roofline" (SURVEY 8d), measured inside the real model (inputs = real activations, every
    layer's working set >> L2 at bs256)."""
    from cotnet_b200.cot_layer import CotLayer, CoXtLayer
    layers = [(n, m) for n, m in model.named_modules() if isinstance(m, (CotLayer, CoXtLayer))]
    ev = {n: [] for n, _ in layers}
    hooks = []
    for n, m in layers:
        def pre(mod, inp, n=n):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev[n].append([e, None])

        def post(mod, inp, out, n=n):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev[n][-1][1] = e
        hooks.append(m.register_forward_pre_hook(pre))
        hooks.append(m.register_forward_hook(post))
    was = model.training
    model.eval()
    xb = x.to(torch.bfloat16)
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            for _ in range(3):
                model(xb)
            for v in ev.values():
                v.clear()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                model(xb)
            e1.record()
            torch.cuda.synchronize()
    finally:
        for h in hooks:
            h.remove()
        model.train(was)
    per = {n: sum(a.elapsed_time(b) for a, b in v) / max(1, len(v)) for n, v in ev.items()}
    return per, e0.elapsed_time(e1) / steps


DUMP_SAMPLE = 1 << 20


def dump_outputs(d, arrays):
    """Each tensor of `arrays` as d/<name>.npy in float32; tensors of more than DUMP_SAMPLE elements as the values at DUMP_SAMPLE
    positions drawn by a fixed seed (the same positions for the same size), which keeps a dump under 64 MB."""
    import numpy as np
    os.makedirs(d, exist_ok=True)
    for name, t in arrays.items():
        flat = t.detach().reshape(-1)
        if flat.numel() > DUMP_SAMPLE:
            idx = torch.randint(0, flat.numel(), (DUMP_SAMPLE,), generator=torch.Generator().manual_seed(flat.numel()))
            flat = flat[idx.to(flat.device)]
        np.save(os.path.join(d, name + ".npy"), flat.float().cpu().numpy())


def main_ours(a):
    from cotnet_b200 import _lib, roofline, trainer
    from cotnet_b200 import dist as cdist
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the product path has no CPU fallback")
    # keep stdout = the one JSON line: NCCL writes its banner ("NCCL version ...") to stdout when NCCL_DEBUG=VERSION
    os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
    if os.environ.get("NCCL_DEBUG", "").upper() in ("VERSION",):
        os.environ["NCCL_DEBUG"] = "WARN"
    rank, local_rank, world = cdist.init_from_env()
    if world != a.gpus and world > 1:
        a.gpus = world
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    _lib.load()
    # the same arguments must compute the same step every run: cuDNN picks its algorithms by heuristics (autotuning by timing can
    # pick a different algorithm, i.e. a different summation order, from run to run) and only deterministic ones
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    torch.manual_seed(1234 + rank)

    B, R = a.batch, a.res
    model = build_model(a.model, zero_init_last_bn=False).to(dev).to(memory_format=torch.channels_last).train()
    if world > 1:
        cdist.broadcast_module_(model, 0)
    # One data-parallel training step = cotnet_b200.trainer.TrainStep (reference: train.py:255-277 + DDP): fp32 master
    # weights / momentum / EMA in flat buffers, bf16 weight copy for the convolutions, gradients gathered into one bucket,
    # NCCL all-reduce overlapped with backward, ONE optimizer(+EMA) kernel; the whole step replays from one CUDA graph.
    ts = trainer.TrainStep(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True,
                           ema_decay=None if a.no_ema else 0.9999, weights=a.weights,
                           bucket_dtype={"bf16": torch.bfloat16, "fp32": torch.float32, "auto": None}[a.bucket],
                           comm_chunks=a.chunks, overlap=not a.no_overlap)
    gen = torch.Generator().manual_seed(1234 + rank)
    host_u8 = torch.randint(0, 256, (B, 3, R, R), generator=gen, dtype=torch.uint8).pin_memory()
    host_lab = torch.randint(0, 1000, (B,), generator=gen, dtype=torch.int64).pin_memory()

    def to_device_batch():
        """pinned uint8 NCHW host batch -> device -> ONE kernel: (x - mean)/std, bf16, channels_last (datasets/loader.py:86-90)"""
        u8 = host_u8.to(dev, non_blocking=True)
        lab = host_lab.to(dev, non_blocking=True)
        return trainer.normalize_u8(u8, IMAGENET_MEAN, IMAGENET_STD, torch.bfloat16), lab

    x_res, lab_res = to_device_batch()           # resident inputs for `value`
    torch.cuda.synchronize()

    if a.fwd_only:
        # diagnostic leg (not the headline): eval-mode bf16 forward of the whole model, no autograd
        model.eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            for _ in range(max(a.warmup, 3)):
                model(x_res)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                logits = model(x_res)
            e1.record()
            torch.cuda.synchronize()
        ms = cdist.max_over_ranks(e0.elapsed_time(e1), dev)
        if a.dump_outputs and rank == 0:
            dump_outputs(a.dump_outputs, {"logits": logits})
        graph_info = {"cuda_graph": False}
        launches, clk, e2e = 0, None, None
        model.train()
    else:
        graph_info = {"cuda_graph": False}
        if a.graph != "off":
            try:
                graph_info = ts.capture(x_res, lab_res, warmup=3, capture_nccl=not a.no_nccl_capture)
            except Exception as e:      # noqa: BLE001 -- never lose the bench line to a capture problem
                graph_info = {"cuda_graph": False, "cuda_graph_error": repr(e)[:300]}
                torch.cuda.synchronize()
        if ts._graph is not None:
            x_res, lab_res = ts.static_inputs        # the graph's static input buffers ARE the resident inputs

        def timed(fn, steps):
            cdist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            cdist.barrier()
            return cdist.max_over_ranks(e0.elapsed_time(e1), dev)

        # ---- value: resident inputs
        for _ in range(max(a.warmup, 3)):
            ts.step(x_res, lab_res)
        clocks = ClockSampler(local_rank)
        if rank == 0:
            clocks.start()
        l0 = _lib.launch_count()
        last = {}

        def timed_step():
            last["loss"] = ts.step(x_res, lab_res)
        ms = timed(timed_step, a.steps)
        launches = _lib.launch_count() - l0
        if a.dump_outputs and rank == 0:
            dump_outputs(a.dump_outputs, dict({"loss": last["loss"]},
                                              **{n: getattr(ts, n) for n in ("P_big", "P_small", "M_big", "M_small", "E_big", "E_small")
                                                 if getattr(ts, n, None) is not None}))
        if ts._graph is not None:      # replayed launches do not pass through the host-side counter: kernels captured x replays
            launches = graph_info.get("libcotb200_kernels_per_replay", 0) * a.steps
        clk = clocks.stop() if rank == 0 else None

        # ---- e2e: host buffers, H2D + normalise + step + loss read back every step
        e2e = None
        if not a.no_e2e:
            def e2e_step():
                x, lab = to_device_batch()
                return float(ts.step(x, lab).item())
            for _ in range(2):
                e2e_step()
            ms_e = timed(e2e_step, a.steps)
            e2e = {"value": world * B * a.steps / (ms_e / 1e3), "unit": "images/s",
                   "h2d_bytes_per_step": host_u8.numel() + host_lab.numel() * 8, "d2h_bytes_per_step": 4,
                   "ms_per_step": ms_e / a.steps}
    value = world * B * a.steps / (ms / 1e3)

    # ---- roofline 1: per-kernel CUDA-event times of OUR kernels over 2 eager steps of the same workload
    hbm, tf_burst, tf_sust, src = peaks_all()
    roof = None
    extra = {}
    if not a.fwd_only:
        _lib.prof_enable(True)            # eager (not graph-replayed) steps: the per-launch events are recorded by the library
        for _ in range(2):
            ts.step_eager(x_res, lab_res)
        torch.cuda.synchronize()
        prof = _lib.prof_report()
        _lib.prof_enable(False)
        if prof and rank == 0:
            cand = {k: v for k, v in prof.items() if v[2] > 0}
            kname, (cnt, tot_ms, tot_bytes) = max(cand.items(), key=lambda kv: kv[1][1])
            if tot_bytes > 0 and tot_ms > 0:
                ach = tot_bytes / (tot_ms / 1e3) / 1e9
                ours_ms = sum(v[1] for v in prof.values()) / 2
                w_frac = sum(v[2] for v in cand.values()) / 1e9 / (sum(v[1] for v in cand.values()) / 1e3) / hbm
                roof = {"bound": "hbm", "kernel": kname, "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm,
                        "peak_source": src, "launches_per_step": cnt // 2,
                        "avg_launch_us": 1e3 * tot_ms / cnt, "algorithmic_bytes_per_launch": tot_bytes / cnt,
                        "kernel_share_of_step": (tot_ms / 2) / (ms / a.steps),
                        "our_kernels_share_of_step": ours_ms / (ms / a.steps),
                        "our_kernels_time_weighted_frac": w_frac,
                        "all_kernels": {k: {"ms_per_step": round(v[1] / 2, 4), "launches_per_step": v[0] // 2,
                                            "GBps": round(v[2] / (v[1] / 1e3) / 1e9, 1) if v[1] > 0 and v[2] > 0 else None}
                                        for k, v in sorted(prof.items())}}
    # ---- roofline 2: whole step against the arithmetic-intensity roofline (SURVEY 8d), and the CoT layers alone (N = 1)
    if rank == 0:
        try:
            model.eval()
            with torch.autocast("cuda", dtype=torch.bfloat16):
                rows = roofline.layer_table(model, x_res[:2], s=2, batch=B)
            model.train()
            sr = roofline.step_roofline(rows, hbm, tf_sust)
            t_step = ms / a.steps
            extra["step_roofline"] = {
                "definition": "sum over layers of max(FLOPs / %.0f TF/s sustained, compulsory bytes / %.0f GB/s): every conv reads "
                              "input+weights once and writes its output once, a CoT block moves only its input and output, "
                              "norm/activation/pool/residual fused away; backward = 2x FLOPs, 2x bytes" % (tf_sust, hbm),
                "fwd_ms": sr["fwd_ms"], "fwd_bwd_ms": sr["fwd_bwd_ms"], "cot_layers_fwd_ms": sr["cot_fwd_ms"],
                "cot_layers_fwd_bwd_ms": sr["cot_fwd_bwd_ms"], "flops_fwd": sr["flops_fwd"],
                "frac": (sr["fwd_ms"] if a.fwd_only else sr["fwd_bwd_ms"]) / t_step, "measured_ms": t_step}
            if world == 1 and not a.no_cot_leg:
                per, fwd_ms = cot_forward_leg(model, x_res, 3)
                cot_ms = sum(per.values())
                rb = roofline.step_roofline([r for r in rows if r["kind"] == "cot"], hbm, tf_burst)
                extra["cot_forward"] = {"cot_layers_ms": cot_ms, "roofline_ms": rb["cot_fwd_ms"], "frac": rb["cot_fwd_ms"] / cot_ms,
                                        "model_forward_ms": fwd_ms, "layers": len(per), "mode": "eval, bf16, no_grad, eager, "
                                        "CUDA events around every CoT layer inside the model; roofline at burst peaks",
                                        "slowest_layer_ms": max(per.values()), "fastest_layer_ms": min(per.values())}
        except Exception as e:          # noqa: BLE001
            extra["step_roofline_error"] = repr(e)[:200]
    # ---- exposed communication: the same captured step without any collective (N > 1)
    if world > 1 and not a.fwd_only and a.exposed_comm:
        try:
            ms_nc = ts.time_without_comm(a.steps, timed)
            extra["comm"] = {"exposed_ms_per_step": ms / a.steps - ms_nc / a.steps, "ms_per_step_without_collectives": ms_nc / a.steps,
                             "bucket_MB": ts.G_big.numel() * ts.G_big.element_size() / 1e6, "bucket_dtype": str(ts.G_big.dtype),
                             "chunks": len(ts.plan["chunks"]), "overlap": ts.overlap}
        except Exception as e:          # noqa: BLE001
            extra["comm_error"] = repr(e)[:200]

    cpu = None
    if rank == 0 and world == 1 and not a.no_cpu_baseline:
        cpu = run_cpu_baseline(a.model, R)

    if rank == 0:
        line = {
            "metric": metric_name(a.model, R, B, a.fwd_only),
            "value": value, "unit": "images/s", "n_gpus": world, "steps": a.steps, "warmup": max(a.warmup, 3),
            "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16", "data": "synthetic",
            "config": {"workload": "%s %dx%d bs%d/GPU %s, bf16 compute over fp32 master weights, channels_last"
                                   % (a.model, R, R, B, "[FORWARD ONLY diagnostic, eval mode]" if a.fwd_only else
                                      "fwd+bwd+SGD-nesterov(+EMA %s)" % ("off" if a.no_ema else "0.9999")),
                       "global_batch": B * world, "parallelism": "dp%d" % world,
                       "l2": "per-step working set (activations, several GB) >> 50 MB L2; no explicit flush needed",
                       "step": "cotnet_b200.trainer.TrainStep: weights %s, gradient bucket %s, %d comm chunk(s), overlap %s"
                               % (a.weights, str(ts.G_big.dtype), len(ts.plan["chunks"]), ts.overlap),
                       "cot_path": "libcotb200 (train_conv_backend=%s): LocalConv fwd/dX/dW, GroupNorm(9 taps) fwd/bwd, bn+SiLU+pool+"
                                   "radix-2 recombination fwd/bwd (also SplitAttnConv2d's tail), fused BatchNorm(+ReLU,+residual), NHWC pooling, "
                                   "gradient fan-in; wgmma: the block's 1x1 convolutions (embed.0 concat-free two-pair GEMM, embed.3, conv1x1) "
                                   "fwd + dgrad + wgrad with BatchNorm statistics in the epilogue, key_embed 3x3 grouped conv on the haloed-tile "
                                   "kernel (dim <= 128), the bottleneck's 1x1 convolutions of stages 1-2, the 7x7 stem as a 4-tap implicit GEMM "
                                   "(+ its weight gradient); gradient gather + SGD/EMA/bf16-copy kernel, uint8->bf16 NHWC normalise; cuDNN: "
                                   "grouped 3x3 at 14x14 / 7x7 and its weight gradients, bottleneck 1x1 convolutions of stages 3-4, fc"
                                   % _train_backend()},
            "e2e": e2e, "gpu_launches": int(launches), "launch_mode": graph_info, "clocks": clk, "roofline": roof, "cpu_baseline": cpu,
        }
        line.update(extra)
        print(json.dumps(line), flush=True)
    if world > 1:
        # Every collective of this process is behind us (the timed region and the two profiled steps end with the gradient all-reduce;
        # the roofline legs of rank 0 launch no collective) and the JSON line is flushed.  Leave WITHOUT the process-group teardown and
        # without the interpreter's exit handlers: with NCCL kernels living inside a CUDA graph (and after a failed optional capture)
        # the communicator teardown can block both ranks for minutes.  torchrun sees exit code 0 from every rank.
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)
    return 0


if __name__ == "__main__":
    args = parse()
    sys.exit(main_reference(args) if args.impl == "reference" else main_ours(args))
