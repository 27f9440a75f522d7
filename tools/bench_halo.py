#!/usr/bin/env python
"""3x3 grouped key convolution (key_embed.0, models/cotnet.py:44) per CoTNet-50 stage shape, bs256, bf16 NHWC: the haloed-tile
wgmma kernel (variants through COTB200_CONV_HALO / COTB200_HALO_MAXPX, one subprocess each) against the per-tap conv mode and
cuDNN's grouped convolution.  CUDA events, inputs rotated through > 126 MB."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
STAGES = [(64, 56), (128, 28), (256, 14), (512, 7)]


def child():
    import torch
    import torch.nn.functional as F
    from cotnet_b200 import tc
    torch.backends.cudnn.benchmark = True
    out = {}
    for C, H in STAGES:
        B = 256
        nset = max(2, int(300e6 // (B * H * H * C * 2)) + 1)
        xs = [torch.randn(B, C, H, H, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last) for _ in range(nset)]
        w = (torch.randn(C, C // 4, 3, 3, device="cuda") / 10).bfloat16()
        wp, bn = tc.prepare_conv3x3_weight(w, 4)
        scale, shift = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
        cs, cq = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
        o = torch.empty_like(xs[0])
        wcl = w.contiguous(memory_format=torch.channels_last)

        def t(fn, iters=20):
            for i in range(3):
                fn(xs[i % nset])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(iters):
                fn(xs[i % nset])
            e1.record()
            torch.cuda.synchronize()
            return round(e0.elapsed_time(e1) / iters * 1e3, 1)
        out["C%d" % C] = {"tc_eval_us": t(lambda x: tc.conv3x3_bf16(x, wp, bn, scale=scale, shift=shift, relu=True, out=o)),
                          "tc_stats_us": t(lambda x: tc.conv3x3_bf16(x, wp, bn, stats=(cs, cq), out=o)),
                          "cudnn_us": t(lambda x: F.conv2d(x, wcl, None, 1, 1, 1, 4)),
                          "roof_us": round(2 * B * H * H * C * 2 / 6485.2e3, 1)}
    print("RESULT " + json.dumps(out), flush=True)


def main():
    if os.environ.get("BENCH_HALO_CHILD"):
        return child()
    res = {}
    for name, env in (("halo_256", {"COTB200_CONV_HALO": "1", "COTB200_HALO_MAXPX": "256"}),
                      ("halo_128", {"COTB200_CONV_HALO": "1", "COTB200_HALO_MAXPX": "128"}),
                      ("per_tap", {"COTB200_CONV_HALO": "0"})):
        e = dict(os.environ, BENCH_HALO_CHILD="1", **env)
        r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=e, capture_output=True, text=True, timeout=600)
        line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
        res[name] = json.loads(line[-1][7:]) if line else {"error": (r.stderr or r.stdout)[-400:]}
        print(name, json.dumps(res[name]), flush=True)
    if len(sys.argv) > 1:
        json.dump(res, open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
