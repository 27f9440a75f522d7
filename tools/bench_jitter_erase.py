"""GPU time of the ColorJitter / vertical-flip kernel and of the random-erasing kernel per batch, beside the reference's way of
doing the same work.  Prints one JSON line per measurement with the GPU name and power limit beside the numbers.

    python tools/bench_jitter_erase.py [--batch 256] [--iters 50] [--cpu-images 64]

* jitter: cotb200_aug_color_jitter on a uint8 [B, 3, 224, 224] batch, every image with all four ops (random order, hue
  included) and a vertical flip on half of them; CUDA events around `iters` launches after warm-up.
* erase: cotb200_aug_erase on the normalised channels_last batch (fp32 and bf16) for each mode at reprob 0.25 and recount 1
  and 3 (the boxes drawn once, the device table uploaded once: kernel time); beside it, ref_loop: a torch restatement of the
  reference's RandomErasing loop (datasets/random_erasing.py: per image a Python draw, per box an allocation, normal_ and
  an indexed copy) on the same fp32 batch and device, host clock around `iters` calls ending in a synchronise.
* cpu_pil_jitter: torchvision ColorJitter((0.4, 0.4, 0.4, 0.1)) on 224 x 224 PIL images, one process, ms per image.
"""
import argparse
import json
import math
import os
import random
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cotnet_b200 import _lib, augment  # noqa: E402
from cotnet_b200.trainer import normalize_u8  # noqa: E402
from tools.bench_augment import gpu_info  # noqa: E402

MEAN = tuple(x * 255 for x in (0.485, 0.456, 0.406))
STD = tuple(x * 255 for x in (0.229, 0.224, 0.225))


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def ref_erase_loop(x, p, mode, count, rnd):
    """The reference's RandomErasing.__call__ on a [B, C, H, W] batch, restated with the same torch calls."""
    B, C, H, W = x.shape
    log_ar = (math.log(0.3), math.log(1 / 0.3))
    for i in range(B):
        if rnd.random() > p:
            continue
        n = 1 if count == 1 else rnd.randint(1, count)
        for _ in range(n):
            for _ in range(10):
                ta = rnd.uniform(0.02, 1 / 3) * H * W / n
                ar = math.exp(rnd.uniform(*log_ar))
                h, w = int(round(math.sqrt(ta * ar))), int(round(math.sqrt(ta / ar)))
                if w < W and h < H:
                    t, l = rnd.randint(0, H - h), rnd.randint(0, W - w)
                    if mode == "pixel":
                        v = torch.empty((C, h, w), dtype=x.dtype, device=x.device).normal_()
                    elif mode == "rand":
                        v = torch.empty((C, 1, 1), dtype=x.dtype, device=x.device).normal_()
                    else:
                        v = torch.zeros((C, 1, 1), dtype=x.dtype, device=x.device)
                    x[i][:, t:t + h, l:l + w] = v
                    break
    return x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-images", type=int, default=64)
    a = ap.parse_args()
    name, power = gpu_info()
    B, S = a.batch, 224
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    g = torch.Generator().manual_seed(0)
    u8 = torch.randint(0, 256, (B, 3, S, S), dtype=torch.uint8, generator=g).to(dev)
    # ---- ColorJitter + vflip
    r = np.random.RandomState(0)
    rec = np.zeros(B, augment.JITTER_DTYPE)
    for n in range(B):
        rec["vflip"][n] = n % 2
        rec["order"][n] = r.permutation(4)
        rec["factor"][n] = r.uniform(0.6, 1.4, 3)
        rec["hue"][n] = r.uniform(-0.1, 0.1)
    jdev = torch.from_numpy(rec.view(np.uint8).copy()).to(dev)
    out = u8.clone()
    st = _lib.stream_ptr(out)

    def jitter():
        _lib.check(lib.cotb200_aug_color_jitter(B, S, rec.ctypes.data, jdev.data_ptr(), out.data_ptr(), st), "aug_color_jitter")

    print(json.dumps(dict(what="jitter", batch=B, size=S, ops="b,c,s,h + vflip 0.5", gpu_ms_per_batch=timed(jitter, a.iters),
                          gpu=name, power_limit=power)), flush=True)
    # ---- random erasing
    for dtype in (torch.float32, torch.bfloat16):
        base = normalize_u8(u8, MEAN, STD, dtype=dtype)
        for mode in ("const", "rand", "pixel"):
            for count in (1, 3):
                er = augment.RandomErasing(0.25, mode, count, seed=1)
                params = er.params(B, S, S, dev)
                nboxes = int(params.header["n_boxes"])
                x = base.clone()
                ms = timed(lambda: er.apply(x, params), a.iters)
                line = dict(what="erase", dtype=str(dtype).replace("torch.", ""), mode=mode, reprob=0.25, recount=count, batch=B,
                            boxes=nboxes, gpu_ms_per_batch=ms, gpu=name, power_limit=power)
                if dtype == torch.float32:
                    xr = base.contiguous()                        # the reference erases its NCHW fp32 batch
                    rnd = random.Random(1)
                    for _ in range(3):
                        ref_erase_loop(xr, 0.25, mode, count, rnd)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(a.iters):
                        ref_erase_loop(xr, 0.25, mode, count, rnd)
                    torch.cuda.synchronize()
                    line["ref_loop_ms_per_batch"] = (time.perf_counter() - t0) * 1e3 / a.iters
                print(json.dumps(line), flush=True)
    # ---- Pillow ColorJitter on one core
    try:
        from PIL import Image
        from torchvision import transforms
        n = a.cpu_images
        imgs = [Image.fromarray(u8[k % B].permute(1, 2, 0).cpu().numpy()) for k in range(n)]
        cj = transforms.ColorJitter(0.4, 0.4, 0.4, 0.1)
        torch.set_num_threads(1)
        t0 = time.perf_counter()
        for im in imgs:
            np.asarray(cj(im))
        print(json.dumps(dict(what="cpu_pil_jitter", images=n, ms_per_image=(time.perf_counter() - t0) * 1e3 / n,
                              note="one process, torchvision ColorJitter((0.4, 0.4, 0.4, 0.1)) on 224 x 224 PIL images")), flush=True)
    except ImportError:
        print(json.dumps(dict(what="cpu_pil_jitter", note="Pillow / torchvision not installed: not measured")), flush=True)


if __name__ == "__main__":
    main()
