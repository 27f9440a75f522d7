"""Generate tests/golden/dropblock.npz from the reference's OWN DropBlock code.  TEST INFRASTRUCTURE ONLY.

Run where the reference tree exists (oracle/ref_import.py finds it):   python tools/make_dropblock_golden.py

``torch.rand_like`` is patched, call by call in forward order (site 0, 1, ...), to return the library's uniforms
(cotnet_b200/dropblock.py:uniforms) for a fixed key, and every drawn u is checked to fall on the same side of gamma in fp32 and
fp64 (the library compares in fp32, an fp64 reference in fp64).  Stored:
* geo_*: models/layers/drop.py:drop_block_fast_2d forward and backward on seeded fp32 tensors over many geometries (H, W from
  3 to 40, block sizes 1 / 3 / 5, counts of 0 and 1 included): the keep mask (from the reference's own pooled mask), its
  count, the scale (the output of an all-ones input), y and dx.
* sites_<model>_<res>: each DropBlock call of the reference model in forward order at a res x res input, batch 2:
  (block_size, gamma_scale, C, H, W).
* step_<model>_*: one fp64 training step of the reference's cotnet50 / se_cotnetd_50 with drop_block_rate 0.1 at 128 px under
  the protocol of tools/make_recipe_golden.py (parameters of make_golden.hybrid_seeded_state rounded to bf16, the bf16-rounded
  normalised step_batch, no mixing, label smoothing 0.1): the loss and every parameter gradient as norm + projection.
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cotnet_b200 import dropblock  # noqa: E402
from oracle import make_golden, ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "dropblock.npz")
KEY = (0x1234ABCD, 0x0F0E0D0C)

# (B, C, H, W, block_size, gamma_scale, rate, site, key): counts of 0 (rate 1 at a small plane) and 1 are searched below
GEOS = [(2, 8, 7, 7, 3, 1.0, 0.1, 0), (2, 16, 14, 14, 5, 0.25, 0.1, 1), (1, 8, 28, 28, 5, 0.25, 0.1, 2),
        (2, 8, 10, 20, 5, 0.25, 0.3, 3), (1, 16, 20, 10, 3, 1.0, 0.2, 4), (1, 8, 40, 40, 5, 0.25, 0.1, 5),
        (3, 8, 3, 3, 3, 1.0, 0.1, 6), (2, 8, 3, 5, 5, 0.25, 0.1, 7), (2, 8, 9, 4, 3, 1.0, 0.5, 8), (1, 24, 13, 17, 1, 1.0, 0.2, 9),
        (2, 8, 7, 7, 3, 1.0, 0.9, 10), (1, 8, 33, 40, 3, 1.0, 0.05, 11), (2, 8, 14, 14, 3, 1.0, 0.1, 12),
        (1, 8, 6, 6, 5, 0.25, 0.1, 13), (1, 8, 3, 3, 3, 1.0, 1.0, 14)]

MODELS = ("cotnet50", "cotnet101", "cotnext50_2x48d", "cotnext101_2x48d", "se_cotnetd_50", "se_cotnetd_101", "se_cotnetd_152")


def _drop_module():
    ref_import.load()
    return importlib.import_module("models.layers.drop")


class _Patch:
    """torch.rand_like -> the library's uniforms for KEY, site = the call's number; F.max_pool2d of the drop module recorded."""

    def __init__(self, drop, key=KEY, first_site=0):
        self.drop, self.key, self.site = drop, key, first_site
        self.pooled = []

    def __enter__(self):
        self.rand_like, self.fast = torch.rand_like, self.drop.drop_block_fast_2d
        self.F = self.drop.F
        patch = self

        def rand_like(x, *a, **k):
            u = dropblock.uniforms(tuple(x.shape), patch.site, patch.key)
            patch.last_u = u
            patch.site += 1
            return torch.from_numpy(u).to(x.dtype)

        def fast(x, drop_prob=0.1, block_size=7, gamma_scale=1.0, *a, **k):
            B, C, H, W = x.shape
            cbs = min(block_size, H, W)
            gamma = gamma_scale * drop_prob * H * W / cbs ** 2 / ((W - block_size + 1) * (H - block_size + 1))
            y = patch.fast(x, drop_prob, block_size, gamma_scale, *a, **k)
            u = patch.last_u
            assert np.array_equal(u < np.float32(gamma), u.astype(np.float64) < gamma), "fp32 / fp64 seed tests disagree"
            return y

        class _F:
            def __getattr__(self, n):
                return getattr(patch.F, n)

            @staticmethod
            def max_pool2d(*a, **k):
                out = patch.F.max_pool2d(*a, **k)
                patch.pooled.append(out.detach().clone())
                return out

        torch.rand_like = rand_like
        self.drop.drop_block_fast_2d = fast
        self.drop.F = _F()
        return self

    def __exit__(self, *a):
        torch.rand_like = self.rand_like
        self.drop.drop_block_fast_2d = self.fast
        self.drop.F = self.F


def _geo_case(drop, B, C, H, W, bs, gs, rate, site, key):
    g = torch.Generator().manual_seed(1000 + site)
    x = torch.randn(B, C, H, W, generator=g).requires_grad_(True)
    dy = torch.randn(B, C, H, W, generator=g)
    with _Patch(drop, key, site) as p:
        y = drop.drop_block_fast_2d(x, rate, bs, gs)
    y.backward(dy)
    keep = (1 - p.pooled[-1]).numpy() != 0
    with _Patch(drop, key, site):
        ones = drop.drop_block_fast_2d(torch.ones(B, C, H, W), rate, bs, gs).numpy()
    count = int(keep.sum())
    scale = ones[keep][0] if count else (keep.size / torch.tensor(0.0).add(1e-7)).item()
    assert np.array_equal(ones != 0, keep)
    return x.detach().numpy(), dy.numpy(), y.detach().numpy(), x.grad.numpy(), keep, count, np.float32(scale)


def _geos(drop):
    rec = {}
    cases = list(GEOS)
    # a count of 1: search a 3x3 plane with block size 3 for a key that keeps exactly one element
    for k in range(20000):
        key = (k, 77)
        try:
            keep, count, _ = dropblock.host_mask((1, 8, 3, 3), 20, key, dropblock.DropBlock(0.25, 3, 1.0))
        except ValueError:
            continue
        if count == 1:
            cases.append((1, 8, 3, 3, 3, 1.0, 0.25, 20, key))
            break
    else:
        raise RuntimeError("no key with a count of 1")
    cases = [c if len(c) == 9 else c + (KEY,) for c in cases]
    counts = []
    for i, (B, C, H, W, bs, gs, rate, site, key) in enumerate(cases):
        x, dy, y, dx, keep, count, scale = _geo_case(drop, B, C, H, W, bs, gs, rate, site, key)
        counts.append(count)
        rec["geo%d_x" % i], rec["geo%d_dy" % i], rec["geo%d_y" % i], rec["geo%d_dx" % i] = x, dy, y, dx
        rec["geo%d_keep" % i], rec["geo%d_count" % i], rec["geo%d_scale" % i] = keep, np.int64(count), scale
    rec["geo_params"] = np.array([[B, C, H, W, bs, gs, rate, site, key[0], key[1]] for (B, C, H, W, bs, gs, rate, site, key) in cases],
                                 dtype=np.float64)
    assert 0 in counts and 1 in counts, counts
    print("geometries", len(cases), "counts", counts)
    return rec


def _sites():
    ns = ref_import.load()
    drop = _drop_module()
    rec = {}
    fns = {"cotnet50": ns.cotnet50, "cotnet101": ns.cotnet101, "cotnext50_2x48d": ns.cotnext50_2x48d}
    import models.cotnet as ref_cotnet
    fns["cotnext101_2x48d"] = ref_cotnet.cotnext101_2x48d
    for n in ("se_cotnetd_50", "se_cotnetd_101", "se_cotnetd_152"):
        fns[n] = getattr(ns.hybrid, n)
    for name in MODELS:
        torch.manual_seed(0)
        m = fns[name](drop_block_rate=0.1).train()
        for res in (128, 224, 320):
            calls = []
            orig = drop.DropBlock2d.forward

            def fwd(self, x):
                calls.append((self.block_size, self.gamma_scale) + tuple(x.shape[1:]))
                return x
            drop.DropBlock2d.forward = fwd
            try:
                with torch.no_grad():
                    m(torch.randn(2, 3, res, res))
            finally:
                drop.DropBlock2d.forward = orig
            rec["sites_%s_%d" % (name, res)] = np.array(calls, dtype=np.float64)
        print(name, "sites", len(calls))
        del m
    return rec


STEP_SEED, STEP_B, STEP_RES, STEP_RATE, STEP_SMOOTHING = 3101, 8, 128, 0.1, 0.1
MEAN = (0.485 * 255, 0.456 * 255, 0.406 * 255)
STD = (0.229 * 255, 0.224 * 255, 0.225 * 255)


def step_input():
    """The normalised, bf16-rounded batch and labels of the step fixture (regenerated by the tests)."""
    from make_recipe_golden import step_batch
    u8, y = step_batch(STEP_SEED, STEP_B, STEP_RES)
    mean = torch.tensor(MEAN, dtype=torch.float32).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=torch.float32).view(1, 3, 1, 1)
    return u8.float().sub_(mean).div_(std).bfloat16(), y


def _step(name):
    ns = ref_import.load()
    drop = _drop_module()
    fn = ns.cotnet50 if name == "cotnet50" else ns.hybrid.se_cotnetd_50
    x, y = step_input()
    torch.manual_seed(0)
    m = make_golden.hybrid_seeded_state(fn(drop_block_rate=STEP_RATE), STEP_SEED)
    with torch.no_grad():
        for t in m.state_dict().values():
            if t.dtype.is_floating_point:
                t.copy_(t.bfloat16().float())
    m = m.double().train()
    with _Patch(drop) as p:
        logits = m(x.double())
    n_sites = p.site
    K = logits.shape[1]
    logp = torch.log_softmax(logits, dim=-1)
    loss = (-(1 - STEP_SMOOTHING) * logp.gather(1, y.view(-1, 1)).squeeze(1) - STEP_SMOOTHING * logp.mean(-1)).mean()
    loss.backward()
    dropped = sum(int((t != 0).sum()) for t in p.pooled)
    assert dropped > 0
    names, gn, gp = [], [], []
    for n, q in m.named_parameters():
        names.append(n)
        gn.append(q.grad.norm().item())
        gp.append((q.grad * make_golden.proj_vector(n, q.shape, STEP_SEED)).sum().item())
    print(name, "step loss", loss.item(), "sites", n_sites, "dropped", dropped, "K", K)
    pre = "step_%s_" % name
    return {pre + "loss": np.float64(loss.item()), pre + "names": np.array(names), pre + "gnorm": np.array(gn),
            pre + "gproj": np.array(gp), pre + "sites": np.int64(n_sites)}


def main():
    rec = {"key": np.array(KEY, dtype=np.int64), "step_seed": np.int64(STEP_SEED), "step_B": np.int64(STEP_B),
           "step_res": np.int64(STEP_RES), "step_rate": np.float64(STEP_RATE), "step_smoothing": np.float64(STEP_SMOOTHING)}
    rec.update(_geos(_drop_module()))
    rec.update(_sites())
    for name in ("cotnet50", "se_cotnetd_50"):
        rec.update(_step(name))
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
