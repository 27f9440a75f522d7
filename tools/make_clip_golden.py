"""Generate tests/golden/clip.npz from the reference's OWN gradient clipping.  TEST INFRASTRUCTURE ONLY.

Run where the reference tree exists (oracle/ref_import.py finds it):   python tools/make_clip_golden.py

utils/clip_grad.py is loaded by file; models/helpers.py:model_parameters through the reference package.  On the toy module of
tests/clip_ref.py (clip_ref.Toy) with seeded fp32 parameters and gradients, stored as `p_<i>` / `g_<i>` in
model.parameters() order:
* head: the indices of model.parameters() that model_parameters(model, exclude_head=True) keeps;
* out_<mode>_<bind|free>_<i>: the gradients after train.py:270-273 (dispatch_clip_grad on model_parameters(model,
  exclude_head='agc' in mode)), with a clip value that binds (about half of the agc units, the norm, about half of the elements)
  and one that does not (1e30); value_<mode>_<bind|free> the value used;
* norm_<bind|free>: what clip_grad_norm_ returns on the same gradients.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import clip_ref  # noqa: E402
from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "clip.npz")
SEED = 2718


def _clip_module():
    spec = importlib.util.spec_from_file_location("ref_clip_grad", os.path.join(ref_import.REF, "utils", "clip_grad.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def inputs(seed=SEED):
    """Seeded parameters (a spread of unit scales) and gradients of clip_ref.Toy, fp32, in model.parameters() order."""
    torch.manual_seed(seed)
    m = clip_ref.Toy()
    g0 = torch.Generator().manual_seed(seed)
    ps, gs = [], []
    for p in m.parameters():
        rows = p.shape[0] if p.dim() > 1 else 1
        scale = torch.exp(torch.randn(rows, generator=g0)).view(-1, *([1] * (p.dim() - 1))) if p.dim() > 1 else torch.exp(torch.randn(1, generator=g0))
        ps.append((torch.randn(p.shape, generator=g0) * scale * 0.1).float())
        gs.append((torch.randn(p.shape, generator=g0) * torch.exp(torch.randn(rows, generator=g0)).view(scale.shape) * 0.01).float())
    return m, ps, gs


def _clip_values(m, ps, gs):
    """Binding values: midway between the two middle agc unit ratios ||g_u|| / max(||p_u||, 1e-3), half the total norm, the
    median |g|."""
    head = clip_ref.model_parameters(m, exclude_head=True)
    ids = [id(p) for p in m.parameters()]
    ratios = []
    for p in head:
        i = ids.index(id(p))
        ratios.append((clip_ref.unitwise_norm(gs[i].double()) / clip_ref.unitwise_norm(ps[i].double()).clamp(min=1e-3)).reshape(-1))
    r = torch.cat(ratios).sort().values
    k = len(r) // 2
    agc = float((r[k - 1] + r[k]) / 2)
    total = float(torch.linalg.vector_norm(torch.cat([g.double().reshape(-1) for g in gs])))
    val = float(torch.cat([g.abs().reshape(-1) for g in gs]).median())
    return {"norm": 0.5 * total, "value": val, "agc": agc}


def main():
    ref_import.load()
    import models.helpers as ref_helpers                       # noqa: E402  (the reference package is on sys.path now)
    cg = _clip_module()
    m, ps, gs = inputs()
    rec = {}
    for i, (p, g) in enumerate(zip(ps, gs)):
        rec["p_%d" % i], rec["g_%d" % i] = p.numpy(), g.numpy()
    params = list(m.parameters())
    kept = ref_helpers.model_parameters(m, exclude_head=True)
    rec["head"] = np.array([[id(q) for q in params].index(id(p)) for p in kept], dtype=np.int64)
    rec["names"] = np.array([n for n, _ in m.named_parameters()])
    binding = _clip_values(m, ps, gs)
    for mode in clip_ref.MODES:
        for tag, value in (("bind", binding[mode]), ("free", 1e30)):
            with torch.no_grad():
                for p, pv, gv in zip(params, ps, gs):
                    p.copy_(pv)
                    p.grad = gv.clone()
            cg.dispatch_clip_grad(ref_helpers.model_parameters(m, exclude_head="agc" in mode), value=value, mode=mode)
            rec["value_%s_%s" % (mode, tag)] = np.float64(value)
            for i, p in enumerate(params):
                rec["out_%s_%s_%d" % (mode, tag, i)] = p.grad.numpy().copy()
            if mode == "norm":
                for p, gv in zip(params, gs):
                    p.grad = gv.clone()
                rec["norm_%s" % tag] = np.float64(torch.nn.utils.clip_grad_norm_(params, value).item())
    bound = [int((rec["out_agc_bind_%d" % i] != rec["g_%d" % i]).any()) for i in range(len(params))]
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, "%d bytes" % os.path.getsize(OUT), "agc-clipped parameters", bound, "values", binding)


if __name__ == "__main__":
    main()
