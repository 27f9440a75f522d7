"""Stored outputs of the reference's own LocalConv kernels, so that the parity tests against them run without the reference.
TEST INFRASTRUCTURE ONLY.

`python -m oracle.ref_golden` (on a GPU, with oracle/_ref built by oracle/build_ref_kernels.py) launches the reference kernels on
the seeded inputs of every case of tests/test_ref_kernels_gpu.py and tests/test_variants_gpu.py and stores, per output array, its
values at 1024 seeded positions (half of them on the spatial border, where
padding bugs live) in tests/golden/ref_kernels.npz, together with the kernel geometries those cases use.  The tests
regenerate the same inputs (seeded CUDA generator) and compare their outputs at the same positions.
"""
import json
import os

import numpy as np
import torch

from oracle import ref_kernels

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_kernels.npz")
SAMPLES = 1024

# (case group, tag, dtype, seed) -- the parametrisations of the tests that compare against the reference kernels
AGG_CASES = [("cfg1", "float"), ("cfg1", "double"), ("selftest_k5", "double"), ("selftest_k1", "double"), ("ragged", "float"),
             ("ragged", "double"), ("s1_b8", "float"), ("s1_b256", "float"), ("s2_b256", "float"), ("s3_b256", "float"),
             ("s4_b256", "float")]
CASES = ([("agg", t, d, 0) for t, d in AGG_CASES]
         + [("agg_bf16", t, "float", 3) for t in ("s1_b8", "s2_b256", "s4_b256", "cfg1")]
         + [("agg", t, "double", 5) for t in ("cfg1", "selftest_k5", "ragged")]
         + [("mix", t, d, 0) for t, d in (("mix_selftest", "double"), ("mix_selftest", "float"), ("mix_s1_b32", "float"))]
         + [("refpad", t, d, 0) for t, d in (("refpad_selftest", "double"), ("refpad_selftest", "float"), ("refpad_k3", "double"),
                                              ("refpad_k3", "float"), ("refpad_s2_b8", "float"))]
         + [("dilate", t, d, 0) for t, d in (("dilate_selftest", "double"), ("dilate_selftest", "float"), ("dilate_s2_b8", "float"))]
         + [("merge", t, d, 0) for t, d in (("merge_selftest", "double"), ("merge_selftest", "float"), ("merge_s1_b8", "float"))])


def sample_index(shape):
    """The stored positions of a tensor of this shape in its contiguous flattening (fixed per shape): SAMPLES / 2 uniform, the
    rest on the border rows / columns of the last two (spatial) dimensions."""
    shape = tuple(int(d) for d in shape)
    numel = 1
    for d in shape:
        numel *= d
    g = torch.Generator().manual_seed(numel)
    if numel <= SAMPLES:
        return torch.arange(numel)
    uni = torch.randint(0, numel, (SAMPLES // 2,), generator=g)
    H, W = shape[-2], shape[-1]
    lead = torch.randint(0, numel // (H * W), (SAMPLES - SAMPLES // 2,), generator=g)
    side = torch.randint(0, 4, lead.shape, generator=g)
    t = torch.randint(0, max(H, W), lead.shape, generator=g)
    h = torch.where(side == 0, torch.zeros_like(t), torch.where(side == 1, torch.full_like(t, H - 1), t % H))
    w = torch.where(side == 2, torch.zeros_like(t), torch.where(side == 3, torch.full_like(t, W - 1), t % W))
    return torch.cat([uni, (lead * H + h) * W + w])


def key(group, tag, dtype, seed, name):
    return "%s/%s/%s/%d/%s" % (group, tag, dtype, seed, name)


class GoldenRef(ref_kernels.RefKernels):
    """make_inputs / make_variant_inputs of RefKernels over the stored geometries, plus the stored reference outputs."""

    def __init__(self):
        self.z = np.load(PATH)
        self.manifest = json.loads(bytes(self.z["manifest"]).decode())

    def ref(self, group, tag, dtype, seed, name):
        return torch.from_numpy(self.z[key(group, tag, dtype, seed, name)].astype(np.float64))


def sampled(t):
    """Values of tensor t (any layout) at the stored positions of its NCHW-contiguous flattening, as fp64 on the CPU."""
    flat = t.detach().contiguous().reshape(-1)
    return flat[sample_index(t.shape).to(flat.device)].double().cpu()


def _run(rk, group, tag, dtype, seed):
    op = "agg" if group == "agg_bf16" else group
    if op in ("agg", "mix"):
        inputs = rk.make_inputs(tag, dtype, op=op, seed=seed)
    else:
        inputs = rk.make_variant_inputs(tag, dtype, op, seed=seed)
    e = inputs[0]
    if group == "agg_bf16":
        inputs = (e,) + tuple(t.to(torch.bfloat16).float() for t in inputs[1:])
    if op == "agg":
        _, x, w, dy = inputs
        outs = {"y": rk.agg_forward(tag, x, w)}
        outs["dx"], outs["dw"] = rk.agg_backward(tag, dy, x, w)
    elif op == "mix":
        _, x, w1, w2, dy = inputs
        outs = {"y": rk.mix_forward(tag, x, w1, w2)}
        outs["dx"], outs["dw1"], outs["dw2"] = rk.mix_backward(tag, dy, x, w1, w2)
    elif op == "refpad":
        _, x, w, dy = inputs
        outs = {"y": rk.refpad_forward(tag, x, w)}
        outs["dx"], outs["dw"] = rk.refpad_backward(tag, dy, x, w)
    elif op == "dilate":
        _, x, w, dil, dy = inputs
        outs = {"y": rk.dilate_forward(tag, x, w, dil)}
        outs["dx"], outs["dw"] = rk.dilate_backward(tag, dy, x, w, dil)
    else:
        _, x, w, dy = inputs
        outs = {"y": rk.merge_forward(tag, x, w)}
        outs["dx"], outs["dw"] = rk.merge_backward(tag, dy, x, w)
    outs["x"] = x                                    # the inputs themselves: a changed random generator shows up as such
    return e, outs


def record(path=PATH):
    rk = ref_kernels.RefKernels()
    arrays, entries = {}, []
    for group, tag, dtype, seed in CASES:
        _, outs = _run(rk, group, tag, dtype, seed)
        for name, t in outs.items():
            v = sampled(t).numpy()
            arrays[key(group, tag, dtype, seed, name)] = v.astype(np.float32 if dtype == "float" else np.float64)
        op = "agg" if group == "agg_bf16" else group
        entries += [k for k in rk.manifest["kernels"] if k["tag"] == tag and k["op"] == op and k not in entries]
    man = {"block": rk.manifest["block"], "kernels": [{k: v for k, v in e.items() if k not in ("file", "sha256")} for e in entries]}
    arrays["manifest"] = np.frombuffer(json.dumps(man).encode(), dtype=np.uint8)
    np.savez_compressed(path, **arrays)
    return path


if __name__ == "__main__":
    import sys
    print(record(sys.argv[1] if len(sys.argv) > 1 else PATH))
