"""Pin the CPU oracle (oracle/) against the golden vectors made from the reference's own module code
and against the identities the reference's self-tests assert (SURVEY.md section 4 / 8c)."""
import os

import numpy as np
import pytest
import torch

from oracle import agg_ref, cot_ref, ref_import

TOL = 1e-9  # the reference self-tests' gate (aggregation_zeropad.py:252-260)


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


@pytest.mark.parametrize("name", ["agg_selftest_k5.npz", "agg_selftest_k1.npz", "agg_cot_k3.npz"])
def test_loops_match_unfold_golden(golden_dir, name):
    g = _load(golden_dir, name)
    k, s, p, d, heads = [int(v) for v in g["meta"]]
    y = agg_ref.agg_zeropad_fwd_loops(g["x"], g["w"], k, s, p, d)
    assert np.abs(y - g["y"]).max() < TOL
    dx, dw = agg_ref.agg_zeropad_bwd_loops(g["cot"], g["x"], g["w"], k, s, p, d)
    assert np.abs(dx - g["gx"]).max() < TOL
    assert np.abs(dw - g["gw"]).max() < TOL


def test_mix_loops_match_unfold_golden(golden_dir):
    g = _load(golden_dir, "agg_mix_selftest.npz")
    y = agg_ref.agg_zeropad_mix_fwd_loops(g["x"], g["w1"], g["w2"], 3, 5, 1, 1, 2, 1)
    assert np.abs(y - g["y"]).max() < TOL
    dx, d1, d2 = agg_ref.agg_zeropad_mix_bwd_loops(g["cot"], g["x"], g["w1"], g["w2"], 3, 5, 1, 1, 2, 1)
    assert np.abs(dx - g["gx"]).max() < TOL
    assert np.abs(d1 - g["gw1"]).max() < TOL
    assert np.abs(d2 - g["gw2"]).max() < TOL


@pytest.mark.parametrize("k,s,p,d,heads", [(3, 2, 1, 1, 1), (3, 1, 2, 2, 2), (5, 2, 2, 1, 1), (7, 1, 3, 1, 1)])
def test_loops_vs_unfold_strided_dilated(k, s, p, d, heads):
    gen = torch.Generator().manual_seed(5)
    N, C, wc, H, W = 2, 6, 3, 9, 8
    Ho, Wo = agg_ref.out_size(H, W, k, s, p, d)
    x = torch.randn(N, C, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn(N, heads, wc, k * k, Ho, Wo, generator=gen, dtype=torch.float64, requires_grad=True)
    cot = torch.randn(N, heads * C, Ho, Wo, generator=gen, dtype=torch.float64)
    y = agg_ref.agg_zeropad_unfold(x, w, k, s, p, d)
    gx, gw = torch.autograd.grad((y * cot).sum(), (x, w))
    y2 = agg_ref.agg_zeropad_fwd_loops(x.detach().numpy(), w.detach().numpy(), k, s, p, d)
    dx2, dw2 = agg_ref.agg_zeropad_bwd_loops(cot.numpy(), x.detach().numpy(), w.detach().numpy(), k, s, p, d)
    assert np.abs(y2 - y.detach().numpy()).max() < TOL
    assert np.abs(dx2 - gx.numpy()).max() < TOL
    assert np.abs(dw2 - gw.numpy()).max() < TOL


def _run_layer(fn, g, training):
    sd = {k[len("param/"):]: torch.from_numpy(g[k]).clone() for k in g.files if k.startswith("param/")}
    x = torch.from_numpy(g["x"]).clone().requires_grad_(training)
    for k, v in sd.items():
        if v.dtype.is_floating_point and "running" not in k:
            v.requires_grad_(training)
    out = fn(x, sd, training=training)
    return x, sd, out


@pytest.mark.parametrize("name,fn", [("cot_layer_d32.npz", cot_ref.cot_layer),
                                     ("cothybrid_layer_d32.npz", cot_ref.cot_layer),
                                     ("coxt_layer_d48.npz", cot_ref.coxt_layer)])
def test_block_restatement_matches_reference_golden(golden_dir, name, fn):
    g = _load(golden_dir, name)
    _, _, out = _run_layer(fn, g, False)
    assert (out - torch.from_numpy(g["out_eval"])).abs().max() < 1e-11
    x, sd, out = _run_layer(fn, g, True)
    assert (out.detach() - torch.from_numpy(g["out_train"])).abs().max() < 1e-11
    (out * torch.from_numpy(g["cotangent"])).sum().backward()
    assert (x.grad - torch.from_numpy(g["grad/x"])).abs().max() < 1e-10
    for k in g.files:
        if k.startswith("grad/") and k != "grad/x":
            ref = torch.from_numpy(g[k])
            got = sd[k[len("grad/"):]].grad
            assert (got - ref).abs().max() < 1e-10 * max(1.0, ref.abs().max().item()), k
        if k.startswith("buf_after/"):
            ref = torch.from_numpy(g[k])
            got = sd[k[len("buf_after/"):]]
            assert (got.double() - ref.double()).abs().max() < 1e-12, k


def test_restatement_vs_live_reference_module(golden_dir):
    """Same check against the reference module at another size: its output is stored in tests/golden/cot_layer_live_7x7.npz
    (oracle/make_golden.py) and, where a reference checkout exists, recomputed live as well."""
    gen = torch.Generator().manual_seed(77)
    sd = cot_ref.init_state_dict("cot", 64, gen)
    x = torch.relu(torch.randn(2, 64, 7, 7, generator=gen, dtype=torch.float64))
    got = cot_ref.cot_layer(x, {k: v.clone() for k, v in sd.items()}, training=False)
    wants = [torch.from_numpy(np.load(os.path.join(golden_dir, "cot_layer_live_7x7.npz"))["y"])]
    if ref_import.available():
        m = ref_import.load().CotLayer(64, 3).double()
        m.load_state_dict(sd, strict=True)
        m.eval()
        with torch.no_grad():
            wants.append(m(x))
    for want in wants:
        assert (got - want).abs().max() < 1e-11


def test_reference_kernel_cubins_are_consistent():
    """oracle/_ref (built from /root/reference by oracle/build_ref_kernels.py): every manifest entry has its cubin and the
    launch geometry the reference uses (block 1024, grid ceil(n / 1024), aggregation_zeropad.py:8,17-18,140-141)."""
    import json
    import os
    from oracle import ref_kernels
    if not ref_kernels.available():
        pytest.skip("oracle/_ref not built")
    man = json.load(open(os.path.join(ref_kernels.HERE, "manifest.json")))
    assert man["block"] == 1024 and len(man["kernels"]) >= 30
    for e in man["kernels"]:
        blob = open(os.path.join(ref_kernels.HERE, e["file"]), "rb").read()
        assert blob[:4] == b"\x7fELF" and e["kernel"].encode() in blob
        if "mix_weight_backward" in e["kernel"]:
            assert e["grid"] == (e["nthreads"] // 2 + 1023) // 1024
        else:
            assert e["grid"] == (e["nthreads"] + 1023) // 1024


@pytest.mark.parametrize("name,fixture", [("cotnet50", "cotnet50_eval_logits.npz"), ("cotnext50_2x48d", "cotnext50_eval_logits.npz")])
def test_oracle_model_matches_reference_golden_logits(golden_dir, name, fixture):
    """oracle/cot_model_ref.py (the CPU baseline and the `--impl reference` arm of bench.py, and the checker of the GPU
    backbone tests) against eval logits of the reference's own cotnet50 / cotnext50_2x48d (oracle/make_golden.py) on the
    same seeded parameters -- runs on every box, the reference tree is not needed."""
    from cotnet_b200 import backbone
    from oracle import cot_model_ref, make_golden
    g = np.load(os.path.join(golden_dir, fixture))
    m = make_golden.hybrid_seeded_state(backbone.MODELS[name](), int(g["seed"]))      # mirror = reference state-dict names
    assert sum(p.numel() for p in m.parameters()) == int(g["n_params"])
    o = cot_model_ref.build(name)
    o.load_reference_state(m.state_dict())
    o.eval()
    with torch.no_grad():
        y = o(torch.from_numpy(g["x"]))
    err = (y - torch.from_numpy(g["logits"])).abs().max().item()
    assert err <= 2e-5, err


# ---------------------------------------------------------------- the other cupy_layers variants (SURVEY 8f rank 4)
def test_refpad_loops_match_unfold_identity():
    """aggregation_refpad.py:223-239: kernel index math (loops) == Unfold(ReflectionPad2d(x)) at the self-test shape and a
    strided / dilated one."""
    for k, s, p, d, H, W in [(5, 1, 2, 1, 9, 9), (3, 2, 1, 1, 9, 8), (3, 1, 2, 2, 8, 7)]:
        gen = torch.Generator().manual_seed(k + s)
        n, c, wc, heads = 2, 8, 4, 2
        Ho, Wo = agg_ref.out_size(H, W, k, s, p, d)
        x = torch.randn(n, c, H, W, generator=gen, dtype=torch.float64)
        w = torch.randn(n, heads, wc, k * k, Ho, Wo, generator=gen, dtype=torch.float64)
        a = agg_ref.agg_refpad_unfold(x, w, k, s, p, d).numpy()
        b = agg_ref.agg_refpad_fwd_loops(x.numpy(), w.numpy(), k, s, p, d)
        assert np.abs(a - b).max() < TOL


def test_dilate_loops_match_unfold_identity():
    """aggregation_zeropad_dilate.py:258-296 (dilation_arr = [1, 1, 2, 4])."""
    gen = torch.Generator().manual_seed(3)
    n, c, wc, heads, H, W = 2, 8, 4, 2, 7, 7
    x = torch.randn(n, c, H, W, generator=gen, dtype=torch.float64)
    w = torch.randn(n, heads, wc, 9, H, W, generator=gen, dtype=torch.float64)
    dil = [1, 1, 2, 4]
    a = agg_ref.agg_dilate_unfold(x, w, dil).numpy()
    b = agg_ref.agg_dilate_fwd_loops(x.numpy(), w.numpy(), dil)
    assert np.abs(a - b).max() < TOL
    # the reference's own formulation of the identity (:266-295): three dilation groups, channel-interleaved
    split = [2, 1, 1]
    w1, w2, w3 = torch.split(w, split, dim=2)
    xs = torch.split(x.view(n, c // 4, 4, H, W), split, dim=2)
    ys = []
    for xi, wi, dd, sp in zip(xs, (w1, w2, w3), (1, 2, 4), split):
        xi = xi.reshape(n, -1, H, W)
        u = torch.nn.Unfold(kernel_size=3, dilation=dd, padding=dd, stride=1)(xi).view(n, xi.shape[1] // sp, sp, 9, H, W)
        ys.append((wi.unsqueeze(2) * u.unsqueeze(1)).sum(-3).view(n, heads * xi.shape[1], H, W).view(n, -1, sp, H, W))
    y2 = torch.cat(ys, dim=2).view(n, -1, H, W)
    assert (y2 - torch.from_numpy(b)).abs().max() < TOL


def test_mix_merge_matches_mix_on_split_weights():
    """aggregation_zeropad_mix_merge.py:332-351: the packed weight is cat([w1.view(n,-1,h,w), w2.view(n,-1,h,w)], 1)."""
    gen = torch.Generator().manual_seed(4)
    n, c, wc, heads, H, W = 2, 8, 4, 2, 6, 6
    x = torch.randn(n, c, H, W, generator=gen, dtype=torch.float64)
    w1 = torch.randn(n, heads, wc, 9, H, W, generator=gen, dtype=torch.float64)
    w2 = torch.randn(n, heads, wc, 25, H, W, generator=gen, dtype=torch.float64)
    w = torch.cat([w1.view(n, -1, H, W), w2.view(n, -1, H, W)], dim=1)
    a = agg_ref.agg_zeropad_mix_merge_unfold(x, w, heads, wc, 3, 5, 1, 1, 2, 1)
    b = agg_ref.agg_zeropad_mix_unfold(x, w1, w2, 3, 5, 1, 1, 2, 1)
    assert (a - b).abs().max() < TOL
    c2 = agg_ref.agg_zeropad_mix_merge_fwd_loops(x.numpy(), w.numpy(), heads, wc, 3, 5, 1, 1, 2, 1)
    assert np.abs(c2 - b.numpy()).max() < TOL


def test_oracle_model_train_step_matches_reference_golden(golden_dir):
    """oracle/cot_model_ref.py (the checker of the GPU model tests and the CPU arm of bench.py) against a TRAINING step of the
    reference's own cotnet50 (fixture from oracle/make_golden.py train: loss + every parameter gradient as norm and fixed random
    projection).  The fixture's own batch (16 x 224^2) in fp64."""
    import zlib  # noqa: F401
    from oracle import cot_model_ref, make_golden
    g = np.load(os.path.join(golden_dir, "cotnet50_train_bf16w.npz"))
    seed = int(g["seed"])
    o = cot_model_ref.build("cotnet50")
    # name-seeded state on a module tree with the REFERENCE's names: the product backbone carries them (tests/test_hybrid_cpu.py,
    # tests/test_patch_cpu.py pin that), the oracle loads from it
    from cotnet_b200 import backbone
    src = make_golden.hybrid_seeded_state(backbone.cotnet50(), seed)
    with torch.no_grad():
        for t in src.state_dict().values():
            if t.dtype.is_floating_point:
                t.copy_(t.bfloat16().float())
    o.load_reference_state(src.state_dict())
    o = o.double()      # fp64 like the fixture: training-mode gradients of this net amplify fp32 rounding to the percent level
    x, y = make_golden.train_batch(seed, int(g["B"]), int(g["res"]))
    x = x.bfloat16().double()
    o.train()
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    loss = torch.nn.functional.cross_entropy(o(x), y)
    loss.backward()
    assert abs(loss.item() - float(g["loss"])) <= 1e-4 * float(g["loss"])
    grads = {k.replace("__", "."): p.grad for k, p in o.named_parameters()}
    worst = 0.0
    floor = 1e-4 * float(np.median(g["gnorm"]))      # biases in front of a BatchNorm have an exactly-zero gradient (fp64: 1e-17)
    for n, gn, gp in zip([str(n) for n in g["names"]], g["gnorm"], g["gproj"]):
        t = grads[n].double()
        r = make_golden.proj_vector(n, t.shape, seed)
        d = max(gn, floor)
        worst = max(worst, abs(t.norm().item() - gn) / d, abs((t * r).sum().item() - gp) / (d * r.norm().item()))
    assert worst <= 1e-6, worst
