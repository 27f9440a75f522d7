"""Generate tests/golden/*.npz from the reference's OWN module code.  TEST INFRASTRUCTURE ONLY.

Run in the build container (needs /root/reference):   python -m oracle.make_golden

* cot_layer_d32.npz / coxt_layer_d48.npz / cothybrid_layer_d32.npz : the reference's unmodified
  ``CotLayer`` / ``CoXtLayer`` / ``CoTLayer`` (imported through ``oracle/ref_import.py``) run in
  fp64 on CPU with seeded, perturbed parameters: eval output, train output, d(out)/dx and
  d(out)/d(param) for a seeded cotangent, and the BN running buffers after the train step.
* agg_selftest_*.npz : the right-hand sides of the reference self-tests
  (aggregation_zeropad.py:238-292, aggregation_zeropad_mix.py:344-383) at their exact shapes,
  evaluated with torch's Unfold -- the reference stores no vectors, this identity is its only pin.
* cotnet50_eval_logits.npz / cotnext50_eval_logits.npz : eval logits of the reference's unmodified ``cotnet50`` /
  ``cotnext50_2x48d`` with seeded parameters: the pin of oracle/cot_model_ref.py (CPU baseline of bench.py).
* se_cotnetd50_eval_logits.npz : eval logits of the reference's unmodified ``se_cotnetd_50`` (models/cotnet_hybrid.py:458)
  on a seeded input with seeded parameters (``hybrid_seeded_state``): the pin of cotnet_b200/backbone_hybrid.py.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import agg_ref, cot_ref, ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def _layer_fixture(cls, kind, dim, B, H, W, seed, fname):
    gen = torch.Generator().manual_seed(seed)
    sd = cot_ref.init_state_dict(kind, dim, gen, dtype=torch.float64, perturb=True)
    x = torch.relu(torch.randn(B, dim, H, W, generator=gen, dtype=torch.float64))
    cot = torch.randn(B, dim, H, W, generator=gen, dtype=torch.float64)

    m = cls(dim, 3).double()
    missing = m.load_state_dict(sd, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    rec = {"x": x.numpy(), "cotangent": cot.numpy()}
    for k_, v_ in sd.items():
        rec["param/" + k_] = v_.numpy()

    m.eval()
    with torch.no_grad():
        rec["out_eval"] = m(x).numpy()

    m.train()
    xg = x.clone().requires_grad_(True)
    out = m(xg)
    rec["out_train"] = out.detach().numpy()
    (out * cot).sum().backward()
    rec["grad/x"] = xg.grad.numpy()
    for n_, p_ in m.named_parameters():
        rec["grad/" + n_] = p_.grad.numpy()
    for n_, b_ in m.named_buffers():
        rec["buf_after/" + n_] = b_.detach().numpy()
    np.savez_compressed(os.path.join(OUT, fname), **rec)
    print("wrote", fname, {k: v.shape for k, v in rec.items() if not k.startswith(("param/", "grad/", "buf_after/"))})


def _agg_fixture(fname, k, heads, n, cx, cw, H, W, seed):
    gen = torch.Generator().manual_seed(seed)
    p = (k - 1 + 1) // 2
    x = torch.randn(n, cx, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
    w = torch.randn(n, heads, cw, k * k, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
    cot = torch.randn(n, heads * cx, H, W, generator=gen, dtype=torch.float64)
    y = agg_ref.agg_zeropad_unfold(x, w, k, 1, p, 1)
    gx, gw = torch.autograd.grad((y * cot).sum(), (x, w))
    np.savez_compressed(os.path.join(OUT, fname), x=x.detach().numpy(), w=w.detach().numpy(), cot=cot.numpy(),
                        y=y.detach().numpy(), gx=gx.numpy(), gw=gw.numpy(),
                        meta=np.array([k, 1, p, 1, heads]))
    print("wrote", fname)


def _mix_fixture(fname, seed):
    gen = torch.Generator().manual_seed(seed)
    n, cx, cw, H, W = 2, 8, 4, 6, 6
    x = torch.randn(n, cx, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
    w1 = torch.randn(n, 1, cw, 9, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
    w2 = torch.randn(n, 1, cw, 25, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
    cot = torch.randn(n, 2 * cx, H, W, generator=gen, dtype=torch.float64)
    y = agg_ref.agg_zeropad_mix_unfold(x, w1, w2, 3, 5, 1, 1, 2, 1)
    gx, g1, g2 = torch.autograd.grad((y * cot).sum(), (x, w1, w2))
    np.savez_compressed(os.path.join(OUT, fname), x=x.detach().numpy(), w1=w1.detach().numpy(),
                        w2=w2.detach().numpy(), cot=cot.numpy(), y=y.detach().numpy(),
                        gx=gx.numpy(), gw1=g1.numpy(), gw2=g2.numpy())
    print("wrote", fname)


def hybrid_seeded_state(model, seed):
    """Deterministic, non-trivial parameters / BatchNorm statistics for a whole-model fixture without shipping a 90 MB state
    dict: every floating-point tensor of `model.state_dict()` is re-initialised from its OWN generator seeded by
    (seed, crc32(name)), so the result depends only on the tensor's name and shape -- not on module definition order.  Used
    identically here (on the reference models) and in the tests (on the mirrors / the oracle model)."""
    import zlib
    with torch.no_grad():
        for name, t in model.state_dict().items():
            if not t.dtype.is_floating_point:
                continue
            gen = torch.Generator().manual_seed((int(seed) * 1000003 + zlib.crc32(name.encode())) % (2 ** 31))
            if name.endswith("running_var"):
                t.copy_(torch.rand(t.shape, generator=gen) * 0.4 + 0.8)
            elif name.endswith("running_mean"):
                t.copy_(torch.randn(t.shape, generator=gen) * 0.1)
            elif t.dim() == 1 and name.endswith("weight"):            # norm-layer scales
                t.copy_(torch.rand(t.shape, generator=gen) * 0.5 + 0.5)
            elif t.dim() == 1:                                          # biases
                t.copy_(torch.randn(t.shape, generator=gen) * 0.1)
            else:
                fan = max(1, t[0].numel())
                t.copy_(torch.randn(t.shape, generator=gen) * (1.0 / fan) ** 0.5)
    return model


def _hybrid_fixture(fname, seed):
    """SE-CoTNetD-50 (models/cotnet_hybrid.py:458-464) eval logits from the reference's own model code."""
    ref = ref_import.load()
    m = hybrid_seeded_state(ref.hybrid.se_cotnetd_50(), seed).eval()
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(seed + 1))
    with torch.no_grad():
        y = m(x)
    np.savez_compressed(os.path.join(OUT, fname), x=x.numpy(), logits=y.numpy(), seed=np.int64(seed),
                        n_params=np.int64(sum(p.numel() for p in m.parameters())))


def _trunk_fixture(fname, entry, seed, res=64):
    """CoTNet-50 / CoTNeXt-50 (models/cotnet.py:266-288) eval logits from the reference's own model code: the pin of
    oracle/cot_model_ref.py (the CPU baseline / reference arm of bench.py) on boxes without the reference tree."""
    ref = ref_import.load()
    m = hybrid_seeded_state(getattr(ref, entry)(), seed).eval()
    x = torch.randn(2, 3, res, res, generator=torch.Generator().manual_seed(seed + 1))
    with torch.no_grad():
        y = m(x)
    np.savez_compressed(os.path.join(OUT, fname), x=x.numpy(), logits=y.numpy(), seed=np.int64(seed),
                        n_params=np.int64(sum(p.numel() for p in m.parameters())))


def proj_vector(name, shape, seed):
    """The fixed random direction a gradient is projected on in the train-step fixtures (regenerated from the tensor's
    name by the tests; storing <grad, r> and ||grad|| per parameter pins every gradient in two floats)."""
    import zlib
    gen = torch.Generator().manual_seed((int(seed) * 7919 + zlib.crc32(name.encode())) % (2 ** 31))
    return torch.randn(shape, generator=gen, dtype=torch.float64)


def train_batch(seed, B, res):
    """Image-like synthetic batch: smooth low-frequency content (bilinearly up-sampled 6x6 noise) + fine noise, per-sample
    contrast and per-sample colour offset.  i.i.d. N(0,1) images all pool to the same descriptor, which makes every
    batch-statistics BatchNorm behind a global pool (se.1, bn1 of SplitAttn) normalise pure noise and the training-mode
    gradients of the net chaotic (fp32 vs fp64 of the SAME code differ by 4 % with i.i.d. images, 1 % with these)."""
    gen = torch.Generator().manual_seed(int(seed) + 17)
    lo = torch.randn(B, 3, 6, 6, generator=gen)
    x = torch.nn.functional.interpolate(lo, size=(res, res), mode="bilinear", align_corners=False) * 2.0
    x = x + 0.5 * torch.randn(B, 3, res, res, generator=gen)
    x = x * (torch.rand(B, 1, 1, 1, generator=gen) * 1.5 + 0.5) + torch.randn(B, 3, 1, 1, generator=gen)
    y = torch.randint(0, 1000, (B,), generator=gen)
    return x, y


def _train_fixture(fname, entry, seed, res, B, round_bf16):
    """Eval logits + one training step (loss, every parameter gradient as norm + fixed random projection, a few updated
    running statistics) of the reference's OWN model code in fp64 on name-seeded parameters.  round_bf16: parameters and
    the batch are rounded to bf16-representable values first (the protocol of SURVEY 8d for bf16 runs)."""
    ref = ref_import.load()
    ctor = getattr(ref, entry) if hasattr(ref, entry) else getattr(ref.hybrid, entry)
    m = hybrid_seeded_state(ctor(), seed)
    if round_bf16:
        with torch.no_grad():
            for t in m.state_dict().values():
                if t.dtype.is_floating_point:
                    t.copy_(t.bfloat16().float())
    m = m.double()
    x, y = train_batch(seed, B, res)
    if round_bf16:
        x = x.bfloat16().float()
    x = x.double()
    m.eval()
    with torch.no_grad():
        logits = m(x)
    m.train()
    loss = torch.nn.functional.cross_entropy(m(x), y)
    loss.backward()
    names, gn, gp = [], [], []
    for n, p_ in m.named_parameters():
        names.append(n)
        gn.append(p_.grad.norm().item())
        gp.append((p_.grad * proj_vector(n, p_.shape, seed)).sum().item())
    sd = m.state_dict()
    rm_names = [k for k in sd if k.endswith("running_mean") or k.endswith("running_var")]
    rm_names = rm_names[:4] + rm_names[-4:]
    np.savez_compressed(os.path.join(OUT, fname), logits=logits.numpy().astype(np.float32), loss=np.float64(loss.item()),
                        names=np.array(names), gnorm=np.array(gn), gproj=np.array(gp), seed=np.int64(seed), res=np.int64(res),
                        B=np.int64(B), round_bf16=np.int64(1 if round_bf16 else 0), rm_names=np.array(rm_names),
                        rm_values=np.concatenate([sd[k].numpy().reshape(-1)[:8] for k in rm_names]),
                        n_params=np.int64(sum(p_.numel() for p_ in m.parameters())))
    print("wrote", fname, "loss", loss.item())


TRAIN_FIXTURES = [("cotnet50_train_bf16w.npz", "cotnet50", 3001, 224, 16, True),
                  ("cotnext50_train_bf16w.npz", "cotnext50_2x48d", 3002, 224, 16, True),
                  ("se_cotnetd101_train.npz", "se_cotnetd_101", 3003, 224, 8, False),
                  ("se_cotnetd152_train_320.npz", "se_cotnetd_152", 3004, 320, 4, False)]


def _live_layer_fixture(fname):
    """CotLayer(64) eval output at 7x7 from the reference's module code (tests/test_oracle.py checks the restatement against it)."""
    ref = ref_import.load()
    gen = torch.Generator().manual_seed(77)
    sd = cot_ref.init_state_dict("cot", 64, gen)
    x = torch.relu(torch.randn(2, 64, 7, 7, generator=gen, dtype=torch.float64))
    m = ref.CotLayer(64, 3).double()
    m.load_state_dict(sd, strict=True)
    m.eval()
    with torch.no_grad():
        y = m(x)
    np.savez_compressed(os.path.join(OUT, fname), y=y.numpy())


HYBRID_TRAIN_SEED = 31


def hybrid_train_inputs():
    return (torch.randn(2, 3, 64, 64, dtype=torch.float64, generator=torch.Generator().manual_seed(5)),
            torch.randn(2, 1000, dtype=torch.float64, generator=torch.Generator().manual_seed(6)))


def hybrid_train_record(m, seed=HYBRID_TRAIN_SEED):
    """One fp64 training step of SE-CoTNetD-50 (seeded state, hybrid_train_inputs): output, every parameter gradient pinned as
    (sum, <grad, proj_vector>, ||grad||^2), and the sums of the running statistics after the step."""
    x, cot = hybrid_train_inputs()
    m.train()
    y = m(x)
    names = [n for n, _ in m.named_parameters()]
    grads = torch.autograd.grad((y * cot).sum(), [p for _, p in m.named_parameters()])
    g = np.array([[t.sum().item(), (t * proj_vector(n, t.shape, seed)).sum().item(), (t * t).sum().item()]
                  for n, t in zip(names, grads)])
    run = np.array([v.sum().item() for k, v in m.state_dict().items() if k.endswith("running_mean") or k.endswith("running_var")])
    return y.detach().numpy(), g, run


def _hybrid_live_fixture(fname, seed=HYBRID_TRAIN_SEED):
    """State-dict layout of SE-CoTNetD-50/101/152 and one training step of SE-CoTNetD-50 from the reference's model code
    (tests/test_hybrid_cpu.py)."""
    import json
    ref = ref_import.load()
    rec = {}
    for name in ("se_cotnetd_50", "se_cotnetd_101", "se_cotnetd_152"):
        sd = getattr(ref.hybrid, name)().state_dict()
        rec["layout/" + name] = np.frombuffer(json.dumps([[k, list(v.shape)] for k, v in sd.items()]).encode(), dtype=np.uint8)
    m = hybrid_seeded_state(ref.hybrid.se_cotnetd_50(zero_init_last_bn=False), seed).double()
    rec["y"], rec["grads"], rec["running"] = hybrid_train_record(m, seed)
    np.savez_compressed(os.path.join(OUT, fname), **rec)


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "train":
        os.makedirs(OUT, exist_ok=True)
        torch.set_num_threads(8)
        for f in TRAIN_FIXTURES:
            if len(sys.argv) > 2 and sys.argv[2] not in f[0]:
                continue
            _train_fixture(*f)
        return
    os.makedirs(OUT, exist_ok=True)
    ref = ref_import.load()
    torch.set_num_threads(4)
    _layer_fixture(ref.CotLayer, "cot", 32, 2, 6, 5, 101, "cot_layer_d32.npz")
    _layer_fixture(ref.CoXtLayer, "coxt", 48, 2, 5, 6, 202, "coxt_layer_d48.npz")
    _layer_fixture(ref.CoTLayer, "cot", 32, 3, 4, 4, 303, "cothybrid_layer_d32.npz")
    # reference self-test shapes: aggregation_zeropad.py:238-246 and :266-274, mix :344-353
    _agg_fixture("agg_selftest_k5.npz", 5, 2, 2, 8, 4, 9, 9, 11)
    _agg_fixture("agg_selftest_k1.npz", 1, 2, 2, 8, 4, 9, 9, 12)
    _agg_fixture("agg_cot_k3.npz", 3, 1, 2, 16, 2, 7, 6, 13)
    _mix_fixture("agg_mix_selftest.npz", 14)
    _hybrid_fixture("se_cotnetd50_eval_logits.npz", 2024)
    _live_layer_fixture("cot_layer_live_7x7.npz")
    _hybrid_live_fixture("se_cotnetd50_train_fp64.npz")
    _trunk_fixture("cotnet50_eval_logits.npz", "cotnet50", 2025)
    _trunk_fixture("cotnext50_eval_logits.npz", "cotnext50_2x48d", 2026)


if __name__ == "__main__":
    main()
