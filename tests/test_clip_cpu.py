"""CPU checks of gradient clipping (train.py:270-273): the torch restatement against the reference's own clip_grad.py
(tests/golden/clip.npz), the AGC unit planner on the real trunks, and the argument checks of the new C entry points."""
import numpy as np
import pytest
import torch

import clip_ref

N_PARAMS = len(list(clip_ref.Toy().parameters()))


@pytest.fixture(scope="module")
def golden(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, "clip.npz"))


def _inputs(g, dtype):
    ps = [torch.from_numpy(g["p_%d" % i]).to(dtype) for i in range(N_PARAMS)]
    gs = [torch.from_numpy(g["g_%d" % i]).to(dtype) for i in range(N_PARAMS)]
    return ps, gs


def test_head_pick_matches_reference(golden):
    m = clip_ref.Toy()
    ids = [id(p) for p in m.parameters()]
    kept = [ids.index(id(p)) for p in clip_ref.model_parameters(m, exclude_head=True)]
    assert kept == golden["head"].tolist()
    names = [str(n) for n in golden["names"]]
    assert [names[i] for i in range(N_PARAMS) if i not in kept] == ["fc.weight", "fc.bias"]


@pytest.mark.parametrize("mode", clip_ref.MODES)
@pytest.mark.parametrize("tag", ["bind", "free"])
@pytest.mark.parametrize("dtype,rtol", [(torch.float32, 1e-6), (torch.float64, 1e-6)])
def test_oracle_matches_reference(golden, mode, tag, dtype, rtol):
    m = clip_ref.Toy()
    ps, gs = _inputs(golden, dtype)
    value = float(golden["value_%s_%s" % (mode, tag)])
    out, norm = clip_ref.clip_model_grads(m, ps, gs, value, mode)
    changed = 0
    for i, o in enumerate(out):
        want = torch.from_numpy(golden["out_%s_%s_%d" % (mode, tag, i)]).double()
        torch.testing.assert_close(o.double(), want, rtol=rtol, atol=1e-12, msg=lambda s: "%s param %d: %s" % (mode, i, s))
        if dtype == torch.float32:
            changed += int(not torch.equal(o, gs[i]))
    if mode == "norm":
        assert abs(float(norm) - float(golden["norm_%s" % tag])) <= 1e-6 * float(golden["norm_%s" % tag])
    if dtype == torch.float32:
        assert (changed > 0) == (tag == "bind"), changed
    if mode == "agc" and tag == "bind":                  # the head is never clipped, and some other parameters are not either
        assert torch.equal(out[-1], gs[-1]) and torch.equal(out[-2], gs[-2])


def test_agc_factor_form_matches_oracle(golden):
    """The factor form the kernels use (factor 1 where the clip does not bind) gives the oracle's gradients exactly."""
    m = clip_ref.Toy()
    ps, gs = _inputs(golden, torch.float32)
    value = float(golden["value_agc_bind"])
    kept = golden["head"].tolist()
    fs = clip_ref.agc_factors([ps[i] for i in kept], [gs[i] for i in kept], value)
    out, _ = clip_ref.clip_model_grads(m, ps, gs, value, "agc")
    for i, f in zip(kept, fs):
        shaped = f.view(-1, *([1] * (gs[i].dim() - 1))) if gs[i].dim() > 1 else f
        assert torch.equal(gs[i] * shaped, out[i]), i


# ------------------------------------------------------------------------------------------------ the AGC unit planner
def _trunk(name):
    from cotnet_b200 import backbone, backbone_hybrid
    fn = {**backbone.MODELS, **backbone_hybrid.MODELS}[name]
    torch.manual_seed(0)
    return fn().to(memory_format=torch.channels_last)


@pytest.mark.parametrize("name", ["cotnet50", "cotnext50_2x48d", "se_cotnetd_50"])
def test_unit_planner_tiles_the_slots(name):
    from cotnet_b200 import trainer
    m = _trunk(name)
    plan = trainer.plan_flat(list(m.named_parameters()))
    units, head = trainer.plan_clip_units(m, plan)
    assert head == ["fc.weight", "fc.bias"]
    params = list(m.parameters())
    count = [p.shape[0] if p.dim() > 1 else 1 for p in params]
    assert len(units) == sum(count[:-2])                  # the head's 1000 rows + 1 bias are left out
    if name == "cotnet50":
        assert sum(count) == 47227 and len(units) == 47227 - 1001
    lengths = {len_ for _, _, len_ in units}
    if name == "cotnet50":                                # the stem's 147-element rows start inside a float4
        assert max(lengths) == 2048 and 147 in lengths
    # every kept parameter's slot is tiled exactly by its units, in order; nothing else is covered
    by_bucket = {0: [], 1: []}
    for b, off, n in units:
        by_bucket[b].append((off, n))
    for b, key in ((0, "big"), (1, "small")):
        covered = sorted(by_bucket[b])
        want = []
        for _, p, off in plan[key]:
            if any(p is q for q in params[-2:]):
                continue
            rows = p.shape[0] if p.dim() > 1 else 1
            want += [(off + r * (p.numel() // rows), p.numel() // rows) for r in range(rows)]
        assert covered == sorted(want)
        assert all(a[0] + a[1] <= c[0] for a, c in zip(covered, covered[1:]))


def test_unit_planner_segments_cover_the_range():
    from cotnet_b200 import trainer
    m = _trunk("cotnet50")
    plan = trainer.plan_flat(list(m.named_parameters()))
    units, _ = trainer.plan_clip_units(m, plan)
    for b, n in ((0, plan["n_big"]), (1, plan["n_small"])):
        mine = [(i, off, ln) for i, (bb, off, ln) in enumerate(units) if bb == b]
        segs = trainer._clip_segments(mine, n, 4096)
        pos = 0
        for off, ln, u in segs:
            assert off == pos and 1 <= ln <= 4096
            pos += ln
        assert pos == n
        seen = {}
        for off, ln, u in segs:
            if u >= 0:
                seen[u] = seen.get(u, 0) + ln
        assert seen == {i: ln for i, _, ln in mine}


def test_unit_planner_refuses_transposed_rows():
    from cotnet_b200 import trainer
    m = clip_ref.Toy()
    with torch.no_grad():
        m.conv2.weight.data = m.conv2.weight.data.flatten(1).t().contiguous().t().view(16, 8, 1, 1)   # dim 0 has stride 1
    plan = trainer.plan_flat(list(m.named_parameters()))
    with pytest.raises(ValueError, match="conv2.weight"):
        trainer.plan_clip_units(m, plan)
    m2 = clip_ref.Toy().to(memory_format=torch.channels_last)                                         # channels_last is fine
    assert len(trainer.plan_clip_units(m2, trainer.plan_flat(list(m2.named_parameters())))[0]) == 8 + 2 + 16 + 16 + 1


def test_trainstep_rejects_unknown_clip_mode():
    from cotnet_b200 import trainer
    with pytest.raises(ValueError, match="clip_mode"):
        trainer.TrainStep(clip_ref.Toy(), clip_grad=1.0, clip_mode="l1")


# ------------------------------------------------------------------------------------------------ C entry points
def test_clip_and_clipped_opt_step_reject_bad_arguments():
    """Validation happens before any CUDA call: the pointers below are never dereferenced."""
    from cotnet_b200 import _lib
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EALIGN, EDTYPE = -5, -1, -4, -2
    assert lib.cotb200_clip_seg_max() == 4096
    # grad_norm
    assert lib.cotb200_grad_norm(8, _lib.BF16, P, P, 8, P, P, 1.0, None, None) == ENULL
    assert lib.cotb200_grad_norm(8, _lib.BF16, P, P, 8, None, P, 1.0, P, None) == ENULL
    assert lib.cotb200_grad_norm(6, _lib.BF16, P, P, 0, None, None, 1.0, P, None) == EINVAL
    assert lib.cotb200_grad_norm(8, _lib.BF16, P, P, 5, P, P, 1.0, P, None) == EINVAL
    assert lib.cotb200_grad_norm(8, _lib.F16, P, P, 0, None, None, 1.0, P, None) == EDTYPE
    assert lib.cotb200_grad_norm(8, _lib.F32, 8, P, 0, None, None, 1.0, P, None) == EALIGN
    # unit_norms
    assert lib.cotb200_unit_norms(4, None, 16, P, _lib.BF16, P, P, None, None, None, 0.01, P, None, None) == ENULL
    assert lib.cotb200_unit_norms(4, P, 16, P, _lib.BF16, P, P, P, None, P, 0.01, P, None, None) == ENULL
    assert lib.cotb200_unit_norms(0, P, 16, P, _lib.BF16, P, P, None, None, None, 0.01, P, None, None) == EINVAL
    assert lib.cotb200_unit_norms(4, P, 16, P, _lib.F64, P, P, None, None, None, 0.01, P, None, None) == EDTYPE
    # the clipped SGD pass: opt_step with rule SGD
    def step(n=8, gdt=_lib.F32, G=P, clip=None):
        return lib.cotb200_opt_step(n, P, gdt, G, None, None, P, _lib.Opt(rule=_lib.OPT_SGD, M=P, state=P), clip, None)
    norm = _lib.Clip(mode=_lib.CLIP_NORM, factor=P)
    assert step(n=6, clip=norm) == EINVAL
    assert step(clip=_lib.Clip(mode=7, factor=P)) == EINVAL
    assert step(clip=_lib.Clip(mode=_lib.CLIP_NORM)) == ENULL
    assert step(clip=_lib.Clip(mode=_lib.CLIP_VALUE, value=0.0)) == EINVAL
    assert step(clip=_lib.Clip(mode=_lib.CLIP_VALUE, value=float("nan"))) == EINVAL
    assert step(clip=_lib.Clip(mode=_lib.CLIP_AGC, factor=P, n_segs=3)) == ENULL
    assert step(clip=_lib.Clip(mode=_lib.CLIP_AGC, factor=P, segs=P, n_segs=0)) == EINVAL
    assert step(G=8, clip=norm) == EALIGN
    assert step(gdt=_lib.F16, clip=norm) == EDTYPE
    assert lib.cotb200_last_error()
