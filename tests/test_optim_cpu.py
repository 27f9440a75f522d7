"""CPU checks of the optimizer rules (solver.opt, optim/optim_factory.py:create_optimizer): the torch restatement against the
reference's own optimizers (tests/golden/optim.npz), the parsing of solver.opt, and the argument checks of the new C entry
points."""
import os

import numpy as np
import pytest
import torch

import optim_ref


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "optim.npz"))


def _cases(g):
    return [(str(c), str(o), float(m)) for c, o, m in zip(g["cases"], g["opts"], g["momenta"])]


def replay(g, opt, momentum, dtype=torch.float64, on_step=None):
    """The golden's 14 steps through optim_ref.Optim in `dtype`: (w, b, optimizer)."""
    w = torch.from_numpy(g["w0"]).to(dtype).clone()
    b = torch.from_numpy(g["b0"]).to(dtype).clone()
    o = optim_ref.Optim(opt, [(float(g["weight_decay"]), [w]), (0.0, [b])], float(g["lr"]), momentum, float(g["eps"]), radam_fp32=True)
    for s in range(1, 15):
        if s == int(g["lr2_step"]):
            o.lr = float(g["lr2"])
        o.step([torch.from_numpy(g["gw_%d" % s]).to(dtype), torch.from_numpy(g["gb_%d" % s]).to(dtype)])
        if on_step:
            on_step(s, w, b, o)
    return w, b, o


EXPECTED_CASES = {"sgd", "momentum", "adam", "adamw", "nadam", "radam", "adadelta", "rmsprop", "rmsproptf", "lookahead_sgd",
                  "lookahead_adamw", "lookahead_rmsproptf"}


def test_golden_covers_every_rule(golden):
    names = {c for c, _, _ in _cases(golden)}
    assert EXPECTED_CASES <= names
    assert int(golden["lr2_step"]) == 8


@pytest.mark.parametrize("case", sorted(EXPECTED_CASES | {"rmsprop_m0", "rmsproptf_m0", "lookahead_radam"}))
def test_restatement_matches_reference(golden, case):
    opt, mom = {c: (o, m) for c, o, m in _cases(golden)}[case]

    def check(s, w, b, o):
        for tag, t in (("w", w), ("b", b)):
            want = torch.from_numpy(golden["%s/%s_%d" % (case, tag, s)])
            torch.testing.assert_close(t, want, rtol=1e-12, atol=1e-14, msg=lambda m: "%s step %d %s: %s" % (case, s, tag, m))
    w, b, o = replay(golden, opt, mom, on_step=check)
    for tag, st in zip("wb", o.state):
        for k, v in st.items():
            key = "%s/state_%s_%s" % (case, k, tag)
            if torch.is_tensor(v):
                want = torch.from_numpy(golden[key])
                assert v.dtype == want.dtype, (key, v.dtype, want.dtype)        # RAdam's moments are fp32 in the reference
                torch.testing.assert_close(v, want, rtol=1e-12, atol=1e-14, msg=lambda m: key + ": " + m)
            elif k in ("step", "m_schedule") and "%s/%s_%s" % (case, k, tag) in golden.files:
                assert v == float(golden["%s/%s_%s" % (case, k, tag)]), (key, v)
    stored = {k.split("/state_")[1].rsplit("_", 1)[0] for k in golden.files if k.startswith(case + "/state_")}
    assert stored == {k for k, v in o.state[0].items() if torch.is_tensor(v)}, stored


def test_radam_rectifies_from_step_6_and_lookahead_syncs_at_6_and_12(golden):
    t = np.arange(1, 15, dtype=np.float64)
    b2t = 0.999 ** t
    n_sma = (2 / (1 - 0.999) - 1) - 2 * t * b2t / (1 - b2t)
    assert (n_sma >= 5).tolist() == [s >= 6 for s in range(1, 15)]
    syncs = []

    def on(s, w, b, o):
        if s % 6 == 0:
            syncs.append(s)
            assert torch.equal(o.state[0]["slow_buffer"], w)
    replay(golden, "lookahead_sgd", 0.9, on_step=on)
    assert syncs == [6, 12]
    # the first synchronisation leaves the fast weights as they are: step 6 of lookahead_sgd equals step 6 of sgd
    for tag in "wb":
        assert np.array_equal(golden["lookahead_sgd/%s_6" % tag], golden["sgd/%s_6" % tag])
        assert not np.array_equal(golden["lookahead_sgd/%s_12" % tag], golden["sgd/%s_12" % tag])


# ------------------------------------------------------------------------------------------------ solver.opt parsing
@pytest.mark.parametrize("name,base,rule,la", [
    ("sgd", "sgd", "OPT_SGD", False), ("SGD", "sgd", "OPT_SGD", False), ("nesterov", "nesterov", "OPT_SGD", False),
    ("momentum", "momentum", "OPT_MOMENTUM", False), ("adam", "adam", "OPT_ADAM", False), ("AdamW", "adamw", "OPT_ADAMW", False),
    ("nadam", "nadam", "OPT_NADAM", False), ("radam", "radam", "OPT_RADAM", False), ("adadelta", "adadelta", "OPT_ADADELTA", False),
    ("rmsprop", "rmsprop", "OPT_RMSPROP", False), ("rmsproptf", "rmsproptf", "OPT_RMSPROPTF", False),
    ("lookahead_sgd", "sgd", "OPT_SGD", True), ("lookahead_adamw", "adamw", "OPT_ADAMW", True),
    ("Lookahead_RMSpropTF", "rmsproptf", "OPT_RMSPROPTF", True), ("foo_adam", "adam", "OPT_ADAM", False),
])
def test_parse_opt(name, base, rule, la):
    from cotnet_b200 import _lib, trainer
    assert trainer.parse_opt(name) == (base, getattr(_lib, rule), la)


def test_parse_opt_sgd_follows_nesterov():
    from cotnet_b200 import _lib, trainer
    assert trainer.parse_opt("sgd", nesterov=False)[1] == _lib.OPT_MOMENTUM
    assert trainer.parse_opt("nesterov", nesterov=False)[1] == _lib.OPT_SGD
    assert trainer.parse_opt("momentum", nesterov=True)[1] == _lib.OPT_MOMENTUM


@pytest.mark.parametrize("name,why", [
    ("adamp", "per-tensor projection"), ("sgdp", "per-tensor projection"), ("lookahead_sgdp", "per-tensor projection"),
    ("novograd", "per-tensor gradient norms"), ("nvnovograd", "per-tensor gradient norms"), ("adafactor", "factored"),
    ("adahessian", "Hessian"), ("fusedsgd", "apex"), ("fusedadamw", "apex"), ("fusedlamb", "apex"), ("lbfgs", "unknown"),
])
def test_parse_opt_rejects_unsupported(name, why):
    from cotnet_b200 import trainer
    with pytest.raises(ValueError, match=why) as e:
        trainer.parse_opt(name)
    for ok in ("adamw", "rmsproptf", "lookahead_"):
        assert ok in str(e.value)


def test_trainstep_rejects_unsupported_opt():
    import clip_ref
    from cotnet_b200 import trainer
    with pytest.raises(ValueError, match="adamp"):
        trainer.TrainStep(clip_ref.Toy(), opt="adamp")


# ------------------------------------------------------------------------------------------------ C entry points
def test_opt_entry_points_reject_bad_arguments():
    """Validation happens before any CUDA call: the pointers below are never dereferenced."""
    from cotnet_b200 import _lib
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EALIGN, EDTYPE = -5, -1, -4, -2

    def opt(**kw):
        base = dict(rule=_lib.OPT_ADAM, eps=1e-8, lookahead_k=0, lookahead_alpha=0.5, M=P, V=P, S=None, state=P)
        base.update(kw)
        return _lib.Opt(**base)

    # prepare
    assert lib.cotb200_opt_prepare(None, P, 1, None) == ENULL
    assert lib.cotb200_opt_prepare(opt(state=None), P, 1, None) == ENULL
    assert lib.cotb200_opt_prepare(opt(), None, 1, None) == ENULL
    assert lib.cotb200_opt_prepare(opt(rule=0), P, 1, None) == EINVAL
    assert lib.cotb200_opt_prepare(opt(rule=10), P, 1, None) == EINVAL
    assert lib.cotb200_opt_prepare(opt(lookahead_k=-1), P, 1, None) == EINVAL

    # opt_step
    def step(o, n=8, gdt=_lib.F32, G=P, clip=None, Pb=None, E=None):
        return lib.cotb200_opt_step(n, P, gdt, G, E, Pb, P, o, clip, None)
    assert step(None) == ENULL
    assert step(opt(state=None)) == ENULL
    assert lib.cotb200_opt_step(8, None, _lib.F32, P, None, None, P, opt(), None, None) == ENULL
    assert step(opt(rule=42)) == EINVAL
    assert step(opt(M=None)) == ENULL                                   # adam needs exp_avg
    assert step(opt(V=None)) == ENULL                                   # and exp_avg_sq
    assert step(opt(rule=_lib.OPT_SGD, M=None, V=None)) == ENULL
    assert step(opt(rule=_lib.OPT_ADADELTA, M=None)) == ENULL
    assert step(opt(lookahead_k=6)) == ENULL                            # Lookahead without slow weights
    assert step(opt(lookahead_k=6, S=P, lookahead_alpha=1.5)) == EINVAL
    assert step(opt(eps=-1.0)) == EINVAL
    assert step(opt(), n=6) == EINVAL
    assert step(opt(), n=0) == EINVAL
    assert step(opt(M=24)) == EALIGN
    assert step(opt(), G=8) == EALIGN
    assert step(opt(), E=8) == EALIGN
    assert step(opt(), Pb=P + 2) == EALIGN
    assert step(opt(), gdt=_lib.F16) == EDTYPE
    assert step(opt(), clip=_lib.Clip(mode=7, factor=P)) == EINVAL
    assert step(opt(), clip=_lib.Clip(mode=_lib.CLIP_NORM)) == ENULL
    assert step(opt(), clip=_lib.Clip(mode=_lib.CLIP_AGC, factor=P, n_segs=3)) == ENULL
    assert step(opt(), clip=_lib.Clip(mode=_lib.CLIP_VALUE, value=0.0)) == EINVAL

    # lookahead_sync
    assert lib.cotb200_lookahead_sync(8, P, None, opt(S=None), None) == ENULL
    assert lib.cotb200_lookahead_sync(8, P, None, None, None) == ENULL
    assert lib.cotb200_lookahead_sync(6, P, None, opt(S=P), None) == EINVAL
    assert lib.cotb200_lookahead_sync(8, P, None, opt(S=P, lookahead_alpha=-0.1), None) == EINVAL
    assert lib.cotb200_lookahead_sync(8, P, None, opt(S=24), None) == EALIGN
    assert lib.cotb200_last_error()


def test_sgd_pass_rejects_bad_arguments():
    """The plain SGD pass as TrainStep launches it (rule SGD, no clip); no pointer below is dereferenced."""
    from cotnet_b200 import _lib
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EDTYPE = -5, -1, -2
    o = _lib.Opt(rule=_lib.OPT_SGD, M=P, state=P)
    assert lib.cotb200_opt_step(6, P, _lib.F32, P, None, None, P, o, None, None) == EINVAL
    assert lib.cotb200_opt_step(8, None, _lib.F32, P, None, None, P, o, None, None) == ENULL
    assert lib.cotb200_opt_step(8, P, _lib.F64, P, None, None, P, o, None, None) == EDTYPE


def test_struct_layouts():
    import ctypes
    from cotnet_b200 import _lib
    assert ctypes.sizeof(_lib.OptState) == 40 and _lib.OptState.c.offset == 16 and _lib.OptState.sync.offset == 32
    assert ctypes.sizeof(_lib.Opt) == 48 and _lib.Opt.M.offset == 16 and _lib.Opt.state.offset == 40
