"""The kernels only the inference path reaches, each against fp64 of its own inputs (tests/stage_ref.py).

CotLayer._forward_tc_eval puts every convolution of the CoT layer on the wgmma kernels with the BatchNorms folded into their
epilogues, and fused._cot_tail_eval runs tail_pool -> cotb200_se_eval -> tail_combine.  No training step runs these
geometries or epilogue forms:

  * the grouped 3x3 key conv at stage 3 (C = 256, 64-channel groups: the haloed kernel with 4 N tiles, R = 14, two M blocks)
    and stage 4 (C = 512, 128-channel groups: conv mode of the GEMM kernel, two samples per M tile);
  * the GEMM epilogues of embed.0 (two operand pairs, scale + shift + ReLU), embed.3 (shift only: its bias) and conv1x1 (scale +
    shift, no ReLU) at the four stages' shapes;
  * cotb200_se_eval (fc1 + folded BatchNorm + ReLU, fc2 + radix-2 __expf softmax) at every branch of its tiling;
  * tail_pool / tail_combine with the eval fold of the running statistics.

With small-integer operands the accumulators are exact, so the epilogue's single fmaf rounding and the bf16 store can be
emulated exactly (stage_ref.epilogue_ref) for arbitrary fp32 scale / shift and the whole output compared with torch.equal; the
same holds for the hidden activations of cotb200_se_eval.  Values that go through __expf, rsqrt or the SiLU are compared within
per-element bounds derived in stage_ref.py."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import stage_ref as S
from cotnet_b200 import _lib, fused
from test_determinism_gpu import _sms
from test_persistent_gpu import conv3x3_halo_launch, conv3x3_tc_launch, kernels_ran, pack_conv3x3

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
ENULL, EINVAL = -5, -1


def _st():
    return torch.cuda.current_stream().cuda_stream


def _cpu_gen(seed):
    return torch.Generator().manual_seed(seed)


def _ints(shape, lo, hi, g, dtype=torch.float32):
    return torch.randint(lo, hi + 1, shape, generator=g).to(dtype).to(DEV)


def _scale_shift(n, g):
    """arbitrary fp32 folded-BatchNorm constants: |scale| in [1/4, 2) of either sign, shift ~ N(0, 2)"""
    sign = torch.randint(0, 2, (n,), generator=g).float() * 2 - 1
    scale = sign * (0.25 + 1.75 * torch.rand(n, generator=g))
    return scale.to(DEV), (2 * torch.randn(n, generator=g)).to(DEV)


# ================================================================================================ the key convolution
# (C, H, B, bn): groups 4 as in CotLayer.key_embed; {-1, 0, 1} operands: |acc| <= 9 * C / 4 (at most 1152), exact
CONV_CASES = [
    (256, 14, 67, 64),      # stage 3: haloed kernel, 4 N tiles, R = 14, MB = 2
    (512, 7, 65, 128),      # stage 4: conv mode, two samples per M tile, odd B -> a half-empty last tile
    (128, 28, 9, 64),       # stage 2, for contrast: haloed kernel, 2 N tiles
]


def _conv_plan(C, H, B, bn):
    assert S.conv_tile(C, 4) == bn
    if bn == 64:
        plan = conv3x3_halo_launch(B, H, H, C, _sms())
        assert plan is not None and plan.info["n_tiles"] == C // 64
        if C == 256:
            assert plan.info["R"] == 14 and -(-(plan.info["R"] * (H + 2)) // 128) == 2     # 14 padded rows of 16: two M blocks
        return plan
    plan = conv3x3_tc_launch(B, H, H, C, bn, False, _sms())
    assert plan.info["bbox"] == 2 and B % 2 == 1, plan
    return plan


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "C%d-%dx%d-B%d-bn%d" % (c[0], c[1], c[1], c[2], c[3]))
def test_key_conv_eval_epilogue_exact(case):
    key_conv_exact(case, _conv_plan(*case))


def key_conv_exact(case, plan):
    """cotb200_conv3x3_bf16 on {-1, 0, 1} operands at (C, H, B, bn), with and without ReLU: torch.equal to the epilogue of the exact
    accumulator, and the planned kernel ran"""
    C, H, B, bn = case
    print("key conv %s: %s" % (case, plan))
    g = _cpu_gen(C + H + B)
    cg = C // 4
    x = _ints((B, H, H, C), -1, 1, g, BF)
    w = _ints((C, cg, 3, 3), -1, 1, g, BF)
    scale, shift = _scale_shift(C, g)
    wp = pack_conv3x3(w, 4, bn)
    lib = _lib.load()
    outs = {}
    with kernels_ran(plan.name):
        for relu in (1, 0):
            D = torch.full((B, H, H, C), float("nan"), dtype=BF, device=DEV)
            _lib.check(lib.cotb200_conv3x3_bf16(B, H, H, C, x.data_ptr(), C, wp.data_ptr(), bn, D.data_ptr(), C, scale.data_ptr(),
                                                shift.data_ptr(), relu, None, None, _st()), "conv3x3_bf16")
            outs[relu] = D
    torch.cuda.synchronize()
    acc = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), padding=1, groups=4).permute(0, 2, 3, 1)
    for relu, D in outs.items():
        S.equal(D, S.epilogue_ref(acc, scale, shift, relu).to(BF), "key conv %s relu=%d (%s)" % (case, relu, plan))


# ================================================================================================ the 1x1 GEMM epilogues
# the CoT layer's three 1x1 convolutions at dim C and H x H, B = 3 (a partial last M tile at every stage)
STAGES = [(64, 56), (128, 28), (256, 14), (512, 7)]
GEMM_FORMS = {
    # name: (K1, K2, N, scale, shift, relu) as functions of C
    "embed0": lambda C: (C, C, C // 2, True, True, True),          # x and k as two operand pairs, folded BN + ReLU
    "embed3": lambda C: (C // 2, 0, 9 * C // 8, False, True, False),  # shift-only: the bias, no BatchNorm
    "conv1x1": lambda C: (C, 0, C, True, True, False),           # folded BN, no ReLU
}


@pytest.mark.parametrize("form", sorted(GEMM_FORMS))
@pytest.mark.parametrize("stage", STAGES, ids=lambda s: "C%d-%dx%d" % (s[0], s[1], s[1]))
def test_gemm_eval_epilogue_exact(stage, form):
    C, H = stage
    gemm_exact(C, 3 * H * H, form)


def gemm_exact(C, M, form, pad_cols=0):
    """cotb200_gemm_bf16 in the epilogue form `form` of a dim-C CoT layer on M rows of {-1, 0, 1} operands: torch.equal to the
    epilogue of the exact accumulator.  pad_cols > 0: D is the left part of a [M, N + pad_cols] buffer (ldd = N + pad_cols) whose
    columns past N hold a pattern the kernel must leave as it is."""
    K1, K2, N, has_scale, has_shift, relu = GEMM_FORMS[form](C)
    g = _cpu_gen(C + K1 + N)
    a1, b1 = _ints((M, K1), -1, 1, g, BF), _ints((N, K1), -1, 1, g, BF)
    a2 = _ints((M, K2), -1, 1, g, BF) if K2 else None
    b2 = _ints((N, K2), -1, 1, g, BF) if K2 else None
    scale, shift = _scale_shift(N, g)
    scale = scale if has_scale else None
    shift = shift if has_shift else None
    ldd = N + pad_cols
    buf = torch.full((M, ldd), float("nan"), dtype=BF, device=DEV)
    if pad_cols:
        buf[:, N:] = _ints((M, pad_cols), -100, 100, g, BF)
    outside = buf[:, N:].clone()
    lib = _lib.load()
    with kernels_ran("tc_gemm_1x1"):
        _lib.check(lib.cotb200_gemm_bf16(M, N, K1, a1.data_ptr(), K1, b1.data_ptr(), K1, K2, _lib.ptr(a2), K2, _lib.ptr(b2), K2,
                                         buf.data_ptr(), ldd, _lib.ptr(scale), _lib.ptr(shift), 1 if relu else 0, None, None, _st()),
                   "gemm_bf16")
    torch.cuda.synchronize()
    acc = a1.double() @ b1.double().t()
    if K2:
        acc = acc + a2.double() @ b2.double().t()
    what = "gemm %s at C=%d (M=%d N=%d K=%d+%d ldd=%d)" % (form, C, M, N, K1, K2, ldd)
    S.equal(buf[:, :N], S.epilogue_ref(acc, scale, shift, relu).to(BF), what)
    S.equal(buf[:, N:], outside, what + ": columns past N")


# ================================================================================================ cotb200_se_eval
# (B, C, A, biases): fc1 is [B, C] x [C, A] (K = C, J = A), fc2 [B, A] x [A, 2C] (K = A, J = 2C); tiles of 16 samples x 32 outputs,
# K staged in chunks of 256 with 16-byte loads when K % 4 == 0
SE_CASES = [
    (1, 64, 32, True),          # stage 1 (attn_chs = max(C / 2, 32))
    (15, 128, 64, False),       # B < 16; b0 = b3 = NULL
    (16, 256, 128, True),       # one whole sample tile
    (17, 512, 256, True),       # a second sample tile with one sample
    (257, 2048, 1024, True),    # many tiles, fc1 K = 8 chunks
    (17, 64, 33, True),         # odd A: the j + 1 < J guard of fc1; fc2 K = 33 on the scalar staging branch
    (16, 257, 300, False),      # fc1 K = 257 (scalar branch, a 1-wide last chunk); fc2 K = 300 (16-byte branch, 44-wide last chunk)
    (15, 300, 257, True),       # fc1 K = 300; fc2 K = 257 (scalar branch); odd A
    (16, 66, 512, True),        # C % 4 != 0 (fc1 scalar branch); fc2 K = 512, two whole chunks
]
SE_IDS = ["B%d-C%d-A%d-%s" % (c[0], c[1], c[2], "bias" if c[3] else "nobias") for c in SE_CASES]
INV_HW_EXACT = 2.0 ** -3


def _se_call(B, C, A, psum, inv_hw, w0, b0, s1, t1, w3, b3):
    lib = _lib.load()
    assert lib.cotb200_se_eval_scratch_bytes(B, A) == B * A * 4
    a = torch.full((B, C, 2), float("nan"), device=DEV)
    z = torch.full((B, A), float("nan"), device=DEV)
    with kernels_ran("se_eval"):
        _lib.check(lib.cotb200_se_eval(B, C, A, psum.data_ptr(), inv_hw, w0.data_ptr(), _lib.ptr(b0), s1.data_ptr(), t1.data_ptr(),
                                       w3.data_ptr(), _lib.ptr(b3), a.data_ptr(), z.data_ptr(), _st()), "se_eval")
    torch.cuda.synchronize()
    return a, z


def _se_exact_inputs(B, C, A, bias, g):
    """integer psum, inv_hw = 2^-3, integer W0 / b0, power-of-two s1 (either sign), integer t1, W3 / b3 integers times 2^-6: every
    product and partial sum of both GEMVs is a dyadic rational that fp32 holds exactly (asserted in the test)"""
    psum = _ints((B, C), -3, 3, g)
    w0 = _ints((A, C), -1, 1, g)
    b0 = _ints((A,), -4, 4, g) if bias else None
    s1 = (2.0 ** -torch.randint(4, 7, (A,), generator=g).float() * (torch.randint(0, 4, (A,), generator=g) > 0).float().mul(2).sub(1)).to(DEV)
    t1 = _ints((A,), -2, 2, g)
    w3 = _ints((2 * C, A), -2, 2, g) * 2.0 ** -6
    b3 = _ints((2 * C,), -4, 4, g) * 2.0 ** -6 if bias else None
    return psum, w0, b0, s1, t1, w3, b3


@pytest.mark.parametrize("case", SE_CASES, ids=SE_IDS)
def test_se_eval_exact_hidden_and_expf_bound(case):
    """hidden activations torch.equal to fp64; the attention weights within the __expf softmax bound of the exact logits"""
    B, C, A, bias = case
    psum, w0, b0, s1, t1, w3, b3 = _se_exact_inputs(B, C, A, bias, _cpu_gen(B * C + A))
    a, z = _se_call(B, C, A, psum, INV_HW_EXACT, w0, b0, s1, t1, w3, b3)
    what = "se_eval %s" % (case,)
    p = psum.double() * INV_HW_EXACT
    zero = lambda n: torch.zeros(n, dtype=torch.float64, device=DEV)          # noqa: E731
    bb0, bb3 = (b0.double() if bias else zero(A)), (b3.double() if bias else zero(2 * C))
    # exactness premise: every partial sum of fc1 is a multiple of 2^-3 below 2^21 in magnitude, every partial sum of fc2 a multiple
    # of 2^-15 below 2^9 (bounded by sum|terms|), so fp32 holds each one exactly
    assert float((p.abs() @ w0.double().abs().t() + bb0.abs()).max()) < 2.0 ** 21
    z1 = p @ w0.double().t() + bb0
    h = torch.relu(z1 * s1.double() + t1.double())
    assert float((h.abs() @ w3.double().abs().t() + bb3.abs()).max()) < 2.0 ** 9
    S.equal(z, h.float(), what + " hidden activations (z_scratch)")
    u = (h @ w3.double().t() + bb3).view(B, C, 2)
    ref, bound = S.softmax2_fast_ref(u, torch.zeros_like(u))
    S.within(a, ref, bound, what + " attention weights")
    # the two outputs of a pair are not interchangeable: the larger logit takes the larger weight
    big = (u[..., 0] - u[..., 1]).abs() > 1e-3
    S.equal((a[..., 0] > a[..., 1])[big], (u[..., 0] > u[..., 1])[big], what + " order of the softmax pair")


def _se_module(C, A, bias, g):
    se = nn.Sequential(nn.Conv2d(C, A, 1, bias=bias), nn.BatchNorm2d(A), nn.ReLU(inplace=True), nn.Conv2d(A, 2 * C, 1, bias=bias))
    with torch.no_grad():
        for m in (se[0], se[3]):
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) / m.weight.shape[1] ** 0.5)
            if bias:
                m.bias.copy_(0.3 * torch.randn(m.bias.shape, generator=g))
        se[1].weight.copy_(0.5 + torch.rand(A, generator=g))
        se[1].bias.copy_(0.3 * torch.randn(A, generator=g))
        se[1].running_mean.copy_(2 * torch.randn(A, generator=g))
        se[1].running_var.copy_(0.1 + 3 * torch.rand(A, generator=g))
    return se.to(DEV).eval()


@pytest.mark.parametrize("case", SE_CASES, ids=SE_IDS)
def test_se_eval_random_vs_mlp_ref(case):
    """random fp32 operands through the library's own fold (fused._se_eval_params), against the fp64 MLP of the module"""
    B, C, A, bias = case
    g = _cpu_gen(7 * B + C + A)
    se = _se_module(C, A, bias, g)
    HW = 49
    psum = (HW * (0.5 + torch.randn(B, C, generator=g))).to(DEV)
    inv_hw = 1.0 / HW
    w0, b0, s1, t1, w3, b3 = fused._se_eval_params(se)
    what = "se_eval %s random" % (case,)
    # the fold against fp64 of the module (stage_ref._mlp_fwd's se_eval bound assumes these)
    fb = S.fold_bound(se[1])
    S.within(s1, fb["scale"], fb["scale_err"], what + " folded scale s1")
    S.within(t1, fb["shift"], fb["shift_err"], what + " folded shift t1")
    a, z = _se_call(B, C, A, psum, inv_hw, w0, b0, s1, t1, w3, b3)
    p = psum.double() * torch.tensor(inv_hw, dtype=torch.float32).double()             # the kernel's operands: fp32 inv_hw
    f = S._mlp_fwd(p, (se[0], se[1], se[3]), "cot", False, se_eval=True)
    S.within(z, f["h"], f["eh"], what + " hidden activations")
    ref, bound = S.mlp_ref(p, (se[0], se[1], se[3]), "cot", False, se_eval=True)
    S.within(a, ref, bound, what + " attention weights")


def test_se_eval_rejects_bad_arguments():
    lib = _lib.load()
    B, C, A = 2, 64, 32
    t = {n: torch.zeros(s, device=DEV) for n, s in (("psum", B * C), ("w0", A * C), ("s1", A), ("t1", A), ("w3", 2 * C * A),
                                                  ("a", B * C * 2), ("z", B * A))}
    ptrs = {n: v.data_ptr() for n, v in t.items()}

    def call(B=B, C=C, A=A, **over):
        p = dict(ptrs, **over)
        return lib.cotb200_se_eval(B, C, A, p["psum"], 0.25, p["w0"], None, p["s1"], p["t1"], p["w3"], None, p["a"], p["z"], _st())
    for name in ptrs:
        assert call(**{name: None}) == ENULL, name
    for dims in (dict(B=0), dict(C=0), dict(A=0), dict(B=-1), dict(C=-3), dict(A=-2)):
        assert call(**dims) == EINVAL, dims
    assert call() == 0
    assert torch.isfinite(t["a"]).all() and bool((t["a"] == 0.5).all())           # zero logits: an even split
    assert [lib.cotb200_se_eval_scratch_bytes(b, a) for b, a in ((1, 1), (3, 33), (257, 1024))] == [4, 3 * 33 * 4, 257 * 1024 * 4]


# ================================================================================================ eval tail: fold, pool, combine
@pytest.mark.parametrize("C,H,B", [(64, 56, 3), (256, 14, 5), (512, 7, 9)])
def test_tail_pool_combine_eval_fold(C, H, B):
    """_bn_eval_fold of the running statistics within a few fp32 ulp of fp64, then tail_pool and tail_combine with that fold"""
    g = _cpu_gen(C + H + B)
    bn = nn.BatchNorm2d(C)
    with torch.no_grad():
        bn.weight.copy_(torch.randn(C, generator=g))
        bn.bias.copy_(torch.randn(C, generator=g))
        bn.running_mean.copy_(2 * torch.randn(C, generator=g))
        bn.running_var.copy_(0.05 + 4 * torch.rand(C, generator=g))
    bn = bn.to(DEV).eval()
    scale, shift, mean, rstd = fused._bn_eval_fold(bn, bn.weight, bn.bias)
    fb = S.fold_bound(bn)
    for name, got in (("rstd", rstd), ("scale", scale), ("shift", shift)):
        S.within(got, fb[name], fb[name + "_err"], "eval fold " + name)
    cl = lambda t: t.to(DEV).to(BF).contiguous(memory_format=torch.channels_last)          # noqa: E731
    u = cl(torch.randn(B, C, H, H, generator=g))
    k = cl(torch.relu(torch.randn(B, C, H, H, generator=g)))
    a = torch.softmax(torch.randn(B, C, 2, generator=g), -1).to(DEV).contiguous()
    lib = _lib.load()
    psum = torch.zeros(B, C, device=DEV)
    out = torch.empty_like(u)
    dt = _lib.dtype_code(u)
    _lib.check(lib.cotb200_tail_pool(dt, B, H * H, C, u.data_ptr(), k.data_ptr(), scale.data_ptr(), shift.data_ptr(), psum.data_ptr(),
                                     _st()), "tail_pool")
    _lib.check(lib.cotb200_tail_combine(dt, B, H * H, C, u.data_ptr(), k.data_ptr(), scale.data_ptr(), shift.data_ptr(), a.data_ptr(),
                                        out.data_ptr(), _st()), "tail_combine")
    torch.cuda.synchronize()
    ps, pe, y, ye = S.tail_pool_ref(u, k, scale, shift, S.SIGMOID_ERR_16)
    S.within(psum, ps, pe, "tail_pool psum (eval fold)")
    o, oe = S.tail_combine_ref(y, ye, k, a)
    S.within(out, o, S.store_bound(o, oe, BF), "tail_combine out (eval fold)")


# ================================================================================================ eval forms of the trunk functions
def _eval_bn(C, g):
    bn = nn.BatchNorm2d(C)
    with torch.no_grad():
        bn.weight.copy_(0.5 + torch.rand(C, generator=g))
        bn.bias.copy_(torch.randn(C, generator=g))
        bn.running_mean.copy_(2 * torch.randn(C, generator=g))
        bn.running_var.copy_(0.1 + 2 * torch.rand(C, generator=g))
    return bn.to(DEV).eval()


def test_conv1x1_eval_residual_path():
    """TcConv1x1Fn in eval with a residual (the bottleneck's conv3 at stage 1): a raw GEMM into a bf16 `pre`, then cotb200_bn_apply
    with _bn_eval_fold's constants.  Integer operands keep `pre` exact; the output is within the apply's bound of fp64."""
    B, K, N, H = 3, 64, 256, 56
    g = _cpu_gen(11)
    cl = lambda t: t.contiguous(memory_format=torch.channels_last)          # noqa: E731
    a = cl(_ints((B, K, H, H), -1, 1, g, BF))
    w = _ints((N, K, 1, 1), -1, 1, g)
    res = cl(torch.randn(B, N, H, H, generator=g).to(DEV).to(BF))
    bn = _eval_bn(N, g)
    with torch.no_grad(), kernels_ran("tc_gemm_1x1", "bn_apply"):
        out = fused.TcConv1x1Fn.apply(a, None, w, None, bn.weight, bn.bias, bn, True, res)
    scale, shift, _, _ = fused._bn_eval_fold(bn, bn.weight, bn.bias)
    fb = S.fold_bound(bn)
    S.within(scale, fb["scale"], fb["scale_err"], "conv1x1 eval fold scale")
    S.within(shift, fb["shift"], fb["shift_err"], "conv1x1 eval fold shift")
    acc = F.conv2d(a.double(), w.double())
    y, err = S.bn_apply_ref(acc, scale, shift, True, res)
    S.within(out, y, S.store_bound(y, err, BF), "conv1x1 eval output (pre exact, + residual, ReLU)")


def test_stem_eval_exact():
    """StemConvBNFn in eval: the 7x7 / s2 stem with _bn_eval_fold in its epilogue; integer operands: torch.equal"""
    B, N = 2, 64
    g = _cpu_gen(12)
    x = _ints((B, 3, 224, 224), -1, 1, g, BF).contiguous(memory_format=torch.channels_last)
    w = _ints((N, 3, 7, 7), -1, 1, g)
    bn = _eval_bn(N, g)
    with torch.no_grad(), kernels_ran("tc_stem7x7"):
        out = fused.StemConvBNFn.apply(x, w, bn.weight, bn.bias, bn, True)
    scale, shift, _, _ = fused._bn_eval_fold(bn, bn.weight, bn.bias)
    acc = F.conv2d(x.double(), w.double(), stride=2, padding=3)
    ref = S.epilogue_ref(acc.permute(0, 2, 3, 1), scale, shift, True).permute(0, 3, 1, 2)
    S.equal(out, ref.to(BF), "stem eval output (integer operands)")
