"""The bf16 training step's fused autograd functions stage by stage, each stage against fp64 of the inputs it actually received
(tests/stage_ref.py): BNActFn, GroupNorm9Fn, FanOutFn, CotTailFn (forward and backward, with its MLP), AggTapFn, Pool3x3S2Fn,
TcConv1x1Fn, TcConv3x3Fn and StemConvBNFn in the configurations the CoT blocks reach, and cotnet50 CoT bottlenecks of stages 1, 2 and
4 parameter by parameter.  The DropBlock functions' checks, the CoXt, SE-CoTNetD, DropBlock, stochastic-depth and stem cases and
the derived-weight accounting are used by test_step_stages_gpu.py.  Not covered: whole-model steps.  Eval-mode flags are checked only under grad, where CotLayer takes _forward_fused and cot_tail takes
CotTailFn; the inference path (_forward_tc_eval, _cot_tail_eval, cotb200_se_eval) is tested in test_eval_kernels_gpu.py,
test_eval_stages_gpu.py and, in whole blocks and networks, test_eval_blocks_gpu.py.

Bounds are per element: 1/2 ulp of the stored dtype plus the fp32 error of the stage, with fp32 sums bounded by gamma(n) * sum|terms|
(gamma_tc(n), 2u per add, on the tensor cores) for the chain length n of the kernel.  Where operands are small integers the GEMM /
convolution outputs are exact and compared with torch.equal.  The glue inside each function is checked exactly: the returned
dgamma / dbeta are the BatchNorm backward's sums, dres is the gated incoming gradient, the tail returns its MLP's gradients, and so on."""
import copy
import zlib

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import stage_ref as S
from cotnet_b200 import _lib, fused

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
CL = torch.channels_last
ONE_ULP = {}          # stage -> [one ulp off, more than one ulp off, total] of bf16 outputs against the correctly rounded fp64 value


@pytest.fixture(autouse=True)
def _no_tf32(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cl(t):
    return t.contiguous(memory_format=CL)


def _ints(shape, g, lo=-3, hi=3, dtype=BF):
    return _cl(torch.randint(lo, hi + 1, shape, generator=g, device=DEV).to(dtype))


def _randn(shape, g, dtype=BF, scale=1.0):
    return _cl((torch.randn(shape, generator=g, device=DEV) * scale).to(dtype))


@pytest.fixture(scope="module", autouse=True)
def _report_one_ulp():
    """after the module: per stage type, the fraction of bf16 outputs exactly one ulp from the correctly rounded fp64 value (and
    how many lie farther, which the bounds allow only where a stage's fp32 error reaches an ulp)"""
    ONE_ULP.clear()
    yield
    for k in sorted(ONE_ULP):
        one, far, n = ONE_ULP[k]
        print("\nbf16 outputs one ulp off, %-10s %.2e (%d of %d; %d farther)" % (k, one / max(n, 1), one, n, far), end="")


def _note(stage, got, exact):
    if got.dtype == BF:
        d = ONE_ULP.setdefault(stage, [0, 0, 0])
        rn = S.bf16(exact.double())
        diff = (got.double() - rn).abs()
        step = S.ulp(torch.maximum(got.double().abs(), rn.abs()), 8)
        d[0] += int(((diff > 0) & (diff <= step)).sum())
        d[1] += int((diff > step).sum())
        d[2] += got.numel()


def _w(got, exact, err, what, stage=None):
    S.within(got, exact, S.store_bound(exact, err, got.dtype), what)
    if stage:
        _note(stage, got, exact)


def _unpack(mask, C):
    bits = torch.arange(8, device=mask.device, dtype=torch.uint8)
    return ((mask.unsqueeze(-1) >> bits) & 1).reshape(mask.shape[0], -1)[:, :C].bool()


def _rows_of(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


# ------------------------------------------------------------------------------------------------ BatchNorm stages
def check_apply(cap, what):
    """_bn_apply_batch: the producer's column sums, the rsqrt prologue, y from the captured scale / shift, mask and running buffers"""
    x, n, ss, sums = cap["x"], cap["n"], cap["ss"], cap["sums"]
    s0, s1, sabs = S.bn_stats_ref(x, n)
    xd = x.double()
    hu = 0.5 * S.ulp(xd.abs() * 1.01, 8) if x.dtype == BF else torch.zeros_like(xd)   # the sums may come from the fp32 accumulator
    S.within(sums[0], s0, S.gamma(n + 1) * sabs + hu.sum((0, 2, 3)), what + " column sums")
    S.within(sums[1], s1, S.gamma(n + 1) * (xd * xd).sum((0, 2, 3)) + (hu * (2 * xd.abs() + hu)).sum((0, 2, 3)), what + " column sq sums")
    m64 = sums[0].double() / n
    e2 = sums[1].double() / n
    var64 = (e2 - m64 * m64).clamp_min(0.0)
    var_err = 3 * S.U32 * (e2 + m64 * m64)
    r64 = 1.0 / torch.sqrt(var64 + cap["eps"])
    S.within(ss[2], m64, S.ulp(m64, 24), what + " mean")
    S.within(ss[3], r64, 0.5 * r64 * var_err / (var64 + cap["eps"]) * 1.01 + 4 * S.ulp(r64, 24), what + " rstd")
    w, b = cap["weight"].double(), cap["bias"].double()
    S.within(ss[0], w * ss[3].double(), S.ulp(w * ss[3].double(), 24), what + " scale")
    sh = b - ss[2].double() * ss[0].double()
    S.within(ss[1], sh, 2 * S.U32 * (b.abs() + (ss[2].double() * ss[0].double()).abs()) * 2 + S.ulp(sh, 24), what + " shift")
    y, err = S.bn_apply_ref(x, ss[0], ss[1], cap["relu"], cap["res"], cap["ds"])
    _w(cap["y"], y, err, what + " y", "bn_apply")
    if cap["mask"] is not None:
        S.equal(_unpack(cap["mask"], x.shape[1]), _rows_of(cap["y"]) > 0, what + " 1-bit mask == (y > 0)")
    if cap["rm0"] is not None:
        mom = cap["momentum"] if cap["momentum"] is not None else 1.0 / cap["nbt"]
        rm = (1 - mom) * cap["rm0"].double() + mom * m64
        bdt = cap["rm1"].dtype                # fp32 update, then the module's buffer dtype
        S.within(cap["rm1"], rm, S.store_bound(rm, 4 * S.U32 * ((1 - mom) * cap["rm0"].double().abs() + mom * m64.abs()) + S.ulp(rm, 24),
                                               bdt), what + " running_mean")
        c = mom * n / max(n - 1, 1)
        rv = (1 - mom) * cap["rv0"].double() + c * var64
        S.within(cap["rv1"], rv, S.store_bound(rv, c * var_err + 4 * S.U32 * ((1 - mom) * cap["rv0"].double().abs() + c * var64)
                                               + S.ulp(rv, 24), bdt), what + " running_var")


def check_bwd(cap, y_fwd, what):
    """_bn_bwd: ReLU decision from the library's own forward output, dres exact, the dgamma / dbeta sums, dx from the captured sums"""
    rc = cap["rcode"]
    gate = None if rc == 0 else (y_fwd > 0)
    if rc == 1:
        S.equal(cap["y"], y_fwd, what + " saved y")
    if rc == 3:
        S.equal(_unpack(cap["y"], y_fwd.shape[1]), _rows_of(y_fwd) > 0, what + " saved mask == (y > 0)")
    r = S.bn_bwd_ref(cap["dy"], cap["x"], gate, cap["scale"], cap["mean"], cap["rstd"], cap["sums"], cap["batch"], cap["ds"])
    M = cap["B"] * cap["HW"]
    if cap["dres"] is not None:
        S.equal(cap["dres"], r["dres"].to(cap["dres"].dtype), what + " dres = dy * relu'")
    if cap["sums"] is not None:
        S.within(cap["sums"][0], r["s0"], S.gamma(M + 1) * r["s0_abs"], what + " dbeta sum")
        S.within(cap["sums"][1], r["s1"], S.gamma(M + 1) * r["s1_abs"], what + " dgamma sum")
    _w(cap["dx"], r["dx"], r["dx_err"], what + " dx", "bn_bwd")


def _bn_glue(call, bwd, i_w, i_b, what):
    g = call.gout
    if g[i_w] is not None:
        S.equal(g[i_w], bwd["sums"][1].to(call.args[i_w].dtype), what + " returned dgamma = the dgamma sum")
    if g[i_b] is not None:
        S.equal(g[i_b], bwd["sums"][0].to(call.args[i_b].dtype), what + " returned dbeta = the dbeta sum")


def check_bnact(call, what="BNActFn"):
    x, weight, bias, res, bn, relu, ds = call.inp
    if call.apply is not None:
        check_apply(call.apply, what)
    else:                                   # eval: running statistics folded by bn_finalize, then bn_apply
        ss = call.saved[2]
        r64 = 1.0 / torch.sqrt(bn.running_var.double() + bn.eps)
        S.within(ss[3], r64, 4 * S.ulp(r64, 24), what + " eval rstd")
        y, err = S.bn_apply_ref(x, ss[0], ss[1], relu, res, ds)
        _w(call.out, y, err, what + " eval y", "bn_apply")
    if call.gout is not None:
        check_bwd(call.bwd, call.out, what + " backward")
        S.equal(call.gout[0], call.bwd["dx"], what + " returned dx")
        _bn_glue(call, call.bwd, 1, 2, what)
        if call.gout[3] is not None:
            S.equal(call.gout[3], call.bwd["dres"], what + " returned dres")


# ------------------------------------------------------------------------------------------------ wgmma functions
def _dw_bound(ref, mag, n_chain, mm, wdtype):
    if mm:      # torch.mm / cuDNN on bf16 operands: bf16 result, any order of the M terms
        err = S.store_bound(ref, S.gamma_tc(n_chain) * mag, BF)
    else:       # wgmma kernel: fp32, the pinned chain
        err = S.gamma_tc(n_chain) * mag
    return S.store_bound(ref, err, wdtype) if wdtype != torch.float32 else err


def check_tc1x1(call, what="TcConv1x1Fn", exact=False):
    a1, a2, weight, _, bn_w, bn_b, bn, relu, res, ds = tuple(call.inp) + (None,) * (10 - len(call.inp))
    N = weight.shape[0]
    K1 = a1.shape[1]
    K2 = 0 if a2 is None else a2.shape[1]
    B, _, H, W = a1.shape
    M = B * H * W
    wb = weight.reshape(N, K1 + K2).to(BF)
    ws = [wb[:, :K1]] + ([wb[:, K1:]] if K2 else [])
    acc, mag = S.gemm_ref([a1] + ([a2] if K2 else []), ws)
    err = S.gamma_tc(K1 + K2 + 1) * mag
    pre = call.apply["x"] if call.apply is not None else (call.saved[3] if bn is not None else call.out)
    if pre is not None:
        if exact:
            S.equal(pre, acc.to(BF), what + " GEMM output (integer operands)")
        _w(pre, acc, err, what + " GEMM output", "gemm")
    if call.apply is not None:
        check_apply(call.apply, what)
    elif bn is not None:                    # eval: BatchNorm folded into the epilogue (no residual) or applied to pre
        scale, mean = call.saved[5], call.saved[7]
        shift = bn_b.double() - mean.double() * scale.double()
        sh_err = 2 * S.U32 * (bn_b.double().abs() + (mean.double() * scale.double()).abs())
        if res is None and ds is None:
            y, yerr = S.bn_apply_ref(acc, scale, shift, relu)
            yerr = yerr + scale.double().abs().view(1, -1, 1, 1) * err + sh_err.view(1, -1, 1, 1)
        else:
            y, yerr = S.bn_apply_ref(pre, scale, shift, relu, res, ds)
            yerr = yerr + sh_err.view(1, -1, 1, 1) * (1 if ds is None else ds.double().abs().view(-1, 1, 1, 1))
        _w(call.out, y, yerr, what + " eval output", "bn_apply")
    if call.gout is None:
        return
    dy = call.gin[0]
    if bn is not None:
        check_bwd(call.bwd, call.out, what + " backward")
        dpre = call.bwd["dx"]
        _bn_glue(call, call.bwd, 4, 5, what)
        if call.gout[8] is not None:
            S.equal(call.gout[8], call.bwd["dres"], what + " returned dres")
    else:
        dpre = dy
    dp = S.rows(dpre)
    for i, (a, wcols) in enumerate(((a1, ws[0]),) + (((a2, ws[1]),) if K2 else ())):
        if call.gout[i] is None:
            continue
        ref = (dp @ wcols.double()).view(B, H, W, -1).permute(0, 3, 1, 2)
        m2 = (dp.abs() @ wcols.double().abs()).view(B, H, W, -1).permute(0, 3, 1, 2)
        if exact and bn is None:
            S.equal(call.gout[i], ref.to(BF), what + " da%d (integer operands)" % (i + 1))
        _w(call.gout[i], ref, S.gamma_tc(N + 1) * m2, what + " da%d" % (i + 1), "gemm_dgrad")
    if call.gout[2] is not None:
        arow = torch.cat([S.rows(a1)] + ([S.rows(a2)] if K2 else []), 1)
        ref, m2 = dp.t() @ arow, dp.abs().t() @ arow.abs()
        mm = S.mm_wgrad(N, K1 + K2, M)
        n = M + 1 if mm else S.wgrad_chain(M, N, K1, K2, _sms())
        got = call.gout[2].reshape(N, K1 + K2)
        if exact and bn is None and not mm:
            S.equal(got.double(), ref, what + " dW (integer operands)")
        S.within(got, ref, _dw_bound(ref, m2, n, mm, got.dtype), what + " dW (%s)" % ("torch.mm" if mm else "wgmma"))
        assert got.dtype == weight.dtype


def check_tc3x3(call, what="TcConv3x3Fn", exact=False):
    x, weight, bn_w, bn_b, bn, groups, relu = call.inp
    C, cg = weight.shape[0], weight.shape[1]
    w64 = weight.to(BF).double()
    acc = F.conv2d(x.double(), w64, padding=1, groups=groups)
    mag = F.conv2d(x.double().abs(), w64.abs(), padding=1, groups=groups)
    err = S.gamma_tc(9 * cg + 1) * mag
    pre = call.apply["x"] if call.apply is not None else call.saved[2]
    if pre is not None:
        if exact:
            S.equal(pre, acc.to(BF), what + " conv output (integer operands)")
        _w(pre, acc, err, what + " conv output", "conv")
    if call.apply is not None:
        check_apply(call.apply, what)
    else:
        scale, mean = call.saved[4], call.saved[6]
        shift = bn_b.double() - mean.double() * scale.double()
        y, yerr = S.bn_apply_ref(acc, scale, shift, relu)
        yerr = yerr + scale.double().abs().view(1, -1, 1, 1) * err + (2 * S.U32 * (bn_b.double().abs() + (mean.double() * scale.double()).abs())).view(1, -1, 1, 1)
        _w(call.out, y, yerr, what + " eval output", "bn_apply")
    if call.gout is None:
        return
    check_bwd(call.bwd, call.out, what + " backward")
    _bn_glue(call, call.bwd, 2, 3, what)
    dpre = call.bwd["dx"].double()
    if call.gout[0] is not None:
        ref = torch.nn.grad.conv2d_input(x.shape, w64, dpre, padding=1, groups=groups)
        m2 = torch.nn.grad.conv2d_input(x.shape, w64.abs(), dpre.abs(), padding=1, groups=groups)
        _w(call.gout[0], ref, S.gamma_tc(9 * cg + 1) * m2, what + " dx", "conv_dgrad")
    if call.gout[1] is not None:     # cuDNN grouped wgrad: bf16 result, M terms per element
        ref = torch.nn.grad.conv2d_weight(x.double(), weight.shape, dpre, padding=1, groups=groups)
        m2 = torch.nn.grad.conv2d_weight(x.double().abs(), weight.shape, dpre.abs(), padding=1, groups=groups)
        M = x.shape[0] * x.shape[2] * x.shape[3]
        S.within(call.gout[1], ref, _dw_bound(ref, m2, M + 1, True, call.gout[1].dtype), what + " dW (cuDNN)")


def check_stem(call, what="StemConvBNFn", exact=False):
    x, weight, bn_w, bn_b, bn, relu = call.inp
    w64 = weight.to(BF).double()
    acc = F.conv2d(x.double(), w64, stride=2, padding=3)
    mag = F.conv2d(x.double().abs(), w64.abs(), stride=2, padding=3)
    err = S.gamma_tc(148) * mag
    pre = call.apply["x"] if call.apply is not None else call.saved[2]
    if pre is not None:
        if exact:
            S.equal(pre, acc.to(BF), what + " conv output (integer operands)")
        _w(pre, acc, err, what + " conv output", "conv")
    if call.apply is not None:
        check_apply(call.apply, what)
    else:
        scale, mean = call.saved[4], call.saved[6]
        shift = bn_b.double() - mean.double() * scale.double()
        y, yerr = S.bn_apply_ref(acc, scale, shift, relu)
        yerr = yerr + scale.double().abs().view(1, -1, 1, 1) * err + (2 * S.U32 * (bn_b.double().abs() + (mean.double() * scale.double()).abs())).view(1, -1, 1, 1)
        _w(call.out, y, yerr, what + " eval output", "bn_apply")
    if call.gout is None:
        return
    check_bwd(call.bwd, call.out, what + " backward")
    _bn_glue(call, call.bwd, 2, 3, what)
    if call.gout[1] is not None:
        dpre = call.bwd["dx"].double()
        ref = torch.nn.grad.conv2d_weight(x.double(), weight.shape, dpre, stride=2, padding=3)
        m2 = torch.nn.grad.conv2d_weight(x.double().abs(), weight.shape, dpre.abs(), stride=2, padding=3)
        B, _, H, W = x.shape
        tc = S.stem_wgrad_tc(H, W, weight.shape[0]) and call.apply is not None
        n = S.stem_wgrad_chain(B, H // 2, W // 2, _sms()) if tc else B * (H // 2) * (W // 2) + 1
        S.within(call.gout[1], ref, _dw_bound(ref, m2, n, not tc, call.gout[1].dtype), what + " dW (%s)" % ("wgmma" if tc else "cuDNN"))


# ------------------------------------------------------------------------------------------------ row functions
def check_gn9(call, what="GroupNorm9Fn"):
    l, gamma_, beta, eps, gc, lbias = call.inp
    _, mean, rstd, _, _ = call.saved
    B, J, H, W = l.shape
    out, err, xh, (m64, m_err, r64, r_err) = S.gn9_ref(l, lbias, gamma_, beta, mean, rstd, gc, eps)
    S.within(mean.view(B, -1), m64, m_err, what + " mean")
    S.within(rstd.view(B, -1), r64, r_err, what + " rstd")
    _w(call.out, out, err, what + " output", "gn9")
    if call.gout is None:
        return
    dg = S.from_storage(call.gin[0].double(), gc)
    r = S.gn9_bwd_ref(dg, xh, gamma_, rstd, 9 * H * W)
    n = H * W + B + 1                       # per-sample column partials, then the B samples
    xh_err = 8 * S.U32 * (r["dgamma_abs"] + r["dbeta_abs"])
    if call.gout[0] is not None:
        _w(call.gout[0], r["dl"], r["dl_err"], what + " dl", "gn9_bwd")
    for i, key, extra in ((1, "dgamma", xh_err), (2, "dbeta", 0.0)):
        S.within(call.gout[i], r[key], S.store_bound(r[key], S.gamma(n) * r[key + "_abs"] + extra, call.gout[i].dtype)
                 if call.gout[i].dtype != torch.float32 else S.gamma(n) * r[key + "_abs"] + extra, what + " " + key)
    if lbias is not None and call.gout[5] is not None:
        e = S.gamma(n) * r["dlbias_abs"] + r["dlbias_err"]
        S.within(call.gout[5], r["dlbias"], e if call.gout[5].dtype == torch.float32 else S.store_bound(r["dlbias"], e, call.gout[5].dtype),
                 what + " dlbias")


def check_tail(call, mods, kind, what="CotTailFn"):
    """forward: pooled descriptor from the captured scale / shift, the fp32 attention MLP against fp64 of that descriptor, output;
    backward: S, the MLP backward at the recorded descriptor and S, dgamma / dbeta, du and dk"""
    u, k = call.inp[0], call.inp[1]
    _, _, scale, shift, mean, rstd, a_c = call.saved
    B, C, H, W = u.shape
    es = S.SIGMOID_ERR_16 if u.dtype != torch.float32 else S.SIGMOID_ERR_32
    z = u.double() * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    ze = 4 * S.U32 * ((u.double() * scale.double().view(1, -1, 1, 1)).abs() + shift.double().abs().view(1, -1, 1, 1))
    y = F.silu(z)
    ye = z.abs() * es + 1.1 * ze + 4 * S.U32 * y.abs()
    t = y + (0 if k is None else k.double())
    p = t.mean((2, 3))
    pe = (ye.sum((2, 3)) + S.gamma(H * W + 1) * t.abs().sum((2, 3))) / (H * W) + S.ulp(p, 24)
    S.within(call.extra["p"], p, pe, what + " pooled mean")
    a, ea = S.mlp_ref(call.extra["p"], mods, kind, call.extra["training"])
    S.within(a_c, a, ea, what + " attention weights (fp32 MLP)")
    a0, a1 = a_c[..., 0].double().view(B, C, 1, 1), a_c[..., 1].double().view(B, C, 1, 1)
    o = a0 * y + (0 if k is None else a1 * k.double())
    oe = a0.abs() * ye + 4 * S.U32 * (o.abs() + (0 if k is None else (a1 * k.double()).abs()))
    _w(call.out, o, oe, what + " output", "tail")
    if call.gout is None:
        return
    # backward, stage by stage: tail_bwd_sums -> S; the fp32 MLP backward at the recorded p and S -> d/dp and the MLP's parameter
    # gradients; tail_bwd_dz_sums + tail_bwd_apply at the recorded d/dp -> dbeta, dgamma, du, dk
    Scap, mg = call.extra["S"], call.extra["mlp_grads"]
    r = S.tail_bwd_ref(u, k, scale, shift, mean, rstd, a_c, call.gin[0], mg[0], call.extra["training"], es)
    S.within(Scap[..., 0], r["S0"], r["S0_err"] + S.ulp(r["S0"], 24), what + " S[..., 0] = sum dout * y")
    if k is not None:
        S.within(Scap[..., 1], r["S1"], r["S1_err"] + S.ulp(r["S1"], 24), what + " S[..., 1] = sum dout * k")
    (dp, e_dp), prm = S.mlp_bwd_ref(call.extra["p"], Scap, mods, kind, call.extra["training"])
    S.within(mg[0], dp, e_dp + S.ulp(dp, 24), what + " MLP d/dp")
    params = call.args[6:]
    assert len(params) == len(prm) == len(mg) - 1
    for i, (pt, (ref, err)) in enumerate(zip(params, prm)):
        got = call.gout[6 + i]
        S.equal(got, mg[1 + i], what + " returned MLP gradient %d = the MLP backward's" % i)
        ref, err = ref.reshape(pt.shape), err.reshape(pt.shape)
        S.within(got, ref, S.store_bound(ref, err, got.dtype), what + " MLP parameter gradient %d" % i)
    for i, key in ((2, "dgamma"), (3, "dbeta")):
        got = call.gout[i]
        S.within(got, r[key], S.store_bound(r[key], r[key + "_err"], got.dtype), what + " returned " + key)
    _w(call.gout[0], r["du"], r["du_err"], what + " du", "tail_bwd")
    if k is not None:
        _w(call.gout[1], r["dk"], r["dk_err"], what + " dk", "tail_bwd")


def check_fanout(call, what="FanOutFn"):
    if call.gout is None:
        return
    gs = [g for g in call.gin if g is not None]
    if len(gs) == 1:
        S.equal(call.gout[0], gs[0], what + " single gradient passed through")
        return
    ref = sum(g.double() for g in gs)
    mag = sum(g.double().abs() for g in gs)
    _w(call.gout[0], ref, S.gamma(len(gs)) * mag, what + " sum of %d gradients" % len(gs), "fan_out")


def check_agg(call, what="AggTapFn"):
    v, w, fold, gc = call.inp
    ref, mag = S.agg_ref(v, w, fold, gc)
    _w(call.out, ref, S.gamma(10) * mag, what + " output", "agg")
    if call.gout is None:
        return
    v64, w64 = v.double().requires_grad_(True), w.double().requires_grad_(True)
    va, wa = v.double().abs().requires_grad_(True), w.double().abs().requires_grad_(True)
    dy = call.gin[0].double()
    dv, dw = torch.autograd.grad((S.agg_ref(v64, w64, fold, gc)[0] * dy).sum(), [v64, w64])
    mv, mw = torch.autograd.grad((S.agg_ref(va, wa, fold, gc)[0] * dy.abs()).sum(), [va, wa])
    _w(call.gout[0], dv, S.gamma(10) * mv, what + " dv", "agg_bwd")
    _w(call.gout[1], dw, S.gamma(17) * mw, what + " dw", "agg_bwd")


def check_pool(call, what="Pool3x3S2Fn"):
    x, mode = call.inp
    B, C, H, W = x.shape
    if mode == 0:
        # NCHW-contiguous reference: ATen's channels_last avg_pool2d backward on CUDA disagrees with its NCHW form (see test_fused_gpu)
        x64 = x.double().contiguous().requires_grad_(True)
        ref = F.avg_pool2d(x64, 3, 2, 1, count_include_pad=True)
        mag = F.avg_pool2d(x.double().abs().contiguous(), 3, 2, 1, count_include_pad=True)
        _w(call.out, ref, S.gamma(10) * mag, what + " avg output", "pool")
        if call.gout is not None:
            dy = call.gin[0].double().contiguous()
            dx = torch.autograd.grad((ref * dy).sum(), x64)[0]
            xa = x.double().abs().contiguous().requires_grad_(True)
            m2 = torch.autograd.grad((F.avg_pool2d(xa, 3, 2, 1, count_include_pad=True) * dy.abs()).sum(), xa)[0]
            _w(call.gout[0], dx, S.gamma(5) * m2, what + " avg dx", "pool_bwd")
        return
    S.equal(call.out, F.max_pool2d(x.double(), 3, 2, 1).to(x.dtype), what + " max output")
    (idx,) = call.saved
    Ho, Wo = call.out.shape[2:]
    xp = F.pad(x.double(), (1, 1, 1, 1), value=float("-inf"))
    dxp = torch.zeros_like(xp)
    dy = call.gin[0].double() if call.gout is not None else None
    for t in range(9):
        kh, kw = divmod(t, 3)
        sel = (idx.permute(0, 3, 1, 2) == t)
        win = xp[:, :, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2]
        assert bool((win[sel] == call.out.double()[sel]).all()), what + " index does not point at the maximum"
        if dy is not None:
            dxp[:, :, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] += dy * sel
    if dy is not None:
        S.equal(call.gout[0], dxp[:, :, 1:H + 1, 1:W + 1].to(x.dtype), what + " max dx routed by the saved index")


def _dropblock_mask(call, x, mask, count, what):
    """the call's mask and count against dropblock.host_mask for the (key, site, DropBlock) its caller passed; returns the keep
    mask [B, C, H, W] (fp64, 0 / 1) and the scale as the kernels apply it: fp32 s rounded to the activation dtype"""
    from cotnet_b200 import dropblock
    e = call.extra
    keep, cnt, s = dropblock.host_mask(tuple(x.shape), e["site"], e["key"], e["spec"])
    m = torch.from_numpy(keep).to(DEV)
    S.equal(_unpack(mask, x.shape[1]), _rows_of(m), what + " mask == host_mask(key, site %d)" % e["site"])
    assert int(count.item()) == cnt, "%s: count %d, host count %d" % (what, int(count.item()), cnt)
    s64 = torch.tensor(float(s), dtype=torch.float64)
    sb = S.bf16(s64) if x.dtype == BF else (s64 if x.dtype == torch.float32 else s64.to(x.dtype).double())
    return m.double(), float(sb)


def check_dropblock(call, what="DropBlockFn"):
    """y = x * M * s: x * s of two bf16 values is exact in fp32 and fp64, so the one rounding to bf16 is the whole error and y is
    compared bit for bit; the backward is the same map on dy"""
    x, mask, count = call.inp
    m, s = _dropblock_mask(call, x, mask, count, what)
    rnd = S.bf16 if x.dtype == BF else S.f32
    S.equal(call.out.double(), rnd(x.double() * m * s), what + " y = bf16(x * M * s)")
    if call.gout is not None:
        S.equal(call.gout[0].double(), rnd(call.gin[0].double() * m * s), what + " dx = bf16(dy * M * s)")


def check_dropblock_res_relu(call, what="DropBlockResReluFn"):
    """y = relu(res + ds[b] * (z * M * s)): z * s is exact in fp32, then one fma (or add): 1/2 ulp of fp32 of |res + ds*a|, then
    the bf16 store.  dres = dy * [y > 0] exactly; dz = dres * ds[b] * M * s: fl(fl(g * s) * d), the first product exact."""
    z, res, mask, count, ds = call.inp
    m, s = _dropblock_mask(call, z, mask, count, what)
    d = ds.double().view(-1, 1, 1, 1) if ds is not None else 1.0
    v = res.double() + d * (z.double() * m * s)
    _w(call.out, torch.relu(v), S.U32 * v.abs(), what + " y", "dropblock_res_relu")
    if call.gout is None:
        return
    dy = call.gin[0].double()
    dres = dy * (call.out > 0).double()
    if call.gout[1] is not None:
        S.equal(call.gout[1].double(), dres, what + " dres = dy * [y > 0]")
    dz = dres * d * m * s
    _w(call.gout[0], dz, S.U32 * dz.abs(), what + " dz", "dropblock_res_relu_bwd")


def check_call(call, mods=None):
    n = call.name
    if n == "BNActFn":
        check_bnact(call)
    elif n == "TcConv1x1Fn":
        check_tc1x1(call)
    elif n == "TcConv3x3Fn":
        check_tc3x3(call)
    elif n == "StemConvBNFn":
        check_stem(call)
    elif n == "GroupNorm9Fn":
        check_gn9(call)
    elif n == "CotTailFn":
        kind, m = mods[id(call.args[6])]
        check_tail(call, m, kind)
    elif n == "FanOutFn":
        check_fanout(call)
    elif n == "AggTapFn":
        check_agg(call)
    elif n == "Pool3x3S2Fn":
        check_pool(call)
    elif n == "DropBlockFn":
        check_dropblock(call)
    elif n == "DropBlockResReluFn":
        check_dropblock_res_relu(call)
    else:
        raise AssertionError("no stage check for " + n)


def tail_mods(model):
    """id(first MLP parameter) -> (kind, (conv0, bn, conv3)) for every tail MLP of the model"""
    out = {}
    for m in model.modules():
        if hasattr(m, "se") and isinstance(m.se, nn.Sequential):
            out[id(m.se[0].weight)] = ("cot", (m.se[0], m.se[1], m.se[3]))
        if hasattr(m, "fc1") and hasattr(m, "bn0"):
            out[id(m.fc1.weight)] = ("split", (m.fc1, m.bn1, m.fc2))
    return out


# ------------------------------------------------------------------------------------------------ function configurations
def _bn(C, g, dtype=torch.float32, eval_mode=False):
    bn = nn.BatchNorm2d(C).to(DEV)
    with torch.no_grad():
        bn.weight.copy_(1 + 0.25 * torch.randn(C, generator=g, device=DEV))
        bn.bias.copy_(0.25 * torch.randn(C, generator=g, device=DEV))
        bn.running_mean.copy_(0.5 * torch.randn(C, generator=g, device=DEV))
        bn.running_var.copy_(0.5 + torch.rand(C, generator=g, device=DEV))
    bn = bn.to(dtype)
    return bn.eval() if eval_mode else bn.train()


TC1X1 = {
    # name: (K1, K2, N, H, bn, relu, res, ds, eval, weight dtype) at B = 2
    "embed0_two_operands": (64, 64, 32, 56, True, True, False, False, False, torch.float32),
    "embed0_coxt_96": (96, 96, 48, 56, True, True, False, False, False, torch.float32),
    "embed3_no_bn": (32, 0, 72, 56, False, False, False, False, False, torch.float32),
    "conv1x1_bn_no_relu": (64, 0, 64, 56, True, False, False, False, False, torch.float32),
    "bn_relu_code2": (64, 0, 64, 56, True, True, False, False, False, torch.float32),
    "bn_relu_res_code3": (64, 0, 256, 56, True, True, True, False, False, torch.float32),
    "bn_relu_res_drop_scale": (64, 0, 256, 56, True, True, True, True, False, torch.float32),
    "relu_false_for_dropblock": (256, 0, 1024, 14, True, False, False, False, False, torch.float32),
    "eval_no_res": (64, 0, 64, 28, True, True, False, False, True, torch.float32),
    "eval_res": (64, 0, 256, 28, True, True, True, False, True, torch.float32),
    "mm_wgrad_branch": (512, 0, 2048, 7, True, True, True, False, False, torch.float32),
    "bf16_weights": (64, 64, 32, 56, True, True, False, False, False, BF),
}


@pytest.mark.parametrize("exact", [True, False], ids=["integers", "randn"])
@pytest.mark.parametrize("name", sorted(TC1X1))
def test_tc_conv1x1(name, exact, monkeypatch):
    K1, K2, N, H, has_bn, relu, has_res, has_ds, ev, wdt = TC1X1[name]
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(name.encode()) % 1000 + exact)
    B = 2
    mk = (lambda s: _ints(s, g)) if exact else (lambda s: _randn(s, g))
    a1 = mk((B, K1, H, H)).requires_grad_(True)
    a2 = mk((B, K2, H, H)).requires_grad_(True) if K2 else None
    w = (torch.randint(-2, 3, (N, K1 + K2, 1, 1), generator=g, device=DEV).float() if exact else
         torch.randn(N, K1 + K2, 1, 1, generator=g, device=DEV) * (K1 + K2) ** -0.5).to(wdt).requires_grad_(True)
    bn = _bn(N, g, eval_mode=ev) if has_bn else None
    res = _randn((B, N, H, H), g).requires_grad_(True) if has_res else None
    ds = torch.tensor([0.0, 1 / 0.8], device=DEV) if has_ds else None
    rec = S.Recorder(monkeypatch)
    out = fused.TcConv1x1Fn.apply(a1, a2, w, None, None if bn is None else bn.weight, None if bn is None else bn.bias, bn, relu, res, ds)
    dy = mk(tuple(out.shape)) if exact and not has_bn else _randn(tuple(out.shape), g)
    out.backward(dy)
    (call,) = rec.calls
    check_tc1x1(call, exact=exact)
    assert call.gout[2].dtype == wdt and w.grad is not None
    S.equal(w.grad, call.gout[2], "w.grad")


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("dim,H", [(64, 56), (128, 28)])
def test_tc_conv3x3(dim, H, train, monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(dim + train)
    B = 2
    x = _ints((B, dim, H, H), g).requires_grad_(True)
    w = torch.randint(-2, 3, (dim, dim // 4, 3, 3), generator=g, device=DEV).to(BF).requires_grad_(True)
    bn = _bn(dim, g, BF, eval_mode=not train)
    rec = S.Recorder(monkeypatch)
    out = fused.TcConv3x3Fn.apply(x, w, bn.weight, bn.bias, bn, 4, True)
    out.backward(_randn(tuple(out.shape), g))
    (call,) = rec.calls
    check_tc3x3(call, exact=True)


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("HW", [(96, 96), (64, 72)], ids=["wgmma_wgrad", "cudnn_wgrad"])
def test_stem(HW, train, monkeypatch):
    H, W = HW
    g = torch.Generator(device=DEV).manual_seed(H + W + train)
    assert S.stem_wgrad_tc(H, W, 64) == (W == 96) and S.stem_tc(H, W, 64)
    x = _ints((2, 3, H, W), g)
    conv = nn.Conv2d(3, 64, 7, 2, 3, bias=False).to(DEV)
    with torch.no_grad():
        conv.weight.copy_(torch.randint(-2, 3, conv.weight.shape, generator=g, device=DEV).float())
    bn = _bn(64, g, eval_mode=not train)
    rec = S.Recorder(monkeypatch)
    out = fused.stem_conv_bn(x, conv, bn, relu=True)
    out.backward(_randn(tuple(out.shape), g))
    (call,) = rec.calls
    assert call.name == "StemConvBNFn"
    check_stem(call, exact=True)
    S.equal(conv.weight.grad, call.gout[1], "stem weight .grad")


@pytest.mark.parametrize("dtype", [BF, torch.float32])
@pytest.mark.parametrize("cfg", ["relu", "plain", "relu_res", "relu_res_ds", "eval_relu", "eval_res"])
def test_bn_act(cfg, dtype, monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(len(cfg))
    B, C, H = 2, 256, 28
    x = _randn((B, C, H, H), g, dtype, 2.0).requires_grad_(True)
    bn = _bn(C, g, dtype, eval_mode=cfg.startswith("eval"))
    res = _randn((B, C, H, H), g, dtype).requires_grad_(True) if "res" in cfg else None
    ds = torch.tensor([1 / 0.9, 0.0], device=DEV) if "ds" in cfg else None
    rec = S.Recorder(monkeypatch)
    out = fused.bn_act(x, bn, relu="relu" in cfg or "res" in cfg, res=res, drop_scale=ds)
    out.backward(_randn(tuple(out.shape), g, dtype))
    (call,) = rec.calls
    check_bnact(call)


@pytest.mark.parametrize("lbias", [True, False])
@pytest.mark.parametrize("C,fold,tap", [(64, 1, True), (64, 1, False), (96, 2, False), (128, 2, True)],
                         ids=["cot64_tap", "cot64_ref_order", "coxt96_fold2", "coxt128_fold2_tap"])
def test_group_norm9(C, fold, tap, lbias, monkeypatch):
    """the CoT layer's tap-major order, the reference order, and the CoXt fold 2 with (C = 128) and without (C = 96) tap order"""
    g = torch.Generator(device=DEV).manual_seed(fold * 4 + 2 * tap + lbias)
    B, H = 2, 28
    wc = C // 8
    gc = fused.tap_chunk(wc, fold) if tap else 0
    assert (gc > 0) == tap
    gn = nn.GroupNorm(wc, 9 * wc).to(DEV)
    with torch.no_grad():
        gn.weight.copy_(1 + 0.25 * torch.randn(9 * wc, generator=g, device=DEV))
        gn.bias.copy_(0.25 * torch.randn(9 * wc, generator=g, device=DEV))
    lb = (0.5 * torch.randn(9 * wc, generator=g, device=DEV)).requires_grad_(True) if lbias else None
    l = _randn((B, 9 * wc, H, H), g, BF, 2.0).requires_grad_(True)
    rec = S.Recorder(monkeypatch)
    out = fused.group_norm9(l, gn, gc, lb)
    out.backward(_randn(tuple(out.shape), g))
    (call,) = rec.calls
    check_gn9(call)


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("kind", ["cot", "split"])
def test_cot_tail(kind, train, monkeypatch):
    """under bf16 autocast, as the training step runs it: the tail's MLP must still be fp32"""
    from cotnet_b200.cot_layer import CotLayer
    g = torch.Generator(device=DEV).manual_seed(train + 2 * (kind == "cot"))
    B, C, H = 4, 128, 28
    if kind == "cot":
        m = CotLayer(C, 3).to(DEV)
        mods = (m.se[0], m.se[1], m.se[3])
    else:
        from cotnet_b200.backbone_hybrid import SplitAttnConv2d
        m = SplitAttnConv2d(C, C, 3, padding=1).to(DEV)
        mods = (m.fc1, m.bn1, m.fc2)
    with torch.no_grad():
        for bnm in [mm for mm in m.modules() if isinstance(mm, nn.BatchNorm2d)]:
            bnm.running_mean.normal_(0, 0.3, generator=g)
            bnm.running_var.uniform_(0.5, 1.5, generator=g)
    m.train(train)
    bnt = m.bn if kind == "cot" else m.bn0
    u = _randn((B, C, H, H), g).requires_grad_(True)
    k = torch.relu(_randn((B, C, H, H), g)).requires_grad_(True) if kind == "cot" else None
    rec = S.Recorder(monkeypatch)
    with torch.autocast("cuda", dtype=BF):
        out = fused.cot_tail(u, k, bnt, m.se) if kind == "cot" else fused.split_attn_tail(u, bnt, m.fc1, m.bn1, m.fc2)
    out.backward(_randn(tuple(out.shape), g))
    (call,) = rec.calls
    check_tail(call, mods, kind)
    for pt in call.args[6:]:
        assert pt.grad is not None and bool((pt.grad != 0).any())


@pytest.mark.parametrize("n", [2, 3])
def test_fan_out(n, monkeypatch):
    """three consumers with two channel slices of a concat (pitch 2C), as the CoT layer's x; two as its k"""
    g = torch.Generator(device=DEV).manual_seed(n)
    B, C, H = 2, 64, 28
    x = _randn((B, C, H, H), g).requires_grad_(True)
    rec = S.Recorder(monkeypatch)
    outs = fused.fan_out(x, n)
    other = _randn((B, C, H, H), g)
    cat = torch.cat([outs[0], other], 1) if n == 3 else outs[0]
    loss = (cat.float() * _randn(tuple(cat.shape), g).float()).sum()
    for o in outs[1:]:
        loss = loss + (o.float() * _randn(tuple(o.shape), g).float()).sum()
    loss.backward()
    (call,) = rec.calls
    check_fanout(call)
    S.equal(x.grad, call.gout[0], "x.grad")


@pytest.mark.parametrize("fold", [1, 2])
def test_agg_tap(fold, monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(fold)
    B, C, H = 2, (64 if fold == 1 else 96), 28
    wc = C // 8
    gc = fused.tap_chunk(wc, fold)
    v = _randn((B, C, H, H), g).requires_grad_(True)
    w = _randn((B, 9 * wc, H, H), g).requires_grad_(True)
    rec = S.Recorder(monkeypatch)
    out = fused.AggTapFn.apply(v, w, fold, gc)
    out.backward(_randn(tuple(out.shape), g))
    (call,) = rec.calls
    check_agg(call)


@pytest.mark.parametrize("mode", [0, 1])
def test_pool(mode, monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(mode)
    x = _randn((2, 64, 56, 56), g).requires_grad_(True)
    rec = S.Recorder(monkeypatch)
    out = fused.Pool3x3S2Fn.apply(x, mode)
    out.backward(_randn(tuple(out.shape), g))
    (call,) = rec.calls
    check_pool(call)


# ------------------------------------------------------------------------------------------------ blocks, parameter by parameter
class ConvRecorder:
    """F.conv2d calls (cuDNN glue: key conv, embed.3, trunk convolutions off the wgmma path) with input (and its storage), weight,
    incoming gradient and, for a weight that is not a leaf (the dense weights CoXtLayer derives), the weight's gradient"""

    def __init__(self, monkeypatch):
        self.calls = []
        conv0 = F.conv2d

        def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
            out = conv0(input, weight, bias, stride, padding, dilation, groups)
            rec = dict(x=input.detach().clone(), ptr=input.data_ptr(), w=weight, b=bias, stride=stride, padding=padding,
                       dilation=dilation, groups=groups, g=None, gw=None, out_ptr=out.data_ptr(), y=out.detach().clone())
            if out.requires_grad:
                out.register_hook(lambda gr: rec.__setitem__("g", gr.detach().clone()))
            if weight.requires_grad and weight.grad_fn is not None:
                weight.register_hook(lambda gr: rec.__setitem__("gw", gr.detach().clone()))
            self.calls.append(rec)
            return out
        monkeypatch.setattr(torch.nn.functional, "conv2d", conv2d)


class TorchBNRecorder:
    """F.batch_norm calls in training mode (BatchNorms the glue runs in plain PyTorch: the split-attention gate's bn1 when DropBlock
    sits after bn0) with input, weight, bias and the gradient of the output"""

    def __init__(self, monkeypatch):
        self.calls = []
        bn0 = F.batch_norm

        def batch_norm(input, running_mean, running_var, weight=None, bias=None, training=False, momentum=0.1, eps=1e-5):
            out = bn0(input, running_mean, running_var, weight, bias, training, momentum, eps)
            rec = dict(x=input.detach().clone(), w=weight, b=bias, training=training, eps=eps, g=None, y=out.detach().clone())
            if out.requires_grad:
                out.register_hook(lambda gr: rec.__setitem__("g", gr.detach().clone()))
            self.calls.append(rec)
            return out
        monkeypatch.setattr(torch.nn.functional, "batch_norm", batch_norm)


def torch_bn_bwd_ref(r):
    """fp64 backward of a recorded training-mode torch BatchNorm from its recorded input and output gradient: dx, dgamma, dbeta and
    bounds.  torch forms the batch statistics in fp32 (Welford): mean within gamma(n+1) mean|x|, var within gamma(2n+2) E[x^2],
    so rstd within e_r = gamma(2n+2) E[x^2] / (2 var) + 2u relative -- E[x^2] / var is the conditioning |x| / std squared -- and
    xhat = (x - mean) rstd within |xhat| e_r + e_m rstd.  The sums of n terms add gamma(n+1); results are stored in the
    parameter / activation dtype (store_bound at the call site)."""
    x, g = r["x"].double(), r["g"].double()
    dims = (0,) + tuple(range(2, x.dim()))
    n = x.numel() // x.shape[1]
    shp = (1, -1) + (1,) * (x.dim() - 2)
    m = x.mean(dims, keepdim=True)
    var = ((x - m) ** 2).mean(dims, keepdim=True)
    rs = 1.0 / torch.sqrt(var + r["eps"])
    e2 = (x * x).mean(dims, keepdim=True)
    e_m = S.gamma(n + 1) * x.abs().mean(dims, keepdim=True)
    e_r = S.gamma(2 * n + 2) * e2 / (2 * (var + r["eps"])) + 2 * S.U32
    xh = (x - m) * rs
    xh_err = xh.abs() * e_r + e_m * rs + 2 * S.U32 * xh.abs()
    gam = r["w"].detach().double().view(shp) if r["w"] is not None else torch.ones_like(rs)
    out = dict(dbeta=g.sum(dims), dbeta_err=S.gamma(n + 1) * g.abs().sum(dims),
               dgamma=(g * xh).sum(dims), dgamma_err=(g.abs() * xh_err).sum(dims) + S.gamma(n + 1) * (g * xh).abs().sum(dims))
    gd = g * gam
    c0, c1 = gd.mean(dims, keepdim=True), (gd * xh).mean(dims, keepdim=True)
    e_c1 = (gd.abs() * xh_err).mean(dims, keepdim=True) + S.gamma(n + 1) * (gd * xh).abs().mean(dims, keepdim=True)
    out["dx"] = rs * (gd - c0 - xh * c1)
    out["dx_err"] = (out["dx"].abs() * e_r + rs * (xh_err * c1.abs() + xh.abs() * e_c1 + S.gamma(n + 1) * gd.abs().mean(dims, keepdim=True)
                                                   + 8 * S.U32 * (gd.abs() + c0.abs() + (xh * c1).abs())))
    return out


def _conv_wgrad_check(r, shape, got, what):
    """a torch convolution's weight gradient `got` (of weight shape `shape`) against fp64 of its recorded input and gradient"""
    kw = dict(stride=r["stride"], padding=r["padding"], dilation=r["dilation"], groups=r["groups"])
    gd = r["g"].double()
    ref = torch.nn.grad.conv2d_weight(r["x"].double(), shape, gd, **kw)
    mag = torch.nn.grad.conv2d_weight(r["x"].double().abs(), shape, gd.abs(), **kw)
    terms = gd.shape[0] * gd.shape[2] * gd.shape[3]
    # cuDNN's bf16 weight gradients may store split-K partial sums in bf16 before adding them: each partial rounds once, within
    # 2^-9 of its magnitude, and the partials' magnitudes sum to at most sum|terms|
    S.within(got, ref, _dw_bound(ref, mag, terms + 1, True, got.dtype) + (2.0 ** -9 * mag if got.dtype == BF else 0.0), what)


def _derived_grad(p, entries, calls, convs, what):
    """the gradient of the dense weight a parameter was derived into, from its one consumer: a TcConv1x1Fn (returned dW, checked
    by check_tc1x1) or a torch convolution (hooked, checked here against fp64); then its restated adjoint"""
    (e,) = entries
    if e["kind"] == "grouped":
        dense = e["dense"]
        srcs = [r for r in convs if r["w"] is dense]
        tcs = [c for c in calls if c.name == "TcConv1x1Fn" and c.args[2] is dense]
    else:
        dense = torch.cat([e["wx"], e["wk"]], 1).detach()
        srcs = [r for r in convs if r["w"].shape[:2] == dense.shape and torch.equal(r["w"].detach().reshape(dense.shape), dense)]
        tcs = [c for c in calls if c.name == "TcConv1x1Fn" and c.args[2].shape[:2] == dense.shape
               and torch.equal(c.inp[2].reshape(dense.shape), dense)]
    assert len(srcs) + len(tcs) == 1, "%s: %d consumers of the dense weight" % (what, len(srcs) + len(tcs))
    if tcs:
        gd = tcs[0].gout[2]
    else:
        r = srcs[0]
        gd = r["gw"]
        assert gd is not None, what + ": the dense weight's gradient was not recorded"
        _conv_wgrad_check(r, tuple(r["w"].shape), gd, what + " dense weight gradient")
    if e["kind"] == "grouped":
        return S.dense_from_grouped_adjoint(gd, e["groups"])
    C = dense.shape[1] // 2
    g2 = gd.reshape(dense.shape)
    return S.coxt_embed0_adjoint(g2[:, :C], g2[:, C:], e["groups"])


def _leaf_of(t):
    """the parameter behind an autocast copy (ToCopyBackward -> AccumulateGrad), or t itself"""
    fn = t.grad_fn
    if fn is not None and type(fn).__name__.startswith("ToCopyBackward"):
        v = getattr(fn.next_functions[0][0], "variable", None)
        return v if v is not None else t
    return t


def account_params(model, calls, convs, what, derived=None, skip=(), bns=()):
    """every trainable parameter's .grad is a recorded returned gradient (bitwise), the fp64 weight (or bias) gradient of its torch
    conv, the fp64 gradient of its torch BatchNorm (bns: TorchBNRecorder.calls), or (derived: DerivedRecorder.of) bit for bit the
    restated adjoint of the gradient of the dense weight it was derived into.  `skip`: names checked elsewhere."""
    owner = {}
    for c in calls:
        for i, a in enumerate(c.args):
            if isinstance(a, torch.Tensor) and c.gout is not None and i < len(c.gout) and c.gout[i] is not None:
                owner.setdefault(id(a), []).append((c, i))
    conv_of = {}
    for r in convs:
        conv_of.setdefault(id(r["w"]), []).append(r)
    derived = derived or {}
    bias_of = {id(_leaf_of(r["b"])): r for r in convs if r["b"] is not None}
    bn_of = {}
    for r in bns:
        if r["training"] and r["g"] is not None:
            for k in ("w", "b"):
                if r[k] is not None:
                    bn_of.setdefault(id(r[k]), []).append((k, r))
    for name, p in model.named_parameters():
        if name in skip:
            continue
        assert p.grad is not None and bool((p.grad != 0).any()), "%s %s: no or zero gradient" % (what, name)
        src = owner.get(id(p), [])
        if len(src) == 1:
            c, i = src[0]
            S.equal(p.grad, c.gout[i], "%s %s: .grad == %s's returned gradient %d" % (what, name, c.name, i))
            continue
        assert not src, "%s %s: %d recorded contributors" % (what, name, len(src))
        if id(p) in derived:
            assert id(p) not in conv_of, "%s %s: used directly and through a derived weight" % (what, name)
            ref = _derived_grad(p, derived[id(p)], calls, convs, "%s %s" % (what, name))
            S.equal(p.grad, ref.to(p.grad.dtype), "%s %s: .grad == the adjoint of its dense weight's gradient" % (what, name))
            continue
        if id(p) in bias_of:
            r = bias_of[id(p)]
            gd = r["g"].double()
            ref = gd.sum((0, 2, 3))
            err = S.gamma(gd.numel() // gd.shape[1] + 1) * gd.abs().sum((0, 2, 3))
            dt = r["y"].dtype                     # under autocast an fp32 bias is used (and differentiated) as a bf16 copy
            S.within(p.grad, ref, S.store_bound(ref, err, dt) if dt != torch.float32 else err + S.ulp(ref, 24),
                     "%s %s: torch conv bias gradient" % (what, name))
            continue
        if id(p) in bn_of:
            ((k, r),) = bn_of[id(p)]
            br = torch_bn_bwd_ref(r)
            key = "dgamma" if k == "w" else "dbeta"
            ref, err = br[key], br[key + "_err"]
            S.within(p.grad, ref, S.store_bound(ref, err, p.grad.dtype) if p.grad.dtype != torch.float32 else err + S.ulp(ref, 24),
                     "%s %s: torch BatchNorm %s" % (what, name, key))
            continue
        (r,) = conv_of.get(id(p), [None])
        assert r is not None, "%s %s: gradient from no recorded call" % (what, name)
        _conv_wgrad_check(r, p.shape, p.grad, "%s %s: torch conv weight gradient" % (what, name))


def _cfg(call):
    """(function, configuration) label of a recorded call, as the expected lists in stage_ref spell them"""
    a = tuple(call.args) + (None,) * 4          # trailing optional arguments the caller left out
    n = call.name
    if n == "BNActFn":
        return "BNActFn(%s%s%s)" % ("relu" if a[5] else "plain", "+res" if a[3] is not None else "", "+ds" if a[6] is not None else "")
    if n == "TcConv1x1Fn":
        return "TcConv1x1Fn(%s,%s%s%s)" % ("two" if a[1] is not None else "one", "nobn" if a[6] is None else ("relu" if a[7] else "bn"),
                                          "+res" if a[8] is not None else "", "+ds" if a[9] is not None else "")
    if n == "FanOutFn":
        return "FanOutFn(%d)" % a[1]
    if n == "GroupNorm9Fn":
        return "GroupNorm9Fn(gc%d%s)" % (a[4], "+lbias" if a[5] is not None else "")
    if n == "AggTapFn":
        return "AggTapFn(fold%d,gc%d)" % (a[2], a[3])
    if n == "CotTailFn":
        return "CotTailFn(%s)" % ("k" if a[1] is not None else "gate")
    if n == "Pool3x3S2Fn":
        return "Pool3x3S2Fn(%s)" % ("avg" if a[1] == 0 else "max")
    return n


@pytest.mark.parametrize("geo", sorted(S.BLOCK_CASES))
def test_bottleneck_stage_by_stage(geo, monkeypatch):
    """one forward and backward of a bf16 CoT bottleneck: (a) the recorded calls, (b) producer -> consumer equality where a call
    consumes another's output unchanged, (c) every call's stage check, (d) every parameter accounted for"""
    from cotnet_b200 import backbone
    case = S.BLOCK_CASES[geo]
    if case["min_pixels"] is not None:
        monkeypatch.setattr(fused, "TC_MIN_PIXELS", case["min_pixels"])
    torch.manual_seed(5)
    model = backbone.cotnet50() if case["model"] == "cotnet50" else backbone.cotnext50_2x48d()
    blk = getattr(model, case["block"].split(".")[0])[int(case["block"].split(".")[1])]
    with torch.no_grad():
        for m in blk.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.25, 0.25)
    blk = blk.to(DEV).to(BF).to(memory_format=CL).train()
    g = torch.Generator(device=DEV).manual_seed(7)
    B, C, H = case["B"], case["cin"], case["H"]
    x = torch.relu(_randn((B, C, H, H), g)).requires_grad_(True)
    ref_blk = copy.deepcopy(blk)
    dy = _randn((B, case["cout"], H // case["stride"], H // case["stride"]), g)
    n0 = _lib.launch_count()
    x0 = x.detach().clone().requires_grad_(True)
    ref_out = ref_blk(x0)
    ref_out.backward(dy)
    n_plain = _lib.launch_count() - n0
    rec = S.Recorder(monkeypatch)
    convs = ConvRecorder(monkeypatch).calls
    n0 = _lib.launch_count()
    out = blk(x)
    out.backward(dy)
    assert _lib.launch_count() - n0 == n_plain, "the recorder changed the launches"
    # the recorder changes nothing
    S.equal(out, ref_out, "block output with / without the recorder")
    S.equal(x.grad, x0.grad, "dX with / without the recorder")
    for (n, p), (_, q) in zip(blk.named_parameters(), ref_blk.named_parameters()):
        S.equal(p.grad, q.grad, "%s.grad with / without the recorder" % n)
    for (n, b), (_, c) in zip(blk.named_buffers(), ref_blk.named_buffers()):
        S.equal(b, c, "%s with / without the recorder" % n)
    # (a)
    assert [_cfg(c) for c in rec.calls] == case["calls"], [_cfg(c) for c in rec.calls]
    # (b) the stated dataflow: (consumer, argument) <- (producer, output) or the block input x, by storage and by value; and no other
    # recorded output (or x) reaches a recorded input
    ptrs = {}
    for i, c in enumerate(rec.calls):
        for o, (pt, snap) in enumerate(zip(c.out_ptr, c.out if isinstance(c.out, tuple) else (c.out,))):
            ptrs.setdefault(pt, []).append(("%d.%d" % (i, o), snap))
    ptrs.setdefault(x.data_ptr(), []).append(("x", x.detach()))
    flow = dict(e.split("<-") for e in case["flow"])
    seen = set()
    for i, c in enumerate(rec.calls):
        for a, arg in enumerate(c.args):
            if not isinstance(arg, torch.Tensor) or arg.data_ptr() not in ptrs:
                continue
            key = "%d.%d" % (i, a)
            cands = {name: snap for name, snap in ptrs[arg.data_ptr()] if name == "x" or int(name.split(".")[0]) < i}
            if not cands:
                continue
            assert key in flow, "%s: %s %s reads %s, which the stated dataflow does not list" % (geo, key, c.name, sorted(cands))
            assert flow[key] in cands, "%s: %s reads %s, not %s" % (geo, key, sorted(cands), flow[key])
            S.equal(c.inp[a], cands[flow[key]], "%s: %s == %s" % (geo, key, flow[key]))
            seen.add(key)
    assert seen == set(flow), "%s: stated edges not found: %s" % (geo, sorted(set(flow) - seen))
    # (c)
    mods = tail_mods(blk)
    for c in rec.calls:
        check_call(c, mods)
    # (d)
    account_params(blk, rec.calls, convs, geo)
