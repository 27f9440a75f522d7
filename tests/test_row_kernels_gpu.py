"""The row kernels (csrc/norm_tail.cu, csrc/gn72.cu, csrc/sum_rows.cu, csrc/pool.cu) through the C ABI, exactly, at every dispatch
geometry of tests/test_row_geometry_cpu.py.

Exact inputs: small integers in every dtype, powers of two for scales and rstd, integer or half-integer means and shifts.  Every
per-element expression of these kernels is then exact in fp32, and so is every column sum below 2^24 in any order of addition, so
the expected result is computed in fp64 on the device and compared with torch.equal: a dropped row chunk, a column chunk reading
another chunk's scale or a drop-path scale applied to the wrong sample changes the bits.  The SiLU is neutralised two ways: z = 0
(silu = 0 and silu' = 1/2 exactly) and z >= 18 (sigmoid = 1 exactly in fp32, so silu = z and silu' = 1).  Where a rsqrt sits in
the path (the statistics prologue) its outputs are checked to a few fp32 ulp and the outputs that use them bit for bit.

A smaller set with random activations checks the arithmetic against fp64, in output ulps per dtype."""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cotnet_b200 import _lib
from test_row_geometry_cpu import CASES, ESIZE, SUM_CASES, assert_coverage, assert_sum_rows_coverage, mask_geo_ok, pick_vec

pytestmark = pytest.mark.gpu

TD = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
EINVAL, ENULL, ETOOBIG = -1, -5, -6
DEV = "cuda"


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _at(shape, dtype, off, fill=float("nan")):
    """a tensor of `shape` that starts `off` elements into a larger buffer (pointer alignment of the C ABI), filled with `fill`"""
    n = int(np.prod(shape))
    base = torch.full((n + off,), fill, dtype=dtype, device=DEV)
    return base[off:].view(shape)


def _ints(shape, dtype, off, g, lo=-4, hi=4):
    t = _at(shape, dtype, off, 0.0)
    t.copy_(torch.randint(lo, hi + 1, shape, generator=g, device=DEV).to(dtype))
    return t


def _cases(kind):
    return [c for c in CASES if c.kind == kind]


def _ids(c):
    return c.name


def _eq(got, want, what):
    want = want.to(got.dtype)
    if not torch.equal(got, want):
        bad = (got.double() != want.double()) | torch.isnan(got.double())
        idx = bad.nonzero()[:4].tolist()
        raise AssertionError("%s: %d of %d elements differ, first %s: got %s want %s" % (
            what, int(bad.sum()), got.numel(), idx, [got[tuple(i)].item() for i in idx], [want[tuple(i)].item() for i in idx]))


def _f32(t64):
    """fp64 -> the fp32 value the kernel holds (one rounding)"""
    return t64.float().double()


def _ulp(v, dtype):
    """unit in the last place of |v| in `dtype` (fp64 tensor)"""
    p = {torch.float32: 23, torch.bfloat16: 7, torch.float16: 10}[dtype]
    tiny = {torch.float32: 2.0 ** -126, torch.bfloat16: 2.0 ** -126, torch.float16: 2.0 ** -14}[dtype]
    e = torch.frexp(v.abs().clamp_min(tiny))[1]
    return torch.ldexp(torch.ones_like(v), e - 1 - p)


def _within(got, want, tol, what):
    err = (got.double() - want).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError("%s: %d of %d beyond the bound, e.g. got %r want %r bound %r (max err/bound %.3g)" % (
            what, int(bad.sum()), got.numel(), got.flatten()[i].item(), want.flatten()[i].item(), tol.flatten()[i].item(),
            (err / tol).max().item()))
    return (err / tol).max().item()


# ------------------------------------------------------------------------------------------------ geometry coverage
def test_live_geometry_coverage():
    """The case list reaches every branch of tests/test_row_geometry_cpu.py on this device's SM count too."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    reached = assert_coverage(sms)
    assert_sum_rows_coverage(sms)
    for kind in sorted(reached):
        print("row-kernel coverage on %d SMs, %s: %s" % (sms, kind, " ".join(sorted(reached[kind]))))


# ------------------------------------------------------------------------------------------------ BatchNorm, exact
def _cols(C):
    return torch.arange(C, device=DEV)


def _dyadic_affine(C):
    """per-column scale = +-2^(c%5 - 2), shift = (c%7 - 3)/2: x*scale + shift is exact for |x| <= 4"""
    c = _cols(C)
    scale = torch.ldexp(torch.ones(C, device=DEV), (c % 5 - 2).int()) * torch.where(c % 3 == 1, -1.0, 1.0)
    shift = (c % 7 - 3).float() * 0.5
    return scale.float().contiguous(), shift.float().contiguous()


def _sample_scales(B):
    """distinct drop-path scales per sample (0, 1/2 and 2: every s_b*z stays exact)"""
    return torch.tensor([2.0, 0.0, 0.5, 1.0, 0.5, 2.0, 0.0][:B] + [2.0] * max(0, B - 7), device=DEV)


def _row_scale(ds, B, HW):
    return ds.double().repeat_interleave(HW).view(-1, 1) if ds is not None else 1.0


def _bn_y_ref(x64, sc64, sh64, res64, relu, rs):
    """the kernel's y: fp32 fma(x, scale, shift) (one rounding), * s_b, + res, ReLU"""
    z = _f32(x64 * sc64 + sh64) * rs
    if res64 is not None:
        z = _f32(z + res64)
    return z.clamp_min(0.0) if relu else z


@pytest.mark.parametrize("case", _cases("bn"), ids=_ids)
def test_bn_exact(case):
    """col_stats; bn_apply and bn_apply_batch with and without residual, ReLU and drop-path scales (and the 1-bit mask where the
    geometry takes one); bn_bwd_sums and bn_bwd_apply for relu codes 0-3, with and without dres and drop-path scales, training and
    eval mode.  Everything bit-exact except the rsqrt-derived statistics (<= 4 fp32 ulp)."""
    lib, st = _lib.load(), _st()
    T, B, HW, C, off = TD[case.dtype], case.B, case.HW, case.C, case.off
    dt, n = _lib.dtype_code(torch.empty(0, dtype=T)), case.B * case.HW
    g = _gen(zlib.crc32(case.name.encode()))
    x, res, dy = (_ints((n, C), T, off, g, -case.amp, case.amp) for _ in range(3))
    x64, res64, dy64 = x.double(), res.double(), dy.double()
    mask_ok = mask_geo_ok(C, pick_vec(C, ESIZE[case.dtype], (off * ESIZE[case.dtype],)))

    # column statistics, accumulated onto 0.5
    sums = torch.full((2, C), 0.5, device=DEV)
    _lib.check(lib.cotb200_col_stats(dt, B, HW, C, _p(x), _p(sums[0]), _p(sums[1]), st), "col_stats")
    _eq(sums[0], 0.5 + x64.sum(0), "col_stats sum")
    _eq(sums[1], 0.5 + (x64 * x64).sum(0), "col_stats sq")
    sums -= 0.5

    # apply with dyadic scale / shift
    sc, sh = _dyadic_affine(C)
    ds = _sample_scales(B)
    for use_res in (False, True):
        for relu in (0, 1):
            for use_ds in (False, True):
                y = _at((n, C), T, off)
                _lib.check(lib.cotb200_bn_apply(dt, B, HW, C, _p(x), _p(res) if use_res else None, _p(sc), _p(sh), relu, _p(y),
                                         _p(ds) if use_ds else None, st), "bn_apply")
                want = _bn_y_ref(x64, sc.double(), sh.double(), res64 if use_res else None, relu,
                                 _row_scale(ds if use_ds else None, B, HW))
                _eq(y, want, "bn_apply res=%d relu=%d ds=%d" % (use_res, relu, use_ds))

    # training-mode apply: statistics from the batch sums
    c = _cols(C)
    w = torch.ldexp(torch.ones(C, device=DEV), (c % 3 - 1).int()).float()
    bias = ((c % 5) - 2).float() * 0.25
    mean64 = sums[0].double() / n
    var64 = (sums[1].double() / n - mean64 * mean64).clamp_min(0.0)
    rstd64 = 1.0 / torch.sqrt(var64 + float(np.float32(1e-5)))
    variants = [(relu, use_res, False) for relu in (0, 1) for use_res in (False, True)] + ([(1, True, True)] if mask_ok else [])
    for update in (0, 1):
        for use_ds in (False, True):
            for relu, use_res, use_mask in variants:
                rm0 = ((c % 3) - 1).float() * 0.5
                rv0 = 1.0 + (c % 4).float() * 0.25
                rm, rv = rm0.clone(), rv0.clone()
                ss = torch.full((4, C), float("nan"), device=DEV)
                y = _at((n, C), T, off)
                mask = torch.full((n, C // 8), 0xA5, dtype=torch.uint8, device=DEV) if use_mask else None
                r = res if use_res else None
                _lib.check(lib.cotb200_bn_apply_batch(dt, B, HW, C, _p(x), _p(r), _p(sums[0]), _p(sums[1]), _p(w), _p(bias), _p(rm), _p(rv),
                                               float(n), 1e-5, 0.25, update, relu, _p(y), _p(ss[0]), _p(ss[1]), _p(ss[2]), _p(ss[3]),
                                               _p(ds) if use_ds else None, _p(mask), st), "bn_apply_batch")
                what = "bn_apply_batch update=%d ds=%d relu=%d res=%d mask=%d" % (update, use_ds, relu, use_res, use_mask)
                _within(ss[2], mean64, _ulp(mean64, torch.float32), what + " mean")
                _within(ss[3], rstd64, 4 * _ulp(rstd64, torch.float32), what + " rstd")
                _eq(ss[0], w.double() * ss[3].double(), what + " scale")          # weight is a power of two
                _eq(ss[1], _f32(bias.double() - ss[2].double() * ss[0].double()), what + " shift")
                want = _bn_y_ref(x64, ss[0].double(), ss[1].double(), None if r is None else r.double(), relu,
                                 _row_scale(ds if use_ds else None, B, HW))
                _eq(y, want, what + " y")
                if update:
                    _eq(rm, _f32(0.75 * rm0.double() + 0.25 * ss[2].double()), what + " running_mean")
                    rv64 = 0.75 * rv0.double() + 0.25 * var64 * (n / max(n - 1, 1))
                    _within(rv, rv64, 4 * _ulp(rv64, torch.float32), what + " running_var")
                else:
                    _eq(rm, rm0, what + " running_mean untouched")
                    _eq(rv, rv0, what + " running_var untouched")
                if use_mask:
                    bits = torch.arange(8, device=DEV, dtype=torch.uint8)
                    m = ((mask.unsqueeze(-1) >> bits) & 1).reshape(n, C).bool()
                    _eq(m, y.double() > 0, what + " mask bits")

    # backward with dyadic mean / rstd / scale / shift, the sign source of each relu code given directly
    mu = ((c % 5) - 2).float()
    rstd = torch.ldexp(torch.ones(C, device=DEV), (c % 3 - 1).int()).float()
    yin = _ints((n, C), T, off, g, -2, 2)
    min_ = torch.randint(0, 256, (n, C // 8), generator=g, device=DEV).to(torch.uint8) if mask_ok else None
    c1 = ((c % 5) - 2).float() * 64.0
    c2 = ((c % 3) - 1).float() * 32.0
    inv_n = 1.0 / 64.0
    xhat = (x64 - mu.double()) * rstd.double()
    for relu in ((0, 1, 2, 3) if mask_ok else (0, 1, 2)):
        if relu == 0:
            gate = torch.ones_like(x64, dtype=torch.bool)
        elif relu == 1:
            gate = yin.double() > 0
        elif relu == 3:
            bits = torch.arange(8, device=DEV, dtype=torch.uint8)
            gate = ((min_.unsqueeze(-1) >> bits) & 1).reshape(n, C).bool()
        for use_ds in (False, True):
            rs = _row_scale(ds if use_ds else None, B, HW)
            if relu == 2:
                gate = (_f32(x64 * sc.double() + sh.double()) * rs) > 0
            gd = torch.where(gate, dy64, 0.0)
            dz = gd * rs
            head = (dt, B, HW, C, _p(dy), _p(x), _p(yin) if relu == 1 else None, _p(min_) if relu == 3 else None, _p(sc),
                    _p(sh) if relu == 2 else None, _p(mu), _p(rstd))
            s = torch.full((2, C), 0.25, device=DEV)
            _lib.check(lib.cotb200_bn_bwd_sums(*head, relu, _p(s[0]), _p(s[1]), _p(ds) if use_ds else None, st), "bn_bwd_sums")
            what = "bn_bwd relu=%d ds=%d" % (relu, use_ds)
            _eq(s[0], 0.25 + dz.sum(0), what + " sum_dz")
            _eq(s[1], 0.25 + (dz * xhat).sum(0), what + " sum_dzx")
            for train in (True, False):
                for use_dres in (False, True):
                    dx, dres = _at((n, C), T, off), (_at((n, C), T, off) if use_dres else None)
                    _lib.check(lib.cotb200_bn_bwd_apply(*head, _p(c1) if train else None, _p(c2) if train else None, inv_n, relu, _p(dx),
                                                 _p(dres), _p(ds) if use_ds else None, st), "bn_bwd_apply")
                    k1 = c1.double() * inv_n if train else 0.0
                    k2 = c2.double() * inv_n if train else 0.0
                    _eq(dx, sc.double() * (dz - k1 - xhat * k2), what + " train=%d dres=%d dx" % (train, use_dres))
                    if use_dres:
                        _eq(dres, gd, what + " dres")

    # codes 1 and 2 agree bit for bit, with and without drop-path scales: code 1 reads the y bn_apply stored, code 2 recomputes
    # its sign from x and the same scale / shift
    for use_ds in (False, True):
        dsp = _p(ds) if use_ds else None
        y = _at((n, C), T, off)
        _lib.check(lib.cotb200_bn_apply(dt, B, HW, C, _p(x), None, _p(sc), _p(sh), 1, _p(y), dsp, st), "bn_apply")
        got = []
        for relu, yp, shp in ((1, _p(y), None), (2, None, _p(sh))):
            head = (dt, B, HW, C, _p(dy), _p(x), yp, None, _p(sc), shp, _p(mu), _p(rstd))
            s, dx = torch.zeros(2, C, device=DEV), _at((n, C), T, off)
            _lib.check(lib.cotb200_bn_bwd_sums(*head, relu, _p(s[0]), _p(s[1]), dsp, st), "bn_bwd_sums")
            _lib.check(lib.cotb200_bn_bwd_apply(*head, _p(s[0]), _p(s[1]), inv_n, relu, _p(dx), None, dsp, st), "bn_bwd_apply")
            got.append((s, dx))
        _eq(got[1][0], got[0][0], "bn_bwd code 2 == code 1 ds=%d sums" % use_ds)
        _eq(got[1][1], got[0][1], "bn_bwd code 2 == code 1 ds=%d dx" % use_ds)


@pytest.mark.parametrize("n,use_batch,update", [(1.0, 1, 1), (2.0, 1, 1), (2.0, 1, 0), (6.0, 0, 0)])
def test_bn_finalize_exact(n, use_batch, update):
    """cotb200_bn_finalize: batch statistics with and without the running-buffer update, n = 1 (unbiased factor n / max(n-1, 1) = 1)
    and n = 2 (factor 2), and eval mode (statistics from the running buffers).  Means are powers of two, so everything but the rsqrt is
    exact."""
    lib, C = _lib.load(), 37
    c = _cols(C)
    mean = torch.where(c % 3 == 0, 0.0, torch.ldexp(torch.ones(C, device=DEV), (c % 4 - 1).int()) * torch.where(c % 2 == 0, 1.0, -1.0))
    var = (c % 5).float() * 0.5
    sum_ = (mean * n).float()
    sq = ((var + mean * mean) * n).float()
    w = torch.ldexp(torch.ones(C, device=DEV), (c % 3 - 1).int()).float()
    b = ((c % 5) - 2).float() * 0.25
    rm0, rv0 = (((c % 3) - 1) * 0.5).float(), (1.0 + (c % 4) * 0.25).float()
    if not use_batch:
        rm0, rv0 = mean.float(), var.float()
    rm, rv = rm0.clone(), rv0.clone()
    out = torch.full((4, C), float("nan"), device=DEV)
    _lib.check(lib.cotb200_bn_finalize(C, _p(sum_), _p(sq), _p(w), _p(b), _p(rm), _p(rv), n, 1e-5, 0.25, use_batch, update, _p(out[0]),
                                _p(out[1]), _p(out[2]), _p(out[3]), _st()), "bn_finalize")
    m64 = mean.double()
    v64 = var.double() if use_batch else rv0.double()
    r64 = 1.0 / torch.sqrt(_f32(v64 + float(np.float32(1e-5))))      # rsqrtf of the fp32 var + eps: 2 ulp
    _eq(out[2], m64, "mean")
    _within(out[3], r64, 2 * _ulp(r64, torch.float32), "rstd")
    _eq(out[0], w.double() * out[3].double(), "scale")
    _eq(out[1], _f32(b.double() - m64 * out[0].double()), "shift")
    if use_batch and update:
        _eq(rm, 0.75 * rm0.double() + 0.25 * m64, "running_mean")
        _eq(rv, 0.75 * rv0.double() + 0.25 * v64 * (n / max(n - 1.0, 1.0)), "running_var")
    else:
        _eq(rm, rm0, "running_mean untouched")
        _eq(rv, rv0, "running_var untouched")


# ------------------------------------------------------------------------------------------------ CoT / split-attention tails, exact
def _tail_params(B, C):
    """columns c % 3 == 0: scale = shift = 0 (z = 0); the others: scale 1 or 2, shift 26..30 (z >= 18, sigmoid(z) = 1 in fp32).
    a[b,c,0] = +-2^k and a[b,c,1] = multiples of 1/4, distinct per sample; dpn integers; pscale 1/2."""
    c = _cols(C)
    sat = c % 3 != 0
    scale = torch.where(sat, torch.ldexp(torch.ones(C, device=DEV), (c % 2).int()), 0.0).float()
    shift = torch.where(sat, 26.0 + (c % 5).float(), 0.0).float()
    b = torch.arange(B, device=DEV).view(B, 1)
    a0 = torch.ldexp(torch.ones(B, C, device=DEV), ((b + c) % 3 - 1).int()) * torch.where((b * 7 + c) % 2 == 0, 1.0, -1.0)
    a1 = ((b * 5 + c) % 7 - 3).float() * 0.25
    a = torch.stack([a0, a1], -1).float().contiguous()
    dpn = ((b * 3 + c * 5) % 9 - 4).float().contiguous()
    return sat, scale, shift, a, dpn


@pytest.mark.parametrize("case", _cases("tail"), ids=_ids)
def test_tail_exact(case):
    """tail_pool, tail_combine, tail_bwd_sums with k and with k == NULL (the radix-1 SplitAttnConv2d); tail_bwd_dz_sums;
    tail_bwd_apply in training and eval mode, with and without dk; per-sample a / dpn distinct for every sample."""
    lib, st = _lib.load(), _st()
    T, B, HW, C, off = TD[case.dtype], case.B, case.HW, case.C, case.off
    dt = _lib.dtype_code(torch.empty(0, dtype=T))
    g = _gen(zlib.crc32(case.name.encode()))
    u, k, dout = (_ints((B, HW, C), T, off, g, -case.amp, case.amp) for _ in range(3))
    u64, k64, d64 = u.double(), k.double(), dout.double()
    sat, scale, shift, a, dpn = _tail_params(B, C)
    z = u64 * scale.double() + shift.double()
    assert bool((z[..., sat] >= 18).all())
    y = torch.where(sat, z, 0.0)                       # silu(z)
    dsilu = torch.where(sat, 1.0, 0.5)                 # silu'(z)
    a0, a1 = a[..., 0].double().unsqueeze(1), a[..., 1].double().unsqueeze(1)
    pscale = 0.5
    dp = (dpn.double() * pscale).unsqueeze(1)
    for use_k in (True, False):
        kp, kk = (k, k64) if use_k else (None, torch.zeros_like(k64))
        what = "k=%d" % use_k
        ps = torch.full((B, C), 0.5, device=DEV)
        _lib.check(lib.cotb200_tail_pool(dt, B, HW, C, _p(u), _p(kp), _p(scale), _p(shift), _p(ps), st), "tail_pool")
        _eq(ps, 0.5 + (y + kk).sum(1), what + " tail_pool")
        out = _at((B, HW, C), T, off)
        _lib.check(lib.cotb200_tail_combine(dt, B, HW, C, _p(u), _p(kp), _p(scale), _p(shift), _p(a), _p(out), st), "tail_combine")
        _eq(out, a0 * y + a1 * kk, what + " tail_combine")
        S = torch.full((B, C, 2), 0.25, device=DEV)
        _lib.check(lib.cotb200_tail_bwd_sums(dt, B, HW, C, _p(dout), _p(u), _p(kp), _p(scale), _p(shift), _p(S), st), "tail_bwd_sums")
        _eq(S[..., 0], 0.25 + (d64 * y).sum(1), what + " tail_bwd_sums S0")
        _eq(S[..., 1], 0.25 + (d64 * kk).sum(1), what + " tail_bwd_sums S1")
    c = _cols(C)
    mu = ((c % 5) - 2).float()
    rstd = torch.ldexp(torch.ones(C, device=DEV), (c % 3 - 1).int()).float()
    xhat = (u64 - mu.double()) * rstd.double()
    dz = (a0 * d64 + dp) * dsilu
    s = torch.full((2, C), 0.5, device=DEV)
    _lib.check(lib.cotb200_tail_bwd_dz_sums(dt, B, HW, C, _p(dout), _p(u), _p(scale), _p(shift), _p(mu), _p(rstd), _p(a), _p(dpn), pscale,
                                     _p(s[0]), _p(s[1]), st), "tail_bwd_dz_sums")
    _eq(s[0], 0.5 + dz.sum((0, 1)), "tail_bwd_dz_sums sum_dz")
    _eq(s[1], 0.5 + (dz * xhat).sum((0, 1)), "tail_bwd_dz_sums sum_dzx")
    c1 = ((c % 5) - 2).float() * 64.0
    c2 = ((c % 3) - 1).float() * 32.0
    for train in (True, False):
        for use_dk in (True, False):
            du, dk = _at((B, HW, C), T, off), (_at((B, HW, C), T, off) if use_dk else None)
            _lib.check(lib.cotb200_tail_bwd_apply(dt, B, HW, C, _p(dout), _p(u), _p(scale), _p(shift), _p(mu), _p(rstd), _p(a), _p(dpn),
                                           _p(c1) if train else None, _p(c2) if train else None, 1.0 / 64.0, pscale, _p(du), _p(dk),
                                           st), "tail_bwd_apply")
            k1 = c1.double() / 64.0 if train else 0.0
            k2 = c2.double() / 64.0 if train else 0.0
            what = "tail_bwd_apply train=%d dk=%d" % (train, use_dk)
            _eq(du, scale.double() * (dz - k1 - xhat * k2), what + " du")
            if use_dk:
                _eq(dk, a1 * d64 + dp, what + " dk")


# ------------------------------------------------------------------------------------------------ GroupNorm over 9 taps, exact
def _gn_pos(J, gc):
    """storage position of reference channel j = g*9 + t"""
    j = torch.arange(J, device=DEV)
    if gc <= 0:
        return j
    gi, t = j // 9, j % 9
    return ((gi // gc) * 9 + t) * gc + gi % gc


def _pre_image(target, HW):
    """an fp32 s with fl(s * fl(1 / (9*HW))) == target: the kernels scale s1, s2 by that inv_n"""
    inv = np.float32(1.0) / np.float32(9.0 * HW)
    s, t = np.float32(target * 9.0 * HW), np.float32(target)
    for _ in range(64):
        k = np.float32(s * inv)
        if k == t:
            return float(s)
        s = np.nextafter(s, np.float32(np.inf if k < t else -np.inf))
    raise AssertionError("no pre-image of %r" % target)


@pytest.mark.parametrize("case", _cases("gn"), ids=_ids)
def test_gn9_exact(case):
    """gn9_stats, gn9_apply, gn9_bwd_sums (s1, s2, dgamma, dbeta exact; dlbias to fp32 rounding: its 1/(9*HW) is not dyadic) and
    gn9_bwd_apply, with and without lbias, on the gn72 fast path or the generic kernels as the case's geometry picks."""
    lib, st = _lib.load(), _st()
    T, B, HW, wc, gc, off = TD[case.dtype], case.B, case.HW, case.C, case.gc, case.off
    dt, J = _lib.dtype_code(torch.empty(0, dtype=T)), 9 * case.C
    g = _gen(zlib.crc32(case.name.encode()))
    l = _ints((B, HW, J), T, off, g, -case.amp, case.amp)
    dg = _ints((B, HW, J), T, off, g, -case.amp, case.amp)
    pos = _gn_pos(J, gc)
    l64, dg_ref = l.double(), dg.double()[..., pos]                  # dg in the reference order
    j = torch.arange(J, device=DEV)
    gi = torch.arange(wc, device=DEV)
    bb = torch.arange(B, device=DEV).view(B, 1)
    mean = ((bb + gi) % 3 - 1).float().contiguous()
    rstd = torch.ldexp(torch.ones(B, wc, device=DEV), ((bb + gi) % 3 - 1).int()).float().contiguous()
    gamma = (torch.ldexp(torch.ones(J, device=DEV), (j % 3 - 1).int()) * torch.where(j % 4 == 1, -1.0, 1.0)).float()
    beta = ((j % 5) - 2).float() * 0.25
    for use_lb in (False, True):
        lb = ((j % 5) - 2).float() if use_lb else None
        lbd = lb.double() if use_lb else torch.zeros(J, device=DEV, dtype=torch.float64)
        what = "lbias=%d" % use_lb
        lv = l64 + lbd
        gs = torch.full((2, B, wc), 0.5, device=DEV)
        _lib.check(lib.cotb200_gn9_stats(dt, B, HW, wc, gc, _p(l), _p(lb), _p(gs[0]), _p(gs[1]), st), "gn9_stats")
        _eq(gs[0], 0.5 + lv.view(B, HW, wc, 9).sum((1, 3)), what + " gn9_stats sum")
        _eq(gs[1], 0.5 + (lv * lv).view(B, HW, wc, 9).sum((1, 3)), what + " gn9_stats sq")
        mj = mean.double().repeat_interleave(9, 1).unsqueeze(1)          # [B, 1, J]
        rj = rstd.double().repeat_interleave(9, 1).unsqueeze(1)
        lhat = (lv - mj) * rj
        out = _at((B, HW, J), T, off)
        _lib.check(lib.cotb200_gn9_apply(dt, B, HW, wc, gc, _p(l), _p(lb), _p(mean), _p(rstd), _p(gamma), _p(beta), _p(out), st), "gn9_apply")
        want = torch.empty_like(lhat)
        want[..., pos] = lhat * gamma.double() + beta.double()
        _eq(out, want, what + " gn9_apply")
        work = torch.zeros(B, 3, J, device=DEV)
        s12 = torch.full((2, B, wc), float("nan"), device=DEV)
        acc = torch.full((3, J), 0.5, device=DEV)
        _lib.check(lib.cotb200_gn9_bwd_sums(dt, B, HW, wc, gc, _p(dg), _p(l), _p(lb), _p(mean), _p(rstd), _p(gamma), _p(work), _p(s12[0]),
                                     _p(s12[1]), _p(acc[0]), _p(acc[1]), _p(acc[2]) if use_lb else None, st), "gn9_bwd_sums")
        D = dg_ref.sum(1)                                                 # [B, J]
        DL = (dg_ref * lhat).sum(1)
        s1 = (D * gamma.double()).view(B, wc, 9).sum(2)
        s2 = (DL * gamma.double()).view(B, wc, 9).sum(2)
        _eq(s12[0], s1, what + " gn9_bwd_sums s1")
        _eq(s12[1], s2, what + " gn9_bwd_sums s2")
        _eq(acc[0], 0.5 + DL.sum(0), what + " gn9_bwd_sums dgamma")
        _eq(acc[1], 0.5 + D.sum(0), what + " gn9_bwd_sums dbeta")
        if use_lb:
            k1, k2 = (s1 / (9.0 * HW)).repeat_interleave(9, 1).unsqueeze(1), (s2 / (9.0 * HW)).repeat_interleave(9, 1).unsqueeze(1)
            terms = rj * (dg_ref * gamma.double() - k1 - lhat * k2)
            mag = (rj * (dg_ref.abs() * gamma.double().abs() + k1.abs() + (lhat * k2).abs())).sum((0, 1))
            _within(acc[2], 0.5 + terms.sum((0, 1)), 2.0 ** -18 * mag + _ulp(torch.full_like(mag, 0.5) + mag, torch.float32),
                    what + " gn9_bwd_sums dlbias")
        # backward apply with s1, s2 whose scaled values k = fl(s * fl(1/(9 HW))) are small dyadic numbers
        kt1 = (((bb + 2 * gi) % 5) - 2).double() * 0.5
        kt2 = (((2 * bb + gi) % 3) - 1).double() * 0.25
        s1in = torch.tensor([[_pre_image(v, HW) for v in row] for row in kt1.tolist()], device=DEV)
        s2in = torch.tensor([[_pre_image(v, HW) for v in row] for row in kt2.tolist()], device=DEV)
        dl = _at((B, HW, J), T, off)
        _lib.check(lib.cotb200_gn9_bwd_apply(dt, B, HW, wc, gc, _p(dg), _p(l), _p(lb), _p(mean), _p(rstd), _p(gamma), _p(s1in), _p(s2in),
                                      _p(dl), st), "gn9_bwd_apply")
        k1 = kt1.repeat_interleave(9, 1).unsqueeze(1)
        k2 = kt2.repeat_interleave(9, 1).unsqueeze(1)
        _eq(dl, rj * (dg_ref * gamma.double() - k1 - lhat * k2), what + " gn9_bwd_apply")


# ------------------------------------------------------------------------------------------------ sum_rows and pool3s2, exact


@pytest.mark.parametrize("name,dtype,rows,C,lds,ldo,off", SUM_CASES, ids=[c[0] for c in SUM_CASES])
def test_sum_rows_exact(name, dtype, rows, C, lds, ldo, off):
    """out = sum of 2-4 row-pitched sources (pitches > C, odd pitches and a misaligned pointer pick every packet width, and one case
    is past the grid cap so that threads take a second item); the output's padding columns keep their bytes."""
    lib, T = _lib.load(), TD[dtype]
    g = _gen(len(name) * 7 + rows)
    src = [_ints((rows, ld), T, off, g)[:, :C] for ld in lds]
    outb = _at((rows, ldo), T, off, 7.0)
    args = []
    for i in range(4):
        args += [_p(src[i]), lds[i]] if i < len(src) else [None, 0]
    _lib.check(lib.cotb200_sum_rows(_lib.dtype_code(outb), rows, C, *args, _p(outb), ldo, _st()), "sum_rows")
    _eq(outb[:, :C], sum(s.double() for s in src), name)
    if ldo > C:
        _eq(outb[:, C:], torch.full((rows, ldo - C), 7.0, device=DEV, dtype=torch.float64), name + " padding")


POOL_CASES = [  # name, dtype, N, H, W, C, element offset
    ("pool_bf16_vec8", "bf16", 2, 8, 8, 64, 0),
    ("pool_f32_oddhw_c3", "f32", 3, 7, 9, 3, 0),
    ("pool_f16_c33_offset", "f16", 2, 9, 6, 33, 1),
    ("pool_bf16_c40_offset", "bf16", 1, 5, 11, 40, 2),
]


def _pool_taps(x64, fill):
    """[N, C, 9, Ho*Wo] taps of the 3x3 / stride 2 / pad 1 windows of NHWC x, padding = fill"""
    N, H, W, C = x64.shape
    xp = F.pad(x64.permute(0, 3, 1, 2), (1, 1, 1, 1), value=fill)
    return F.unfold(xp, 3, stride=2).view(N, C, 9, -1)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name,dtype,N,H,W,C,off", POOL_CASES, ids=[c[0] for c in POOL_CASES])
def test_pool3s2_exact(name, dtype, N, H, W, C, off, mode):
    """average (sum * fl(1/9), as the kernel rounds it) and max (first maximum in scan order; integer inputs tie often) forward and
    their gather backward, at odd C and misaligned pointers"""
    lib, T, st = _lib.load(), TD[dtype], _st()
    dt = _lib.dtype_code(torch.empty(0, dtype=T))
    g = _gen(len(name) + 31 * mode)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    x = _ints((N, H, W, C), T, off, g)
    dy = _ints((N, Ho, Wo, C), T, off, g)
    y = _at((N, Ho, Wo, C), T, off)
    idx = torch.full((N, Ho, Wo, C), 0xEE, dtype=torch.uint8, device=DEV) if mode else None
    _lib.check(lib.cotb200_pool3s2_fwd(dt, mode, N, H, W, C, _p(x), _p(y), _p(idx), st), "pool3s2_fwd")
    ninth = torch.tensor(1.0 / 9.0, dtype=torch.float32, device=DEV)
    if mode == 0:
        taps = _pool_taps(x.double(), 0.0)
        want = (taps.sum(2).float() * ninth).double()
    else:
        taps = _pool_taps(x.double(), float("-inf"))
        want = taps.max(2).values
        first = ((taps == want.unsqueeze(2)).double() * torch.arange(9, 0, -1, device=DEV, dtype=torch.float64).view(1, 1, 9, 1)).argmax(2)
        _eq(idx, first.view(N, C, Ho, Wo).permute(0, 2, 3, 1).to(torch.uint8), name + " argmax")
    _eq(y, want.view(N, C, Ho, Wo).permute(0, 2, 3, 1), name + " fwd")
    dx = _at((N, H, W, C), T, off)
    _lib.check(lib.cotb200_pool3s2_bwd(dt, mode, N, H, W, C, _p(dy), _p(idx), _p(dx), st), "pool3s2_bwd")
    cols = dy.double().permute(0, 3, 1, 2).reshape(N, C, 1, Ho * Wo).expand(N, C, 9, Ho * Wo)
    if mode == 1:
        cols = cols * F.one_hot(first, 9).permute(0, 1, 3, 2).double()
    back = F.fold(cols.reshape(N, C * 9, Ho * Wo), (H + 2, W + 2), 3, stride=2)[:, :, 1:H + 1, 1:W + 1]
    if mode == 0:
        back = (back.float() * ninth).double()
    _eq(dx, back.permute(0, 2, 3, 1), name + " bwd")


# ------------------------------------------------------------------------------------------------ rejections
def test_rejections_launch_nothing():
    """ETOOBIG for B*HW >= 2^31 rows (checked on the host before any pointer is used), EINVAL for the 1-bit mask at C % 8 != 0 or
    at a column chunk that is not a multiple of 8 (vec 1: 264 channels in chunks of 132), for relu codes outside 0-3, for a mask
    next to relu != 1 (forward) or != 3 (backward), and for gn9 with gc not dividing wc.  None of them launches a kernel."""
    lib, st = _lib.load(), _st()
    bf = _lib.BF16
    x = torch.zeros(4096, device=DEV, dtype=torch.bfloat16)
    xo = x[1:]                                                       # 2-byte aligned only: vec 1
    f = torch.zeros(4096, device=DEV)
    m = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    P = _p
    big = (65536, 32768)                                             # 2^31 rows

    def apply_batch(B, HW, C, xp, relu, mask):
        return lib.cotb200_bn_apply_batch(bf, B, HW, C, xp, xp, P(f), P(f), None, None, None, None, 4.0, 1e-5, 0.1, 0, relu, xp,
                                          P(f), P(f), P(f), P(f), None, mask, st)

    def bwd_sums(B, HW, C, xp, relu, mask, y=None):
        return lib.cotb200_bn_bwd_sums(bf, B, HW, C, xp, xp, y, mask, P(f), P(f), P(f), P(f), relu, P(f), P(f), None, st)

    def bwd_apply(B, HW, C, xp, relu, mask, y=None):
        return lib.cotb200_bn_bwd_apply(bf, B, HW, C, xp, xp, y, mask, P(f), P(f), P(f), P(f), P(f), P(f), 0.25, relu, xp, None, None, st)

    checks = [
        ("col_stats rows", ETOOBIG, lambda: lib.cotb200_col_stats(bf, *big, 8, P(x), P(f), P(f), st)),
        ("bn_apply rows", ETOOBIG, lambda: lib.cotb200_bn_apply(bf, *big, 8, P(x), None, P(f), P(f), 1, P(x), None, st)),
        ("bn_apply_batch rows", ETOOBIG, lambda: apply_batch(*big, 8, P(x), 1, None)),
        ("bn_bwd_sums rows", ETOOBIG, lambda: bwd_sums(*big, 8, P(x), 0, None)),
        ("bn_bwd_apply rows", ETOOBIG, lambda: bwd_apply(*big, 8, P(x), 0, None)),
        ("pool3s2_fwd rows", ETOOBIG, lambda: lib.cotb200_pool3s2_fwd(bf, 0, *big, 4, 8, P(x), P(x), None, st)),
        ("pool3s2_bwd rows", ETOOBIG, lambda: lib.cotb200_pool3s2_bwd(bf, 1, *big, 4, 8, P(x), P(m), P(x), st)),
        ("apply_batch mask C%8", EINVAL, lambda: apply_batch(1, 4, 12, P(x), 1, P(m))),
        ("bwd_sums mask C%8", EINVAL, lambda: bwd_sums(1, 4, 12, P(x), 3, P(m))),
        ("bwd_apply mask C%8", EINVAL, lambda: bwd_apply(1, 4, 12, P(x), 3, P(m))),
        ("apply_batch mask chunk of 132", EINVAL, lambda: apply_batch(1, 4, 264, P(xo), 1, P(m))),
        ("bwd_sums mask chunk of 132", EINVAL, lambda: bwd_sums(1, 4, 264, P(xo), 3, P(m))),
        ("bwd_apply mask chunk of 132", EINVAL, lambda: bwd_apply(1, 4, 264, P(xo), 3, P(m))),
        ("bwd_sums relu 4", EINVAL, lambda: bwd_sums(1, 4, 8, P(x), 4, None)),
        ("bwd_sums relu -1", EINVAL, lambda: bwd_sums(1, 4, 8, P(x), -1, None)),
        ("bwd_apply relu 4", EINVAL, lambda: bwd_apply(1, 4, 8, P(x), 4, None)),
        ("apply_batch mask relu 0", EINVAL, lambda: apply_batch(1, 4, 8, P(x), 0, P(m))),
        ("bwd_sums mask relu 1", EINVAL, lambda: bwd_sums(1, 4, 8, P(x), 1, P(m), P(x))),
        ("bwd_apply mask relu 1", EINVAL, lambda: bwd_apply(1, 4, 8, P(x), 1, P(m), P(x))),
        ("gn9_stats gc", EINVAL, lambda: lib.cotb200_gn9_stats(bf, 1, 4, 12, 8, P(x), None, P(f), P(f), st)),
        ("gn9_apply gc", EINVAL, lambda: lib.cotb200_gn9_apply(bf, 1, 4, 12, 8, P(x), None, P(f), P(f), P(f), P(f), P(x), st)),
        ("gn9_bwd_sums gc", EINVAL, lambda: lib.cotb200_gn9_bwd_sums(bf, 1, 4, 12, 8, P(x), P(x), None, P(f), P(f), P(f), P(f), P(f),
                                                                     P(f), P(f), P(f), None, st)),
        ("gn9_bwd_apply gc", EINVAL, lambda: lib.cotb200_gn9_bwd_apply(bf, 1, 4, 12, 8, P(x), P(x), None, P(f), P(f), P(f), P(f), P(f),
                                                                       P(x), st)),
        ("sum_rows one source", ENULL, lambda: lib.cotb200_sum_rows(bf, 4, 8, P(x), 8, None, 0, None, 0, None, 0, P(x), 8, st)),
        ("sum_rows pitch < C", EINVAL, lambda: lib.cotb200_sum_rows(bf, 4, 8, P(x), 8, P(x), 4, None, 0, None, 0, P(x), 8, st)),
    ]
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    got = [(name, fn()) for name, _, fn in checks]
    torch.cuda.synchronize()
    assert [(name, rc) for name, rc in got] == [(name, want) for name, want, _ in checks]
    assert _lib.launch_count() == n0, "a rejected call launched a kernel"
    assert (x == 0).all() and (f == 0).all() and (m == 0).all()


# ------------------------------------------------------------------------------------------------ realistic values against fp64
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
# fp32 arithmetic error, relative to the magnitude of the terms (derived, not measured):
#   ELEM_SLACK for an element computed from its inputs by a few fp32 operations (<= 8 roundings of the largest term),
#   SUM_SLACK for a column or sample sum: a sequential chain of up to 128 additions per thread before the tree reductions.
ELEM_SLACK = 2.0 ** -20
SUM_SLACK = 2.0 ** -17


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_bn_realistic(dtype):
    """col_stats + bn_apply_batch + bn_bwd_sums + bn_bwd_apply on random activations against fp64.  y and dx within 2 output ulp of
    the fp64 value plus ELEM_SLACK of the magnitude of the terms (dx from the published sums, which are checked to SUM_SLACK); rstd
    within 2^-21 relative (4 fp32 ulp) for centred data, which keeps y inside ELEM_SLACK, and within 1e-4 for the
    shifted-mean columns (|mean|/std = 8): the kernels compute var = E[x^2] - mean^2 in fp32, which loses about log2(1 + 64) bits
    here.  Measured on an H100 SXM (132 SMs, 700 W): 1.5e-7 centred, 7.7e-6 shifted at most over the three dtypes."""
    lib, st = _lib.load(), _st()
    dt = _lib.dtype_code(torch.empty(0, dtype=dtype))
    B, HW, C = 4, 784, 96
    n = B * HW
    g = _gen(5)
    c = _cols(C)
    shifted = c >= C // 2
    mu_true = torch.where(shifted, 8.0 * torch.where(c % 2 == 0, 1.0, -1.0), 0.1)
    x = (torch.randn(n, C, generator=g, device=DEV) + mu_true).to(dtype)
    res = torch.randn(n, C, generator=g, device=DEV).to(dtype)
    dy = torch.randn(n, C, generator=g, device=DEV).to(dtype)
    x64, res64, dy64 = x.double(), res.double(), dy.double()
    sums = torch.zeros(2, C, device=DEV)
    _lib.check(lib.cotb200_col_stats(dt, B, HW, C, _p(x), _p(sums[0]), _p(sums[1]), st), "col_stats")
    w = torch.rand(C, generator=g, device=DEV) + 0.5
    b = torch.randn(C, generator=g, device=DEV) * 0.3
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    ss = torch.empty(4, C, device=DEV)
    y = torch.empty_like(x)
    _lib.check(lib.cotb200_bn_apply_batch(dt, B, HW, C, _p(x), _p(res), _p(sums[0]), _p(sums[1]), _p(w), _p(b), _p(rm), _p(rv), float(n),
                                   1e-5, 0.1, 1, 1, _p(y), _p(ss[0]), _p(ss[1]), _p(ss[2]), _p(ss[3]), None, None, st), "bn_apply_batch")
    mean64 = x64.mean(0)
    var64 = x64.var(0, unbiased=False)
    rstd64 = 1.0 / torch.sqrt(var64 + 1e-5)
    rel = (ss[3].double() - rstd64).abs() / rstd64
    print("rstd relative error, %s: centred %.3g, |mean|/std = 8: %.3g" % (dtype, rel[~shifted].max().item(), rel[shifted].max().item()))
    assert rel[~shifted].max().item() <= 2.0 ** -21 and rel[shifted].max().item() <= 1e-4
    # y on the centred columns (the shifted ones carry the rstd error above)
    sc64, sh64 = w.double() * rstd64, b.double() - mean64 * w.double() * rstd64
    y64 = (x64 * sc64 + sh64 + res64).clamp_min(0.0)
    mag = (x64 * sc64).abs() + (mean64 * sc64).abs() + b.double().abs() + res64.abs()
    tol = 2 * _ulp(y64, dtype) + ELEM_SLACK * mag
    r = _within(y[:, ~shifted], y64[:, ~shifted], tol[:, ~shifted], "bn y")
    # backward from the published statistics
    scale, mu, rstd = ss[0], ss[2], ss[3]
    s = torch.zeros(2, C, device=DEV)
    head = (dt, B, HW, C, _p(dy), _p(x), _p(y), None, _p(scale), None, _p(mu), _p(rstd))
    _lib.check(lib.cotb200_bn_bwd_sums(*head, 1, _p(s[0]), _p(s[1]), None, st), "bn_bwd_sums")
    dx = torch.empty_like(x)
    _lib.check(lib.cotb200_bn_bwd_apply(*head, _p(s[0]), _p(s[1]), 1.0 / n, 1, _p(dx), None, None, st), "bn_bwd_apply")
    dz = torch.where(y.double() > 0, dy64, 0.0)
    xhat = (x64 - mu.double()) * rstd.double()
    S0, S1 = dz.sum(0), (dz * xhat).sum(0)
    r0 = _within(s[0], S0, SUM_SLACK * dz.abs().sum(0) + 1e-30, "sum_dz")
    r1 = _within(s[1], S1, SUM_SLACK * (dz * xhat).abs().sum(0) + 1e-30, "sum_dzx")
    P0, P1 = s[0].double(), s[1].double()
    dx64 = scale.double() * (dz - P0 / n - xhat * P1 / n)
    mag = scale.double().abs() * (dz.abs() + P0.abs() / n + (xhat * P1).abs() / n)
    r2 = _within(dx, dx64, 2 * _ulp(dx64, dtype) + ELEM_SLACK * mag, "bn dx")
    print("bn %s: y at %.2f, sums at %.2f / %.2f, dx at %.2f of the bound" % (dtype, r, r0, r1, r2))


# tanh.approx.f32: the comment of sigmoid_t (norm_tail.cu) gives ~2.5e-4 absolute error of the 16-bit kernels' sigmoid
# (0.5 * tanh, whose approximation is good to 2^-11 relative); 4e-4 leaves room.  fp32 keeps ex2 + an approximate reciprocal, 2 ulp each.
SIGMOID_ABS = {torch.float32: 2.0 ** -20, torch.bfloat16: 4e-4, torch.float16: 4e-4}


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_tail_realistic(dtype):
    """tail_combine, tail_pool and the training-mode tail backward (dz_sums + apply) on random activations against fp64, with the
    sigmoid error bound of each dtype (SIGMOID_ABS) carried through silu = z*s and silu' = s*(1 + z*(1 - s))."""
    lib, st = _lib.load(), _st()
    dt = _lib.dtype_code(torch.empty(0, dtype=dtype))
    B, HW, C = 3, 196, 128
    g = _gen(6)
    u = (torch.randn(B, HW, C, generator=g, device=DEV) * 2).to(dtype)
    k = torch.randn(B, HW, C, generator=g, device=DEV).to(dtype)
    dout = torch.randn(B, HW, C, generator=g, device=DEV).to(dtype)
    scale = (torch.rand(C, generator=g, device=DEV) + 0.5)
    shift = torch.randn(C, generator=g, device=DEV) * 0.5
    a = torch.softmax(torch.randn(B, C, 2, generator=g, device=DEV), -1).contiguous()
    dpn = torch.randn(B, C, generator=g, device=DEV)
    u64, k64, d64 = u.double(), k.double(), dout.double()
    z = _f32(u64 * scale.double() + shift.double())
    sg = torch.sigmoid(z)
    y = z * sg
    eps_s = SIGMOID_ABS[dtype]
    a0, a1 = a[..., 0].double().unsqueeze(1), a[..., 1].double().unsqueeze(1)
    out = torch.empty_like(u)
    _lib.check(lib.cotb200_tail_combine(dt, B, HW, C, _p(u), _p(k), _p(scale), _p(shift), _p(a), _p(out), st), "tail_combine")
    want = a0 * y + a1 * k64
    tol = 2 * _ulp(want, dtype) + a0.abs() * z.abs() * eps_s + ELEM_SLACK * ((a0 * y).abs() + (a1 * k64).abs())
    r1 = _within(out, want, tol, "tail_combine")
    ps = torch.zeros(B, C, device=DEV)
    _lib.check(lib.cotb200_tail_pool(dt, B, HW, C, _p(u), _p(k), _p(scale), _p(shift), _p(ps), st), "tail_pool")
    rp = _within(ps, (y + k64).sum(1), (z.abs() * eps_s).sum(1) + SUM_SLACK * (y.abs() + k64.abs()).sum(1), "tail_pool")
    mu = torch.randn(C, generator=g, device=DEV) * 0.1
    rstd = torch.rand(C, generator=g, device=DEV) + 0.5
    s = torch.zeros(2, C, device=DEV)
    pscale = 1.0 / HW
    _lib.check(lib.cotb200_tail_bwd_dz_sums(dt, B, HW, C, _p(dout), _p(u), _p(scale), _p(shift), _p(mu), _p(rstd), _p(a), _p(dpn), pscale,
                                     _p(s[0]), _p(s[1]), st), "tail_bwd_dz_sums")
    g0 = a0 * d64 + dpn.double().unsqueeze(1) * pscale
    ds_ = sg * (1 + z * (1 - sg))
    dz = g0 * ds_
    dz_err = g0.abs() * eps_s * (1 + 2 * z.abs()) + ELEM_SLACK * dz.abs()      # |d silu'/ds| <= 1 + 2|z|
    xhat = (u64 - mu.double()) * rstd.double()
    _within(s[0], dz.sum((0, 1)), dz_err.sum((0, 1)) + SUM_SLACK * dz.abs().sum((0, 1)), "tail sum_dz")
    _within(s[1], (dz * xhat).sum((0, 1)), (dz_err * xhat.abs()).sum((0, 1)) + SUM_SLACK * (dz * xhat).abs().sum((0, 1)), "tail sum_dzx")
    n = B * HW
    du = torch.empty_like(u)
    _lib.check(lib.cotb200_tail_bwd_apply(dt, B, HW, C, _p(dout), _p(u), _p(scale), _p(shift), _p(mu), _p(rstd), _p(a), _p(dpn), _p(s[0]),
                                   _p(s[1]), 1.0 / n, pscale, _p(du), None, st), "tail_bwd_apply")
    S0, S1 = s[0].double(), s[1].double()                # the sums as published: this checks the apply's arithmetic
    want = scale.double() * (dz - S0 / n - xhat * S1 / n)
    tol = 2 * _ulp(want, dtype) + scale.double() * (dz_err + ELEM_SLACK * (dz.abs() + S0.abs() / n + (xhat * S1).abs() / n))
    r2 = _within(du, want, tol, "tail du")
    print("tail %s: combine at %.2f, pool at %.2f, du at %.2f of the bound" % (dtype, r1, rp, r2))


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_gn9_realistic(dtype):
    """gn9_stats -> mean / rstd in fp64 -> gn9_apply on random logits (fast path, gc = 8) against fp64, within 2 output ulp plus
    ELEM_SLACK of the magnitude; the statistics to SUM_SLACK of the sums of |l| and l^2."""
    lib, st = _lib.load(), _st()
    dt = _lib.dtype_code(torch.empty(0, dtype=dtype))
    B, HW, wc, gc = 2, 196, 16, 8
    J = 9 * wc
    g = _gen(7)
    l = (torch.randn(B, HW, J, generator=g, device=DEV) * 3 + 1).to(dtype)
    lb = torch.randn(J, generator=g, device=DEV) * 0.5
    gamma = torch.rand(J, generator=g, device=DEV) + 0.5
    beta = torch.randn(J, generator=g, device=DEV) * 0.2
    lv = l.double() + lb.double()
    gs = torch.zeros(2, B, wc, device=DEV)
    _lib.check(lib.cotb200_gn9_stats(dt, B, HW, wc, gc, _p(l), _p(lb), _p(gs[0]), _p(gs[1]), st), "gn9_stats")
    lg = lv.view(B, HW, wc, 9)
    _within(gs[0], lg.sum((1, 3)), SUM_SLACK * lg.abs().sum((1, 3)), "gn9 sum")
    _within(gs[1], (lg * lg).sum((1, 3)), SUM_SLACK * (lg * lg).sum((1, 3)), "gn9 sq")
    m64 = lg.mean((1, 3))
    r64 = 1.0 / torch.sqrt(lg.var((1, 3), unbiased=False) + 1e-5)
    mean, rstd = m64.float(), r64.float()
    out = torch.empty_like(l)
    _lib.check(lib.cotb200_gn9_apply(dt, B, HW, wc, gc, _p(l), _p(lb), _p(mean), _p(rstd), _p(gamma), _p(beta), _p(out), st), "gn9_apply")
    mj, rj = mean.double().repeat_interleave(9, 1).unsqueeze(1), rstd.double().repeat_interleave(9, 1).unsqueeze(1)
    want = torch.empty_like(lv)
    pos = _gn_pos(J, gc)
    want[..., pos] = (lv - mj) * rj * gamma.double() + beta.double()
    mag = torch.empty_like(lv)
    mag[..., pos] = (lv.abs() + mj.abs()) * rj * gamma.double() + beta.double().abs()
    r = _within(out, want, 2 * _ulp(want, dtype) + ELEM_SLACK * mag, "gn9_apply")
    print("gn9 %s: apply at %.2f of the bound" % (dtype, r))
