"""Which kernel serves a call of the other LocalConv variants, mirrored in Python and checked without a GPU.

cotb200_agg_refpad_* and cotb200_agg_zeropad_dilate_* (csrc/agg_variants.cu) and cotb200_agg_zeropad_mix_merge_*
(csrc/agg_zeropad.cu) pick their kernels from the geometry and the dtype alone.  This file holds

  * a Python copy of that dispatch: for a descriptor, a dtype and an SM count, the launches a call makes, each with its
    profiler record, its kernel and sub-branch, its grid and the grid-stride passes of its busiest thread.  mix_merge runs
    through fwd_impl / bwd_impl, whose copy is test_agg_geometry_cpu's;
  * source anchors: the literal conditions the copy follows must still be in the .cu files, so an edit to the dispatch fails
    here until the copy follows it;
  * VCASES, the named calls tests/test_variant_kernels_gpu.py runs on the GPU, and a check that together they reach every
    reachable (kernel, sub-branch) pair in every dtype, and run every kernel past its first grid-stride pass at 132 and 114 SMs;
  * the operand ranges that keep every output of an integer case exact, from the largest number of products a sum can have;
  * the argument checks of the six entry points through the C ABI; they return before any launch."""
import ctypes
import os
from collections import Counter, namedtuple

import pytest
import torch

import test_agg_geometry_cpu as tg
from cotnet_b200 import _lib
from oracle.agg_ref import _reflect

SMS_H100 = tg.SMS_H100
ES = tg.ES
DTYPES = ("fp32", "fp64", "bf16", "fp16")
THREADS = 256


def _cdiv(a, b):
    return -(-a // b)


# ================================================================================================ launches
class Launch(namedtuple("Launch", "prof kernel tags total per_sm")):
    """One kernel launch.  prof: the profiler record it opens (None when it runs inside the previous launch's record);
    kernel / tags: the kernel and its sub-branches; total, per_sm: the grid-stride work items and grid_stride_blocks' cap."""

    def grid(self, sms):
        return min(max(1, _cdiv(self.total, THREADS)), sms * self.per_sm)

    def passes(self, sms):
        """grid-stride iterations of the busiest thread"""
        return _cdiv(self.total, self.grid(sms) * THREADS)

    def names(self):
        return {self.kernel} | {"%s/%s" % (self.kernel, t) for t in self.tags}


class VDesc:
    """struct cotb200_agg_desc of one variant call (NCHW).  op: "refpad", "dilate" or "merge"; k2 / p2: the second kernel of
    mix_merge; dil: the dilation of each weight channel."""

    def __init__(self, op, N, C, H, W, wc, k=3, heads=1, s=1, d=1, p=None, k2=5, p2=None, dil=None):
        kh, kw = (k, k) if isinstance(k, int) else k
        ph, pw = (d * (kh // 2), d * (kw // 2)) if p is None else ((p, p) if isinstance(p, int) else p)
        self.op, self.n, self.c, self.h, self.w, self.heads, self.wc = op, N, C, H, W, heads, wc
        self.kh, self.kw, self.sh, self.sw, self.ph, self.pw, self.dh, self.dw = kh, kw, s, s, ph, pw, d, d
        if op == "dilate":                       # what aggregation_zeropad_dilate passes: 3x3, stride 1, output = input
            assert kh == kw == 3 and dil is not None and len(dil) == wc
            self.sh = self.sw = self.dh = self.dw = 1
            self.ph = self.pw = 0
            self.ho, self.wo = H, W
        else:
            self.ho = (H + 2 * ph - (d * (kh - 1) + 1)) // s + 1
            self.wo = (W + 2 * pw - (d * (kw - 1) + 1)) // s + 1
        self.k2 = k2
        self.p2 = k2 // 2 * d if p2 is None else p2
        self.dil = tuple(dil) if dil is not None else None

    def agg_desc(self):
        """the zeropad descriptor of mix_merge's first kernel (test_agg_geometry_cpu.Desc)"""
        return tg.Desc(self.n, self.c, self.h, self.w, self.wc, k=(self.kh, self.kw), heads=self.heads, s=self.sh, d=self.dh,
                       p=(self.ph, self.pw))

    def fields(self):
        return dict(n=self.n, c=self.c, h=self.h, w=self.w, heads=self.heads, wc=self.wc, kh=self.kh, kw=self.kw, sh=self.sh,
                    sw=self.sw, ph=self.ph, pw=self.pw, dh=self.dh, dw=self.dw, ho=self.ho, wo=self.wo, layout=0, gc=0, fold=1)

    def __repr__(self):
        s = "%s(N=%d C=%d %dx%d wc=%d heads=%d k=%dx%d s=%d d=%d p=%d,%d" % (
            self.op, self.n, self.c, self.h, self.w, self.wc, self.heads, self.kh, self.kw, self.sh, self.dh, self.ph, self.pw)
        if self.op == "merge":
            s += " k2=%d p2=%d" % (self.k2, self.p2)
        if self.op == "dilate":
            s += " dil=%s" % (list(self.dil),)
        return s + ")"


LIM31 = 1 << 31


# ---- refpad (agg_variants.cu: cotb200_agg_refpad_fwd / _bwd)
def reflect_sources(i, n, pad):
    """reflect_sources: the un-shifted padded coordinates that reflect onto i"""
    src = [i]
    if 1 <= i <= pad:
        src.append(-i)
    if n - 1 - pad <= i <= n - 2:
        src.append(2 * (n - 1) - i)
    return src


def _has_src3(n, pad):
    return any(len(reflect_sources(i, n, pad)) == 3 for i in range(n))


def refpad_fwd(d):
    total = d.n * d.heads * d.c * d.ho * d.wo
    rep = d.c // d.wc
    small = total < LIM31 and d.n * d.heads * d.wc * d.kh * d.kw * d.ho * d.wo < LIM31 and d.h * d.w < 1 << 24
    if small and d.kh == d.kw and d.kh in (3, 5, 7):
        return [Launch("agg_refpad_fwd", "refpad_fwd_fast", frozenset({"K%d" % d.kh}), total // rep, 16)]
    tags = {"large"} if not small else {"rect" if d.kh != d.kw else "square"}
    return [Launch("agg_refpad_fwd", "refpad_fwd_generic", frozenset(tags), total, 16)]


def _stride_dil(d):
    return (d.sh > 1 or d.sw > 1) and (d.dh > 1 or d.dw > 1)


def refpad_bwd(d, dx, dw):
    out = []
    if dx:
        t = set()
        if _has_src3(d.h, d.ph) and _has_src3(d.w, d.pw):
            t.add("src3x3")
        if _stride_dil(d):
            t.add("stride-dil")
        if d.heads > 1:
            t.add("heads")
        if d.kh != d.kw:
            t.add("rect")
        out.append(Launch("agg_refpad_dx", "refpad_dx", frozenset(t), d.n * d.c * d.h * d.w, 16))
    if dw:
        t = set()
        if d.wc == 1:
            t.add("wc1")
        if d.wc == d.c:
            t.add("wcC")
        if _stride_dil(d):
            t.add("stride-dil")
        out.append(Launch("agg_refpad_dw", "refpad_dw", frozenset(t), d.n * d.heads * d.wc * d.kh * d.kw * d.ho * d.wo, 16))
    return out


# ---- dilate (agg_variants.cu: cotb200_agg_zeropad_dilate_fwd / _bwd)
def _dilate_tags(d):
    t = set()
    if any(v >= d.h or v >= d.w for v in d.dil):
        t.add("beyond")                          # every tap but the centre falls off the plane
    if 1 in d.dil and any(v >= max(d.h, d.w) for v in d.dil):
        t.add("mixed")                           # dilation 1 next to one that covers the whole plane
    if d.heads > 1:
        t.add("heads")
    return t


def dilate_fwd(d):
    total = d.n * d.heads * d.c * d.h * d.w
    t = _dilate_tags(d)
    if total < LIM31 and d.n * d.heads * d.wc * 9 * d.h * d.w < LIM31:
        return [Launch("agg_dilate_fwd", "dilate_fwd_fast", frozenset(t), total // (d.c // d.wc), 16)]
    return [Launch("agg_dilate_fwd", "dilate_fwd_kernel", frozenset(t | {"large"}), total, 16)]


def dilate_bwd(d, dx, dw):
    t = frozenset(_dilate_tags(d))
    out = []
    if dx:
        out.append(Launch("agg_dilate_dx", "dilate_dx", t, d.n * d.c * d.h * d.w, 16))
    if dw:
        out.append(Launch("agg_dilate_dw", "dilate_dw", t, d.n * d.heads * d.wc * 9 * d.h * d.w, 16))
    return out


# ---- mix_merge (agg_zeropad.cu: cotb200_agg_zeropad_mix_merge_fwd / _bwd over fwd_impl / bwd_impl)
class _Capture(tg.Pred):
    """test_agg_geometry_cpu's Pred that also keeps each launch's grid-stride size"""

    def __init__(self):
        super().__init__()
        self.loops = []

    def add(self, name, *tags, loop=None):
        assert loop is not None, "%s: mix_merge reaches only grid-stride kernels" % name
        super().add(name, *tags, loop=loop)
        self.loops.append(loop)


def merge_geos(d):
    """resolve_mix + merge_strides: both halves, outputs interleaved per sample, weights packed per sample"""
    a = d.agg_desc()
    b = tg.Desc(d.n, d.c, d.h, d.w, d.wc, k=d.k2, heads=d.heads, s=d.sh, d=d.dh, p=d.p2)
    assert b.ho * b.wo == a.ho * a.wo, "the two kernels of mix_merge must give one output size"
    g1, g2 = tg.resolve(a), tg.resolve(b)
    g1.y_sn *= 2
    g2.y_sn *= 2
    plane = g1.HO * g1.WO
    tot = g1.heads * g1.wc * (g1.K2 + g2.K2) * plane
    g1.w_sn = g2.w_sn = tot
    return g1, g2, g1.heads * g1.wc * g1.K2 * plane, g1.heads * g1.C * plane


FWD_BRANCH = {"agg_fwd_nchw_k3": "nchw_k3", "agg_fwd_nchw_k5": "nchw_k5", "agg_fwd_generic": "generic"}


def _merge_launches(P, kernel, branch_of, extra):
    out = []
    for (name, _), (total, per_sm) in zip(P.launches, P.loops):
        out.append(Launch(name, kernel, frozenset({branch_of(name)} | extra), total, per_sm))
    return out


def merge_fwd(d, dt):
    g1, g2, off2, half = merge_geos(d)
    es = ES[dt]
    P = _Capture()
    tg.fwd_impl(P, g1, es, (0, 0, 0))
    tg.fwd_impl(P, g2, es, (0, off2, half))
    return _merge_launches(P, "merge_fwd", FWD_BRANCH.__getitem__, {"n>2"} if d.n > 2 else set())


def merge_bwd(d, dt, dx, dw):
    g1, g2, off2, half = merge_geos(d)
    es = ES[dt]
    call = "dxdw" if dx and dw else ("dx" if dx else "dw")
    extra = {"n>2"} if d.n > 2 else set()
    if es >= 4 and tg.is_same3(g1, 3) and tg.is_same3(g2, 5) and tg.fits32(g2):
        P = _Capture()
        tg.bwd_impl(P, g1, es, (0, 0, 0, 0 if dx else None, 0 if dw else None), dx, dw)
        tg.bwd_impl(P, g2, es, (half, 0, off2, 0 if dx else None, off2 if dw else None), dx, dw, acc_dx=dx)
        return _merge_launches(P, "merge_bwd", lambda _: "fused-" + call, extra)
    tags = frozenset({"generic2-" + call} | extra)
    out = []
    if dx:
        out.append(Launch("agg_mix_merge_dx", "merge_bwd", tags, g1.N * g1.C * g1.H * g1.W, 16))
    if dw:                                     # two agg_dw_generic launches inside one profiler record
        out.append(Launch("agg_mix_merge_dw", "merge_bwd", tags, g1.N * g1.heads * g1.wc * g1.K2 * g1.HO * g1.WO, 16))
        out.append(Launch(None, "merge_bwd", tags, g2.N * g2.heads * g2.wc * g2.K2 * g2.HO * g2.WO, 16))
    return out


BWD_VARIANTS = tg.BWD_VARIANTS                 # ("dxdw", True, True), ("dx", True, False), ("dw", False, True)


def predict(c):
    """{call: [Launch]}: the forward and the backward with both gradients, dX only and dW only"""
    d = c.desc
    if d.op == "refpad":
        out = {"fwd": refpad_fwd(d)}
        out.update((v, refpad_bwd(d, dx, dw)) for v, dx, dw in BWD_VARIANTS)
    elif d.op == "dilate":
        out = {"fwd": dilate_fwd(d)}
        out.update((v, dilate_bwd(d, dx, dw)) for v, dx, dw in BWD_VARIANTS)
    else:
        out = {"fwd": merge_fwd(d, c.dt)}
        out.update((v, merge_bwd(d, c.dt, dx, dw)) for v, dx, dw in BWD_VARIANTS)
    return out


def profile_names(launches):
    """{profiler record: count} of one call"""
    return dict(Counter(l.prof for l in launches if l.prof))


def case_names(c):
    out = set()
    for launches in predict(c).values():
        for l in launches:
            out |= l.names()
    return out


# ================================================================================================ operand bounds
def refpad_dx_terms(d):
    """the largest number of products in one dX sum of refpad_dx_kernel: heads x (source, tap) pairs per axis"""
    def axis(n, pad, k, s, dd, no):
        best = 0
        for i in range(n):
            cnt = 0
            for src in reflect_sources(i, n, pad):
                for kk in range(k):
                    hs = src + pad - kk * dd
                    cnt += hs >= 0 and hs % s == 0 and hs // s < no
            best = max(best, cnt)
        return best
    return d.heads * axis(d.h, d.ph, d.kh, d.sh, d.dh, d.ho) * axis(d.w, d.pw, d.kw, d.sw, d.dw, d.wo)


def max_terms(d):
    """the largest number of products summed into one output element of the forward, dX or dW"""
    rep = d.c // d.wc
    if d.op == "refpad":
        return max(d.kh * d.kw, refpad_dx_terms(d), rep)
    if d.op == "dilate":
        return max(9 * d.heads, rep)
    k1, k2 = d.kh * d.kw, d.k2 * d.k2
    return max(k1, k2, d.heads * (k1 + k2), rep)


EXACT_LIMIT = {"bf16": 1 << 8, "fp16": 1 << 11, "fp32": 1 << 24, "fp64": 1 << 53}
AMP_MAX = 3


def amplitude(c):
    """largest a <= AMP_MAX such that operands drawn from [-a, a] keep every sum (and so every fp32 partial sum and the final
    rounding to the storage type) exact: max_terms * a^2 <= 2^8 (bf16), 2^11 (fp16), 2^24 (fp32)"""
    n = max_terms(c.desc)
    for a in range(AMP_MAX, 0, -1):
        if n * a * a <= EXACT_LIMIT[c.dt]:
            return a
    raise AssertionError("%s: %d products per sum are not exact in %s even at amplitude 1" % (c.name, n, c.dt))


# ================================================================================================ cases
VCase = namedtuple("VCase", "name dt desc kind expect")


def vcase(name, dt, desc, expect=(), kind="int"):
    return VCase(name, dt, desc, kind, frozenset(expect))


def R(*a, **k):
    return VDesc("refpad", *a, **k)


def DL(*a, **k):
    return VDesc("dilate", *a, **k)


def M(*a, **k):
    return VDesc("merge", *a, **k)


# Small geometries, each run in all four dtypes
SMALL = [
    ("refpad-k3-heads2", R(2, 8, 7, 6, 4, heads=2, p=1), {"refpad_fwd_fast/K3", "refpad_dx/heads"}),
    # pad = H - 1 = W - 1: the middle pixel gathers from three padded positions on both axes; wc = 1
    ("refpad-k5-pad-max", R(2, 3, 5, 5, 1, k=5, p=4), {"refpad_fwd_fast/K5", "refpad_dx/src3x3", "refpad_dw/wc1"}),
    ("refpad-k7-wcC", R(2, 6, 9, 8, 6, k=7, p=3), {"refpad_fwd_fast/K7", "refpad_dw/wcC"}),
    # stride 2 with dilation 2: the hs % SH skips of the dX kernel on a dilated grid
    ("refpad-k3-s2-d2", R(2, 8, 9, 10, 2, s=2, d=2, p=2), {"refpad_fwd_fast/K3", "refpad_dx/stride-dil", "refpad_dw/stride-dil"}),
    ("refpad-rect-3x5", R(2, 6, 6, 9, 3, k=(3, 5), heads=2, p=(1, 2)), {"refpad_fwd_generic/rect", "refpad_dx/rect"}),
    ("refpad-k4-s2", R(2, 4, 8, 7, 2, k=4, s=2, p=2), {"refpad_fwd_generic/square"}),
    # dilation 1 next to one >= W = 9 and one >= H = 7 (only the centre tap stays on the plane)
    ("dilate-mixed-heads2", DL(2, 8, 7, 9, 4, heads=2, dil=(1, 9, 2, 7)), {"dilate_fwd_fast/mixed", "dilate_dx/beyond",
                                                                           "dilate_dw/heads"}),
    ("dilate-wc1-beyond", DL(3, 3, 5, 6, 1, dil=(6,)), {"dilate_fwd_fast/beyond", "dilate_dw/beyond"}),
    ("dilate-mixed", DL(2, 6, 6, 6, 2, dil=(1, 6)), {"dilate_dx/mixed", "dilate_dw/mixed"}),
    # 3x3 / 5x5 same-pad, heads 1, N = 3: the register-resident forwards, the fused backward for fp32 / fp64
    ("merge-same-n3", M(3, 8, 7, 7, 4), {"merge_fwd/n>2", "merge_bwd/n>2"}),
    ("merge-heads2", M(2, 8, 6, 5, 2, heads=2), {"merge_fwd/generic", "merge_bwd/generic2-dxdw"}),
    ("merge-s2-n3", M(3, 4, 9, 8, 2, s=2, p=1, p2=2), {"merge_fwd/generic", "merge_bwd/generic2-dw"}),
]

# Past the first grid-stride pass (grid_stride_blocks caps the grid at num_sms x 16 CTAs of 256 threads, x 8 for the
# register-resident zeropad kernels), with more than one input channel per weight channel, so that rep is walked on later passes
LOOPS = [
    ("loop-refpad-k3", "bf16", R(2, 16, 192, 192, 8, p=1), {"refpad_fwd_fast/K3"}),
    ("loop-refpad-rect", "fp32", R(2, 8, 192, 192, 4, k=(3, 5), p=(1, 2)), {"refpad_fwd_generic/rect"}),
    ("loop-dilate", "fp16", DL(2, 16, 192, 192, 8, dil=(1, 2, 5, 192, 3, 1, 64, 7)), {"dilate_fwd_fast/mixed"}),
    ("loop-merge-fp32", "fp32", M(4, 16, 96, 96, 8), {"merge_fwd/nchw_k5", "merge_bwd/fused-dxdw"}),
    ("loop-merge-bf16", "bf16", M(4, 16, 96, 96, 8), {"merge_fwd/nchw_k3", "merge_bwd/generic2-dxdw"}),
    ("loop-merge-fp64", "fp64", M(4, 16, 96, 96, 2), {"merge_fwd/generic", "merge_bwd/fused-dx"}),
]

# Random operands: the widen-and-round steps of each variant in each dtype, against fp64 under a unit-roundoff bound
FLOATS = [
    ("float-refpad", R(2, 8, 7, 6, 4, heads=2, p=1)),
    ("float-refpad-generic", R(2, 6, 6, 9, 3, k=(3, 5), p=(1, 2))),
    ("float-dilate", DL(2, 8, 7, 9, 4, heads=2, dil=(1, 9, 2, 3))),
    ("float-merge", M(3, 8, 7, 7, 4)),
]

VCASES = (
    [vcase("%s-%s" % (n, dt), dt, d, e) for n, d, e in SMALL for dt in DTYPES]
    + [vcase(n, dt, d, e) for n, dt, d, e in LOOPS]
    + [vcase("%s-%s" % (n, dt), dt, d, kind="float") for n, d in FLOATS for dt in DTYPES]
)

# Every (kernel, sub-branch) pair of the dispatch
ALL_PAIRS = (
    {"refpad_fwd_fast/K%d" % k for k in (3, 5, 7)}
    | {"refpad_fwd_generic/rect", "refpad_fwd_generic/square", "refpad_fwd_generic/large"}
    | {"refpad_dx/%s" % t for t in ("src3x3", "stride-dil", "heads", "rect")}
    | {"refpad_dw/%s" % t for t in ("wc1", "wcC", "stride-dil")}
    | {"%s/%s" % (k, t) for k in ("dilate_fwd_fast", "dilate_dx", "dilate_dw") for t in ("beyond", "mixed", "heads")}
    | {"dilate_fwd_kernel/large"}
    | {"merge_fwd/%s" % t for t in ("nchw_k3", "nchw_k5", "generic", "n>2")}
    | {"merge_bwd/%s-%s" % (b, v) for b in ("fused", "generic2") for v in ("dxdw", "dx", "dw")} | {"merge_bwd/n>2"}
)
# Pairs that need a tensor of >= 2^31 elements (multi-GB): reached by the mirror only (test_exemptions_need_2g_elements)
EXEMPT = {"refpad_fwd_generic/large", "dilate_fwd_kernel/large"}
# Pairs a dtype cannot reach
UNREACHABLE = {
    # the register-resident zeropad kernels accumulate in fp32: fp64 takes agg_fwd_generic
    "fp64": {"merge_fwd/nchw_k3", "merge_fwd/nchw_k5"},
    # 16-bit dX must be summed over both halves before its one rounding: agg_dx_generic2, never the fused pair
    "bf16": {"merge_bwd/fused-dxdw", "merge_bwd/fused-dx", "merge_bwd/fused-dw"},
    "fp16": {"merge_bwd/fused-dxdw", "merge_bwd/fused-dx", "merge_bwd/fused-dw"},
}
# The kernel of each profiler record: every one must run >= 2 grid-stride passes in some case at both SM counts
LOOP_KERNELS = {"agg_refpad_fwd/refpad_fwd_fast", "agg_refpad_fwd/refpad_fwd_generic", "agg_refpad_dx/refpad_dx",
                "agg_refpad_dw/refpad_dw", "agg_dilate_fwd/dilate_fwd_fast", "agg_dilate_dx/dilate_dx", "agg_dilate_dw/dilate_dw",
                "agg_fwd_nchw_k3/merge_fwd", "agg_fwd_nchw_k5/merge_fwd", "agg_fwd_generic/merge_fwd",
                "agg_bwd_nchw_dxdw/merge_bwd", "agg_bwd_nchw_dx/merge_bwd", "agg_bwd_nchw_dw/merge_bwd",
                "agg_dx_generic/merge_bwd", "agg_dw_generic/merge_bwd", "agg_mix_merge_dx/merge_bwd", "agg_mix_merge_dw/merge_bwd",
                "None/merge_bwd"}


def required(dt):
    return ALL_PAIRS - EXEMPT - UNREACHABLE.get(dt, set())


def case_bytes(c):
    """device bytes of the operands and outputs of a case in its dtype"""
    d = c.desc
    x = d.n * d.c * d.h * d.w
    K2 = d.kh * d.kw + (d.k2 * d.k2 if d.op == "merge" else 0)
    w = d.n * d.heads * d.wc * K2 * d.ho * d.wo
    y = d.n * d.heads * d.c * d.ho * d.wo * (2 if d.op == "merge" else 1)
    return 2 * (x + w + y) * ES[c.dt]


def oracle_elements(c):
    """elements of the largest fp64 intermediate of the Unfold oracle for one sample (the GPU test runs it sample by sample)"""
    d = c.desc
    K2 = max(d.kh * d.kw, d.k2 * d.k2 if d.op == "merge" else 0)
    return d.heads * d.c * K2 * d.ho * d.wo


# ================================================================================================ tests
def _src(name):
    with open(os.path.join(tg.CSRC, name)) as f:
        return f.read()


ANCHORS = {
    "agg_variants.cu": [
        # vresolve
        "if (d->layout != COTB200_NCHW) { set_error(\"%s supports the NCHW layout only (the reference contract)\", what); return COTB200_ELAYOUT; }",
        "if (d->n <= 0 || d->c <= 0 || d->h <= 0 || d->w <= 0 || d->heads <= 0 || d->wc <= 0 || d->kh <= 0 || d->kw <= 0 || d->ho <= 0 || d->wo <= 0) {",
        "if (d->c % d->wc) {",
        "if (d->kh != 3 || d->kw != 3) {",
        "if (d->ho != d->h || d->wo != d->w) {",
        "if (d->sh <= 0 || d->sw <= 0 || d->dh <= 0 || d->dw <= 0 || d->ph < 0 || d->pw < 0) {",
        "if (d->ph >= d->h || d->pw >= d->w) {",
        "if (span_h < 0 || span_w < 0) {",
        "const int ho = span_h / d->sh + 1, wo = span_w / d->sw + 1;",
        "if (ho * wo != d->ho * d->wo) {",
        # refpad
        "const long long total = (long long)g.N * g.heads * g.C * g.HO * g.WO;",
        "const long long items = total / g.rep;",
        "const bool small = total < (1LL << 31) && (long long)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO < (1LL << 31) && g.H * g.W < (1 << 24);",
        "if (small && g.KH == g.KW && (g.KH == 3 || g.KH == 5 || g.KH == 7)) {",
        "if (g.KH == 3) refpad_fwd_fast<T, 3><<<grid_stride_blocks(items, 256, 16), 256, 0, st>>>",
        "else if (g.KH == 5) refpad_fwd_fast<T, 5><<<grid_stride_blocks(items, 256, 16), 256, 0, st>>>",
        "else refpad_fwd_fast<T, 7><<<grid_stride_blocks(items, 256, 16), 256, 0, st>>>",
        "refpad_fwd_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>",
        "const long long total = (long long)g.N * g.C * g.H * g.W;\n      COTB200_PROF(\"agg_refpad_dx\");\n"
        "      refpad_dx_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>",
        "const long long total = (long long)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO;\n      COTB200_PROF(\"agg_refpad_dw\");\n"
        "      refpad_dw_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>",
        "if (i >= 1 && i <= pad) src[k++] = -i;",
        "if (i <= n - 2 && i >= n - 1 - pad) src[k++] = 2 * (n - 1) - i;",
        # dilate
        "const long long total = (long long)g.N * g.heads * g.C * g.H * g.W;",
        "if (total < (1LL << 31) && (long long)g.N * g.heads * g.wc * 9 * g.H * g.W < (1LL << 31))\n"
        "      dilate_fwd_fast<T><<<grid_stride_blocks(total / g.rep, 256, 16), 256, 0, st>>>",
        "dilate_fwd_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>",
        "const long long total = (long long)g.N * g.C * g.H * g.W;\n      COTB200_PROF(\"agg_dilate_dx\");\n"
        "      dilate_dx_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>",
        "const long long total = (long long)g.N * g.heads * g.wc * 9 * g.H * g.W;\n      COTB200_PROF(\"agg_dilate_dw\");\n"
        "      dilate_dw_kernel<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>",
        "COTB200_PROF_B(\"agg_refpad_fwd\"",
        "COTB200_PROF_B(\"agg_dilate_fwd\"",
    ],
    "agg_zeropad.cu": [
        "if (d->layout != COTB200_NCHW) { set_error(\"agg_zeropad_mix supports the NCHW layout only\"); return COTB200_ELAYOUT; }",
        "d2.kh = k2h; d2.kw = k2w; d2.ph = p2h; d2.pw = p2w;",
        "g1.y_sn *= 2; g2.y_sn *= 2;",
        "const long long tot = (long long)g1.heads * g1.wc * (g1.K2 + g2.K2) * plane;",
        "off2 = (long long)g1.heads * g1.wc * g1.K2 * plane;",
        "g1.w_sn = tot; g2.w_sn = tot;",
        "rc = fwd_impl<T>(g1, (const T*)x, (const T*)w, (T*)y, st);",
        "return fwd_impl<T>(g2, (const T*)x, (const T*)w + off2, (T*)y + half, st);",
        "if (sizeof(T) >= 4 && is_same3(g1, 3) && is_same3(g2, 5) && fits32(g2)) {\n"
        "      rc = bwd_impl<T>(g1, (const T*)dy, (const T*)x, (const T*)w, (T*)dx, (T*)dw, false, st);",
        "return bwd_impl<T>(g2, (const T*)dy + half, (const T*)x, (const T*)w + off2, (T*)dx, dw ? (T*)dw + off2 : (T*)nullptr, dx != nullptr, st);",
        "COTB200_PROF(\"agg_mix_merge_dx\");\n      agg_dx_generic2<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)w, g1,",
        "COTB200_PROF(\"agg_mix_merge_dw\");\n      const long long t1 = (long long)g1.N * g1.heads * g1.wc * g1.K2 * g1.HO * g1.WO;\n"
        "      agg_dw_generic<T><<<grid_stride_blocks(t1, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)x, (T*)dw, g1, t1);",
        "const long long t2 = (long long)g2.N * g2.heads * g2.wc * g2.K2 * g2.HO * g2.WO;\n"
        "      agg_dw_generic<T><<<grid_stride_blocks(t2, 256, 16), 256, 0, st>>>((const T*)dy + half, (const T*)x, (T*)dw + off2, g2, t2);",
        "if (span_h < 0 || span_w < 0) {",
    ],
}


@pytest.mark.parametrize("fname", sorted(ANCHORS))
def test_dispatch_anchors(fname):
    """the conditions the mirror copies are still the ones in the sources (whitespace-insensitive)"""
    missing = tg._missing_anchors(fname, ANCHORS[fname])
    assert not missing, "%s no longer contains (update the mirror in this file): %s" % (fname, missing)


def test_case_names_unique_and_valid():
    names = [c.name for c in VCASES]
    assert len(names) == len(set(names))
    for c in VCASES:
        d = c.desc
        assert c.dt in ES and c.kind in ("int", "float") and d.c % d.wc == 0 and d.ho > 0 and d.wo > 0
        if d.op == "refpad":
            assert d.ph < d.h and d.pw < d.w
        if d.op == "merge":
            merge_geos(d)


@pytest.mark.parametrize("c", VCASES, ids=lambda c: c.name)
def test_case_reaches_what_it_exists_for(c):
    got = case_names(c)
    assert c.expect <= got, "%s: expected %s; the calls reach %s" % (c.name, sorted(c.expect - got), sorted(got))
    assert case_bytes(c) < 100e6 and oracle_elements(c) < 8e6, (case_bytes(c), oracle_elements(c))
    if c.kind == "int":
        amplitude(c)


def test_cases_cover_every_branch_in_every_dtype():
    """every reachable (kernel, sub-branch) pair in fp32, fp64, bf16 and fp16"""
    missing = []
    for dt in DTYPES:
        got = set()
        for c in VCASES:
            if c.dt == dt:
                got |= case_names(c)
        missing += ["%s %s" % (dt, p) for p in sorted(required(dt) - got)]
        assert not (EXEMPT & got), (dt, EXEMPT & got)
        assert not (UNREACHABLE.get(dt, set()) & got), (dt, UNREACHABLE[dt] & got)
    assert not missing, missing


def test_every_kernel_takes_a_second_grid_stride_pass():
    """each kernel (every profiler record and what runs inside it) runs >= 2 grid-stride passes in some case at 132 and at 114 SMs"""
    looped = {}
    for c in VCASES:
        for launches in predict(c).values():
            for l in launches:
                key = "%s/%s" % (l.prof, l.kernel)
                looped.setdefault(key, set()).update(s for s in SMS_H100 if l.passes(s) >= 2)
    assert set(looped) == LOOP_KERNELS, sorted(set(looped) ^ LOOP_KERNELS)
    short = sorted(k for k, s in looped.items() if s != set(SMS_H100))
    assert not short, short


def test_loop_cases_walk_rep_on_later_passes():
    """the 2-pass cases of the register-resident forwards share each weight channel between input channels (rep > 1)"""
    for c in VCASES:
        if c.name.startswith("loop-"):
            assert c.desc.c // c.desc.wc > 1, c.name
            for l in predict(c)["fwd"]:
                assert all(l.passes(s) >= 2 for s in SMS_H100), (c.name, l)


def test_exemptions_need_2g_elements():
    """the exempt branches are reached only by tensors of >= 2^31 elements; no case allocates one"""
    big = R(1, 1 << 11, 1 << 10, 1 << 10, 1 << 11)                          # 2^31 output elements
    assert refpad_fwd(big)[0].names() >= {"refpad_fwd_generic", "refpad_fwd_generic/large"}
    big_w = R(2, 8, 4096, 4096, 8, k=3, p=1)                                 # weights of 2 x 8 x 9 x 2^24 > 2^31
    assert "refpad_fwd_generic/large" in refpad_fwd(big_w)[0].names()
    assert "refpad_fwd_generic/large" in refpad_fwd(R(1, 1, 4096, 4096, 1, k=3, p=1))[0].names()   # H * W = 2^24
    assert "refpad_fwd_generic/large" not in refpad_fwd(R(1, 1, 4095, 4096, 1, k=3, p=1))[0].names()
    assert "dilate_fwd_kernel/large" in dilate_fwd(DL(1, 1 << 11, 1 << 10, 1 << 10, 1 << 11, dil=(1,) * (1 << 11)))[0].names()
    assert "dilate_fwd_kernel/large" in dilate_fwd(DL(2, 8, 4096, 4096, 8, dil=(1,) * 8))[0].names()
    for c in VCASES:
        d = c.desc
        assert d.n * d.heads * d.c * d.ho * d.wo * 2 < LIM31


def test_grid_and_passes():
    """Launch.grid / passes follow grid_stride_blocks: at most num_sms x per_sm CTAs, the loop covers the rest"""
    l = Launch("x", "k", frozenset(), 540672, 16)
    assert l.grid(132) == 2112 and l.passes(132) == 1 and l.grid(114) == 1824 and l.passes(114) == 2
    assert Launch("x", "k", frozenset(), 540673, 16).passes(132) == 2
    assert Launch("x", "k", frozenset(), 1, 16).grid(132) == 1
    assert tg._missing_anchors("common.cuh", tg.GRID_ANCHORS["common.cuh"]) == []


def test_amplitudes_keep_every_sum_exact():
    for c in VCASES:
        if c.kind == "int":
            a = amplitude(c)
            assert max_terms(c.desc) * a * a <= EXACT_LIMIT[c.dt]
    # the dX count of the pad = H - 1 case: on each axis the middle pixel is its own source (5 taps reach it) and the
    # reflection of two padded positions (3 taps each)
    d = R(2, 3, 5, 5, 1, k=5, p=4)
    assert refpad_dx_terms(d) == 11 * 11


def test_refpad_dx_terms_match_a_brute_force_count():
    """refpad_dx_terms against counting, per input pixel, the (output, tap) pairs of the forward that read it"""
    for d in (R(1, 1, 5, 5, 1, k=5, p=4), R(1, 1, 9, 10, 1, s=2, d=2, p=2), R(1, 1, 6, 9, 1, k=(3, 5), heads=2, p=(1, 2)),
              R(1, 1, 8, 7, 1, k=4, s=2, p=2)):
        cnt = Counter()
        for ho in range(d.ho):
            for wo in range(d.wo):
                for kh in range(d.kh):
                    for kw in range(d.kw):
                        hi = _reflect(-d.ph + ho * d.sh + kh * d.dh, d.h)
                        wi = _reflect(-d.pw + wo * d.sw + kw * d.dw, d.w)
                        cnt[hi, wi] += d.heads
        assert refpad_dx_terms(d) == max(cnt.values()), d


def test_refpad_oracle_takes_rectangular_geometry():
    """oracle.agg_refpad_unfold with (height, width) kernel, padding, stride and dilation == the tap-by-tap loops"""
    import numpy as np
    from oracle import agg_ref
    g = torch.Generator().manual_seed(3)
    for k, s, p, dd, H, W in (((3, 5), 1, (1, 2), 1, 6, 9), ((3, 5), (2, 1), (2, 1), (1, 2), 7, 8), (4, 2, 2, 1, 8, 7)):
        Ho, Wo = agg_ref.out_size(H, W, k, s, p, dd)
        kk = (k, k) if isinstance(k, int) else k
        x = torch.randn(2, 6, H, W, generator=g, dtype=torch.float64)
        w = torch.randn(2, 2, 3, kk[0] * kk[1], Ho, Wo, generator=g, dtype=torch.float64)
        want = agg_ref.agg_refpad_fwd_loops(x.numpy(), w.numpy(), k, s, p, dd)
        got = agg_ref.agg_refpad_unfold(x, w, k, s, p, dd)
        assert np.abs(got.numpy() - want).max() < 1e-12, (k, s, p, dd)


# ------------------------------------------------------------------------------------------------ argument checks (C ABI)
EINVAL, EDTYPE, ELAYOUT, ENULL = -1, -2, -3, -5
P = 256                                          # a non-NULL pointer the library never dereferences (no launch happens)


def _adesc(**kw):
    """a valid 3x3 "same" descriptor with the fields of kw changed.  dtype 7 by default: a check that does not fire ends in the
    dtype switch (EDTYPE), so no case here can launch a kernel on the pointers, which are not device memory"""
    base = dict(n=1, c=4, h=6, w=6, heads=1, wc=2, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1, dh=1, dw=1, ho=6, wo=6, dtype=7, layout=0,
                gc=0, fold=1)
    base.update(kw)
    d = _lib.AggDesc()
    for k, v in base.items():
        setattr(d, k, v)
    return d


def _calls(lib, d, ptrs=(P, P, P, P, P)):
    """rc of the forward and the backward of each variant for descriptor d (None: NULL desc)"""
    x, w, y, dil, dxw = ptrs
    dp = None if d is None else ctypes.byref(d)
    return {
        "refpad_fwd": lib.cotb200_agg_refpad_fwd(dp, x, w, y, None),
        "refpad_bwd": lib.cotb200_agg_refpad_bwd(dp, y, x, w, dxw, dxw, None),
        "dilate_fwd": lib.cotb200_agg_zeropad_dilate_fwd(dp, x, w, dil, y, None),
        "dilate_bwd": lib.cotb200_agg_zeropad_dilate_bwd(dp, y, x, w, dil, dxw, dxw, None),
        "merge_fwd": lib.cotb200_agg_zeropad_mix_merge_fwd(dp, 5, 5, 2, 2, x, w, y, None),
        "merge_bwd": lib.cotb200_agg_zeropad_mix_merge_bwd(dp, 5, 5, 2, 2, y, x, w, dxw, dxw, None),
    }


def _expect(lib, d, want, only=None, ptrs=(P, P, P, P, P)):
    n0 = lib.cotb200_launch_count()
    got = _calls(lib, d, ptrs)
    assert lib.cotb200_launch_count() == n0, "an argument check launched a kernel"
    for k, rc in got.items():
        if only is None or k in only:
            assert rc == want, "%s: rc %d, want %d (%s)" % (k, rc, want, lib.cotb200_last_error().decode())


def test_variant_argument_checks():
    lib = _lib.load()
    # dtype 7: every geometry check passes, the dtype switch refuses
    _expect(lib, _adesc(), EDTYPE)
    _expect(lib, _adesc(dtype=4), EDTYPE)
    # non-positive dimensions
    for f in ("n", "c", "h", "w", "heads", "wc", "kh", "kw", "ho", "wo"):
        _expect(lib, _adesc(**{f: 0}), EINVAL)
        _expect(lib, _adesc(**{f: -1}), EINVAL)
    # c % wc
    _expect(lib, _adesc(c=5, wc=2), EINVAL)
    # dilate: 3x3 only (the weight channels of dilate are 3x3 whatever the other fields say), output size = input size
    _expect(lib, _adesc(kh=5, kw=5, ph=2, pw=2), EINVAL, only=("dilate_fwd", "dilate_bwd"))
    _expect(lib, _adesc(kw=5, pw=2), EINVAL, only=("dilate_fwd", "dilate_bwd"))
    _expect(lib, _adesc(ho=4, wo=9), EINVAL, only=("dilate_fwd", "dilate_bwd"))
    _expect(lib, _adesc(ho=6, wo=5), EINVAL, only=("dilate_fwd", "dilate_bwd"))
    # dilate ignores stride, padding and dilation fields (the reference's kernel is stride 1, pad = dilation)
    _expect(lib, _adesc(sh=0, ph=-3, dh=0), EDTYPE, only=("dilate_fwd", "dilate_bwd"))
    # refpad / mix_merge: bad stride, dilation, padding
    for kw in (dict(sh=0), dict(sw=-1), dict(dh=0), dict(dw=0), dict(ph=-1), dict(pw=-1)):
        _expect(lib, _adesc(**kw), EINVAL, only=("refpad_fwd", "refpad_bwd", "merge_fwd", "merge_bwd"))
    # reflect padding >= H or >= W (one reflection, like nn.ReflectionPad2d); zero padding of mix_merge has no such limit
    _expect(lib, _adesc(h=3, ph=3, ho=7), EINVAL, only=("refpad_fwd", "refpad_bwd"))
    _expect(lib, _adesc(w=2, pw=2, wo=4), EINVAL, only=("refpad_fwd", "refpad_bwd"))
    _expect(lib, _adesc(h=4, w=4, ph=3, pw=3, ho=8, wo=8), EDTYPE, only=("refpad_fwd", "refpad_bwd"))
    # the weight plane must hold the output: (H + 2p - span) / s + 1 per axis
    _expect(lib, _adesc(ho=5, wo=6), EINVAL, only=("refpad_fwd", "refpad_bwd", "merge_fwd", "merge_bwd"))
    _expect(lib, _adesc(ho=4, wo=9), EDTYPE, only=("refpad_fwd", "refpad_bwd"))     # same plane, other factors
    # a window larger than the padded input on both axes: sizes (3 - 7) / 1 + 1 = -3 and (5 - 7) / 1 + 1 = -1, whose product
    # equals a 1 x 3 weight plane; and a stride that rounds an overhanging window up to one output position
    _expect(lib, _adesc(h=3, w=5, kh=7, kw=7, ph=0, pw=0, ho=1, wo=3), EINVAL,
            only=("refpad_fwd", "refpad_bwd", "merge_fwd", "merge_bwd"))
    _expect(lib, _adesc(h=2, w=2, kh=5, kw=5, ph=1, pw=1, sh=2, sw=2, ho=1, wo=1), EINVAL,
            only=("refpad_fwd", "refpad_bwd", "merge_fwd", "merge_bwd"))
    # mix_merge: the second kernel must give the same output size
    assert lib.cotb200_agg_zeropad_mix_merge_fwd(ctypes.byref(_adesc()), 5, 5, 1, 1, P, P, P, None) == EINVAL
    assert lib.cotb200_agg_zeropad_mix_merge_fwd(ctypes.byref(_adesc()), 5, 5, 2, 2, P, P, P, None) == EDTYPE
    # NHWC layouts
    _expect(lib, _adesc(layout=1), ELAYOUT)
    _expect(lib, _adesc(layout=2, gc=1), ELAYOUT)
    # NULL descriptor and NULL tensors
    _expect(lib, None, ENULL)
    for i in range(3):                           # x, w, then y (the forwards) / dy (the backwards)
        ptrs = [P] * 5
        ptrs[i] = None
        _expect(lib, _adesc(), ENULL, ptrs=tuple(ptrs))
    _expect(lib, _adesc(), ENULL, only=("dilate_fwd", "dilate_bwd"), ptrs=(P, P, P, None, P))
    assert lib.cotb200_agg_refpad_bwd(ctypes.byref(_adesc()), None, P, P, P, P, None) == ENULL
    assert lib.cotb200_agg_refpad_bwd(ctypes.byref(_adesc()), P, P, None, P, None, None) == ENULL     # dX without w
    assert lib.cotb200_agg_refpad_bwd(ctypes.byref(_adesc()), P, None, P, None, P, None) == ENULL     # dW without x
    assert lib.cotb200_agg_refpad_bwd(ctypes.byref(_adesc()), P, None, P, P, None, None) == EDTYPE    # dX alone needs no x
    assert lib.cotb200_agg_zeropad_mix_merge_bwd(ctypes.byref(_adesc()), 5, 5, 2, 2, P, P, None, P, None, None) == ENULL
    assert lib.cotb200_agg_zeropad_mix_merge_bwd(ctypes.byref(_adesc()), 5, 5, 2, 2, P, None, P, None, P, None) == ENULL
    assert lib.cotb200_agg_zeropad_dilate_bwd(ctypes.byref(_adesc()), P, None, P, P, P, None, None) == EDTYPE
    assert lib.cotb200_last_error()
