"""The persistent TMA / wgmma kernels past their first ring wrap, against fp64 references of the whole output.

Every persistent kernel of the hot path loops `for (tile = blockIdx.x; tile < total; tile += gridDim.x)` and feeds its tiles
through an mbarrier ring whose stage index and phase bit keep running from one tile to the next.  At the bench's batch size every
CTA handles tens of tiles; the small shapes of the other tests give each CTA one tile.  Each case below

  * computes its launch plan from Python copies of the host-side planning (checked against the CUDA sources and for both H100
    SM counts by test_persistent_geometry_cpu.py), picks the smallest size that reaches the regime and asserts it:
      - the busiest CTA walks at least 2 * stages + 1 tiles, so every ring stage is reused at both phase parities;
      - total % grid != 0 (a ragged last round);
      - plus the feature the case is about (a partial last tile arriving mid-CTA, an N-tile change inside a CTA, ...);
  * draws its operands as small integers wherever the output stays exactly representable (bounds in the comments), so the whole
    output is compared with torch.equal against an fp64 reference: a stale stage, a row written by the wrong tile or a dropped
    k-block fails outright instead of hiding in a tolerance;
  * checks, with the library's profiler, that the intended kernel ran (a silent fallback would test something else).

Statistics outputs (fp32 sums over many tiles) use the determinism suite's tolerance rule; one float-random case per kernel checks
the numerics (scale / shift rounding, fp32 paths) with tolerances."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from cotnet_b200 import _lib
from test_determinism_gpu import TC_BK, TC_BM, TOL, _cdiv, _sms, pick_bn, pick_bn_wide, tc_grid

pytestmark = pytest.mark.gpu

SMS_H100 = (132, 114)           # SXM, PCIe: the geometry test plans every case for both
MEM_LIMIT = 8e9                 # rough peak device bytes of one case (inputs, outputs, chunked references)


# ================================================================================================ launch plans (Python copies)
class Plan:
    """One persistent launch: `grid` CTAs walk `total` tiles round-robin through a ring of `stages` slots; a tile takes `per_tile`
    ring slots (k-blocks of the GEMM kernel, 1 elsewhere)."""

    def __init__(self, name, grid, total, stages, per_tile=1, **info):
        self.name, self.grid, self.total, self.stages, self.per_tile, self.info = name, grid, total, stages, per_tile, info

    @property
    def max_tiles(self):
        return _cdiv(self.total, self.grid)

    @property
    def wraps(self):
        """times the busiest CTA's ring index returns to stage 0"""
        return (self.max_tiles * self.per_tile - 1) // self.stages

    def problems(self):
        p = []
        if self.max_tiles < 2 * self.stages + 1:
            p.append("tiles/CTA %d < 2*stages+1 = %d" % (self.max_tiles, 2 * self.stages + 1))
        if self.total % self.grid == 0:
            p.append("total %% grid == 0")
        return p

    def __str__(self):
        extra = "".join(" %s=%s" % kv for kv in sorted(self.info.items()))
        return "%s: grid=%d total=%d tiles/CTA<=%d stages=%d ring wraps=%d%s" % (
            self.name, self.grid, self.total, self.max_tiles, self.stages, self.wraps, extra)


def _mid_cta(tiles, plan):
    """some tile of `tiles` is not the first tile of its CTA"""
    return any(t // plan.grid >= 1 for t in tiles)


def _rup(a, b):
    return _cdiv(a, b) * b


# cotnet_b200/csrc/tc_gemm.cu: TC_STAGES, tc_launch (per_sm, stages, grid)
TC_STAGES = 6


def tc_launch(name, N, bn, m_tiles, nkb, colstats, sms):
    out_bytes = 2 * TC_BM * 128 + ((2 * 4 * 256 * 4 + 2 * N * 4) if colstats else 0)
    stage_bytes = TC_BM * TC_BK * 2 + _rup(bn * TC_BK * 2, 1024)
    per_sm = 2
    stages = (104 * 1024 - out_bytes) // stage_bytes
    if stages < 2 or bn > 128:
        per_sm = 1
        stages = (200 * 1024 - out_bytes) // stage_bytes
    stages = max(2, min(stages, TC_STAGES))
    n_tiles = _cdiv(N, bn)
    total = m_tiles * n_tiles
    grid = min(per_sm * sms, total)
    if colstats:
        assert grid == tc_grid(N, bn, m_tiles, True, sms)
    return Plan(name, grid, total, stages, nkb, inst="<2,2>" if per_sm == 2 else "<4,1>", bn=bn, n_tiles=n_tiles)


# conv3x3_halo_launch (R, items, stages, grid = (sms / n_tiles) * n_tiles); the plan is that of one N tile: step = grid / n_tiles
# CTAs walk its `items` work items
HC_WBYTES = 9 * 64 * 128


def conv3x3_halo_launch(B, H, W, C, sms):
    Wpad = W + 2
    R = 0
    for r in range(1, H + 1):
        if H % r == 0 and r * Wpad <= 256 and r * W <= 256:
            R = r
    n_tiles = C // 64
    if R == 0 or n_tiles > sms:
        return None
    MB = _cdiv(R * Wpad, 128)
    a_stage = _rup(max((R + 2) * Wpad, MB * 128 + 2 * Wpad + 2) * 128, 1024)
    out_bytes = _rup(R * W * 128, 1024)
    stages = min((220 * 1024 - HC_WBYTES - out_bytes) // a_stage, 4)
    if stages < 2:
        return None
    items = B * (H // R)
    grid = min((sms // n_tiles) * n_tiles, items * n_tiles)
    return Plan("tc_conv3x3_halo", grid // n_tiles, items, stages, R=R, n_tiles=n_tiles)


def conv3x3_tc_launch(B, H, W, C, bn, colstats, sms):
    """conv mode of tc_gemm_kernel (cotb200_conv3x3_bf16 when the haloed-tile kernel does not take the call)"""
    if H * W <= TC_BM // 2:
        bbox, hbox = TC_BM // (H * W), H
        m_tiles = _cdiv(B, bbox)
    else:
        bbox, hbox = 1, max(1, min(TC_BM // W, H))
        while H % hbox:
            hbox -= 1
        m_tiles = B * (H // hbox)
    p = tc_launch("tc_conv3x3", C, bn, m_tiles, 9 * (bn // 64), colstats, sms)
    p.info.update(bbox=bbox, hbox=hbox)
    return p


def stem_launch(B, H, W, N, colstats, sms):
    Wh = W // 2
    wtiles = _cdiv(Wh, TC_BM)
    while Wh % wtiles:
        wtiles += 1
    return tc_launch("tc_stem7x7", N, pick_bn_wide(N), B * (H // 2) * wtiles, 4, colstats, sms)


# cotnet_b200/csrc/tc_wgrad.cu: cotb200_stem7x7s2_wgrad_bf16 (splits = CTAs, one output row per ring stage)
WG_STAGES = 4


def stem_wgrad_launch(B, H, W, sms):
    kb_total = B * (H // 2)
    per = _cdiv(kb_total, min(sms, kb_total))
    stages = min((216 * 1024) // (6 * 128 * (W // 2)), WG_STAGES)
    return Plan("tc_stem_wgrad", _cdiv(kb_total, per), kb_total, stages)


# cotnet_b200/csrc/agg_tma.cu: AT_MAX_STAGES, at_setup (TH, bands, stages, grid); mode 0 fwd, 1 dX, 2 dW
AT_MAX_STAGES = 4
AT_NAMES = {0: "agg3_fwd_tma", 1: "agg3_dx_tma", 2: "agg3_dw_tma"}


def at_setup(mode, es, N, C, H, W, wc):
    vec = 16 // es
    slabs = C * es // 128
    J = 9 * wc
    whalo = 1 if mode == 1 else 0
    CQ = C // vec
    TH = 0
    for th in range(1, min(H, 254) + 1):
        xb = slabs * _rup((th + 2) * (W + 2) * 128, 1024)
        if mode == 2:
            bb = slabs * _rup(th * W * 128, 1024)
        else:
            bb = _rup((th + 2 * whalo) * (W + 2 * whalo) * J * es, 1024)
        if xb + bb > 72 * 1024:
            break
        if mode != 2 and th * W * CQ > 2 * 896:
            break
        TH = th
        if th * W * CQ >= 896:
            break
    if not TH:
        return None                      # the second-generation kernels take the call
    slab_bytes = _rup((TH + 2) * (W + 2) * 128, 1024)
    if mode == 2:
        w_stage = slabs * _rup(TH * W * 128, 1024)
    else:
        w_stage = _rup((TH + 2 * whalo) * (W + 2 * whalo) * J * es, 1024)
    stages = min((200 * 1024) // (slabs * slab_bytes + w_stage), AT_MAX_STAGES)
    if stages < 2:
        return None
    bands = _cdiv(H, TH)
    return TH, bands, stages


def at_plan(mode, es, N, C, H, W, wc, sms):
    """the plan of the TMA kernel, or None when at_setup declines the geometry"""
    if at_setup(mode, es, N, C, H, W, wc) is None:
        return None
    TH, bands, stages = at_setup(mode, es, N, C, H, W, wc)
    total = N * bands
    return Plan(AT_NAMES[mode], min(sms, total), total, stages, TH=TH, bands=bands)


# cotnet_b200/csrc/agg_nchw_tma.cu: nchw_tma_launch (tile = (sample, weight channel, band))
NT_MAX_STAGES = 4
NT_COMPUTE_THREADS = 384
NT_NAMES = {0: "agg3_fwd_nchw_tma", 1: "agg3_dx_nchw_tma", 2: "agg3_dw_nchw_tma"}


def nchw_tma_launch(mode, es, N, C, H, W, wc, sms):
    rep, al = C // wc, 16 // es
    pxv = 4 if W % 4 == 0 else (2 if W % 2 == 0 and es == 4 else 0)
    assert pxv and 1 <= rep <= 16 and H * W > 256
    halo = max(pxv, al)
    BWa, BWb = _rup(W + 2 * halo, al), _rup(W, al)
    nsplit = 1 if mode == 2 else (2 if rep % 2 == 0 else 1)
    nq = W // pxv
    budget = 200 * 1024
    TH = stages = 0
    for th in range(1, min(H, 32) + 1):
        a = _rup(rep * (th + 2) * BWa * es, 128)
        b = _rup(9 * th * BWb * es if mode == 0 else 9 * (th + 2) * BWa * es if mode == 1 else rep * th * BWb * es, 128)
        if (a + b) * 2 > budget:
            break
        TH, stages = th, budget // (a + b)
        if th * nq * nsplit >= NT_COMPUTE_THREADS:
            break
    assert TH
    stages = min(stages, NT_MAX_STAGES)
    bands = _cdiv(H, TH)
    total = N * wc * bands
    return Plan(NT_NAMES[mode], min(sms, total), total, stages, TH=TH, bands=bands)


# cotnet_b200/csrc/gn72.cu: gn72_stats_launch (X walkers per sample over ntiles tiles, two-stage bulk-copy ring)
def gn72_stats_launch(B, HW, wc, es, sms):
    tb = 256 if es == 2 else 128
    ntiles = _cdiv(HW * (wc // 8), tb)
    X = max(1, min(_cdiv(4 * sms, B), ntiles))
    return Plan("gn72_stats", X, ntiles, 2, per_sample_ctas=X)


def _search(make, first=1, limit=100000):
    """smallest size n >= first for which make(n) returns (plans, ok, sizes) with every plan in its regime and ok true"""
    for n in range(first, limit):
        plans, ok, sizes = make(n)
        if ok and not any(p.problems() for p in plans):
            return plans, sizes
    raise AssertionError("no size up to %d reaches the regime" % limit)


def _describe(plans):
    return "; ".join(str(p) for p in plans)


def _assert_regime(plans, **features):
    for p in plans:
        assert not p.problems(), "%s: %s" % (p, ", ".join(p.problems()))
    for what, ok in features.items():
        assert ok, "%s not reached: %s" % (what, _describe(plans))


# ================================================================================================ cases and their sizes
# GEMM: (N, K1, K2, epilogue); epilogue "none", "affine" (power-of-two scale, integer shift, ReLU), "stats" (+ column statistics),
# "float" (random bf16 operands, random fp32 scale / shift).  Integer operands in {-1, 0, 1}, K1 + K2 <= 256: |D| <= 256 (the
# scale is at most 1, the shift at most 4 and the ReLU only clips).
GEMM_CASES = [
    (64, 64, 0, "none"),                 # <2,2>, 3 stages
    (640, 128, 0, "affine"),             # <2,2>, N tiles of 128: 5 N tiles on a grid they do not divide -> n0 changes in a CTA
    (640, 128, 0, "stats"),              # one CTA per SM (statistics smem), N-tile changes, s_tot over many tiles
    (256, 128, 128, "stats"),            # <4,1> (bn = 256), two operand pairs
    (320, 128, 64, "affine"),            # <4,1> with bn = 192: the second N tile is partly outside N (zero-filled B, clipped store)
    (640, 128, 0, "float"),
]
N_TILE_CHANGE = 640                      # the cases with this N must see n0 change inside a CTA


def gemm_sizes(case, sms):
    N, K1, K2, epi = case
    bn = pick_bn(N, K1 + K2)
    n_tiles = _cdiv(N, bn)
    nkb = _cdiv(K1, TC_BK) + _cdiv(K2, TC_BK)
    colstats = epi == "stats"

    def make(mt):
        M = mt * TC_BM - 40                                          # partial last row tile
        p = tc_launch("tc_gemm_1x1", N, bn, mt, nkb, colstats, sms)
        partial = range((mt - 1) * n_tiles, mt * n_tiles)
        ok = _mid_cta(partial, p) and (N != N_TILE_CHANGE or p.grid % n_tiles != 0)
        mem = M * (K1 + K2 + N) * 2 + N * (K1 + K2) * 2 + 3 * 65536 * N * 8
        return [p], ok, dict(M=M, bn=bn, n_tiles=n_tiles, mem=mem)

    return _search(make)


# 3x3 convolutions: (C, groups, bn, H, W, transposed weight (data gradient), statistics, operands).  cg = C / groups = 16 with
# {-1, 0, 1} operands: |D| <= 9 * 16 = 144.  bn = 64 is the haloed-tile kernel, bn in {128, 192, 256} conv mode of the GEMM kernel
# (the weight is packed for that N tile: zero outside each output channel's group).
CONV_CASES = [
    (64, 4, 64, 56, 56, False, True, "int"),
    (128, 8, 64, 28, 28, True, False, "int"),                # two N tiles of the haloed kernel, data gradient
    (128, 8, 128, 28, 28, False, True, "int"),
    (192, 12, 192, 14, 14, True, True, "int"),
    (256, 16, 256, 7, 7, False, True, "int"),                # two samples per tile, B odd: a partial last tile
    (64, 4, 64, 56, 56, False, True, "float"),
    (128, 8, 128, 28, 28, False, True, "float"),
]


def conv_sizes(case, sms):
    C, groups, bn, H, W, _, stats, _ = case

    def make(B):
        if bn == 64:
            p = conv3x3_halo_launch(B, H, W, C, sms)
            ok = p is not None
            plans = [p] if ok else []
        else:
            p = conv3x3_tc_launch(B, H, W, C, bn, stats, sms)
            plans = [p]
            ok = p.info["bbox"] == 1 or (B % p.info["bbox"] != 0 and _mid_cta([p.total - 1], p))
        return plans, ok, dict(B=B, mem=B * H * W * C * (2 * 2 + 3 * 8))

    return _search(make)


# stem: 7x7 / s2 / p3 of a 224x224 image, N = 64; {-1, 0, 1} operands: |D| <= 147; the weight gradient sums at most
# B * 112 * 112 products of {-1, 0, 1}: integers below 2^24
STEM_CASES = [(224, 224, 64, "int"), (224, 224, 64, "float")]


def stem_sizes(case, sms):
    H, W, N, _ = case

    def make(B):
        plans = [stem_launch(B, H, W, N, True, sms), stem_wgrad_launch(B, H, W, sms)]
        return plans, True, dict(B=B, mem=B * H * W * 3 * 8 * 3 + B * (H // 2) * (W // 2) * N * (2 * 2 + 8 * 2))

    return _search(make)


# TMA LocalConv, NHWC_TAP: (dtype size, C, wc, H, W, fold, gc, operands).  x, w, dY in {-2..2}: |y|, |dX| <= 9 * 4 = 36 and
# |dW| <= (C / fold) / (wc / fold) * 4 = 32 (8 sharers): exact in every storage type.
AGG_CASES = [
    ("bf16", 64, 8, 56, 56, 1, 8, "int"),     # the stage-1 shape of the block
    ("fp16", 64, 8, 57, 57, 1, 8, "int"),     # H % TH != 0: partial last band
    ("fp32", 64, 8, 56, 56, 1, 8, "int"),     # TH = 1, three stages; the haloed fp32 weight band of dX does not fit a stage
    ("bf16", 128, 16, 28, 28, 2, 8, "int"),   # CoXt fold = 2
    ("bf16", 64, 8, 56, 56, 1, 8, "float"),
]
DTYPES = {"bf16": (torch.bfloat16, 2), "fp16": (torch.float16, 2), "fp32": (torch.float32, 4)}


def agg_sizes(case, sms):
    dt, C, wc, H, W, _, _, _ = case
    es = DTYPES[dt][1]

    def make(N):
        plans = [p for p in (at_plan(m, es, N, C, H, W, wc, sms) for m in (0, 1, 2)) if p is not None]
        ok = plans[0].name == "agg3_fwd_tma" and plans[-1].name == "agg3_dw_tma"

        if H % 2:                                                # odd H: a partial last band, which must arrive mid-CTA
            for p in plans:
                th, bands = p.info["TH"], p.info["bands"]
                ok = ok and H % th != 0 and _mid_cta([n * bands + bands - 1 for n in range(N)], p)
        return plans, ok, dict(N=N, mem=N * H * W * (2 * C + 9 * wc) * (es * 3 + 8 * 4))

    return _search(make)


# NCHW TMA LocalConv: (dtype size, C, wc, H, W); {-2..2} operands, 8 sharers per weight channel: exact
NCHW_CASES = [("fp32", 64, 8, 56, 56), ("bf16", 64, 8, 56, 56)]


def nchw_sizes(case, sms):
    dt, C, wc, H, W = case
    es = DTYPES[dt][1]

    def make(N):
        return [nchw_tma_launch(m, es, N, C, H, W, wc, sms) for m in (0, 1, 2)], True, dict(N=N, mem=N * H * W * (2 * C + 9 * wc) * (es * 3 + 8 * 4))

    return _search(make)


# GroupNorm over 9 taps, blocks of 72: (dtype size, wc, H); stats walk their tiles with a two-stage ring (prefetch of tile + X)
GN_CASES = [("bf16", 16, 56), ("fp32", 16, 56)]


def gn_sizes(case, sms):
    dt, wc, H = case
    es = DTYPES[dt][1]

    def make(B):
        return [gn72_stats_launch(B, H * H, wc, es, sms)], True, dict(B=B, mem=B * H * H * 9 * wc * (es * 4 + 8 * 6))

    return _search(make)


ALL_CASES = ([(gemm_sizes, c) for c in GEMM_CASES] + [(conv_sizes, c) for c in CONV_CASES] + [(stem_sizes, c) for c in STEM_CASES]
             + [(agg_sizes, c) for c in AGG_CASES] + [(nchw_sizes, c) for c in NCHW_CASES] + [(gn_sizes, c) for c in GN_CASES])


# ================================================================================================ helpers
@contextlib.contextmanager
def kernels_ran(*names):
    """the library's profiler around the calls (eager only, never under capture): every name must have been launched"""
    torch.cuda.synchronize()
    _lib.prof_enable(True)
    try:
        yield
        rep = _lib.prof_report()
    finally:
        _lib.prof_enable(False)
    for n in names:
        assert n in rep, "kernel %s did not run (launched: %s)" % (n, sorted(rep))


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ints(shape, lo, hi, g, dtype):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").to(dtype)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _equal_exact(got, ref, what):
    """got (any float dtype) == ref (fp64) element for element"""
    g = got.double()
    bad = g != ref
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %r want %r" % (
            what, int(bad.sum()), bad.numel(), idx, float(g[tuple(idx)]), float(ref[tuple(idx)])))


def _close(got, ref, absterms, what, rel):
    """|got - ref| <= rel * |ref| + TOL * sum|terms|: the storage rounding of the output plus fp32 accumulation"""
    err = (got.double() - ref).abs()
    lim = rel * ref.abs() + TOL * absterms
    bad = ~(err <= lim)
    assert not bool(bad.any()), "%s: %d of %d elements off; worst err/limit %.3g" % (
        what, int(bad.sum()), bad.numel(), float((err / lim.clamp_min(1e-30)).max()))


def _sums_close(got, ref, absterms, what):
    """fp32 sums over many tiles: the determinism suite's rule |got - ref| <= TOL * sum|terms|"""
    _close(got, ref, absterms, what, 0.0)


def _chunks(n, step):
    return [(i, min(n, i + step)) for i in range(0, n, step)]


# ================================================================================================ GEMM
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: "N%d-K%d+%d-%s" % c)
def test_gemm_bf16(case):
    N, K1, K2, epi = case
    (plan,), sz = gemm_sizes(case, _sms())
    M = sz["M"]
    _assert_regime([plan], partial_tile_mid_cta=M % TC_BM != 0 and _mid_cta([plan.total - 1], plan),
                   n_tile_change=N != N_TILE_CHANGE or plan.grid % sz["n_tiles"] != 0)
    print("gemm %s M=%d: %s" % (case, M, plan))
    g = _gen(M + N + K1 + K2)
    flt = epi == "float"
    if flt:
        mk = lambda s: torch.randn(s, generator=g, device="cuda").bfloat16()
        a1, b1 = mk((M, K1)), (torch.randn(N, K1, generator=g, device="cuda") / K1 ** 0.5).bfloat16()
    else:
        a1, b1 = _ints((M, K1), -1, 1, g, torch.bfloat16), _ints((N, K1), -1, 1, g, torch.bfloat16)
    a2 = _ints((M, K2), -1, 1, g, torch.bfloat16) if K2 else None
    b2 = _ints((N, K2), -1, 1, g, torch.bfloat16) if K2 else None
    scale = shift = None
    relu = 0
    if epi in ("affine", "stats"):
        scale = 2.0 ** -torch.randint(0, 3, (N,), generator=g, device="cuda").float()      # 1, 1/2, 1/4
        shift = torch.randint(-4, 5, (N,), generator=g, device="cuda").float()
        relu = 1 if epi == "affine" else 0
    elif flt:
        scale = 0.5 + torch.rand(N, generator=g, device="cuda")
        shift = torch.randn(N, generator=g, device="cuda")
        relu = 1
    D = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
    cs = torch.zeros(N, device="cuda") if epi == "stats" else None
    cq = torch.zeros(N, device="cuda") if epi == "stats" else None
    lib = _lib.load()
    with kernels_ran("tc_gemm_1x1"):
        _lib.check(lib.cotb200_gemm_bf16(M, N, K1, a1.data_ptr(), K1, b1.data_ptr(), K1, K2, _lib.ptr(a2), K2, _lib.ptr(b2), K2,
                                         D.data_ptr(), N, _lib.ptr(scale), _lib.ptr(shift), relu, _lib.ptr(cs), _lib.ptr(cq), _st()),
                   "gemm_bf16")
    torch.cuda.synchronize()
    what = "gemm %s (%s)" % (case, plan)
    s_ref = torch.zeros(N, dtype=torch.float64, device="cuda")
    q_ref = torch.zeros_like(s_ref)
    for i0, i1 in _chunks(M, 1 << 16):
        acc = a1[i0:i1].double() @ b1.double().t()
        if K2:
            acc += a2[i0:i1].double() @ b2.double().t()
        ref = acc * scale.double() + shift.double() if scale is not None else acc
        if relu:
            ref = ref.clamp_min(0.0)
        if flt:
            absterms = (a1[i0:i1].double().abs() @ b1.double().abs().t()) * scale.double() + shift.double().abs()
            _close(D[i0:i1], ref, absterms, what + " rows %d.." % i0, 2.0 ** -8)
        else:
            _equal_exact(D[i0:i1], ref, what + " rows %d.." % i0)
        d = D[i0:i1].double()
        s_ref += d.sum(0)
        q_ref += (d * d).sum(0)
    if cs is not None:
        d_abs = torch.zeros_like(s_ref)
        for i0, i1 in _chunks(M, 1 << 16):
            d_abs += D[i0:i1].double().abs().sum(0)
        _sums_close(cs, s_ref, d_abs, what + " col_sum")
        _sums_close(cq, q_ref, q_ref, what + " col_sqsum")


# ================================================================================================ 3x3 convolutions
def pack_conv3x3(w, groups, bn, transpose=False):
    """[C, C/groups, 3, 3] -> Wp [C, 9 * bn] bf16 for an N tile of bn columns: Wp[n, tap * bn + j] = weight of output channel n for
    input channel (n0(n) + j) at tap, zero where that channel is outside n's group (include/cotb200.h).  transpose: the weight of
    the data-gradient convolution (taps flipped, in / out swapped per group)."""
    C, cg = w.shape[0], w.shape[1]
    w = w.double().view(groups, cg, cg, 3, 3)
    if transpose:
        w = w.permute(0, 2, 1, 3, 4).flip(3, 4)
    w = w.reshape(C, cg, 9)
    n = torch.arange(C, device=w.device)
    idx = ((n // cg) * cg - (n // bn) * bn)[:, None] + torch.arange(cg, device=w.device)[None, :]
    Wp = torch.zeros(C, 9, bn, dtype=torch.float64, device=w.device)
    Wp.scatter_(2, idx[:, None, :].expand(C, 9, cg), w.permute(0, 2, 1))
    return Wp.reshape(C, 9 * bn).bfloat16().contiguous()


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "C%d-g%d-bn%d-%dx%d-%s-%s-%s" % (
    c[0], c[1], c[2], c[3], c[4], "dgrad" if c[5] else "fwd", "stats" if c[6] else "nostats", c[7]))
def test_conv3x3_bf16(case):
    C, groups, bn, H, W, transpose, stats, kind = case
    (plan,), sz = conv_sizes(case, _sms())
    B = sz["B"]
    _assert_regime([plan])
    print("conv3x3 %s B=%d: %s" % (case, B, plan))
    cg = C // groups
    g = _gen(C + groups + bn + H + transpose)
    flt = kind == "float"
    if flt:
        x = torch.randn(B, H, W, C, generator=g, device="cuda").bfloat16()
        w = (torch.randn(C, cg, 3, 3, generator=g, device="cuda") / (3 * cg ** 0.5)).bfloat16()
        scale, shift = 0.5 + torch.rand(C, generator=g, device="cuda"), torch.randn(C, generator=g, device="cuda")
    else:
        x, w = _ints((B, H, W, C), -1, 1, g, torch.bfloat16), _ints((C, cg, 3, 3), -1, 1, g, torch.bfloat16)
        scale = 2.0 ** -torch.randint(0, 3, (C,), generator=g, device="cuda").float()
        shift = torch.randint(-4, 5, (C,), generator=g, device="cuda").float()
    relu = 1 if not stats else 0
    wp = pack_conv3x3(w, groups, bn, transpose)
    D = torch.full((B, H, W, C), float("nan"), dtype=torch.bfloat16, device="cuda")
    cs = torch.zeros(C, device="cuda") if stats else None
    cq = torch.zeros(C, device="cuda") if stats else None
    lib = _lib.load()
    with kernels_ran(plan.name):
        _lib.check(lib.cotb200_conv3x3_bf16(B, H, W, C, x.data_ptr(), C, wp.data_ptr(), bn, D.data_ptr(), C, scale.data_ptr(),
                                            shift.data_ptr(), relu, _lib.ptr(cs), _lib.ptr(cq), _st()), "conv3x3_bf16")
    torch.cuda.synchronize()
    what = "conv3x3 %s (%s)" % (case, plan)
    s_ref = torch.zeros(C, dtype=torch.float64, device="cuda")
    q_ref, d_abs = torch.zeros_like(s_ref), torch.zeros_like(s_ref)

    def conv(xx, ww):
        if transpose:        # data gradient: the adjoint of the forward convolution with w
            return F.conv_transpose2d(xx, ww, padding=1, groups=groups)
        return F.conv2d(xx, ww, padding=1, groups=groups)

    for b0, b1 in _chunks(B, max(1, (1 << 21) // (H * W * C) * 8)):
        xc = x[b0:b1].permute(0, 3, 1, 2).double()
        acc = conv(xc, w.double()).permute(0, 2, 3, 1)
        ref = acc * scale.double() + shift.double()
        if relu:
            ref = ref.clamp_min(0.0)
        if flt:
            absterms = conv(xc.abs(), w.double().abs()).permute(0, 2, 3, 1) * scale.double() + shift.double().abs()
            _close(D[b0:b1], ref, absterms, what + " samples %d.." % b0, 2.0 ** -8)
        else:
            _equal_exact(D[b0:b1], ref, what + " samples %d.." % b0)
        d = D[b0:b1].double().reshape(-1, C)
        s_ref += d.sum(0)
        q_ref += (d * d).sum(0)
        d_abs += d.abs().sum(0)
    if stats:
        _sums_close(cs, s_ref, d_abs, what + " col_sum")
        _sums_close(cq, q_ref, q_ref, what + " col_sqsum")


# ================================================================================================ stem
def _stem_windows(scratch, B, Hh, Wh):
    """[B*Hh*Wh, 256] windows of the space-to-depth image [B, Hh, Wh + 4, 16] (K order of the packed stem weight)"""
    P = scratch.view(torch.bfloat16).view(B, Hh, Wh + 4, 16).double()
    Pp = F.pad(P, (0, 0, 0, 0, 2, 1))
    return torch.stack([torch.stack([Pp[:, a:a + Hh, c:c + Wh, :] for c in range(4)], 3).reshape(B, Hh, Wh, 64)
                        for a in range(4)], 3).reshape(B * Hh * Wh, 256)


@pytest.mark.parametrize("case", STEM_CASES, ids=lambda c: "%dx%d-N%d-%s" % c)
def test_stem7x7s2_and_wgrad(case):
    from cotnet_b200 import tc
    H, W, N, kind = case
    plans, sz = stem_sizes(case, _sms())
    B = sz["B"]
    _assert_regime(plans)
    print("stem %s B=%d: %s" % (case, B, _describe(plans)))
    Hh, Wh = H // 2, W // 2
    g = _gen(H + N + len(kind))
    flt = kind == "float"
    if flt:
        x = torch.randn(B, H, W, 3, generator=g, device="cuda").bfloat16()
        w = (torch.randn(N, 3, 7, 7, generator=g, device="cuda") / 12).bfloat16()
        dy = torch.randn(B * Hh * Wh, N, generator=g, device="cuda").bfloat16()
    else:
        x, w = _ints((B, H, W, 3), -1, 1, g, torch.bfloat16), _ints((N, 3, 7, 7), -1, 1, g, torch.bfloat16)
        dy = _ints((B * Hh * Wh, N), -1, 1, g, torch.bfloat16)
    wm = tc.prepare_stem_weight(w)
    lib = _lib.load()
    scratch = torch.empty(int(lib.cotb200_stem7x7s2_scratch_bytes(B, H, W)), dtype=torch.uint8, device="cuda")
    D = torch.full((B, Hh, Wh, N), float("nan"), dtype=torch.bfloat16, device="cuda")
    cs, cq = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    dwm = torch.zeros(N, 256, device="cuda")
    with kernels_ran("tc_stem7x7", "tc_stem_wgrad"):
        _lib.check(lib.cotb200_stem7x7s2_bf16(B, H, W, x.data_ptr(), wm.data_ptr(), N, D.data_ptr(), N, None, None, 0, cs.data_ptr(),
                                              cq.data_ptr(), scratch.data_ptr(), _st()), "stem7x7s2_bf16")
        _lib.check(lib.cotb200_stem7x7s2_wgrad_bf16(B, H, W, dy.data_ptr(), N, N, scratch.data_ptr(), dwm.data_ptr(), _st()),
                   "stem7x7s2_wgrad_bf16")
    torch.cuda.synchronize()
    what = "stem %s (%s)" % (case, _describe(plans))
    s_ref = torch.zeros(N, dtype=torch.float64, device="cuda")
    q_ref, d_abs = torch.zeros_like(s_ref), torch.zeros_like(s_ref)
    for b0, b1 in _chunks(B, 4):
        xc = x[b0:b1].permute(0, 3, 1, 2).double()
        ref = F.conv2d(xc, w.double(), stride=2, padding=3).permute(0, 2, 3, 1)
        if flt:
            absterms = F.conv2d(xc.abs(), w.double().abs(), stride=2, padding=3).permute(0, 2, 3, 1)
            _close(D[b0:b1], ref, absterms, what + " samples %d.." % b0, 2.0 ** -8)
        else:
            _equal_exact(D[b0:b1], ref, what + " samples %d.." % b0)
        d = D[b0:b1].double().reshape(-1, N)
        s_ref += d.sum(0)
        q_ref += (d * d).sum(0)
        d_abs += d.abs().sum(0)
    _sums_close(cs, s_ref, d_abs, what + " col_sum")
    _sums_close(cq, q_ref, q_ref, what + " col_sqsum")
    win = _stem_windows(scratch, B, Hh, Wh)
    ref = dy.double().t() @ win
    if flt:
        _sums_close(dwm, ref, dy.double().abs().t() @ win.abs(), what + " wgrad")
    else:
        _equal_exact(dwm, ref, what + " wgrad")


# ================================================================================================ TMA LocalConv (NHWC_TAP)
def _tap_pos(C, wc, fold, gc, device="cuda"):
    """[9, C] storage column (tap-major chunks of gc weight channels) of the weight that input channel c uses at tap t"""
    Cf, wcf = C // fold, wc // fold
    c = torch.arange(C, device=device)
    gch = (c // Cf) * wcf + (c % Cf) % wcf
    t = torch.arange(9, device=device)[:, None]
    return (gch // gc) * 9 * gc + t * gc + gch % gc


# (tap, dh, dw) of the 3x3 window
TAPS = [(t, t // 3 - 1, t % 3 - 1) for t in range(9)]


def agg_fwd_ref(x, w, pos):
    """y[n,h,w,c] = sum_t w[n,h,w,pos[t,c]] * x[n,h+dh,w+dw,c] (zero padding), fp64"""
    N, H, W, C = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    y = torch.zeros_like(x)
    for t, dh, dw in TAPS:
        y += w[..., pos[t]] * xp[:, 1 + dh:1 + dh + H, 1 + dw:1 + dw + W, :]
    return y


def agg_dx_ref(dy, w, pos):
    """dx[n,h,w,c] = sum_t w[n,h-dh,w-dw,pos[t,c]] * dy[n,h-dh,w-dw,c]"""
    N, H, W, C = dy.shape
    dx = torch.zeros_like(dy)
    for t, dh, dw in TAPS:
        p = F.pad(w[..., pos[t]] * dy, (0, 0, 1, 1, 1, 1))
        dx += p[:, 1 - dh:1 - dh + H, 1 - dw:1 - dw + W, :]
    return dx


def agg_dw_ref(x, dy, pos, J):
    """dw[n,h,w,pos[t,c]] += x[n,h+dh,w+dw,c] * dy[n,h,w,c]"""
    N, H, W, C = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    dw = torch.zeros(N, H, W, J, dtype=x.dtype, device=x.device)
    for t, dh, dw_ in TAPS:
        dw.index_add_(3, pos[t], xp[:, 1 + dh:1 + dh + H, 1 + dw_:1 + dw_ + W, :] * dy)
    return dw


def _desc(N, C, H, W, wc, dtype, layout, gc=0, fold=1):
    d = _lib.AggDesc()
    d.n, d.c, d.h, d.w, d.heads, d.wc = N, C, H, W, 1, wc
    d.kh = d.kw = 3
    d.sh = d.sw = d.dh = d.dw = 1
    d.ph = d.pw = 1
    d.ho, d.wo = H, W
    d.dtype, d.layout, d.gc, d.fold = _lib.dtype_code(torch.empty(0, dtype=dtype)), layout, gc, fold
    return d


@pytest.mark.parametrize("case", AGG_CASES, ids=lambda c: "%s-C%d-wc%d-%dx%d-fold%d-gc%d-%s" % c)
def test_agg_tma_fwd_dx_dw(case):
    dt, C, wc, H, W, fold, gc, kind = case
    plans, sz = agg_sizes(case, _sms())
    N = sz["N"]
    dtype = DTYPES[dt][0]
    _assert_regime(plans, partial_band=H % 2 == 0 or all(H % p.info["TH"] for p in plans))
    print("agg tma %s %s N=%d: %s" % (case, dtype, N, _describe(plans)))
    J = 9 * wc
    g = _gen(C + wc + H + fold + len(kind))
    flt = kind == "float"
    if flt:
        mk = lambda s: torch.randn(s, generator=g, device="cuda").to(dtype)
    else:
        mk = lambda s: _ints(s, -2, 2, g, dtype)
    x, w, dy = mk((N, H, W, C)), mk((N, H, W, J)), mk((N, H, W, C))
    y, dx, dw = (torch.full(s, float("nan"), dtype=dtype, device="cuda") for s in ((N, H, W, C), (N, H, W, C), (N, H, W, J)))
    d = _desc(N, C, H, W, wc, dtype, _lib.NHWC_TAP, gc, fold)
    lib = _lib.load()
    with kernels_ran(*[p.name for p in plans]):
        _lib.check(lib.cotb200_agg_zeropad_fwd(d, x.data_ptr(), w.data_ptr(), y.data_ptr(), _st()), "agg fwd")
        _lib.check(lib.cotb200_agg_zeropad_bwd(d, dy.data_ptr(), x.data_ptr(), w.data_ptr(), dx.data_ptr(), dw.data_ptr(), _st()), "agg bwd")
    torch.cuda.synchronize()
    what = "agg tma %s %s (%s)" % (case, dtype, _describe(plans))
    pos = _tap_pos(C, wc, fold, gc)
    rel = 0.0 if dtype == torch.float32 else 2.0 ** -8
    for n0, n1 in _chunks(N, 8):
        xs, ws, ds = (t[n0:n1].double() for t in (x, w, dy))
        refs = [("y", y, agg_fwd_ref(xs, ws, pos)), ("dX", dx, agg_dx_ref(ds, ws, pos)), ("dW", dw, agg_dw_ref(xs, ds, pos, J))]
        if flt:
            xa, wa, da = xs.abs(), ws.abs(), ds.abs()
            absterms = [agg_fwd_ref(xa, wa, pos), agg_dx_ref(da, wa, pos), agg_dw_ref(xa, da, pos, J)]
            for (name, got, ref), ab in zip(refs, absterms):
                _close(got[n0:n1], ref, ab, "%s %s samples %d.." % (what, name, n0), rel)
        else:
            for name, got, ref in refs:
                _equal_exact(got[n0:n1], ref, "%s %s samples %d.." % (what, name, n0))


# ================================================================================================ NCHW TMA LocalConv
def nchw_refs(x, w, dy, wc):
    """fwd / dX / dW of LocalConv 3x3 on NCHW: channel c uses weight channel c % wc; w [N, wc, 9, H, W]; fp64"""
    N, C, H, W = x.shape
    rep = C // wc
    wr = w.unsqueeze(1).expand(N, rep, wc, 9, H, W).reshape(N, C, 9, H, W)
    xp = F.pad(x, (1, 1, 1, 1))
    y, dx = torch.zeros_like(x), torch.zeros_like(x)
    dw = torch.zeros(N, wc, 9, H, W, dtype=x.dtype, device=x.device)
    for t in range(9):
        dh, dw_ = t // 3 - 1, t % 3 - 1
        xs = xp[:, :, 1 + dh:1 + dh + H, 1 + dw_:1 + dw_ + W]
        y += wr[:, :, t] * xs
        dx += F.pad(wr[:, :, t] * dy, (1, 1, 1, 1))[:, :, 1 - dh:1 - dh + H, 1 - dw_:1 - dw_ + W]
        dw[:, :, t] = (xs * dy).view(N, rep, wc, H, W).sum(1)
    return y, dx, dw


@pytest.mark.parametrize("case", NCHW_CASES, ids=lambda c: "%s-C%d-wc%d-%dx%d" % c)
def test_agg_nchw_tma(case):
    dt, C, wc, H, W = case
    plans, sz = nchw_sizes(case, _sms())
    N = sz["N"]
    _assert_regime(plans)
    dtype = DTYPES[dt][0]
    print("agg nchw tma %s N=%d: %s" % (case, N, _describe(plans)))
    g = _gen(C + wc + H + len(dt))
    x, dy = _ints((N, C, H, W), -2, 2, g, dtype), _ints((N, C, H, W), -2, 2, g, dtype)
    w = _ints((N, wc, 9, H, W), -2, 2, g, dtype)
    y, dx = (torch.full((N, C, H, W), float("nan"), dtype=dtype, device="cuda") for _ in range(2))
    dw = torch.full((N, wc, 9, H, W), float("nan"), dtype=dtype, device="cuda")
    d = _desc(N, C, H, W, wc, dtype, _lib.NCHW)
    lib = _lib.load()
    with kernels_ran(*NT_NAMES.values()):
        _lib.check(lib.cotb200_agg_zeropad_fwd(d, x.data_ptr(), w.data_ptr(), y.data_ptr(), _st()), "agg fwd")
        _lib.check(lib.cotb200_agg_zeropad_bwd(d, dy.data_ptr(), x.data_ptr(), w.data_ptr(), dx.data_ptr(), dw.data_ptr(), _st()), "agg bwd")
    torch.cuda.synchronize()
    what = "agg nchw tma %s (%s)" % (case, _describe(plans))
    for n0, n1 in _chunks(N, 8):
        refs = nchw_refs(x[n0:n1].double(), w[n0:n1].double(), dy[n0:n1].double(), wc)
        for name, got, ref in zip(("y", "dX", "dW"), (y, dx, dw), refs):
            _equal_exact(got[n0:n1], ref, "%s %s samples %d.." % (what, name, n0))


# ================================================================================================ GroupNorm blocks of 72
@pytest.mark.parametrize("case", GN_CASES, ids=lambda c: "%s-wc%d-%dx%d" % (c[0], c[1], c[2], c[2]))
def test_gn72_stats_apply_bwd(case):
    """stats (persistent walkers with a prefetching two-stage ring), apply, bwd sums and bwd apply at a batch where every stats CTA
    walks many tiles, against fp64 GroupNorm (normalisation is not integer-exact: tolerances of test_groupnorm9)"""
    from cotnet_b200 import fused
    dt, wc, H = case
    (plan,), sz = gn_sizes(case, _sms())
    B = sz["B"]
    _assert_regime([plan])
    dtype = DTYPES[dt][0]
    tol = 3e-2 if dt == "bf16" else 2e-4
    print("gn72 %s B=%d: %s" % (case, B, plan))
    J, gc = 9 * wc, 8
    g = _gen(wc + H + len(dt))
    gn = torch.nn.GroupNorm(wc, J).cuda()
    with torch.no_grad():
        gn.weight.uniform_(0.5, 1.5, generator=g)
        gn.bias.normal_(0, 0.3, generator=g)
    cl = lambda t: t.contiguous(memory_format=torch.channels_last)
    l = cl((torch.randn(B, J, H, H, generator=g, device="cuda") * 2 + 0.5).to(dtype)).requires_grad_(True)
    cot = cl(torch.randn(B, J, H, H, generator=g, device="cuda").to(dtype))
    lbias = (torch.randn(J, generator=g, device="cuda") * 0.7).requires_grad_(True)
    to_tap = lambda t: t.view(B, wc // gc, gc, 9, H, H).permute(0, 1, 3, 2, 4, 5).reshape(B, J, H, H)
    from_tap = lambda t: t.view(B, wc // gc, 9, gc, H, H).permute(0, 1, 3, 2, 4, 5).reshape(B, J, H, H)
    with kernels_ran("gn72_stats", "gn72_apply", "gn72_bwd_sums", "gn72_bwd_apply"):
        out_t = fused.group_norm9(l, gn, gc, lbias)
        got = torch.autograd.grad(out_t, (l, gn.weight, gn.bias, lbias), cl(to_tap(cot)))
    what = "gn72 %s (%s)" % (case, plan)
    lr = l.detach().double().requires_grad_(True)
    br = lbias.detach().double().requires_grad_(True)
    gnr = torch.nn.GroupNorm(wc, J).cuda().double()
    gnr.load_state_dict(gn.state_dict())
    ref = gnr(lr + br.view(1, J, 1, 1))
    refs = torch.autograd.grad(ref, (lr, gnr.weight, gnr.bias, br), cot.double())
    for a, b, name in zip((from_tap(out_t),) + tuple(got), (ref,) + tuple(refs), ("out", "dl", "dgamma", "dbeta", "dlbias")):
        err = (a.double() - b).abs().max().item()
        scale = max(1.0, b.abs().max().item())
        assert err <= tol * scale, "%s %s: err %.3e scale %.3e" % (what, name, err, scale)
