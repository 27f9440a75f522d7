"""The launch geometry of the row kernels (csrc/norm_tail.cu, csrc/gn72.cu), mirrored in Python and checked without a GPU: the mirror
matches the sources, and the named cases of tests/test_row_kernels_gpu.py reach every dispatch branch of those kernels -- every packet
width, padded thread columns, a ragged last row chunk, a single CTA, less than one wave and six waves of CTAs, 2 / 3 / 8 column
chunks (with and without the 1-bit mask), the gn72 fast path with its statistics walkers past the first turn of their two-stage
ring and with several CTAs per sample, the generic GroupNorm kernels, and sum_rows past its grid-stride cap -- on both H100 SM
counts.  The GPU file imports CASES and SUM_CASES and repeats the coverage assertions with the live SM count."""
import os
from collections import namedtuple

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cotnet_b200", "csrc")
SMS_H100 = (132, 114)          # H100 SXM, H100 PCIe
NT_THREADS = 256
ESIZE = {"f32": 4, "bf16": 2, "f16": 2}


# ------------------------------------------------------------------------------------------------ mirror of the host code
def pick_vec(C, esize, offsets=(0,)):
    """pick_vec<T>: the widest packet (<= 16 bytes) that divides C and to which every given pointer (byte offsets) is aligned."""
    vec = 16 // esize
    while vec >= 1:
        if C % vec == 0 and all(o % (vec * esize) == 0 for o in offsets):
            return vec
        vec //= 2
    return 1


def col_chunk(C, vec):
    """col_chunk: the column chunk width (a multiple of vec dividing C, at most 256 packets), C itself, or 0."""
    if C // vec <= NT_THREADS:
        return C
    for nz in range(2, 65):
        if C % nz == 0 and (C // nz) % vec == 0 and (C // nz) // vec <= NT_THREADS:
            return C // nz
    return 0


def mask_geo_ok(C, vec):
    cw = col_chunk(C, vec)
    return C % 8 == 0 and cw != 0 and cw % 8 == 0


def gn72_ok(wc, gc, permuting, offsets):
    if wc not in (8, 16, 32, 64):
        return False
    if permuting and gc != 8:
        return False
    return all(o % 16 == 0 for o in offsets)


def gn72_grid(dtype, B, HW, wc, sms):
    """gn72.cu launches: (tiles per sample, statistics walkers per sample X, CTAs per sample of apply / bwd_apply, of bwd_sums)"""
    tb = 256 if ESIZE[dtype] == 2 else 128          # blocks of 72 per tile
    bps = HW * (wc // 8)
    ntiles = (bps + tb - 1) // tb
    X = max(1, min((4 * sms + B - 1) // B, ntiles))
    pr = tb // (wc // 8)                             # pixels per bwd_sums tile
    return ntiles, X, (bps + tb - 1) // tb, (HW + pr - 1) // pr


Geo = namedtuple("Geo", "B HW C vec cq cq_pad ry rows_per_cta gx waves")


def make_geo(B, HW, C, vec, sms):
    """make_geo: None where the C ABI returns EINVAL; waves = the k of the k * SM-count CTA target that was taken (0: none, the
    row chunk was raised to min_rows)."""
    cq = C // vec
    cq_pad = 1
    while cq_pad < cq:
        cq_pad <<= 1
    if cq_pad > NT_THREADS:
        return None
    ry = NT_THREADS // cq_pad
    min_rows = max(ry * 2, 24)
    rows, waves = HW, 0
    for k in range(6, 0, -1):
        per_b = (sms * k + B - 1) // B
        rows = (HW + per_b - 1) // per_b
        if rows >= min_rows:
            waves = k
            break
    rows = min(max(rows, min_rows), HW)
    return Geo(B, HW, C, vec, cq, cq_pad, ry, rows, (HW + rows - 1) // rows, waves)


# ------------------------------------------------------------------------------------------------ the cases of the GPU file
# kind: "bn" (col_stats, bn_apply(_batch), bn_bwd_*: rows flattened to B*HW, columns chunked), "tail" (the CoT / split-attention
# tail kernels: one row range per sample), "gn" (the gn9_* entry points; C = wc, gc the storage order).  off: element offset of
# every data pointer into a larger buffer.  amp: the data are integers in [-amp, amp] (exact_sum_bound).  expect: the branches the
# case is there for.
Case = namedtuple("Case", "name kind dtype B HW C off gc amp expect")


def _c(name, kind, dtype, B, HW, C, off=0, gc=0, amp=4, expect=()):
    return Case(name, kind, dtype, B, HW, C, off, gc, amp, frozenset(expect))


CASES = [
    # BatchNorm
    _c("bn_bf16_vec8_six_waves", "bn", "bf16", 3, 16896, 64, amp=3, expect={"vec8", "six_waves", "B_odd", "mask"}),
    _c("bn_f16_vec4_offset_one_wave", "bn", "f16", 1, 1000, 64, off=4,
       expect={"vec4", "vec_by_offset", "under_one_wave", "ragged_rows", "B1", "mask"}),
    _c("bn_f32_vec2_cqpad", "bn", "f32", 5, 77, 202, expect={"vec2", "cq_pad>cq", "B_odd"}),
    _c("bn_f16_vec2_parity", "bn", "f16", 2, 61, 66, expect={"vec2", "cq_pad>cq"}),
    _c("bn_bf16_vec1_c3_single_cta", "bn", "bf16", 2, 50, 3, expect={"vec1", "cq_pad>cq", "single_cta"}),
    _c("bn_bf16_vec8_ragged", "bn", "bf16", 7, 99, 256, expect={"vec8", "ragged_rows", "under_one_wave", "B_odd", "mask"}),
    _c("bn_f32_two_chunks_mask", "bn", "f32", 3, 37, 2048, expect={"vec4", "chunks2", "mask_chunked", "B_odd"}),
    _c("bn_f32_vec1_three_chunks_mask", "bn", "f32", 2, 29, 600, off=1,
       expect={"vec1", "vec_by_offset", "chunks3", "mask_chunked"}),
    _c("bn_bf16_vec1_eight_chunks_mask", "bn", "bf16", 1, 45, 2048, off=1,
       expect={"vec1", "vec_by_offset", "chunks8", "mask_chunked", "B1"}),
    _c("bn_f16_vec8_c200", "bn", "f16", 3, 40, 200, expect={"vec8", "cq_pad>cq", "mask"}),
    # CoT / split-attention tails (each test runs with k present and with k == NULL)
    _c("tail_bf16_vec8", "tail", "bf16", 3, 196, 64, expect={"vec8", "B_odd"}),
    _c("tail_f32_vec4_over_six_waves", "tail", "f32", 801, 8, 64, expect={"vec4", "over_six_waves", "B_odd"}),
    _c("tail_f16_vec2_offset_ragged", "tail", "f16", 1, 500, 64, off=2,
       expect={"vec2", "vec_by_offset", "ragged_rows", "under_one_wave", "B1"}),
    _c("tail_bf16_vec8_c200_cqpad", "tail", "bf16", 5, 49, 200, expect={"vec8", "cq_pad>cq", "B_odd"}),
    _c("tail_f32_vec1_c3_single_cta", "tail", "f32", 1, 20, 3, expect={"vec1", "single_cta", "cq_pad>cq", "B1"}),
    _c("tail_f16_vec4_c100", "tail", "f16", 4, 150, 100, expect={"vec4", "cq_pad>cq"}),
    _c("tail_f32_vec1_offset", "tail", "f32", 3, 64, 96, off=1, expect={"vec1", "vec_by_offset"}),
    # GroupNorm over 9 taps (C = wc)
    _c("gn72_bf16_wc8", "gn", "bf16", 3, 50, 8, gc=8, expect={"gn72", "gc8", "B_odd"}),
    _c("gn72_f32_wc64", "gn", "f32", 2, 33, 64, gc=8, expect={"gn72", "gc8", "gn72_multi_cta_f32"}),
    # 5 tiles per sample for one statistics walker: both ring stages reused at both mbarrier parities, a partial last tile, 5 CTAs
    # per sample in apply / bwd_sums / bwd_apply, and more samples than the 256 threads of gn_bwd_finish
    _c("gn72_bf16_wc8_ring_wrap", "gn", "bf16", 531, 1025, 8, gc=8, amp=1,
       expect={"gn72", "gc8", "B_odd", "gn72_multi_tile", "gn72_ring_wrap", "gn72_multi_cta_16bit", "gn_finish_strided"}),
    _c("gn72_f16_wc16", "gn", "f16", 1, 70, 16, gc=8, expect={"gn72", "gc8", "B1"}),
    _c("gn_generic_bf16_wc8_gc0", "gn", "bf16", 3, 41, 8, gc=0, expect={"gn_generic", "gc0", "vec8", "cq_pad>cq"}),
    _c("gn_generic_f32_wc24_gc8", "gn", "f32", 2, 45, 24, gc=8, expect={"gn_generic", "gn_stats_generic", "gc8", "vec4"}),
    _c("gn_generic_bf16_wc8_gc8_offset", "gn", "bf16", 3, 30, 8, off=1, gc=8,
       expect={"gn_generic", "gn_stats_generic", "gc8", "vec1", "vec_by_offset"}),
    _c("gn_generic_f16_wc4_gc0", "gn", "f16", 1, 60, 4, gc=0, expect={"gn_generic", "gn_stats_generic", "gc0", "vec4", "B1"}),
]

# branches every family's cases must reach together
REQUIRED = {
    "bn": {"vec8", "vec4", "vec2", "vec1", "vec_by_offset", "cq_pad>cq", "ragged_rows", "single_cta", "under_one_wave", "six_waves",
           "chunks2", "chunks3", "chunks8", "mask", "mask_chunked", "B1", "B_odd", "f32", "bf16", "f16"},
    "tail": {"vec8", "vec4", "vec2", "vec1", "vec_by_offset", "cq_pad>cq", "ragged_rows", "single_cta", "under_one_wave",
             "over_six_waves", "B1", "B_odd", "f32", "bf16", "f16"},
    "gn": {"gn72", "gn_generic", "gn_stats_generic", "gc0", "gc8", "vec8", "vec4", "vec1", "vec_by_offset", "B1", "B_odd",
           "f32", "bf16", "f16", "gn72_multi_tile", "gn72_ring_wrap", "gn72_multi_cta_16bit", "gn72_multi_cta_f32",
           "gn_finish_strided"},
}


def _geo_branches(g, sms, vec_plain):
    out = {"vec%d" % g.vec}
    if g.vec < vec_plain:
        out.add("vec_by_offset")
    if g.cq_pad > g.cq:
        out.add("cq_pad>cq")
    if g.HW % g.rows_per_cta:
        out.add("ragged_rows")
    ctas = g.gx * g.B
    if ctas == 1:
        out.add("single_cta")
    if ctas < sms:
        out.add("under_one_wave")
    if g.waves == 6:
        out.add("six_waves")
    if ctas > 6 * sms:
        out.add("over_six_waves")
    return out


def plan(case, sms):
    """(geometries, branches) of one case on `sms` SMs: the geometry of every launch of the case's row kernels."""
    es = ESIZE[case.dtype]
    off = case.off * es
    br = {case.dtype}
    if case.B == 1:
        br.add("B1")
    elif case.B % 2:
        br.add("B_odd")
    geos = []
    if case.kind == "bn":
        vec, plain = pick_vec(case.C, es, (off,)), pick_vec(case.C, es)
        cw = col_chunk(case.C, vec)
        assert cw, case
        g = make_geo(1, case.B * case.HW, cw, vec, sms)
        geos = [g] * (case.C // cw)
        br |= _geo_branches(g, sms, plain)
        if case.C // cw > 1:
            br.add("chunks%d" % (case.C // cw))
        if mask_geo_ok(case.C, vec):
            br.add("mask_chunked" if case.C // cw > 1 else "mask")
    elif case.kind == "tail":
        vec, plain = pick_vec(case.C, es, (off,)), pick_vec(case.C, es)
        g = make_geo(case.B, case.HW, case.C, vec, sms)
        geos = [g]
        br |= _geo_branches(g, sms, plain)
    else:
        J = 9 * case.C
        br.add("gc%d" % case.gc)
        if case.C % 8 == 0:
            ntiles, X, cta_apply, cta_sums = gn72_grid(case.dtype, case.B, case.HW, case.C, sms)
        if case.B > 256:
            br.add("gn_finish_strided")
        if not gn72_ok(case.C, case.gc, False, (off,)):
            br.add("gn_stats_generic")
        else:
            walker0 = (ntiles + X - 1) // X           # tiles of the first walker of a sample
            if walker0 >= 2:
                br.add("gn72_multi_tile")
            if walker0 >= 4:                          # stage 0 and stage 1 each refilled at mbarrier parity 0 and 1
                br.add("gn72_ring_wrap")
        if gn72_ok(case.C, case.gc, True, (off,)):
            br.add("gn72")
            if cta_apply > 1 and cta_sums > 1:
                br.add("gn72_multi_cta_16bit" if ESIZE[case.dtype] == 2 else "gn72_multi_cta_f32")
        else:
            br.add("gn_generic")
            vec, plain = pick_vec(J, es, (off,)), pick_vec(J, es)
            g = make_geo(case.B, case.HW, J, vec, sms)
            geos = [g]
            br |= _geo_branches(g, sms, plain)
    assert all(g is not None for g in geos), case
    return geos, br


def coverage(sms):
    """{kind: set of branches reached} and the list of (case, expected branch missing) on `sms` SMs."""
    reached = {k: set() for k in REQUIRED}
    missing = []
    for case in CASES:
        _, br = plan(case, sms)
        reached[case.kind] |= br
        missing += [(case.name, b) for b in sorted(case.expect - br)]
    return reached, missing


def assert_coverage(sms):
    reached, missing = coverage(sms)
    assert not missing, "cases that no longer reach their branch on %d SMs: %s" % (sms, missing)
    for kind, need in REQUIRED.items():
        assert need <= reached[kind], "%s: branches without a case on %d SMs: %s" % (kind, sms, sorted(need - reached[kind]))
    named = {k: set() for k in REQUIRED}
    for case in CASES:
        named[case.kind] |= case.expect | {case.dtype}
    for kind, need in REQUIRED.items():
        assert need <= named[kind], "%s: branches no case names: %s" % (kind, sorted(need - named[kind]))
    return reached


def exact_sum_bound(case):
    """The largest sum over |term| / granularity among the sums the GPU file checks bit for bit.  All terms are multiples of the
    granularity, so the sums are exact in fp32, in any order, while this stays below 2^24.  a = case.amp.
      bn:   col_stats x^2 <= a^2 (granularity 1) over B*HW rows; bwd dz*xhat with dz = s_b*dy (s_b <= 2, granularity 1/2) and
            xhat = (x - mu)*rstd (|mu| <= 2, rstd in {1/2, 1, 2}): <= 2a * 2(a+2) at granularity 1/4, over B*HW rows.
      tail: pool y + k, y = z <= 30 + 2a (granularity 1) over HW rows; dz_sums dz*xhat with dz = (a0*dout + dpn/2)*silu'
            (a0 <= 2 at 1/2, silu' in {1/2, 1}): <= (2a + 2) * 2(a+2) at granularity 1/8, over B*HW rows.
      gn:   stats (l + lbias)^2 <= (a+2)^2 over 9*HW; dgamma dg*lhat, lhat = (l + lbias - mean)*rstd (|lbias| <= 2, |mean| <= 1):
            <= a * 2(a+3) at granularity 1/2 over B*HW; s2 = sum_t gamma*dg*lhat (gamma <= 2 at 1/2): granularity 1/4 over 9*HW."""
    a, n = case.amp, case.B * case.HW
    if case.kind == "bn":
        return max(n * a * a, n * 2 * a * 2 * (a + 2) * 4)
    if case.kind == "tail":
        return max(case.HW * (30 + 3 * a), n * (2 * a + 2) * 2 * (a + 2) * 8)
    return max(9 * case.HW * (a + 2) ** 2, n * a * 2 * (a + 3) * 2, 9 * case.HW * 2 * a * 2 * (a + 3) * 4)


# sum_rows: name, dtype, rows, C, source pitches, output pitch, element offset
SUM_CASES = [
    ("sum2_bf16_vec8", "bf16", 300, 64, (72, 128), 80, 0),
    ("sum3_f32_vec4", "f32", 257, 96, (100, 96, 192), 104, 0),
    ("sum4_f16_vec1_offset", "f16", 131, 40, (48, 56, 40, 64), 48, 1),
    ("sum4_bf16_vec2_pitch", "bf16", 77, 64, (66, 64, 70, 64), 66, 0),
    ("sum3_f32_c3", "f32", 500, 3, (5, 3, 7), 4, 0),
    ("sum2_bf16_grid_stride", "bf16", 20000, 256, (256, 264), 264, 0),
]


def sum_rows_grid(dtype, rows, C, lds, ldo, off, sms):
    """cotb200_sum_rows: (packet width, packets, threads of the capped grid)"""
    es = ESIZE[dtype]
    vec = 16 // es
    while vec > 1 and not (C % vec == 0 and (off * es) % (vec * es) == 0 and all(ld % vec == 0 for ld in tuple(lds) + (ldo,))):
        vec //= 2
    total = rows * (C // vec)
    return vec, total, min((total + 255) // 256, 16 * sms) * 256


def assert_sum_rows_coverage(sms):
    """every packet width, and one case whose grid-stride loop gives threads a second item"""
    plans = {c[0]: sum_rows_grid(*c[1:], sms) for c in SUM_CASES}
    assert {v for v, _, _ in plans.values()} == {8, 4, 2, 1}, plans
    _, total, threads = plans["sum2_bf16_grid_stride"]
    assert total > threads, "sum_rows: no case past the grid-stride cap on %d SMs (%d packets, %d threads)" % (sms, total, threads)


# ------------------------------------------------------------------------------------------------ tests
def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_mirror_matches_the_sources():
    """The lines of norm_tail.cu / gn72.cu the mirror above restates."""
    s = _src("norm_tail.cu")
    for snippet in ("static constexpr int NT_THREADS = 256;",
                    "for (int vec = 16 / (int)sizeof(T); vec >= 1; vec >>= 1) {",
                    "if (C / vec <= NT_THREADS) return C;",
                    "for (int nz = 2; nz <= 64; ++nz)",
                    "if (C % nz == 0 && (C / nz) % vec == 0 && (C / nz) / vec <= NT_THREADS) return C / nz;",
                    "return C % 8 == 0 && cw && cw % 8 == 0;",
                    "while (g.cq_pad < g.cq) g.cq_pad <<= 1;",
                    "if (g.cq_pad > NT_THREADS)",
                    "g.ry = NT_THREADS / g.cq_pad;",
                    "int min_rows = g.ry * 2;", "if (min_rows < 24) min_rows = 24;",
                    "for (int k = 6; k >= 1; --k) {",
                    "const long long ctas = (long long)sms * k;",
                    "const int per_b = (int)((ctas + B - 1) / B);",
                    "const int r = (HW + per_b - 1) / per_b;",
                    "if (r >= min_rows) break;",
                    "if (rows < min_rows) rows = min_rows;", "if (rows > HW) rows = HW;",
                    "#define NT_GRID dim3((g.HW + g.rows_per_cta - 1) / g.rows_per_cta, g.B)"):
        assert snippet in s, snippet
    g = _src("gn72.cu")
    for snippet in ("if (wc != 8 && wc != 16 && wc != 32 && wc != 64) return false;", "if (permuting && gc != 8) return false;",
                    "return aligned16(p0) && (!p1 || aligned16(p1)) && (!p2 || aligned16(p2));",
                    "static constexpr int TB = sizeof(T) == 2 ? 256 : 128;", "g.nchunk = wc / 8; g.J = 9 * wc; g.bps = HW * g.nchunk;",
                    "const int ntiles = (g.bps + TB - 1) / TB;", "int X = (4 * num_sms() + B - 1) / B;", "if (X > ntiles) X = ntiles;",
                    "for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {",
                    "mbar_wait(smem_u32(&bar[stage]), (it >> 1) & 1);", "const int PR = TB / g.nchunk;",
                    "<<<dim3((g.bps + TB - 1) / TB, B), TB, smem, st>>>", "<<<dim3((HW + PR - 1) / PR, B), G7_SUM_THREADS, smem, st>>>",
                    "static constexpr int G7_FIN_THREADS = 256;", "for (int b = tid; b < B; b += G7_FIN_THREADS) {"):
        assert snippet in g, snippet
    r = _src("sum_rows.cu")
    for snippet in ("int vec = 16 / (int)sizeof(T);", "if (((uintptr_t)s.p[k] & m) || (s.ld[k] % v)) return false;",
                    "return !((uintptr_t)out & m) && !(ldo % v);", "item < total; item += (long long)gridDim.x * 256"):
        assert snippet in r, snippet


def test_sum_rows_grid_matches_the_sources():
    """sum_rows_grid's capped grid: the (threads, per_sm) of the sum_rows launch and grid_stride_blocks in common.cuh."""
    assert "const int blocks = grid_stride_blocks(total, 256, 16);" in _src("sum_rows.cu")
    c = _src("common.cuh")
    for snippet in ("const long long need = (items + threads - 1) / threads;", "const long long cap = (long long)num_sms() * per_sm;",
                    "return (int)(need < 1 ? 1 : need < cap ? need : cap);"):
        assert snippet in c, snippet


def test_mirror_known_geometry():
    """hand-checked anchors: the 2048-channel fp32 bn3 of layer 4 runs in two chunks of 256 packets; the stage-1 bf16 BatchNorm of
    the benchmark batch (256 x 56 x 56 rows, 64 channels) gets six waves of 132 CTAs."""
    assert (pick_vec(2048, 4), col_chunk(2048, 4)) == (4, 1024)
    assert col_chunk(600, 1) == 200 and col_chunk(2048, 1) == 256 and col_chunk(264, 1) == 132
    assert not mask_geo_ok(264, 1) and mask_geo_ok(264, 8) and not mask_geo_ok(12, 4)
    g = make_geo(1, 256 * 56 * 56, 64, 8, 132)
    assert (g.cq, g.cq_pad, g.ry, g.waves, g.gx) == (8, 8, 32, 6, 792)
    assert pick_vec(64, 2, (4,)) == 2 and pick_vec(64, 2, (8,)) == 4 and pick_vec(3, 4) == 1


@pytest.mark.parametrize("sms", SMS_H100)
def test_cases_reach_every_branch(sms):
    assert_coverage(sms)
    assert_sum_rows_coverage(sms)


@pytest.mark.parametrize("sms", SMS_H100)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_reaches_its_branches(case, sms):
    geos, br = plan(case, sms)
    assert case.expect <= br, "%s on %d SMs misses %s (geometry %s)" % (case.name, sms, sorted(case.expect - br), geos)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_exact_sums_stay_below_2_24(case):
    assert exact_sum_bound(case) < (1 << 24), (case.name, exact_sum_bound(case))
