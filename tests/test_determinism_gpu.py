"""The deterministic cross-CTA reductions (det_finish, csrc/common.cuh) under every reducing entry point of the library.

Each CTA stores its partial sums to its own scratch row; the last CTA of a block of `fan` rows adds that block in row order, the
last block adds the block totals.  The order depends on the slot count only, so the same inputs must give the same bits on every
run, on every stream and inside a replayed CUDA graph.  Every case below calls the C ABI directly (so the launch geometry is
exactly the one chosen here), asserts the regime its geometry reaches, and checks

  1. the sum against an fp64 reference of the same terms, per element, to fp32 accumulation accuracy;
  2. that the outputs are accumulated (+=) into a pre-filled value;
  3. bit-identical results over eager repeats, under a concurrent load on another stream, and on two streams at once;
  4. bit-identical results of CUDA-graph replays (the tickets are reset by the graph's own memset node).

Regimes of the slot count nslots of one reduction:  R1 = 1 slot;  R2 = 2..16 slots, one block;  R3 = 17..1008 slots, blocks of
16, the last one partial;  R4 = more than 1008 slots, fan > 16.  Only cotb200_tail_bwd_dz_sums reduces over the whole
[B x row-chunk] grid without flattening the batch, so only it reaches R4: the flattened row kernels stop at 6 CTAs per SM, the
per-sample ones at 6 * SMs / B per sample, gn72 at 4 * SMs / B per sample (bwd: HW / pixels-per-tile), the GEMM and convolution
epilogues at 2 CTAs per SM (all R3 at most).  The weight gradients add their split-K partials in split order in a separate
kernel; their regimes are splits == 1 and splits > 1.

The model-level tests at the end check that whole training steps (eager and CUDA graph) are bitwise reproducible."""
import copy

import pytest
import torch

from cotnet_b200 import _lib

pytestmark = pytest.mark.gpu

# Per-element tolerance: |(out - prefill) - ref| <= TOL * (sum|terms| + |prefill|).  Recursive fp32 summation of a chain of
# n additions is off by at most n * 2^-24 * sum|terms| (first order).  The longest serial chain of the cases below is about 200
# additions (rows of one thread + the row lanes of the CTA + a 16/17-row block + up to 63 block totals + the final +=; for the
# weight gradients the wgmma k-steps of one split + the splits), i.e. <= 1.2e-5.  A dropped or doubly added partial moves a
# sum by about sum/nslots >= 1e-3 * sum of the positive-mean terms used here, far outside.
TOL = 2e-5
PREFILL = 0.75                  # the known non-zero value accumulated outputs start from (exact in fp32)


# ================================================================================================ launch geometry (Python copies)
# cotnet_b200/csrc/common.cuh: det_fan, det_blocks
DET_TICKETS_PER_GROUP = 64


def det_fan(nslots):
    f = (nslots + DET_TICKETS_PER_GROUP - 2) // (DET_TICKETS_PER_GROUP - 1)
    return 16 if f < 16 else f


def det_blocks(nslots):
    return (nslots + det_fan(nslots) - 1) // det_fan(nslots)


def regime(nslots):
    if nslots == 1:
        return "R1"
    if nslots <= 16:
        return "R2"
    return "R3" if nslots <= 16 * (DET_TICKETS_PER_GROUP - 1) else "R4"


def _cdiv(a, b):
    return (a + b - 1) // b


# cotnet_b200/csrc/norm_tail.cu: pick_vec (aligned tensors), make_geo, col_chunk, det_geo (slots of one reduction)
NT_THREADS = 256


def pick_vec(C, esize):
    vec = 16 // esize
    while vec > 1 and C % vec:
        vec //= 2
    return vec


def make_geo(B, HW, C, vec, sms):
    """(rows_per_cta, ry, gx): gx = row chunks per sample = grid.x of the row kernels"""
    cq = C // vec
    cq_pad = 1
    while cq_pad < cq:
        cq_pad <<= 1
    assert cq_pad <= NT_THREADS
    ry = NT_THREADS // cq_pad
    min_rows = max(2 * ry, 24)
    rows = HW
    for k in range(6, 0, -1):
        per_b = _cdiv(sms * k, B)
        rows = _cdiv(HW, per_b)
        if rows >= min_rows:
            break
    rows = min(max(rows, min_rows), HW)
    return rows, ry, _cdiv(HW, rows)


def col_chunk(C, vec):
    if C // vec <= NT_THREADS:
        return C
    for nz in range(2, 65):
        if C % nz == 0 and (C // nz) % vec == 0 and (C // nz) // vec <= NT_THREADS:
            return C // nz
    return 0


def rows_slots(kind, B, HW, C, esize, sms):
    """Slots of one reduction of a row kernel.  kind: 'flat' (col_stats, bn_bwd_sums: [B, HW] flattened to rows, one group per
    column chunk), 'sample' (tail_pool, tail_bwd_sums, generic gn9: one group per sample), 'grid' (tail_bwd_dz_sums: one group
    over the whole [gx, B] grid)."""
    vec = pick_vec(C, esize)
    if kind == "flat":
        _, _, gx = make_geo(1, B * HW, col_chunk(C, vec), vec, sms)
        return gx
    _, _, gx = make_geo(B, HW, C, vec, sms)
    return gx * B if kind == "grid" else gx


# cotnet_b200/csrc/gn72.cu: gn72_ok, gn72_stats_launch (X), gn72_bwd_sums_launch (HW / PR)
def gn72_ok(wc, gc, permuting):
    return wc in (8, 16, 32, 64) and (not permuting or gc == 8)


def gn72_stats_slots(B, HW, wc, esize, sms):
    tb = 256 if esize == 2 else 128
    ntiles = _cdiv(HW * (wc // 8), tb)
    return max(1, min(_cdiv(4 * sms, B), ntiles))


def gn72_bwd_slots(HW, wc, esize):
    tb = 256 if esize == 2 else 128
    return _cdiv(HW, tb // (wc // 8))


# cotnet_b200/csrc/tc_gemm.cu: TC_* constants, pick_bn, tc_launch (grid), conv3x3_halo_launch (grid), conv mode m_tiles
TC_BM, TC_BK = 128, 64


def pick_bn_wide(N):
    parts = _cdiv(N, 256)
    return min((_cdiv(N, parts) + 63) & ~63, 256)


def pick_bn(N, K=1 << 30):
    if K <= 128 and N > 128:
        parts = _cdiv(N, 128)
        return min((_cdiv(N, parts) + 63) & ~63, 128)
    return pick_bn_wide(N)


def tc_grid(N, bn, m_tiles, stats, sms):
    out_bytes = 2 * TC_BM * 128 + ((2 * 4 * 256 * 4 + 2 * N * 4) if stats else 0)
    stage_bytes = TC_BM * TC_BK * 2 + ((bn * TC_BK * 2 + 1023) & ~1023)
    per_sm = 2
    if (104 * 1024 - out_bytes) // stage_bytes < 2 or bn > 128:
        per_sm = 1
    return min(per_sm * sms, m_tiles * _cdiv(N, bn))


def conv3x3_slots(B, H, W, C, bn, sms):
    """(path, grid) of cotb200_conv3x3_bf16 with dense NHWC operands"""
    Wp = W + 2
    if bn == 64 and C % 64 == 0 and Wp <= 256:
        R = 0
        for r in range(1, H + 1):
            if H % r == 0 and r * Wp <= 256 and r * W <= 256:
                R = r
        n_tiles = C // 64
        if R and n_tiles <= sms:
            MB = _cdiv(R * Wp, 128)
            a_stage = (max((R + 2) * Wp, MB * 128 + 2 * Wp + 2) * 128 + 1023) & ~1023
            out_bytes = (R * W * 128 + 1023) & ~1023
            if min((220 * 1024 - 9 * 64 * 128 - out_bytes) // a_stage, 4) >= 2:
                return "halo", min((sms // n_tiles) * n_tiles, B * (H // R) * n_tiles)
    if H * W <= TC_BM // 2:
        m_tiles = _cdiv(B, TC_BM // (H * W))
    else:
        hb = max(1, min(TC_BM // W, H))
        while H % hb:
            hb -= 1
        m_tiles = B * (H // hb)
    return "tc", tc_grid(C, bn, m_tiles, True, sms)


def stem_slots(B, H, W, N, sms):
    Wh = W // 2
    wtiles = _cdiv(Wh, TC_BM)
    while Wh % wtiles:
        wtiles += 1
    return tc_grid(N, pick_bn_wide(N), B * (H // 2) * wtiles, True, sms)


# cotnet_b200/csrc/tc_wgrad.cu: cotb200_wgrad_bf16 and cotb200_stem7x7s2_wgrad_bf16 (splits)
def wgrad_splits(M, R, Cc, sms):
    tiles = _cdiv(R, 128) * _cdiv(_cdiv(Cc, 64) * 64, 256)
    kb_total = _cdiv(M, 64)
    splits = max(1, min(_cdiv(sms, tiles), (kb_total + 3) // 4))
    return _cdiv(kb_total, _cdiv(kb_total, splits))


def stem_wgrad_splits(B, H, sms):
    kb_total = B * (H // 2)
    splits = min(sms, kb_total)
    return _cdiv(kb_total, _cdiv(kb_total, splits))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _geo_str(nslots):
    fan, nblk = det_fan(nslots), det_blocks(nslots)
    return "nslots=%d fan=%d blocks=%d last_block=%d" % (nslots, fan, nblk, nslots - (nblk - 1) * fan)


# ================================================================================================ harness
class Case:
    """outs: [(shape, dtype, prefill, accumulated)]; call(outs, stream_handle) issues the library call(s);
    reference(outs) -> [(out index, fp64 reference, fp64 sum|terms|, sensitive)] -- `sensitive` outputs are cross-CTA sums whose
    every slot holds a visible share (checked against nslots)."""

    def __init__(self, nslots, outs, call, reference, det=True):
        self.nslots, self.outs, self.call, self.reference, self.det = nslots, outs, call, reference, det

    def new_outs(self):
        return [torch.empty(s, dtype=dt, device="cuda") for s, dt, _, _ in self.outs]

    def fill(self, outs):
        for o, (_, _, p, _) in zip(outs, self.outs):
            o.fill_(p)

    def run(self, outs):
        self.fill(outs)
        self.call(outs, torch.cuda.current_stream().cuda_stream)


_LOAD = {}


def _load_on(stream):
    """A few large bf16 matmuls on `stream`: they occupy the SMs while the call under test runs, so its CTAs finish in another order."""
    if "a" not in _LOAD:
        g = torch.Generator(device="cuda").manual_seed(99)
        _LOAD["a"] = torch.randn(8192, 8192, generator=g, device="cuda").bfloat16()
    a = _LOAD["a"]
    with torch.cuda.stream(stream):
        for _ in range(3):
            _LOAD["c"] = a @ a


def _snap(outs):
    return [o.clone() for o in outs]


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def _check_exact(case, outs, what):
    for i, ref, absterms, sensitive in case.reference(outs):
        _, _, pre, acc = case.outs[i]
        got = outs[i].double() - (pre if acc else 0.0)
        lim = TOL * (absterms + (abs(pre) if acc else 0.0))
        err = (got - ref).abs()
        bad = ~(err <= lim)
        assert not bool(bad.any()), "%s output %d: %d of %d elements off; worst err/limit %.3g" % (
            what, i, int(bad.sum()), bad.numel(), float((err / lim.clamp_min(1e-30)).max()))
        if sensitive:
            # one slot's share (about |sum| / nslots) must be far above the tolerance, or a lost partial would go unnoticed
            m = absterms > 0
            share = ref.abs()[m] / case.nslots
            assert bool((share > 4 * lim[m]).all()), "%s output %d: a slot's share is not above the tolerance" % (what, i)


def run_case(case, what):
    torch.cuda.synchronize()
    main = torch.cuda.current_stream()
    # 1 + 2: exact, accumulated
    first = case.new_outs()
    case.run(first)
    torch.cuda.synchronize()
    _check_exact(case, first, what)
    # 3a: eager repeats
    for r in range(4):
        o = case.new_outs()
        case.run(o)
        assert _equal(o, first), "%s: eager repeat %d differs bitwise" % (what, r)
    # 3b: under a concurrent load on another stream
    side = torch.cuda.Stream()
    side.wait_stream(main)
    o = case.new_outs()
    case.fill(o)
    _load_on(side)
    case.call(o, main.cuda_stream)
    main.wait_stream(side)
    assert _equal(o, first), "%s: repeat under a concurrent load differs bitwise" % what
    # 3c: the same call on two streams at once, separate outputs
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    o1, o2 = case.new_outs(), case.new_outs()
    case.fill(o1)
    case.fill(o2)
    s1.wait_stream(main)
    s2.wait_stream(main)
    with torch.cuda.stream(s1):
        case.call(o1, s1.cuda_stream)
    with torch.cuda.stream(s2):
        case.call(o2, s2.cuda_stream)
    main.wait_stream(s1)
    main.wait_stream(s2)
    assert _equal(o1, first) and _equal(o2, first), "%s: concurrent calls on two streams differ bitwise" % what
    # 4: graph replay ("fill outputs; call"), three replays, each bit-identical to eager
    og = case.new_outs()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        case.run(og)
    for r in range(3):
        for o_ in og:
            o_.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert _equal(og, first), "%s: graph replay %d differs bitwise from eager" % (what, r)
    del g
    torch.cuda.synchronize()
    print("%s: %s" % (what, _geo_str(case.nslots) if case.det else "splits=%d" % case.nslots))


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _pos_mean(shape, g, dtype, spread=1.0):
    """1 + spread * randn: every CTA's partial is a visible share of the total"""
    return (1.0 + spread * torch.randn(shape, generator=g, device="cuda")).to(dtype)


def _d(t):
    return t.double()


_DT = {torch.float32: (_lib.F32, 4), torch.bfloat16: (_lib.BF16, 2)}


# ================================================================================================ row kernels (norm_tail.cu)
COL_STATS = [  # (dtype, B, HW, C, regime)
    (torch.bfloat16, 2, 10, 64, "R1"),
    (torch.bfloat16, 3, 100, 96, "R2"),
    (torch.bfloat16, 8, 3136, 64, "R3"),
    (torch.float32, 4, 196, 2048, "R3"),          # two column chunks of 1024: one scratch + ticket set per chunk
]


@pytest.mark.parametrize("dtype,B,HW,C,reg", COL_STATS)
def test_col_stats(dtype, B, HW, C, reg):
    code, es = _DT[dtype]
    nslots = rows_slots("flat", B, HW, C, es, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    g = _gen(B * HW + C)
    x = _pos_mean((B, HW, C), g, dtype)
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_col_stats(code, B, HW, C, x.data_ptr(), o[0].data_ptr(), o[1].data_ptr(), st), "col_stats")

    def reference(o):
        xd = _d(x).view(-1, C)
        return [(0, xd.sum(0), xd.abs().sum(0), True), (1, (xd * xd).sum(0), (xd * xd).sum(0), True)]

    run_case(Case(nslots, [((C,), torch.float32, PREFILL, True)] * 2, call, reference), "col_stats %s" % reg)


BN_BWD = [  # (two gradients, relu, dtype, B, HW, C, regime)
    (False, 0, torch.bfloat16, 1, 16, 64, "R1"),
    (False, 1, torch.bfloat16, 3, 100, 96, "R2"),
    (False, 2, torch.bfloat16, 8, 3136, 64, "R3"),
    (True, 1, torch.bfloat16, 8, 784, 128, "R3"),
    (True, 2, torch.float32, 4, 196, 2048, "R3"),   # column chunks
    (True, 0, torch.bfloat16, 2, 12, 256, "R1"),
]


@pytest.mark.parametrize("two,relu,dtype,B,HW,C,reg", BN_BWD)
def test_bn_bwd_sums(two, relu, dtype, B, HW, C, reg):
    code, es = _DT[dtype]
    nslots = rows_slots("flat", B, HW, C, es, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    g = _gen(B * HW + C + relu)
    dy = _pos_mean((B, HW, C), g, dtype)
    dy2 = _pos_mean((B, HW, C), g, dtype) if two else None
    x = _pos_mean((B, HW, C), g, dtype)
    y = _pos_mean((B, HW, C), g, dtype)               # relu 1: mask [y > 0] (about 84 % of the elements)
    scale = 0.5 + torch.rand(C, generator=g, device="cuda")
    shift = torch.randn(C, generator=g, device="cuda")
    mu = -0.5 + 0.1 * torch.randn(C, generator=g, device="cuda")   # not the batch mean: dz * xhat keeps a positive mean
    rstd = 0.6 + 0.4 * torch.rand(C, generator=g, device="cuda")
    lib = _lib.load()

    def call(o, st):
        args = (x.data_ptr(), y.data_ptr(), scale.data_ptr(), shift.data_ptr(), mu.data_ptr(), rstd.data_ptr(), relu,
                o[0].data_ptr(), o[1].data_ptr(), st)
        if two:
            rc = lib.cotb200_bn_bwd_sums2(code, B, HW, C, dy.data_ptr(), dy2.data_ptr(), *args)
        else:
            rc = lib.cotb200_bn_bwd_sums(code, B, HW, C, dy.data_ptr(), *args)
        _lib.check(rc, "bn_bwd_sums")

    def reference(o):
        dz = _d(dy) + (_d(dy2) if two else 0.0)
        xd = _d(x)
        if relu == 1:
            dz = dz * (_d(y) > 0)
        elif relu == 2:
            dz = dz * (xd * _d(scale) + _d(shift) > 0)    # the sign of the fp32 fma is the sign of the exact value
        xh = (xd - _d(mu)) * _d(rstd)
        xa = (xd.abs() + _d(mu).abs()) * _d(rstd)
        dz, xh, xa = dz.view(-1, C), xh.view(-1, C), xa.view(-1, C)
        return [(0, dz.sum(0), dz.abs().sum(0), True), (1, (dz * xh).sum(0), (dz.abs() * xa).sum(0), True)]

    run_case(Case(nslots, [((C,), torch.float32, PREFILL, True)] * 2, call, reference),
             "bn_bwd_sums%s relu=%d %s" % ("2" if two else "", relu, reg))


# The tail kernels compute y = silu(u*scale + shift) with an approximate sigmoid.  The sums are checked on terms whose value is
# exact: bf16 with scale = shift = 0 (z = 0, sigmoid = 0.5 exactly, y = 0), fp32 with z = u + 40 (sigmoid saturates to 1, y = z).
# The numerics of the sigmoid itself are covered by test_fused_gpu.
def _tail_inputs(dtype, B, HW, C, seed, with_k=True):
    g = _gen(seed)
    u = _pos_mean((B, HW, C), g, dtype)
    k = _pos_mean((B, HW, C), g, dtype) if with_k else None
    dout = _pos_mean((B, HW, C), g, dtype)
    if dtype == torch.bfloat16:
        scale, shift = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    else:
        scale, shift = torch.ones(C, device="cuda"), torch.full((C,), 40.0, device="cuda")
    return g, u, k, dout, scale, shift


def _tail_y(u, dtype):
    """(y, |y| bound, silu'(z)) of the exact-valued regimes above, fp64"""
    if dtype == torch.bfloat16:
        return torch.zeros_like(_d(u)), torch.zeros_like(_d(u)), 0.5
    z = _d(u) + 40.0
    return z, z.abs(), 1.0


TAIL_POOL = [  # (dtype, with k, B, HW, C, regime)
    (torch.bfloat16, True, 3, 20, 64, "R1"),        # three per-sample groups of one slot
    (torch.bfloat16, False, 16, 196, 64, "R2"),     # radix-1 form (k = NULL), 16 groups
    (torch.bfloat16, True, 4, 3136, 256, "R3"),
    (torch.float32, True, 3, 784, 128, "R3"),
]


@pytest.mark.parametrize("dtype,with_k,B,HW,C,reg", TAIL_POOL)
def test_tail_pool(dtype, with_k, B, HW, C, reg):
    code, es = _DT[dtype]
    nslots = rows_slots("sample", B, HW, C, es, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    _, u, k, _, scale, shift = _tail_inputs(dtype, B, HW, C, B + HW + C, with_k)
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_tail_pool(code, B, HW, C, u.data_ptr(), _lib.ptr(k), scale.data_ptr(), shift.data_ptr(),
                                         o[0].data_ptr(), st), "tail_pool")

    def reference(o):
        y, ya, _ = _tail_y(u, dtype)
        t = y + (_d(k) if with_k else 0.0)
        ta = ya + (_d(k).abs() if with_k else 0.0)
        return [(0, t.sum(1), ta.sum(1), True)]

    run_case(Case(nslots, [((B, C), torch.float32, PREFILL, True)], call, reference), "tail_pool %s" % reg)


TAIL_BWD = [  # (dtype, B, HW, C, regime)
    (torch.bfloat16, 5, 16, 64, "R1"),
    (torch.bfloat16, 64, 196, 64, "R2"),
    (torch.bfloat16, 4, 3136, 256, "R3"),
    (torch.float32, 3, 784, 128, "R3"),
]


@pytest.mark.parametrize("dtype,B,HW,C,reg", TAIL_BWD)
def test_tail_bwd_sums(dtype, B, HW, C, reg):
    code, es = _DT[dtype]
    nslots = rows_slots("sample", B, HW, C, es, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    _, u, k, dout, scale, shift = _tail_inputs(dtype, B, HW, C, 7 * B + HW + C)
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_tail_bwd_sums(code, B, HW, C, dout.data_ptr(), u.data_ptr(), k.data_ptr(), scale.data_ptr(),
                                             shift.data_ptr(), o[0].data_ptr(), st), "tail_bwd_sums")

    def reference(o):
        y, ya, _ = _tail_y(u, dtype)
        d = _d(dout)
        ref = torch.stack([(d * y).sum(1), (d * _d(k)).sum(1)], -1)
        absterms = torch.stack([(d.abs() * ya).sum(1), (d * _d(k)).abs().sum(1)], -1)
        return [(0, ref, absterms, True)]

    run_case(Case(nslots, [((B, C, 2), torch.float32, PREFILL, True)], call, reference), "tail_bwd_sums %s" % reg)


# R4: the shapes of the wide-fan path depend on the SM count (make_geo); the first candidate that reaches it is used.
DZ_R4_CANDIDATES = [(256, 100), (512, 49), (384, 49), (1024, 49)]


def _dz_shape(reg, C, es, sms):
    if reg != "R4":
        return {"R1": (1, 20), "R2": (2, 196), "R3": (8, 3136)}[reg]
    for B, HW in DZ_R4_CANDIDATES:
        if regime(rows_slots("grid", B, HW, C, es, sms)) == "R4":
            return B, HW
    raise AssertionError("no candidate shape reaches R4 on %d SMs" % sms)


@pytest.mark.parametrize("dtype,C,reg", [(torch.bfloat16, 64, "R1"), (torch.bfloat16, 128, "R2"), (torch.float32, 64, "R3"),
                                         (torch.bfloat16, 256, "R4")])
def test_tail_bwd_dz_sums(dtype, C, reg):
    code, es = _DT[dtype]
    B, HW = _dz_shape(reg, C, es, _sms())
    nslots = rows_slots("grid", B, HW, C, es, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    g, u, _, dout, scale, shift = _tail_inputs(dtype, B, HW, C, 11 * B + HW + C, with_k=False)
    mu = -0.5 + 0.1 * torch.randn(C, generator=g, device="cuda")
    rstd = 0.6 + 0.4 * torch.rand(C, generator=g, device="cuda")
    a = 0.5 + torch.rand(B, C, 2, generator=g, device="cuda")
    dpn = torch.rand(B, C, generator=g, device="cuda")
    pscale = 0.25
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_tail_bwd_dz_sums(code, B, HW, C, dout.data_ptr(), u.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                                                mu.data_ptr(), rstd.data_ptr(), a.data_ptr(), dpn.data_ptr(), pscale,
                                                o[0].data_ptr(), o[1].data_ptr(), st), "tail_bwd_dz_sums")

    def reference(o):
        _, _, ds = _tail_y(u, dtype)
        dz = (_d(a[:, None, :, 0]) * _d(dout) + _d(dpn[:, None, :]) * pscale) * ds
        dza = (_d(a[:, None, :, 0]) * _d(dout).abs() + _d(dpn[:, None, :]) * pscale) * ds
        xh = (_d(u) - _d(mu)) * _d(rstd)
        xa = (_d(u).abs() + _d(mu).abs()) * _d(rstd)
        return [(0, dz.sum((0, 1)), dza.sum((0, 1)), True), (1, (dz * xh).sum((0, 1)), (dza * xa).sum((0, 1)), True)]

    run_case(Case(nslots, [((C,), torch.float32, PREFILL, True)] * 2, call, reference),
             "tail_bwd_dz_sums %s B=%d HW=%d" % (reg, B, HW))


# ================================================================================================ GroupNorm over 9 taps
def _tap_pos(wc, gc):
    """storage position of reference column j = g*9 + t (gc > 0: tap-major chunks of gc weight channels)"""
    j = torch.arange(9 * wc, device="cuda")
    if gc <= 0:
        return j
    gi, t = j // 9, j % 9
    return ((gi // gc) * 9 + t) * gc + gi % gc


GN_STATS = [  # (wc, dtype, B, HW, regime): wc in {8, 16, 32, 64} takes the gn72 kernels, other widths the generic ones
    (16, torch.bfloat16, 3, 49, "R1"),
    (8, torch.bfloat16, 64, 784, "R2"),
    (16, torch.bfloat16, 2, 3136, "R3"),
    (16, torch.float32, 3, 3136, "R3"),
    (24, torch.bfloat16, 3, 20, "R1"),
    (24, torch.bfloat16, 16, 196, "R2"),
    (24, torch.bfloat16, 4, 784, "R3"),
]


@pytest.mark.parametrize("wc,dtype,B,HW,reg", GN_STATS)
def test_gn9_stats(wc, dtype, B, HW, reg):
    code, es = _DT[dtype]
    J = 9 * wc
    fast = gn72_ok(wc, 0, False)
    nslots = gn72_stats_slots(B, HW, wc, es, _sms()) if fast else rows_slots("sample", B, HW, J, es, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    g = _gen(B * HW + wc)
    l = _pos_mean((B, HW, J), g, dtype)
    lbias = 0.2 * torch.randn(J, generator=g, device="cuda")
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_gn9_stats(code, B, HW, wc, 0, l.data_ptr(), lbias.data_ptr(), o[0].data_ptr(), o[1].data_ptr(), st),
                   "gn9_stats")

    def reference(o):
        f = (_d(l) + _d(lbias)).view(B, HW, wc, 9)
        fa = (_d(l).abs() + _d(lbias).abs()).view(B, HW, wc, 9)
        return [(0, f.sum((1, 3)), fa.sum((1, 3)), True), (1, (f * f).sum((1, 3)), (fa * fa).sum((1, 3)), True)]

    run_case(Case(nslots, [((B, wc), torch.float32, PREFILL, True)] * 2, call, reference),
             "gn9_stats %s wc=%d %s" % ("gn72" if fast else "generic", wc, reg))


GN_BWD = [  # (wc, gc, dtype, B, HW, regime): gn72 needs gc == 8 and wc in {8, 16, 32, 64}
    (16, 8, torch.bfloat16, 3, 100, "R1"),
    (16, 8, torch.bfloat16, 3, 784, "R2"),
    (16, 8, torch.bfloat16, 2, 3136, "R3"),
    (8, 8, torch.float32, 3, 3136, "R3"),
    (16, 0, torch.bfloat16, 3, 20, "R1"),
    (16, 0, torch.bfloat16, 16, 196, "R2"),
    (16, 0, torch.bfloat16, 4, 784, "R3"),
    (24, 8, torch.bfloat16, 3, 784, "R3"),          # generic kernels with the tap-major storage order
]


@pytest.mark.parametrize("wc,gc,dtype,B,HW,reg", GN_BWD)
def test_gn9_bwd_sums(wc, gc, dtype, B, HW, reg):
    code, es = _DT[dtype]
    J = 9 * wc
    fast = gn72_ok(wc, gc, True)
    nslots = gn72_bwd_slots(HW, wc, es) if fast else rows_slots("sample", B, HW, J, es, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    g = _gen(B * HW + wc + gc)
    l = _pos_mean((B, HW, J), g, dtype)
    dg = _pos_mean((B, HW, J), g, dtype)           # storage order (gc)
    lbias = 0.2 * torch.randn(J, generator=g, device="cuda")
    mean = -0.5 + 0.1 * torch.randn(B, wc, generator=g, device="cuda")   # not the group mean: sums of dg*lhat keep a positive mean
    rstd = 0.6 + 0.4 * torch.rand(B, wc, generator=g, device="cuda")
    gamma = 0.5 + torch.rand(J, generator=g, device="cuda")
    lib = _lib.load()
    # outputs: work [B, 3, J] (documented as zeroed by the caller), s1, s2 [B, wc] (written), dgamma, dbeta, dlbias [J] (accumulated)
    nan = float("nan")
    outs = [((B, 3, J), torch.float32, 0.0, True), ((B, wc), torch.float32, nan, False), ((B, wc), torch.float32, nan, False),
            ((J,), torch.float32, PREFILL, True), ((J,), torch.float32, PREFILL, True), ((J,), torch.float32, PREFILL, True)]

    def call(o, st):
        _lib.check(lib.cotb200_gn9_bwd_sums(code, B, HW, wc, gc, dg.data_ptr(), l.data_ptr(), lbias.data_ptr(), mean.data_ptr(),
                                            rstd.data_ptr(), gamma.data_ptr(), *[t.data_ptr() for t in o], st), "gn9_bwd_sums")

    def reference(o):
        d = _d(dg)[:, :, _tap_pos(wc, gc)]                        # reference column order
        da = d.abs()
        ld = _d(l)
        gi = torch.arange(J, device="cuda") // 9
        mn = _d(mean)[:, gi][:, None, :] - _d(lbias)             # l + lbias - mean = l - mn
        rs = _d(rstd)[:, gi][:, None, :]
        mna = _d(mean).abs()[:, gi][:, None, :] + _d(lbias).abs()
        lh, lha = (ld - mn) * rs, (ld.abs() + mna) * rs
        D, Da = d.sum(1), da.sum(1)                               # [B, J]
        DL, DLa = (d * lh).sum(1), (da * lha).sum(1)
        LH, LHa = lh.sum(1), lha.sum(1)
        if fast:   # the gn72 kernel sums raw l; gn_bwd_finish applies mean / rstd analytically
            work = torch.stack([D, (d * ld).sum(1), ld.sum(1)], 1)
            work_a = torch.stack([Da, (da * ld.abs()).sum(1), ld.abs().sum(1)], 1)
        else:
            work, work_a = torch.stack([D, DL, LH], 1), torch.stack([Da, DLa, LHa], 1)
        ga = _d(gamma)
        s1, s1a = (D * ga).view(B, wc, 9).sum(-1), (Da * ga).view(B, wc, 9).sum(-1)
        s2, s2a = (DL * ga).view(B, wc, 9).sum(-1), (DLa * ga).view(B, wc, 9).sum(-1)
        n = 9.0 * HW
        rsj = _d(rstd)[:, gi]
        dlb = (rsj * (ga * D - HW * s1[:, gi] / n - s2[:, gi] / n * LH)).sum(0)
        dlba = (rsj * (ga * Da + HW * s1a[:, gi] / n + s2a[:, gi] / n * LHa)).sum(0)
        # the finish kernel re-derives sum dg*lhat and sum lhat from the raw sums (fast path): allow for that cancellation
        return [(0, work, work_a, True), (1, s1, s1a, False), (2, s2, s2a, False),
                (3, DL.sum(0), DLa.sum(0), False), (4, D.sum(0), Da.sum(0), False), (5, dlb, dlba, False)]

    run_case(Case(nslots, outs, call, reference), "gn9_bwd_sums %s wc=%d gc=%d %s" % ("gn72" if fast else "generic", wc, gc, reg))


# ================================================================================================ tensor-core epilogues
def _stats_ref(D, C):
    """column sums / sums of squares of the STORED bf16 output, fp64"""
    d = _d(D).reshape(-1, C)
    return [(1, d.sum(0), d.abs().sum(0), True), (2, (d * d).sum(0), (d * d).sum(0), True)]


GEMM = [  # (M, N, K1, K2, regime)
    (100, 64, 64, 0, "R1"),
    (1000, 64, 64, 0, "R2"),
    (25088, 64, 64, 0, "R3"),
    (3000, 192, 64, 64, "R3"),                      # two products, two N tiles of 128
    (6272, 256, 128, 128, "R3"),                    # one 256-column tile, one CTA per SM
]


@pytest.mark.parametrize("M,N,K1,K2,reg", GEMM)
def test_gemm_bf16_stats(M, N, K1, K2, reg):
    nslots = tc_grid(N, pick_bn(N, K1 + K2), _cdiv(M, TC_BM), True, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    g = _gen(M + N + K1 + K2)
    a1 = _pos_mean((M, K1), g, torch.bfloat16)
    b1 = _pos_mean((N, K1), g, torch.float32).div_(K1 + K2).bfloat16()
    a2 = _pos_mean((M, K2), g, torch.bfloat16) if K2 else None
    b2 = _pos_mean((N, K2), g, torch.float32).div_(K1 + K2).bfloat16() if K2 else None
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_gemm_bf16(M, N, K1, a1.data_ptr(), K1, b1.data_ptr(), K1, K2, _lib.ptr(a2), K2, _lib.ptr(b2), K2,
                                         o[0].data_ptr(), N, None, None, 0, o[1].data_ptr(), o[2].data_ptr(), st), "gemm_bf16")

    outs = [((M, N), torch.bfloat16, float("nan"), False), ((N,), torch.float32, PREFILL, True), ((N,), torch.float32, PREFILL, True)]
    run_case(Case(nslots, outs, call, lambda o: _stats_ref(o[0], N)), "gemm_bf16 stats %s" % reg)


CONV = [  # (B, H, W, C, groups, regime)
    (1, 8, 8, 64, 4, "R1"),                         # haloed-tile kernel, one work item
    (8, 14, 14, 128, 1, "R2"),                      # N tile 128: conv mode of the GEMM kernel
    (4, 56, 56, 64, 4, "R3"),                       # haloed-tile kernel
    (4, 28, 28, 128, 4, "R3"),                      # haloed-tile kernel, two N tiles: zeros in the other tile's columns
]


@pytest.mark.parametrize("B,H,W,C,groups,reg", CONV)
def test_conv3x3_bf16_stats(B, H, W, C, groups, reg):
    from cotnet_b200 import tc
    cg = C // groups
    g = _gen(B + H + C + groups)
    x = _pos_mean((B, H, W, C), g, torch.bfloat16)
    w = _pos_mean((C, cg, 3, 3), g, torch.float32).div_(9 * cg).bfloat16()
    wp, bn = tc.prepare_conv3x3_weight(w, groups)
    path, nslots = conv3x3_slots(B, H, W, C, bn, _sms())
    assert regime(nslots) == reg, (path, _geo_str(nslots))
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_conv3x3_bf16(B, H, W, C, x.data_ptr(), C, wp.data_ptr(), bn, o[0].data_ptr(), C, None, None, 0,
                                            o[1].data_ptr(), o[2].data_ptr(), st), "conv3x3_bf16")

    outs = [((B, H, W, C), torch.bfloat16, float("nan"), False), ((C,), torch.float32, PREFILL, True), ((C,), torch.float32, PREFILL, True)]
    run_case(Case(nslots, outs, call, lambda o: _stats_ref(o[0], C)), "conv3x3_bf16 stats (%s) %s" % (path, reg))


@pytest.mark.parametrize("B,H,W,N,reg", [(1, 32, 32, 64, "R2"), (2, 64, 64, 64, "R3"), (2, 96, 64, 32, "R3")])
def test_stem7x7s2_stats(B, H, W, N, reg):
    from cotnet_b200 import tc
    nslots = stem_slots(B, H, W, N, _sms())
    assert regime(nslots) == reg, _geo_str(nslots)
    g = _gen(B + H + W + N)
    x = _pos_mean((B, H, W, 3), g, torch.bfloat16)
    wm = tc.prepare_stem_weight(_pos_mean((N, 3, 7, 7), g, torch.float32).div_(147).bfloat16())
    lib = _lib.load()
    scratch = torch.empty(int(lib.cotb200_stem7x7s2_scratch_bytes(B, H, W)), dtype=torch.uint8, device="cuda")

    def call(o, st):
        _lib.check(lib.cotb200_stem7x7s2_bf16(B, H, W, x.data_ptr(), wm.data_ptr(), N, o[0].data_ptr(), N, None, None, 0,
                                              o[1].data_ptr(), o[2].data_ptr(), scratch.data_ptr(), st), "stem7x7s2_bf16")

    outs = [((B, H // 2, W // 2, N), torch.bfloat16, float("nan"), False), ((N,), torch.float32, PREFILL, True),
            ((N,), torch.float32, PREFILL, True)]
    run_case(Case(nslots, outs, call, lambda o: _stats_ref(o[0], N)), "stem7x7s2 stats %s" % reg)


# ================================================================================================ split-K weight gradients
WGRAD = [  # (M, R, C1, C2, transpose, split regime)
    (200, 64, 64, 0, 0, "splits=1"),
    (200, 64, 64, 0, 1, "splits=1"),
    (8192, 64, 128, 0, 0, "splits>1"),
    (8192, 128, 64, 0, 1, "splits>1"),
    (4096, 64, 64, 64, 0, "splits>1"),              # two B operands
]


@pytest.mark.parametrize("M,R,C1,C2,transpose,reg", WGRAD)
def test_wgrad_bf16_split_sums(M, R, C1, C2, transpose, reg):
    Cc = C1 + C2
    splits = wgrad_splits(M, R, Cc, _sms())
    assert (splits == 1) == (reg == "splits=1"), splits
    g = _gen(M + R + C1 + C2 + transpose)
    A = _pos_mean((M, R), g, torch.bfloat16)
    B1 = _pos_mean((M, C1), g, torch.bfloat16)
    B2 = _pos_mean((M, C2), g, torch.bfloat16) if C2 else None
    shape = (Cc, R) if transpose else (R, Cc)
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_wgrad_bf16(M, R, A.data_ptr(), R, C1, B1.data_ptr(), C1, C2, _lib.ptr(B2), C2, o[0].data_ptr(),
                                          shape[1], transpose, st), "wgrad_bf16")

    def reference(o):
        Bm = torch.cat([B1, B2], 1) if C2 else B1
        ref, refa = _d(A).t() @ _d(Bm), _d(A).abs().t() @ _d(Bm).abs()
        return [(0, ref.t() if transpose else ref, refa.t() if transpose else refa, True)]

    case = Case(splits, [(shape, torch.float32, PREFILL, True)], call, reference, det=False)
    run_case(case, "wgrad_bf16 transpose=%d %s (%d splits)" % (transpose, reg, splits))


@pytest.mark.parametrize("B,H,W,N,reg", [(1, 2, 32, 64, "splits=1"), (2, 64, 64, 64, "splits>1"), (3, 32, 96, 32, "splits>1")])
def test_stem7x7s2_wgrad_split_sums(B, H, W, N, reg):
    from cotnet_b200 import tc
    splits = stem_wgrad_splits(B, H, _sms())
    assert (splits == 1) == (reg == "splits=1"), splits
    g = _gen(B + H + W + N)
    x = _pos_mean((B, 3, H, W), g, torch.bfloat16).contiguous(memory_format=torch.channels_last)
    wm = tc.prepare_stem_weight(_pos_mean((N, 3, 7, 7), g, torch.float32).div_(147).bfloat16())
    _, scratch = tc.stem7x7s2_bf16(x, wm, return_scratch=True)
    Hh, Wh = H // 2, W // 2
    dy = _pos_mean((B * Hh * Wh, N), g, torch.bfloat16)
    lib = _lib.load()

    def call(o, st):
        _lib.check(lib.cotb200_stem7x7s2_wgrad_bf16(B, H, W, dy.data_ptr(), N, N, scratch.data_ptr(), o[0].data_ptr(), st),
                   "stem7x7s2_wgrad_bf16")

    def reference(o):
        # windows of the space-to-depth image [B, Hh, Wh + 4, 16]: output pixel (oh, ow), tap row a -> image row oh - 2 + a
        # (zero outside), cells ow .. ow + 3 (64 values)
        P = _d(scratch.view(torch.bfloat16).view(B, Hh, Wh + 4, 16))
        Pp = torch.nn.functional.pad(P, (0, 0, 0, 0, 2, 1))
        win = torch.stack([torch.stack([Pp[:, a:a + Hh, c:c + Wh, :] for c in range(4)], 3).reshape(B, Hh, Wh, 64)
                           for a in range(4)], 3).reshape(B * Hh * Wh, 256)
        return [(0, _d(dy).t() @ win, _d(dy).abs().t() @ win.abs(), True)]

    case = Case(splits, [((N, 256), torch.float32, PREFILL, True)], call, reference, det=False)
    run_case(case, "stem7x7s2_wgrad %s (%d splits)" % (reg, splits))


# ================================================================================================ two reductions on forked streams
def test_graph_with_forked_reductions():
    """One captured graph, two reducing calls on forked streams (each with its own scratch and tickets); every replay is
    bit-identical to the eager results."""
    lib = _lib.load()
    g = _gen(5)
    B, HW, C = 8, 3136, 64
    x = _pos_mean((B, HW, C), g, torch.bfloat16)
    l = _pos_mean((2, 3136, 144), g, torch.bfloat16)
    lbias = 0.2 * torch.randn(144, generator=g, device="cuda")

    def calls(o, st_a, st_b):
        _lib.check(lib.cotb200_col_stats(_lib.BF16, B, HW, C, x.data_ptr(), o[0].data_ptr(), o[1].data_ptr(), st_a), "col_stats")
        _lib.check(lib.cotb200_gn9_stats(_lib.BF16, 2, 3136, 16, 0, l.data_ptr(), lbias.data_ptr(), o[2].data_ptr(), o[3].data_ptr(),
                                         st_b), "gn9_stats")

    def outs():
        return [torch.full((C,), PREFILL, device="cuda"), torch.full((C,), PREFILL, device="cuda"),
                torch.full((2, 16), PREFILL, device="cuda"), torch.full((2, 16), PREFILL, device="cuda")]

    eager = outs()
    st = torch.cuda.current_stream().cuda_stream
    calls(eager, st, st)
    torch.cuda.synchronize()
    og = outs()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        main = torch.cuda.current_stream()
        for o_ in og:
            o_.fill_(PREFILL)
        side = torch.cuda.Stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            _lib.check(lib.cotb200_gn9_stats(_lib.BF16, 2, 3136, 16, 0, l.data_ptr(), lbias.data_ptr(), og[2].data_ptr(),
                                             og[3].data_ptr(), side.cuda_stream), "gn9_stats")
        _lib.check(lib.cotb200_col_stats(_lib.BF16, B, HW, C, x.data_ptr(), og[0].data_ptr(), og[1].data_ptr(), main.cuda_stream),
                   "col_stats")
        main.wait_stream(side)
    for r in range(3):
        for o_ in og:
            o_.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert _equal(og, eager), "forked graph replay %d differs bitwise from eager" % r


# ================================================================================================ model level
@pytest.fixture
def deterministic_cudnn():
    """cuDNN on heuristically chosen, deterministic algorithms (as bench.py runs it)"""
    old = (torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic)
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = old


TS_KW = dict(lr=0.002, momentum=0.9, weight_decay=1e-3, nesterov=True, ema_decay=0.99, amp_dtype=torch.bfloat16, weights="bf16")
WARMUP, STEPS = 2, 3


def _model_and_batch(mode):
    """the small CoT network of test_trainer_gpu; `train` switches its BatchNorms to batch statistics (the column-sum kernels)"""
    from test_trainer_gpu import _small_model
    m = _small_model().train(mode == "train")
    g0 = torch.Generator().manual_seed(6)
    x = torch.randn(8, 3, 96, 96, generator=g0).cuda().to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (8,), generator=g0).cuda()
    return m, x, y


def _state(ts, losses):
    st = {"loss": torch.stack([l_.detach().float().reshape(()) for l_ in losses])}
    for kind, d in (("master", ts.master_state()), ("grad", ts.grads()), ("ema", ts.ema_state())):
        for n, t in d.items():
            st["%s:%s" % (kind, n)] = t.detach().clone()
    for n in ("M_big", "M_small"):
        st["momentum:" + n] = getattr(ts, n).clone()
    for n, b in ts.model.named_buffers():                   # BatchNorm running statistics (train mode)
        st["buffer:" + n] = b.detach().clone()
    return st


def _run_eager(m0, x, y):
    from cotnet_b200 import trainer
    ts = trainer.TrainStep(copy.deepcopy(m0), **TS_KW)
    for _ in range(WARMUP):
        ts.step_eager(x, y)
    losses = [ts.step_eager(x, y).clone() for _ in range(STEPS)]
    torch.cuda.synchronize()
    return _state(ts, losses)


def _run_graph(m0, x, y):
    from cotnet_b200 import trainer
    ts = trainer.TrainStep(copy.deepcopy(m0), **TS_KW)
    info = ts.capture(x, y, warmup=WARMUP)
    assert info["cuda_graph"]
    losses = [ts.step(x, y).clone() for _ in range(STEPS)]
    torch.cuda.synchronize()
    return _state(ts, losses)


def _first_difference(a, b):
    for k in a:
        if not torch.equal(a[k], b[k]):
            return k
    return None


@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("pair", ["eager-eager", "graph-graph", "graph-eager"])
def test_train_step_bitwise_reproducible(pair, mode, deterministic_cudnn):
    """Three bf16 training steps (after the same warm-up steps) from the same state and batch: loss, gradients, master weights,
    momentum and EMA are bitwise equal between two eager TrainSteps, two separately captured graphs, and graph against eager."""
    m0, x, y = _model_and_batch(mode)
    run = {"eager": _run_eager, "graph": _run_graph}
    ka, kb = pair.split("-")
    sa = run[ka](m0, x, y)
    sb = run[kb](m0, x, y)
    assert sa.keys() == sb.keys()
    diff = _first_difference(sa, sb)
    assert diff is None, "%s: first tensor that differs bitwise: %s" % (pair, diff)
