"""The launch plans copied into tests/test_persistent_gpu.py, checked without a GPU: the constants they rest on match the CUDA sources,
and every case of that file reaches its regime (every ring stage reused at both phase parities, a ragged last round, the case's
feature) on both H100 SM counts within the per-case memory budget."""
import os
import re

import pytest

import test_persistent_gpu as tp

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cotnet_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _const(text, name):
    m = re.search(r"static constexpr int %s = (\d+);" % name, text)
    assert m, name
    return int(m.group(1))


def test_tc_gemm_constants():
    s = _src("tc_gemm.cu")
    assert (_const(s, "TC_BM"), _const(s, "TC_BK"), _const(s, "TC_STAGES")) == (tp.TC_BM, tp.TC_BK, tp.TC_STAGES)
    # tc_launch: two CTAs per SM under 104 KB, else one under 200 KB; the statistics smem; the grid of resident CTAs
    for snippet in ("p.stages = (104 * 1024 - out_bytes) / stage_bytes;", "if (p.stages < 2 || p.bn > 128) {",
                    "p.stages = (200 * 1024 - out_bytes) / stage_bytes;", "2 * 4 * 256 * 4 + 2 * p.N * 4",
                    "int grid = per_sm * num_sms();", "p.bn = pick_bn(N, K1 + K2);", "p.bn = pick_bn_wide(N); p.mode = 2;"):
        assert snippet in s, snippet
    # conv3x3_halo_launch: the 256-pixel cap, its 4 stages, the 220 KB budget, the grid bound to whole N-tile sets
    assert "static constexpr int HC_WBYTES = 9 * 64 * 128;" in s
    for snippet in ("r * Wpad <= maxpx && r * W <= 256", "const int maxpx = 256;", "if (p.stages > 4) p.stages = 4;",
                    "p.stages = (220 * 1024 - HC_WBYTES - out_bytes) / p.a_stage_bytes;",
                    "int grid = (num_sms() / p.n_tiles) * p.n_tiles;", "while (H % hb) --hb;"):
        assert snippet in s, snippet


def test_tma_localconv_constants():
    s = _src("agg_tma.cu")
    assert _const(s, "AT_MAX_STAGES") == tp.AT_MAX_STAGES
    for snippet in ("if (xb + bb > 72 * 1024) break;", "th * a.W * CQ > 2 * 896", "if ((long long)th * a.W * CQ >= 896) break;",
                    "p.stages = (int)((200 * 1024) / p.stage_bytes);", "L.grid = num_sms();", "p.whalo = mode == 1 ? 1 : 0;"):
        assert snippet in s, snippet
    n = _src("agg_nchw_tma.cu")
    assert (_const(n, "NT_MAX_STAGES"), _const(n, "NT_COMPUTE_THREADS")) == (tp.NT_MAX_STAGES, tp.NT_COMPUTE_THREADS)
    for snippet in ("const int budget = 200 * 1024;", "for (int th = 1; th <= H && th <= 32; ++th) {", "if (stage * 2 > budget) break;",
                    "p.total_tiles = N * wc * p.bands;", "int grid = num_sms();"):
        assert snippet in n, snippet


def test_wgrad_and_gn72_constants():
    w = _src("tc_wgrad.cu")
    assert _const(w, "WG_STAGES") == tp.WG_STAGES
    for snippet in ("int splits = num_sms();", "const int stage_bytes = 6 * box_bytes;", "p.stages = (216 * 1024) / stage_bytes;"):
        assert snippet in w, snippet
    g = _src("gn72.cu")
    for snippet in ("int X = (4 * num_sms() + B - 1) / B;", "if (X > ntiles) X = ntiles;",
                    "static constexpr int TB = sizeof(T) == 2 ? 256 : 128;",
                    "if (tid == 0 && tile + (int)gridDim.x < ntiles) issue(tile + gridDim.x, stage ^ 1);"):
        assert snippet in g, snippet


@pytest.mark.parametrize("sms", tp.SMS_H100)
@pytest.mark.parametrize("sizes,case", tp.ALL_CASES, ids=lambda v: v.__name__ if callable(v) else "-".join(str(e) for e in v))
def test_every_case_reaches_its_regime(sizes, case, sms):
    plans, sz = sizes(case, sms)
    assert plans
    for p in plans:
        assert not p.problems(), "%s: %s" % (p, p.problems())
        assert p.wraps >= 2, str(p)
    assert sz["mem"] < tp.MEM_LIMIT, (case, sz)


def test_plans_against_known_geometry():
    """hand-checked anchors on 132 SMs: the stage-1 TMA LocalConv of the bench (bs256: 256 x 28 bands on 132 CTAs, 4 stages) and
    the stage-1 1x1 GEMM (M = 802816, N = 64, K = 64: 6272 row tiles on 264 CTAs)"""
    p = tp.at_plan(0, 2, 256, 64, 56, 56, 8, 132)
    assert (p.info["TH"], p.info["bands"], p.stages, p.grid, p.total) == (2, 28, 4, 132, 7168)
    bn = tp.pick_bn(64, 64)
    p = tp.tc_launch("tc_gemm_1x1", 64, bn, 802816 // 128, 1, False, 132)
    assert (p.grid, p.total, p.max_tiles) == (264, 6272, 24)
    p = tp.tc_launch("tc_gemm_1x1", 640, tp.pick_bn(640, 128), 10, 2, False, 132)
    assert p.info["n_tiles"] == 5 and p.info["bn"] == 128
