"""The block geometry of the deterministic cross-CTA reductions (det_fan / det_blocks / det_floats in csrc/common.cuh), checked on
the real header: a host-only program compiled with nvcc walks every slot count from 1 to 2^20."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NMAX = 1 << 20

HARNESS = r"""
#include "common.cuh"
#include <cstdio>
using namespace cotb200;
int main() {
  long long bad = 0;
  int prev_fan = -1, prev_blk = -1;
  for (int n = 1; n <= %(nmax)d; ++n) {
    const int fan = det_fan(n), blk = det_blocks(n);
    const char* why = nullptr;
    if (fan < 16) why = "fan below 16";
    else if (blk < 1 || 1 + blk > DET_TICKETS_PER_GROUP) why = "more blocks than first-level tickets";
    else if ((long long)blk * fan < n) why = "blocks do not cover the slots";
    else if ((long long)(blk - 1) * fan >= n) why = "last block empty";
    else if (det_floats(n, 1) != (size_t)n + blk || det_floats(n, 3) != 3 * ((size_t)n + blk)) why = "scratch misses rows";
    else if ((n - 1) / fan != blk - 1) why = "last slot outside the last block";
    if (why) { if (bad < 8) printf("FAIL %%d fan=%%d blocks=%%d: %%s\n", n, fan, blk, why); ++bad; }
    if (fan != prev_fan || blk != prev_blk) { printf("G %%d %%d %%d\n", n, fan, blk); prev_fan = fan; prev_blk = blk; }
  }
  printf("DONE %%lld\n", bad);
  return bad != 0;
}
"""


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def header_geometry(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("det_geometry")
    src, exe = str(d / "harness.cu"), str(d / "harness")
    with open(src, "w") as f:
        f.write(HARNESS % {"nmax": NMAX})
    cc = subprocess.run([nvcc, "-std=c++17", "-O2", "-I", os.path.join(ROOT, "cotnet_b200", "csrc"), src, "-o", exe],
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    run = subprocess.run([exe], capture_output=True, text=True)
    return run.returncode, run.stdout


def test_blocks_partition_every_slot_count(header_geometry):
    """fan >= 16; at most 63 blocks, so 1 + block index stays inside the 64 tickets of a group; the blocks partition [0, nslots)
    with a non-empty last block; det_floats holds the nslots rows and the block totals."""
    rc, out = header_geometry
    fails = [ln for ln in out.splitlines() if ln.startswith("FAIL")]
    assert rc == 0 and not fails and "DONE 0" in out, "\n".join(fails[:8]) or out[-400:]


def test_python_copy_matches_header(header_geometry):
    """det_fan / det_blocks as copied into tests/test_determinism_gpu.py (its regime labels rest on them) agree with the header at
    every slot count, and the wide fan starts right after 16 * 63 = 1008 slots."""
    from test_determinism_gpu import det_blocks, det_fan
    _, out = header_geometry
    runs = [tuple(int(v) for v in ln.split()[1:]) for ln in out.splitlines() if ln.startswith("G ")]
    assert runs and runs[0] == (1, 16, 1)
    bounds = [n for n, _, _ in runs] + [NMAX + 1]
    for (n0, fan, blk), n1 in zip(runs, bounds[1:]):
        for n in range(n0, n1):
            assert (det_fan(n), det_blocks(n)) == (fan, blk), n
    assert det_fan(1008) == 16 and det_fan(1009) == 17
    assert (det_fan(1024), det_blocks(1024), 1024 - 60 * 17) == (17, 61, 4)
