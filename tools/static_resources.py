#!/usr/bin/env python
"""Per-kernel registers / spills / static shared memory from `ptxas -v` for every kernel of libcotb200 (bf16 and fp32
instantiations of the widest vector width), written as a markdown table.  Needs nvcc only (no GPU).

    python tools/static_resources.py profiles/r01_static_resources.md"""
import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cotnet_b200", "csrc")


def demangle(names):
    p = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return p.stdout.splitlines()


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "r01_static_resources.md")
    rows = []
    for src in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        p = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                            "-Xptxas", "-v", "-c", "-o", "/dev/null", src], capture_output=True, text=True)
        text = p.stderr
        for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'\n[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                             r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers(?:, used (\d+) barriers)?(?:, (\d+) bytes smem)?", text):
            rows.append((os.path.basename(src), m.group(1), int(m.group(5)), int(m.group(3)) + int(m.group(4)), int(m.group(7) or 0)))
    names = demangle([r[1] for r in rows])
    keep = []
    for (src, _, regs, spill, smem), dn in zip(rows, names):
        short = re.sub(r"^void ", "", dn)
        short = re.sub(r"\(.*", "", short).replace("cotb200::", "")
        if "double" in short or "__half" in short:
            continue
        # widest vector instantiation only: <T, 8, ...> for bf16, <T, 4, ...> for float, or kernels without a VEC parameter
        m = re.match(r"(\w+)<(__nv_bfloat16|float)(?:, \(int\)(\d+))?", short)
        if m and m.group(3) is not None:
            vec = int(m.group(3))
            if (m.group(2) == "__nv_bfloat16" and vec not in (8, 4)) or (m.group(2) == "float" and vec not in (4,)):
                continue
        keep.append((src, short.replace("(int)", "").replace("(bool)", ""), regs, spill, smem))
    with open(out, "w") as f:
        f.write("# static resources of the libcotb200 kernels (`ptxas -v`, sm_90a; bf16 / fp32 instantiations)\n\n")
        f.write("65 536 registers and 227 KB of shared memory per SM: `regs x threads` bounds the resident CTAs of the register-heavy\n"
                "kernels (LocalConv gen 2, fused NCHW backward), dynamic shared memory those of the TMA / bulk-copy pipelines.\n\n")
        f.write("| source | kernel | registers | spill bytes | static smem |\n|---|---|---|---|---|\n")
        for src, short, regs, spill, smem in sorted(keep):
            f.write("| %s | `%s` | %d | %d | %d |\n" % (src, short[:110], regs, spill, smem))
    print(out, len(keep), "kernels")


if __name__ == "__main__":
    main()
