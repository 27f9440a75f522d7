"""Build libcotb200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m cotnet_b200.build [--force] [--verbose]

The shared library is the C-ABI boundary declared in include/cotb200.h; it links only the CUDA
runtime (static) -- no torch, no cuBLAS/cuDNN.  The .so is a git-ignored build product.
"""
import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libcotb200.so")

def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(os.path.dirname(HERE), "include", "cotb200.h")]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into cotnet_b200/libcotb200.so.  Returns the path."""
    if not force and not _stale():
        return OUT
    nvcc = _nvcc()
    if nvcc is None:
        if os.path.exists(OUT):
            return OUT  # no toolchain: use the library built earlier
        raise RuntimeError("nvcc not found and no prebuilt libcotb200.so present")
    objs = []
    tmp = os.path.join(HERE, "build")
    os.makedirs(tmp, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(tmp, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(
                [os.path.getmtime(src)] + [os.path.getmtime(p) for p in glob.glob(os.path.join(CSRC, "*.cuh"))]
                + [os.path.getmtime(os.path.join(os.path.dirname(HERE), "include", "cotb200.h"))]):
            continue
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
               "-Xcompiler", "-fPIC", "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out))
    link = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static", "-o", OUT] + objs
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s" % r.stdout)
    return OUT


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
