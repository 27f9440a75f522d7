"""A minimal stand-in for CuPy so that the REFERENCE's own operator code (cupy_layers/*.py, unmodified) runs its own CUDA
kernels on the GPU box.  TEST / MEASUREMENT INFRASTRUCTURE ONLY (tools/bench_reference_gpu.py, tests).

The reference touches exactly two CuPy entry points (cupy_layers/utils.py:14-18):
    @cupy.memoize(for_each_device=True)           -> a per-(device, arguments) memo decorator
    cupy.cuda.compile_with_cache(code)            -> NVRTC compile of the substituted kernel source; .get_function(name)
and launches the returned function as  f(block=(..), grid=(..), args=[ptr, ...], stream=Stream(ptr=...))
(cupy_layers/aggregation_zeropad.py:140-143).  Here the compile step is `nvcc -cubin -arch=sm_90a` (NVRTC and nvcc share
the front end; the image has no CuPy) and the launch goes through the CUDA driver API with ctypes.  The kernel SOURCE is
the reference's string, untouched; it lives only in a temporary directory.
"""
import ctypes
import os
import subprocess
import sys
import tempfile
import types

import torch

_cu = None


def _driver():
    global _cu
    if _cu is None:
        _cu = ctypes.CDLL("libcuda.so.1")
    return _cu


def _check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed with CUresult %d" % (what, rc))


class _Function:
    def __init__(self, mod, name):
        self.fn = ctypes.c_void_p()
        _check(_driver().cuModuleGetFunction(ctypes.byref(self.fn), mod, name.encode()), "cuModuleGetFunction")

    def __call__(self, block, grid, args, stream=None):
        vals = [ctypes.c_void_p(int(a)) for a in args]
        argv = (ctypes.c_void_p * len(vals))(*[ctypes.cast(ctypes.pointer(v), ctypes.c_void_p) for v in vals])
        st = ctypes.c_void_p(getattr(stream, "ptr", 0) or 0)
        _check(_driver().cuLaunchKernel(self.fn, grid[0], grid[1], grid[2], block[0], block[1], block[2], 0, st, argv, None),
               "cuLaunchKernel")


class _Module:
    def __init__(self, cubin):
        self.blob = cubin
        self.mod = ctypes.c_void_p()
        torch.zeros(1, device="cuda")                                  # torch's primary context is current
        _check(_driver().cuModuleLoadData(ctypes.byref(self.mod), cubin), "cuModuleLoadData")

    def get_function(self, name):
        return _Function(self.mod, name)


def compile_with_cache(code):
    with tempfile.TemporaryDirectory() as td:
        src, dst = os.path.join(td, "k.cu"), os.path.join(td, "k.cubin")
        open(src, "w").write(code)
        subprocess.run(["nvcc", "-cubin", "-arch=sm_90a", "-O3", "-o", dst, src], check=True, capture_output=True)
        return _Module(open(dst, "rb").read())


def memoize(for_each_device=False):
    def deco(f):
        memo = {}

        def wrapped(*a, **k):
            key = (torch.cuda.current_device() if for_each_device else -1, a, tuple(sorted(k.items())))
            if key not in memo:
                memo[key] = f(*a, **k)
            return memo[key]
        return wrapped
    return deco


def install():
    """Put the stand-in into sys.modules as `cupy` (refuses to shadow a real CuPy)."""
    if "cupy" in sys.modules and not getattr(sys.modules["cupy"], "_cotb200_shim", False):
        raise RuntimeError("a real cupy is already imported")
    m = types.ModuleType("cupy")
    m._cotb200_shim = True
    m.memoize = memoize
    m.cuda = types.SimpleNamespace(compile_with_cache=compile_with_cache)
    sys.modules["cupy"] = m
    return m
