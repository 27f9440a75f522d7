"""CPU-side checks of the C-ABI boundary: the library builds/loads, exports every symbol declared in
include/cotb200.h, and rejects bad arguments with the documented codes (no kernel is launched)."""
import ctypes
import os
import re

import pytest

from cotnet_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "cotb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cotb200_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    declared = _declared_symbols()
    assert declared, "no symbols parsed from the header"
    for name in declared:
        assert hasattr(lib, name), "libcotb200.so does not export %s" % name
    # and the Python binding table covers the header exactly
    assert sorted(_lib.SYMBOLS) == declared


def test_version_and_struct_size():
    lib = _lib.load()
    assert lib.cotb200_version() == 100
    assert ctypes.sizeof(_lib.AggDesc) == 20 * 4 + 6 * 8


def _desc(**kw):
    d = _lib.AggDesc()
    base = dict(n=2, c=8, h=9, w=9, heads=1, wc=4, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1, dh=1, dw=1, ho=9, wo=9,
                dtype=_lib.F32, layout=_lib.NCHW)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw,code", [
    (dict(c=7), -1),            # c % wc != 0           (aggregation_zeropad.py:189)
    (dict(ho=8), -1),           # Ho*Wo mismatch        (aggregation_zeropad.py:122)
    (dict(n=0), -1),
    (dict(layout=9), -3),
])
def test_argument_errors(kw, code):
    lib = _lib.load()
    rc = lib.cotb200_agg_zeropad_fwd(_desc(**kw), 16, 16, 16, None)
    assert rc == code
    assert lib.cotb200_last_error()


def test_null_pointer_and_dtype_errors():
    lib = _lib.load()
    assert lib.cotb200_agg_zeropad_fwd(_desc(), None, 16, 16, None) == -5
    assert lib.cotb200_agg_zeropad_fwd(_desc(dtype=11), 16, 16, 16, None) == -2
    assert lib.cotb200_agg_zeropad_mix_fwd(_desc(layout=_lib.NHWC), 5, 5, 2, 2, 16, 16, 16, 16, None) == -3
    with pytest.raises(RuntimeError):
        _lib.check(-1, "unit")


def test_ops_refuse_cpu_tensors_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cotnet_b200 import aggregation_zeropad
    x = torch.randn(1, 4, 5, 5)
    w = torch.randn(1, 1, 2, 9, 5, 5)
    with pytest.raises(RuntimeError, match="no CPU implementation"):
        aggregation_zeropad(x, w, 3, 1, 1, 1)


def test_row_kernel_argument_errors():
    """Argument validation of the normalisation / fan-in entry points (returns before any CUDA call)."""
    lib = _lib.load()
    P = 16          # any non-NULL "pointer": these calls must fail in validation, nothing is dereferenced
    ENULL, EINVAL, EDTYPE = -5, -1, -2
    # sum_rows: NULL operands, a third source without the second, pitch smaller than the row, fp64
    assert lib.cotb200_sum_rows(_lib.BF16, 10, 8, None, 8, P, 8, None, 0, None, 0, P, 8, None) == ENULL
    assert lib.cotb200_sum_rows(_lib.BF16, 10, 8, P, 8, P, 8, None, 0, P, 8, P, 8, None) == EINVAL
    assert lib.cotb200_sum_rows(_lib.BF16, 10, 8, P, 4, P, 8, None, 0, None, 0, P, 8, None) == EINVAL
    assert lib.cotb200_sum_rows(_lib.BF16, 10, 8, P, 8, P, 8, None, 0, None, 0, P, 4, None) == EINVAL
    assert lib.cotb200_sum_rows(_lib.F64, 10, 8, P, 8, P, 8, None, 0, None, 0, P, 8, None) == EDTYPE
    # GroupNorm(9 taps): chunk width must divide the weight channels; bwd_sums needs its workspace
    assert lib.cotb200_gn9_stats(_lib.BF16, 2, 9, 12, 8, P, None, P, P, None) == EINVAL
    assert lib.cotb200_gn9_apply(_lib.BF16, 2, 9, 12, 8, P, None, P, P, P, P, P, None) == EINVAL
    assert lib.cotb200_gn9_bwd_sums(_lib.BF16, 2, 9, 16, 8, P, P, None, P, P, P, None, P, P, P, P, None, None) == ENULL
    assert lib.cotb200_last_error()


def test_bn_argument_errors():
    """Argument validation of the BatchNorm entry points (returns before any CUDA call)."""
    lib = _lib.load()
    P = 16          # any non-NULL "pointer": these calls must fail in validation, nothing is dereferenced
    ENULL, EINVAL, EDTYPE = -5, -1, -2
    # BatchNorm backward: relu code 1 needs y, code 2 needs scale AND shift, code 3 needs the mask, a mask needs code 3, other
    # codes are rejected
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 1, 4, 8, P, P, None, None, P, P, P, P, 1, P, P, None, None) == ENULL
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 1, 4, 8, P, P, None, None, P, None, P, P, 2, P, P, None, None) == ENULL
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 1, 4, 8, P, P, P, None, P, P, P, P, 3, P, P, None, None) == ENULL
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 1, 4, 8, P, P, P, P, P, P, P, P, 1, P, P, None, None) == EINVAL
    assert lib.cotb200_bn_bwd_sums(_lib.BF16, 1, 4, 8, P, P, P, None, P, P, P, P, 4, P, P, None, None) == EINVAL
    assert lib.cotb200_bn_bwd_apply(_lib.BF16, 1, 4, 8, P, P, None, None, P, None, P, P, None, None, 0.25, 2, P, None, None,
                                    None) == ENULL
    assert lib.cotb200_bn_bwd_apply(_lib.BF16, 1, 4, 8, P, P, None, P, P, P, P, P, None, None, 0.25, 2, P, None, None,
                                    None) == EINVAL
    assert lib.cotb200_bn_bwd_apply(_lib.BF16, 1, 4, 8, P, P, P, None, P, P, P, P, None, None, 0.25, 4, P, None, None,
                                    None) == EINVAL
    assert lib.cotb200_bn_bwd_apply(_lib.F64, 1, 4, 8, P, P, P, None, P, P, P, P, None, None, 0.25, 1, P, None, None, None) == EDTYPE
    # BatchNorm forward with in-kernel finalisation: running buffers required when they are to be updated; the 1-bit mask
    # needs the ReLU
    assert lib.cotb200_bn_apply_batch(_lib.BF16, 1, 4, 8, P, None, P, P, None, None, None, None, 4.0, 1e-5, 0.1, 1, 1, P, P, P, P, P,
                                      None, None, None) == ENULL
    assert lib.cotb200_bn_apply_batch(_lib.BF16, 1, 4, 8, P, P, P, P, None, None, None, None, 4.0, 1e-5, 0.1, 0, 0, P, P, P, P, P,
                                      None, P, None) == EINVAL
    assert lib.cotb200_last_error()
