"""ctypes binding of libcotb200.so (the C ABI in include/cotb200.h).

PyTorch is only plumbing here: it owns device memory and streams; every kernel is reached through the
plain-C entry points with raw device pointers.  There is NO CPU or eager fallback: if the library
cannot be loaded the import of any op raises, loudly.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libcotb200.so")

F32, F64, BF16, F16 = 0, 1, 2, 3
NCHW, NHWC, NHWC_TAP = 0, 1, 2

_DTYPES = {torch.float32: F32, torch.float64: F64, torch.bfloat16: BF16, torch.float16: F16}


class AggDesc(ctypes.Structure):
    """struct cotb200_agg_desc (include/cotb200.h)."""
    _fields_ = [(n, ctypes.c_int) for n in (
        "n", "c", "h", "w", "heads", "wc", "kh", "kw", "sh", "sw", "ph", "pw", "dh", "dw", "ho", "wo",
        "dtype", "layout", "gc", "fold")] + [(n, ctypes.c_longlong) for n in (
            "x_sn", "x_sp", "w_sn", "w_sp", "y_sn", "y_sp")]


class MixRow(ctypes.Structure):
    """struct cotb200_mix_row (include/cotb200.h): the Mixup / CutMix of one output row."""
    _fields_ = [("mode", ctypes.c_int), ("partner", ctypes.c_int), ("lam", ctypes.c_float), ("one_minus_lam", ctypes.c_float),
                ("target_lam", ctypes.c_float), ("y0", ctypes.c_int), ("y1", ctypes.c_int), ("x0", ctypes.c_int), ("x1", ctypes.c_int)]


CLIP_NORM, CLIP_VALUE, CLIP_AGC = 1, 2, 3


class ClipUnit(ctypes.Structure):
    """struct cotb200_clip_unit (include/cotb200.h): one AGC unit of a flat range."""
    _fields_ = [("offset", ctypes.c_longlong), ("numel", ctypes.c_int), ("range", ctypes.c_int)]


class ClipSeg(ctypes.Structure):
    """struct cotb200_clip_seg (include/cotb200.h): one warp's piece of the optimizer's flat range, with its AGC unit (-1: none)."""
    _fields_ = [("offset", ctypes.c_longlong), ("numel", ctypes.c_int), ("unit", ctypes.c_int)]


class Clip(ctypes.Structure):
    """struct cotb200_clip (include/cotb200.h): the clip of one cotb200_sgd_ema_step_clip call."""
    _fields_ = [("mode", ctypes.c_int), ("value", ctypes.c_float), ("factor", ctypes.c_void_p), ("segs", ctypes.c_void_p),
                ("n_segs", ctypes.c_int), ("pad_", ctypes.c_int)]


OPT_SGD, OPT_MOMENTUM, OPT_ADAM, OPT_ADAMW, OPT_NADAM, OPT_RADAM, OPT_ADADELTA, OPT_RMSPROP, OPT_RMSPROPTF = range(1, 10)


class OptState(ctypes.Structure):
    """struct cotb200_opt_state (include/cotb200.h): the device scalars of one optimizer."""
    _fields_ = [("t", ctypes.c_double), ("m_schedule", ctypes.c_double), ("c", ctypes.c_float * 4), ("sync", ctypes.c_int),
                ("slow_init", ctypes.c_int)]


class Opt(ctypes.Structure):
    """struct cotb200_opt (include/cotb200.h): the optimizer of one cotb200_opt_step call."""
    _fields_ = [("rule", ctypes.c_int), ("eps", ctypes.c_float), ("lookahead_k", ctypes.c_int), ("lookahead_alpha", ctypes.c_float),
                ("M", ctypes.c_void_p), ("V", ctypes.c_void_p), ("S", ctypes.c_void_p), ("state", ctypes.c_void_p)]


_lock = threading.Lock()
_lib = None

_VP = ctypes.c_void_p
_DP = ctypes.POINTER(AggDesc)

# name -> (restype, argtypes); every symbol declared in include/cotb200.h must be listed here
SYMBOLS = {
    "cotb200_version": (ctypes.c_int, []),
    "cotb200_last_error": (ctypes.c_char_p, []),
    "cotb200_launch_count": (ctypes.c_longlong, []),
    "cotb200_prof_enable": (None, [ctypes.c_int]),
    "cotb200_prof_report": (ctypes.c_int, [ctypes.c_char_p, ctypes.c_int]),
    "cotb200_agg_zeropad_fwd": (ctypes.c_int, [_DP, _VP, _VP, _VP, _VP]),
    "cotb200_agg_zeropad_bwd": (ctypes.c_int, [_DP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "cotb200_agg_zeropad_mix_fwd": (ctypes.c_int, [_DP] + [ctypes.c_int] * 4 + [_VP] * 5),
    "cotb200_agg_zeropad_mix_bwd": (ctypes.c_int, [_DP] + [ctypes.c_int] * 4 + [_VP] * 8),
    "cotb200_agg_refpad_fwd": (ctypes.c_int, [_DP, _VP, _VP, _VP, _VP]),
    "cotb200_agg_refpad_bwd": (ctypes.c_int, [_DP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "cotb200_agg_zeropad_dilate_fwd": (ctypes.c_int, [_DP, _VP, _VP, _VP, _VP, _VP]),
    "cotb200_agg_zeropad_dilate_bwd": (ctypes.c_int, [_DP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "cotb200_agg_zeropad_mix_merge_fwd": (ctypes.c_int, [_DP] + [ctypes.c_int] * 4 + [_VP] * 4),
    "cotb200_agg_zeropad_mix_merge_bwd": (ctypes.c_int, [_DP] + [ctypes.c_int] * 4 + [_VP] * 6),
    "cotb200_col_stats": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 4),
    "cotb200_tail_pool": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 6),
    "cotb200_tail_combine": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 7),
    "cotb200_tail_bwd_sums": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 7),
    "cotb200_tail_bwd_dz_sums": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 8 + [ctypes.c_float] + [_VP] * 3),
    "cotb200_tail_bwd_apply": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 10 + [ctypes.c_float] * 2 + [_VP] * 3),
    "cotb200_bn_apply": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 4 + [ctypes.c_int] + [_VP] * 3),
    "cotb200_bn_apply_batch": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 8 + [ctypes.c_float] * 3 + [ctypes.c_int] * 2 + [_VP] * 8),
    "cotb200_bn_bwd_sums": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 8 + [ctypes.c_int] + [_VP] * 4),
    "cotb200_bn_bwd_apply": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 10 + [ctypes.c_float, ctypes.c_int] + [_VP] * 4),
    "cotb200_bn_finalize": (ctypes.c_int, [ctypes.c_int] + [_VP] * 6 + [ctypes.c_float] * 3 + [ctypes.c_int] * 2 + [_VP] * 5),
    "cotb200_gn9_stats": (ctypes.c_int, [ctypes.c_int] * 5 + [_VP] * 5),
    "cotb200_gn9_apply": (ctypes.c_int, [ctypes.c_int] * 5 + [_VP] * 8),
    "cotb200_gn9_bwd_sums": (ctypes.c_int, [ctypes.c_int] * 5 + [_VP] * 13),
    "cotb200_gn9_bwd_apply": (ctypes.c_int, [ctypes.c_int] * 5 + [_VP] * 10),
    "cotb200_sum_rows": (ctypes.c_int, [ctypes.c_int, ctypes.c_longlong, ctypes.c_int]
                         + [_VP, ctypes.c_longlong] * 5 + [_VP]),
    "cotb200_pool3s2_fwd": (ctypes.c_int, [ctypes.c_int] * 6 + [_VP] * 4),
    "cotb200_pool3s2_bwd": (ctypes.c_int, [ctypes.c_int] * 6 + [_VP] * 4),
    "cotb200_gemm_bf16": (ctypes.c_int, [ctypes.c_int] * 3 + [_VP, ctypes.c_longlong, _VP, ctypes.c_longlong]
                          + [ctypes.c_int, _VP, ctypes.c_longlong, _VP, ctypes.c_longlong]
                          + [_VP, ctypes.c_longlong, _VP, _VP, ctypes.c_int, _VP, _VP, _VP]),
    "cotb200_conv3x3_bf16": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP, ctypes.c_longlong, _VP, ctypes.c_int, _VP,
                                                                 ctypes.c_longlong, _VP, _VP, ctypes.c_int, _VP, _VP, _VP]),
    "cotb200_stem7x7s2_scratch_bytes": (ctypes.c_longlong, [ctypes.c_int] * 3),
    "cotb200_stem7x7s2_bf16": (ctypes.c_int, [ctypes.c_int] * 3 + [_VP, _VP, ctypes.c_int, _VP, ctypes.c_longlong, _VP, _VP, ctypes.c_int,
                                              _VP, _VP, _VP, _VP]),
    "cotb200_stem7x7s2_wgrad_bf16": (ctypes.c_int, [ctypes.c_int] * 3 + [_VP, ctypes.c_longlong, ctypes.c_int, _VP, _VP, _VP]),
    "cotb200_wgrad_bf16": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, _VP, ctypes.c_longlong, ctypes.c_int, _VP, ctypes.c_longlong,
                                          ctypes.c_int, _VP, ctypes.c_longlong, _VP, ctypes.c_longlong, ctypes.c_int, _VP]),
    "cotb200_se_eval_scratch_bytes": (ctypes.c_longlong, [ctypes.c_int] * 2),
    "cotb200_se_eval": (ctypes.c_int, [ctypes.c_int] * 3 + [_VP, ctypes.c_float] + [_VP] * 9),
    "cotb200_gather_chunk": (ctypes.c_int, []),
    "cotb200_multi_gather": (ctypes.c_int, [_VP, _VP, ctypes.c_int, ctypes.c_int, _VP, ctypes.c_float, _VP]),
    "cotb200_sgd_ema_step": (ctypes.c_int, [ctypes.c_longlong, _VP, _VP, ctypes.c_int, _VP, _VP, _VP, _VP, ctypes.c_int, _VP]),
    "cotb200_multi_lerp": (ctypes.c_int, [_VP, ctypes.c_int, _VP, _VP]),
    "cotb200_clip_seg_max": (ctypes.c_int, []),
    "cotb200_grad_norm": (ctypes.c_int, [ctypes.c_longlong, ctypes.c_int, _VP, _VP, ctypes.c_longlong, _VP, _VP, ctypes.c_float, _VP, _VP]),
    "cotb200_unit_norms": (ctypes.c_int, [ctypes.c_int, _VP, ctypes.c_longlong, _VP, ctypes.c_int, _VP, _VP, _VP, _VP, _VP, ctypes.c_float,
                                          _VP, _VP, _VP]),
    "cotb200_sgd_ema_step_clip": (ctypes.c_int, [ctypes.c_longlong, _VP, _VP, ctypes.c_int, _VP, _VP, _VP, _VP, ctypes.c_int,
                                                 ctypes.POINTER(Clip), _VP]),
    "cotb200_opt_prepare": (ctypes.c_int, [ctypes.POINTER(Opt), _VP, ctypes.c_int, _VP]),
    "cotb200_opt_step": (ctypes.c_int, [ctypes.c_longlong, _VP, ctypes.c_int, _VP, _VP, _VP, _VP, ctypes.POINTER(Opt), ctypes.POINTER(Clip),
                                        _VP]),
    "cotb200_lookahead_sync": (ctypes.c_int, [ctypes.c_longlong, _VP, _VP, ctypes.POINTER(Opt), _VP]),
    "cotb200_u8_to_nhwc": (ctypes.c_int, [ctypes.c_int] * 5 + [_VP, _VP, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float),
                                          _VP, _VP, _VP]),
    "cotb200_u8_mix_rows_to_nhwc": (ctypes.c_int, [ctypes.c_int] * 6 + [_VP, _VP, ctypes.POINTER(ctypes.c_float),
                                                                      ctypes.POINTER(ctypes.c_float), _VP, _VP, ctypes.POINTER(MixRow),
                                                                      _VP, _VP]),
    "cotb200_soft_ce": (ctypes.c_int, [ctypes.c_int] * 3 + [_VP, ctypes.c_longlong, _VP, ctypes.c_int, _VP, ctypes.c_float, _VP, _VP, _VP]),
    "cotb200_soft_ce_bwd": (ctypes.c_int, [ctypes.c_int] * 3 + [_VP, ctypes.c_longlong, _VP, ctypes.c_int, _VP, ctypes.c_float, _VP, _VP,
                                                                 _VP, ctypes.c_longlong, _VP]),
    "cotb200_jsd_ce": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP, ctypes.c_longlong, _VP, ctypes.c_float, ctypes.c_float, _VP, _VP, _VP]),
    "cotb200_jsd_ce_bwd": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP, ctypes.c_longlong, _VP, ctypes.c_float, ctypes.c_float, _VP, _VP,
                                                                _VP, ctypes.c_longlong, _VP]),
    "cotb200_topk_hits": (ctypes.c_int, [ctypes.c_int] * 3 + [_VP, ctypes.c_longlong, _VP, _VP, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                                               _VP, _VP]),
    "cotb200_aug_resize_crop": (ctypes.c_int, [ctypes.c_int] * 2 + [_VP, ctypes.c_longlong, _VP, _VP, _VP, ctypes.c_longlong, _VP, _VP]),
    "cotb200_aug_randaug": (ctypes.c_int, [ctypes.c_int] * 2 + [_VP] * 4),
    "cotb200_aug_color_jitter": (ctypes.c_int, [ctypes.c_int] * 2 + [_VP] * 4),
    "cotb200_aug_erase": (ctypes.c_int, [ctypes.c_int] * 5 + [_VP] * 4),
    "cotb200_dropblock_mask": (ctypes.c_int, [ctypes.c_int] * 5 + [ctypes.c_float, ctypes.c_int] + [_VP] * 4),
    "cotb200_dropblock_apply": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 5),
    "cotb200_dropblock_res_relu": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 8),
    "cotb200_dropblock_res_relu_bwd": (ctypes.c_int, [ctypes.c_int] * 4 + [_VP] * 8),
}


def lib_path():
    return _LIB_PATH


def load():
    """Load (building first if the sources are newer and nvcc exists) and return the ctypes library."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        from . import build as _build
        try:
            _build.build()
        except Exception as e:  # no nvcc and no prebuilt .so
            raise RuntimeError(
                "cotnet_b200: libcotb200.so is missing and could not be built (%s). "
                "There is no CPU fallback: run `python -m cotnet_b200.build` on a box with nvcc." % e) from e
        lib = ctypes.CDLL(_LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc, what):
    if rc != 0:
        msg = load().cotb200_last_error().decode("utf-8", "replace")
        raise RuntimeError("cotb200 %s failed (rc=%d): %s" % (what, rc, msg))


def dtype_code(t: torch.Tensor) -> int:
    try:
        return _DTYPES[t.dtype]
    except KeyError:
        raise TypeError("cotb200: unsupported dtype %s (float32/float64/bfloat16/float16)" % t.dtype)


def stream_ptr(t: torch.Tensor) -> int:
    """Current stream of t's device.  The C ABI launches on the CURRENT device (like the reference's
    `with torch.cuda.device_of(input)`, cupy_layers/aggregation_zeropad.py:129): a tensor that lives on another
    device would be launched with a foreign stream, so that is refused loudly instead of guarded silently."""
    if t.device.index is not None and t.device.index != torch.cuda.current_device():
        raise RuntimeError("cotb200: tensor on %s but the current CUDA device is cuda:%d; wrap the call in "
                           "`with torch.cuda.device_of(tensor):` (one process per GPU is the supported layout)"
                           % (t.device, torch.cuda.current_device()))
    return torch.cuda.current_stream(t.device).cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()


class DeviceCopy:
    """A device copy of a host table that kernels read (a Mixup / CutMix row table, an erase table).  The copy is made from a
    freshly pinned buffer of torch's caching host allocator, which does not hand that buffer out again before the copy has
    finished: the next table never races it.  The copy is issued on the stream current at creation; every consumer takes it
    through on_stream(), which orders its own current stream after that copy (an event wait) and tells the allocator that stream
    uses the memory, so creating and consuming on different streams is safe."""

    def __init__(self, host, device):
        self.dev = torch.frombuffer(bytearray(host), dtype=torch.uint8).pin_memory().to(device, non_blocking=True)
        self._copied = torch.cuda.Event()
        self._copied.record(torch.cuda.current_stream(self.dev.device))

    def on_stream(self, device, what):
        """The device copy, ready for use on `device`'s current stream."""
        if self.dev.device != torch.device(device):
            raise ValueError("%s: the device copy lives on %s, not %s" % (what, self.dev.device, device))
        st = torch.cuda.current_stream(self.dev.device)
        st.wait_event(self._copied)
        self.dev.record_stream(st)
        return self.dev


def launch_count() -> int:
    return int(load().cotb200_launch_count())


def require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError("cotb200 %s: tensor is on %s; the H100 kernels need CUDA tensors (no CPU fallback)" % (what, t.device))


def prof_enable(on: bool):
    load().cotb200_prof_enable(1 if on else 0)


def prof_report():
    """{kernel name: (launches, total_ms, total ALGORITHMIC bytes)} of the launches recorded since prof_enable(True)."""
    lib = load()
    n = lib.cotb200_prof_report(None, 0)
    buf = ctypes.create_string_buffer(n + 16)
    lib.cotb200_prof_report(buf, n + 16)
    out = {}
    for line in buf.value.decode().splitlines():
        name, cnt, ms, nbytes = line.rsplit(" ", 3)
        out[name] = (int(cnt), float(ms), float(nbytes))
    return out
