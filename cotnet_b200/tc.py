"""Thin torch-side wrappers of the wgmma GEMM / implicit-GEMM conv entry points (include/cotb200.h).

These are plumbing for the fused CoT block and for the unit tests: they allocate outputs with torch, pass raw
pointers + the current stream to the C ABI, and never fall back to cuBLAS/cuDNN."""
import torch

from . import _lib


def _rows(t: torch.Tensor):
    """[M, K] view of a 2-D tensor or of a channels_last 4-D activation ([B,C,H,W] with NHWC memory)."""
    if t.dim() == 2:
        assert t.stride(1) == 1
        return t.shape[0], t.shape[1], t.stride(0)
    assert t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last)
    B, C, H, W = t.shape
    return B * H * W, C, C


def gemm_bf16(a1, b1, a2=None, b2=None, scale=None, shift=None, relu=False, stats=None, out=None):
    """D[M,N] = epi(a1 @ b1.T (+ a2 @ b2.T)); bf16 in/out, fp32 accumulate.  stats=(col_sum, col_sqsum) fp32 [N],
    accumulated in place.  a* may be 2-D row-major or channels_last activations (rows = pixels)."""
    M, K1, lda1 = _rows(a1)
    N, K1b = b1.shape
    assert K1 == K1b and a1.dtype == torch.bfloat16 and b1.dtype == torch.bfloat16 and b1.stride(1) == 1
    K2, lda2, ldb2 = 0, 0, 0
    if a2 is not None:
        M2, K2, lda2 = _rows(a2)
        assert M2 == M and b2.shape == (N, K2) and b2.stride(1) == 1
        ldb2 = b2.stride(0)
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=a1.device)
    assert out.stride(-1) == 1
    cs, cq = (stats if stats is not None else (None, None))
    rc = _lib.load().cotb200_gemm_bf16(M, N, K1, a1.data_ptr(), lda1, b1.data_ptr(), b1.stride(0), K2, _lib.ptr(a2), lda2,
                                       _lib.ptr(b2), ldb2, out.data_ptr(), out.stride(0), _lib.ptr(scale), _lib.ptr(shift),
                                       1 if relu else 0, _lib.ptr(cs), _lib.ptr(cq), _lib.stream_ptr(a1))
    _lib.check(rc, "gemm_bf16")
    return out


def wgrad_bf16(dy, a1, a2=None, out=None):
    """dW [N, K1 (+K2)] fp32 = dy[M, N]^T @ [a1 | a2][M, K]: the weight gradient of a 1x1 convolution with output gradient dy and
    input(s) a1 (, a2).  Operands: 2-D row-major or channels_last activations (rows = pixels), bf16.  `out` (fp32, zeroed) may be
    given; the kernel ADDS into it."""
    M, N, ldy = _rows(dy)
    M1, K1, lda1 = _rows(a1)
    assert M1 == M and dy.dtype == torch.bfloat16 and a1.dtype == torch.bfloat16
    K2, lda2 = 0, 0
    if a2 is not None:
        M2, K2, lda2 = _rows(a2)
        assert M2 == M and a2.dtype == torch.bfloat16
    K = K1 + K2
    if out is None:
        out = torch.zeros((N, K), dtype=torch.float32, device=dy.device)
    assert out.shape == (N, K) and out.dtype == torch.float32 and out.stride(1) == 1 and out.data_ptr() % 16 == 0
    lib = _lib.load()
    if a2 is not None and K1 % 64:
        # the two-source form takes 64-channel boxes from a1 then a2: an a1 that does not end on a box boundary (CoXt, C = 96 ...)
        # runs as two single-source launches into the two column ranges of `out`
        wgrad_bf16(dy, a1, None, out=out[:, :K1])
        wgrad_bf16(dy, a2, None, out=out[:, K1:])
        return out
    # orientation: rows of the MMA tile (128 per CTA) from dy or from the input -- whichever needs fewer tiles
    t0 = ((N + 127) // 128) * ((K + 255) // 256)
    t1 = ((K + 127) // 128) * ((N + 255) // 256)
    if a2 is None and t1 < t0:
        rc = lib.cotb200_wgrad_bf16(M, K1, a1.data_ptr(), lda1, N, dy.data_ptr(), ldy, 0, None, 0, out.data_ptr(), out.stride(0), 1,
                                    _lib.stream_ptr(dy))
    else:
        rc = lib.cotb200_wgrad_bf16(M, N, dy.data_ptr(), ldy, K1, a1.data_ptr(), lda1, K2, _lib.ptr(a2), lda2, out.data_ptr(),
                                    out.stride(0), 0, _lib.stream_ptr(dy))
    _lib.check(rc, "wgrad_bf16")
    return out


_CONV_IDX = {}


def conv_tile(C, groups):
    """N tile (output channels per CTA) used by conv3x3_bf16 for a grouped conv, or None if unsupported."""
    cg = C // groups
    for bn in (64, 128, 192, 256):
        if C % bn == 0 and (bn % cg == 0):
            return bn
    return None


def prepare_conv3x3_weight(weight, groups, transpose_for_dgrad=False):
    """[C, C/groups, 3, 3] -> Wp [C, 9*bn] bf16 (dense inside each N tile, zero outside the group); see cotb200.h.
    transpose_for_dgrad: build the weight of the data-gradient convolution (taps flipped, in/out swapped per group)."""
    C, cg = weight.shape[0], weight.shape[1]
    bn = conv_tile(C, groups)
    assert bn is not None, "unsupported grouped-conv geometry for the wgmma path"
    w = weight.detach().float().view(groups, cg, cg, 3, 3)            # [g, out, in, kh, kw]
    if transpose_for_dgrad:
        w = w.permute(0, 2, 1, 3, 4).flip(3, 4)                       # dX = conv(dY, W^T flipped)
    w = w.reshape(C, cg, 9)
    Wp = torch.zeros(C, 9, bn, dtype=torch.float32, device=weight.device)
    key = (C, cg, bn, str(weight.device))
    idx3 = _CONV_IDX.get(key)
    if idx3 is None:                                                   # shape-only index tensor: built once (5 tiny launches per call otherwise)
        n = torch.arange(C, device=weight.device)
        off = (n // cg) * cg - (n // bn) * bn                          # first input channel of n's group inside the tile
        idx = off[:, None] + torch.arange(cg, device=weight.device)[None, :]      # [C, cg]
        idx3 = idx[:, None, :].expand(C, 9, cg).contiguous()
        _CONV_IDX[key] = idx3
    Wp.scatter_(2, idx3, w.permute(0, 2, 1))
    return Wp.reshape(C, 9 * bn).to(torch.bfloat16).contiguous(), bn


def conv3x3_bf16(x, wp, bn, scale=None, shift=None, relu=False, stats=None, out=None):
    """x: channels_last bf16 [B,C,H,W]; returns channels_last bf16 [B,C,H,W]."""
    assert x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=torch.channels_last)
    B, C, H, W = x.shape
    if out is None:
        out = torch.empty_like(x, memory_format=torch.channels_last)
    cs, cq = (stats if stats is not None else (None, None))
    rc = _lib.load().cotb200_conv3x3_bf16(B, H, W, C, x.data_ptr(), C, wp.data_ptr(), bn, out.data_ptr(), C, _lib.ptr(scale),
                                          _lib.ptr(shift), 1 if relu else 0, _lib.ptr(cs), _lib.ptr(cq), _lib.stream_ptr(x))
    _lib.check(rc, "conv3x3_bf16")
    return out


def prepare_stem_weight(weight):
    """[N, 3, 7, 7] -> Wm [N, 256] bf16 for cotb200_stem7x7s2_bf16: Wm[n, a*64 + a2*16 + (di*2+dj)*3 + c] =
    weight[n, c, 2a+di-1, 2a2+dj-1] (zero where an index is -1, and for the 4 pad channels of every cell)."""
    N = weight.shape[0]
    assert tuple(weight.shape[1:]) == (3, 7, 7)
    wp = torch.zeros(N, 3, 8, 8, dtype=torch.float32, device=weight.device)
    wp[:, :, 1:, 1:] = weight.detach().float()                       # index u = kh + 1 = 2a + di
    w6 = wp.view(N, 3, 4, 2, 4, 2).permute(0, 2, 4, 3, 5, 1)         # [n, a, a2, di, dj, c]
    wm = torch.zeros(N, 4, 4, 16, dtype=torch.float32, device=weight.device)
    wm[..., :12] = w6.reshape(N, 4, 4, 12)
    return wm.reshape(N, 256).to(torch.bfloat16).contiguous()


def stem7x7s2_bf16(x, wm, scale=None, shift=None, relu=False, stats=None, out=None, return_scratch=False):
    """x: channels_last bf16 [B,3,H,W] -> channels_last bf16 [B,N,H/2,W/2] = conv 7x7 / stride 2 / pad 3 with the prepared weight
    wm (prepare_stem_weight).  Returns None when the library cannot take the geometry (COTB200_EUNSUPPORTED)."""
    assert x.dim() == 4 and x.shape[1] == 3 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=torch.channels_last)
    B, _, H, W = x.shape
    N = wm.shape[0]
    lib = _lib.load()
    if out is None:
        out = torch.empty((B, N, H // 2, W // 2), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    scratch = torch.empty(int(lib.cotb200_stem7x7s2_scratch_bytes(B, H, W)), dtype=torch.uint8, device=x.device)
    cs, cq = (stats if stats is not None else (None, None))
    rc = lib.cotb200_stem7x7s2_bf16(B, H, W, x.data_ptr(), wm.data_ptr(), N, out.data_ptr(), N, _lib.ptr(scale), _lib.ptr(shift),
                                    1 if relu else 0, _lib.ptr(cs), _lib.ptr(cq), scratch.data_ptr(), _lib.stream_ptr(x))
    if rc == -7:
        return None
    _lib.check(rc, "stem7x7s2_bf16")
    return (out, scratch) if return_scratch else out


def unpack_stem_weight_grad(dwm):
    """[N, 256] gradient in the packed layout of prepare_stem_weight -> [N, 3, 7, 7] (the inverse gather: packed entries that stand for
    kernel index -1 or for the pad channels have no counterpart and are dropped)."""
    N = dwm.shape[0]
    g = dwm.view(N, 4, 4, 16)[..., :12].reshape(N, 4, 4, 2, 2, 3)       # [n, a, a2, di, dj, c]
    g = g.permute(0, 5, 1, 3, 2, 4).reshape(N, 3, 8, 8)                  # [n, c, 2a+di, 2a2+dj]
    return g[:, :, 1:, 1:].contiguous()


def stem7x7s2_wgrad(dy, scratch, x_shape, N):
    """dW [N, 3, 7, 7] fp32 of the stem convolution from dy (channels_last bf16 [B, N, H/2, W/2]) and the space-to-depth scratch image
    of the forward call; None when the library cannot take the geometry."""
    B, _, H, W = x_shape
    assert dy.dtype == torch.bfloat16 and dy.is_contiguous(memory_format=torch.channels_last)
    dwm = torch.zeros(N, 256, dtype=torch.float32, device=dy.device)
    rc = _lib.load().cotb200_stem7x7s2_wgrad_bf16(B, H, W, dy.data_ptr(), N, N, scratch.data_ptr(), dwm.data_ptr(), _lib.stream_ptr(dy))
    if rc == -7:
        return None
    _lib.check(rc, "stem7x7s2_wgrad_bf16")
    return unpack_stem_weight_grad(dwm)
