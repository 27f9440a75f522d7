"""DropBlock of the reference trunks (``drop_block_rate`` of create_model; models/layers/drop.py:70-131 ``drop_block_fast_2d``,
models/resnet.py:397-401 ``drop_blocks``).

Stages 1-2 have none, stage 3 ``DropBlock2d(rate, 5, 0.25)`` and stage 4 ``DropBlock2d(rate, 3, 1.0)``, one per stage shared by
its blocks.  A block applies it after ``bn1`` (before the ReLU), after ``bn0`` of a split-attention ``conv2`` (before the SiLU) and
after ``bn3`` (before drop path, the residual add and the ReLU); only in training mode with rate > 0.

For x [B, C, H, W] with cbs = min(block_size, H, W):
    gamma = gamma_scale * rate * H*W / cbs**2 / ((W - block_size + 1) * (H - block_size + 1))
    seed  = u < fp32(gamma),  M = 1 - max_pool2d(seed, cbs, stride 1, padding cbs // 2),  s = numel / (sum(M) + 1e-7)
    y     = x * M * s
The uniforms u are the library's own stream (include/cotb200.h, "DropBlock"), not torch.rand_like's: Philox4x32-10 keyed by
one [2] int64 draw per training forward, counted by the element's logical NCHW index and the site's number.  ``uniforms`` below
restates it on the host; the unfused (CPU / fp64 / NCHW) path uses it, so one key gives the same mask on both paths.  The
channels_last CUDA path draws, pools and counts the mask in cotb200_dropblock_mask and applies it in cotb200_dropblock_apply
(bn1, bn0) or in cotb200_dropblock_res_relu together with drop path, the residual add and the ReLU (bn3).  On a CUDA tensor
that is not channels_last the unfused path copies the key to the host at every site (a device sync; not capturable in a CUDA
graph) and draws the mask in numpy: it is a reference path, and CUDA training with DropBlock wants channels_last activations.
"""
import numpy as np
import torch
from torch.autograd import Function

from . import _lib, fused

_M0, _M1, _W0, _W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(q, site, k0, k1):
    """The four 32-bit outputs (as uint64 arrays) of Philox4x32-10 at counters (q mod 2^32, q >> 32, site, 0), key (k0, k1)."""
    q = np.asarray(q, dtype=np.uint64)
    c0, c1 = q & _LO, q >> np.uint64(32)
    c2, c3 = np.full_like(q, site), np.zeros_like(q)
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & _LO,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & _LO)
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def key_words(key):
    """(k0, k1): the low 32 bits of the two int64 words of a DropBlock key."""
    k = key.detach().cpu().tolist() if torch.is_tensor(key) else list(key)
    return int(k[0]) & 0xFFFFFFFF, int(k[1]) & 0xFFFFFFFF


def uniforms(shape, site, key):
    """fp32 uniforms u of site `site` for a tensor of NCHW shape `shape`, element e = the logical NCHW index."""
    n = int(np.prod(shape))
    k0, k1 = key_words(key)
    r = np.stack(philox4x32_10(np.arange((n + 3) // 4, dtype=np.uint64), site, k0, k1), axis=1).reshape(-1)[:n]
    return ((r >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)).reshape(shape)


def scale_of(count, numel):
    """torch's fp32  numel / (mask.float().sum() + 1e-7)  (reciprocal, then the product) for an exact count."""
    return np.float32(numel) * (np.float32(1.0) / (np.float32(count) + np.float32(1e-7)))


class DropBlock:
    """DropBlock2d(rate, block_size, gamma_scale) with the reference's defaults (fast, per sample, no noise).  No parameters
    or buffers: a model's state dict does not change."""

    def __init__(self, rate, block_size, gamma_scale):
        self.rate, self.block_size, self.gamma_scale = float(rate), int(block_size), float(gamma_scale)

    def __repr__(self):
        return "DropBlock(rate=%g, block_size=%d, gamma_scale=%g)" % (self.rate, self.block_size, self.gamma_scale)

    def geometry(self, H, W, site):
        """(cbs, gamma) at an H x W plane; ValueError where the reference would fail: an even clipped block size (its pooled
        mask is one pixel larger than x) or no valid block position (division by zero)."""
        bs = self.block_size
        cbs = min(bs, H, W)
        if cbs % 2 == 0:
            raise ValueError("DropBlock site %d: block size %d clipped to %d at %dx%d is even; the pooled mask would not match the "
                             "input (use a larger image)" % (site, bs, cbs, H, W))
        den = (W - bs + 1) * (H - bs + 1)
        if den == 0:
            raise ValueError("DropBlock site %d: no valid %dx%d block position at %dx%d (use a larger image)" % (site, bs, bs, H, W))
        return cbs, self.gamma_scale * self.rate * (H * W) / cbs ** 2 / den


def stage_drop_blocks(rate):
    """models/resnet.py:397-401: one DropBlock (or None) per stage."""
    rate = float(rate)
    return [None, None, DropBlock(rate, 5, 0.25) if rate else None, DropBlock(rate, 3, 1.0) if rate else None]


def host_mask(shape, site, key, spec):
    """(keep mask M as a bool NCHW array, exact kept count, fp32 scale) of one site, restated on the host."""
    B, C, H, W = shape
    cbs, gamma = spec.geometry(H, W, site)
    seed = uniforms(shape, site, key) < np.float32(gamma)
    pad = cbs // 2
    p = np.pad(seed, ((0, 0), (0, 0), (0, 0), (pad, pad)))
    row = np.zeros_like(seed)
    for d in range(cbs):
        row |= p[..., d:d + W]
    p = np.pad(row, ((0, 0), (0, 0), (pad, pad), (0, 0)))
    blk = np.zeros_like(seed)
    for d in range(cbs):
        blk |= p[..., d:d + H, :]
    keep = ~blk
    count = int(keep.sum())
    return keep, count, scale_of(count, keep.size)


def _unfused(x, key, site, spec):
    """drop_block_fast_2d with the host-restated uniforms: x * M * s in x's dtype, as the reference composes it."""
    keep, _, scale = host_mask(tuple(x.shape), site, key, spec)
    m = torch.from_numpy(keep).to(device=x.device, dtype=x.dtype)
    return x * m * torch.tensor(float(scale), dtype=torch.float32).to(device=x.device, dtype=x.dtype)


def device_mask(x, key, site, spec):
    """(mask [B*H*W, C/8] uint8, count int32 [1]) of one site of the channels_last CUDA tensor x (cotb200_dropblock_mask).
    The count accumulator comes from the step's zeroed scratch (fused._zeros), so a captured graph clears it at every replay."""
    B, C, H, W = x.shape
    cbs, gamma = spec.geometry(H, W, site)
    if C % 8:
        raise ValueError("DropBlock site %d: the CUDA kernels need C %% 8 == 0 (C = %d)" % (site, C))
    mask = torch.empty(B * H * W, C // 8, dtype=torch.uint8, device=x.device)
    count = fused._zeros((1,), x.device).view(torch.int32)
    key = key.to(device=x.device, dtype=torch.int64).contiguous()
    _lib.check(_lib.load().cotb200_dropblock_mask(B, C, H, W, cbs, float(np.float32(gamma)), site, key.data_ptr(), mask.data_ptr(),
                                                  count.data_ptr(), _lib.stream_ptr(x)), "dropblock_mask")
    return mask, count


def _apply(t, mask, count):
    B, C, H, W = t.shape
    y = torch.empty_like(t, memory_format=torch.channels_last)
    _lib.check(_lib.load().cotb200_dropblock_apply(_lib.dtype_code(t), B, H * W, C, t.data_ptr(), mask.data_ptr(), count.data_ptr(),
                                                   y.data_ptr(), _lib.stream_ptr(t)), "dropblock_apply")
    return y


class DropBlockFn(Function):
    """y = x * M * s on a channels_last CUDA tensor; dx = dy * M * s (the same kernel)."""

    @staticmethod
    def forward(ctx, x, mask, count):
        ctx.save_for_backward(mask, count)
        return _apply(x.detach().contiguous(memory_format=torch.channels_last), mask, count)

    @staticmethod
    def backward(ctx, dy):
        mask, count = ctx.saved_tensors
        return _apply(dy.contiguous(memory_format=torch.channels_last), mask, count), None, None


class DropBlockResReluFn(Function):
    """The bn3 site of a bottleneck: y = relu(res + ds[b] * (z * M * s)) (models/cotnet.py:248-262), its 1-bit ReLU mask kept for
    the backward: dres = dy * [y > 0], dz = dres * ds[b] * M * s."""

    @staticmethod
    def forward(ctx, z, res, mask, count, ds):
        assert fused._is_cl(z) and fused._is_cl(res) and z.shape == res.shape and z.dtype == res.dtype
        B, C, H, W = z.shape
        z, res = z.detach(), res.detach()
        y = torch.empty_like(z, memory_format=torch.channels_last)
        rmask = torch.empty(B * H * W, C // 8, dtype=torch.uint8, device=z.device)
        _lib.check(_lib.load().cotb200_dropblock_res_relu(_lib.dtype_code(z), B, H * W, C, z.data_ptr(), res.data_ptr(), mask.data_ptr(),
                                                          count.data_ptr(), _lib.ptr(ds), y.data_ptr(), rmask.data_ptr(),
                                                          _lib.stream_ptr(z)), "dropblock_res_relu")
        ctx.save_for_backward(rmask, mask, count, ds)
        return y

    @staticmethod
    def backward(ctx, dy):
        rmask, mask, count, ds = ctx.saved_tensors
        dy = dy.contiguous(memory_format=torch.channels_last)
        B, C, H, W = dy.shape
        dz = torch.empty_like(dy, memory_format=torch.channels_last)
        dres = torch.empty_like(dy, memory_format=torch.channels_last) if ctx.needs_input_grad[1] else None
        _lib.check(_lib.load().cotb200_dropblock_res_relu_bwd(_lib.dtype_code(dy), B, H * W, C, dy.data_ptr(), rmask.data_ptr(),
                                                              mask.data_ptr(), count.data_ptr(), _lib.ptr(ds), _lib.ptr(dres),
                                                              dz.data_ptr(), _lib.stream_ptr(dy)), "dropblock_res_relu_bwd")
        return dz, dres, None, None, None


def drop_block(x, key, site, spec):
    """DropBlock of site `site` on x: the CUDA kernels for channels_last CUDA tensors, else the reference's formula with the
    host-restated uniforms."""
    if fused.supported(x):
        mask, count = device_mask(x, key, site, spec)
        return DropBlockFn.apply(x, mask, count)
    return _unfused(x, key, site, spec)


def drop_block_res_relu(z, res, key, site, spec, drop_scale=None):
    """relu(res + drop_scale[b] * drop_block(z)) for channels_last CUDA z and res (the fused bn3 site)."""
    mask, count = device_mask(z, key, site, spec)
    return DropBlockResReluFn.apply(z, res, mask, count, fused._drop_scale(drop_scale, z))
