"""Which LocalConv kernel serves a call, mirrored in Python and checked without a GPU.

cotb200_agg_zeropad_fwd / _bwd (csrc/agg_zeropad.cu: fwd_impl, bwd_impl) and the mix pair try a cascade of kernels; the first one
whose conditions hold on geometry, dtype, layout, pointer alignment and strides takes the call.  This file holds

  * a Python copy of that cascade (resolve, is_same3, fits32, nhwc_vec, nhwc2_ok and the extra conditions of nhwc2_fwd / _dx / _dw,
    nchw2_pxv with its N*wc and stride tests, nchw_plane_launch's plane window and shared-memory loop, the NCHW and NHWC TMA
    eligibility; the NHWC TMA tile planning is test_persistent_gpu.at_setup) that predicts the exact multiset of profiler names a
    call launches and the sub-branch each launch takes;
  * source anchors: the literal conditions the copy follows must still be in the .cu files, so an edit to the dispatch fails here
    until the copy follows it;
  * CASES, the named calls tests/test_agg_kernels_gpu.py runs on the GPU, and a check that together they reach every branch of the
    cascade (REQUIRED);
  * the production table: every CoT / CoXt layer's LocalConv call of the models at the resolutions of their goldens and of bench.py,
    mapped to its kernels, pinned as hand-checked values, with each (kernel, sub-branch) pair present in CASES at the same geometry;
  * the fp64 reference the GPU test compares against, written from the header's definitions (weight channel of input channel c with
    the CoXt fold, NHWC_TAP weight order), checked here against oracle/agg_ref."""
import math
import os
import re
from collections import Counter, namedtuple

import pytest
import torch
import torch.nn.functional as F

import test_persistent_gpu as tp

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cotnet_b200", "csrc")
SMS_H100 = tp.SMS_H100
NCHW, NHWC, TAP = 0, 1, 2                        # COTB200_NCHW / NHWC / NHWC_TAP
ES = {"fp32": 4, "fp64": 8, "bf16": 2, "fp16": 2}
LIM31 = (1 << 31) - 1


def _cdiv(a, b):
    return -(-a // b)


# ================================================================================================ descriptors
class Desc:
    """struct cotb200_agg_desc.  p defaults to "same" padding; pitches of 0 select the dense default (NHWC layouts only)."""

    def __init__(self, N, C, H, W, wc, k=3, heads=1, s=1, d=1, p=None, layout=NCHW, gc=0, fold=1,
                 x_sn=0, x_sp=0, w_sn=0, w_sp=0, y_sn=0, y_sp=0):
        kh, kw = (k, k) if isinstance(k, int) else k
        p = (d * (kh // 2), d * (kw // 2)) if p is None else ((p, p) if isinstance(p, int) else p)
        self.n, self.c, self.h, self.w, self.heads, self.wc = N, C, H, W, heads, wc
        self.kh, self.kw, self.sh, self.sw, self.dh, self.dw = kh, kw, s, s, d, d
        self.ph, self.pw = p
        self.ho = (H + 2 * self.ph - (d * (kh - 1) + 1)) // s + 1
        self.wo = (W + 2 * self.pw - (d * (kw - 1) + 1)) // s + 1
        self.layout, self.gc, self.fold = layout, gc, fold
        self.x_sn, self.x_sp, self.w_sn, self.w_sp, self.y_sn, self.y_sp = x_sn, x_sp, w_sn, w_sp, y_sn, y_sp

    def key(self):
        return tuple(sorted(vars(self).items()))

    def __repr__(self):
        return "Desc(%s)" % ", ".join("%s=%s" % kv for kv in vars(self).items() if kv[1] or kv[0] in ("n", "c"))


class Geo:
    pass


def resolve(d):
    """resolve(): the kernels' view of a descriptor (element strides, fold, rep)."""
    if d.c % d.wc:
        raise ValueError("c % wc")
    g = Geo()
    g.N, g.C, g.H, g.W, g.heads, g.wc = d.n, d.c, d.h, d.w, d.heads, d.wc
    g.KH, g.KW, g.SH, g.SW, g.PH, g.PW, g.DH, g.DW = d.kh, d.kw, d.sh, d.sw, d.ph, d.pw, d.dh, d.dw
    g.HO, g.WO, g.K2, g.rep, g.layout = d.ho, d.wo, d.kh * d.kw, d.c // d.wc, d.layout
    g.gc = d.gc if d.gc > 0 else 1
    g.fold = d.fold if d.fold > 0 else 1
    if d.c % g.fold or d.wc % g.fold or (d.c // g.fold) % (d.wc // g.fold):
        raise ValueError("fold")
    g.Cf, g.wcf = d.c // g.fold, d.wc // g.fold
    J = d.heads * d.wc * g.K2
    if d.layout == NCHW:
        g.x_sw, g.x_sn = 1, g.C * g.H * g.W
        g.w_sw, g.w_sn = 1, g.wc * g.K2 * g.HO * g.WO * g.heads
        g.y_sw, g.y_sn = 1, g.HO * g.WO * g.C * g.heads
    else:
        if d.layout == TAP and g.wc % g.gc:
            raise ValueError("gc")
        g.x_sw = d.x_sp or g.C
        g.x_sn = d.x_sn or g.x_sw * g.W * g.H
        g.w_sw = d.w_sp or J
        g.w_sn = d.w_sn or g.w_sw * g.WO * g.HO
        g.y_sw = d.y_sp or g.C * g.heads
        g.y_sn = d.y_sn or g.y_sw * g.WO * g.HO
    return g


def is_same3(g, K):
    return (g.KH == K and g.KW == K and g.SH == 1 and g.SW == 1 and g.DH == 1 and g.DW == 1 and g.PH == K // 2 and g.PW == K // 2
            and g.heads == 1)


def fits32(g):
    return (g.N * g.C * g.heads * g.HO * g.WO < 1 << 31 and g.N * g.heads * g.wc * g.K2 * g.HO * g.WO < 1 << 31
            and g.N * g.C * g.H * g.W < 1 << 31)


def _aligned(offs, es, nbytes):
    """pointers at element offsets `offs` (None = NULL) of 256-byte aligned allocations are nbytes-aligned"""
    return all(o is None or (o * es) % nbytes == 0 for o in offs)


# ================================================================================================ the cascade, kernel by kernel
class Pred:
    """The launches of one call: [(profiler name, frozenset of sub-branch tags)] plus call-level tags (declines on the way)."""

    def __init__(self):
        self.launches, self.tags = [], set()

    def add(self, name, *tags, loop=None):
        t = set(tags)
        if loop is not None:                     # grid-stride kernel: (total threads, CTAs per SM of grid_stride_blocks' cap)
            total, per_sm = loop
            for sms in SMS_H100:
                grid = min(max(1, _cdiv(total, 256)), sms * per_sm)
                if total > grid * 256:
                    t.add("loop2@%d" % sms)
        self.launches.append((name, frozenset(t)))

    def names(self):
        return Counter(n for n, _ in self.launches)

    def all_tags(self):
        out = set(self.tags)
        for n, t in self.launches:
            out.add(n)
            out |= {n + "/" + x for x in t}
        return out


def nhwc_vec(g, es, offs):
    """nhwc_vec<T>: the packet width of the first-generation NHWC kernels, 0 if none"""
    if not is_same3(g, 3) or not fits32(g):
        return 0
    vec = 16 // es
    while vec >= 1:
        nb = vec * es
        ok = not (g.layout == TAP and vec != g.gc) and not (nb < 4 and vec != 1) and g.wcf % vec == 0
        ok = ok and _aligned(offs, es, nb) and all((s * es) % nb == 0 for s in (g.x_sw, g.x_sn, g.w_sw, g.w_sn, g.y_sw, g.y_sn))
        if ok:
            return vec
        vec //= 2
    return 0


def at_ok(mode, g, es, offs):
    """agg_tma.cu at_setup: the persistent TMA kernels take the call (mode 0 fwd, 1 dX, 2 dW)"""
    V = 16 // es
    if es == 8 or g.layout != TAP:
        return False
    if (g.C * es) % 128 or g.wcf % V or g.gc < V or g.gc % V or g.wc % g.gc:
        return False
    if not _aligned(offs, es, 16) or any((s * es) % 16 for s in (g.x_sn, g.x_sw, g.w_sn, g.w_sw, g.y_sn, g.y_sw)):
        return False
    if g.W + 2 > 256:
        return False
    J = 9 * g.wc
    jboxes = _cdiv(J, 256)
    while J % jboxes:
        jboxes += 1
    if ((J // jboxes) * es) % 16:
        return False
    if (g.y_sw, g.x_sw, g.w_sw)[mode] > LIM31:
        return False
    return tp.at_setup(mode, es, g.N, g.C, g.H, g.W, g.wc) is not None


def nhwc2_ok(g, es, offs, need_tap):
    V = 16 // es
    if es == 8 or g.layout == NCHW or (need_tap and g.layout != TAP):
        return False
    if g.wcf % V or g.C % V:
        return False
    if g.layout == TAP and (g.gc < V or g.gc % V or g.wc % g.gc):
        return False
    if not _aligned(offs, es, 16):
        return False
    if any(s > LIM31 or (s * es) % 16 for s in (g.x_sn, g.x_sw, g.w_sn, g.w_sw, g.y_sn, g.y_sw)):
        return False
    if any(g.H * g.W * sp > LIM31 for sp in (g.x_sw, g.w_sw, g.y_sw)):
        return False
    return g.N * g.H <= 65535 * 32768


def _nhwc2_rows(g, px):
    """(interior rows exist, edge rows exist) of agg3_nhwc2_kernel's interior / CHECK split"""
    interior = g.H >= 3 and any(w0 >= 1 and w0 + px < g.W for w0 in range(0, g.W, px))
    return interior, True


def nhwc2_fwd(P, g, es, offs):
    if not nhwc2_ok(g, es, offs, False) or g.N * g.H > LIM31:
        return False
    px = 2 if g.W % 2 == 0 else 1
    if g.N * g.H > 65535:
        P.tags.add("nhwc2_fwd-declined/grid.y")
        return False
    P.add("agg3_fwd_nhwc2", *_nhwc2_tags(g, px))
    return True


def _nhwc2_tags(g, px):
    interior, _ = _nhwc2_rows(g, px)
    return ("px%d" % px, "tap" if g.layout == TAP else "plain", "fold%d" % g.fold, "interior" if interior else "edge-only")


def nhwc2_dx(P, g, es, offs):
    if not nhwc2_ok(g, es, offs, True):
        return False
    px = 2 if g.W % 2 == 0 else 1
    if g.N * g.H > 65535:
        P.tags.add("nhwc2_dx-declined/grid.y")
        return False
    P.add("agg3_dx_nhwc2", *_nhwc2_tags(g, px))
    return True


def nhwc2_dw(P, g, es, offs):
    if not nhwc2_ok(g, es, offs, True):
        return False
    V = 16 // es
    if g.C // g.wc != 8:
        P.tags.add("nhwc2_dw-declined/rep")
        return False
    GQ = g.wc // V
    gqw = 4 if GQ >= 4 else GQ
    if GQ % gqw or gqw not in (1, 2, 4):
        P.tags.add("nhwc2_dw-declined/gqw")
        return False
    if g.fold > 1 and (g.wc // g.fold) % (gqw * V):
        P.tags.add("nhwc2_dw-declined/fold")
        return False
    if g.N * g.H > 65535:
        P.tags.add("nhwc2_dw-declined/grid.y")
        return False
    P.add("agg3_dw_nhwc2", "gqw%d" % gqw, "fold%d" % g.fold, *_nhwc2_tags(g, 1)[3:])
    return True


def nchw_tma_ok(es, N, C, H, W, wc, a_sn, b_sn, out_sn, offs):
    """agg_nchw_tma.cu nchw_tma_launch's conditions.  With rep <= 16 and W + 2 * halo <= 256 a one-row tile always fits its
    budget at >= 2 stages (test_nchw_tma_first_tile_fits), so these are all of them."""
    if es == 8 or C % wc:
        return False
    rep, al = C // wc, 16 // es
    pxv = 4 if W % 4 == 0 else (2 if W % 2 == 0 and es == 4 else 0)
    if not pxv or rep > 16:
        return False
    if (W * es) % 16 or (H * W * es) % 16 or (a_sn * es) % 16 or (b_sn * es) % 16 or (out_sn * es) % (pxv * es):
        return False
    return _aligned(offs, es, 16) and W + 2 * max(pxv, al) <= 256


def nchw2_pxv(es, W, offs):
    if es == 8:
        return 0
    for pxv in (4, 2):
        if W % pxv == 0 and _aligned(offs, es, pxv * es):
            return pxv
    return 0


def nchw2_fwd(P, g, es, offs):
    pxv = nchw2_pxv(es, g.W, offs)
    if pxv and g.N * g.wc > 65535:
        P.tags.add("nchw2-declined/N*wc")
    if not pxv or g.N * g.wc > 65535 or g.y_sn % pxv:
        return False
    P.add("agg3_fwd_nchw2", "pxv%d" % pxv)
    return True


def nchw2_bwd(P, g, es, offs, dx, dw):
    pxv = nchw2_pxv(es, g.W, offs)
    if pxv and g.N * g.wc > 65535:
        P.tags.add("nchw2-declined/N*wc")
    if not pxv or g.N * g.wc > 65535 or g.y_sn % pxv:
        return False
    P.add("agg3_bwd_nchw2_" + ("dxdw" if dx and dw else ("dx" if dx else "dw")), "pxv%d" % pxv)
    return True


PLANE_SMEM = 96 * 1024


def plane_launch(P, g, es, mode):
    """agg_nchw_plane.cu nchw_plane_launch: CTAs own ipc (sample, weight channel) items, their rep planes staged in shared memory"""
    HW = g.H * g.W
    if es == 8 or HW > 256 or HW < 100 or g.C % g.wc:
        return False
    PP = (g.H + 2) * (g.W + 2)
    per = g.rep * PP * (2 if mode & 2 else 1) * 4
    ipc = 256 // HW
    while ipc > 1 and ipc * per > PLANE_SMEM:
        ipc -= 1
    if ipc * per > PLANE_SMEM:
        P.tags.add("plane-declined/smem")
        return False
    if g.N * g.wc > 2000000000:
        return False
    tags = ["ipc%d" % ipc]
    if ipc > 1:
        tags.append("ipc>1")
    if ipc < 256 // HW:
        tags.append("ipc-lowered")
    P.add({1: "agg3_dx_plane", 2: "agg3_dw_plane", 3: "agg3_dxdw_plane"}[mode], *tags)
    return True


def fwd_impl(P, g, es, offs):
    """fwd_impl: offs = element offsets of (x, w, y)"""
    if g.layout != NCHW and is_same3(g, 3):
        if at_ok(0, g, es, offs):
            P.add("agg3_fwd_tma")
            return
        if nhwc2_fwd(P, g, es, offs):
            return
    if g.layout == NCHW and g.fold == 1 and fits32(g) and is_same3(g, 3) and g.w_sn == g.wc * 9 * g.H * g.W:
        if g.x_sn == g.C * g.H * g.W and nchw_tma_ok(es, g.N, g.C, g.H, g.W, g.wc, g.x_sn, 0, g.y_sn, offs):
            P.add("agg3_fwd_nchw_tma")
            return
        if nchw2_fwd(P, g, es, offs):
            return
    if g.layout == NCHW and g.fold == 1 and fits32(g) and (is_same3(g, 3) or is_same3(g, 5)) and es != 8:
        P.add("agg_fwd_nchw_k%d" % g.KH, loop=(g.N * g.wc * g.H * g.W, 8))
        return
    if g.layout != NCHW and es != 8:
        vec = nhwc_vec(g, es, offs)
        if vec:
            P.add("agg3_fwd_nhwc", "vec%d" % vec, "tap" if g.layout == TAP else "plain", "fold%d" % g.fold,
                  loop=(g.N * g.H * g.W * (g.C // vec), 8))
            return
    P.add("agg_fwd_generic", *_generic_tags(g), loop=(g.N * g.heads * g.C * g.HO * g.WO, 16))


def _generic_tags(g):
    t = {"layout%d" % g.layout, "fold%d" % g.fold}
    if g.heads > 1:
        t.add("heads")
    if g.SH > 1 or g.SW > 1:
        t.add("stride")
    if g.DH > 1 or g.DW > 1:
        t.add("dilation")
    if g.KH >= 7 or g.KW >= 7:
        t.add("k7")
    if g.H != g.W:
        t.add("rect")
    return sorted(t)


def bwd_impl(P, g, es, offs, dx, dw, acc_dx=False):
    """bwd_impl: offs = element offsets of (dy, x, w, dx, dw) (None where NULL); dx / dw: gradient wanted"""
    if not dx and not dw:
        return
    o_dy, o_x, o_w, o_dx, o_dw = offs
    if (g.layout == NCHW and g.fold == 1 and fits32(g) and is_same3(g, 3) and not acc_dx and g.w_sn == g.wc * 9 * g.H * g.W):
        if g.H * g.W <= 256 and plane_launch(P, g, es, 3 if dx and dw else (1 if dx else 2)):
            return
        if g.x_sn == g.C * g.H * g.W:
            done_dx, done_dw = not dx, not dw
            if dx and nchw_tma_ok(es, g.N, g.C, g.H, g.W, g.wc, g.y_sn, 0, g.x_sn, (o_dy, o_w, o_dx)):
                P.add("agg3_dx_nchw_tma")
                done_dx = True
            if dw and nchw_tma_ok(es, g.N, g.C, g.H, g.W, g.wc, g.x_sn, g.y_sn, g.w_sn, (o_x, o_dy, o_dw)):
                P.add("agg3_dw_nchw_tma")
                done_dw = True
            if done_dx and done_dw:
                return
            if nchw2_bwd(P, g, es, (o_dy, o_x, o_w, None if done_dx else o_dx, None if done_dw else o_dw),
                         dx and not done_dx, dw and not done_dw):
                return
            dx, dw = dx and not done_dx, dw and not done_dw
    if g.layout == NCHW and g.fold == 1 and fits32(g) and (is_same3(g, 3) or is_same3(g, 5)) and es != 8:
        tags = ["K%d" % g.KH] + (["ACC_DX"] if acc_dx and dx else [])
        P.add("agg_bwd_nchw_" + ("dxdw" if dx and dw else ("dx" if dx else "dw")), *tags, loop=(g.N * g.wc * g.H * g.W, 8))
        return
    if g.layout == TAP and not acc_dx and is_same3(g, 3):
        if dx and at_ok(1, g, es, (o_dy, o_w, o_dx)):
            P.add("agg3_dx_tma")
            dx = False
        if dw and at_ok(2, g, es, (o_x, o_dy, o_dw)):
            P.add("agg3_dw_tma")
            dw = False
        if dx and nhwc2_dx(P, g, es, (o_dy, o_w, o_dx)):
            dx = False
        if dw and nhwc2_dw(P, g, es, (o_dy, o_x, o_dw)):
            dw = False
        if not dx and not dw:
            return
    if g.layout != NCHW and not acc_dx and es != 8:
        vec = nhwc_vec(g, es, (o_dy, o_x, o_w))
        if vec and _aligned((o_dx if dx else None, o_dw if dw else None), es, vec * es):
            tags = ("vec%d" % vec, "tap" if g.layout == TAP else "plain", "fold%d" % g.fold)
            if dx:
                P.add("agg3_dx_nhwc", *tags, loop=(g.N * g.H * g.W * (g.C // vec), 8))
            if dw:
                P.add("agg3_dw_nhwc", *tags, loop=(g.N * g.H * g.W * (g.wc // vec), 8))
            return
    gt = _generic_tags(g)
    if dx:
        P.add("agg_dx_generic", *(gt + (["ACCUM"] if acc_dx else [])), loop=(g.N * g.C * g.H * g.W, 16))
    if dw:
        P.add("agg_dw_generic", *gt, loop=(g.N * g.heads * g.wc * g.K2 * g.HO * g.WO, 16))


# ---- entry points
def predict_fwd(d, dt, offs):
    P = Pred()
    fwd_impl(P, resolve(d), ES[dt], (offs["x"], offs["w"], offs["y"]))
    return P


def predict_bwd(d, dt, offs, dx, dw):
    P = Pred()
    bwd_impl(P, resolve(d), ES[dt], (offs["dy"], offs["x"], offs["w"], offs["dx"] if dx else None, offs["dw"] if dw else None),
             dx, dw)
    return P


MIX_K2, MIX_P2 = 5, 2           # the second kernel of the mix op in every case here: 5x5, "same" padding


def mix_geos(d):
    """resolve_mix: both halves, their outputs interleaved per sample in one [n, 2*heads*c, ho, wo] tensor"""
    d2 = Desc(d.n, d.c, d.h, d.w, d.wc, k=MIX_K2, heads=d.heads, s=d.sh, d=d.dh, p=MIX_P2, fold=d.fold)
    g1, g2 = resolve(d), resolve(d2)
    g1.y_sn *= 2
    g2.y_sn *= 2
    return g1, g2


def predict_mix_fwd(d, dt, offs):
    P = Pred()
    g1, g2 = mix_geos(d)
    es = ES[dt]
    half = g1.heads * g1.C * g1.HO * g1.WO
    if es != 8 and is_same3(g1, 3) and is_same3(g2, 5) and fits32(g2) and 2 * half * g1.N < 1 << 31:
        P.add("agg_mix_fwd_nchw", loop=(g1.N * g1.wc * g1.H * g1.W, 8))
        return P
    fwd_impl(P, g1, es, (offs["x"], offs["w1"], offs["y"]))
    fwd_impl(P, g2, es, (offs["x"], offs["w2"], offs["y"] + half))
    return P


def predict_mix_bwd(d, dt, offs, dx, dw):
    P = Pred()
    g1, g2 = mix_geos(d)
    es = ES[dt]
    half = g1.heads * g1.C * g1.HO * g1.WO
    o_dx = offs["dx"] if dx else None
    o_dw1, o_dw2 = (offs["dw1"], offs["dw2"]) if dw else (None, None)
    if es >= 4 and is_same3(g1, 3) and is_same3(g2, 5) and fits32(g2):
        bwd_impl(P, g1, es, (offs["dy"], offs["x"], offs["w1"], o_dx, o_dw1), dx, dw)
        bwd_impl(P, g2, es, (offs["dy"] + half, offs["x"], offs["w2"], o_dx, o_dw2), dx, dw, acc_dx=dx)
        return P
    if dx:
        P.add("agg_mix_dx", loop=(g1.N * g1.C * g1.H * g1.W, 16))
    bwd_impl(P, g1, es, (offs["dy"], offs["x"], offs["w1"], None, o_dw1), False, dw)
    bwd_impl(P, g2, es, (offs["dy"] + half, offs["x"], offs["w2"], None, o_dw2), False, dw)
    return P


# ================================================================================================ cases
TENSORS = ("x", "w", "y", "dy", "dx", "dw")
MIX_TENSORS = ("x", "w1", "w2", "y", "dy", "dx", "dw1", "dw2")
BWD_VARIANTS = (("dxdw", True, True), ("dx", True, False), ("dw", False, True))
Case = namedtuple("Case", "name dt desc op kind offs expect")


def case(name, dt, desc, expect=(), op="agg", kind="int", off=0):
    names = MIX_TENSORS if op == "mix" else TENSORS
    offs = dict.fromkeys(names, off) if isinstance(off, int) else {n: off.get(n, 0) for n in names}
    return Case(name, dt, desc, op, kind, offs, frozenset(expect))


def predict(c):
    """{call: Pred} of the calls a case makes: the forward and the backward with both gradients, dX only and dW only"""
    if c.op == "mix":
        out = {"fwd": predict_mix_fwd(c.desc, c.dt, c.offs)}
        out.update((v, predict_mix_bwd(c.desc, c.dt, c.offs, dx, dw)) for v, dx, dw in BWD_VARIANTS)
    else:
        out = {"fwd": predict_fwd(c.desc, c.dt, c.offs)}
        out.update((v, predict_bwd(c.desc, c.dt, c.offs, dx, dw)) for v, dx, dw in BWD_VARIANTS)
    return out


def case_tags(c):
    t = set()
    for p in predict(c).values():
        t |= p.all_tags()
    return t


def _pitch(N, C, H, W, wc, heads=1, k=3, extra=8, **kw):
    """NHWC pitches larger than dense: every pixel row and every sample of x, w and y padded by `extra` elements"""
    J = heads * wc * (k * k)
    return dict(x_sp=C + extra, x_sn=H * W * (C + extra) + extra, w_sp=J + extra, w_sn=H * W * (J + extra) + 2 * extra,
                y_sp=heads * C + extra, y_sn=H * W * (heads * C + extra) + 3 * extra, **kw)


def D(N, C, H, W, wc, **kw):
    return Desc(N, C, H, W, wc, **kw)


def DP(N, C, H, W, wc, extra=8, **kw):
    """NHWC descriptor with pitches"""
    pk = _pitch(N, C, H, W, wc, heads=kw.get("heads", 1), k=kw.get("k", 3), extra=extra)
    return Desc(N, C, H, W, wc, **dict(kw, **pk))


# Production geometries (bf16, dense, "same" 3x3, heads 1): the descriptor fused.AggTapFn builds for each CoT / CoXt layer
# (gc = fused.tap_chunk(C // 8, fold)), at a batch of 2.
PROD_GEOS = {
    # (C, H, W, fold): gc
    (64, 56, 56, 1): 8, (128, 28, 28, 1): 8, (256, 14, 14, 1): 8, (512, 7, 7, 1): 8,
    (256, 40, 40, 1): 8, (256, 20, 20, 1): 8, (512, 20, 20, 1): 8, (512, 10, 10, 1): 8,
    (96, 56, 56, 2): 0, (192, 28, 28, 2): 0, (384, 14, 14, 2): 8, (768, 7, 7, 2): 8,
}


def _prod_desc(C, H, W, fold, gc, N=2):
    return Desc(N, C, H, W, C // 8, layout=TAP if gc else NHWC, gc=gc, fold=fold)


CASES = [
    # ---- production geometries at batch 2
    *[case("prod-C%d-%dx%d-fold%d" % (C, H, W, fold), "bf16", _prod_desc(C, H, W, fold, gc)) for (C, H, W, fold), gc in PROD_GEOS.items()],
    # ---- second-generation NHWC kernels (W + 2 > 256, the channel slab budget or C * 2 % 128 keep the TMA kernels out)
    case("nhwc2-tap-gqw1", "bf16", D(1, 64, 3, 256, 8, layout=TAP, gc=8),
         {"agg3_fwd_nhwc2/px2", "agg3_fwd_nhwc2/tap", "agg3_fwd_nhwc2/interior", "agg3_dx_nhwc2/px2", "agg3_dw_nhwc2/gqw1"}),
    case("nhwc2-tap-gqw2-px1", "bf16", D(1, 128, 4, 255, 16, layout=TAP, gc=8),
         {"agg3_fwd_nhwc2/px1", "agg3_dx_nhwc2/px1", "agg3_dw_nhwc2/gqw2"}),
    case("nhwc2-tap-gqw4", "fp16", D(1, 256, 3, 256, 32, layout=TAP, gc=8), {"agg3_dw_nhwc2/gqw4"}),
    case("nhwc2-tap-gqw4-fold2", "bf16", D(1, 512, 3, 40, 64, layout=TAP, gc=8, fold=2),
         {"agg3_fwd_nhwc2/fold2", "agg3_dx_nhwc2/fold2", "agg3_dw_nhwc2/fold2", "agg3_dw_nhwc2/gqw4"}),
    case("nhwc2-tap-edge-rows", "bf16", D(2, 64, 2, 256, 8, layout=TAP, gc=8),
         {"agg3_fwd_nhwc2/edge-only", "agg3_dx_nhwc2/edge-only", "agg3_dw_nhwc2/edge-only"}),
    case("nhwc2-tap-fp32", "fp32", D(1, 32, 3, 256, 4, layout=TAP, gc=4), {"agg3_dw_nhwc2/gqw1", "agg3_fwd_nhwc2/interior"}),
    case("nhwc2-plain-fwd", "bf16", D(2, 64, 5, 6, 8, layout=NHWC),
         {"agg3_fwd_nhwc2/plain", "agg3_fwd_nhwc2/interior", "agg3_dx_nhwc/vec8", "agg3_dx_nhwc/plain", "agg3_dw_nhwc/vec8"}),
    case("nhwc2-dw-rep3", "bf16", D(2, 72, 4, 6, 24, layout=TAP, gc=8),
         {"agg3_fwd_nhwc2/tap", "agg3_dx_nhwc2/px2", "nhwc2_dw-declined/rep", "agg3_dw_nhwc/vec8", "agg3_dw_nhwc/tap"}),
    case("nhwc2-dw-gqw3", "bf16", D(1, 192, 2, 256, 24, layout=TAP, gc=8), {"nhwc2_dw-declined/gqw", "agg3_dw_nhwc/tap"}),
    case("nhwc2-dw-fold", "bf16", D(1, 256, 3, 256, 32, layout=TAP, gc=8, fold=2),
         {"nhwc2_dw-declined/fold", "agg3_dw_nhwc/fold2", "agg3_dx_nhwc2/fold2"}),
    case("nhwc2-pitch", "bf16", DP(2, 64, 3, 256, 8, layout=TAP, gc=8), {"agg3_fwd_nhwc2/tap", "agg3_dw_nhwc2/gqw1"}),
    case("tma-pitch", "bf16", DP(2, 64, 8, 8, 8, layout=TAP, gc=8), {"agg3_fwd_tma", "agg3_dx_tma", "agg3_dw_tma"}),
    # ---- first-generation packet kernels: widths 8 / 4 / 2 / 1, TAP order (vec == gc) and plain order
    case("pk-plain-v4", "bf16", D(2, 48, 5, 7, 12, layout=NHWC), {"agg3_fwd_nhwc/vec4", "agg3_dx_nhwc/vec4", "agg3_dw_nhwc/plain"}),
    case("pk-plain-v1", "bf16", D(2, 24, 4, 5, 3, layout=NHWC), {"agg3_fwd_nhwc/vec1", "agg3_dw_nhwc/vec1"}),
    case("pk-plain-v2-offset", "bf16", D(2, 64, 4, 5, 8, layout=NHWC), {"agg3_fwd_nhwc/vec2", "agg3_dx_nhwc/vec2"}, off=2),
    case("pk-plain-v1-offset", "fp16", D(2, 64, 3, 4, 8, layout=NHWC), {"agg3_fwd_nhwc/vec1", "agg3_dw_nhwc/vec1"}, off=1),
    case("pk-tap-v4", "bf16", D(2, 32, 5, 5, 4, layout=TAP, gc=4), {"agg3_fwd_nhwc/vec4", "agg3_fwd_nhwc/tap", "agg3_dx_nhwc/vec4"}),
    case("pk-tap-v2", "bf16", D(2, 16, 4, 3, 2, layout=TAP, gc=2), {"agg3_fwd_nhwc/vec2", "agg3_dw_nhwc/tap"}),
    case("pk-tap-v1", "bf16", D(2, 8, 3, 4, 1, layout=TAP, gc=1), {"agg3_fwd_nhwc/vec1", "agg3_dx_nhwc/tap"}),
    case("pk-tap-v2-fold2", "fp16", DP(2, 16, 4, 5, 4, layout=TAP, gc=2, fold=2, extra=2),
         {"agg3_fwd_nhwc/fold2", "agg3_dw_nhwc/fold2", "agg3_dx_nhwc/tap"}),
    case("pk-fp32-plain-v2", "fp32", D(2, 16, 4, 6, 2, layout=NHWC), {"agg3_fwd_nhwc/vec2", "agg3_dw_nhwc/vec2"}),
    case("pk-fp32-plain-v1", "fp32", D(2, 9, 3, 5, 3, layout=NHWC), {"agg3_fwd_nhwc/vec1"}),
    case("pk-fp32-tap-v4", "fp32", D(2, 48, 4, 6, 16, layout=TAP, gc=4), {"agg3_dw_nhwc/vec4", "agg3_fwd_nhwc2/tap"}),
    case("pk-fp32-plain-v4", "fp32", D(2, 16, 4, 5, 4, layout=NHWC), {"agg3_dx_nhwc/vec4", "agg3_dw_nhwc/vec4"}),
    case("pk-fp32-tap-v1-pitch", "fp32", DP(2, 6, 3, 5, 3, layout=TAP, gc=1, extra=3), {"agg3_fwd_nhwc/vec1", "agg3_dw_nhwc/tap"}),
    case("pk-plain-v4-pitch", "bf16", DP(2, 48, 5, 7, 12, layout=NHWC, extra=4), {"agg3_fwd_nhwc/vec4", "agg3_dw_nhwc/vec4"}),
    # ---- limits: nhwc2's grid.y (N * H > 65535) -> first-generation kernels at full width, both orders
    case("limit-nhwc2-plain", "bf16", D(21846, 8, 3, 2, 8, layout=NHWC),
         {"nhwc2_fwd-declined/grid.y", "agg3_fwd_nhwc/vec8", "agg3_fwd_nhwc/plain"}),
    case("limit-nhwc2-tap", "bf16", D(21846, 8, 3, 2, 8, layout=TAP, gc=8),
         {"nhwc2_fwd-declined/grid.y", "nhwc2_dx-declined/grid.y", "agg3_fwd_nhwc/vec8", "agg3_fwd_nhwc/tap", "agg3_dx_nhwc/vec8",
          "agg3_dx_nhwc/tap", "agg3_dw_nhwc/vec8"}),
    # ---- NCHW: TMA, second generation (PXV 4 / 2), small-plane backward, first generation K 3 / 5
    case("nchw-tma-small", "fp32", D(2, 32, 8, 8, 8), {"agg3_fwd_nchw_tma", "agg3_dx_nchw_tma", "agg3_dw_nchw_tma"}),
    case("nchw2-pxv4", "bf16", D(2, 32, 6, 12, 8), {"agg3_fwd_nchw2/pxv4", "agg3_bwd_nchw2_dxdw/pxv4", "agg3_bwd_nchw2_dx",
                                                   "agg3_bwd_nchw2_dw"}),
    case("nchw2-pxv2", "fp16", D(2, 24, 7, 10, 8), {"agg3_fwd_nchw2/pxv2", "agg3_bwd_nchw2_dxdw/pxv2"}),
    case("nchw2-pxv2-fp32", "fp32", D(2, 16, 5, 14, 4), {"agg3_fwd_nchw2/pxv2", "agg3_bwd_nchw2_dx/pxv2", "agg3_bwd_nchw2_dw/pxv2"}),
    case("nchw2-pxv4-fp32-rep32", "fp32", D(1, 64, 6, 8, 2), {"agg3_fwd_nchw2/pxv4", "agg3_bwd_nchw2_dxdw/pxv4"}),
    case("nchw2-pxv2-offset", "bf16", D(2, 16, 6, 12, 4), {"agg3_fwd_nchw2/pxv2", "agg3_bwd_nchw2_dxdw/pxv2"}, off=2),
    case("plane-14x14", "bf16", D(2, 64, 14, 14, 8), {"agg3_dxdw_plane/ipc1", "agg3_dx_plane", "agg3_dw_plane", "agg3_fwd_nchw2/pxv2"}),
    case("plane-ipc2", "fp16", D(3, 32, 10, 10, 4), {"agg3_dxdw_plane/ipc>1", "agg3_dx_plane/ipc>1", "agg3_dw_plane/ipc>1"}),
    case("plane-fp32-rect", "fp32", D(2, 16, 8, 16, 2), {"agg3_dxdw_plane/ipc>1", "agg3_fwd_nchw_tma"}),
    case("plane-ipc-lowered", "bf16", D(3, 86, 10, 10, 2), {"agg3_dxdw_plane/ipc-lowered", "agg3_dw_plane/ipc-lowered"}),
    case("plane-declined", "bf16", D(2, 86, 10, 10, 1),
         {"plane-declined/smem", "agg3_bwd_nchw2_dxdw/pxv2", "agg3_bwd_nchw2_dw/pxv2", "agg3_dx_plane/ipc-lowered"}),
    case("nchw-k3", "bf16", D(2, 16, 7, 7, 4), {"agg_fwd_nchw_k3", "agg_bwd_nchw_dxdw/K3", "agg_bwd_nchw_dx/K3", "agg_bwd_nchw_dw/K3"}),
    case("nchw-k3-fp32", "fp32", D(2, 12, 5, 9, 3), {"agg_fwd_nchw_k3", "agg_bwd_nchw_dxdw/K3"}),
    case("nchw-k5", "fp32", D(2, 16, 9, 11, 4, k=5), {"agg_fwd_nchw_k5", "agg_bwd_nchw_dxdw/K5", "agg_bwd_nchw_dx/K5",
                                                        "agg_bwd_nchw_dw/K5"}),
    case("nchw-k5-bf16", "bf16", D(2, 16, 12, 12, 8, k=5), {"agg_fwd_nchw_k5", "agg_bwd_nchw_dxdw/K5"}),
    case("limit-nchw2", "bf16", D(4097, 16, 4, 4, 16), {"nchw2-declined/N*wc", "agg_fwd_nchw_k3", "agg_bwd_nchw_dxdw/K3"}),
    # ---- grid-stride loops past grid_stride_blocks' cap on both SM counts
    case("loop-nchw-k5", "fp32", D(4, 32, 72, 72, 16, k=5),
         {"agg_fwd_nchw_k5/loop2@132", "agg_fwd_nchw_k5/loop2@114", "agg_bwd_nchw_dxdw/loop2@132"}),
    case("loop-nhwc-v4", "bf16", D(8, 48, 56, 56, 12, layout=NHWC),
         {"agg3_fwd_nhwc/loop2@132", "agg3_dx_nhwc/loop2@132", "agg3_dx_nhwc/loop2@114"}),
    case("loop-generic", "fp32", D(2, 64, 48, 48, 8, heads=2), {"agg_fwd_generic/loop2@132", "agg_dw_generic/loop2@114"}),
    # ---- generic kernels: heads 2, stride 2, dilation 2, k = 7, rectangular maps, fp64, on every layout
    case("gen-nchw-heads2", "fp32", D(2, 12, 5, 7, 4, heads=2), {"agg_fwd_generic/heads", "agg_dx_generic/layout0", "agg_dw_generic/rect"}),
    case("gen-nchw-s2", "bf16", D(2, 8, 9, 6, 4, s=2, p=1), {"agg_fwd_generic/stride", "agg_dx_generic/stride"}),
    case("gen-nchw-d2", "fp16", D(2, 8, 8, 7, 2, d=2), {"agg_fwd_generic/dilation", "agg_dw_generic/dilation"}),
    case("gen-nchw-k7", "bf16", D(2, 8, 9, 8, 4, k=7), {"agg_fwd_generic/k7", "agg_dx_generic/k7", "agg_dw_generic/k7"}),
    case("gen-nchw-fold2", "fp32", D(2, 16, 6, 6, 4, fold=2), {"agg_fwd_generic/fold2", "agg_dw_generic/fold2"}),
    case("gen-nchw-fp64", "fp64", D(2, 12, 6, 5, 4), {"agg_fwd_generic/layout0", "agg_dw_generic/layout0"}),
    case("gen-nhwc-heads2-pitch", "bf16", DP(2, 16, 5, 6, 4, heads=2, layout=NHWC),
         {"agg_fwd_generic/heads", "agg_dx_generic/layout1", "agg_dw_generic/heads"}),
    case("gen-nhwc-k7-s2", "fp32", D(2, 8, 11, 9, 2, k=7, s=2, p=2, layout=NHWC), {"agg_fwd_generic/k7", "agg_dw_generic/stride"}),
    case("gen-nhwc-fp64-fold2", "fp64", DP(2, 16, 5, 4, 4, fold=2, layout=NHWC, extra=1),
         {"agg_fwd_generic/fold2", "agg_dw_generic/layout1"}),
    case("gen-tap-s2-d2", "fp32", D(2, 16, 9, 8, 8, s=2, d=2, layout=TAP, gc=4),
         {"agg_fwd_generic/layout2", "agg_dx_generic/dilation", "agg_dw_generic/layout2"}),
    case("gen-tap-heads2-pitch", "bf16", DP(2, 16, 4, 6, 8, heads=2, layout=TAP, gc=4), {"agg_dw_generic/heads", "agg_dx_generic/heads"}),
    case("gen-tap-fp64-fold2", "fp64", D(2, 32, 5, 6, 8, fold=2, layout=TAP, gc=4), {"agg_fwd_generic/layout2", "agg_dw_generic/fold2"}),
    case("gen-tap-offset", "bf16", D(2, 64, 4, 5, 8, layout=TAP, gc=8), {"agg_fwd_generic/layout2", "agg_dx_generic/layout2"}, off=4),
    case("gen-tap-fp32-gc8", "fp32", D(2, 16, 4, 5, 8, layout=TAP, gc=8, fold=1), {"nhwc2_dw-declined/rep", "agg_dw_generic/layout2"}),
    # ---- the mix op (3x3 and 5x5 halves, NCHW)
    case("mix-fp32-plane", "fp32", D(2, 16, 12, 12, 4), {"agg_mix_fwd_nchw", "agg3_dxdw_plane", "agg_bwd_nchw_dxdw/ACC_DX",
                                                          "agg_bwd_nchw_dx/ACC_DX", "agg_bwd_nchw_dw/K5"}, op="mix"),
    case("mix-fp32-tma", "fp32", D(2, 16, 8, 8, 4), {"agg3_dx_nchw_tma", "agg3_dw_nchw_tma", "agg_bwd_nchw_dxdw/K5"}, op="mix"),
    case("mix-bf16", "bf16", D(2, 16, 10, 10, 4), {"agg_mix_fwd_nchw", "agg_mix_dx", "agg3_dw_plane", "agg_bwd_nchw_dw/K5"}, op="mix"),
    case("mix-fp16-rect", "fp16", D(2, 8, 6, 9, 2), {"agg_mix_dx", "agg_bwd_nchw_dw/K3", "agg_bwd_nchw_dw/K5"}, op="mix"),
    case("mix-fp64", "fp64", D(2, 8, 5, 6, 4), {"agg_fwd_generic", "agg_dx_generic/ACCUM", "agg_dw_generic"}, op="mix"),
    # ---- float operands: the widen-and-round steps of each family against fp64 under a tolerance
    case("float-nhwc2", "bf16", D(1, 64, 3, 256, 8, layout=TAP, gc=8), {"agg3_fwd_nhwc2", "agg3_dw_nhwc2"}, kind="float"),
    case("float-packet", "fp16", D(2, 48, 5, 7, 12, layout=NHWC), {"agg3_fwd_nhwc", "agg3_dw_nhwc"}, kind="float"),
    case("float-nchw2", "bf16", D(2, 32, 6, 12, 8), {"agg3_fwd_nchw2", "agg3_bwd_nchw2_dxdw"}, kind="float"),
    case("float-plane", "bf16", D(2, 64, 14, 14, 8), {"agg3_dxdw_plane"}, kind="float"),
    case("float-nchw-k3", "fp32", D(2, 16, 7, 7, 4), {"agg_fwd_nchw_k3", "agg_bwd_nchw_dxdw"}, kind="float"),
    case("float-nchw-k5", "bf16", D(2, 16, 9, 11, 4, k=5), {"agg_fwd_nchw_k5", "agg_bwd_nchw_dxdw"}, kind="float"),
    case("float-generic", "bf16", D(2, 16, 5, 6, 4, heads=2, layout=NHWC), {"agg_fwd_generic", "agg_dx_generic"}, kind="float"),
    case("float-mix", "bf16", D(2, 16, 10, 10, 4), {"agg_mix_fwd_nchw", "agg_mix_dx"}, op="mix", kind="float"),
]

ENTRY_NAMES = [
    "agg3_fwd_tma", "agg3_dx_tma", "agg3_dw_tma", "agg3_fwd_nhwc2", "agg3_dx_nhwc2", "agg3_dw_nhwc2", "agg3_fwd_nhwc", "agg3_dx_nhwc",
    "agg3_dw_nhwc", "agg3_fwd_nchw_tma", "agg3_dx_nchw_tma", "agg3_dw_nchw_tma", "agg3_fwd_nchw2", "agg3_bwd_nchw2_dxdw",
    "agg3_bwd_nchw2_dx", "agg3_bwd_nchw2_dw", "agg3_dxdw_plane", "agg3_dx_plane", "agg3_dw_plane", "agg_fwd_nchw_k3",
    "agg_fwd_nchw_k5", "agg_bwd_nchw_dxdw", "agg_bwd_nchw_dx", "agg_bwd_nchw_dw", "agg_fwd_generic", "agg_dx_generic", "agg_dw_generic",
    "agg_mix_fwd_nchw", "agg_mix_dx"]

REQUIRED = set(ENTRY_NAMES)
for _k in ("fwd", "dx", "dw"):
    REQUIRED |= {"agg3_%s_nhwc/vec%d" % (_k, v) for v in (8, 4, 2, 1)}
    REQUIRED |= {"agg3_%s_nhwc/%s" % (_k, o) for o in ("tap", "plain")}
    REQUIRED |= {"agg3_%s_nhwc/fold2" % _k, "agg3_%s_nhwc/fold1" % _k}
for _k in ("fwd", "dx"):
    REQUIRED |= {"agg3_%s_nhwc2/%s" % (_k, t) for t in ("px2", "px1", "fold1", "fold2", "interior", "edge-only")}
REQUIRED |= {"agg3_fwd_nhwc2/plain", "agg3_fwd_nhwc2/tap"}
REQUIRED |= {"agg3_dw_nhwc2/%s" % t for t in ("gqw1", "gqw2", "gqw4", "fold1", "fold2", "interior", "edge-only")}
REQUIRED |= {"nhwc2_dw-declined/rep", "nhwc2_dw-declined/fold", "nhwc2_dw-declined/gqw"}
REQUIRED |= {"agg3_fwd_nchw2/pxv4", "agg3_fwd_nchw2/pxv2"}
REQUIRED |= {"agg3_bwd_nchw2_%s/pxv%d" % (k, v) for k in ("dxdw", "dx", "dw") for v in (4, 2)}
REQUIRED |= {"agg3_%s_plane/%s" % (k, t) for k in ("dxdw", "dx", "dw") for t in ("ipc1", "ipc>1", "ipc-lowered")}
REQUIRED |= {"plane-declined/smem"}
REQUIRED |= {"agg_bwd_nchw_%s/K%d" % (k, K) for k in ("dxdw", "dx", "dw") for K in (3, 5)}
REQUIRED |= {"agg_bwd_nchw_dxdw/ACC_DX", "agg_bwd_nchw_dx/ACC_DX"}
for _k in ("fwd", "dx", "dw"):
    REQUIRED |= {"agg_%s_generic/%s" % (_k, t) for t in ("heads", "stride", "dilation", "k7", "rect", "layout0", "layout1", "layout2",
                                                          "fold2")}
REQUIRED |= {"agg_dx_generic/ACCUM"}
# (agg3_dw_nhwc2's own grid.y limit is not among them: it is reached only where the TMA kernel declines a rep-8 call, which takes
# W + 2 > 256 or a 17-pixel row of 512 channels, times 65536 rows -- gigabytes)
REQUIRED |= {"nhwc2_fwd-declined/grid.y", "nhwc2_dx-declined/grid.y", "nchw2-declined/N*wc"}
REQUIRED |= {"%s/loop2@%d" % (n, s) for n in ("agg_fwd_nchw_k5", "agg3_fwd_nhwc", "agg_fwd_generic") for s in SMS_H100}
# the same kernels with pitches larger than dense (the case's descriptor has pitches) and with pointer offsets: see test_pitch_coverage
PITCHED_KERNELS = {"agg3_fwd_tma", "agg3_dx_tma", "agg3_dw_tma", "agg3_fwd_nhwc2", "agg3_dx_nhwc2", "agg3_dw_nhwc2", "agg3_fwd_nhwc",
                   "agg3_dx_nhwc", "agg3_dw_nhwc", "agg_fwd_generic", "agg_dx_generic", "agg_dw_generic"}
FLOAT_FAMILIES = {"agg3_fwd_nhwc2", "agg3_fwd_nhwc", "agg3_fwd_nchw2", "agg3_dxdw_plane", "agg_fwd_nchw_k3", "agg_fwd_nchw_k5",
                  "agg_fwd_generic", "agg_mix_fwd_nchw", "agg_mix_dx"}


# ================================================================================================ fp64 reference (header semantics)
def weight_channel(C, wc, fold):
    """include/cotb200.h: input channel c uses weight channel (c/(C/F))*(wc/F) + (c%(C/F))%(wc/F) (F = fold; c % wc when F = 1)"""
    F_ = max(fold, 1)
    Cf, wcf = C // F_, wc // F_
    c = torch.arange(C)
    return (c // Cf) * wcf + (c % Cf) % wcf


def weight_column(heads, wc, K2, layout, gc):
    """[heads, wc, K2] column of (head, g, tap) in an NHWC weight row (include/cotb200.h): head*wc*K2 + g*K2 + tap, or with NHWC_TAP
    head*wc*K2 + ((g/gc)*K2 + tap)*gc + g%gc"""
    h = torch.arange(heads)[:, None, None]
    g = torch.arange(wc)[None, :, None]
    t = torch.arange(K2)[None, None, :]
    if layout == TAP:
        return h * wc * K2 + ((g // gc) * K2 + t) * gc + g % gc
    return h * wc * K2 + g * K2 + t


def agg_ref(x, w, d):
    """y[n, head*C + c, ho, wo] = sum_tap w[n, head, wch(c), tap, ho, wo] * x[n, c, ho*s - p + kh*d, wo*s - p + kw*d] (zero outside),
    canonical layouts x [N,C,H,W], w [N,heads,wc,K2,Ho,Wo]; differentiable"""
    N, C = x.shape[:2]
    unf = F.unfold(x, (d.kh, d.kw), dilation=(d.dh, d.dw), padding=(d.ph, d.pw), stride=(d.sh, d.sw))
    unf = unf.view(N, 1, C, d.kh * d.kw, d.ho, d.wo)
    wsel = w[:, :, weight_channel(C, d.wc, d.fold).to(w.device)]
    return (wsel * unf).sum(3).reshape(N, d.heads * C, d.ho, d.wo)


def mix_descs(d):
    d2 = Desc(d.n, d.c, d.h, d.w, d.wc, k=MIX_K2, heads=d.heads, s=d.sh, d=d.dh, p=MIX_P2)
    return d, d2


def mix_ref(x, w1, w2, d):
    d1, d2 = mix_descs(d)
    return torch.cat([agg_ref(x, w1, d1), agg_ref(x, w2, d2)], 1)


# ================================================================================================ tests
def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


ANCHORS = {
    "agg_zeropad.cu": [
        "if (d->c % g.fold || d->wc % g.fold || (d->c / g.fold) % (d->wc / g.fold)) {",
        "g.x_sc = 1; g.x_sw = d->x_sp ? d->x_sp : g.C; g.x_sh = g.x_sw * g.W; g.x_sn = d->x_sn ? d->x_sn : g.x_sh * g.H;",
        "g.w_sw = d->w_sp ? d->w_sp : J; g.w_sh = g.w_sw * g.WO; g.w_sn = d->w_sn ? d->w_sn : g.w_sh * g.HO;",
        "g.y_sc = 1; g.y_sw = d->y_sp ? d->y_sp : (long long)g.C * g.heads; g.y_sh = g.y_sw * g.WO;",
        "return g.KH == K && g.KW == K && g.SH == 1 && g.SW == 1 && g.DH == 1 && g.DW == 1 && g.PH == K / 2 && g.PW == K / 2 &&\n"
        "         g.heads == 1;",
        "return a < (1LL << 31) && b < (1LL << 31) && c < (1LL << 31);",
        "if (!is_same3(g, 3) || !fits32(g)) return 0;",
        "for (int vec = 16 / (int)sizeof(T); vec >= 1; vec >>= 1) {",
        "if (g.layout == COTB200_NHWC_TAP && vec != g.gc) continue;",
        "if (bytes < 4 && vec != 1) continue;",
        "if (g.wcf % vec) continue;",
        "if (!oks(g.x_sw) || !oks(g.x_sn) || !oks(g.w_sw) || !oks(g.w_sn) || !oks(g.y_sw) || !oks(g.y_sn)) continue;",
        "if (agg_tma_fwd<T>(nhwc2_args(g), x, w, y, st, &rc2)) return rc2;",
        "if (nhwc2_fwd<T>(nhwc2_args(g), x, w, y, st, &rc2)) return rc2;",
        "if (g.layout == COTB200_NCHW && nofold(g) && fits32(g) && is_same3(g, 3) && g.w_sn == (long long)g.wc * 9 * g.H * g.W) {",
        "if (g.x_sn == (long long)g.C * g.H * g.W &&\n        nchw_tma_launch<T>(0, g.N, g.C, g.H, g.W, g.wc, g.x_sn, 0, g.y_sn, x, w, y, st, &rc2)) return rc2;",
        "if (nchw2_fwd<T>(g.N, g.C, g.H, g.W, g.wc, g.y_sn, x, w, y, st, &rc2)) return rc2;",
        "if (g.layout == COTB200_NCHW && nofold(g) && fits32(g) && (is_same3(g, 3) || is_same3(g, 5))) {",
        "const int vec = nhwc_vec<T>(g, x, w, y);",
        "const int total = g.N * g.H * g.W * (g.C / vec);",
        "if (g.layout == COTB200_NCHW && nofold(g) && fits32(g) && is_same3(g, 3) && !acc_dx && g.w_sn == (long long)g.wc * 9 * g.H * g.W) {",
        "if (g.H * g.W <= 256 && nchw_plane_launch<T>(dx && dw ? 3 : (dx ? 1 : 2), g.N, g.C, g.H, g.W, g.wc, g.x_sn, g.y_sn, g.w_sn, dy, x, w,",
        "if (dx && nchw_tma_launch<T>(1, g.N, g.C, g.H, g.W, g.wc, g.y_sn, 0, g.x_sn, dy, w, dx, st, &rc2)) { if (rc2) return rc2; done_dx = 1; }",
        "if (dw && nchw_tma_launch<T>(2, g.N, g.C, g.H, g.W, g.wc, g.x_sn, g.y_sn, g.w_sn, x, dy, dw, st, &rc2)) { if (rc2) return rc2; done_dw = 1; }",
        "if (nchw2_bwd<T>(g.N, g.C, g.H, g.W, g.wc, g.y_sn, dy, x, w, done_dx ? nullptr : dx, done_dw ? nullptr : dw, st, &rc2)) return rc2;",
        "if (g.layout == COTB200_NHWC_TAP && !acc_dx && is_same3(g, 3)) {",
        "if (dx && agg_tma_dx<T>(nhwc2_args(g), dy, w, dx, st, &rc2)) { if (rc2) return rc2; dx = nullptr; }",
        "if (dw && agg_tma_dw<T>(nhwc2_args(g), dy, x, dw, st, &rc2)) { if (rc2) return rc2; dw = nullptr; }",
        "if (dx && nhwc2_dx<T>(nhwc2_args(g), dy, w, dx, st, &rc2)) { if (rc2) return rc2; dx = nullptr; }",
        "if (dw && nhwc2_dw<T>(nhwc2_args(g), dy, x, dw, st, &rc2)) { if (rc2) return rc2; dw = nullptr; }",
        "if (g.layout != COTB200_NCHW && !acc_dx) {",
        "const int vec = nhwc_vec<T>(g, dy, x, w);",
        "if (vec && okp(dx) && okp(dw)) {",
        "const int total = g.N * g.H * g.W * (g.wc / V);",
        "const long long total = (long long)g.N * g.heads * g.wc * g.K2 * g.HO * g.WO;",
        "g1.y_sn *= 2; g2.y_sn *= 2;",
        "if (is_same3(g1, 3) && is_same3(g2, 5) && fits32(g2) && 2 * half * g1.N < (1LL << 31)) {",
        "if (sizeof(T) >= 4 && is_same3(g1, 3) && is_same3(g2, 5) && fits32(g2)) {",
        "return bwd_impl<T>(g2, (const T*)dy + half, (const T*)x, (const T*)w2, (T*)dx, (T*)dw2, dx != nullptr, st);",
        "rc = bwd_impl<T>(g1, (const T*)dy, (const T*)x, (const T*)w1, (T*)nullptr, (T*)dw1, false, st);",
    ],
    "agg_nhwc2.cu": [
        "if (wcf % VEC || a.C % VEC) return false;",
        "if (tap && (a.gc < VEC || a.gc % VEC || a.wc % a.gc)) return false;",
        "for (long long s : strides) if (s > lim || (s * (long long)sizeof(T)) % 16) return false;",
        "if ((long long)a.H * a.W * a.x_sp > lim || (long long)a.H * a.W * a.w_sp > lim || (long long)a.H * a.W * a.y_sp > lim) return false;",
        "if ((long long)a.N * a.H > 65535LL * 32768) return false;",
        "if ((long long)a.N * a.H > 2147483647LL) return 0;",
        "const int px = (a.W % 2 == 0) ? 2 : 1;",
        "if (grid.y > 65535) {   // fold rows into x when the batch is huge",
        "if (grid.y > 65535) return 0;",
        "if (a.C / a.wc != 8) return 0;",
        "int gqw = GQ >= 4 ? 4 : GQ;",
        "if (GQ % gqw || (gqw != 1 && gqw != 2 && gqw != 4)) return 0;",
        "if (a.fold > 1 && (a.wc / a.fold) % (gqw * VEC)) return 0;",
        "const bool interior = h >= 1 && h + 1 < g.H && w0 >= 1 && w0 + PX < g.W;",
    ],
    "agg_nchw2.cu": [
        "for (int pxv = 4; pxv >= 2; pxv >>= 1) {",
        "if (W % pxv) continue;",
        "if (!pxv || (long long)N * wc > 65535 || (y_sn * (long long)sizeof(T)) % (pxv * sizeof(T))) return 0;",
        "if (!pxv || (long long)N * wc > 65535 || (dy_sn * (long long)sizeof(T)) % (pxv * sizeof(T))) return 0;",
        "COTB200_PROF_B(dx && dw ? \"agg3_bwd_nchw2_dxdw\" : (dx ? \"agg3_bwd_nchw2_dx\" : \"agg3_bwd_nchw2_dw\")",
    ],
    "agg_nchw_plane.cu": [
        "if (HW > 256 || HW < 100 || C % wc) return 0;",
        "int ipc = 256 / HW;",
        "const int PP = (H + 2) * (W + 2);",
        "while (ipc > 1 && (size_t)ipc * rep * PP * (dwm ? 2 : 1) * sizeof(float) > 96 * 1024) --ipc;",
        "if (smem > 96 * 1024) return 0;",
        "if (items_ll > 2000000000LL) return 0;",
    ],
    "agg_nchw_tma.cu": [
        "if (W % 4 == 0) pxv = 4; else if (W % 2 == 0 && es == 4) pxv = 2;",
        "if (!pxv || rep > 16 || rep < 1) return 0;",
        "if (((long long)W * es) % 16 || ((long long)H * W * es) % 16) return 0;",
        "if ((a_sn * es) % 16 || (b_sn * es) % 16 || (out_sn * es) % (pxv * es)) return 0;",
        "if (!aligned16(A) || !aligned16(Bp) || !aligned16(out)) return 0;",
        "if (W + 2 * (pxv > al ? pxv : al) > 256 || H < 1 || N < 1) return 0;",
    ],
    "agg_tma.cu": [
        "if (a.layout != COTB200_NHWC_TAP) return false;",
        "if ((a.C * (int)sizeof(T)) % 128 || wcf % VEC || a.gc < VEC || a.gc % VEC || a.wc % a.gc) return false;",
        "if (((uintptr_t)A | (uintptr_t)Bp | (uintptr_t)out) & 15) return false;",
        "for (long long sv : strides) if ((sv * (long long)sizeof(T)) % 16) return false;",
        "if (a.W + 2 > 256) return false;",
        "p.jboxes = (p.J + 255) / 256;",
        "while (p.J % p.jboxes) ++p.jboxes;",
        "if ((p.jbox * (int)sizeof(T)) % 16) return false;",
        "if (o_sp > 2147483647LL) return false;",
    ],
}


# Pred.add's loop=(total, per_sm): grid_stride_blocks (common.cuh) and the (threads, per_sm) each grid-stride launch passes it
GRID_ANCHORS = {
    "common.cuh": [
        "inline int grid_stride_blocks(long long items, int threads, int per_sm) {",
        "const long long need = (items + threads - 1) / threads;",
        "const long long cap = (long long)num_sms() * per_sm;",
        "return (int)(need < 1 ? 1 : need < cap ? need : cap);",
    ],
    "agg_zeropad.cu": [
        "const int grid = grid_stride_blocks(total, 256, 8);",
        "agg_fwd_generic<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>(x, w, y, g, total);",
        "agg_dw_generic<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>(dy, x, dw, g, total);",
        "agg_dx_generic2<T><<<grid_stride_blocks(total, 256, 16), 256, 0, st>>>((const T*)dy, (const T*)w1, g1, (const T*)dy + half,",
        "agg_mix_fwd_nchw_fast<T><<<grid_stride_blocks(total, 256, 8), 256, 0, st>>>(",
    ],
}


def _missing_anchors(fname, anchors):
    squash = lambda s: re.sub(r"\s+", " ", s)
    src = squash(_src(fname))
    return [a for a in anchors if squash(a) not in src]


@pytest.mark.parametrize("fname", sorted(ANCHORS))
def test_dispatch_anchors(fname):
    """the conditions the mirror copies are still the ones in the sources (whitespace-insensitive)"""
    missing = _missing_anchors(fname, ANCHORS[fname])
    assert not missing, "%s no longer contains (update the mirror in this file): %s" % (fname, missing)


def test_grid_stride_anchors():
    """the grid-stride sizing the mirror copies (whitespace-insensitive)"""
    for fname, anchors in sorted(GRID_ANCHORS.items()):
        missing = _missing_anchors(fname, anchors)
        assert not missing, "%s no longer contains (update the mirror in this file): %s" % (fname, missing)


def test_every_launch_name_is_profiled():
    """the profiler names the mirror predicts are the names the sources record"""
    src = "".join(_src(f) for f in ("agg_zeropad.cu", "agg_nhwc2.cu", "agg_nchw2.cu", "agg_nchw_plane.cu", "agg_nchw_tma.cu",
                                    "agg_tma.cu"))
    for n in ENTRY_NAMES:
        assert '"%s"' % n in src, n


def test_nchw_tma_first_tile_fits():
    """nchw_tma_launch's tile loop always finds a one-row tile with >= 2 stages once its early conditions hold (rep <= 16,
    W + 2 * halo <= 256), so nchw_tma_ok needs no copy of the loop"""
    for es in (2, 4):
        al = 16 // es
        for pxv in ((4, 2) if es == 4 else (4,)):
            halo = max(pxv, al)
            BWa = tp._rup(256, al)                      # W + 2 * halo <= 256
            BWb = tp._rup(256 - 2 * halo, al)
            rep = 16
            for mode in (0, 1, 2):
                a = tp._rup(rep * 3 * BWa * es, 128)
                b = tp._rup(9 * BWb * es if mode == 0 else 9 * 3 * BWa * es if mode == 1 else rep * BWb * es, 128)
                assert (a + b) * 2 <= 200 * 1024 and (200 * 1024) // (a + b) >= 2


def test_case_names_unique_and_valid():
    names = [c.name for c in CASES]
    assert len(names) == len(set(names))
    for c in CASES:
        resolve(c.desc)
        assert c.dt in ES and c.kind in ("int", "float") and c.op in ("agg", "mix")
        if c.op == "mix":
            assert c.desc.layout == NCHW and c.desc.kh == 3 and c.desc.ph == 1


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.name)
def test_case_reaches_what_it_exists_for(c):
    got = case_tags(c)
    assert c.expect <= got, "%s: expected %s; the calls reach %s" % (c.name, sorted(c.expect - got), sorted(got))
    assert case_bytes(c) < 400e6, case_bytes(c)


def test_cases_cover_every_branch():
    got = set()
    for c in CASES:
        got |= case_tags(c)
    missing = REQUIRED - got
    assert not missing, sorted(missing)


def test_pitch_coverage():
    """every NHWC kernel runs at least once with pitches larger than dense, and every packet width is also reached through pointer
    offsets that lower it"""
    pitched, offset_vecs = set(), set()
    for c in CASES:
        tags = case_tags(c)
        if c.desc.layout != NCHW and c.desc.x_sp:
            pitched |= tags & PITCHED_KERNELS
        if any(c.offs.values()):
            offset_vecs |= {t for t in tags if "/vec" in t or "/pxv" in t or t.startswith("agg_fwd_generic")}
    assert PITCHED_KERNELS <= pitched, sorted(PITCHED_KERNELS - pitched)
    for t in ("agg3_fwd_nhwc/vec2", "agg3_fwd_nhwc/vec1", "agg3_bwd_nchw2_dxdw/pxv2", "agg_fwd_generic"):
        assert t in offset_vecs, t


def test_float_cases_cover_every_family():
    fam = set()
    for c in CASES:
        if c.kind == "float":
            fam |= case_tags(c) & FLOAT_FAMILIES
    assert fam == FLOAT_FAMILIES, sorted(FLOAT_FAMILIES - fam)


# ------------------------------------------------------------------------------------------------ operand bounds
INT_LIMIT = {"bf16": 256, "fp16": 2048, "fp32": 1 << 22, "fp64": 1 << 40}


def amplitude(c):
    """largest a in {2, 1} for operands drawn from [-a, a] such that every output is an integer the storage type holds:
    |y| <= K2 * a^2, |dX| <= heads * K2 * a^2 (both mix halves: (9 + 25) * a^2), |dW| <= rep * a^2"""
    d = c.desc
    K2 = d.kh * d.kw + (MIX_K2 * MIX_K2 if c.op == "mix" else 0)
    worst = max(d.heads * K2, d.c // d.wc)
    for a in (2, 1):
        if worst * a * a <= INT_LIMIT[c.dt]:
            return a
    raise AssertionError("%s: outputs not exact even at amplitude 1" % c.name)


def tensor_extent(c):
    """{tensor: (shape of the described slice, strides, elements of the whole buffer from its offset)}"""
    d = c.desc
    out = {}
    if c.op == "mix":
        shapes = {"x": (d.n, d.c, d.h, d.w), "w1": (d.n, d.heads, d.wc, 9, d.ho, d.wo), "w2": (d.n, d.heads, d.wc, 25, d.ho, d.wo),
                  "y": (d.n, 2 * d.heads * d.c, d.ho, d.wo)}
        shapes.update(dy=shapes["y"], dx=shapes["x"], dw1=shapes["w1"], dw2=shapes["w2"])
        for k, s in shapes.items():
            out[k] = (s, _dense_strides(s), math.prod(s))
        return out
    g = resolve(d)
    J = d.heads * d.wc * d.kh * d.kw
    if d.layout == NCHW:
        shapes = {"x": (d.n, d.c, d.h, d.w), "w": (d.n, d.heads, d.wc, d.kh * d.kw, d.ho, d.wo), "y": (d.n, d.heads * d.c, d.ho, d.wo)}
        for k, s in shapes.items():
            out[k] = (s, _dense_strides(s), math.prod(s))
    else:
        for k, (H, W, Cn, sp, sn) in {"x": (d.h, d.w, d.c, g.x_sw, g.x_sn), "w": (d.ho, d.wo, J, g.w_sw, g.w_sn),
                                      "y": (d.ho, d.wo, d.heads * d.c, g.y_sw, g.y_sn)}.items():
            s = (d.n, H, W, Cn)
            st = (sn, W * sp, sp, 1)
            out[k] = (s, st, (d.n - 1) * sn + (H * W - 1) * sp + Cn + (sn - H * W * sp if sn > H * W * sp else 0))
    out["dy"], out["dx"], out["dw"] = out["y"], out["x"], out["w"]
    return out


def _dense_strides(s):
    st, acc = [], 1
    for n in reversed(s):
        st.append(acc)
        acc *= n
    return tuple(reversed(st))


def case_bytes(c):
    es = ES[c.dt]
    return sum((c.offs[k] + n) * es for k, (_, _, n) in tensor_extent(c).items())


def test_amplitudes_exact():
    for c in CASES:
        if c.kind == "int":
            amplitude(c)


# ------------------------------------------------------------------------------------------------ the reference
def test_reference_matches_oracle_nchw():
    """agg_ref (header semantics) == oracle.agg_ref's unfold restatement for NCHW, fold 1, and == the reference's batch-fold view for
    fold 2 (channel halves folded into the batch, the weight channels split the same way)"""
    from oracle import agg_ref as oracle
    gen = torch.Generator().manual_seed(7)
    for kw in (dict(k=3), dict(k=5), dict(k=3, s=2, p=1), dict(k=3, d=2), dict(k=3, heads=2), dict(k=(3, 5), p=(1, 0))):
        d = Desc(2, 12, 7, 9, 4, **kw)
        x = torch.randn(2, 12, 7, 9, generator=gen, dtype=torch.float64)
        w = torch.randn(2, d.heads, 4, d.kh * d.kw, d.ho, d.wo, generator=gen, dtype=torch.float64)
        want = oracle.agg_zeropad_unfold(x, w, (d.kh, d.kw), (d.sh, d.sw), (d.ph, d.pw), (d.dh, d.dw))
        assert torch.allclose(agg_ref(x, w, d), want, rtol=0, atol=1e-12), kw
    d = Desc(2, 16, 6, 5, 4, fold=2)
    x = torch.randn(2, 16, 6, 5, generator=gen, dtype=torch.float64)
    w = torch.randn(2, 1, 4, 9, 6, 5, generator=gen, dtype=torch.float64)
    want = oracle.agg_zeropad_unfold(x.reshape(4, 8, 6, 5), w.reshape(4, 1, 2, 9, 6, 5), 3, 1, 1, 1).reshape(2, 16, 6, 5)
    assert torch.allclose(agg_ref(x, w, d), want, rtol=0, atol=1e-12)
    d = Desc(2, 8, 6, 7, 4)
    w2 = torch.randn(2, 1, 4, 25, 6, 7, generator=gen, dtype=torch.float64)
    x = torch.randn(2, 8, 6, 7, generator=gen, dtype=torch.float64)
    w = torch.randn(2, 1, 4, 9, 6, 7, generator=gen, dtype=torch.float64)
    assert torch.allclose(mix_ref(x, w, w2, d), oracle.agg_zeropad_mix_unfold(x, w, w2, 3, 5, 1, 1, 2, 1), rtol=0, atol=1e-12)


def test_tap_columns_follow_the_header():
    """NHWC_TAP: tap-major chunks of gc weight channels; the plain order is the channels_last view of [heads, wc, K2]"""
    col = weight_column(1, 16, 9, TAP, 8)
    assert col[0, 0, 0] == 0 and col[0, 1, 0] == 1 and col[0, 0, 1] == 8 and col[0, 8, 0] == 72 and col[0, 15, 8] == 143
    assert sorted(col.flatten().tolist()) == list(range(144))
    assert (weight_column(2, 4, 9, NHWC, 0).flatten() == torch.arange(72)).all()
    assert weight_channel(96, 12, 2).tolist()[:14] == [0, 1, 2, 3, 4, 5, 0, 1, 2, 3, 4, 5, 0, 1]
    assert weight_channel(96, 12, 2).tolist()[48:50] == [6, 7]


# ------------------------------------------------------------------------------------------------ the production table
# model: (resolution, [(kind, C, H, W, layers)]) -- the CoT / CoXt layers of the model (cot_layers() order of stages)
PRODUCTION_MODELS = {
    "cotnet50": (224, [(64, 56, 56, 1, 3), (128, 28, 28, 1, 4), (256, 14, 14, 1, 6), (512, 7, 7, 1, 3)]),
    "cotnext50_2x48d": (224, [(96, 56, 56, 2, 3), (192, 28, 28, 2, 4), (384, 14, 14, 2, 6), (768, 7, 7, 2, 3)]),
    "se_cotnetd_50": (224, [(256, 14, 14, 1, 3), (512, 7, 7, 1, 3)]),
    "se_cotnetd_101": (224, [(256, 14, 14, 1, 12), (512, 7, 7, 1, 3)]),
    "se_cotnetd_152": (320, [(256, 40, 40, 1, 1), (256, 20, 20, 1, 17), (512, 20, 20, 1, 1), (512, 10, 10, 1, 2)]),
}

# hand-checked: (C, H, W, fold) -> (eval and training forward, training backward with dX and dW) at the bench's batch of 256
PRODUCTION_TABLE = {
    (64, 56, 56, 1): ("agg3_fwd_tma", ("agg3_dx_tma", "agg3_dw_tma")),
    (128, 28, 28, 1): ("agg3_fwd_tma", ("agg3_dx_tma", "agg3_dw_tma")),
    (256, 14, 14, 1): ("agg3_fwd_tma", ("agg3_dx_tma", "agg3_dw_tma")),
    (512, 7, 7, 1): ("agg3_fwd_tma", ("agg3_dx_tma", "agg3_dw_tma")),
    # 40 x 40 rows of 256 / 512 channels: the one-row tile of x (4 or 8 slabs of 42 x 3 pixels) plus its weights exceed 72 KB
    (256, 40, 40, 1): ("agg3_fwd_nhwc2", ("agg3_dx_nhwc2", "agg3_dw_nhwc2")),
    # dX's haloed weight band (3 x 22 pixels x 288 weights) does not fit a 72 KB stage next to x: dX on nhwc2
    (256, 20, 20, 1): ("agg3_fwd_tma", ("agg3_dx_nhwc2", "agg3_dw_tma")),
    (512, 20, 20, 1): ("agg3_fwd_nhwc2", ("agg3_dx_nhwc2", "agg3_dw_nhwc2")),
    (512, 10, 10, 1): ("agg3_fwd_tma", ("agg3_dx_nhwc2", "agg3_dw_tma")),
    # CoXt stages 1-2: wc / fold = 6 / 12 is no multiple of 8, so tap_chunk gives the plain order: packet kernels of width 2 / 4
    (96, 56, 56, 2): ("agg3_fwd_nhwc", ("agg3_dx_nhwc", "agg3_dw_nhwc")),
    (192, 28, 28, 2): ("agg3_fwd_nhwc", ("agg3_dx_nhwc", "agg3_dw_nhwc")),
    (384, 14, 14, 2): ("agg3_fwd_tma", ("agg3_dx_nhwc2", "agg3_dw_tma")),
    (768, 7, 7, 2): ("agg3_fwd_tma", ("agg3_dx_nhwc2", "agg3_dw_tma")),
}


def production_calls(C, H, W, fold, N=256):
    from cotnet_b200 import fused
    gc = fused.tap_chunk(C // 8, fold)
    d = _prod_desc(C, H, W, fold, gc, N)
    offs = dict.fromkeys(TENSORS, 0)
    return predict_fwd(d, "bf16", offs), predict_bwd(d, "bf16", offs, True, True)


def _strip_loops(launches):
    return {(n, frozenset(t for t in tags if not t.startswith("loop2@"))) for n, tags in launches}


def test_production_geometries_follow_the_models():
    """PRODUCTION_MODELS is what the models build: every CoT / CoXt layer's input shape at the model's resolution (the layers
    replaced by a shape recorder, the rest of the network run on the CPU at batch 1)"""
    from cotnet_b200 import backbone, backbone_hybrid, cot_layer
    seen = []

    def rec(self, x):
        seen.append((x.shape[1], x.shape[2], x.shape[3], getattr(self, "dw_group", 1)))
        return x

    mp = pytest.MonkeyPatch()
    mp.setattr(cot_layer.CotLayer, "forward", rec)
    mp.setattr(cot_layer.CoXtLayer, "forward", rec)
    try:
        for name, (res, layers) in PRODUCTION_MODELS.items():
            ctor = getattr(backbone, name, None) or backbone_hybrid.MODELS[name]
            m = ctor().eval()
            seen.clear()
            with torch.no_grad():
                m(torch.zeros(1, 3, res, res))
            got = sorted(Counter(seen).items(), key=lambda kv: (-kv[0][1], kv[0][0]))
            assert [k + (v,) for k, v in got] == layers, (name, got)
    finally:
        mp.undo()


def test_production_table():
    """every production call maps to the pinned kernels, and each (kernel, sub-branch) pair it takes is run by a case of CASES at
    that exact C, wc, fold, gc and H x W"""
    geos = {(C, H, W, f) for _, layers in PRODUCTION_MODELS.values() for C, H, W, f, _ in layers}
    assert geos == set(PRODUCTION_TABLE) == set(PROD_GEOS)
    for (C, H, W, fold), (fwd_name, bwd_names) in PRODUCTION_TABLE.items():
        from cotnet_b200 import fused
        assert PROD_GEOS[(C, H, W, fold)] == fused.tap_chunk(C // 8, fold)
        pf, pb = production_calls(C, H, W, fold)
        assert list(pf.names()) == [fwd_name], (C, H, W, fold, pf.launches)
        assert sorted(pb.names()) == sorted(bwd_names) and all(v == 1 for v in pb.names().values()), (C, H, W, fold, pb.launches)
        want = _strip_loops(pf.launches) | _strip_loops(pb.launches)
        have = set()
        for c in CASES:
            d = c.desc
            if (c.dt == "bf16" and c.op == "agg" and (d.c, d.h, d.w, d.fold, d.wc, d.gc) == (C, H, W, fold, C // 8, PROD_GEOS[(C, H, W, fold)])
                    and d.layout == (TAP if d.gc else NHWC) and not any(c.offs.values()) and not d.x_sp):
                P = predict(c)
                have |= _strip_loops(P["fwd"].launches) | _strip_loops(P["dxdw"].launches)
        assert want <= have, (C, H, W, fold, sorted(want - have))


def test_production_sub_branches():
    """the sub-branches the production calls take (the CoXt stages 1-2 on the packet kernels at width 2 and 4 with fold 2)"""
    pf, pb = production_calls(96, 56, 56, 2)
    assert _strip_loops(pf.launches) == {("agg3_fwd_nhwc", frozenset({"vec2", "plain", "fold2"}))}
    assert _strip_loops(pb.launches) == {("agg3_dx_nhwc", frozenset({"vec2", "plain", "fold2"})),
                                         ("agg3_dw_nhwc", frozenset({"vec2", "plain", "fold2"}))}
    pf, _ = production_calls(192, 28, 28, 2)
    assert _strip_loops(pf.launches) == {("agg3_fwd_nhwc", frozenset({"vec4", "plain", "fold2"}))}
    pf, pb = production_calls(512, 20, 20, 1)
    assert _strip_loops(pb.launches) == {("agg3_dx_nhwc2", frozenset({"px2", "tap", "fold1", "interior"})),
                                         ("agg3_dw_nhwc2", frozenset({"gqw4", "fold1", "interior"}))}
