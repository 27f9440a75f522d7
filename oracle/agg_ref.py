"""CPU restatement of the LocalConv ("aggregation_zeropad") operator.  TEST INFRASTRUCTURE ONLY.

Two independent restatements of the same operator:

* ``*_loops``  -- numpy, follows the reference CUDA kernels' index math tap by tap:
    forward          cupy_layers/aggregation_zeropad.py:20-46
    input backward   cupy_layers/aggregation_zeropad.py:48-79
    weight backward  cupy_layers/aggregation_zeropad.py:81-110
    mix forward      cupy_layers/aggregation_zeropad_mix.py:20-74
    mix backward     cupy_layers/aggregation_zeropad_mix.py:76-207
* ``*_unfold`` -- torch, the identity the reference's self-tests assert the kernels equal
    (cupy_layers/aggregation_zeropad.py:249-251, aggregation_zeropad_mix.py:360-366);
    differentiable, so autograd gives dX / dW.

``tests/test_oracle.py`` pins one against the other at the reference self-test shapes with
the reference's own gate (max-abs < 1e-9 in fp64).

Layouts are the reference's: x [N,C,H,W]; w [N,heads,wc,kh*kw,Ho,Wo]; out [N,heads*C,Ho,Wo].
"""
import numpy as np
import torch


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def out_size(H, W, k, s, p, d):
    k, s, p, d = _pair(k), _pair(s), _pair(p), _pair(d)
    # aggregation_zeropad.py:119-120
    Ho = int((H + 2 * p[0] - (d[0] * (k[0] - 1) + 1)) / s[0] + 1)
    Wo = int((W + 2 * p[1] - (d[1] * (k[1] - 1) + 1)) / s[1] + 1)
    return Ho, Wo


# --------------------------------------------------------------------------- numpy loops
def agg_zeropad_fwd_loops(x, w, k=3, s=1, p=0, d=1):
    """aggregation_zeropad.py:20-46.  out[n, head*C + c, h, w] = sum_tap w[n,head,c%wc,tap,h,w] * x[n,c,h_in,w_in]."""
    k, s, p, d = _pair(k), _pair(s), _pair(p), _pair(d)
    N, C, H, W = x.shape
    _, heads, wc, K2, Ho, Wo = w.shape
    assert K2 == k[0] * k[1] and C % wc == 0
    out = np.zeros((N, heads, C, Ho, Wo), dtype=np.result_type(x.dtype, w.dtype))
    cidx = np.arange(C) % wc
    for kh in range(k[0]):
        for kw in range(k[1]):
            tap = kh * k[1] + kw
            # valid output range for this tap
            hs = [h for h in range(Ho) if 0 <= -p[0] + h * s[0] + kh * d[0] < H]
            ws = [q for q in range(Wo) if 0 <= -p[1] + q * s[1] + kw * d[1] < W]
            if not hs or not ws:
                continue
            hs = np.array(hs)
            ws = np.array(ws)
            hin = -p[0] + hs * s[0] + kh * d[0]
            win = -p[1] + ws * s[1] + kw * d[1]
            xs = x[:, :, hin[:, None], win[None, :]]                      # [N,C,h,w]
            wt = w[:, :, :, tap][:, :, :, hs[:, None], ws[None, :]]       # [N,heads,wc,h,w]
            wt = wt[:, :, cidx]                                           # [N,heads,C,h,w]
            out[:, :, :, hs[:, None], ws[None, :]] += wt * xs[:, None]
    return out.reshape(N, heads * C, Ho, Wo)


def agg_zeropad_bwd_loops(dy, x, w, k=3, s=1, p=0, d=1):
    """aggregation_zeropad.py:48-110 -> (dX [N,C,H,W], dW like w)."""
    k, s, p, d = _pair(k), _pair(s), _pair(p), _pair(d)
    N, C, H, W = x.shape
    _, heads, wc, K2, Ho, Wo = w.shape
    dy5 = dy.reshape(N, heads, C, Ho, Wo)
    dx = np.zeros_like(x, dtype=np.result_type(x.dtype, w.dtype))
    dw = np.zeros_like(w, dtype=np.result_type(x.dtype, w.dtype))
    cidx = np.arange(C) % wc
    for kh in range(k[0]):
        for kw in range(k[1]):
            tap = kh * k[1] + kw
            hs = [h for h in range(Ho) if 0 <= -p[0] + h * s[0] + kh * d[0] < H]
            ws = [q for q in range(Wo) if 0 <= -p[1] + q * s[1] + kw * d[1] < W]
            if not hs or not ws:
                continue
            hs = np.array(hs)
            ws = np.array(ws)
            hin = -p[0] + hs * s[0] + kh * d[0]
            win = -p[1] + ws * s[1] + kw * d[1]
            g = dy5[:, :, :, hs[:, None], ws[None, :]]                    # [N,heads,C,h,w]
            wt = w[:, :, :, tap][:, :, :, hs[:, None], ws[None, :]][:, :, cidx]
            # dX (kernel :48-79): sum over heads of w * dY at the output positions that read this input
            dx[:, :, hin[:, None], win[None, :]] += (wt * g).sum(1)   # (hin, win) unique within one tap
            # dW (kernel :81-110): sum over the C/wc channels sharing weight channel cw
            xs = x[:, :, hin[:, None], win[None, :]]                      # [N,C,h,w]
            prod = g * xs[:, None]                                        # [N,heads,C,h,w]
            prod = prod.reshape(N, heads, C // wc, wc, len(hs), len(ws)).sum(2)
            dw[:, :, :, tap][:, :, :, hs[:, None], ws[None, :]] = prod
    return dx, dw


def agg_zeropad_mix_fwd_loops(x, w1, w2, k1=3, k2=5, s=1, p1=0, p2=0, d=1):
    """aggregation_zeropad_mix.py:20-74: channel order [n, (kernel_idx*heads + head)*C + c]."""
    N, C, H, W = x.shape
    heads = w1.shape[1]
    y1 = agg_zeropad_fwd_loops(x, w1, k1, s, p1, d)
    y2 = agg_zeropad_fwd_loops(x, w2, k2, s, p2, d)
    return np.concatenate([y1, y2], axis=1)


def agg_zeropad_mix_bwd_loops(dy, x, w1, w2, k1=3, k2=5, s=1, p1=0, p2=0, d=1):
    """aggregation_zeropad_mix.py:76-207.  NOTE: the reference's dX kernel hard-codes head=0
    (:88); for heads==1 (the only configuration its self-test and callers use) that is the
    full gradient, which is what is restated here for any heads."""
    N, C, H, W = x.shape
    heads = w1.shape[1]
    half = heads * C
    dx1, dw1 = agg_zeropad_bwd_loops(dy[:, :half], x, w1, k1, s, p1, d)
    dx2, dw2 = agg_zeropad_bwd_loops(dy[:, half:], x, w2, k2, s, p2, d)
    return dx1 + dx2, dw1, dw2


# --------------------------------------------------------------------------- torch Unfold identity
def agg_zeropad_unfold(x, w, k=3, s=1, p=0, d=1):
    """aggregation_zeropad.py:247-251 (the self-test's right-hand side), any dtype, differentiable."""
    N, C, H, W = x.shape
    _, heads, wc, K2, Ho, Wo = w.shape
    unfold = torch.nn.Unfold(kernel_size=k, dilation=d, padding=p, stride=s)
    x2 = unfold(x).view(N, C // wc, wc, K2, Ho, Wo)
    y = (w.unsqueeze(2) * x2.unsqueeze(1)).sum(-3)
    return y.view(N, heads * C, Ho, Wo)


def agg_zeropad_mix_unfold(x, w1, w2, k1=3, k2=5, s=1, p1=0, p2=0, d=1):
    """aggregation_zeropad_mix.py:360-366."""
    return torch.cat([agg_zeropad_unfold(x, w1, k1, s, p1, d),
                      agg_zeropad_unfold(x, w2, k2, s, p2, d)], dim=1)


# =========================================================================== the other cupy_layers variants (SURVEY 8f rank 4)
def _reflect(i, n):
    """aggregation_refpad.py:42-45 (applied to out-of-range indices; identity in range)."""
    if i < 0:
        i = -i
    if i >= n:
        i = 2 * (n - 1) - i
    return i


def agg_refpad_fwd_loops(x, w, k=3, s=1, p=0, d=1):
    """aggregation_refpad.py:21-55: the zero-pad forward with reflected input indices instead of skipped taps."""
    k, s, p, d = _pair(k), _pair(s), _pair(p), _pair(d)
    N, C, H, W = x.shape
    _, heads, wc, K2, Ho, Wo = w.shape
    out = np.zeros((N, heads, C, Ho, Wo), dtype=np.result_type(x.dtype, w.dtype))
    cidx = np.arange(C) % wc
    for kh in range(k[0]):
        for kw in range(k[1]):
            tap = kh * k[1] + kw
            hin = np.array([_reflect(-p[0] + h * s[0] + kh * d[0], H) for h in range(Ho)])
            win = np.array([_reflect(-p[1] + q * s[1] + kw * d[1], W) for q in range(Wo)])
            xs = x[:, :, hin[:, None], win[None, :]]                      # [N,C,Ho,Wo]
            wt = w[:, :, :, tap][:, :, cidx]                              # [N,heads,C,Ho,Wo]
            out += wt * xs[:, None]
    return out.reshape(N, heads * C, Ho, Wo)


def agg_refpad_unfold(x, w, k=3, s=1, p=0, d=1):
    """aggregation_refpad.py:236-239 (the self-test's right-hand side): Unfold of the ReflectionPad2d'ed input.
    k, s, p, d are ints or (height, width) pairs."""
    N, C, H, W = x.shape
    _, heads, wc, K2, Ho, Wo = w.shape
    ph, pw = _pair(p)
    unfold = torch.nn.Unfold(kernel_size=_pair(k), dilation=_pair(d), padding=0, stride=_pair(s))
    x2 = unfold(torch.nn.ReflectionPad2d((pw, pw, ph, ph))(x)).view(N, C // wc, wc, K2, Ho, Wo)
    return (w.unsqueeze(2) * x2.unsqueeze(1)).sum(-3).view(N, heads * C, Ho, Wo)


def agg_dilate_fwd_loops(x, w, dil):
    """aggregation_zeropad_dilate.py:20-57: 3x3, stride 1, weight channel g = c % wc uses dilation = padding = int(dil[g])."""
    N, C, H, W = x.shape
    _, heads, wc, K2, Ho, Wo = w.shape
    assert K2 == 9 and (Ho, Wo) == (H, W)
    out = np.zeros((N, heads, C, H, W), dtype=np.result_type(x.dtype, w.dtype))
    for c in range(C):
        g = c % wc
        dd = int(dil[g])
        for kh in range(3):
            for kw in range(3):
                hs = np.array([h for h in range(H) if 0 <= h + (kh - 1) * dd < H], dtype=np.int64)
                ws = np.array([q for q in range(W) if 0 <= q + (kw - 1) * dd < W], dtype=np.int64)
                if hs.size == 0 or ws.size == 0:
                    continue
                xs = x[:, c][:, (hs + (kh - 1) * dd)[:, None], (ws + (kw - 1) * dd)[None, :]]       # [N,h,w]
                wt = w[:, :, g, kh * 3 + kw][:, :, hs[:, None], ws[None, :]]                        # [N,heads,h,w]
                out[:, :, c][:, :, hs[:, None], ws[None, :]] += wt * xs[:, None]
    return out.reshape(N, heads * C, H, W)


def agg_dilate_unfold(x, w, dil):
    """The identity of aggregation_zeropad_dilate.py:258-296, written per weight channel: the channels {c : c % wc == g}
    are a LocalConv with one weight channel, dilation = padding = dil[g].  Differentiable (torch)."""
    N, C, H, W = x.shape
    _, heads, wc, K2, Ho, Wo = w.shape
    out = x.new_zeros(N, heads, C, H, W)
    for g in range(wc):
        dd = int(dil[g])
        xg = x[:, g::wc]                                                  # [N, C/wc, H, W]
        unfold = torch.nn.Unfold(kernel_size=3, dilation=dd, padding=dd, stride=1)
        x2 = unfold(xg).view(N, C // wc, 9, H, W)
        yg = (w[:, :, g].unsqueeze(2) * x2.unsqueeze(1)).sum(-3)          # [N, heads, C/wc, H, W]
        idx = torch.arange(g, C, wc, device=x.device)
        out = out.index_add(2, idx, yg)
    return out.view(N, heads * C, H, W)


def split_merged_weight(w, heads, wc, k1=3, k2=5):
    """aggregation_zeropad_mix_merge.py:35-36,52-54,334-338: [N, heads*wc*(k1^2+k2^2), Ho, Wo] -> (w1, w2) 6-D views."""
    N, _, Ho, Wo = w.shape
    n1 = heads * wc * k1 * k1
    return (w[:, :n1].reshape(N, heads, wc, k1 * k1, Ho, Wo), w[:, n1:].reshape(N, heads, wc, k2 * k2, Ho, Wo))


def agg_zeropad_mix_merge_unfold(x, w, heads, wc, k1=3, k2=5, s=1, p1=0, p2=0, d=1):
    """aggregation_zeropad_mix_merge.py:344-351: the mix identity on the two halves of the packed weight."""
    w1, w2 = split_merged_weight(w, heads, wc, k1, k2)
    return agg_zeropad_mix_unfold(x, w1, w2, k1, k2, s, p1, p2, d)


def agg_zeropad_mix_merge_fwd_loops(x, w, heads, wc, k1=3, k2=5, s=1, p1=0, p2=0, d=1):
    N, _, Ho, Wo = w.shape
    n1 = heads * wc * k1 * k1
    w1 = np.ascontiguousarray(w[:, :n1]).reshape(N, heads, wc, k1 * k1, Ho, Wo)
    w2 = np.ascontiguousarray(w[:, n1:]).reshape(N, heads, wc, k2 * k2, Ho, Wo)
    return agg_zeropad_mix_fwd_loops(x, w1, w2, k1, k2, s, p1, p2, d)
