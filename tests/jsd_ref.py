"""fp64 restatement of the reference's JsdCrossEntropy (loss/jsd.py) and its gradient, what cotb200_jsd_ce / _bwd compute.

logits z [S*B, K] split-major, labels y [>= B] (the first B read).  With p_s = softmax(z_s) of the B x K block of split s and
m = clamp(mean_s p_s, 1e-7, 1):
    loss = CE_smooth(z_0, y) + alpha/S * sum_s sum_{b,c} (xlogy(p_sbc, p_sbc) - p_sbc log m_bc) / B.
The gradient is written out: dL/dp_s = alpha/(S*B) (log p_s - log m + [clamp binds]), then the softmax Jacobian of each split,
plus the cross-entropy gradient on split 0.  Where p underflows to 0 the xlogy limit makes the term 0 (the reference's autograd
gives NaN there).
"""
import numpy as np

CLAMP_LO, CLAMP_HI = 1e-7, 1.0


def _log_softmax(z):
    mx = z.max(axis=1, keepdims=True)
    return z - mx - np.log(np.exp(z - mx).sum(axis=1, keepdims=True))


def jsd_ce(z, y, S, smoothing=0.0, alpha=12.0, clamp=(CLAMP_LO, CLAMP_HI)):
    """(loss, dloss/dz) in fp64.  `clamp` bounds the mixture (the kernels compare in fp32: pass (np.float32(1e-7), 1.0))."""
    z = np.asarray(z, np.float64)
    N, K = z.shape
    B = N // S
    y = np.asarray(y)[:B]
    lp = _log_softmax(z).reshape(S, B, K)
    p = np.exp(lp)
    msum = p[0].copy()
    for s in range(1, S):
        msum += p[s]
    m = msum / S
    lo, hi = clamp
    passes = (m >= lo) & (m <= hi)
    lm = np.log(np.clip(m, lo, hi))
    off = smoothing / K
    t = np.full((B, K), off)
    t[np.arange(B), y] += 1.0 - smoothing
    ce = -(t * lp[0]).sum(axis=1)
    kl = (p * lp - p * lm).sum(axis=(0, 2))                          # p * lp -> 0 as p underflows to 0: xlogy's limit
    loss = (ce + alpha / S * kl).mean()
    gp = alpha / (S * B) * (lp - lm + np.where(passes, 0.0, 1.0))
    dz = p * (gp - (p * gp).sum(axis=2, keepdims=True))
    dz[0] += (p[0] - t) / B
    return loss, dz.reshape(N, K)
