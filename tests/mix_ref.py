"""numpy restatement of what a per-sample Mixup / CutMix row table (struct cotb200_mix_row, trainer.MixRows) means: the mixed
uint8 batch of FastCollateMixup's _mix_elem_collate / _mix_pair_collate (datasets/mixup.py:223-280) and the soft targets of
mixup_target (:17-27), what cotb200_u8_mix_rows_to_nhwc and cotb200_soft_ce_rows compute.

rows: a sequence of objects with mode, partner, lam, one_minus_lam, target_lam, y0, y1, x0, x1 (a ctypes array of _lib.MixRow).
"""
import numpy as np


def mixed_batch(x, rows):
    """uint8 [N_in, C, H, W] -> uint8 [len(rows), C, H, W]: output row n from input rows n and rows[n].partner.  Mixup is numpy's
    fp32 arithmetic (two rounded products, a rounded sum, np.rint: ties to even)."""
    out = np.empty((len(rows),) + x.shape[1:], dtype=np.uint8)
    for n, r in enumerate(rows):
        a, p = x[n], x[r.partner]
        if r.mode == 0:
            out[n] = a
        elif r.mode == 1:
            out[n] = np.rint(a.astype(np.float32) * np.float32(r.lam) + p.astype(np.float32) * np.float32(r.one_minus_lam))
        elif r.mode == 2:
            out[n] = a
            out[n][:, r.y0:r.y1, r.x0:r.x1] = p[:, r.y0:r.y1, r.x0:r.x1]
        else:
            raise ValueError("unknown mode %d" % r.mode)
    return out


def soft_targets(labels, rows, num_classes, smoothing):
    """float64 [len(rows), K]: target_lam * onehot(labels[n]) + (1 - target_lam) * onehot(labels[partner]), smoothed."""
    off = smoothing / num_classes
    on = 1.0 - smoothing + off
    eye = np.eye(num_classes) * (on - off) + off
    return np.stack([r.target_lam * eye[labels[n]] + (1.0 - r.target_lam) * eye[labels[r.partner]] for n, r in enumerate(rows)])
