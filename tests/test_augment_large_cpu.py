"""CPU checks of the augmentation above 256 x 256 (the thread-block-cluster entry points cotb200_aug_randaug_cluster and
cotb200_aug_color_jitter_cluster): they reject bad arguments before any CUDA call, oracle/aug_ref.py and tests/jitter_ref.py
reproduce the reference's PIL outputs at 288 and 320 in tests/golden/augment_large.npz byte for byte, and se_cotnetd_152_L is
the reference's model of that name."""
import os
import random

import numpy as np
import pytest
import torch

from cotnet_b200 import _lib, augment
import jitter_ref
from oracle import aug_ref, ref_import

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augment_large.npz")
FAKE = 1 << 20                                          # never dereferenced: validation fails first
EINVAL, ENULL, EUNSUPPORTED = -1, -5, -7


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _draw(tf, s, H, W):
    return tf.draw_one(H, W, random.Random(s), np.random.RandomState(s), torch.Generator().manual_seed(s))


def _cases(gold, prefix):
    k = 0
    while "%s_%d" % (prefix, k) in gold:
        yield k, [int(v) for v in gold["%s_%d_size" % (prefix, k)]], gold["%s_%d" % (prefix, k)]
        k += 1


# ---------------------------------------------------------------- C-ABI argument errors (no kernel is launched)
def _rec():
    r = np.zeros(1, augment.SAMPLE_DTYPE)
    r["ops"]["op"] = -1
    return r


def _jrec(**kw):
    r = np.zeros(1, augment.JITTER_DTYPE)
    r["order"] = [0, 1, 2, 3]
    r["factor"] = [1.1, 0.9, 1.2]
    r["hue"] = 0.1
    for k, v in kw.items():
        r[k][0] = v
    return r


def test_capi_randaug_cluster_rejects_bad_arguments():
    f = _lib.load().cotb200_aug_randaug_cluster
    for op, extra in ((16, {}), (-2, {}), (3, {"filter": 2}), (4, {"v": [-1, 0, 0, 0]}), (7, {"factor": float("nan")}),
                      (11, {"m": [float("inf"), 0, 0, 0, 1, 0]})):
        r = _rec()
        r["ops"]["op"][0, 1] = op
        for k, v in extra.items():
            r["ops"][k][0, 1] = v
        assert f(1, 320, r.ctypes.data, FAKE, FAKE, None) == EINVAL, (op, extra)
    assert f(1, 8, None, FAKE, FAKE, None) == ENULL
    assert f(1, 320, _rec().ctypes.data, None, FAKE, None) == ENULL
    assert f(1, 320, _rec().ctypes.data, FAKE, None, None) == ENULL
    for N, S in ((0, 320), (-1, 320), (1, 0), (1, -5)):
        assert f(N, S, _rec().ctypes.data, FAKE, FAKE, None) == EINVAL, (N, S)
    assert f(1, 513, _rec().ctypes.data, FAKE, FAKE, None) == EUNSUPPORTED
    assert augment.CLUSTER_MAX_S == 512 and augment.ONE_CTA_MAX_S == 256


def test_capi_color_jitter_cluster_rejects_bad_arguments():
    f = _lib.load().cotb200_aug_color_jitter_cluster
    for bad in (dict(order=[0, 1, 2, 4]), dict(order=[0, -2, 1, 2]), dict(order=[0, 1, 1, 2]), dict(order=[3, -1, -1, 3]),
                dict(factor=[-0.1, 1, 1]), dict(factor=[1, float("nan"), 1]), dict(factor=[1, 1, float("inf")]),
                dict(hue=0.5000001), dict(hue=-0.6), dict(hue=float("nan")), dict(vflip=2), dict(vflip=-1)):
        assert f(1, 320, _jrec(**bad).ctypes.data, FAKE, FAKE, None) == EINVAL, bad
    assert f(1, 8, None, FAKE, FAKE, None) == ENULL
    assert f(1, 320, _jrec().ctypes.data, None, FAKE, None) == ENULL
    assert f(1, 320, _jrec().ctypes.data, FAKE, None, None) == ENULL
    for N, S in ((0, 320), (-1, 320), (1, 0), (1, -5)):
        assert f(N, S, _jrec().ctypes.data, FAKE, FAKE, None) == EINVAL, (N, S)
    assert f(1, 513, _jrec().ctypes.data, FAKE, FAKE, None) == EUNSUPPORTED


def test_dispatch_by_size():
    assert [augment.uses_cluster_kernels(S) for S in (1, 224, 256, 257, 288, 320, 512)] == [False] * 3 + [True] * 4


# ---------------------------------------------------------------- the oracles against the reference's PIL outputs
@pytest.mark.parametrize("S", [288, 320])
def test_aug_ref_train_equals_fixture(gold, S):
    tf = augment.TrainAugment(size=S)
    n = 0
    for k, (H, W, seed, iseed), want in _cases(gold, "train_%d" % S):
        got = aug_ref.train_sample(aug_ref.source_image(iseed, H, W), _draw(tf, seed, H, W), S)
        np.testing.assert_array_equal(got, want, err_msg="train %d image %d" % (S, k))
        n += 1
    assert n >= 4


def test_jitter_ref_equals_fixture(gold):
    tf = augment.TrainAugment(size=320, auto_augment=None, color_jitter=0.4, vflip=0.5)
    n = 0
    for k, (H, W, seed, iseed), want in _cases(gold, "jout_320"):
        p = _draw(tf, seed, H, W)
        got = jitter_ref.train_sample_jitter(aug_ref.source_image(iseed, H, W), p, 320)
        np.testing.assert_array_equal(got, want, err_msg="jitter image %d" % k)
        n += 1
    assert n >= 4


@pytest.mark.parametrize("S", [288, 320])
def test_aug_ref_eval_equals_fixture(gold, S):
    crop_pct = float(gold["eval_%d_crop_pct" % S])
    n = 0
    for k, (H, W, iseed), want in _cases(gold, "eval_%d" % S):
        got = aug_ref.eval_transform(aug_ref.source_image(iseed, H, W), S, crop_pct).transpose(2, 0, 1)
        np.testing.assert_array_equal(got, want, err_msg="eval %d image %d" % (S, k))
        n += 1
    assert n >= 2


# ---------------------------------------------------------------- se_cotnetd_152_L
@pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")
def test_se_cotnetd_152_L_is_the_reference_model():
    from cotnet_b200 import backbone_hybrid as bh
    ns = ref_import.load()
    ref, m = ns.hybrid.se_cotnetd_152_L(), bh.se_cotnetd_152_L()
    m.load_state_dict(ref.state_dict(), strict=True)
    assert abs(sum(p.numel() for p in m.parameters()) / 1e6 - 55.8) < 0.06
