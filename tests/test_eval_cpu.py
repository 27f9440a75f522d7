"""Validation host logic on CPU: the argument checks of cotb200_topk_hits (no kernel is launched), the rank rule against torch's
topk on tie-free rows, and TrainStep.distribute_bn over 2 gloo ranks against the reference's per-buffer arithmetic."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from cotnet_b200 import _lib


def rank_rule_counts(z, y, ks, valid=None):
    """numpy statement of the rank rule (include/cotb200.h, cotb200_topk_hits): [hits at each k, rows counted, bad labels]."""
    z = np.asarray(z, dtype=np.float64)
    B, K = z.shape
    n = B if valid is None else min(max(int(valid), 0), B)
    out = np.zeros(len(ks) + 2, dtype=np.int64)
    for b in range(n):
        out[len(ks)] += 1
        if not 0 <= y[b] < K:
            out[len(ks) + 1] += 1
            continue
        zy = z[b, y[b]]
        if np.isnan(zy):
            continue
        r = int(np.sum(z[b] > zy)) + int(np.sum(z[b, :y[b]] == zy))
        out[:len(ks)] += np.array([r < k for k in ks], dtype=np.int64)
    return out


def accuracy_counts(output, target, topk):
    """utils/meters.py:12-19 accuracy(): hit counts of output.topk(maxk) + eq."""
    _, pred = output.topk(max(topk), 1, True, True)
    correct = pred.t().eq(target.reshape(1, -1).expand_as(pred.t()))
    return [int(correct[:k].reshape(-1).float().sum(0)) for k in topk]


def test_topk_hits_argument_errors():
    lib = _lib.load()
    P = 16
    ENULL, EINVAL, EDTYPE = -5, -1, -2
    ks = (ctypes.c_int * 2)(1, 5)
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, None, 10, P, None, 2, ks, P, None) == ENULL
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, P, 10, None, None, 2, ks, P, None) == ENULL
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, P, 10, P, None, 2, None, P, None) == ENULL
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, P, 10, P, None, 2, ks, None, None) == ENULL
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, P, 10, P, None, 0, ks, P, None) == EINVAL             # nk = 0
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, P, 10, P, None, 5, (ctypes.c_int * 5)(1, 2, 3, 4, 5), P, None) == EINVAL
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, P, 10, P, None, 2, (ctypes.c_int * 2)(0, 5), P, None) == EINVAL
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, P, 10, P, None, 2, (ctypes.c_int * 2)(1, 11), P, None) == EINVAL
    assert lib.cotb200_topk_hits(_lib.BF16, 4, 10, P, 9, P, None, 2, ks, P, None) == EINVAL              # ld < K
    assert lib.cotb200_topk_hits(_lib.BF16, 0, 10, P, 10, P, None, 2, ks, P, None) == EINVAL
    assert lib.cotb200_topk_hits(_lib.F64, 4, 10, P, 10, P, None, 2, ks, P, None) == EDTYPE
    assert lib.cotb200_topk_hits(7, 4, 10, P, 10, P, None, 2, ks, P, None) == EDTYPE
    assert lib.cotb200_last_error()


@pytest.mark.parametrize("K,ks", [(10, (1, 5)), (1000, (1, 5)), (1001, (1, 2, 3, 10))])
def test_rank_rule_equals_torch_topk_without_ties(K, ks):
    g = torch.Generator().manual_seed(K)
    B = 64
    z = torch.randn(B, K, generator=g, dtype=torch.float64)
    assert all(len(set(r.tolist())) == K for r in z)                    # tie-free rows
    y = torch.randint(0, K, (B,), generator=g)
    # make some rows hits at every k and some misses at every k
    z[0, y[0]] = 100.0
    z[1, y[1]] = -100.0
    want = accuracy_counts(z, y, ks)
    got = rank_rule_counts(z.numpy(), y.numpy(), ks)
    assert got[:len(ks)].tolist() == want and got[len(ks)] == B and got[len(ks) + 1] == 0
    assert got[0] >= 1 and got[0] < B
    # the rank rule on a prefix counts only that prefix
    assert rank_rule_counts(z.numpy(), y.numpy(), ks, valid=7)[:len(ks)].tolist() == accuracy_counts(z[:7], y[:7], ks)


def test_rank_rule_ties_nan_and_bad_labels():
    z = np.array([[1.0, 2.0, 2.0, 0.0],     # label 2 ties with class 1 (lower index wins): rank 1
                  [1.0, 2.0, 2.0, 0.0],     # label 1 wins the tie: rank 0
                  [np.nan, 1.0, 0.5, 3.0],  # NaN competitor never outranks: label 2 has rank 2 (1.0 and 3.0)
                  [1.0, np.nan, 0.5, 3.0],  # NaN label logit: miss
                  [1.0, 2.0, 3.0, 4.0]])    # label -1: bad
    y = np.array([2, 1, 2, 1, -1])
    assert rank_rule_counts(z, y, (1, 2, 3)).tolist() == [1, 2, 3, 5, 1]


# ------------------------------------------------------------------------------------------------ distribute_bn over gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _bn_worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from cotnet_b200 import dist as cdist, trainer
    cdist.init_from_env(backend="gloo")

    class HostTrainStep(trainer.TrainStep):
        _host_logic_only = True                   # CPU model over gloo: distribute_bn launches no kernel

    torch.manual_seed(3)
    net = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3), torch.nn.BatchNorm2d(8), torch.nn.ReLU(), torch.nn.Conv2d(8, 6, 1),
                              torch.nn.BatchNorm2d(6), torch.nn.Flatten(), torch.nn.Linear(6 * 4 * 4, 5))
    ts = HostTrainStep(net, ema_decay=0.9, amp_dtype=None, weights="fp32")
    names = [n for n, _ in net.named_buffers()]
    out = {}
    for mode in ("reduce", "broadcast"):
        g = torch.Generator().manual_seed(100 * rank + (mode == "broadcast"))
        with torch.no_grad():
            for n, b, e in zip(names, net.buffers(), ts.ema_buffers):
                if b.dtype.is_floating_point:
                    b.copy_(torch.rand(b.shape, generator=g) * 3 + 0.1)
                    e.copy_(torch.rand(b.shape, generator=g) * 3 + 0.1)
                else:
                    b.fill_(10 + rank)
                    e.fill_(20 + rank)
        bufs = list(net.buffers()) + list(ts.ema_buffers)
        ptrs = [t.data_ptr() for t in bufs]
        want = []
        for t, n in zip(bufs, names + names):                              # utils/distributed.py:57-67, buffer by buffer
            r = t.clone()
            if "running_mean" in n or "running_var" in n:
                if mode == "reduce":
                    dist.all_reduce(r, op=dist.ReduceOp.SUM)
                    r /= float(world)
                else:
                    dist.broadcast(r, 0)
            want.append(r)
        before = [t.clone() for t in bufs]
        ts.distribute_bn(reduce=(mode == "reduce"), ema=True)
        out[mode] = dict(
            exact=all(torch.equal(t, w) for t, w in zip(bufs, want)),
            ptrs=[t.data_ptr() for t in bufs] == ptrs,
            counters=all(torch.equal(t, b) for t, b, n in zip(bufs, before, names + names) if n.endswith("num_batches_tracked")),
            changed=sum(not torch.equal(t, b) for t, b in zip(bufs, before)),
            values=[t.tolist() for t, n in zip(bufs, names + names) if "running" in n])
    q.put((rank, out))
    dist.destroy_process_group()


def test_distribute_bn_two_rank_gloo():
    world = 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_bn_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    for rank, out in res:
        for mode in ("reduce", "broadcast"):
            o = out[mode]
            assert o["exact"] and o["ptrs"] and o["counters"], (rank, mode)
        # 2 BatchNorms x (mean, var) in the model and in the EMA copies; rank 0 keeps its values when broadcasting
        assert out["reduce"]["changed"] == 8
        assert out["broadcast"]["changed"] == (0 if rank == 0 else 8)
    for mode in ("reduce", "broadcast"):
        assert res[0][1][mode]["values"] == res[1][1][mode]["values"]
