"""TrainStep(virtual_ranks=K) without a GPU: argument validation (of the step's batch / mix / augmentation-split shapes and of
cotb200_multi_gather_acc, whose pointers are never dereferenced), the micro-batch gradient sum and per-rank BatchNorm buffers of
the host logic, and distribute_bn over K sets x 2 gloo ranks against the reference's arithmetic."""
import copy
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp


def _host_step_class():
    from cotnet_b200 import trainer

    class HostTrainStep(trainer.TrainStep):
        """The product's plumbing on CPU tensors: the kernel launches replaced by torch ops (the store gather, the fp32 accumulate /
        emit gather, plain SGD-nesterov)."""
        _host_logic_only = True

        def _launch_gather(self, tab, ent, bucket, grads):
            for (_, off, n, _), g in zip(ent, grads):
                bucket[off:off + n] = g.reshape(-1).to(bucket.dtype)

        def _launch_gather_acc(self, tab, ent, acc, dst, grads):
            it = iter(grads)
            for ptr, off, n, _ in ent:
                s = acc[off:off + n]
                if ptr:
                    s = s + next(it).reshape(-1).float()
                (acc if dst is None else dst)[off:off + n] = s.to(acc.dtype if dst is None else dst.dtype)

        def optimizer_step(self):
            for P, M, G, h in ((self.P_big, self.M_big, self.G_big, self.hyper), (self.P_small, self.M_small, self.G_small, self.hyper_small)):
                lr, mu, wd, _, gs = [float(v) for v in h]
                g = G.float() * gs + wd * P
                M.mul_(mu).add_(g)
                P.sub_(lr * (g + mu * M))
    return HostTrainStep


def _net(seed=7):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 4, 3), torch.nn.BatchNorm2d(4), torch.nn.ReLU(), torch.nn.Flatten(),
                               torch.nn.Linear(4 * 6 * 6, 5))


def _ts(K, **kw):
    base = dict(lr=0.1, momentum=0.9, weight_decay=1e-2, ema_decay=0.9, amp_dtype=None, weights="fp32", virtual_ranks=K)
    base.update(kw)
    return _host_step_class()(_net(), **base)


# ------------------------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("K", [0, -1, 1.5, True, "2"])
def test_virtual_ranks_rejects_bad_values(K):
    from cotnet_b200 import trainer
    with pytest.raises(ValueError, match="virtual_ranks"):
        trainer.TrainStep(_net(), virtual_ranks=K)


def test_step_rejects_bad_batch_mix_and_split_shapes():
    ts = _ts(2)
    x, y = torch.randn(8, 3, 8, 8), torch.randint(0, 5, (8,))
    with pytest.raises(ValueError, match="virtual ranks"):
        ts.step(x[:7], y[:7])                                        # rows not divisible by K
    with pytest.raises(ValueError, match="virtual ranks"):
        ts.step(x, y[:7])
    with pytest.raises(ValueError, match="list of 2"):
        ts.step(x, y, mix=object())                                  # one table for two ranks
    with pytest.raises(ValueError, match="list of 2"):
        ts.step(x, y, mix=[object()])
    with pytest.raises(ValueError, match="list of 2"):
        ts.step(x, y, mix=[object(), None])
    with pytest.raises(ValueError, match="rank"):
        ts.rank_buffers(2)
    jsd = _ts(2, jsd_splits=2)
    with pytest.raises(ValueError, match="augmentation splits"):
        jsd.step(x[:6], y[:6])                                       # rank batch of 3 is not 2 splits
    with pytest.raises(ValueError, match="does not mix"):
        jsd.step(x, y, mix=[object(), object()])
    assert torch.equal(ts.P_big, _ts(2).P_big) and ts.G_big.abs().sum() == 0    # nothing ran


def test_multi_gather_acc_rejects_bad_arguments():
    """Validation happens before any CUDA call: the pointers below are never dereferenced."""
    from cotnet_b200 import _lib
    lib = _lib.load()
    P = 64
    ENULL, EINVAL, EALIGN, EDTYPE = -5, -1, -4, -2

    def call(segs=P, blocks=P, nb=1, acc=P, dt=_lib.F32, dst=2 * P):
        return lib.cotb200_multi_gather_acc(segs, blocks, nb, acc, dt, dst, 1.0, None)
    assert call(segs=None) == ENULL
    assert call(blocks=None) == ENULL
    assert call(acc=None) == ENULL
    assert call(nb=0) == EINVAL
    assert call(nb=-3) == EINVAL
    assert call(acc=P + 4) == EALIGN                                 # fp32-aligned but not 16-byte aligned
    assert call(dt=_lib.F16) == EDTYPE
    assert call(dt=_lib.F64) == EDTYPE
    assert call(dt=_lib.BF16, dst=P) == EINVAL                       # a bf16 bucket cannot be the fp32 accumulator
    assert b"multi_gather_acc" in lib.cotb200_last_error()


# ------------------------------------------------------------------------------------------------ host logic, one process
def test_host_logic_sums_gradients_and_keeps_buffers_per_rank():
    K = 3
    ts = _ts(K)
    ref = copy.deepcopy(_net())
    g0 = torch.Generator().manual_seed(1)
    for step in range(2):                                            # forward_backward only: the weights stay the reference's
        x, y = torch.randn(4 * K, 3, 8, 8, generator=g0), torch.randint(0, 5, (4 * K,), generator=g0)
        ts.forward_backward(x, y)
        B = 4
        want_g, want_b = {}, []
        for k in range(K):                                           # rank k starts from its own buffers of the previous step
            rk = copy.deepcopy(ref)
            if step:
                with torch.no_grad():
                    for n, b in rk.named_buffers():
                        b.copy_(prev[k][n])
            rk.zero_grad(set_to_none=True)
            torch.nn.functional.cross_entropy(rk(x[k * B:(k + 1) * B]), y[k * B:(k + 1) * B]).backward()
            for n, p in rk.named_parameters():
                want_g[n] = p.grad.clone() if k == 0 else want_g[n] + p.grad
            want_b.append({n: b.clone() for n, b in rk.named_buffers()})
        prev = want_b
        got = ts.grads()
        for n in want_g:
            assert torch.equal(got[n], want_g[n]), n                 # the fp32 sum in rank order
        for k in range(K):
            rb = ts.rank_buffers(k)
            for n in want_b[k]:
                assert torch.equal(rb[n], want_b[k][n]), (k, n)
        # outside the step the module's own buffers are rank 0's, in their original storage
        assert all(b.data_ptr() == t.data_ptr() for b, t in zip(ts.model.buffers(), ts.rank_buffers(0).values()))
    assert float(ts.hyper[4]) == pytest.approx(1.0 / K)


def test_distribute_bn_local_sets():
    ts = _ts(3)
    g0 = torch.Generator().manual_seed(2)
    vals = []
    for k in range(3):
        rb, eb = ts.rank_buffers(k), ts.rank_buffers(k, ema=True)
        with torch.no_grad():
            for d in (rb, eb):
                d["1.running_mean"].copy_(torch.randn(4, generator=g0))
                d["1.running_var"].copy_(torch.rand(4, generator=g0) + 0.5)
                d["1.num_batches_tracked"].fill_(k + 1)
        vals.append({n: (rb[n].clone(), eb[n].clone()) for n in rb})
    ts.distribute_bn()
    for n in ("1.running_mean", "1.running_var"):
        for e in (0, 1):
            want = (vals[0][n][e] + vals[1][n][e] + vals[2][n][e]) / 3.0
            for k in range(3):
                assert torch.equal(ts.rank_buffers(k, ema=bool(e))[n], want), (n, e, k)
    assert [int(ts.rank_buffers(k)["1.num_batches_tracked"]) for k in range(3)] == [1, 2, 3]
    assert torch.equal(ts.model[1].running_mean, ts.rank_buffers(1)["1.running_mean"])


# ------------------------------------------------------------------------------------------------ distribute_bn over gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _set_values(r, k, n):
    g = torch.Generator().manual_seed(1000 * r + 10 * k + (0 if "mean" in n else 1))
    return torch.randn(4, generator=g) if "mean" in n else torch.rand(4, generator=g) + 0.5


def _dist_worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from cotnet_b200 import dist as cdist
    cdist.init_from_env(backend="gloo")
    K = 2
    ts = _ts(K)
    assert ts.world == world and abs(float(ts.hyper[4]) - 1.0 / (K * world)) < 1e-9      # gloo SUM: 1/(K world) in the update
    names = ("1.running_mean", "1.running_var")
    out = {}
    for reduce in (True, False):
        with torch.no_grad():
            for k in range(K):
                for e in (False, True):
                    for n in names:
                        ts.rank_buffers(k, ema=e)[n].copy_(_set_values(rank, k, n) + (100.0 if e else 0.0))
        ts.distribute_bn(reduce=reduce)
        out[reduce] = {(k, e, n): ts.rank_buffers(k, ema=e)[n].tolist() for k in range(K) for e in (False, True) for n in names}
    q.put((rank, out))
    dist.destroy_process_group()


def test_distribute_bn_two_sets_two_gloo_ranks():
    world, K = 2, 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dist_worker, args=(r, world, port, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=120) for _ in range(world))
        for p in procs:
            p.join(60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(10)
    for e in (False, True):
        off = 100.0 if e else 0.0
        for n in ("1.running_mean", "1.running_var"):
            v = {(r, k): _set_values(r, k, n) + off for r in range(world) for k in range(K)}
            local = [v[(r, 0)] + v[(r, 1)] for r in range(world)]           # the local sum first, in rank order
            want = (local[0] + local[1]) / float(K * world)
            plain = sum(v.values()) / float(K * world)                      # the reference's SUM over 4 ranks, / 4
            for r in range(world):
                for k in range(K):
                    got = torch.tensor(res[r][True][(k, e, n)])
                    assert torch.equal(got, want), (r, k, e, n)
                    assert torch.allclose(got, plain, rtol=1e-6, atol=1e-6)
                    # broadcast: global rank 0's set 0 everywhere
                    assert torch.equal(torch.tensor(res[r][False][(k, e, n)]), v[(0, 0)]), (r, k, e, n)
