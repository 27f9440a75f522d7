"""TrainStep(virtual_ranks=K) on the GPU: cotb200_multi_gather_acc bit-exact against torch fp32 adds, K = 1 identical to the
plain step, K virtual ranks bit-identical to their definition (K micro-batches of a one-rank step, their gradients summed in
fp32, one update at grad_scale 1/K, buffers and their EMA kept per rank), graph replay against the eager step, two virtual ranks
against two real gloo ranks, and EvalStep on rank 0's buffers before distribute_bn and on the averaged ones after it."""
import copy
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
CL = torch.channels_last
MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


@pytest.fixture
def deterministic(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("dst_kind", ["f32", "bf16", "acc"])
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_multi_gather_acc_bit_exact(K, dst_kind):
    """K phases -- store (cotb200_multi_gather), add, ..., emit -- against torch fp32 adds in the same order: fp32 / bf16 / fp16
    sources, fp32 / bf16 buckets and the fp32 bucket as its own accumulator, segments longer than a gather chunk, offsets that
    break the 16-byte packets, segments without a source in some phases; the slot padding is never written."""
    from cotnet_b200 import _lib, trainer
    lib = _lib.load()
    chunk = lib.cotb200_gather_chunk()
    st = torch.cuda.current_stream().cuda_stream
    shapes = [(3,), (chunk + 5,), (7, 9), (2 * chunk + 3,), (64, 3, 7, 7), (1,), (1000,)]
    pads = [0, 1, 8, 3, 5, 8, 2]                                     # gaps before each slot: odd offsets take the scalar path
    offs, o = [], 0
    for s, p in zip(shapes, pads):
        o += p
        offs.append(o)
        o += int(torch.tensor(s).prod())
    n = o + 7
    g0 = torch.Generator(device="cuda").manual_seed(10 + K)
    dtypes = [torch.float32, torch.bfloat16, torch.float16]
    scale = 0.5 if K % 2 else 1.0
    sentinel = 7.0
    dst_dtype = torch.bfloat16 if dst_kind == "bf16" else torch.float32
    acc = torch.full((n,), sentinel, device="cuda")
    dst = acc if dst_kind == "acc" else torch.full((n,), sentinel, device="cuda", dtype=dst_dtype)
    want = None
    tabs = []
    for k in range(K):
        srcs = [torch.randn(*s, device="cuda", generator=g0).to(dtypes[(i + k) % 3]) for i, s in enumerate(shapes)]
        absent = {i for i in range(len(shapes)) if k > 0 and (i + k) % 4 == 0}      # no gradient in this phase
        ents = [(0 if i in absent else t.data_ptr(), off, t.numel(), _lib.dtype_code(t)) for i, (t, off) in enumerate(zip(srcs, offs))]
        tab = trainer._GatherTable(len(ents), sum((t.numel() + chunk - 1) // chunk for t in srcs), torch.device("cuda"))
        tabs.append(tab)
        nb = tab.fill(ents, chunk)
        tab.upload(False)
        target = dst if K == 1 else acc
        if k == 0:
            _lib.check(lib.cotb200_multi_gather(tab.seg_d.data_ptr(), tab.blk_d.data_ptr(), nb, _lib.dtype_code(target), target.data_ptr(),
                                                scale, st), "multi_gather")
        else:
            out = dst if k == K - 1 else None
            _lib.check(lib.cotb200_multi_gather_acc(tab.seg_d.data_ptr(), tab.blk_d.data_ptr(), nb, acc.data_ptr(),
                                                    _lib.dtype_code(dst) if out is not None else _lib.F32, _lib.ptr(out), scale, st),
                       "multi_gather_acc")
        parts = [None if i in absent else t.float().reshape(-1) * scale for i, t in enumerate(srcs)]
        if k == 0:
            want = parts
        else:
            want = [w if p is None else w + p for w, p in zip(want, parts)]
    torch.cuda.synchronize()
    for w, off in zip(want, offs):
        assert torch.equal(dst[off:off + w.numel()], w.to(dst.dtype)), off
    covered = torch.zeros(n, dtype=torch.bool, device="cuda")
    for w, off in zip(want, offs):
        covered[off:off + w.numel()] = True
    assert bool((dst[~covered] == sentinel).all())                  # padding untouched


# ------------------------------------------------------------------------------------------------ models and batches
def _model(seed=0, **kw):
    from cotnet_b200 import backbone
    torch.manual_seed(seed)
    return backbone.CoTResNet([1, 1, 1, 1], num_classes=16, zero_init_last_bn=False, **kw).cuda().to(memory_format=CL).train()


def _batch(seed, B, res=96, classes=16):
    from cotnet_b200 import trainer
    g0 = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (B, 3, res, res), generator=g0, dtype=torch.uint8).cuda()
    return trainer.normalize_u8(x, MEAN, STD), torch.randint(0, classes, (B,), generator=g0).cuda()


def _bufs(ts, k, ema=False):
    return {n: t.clone() for n, t in ts.rank_buffers(k, ema).items()}


def _state(ts):
    out = {"P_big": ts.P_big, "P_small": ts.P_small, "M_big": ts.M_big, "M_small": ts.M_small}
    for name in ("V_big", "V_small", "E_big", "E_small", "Pb"):
        if getattr(ts, name) is not None:
            out[name] = getattr(ts, name)
    return {k: v.clone() for k, v in out.items()}


def _assert_same(a, b, what):
    differ = [k for k in a if not torch.equal(a[k], b[k])]
    assert not differ, (what, differ[:5])


# ------------------------------------------------------------------------------------------------ K = 1 is the plain step
def test_one_virtual_rank_is_the_plain_step(deterministic):
    from cotnet_b200 import trainer
    kw = dict(lr=0.01, momentum=0.9, weight_decay=1e-3, ema_decay=0.99, label_smoothing=0.1)
    m1 = _model(drop_path_rate=0.1)
    m2 = copy.deepcopy(m1)
    t1, t2 = trainer.TrainStep(m1, **kw), trainer.TrainStep(m2, virtual_ranks=1, **kw)
    assert t2.G_acc is t2.G_big                                      # no accumulator
    x, y = _batch(1, 8)
    infos = []
    for t in (t1, t2):
        torch.manual_seed(5)
        infos.append(t.capture(x, y, warmup=1))
        for s in range(3):
            t.step(*_batch(2 + s, 8))
    assert infos[0]["libcotb200_kernels_per_replay"] == infos[1]["libcotb200_kernels_per_replay"]
    _assert_same(_state(t1), _state(t2), "state")
    _assert_same(_bufs(t1, 0), _bufs(t2, 0), "buffers")
    _assert_same(_bufs(t1, 0, True), _bufs(t2, 0, True), "ema buffers")


# ------------------------------------------------------------------------------------------------ K ranks == their definition
def _definition_step(ref, K, x, y, rank_bufs, rank_ema):
    """One step of K ranks built from a one-rank TrainStep `ref`: per rank its buffers, forward_backward on its slice, the
    gradients summed in fp32 in rank order, one optimizer_step at grad_scale 1/K; the buffers' EMA per rank."""
    B, L = x.shape[0] // K, y.shape[0] // K
    model_bufs = list(ref.model.buffers())
    gb, gs, losses = None, None, []
    for k in range(K):
        with torch.no_grad():
            for b, v in zip(model_bufs, rank_bufs[k]):
                b.copy_(v)
        losses.append(ref.forward_backward(x[k * B:(k + 1) * B], y[k * L:(k + 1) * L]).detach().clone())
        with torch.no_grad():
            gb = ref.G_big.float().clone() if k == 0 else gb + ref.G_big.float()
            gs = ref.G_small.clone() if k == 0 else gs + ref.G_small
            rank_bufs[k] = [b.clone() for b in model_bufs]
    with torch.no_grad():
        ref.G_big.copy_(gb.to(ref.G_big.dtype))
        ref.G_small.copy_(gs)
        ref.hyper[4] = ref.hyper_small[4] = 1.0 / K
        for b, v in zip(model_bufs, rank_bufs[0]):
            b.copy_(v)
        for e, v in zip(ref.ema_buffers, rank_ema[0]):
            e.copy_(v)
        ref.optimizer_step()
        rank_ema[0] = [e.clone() for e in ref.ema_buffers]
        st = torch.cuda.current_stream().cuda_stream
        for k in range(1, K):                                        # the EMA of rank k's buffers: the same lerp kernel
            for b, v in zip(model_bufs, rank_bufs[k]):
                b.copy_(v)
            for e, v in zip(ref.ema_buffers, rank_ema[k]):
                e.copy_(v)
            ref.lib.cotb200_multi_lerp(ref._lerp_tab.data_ptr(), ref._lerp_n, ref.hyper.data_ptr(), st)
            rank_ema[k] = [e.clone() for e in ref.ema_buffers]
    loss = losses[0]
    for lk in losses[1:]:
        loss = loss + lk
    return loss / K


CASES = [  # K, bucket, opt, clip mode, jsd splits
    (2, torch.bfloat16, "sgd", "agc", 0),
    (3, torch.float32, "adamw", "norm", 0),
    (2, torch.float32, "adamw", "agc", 0),
    (3, torch.bfloat16, "sgd", "norm", 0),
    (2, torch.bfloat16, "sgd", "norm", 2),                          # a CoTNet trunk with drop rates and the JSD splits
]


@pytest.mark.parametrize("K,bucket,opt,clip_mode,jsd", CASES)
def test_virtual_ranks_equal_their_definition(K, bucket, opt, clip_mode, jsd, deterministic):
    from cotnet_b200 import trainer
    B = 4
    m = _model(drop_path_rate=0.2, drop_block_rate=0.2)
    n_blocks = len(m.blocks())
    g0 = torch.Generator().manual_seed(3)
    m.fixed_drop_path_scales = (torch.rand(n_blocks, B, generator=g0) > 0.3).float().cuda() / 0.7
    m.fixed_drop_block_key = torch.tensor([11, 12])
    mr = copy.deepcopy(m)
    kw = dict(lr=0.02, momentum=0.9, weight_decay=1e-3, ema_decay=0.9, bucket_dtype=bucket, opt=opt, clip_grad=0.05,
              clip_mode=clip_mode, label_smoothing=0.1, jsd_splits=jsd)
    ts = trainer.TrainStep(m, virtual_ranks=K, **kw)
    ref = trainer.TrainStep(mr, **kw)
    rank_bufs = [[b.clone() for b in mr.buffers()] for _ in range(K)]
    rank_ema = [[e.clone() for e in ref.ema_buffers] for _ in range(K)]
    for step in range(2):
        x, y = _batch(20 + step, K * B)
        loss = ts.step_eager(x, y)
        loss_ref = _definition_step(ref, K, x, y, rank_bufs, rank_ema)
        assert torch.equal(loss, loss_ref), (step, loss.item(), loss_ref.item())
    _assert_same(_state(ts), _state(ref), "state")
    names = [n for n, _ in m.named_buffers()]
    for k in range(K):
        _assert_same(_bufs(ts, k), dict(zip(names, rank_bufs[k])), "buffers of rank %d" % k)
        _assert_same(_bufs(ts, k, True), dict(zip(names, rank_ema[k])), "EMA buffers of rank %d" % k)
    assert not torch.equal(ts.rank_buffers(0)[names[0]], ts.rank_buffers(1)[names[0]])   # the ranks saw different batches


# ------------------------------------------------------------------------------------------------ graph replay == eager
@pytest.mark.parametrize("mode", ["batch", "elem"])
def test_graph_replay_equals_eager(mode, deterministic):
    from cotnet_b200 import trainer
    K, B, res = 2, 4, 96
    kw = dict(lr=0.02, momentum=0.9, weight_decay=1e-3, ema_decay=0.9, label_smoothing=0.1, virtual_ranks=K)

    def draws(seed):
        mixers = [trainer.MixupCutmix(mode=mode, num_classes=16, seed=seed + k) for k in range(K)]
        g0 = torch.Generator().manual_seed(seed)
        while True:
            x_u8 = torch.randint(0, 256, (K * B, 3, res, res), generator=g0, dtype=torch.uint8).cuda()
            y = torch.randint(0, 16, (K * B,), generator=g0).cuda()
            mix = [mx.draw(B, res, res) for mx in mixers]
            x = torch.cat([trainer.normalize_u8(x_u8[k * B:(k + 1) * B].contiguous(), MEAN, STD, mix=mix[k]) for k in range(K)])
            yield x, y, mix

    # fixed stochastic-depth scales and DropBlock key: the captured step against the eager step
    m1 = _model(drop_path_rate=0.2, drop_block_rate=0.2)
    m1.fixed_drop_path_scales = torch.tensor([1.0, 0.0, 1.25, 1.25], device="cuda").view(1, 4).repeat(len(m1.blocks()), 1)
    m1.fixed_drop_block_key = torch.tensor([3, 4], device="cuda")          # no host copy inside the captured graph
    m2 = copy.deepcopy(m1)
    t1, t2 = trainer.TrainStep(m1, **kw), trainer.TrainStep(m2, **kw)
    d1 = draws(7)
    x, y, mix = next(d1)
    info = t1.capture(x, y, warmup=2, mix=mix)
    for _ in range(2):
        t2.step_eager(x, y, mix)
    la, lb = [], []
    for step in range(4):
        x, y, mix = next(d1)
        for t in (t1, t2):
            t.set_lr(0.02 / (step + 1))
        la.append(t1.step(x, y, mix=mix).item())
        lb.append(t2.step_eager(x, y, mix).item())
    assert la == lb, (la, lb)
    _assert_same(_state(t1), _state(t2), "state")
    for k in range(K):
        _assert_same(_bufs(t1, k), _bufs(t2, k), "buffers")
        _assert_same(_bufs(t1, k, True), _bufs(t2, k, True), "ema buffers")
    with pytest.raises(ValueError, match="list of 2"):
        t1.step(x, y, mix=mix[0])

    # drawn stochastic depth and DropBlock: two runs of the captured step are bit-identical
    runs = []
    for _ in range(2):
        t = trainer.TrainStep(_model(drop_path_rate=0.2, drop_block_rate=0.2), **kw)
        d = draws(9)
        x, y, mix = next(d)
        torch.manual_seed(13)
        t.capture(x, y, warmup=1, mix=mix)
        losses = []
        for step in range(3):
            x, y, mix = next(d)
            t.set_lr(0.01 * (step + 1))
            losses.append(t.step(x, y, mix=mix).item())
        runs.append((losses, _state(t), _bufs(t, 1)))
    assert runs[0][0] == runs[1][0]
    _assert_same(runs[0][1], runs[1][1], "state")
    _assert_same(runs[0][2], runs[1][2], "rank 1 buffers")
    assert info["cuda_graph"]


# ------------------------------------------------------------------------------------------------ virtual ranks == real ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _real_rank(rank, world, port, path):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    from cotnet_b200 import dist as cdist
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    cdist.init_from_env(backend="gloo")
    torch.cuda.set_device(0)
    out = _run_two_ranks(rank)
    torch.save(out, path)
    dist.destroy_process_group()


def _run_two_ranks(rank):
    """rank None: one process with two virtual ranks; rank r: real rank r of two."""
    from cotnet_b200 import trainer
    B = 4
    kw = dict(lr=0.02, momentum=0.9, weight_decay=1e-3, ema_decay=0.9, bucket_dtype=torch.float32, opt="adamw")
    ts = trainer.TrainStep(_model(), virtual_ranks=2 if rank is None else 1, **kw)
    for step in range(2):
        x, y = _batch(40 + step, 2 * B, res=64)
        if rank is not None:
            x, y = x[rank * B:(rank + 1) * B].contiguous(memory_format=CL), y[rank * B:(rank + 1) * B]
        ts.step_eager(x, y)
    before = [_bufs(ts, k) for k in range(2 if rank is None else 1)]
    ts.distribute_bn()
    torch.cuda.synchronize()
    cpu = lambda d: {k: v.cpu() for k, v in d.items()}              # noqa: E731
    return dict(state=cpu(_state(ts)), before=[cpu(b) for b in before],
                after=[cpu(_bufs(ts, k)) for k in range(2 if rank is None else 1)],
                ema_after=[cpu(_bufs(ts, k, True)) for k in range(2 if rank is None else 1)])


def test_virtual_ranks_equal_real_ranks(tmp_path, deterministic):
    world = 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    paths = [str(tmp_path / ("rank%d.pt" % r)) for r in range(world)]
    procs = [ctx.Process(target=_real_rank, args=(r, world, port, paths[r])) for r in range(world)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(600)
            assert p.exitcode == 0, p.exitcode
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)
    real = [torch.load(p) for p in paths]
    virt = _run_two_ranks(None)
    for r in range(world):
        _assert_same(real[r]["state"], virt["state"], "weights / optimizer state / EMA of rank %d" % r)
        _assert_same(real[r]["before"][0], virt["before"][r], "buffers of rank %d before distribute_bn" % r)
        _assert_same(real[r]["after"][0], virt["after"][r], "buffers of rank %d after distribute_bn" % r)
        _assert_same(real[r]["ema_after"][0], virt["ema_after"][r], "EMA buffers of rank %d after distribute_bn" % r)


# ------------------------------------------------------------------------------------------------ EvalStep after K > 1 training
def test_eval_step_reads_rank_zero_then_the_averages(deterministic):
    from cotnet_b200 import evaler, trainer
    K, B = 2, 4
    m = _model()
    ts = trainer.TrainStep(m, virtual_ranks=K, lr=0.02, ema_decay=0.9)
    for step in range(2):
        ts.step_eager(*_batch(60 + step, K * B, res=64))
    with torch.no_grad():                                            # make rank 1 clearly different
        for n, t in ts.rank_buffers(1).items():
            if "running_mean" in n:
                t.add_(0.5)
        for n, t in ts.rank_buffers(1, ema=True).items():
            if "running_mean" in n:
                t.add_(0.5)
    ev = evaler.EvalStep(m, 8, 64, train_step=ts)
    ev.capture()
    xe, ye = _batch(70, 8, res=64)

    def eager(which):
        """The eval forward with the module's buffers (live) or the EMA state bound, outside any graph."""
        evaler.drop_weight_caches(m)
        m.eval()
        try:
            with torch.no_grad(), ev._bound(which), torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False):
                return m(xe).float()
        finally:
            m.train()
            evaler.drop_weight_caches(m)

    def rel(a, b):
        return ((a - b).norm() / b.norm()).item()

    for which in ("live", "ema"):
        mod0 = eager(which)
        got = ev.run(xe, ye, which=which).float().clone()
        assert rel(got, mod0) <= 1e-3, (which, rel(got, mod0))
        # rank 1's buffers give other logits: the graph did not read them
        saved = [t.clone() for t in (ts.ema_buffers if which == "ema" else ts._buf_sets[0])]
        src = ts._ema_sets[1] if which == "ema" else ts._buf_sets[1]
        dst = ts.ema_buffers if which == "ema" else ts._buf_sets[0]
        with torch.no_grad():
            for d, s in zip(dst, src):
                d.copy_(s)
            mod1 = eager(which)
            for d, s in zip(dst, saved):
                d.copy_(s)
        assert rel(mod1, mod0) >= 1e-2, (which, rel(mod1, mod0))
    ts.distribute_bn()
    for k in range(K):
        for which in (False, True):
            _assert_same(_bufs(ts, 0, which), _bufs(ts, k, which), "averaged sets")
    for which in ("live", "ema"):
        got = ev.run(xe, ye, which=which).float().clone()
        want = eager(which)
        assert rel(got, want) <= 1e-3, (which, rel(got, want))
