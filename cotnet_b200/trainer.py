"""One data-parallel training step of a CoT network, H100-native (SURVEY.md section 8e + 8f rank 3).

Mirrors the body of the reference's training loop -- forward under autocast, loss, backward, ``optimizer.step()``,
``model_ema.update(model)`` (/root/reference/train.py:255-277) -- and what DistributedDataParallel does around it
(train.py:113-115): gradients averaged over the ranks.  Same results, different plumbing:

* **Flat state.**  fp32 master weights ``P``, momentum ``M``, optional EMA ``E`` live in flat buffers; the >=2-D weights
  the convolutions read are a bf16 copy ``Pb`` written by the optimizer kernel (the reference's AMP path casts every
  weight every step).  1-D parameters (BatchNorm / GroupNorm affine, biases) stay fp32 and un-decayed, exactly the split
  of ``optim_factory.add_weight_decay`` (optim/optim_factory.py:18-30).
* **No accumulate kernels.**  ``p.grad`` is None when backward starts, so autograd hands every gradient over without an
  ``add_``; ONE gather launch (``cotb200_multi_gather``, pointer table) packs them into the flat bucket.
* **Bucketed overlap.**  The bucket is cut into ``comm_chunks`` ranges in forward order; when the last gradient of a range
  has been produced (post-accumulate hook) the range is gathered and all-reduced (NCCL, AVG) on a side stream while the
  backward of the earlier layers is still running.  Everything -- forward, backward, gathers, NCCL, optimizer -- is
  captured in ONE CUDA graph (fork/join through events); if NCCL cannot be captured the collectives run eagerly between
  a fwd+bwd graph and an optimizer graph.
* **One optimizer pass.**  ``cotb200_sgd_ema_step``: SGD-nesterov + weight decay + EMA + bf16 copy, hyper-parameters read
  from device memory (LR schedules work under graph replay); ``cotb200_multi_lerp`` for the EMA of the buffers.

There is no CPU fallback of the kernels; the planning logic (``plan_flat``) is pure Python and unit-tested on CPU.
"""
import ctypes

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F

from . import _lib, fused

#: COTB200_BOOKKEEPING=0: one `num_batches_tracked += 1` kernel per BatchNorm instead of one multi-tensor add per step.
#: COTB200_ARENA_ESCAPE=1 (opt-in): BatchNorm / GroupNorm gradient sums from the pre-zeroed step arena instead of torch.zeros (~140 fill
#: launches per step less).  Off by default: the gradients of 1-D parameters would then alias memory that the next step_begin()
#: recycles.
import os as _os
_BOOKKEEPING = _os.environ.get("COTB200_BOOKKEEPING", "1") != "0"
_ARENA_ESCAPE = _os.environ.get("COTB200_ARENA_ESCAPE", "0") != "0"

ALIGN = 8          # elements: every parameter slot starts 16-byte aligned in the bf16 bucket (32 B in fp32)


def plan_flat(named_params, comm_chunks=3):
    """Partition parameters like optim_factory.add_weight_decay (big = decayed >=2-D weights, small = 1-D / bias) and lay
    each group out in a flat buffer.  Returns dict(big=[(name, p, offset)], small=[...], n_big, n_small,
    chunks=[(lo, hi, [indices into big])]) with chunk boundaries on parameter boundaries, in forward (registration) order."""
    big, small = [], []
    ob = os_ = 0
    for name, p in named_params:
        if not p.requires_grad:
            continue
        n = p.numel()
        slot = (n + ALIGN - 1) // ALIGN * ALIGN
        if p.dim() == 1 or name.endswith(".bias"):
            small.append((name, p, os_))
            os_ += slot
        else:
            big.append((name, p, ob))
            ob += slot
    chunks = []
    if big:
        k = max(1, min(comm_chunks, len(big)))
        target = ob / k
        lo_i, lo = 0, 0
        for c in range(k):
            if c == k - 1:
                hi_i = len(big)
            else:
                hi_i = lo_i
                while hi_i < len(big) - (k - 1 - c) and (hi_i == lo_i or big[hi_i][2] < (c + 1) * target):
                    hi_i += 1
            hi = big[hi_i][2] if hi_i < len(big) else ob
            chunks.append((lo, hi, list(range(lo_i, hi_i))))
            lo_i, lo = hi_i, hi
    return {"big": big, "small": small, "n_big": ob, "n_small": os_, "chunks": chunks}


class _Seg(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("offset", ctypes.c_longlong), ("numel", ctypes.c_longlong),
                ("dtype", ctypes.c_int), ("pad_", ctypes.c_int)]


class _Seg2(ctypes.Structure):
    _fields_ = [("dst", ctypes.c_void_p), ("src", ctypes.c_void_p), ("numel", ctypes.c_longlong),
                ("dtype", ctypes.c_int), ("pad_", ctypes.c_int)]


def _strided_view(flat, p, off):
    return torch.as_strided(flat, p.size(), p.stride(), off)


class _GatherTable:
    """Pinned host table + device copy for one gather launch (the copy is issued on the launch stream, so under CUDA-graph
    capture it becomes a memcpy node that re-reads the same pinned table at every replay)."""

    def __init__(self, n_tensors, max_blocks, device):
        self.seg_h = torch.zeros(n_tensors * ctypes.sizeof(_Seg), dtype=torch.uint8).pin_memory()
        self.blk_h = torch.zeros(max_blocks * 2, dtype=torch.int32).pin_memory()
        self.seg_d = torch.zeros_like(self.seg_h, device=device)
        self.blk_d = torch.zeros_like(self.blk_h, device=device)
        self.done = None                     # event after the last H2D copy (eager mode: host table reuse)

    def fill(self, entries, chunk):
        """entries: [(ptr, offset, numel, dtype_code)] -> number of blocks."""
        if self.done is not None:
            self.done.synchronize()          # the previous (eager) upload has finished reading the pinned table
            self.done = None
        segs = (_Seg * len(entries)).from_address(self.seg_h.data_ptr())
        for i, (ptr, off, n, dt) in enumerate(entries):
            segs[i].ptr, segs[i].offset, segs[i].numel, segs[i].dtype = ptr, off, n, dt
        per = np.array([(e[2] + chunk - 1) // chunk for e in entries], dtype=np.int64)
        nb = int(per.sum())
        blk = self.blk_h.numpy()[:2 * nb].reshape(nb, 2)
        blk[:, 0] = np.repeat(np.arange(len(entries), dtype=np.int32), per)
        starts = np.repeat(np.cumsum(per) - per, per)
        blk[:, 1] = (np.arange(nb, dtype=np.int64) - starts).astype(np.int32)
        return nb

    def upload(self, capturing):
        self.seg_d.copy_(self.seg_h, non_blocking=True)
        self.blk_d.copy_(self.blk_h, non_blocking=True)
        if not capturing:
            self.done = torch.cuda.Event()
            self.done.record()


class TrainStep:
    #: tests/test_dist_cpu.py drives the bucket / chunk / hook / all-reduce logic on CPU tensors over gloo through a subclass
    #: that sets this flag and replaces the two kernel-launching methods (_launch_gather, optimizer_step) with torch ops.
    #: The product class refuses CPU models.
    _host_logic_only = False

    def __init__(self, model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=None,
                 loss_fn=None, amp_dtype=torch.bfloat16, weights="bf16", bucket_dtype=None, comm_chunks=3, overlap=True,
                 process_group=None, label_smoothing=0.):
        """label_smoothing > 0, or a `mix` given to the step, selects the soft-target loss (soft_target_cross_entropy) that the
        reference recipe trains with (train.py:198-209); otherwise the loss is `loss_fn` (default F.cross_entropy)."""
        self.model = model
        self.loss_fn = loss_fn or (lambda out, lab: F.cross_entropy(out.float(), lab))
        self.label_smoothing = float(label_smoothing)
        self._gmix = None
        self.amp_dtype = amp_dtype
        self.nesterov = bool(nesterov)
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        dev = next(model.parameters()).device
        self._cuda = dev.type == "cuda"
        if not self._cuda and not self._host_logic_only:
            raise RuntimeError("TrainStep: the model must live on a CUDA device (libcotb200 has no CPU path)")
        self.dev = dev
        self.lib = _lib.load() if self._cuda else None
        self.chunk_elems = int(self.lib.cotb200_gather_chunk()) if self._cuda else 8192
        self.overlap = bool(overlap) and self.world > 1
        plan = plan_flat(list(model.named_parameters()), comm_chunks if self.overlap else 1)
        self.plan = plan
        nb, ns = plan["n_big"], plan["n_small"]
        self.weights_bf16 = (weights == "bf16")
        if bucket_dtype is None:
            bucket_dtype = torch.bfloat16 if self.weights_bf16 else torch.float32
        self.bucket_dtype = bucket_dtype
        f32 = dict(dtype=torch.float32, device=dev)
        with torch.no_grad():
            self.P_big, self.P_small = torch.zeros(nb, **f32), torch.zeros(ns, **f32)
            self.M_big, self.M_small = torch.zeros(nb, **f32), torch.zeros(ns, **f32)
            self.Pb = torch.zeros(nb, dtype=torch.bfloat16, device=dev) if self.weights_bf16 else None
            self.G_big = torch.zeros(nb, dtype=bucket_dtype, device=dev)
            self.G_small = torch.zeros(ns, **f32)
            for _, p, off in plan["big"]:
                _strided_view(self.P_big, p, off).copy_(p.detach())
                if self.weights_bf16:
                    _strided_view(self.Pb, p, off).copy_(p.detach())
                    p.data = _strided_view(self.Pb, p, off)
                else:
                    p.data = _strided_view(self.P_big, p, off)
                p.grad = None
            for _, p, off in plan["small"]:
                _strided_view(self.P_small, p, off).copy_(p.detach())
                p.data = _strided_view(self.P_small, p, off)
                p.grad = None
            self.ema = ema_decay is not None
            self.E_big = self.P_big.clone() if self.ema else None
            self.E_small = self.P_small.clone() if self.ema else None
            self.ema_buffers = None
            if self.ema:
                bufs = [b for _, b in model.named_buffers()]
                self.ema_buffers = [b.detach().clone() for b in bufs]
                segs = (_Seg2 * max(1, len(bufs)))()
                keep = 0
                for b, e in zip(bufs, self.ema_buffers):
                    if b.dtype == torch.float32:
                        code = _lib.F32
                    elif b.dtype == torch.int64:
                        code = 100
                    else:
                        continue
                    segs[keep].dst, segs[keep].src, segs[keep].numel, segs[keep].dtype = e.data_ptr(), b.data_ptr(), b.numel(), code
                    keep += 1
                self._lerp_tab = None
                if keep:
                    raw = torch.frombuffer(bytearray(bytes(segs)), dtype=torch.uint8)[:keep * ctypes.sizeof(_Seg2)]
                    self._lerp_tab = raw.to(dev)
                self._lerp_n = keep
        self.hyper = torch.tensor([lr, momentum, weight_decay, ema_decay if self.ema else 0.0, 1.0], **f32)
        self.hyper_small = self.hyper.clone()
        self.hyper_small[2] = 0.0                                   # no weight decay on 1-D parameters / biases
        if self.world > 1 and dist.get_backend(process_group) != "nccl":
            self.hyper[4] = self.hyper_small[4] = 1.0 / self.world  # SUM all-reduce: the optimizer kernel applies 1/world
        # gather tables: one per comm chunk of the big bucket + one for the small bucket
        def blocks_of(items):
            return sum((p.numel() + self.chunk_elems - 1) // self.chunk_elems for _, p, _ in items)
        if self._cuda:
            self._tabs = [_GatherTable(len(idx), blocks_of([plan["big"][i] for i in idx]), dev) for _, _, idx in plan["chunks"]]
            self._tab_small = _GatherTable(max(1, len(plan["small"])), max(1, blocks_of(plan["small"])), dev)
        else:
            self._tabs, self._tab_small = [None] * len(plan["chunks"]), None
        self._chunk_of = {}
        for c, (_, _, idx) in enumerate(plan["chunks"]):
            for i in idx:
                self._chunk_of[id(plan["big"][i][1])] = c
        self._pending = [0] * len(plan["chunks"])
        self._flushed = [False] * len(plan["chunks"])
        self._capturing = False
        self.comm_stream = torch.cuda.Stream(device=dev) if (self.world > 1 and self._cuda) else None
        self._graph = None
        self.exposed_comm_ms = None
        if self.overlap:
            for _, p, _ in plan["big"]:
                p.register_post_accumulate_grad_hook(self._on_grad)

    # ------------------------------------------------------------------ hyper-parameters
    def set_lr(self, lr):
        self.hyper[0:1].fill_(lr)
        self.hyper_small[0:1].fill_(lr)

    # ------------------------------------------------------------------ gradient plumbing
    def _on_grad(self, p):
        c = self._chunk_of.get(id(p))
        if c is None or self._flushed[c]:
            return
        self._pending[c] -= 1
        if self._pending[c] == 0:
            self._flush_chunk(c)

    def _entries(self, items):
        ent, missing = [], False
        for _, p, off in items:
            g = p.grad
            if g is None:
                missing = True
                continue
            if any(a_ != b_ for a_, b_, n_ in zip(g.stride(), p.stride(), p.shape) if n_ != 1):   # same memory order? (size-1 dims are free)
                t = torch.empty_strided(p.size(), p.stride(), dtype=g.dtype, device=g.device)
                t.copy_(g)
                p.grad = g = t
            ent.append((g.data_ptr(), off, g.numel(), _lib.dtype_code(g)))
        return ent, missing

    def _gather(self, tab, items, bucket, lo, hi):
        ent, missing = self._entries(items)
        if missing:
            bucket[lo:hi].zero_()
        if not ent:
            return
        self._launch_gather(tab, ent, bucket, [p.grad for _, p, _ in items if p.grad is not None])

    def _launch_gather(self, tab, ent, bucket, grads):
        nb = tab.fill(ent, self.chunk_elems)
        tab.upload(self._capturing)
        st = torch.cuda.current_stream(self.dev).cuda_stream
        _lib.check(self.lib.cotb200_multi_gather(tab.seg_d.data_ptr(), tab.blk_d.data_ptr(), nb, _lib.dtype_code(bucket),
                                                 bucket.data_ptr(), 1.0, st), "multi_gather")

    def _all_reduce(self, t):
        if dist.get_backend(self.pg) == "nccl":
            dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.pg)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.pg)

    def _all_reduce_side(self, t):
        """All-reduce on the communication stream, ordered after everything issued so far on the current stream."""
        if self.comm_stream is None:
            self._all_reduce(t)
            return
        self.comm_stream.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.comm_stream):
            self._all_reduce(t)

    def _flush_chunk(self, c):
        """Gather chunk c of the big bucket on the current (backward) stream and all-reduce it on the side stream."""
        lo, hi, idx = self.plan["chunks"][c]
        self._flushed[c] = True
        self._gather(self._tabs[c], [self.plan["big"][i] for i in idx], self.G_big, lo, hi)
        if self.world > 1:
            self._all_reduce_side(self.G_big[lo:hi])

    def _finish_grads(self):
        for c in range(len(self.plan["chunks"])):
            if not self._flushed[c]:
                self._flush_chunk(c)
        if self.plan["small"]:
            self._gather(self._tab_small, self.plan["small"], self.G_small, 0, self.plan["n_small"])
            if self.world > 1:
                self._all_reduce_side(self.G_small)
        if self.world > 1 and self.comm_stream is not None:
            torch.cuda.current_stream(self.dev).wait_stream(self.comm_stream)

    # ------------------------------------------------------------------ the step
    def _loss(self, out, lab, mix_dev):
        if mix_dev is None and self.label_smoothing == 0.:
            return self.loss_fn(out, lab)
        return SoftTargetCrossEntropyFn.apply(out, lab, mix_dev, self.label_smoothing)

    def forward_backward(self, x, lab, mix=None):
        """mix: None, a MixParams (MixupCutmix.draw) or its 32-byte device struct -- the loss reads the mixed targets' lam from it."""
        mix_dev = mix.on_stream(self.dev) if isinstance(mix, MixParams) else mix
        if self._cuda:
            fused.step_begin(self.dev)
            # every gradient of this step is gathered into the flat bucket before the next step_begin(): the BatchNorm gradient sums
            # may live in the step arena, and the ~100 `num_batches_tracked += 1` kernels become one multi-tensor add after the forward
            if _ARENA_ESCAPE:
                fused.arena_escape_ok(True)
            if _BOOKKEEPING:
                fused.defer_bn_counters(True)
        for _, p, _ in self.plan["big"]:
            p.grad = None
        for _, p, _ in self.plan["small"]:
            p.grad = None
        for c, (_, _, idx) in enumerate(self.plan["chunks"]):
            self._pending[c] = len(idx)
            self._flushed[c] = False
        with torch.autocast(self.dev.type, dtype=self.amp_dtype, enabled=self.amp_dtype is not None):
            out = self.model(x)
            loss = self._loss(out, lab, mix_dev)
        if self._cuda:
            fused.flush_bn_counters()
            fused.defer_bn_counters(False)
        loss.backward()
        self._finish_grads()
        if self._cuda:
            fused.arena_escape_ok(False)
        return loss

    def optimizer_step(self):
        st = torch.cuda.current_stream(self.dev).cuda_stream
        lib = self.lib
        if self.plan["n_big"]:
            _lib.check(lib.cotb200_sgd_ema_step(self.plan["n_big"], self.P_big.data_ptr(), self.M_big.data_ptr(),
                                                _lib.dtype_code(self.G_big), self.G_big.data_ptr(), _lib.ptr(self.E_big),
                                                _lib.ptr(self.Pb), self.hyper.data_ptr(), 1 if self.nesterov else 0, st),
                       "sgd_ema_step")
        if self.plan["n_small"]:
            _lib.check(lib.cotb200_sgd_ema_step(self.plan["n_small"], self.P_small.data_ptr(), self.M_small.data_ptr(), _lib.F32,
                                                self.G_small.data_ptr(), _lib.ptr(self.E_small), None,
                                                self.hyper_small.data_ptr(), 1 if self.nesterov else 0, st), "sgd_ema_step")
        if self.ema and self._lerp_n:
            _lib.check(lib.cotb200_multi_lerp(self._lerp_tab.data_ptr(), self._lerp_n, self.hyper.data_ptr(), st), "multi_lerp")

    def step_eager(self, x, lab, mix=None):
        loss = self.forward_backward(x, lab, mix)
        self.optimizer_step()
        return loss

    # ------------------------------------------------------------------ CUDA graph
    def capture(self, x, lab, warmup=3, capture_nccl=True, mix=None):
        """Warm up (cuDNN autotune, allocator) and capture the whole step.  Returns a dict describing the launch mode.
        With `mix` (a MixParams) the graph's loss reads a static copy of the mixing parameters that step(mix=) refreshes."""
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self.step_eager(x, lab, mix)
        torch.cuda.current_stream(self.dev).wait_stream(side)
        torch.cuda.synchronize(self.dev)
        for t in self._tabs + [self._tab_small]:
            t.done = None
        self._gx, self._glab = x.clone(), lab.clone()
        self._gmix = None if mix is None else mix.dev.clone()
        info = {"cuda_graph": True}
        lc0 = _lib.launch_count()
        try:
            if self.world > 1 and not capture_nccl:
                raise RuntimeError("NCCL capture disabled")
            g = torch.cuda.CUDAGraph()
            self._capturing = True
            with torch.cuda.graph(g):
                self._gloss = self.step_eager(self._gx, self._glab, self._gmix)
            self._capturing = False
            self._graph = ("one", g)
            info["graphs"] = "fwd+bwd+gather%s+optimizer in ONE graph" % ("+NCCL (side-stream branches)" if self.world > 1 else "")
        except Exception as e:          # noqa: BLE001 -- NCCL not capturable here: collectives run eagerly between two graphs
            self._capturing = False
            torch.cuda.synchronize(self.dev)
            if self.world == 1:
                raise
            info["nccl_capture_error"] = repr(e)[:200]
            lc0 = _lib.launch_count()
            saved_overlap, self.overlap = self.overlap, False
            world, self.world = self.world, 1                  # capture the gathers without any collective
            g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            self._capturing = True
            with torch.cuda.graph(g1):
                self._gloss = self.forward_backward(self._gx, self._glab, self._gmix)
            with torch.cuda.graph(g2):
                self.optimizer_step()
            self._capturing = False
            self.world, self.overlap = world, saved_overlap
            self._graph = ("two", g1, g2)
            info["graphs"] = "fwd+bwd+gather graph -> eager NCCL all-reduce of the flat buckets -> optimizer graph"
        info["libcotb200_kernels_per_replay"] = _lib.launch_count() - lc0
        return info

    def step(self, x=None, lab=None, mix=None):
        """One step; (x, lab) and the mixing parameters `mix` (MixupCutmix.draw) are copied into the graph's static inputs
        when a graph is active and they are given.  A graph captured with `mix` needs one at every step (it would otherwise replay
        the previous step's lam and box), and a graph captured without it refuses one."""
        if self._graph is None:
            return self.step_eager(x, lab, mix)
        if x is not None and x is not self._gx:
            self._gx.copy_(x, non_blocking=True)
            self._glab.copy_(lab, non_blocking=True)
        if (mix is None) != (self._gmix is None):
            raise ValueError("TrainStep.step: this graph was captured %s mixing parameters; pass mix= %s"
                             % (("without", "to capture() first") if mix is not None else ("with", "(MixupCutmix.draw) at every step")))
        if mix is not None:
            self._gmix.copy_(mix.on_stream(self.dev), non_blocking=True)
        if self._graph[0] == "one":
            self._graph[1].replay()
        else:
            self._graph[1].replay()
            self._all_reduce(self.G_big)
            if self.plan["small"]:
                self._all_reduce(self.G_small)
            self._graph[2].replay()
        return self._gloss

    def time_without_comm(self, steps, timed):
        """Step time (ms for `steps` steps, via the caller's `timed`) of the SAME step with every collective removed: what the
        bench subtracts to report the exposed (non-overlapped) communication time.  Captures a second graph when graphs are
        in use.  The weights still move (identical arithmetic per rank, no averaging), so call it after the real timing."""
        world, self.world = self.world, 1
        try:
            if self._graph is None:
                return timed(lambda: self.step_eager(self._gx, self._glab, self._gmix), steps)
            if self._graph[0] == "two":
                def run():
                    self._graph[1].replay()
                    self._graph[2].replay()
                return timed(run, steps)
            torch.cuda.synchronize(self.dev)
            g = torch.cuda.CUDAGraph()
            self._capturing = True
            with torch.cuda.graph(g):
                self.step_eager(self._gx, self._glab, self._gmix)
            self._capturing = False
            for _ in range(2):
                g.replay()
            return timed(g.replay, steps)
        finally:
            self._capturing = False
            self.world = world

    @property
    def static_inputs(self):
        return self._gx, self._glab

    # ------------------------------------------------------------------ state
    def master_state(self):
        """name -> fp32 master tensor (views) of every parameter."""
        out = {}
        for n, p, off in self.plan["big"]:
            out[n] = _strided_view(self.P_big, p, off)
        for n, p, off in self.plan["small"]:
            out[n] = _strided_view(self.P_small, p, off)
        return out

    def ema_state(self):
        """state_dict of the EMA model (parameters from the flat EMA buffers, buffers from their EMA copies)."""
        if not self.ema:
            return None
        out = {}
        for n, p, off in self.plan["big"]:
            out[n] = _strided_view(self.E_big, p, off)
        for n, p, off in self.plan["small"]:
            out[n] = _strided_view(self.E_small, p, off)
        for (n, _), e in zip(self.model.named_buffers(), self.ema_buffers):
            out[n] = e
        return out

    def grads(self):
        """name -> gradient view into the flat buckets (after forward_backward / a step)."""
        out = {}
        for n, p, off in self.plan["big"]:
            out[n] = _strided_view(self.G_big, p, off)
        for n, p, off in self.plan["small"]:
            out[n] = _strided_view(self.G_small, p, off)
        return out


def normalize_u8(x_u8, mean, std, dtype=torch.bfloat16, mix=None):
    """uint8 NCHW batch [N,C,H,W] (CUDA) -> (x - mean)/std as a channels_last tensor of `dtype`: the PrefetchLoader's
    normalisation (datasets/loader.py:86-90) + the layout / precision the AMP forward wants, in ONE kernel.
    mix: a MixParams of MixupCutmix.draw -- the batch is Mixup / CutMix-ed first, on the uint8 values, exactly like
    FastCollateMixup (datasets/mixup.py:282-299), in the same kernel."""
    assert x_u8.is_cuda and x_u8.dtype == torch.uint8 and x_u8.dim() == 4 and x_u8.is_contiguous()
    N, C, H, W = x_u8.shape
    y = torch.empty((N, C, H, W), dtype=dtype, device=x_u8.device, memory_format=torch.channels_last)
    mean = [float(m) for m in mean]
    std = [float(s) for s in std]
    assert len(mean) == C and len(std) == C
    mh, sh = (ctypes.c_float * C)(*mean), (ctypes.c_float * C)(*std)
    md = sd = None
    if not (C == 3 and (H * W) % 4 == 0):
        md = torch.tensor(mean, dtype=torch.float32, device=x_u8.device)
        sd = torch.tensor(std, dtype=torch.float32, device=x_u8.device)
    if mix is None:
        rc = _lib.load().cotb200_u8_to_nhwc(_lib.dtype_code(y), N, C, H, W, x_u8.data_ptr(), y.data_ptr(), mh, sh, _lib.ptr(md),
                                            _lib.ptr(sd), _lib.stream_ptr(x_u8))
        _lib.check(rc, "u8_to_nhwc")
        return y
    mix.check(N, H, W)
    rc = _lib.load().cotb200_u8_mix_to_nhwc(_lib.dtype_code(y), N, C, H, W, x_u8.data_ptr(), y.data_ptr(), mh, sh, _lib.ptr(md),
                                            _lib.ptr(sd), mix.on_stream(x_u8.device).data_ptr(), _lib.stream_ptr(x_u8))
    _lib.check(rc, "u8_mix_to_nhwc")
    return y


# ---------------------------------------------------------------------------------------------------- the training recipe
class MixParams:
    """One step's batch Mixup / CutMix parameters (struct cotb200_mix): `host` holds the values (a ctypes _lib.Mix), `dev` a
    device copy that the kernels read, `target_lam` the float64 lam of the draw (the struct holds it rounded to fp32).
    The device copy is made from a freshly pinned buffer of torch's caching host allocator, which does not hand that buffer out
    again before the copy has finished: the next draw() never races it.  The copy is issued on the stream current at draw();
    every consumer takes the struct through on_stream(), which orders its own current stream after that copy (an event wait)
    and tells the allocator that stream uses the memory, so drawing and consuming on different streams is safe."""
    MODES = (0, 1, 2)

    def __init__(self, host, device=None, target_lam=None):
        self.host = host
        self.target_lam = float(host.target_lam if target_lam is None else target_lam)
        self.dev = self._copied = None
        if device is not None:
            self.dev = torch.frombuffer(bytearray(bytes(host)), dtype=torch.uint8).pin_memory().to(device, non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record(torch.cuda.current_stream(self.dev.device))

    mode = property(lambda self: self.host.mode)
    box = property(lambda self: (self.host.y0, self.host.y1, self.host.x0, self.host.x1))

    def check(self, N, H, W):
        h = self.host
        if h.mode not in self.MODES:
            raise ValueError("mix: unknown mode %d (0 none, 1 mixup, 2 cutmix)" % h.mode)
        if N % 2:
            raise ValueError("mix: batch size %d must be even (the partner of sample n is N-1-n)" % N)
        if h.mode == 2 and not (0 <= h.y0 <= h.y1 <= H and 0 <= h.x0 <= h.x1 <= W):
            raise ValueError("mix: CutMix box %s outside the %dx%d image" % (self.box, H, W))

    def on_stream(self, device):
        """The device struct, ready for use on `device`'s current stream."""
        if self.dev is None or self.dev.device != torch.device(device):
            raise ValueError("mix: no device copy on %s (MixupCutmix(device=...))" % device)
        st = torch.cuda.current_stream(self.dev.device)
        st.wait_event(self._copied)
        self.dev.record_stream(st)
        return self.dev


class MixupCutmix:
    """Batch-mode Mixup / CutMix of the reference configs (FastCollateMixup, datasets/mixup.py; mode 'batch', correct_lam,
    no cutmix_minmax), drawing its parameters from its own np.random.RandomState(seed) in the reference's call order:
    rand < prob, rand < switch_prob, beta, randint (box centre row), randint (box centre column).
    `enabled = False` turns mixing off (mixup_off_epoch); draws then give lam = 1 without consuming random numbers."""

    def __init__(self, mixup_alpha=0.8, cutmix_alpha=1.0, prob=1.0, switch_prob=0.5, label_smoothing=0.1, num_classes=1000,
                 seed=0, correct_lam=True, device="cuda"):
        if not (mixup_alpha > 0. or cutmix_alpha > 0.):
            raise ValueError("MixupCutmix: mixup_alpha or cutmix_alpha must be > 0")
        self.mixup_alpha, self.cutmix_alpha = float(mixup_alpha), float(cutmix_alpha)
        self.prob, self.switch_prob = float(prob), float(switch_prob)
        self.label_smoothing, self.num_classes = float(label_smoothing), int(num_classes)
        self.correct_lam = bool(correct_lam)
        self.rng = np.random.RandomState(seed)
        self.enabled = True
        self.device = None if device is None else torch.device(device)

    def _params_per_batch(self):                                    # datasets/mixup.py:143-159
        lam, use_cutmix = 1., False
        if self.enabled and self.rng.rand() < self.prob:
            if self.mixup_alpha > 0. and self.cutmix_alpha > 0.:
                use_cutmix = self.rng.rand() < self.switch_prob
                lam_mix = (self.rng.beta(self.cutmix_alpha, self.cutmix_alpha) if use_cutmix
                           else self.rng.beta(self.mixup_alpha, self.mixup_alpha))
            elif self.mixup_alpha > 0.:
                lam_mix = self.rng.beta(self.mixup_alpha, self.mixup_alpha)
            else:
                use_cutmix = True
                lam_mix = self.rng.beta(self.cutmix_alpha, self.cutmix_alpha)
            lam = float(lam_mix)
        return lam, bool(use_cutmix)

    def draw(self, B, H, W):
        """Parameters of the next batch of B images of H x W as a MixParams (host struct + device copy)."""
        if B % 2:
            raise ValueError("MixupCutmix: batch size %d must be even" % B)
        lam, use_cutmix = self._params_per_batch()
        m = _lib.Mix()
        if use_cutmix:                                              # rand_bbox + cutmix_bbox_and_lam (:30-87), margin 0
            ratio = np.sqrt(1 - lam)
            cut_h, cut_w = int(H * ratio), int(W * ratio)
            cy, cx = self.rng.randint(0, H), self.rng.randint(0, W)
            m.y0, m.y1 = int(np.clip(cy - cut_h // 2, 0, H)), int(np.clip(cy + cut_h // 2, 0, H))
            m.x0, m.x1 = int(np.clip(cx - cut_w // 2, 0, W)), int(np.clip(cx + cut_w // 2, 0, W))
            if self.correct_lam:
                lam = 1. - (m.y1 - m.y0) * (m.x1 - m.x0) / float(H * W)
        m.mode = 0 if lam == 1. else (2 if use_cutmix else 1)
        # numpy 2 weak scalars: float32 pixels * python float multiplies by the float rounded to fp32 (:296)
        m.lam, m.one_minus_lam = float(np.float32(lam)), float(np.float32(1 - lam))
        m.target_lam = lam
        return MixParams(m, self.device, lam)


class SoftTargetCrossEntropyFn(torch.autograd.Function):
    """SoftTargetCrossEntropy()(logits, mixup_target(labels, K, lam, smoothing)) (loss/cross_entropy.py:29-36,
    datasets/mixup.py:17-27) on cotb200_soft_ce / cotb200_soft_ce_bwd; lam is read on the device from `mix_dev` (the struct of
    a MixParams; None = no mixing, i.e. LabelSmoothingCrossEntropy, and plain cross entropy with smoothing 0).  logits
    [B, K] fp32 / bf16 / fp16 with unit column stride; labels int64 [B].  Returns the fp32 batch mean."""

    @staticmethod
    def forward(ctx, logits, labels, mix_dev, smoothing):
        assert logits.is_cuda and logits.dim() == 2 and logits.stride(1) == 1 and labels.dtype == torch.int64
        B, K = logits.shape
        logits, labels = logits.detach(), labels.contiguous()
        rows = torch.empty(2, B, dtype=torch.float32, device=logits.device)
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        lib, st, dt = _lib.load(), _lib.stream_ptr(logits), _lib.dtype_code(logits)
        _lib.check(lib.cotb200_soft_ce(dt, B, K, logits.data_ptr(), logits.stride(0), labels.data_ptr(), _lib.ptr(mix_dev),
                                       float(smoothing), rows.data_ptr(), loss.data_ptr(), st), "soft_ce")
        ctx.save_for_backward(logits, labels, mix_dev, rows)
        ctx.smoothing = float(smoothing)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        logits, labels, mix_dev, rows = ctx.saved_tensors
        B, K = logits.shape
        dloss = dloss.float().contiguous()
        dz = torch.empty(B, K, dtype=torch.float32, device=logits.device)
        lib, st, dt = _lib.load(), _lib.stream_ptr(logits), _lib.dtype_code(logits)
        _lib.check(lib.cotb200_soft_ce_bwd(dt, B, K, logits.data_ptr(), logits.stride(0), labels.data_ptr(), _lib.ptr(mix_dev),
                                           ctx.smoothing, rows.data_ptr(), dloss.data_ptr(), dz.data_ptr(), K, st), "soft_ce_bwd")
        return dz.to(logits.dtype), None, None, None


def soft_target_cross_entropy(logits, labels, mix=None, smoothing=0.):
    """The recipe's loss: mean over the batch of -sum_c t_c log softmax(logits)_c with t = mixup_target(labels, K, mix.target_lam,
    smoothing).  mix: None or a MixParams (MixupCutmix.draw)."""
    return SoftTargetCrossEntropyFn.apply(logits, labels, None if mix is None else mix.on_stream(logits.device), smoothing)
