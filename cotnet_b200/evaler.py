"""Validation on the library's kernels: the reference's evaler (evaler/evaler.py:37-57, utils/meters.py:12-19) as a CUDA graph.

The reference evaluates with ``model.eval()``, ``no_grad`` and autocast, computes top-1 / top-5 with ``output.topk(5)`` + ``eq``
and synchronises after every batch; at the end of the epoch it does the same again for the EMA model (train.py:346-355).
``EvalStep`` captures the eval-mode forward at a fixed batch size into a CUDA graph whose last node is ``cotb200_topk_hits``: the
hit counts accumulate as int64 on the device, so a whole validation pass runs without a host synchronisation, and the short last
batch is handled by a device-side row count.  ``result()`` does one all-reduce and one device-to-host copy.

Up to two graphs, sharing one memory pool (they never run at the same time):

* ``"live"`` reads the model's own parameters and buffers in place (under a ``TrainStep``: the flat ``Pb`` / ``P_small`` and the
  model's buffers).  Nothing is copied.
* ``"ema"`` (a ``TrainStep`` built with ``ema_decay``) reads the flat EMA state: its first node rounds ``E_big`` to a bf16 ``Eb``
  (round to nearest even, what ``.to(torch.bfloat16)`` gives; with ``weights="fp32"`` the graph reads ``E_big`` itself), plus
  ``E_small`` and ``ema_buffers``.  During that capture the parameters' ``.data`` and the buffers are rebound to those tensors
  and restored afterwards: the graph bakes the pointers it was captured with.

Rules of the road, checked or enforced by ``capture()``:

* The eval forward must not touch what a training graph owns.  The pre-zeroed step arena of ``fused`` is switched off while
  capturing, so every accumulator of the eval graph is a memset node of its own pool.
* The inference paths cache bf16 / BatchNorm-folded copies of the weights keyed by the tensors' version counters, which the
  optimizer kernels (raw pointer writes) and ``.data`` rebinding do not bump.  The caches are dropped before each capture, so the
  graph recomputes them from the live (or EMA) tensors at every replay, and again after it, so that eager code never reuses a
  graph-owned copy.
* BatchNorm runs on running statistics in eval mode; ``capture()`` checks that no buffer changed.
"""
import contextlib
import ctypes

import torch
import torch.distributed as dist

from . import _lib, fused
from .trainer import _strided_view

#: per-module attributes holding eval-mode copies of weights (cot_layer.CotLayer._tc_params, fused._se_eval_params)
_WEIGHT_CACHES = ("_tc_cache", "_cotb200_eval_cache")


def topk_hits(logits, labels, counts, topk=(1, 5), valid=None):
    """counts += [hits at each k of topk..., rows counted, rows with a label outside [0, K)] (cotb200_topk_hits, the rank rule of
    include/cotb200.h).  logits [B, K] fp32 / bf16 / fp16 with unit column stride; labels int64 [B]; counts int64 [len(topk) + 2]
    on the device; valid: None (all B rows) or a device int32 [1] with the number of leading rows to count.  Returns counts."""
    _lib.require_cuda(logits, "topk_hits")
    if logits.dim() != 2 or logits.stride(1) != 1:
        raise ValueError("topk_hits: logits must be [B, K] with unit column stride")
    if labels.dtype != torch.int64 or labels.dim() != 1 or labels.shape[0] != logits.shape[0] or not labels.is_contiguous():
        raise ValueError("topk_hits: labels must be a contiguous int64 [B]")
    if counts.dtype != torch.int64 or counts.numel() != len(topk) + 2 or not counts.is_contiguous():
        raise ValueError("topk_hits: counts must be a contiguous int64 [len(topk) + 2]")
    if valid is not None and (valid.dtype != torch.int32 or valid.numel() != 1):
        raise ValueError("topk_hits: valid must be a device int32 [1]")
    B, K = logits.shape
    ks = (ctypes.c_int * len(topk))(*[int(k) for k in topk])
    _lib.check(_lib.load().cotb200_topk_hits(_lib.dtype_code(logits), B, K, logits.data_ptr(), logits.stride(0), labels.data_ptr(),
                                             _lib.ptr(valid), len(topk), ks, counts.data_ptr(), _lib.stream_ptr(logits)), "topk_hits")
    return counts


def drop_weight_caches(model):
    """Forget the eval-mode weight copies cached on the modules of `model` (see the module docstring)."""
    for m in model.modules():
        for name in _WEIGHT_CACHES:
            m.__dict__.pop(name, None)


class EvalStep:
    """Graph-captured validation step of `model` at batch size `batch` and resolution `res` (int or (H, W)).

    train_step: the TrainStep that owns the model's weights (needed for the "ema" graph; None for a model loaded only to be
    evaluated).  topk: up to four values of k (the reference reports top-1 and top-5).  Inputs are the normalised,
    channels_last batch (trainer.normalize_u8(..., mix=None) turns the loader's uint8 batch into it); labels int64 on the device."""

    def __init__(self, model, batch, res, amp_dtype=torch.bfloat16, train_step=None, topk=(1, 5)):
        if not 1 <= len(topk) <= 4:
            raise ValueError("EvalStep: 1 to 4 values of k, got %r" % (topk,))
        self.model = model
        self.ts = train_step
        if train_step is not None and train_step.model is not model:
            raise ValueError("EvalStep: train_step belongs to another model")
        self.dev = next(model.parameters()).device
        _lib.require_cuda(next(model.parameters()), "EvalStep")
        self.batch = int(batch)
        H, W = (res, res) if isinstance(res, int) else res
        self.amp_dtype = amp_dtype
        self.topk = tuple(int(k) for k in topk)
        self.x = torch.zeros(self.batch, 3, H, W, dtype=amp_dtype or torch.float32,
                             device=self.dev).contiguous(memory_format=torch.channels_last)
        self.labels = torch.zeros(self.batch, dtype=torch.int64, device=self.dev)
        self.valid = torch.full((1,), self.batch, dtype=torch.int32, device=self.dev)
        self.counts = {}
        self.logits = {}                     # static outputs: which -> [batch, K] (rows >= the valid count are stale)
        self._graphs = {}
        self._pool = None
        self._eb = None

    @property
    def has_ema(self):
        return self.ts is not None and self.ts.ema

    # ------------------------------------------------------------------ capture
    def _body(self, which):
        with torch.no_grad(), torch.autocast(self.dev.type, dtype=self.amp_dtype, enabled=self.amp_dtype is not None,
                                             cache_enabled=False):
            if which == "ema" and self._eb is not None:
                self._eb.copy_(self.ts.E_big)
            out = self.model(self.x)
        topk_hits(out, self.labels, self.counts[which], self.topk, self.valid)
        return out

    @contextlib.contextmanager
    def _bound(self, which):
        """The model's parameters and buffers rebound to the EMA state for the duration of the block ("ema"), or untouched."""
        if which == "live":
            yield
            return
        ts = self.ts
        big = self._eb if self._eb is not None else ts.E_big
        saved = []
        try:
            for _, p, off in ts.plan["big"]:
                saved.append((p, p.data))
                p.data = _strided_view(big, p, off)
            for _, p, off in ts.plan["small"]:
                saved.append((p, p.data))
                p.data = _strided_view(ts.E_small, p, off)
            for (_, b), e in zip(self.model.named_buffers(), ts.ema_buffers):
                saved.append((b, b.data))
                b.data = e
            yield
        finally:
            for t, d in reversed(saved):
                t.data = d

    def capture(self, warmup=2):
        """Warm up and capture the "live" graph, and the "ema" graph when the TrainStep keeps an EMA.  Returns a dict describing
        what was captured."""
        model = self.model
        modes, arena_was = [(m, m.training) for m in model.modules()], fused._ARENA.active
        ptrs = [p.data_ptr() for p in model.parameters()] + [b.data_ptr() for b in model.buffers()]
        bufs = list(model.buffers()) + (list(self.ts.ema_buffers) if self.has_ema else [])
        before = [b.clone() for b in bufs]
        which_all = ("live", "ema") if self.has_ema else ("live",)
        if self.has_ema and self.ts.weights_bf16 and self._eb is None:
            self._eb = torch.empty_like(self.ts.E_big, dtype=torch.bfloat16)
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()
        lc0 = _lib.launch_count()
        model.eval()
        fused.step_arena_off()
        try:
            assert not any(m.training for m in model.modules())
            for which in which_all:
                self.counts[which] = torch.zeros(len(self.topk) + 2, dtype=torch.int64, device=self.dev)
                with self._bound(which):
                    side = torch.cuda.Stream(device=self.dev)
                    side.wait_stream(torch.cuda.current_stream(self.dev))
                    with torch.cuda.stream(side):
                        for _ in range(warmup):
                            self._body(which)
                    torch.cuda.current_stream(self.dev).wait_stream(side)
                    torch.cuda.synchronize(self.dev)
                    drop_weight_caches(model)
                    g = torch.cuda.CUDAGraph()
                    try:
                        with torch.cuda.graph(g, pool=self._pool):
                            self.logits[which] = self._body(which)
                    finally:
                        drop_weight_caches(model)
                self.counts[which].zero_()
                self._graphs[which] = g
        finally:
            fused._ARENA.active = arena_was
            for m, t in modes:
                m.training = t
        if [p.data_ptr() for p in model.parameters()] + [b.data_ptr() for b in model.buffers()] != ptrs:
            raise RuntimeError("EvalStep.capture: a parameter or buffer moved")
        if not all(torch.equal(a, b) for a, b in zip(before, bufs)):
            raise RuntimeError("EvalStep.capture: the eval forward changed a buffer (BatchNorm running statistics)")
        return {"graphs": list(which_all), "libcotb200_launches": _lib.launch_count() - lc0,
                "K": int(self.logits["live"].shape[1])}

    # ------------------------------------------------------------------ run / result
    def run(self, x, labels, valid=None, which="live"):
        """Count one batch: x [n, C, H, W] (n <= batch) and labels int64 [n] on the device are copied into the static inputs and the
        graph is replayed.  valid: the number of leading rows to count (default n), a Python int or a device int32 [1].  No host
        synchronisation."""
        g = self._graphs.get(which)
        if g is None:
            raise ValueError("EvalStep.run: no %r graph (capture() first%s)" % (which, "" if which == "live" else
                                                                                  "; 'ema' needs a TrainStep with ema_decay"))
        n = x.shape[0]
        if n > self.batch or labels.shape[0] != n:
            raise ValueError("EvalStep.run: batch of %d images / %d labels for a graph of %d" % (n, labels.shape[0], self.batch))
        self.x[:n].copy_(x, non_blocking=True)
        self.labels[:n].copy_(labels, non_blocking=True)
        if valid is None:
            valid = n
        if isinstance(valid, torch.Tensor):
            self.valid.copy_(valid.reshape(1), non_blocking=True)
        else:
            self.valid.fill_(min(int(valid), n))
        g.replay()
        return self.logits[which]

    def result(self, which="live", all_reduce=True):
        """{"top1", "top5" (one entry per k, in percent), "n", "bad_labels"} of everything counted since the last result(), summed
        over the process group (one int64 SUM all-reduce) when `all_reduce` and torch.distributed is initialised; resets the
        counters.  One device-to-host copy."""
        c = self.counts[which]
        if all_reduce and dist.is_available() and dist.is_initialized():
            dist.all_reduce(c, op=dist.ReduceOp.SUM, group=self.ts.pg if self.ts is not None else None)
        h = c.cpu().tolist()
        c.zero_()
        n = h[len(self.topk)]
        out = {"top%d" % k: (100.0 * h[i] / n if n else float("nan")) for i, k in enumerate(self.topk)}
        out.update(n=n, bad_labels=h[len(self.topk) + 1])
        return out
