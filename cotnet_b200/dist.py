"""Data-parallel plumbing for the CoT path (SURVEY.md section 8e): one process per GPU, batch sharded by rank,
no data-path collective in the forward; the only collective is the gradient all-reduce (NCCL over NVLink on
the GPU box, gloo in the CPU tests).  Replaces the reference's launch/reduce helpers:
    init_process_group('nccl', 'env://')         /root/reference/train.py:222-226
    scaled_all_reduce / sum_tensor               /root/reference/utils/distributed.py:20-48
"""
import os

import torch
import torch.distributed as dist


def env_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))


def init_from_env(backend=None):
    """Initialise torch.distributed from RANK/LOCAL_RANK/WORLD_SIZE/MASTER_* when WORLD_SIZE > 1."""
    rank, local_rank, world = env_world()
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = {}
        if backend == "nccl":
            torch.cuda.set_device(local_rank)
            kw["device_id"] = torch.device("cuda", local_rank)
        dist.init_process_group(backend=backend, init_method="env://", rank=rank, world_size=world, **kw)
    return rank, local_rank, world


def shard_range(total, rank, world):
    """Contiguous [lo, hi) slice of `total` units owned by `rank` (remainder spread over the first ranks)."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def max_over_ranks(value: float, device) -> float:
    """Timing reduction the bench contract asks for: the slowest rank defines the step time."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def sum_over_ranks(value: float, device) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


def barrier():
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()


def allreduce_grads_(params, world):
    """Average gradients across ranks with ONE flattened all-reduce per dtype (the reference lets DDP bucket
    them, train.py:113-115).  Used by the bench when the model is not wrapped in DDP."""
    if world == 1:
        return
    by_dtype = {}
    for p in params:
        if p.grad is not None:
            by_dtype.setdefault(p.grad.dtype, []).append(p.grad)
    for grads in by_dtype.values():
        flat = torch.cat([g.reshape(-1) for g in grads])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
        flat.div_(world)
        off = 0
        for g in grads:
            n = g.numel()
            g.copy_(flat[off:off + n].view_as(g))
            off += n


def broadcast_module_(module, src=0):
    """Make every rank start from rank `src`'s parameters and buffers (what DDP does at construction)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return
    with torch.no_grad():
        for t in list(module.parameters()) + list(module.buffers()):
            if t.is_floating_point() or t.dtype in (torch.int64, torch.int32):
                dist.broadcast(t.data, src)


class FlatGrads:
    """All gradients of a replica in ONE flat buffer: every `p.grad` is a view (same strides as `p`) into `flat`, so
    backward accumulates straight into the bucket, `zero_()` is one memset and the data-parallel reduction is ONE
    all-reduce(mean) per step -- the gradients of CoTNet-50 are 89 MB, a fraction of a millisecond on NVLink, so there is nothing to
    gain from DDP's bucketed overlap, and without DDP's autograd hooks the whole fwd+bwd replays from a CUDA graph
    (the collective is issued eagerly between the fwd+bwd graph and the optimizer graph)."""

    def __init__(self, params):
        self.params = [p for p in params if p.requires_grad]
        dtypes = {p.dtype for p in self.params}
        if len(dtypes) != 1:
            raise ValueError("FlatGrads: parameters must share one dtype, got %s" % sorted(map(str, dtypes)))
        total = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(total, dtype=self.params[0].dtype, device=self.params[0].device)
        off = 0
        for p in self.params:
            if not (p.is_contiguous() or (p.dim() == 4 and p.is_contiguous(memory_format=torch.channels_last))):
                raise ValueError("FlatGrads: parameter is neither contiguous nor channels_last")
            p.grad = torch.as_strided(self.flat, p.size(), p.stride(), off)
            off += p.numel()

    def zero_(self):
        self.flat.zero_()

    def attached(self):
        """True while every p.grad still aliases the bucket (zero_grad(set_to_none=True) would detach them)."""
        lo, hi = self.flat.data_ptr(), self.flat.data_ptr() + self.flat.numel() * self.flat.element_size()
        return all(p.grad is not None and lo <= p.grad.data_ptr() < hi for p in self.params)

    def all_reduce_mean_(self):
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return
        if dist.get_backend() == "nccl":
            dist.all_reduce(self.flat, op=dist.ReduceOp.AVG)
        else:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
            self.flat.div_(dist.get_world_size())
