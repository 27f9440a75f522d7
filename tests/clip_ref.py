"""Restatement in torch of the reference's gradient clipping (utils/clip_grad.py, models/helpers.py:270-275) and of the update
that follows it, for the tests of the clip path.  TEST INFRASTRUCTURE ONLY.

Functional: every function takes the gradients as a list of tensors and returns new ones; the dtype of the inputs (fp32 or
fp64) is the dtype of the arithmetic.  Pinned to the reference's own code by tests/golden/clip.npz (tools/make_clip_golden.py).
"""
import torch
import torch.nn as nn

MODES = ("norm", "value", "agc")


def model_parameters(model, exclude_head=False):
    """models/helpers.py:270-275: the classifier head is `the last two of model.parameters()`."""
    ps = list(model.parameters())
    return ps[:-2] if exclude_head else ps


def unitwise_norm(x):
    """utils/clip_grad.py:3-9 with norm_type 2: the whole tensor for ndim <= 1, else one norm per index of dim 0 (keepdim)."""
    if x.ndim <= 1:
        return torch.linalg.vector_norm(x)
    return torch.linalg.vector_norm(x, dim=tuple(range(1, x.ndim)), keepdim=True)


def clip_grad_norm(grads, max_norm):
    """torch.nn.utils.clip_grad_norm_(norm_type=2, error_if_nonfinite=False): (clipped grads, total norm)."""
    total = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(g) for g in grads]))
    coef = torch.clamp((total + 1e-6).reciprocal() * max_norm, max=1.0)       # `max_norm / tensor` is reciprocal() * max_norm
    return [g * coef for g in grads], total


def clip_grad_value(grads, value):
    return [torch.clamp(g, -value, value) for g in grads]


def adaptive_clip_grad(params, grads, clip_factor, eps=1e-3):
    """utils/clip_grad.py:12-24 (norm_type 2) on (parameter, gradient) pairs."""
    out = []
    for p, g in zip(params, grads):
        max_norm = unitwise_norm(p).clamp(min=eps) * clip_factor
        grad_norm = unitwise_norm(g)
        out.append(torch.where(grad_norm < max_norm, g, g * (max_norm / grad_norm.clamp(min=1e-6))))
    return out


def agc_factors(params, grads, clip_factor, eps=1e-3):
    """Per parameter, the factor of each unit (1 where the clip does not bind): shape [shape[0]] for >= 2-D, [1] otherwise."""
    out = []
    for p, g in zip(params, grads):
        max_norm = unitwise_norm(p).clamp(min=eps) * clip_factor
        grad_norm = unitwise_norm(g)
        f = torch.where(grad_norm < max_norm, torch.ones_like(grad_norm), max_norm / grad_norm.clamp(min=1e-6))
        out.append(f.reshape(-1))
    return out


def dispatch_clip_grad(params, grads, value, mode="norm"):
    """utils/clip_grad.py:26-41 on the gradients of `params` (what train.py:271 passes): (clipped grads, total norm or None)."""
    if mode == "norm":
        return clip_grad_norm(grads, value)
    if mode == "value":
        return clip_grad_value(grads, value), None
    if mode == "agc":
        return adaptive_clip_grad(params, grads, value), None
    raise ValueError("unknown clip mode %r" % mode)


def clip_model_grads(model, params, grads, value, mode):
    """train.py:270-273 on name-free lists: `params` / `grads` follow model.parameters(); agc leaves the head out
    (model_parameters(exclude_head=True)).  Returns (clipped grads for every parameter, total norm or None)."""
    pick = model_parameters(model, exclude_head=(mode == "agc"))
    ids = [id(p) for p in model.parameters()]
    idx = [ids.index(id(p)) for p in pick]
    clipped, norm = dispatch_clip_grad([params[i] for i in idx], [grads[i] for i in idx], value, mode)
    out = list(grads)
    for i, g in zip(idx, clipped):
        out[i] = g
    return out, norm


def sgd_ema(p, m, e, g, lr, mu, wd, dec, nesterov=True):
    """torch.optim.SGD (momentum, weight decay, nesterov) then ModelEmaV2.update, in the dtype of the inputs: (p, m, e)."""
    d = g + wd * p
    m = mu * m + d
    step = d + mu * m if nesterov else m
    p = p - lr * step
    e = None if e is None else dec * e + (1.0 - dec) * p
    return p, m, e


class Toy(nn.Module):
    """The module of the golden: a 7x7 stem whose 147-element rows cross float4 boundaries, 1x1 and grouped 3x3 convolutions,
    BatchNorm affines, a bias, and a classifier head `fc` registered last."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 8, 7, bias=False)
        self.bn1 = nn.BatchNorm2d(8)
        self.conv2 = nn.Conv2d(8, 16, 1, bias=False)
        self.conv3 = nn.Conv2d(16, 16, 3, groups=4, bias=True)
        self.fc = nn.Linear(32, 10)
