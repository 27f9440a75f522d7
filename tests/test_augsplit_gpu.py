"""The augmentation splits and the JSD loss on the GPU: TrainAugment(num_splits=S) batches byte-equal to the reference's
AugMixDataset + fast_collate (tests/golden/augsplit.npz), random erasing that spares the clean split, cotb200_jsd_ce / _bwd
against the fp64 restatement tests/jsd_ref.py, and TrainStep(jsd_splits=S) against a plain PyTorch loop and under graph replay."""
import copy
import os
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cotnet_b200 import _lib, augment, trainer
import jsd_ref
from oracle import aug_ref

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "augsplit.npz")
CASES = {"s2_rand_v0": (2, "rand-m15-mstd0.5-n2", 0.), "s2_cj_v5": (2, None, 0.5), "s3_rand_v5": (3, "rand-m15-mstd0.5-n2", 0.5),
         "s3_cj_v0": (3, None, 0.), "s2_rand_v5": (2, "rand-m15-mstd0.5-n2", 0.5), "s2_cj_v0": (2, None, 0.),
         "s3_rand_v0": (3, "rand-m15-mstd0.5-n2", 0.), "s3_cj_v5": (3, None, 0.5)}
MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


@pytest.fixture(scope="module")
def gold():
    return aug_ref.load_golden(GOLD)


def _split_batch(gold, case):
    S, aa, vflip = CASES[case]
    seed, B, size = (int(v) for v in gold["o_%s_meta" % case])
    tf = augment.TrainAugment(size=size, auto_augment=aa, color_jitter=0.4, vflip=vflip, num_splits=S)
    src = gold["o_src"]
    imgs = [aug_ref.source_image(int(s), int(H), int(W)) for H, W, s in src]
    draws = tf.draw([(int(H), int(W)) for H, W, _ in src], random.Random(seed), np.random.RandomState(seed),
                    torch.Generator().manual_seed(seed))
    out, lab = tf(tf.collate_draws(imgs, [3, 5], draws))
    return out, lab, gold["o_%s" % case].reshape(S * B, 3, size, size), S, B


@pytest.mark.parametrize("case", sorted(CASES))
def test_split_batch_equals_reference(gold, case):
    out, lab, want, S, B = _split_batch(gold, case)
    torch.cuda.synchronize()
    assert lab.tolist() == [3, 5] * S
    got = out.cpu().numpy()
    for n in range(S * B):
        assert np.array_equal(got[n], want[n]), (case, n, int((got[n] != want[n]).sum()))


@pytest.mark.parametrize("case", ["s2_rand_v5", "s3_cj_v0"])
def test_random_erasing_spares_the_clean_split(gold, case):
    out, _, _, S, B = _split_batch(gold, case)
    x = trainer.normalize_u8(out, MEAN, STD, dtype=torch.float32)
    before = x.clone()
    augment.RandomErasing(probability=1.0, mode="pixel", max_count=2, num_splits=S, seed=3)(x)
    assert torch.equal(x[:B], before[:B])
    for n in range(B, S * B):
        assert not torch.equal(x[n], before[n]), n


# ------------------------------------------------------------------------------------------------ JSD kernels
def _logits(S, B, K, ld, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randn(S * B, ld, generator=g, device="cuda") * 3
    z = buf[:, :K]
    for s in range(S):                   # sample 0: one-hot-like in every split (mixture exactly 1 and below 1e-7)
        z[s * B].fill_(0.)
        z[s * B, 0] = 40.
    z[1 + B, 3] = -800.                  # sample 1, split 1: a probability that underflows to 0
    return buf.to(dtype)[:, :K]


def _run(z, labels, S, smoothing, alpha=12.0):
    N, K = z.shape
    B = N // S
    lib, st = _lib.load(), torch.cuda.current_stream().cuda_stream
    rows = torch.empty(N + B, device="cuda")
    loss = torch.empty((), device="cuda")
    _lib.check(lib.cotb200_jsd_ce(_lib.dtype_code(z), S, B, K, z.data_ptr(), z.stride(0), labels.data_ptr(), smoothing, alpha,
                                  rows.data_ptr(), loss.data_ptr(), st), "jsd_ce")
    one = torch.full((), 1.7, device="cuda")
    dz = torch.empty(N, K + 8, device="cuda")
    _lib.check(lib.cotb200_jsd_ce_bwd(_lib.dtype_code(z), S, B, K, z.data_ptr(), z.stride(0), labels.data_ptr(), smoothing, alpha,
                                      rows.data_ptr(), one.data_ptr(), dz.data_ptr(), dz.stride(0), st), "jsd_ce_bwd")
    return loss, dz[:, :K], rows


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
@pytest.mark.parametrize("K", [1000, 37])
def test_jsd_kernels_match_fp64(dtype, S, smoothing, K):
    B = 64
    z = _logits(S, B, K, K + 24, dtype, seed=K + S)
    assert z.stride(0) == K + 24
    labels = torch.randint(0, K, (S * B,), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
    loss, dz, _ = _run(z, labels, S, smoothing)
    want, gd = jsd_ref.jsd_ce(z.double().cpu().numpy(), labels.cpu().numpy(), S, smoothing, clamp=(float(np.float32(1e-7)), 1.0))
    assert abs(loss.item() - want) <= 1e-5 * abs(want), (loss.item(), want)
    err = np.abs(dz.double().cpu().numpy() - 1.7 * gd).max()
    assert np.isfinite(dz.cpu().numpy()).all()
    assert err <= 1e-6, err                  # the kernel's own fp32 gradient, before any cast to the logits' dtype
    # through autograd: the gradient in the logits' dtype
    zg = z.detach().clone().requires_grad_(True)
    lz = trainer.jsd_cross_entropy(zg, labels, S, smoothing)
    (gz,) = torch.autograd.grad(lz * 1.7, [zg])
    assert gz.dtype == dtype
    gerr = np.abs(gz.double().cpu().numpy() - 1.7 * gd).max()
    assert gerr <= (1e-6 if dtype == torch.float32 else 0.5 ** 8 * np.abs(1.7 * gd).max() + 1e-6), gerr
    # repeats are bit-identical
    loss2, dz2, _ = _run(z, labels, S, smoothing)
    assert torch.equal(loss, loss2) and torch.equal(dz, dz2)


def test_jsd_invalid_label_is_nan():
    S, B, K = 3, 4, 10
    z = torch.randn(S * B, K, device="cuda")
    labels = torch.tensor([1, 2, 10, 3], device="cuda")
    loss, dz, rows = _run(z, labels, S, 0.1)
    assert torch.isnan(loss) and torch.isnan(rows[S * B + 2]) and not torch.isnan(rows[S * B:]).all()
    for s in range(S):
        assert torch.isnan(dz[2 + s * B]).all() and not torch.isnan(dz[s * B]).any()
    labels[2] = -1
    assert torch.isnan(trainer.jsd_cross_entropy(z, labels, S, 0.1))


# ------------------------------------------------------------------------------------------------ the loss in a training step
def _small_model():
    """tests/test_trainer_gpu.py:_small_model: a 4-block CoT network with perturbed running statistics, BatchNorm in eval mode."""
    from cotnet_b200 import backbone
    torch.manual_seed(0)
    m = backbone.CoTResNet([1, 1, 1, 1], zero_init_last_bn=False)
    g0 = torch.Generator().manual_seed(11)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.2, generator=g0)
                mod.running_var.uniform_(0.6, 1.6, generator=g0)
    return m.cuda().to(memory_format=torch.channels_last).eval()


def _torch_jsd(out, y, S, smoothing, alpha=12.0):
    """loss/jsd.py in torch ops: LabelSmoothingCrossEntropy on the clean split + alpha * mean_s KL(p_s || clamped mixture)."""
    B = out.shape[0] // S
    splits = torch.split(out, B)
    lp = F.log_softmax(splits[0], dim=-1)
    ce = ((1 - smoothing) * -lp.gather(1, y[:B, None])[:, 0] + smoothing * -lp.mean(-1)).mean()
    probs = [F.softmax(z, dim=1) for z in splits]
    logm = torch.clamp(torch.stack(probs).mean(0), 1e-7, 1).log()
    return ce + alpha * sum(F.kl_div(logm, p, reduction="batchmean") for p in probs) / S


def _ref_groups(model, wd):
    decay, no_decay = [], []
    for name, p in model.named_parameters():
        (no_decay if (p.dim() == 1 or name.endswith(".bias")) else decay).append(p)
    return [{"params": no_decay, "weight_decay": 0.0}, {"params": decay, "weight_decay": wd}]


@pytest.fixture
def _no_tf32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _split_inputs(g0, S=3, B=4, res=96):
    x = torch.randn(B, 3, res, res, generator=g0)
    x = torch.cat([x] + [x + 0.3 * torch.randn(B, 3, res, res, generator=g0) for _ in range(S - 1)])
    y = torch.randint(0, 1000, (B,), generator=g0).repeat(S)
    return x.cuda().contiguous(memory_format=torch.channels_last), y.cuda()


def test_jsd_trainstep_matches_plain_pytorch_loop_fp32(_no_tf32):
    """fp32 weights, no autocast: TrainStep(jsd_splits=3, label_smoothing=0.1) == forward / JsdCrossEntropy / SGD(nesterov) /
    ModelEmaV2, with the thresholds of tests/test_trainer_gpu.py's plain-loop test."""
    lr, mu, wd, dec = 0.05, 0.9, 1e-3, 0.99
    m1 = _small_model()
    m2 = copy.deepcopy(m1)
    opt = torch.optim.SGD(_ref_groups(m2, wd), lr=lr, momentum=mu, nesterov=True)
    ts = trainer.TrainStep(m1, lr=lr, momentum=mu, weight_decay=wd, nesterov=True, ema_decay=dec, amp_dtype=None, weights="fp32",
                           jsd_splits=3, label_smoothing=0.1)
    g0 = torch.Generator().manual_seed(5)
    for step in range(3):
        x, y = _split_inputs(g0)
        l1 = ts.step_eager(x, y)
        opt.zero_grad(set_to_none=True)
        l2 = _torch_jsd(m2(x), y, 3, 0.1)
        l2.backward()
        opt.step()
        assert abs(l1.item() - l2.item()) <= 2e-4 * max(1.0, abs(l2.item())), (step, l1.item(), l2.item())
    ms = ts.master_state()
    rels = sorted(((ms[n] - p2).norm() / p2.norm().clamp_min(1e-6)).item() for n, p2 in m2.named_parameters())
    assert rels[len(rels) // 2] <= 5e-5 and rels[(9 * len(rels)) // 10] <= 3e-2 and rels[-1] <= 1e-1, (
        rels[len(rels) // 2], rels[(9 * len(rels)) // 10], rels[-1])


def test_jsd_graph_replay_equals_eager_and_launches_like_label_smoothing(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    m1 = _small_model()
    m2, m3 = copy.deepcopy(m1), copy.deepcopy(m1)
    kw = dict(lr=0.002, momentum=0.9, weight_decay=1e-3, nesterov=True, ema_decay=0.99, amp_dtype=torch.bfloat16, weights="bf16",
              label_smoothing=0.1)
    t1, t2 = trainer.TrainStep(m1, jsd_splits=3, **kw), trainer.TrainStep(m2, jsd_splits=3, **kw)
    x, y = _split_inputs(torch.Generator().manual_seed(6))
    x = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    info = t1.capture(x, y, warmup=2)
    for _ in range(2):
        t2.step_eager(x, y)
    la, lb = [], []
    for lr in (0.002, 0.01, 0.0005):
        t1.set_lr(lr)
        t2.set_lr(lr)
        la.append(t1.step(x, y).item())
        lb.append(t2.step_eager(x, y).item())
    assert la == lb, (la, lb)
    s1, s2 = t1.master_state(), t2.master_state()
    assert all(torch.equal(s1[n], s2[n]) for n in s1)
    # the same number of library launches as the label-smoothing graph at the same total batch
    t3 = trainer.TrainStep(m3, **kw)
    info3 = t3.capture(x, y, warmup=1)
    assert info["libcotb200_kernels_per_replay"] == info3["libcotb200_kernels_per_replay"], (info, info3)


def test_jsd_trainstep_argument_errors():
    m = _small_model()
    ts = trainer.TrainStep(m, jsd_splits=3, label_smoothing=0.1, amp_dtype=None, weights="fp32")
    x, y = _split_inputs(torch.Generator().manual_seed(1), S=3, B=2, res=64)
    with pytest.raises(ValueError):
        ts.step_eager(x[:5], y[:5])
    mix = trainer.MixupCutmix(num_classes=1000, seed=0).draw(6, 64, 64)
    with pytest.raises(ValueError):
        ts.step_eager(x, y, mix)
    assert torch.isfinite(ts.step_eager(x, y))


def test_aug_splits_without_jsd_is_label_smoothing_over_all_rows():
    """aug_splits without loss.jsd: the reference trains LabelSmoothingCrossEntropy over all S*B rows of the split batch."""
    S, B, K = 3, 8, 1000
    z = torch.randn(S * B, K, device="cuda", requires_grad=True)
    y = torch.randint(0, K, (B,), device="cuda").repeat(S)
    loss = trainer.soft_target_cross_entropy(z, y, None, 0.1)
    zd = z.detach().double()
    lp = F.log_softmax(zd, -1)
    want = (0.9 * -lp.gather(1, y[:, None])[:, 0] + 0.1 * -lp.mean(-1)).mean()
    assert abs(loss.item() - want.item()) <= 1e-5 * want.item()
