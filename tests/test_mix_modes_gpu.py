"""Per-sample Mixup / CutMix on the GPU: cotb200_u8_mix_rows_to_nhwc against the reference's own mixed batches
(tests/golden/mix_modes.npz) on the fast and the generic path and against the numpy restatement, cotb200_soft_ce with a row table
against fp64 SoftTargetCrossEntropy, and row tables in a captured training step."""
import ctypes
import os

import numpy as np
import pytest
import torch

import mix_ref
from cotnet_b200 import _lib, backbone, trainer
from test_mix_modes_cpu import ALPHAS, MODES, NUM_CLASSES, mixed_batch, mixer

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mix_modes.npz"))
MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


def _rows(n_in, spec):
    """A MixRows from (mode, partner, lam, target_lam, box) tuples, weights rounded like MixupCutmix's."""
    rows = (_lib.MixRow * len(spec))()
    for r, (mode, partner, lam, tl, box) in zip(rows, spec):
        r.mode, r.partner, r.lam, r.one_minus_lam, r.target_lam = mode, partner, lam, float(np.float32(1) - np.float32(lam)), tl
        r.y0, r.y1, r.x0, r.x1 = box
    return trainer.MixRows(rows, n_in, "cuda")


# ------------------------------------------------------------------------------------------------ input kernel
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("case", ["%s_%s" % (m, a) for m in MODES for a in ALPHAS] + ["%s_both_generic" % m for m in MODES])
def test_rows_kernel_equals_reference_mixed_batch(case, dtype):
    """normalize_u8(x, mix=draw) == normalize_u8(the reference's mixed uint8 batch), bit for bit: 3 x 16 x 20 takes the fast path,
    3 x 15 x 19 the generic one."""
    mode, aset = case.split("_")[:2]
    out, seed = GOLDEN["out_" + case], int(GOLDEN["seed_" + case])
    x, _ = mixed_batch(seed, (out.shape[0] * (2 if mode == "half" else 1),) + out.shape[1:])
    t = mixer(mode, aset, 1.0, seed, "cuda").draw(x.shape[0], x.shape[2], x.shape[3])
    got = trainer.normalize_u8(torch.from_numpy(x).cuda(), MEAN, STD, dtype, mix=t)
    want = trainer.normalize_u8(torch.from_numpy(out).cuda(), MEAN, STD, dtype)
    assert got.shape == want.shape and torch.equal(got, want)


@pytest.mark.parametrize("shape", [(8, 3, 16, 20), (4, 3, 15, 19), (4, 5, 8, 8)])
def test_rows_kernel_mode0_batch_and_any_partner_tables(shape):
    """A table of mode-0 rows equals plain normalize_u8; a batch-shaped table (partner N-1-n, one draw on every row) and a table
    of every row kind with any partners equal the numpy restatement -- fp32 and bf16, bit for bit."""
    N, C, H, W = shape
    x = torch.from_numpy(np.random.RandomState(N * H).randint(0, 256, size=shape).astype(np.uint8)).cuda()
    mean, std = (MEAN + [100.0, 50.0])[:C], (STD + [60.0, 70.0])[:C]
    box = (3, H - 2, 2, W - 5)
    spec = [(n % 3, (n * 5 + 1) % N, 0.37 + 0.05 * n, 0.5, box) for n in range(N)]
    for dtype in (torch.float32, torch.bfloat16):
        plain = trainer.normalize_u8(x, mean, std, dtype)
        zero = _rows(N, [(0, N - 1 - n, 1.0, 1.0, (0, 0, 0, 0)) for n in range(N)])
        assert torch.equal(trainer.normalize_u8(x, mean, std, dtype, mix=zero), plain)
        batch = [_rows(N, [(mode, N - 1 - n, lam, lam, box) for n in range(N)]) for mode, lam in ((1, 0.37), (2, 0.8))]
        for t in batch + [_rows(N, spec)]:
            want = mix_ref.mixed_batch(x.cpu().numpy(), t.host)
            assert torch.equal(trainer.normalize_u8(x, mean, std, dtype, mix=t),
                               trainer.normalize_u8(torch.from_numpy(want).cuda(), mean, std, dtype))


def test_rows_kernel_device_partner_out_of_range_is_nan():
    """A device table whose partner differs from the validated host copy: that row is NaN, the others are untouched."""
    N, C, H, W = 4, 3, 8, 8
    x = torch.randint(0, 256, (N, C, H, W), dtype=torch.uint8, device="cuda")
    t = _rows(N, [(1, N - 1 - n, 0.3, 0.3, (0, 0, 0, 0)) for n in range(N)])
    good = trainer.normalize_u8(x, MEAN, STD, torch.float32, mix=t)
    bad = (_lib.MixRow * N).from_buffer_copy(bytes(t.host))
    bad[1].partner = 1 << 20
    t.dev.copy_(torch.frombuffer(bytearray(bytes(bad)), dtype=torch.uint8))
    got = trainer.normalize_u8(x, MEAN, STD, torch.float32, mix=t)
    assert torch.isnan(got[1]).all() and torch.equal(got[[0, 2, 3]], good[[0, 2, 3]])


# ------------------------------------------------------------------------------------------------ loss
def _soft_ce_ref(z, labels, rows, smoothing):
    t = torch.from_numpy(mix_ref.soft_targets(labels.cpu().numpy(), rows, z.shape[1], smoothing)).to(z.device)
    return torch.sum(-t * torch.log_softmax(z, dim=-1), dim=-1).mean()                  # loss/cross_entropy.py:34-36


@pytest.mark.parametrize("mode", ["elem", "half"])
@pytest.mark.parametrize("K", [10, 1000, 1001])
@pytest.mark.parametrize("B", [2, 256])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_soft_ce_rows_matches_fp64(mode, K, B, dtype):
    """Loss and gradient against fp64 SoftTargetCrossEntropy on the table's targets; 'half' has B logit rows and 2B labels."""
    g = torch.Generator(device="cuda").manual_seed(K + B)
    n_in = 2 * B if mode == "half" else B
    t = mixer(mode, "both", 1.0, K + B, "cuda").draw(n_in, 32, 32)
    z = (torch.randn(B, K, generator=g, device="cuda") * 3).to(dtype).requires_grad_(True)
    labels = torch.randint(0, K, (n_in,), generator=g, device="cuda")
    loss = trainer.soft_target_cross_entropy(z, labels, t, 0.1)
    (gz,) = torch.autograd.grad(loss * 1.7, [z])
    zd = z.detach().double().requires_grad_(True)
    want = _soft_ce_ref(zd, labels, t.host, 0.1)
    (gd,) = torch.autograd.grad(want * 1.7, [zd])
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item()), (loss.item(), want.item())
    assert gz.dtype == dtype
    err = (gz.double() - gd).abs().max().item()
    assert err <= (1e-6 if dtype == torch.float32 else 0.5 ** 8 * gd.abs().max().item() + 1e-6), err
    assert torch.equal(loss, trainer.soft_target_cross_entropy(z, labels, t, 0.1))


def test_soft_ce_rows_partner_out_of_range_is_nan():
    z = torch.randn(4, 10, device="cuda")
    labels = torch.tensor([1, 2, 3, 4], device="cuda")
    t = _rows(4, [(1, 3 - n, 0.5, 0.5, (0, 0, 0, 0)) for n in range(4)])
    assert torch.isfinite(trainer.soft_target_cross_entropy(z, labels, t, 0.1))
    bad = (_lib.MixRow * 4).from_buffer_copy(bytes(t.host))
    bad[2].partner = 4
    t.dev.copy_(torch.frombuffer(bytearray(bytes(bad)), dtype=torch.uint8))
    assert torch.isnan(trainer.soft_target_cross_entropy(z, labels, t, 0.1))


# ------------------------------------------------------------------------------------------------ the training step
def _model(**kw):
    torch.manual_seed(0)
    return backbone.CoTResNet([1, 1, 1, 1], num_classes=100, **kw).cuda().to(memory_format=torch.channels_last)


def _batch(seed, B=8, res=96):
    g0 = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (B, 3, res, res), generator=g0, dtype=torch.uint8).cuda()
    return x, torch.randint(0, 100, (B,), generator=g0).cuda()


def test_graph_replays_follow_each_steps_row_table(monkeypatch):
    """With fixed drop-path masks and lr 0, a graph captured with an 'elem' table gives, for each of several tables, the eager
    step's loss bit for bit, and the losses differ from table to table."""
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    xu, lab = _batch(1)
    x = trainer.normalize_u8(xu, MEAN, STD)
    mc = trainer.MixupCutmix(seed=4, mode="elem")
    tables = [mc.draw(8, 96, 96) for _ in range(5)]
    tsg, tse = [trainer.TrainStep(_model(drop_path_rate=0.5), lr=0.0, momentum=0.0, weight_decay=0.0, label_smoothing=0.1)
                for _ in range(2)]
    for t in (tsg, tse):
        t.model.fixed_drop_path_scales = torch.tensor([1.0, 0.0, 1.5, 2.0], device="cuda").repeat_interleave(2).view(1, 8).repeat(4, 1)
    tsg.capture(x, lab, warmup=1, mix=tables[0])
    tse.step_eager(x, lab, tables[0])
    lg = [tsg.step(x, lab, mix=t).item() for t in tables[1:]]
    le = [tse.step_eager(x, lab, t).item() for t in tables[1:]]
    assert lg == le and len(set(lg)) == len(lg), (lg, le)


def test_identically_seeded_elem_runs_are_bit_identical(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    runs = []
    for _ in range(2):
        ts = trainer.TrainStep(_model(drop_path_rate=0.1, drop_rate=0.25), lr=0.01, label_smoothing=0.1)
        mc = trainer.MixupCutmix(seed=5, mode="elem", cutmix_minmax=[0.2, 0.8])
        xu, lab = _batch(2)
        torch.manual_seed(9)
        t = mc.draw(8, 96, 96)
        ts.capture(trainer.normalize_u8(xu, MEAN, STD, mix=t), lab, warmup=1, mix=t)
        losses = []
        for step in range(3):
            xu, lab = _batch(3 + step)
            t = mc.draw(8, 96, 96)
            losses.append(ts.step(trainer.normalize_u8(xu, MEAN, STD, mix=t), lab, mix=t).item())
        torch.cuda.synchronize()
        runs.append((losses, {k: v.clone() for k, v in ts.master_state().items()}))
    assert runs[0][0] == runs[1][0]
    assert all(torch.equal(runs[0][1][k], runs[1][1][k]) for k in runs[0][1])


def test_half_step_and_graph_table_sizes(monkeypatch):
    """'half': B/2 mixed images and the B labels, eager and replayed; a graph refuses a table of another size (output rows,
    input rows), and a graph captured with a batch draw follows an 'elem' table of its size bit for bit."""
    xu, lab = _batch(6)
    mc = trainer.MixupCutmix(seed=1, mode="half")
    t = mc.draw(8, 96, 96)
    x = trainer.normalize_u8(xu, MEAN, STD, mix=t)
    assert x.shape[0] == 4
    assert np.isfinite(trainer.TrainStep(_model(), lr=0.01, label_smoothing=0.1).step_eager(x, lab, t).item())
    ts = trainer.TrainStep(_model(), lr=0.01, label_smoothing=0.1)
    ts.capture(x, lab, warmup=1, mix=t)
    t2 = mc.draw(8, 96, 96)
    assert torch.isfinite(ts.step(trainer.normalize_u8(xu, MEAN, STD, mix=t2), lab, mix=t2))
    with pytest.raises(ValueError, match="captured with a table of 4 rows from 8 images, not 8 from 8"):
        ts.step(x, lab, mix=trainer.MixupCutmix(seed=1).draw(8, 96, 96))
    with pytest.raises(ValueError, match="captured with a table of 4 rows from 8 images, not 8 from 8"):
        ts.step(x, lab, mix=trainer.MixupCutmix(seed=1, mode="elem").draw(8, 96, 96))
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    tsg, tse = [trainer.TrainStep(_model(), lr=0.0, momentum=0.0, weight_decay=0.0, label_smoothing=0.1) for _ in range(2)]
    p = trainer.MixupCutmix(seed=2).draw(8, 96, 96)
    xb = trainer.normalize_u8(xu, MEAN, STD, mix=p)
    tsg.capture(xb, lab, warmup=1, mix=p)
    tse.step_eager(xb, lab, p)
    with pytest.raises(ValueError, match="captured with a table of 8 rows from 8 images, not 4 from 8"):
        tsg.step(xb, lab, mix=t2)
    e = trainer.MixupCutmix(seed=2, mode="elem").draw(8, 96, 96)
    xe = trainer.normalize_u8(xu, MEAN, STD, mix=e)
    lg, le = tsg.step(xe, lab, mix=e).item(), tse.step_eager(xe, lab, e).item()
    assert lg == le and lg != tse.step_eager(xb, lab, p).item(), (lg, le)
    assert ctypes.sizeof(_lib.MixRow) * 4 == t.dev.numel()
