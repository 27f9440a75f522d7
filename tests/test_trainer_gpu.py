"""Train-step plumbing (cotnet_b200/trainer.py, csrc/optim.cu) on the GPU: the flat-state kernels against torch's own
optimizer / EMA arithmetic, the uint8 normalise kernel against the loader's formula, TrainStep against a plain PyTorch loop
(the reference's train.py:255-277 with optim.SGD(nesterov) + add_weight_decay + ModelEmaV2), CUDA-graph replay against the
eager step, and the BENCH PATH itself (bf16 weights, autocast, channels_last, CUDA graph, gradient bucket) against golden
train-step fixtures made from the reference's own model code (oracle/make_golden.py train)."""
import copy
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import make_golden

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")


@pytest.fixture(autouse=True)
def _no_tf32():
    """fp32 parity is judged without TF32 (the oracle / goldens are exact)."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _record(name, payload):
    try:
        os.makedirs(OUT, exist_ok=True)
        path = os.path.join(OUT, "parity_measured.json")
        data = json.load(open(path)) if os.path.exists(path) else {}
        data[name] = payload
        json.dump(data, open(path, "w"), indent=1)
    except Exception:
        pass


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("nesterov", [True, False])
def test_sgd_ema_kernel_matches_torch(gdt, nesterov):
    from cotnet_b200 import _lib
    lib = _lib.load()
    n = 4 * 12345
    g0 = torch.Generator(device="cuda").manual_seed(1)
    P = torch.randn(n, device="cuda", generator=g0)
    E = P.clone()
    M = torch.zeros(n, device="cuda")
    Pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    lr, mu, wd, dec = 0.1, 0.9, 1e-2, 0.99
    hyper = torch.tensor([lr, mu, wd, dec, 1.0], device="cuda")
    p_ref = torch.nn.Parameter(P.clone())
    opt = torch.optim.SGD([p_ref], lr=lr, momentum=mu, weight_decay=wd, nesterov=nesterov)
    e_ref = P.clone()
    for step in range(3):
        G = torch.randn(n, device="cuda", generator=g0).to(gdt)
        rc = lib.cotb200_sgd_ema_step(n, P.data_ptr(), M.data_ptr(), _lib.dtype_code(G), G.data_ptr(), E.data_ptr(), Pb.data_ptr(),
                                      hyper.data_ptr(), 1 if nesterov else 0, torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "sgd_ema_step")
        p_ref.grad = G.float()
        opt.step()
        e_ref = dec * e_ref + (1.0 - dec) * p_ref.detach()               # utils/model_ema.py:52-53
    assert torch.allclose(P, p_ref.detach(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(E, e_ref, rtol=1e-5, atol=1e-6)
    assert torch.equal(Pb, P.to(torch.bfloat16))
    assert torch.allclose(M, opt.state[p_ref]["momentum_buffer"], rtol=1e-5, atol=1e-6)


def test_sgd_ema_kernel_argument_errors():
    from cotnet_b200 import _lib
    lib = _lib.load()
    t = torch.zeros(64, device="cuda")
    h = torch.zeros(5, device="cuda")
    assert lib.cotb200_sgd_ema_step(6, t.data_ptr(), t.data_ptr(), _lib.F32, t.data_ptr(), None, None, h.data_ptr(), 1, None) == -1
    assert lib.cotb200_sgd_ema_step(8, None, t.data_ptr(), _lib.F32, t.data_ptr(), None, None, h.data_ptr(), 1, None) == -5
    assert lib.cotb200_sgd_ema_step(8, t.data_ptr(), t.data_ptr(), _lib.F64, t.data_ptr(), None, None, h.data_ptr(), 1, None) == -2


@pytest.mark.parametrize("bucket", [torch.float32, torch.bfloat16])
def test_multi_gather(bucket):
    from cotnet_b200 import _lib, trainer
    lib = _lib.load()
    chunk = lib.cotb200_gather_chunk()
    g0 = torch.Generator(device="cuda").manual_seed(2)
    shapes = [(3,), (chunk + 5,), (7, 9), (2 * chunk,), (64, 3, 7, 7), (1,)]
    srcs = [torch.randn(*s, device="cuda", generator=g0).to(torch.bfloat16 if i % 2 else torch.float32) for i, s in enumerate(shapes)]
    offs, o = [], 0
    for t in srcs:
        offs.append(o)
        o += (t.numel() + 7) // 8 * 8
    flat = torch.full((o,), 7.0, device="cuda", dtype=bucket)
    tab = trainer._GatherTable(len(srcs), sum((t.numel() + chunk - 1) // chunk for t in srcs), torch.device("cuda"))
    nb = tab.fill([(t.data_ptr(), off, t.numel(), _lib.dtype_code(t)) for t, off in zip(srcs, offs)], chunk)
    tab.upload(False)
    _lib.check(lib.cotb200_multi_gather(tab.seg_d.data_ptr(), tab.blk_d.data_ptr(), nb, _lib.dtype_code(flat), flat.data_ptr(), 0.5,
                                        torch.cuda.current_stream().cuda_stream), "multi_gather")
    for t, off in zip(srcs, offs):
        want = (t.float() * 0.5).to(bucket)
        assert torch.equal(flat[off:off + t.numel()], want.reshape(-1))
    assert float(flat[offs[1] - 1]) == 7.0                    # padding between slots untouched


def test_multi_lerp():
    from cotnet_b200 import _lib, trainer
    lib = _lib.load()
    a, b = torch.randn(1000, device="cuda"), torch.randn(1000, device="cuda")
    ai = torch.tensor([0, 5, 20000], device="cuda"), torch.tensor([1, 7, 50000], device="cuda")
    want = 0.9 * a + 0.1 * b
    wanti = (0.9 * ai[0] + (1.0 - 0.9) * ai[1]).to(torch.int64)      # the reference's float round trip (model_ema.py:50,53)
    segs = (trainer._Seg2 * 2)()
    segs[0].dst, segs[0].src, segs[0].numel, segs[0].dtype = a.data_ptr(), b.data_ptr(), 1000, _lib.F32
    segs[1].dst, segs[1].src, segs[1].numel, segs[1].dtype = ai[0].data_ptr(), ai[1].data_ptr(), 3, 100
    tab = torch.frombuffer(bytearray(bytes(segs)), dtype=torch.uint8).cuda()
    hyper = torch.tensor([0, 0, 0, 0.9, 1.0], device="cuda")
    _lib.check(lib.cotb200_multi_lerp(tab.data_ptr(), 2, hyper.data_ptr(), torch.cuda.current_stream().cuda_stream), "multi_lerp")
    assert torch.allclose(a, want, rtol=1e-6, atol=1e-7)
    assert torch.equal(ai[0], wanti)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(4, 3, 32, 32), (2, 3, 17, 13), (2, 5, 8, 8)])
def test_normalize_u8(dtype, shape):
    from cotnet_b200 import trainer
    g0 = torch.Generator().manual_seed(3)
    x = torch.randint(0, 256, shape, generator=g0, dtype=torch.uint8).cuda()
    C = shape[1]
    mean = [0.485 * 255, 0.456 * 255, 0.406 * 255, 100.0, 50.0][:C]
    std = [0.229 * 255, 0.224 * 255, 0.225 * 255, 60.0, 70.0][:C]
    y = trainer.normalize_u8(x, mean, std, dtype)
    m = torch.tensor(mean, device="cuda").view(1, C, 1, 1)
    s = torch.tensor(std, device="cuda").view(1, C, 1, 1)
    want = x.float().sub_(m).div_(s)                                     # datasets/loader.py:88-90
    assert y.shape == x.shape and y.dtype == dtype and y.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(y.float(), want.to(dtype).float())


# ------------------------------------------------------------------------------------------------ TrainStep vs a plain PyTorch loop
def _ref_groups(model, wd):
    decay, no_decay = [], []
    for name, p in model.named_parameters():                             # optim/optim_factory.py:18-30
        (no_decay if (p.dim() == 1 or name.endswith(".bias")) else decay).append(p)
    return [{"params": no_decay, "weight_decay": 0.0}, {"params": decay, "weight_decay": wd}]


def _small_model():
    """A 4-block CoT network with its BatchNorms in EVAL mode (running statistics, perturbed): the plumbing tests compare two
    implementations of the same step to 1e-4, which needs a well-conditioned network -- with batch statistics the
    training-mode gradients of these nets amplify fp32 rounding to the percent level (see the bench-path test below)."""
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


def test_trainstep_matches_plain_pytorch_loop_fp32():
    """fp32 weights, no autocast: TrainStep == forward/backward + optim.SGD(nesterov, add_weight_decay) + ModelEmaV2.update."""
    from cotnet_b200 import trainer
    lr, mu, wd, dec = 0.05, 0.9, 1e-3, 0.99
    m1 = _small_model()
    m2 = copy.deepcopy(m1)
    ema2 = copy.deepcopy(m2)
    opt = torch.optim.SGD(_ref_groups(m2, wd), lr=lr, momentum=mu, nesterov=True)
    ts = trainer.TrainStep(m1, lr=lr, momentum=mu, weight_decay=wd, nesterov=True, ema_decay=dec, amp_dtype=None, weights="fp32")
    g0 = torch.Generator().manual_seed(5)
    for step in range(3):
        x = torch.randn(8, 3, 96, 96, generator=g0).cuda().contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 1000, (8,), generator=g0).cuda()
        l1 = ts.step_eager(x, y)
        opt.zero_grad(set_to_none=True)
        l2 = torch.nn.functional.cross_entropy(m2(x), y)
        l2.backward()
        opt.step()
        with torch.no_grad():                                            # utils/model_ema.py:45-53
            for ev, mv in zip(ema2.state_dict().values(), m2.state_dict().values()):
                ev.copy_(dec * ev + (1.0 - dec) * mv)
        assert abs(l1.item() - l2.item()) <= 2e-4 * max(1.0, abs(l2.item())), (step, l1.item(), l2.item())
    ms, es = ts.master_state(), ts.ema_state()
    rels = sorted(((ms[n] - p2).norm() / p2.norm().clamp_min(1e-6)).item() for n, p2 in m2.named_parameters())
    # two runs of the same fp32 kernels differ in atomic accumulation order; the GroupNorm'ed / softmax-gated CoT layers amplify that
    # for a few parameters (fp32 vs fp64 of one implementation shows the same spread), hence median + worst
    # measured over ten GPU runs of the same code (calls A..Q2): median 1e-5 .. 2e-5 every time; 90th percentile <= 2e-3 in nine runs and
    # 1.5e-2 in one; worst 2e-3 .. 3e-2.  The tail is made of 1-D parameters (most parameters of this net by count: BatchNorm / GroupNorm
    # affines, biases) whose norm is still ~lr * |grad| after three steps, so their RELATIVE error is the relative error of a gradient
    # (atomics-ordered fp32 sums through GroupNorm / softmax gates), not of a weight.  The step itself is pinned by the per-step loss (2e-4).
    assert rels[len(rels) // 2] <= 5e-5 and rels[(9 * len(rels)) // 10] <= 3e-2 and rels[-1] <= 1e-1, (
        rels[len(rels) // 2], rels[(9 * len(rels)) // 10], rels[-1])
    sd_e = ema2.state_dict()
    for n, e in es.items():
        ref = sd_e[n]
        if ref.dtype.is_floating_point:
            assert ((e - ref).norm() / ref.norm().clamp_min(1e-6)).item() <= 5e-3, n
        else:
            assert torch.equal(e, ref), n


def test_trainstep_graph_replay_equals_eager():
    """The captured step (one CUDA graph: forward, backward, gather, optimizer, EMA) against the eager step from the same
    state and batch.  Bit equality is not attainable: the statistics kernels accumulate with fp32 atomics whose order
    changes from run to run (two EAGER runs differ the same way); the gate is 5e-3 relative on the loss, 1e-4 median / 2e-2
    worst relative L2 over the master weights after four small steps (bf16 activations)."""
    from cotnet_b200 import trainer
    m1 = _small_model()
    m2 = copy.deepcopy(m1)
    kw = dict(lr=0.002, momentum=0.9, weight_decay=1e-3, nesterov=True, ema_decay=0.99, amp_dtype=torch.bfloat16, weights="bf16")
    t1, t2 = trainer.TrainStep(m1, **kw), trainer.TrainStep(m2, **kw)
    g0 = torch.Generator().manual_seed(6)
    x = torch.randn(8, 3, 96, 96, generator=g0).cuda().to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (8,), generator=g0).cuda()
    info = t1.capture(x, y, warmup=2)
    assert info["cuda_graph"] and info["libcotb200_kernels_per_replay"] > 20
    for _ in range(2):
        t2.step_eager(x, y)                                              # the same 2 warm-up steps, eagerly
    la = [t1.step(x, y).item() for _ in range(2)]
    lb = [t2.step_eager(x, y).item() for _ in range(2)]
    for a_, b_ in zip(la, lb):
        assert abs(a_ - b_) <= 5e-3 * max(1.0, abs(b_)), (la, lb)
    s1, s2 = t1.master_state(), t2.master_state()
    rels = sorted(((s1[n] - s2[n]).norm() / s2[n].norm().clamp_min(1e-6)).item() for n in s1)
    _record("graph_vs_eager", {"loss_graph": la, "loss_eager": lb, "median_master_rel_l2": rels[len(rels) // 2], "worst_master_rel_l2": rels[-1]})
    assert rels[len(rels) // 2] <= 1e-4 and rels[-1] <= 2e-1, (rels[len(rels) // 2], rels[-1])    # worst = a near-zero bias vector


# ------------------------------------------------------------------------------------------------ bench path vs golden train steps
def _grad_errors(grads, g):
    """grads: name -> tensor.  Returns (worst norm rel err, worst normalised projection err, median both)."""
    names = [str(n) for n in g["names"]]
    seed = int(g["seed"])
    en, ep = [], []
    floor = 1e-2 * float(np.median(g["gnorm"]))      # biases in front of a BatchNorm have an exactly-zero gradient (fp64: 1e-17)
    for n, gn, gp in zip(names, g["gnorm"], g["gproj"]):
        t = grads[n].detach().double().cpu()
        r = make_golden.proj_vector(n, t.shape, seed)
        d = max(gn, floor)
        en.append(abs(t.norm().item() - gn) / d)
        ep.append(abs((t * r).sum().item() - gp) / (d * r.norm().item()))
    en, ep = np.array(en), np.array(ep)
    return dict(worst_norm=float(en.max()), worst_proj=float(ep.max()), median_norm=float(np.median(en)), median_proj=float(np.median(ep)),
                worst_norm_at=names[int(en.argmax())], worst_proj_at=names[int(ep.argmax())])


@pytest.mark.parametrize("model_name,fixture", [("cotnet50", "cotnet50_train_bf16w.npz"), ("cotnext50_2x48d", "cotnext50_train_bf16w.npz")])
def test_bench_path_matches_reference_golden(model_name, fixture, monkeypatch):
    """EXACTLY what bench.py times -- TrainStep with bf16 weight copies, bf16 autocast, channels_last, the whole step
    replayed from a CUDA graph, gradients read from the flat bucket -- at 224x224, bs16, against loss and per-parameter
    gradients of the reference's own model code (fp64) on the same bf16-representable weights and batch (lr = 0 keeps the
    weights at the seeded values through the warm-up steps).

    What can be asserted: training-mode gradients of these networks are ill-conditioned -- every batch-statistics BatchNorm
    projects the scale / shift directions out of its incoming gradient, and rounding of the (large) projected-out part leaks
    into the (small) remainder.  fp32 against fp64 of the SAME code already differs by 1-2 % per parameter
    (tests/test_oracle.py runs the oracle in fp64 for that reason); any bf16 pipeline sits at tens of percent.  The gate is
    therefore RELATIVE: the bench path must be as close to the fp64 reference as the plain eager graph of the same modules
    under torch.autocast (= the reference's own AMP path, with only the LocalConv op on our kernel) is, within 2.5x (the measured run-to-run spread, see the assertion), and the
    loss within 1 %.  Eval-mode logits (well-conditioned) are held to 1e-2 relative L2 and top-1 agreement."""
    import bench
    from cotnet_b200 import trainer
    g = np.load(os.path.join(GOLDEN, fixture))
    m = make_golden.hybrid_seeded_state(bench.build_model(model_name, zero_init_last_bn=False), int(g["seed"]))
    with torch.no_grad():
        for t in m.state_dict().values():
            if t.dtype.is_floating_point:
                t.copy_(t.bfloat16().float())
    x, y = make_golden.train_batch(int(g["seed"]), int(g["B"]), int(g["res"]))
    x = x.bfloat16().cuda()
    y = y.cuda()
    # (a) plain eager AMP arm: NCHW tensors take the modules' un-fused PyTorch branch (cuDNN / ATen + the LocalConv op)
    mp_ = copy.deepcopy(m).cuda().train()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss_plain = torch.nn.functional.cross_entropy(mp_(x.float()).float(), y)
    loss_plain.backward()
    errs_plain = _grad_errors({n: p.grad for n, p in mp_.named_parameters()}, g)
    del mp_
    # (b) the bench path.  The batch here is 16, not 256: lift the pixel threshold so that every layer takes the backend the bs256 bench
    # takes (all-wgmma 1x1 convolutions + haloed key conv), i.e. the code under test is the code that is timed
    from cotnet_b200 import cot_layer as _cl, fused as _fu
    monkeypatch.setattr(_cl.CotLayer, "tc_min_pixels", 0)
    monkeypatch.setattr(_fu, "TC_MIN_PIXELS", 0)
    m = m.cuda().to(memory_format=torch.channels_last)
    xc = x.contiguous(memory_format=torch.channels_last)
    m.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        logits = m(xc).float().cpu()
    ref = torch.from_numpy(g["logits"])
    rel_logits = ((logits - ref).norm() / ref.norm()).item()
    top1 = (logits.argmax(1) == ref.argmax(1)).float().mean().item()
    m.train()
    ts = trainer.TrainStep(m, lr=0.0, momentum=0.9, weight_decay=1e-4, nesterov=True, ema_decay=0.9999, weights="bf16")
    info = ts.capture(xc, y, warmup=2)
    loss = ts.step(xc, y).item()
    errs = _grad_errors(ts.grads(), g)
    loss_eager = ts.step_eager(xc, y).item()
    errs_eager = _grad_errors(ts.grads(), g)
    lref = float(g["loss"])
    _record("bench_path_" + model_name, dict(bench_graph=errs, bench_eager=errs_eager, plain_amp=errs_plain, loss_graph=loss, loss_eager=loss_eager,
                                             loss_plain_amp=loss_plain.item(), loss_ref=lref, rel_l2_eval_logits=rel_logits,
                                             top1_agreement=top1, graph=info))
    assert info["cuda_graph"]
    assert rel_logits <= 1e-2 and top1 >= 0.75, (rel_logits, top1)      # 16 random-weight samples: near-ties flip the arg-max
    assert abs(loss - lref) <= 1e-2 * lref and abs(loss_eager - lref) <= 1e-2 * lref, (loss, loss_eager, lref)
    # the plain AMP graph uses cuDNN / ATen reductions whose order may change between runs (BatchNorm statistics differ in the last
    # bits -> bf16 roundings flip), so its own error moves from run to run; the factor covers that spread.
    for e_ in (errs, errs_eager):
        assert e_["median_norm"] <= 2.5 * errs_plain["median_norm"] + 1e-2, (e_, errs_plain)
        assert e_["median_proj"] <= 2.5 * errs_plain["median_proj"] + 1e-2, (e_, errs_plain)


@pytest.mark.parametrize("model_name,fixture", [("se_cotnetd_101", "se_cotnetd101_train.npz"), ("se_cotnetd_152", "se_cotnetd152_train_320.npz")])
def test_hybrids_match_reference_golden_fp32(model_name, fixture):
    """BASELINE configs 4 / 5: SE-CoTNetD-101 @224 and SE-CoTNetD-152 @320 -- eval logits and one training step (loss, every
    parameter gradient) in fp32 channels_last on the fused path (CoT layers, SplitAttn tail, BatchNorm glue, pooling on
    libcotb200) against the reference's own model code in fp64."""
    import bench
    g = np.load(os.path.join(GOLDEN, fixture))
    m = make_golden.hybrid_seeded_state(bench.build_model(model_name, zero_init_last_bn=False), int(g["seed"]))
    assert sum(p.numel() for p in m.parameters()) == int(g["n_params"])
    m = m.cuda().to(memory_format=torch.channels_last)
    x, y = make_golden.train_batch(int(g["seed"]), int(g["B"]), int(g["res"]))
    x = x.cuda().contiguous(memory_format=torch.channels_last)
    y = y.cuda()
    m.eval()
    with torch.no_grad():
        logits = m(x).cpu()
    ref = torch.from_numpy(g["logits"])
    assert torch.allclose(logits, ref, atol=2e-3, rtol=2e-3), (logits - ref).abs().max().item()
    m.train()
    loss = torch.nn.functional.cross_entropy(m(x), y)
    loss.backward()
    errs = _grad_errors({n: p.grad for n, p in m.named_parameters()}, g)
    _record("hybrid_fp32_" + model_name, dict(errs, loss=loss.item(), loss_ref=float(g["loss"])))
    assert abs(loss.item() - float(g["loss"])) <= 1e-4 * float(g["loss"])
    # fp32 vs fp64 of training-mode gradients: percent-level per parameter is the conditioning of the net, not of the kernels
    # (the CPU oracle in fp32 shows the same, tests/test_oracle.py); medians are at 1e-3
    assert errs["median_norm"] <= 5e-3 and errs["median_proj"] <= 2e-3, errs
    assert errs["worst_norm"] <= 2.5e-1 and errs["worst_proj"] <= 5e-2, errs
    sd = m.state_dict()
    off = 0
    for k in [str(k) for k in g["rm_names"]]:
        want = torch.from_numpy(g["rm_values"][off:off + min(8, sd[k].numel())])
        off += min(8, sd[k].numel())
        assert torch.allclose(sd[k].reshape(-1)[:want.numel()].double().cpu(), want, atol=1e-4, rtol=1e-3), k


def test_hybrid_bf16_train_step_runs_and_tracks_golden():
    """SE-CoTNetD-101 on the bench path (bf16, graph): loss within 2 % of the fp64 reference, gradient medians within budget."""
    import bench
    from cotnet_b200 import trainer
    g = np.load(os.path.join(GOLDEN, "se_cotnetd101_train.npz"))
    m = make_golden.hybrid_seeded_state(bench.build_model("se_cotnetd_101", zero_init_last_bn=False), int(g["seed"]))
    m = m.cuda().to(memory_format=torch.channels_last).train()
    x, y = make_golden.train_batch(int(g["seed"]), int(g["B"]), int(g["res"]))
    x = x.bfloat16().cuda().contiguous(memory_format=torch.channels_last)
    ts = trainer.TrainStep(m, lr=0.0, weights="bf16")
    ts.capture(x, y.cuda(), warmup=2)
    loss = ts.step(x, y.cuda()).item()
    errs = _grad_errors(ts.grads(), g)
    _record("hybrid_bf16_se_cotnetd_101", dict(errs, loss=loss, loss_ref=float(g["loss"])))
    assert abs(loss - float(g["loss"])) <= 1e-2 * float(g["loss"])
    assert errs["median_norm"] <= 2.5e-1 and errs["median_proj"] <= 5e-2, errs     # bf16 training-mode gradients: see the bench-path test


# ------------------------------------------------------------------------------------------------ SplitAttn tail
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-4), (torch.bfloat16, 3e-2)])
@pytest.mark.parametrize("training", [True, False])
def test_split_attn_fused_vs_plain(dtype, tol, training):
    """SplitAttnConv2d (radix 1): the fused tail path (channels_last CUDA) against the module's own plain-PyTorch branch."""
    from cotnet_b200 import backbone_hybrid as bh
    torch.manual_seed(7)
    m = bh.SplitAttnConv2d(64, 64, 3, stride=1, padding=1, radix=1).cuda()
    with torch.no_grad():
        for bn in (m.bn0, m.bn1):
            bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(0, 0.2); bn.running_mean.normal_(0, 0.3); bn.running_var.uniform_(0.5, 2.0)
    m.train(training)
    m2 = copy.deepcopy(m)
    x = torch.randn(8, 64, 14, 14, device="cuda")
    cot = torch.randn(8, 64, 14, 14, device="cuda")
    xa = x.clone().requires_grad_(True)                                   # NCHW-contiguous -> plain branch (fp32 reference)
    ya = m2(xa)
    (ya * cot).sum().backward()
    mb = m.to(dtype).to(memory_format=torch.channels_last)
    xb = x.to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    yb = mb(xb)
    (yb.float() * cot).sum().backward()
    rel = lambda a_, b_, fl=1e-12: ((a_.float() - b_.float()).norm() / b_.float().norm().clamp_min(fl)).item()   # noqa: E731
    assert rel(yb, ya) <= tol, rel(yb, ya)
    assert rel(xb.grad, xa.grad) <= 4 * tol, rel(xb.grad, xa.grad)
    # fc1.bias sits in front of a batch-statistics BatchNorm: its true gradient is exactly zero, both sides hold rounding noise.
    # Parameters are judged relative to max(their own gradient norm, 1 % of the largest gradient norm of the module).
    floor = 1e-2 * max(p_.grad.float().norm().item() for p_ in m2.parameters())
    for (n, pa), (_, pb) in zip(m2.named_parameters(), mb.named_parameters()):
        assert rel(pb.grad, pa.grad, floor) <= 6 * tol, (n, rel(pb.grad, pa.grad, floor))
    if training:
        assert torch.allclose(mb.bn0.running_mean.float(), m2.bn0.running_mean, atol=5 * tol, rtol=5 * tol)
        assert torch.allclose(mb.bn1.running_var.float(), m2.bn1.running_var, atol=5 * tol, rtol=5 * tol)


def test_forked_block_outputs_model_level():
    """COTB200_FORK=1 (opt-in): every bottleneck hands its output to the next one as two aliases and bn3's backward kernels sum the two
    incoming gradients (cotb200_bn_bwd_{sums,apply}2).  Same loss and gradients as the default graph (autograd add).  Training-mode
    gradients of these nets are ill-conditioned (batch-statistics BatchNorms, atomics-ordered sums: two runs of the SAME graph differ at
    the percent level), so the gate is relative: forked vs default must be as close as default vs default."""
    from cotnet_b200 import backbone
    torch.manual_seed(3)
    m0 = backbone.CoTResNet([2, 1, 1, 1], num_classes=16, zero_init_last_bn=False).cuda().to(memory_format=torch.channels_last).train()
    x = torch.randn(16, 3, 96, 96, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 16, (16,), device="cuda")

    def run(fork):
        m = copy.deepcopy(m0)
        for blk in m.modules():
            if isinstance(blk, backbone.Bottleneck):
                blk.fork_output = fork
        m.layer4[-1].fork_output = False
        loss = torch.nn.functional.cross_entropy(m(x), y)          # fp32, no autocast: the plumbing is what is under test
        loss.backward()
        return loss.item(), {n: p.grad.float() for n, p in m.named_parameters()}

    def med(ga, gb):
        rels = sorted(((ga[n] - g).norm() / g.norm().clamp_min(1e-6)).item() for n, g in gb.items())
        return rels[len(rels) // 2]

    la, ga = run(False)
    lb, gb = run(False)
    lc, gc = run(True)
    assert abs(lc - la) <= 1e-4 * abs(la) + 2 * abs(lb - la), (la, lb, lc)
    noise, diff = med(gb, ga), med(gc, ga)
    assert diff <= 3 * noise + 1e-3, (diff, noise)
