"""CPU checks of the eval dispatch mirror in tests/stage_ref.py: the stated call lists of the eval block cases follow the generators,
the cases' geometry is their blocks' in the models, the output-size rule of the stride-2 stages, and the whole-network lists the
GPU tests compare against.  The source lines the generators restate are pinned by test_stage_grads_cpu.test_mirror_source_anchors."""
import pytest
import torch
import torch.nn as nn

import stage_ref as S


@pytest.mark.parametrize("geo", sorted(S.EVAL_BLOCK_CASES))
def test_eval_call_lists_follow_the_mirror(geo):
    c = S.EVAL_BLOCK_CASES[geo]
    assert S.eval_case_calls(c) == c["calls"]


def _models():
    from cotnet_b200 import backbone, backbone_hybrid
    return {"cotnet50": backbone.cotnet50(), "cotnext50_2x48d": backbone.cotnext50_2x48d(), "se_cotnetd_50": backbone_hybrid.se_cotnetd_50(),
            "se_cotnetd_152": backbone_hybrid.se_cotnetd_152()}


def test_eval_block_cases_match_the_models():
    """each block case's input / width / output channels, stride and conv2 kind are its block's in the model"""
    from cotnet_b200.backbone_hybrid import SplitAttnConv2d
    from cotnet_b200.cot_layer import CoXtLayer
    models = _models()
    for geo, c in S.EVAL_BLOCK_CASES.items():
        m = models[c["model"]]
        if c["kind"] == "stem":
            assert isinstance(m.conv1, nn.Sequential) == (c["model"] in S.HYBRID), geo
            continue
        stage, i = c["block"].split(".")
        blk = getattr(m, stage)[int(i)]
        assert (blk.conv1.in_channels, blk.conv1.out_channels, blk.conv3.out_channels) == (c["cin"], c["width"], c["cout"]), geo
        if c["model"] in S.HYBRID:
            assert isinstance(blk.conv2, SplitAttnConv2d) == S.hybrid_split(c["width"], int(i), c4_idx=S.HYBRID[c["model"]]["c4_idx"]), geo
            assert (2 if int(i) == 0 else 1) == c["stride"], geo
        else:
            assert isinstance(blk.conv2, CoXtLayer) == (c["model"] != "cotnet50") and blk.stride == c["stride"], geo
        # the case's input height and width are ones the block sees for some image size
        sizes = {S.model_blocks(c["model"], h0)[[n for n, *_ in S.model_blocks(c["model"], 224)].index(c["block"])][5]
                 for h0 in range(32, 1100)}
        assert c["H"] in sizes and c["W"] in sizes, geo


@pytest.mark.parametrize("H0,W0", [(224, 224), (232, 200), (225, 225), (96, 72), (320, 320), (256, 256)])
@pytest.mark.parametrize("model", ["cotnet50", "se_cotnetd_50", "se_cotnetd_152"])
def test_model_blocks_follow_the_modules(model, H0, W0):
    """every block's input size in model_blocks is the one the trunk's own torch modules give, odd sizes included: a CPU forward of
    the trunk with its CoT layers (stride 1, shape-preserving, GPU-only kernels) replaced by identities"""
    from cotnet_b200.cot_layer import CotLayer, CoXtLayer
    m = _models()[model].eval()
    for blk in m.blocks():
        if isinstance(blk.conv2, (CotLayer, CoXtLayer)):
            blk.conv2 = nn.Identity()
    sizes = []
    for name, blk in m.named_modules():
        if name.count(".") == 1 and name.startswith("layer"):
            blk.register_forward_pre_hook(lambda mod, a, n=name: sizes.append((n, tuple(a[0].shape[2:]))))
    with torch.no_grad():
        m(torch.zeros(1, 3, H0, W0))
    want = [(n, (H, W)) for n, _, _, _, _, H, W, _ in S.model_blocks(model, H0, W0)]
    assert sizes == want


def test_output_size_rule():
    assert [S.conv_out(h, 2) for h in (224, 225, 232, 200, 58, 50, 29, 25, 15, 13, 7)] == [112, 113, 116, 100, 29, 25, 15, 13, 8, 7, 4]
    assert [(H, W) for n, _, _, _, _, H, W, s in S.model_blocks("cotnet50", 232, 200) if n.endswith(".0")] == [(58, 50), (58, 50),
                                                                                                               (29, 25), (15, 13)]
    assert S.model_blocks("cotnet50", 232, 200)[-1][5:7] == (8, 7)


@pytest.mark.parametrize("model", ["cotnet50", "cotnext50_2x48d", "se_cotnetd_50"])
def test_eval_model_calls(model):
    """the whole-network lists: every CoT layer of cotnet50 / se_cotnetd_50 on the wgmma eval path at 224, 232x200 and B = 2; the
    trunk 1x1 convolutions of stage 1 move to wgmma with TC_MIN_PIXELS = 0; CoXt's embed.0 follows the weight dtype"""
    for (H0, W0) in ((224, 224), (232, 200)):
        stem, blocks = S.eval_model_calls(model, 2, H0, W0, True)
        assert len(blocks) == 16
        flat = sum(blocks, [])
        assert "TcConv1x1Fn(one,relu)" not in flat and "FanOutFn(3)" not in flat       # 12544 pixels at most: below the threshold
        if model == "cotnext50_2x48d":
            assert flat.count("TcConv1x1Fn(two,relu)") == 16
            assert S.eval_model_calls(model, 2, H0, W0, False)[1][0].count("TcConv1x1Fn(two,relu)") == 0
        else:
            n_cot = 16 if model == "cotnet50" else 6                                   # se_cotnetd_50: layer3.0/2/4 and layer4
            assert flat.count("conv3x3_bf16") == n_cot and flat.count("cot_tail_eval") == n_cot
        stem0, blocks0 = S.eval_model_calls(model, 2, H0, W0, True, 0)
        assert blocks0[0][0] == "TcConv1x1Fn(one,relu)" and blocks0[0][-1] == "TcConv1x1Fn(one,relu+res)"
        assert stem0 == stem
    assert S.eval_model_calls("cotnet50", 2, 225, 225, True)[0] == ["BNActFn(relu)", "Pool3x3S2Fn(max)"]


def test_eval_model_calls_se_cotnetd_152():
    """se_cotnetd_152 at 320 and 256, B = 2: every CoT layer (the 18 even stage-3 blocks and stage 4) on the wgmma eval path, the
    BlurPools are torch glue (no recorded pool), the CoT layers of layer3.0 / layer4.0 at the stage's input size"""
    for res in (320, 256):
        stem, blocks = S.eval_model_calls("se_cotnetd_152", 2, res, res, True)
        assert len(blocks) == 50 and stem == ["BNActFn(relu)"] * 3
        flat = sum(blocks, [])
        assert flat.count("conv3x3_bf16") == 21 and flat.count("CotTailFn(gate)") == 29
        assert not any(c.startswith("Pool3x3S2Fn") for c in flat)
        assert blocks[11] == ["BNActFn(relu)"] + S.EVAL_LAYER_TC + ["GroupNorm9Fn(gc8)", "AggTapFn(fold1,gc8)", "cot_tail_eval",
                                                                   "BNActFn(plain)", "BNActFn(relu+res)"]
    # the stage-by-stage eval cases cover every key-conv geometry of the trunk at both sizes
    geos = {(bl[3], bl[5]) for res in (320, 256) for bl in S.model_blocks("se_cotnetd_152", res)
            if not S.hybrid_split(bl[3], bl[1], c4_idx=S.HYBRID["se_cotnetd_152"]["c4_idx"])}
    cases = {(c["width"], c["H"]) for c in S.EVAL_BLOCK_CASES.values() if c["model"] == "se_cotnetd_152" and c["kind"] == "block"}
    assert geos == {(256, 40), (256, 20), (512, 20), (512, 10), (256, 32), (256, 16), (512, 16), (512, 8)} and geos <= cases
