"""SE-CoTNetD-152 at the reference's largest data configs, 256 x 256 (cot_s, se_cotnetd_152) and 320 x 320 (cot_l,
se_cotnetd_152_L), stage by stage.  The trunk pools every stride-2 block with a BlurPool after conv2 (avd, avd_first=False), so its
CoT layers run at geometries the 224-class models never reach: 40x40, 20x20 and 10x10 at 320, 32x32, 16x16 and 8x8 at 256.

  * one eager TrainStep(weights="bf16").forward_backward at each size with drop path at the config's 0.15: the whole call list
    against stage_ref.model_calls, every stage, every BlurPool, block-to-block dataflow, the gradient at every block input, the
    flat buckets (test_step_stages_gpu.train_step_stage_by_stage);
  * one eval forward of se_cotnetd_152_L at 320 through test_eval_blocks_gpu's network check, with the captured EvalStep's logits
    bit-equal to the eager ones;
  * the wgmma key convolution and the CoT layer's GEMM epilogues at every geometry of the trunk, on small-integer operands (exact
    accumulators, torch.equal), each with its launch plan asserted and the planned kernel seen by the profiler.

The block cases of the same trunk are in stage_ref.STEP_BLOCK_CASES and EVAL_BLOCK_CASES."""
import pytest

import stage_ref as S
from test_determinism_gpu import TC_BM, _cdiv, _sms, pick_bn
from test_eval_blocks_gpu import eval_network_stage_by_stage
from test_eval_kernels_gpu import GEMM_FORMS, gemm_exact, key_conv_exact
from test_persistent_gpu import conv3x3_halo_launch, conv3x3_tc_launch
from test_step_stages_gpu import train_step_stage_by_stage

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ whole networks
@pytest.mark.parametrize("res", [256, 320])
def test_train_step_se_cotnetd_152(res, monkeypatch):
    train_step_stage_by_stage("se_cotnetd_152_%d" % res, "se_cotnetd_152", None, monkeypatch, B=2, H0=res, drop_path=0.15,
                              drop_block=0.0)


def test_eval_se_cotnetd_152_L_320(monkeypatch):
    eval_network_stage_by_stage("se_cotnetd_152_L_320", "se_cotnetd_152_L", 320, 320, True, None, monkeypatch, bn3_gain=0.05)


# ------------------------------------------------------------------------------------------------ the key convolution
# (C, H, B): every CoT-layer geometry of the trunk; dim 256 (64-channel tiles) on the haloed kernel with R rows per item and two M
# blocks, dim 512 (128-channel tiles) in conv mode: 100-row bands of 5 rows, 100-row tiles of one 10x10 sample, 128-row bands of 8
# rows, two 8x8 samples per tile (odd B: a half-empty last tile)
HALO_CASES = {(256, 40, 3): 5, (256, 20, 5): 10, (256, 32, 3): 4, (256, 16, 5): 8}
CONV_MODE_CASES = {(512, 20, 3): (1, 5, 100), (512, 10, 5): (1, 10, 100), (512, 16, 3): (1, 8, 128), (512, 8, 7): (2, 8, 128)}


@pytest.mark.parametrize("case", sorted(HALO_CASES), ids=lambda c: "C%d-%dx%d-B%d" % (c[0], c[1], c[1], c[2]))
def test_key_conv_haloed_exact(case):
    C, H, B = case
    assert S.conv_tile(C, 4) == 64
    plan = conv3x3_halo_launch(B, H, H, C, _sms())
    R = plan.info["R"]
    assert R == HALO_CASES[case] and _cdiv(R * (H + 2), 128) == 2 and plan.info["n_tiles"] == C // 64, plan
    key_conv_exact((C, H, B, 64), plan)


@pytest.mark.parametrize("case", sorted(CONV_MODE_CASES), ids=lambda c: "C%d-%dx%d-B%d" % (c[0], c[1], c[1], c[2]))
def test_key_conv_conv_mode_exact(case):
    C, H, B = case
    assert S.conv_tile(C, 4) == 128                    # the haloed kernel takes 64-channel tiles only
    plan = conv3x3_tc_launch(B, H, H, C, 128, False, _sms())
    bbox, hbox, rows = CONV_MODE_CASES[case]
    assert (plan.info["bbox"], plan.info["hbox"], bbox * hbox * H) == (bbox, hbox, rows) and rows <= TC_BM, plan
    key_conv_exact((C, H, B, 128), plan)


# ------------------------------------------------------------------------------------------------ the 1x1 GEMM epilogues
# the CoT layer's embed.0, embed.3 and conv1x1 at the trunk's CoT geometries (dim, H, B); embed.3 at dim 256 is N = 288 with
# K = 128: three 128-wide N tiles, the last one 32 wide, written into a wider D whose columns past N must stay as they are.  B
# leaves a partial last M tile wherever H * H is not a multiple of 128.  The bs64 step's layer3.0 at 320 (102400 rows) too.
GEMM_CASES = [(256, 40, 3), (256, 32, 2), (256, 20, 3), (512, 20, 3), (512, 16, 2), (512, 10, 5), (512, 8, 5)]


@pytest.mark.parametrize("form", sorted(GEMM_FORMS))
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: "C%d-%dx%d-B%d" % (c[0], c[1], c[1], c[2]))
def test_gemm_epilogue_exact(case, form):
    C, H, B = case
    K1, K2, N, _, _, _ = GEMM_FORMS[form](C)
    M = B * H * H
    bn = pick_bn(N, K1 + K2)
    if form == "embed3" and C == 256:
        assert (N, bn, _cdiv(N, bn), N % bn) == (288, 128, 3, 32)
    gemm_exact(C, M, form, pad_cols=64)


def test_gemm_embed3_bs64_layer3_320():
    """the embed.3 GEMM of the bs64 training step's layer3.0 at 320: M = 64 * 40 * 40 = 102400, N = 288 in three tiles"""
    assert 64 * 40 * 40 >= S.TC_MIN_PIXELS
    gemm_exact(256, 64 * 40 * 40, "embed3", pad_cols=64)
