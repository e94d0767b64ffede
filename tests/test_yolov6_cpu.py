"""CPU: YOLOv6 N/S/M/L packer, folds and plan validation.

The graphs restate meituan/YOLOv6 0.4.0 (configs/yolov6{n,s,m,l}.py); with no upstream file available, the published deployed-model counts
are their anchor.  The published GFLOP figures (thop, 2 * MAC at 640x640) count a ConvTranspose2d(k=2, s=2) at output elements x Cin x 4
MACs, four times its algorithmic MACs; the plan counts algorithmic FLOP, so the check adds the difference back."""

import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import plan
import plan_footprint as fp
import yolov6_oracle as o6


def _fused_params(W):
    """parameters of the deployed graph: conv / transposed-conv weights + one bias per output channel (the RepVGG 1x1 and identity
    branches fold into the 3x3) + BottleRep alphas."""
    n = 0
    for k, v in W.state_dict.items():
        if k.endswith(".weight") and v.ndim == 4 and ".rbr_1x1." not in k:
            n += v.size + (v.shape[1] if "upsample_transpose" in k else v.shape[0])
        elif k.endswith(".alpha"):
            n += v.size
    return n


def _transpose_flops(pb):
    return sum(2 * pb.buffers[p.a_buf][3] * pb.buffers[p.a_buf][4] * p.Kc * p.N for t, p, _ in pb.ops
               if t == plan.OP_GEMM and p.up2 == 1)


PUBLISHED = [("n", 11.4, 4.7), ("s", 45.3, 18.5), ("m", 85.8, 34.9), ("l", 150.7, 59.6)]


@pytest.mark.parametrize("scale,gflop,mparams", PUBLISHED)
def test_yolov6_flops_match_published_counts(scale, gflop, mparams):
    W = plan.synth_weights("yolov6", 0)
    pb = plan.build_yolov6(W, scale)
    thop = pb.flops_per_img + 3 * _transpose_flops(pb)
    assert abs(thop / 1e9 - gflop) < 0.05, thop / 1e9
    reg_max = 16 if scale in "ml" else 0
    assert pb.model_kind == plan.MODEL_YOLOV6 and pb.meta[:3] == [80, 8400, reg_max] and len(pb.outputs) == 3
    gemm_acts = {p.act for t, p, _ in pb.ops if t == plan.OP_GEMM and not pb.buffers[p.out_buf][2] and p.up2 == 0}
    assert gemm_acts == ({plan.ACT_SILU, plan.ACT_RELU})
    stem = pb.ops[0]
    assert stem[0] == plan.OP_STEMCONV and stem[1].act == (plan.ACT_SILU if scale == "l" else plan.ACT_RELU)
    assert sum(1 for t, p, _ in pb.ops if t == plan.OP_GEMM and p.up2 == 1) == 2          # the two BiFusion transposed convs
    n_scaled = sum(1 for op in pb.ops if op[0] == plan.OP_GEMM and op[2][0] != 0.0)
    assert n_scaled == ({"m": 2 + 3 + 5 + 2 + 4 * 3, "l": 3 + 6 + 9 + 3 + 4 * 6}.get(scale, 0))   # BottleReps with their alpha


@pytest.mark.parametrize("scale,gflop,mparams", [
    pytest.param(*PUBLISHED[0], marks=pytest.mark.xfail(strict=True, reason=(
        "the N restatement has 4.647 M parameters, 0.003 M under the published 4.7 M's rounding interval, while N's FLOP count and "
        "S / M / L's parameter counts match; no single structural change found reaches 4.65 M"))),
    *PUBLISHED[1:]])
def test_yolov6_params_match_published_counts(scale, gflop, mparams):
    W = plan.synth_weights("yolov6", 0)
    plan.build_yolov6(W, scale)
    assert abs(_fused_params(W) / 1e6 - mparams) < 0.05, _fused_params(W) / 1e6


def test_activation_arguments_choose_the_epilogues():
    pb = plan.build_yolov6(plan.synth_weights("yolov6", 0), "s", act_body="silu", act_neck="silu", act_head="relu", in_h=320, in_w=320)
    assert {p.act for t, p, _ in pb.ops if t == plan.OP_GEMM and not pb.buffers[p.out_buf][2] and p.up2 == 0} == {plan.ACT_SILU, plan.ACT_RELU}
    pb = plan.build_yolov6(plan.synth_weights("yolov6", 0), "s", act_body="silu", act_neck="silu", act_head="silu", in_h=320, in_w=320)
    assert {p.act for t, p, _ in pb.ops if t == plan.OP_GEMM and not pb.buffers[p.out_buf][2] and p.up2 == 0} == {plan.ACT_SILU}


@pytest.mark.parametrize("scale", ["s", "m"])
def test_packer_repvgg_folds_equal_oracle_fuse(scale):
    """RepVGG (3x3 + 1x1 + identity BN) folded by the packer equals the oracle's fuse() to 1e-5, with and without the identity branch."""
    W = plan.synth_weights("yolov6", 2)
    plan.build_yolov6(W, scale, in_h=320, in_w=320)
    fused = o6.build(W.state_dict, scale).fuse()
    mods = dict(fused.named_modules())
    checked = {True: 0, False: 0}
    for name, m in mods.items():
        if isinstance(m, o6.RepVGGBlock):
            r = m.rbr_reparam
            idt = r.in_channels == r.out_channels and r.stride == (1, 1)
            w, b = W.repconv(name, r.out_channels, r.in_channels, plan.BN_EPS_YOLO, keys=("conv", "bn"), identity=idt)
            assert np.abs(w - r.weight.detach().numpy()).max() < 1e-5 and np.abs(b - r.bias.detach().numpy()).max() < 1e-5, name
            checked[idt] += 1
    assert checked[True] > 0 and checked[False] > 0


def test_yolov7_repconv_fold_is_unchanged():
    """The YOLOv7 call of the shared fold (Sequential keys, no identity) gives what it gave before it learned the YOLOv6 names."""
    W = plan.synth_weights("yolov7", 2)
    plan.build_yolov7(W, "base")
    w, b = W.repconv("model.102", 256, 128, plan.BN_EPS_YOLO)
    wd, bd = W._conv_bn64("model.102.rbr_dense", 256, 128, 3, plan.BN_EPS_YOLO, conv_key="0", bn_key="1")
    w1, b1 = W._conv_bn64("model.102.rbr_1x1", 256, 128, 1, plan.BN_EPS_YOLO, conv_key="0", bn_key="1")
    wd[:, :, 1, 1] += w1[:, :, 0, 0]
    assert np.array_equal(w, wd.astype(np.float32)) and np.array_equal(b, (bd + b1).astype(np.float32))


@pytest.mark.parametrize("scale", ["n", "s", "m", "l"])
def test_oracle_fused_equals_training_form(scale):
    W = plan.synth_weights("yolov6", 1)
    plan.build_yolov6(W, scale, in_h=320, in_w=320)
    x = torch.rand(1, 3, 320, 320)
    with torch.no_grad():
        a = o6.build(W.state_dict, scale)(x).numpy()
        b = o6.build(W.state_dict, scale).fuse()(x).numpy()
    assert a.shape == (1, 2100, 85) and np.all(a[..., 4] == 1.0)
    assert np.abs(a[..., 5:] - b[..., 5:]).max() < 1e-4
    assert np.abs(a[..., :4] - b[..., :4]).max() < 1e-4 * max(1.0, float(np.abs(a[..., :4]).max()))


def test_deployed_checkpoint_packs_the_training_form_plan():
    """A state_dict after upstream's fuse (rbr_reparam, ConvModule convs with a bias, no BN) packs the same network."""
    W = plan.synth_weights("yolov6", 6)
    ref = plan.build_yolov6(W, "n", in_h=320, in_w=320)
    sd = {k: v.detach().numpy() for k, v in o6.build(W.state_dict, "n").fuse().state_dict().items()}
    assert any(".rbr_reparam." in k for k in sd) and not any(".rbr_dense." in k for k in sd)
    got = plan.build_yolov6(plan.Weights(sd), "n", in_h=320, in_w=320)
    assert [(t, p) for t, p, _ in ref.ops] == [(t, p) for t, p, _ in got.ops]
    for a, b in zip(ref.tensors, got.tensors):
        assert a.shape == b.shape and np.abs(a.astype(np.float32) - b.astype(np.float32)).max() <= 2e-3 * max(1.0, float(np.abs(a).max()))


@pytest.mark.skipif(torch.cuda.is_available(), reason="load-time validation is observed through the missing-device error")
def test_plan_validator_rejects_bad_yolov6_fields(tmp_path):
    pb = plan.build_yolov6(plan.synth_weights("yolov6", 0), "m", in_h=320, in_w=320)
    good = tmp_path / "v6m.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    pl = fp.parse(raw)
    meta2 = 8 + 4 * fp.HEADER_FIELDS.index("meta2")
    up = next(i for i, (t, p, _) in enumerate(pb.ops) if t == plan.OP_GEMM and p.up2 == 1)
    res = next(i for i, (t, p, _) in enumerate(pb.ops) if t == plan.OP_GEMM and p.res_buf >= 0)
    cases = [
        ("reg_max", fp.corrupt(raw, meta2, "<I", 8), "reg_max"),
        ("narrow level", fp.corrupt(raw, pl.out_off(0) + 8, "<I", 72 + 79), "columns wide"),
        ("transposed Cout", fp.corrupt(raw, pl.field_off(up, "N"), "<i", pb.ops[up][1].N - 16), "transposed conv"),
        ("transposed geometry", fp.corrupt(raw, pl.field_off(up, "out_buf"), "<i", pb.ops[up][1].a_buf), "transposed conv"),
        ("residual scale", fp.corrupt(raw, pl.field_off(res, "res_scale"), "<f", float("inf")), "residual scale"),
    ]
    for name, data, msg in cases:
        bad = tmp_path / "bad.b200w"
        bad.write_bytes(data)
        err = fp.engine_error(bad)
        assert err is not None and "plan" in err and msg in err, (name, err)
