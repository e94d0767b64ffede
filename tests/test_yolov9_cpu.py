"""CPU: YOLOv9-T/S/M/C packer, folds, the aligned channel layout and plan validation.

The graphs restate WongKinYiu/yolov9 v0.1's converted (GELAN) models; with no upstream file available, the published counts are their
anchor: parameters of the fused graph (grouped convs at their grouped size, the 16 fixed DFL weights included) and 2 * MAC at 640x640."""

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import adas_b200  # noqa: F401
from adas_b200 import plan
import plan_footprint as fp
import yolov9_oracle as o9

PUBLISHED = [("t", 2.002, 7.71), ("s", 7.106, 26.38), ("m", 19.979, 76.31), ("c", 25.289, 102.14)]


@pytest.mark.parametrize("scale,mparams,gflop", PUBLISHED)
def test_yolov9_counts_match_the_published_figures(scale, mparams, gflop):
    W = plan.synth_weights("yolov9", 0, variant=scale)
    pb = plan.build_yolov9(W, scale)
    assert abs(pb.flops_per_img / 1e9 - gflop) < 0.005, pb.flops_per_img / 1e9
    fused = o9.build(W.state_dict, scale).fuse()
    assert abs(o9.fused_params(fused) / 1e6 - mparams) < 0.0005, o9.fused_params(fused) / 1e6
    assert o9.flops(fused) == pb.flops_per_img
    assert pb.model_kind == plan.MODEL_YOLOV8 and pb.meta[:2] == [80, 8400] and len(pb.outputs) == 3
    n_pool = sum(1 for op in pb.ops if op[0] == plan.OP_AVGPOOL2)
    assert n_pool == (10 if scale == "c" else 5)                     # ADown: one per half; AConv: one
    assert sum(1 for op in pb.ops if op[0] == plan.OP_AVGPOOL2 and op[1].fill == 1) == (5 if scale == "c" else 0)


def test_grouped_conv_packs_as_block_diagonal():
    rng = np.random.default_rng(0)
    w = rng.standard_normal((64, 16, 3, 3)).astype(np.float32)
    x = torch.from_numpy(rng.standard_normal((1, 64, 9, 11)).astype(np.float32))
    d = plan.grouped_to_dense(w, 4)
    assert d.shape == (64, 64, 3, 3)
    ref = F.conv2d(x, torch.from_numpy(w), padding=1, groups=4)
    got = F.conv2d(x, torch.from_numpy(d), padding=1)
    assert torch.allclose(ref, got, atol=1e-5)
    assert plan.grouped_to_dense(w, 1) is w


@pytest.mark.parametrize("scale", ["s", "m"])
def test_packer_folds_equal_oracle_fuse(scale):
    """RepConvN (3x3 + 1x1 on the centre tap) and Conv + BN folded by the packer equal the oracle's fuse() to 1e-5."""
    W = plan.synth_weights("yolov9", 2, variant=scale)
    plan.build_yolov9(W, scale, in_h=320, in_w=320)
    fused = o9.build(W.state_dict, scale).fuse()
    n_rep = n_conv = 0
    for name, m in fused.named_modules():
        if isinstance(m, o9.RepConvN):
            c = m.conv
            w, b = W.repconvn(name, c.out_channels, c.in_channels, plan.BN_EPS_YOLO)
            n_rep += 1
        elif isinstance(m, o9.Conv):
            c = m.conv
            w, b = W.conv_bn(name, c.out_channels, c.in_channels // c.groups, c.kernel_size[0], plan.BN_EPS_YOLO)
            n_conv += 1
        else:
            continue
        assert np.abs(w - c.weight.detach().numpy()).max() < 1e-5 and np.abs(b - c.bias.detach().numpy()).max() < 1e-5, name
    assert n_rep == plan.yolov9_repconvn_count(scale) and n_conv > 0


@pytest.mark.parametrize("scale", ["t", "s", "m", "c"])
def test_oracle_fused_equals_training_form(scale):
    W = plan.synth_weights("yolov9", 1, variant=scale)
    plan.build_yolov9(W, scale, in_h=320, in_w=320)
    x = torch.rand(1, 3, 320, 320)
    with torch.no_grad():
        a = o9.build(W.state_dict, scale)(x).numpy()
        b = o9.build(W.state_dict, scale).fuse()(x).numpy()
    assert a.shape == (1, 84, 2100)
    assert np.abs(a[:, 4:] - b[:, 4:]).max() < 1e-4
    assert np.abs(a[:, :4] - b[:, :4]).max() < 1e-4 * max(1.0, float(np.abs(a[:, :4]).max()))


def test_fused_checkpoint_packs_the_training_form_plan():
    """A state_dict after upstream's fuse (RepConvN `conv`, Conv with a bias, no BN) packs the same network."""
    W = plan.synth_weights("yolov9", 6, variant="m")
    ref = plan.build_yolov9(W, "m", in_h=320, in_w=320)
    sd = {k: v.detach().numpy() for k, v in o9.build(W.state_dict, "m").fuse().state_dict().items()}
    assert not any(".conv1." in k or ".bn." in k for k in sd)
    got = plan.build_yolov9(plan.Weights(sd), "m", in_h=320, in_w=320)
    assert [(t, p) for t, p, _ in ref.ops] == [(t, p) for t, p, _ in got.ops]
    for a, b in zip(ref.tensors, got.tensors):
        assert a.shape == b.shape and np.abs(a.astype(np.float32) - b.astype(np.float32)).max() <= 2e-3 * max(1.0, float(np.abs(a).max()))


def _gemm_weights(pb, shape):
    return [pb.tensors[op[1].w_tensor].astype(np.float32) for op in pb.ops if op[0] == plan.OP_GEMM and pb.tensors[op[1].w_tensor].shape == shape]


def test_yolov9m_aligned_layout_equals_the_oracle_weights():
    """YOLOv9-M's 180 / 90-channel members sit at multiples of 8: model.6's first 1x1 conv writes its two 180-channel chunks as row
    blocks [0, 180) and [184, 364) of one GEMM, its cv4 and the RepNCSP cv3 read their inputs around zero columns; packed weights equal
    the oracle's fused convs with the gaps zero."""
    W = plan.synth_weights("yolov9", 3, variant="m")
    pb = plan.build_yolov9(W, "m", in_h=320, in_w=320)
    fused = dict(o9.build(W.state_dict, "m").fuse().named_modules())
    h = lambda name: fused[name].conv.weight.detach().numpy()[:, :, 0, 0].astype(np.float16).astype(np.float32)
    # model.6.cv1: Conv(360, 360, 1) -> rows [0, 180) and [184, 364) of a 368-row GEMM
    w = _gemm_weights(pb, (368, 360))[0]
    ref = h("model.6.cv1")
    assert np.array_equal(w[:180], ref[:180]) and np.array_equal(w[184:364], ref[180:]) and not w[180:184].any() and not w[364:].any()
    # model.6.cv4: Conv(720, 360, 1) on members at 0, 184, 368, 552 of a 736-channel concat
    w = _gemm_weights(pb, (360, 736))[0]
    ref = h("model.6.cv4")
    for i in range(4):
        assert np.array_equal(w[:, 184 * i:184 * i + 180], ref[:, 180 * i:180 * (i + 1)]) and not w[:, 184 * i + 180:184 * (i + 1)].any()
    # model.6.cv2.0.cv3: Conv(180, 180, 1) on [m (90 of 96), cv2 (90 of 96)], 184 stored rows
    w = _gemm_weights(pb, (184, 192))[0]
    ref = h("model.6.cv2.0.cv3")
    assert np.array_equal(w[:180, :90], ref[:, :90]) and np.array_equal(w[:180, 96:186], ref[:, 90:])
    assert not w[:, 90:96].any() and not w[:, 186:].any() and not w[180:].any()
    # every GEMM reads and writes at multiples of 8 channels
    assert all(op[1].a_coff % 8 == 0 and op[1].out_coff % 8 == 0 for op in pb.ops if op[0] == plan.OP_GEMM)


@pytest.mark.skipif(torch.cuda.is_available(), reason="load-time validation is observed through the missing-device error")
def test_plan_validator_rejects_bad_avgpool2_ops(tmp_path):
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 16, 16)
    xin = pb.new_padded(16, 16, 64)
    out = pb.new_padded(16, 16, 32)
    other = pb.new_padded(8, 8, 32)
    f32 = pb.new_padded(16, 16, 32, f32=True)
    pb.avgpool2(pb.sub(xin, 8, 16), 1, out=pb.sub(out, 8, 16))
    good = tmp_path / "ap.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    p = lambda name: fp.parse(raw).field_off(0, name)
    cases = [
        ("input index", fp.corrupt(raw, p("in_buf"), "<i", 99), "index out of range"),
        ("output index", fp.corrupt(raw, p("out_buf"), "<i", -1), "index out of range"),
        ("fp32 output", fp.corrupt(raw, p("out_buf"), "<i", f32.buf), "fp16"),
        ("geometry", fp.corrupt(raw, p("out_buf"), "<i", other.buf), "H x W"),
        ("channels", fp.corrupt(raw, p("C"), "<i", 12), "multiples of 8"),
        ("input offset", fp.corrupt(raw, p("in_coff"), "<i", 4), "multiples of 8"),
        ("output offset", fp.corrupt(raw, p("out_coff"), "<i", 12), "multiples of 8"),
        ("input slice", fp.corrupt(raw, p("in_coff"), "<i", 56), "exceeds"),
        ("output slice", fp.corrupt(raw, p("out_coff"), "<i", 24), "exceeds"),
        ("in place", fp.corrupt(fp.corrupt(raw, p("out_buf"), "<i", xin.buf), p("out_coff"), "<i", 16), "overlaps"),
        ("fill", fp.corrupt(raw, p("fill"), "<i", 2), "fill"),
    ]
    for name, data, msg in cases:
        bad = tmp_path / "bad.b200w"
        bad.write_bytes(data)
        err = fp.engine_error(bad)
        assert err is not None and "plan" in err and msg in err, (name, err)
