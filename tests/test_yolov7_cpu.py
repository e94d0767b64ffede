"""CPU: YOLOv7 / YOLOv7-tiny packer, folds, ONNX recognition and the plan-carried anchor table.

The graphs restate cfg/training/yolov7.yaml and yolov7-tiny.yaml; with no upstream file available, the published counts are their
anchor (FLOP = 2 * MAC of the fused graph at 640x640).  ONNX files are written by torch's exporter from the oracle (tests/yolov7_oracle.py)
after the upstream-style fuse(), at 320x320 to keep CPU time short."""
import os

import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import onnx_import, plan
import plan_footprint as fp
import test_onnx_import as toi
import yolov7_oracle as o7


def _fused_params(W):
    """parameters of the fused graph: every conv weight + one bias per output channel (RepConv's 1x1 folds into its 3x3)."""
    return sum(v.size + v.shape[0] for k, v in W.state_dict.items() if k.endswith(".weight") and v.ndim == 4 and ".rbr_1x1." not in k)


@pytest.mark.parametrize("scale,gflop,mparams", [("tiny", 13.8, 6.2), ("base", 104.7, 36.9)])
def test_yolov7_graph_matches_published_counts(scale, gflop, mparams):
    W = plan.synth_weights("yolov7", 0)
    pb = plan.build_yolov7(W, scale)
    assert abs(pb.flops_per_img / 1e9 - gflop) < 0.3
    assert abs(_fused_params(W) / 1e6 - mparams) < 0.1
    assert pb.model_kind == plan.MODEL_YOLOV5 and pb.meta[:3] == [80, 25200, 0] and len(pb.outputs) == 3
    anc = plan.YOLOV7_ANCHORS if scale == "base" else plan.YOLOV5_ANCHORS
    assert np.array_equal(pb.tensors[pb.meta[3] - 1], np.asarray(anc, np.float32).reshape(18))
    acts = {op[1].act for op in pb.ops if op[0] == plan.OP_GEMM and not pb.buffers[op[1].out_buf][2]}
    assert acts == {plan.ACT_LEAKY if scale == "tiny" else plan.ACT_SILU}
    stem = pb.ops[0]                               # the image conv runs in stem_conv.cu: stride 1 (base, field 1) or 2 (tiny, field 0)
    assert stem[0] == plan.OP_STEMCONV and stem[1].Cout == 32 and stem[1].stride == (1 if scale == "base" else 0)


def test_tiny_silu_variant():
    pb = plan.build_yolov7(plan.synth_weights("yolov7", 0), "tiny", act="silu")
    assert {p.act for t, p, _ in pb.ops if t == plan.OP_GEMM and p.act != plan.ACT_NONE} == {plan.ACT_SILU}


def test_packer_folds_equal_oracle_fuse():
    """RepConv (BN-folded 3x3 + BN-folded 1x1 on the centre tap) and IDetect (w' = im w, b' = im (b + w ia)) against the oracle's fuse()."""
    for scale, det in (("base", 105), ("tiny", 77)):
        W = plan.synth_weights("yolov7", 2)
        plan.build_yolov7(W, scale)
        fused = o7.build(W.state_dict, scale).fuse()
        if scale == "base":
            for i, (cin, cout) in enumerate(((128, 256), (256, 512), (512, 1024))):
                w, b = W.repconv(f"model.{102 + i}", cout, cin, plan.BN_EPS_YOLO)
                r = fused.model[102 + i].rbr_reparam
                assert np.abs(w - r.weight.detach().numpy()).max() < 1e-5 and np.abs(b - r.bias.detach().numpy()).max() < 1e-5
        for li, conv in enumerate(fused.model[det].m):
            w, b = W.implicit_head(f"model.{det}", li, 255, conv.in_channels)
            assert np.abs(w - conv.weight.detach().numpy()).max() < 1e-5 and np.abs(b - conv.bias.detach().numpy()).max() < 1e-5


@pytest.mark.parametrize("scale", ["tiny", "base"])
def test_oracle_fused_equals_training_form(scale):
    W = plan.synth_weights("yolov7", 1)
    plan.build_yolov7(W, scale, in_h=320, in_w=320)
    x = torch.rand(1, 3, 320, 320)
    with torch.no_grad():
        a = o7.build(W.state_dict, scale)(x).numpy()
        b = o7.build(W.state_dict, scale).fuse()(x).numpy()
    assert a.shape == (1, 6300, 85)
    assert np.abs(a[..., 4:] - b[..., 4:]).max() < 1e-4                    # fp32 rounding of the reordered sums
    assert np.abs(a[..., :4] - b[..., :4]).max() < 1e-4 * max(1.0, float(np.abs(a[..., :4]).max()))


def _export_v7(tmp_path, scale, seed, name, act=None, anchors=None):
    W = plan.synth_weights("yolov7", seed)
    ref = plan.build_yolov7(W, scale, in_h=320, in_w=320, act=act, anchors=anchors)
    path = str(tmp_path / f"{name}.onnx")
    toi._export(o7.build(W.state_dict, scale, act=act, anchors=anchors).fuse(), (1, 3, 320, 320), path)
    return W, ref, path


@pytest.mark.parametrize("scale,act", [("tiny", "leaky"), ("base", "silu"), ("tiny", "silu")])
def test_fused_export_is_recognised_and_packs_the_state_dict_plan(tmp_path, scale, act):
    W, ref, path = _export_v7(tmp_path, scale, 3, f"v7{scale}{act}", act=act)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.act, spec.nc, spec.in_h, spec.in_w) == ("yolov7", scale, act, 80, 320, 320)
    got = onnx_import.build_plan(m, spec)
    toi._assert_same_plan(ref, got, f"yolov7-{scale} {act}")


def test_export_with_custom_anchors_puts_them_in_the_plan(tmp_path):
    anchors = tuple(tuple(float(v) * 1.5 for v in lvl) for lvl in o7.V5_ANCHORS)
    W, ref, path = _export_v7(tmp_path, "tiny", 4, "v7anchors", anchors=anchors)
    got = onnx_import.build_plan(onnx_import.read_onnx(path))
    assert np.array_equal(got.tensors[got.meta[3] - 1], np.asarray(anchors, np.float32).reshape(18))
    toi._assert_same_plan(ref, got, "yolov7-tiny custom anchors")


def test_yolov8s_export_is_still_yolov8(tmp_path):
    """YOLOv8s starts with a (32, 3, 3, 3) stride-2 conv exactly like YOLOv7-tiny."""
    W = plan.synth_weights("yolov8", 5)
    plan.build_yolov8(W, "s", in_h=320, in_w=320)
    path = str(tmp_path / "v8s.onnx")
    toi._export(toi._fuse_conv_bn(toi.nets.build("yolov8", W.state_dict, scale="s")), (1, 3, 320, 320), path)
    spec = onnx_import.recognise(onnx_import.read_onnx(path))
    assert (spec.kind, spec.scale, spec.nc) == ("yolov8", "s", 80)


def test_out_of_scope_yolov7_file_names_the_supported_variants(tmp_path):
    """A YOLOv7-X-like file: 40-channel stem, MP blocks (2x2 max pool), three detection convs."""
    class XLike(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.stem = torch.nn.Conv2d(3, 40, 3, 1, 1)
            self.m = torch.nn.ModuleList(torch.nn.Conv2d(40, 255, 1) for _ in range(3))

        def forward(self, x):
            y = torch.nn.functional.max_pool2d(torch.nn.functional.silu(self.stem(x)), 2, 2)
            return [m(y) for m in self.m]
    path = str(tmp_path / "v7x_like.onnx")
    toi._export(XLike(), (1, 3, 64, 64), path)
    with pytest.raises(Exception, match="YOLOv7 and YOLOv7-tiny"):
        onnx_import.recognise(onnx_import.read_onnx(path))


def test_checkpoint_conversion(tmp_path):
    from adas_b200 import convert
    W = plan.synth_weights("yolov7", 6)
    ref = plan.build_yolov7(W, "tiny")
    ckpt = str(tmp_path / "v7t.pth")
    torch.save({"model": {k: torch.from_numpy(np.asarray(v)) for k, v in W.state_dict.items()}}, ckpt)
    got = convert.plan_from_state_dict(convert.load_checkpoint_state_dict(ckpt), "yolov7", scale="tiny")
    assert ref.ops == got.ops and all(np.array_equal(a, b) for a, b in zip(ref.tensors, got.tensors))
    assert convert.main([ckpt, "--kind", "yolov7", "--scale", "tiny"]) == 0
    # an upstream checkpoint carries IDetect's anchor_grid buffer: its anchors go into the plan
    sd = dict(W.state_dict)
    sd["model.77.anchor_grid"] = np.arange(1, 19, dtype=np.float32).reshape(3, 1, 3, 1, 1, 2)
    pb = convert.plan_from_state_dict(sd, "yolov7", scale="tiny")
    assert np.array_equal(pb.tensors[pb.meta[3] - 1], np.arange(1, 19, dtype=np.float32))


@pytest.mark.skipif(torch.cuda.is_available(), reason="load-time validation is observed through the missing-device error")
def test_anchor_table_and_activation_validation(tmp_path):
    # a plan without an anchor table (every YOLOv5 plan) validates and decodes with the YOLOv5 table
    v5 = tmp_path / "v5n.b200w"
    plan.build_yolov5(plan.synth_weights("yolov5", 0), "n").write(str(v5))
    assert "no CUDA device" in fp.engine_error(v5)
    assert np.array_equal(plan.read_anchors(str(v5)), np.asarray(plan.YOLOV5_ANCHORS, np.float32).reshape(3, 3, 2))
    v7 = tmp_path / "v7.b200w"
    pb = plan.build_yolov7(plan.synth_weights("yolov7", 0), "tiny", in_h=320, in_w=320, anchors=plan.YOLOV7_ANCHORS)
    pb.write(str(v7))
    assert "no CUDA device" in fp.engine_error(v7)
    assert np.array_equal(plan.read_anchors(str(v7)), np.asarray(plan.YOLOV7_ANCHORS, np.float32).reshape(3, 3, 2))
    # a non-positive anchor, an anchor index outside the tensors, an anchor table on a lite plan: rejected at load
    raw = v7.read_bytes()
    pl = fp.parse(raw)
    blob = pl.header[-2]
    off = pl.tensors[pb.meta[3] - 1][0]
    meta3 = 8 + 4 * 2 + 4 * 3 + 4 * 4 + 4 * 3
    for name, data in (("negative anchor", fp.corrupt(raw, blob + off + 8, "<f", -4.0)),
                       ("nan anchor", fp.corrupt(raw, blob + off, "<f", float("nan"))),
                       ("anchor index", fp.corrupt(raw, meta3, "<I", 100000)),
                       ("lite flag", fp.corrupt(raw, meta3 - 4, "<I", 1))):
        bad = tmp_path / "bad.b200w"
        bad.write_bytes(data)
        err = fp.engine_error(bad)
        assert err is not None and "plan" in err and "anchor" in err, (name, err)
    # activation ids above 3 are rejected (GEMM and stem conv)
    for image in (False, True):
        b1 = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, 16, 16)
        x = b1.image if image else b1.new_padded(16, 16, 64)
        b1.conv(x, np.ones((32, 3 if image else 64, 3, 3), np.float32), np.zeros(32, np.float32), 3, 1, 4)
        p = tmp_path / f"act{int(image)}.b200w"
        b1.write(str(p))
        assert b1.ops[-1][0] == (plan.OP_STEMCONV if image else plan.OP_GEMM)
        assert "unknown activation 4" in fp.engine_error(p)
        b1.ops[-1][1].act = plan.ACT_LEAKY
        b1.write(str(p))
        assert "no CUDA device" in fp.engine_error(p)
