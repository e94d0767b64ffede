"""CPU: YOLOv7 P6 models (W6 / E6 / D6 / E6E) -- packer, the ReOrg stem fold, folds against the oracle's fuse(), the training-form checkpoint
decision and the plan validator's 4-level rules.

The graphs restate cfg/deploy/yolov7-{w6,e6,d6,e6e}.yaml (tests/yolov7_p6_oracle.py); with no upstream file available, the published yolov7
README figures at 1280x1280 are their anchor.  Those figures are the deploy graph's: they do not include the training-form aux head
(IAuxDetect's extra level convs), whose parameters the counts below would otherwise exceed."""
import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import onnx_import, plan
import plan_footprint as fp
import test_onnx_import as toi
import yolov7_p6_oracle as o6

DET = {"w6": 118, "e6": 140, "d6": 162, "e6e": 261}


def _fused_params(W):
    """parameters of the fused graph: every conv weight + one bias per output channel."""
    return sum(v.size + v.shape[0] for k, v in W.state_dict.items() if k.endswith(".weight") and v.ndim == 4)


_D6_GAP = ("D6 restated like W6 / E6 / E6E (96-channel stem, ELANs of 8 chained 3x3 convs keeping every other one, E6's head ELAN "
           "widths) gives 133.76 M / 701.7 GFLOP against the published 154.7 M / 806.8 G.  Of the 64 ways of widening some of the six head "
           "ELANs by 1.5x, none gives both figures (closest: 152.0 M / 806.7 G and 154.7 M / 794.6 G), so the gap is a structural "
           "difference not found here; a D6 checkpoint with other shapes is refused by key and shape")


@pytest.mark.parametrize("scale,gflop,mparams", [("w6", 360.0, 70.4), ("e6", 515.2, 97.2),
                                                 pytest.param("d6", 806.8, 154.7, marks=pytest.mark.xfail(reason=_D6_GAP, strict=True)),
                                                 ("e6e", 843.2, 151.7)])
def test_p6_graph_matches_published_counts(scale, gflop, mparams):
    """FLOP = 2 * MAC of the fused graph's convolutions at 1280x1280.  The restated graphs come out 0.1-0.2 % under the published
    FLOP (359.7 / 514.4 / 842.2 G), about what the pools, upsamples, concats and adds the published figures may count amount to."""
    W = plan.synth_weights("yolov7", 0)
    pb = plan.build_yolov7(W, scale)
    assert (pb.in_h, pb.in_w) == (1280, 1280)
    assert pb.model_kind == plan.MODEL_YOLOV5 and pb.meta[:3] == [80, 102000, 0] and [o[3] for o in pb.outputs] == [8, 16, 32, 64]
    assert np.array_equal(pb.tensors[pb.meta[3] - 1], np.asarray(plan.YOLOV7_P6_ANCHORS, np.float32).reshape(24))
    stem = pb.ops[0]                      # ReOrg + 3x3 as one 6x6 stride-2 pad-2 conv in stem_conv.cu
    assert stem[0] == plan.OP_STEMCONV and (stem[1].Cout, stem[1].k, stem[1].pad) == ({"w6": 64, "d6": 96}.get(scale, 80), 6, 2) and stem[1].stride == 0
    assert 0 <= gflop - pb.flops_per_img / 1e9 < 0.002 * gflop
    assert abs(_fused_params(W) / 1e6 - mparams) < 0.05


def test_out_of_scope_scales_are_refused():
    with pytest.raises(AssertionError, match="YOLOv7-X is not supported"):
        plan.build_yolov7(plan.synth_weights("yolov7", 0), "x")
    with pytest.raises(AssertionError, match="multiple of 64"):
        plan.build_yolov7(plan.synth_weights("yolov7", 0), "w6", in_h=320, in_w=352)


def test_reorg_fold_equals_reorg_then_3x3():
    rng = np.random.default_rng(0)
    w = rng.standard_normal((16, 12, 3, 3))
    x = torch.from_numpy(rng.standard_normal((2, 3, 38, 46)))
    ref = torch.nn.functional.conv2d(o6.ReOrg()(x), torch.from_numpy(w), padding=1)
    got = torch.nn.functional.conv2d(x, torch.from_numpy(plan.reorg_stem_weights(w)), stride=2, padding=2)
    assert got.shape == ref.shape and float((got - ref).abs().max()) < 1e-12


@pytest.mark.parametrize("scale", ["w6", "e6", "d6", "e6e"])
def test_packer_folds_equal_oracle_fuse(scale):
    W = plan.synth_weights("yolov7", 2)
    pb = plan.build_yolov7(W, scale, in_h=256, in_w=256)
    fused = o6.build(W.state_dict, scale).fuse()
    det = fused.model[DET[scale]]
    for li, conv in enumerate(det.m):
        w, b = W.implicit_head(f"model.{DET[scale]}", li, 255, conv.in_channels)
        assert np.abs(w - conv.weight.detach().numpy()).max() < 1e-5 and np.abs(b - conv.bias.detach().numpy()).max() < 1e-5
    stem = fused.model[1].conv
    w6 = np.zeros((stem.out_channels, 4, 6, 6), np.float32)
    w6[:, :3] = plan.reorg_stem_weights(stem.weight.detach().numpy())
    KR = 32
    packed = pb.tensors[pb.ops[0][1].w_tensor].astype(np.float32).reshape(stem.out_channels, 6, KR)[:, :, :24]
    assert np.array_equal(packed, np.transpose(w6, (0, 2, 3, 1)).reshape(stem.out_channels, 6, 24).astype(np.float16).astype(np.float32))


@pytest.mark.parametrize("scale", ["w6", "e6", "d6", "e6e"])
def test_oracle_fused_equals_training_form(scale):
    W = plan.synth_weights("yolov7", 1)
    plan.build_yolov7(W, scale, in_h=256, in_w=256)
    x = torch.rand(1, 3, 256, 256)
    with torch.no_grad():
        a = o6.build(W.state_dict, scale)(x).numpy()
        b = o6.build(W.state_dict, scale).fuse()(x).numpy()
    assert a.shape == (1, 3 * (32 * 32 + 16 * 16 + 8 * 8 + 4 * 4), 85)
    assert np.abs(a[..., 4:] - b[..., 4:]).max() < 1e-4
    assert np.abs(a[..., :4] - b[..., :4]).max() < 1e-4 * max(1.0, float(np.abs(a[..., :4]).max()))


def test_training_form_checkpoint_packs_its_main_path(tmp_path):
    """A training-form W6 checkpoint: IAuxDetect at model.122 with the aux level convs model.118 .. 121 before it and an `m2` list.  The
    main path keeps the deploy numbering, so the checkpoint packs by ignoring the aux keys and gives the deploy plan."""
    from adas_b200 import convert
    W = plan.synth_weights("yolov7", 6)
    ref = plan.build_yolov7(W, "w6", in_h=256, in_w=256)
    sd = {}
    for k, v in W.state_dict.items():
        sd[k.replace("model.118.", "model.122.")] = v
    rng = np.random.default_rng(0)
    for li, (c, src) in enumerate(((320, 128), (640, 256), (960, 384), (1280, 512))):
        sd[f"model.{118 + li}.conv.weight"] = rng.standard_normal((c, src, 3, 3)).astype(np.float32)
        sd[f"model.122.m2.{li}.weight"] = rng.standard_normal((255, c, 1, 1)).astype(np.float32)
    sd["model.122.anchor_grid"] = np.arange(1, 25, dtype=np.float32).reshape(4, 1, 3, 1, 1, 2)
    got = plan.build_yolov7(plan.Weights(sd), "w6", in_h=256, in_w=256)
    assert ref.ops == got.ops and all(np.array_equal(a, b) for a, b in zip(ref.tensors[:-1], got.tensors[:-1]))
    assert np.array_equal(got.tensors[got.meta[3] - 1], np.arange(1, 25, dtype=np.float32))
    ckpt = str(tmp_path / "w6.pth")
    torch.save({"model": {k: torch.from_numpy(np.asarray(v)) for k, v in W.state_dict.items()}}, ckpt)
    full = convert.plan_from_state_dict(convert.load_checkpoint_state_dict(ckpt), "yolov7", scale="w6")
    assert (full.in_h, full.in_w, len(full.outputs)) == (1280, 1280, 4)
    assert convert.main([ckpt, "--kind", "yolov7", "--scale", "w6", "--out", str(tmp_path / "w6.b200w")]) == 0
    assert plan.read_anchors(str(tmp_path / "w6.b200w")).shape == (4, 3, 2)


def _write(pb, tmp_path, name):
    p = tmp_path / f"{name}.b200w"
    pb.write(str(p))
    return p


@pytest.mark.skipif(torch.cuda.is_available(), reason="load-time validation is observed through the missing-device error")
def test_four_level_plan_validation(tmp_path):
    W = plan.synth_weights("yolov7", 0)
    pb = plan.build_yolov7(W, "w6", in_h=256, in_w=256)
    ok = _write(pb, tmp_path, "w6")
    assert "no CUDA device" in fp.engine_error(ok)
    assert np.array_equal(plan.read_anchors(str(ok)), np.asarray(plan.YOLOV7_P6_ANCHORS, np.float32).reshape(4, 3, 2))

    def bad(name, edit, expect):
        b = plan.build_yolov7(plan.Weights(W.state_dict), "w6", in_h=256, in_w=256)
        edit(b)
        err = fp.engine_error(_write(b, tmp_path, name))
        assert err is not None and expect in err, (name, err)

    bad("anchors18", lambda b: b.tensors.__setitem__(b.meta[3] - 1, np.ones(18, np.float32)), "anchor table")
    bad("no_anchors", lambda b: b.meta.__setitem__(3, 0), "needs its own anchor table")
    bad("lite", lambda b: b.meta.__setitem__(2, 1), "anchor table")
    bad("strides", lambda b: b.outputs.__setitem__(3, b.outputs[3][:3] + (128,)), "stride 128")
    bad("grid", lambda b: b.outputs.__setitem__(3, (b.outputs[2][0],) + b.outputs[3][1:]), "has stride 64 and a 8x8 grid")
    bad("meta1", lambda b: b.meta.__setitem__(1, b.meta[1] + 3), "levels hold 4080 anchors")
    # 4 levels on a YOLOv8, YOLOv6 or lite plan
    for name, b, expect in (("v8", plan.build_yolov8(plan.synth_weights("yolov8", 0), "n", in_h=256, in_w=256), "YOLOv8 head has 3 levels"),
                            ("v6", plan.build_yolov6(plan.synth_weights("yolov6", 0, variant="n"), "n", in_h=256, in_w=256), "YOLOv6 head has 3 levels"),
                            ("lite", plan.build_yolov5(plan.synth_weights("yolov5", 0), "n", in_h=256, in_w=256, lite=True), "4 without the lite flag")):
        assert "no CUDA device" in fp.engine_error(_write(b, tmp_path, name + "_ok"))
        b.outputs.append(b.outputs[-1][:3] + (64,))
        err = fp.engine_error(_write(b, tmp_path, name))
        assert err is not None and expect in err, (name, err)
    # stem conv widths: 80 and 96 are supported, 40 is not
    for cout, expect in ((80, "no CUDA device"), (96, "no CUDA device"), (40, "bad stem conv")):
        b = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, 64, 64)
        w = np.zeros((cout, 4, 6, 6), np.float32)
        b.stem_conv(b.image, w, np.zeros(cout, np.float32), 6, 2, 2, plan.ACT_SILU, b.new_padded(32, 32, (cout + 7) // 8 * 8))
        assert expect in fp.engine_error(_write(b, tmp_path, f"stem{cout}"))


def _export_p6(tmp_path, scale, seed, anchors=None, size=256):
    W = plan.synth_weights("yolov7", seed)
    ref = plan.build_yolov7(W, scale, in_h=size, in_w=size, anchors=anchors)
    path = str(tmp_path / f"{scale}.onnx")
    toi._export(o6.build(W.state_dict, scale, anchors=anchors).fuse(), (1, 3, size, size), path)
    return ref, path


@pytest.mark.parametrize("scale", ["w6", "e6", "d6", "e6e"])
def test_p6_onnx_round_trip(tmp_path, scale):
    """An export after upstream's fuse() (ReOrg as Slice / Concat, 4 detection convs) is recognised and packs the state_dict plan; E6
    carries custom anchors, which reach the plan through the export's anchor tensors."""
    anchors = tuple(tuple(float(v) * 1.25 for v in lvl) for lvl in o6.P6_ANCHORS) if scale == "e6" else None
    ref, path = _export_p6(tmp_path, scale, 7, anchors)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.act, spec.nc, spec.in_h, spec.in_w) == ("yolov7", scale, "silu", 80, 256, 256)
    assert onnx_import.reorg_slices(m, next(n for n in m.nodes if n.op_type == "Conv")) == [(0, 0), (1, 0), (0, 1), (1, 1)]
    assert len(onnx_import.OnnxWeights(m).convs) == onnx_import._P6_CONVS[scale]      # the count that tells E6 from E6E without names
    got = onnx_import.build_plan(m, spec)
    toi._assert_same_plan(ref, got, f"yolov7-{scale}")
    want = np.asarray(anchors or plan.YOLOV7_P6_ANCHORS, np.float32).reshape(24)
    assert np.array_equal(got.tensors[got.meta[3] - 1], want)


class _ReOrgNet(torch.nn.Module):
    """A ReOrg stem in a given slice order, Conv(12, c, 3), and `levels` detection convs."""
    def __init__(self, c, levels, order):
        super().__init__()
        self.order = order
        self.stem = torch.nn.Conv2d(12, c, 3, 1, 1)
        self.m = torch.nn.ModuleList(torch.nn.Conv2d(c, 255, 1) for _ in range(levels))

    def forward(self, x):
        y = torch.nn.functional.silu(self.stem(torch.cat([x[..., dy::2, dx::2] for dy, dx in self.order], 1)))
        outs = []
        for m in self.m:
            outs.append(m(y))
            y = torch.nn.functional.max_pool2d(y, 2, 2)
        return outs


@pytest.mark.parametrize("c,levels,order,match", [
    (64, 4, ((0, 0), (0, 1), (1, 0), (1, 1)), "not upstream's ReOrg"),      # columns before rows
    (48, 4, ((0, 0), (1, 0), (0, 1), (1, 1)), "P6 stem"),                   # no P6 model has a 48-channel stem
    (64, 3, ((0, 0), (1, 0), (0, 1), (1, 1)), "3 detection levels"),        # a ReOrg stem with a P5 head
])
def test_p6_recognition_guards(tmp_path, c, levels, order, match):
    path = str(tmp_path / "reorg.onnx")
    toi._export(_ReOrgNet(c, levels, order), (1, 3, 128, 128), path)
    with pytest.raises(Exception, match=match) as e:
        onnx_import.recognise(onnx_import.read_onnx(path))
    assert "YOLOv7 and YOLOv7-tiny" in str(e.value)
