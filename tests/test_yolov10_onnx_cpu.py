"""CPU: YOLOv10 files -- ONNX recognition and packing with module names kept (fused before export) and lost (exporter-folded BatchNorm),
a file with upstream's top-k tail, the guards that keep YOLOv8 / YOLOv9 files what they are and still refuse YOLOv6-Lite, and the
refusals of out-of-scope YOLOv10 files.  ONNX files are written by torch's exporter from the oracle (tests/yolov10_oracle.py) at 320x320
to keep CPU time short."""
import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import onnx_import, plan
import test_onnx_import as toi
import yolov10_oracle as o10
import yolov9_oracle as o9


@pytest.mark.parametrize("names", ["kept", "lost"])
@pytest.mark.parametrize("scale", ["n", "s", "m", "b", "l", "x"])
def test_export_is_recognised_and_packs_the_state_dict_plan(tmp_path, scale, names):
    W = plan.synth_weights("yolov10", 3, variant=scale)
    ref = plan.build_yolov10(W, scale, in_h=320, in_w=320)
    model = o10.build(W.state_dict, scale)
    path = str(tmp_path / f"v10{scale}_{names}.onnx")
    toi._export(model.fuse() if names == "kept" else model, (1, 3, 320, 320), path)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.nc, spec.in_h, spec.in_w) == ("yolov10", scale, 80, 320, 320)
    got = onnx_import.build_plan(m, spec)
    assert onnx_import.OnnxWeights(m).convs[0][0].startswith("model.0.") == (names == "kept")
    toi._assert_same_plan(ref, got, f"yolov10-{scale} names {names}")


def _with_top_k_tail(m):
    """Upstream's end-to-end tail appended to the [1, 4 + nc, A] output (xyxy boxes, best class score and index of the top 300 anchors),
    with the module names of `m` unchanged."""
    net = m.forward

    def forward(x):
        y = net(x).transpose(1, 2)
        xy, wh, cls = y[..., :2], y[..., 2:4], y[..., 4:]
        xyxy = torch.cat((xy - wh / 2, xy + wh / 2), -1)
        score, idx = cls.max(-1)
        s, i = score.topk(300, dim=1)
        return torch.cat((xyxy.gather(1, i[..., None].expand(-1, -1, 4)), s[..., None], idx.gather(1, i)[..., None].float()), -1)

    m.forward = forward
    return m


@pytest.mark.parametrize("names", ["kept", "lost"])
def test_a_file_with_the_top_k_tail_packs_the_same_plan(tmp_path, names):
    W = plan.synth_weights("yolov10", 4, variant="s")
    ref = plan.build_yolov10(W, "s", in_h=320, in_w=320)
    model = o10.build(W.state_dict, "s")
    path = str(tmp_path / "v10s_topk.onnx")
    toi._export(_with_top_k_tail(model.fuse() if names == "kept" else model), (1, 3, 320, 320), path)
    m = onnx_import.read_onnx(path)
    assert len(m.outputs) == 1
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.nc) == ("yolov10", "s", 80)
    toi._assert_same_plan(ref, onnx_import.build_plan(m, spec), f"yolov10-s top-k tail, names {names}")


def test_yolov8_and_yolov9_exports_keep_their_kinds(tmp_path):
    W = plan.synth_weights("yolov8", 5)
    plan.build_yolov8(W, "s", in_h=320, in_w=320)
    path = str(tmp_path / "v8s.onnx")
    toi._export(toi._fuse_conv_bn(toi.nets.build("yolov8", W.state_dict, scale="s")), (1, 3, 320, 320), path)
    spec = onnx_import.recognise(onnx_import.read_onnx(path))
    assert (spec.kind, spec.scale) == ("yolov8", "s")
    W = plan.synth_weights("yolov9", 5, variant="t")
    plan.build_yolov9(W, "t", in_h=320, in_w=320)
    path = str(tmp_path / "v9t.onnx")
    toi._export(o9.build(W.state_dict, "t").fuse(), (1, 3, 320, 320), path)
    spec = onnx_import.recognise(onnx_import.read_onnx(path))
    assert (spec.kind, spec.scale) == ("yolov9", "t")


class _Small(torch.nn.Module):
    """A YOLOv10-like file: stem conv, a depthwise conv, a softmax, `n_1x1` further 1x1 convs; optionally a second output or a
    transposed conv (a YOLOv6-Lite-like file)."""
    def __init__(self, stem=16, n_1x1=4, two_outputs=False, transposed=False):
        super().__init__()
        self.stem = torch.nn.Conv2d(3, stem, 3, 2, 1)
        self.dw = torch.nn.Conv2d(stem, stem, 3, 1, 1, groups=stem)
        self.c = torch.nn.ModuleList(torch.nn.Conv2d(stem, stem, 1) for _ in range(n_1x1))
        self.up = torch.nn.ConvTranspose2d(stem, stem, 2, 2) if transposed else None
        self.two = two_outputs

    def forward(self, x):
        y = self.dw(self.stem(x))
        y = y * y.flatten(2).softmax(-1).view_as(y)
        for c in self.c:
            y = torch.relu(c(y))
        if self.up is not None:
            y = self.up(y)
        return (y, y + 1) if self.two else y


@pytest.mark.parametrize("kw,shape,what", [
    (dict(two_outputs=True), (1, 3, 64, 64), "outputs"),
    (dict(), (1, 3, 80, 80), "multiple of 32"),
    (dict(stem=24), (1, 3, 64, 64), "stem"),
    (dict(n_1x1=10), (1, 3, 64, 64), "convolutions"),
    # YOLOv10-N without names has 82 convolutions (83 with RepVGGDW's branches apart); 24 more are the one-to-many head
    (dict(n_1x1=plan.yolov10_conv_count("n") + 24 - 2), (1, 3, 64, 64), "one-to-many"),
])
def test_out_of_scope_yolov10_files_name_the_supported_variants(tmp_path, kw, shape, what):
    path = str(tmp_path / "bad.onnx")
    toi._export(_Small(**kw), shape, path)
    with pytest.raises(Exception, match="YOLOv10-N / S / M / B / L / X") as e:
        onnx_import.recognise(onnx_import.read_onnx(path))
    assert what in str(e.value)


def test_a_yolov6_lite_like_file_is_still_refused_by_the_yolov6_path(tmp_path):
    path = str(tmp_path / "lite.onnx")
    toi._export(_Small(transposed=True), (1, 3, 64, 64), path)
    with pytest.raises(Exception, match="YOLOv6-Lite"):
        onnx_import.recognise(onnx_import.read_onnx(path))


def test_conv_counts_match_the_packed_graphs():
    for sc in plan.YOLOV10_SCALES:
        pb = plan.build_yolov10(plan.synth_weights("yolov10", 0, variant=sc), sc, in_h=64, in_w=64)
        n = sum(1 for t, _, _ in pb.ops if t in (plan.OP_GEMM, plan.OP_DWCONV, plan.OP_STEMCONV))
        assert n == plan.yolov10_conv_count(sc), sc


def test_class_branch_wider_than_its_input_and_not_a_multiple_of_8():
    """nc = 70 on YOLOv10-N: c3 = max(64, 70) = 70 is stored as 72 channels; the depthwise weights, bias and the 1x1 rows past 70 are zero."""
    W = plan.synth_weights("yolov10", 0, variant="n")
    pb = plan.build_yolov10(W, "n", nc=70, in_h=320, in_w=320)
    assert pb.meta[:2] == [70, 2100] and all(o[2] == 64 + 72 for o in pb.outputs)
    dw72 = [p for t, p, _ in pb.ops if t == plan.OP_DWCONV and p.C == 72]
    assert len(dw72) == 3                                                  # one2one_cv3.i.1.0 per level
    for p in dw72:
        assert not pb.tensors[p.w_tensor][:, 70:].astype(np.float32).any() and not pb.tensors[p.bias_tensor][70:].any()
    # per level the 1x1 c3 -> c3 and c3 -> nc convs: 72 x 72 packed, zero past 70 rows and input channels
    gemms = [pb.tensors[p.w_tensor] for t, p, _ in pb.ops if t == plan.OP_GEMM and pb.tensors[p.w_tensor].shape == (72, 72)]
    assert len(gemms) == 6 and all(not g[70:].astype(np.float32).any() and not g[:, 70:].astype(np.float32).any() for g in gemms)
