"""CPU: YOLOv6 files -- ONNX recognition and packing, the per-conv activation check, the guards that keep YOLOv8 / YOLOv7 files and
out-of-scope YOLOv6 variants where they belong, and checkpoint conversion.  ONNX files are written by torch's exporter from the fused
oracle (tests/yolov6_oracle.py) at 320x320 to keep CPU time short."""
import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import onnx_import, plan
import test_onnx_import as toi
import yolov6_oracle as o6
import yolov7_oracle as o7


def _export_v6(tmp_path, scale, seed, name, model_fn=None):
    W = plan.synth_weights("yolov6", seed)
    ref = plan.build_yolov6(W, scale, in_h=320, in_w=320)
    model = o6.build(W.state_dict, scale).fuse()
    if model_fn is not None:
        model_fn(model)
    path = str(tmp_path / f"{name}.onnx")
    toi._export(model, (1, 3, 320, 320), path)
    return W, ref, path


@pytest.mark.parametrize("scale", ["n", "s", "m", "l"])
def test_fused_export_is_recognised_and_packs_the_state_dict_plan(tmp_path, scale):
    W, ref, path = _export_v6(tmp_path, scale, 3, f"v6{scale}")
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    reg_max = 16 if scale in "ml" else 0
    assert (spec.kind, spec.scale, spec.nc, spec.reg_max, spec.in_h, spec.in_w) == ("yolov6", scale, 80, reg_max, 320, 320)
    assert spec.acts == (("silu" if scale == "l" else "relu"), "relu", "silu")
    got = onnx_import.build_plan(m, spec)
    toi._assert_same_plan(ref, got, f"yolov6-{scale}")


def test_yolov8_exports_are_still_yolov8(tmp_path):
    for scale in ("n", "s"):
        W = plan.synth_weights("yolov8", 5)
        plan.build_yolov8(W, scale, in_h=320, in_w=320)
        path = str(tmp_path / f"v8{scale}.onnx")
        toi._export(toi._fuse_conv_bn(toi.nets.build("yolov8", W.state_dict, scale=scale)), (1, 3, 320, 320), path)
        spec = onnx_import.recognise(onnx_import.read_onnx(path))
        assert (spec.kind, spec.scale) == ("yolov8", scale)


def test_yolov7_tiny_export_is_still_yolov7(tmp_path):
    W = plan.synth_weights("yolov7", 3)
    plan.build_yolov7(W, "tiny", in_h=320, in_w=320)
    path = str(tmp_path / "v7t.onnx")
    toi._export(o7.build(W.state_dict, "tiny").fuse(), (1, 3, 320, 320), path)
    spec = onnx_import.recognise(onnx_import.read_onnx(path))
    assert (spec.kind, spec.scale) == ("yolov7", "tiny")


class _Lite(torch.nn.Module):
    """A YOLOv6-Lite-like file: depthwise convs and a transposed-conv upsample."""
    def __init__(self):
        super().__init__()
        self.stem = torch.nn.Conv2d(3, 16, 3, 2, 1)
        self.dw = torch.nn.Conv2d(16, 16, 3, 1, 1, groups=16)
        self.up = torch.nn.ConvTranspose2d(16, 16, 2, 2)

    def forward(self, x):
        return self.up(torch.relu(self.dw(torch.relu(self.stem(x)))))


class _P6(torch.nn.Module):
    """A P6-like head: four levels of detect.cls_preds / reg_preds behind a transposed conv."""
    def __init__(self):
        super().__init__()
        self.stem = torch.nn.Conv2d(3, 16, 3, 2, 1)
        self.up = torch.nn.ConvTranspose2d(16, 16, 2, 2)
        self.detect = torch.nn.Module()
        self.detect.cls_preds = torch.nn.ModuleList(torch.nn.Conv2d(16, 80, 1) for _ in range(4))
        self.detect.reg_preds = torch.nn.ModuleList(torch.nn.Conv2d(16, 4, 1) for _ in range(4))

    def forward(self, x):
        y = self.up(torch.relu(self.stem(x)))
        return [c(y) for c in self.detect.cls_preds] + [r(y) for r in self.detect.reg_preds]


@pytest.mark.parametrize("cls,what", [(_Lite, "YOLOv6-Lite"), (_P6, "P6")])
def test_out_of_scope_yolov6_files_name_the_supported_variants(tmp_path, cls, what):
    path = str(tmp_path / f"{what}.onnx")
    toi._export(cls(), (1, 3, 64, 64), path)
    with pytest.raises(Exception, match="YOLOv6-N / S / M / L") as e:
        onnx_import.recognise(onnx_import.read_onnx(path))
    assert what in str(e.value)


def test_altered_activation_is_rejected_naming_the_conv(tmp_path):
    """One neck reduce layer switched from ReLU to SiLU: the file is refused and the message names that convolution."""
    def alter(model):
        model.neck.reduce_layer1.block.act = torch.nn.SiLU()
    _, _, path = _export_v6(tmp_path, "n", 4, "v6n_altered", alter)
    with pytest.raises(Exception, match=r"neck\.reduce_layer1\.block\.conv\.weight"):
        onnx_import.recognise(onnx_import.read_onnx(path))


@pytest.mark.parametrize("form", ["training", "deployed"])
def test_checkpoint_conversion(tmp_path, form):
    from adas_b200 import convert
    W = plan.synth_weights("yolov6", 6)
    ref = plan.build_yolov6(W, "m")
    sd = W.state_dict if form == "training" else {k: v.numpy() for k, v in o6.build(W.state_dict, "m").fuse().state_dict().items()}
    ckpt = str(tmp_path / f"v6m_{form}.pth")
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, ckpt)
    got = convert.plan_from_state_dict(convert.load_checkpoint_state_dict(ckpt), "yolov6", scale="m")
    toi._assert_same_plan(ref, got, f"yolov6-m {form} checkpoint")
    assert convert.main([ckpt, "--kind", "yolov6", "--scale", "m", "--out", str(tmp_path / "v6m.b200w")]) == 0
