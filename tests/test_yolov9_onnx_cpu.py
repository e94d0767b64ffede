"""CPU: YOLOv9 files -- ONNX recognition and packing with module names kept (fused before export) and lost (exporter-folded BatchNorm),
the guards that keep YOLOv8 files YOLOv8 and refuse out-of-scope YOLOv9 variants, and checkpoint conversion.  ONNX files are written by
torch's exporter from the oracle (tests/yolov9_oracle.py) at 320x320 to keep CPU time short."""
import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import onnx_import, plan
import test_onnx_import as toi
import yolov9_oracle as o9


@pytest.mark.parametrize("names", ["kept", "lost"])
@pytest.mark.parametrize("scale", ["t", "s", "m", "c"])
def test_export_is_recognised_and_packs_the_state_dict_plan(tmp_path, scale, names):
    W = plan.synth_weights("yolov9", 3, variant=scale)
    ref = plan.build_yolov9(W, scale, in_h=320, in_w=320)
    model = o9.build(W.state_dict, scale)
    path = str(tmp_path / f"v9{scale}_{names}.onnx")
    toi._export(model.fuse() if names == "kept" else model, (1, 3, 320, 320), path)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.nc, spec.in_h, spec.in_w) == ("yolov9", scale, 80, 320, 320)
    w = onnx_import.OnnxWeights(m)
    got = plan.build_yolov9(w, scale, in_h=320, in_w=320)
    assert (w.used_anonymous > 100) == (names == "lost")
    toi._assert_same_plan(ref, got, f"yolov9-{scale} names {names}")


def test_yolov8_exports_are_still_yolov8(tmp_path):
    W = plan.synth_weights("yolov8", 5)
    plan.build_yolov8(W, "s", in_h=320, in_w=320)
    path = str(tmp_path / "v8s.onnx")
    toi._export(toi._fuse_conv_bn(toi.nets.build("yolov8", W.state_dict, scale="s")), (1, 3, 320, 320), path)
    spec = onnx_import.recognise(onnx_import.read_onnx(path))
    assert (spec.kind, spec.scale) == ("yolov8", "s")


class _Small(torch.nn.Module):
    """A YOLOv9-like file: stem conv, 2x2 stride-1 average pool, `n_grouped` group-4 convs, optionally a second output."""
    def __init__(self, stem=16, n_grouped=6, two_outputs=False):
        super().__init__()
        self.stem = torch.nn.Conv2d(3, stem, 3, 2, 1)
        self.g = torch.nn.ModuleList(torch.nn.Conv2d(stem, stem, 3, 1, 1, groups=4) for _ in range(n_grouped))
        self.plain = torch.nn.Conv2d(stem, 64, 1)
        self.two = two_outputs

    def forward(self, x):
        y = torch.nn.functional.avg_pool2d(self.stem(x), 2, 1, 0)
        for g in self.g:
            y = torch.relu(g(y))
        return (self.plain(y), y) if self.two else self.plain(y)


@pytest.mark.parametrize("kw,shape,what", [
    (dict(stem=64), (1, 3, 64, 64), "convolutions"),                       # E-like: the C stem with another graph behind it
    (dict(n_grouped=0), (1, 3, 64, 64), "grouped"),                         # ultralytics' YOLOv9: a plain Detect head
    (dict(two_outputs=True), (1, 3, 64, 64), "outputs"),                    # the auxiliary branch's second output
    (dict(), (1, 3, 80, 80), "multiple of 32"),
])
def test_out_of_scope_yolov9_files_name_the_supported_variants(tmp_path, kw, shape, what):
    path = str(tmp_path / "bad.onnx")
    toi._export(_Small(**kw), shape, path)
    with pytest.raises(Exception, match="YOLOv9-T / S / M / C") as e:
        onnx_import.recognise(onnx_import.read_onnx(path))
    assert what in str(e.value)


@pytest.mark.parametrize("form", ["training", "fused"])
def test_checkpoint_conversion(tmp_path, form):
    from adas_b200 import convert
    W = plan.synth_weights("yolov9", 6, variant="t")
    ref = plan.build_yolov9(W, "t")
    sd = W.state_dict if form == "training" else {k: v.numpy() for k, v in o9.build(W.state_dict, "t").fuse().state_dict().items()}
    ckpt = str(tmp_path / f"v9t_{form}.pth")
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, ckpt)
    got = convert.plan_from_state_dict(convert.load_checkpoint_state_dict(ckpt), "yolov9", scale="t")
    toi._assert_same_plan(ref, got, f"yolov9-t {form} checkpoint")
    assert convert.main([ckpt, "--kind", "yolov9", "--scale", "t", "--out", str(tmp_path / "v9t.b200w")]) == 0
