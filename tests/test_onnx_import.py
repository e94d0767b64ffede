"""ONNX ingestion (adas_b200.onnx_import): the wire-format reader, the parameter matching rules and the architecture recognition,
checked on files written by torch's own exporter from the oracle networks (seeded weights) -- CPU only.

The plan built from the ONNX file must be the plan built from the state_dict: same ops, same buffers, same packed tensors (the
BatchNorm fold is done by the exporter in fp32 and by plan.Weights in fp64, so packed fp16 weights may differ by one ulp)."""
import os
import struct
import sys
import warnings

import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import onnx_import, plan

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import nets  # noqa: E402


def _export(model, shape, path):
    """torch.onnx.export (TorchScript exporter) without the `onnx` package: its only use there is splicing onnx-script functions."""
    from torch.onnx._internal.torchscript_exporter import onnx_proto_utils
    onnx_proto_utils._add_onnxscript_fn = lambda model_bytes, custom_opsets: model_bytes
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        torch.onnx.export(model.eval(), torch.zeros(*shape), path, opset_version=12, dynamo=False, input_names=["images"])


def _fuse_conv_bn(model):
    """What ultralytics / yolov5 do before exporting (fuse_conv_and_bn): BN folded into the conv, module names kept."""
    for m in model.modules():
        if isinstance(m, nets.Conv) and isinstance(m.bn, torch.nn.BatchNorm2d):
            w = m.conv.weight.detach().double()
            s = m.bn.weight.detach().double() / torch.sqrt(m.bn.running_var.detach().double() + m.bn.eps)
            fused = torch.nn.Conv2d(m.conv.in_channels, m.conv.out_channels, m.conv.kernel_size, m.conv.stride, m.conv.padding, bias=True)
            fused.weight.data = (w * s[:, None, None, None]).float()
            fused.bias.data = (m.bn.bias.detach().double() - m.bn.running_mean.detach().double() * s).float()
            m.conv, m.bn = fused, torch.nn.Identity()
    return model


def _assert_same_plan(pa, pb_, what):
    assert pa.ops == pb_.ops, f"{what}: op lists differ"
    assert pa.buffers == pb_.buffers and pa.outputs == pb_.outputs and list(pa.meta) == list(pb_.meta)
    assert len(pa.tensors) == len(pb_.tensors)
    worst = 0.0
    for ta, tb in zip(pa.tensors, pb_.tensors):
        assert ta.dtype == tb.dtype and ta.shape == tb.shape
        a, b = ta.astype(np.float64), tb.astype(np.float64)
        tol = 2.0 ** -10 * np.maximum(np.abs(a), np.abs(b)) + 1e-7        # one fp16 ulp (relative) / fp32 noise
        assert np.all(np.abs(a - b) <= tol), f"{what}: packed tensor differs by {np.abs(a - b).max()}"
        worst = max(worst, float(np.abs(a - b).max()))
    return worst


def test_wire_format_reader_on_a_hand_built_model(tmp_path):
    def vint(x):
        out = b""
        while True:
            b7 = x & 0x7F
            x >>= 7
            out += bytes([b7 | (0x80 if x else 0)])
            if not x:
                return out

    def ld(fno, payload):
        return vint((fno << 3) | 2) + vint(len(payload)) + payload

    def vi(fno, x):
        return vint(fno << 3) + vint(x & ((1 << 64) - 1))

    w = np.arange(2 * 3 * 1 * 1, dtype=np.float32).reshape(2, 3, 1, 1) - 2.5
    tensor_raw = b"".join(vi(1, d) for d in w.shape) + vi(2, 1) + ld(8, b"model.0.conv.weight") + ld(9, w.tobytes())
    bias = ld(1, vint(2)) + vi(2, 1) + ld(4, struct.pack("<2f", 0.5, -1.0)) + ld(8, b"model.0.conv.bias")    # packed dims + float_data
    attr = ld(1, b"strides") + ld(8, vint(2) + vint(2)) + vi(20, 7)
    attr_neg = ld(1, b"axis") + vi(3, -1)
    node = ld(1, b"images") + ld(1, b"model.0.conv.weight") + ld(1, b"model.0.conv.bias") + ld(2, b"y") + ld(3, b"/conv") + ld(4, b"Conv") + ld(5, attr) + ld(5, attr_neg)
    dim = lambda n: ld(1, vi(1, n))
    vinfo = ld(1, b"images") + ld(2, ld(1, vi(1, 1) + ld(2, dim(1) + dim(3) + dim(8) + dim(8))))
    graph = ld(1, node) + ld(2, b"g") + ld(5, tensor_raw) + ld(5, bias) + ld(11, vinfo) + ld(12, ld(1, b"y"))
    model = vi(1, 8) + ld(2, b"unit-test") + ld(7, graph) + ld(8, ld(1, b"") + vi(2, 12))
    p = tmp_path / "tiny.onnx"
    p.write_bytes(model)
    m = onnx_import.read_onnx(str(p))
    assert m.producer == "unit-test" and m.opset == 12
    assert [n.op_type for n in m.nodes] == ["Conv"] and m.nodes[0].inputs == ["images", "model.0.conv.weight", "model.0.conv.bias"]
    assert m.nodes[0].attrs == {"strides": [2, 2], "axis": -1}
    assert np.array_equal(m.initializers["model.0.conv.weight"], w)
    assert np.array_equal(m.initializers["model.0.conv.bias"], np.array([0.5, -1.0], np.float32))
    assert m.inputs == [("images", [1, 3, 8, 8])] and m.outputs[0][0] == "y"
    with pytest.raises(Exception):
        onnx_import.read_onnx(str(tmp_path / "missing.onnx"))


@pytest.mark.parametrize("kind,scale", [("yolov8", "n"), ("yolov5", "n")])
def test_yolo_fused_export_matches_state_dict_plan(tmp_path, kind, scale):
    """ultralytics-style file: Conv+BN fused in PyTorch before export, module names kept -> matched by name."""
    W = plan.synth_weights(kind, 3)
    build = plan.build_yolov8 if kind == "yolov8" else plan.build_yolov5
    ref = build(W, scale)
    model = _fuse_conv_bn(nets.build(kind, W.state_dict, scale=scale))
    path = str(tmp_path / f"{kind}{scale}.onnx")
    _export(model, (1, 3, 640, 640), path)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.nc, spec.in_h, spec.in_w) == (kind, scale, 80, 640, 640)
    w = onnx_import.OnnxWeights(m)
    got = build(w, scale)
    assert w.used_anonymous == 0
    worst = _assert_same_plan(ref, got, f"{kind}{scale} fused")
    print(f"[onnx] {kind}{scale} by-name plan: {len(got.ops)} ops, {len(got.tensors)} tensors, max packed |diff| {worst:.2e}")
    # the cached conversion writes a loadable plan file and reuses it
    out = onnx_import.plan_from_onnx(path, str(tmp_path / "cached.b200w"))
    assert open(out, "rb").read(8) == b"B200PLAN"
    t0 = os.path.getmtime(out)
    assert onnx_import.plan_from_onnx(path, out) == out and os.path.getmtime(out) == t0


def test_yolov5_exporter_folded_bn_is_matched_in_graph_order(tmp_path):
    """torch.onnx.export folds eval-mode BatchNorm itself: the folded tensors are anonymous and are taken in execution order."""
    W = plan.synth_weights("yolov5", 4)
    ref = plan.build_yolov5(W, "n")
    path = str(tmp_path / "v5n_unfused.onnx")
    _export(nets.build("yolov5", W.state_dict, scale="n"), (1, 3, 640, 640), path)
    m = onnx_import.read_onnx(path)
    w = onnx_import.OnnxWeights(m)
    got = plan.build_yolov5(w, "n")
    assert w.used_anonymous > 50
    _assert_same_plan(ref, got, "yolov5n exporter-folded")


def test_ufldv2_reference_style_export(tmp_path):
    """convertPytorchToONNX.py-style file: anonymous folded backbone convs (graph order) + named pool / LayerNorm / Linear tensors."""
    W = plan.synth_weights("ufldv2", 5)
    ref = plan.build_ufldv2(W, "18")
    path = str(tmp_path / "ufldv2_18.onnx")
    _export(nets.build("ufldv2", W.state_dict, backbone="18"), (1, 3, 320, 1600), path)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.in_h, spec.in_w) == ("ufldv2", "18", 320, 1600)
    assert len(m.outputs) == 4                       # ultrafastLaneDetectorV2.py:93-94 requires four outputs
    got = onnx_import.build_plan(m, spec)
    worst = _assert_same_plan(ref, got, "ufldv2-18")
    print(f"[onnx] ufldv2-18 plan from ONNX: {len(got.ops)} ops, max packed |diff| {worst:.2e}")
    os.remove(path)                                  # 0.8 GB (the 2048 -> 91224 classifier): do not leave it in the pytest tmp dir


def test_ufldv2_tusimple_export_is_recognised(tmp_path):
    """A TuSimple export (320x800 input, no LayerNorm before the classifier, 100x56 / 100x41 heads): the plan carries dataset id 1."""
    W = plan.synth_weights("ufldv2", 6)
    ref = plan.build_ufldv2(W, "18", "tusimple")
    cfg = {k: v for k, v in plan.UFLD_TUSIMPLE.items() if k not in ("dataset", "crop_ratio")}
    path = str(tmp_path / "tusimple_18.onnx")
    _export(nets.build("ufldv2", W.state_dict, backbone="18", **cfg), (1, 3, 320, 800), path)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.in_h, spec.in_w) == ("ufldv2", "18", 320, 800)
    got = onnx_import.build_plan(m, spec)
    assert got.meta[:7] == ref.meta[:7] and got.meta[6] == 1
    _assert_same_plan(ref, got, "ufldv2-18 tusimple")
    os.remove(path)


def test_wrong_architecture_is_reported(tmp_path):
    W = plan.synth_weights("yolov5", 6)
    plan.build_yolov5(W, "n")                     # materialises the seeded state_dict
    path = str(tmp_path / "v5n.onnx")
    _export(nets.build("yolov5", W.state_dict, scale="n"), (1, 3, 640, 640), path)
    m = onnx_import.read_onnx(path)
    with pytest.raises(Exception, match="expected a|no parameters left|expected"):
        plan.build_yolov5(onnx_import.OnnxWeights(m), "s")


def test_checkpoint_conversion_matches_seeded_plan(tmp_path):
    """convert.py on a reference-style checkpoint ({'model': state_dict} with DataParallel 'module.' prefixes,
    convertPytorchToONNX.py:77-84) and on an ONNX file, through the command-line entry point."""
    from adas_b200 import convert
    W = plan.synth_weights("yolov5", 7)
    ref = plan.build_yolov5(W, "n")
    ckpt = str(tmp_path / "v5n.pth")
    torch.save({"model": {"module." + k: torch.from_numpy(np.asarray(v)) for k, v in W.state_dict.items()}}, ckpt)
    sd = convert.load_checkpoint_state_dict(ckpt)
    assert set(sd) == set(W.state_dict)
    got = convert.plan_from_state_dict(sd, "yolov5", scale="n")
    assert ref.ops == got.ops and all(np.array_equal(a, b) for a, b in zip(ref.tensors, got.tensors))     # same fold -> identical bytes
    assert convert.main([ckpt, "--kind", "yolov5", "--scale", "n"]) == 0
    assert open(str(tmp_path / "v5n.b200w"), "rb").read(8) == b"B200PLAN"
    with pytest.raises(Exception, match="--kind is required"):
        convert.convert(ckpt)
    onnx_path = str(tmp_path / "v5n_fused.onnx")
    _export(_fuse_conv_bn(nets.build("yolov5", W.state_dict, scale="n")), (1, 3, 640, 640), onnx_path)
    out = convert.convert(onnx_path)
    assert out.endswith("v5n_fused.b200w") and os.path.getsize(out) > 1_000_000


def test_engine_accepts_onnx_path_and_fails_loudly_without_a_device(tmp_path, monkeypatch):
    """`B200Engine("model.onnx")` converts and caches the plan, then hands it to the C ABI; on a machine without an sm_90 device the library
    must raise (there is no CPU fallback on the product path)."""
    if torch.cuda.is_available():
        pytest.skip("needs a machine without a GPU")
    from adas_b200.coreEngine import B200Engine
    W = plan.synth_weights("yolov5", 8)
    plan.build_yolov5(W, "n")
    path = str(tmp_path / "v5n.onnx")
    _export(_fuse_conv_bn(nets.build("yolov5", W.state_dict, scale="n")), (1, 3, 640, 640), path)
    monkeypatch.setenv("ADAS_B200_PLAN_CACHE", str(tmp_path / "cache"))
    with pytest.raises(Exception) as ei:
        B200Engine(path, device=0)
    assert "onnx" not in str(ei.value).lower() or "cuda" in str(ei.value).lower()       # the failure is the device, not the conversion
    cached = os.listdir(str(tmp_path / "cache"))
    assert len(cached) == 1 and cached[0].startswith("v5n-") and cached[0].endswith(".b200w")
    with pytest.raises(Exception, match="can't not found"):
        B200Engine(str(tmp_path / "missing.onnx"))
    with pytest.raises(AssertionError):
        B200Engine(__file__)                           # wrong suffix: same assertion style as coreEngine.py:12-14


def test_truncated_or_foreign_files_are_rejected_cleanly(tmp_path):
    W = plan.synth_weights("yolov5", 9)
    plan.build_yolov5(W, "n")
    path = str(tmp_path / "v5n.onnx")
    _export(_fuse_conv_bn(nets.build("yolov5", W.state_dict, scale="n")), (1, 3, 640, 640), path)
    blob = open(path, "rb").read()
    rng = np.random.default_rng(0)
    for k, cut in enumerate([10, 1000, len(blob) // 3, len(blob) - 7]):
        p = tmp_path / f"cut{k}.onnx"
        p.write_bytes(blob[:cut])
        with pytest.raises(Exception):
            onnx_import.build_plan(onnx_import.read_onnx(str(p)))
    junk = tmp_path / "junk.onnx"
    junk.write_bytes(rng.integers(0, 256, 4096, dtype=np.uint8).tobytes())
    with pytest.raises(Exception):
        onnx_import.build_plan(onnx_import.read_onnx(str(junk)))
    with pytest.raises(Exception, match="can't not found"):
        onnx_import.read_onnx(str(tmp_path / "nope.onnx"))
