"""GPU: YOLOv7 / YOLOv7-tiny on the device -- the LeakyReLU(0.1) epilogue of every conv kernel, the stride-1 direct image stem, and
both networks end to end against the fp32 oracle (tests/yolov7_oracle.py) with the plan-carried anchor table."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
from gpu_util import cached_plan, from_padded, halo_is_zero, to_padded, yolo_blob
from oracle import post
import yolov7_oracle as o7

pytestmark = pytest.mark.gpu
torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))


def _leaky(t):
    return F.leaky_relu(t, 0.1)


def _run_leaky_conv(tmp_path, impl, B, cin, cout, H, W, k, s, residual=None, tile=None, no_slab=False, seed=0):
    """One LeakyReLU conv through the C ABI against torch on the fp16-rounded operands; returns (relative error, output buffer)."""
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
    xin = pb.new_padded(H, W, cin)
    w = (rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
    b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    pd = k // 2
    Ho, Wo = (H + 2 * pd - k) // s + 1, (W + 2 * pd - k) // s + 1
    res_view = pb.new_padded(Ho, Wo, cout) if residual else None
    out = pb.conv(xin, w, b, k, s, plan.ACT_LEAKY, res=res_view, res_pre_act=(residual == "pre"), tile=tile, no_slab=no_slab)
    path = str(tmp_path / f"leaky_{impl}_{seed}_{int(no_slab)}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, device=0, max_batch=B, conv_impl=impl)
    x = rng.standard_normal((B, cin, H, W)).astype(np.float32)
    eng.write_buffer(xin.buf, to_padded(x, cin))
    r = None
    if residual:
        r = rng.standard_normal((B, cout, Ho, Wo)).astype(np.float32)
        eng.write_buffer(res_view.buf, to_padded(r, cout))
    for _ in range(3):          # eager, graph capture, graph replay
        eng.run(B)
    got_buf = eng.read_buffer(out.buf, B).copy()
    got = from_padded(got_buf, B, Ho, Wo, out.coff, cout)
    ref = F.conv2d(torch.from_numpy(x).half().float(), torch.from_numpy(w).half().float(), torch.from_numpy(b), stride=s, padding=pd)
    rt = torch.from_numpy(r).half().float() if residual else None
    ref = _leaky(ref + rt if residual == "pre" else ref)
    if residual == "post":
        ref = ref + rt
    ref = ref.numpy()
    assert halo_is_zero(got_buf, B, Ho, Wo), "conv wrote into the zero halo"
    eng.close()
    return float(np.abs(got - ref).max()) / max(1.0, float(np.abs(ref).max())), got_buf


LEAKY_CASES = [
    # B cin cout H W k s residual
    (2, 192, 64, 17, 23, 1, 1, None),          # 1x1, K tail, ragged M
    (2, 64, 128, 20, 24, 3, 1, None),          # 3x3 taps, one k-block
    (1, 128, 256, 40, 40, 3, 1, "post"),       # 3x3, two k-blocks, residual after the activation
    (2, 256, 128, 12, 52, 3, 1, "pre"),        # residual before the activation
    (2, 64, 128, 32, 48, 3, 2, None),          # stride 2 through the strided TMA map
    (1, 128, 256, 20, 28, 1, 2, None),         # 1x1 stride 2
    (1, 32, 64, 40, 40, 3, 1, None),           # 32-channel 3x3 (YOLOv7-tiny): im2col + GEMM
    (1, 32, 64, 40, 40, 3, 2, None),           # 32-channel stride-2 3x3 (YOLOv7 layer 1)
]


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("case", LEAKY_CASES)
def test_leaky_conv_parity(tmp_path, impl, case):
    B, cin, cout, H, W, k, s, residual = case
    err, _ = _run_leaky_conv(tmp_path, impl, B, cin, cout, H, W, k, s, residual, seed=cin + cout + k)
    assert err < 4e-3, f"impl {impl} case {case}: relative error {err}"


LEAKY_TILES = [
    # (B cin cout H W k s residual), (BN, MT)
    ((2, 256, 256, 40, 40, 3, 1, "post"), (256, 1)),
    ((2, 256, 256, 40, 40, 3, 1, None), (128, 2)),
    ((2, 128, 128, 48, 80, 3, 1, "pre"), (128, 4)),
    ((1, 256, 320, 40, 40, 3, 1, None), (160, 1)),
    ((2, 256, 512, 40, 40, 3, 2, None), (128, 2)),
    ((2, 320, 128, 80, 80, 1, 1, None), (128, 3)),
    ((2, 64, 80, 20, 20, 1, 1, None), (80, 1)),
]


@pytest.mark.parametrize("case,tile", LEAKY_TILES)
def test_leaky_conv_tiles_slab_and_per_tap(tmp_path, case, tile):
    """Each (BN, MT) tile, and for 3x3 stride-1 convs slab mode against one activation tile per tap: same bits."""
    B, cin, cout, H, W, k, s, residual = case
    seed = cin + cout + tile[0] + tile[1]
    err, slab = _run_leaky_conv(tmp_path, 0, B, cin, cout, H, W, k, s, residual, tile=tile, seed=seed)
    assert err < 4e-3, (case, tile, err)
    if k == 3 and s == 1:
        err2, tap = _run_leaky_conv(tmp_path, 0, B, cin, cout, H, W, k, s, residual, tile=tile, no_slab=True, seed=seed)
        assert np.array_equal(slab.view(np.uint16), tap.view(np.uint16))


@pytest.mark.parametrize("cout,act", [(16, 1), (32, 3), (48, 0), (64, 3), (32, 1), (16, 3)])
def test_stem_conv_direct_stride1(tmp_path, cout, act):
    """stem_conv.cu at stride 1 (YOLOv7's Conv(3, 32, 3, 1) at full resolution): every supported Cout, LeakyReLU, widths that are not a
    multiple of the 16-pixel warp tile, batch > 1; frame 0 alone gives the same bits."""
    rng = np.random.default_rng(200 + cout + act)
    for (B, H, W) in ((2, 64, 96), (3, 36, 50)):
        pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
        w = (rng.standard_normal((cout, 3, 3, 3)) * np.sqrt(2.0 / 27)).astype(np.float32)
        b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
        out = pb.conv(pb.image, w, b, 3, 1, act)
        assert [op[0] for op in pb.ops] == [plan.OP_STEMCONV] and pb.ops[0][1].stride == 1
        path = str(tmp_path / f"stem1_{cout}_{act}_{H}.b200w")
        pb.write(path)
        eng = _capi.Engine(path, 0, max_batch=B)
        x = rng.standard_normal((B, 3, H, W)).astype(np.float32)
        eng.write_buffer(pb.image.buf, to_padded(x, 4))
        for _ in range(3):
            eng.run(B)
        got_buf = eng.read_buffer(out.buf, B).copy()
        got = from_padded(got_buf, B, H, W, 0, cout)
        ref = F.conv2d(torch.from_numpy(x).half().float(), torch.from_numpy(w).half().float(), torch.from_numpy(b), stride=1, padding=1)
        ref = {0: lambda t: t, 1: F.silu, 3: _leaky}[act](ref).numpy()
        err = float(np.abs(got - ref).max()) / max(1.0, float(np.abs(ref).max()))
        assert err < 2e-3, (cout, act, H, err)
        assert halo_is_zero(got_buf, B, H, W)
        eng1 = _capi.Engine(path, 0, max_batch=1)
        eng1.write_buffer(pb.image.buf, to_padded(x[:1], 4))
        eng1.run(1)
        assert np.array_equal(eng1.read_buffer(out.buf, 1), got_buf[:got_buf.shape[0] // B])
        eng1.close(); eng.close()


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("scale", ["tiny", "base"])
def test_yolov7_engine_vs_oracle_and_batch_invariance(scale, impl):
    path, sd, _ = cached_plan("yolov7", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=3, conv_impl=impl)
    x = yolo_blob([synth.frame(s) for s in (0, 1, 2)])
    raw = eng.infer(x)[0]
    with torch.no_grad():
        ref = o7.build(sd, scale)(torch.from_numpy(x[:2])).numpy()
    assert raw.shape == (3, 25200, 85)
    e_prob = float(np.abs(raw[:2, :, 4:] - ref[..., 4:]).max())
    e_box = float(np.abs(raw[:2, :, :4] - ref[..., :4]).max())
    print(f"[parity] yolov7-{scale} impl{impl}: prob {e_prob:.2e}, box {e_box:.3f} px")
    assert e_prob < 1e-3          # float scores within 1e-3 of the fp32 oracle
    assert e_box < 0.5            # boxes within half a pixel of the 640-px input
    raw1 = eng.infer(x[1:2])[0]
    assert np.array_equal(raw1[0], raw[1]), "batch-1 frame differs from the same frame in a batch of 3"
    eng.close()


@pytest.mark.parametrize("scale", ["tiny", "base"])
def test_yolov7_fused_detect_matches_reference_postprocessing(scale):
    path, sd, _ = cached_plan("yolov7", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=4)
    frames = np.stack([synth.frame(s) for s in (4, 5, 6, 7)])
    boxes, scores, cls, idx, counts, ncand = eng.yolo_detect(frames, 0.4, 0.45, max_det=1024)
    x = _capi.yolo_preprocess(frames, (640, 640))
    raw = eng.infer(x)[0]
    geom = post.letterbox_geom(720, 1280, 640, 640)
    for b in range(4):
        r = post.yolo_postprocess(raw[b], "v5", geom, 0.4, 0.45)     # the reference's v5/v6/v7 host post-processing
        n = int(counts[b])
        assert ncand[b] == r["n_cand"] and np.array_equal(idx[b, :n], r["idx"]) and np.array_equal(boxes[b, :n], r["boxes"])
        assert np.array_equal(scores[b, :n], r["scores"]) and np.array_equal(cls[b, :n], r["cls"])
    with torch.no_grad():
        ref = o7.build(sd, scale)(torch.from_numpy(x)).numpy()
    n_cand = n_margin = 0
    for b in range(4):
        mx_ref, mx_gpu = (ref[b, :, 5:] * ref[b, :, 4:5]).max(1), (raw[b, :, 5:] * raw[b, :, 4:5]).max(1)
        sure = np.abs(mx_ref - 0.4) > 1e-3
        cand = mx_ref > 0.4
        assert np.array_equal(cand[sure], (mx_gpu > 0.4)[sure])
        assert np.abs(mx_ref[cand] - mx_gpu[cand]).max(initial=0.0) < 1e-3
        n_cand += int(cand.sum())
        n_margin += int((~sure & (cand | (mx_gpu > 0.4))).sum())
    print(f"[parity] yolov7-{scale} candidates: {n_cand} over 4 frames, {n_margin} inside the 1e-3 margin, detections {counts.tolist()}")
    # the tiny net's LeakyReLU activations carry far more fp16 noise at the head than the SiLU nets (plan.SYNTH_PROFILES): its head gain
    # is small, its scores crowd the threshold, and ~15 % of its candidates sit inside the 1e-3 margin (CPU fp16 emulation)
    assert n_cand > 50 and n_margin <= (0.05 if scale == "base" else 0.20) * n_cand
    eng.close()


def test_yolo_detector_runs_a_yolov7_onnx_file(tmp_path):
    """YoloDetector(ObjectModelType.YOLOV7) on an exported .onnx file: converted, loaded and decoded with the plan's anchors."""
    import test_onnx_import as toi
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    W = plan.synth_weights("yolov7", 0)
    plan.build_yolov7(W, "tiny")
    onnx_path = str(tmp_path / "yolov7-tiny.onnx")
    toi._export(o7.build(W.state_dict, "tiny").fuse(), (1, 3, 640, 640), onnx_path)
    os.environ["ADAS_B200_PLAN_CACHE"] = str(tmp_path / "cache")
    try:
        YoloDetector.set_defaults({"model_path": onnx_path, "model_type": ObjectModelType.YOLOV7, "classes_path": None, "box_score": 0.4,
                                   "box_nms_iou": 0.45})
        det = YoloDetector(logger=None, max_batch=2)
    finally:
        os.environ.pop("ADAS_B200_PLAN_CACHE", None)
    out = det.engine.engine_inference(yolo_blob([synth.frame(3)]))
    assert out[0].shape == (1, 25200, 85)
    fr = [synth.frame(3), synth.frame(4)]
    det.DetectFrame(fr[0])
    single = [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in det.object_info]
    both = det.DetectFrames(fr)
    assert single == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]
    boxes, scores, cls, idx, counts, _ = det.engine.handle.yolo_detect(np.stack(fr), 0.4, 0.45, 1024)
    n = int(counts[0])
    assert n > 0 and [(r.conf, r.label) for r in det.object_info] == [(float(scores[0, i]), f"class{int(cls[0, i])}") for i in range(n)]
