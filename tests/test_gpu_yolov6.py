"""GPU: YOLOv6 on the device -- the 2x2 transposed-conv store and the scaled residual of both GEMM epilogues, and YOLOv6-N/S/M/L end to
end against the fp32 oracle (tests/yolov6_oracle.py) through the anchor-free v6 head decode."""
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
import yolov6_oracle as o6

pytestmark = pytest.mark.gpu
torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))


def _run_transpose(tmp_path, impl, B, cout, H, W, coff, tile=None, seed=0):
    """ConvTranspose2d(cout, cout, 2, 2) of an H x W map into channels [coff, coff + cout) of a 2H x 2W buffer; returns (error, buffer)."""
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV6, 3, 2 * H, 2 * W)
    xin = pb.new_padded(H, W, cout)
    cat = pb.new_padded(2 * H, 2 * W, coff + cout + 8)
    w = (rng.standard_normal((cout, cout, 2, 2)) * np.sqrt(1.0 / cout)).astype(np.float32)
    b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    pb.conv_transpose2x2(xin, w, b, pb.sub(cat, coff, cout), tile=tile)
    path = str(tmp_path / f"tr_{impl}_{cout}_{H}_{seed}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, device=0, max_batch=B, conv_impl=impl)
    x = rng.standard_normal((B, cout, H, W)).astype(np.float32)
    eng.write_buffer(xin.buf, to_padded(x, cout))
    for _ in range(3):
        eng.run(B)
    buf = eng.read_buffer(cat.buf, B).copy()
    eng.close()
    got = from_padded(buf, B, 2 * H, 2 * W, coff, cout)
    ref = F.conv_transpose2d(torch.from_numpy(x).half().float(), torch.from_numpy(w).half().float(), torch.from_numpy(b), stride=2).numpy()
    assert halo_is_zero(buf, B, 2 * H, 2 * W), "transposed conv wrote into the zero halo"
    other = buf.reshape(B, 2 * H + 2, 2 * W + 2, -1).astype(np.float32)
    assert not other[..., :coff].any() and not other[..., coff + cout:].any(), "transposed conv wrote outside its channel slice"
    return float(np.abs(got - ref).max()) / max(1.0, float(np.abs(ref).max())), buf


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("cout,H,W,coff", [(16, 13, 21, 0), (32, 20, 20, 16), (64, 10, 30, 64), (128, 20, 20, 128), (256, 7, 9, 256)])
def test_transposed_store_matches_torch(tmp_path, impl, cout, H, W, coff):
    err, _ = _run_transpose(tmp_path, impl, 2, cout, H, W, coff, seed=cout + H)
    assert err < 2e-3, (impl, cout, H, W, err)


@pytest.mark.parametrize("cout,tile", [(64, (64, 1)), (64, (128, 3)), (128, (256, 1)), (256, (128, 4)), (32, (128, 2))])
def test_transposed_store_tiles_are_bit_identical(tmp_path, cout, tile):
    _, ref = _run_transpose(tmp_path, 0, 2, cout, 20, 20, 8, seed=7)
    _, got = _run_transpose(tmp_path, 0, 2, cout, 20, 20, 8, tile=tile, seed=7)
    assert np.array_equal(ref.view(np.uint16), got.view(np.uint16)), tile


def _run_scaled_residual(tmp_path, impl, alpha, k=3, cin=64, cout=64, B=2, H=18, W=26, seed=0):
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV6, 3, H, W)
    xin = pb.new_padded(H, W, cin)
    res = pb.new_padded(H, W, cout)
    w = (rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
    b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    out = pb.conv(xin, w, b, k, 1, plan.ACT_RELU, res=res, res_scale=alpha)
    path = str(tmp_path / f"rs_{impl}_{alpha}_{seed}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, device=0, max_batch=B, conv_impl=impl)
    x = rng.standard_normal((B, cin, H, W)).astype(np.float32)
    r = rng.standard_normal((B, cout, H, W)).astype(np.float32)
    eng.write_buffer(xin.buf, to_padded(x, cin))
    eng.write_buffer(res.buf, to_padded(r, cout))
    for _ in range(3):
        eng.run(B)
    buf = eng.read_buffer(out.buf, B).copy()
    eng.close()
    got = from_padded(buf, B, H, W, 0, cout)
    ref = F.relu(F.conv2d(torch.from_numpy(x).half().float(), torch.from_numpy(w).half().float(), torch.from_numpy(b), padding=k // 2))
    ref = (ref + (alpha if alpha is not None else 1.0) * torch.from_numpy(r).half().float()).numpy()
    return float(np.abs(got - ref).max()) / max(1.0, float(np.abs(ref).max())), buf


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("alpha", [0.7, 1.3])
def test_scaled_residual_matches_torch(tmp_path, impl, alpha):
    err, _ = _run_scaled_residual(tmp_path, impl, alpha, seed=int(alpha * 10))
    assert err < 3e-3, (impl, alpha, err)


@pytest.mark.parametrize("impl", [1, 0])
def test_residual_scale_one_is_the_plain_residual(tmp_path, impl):
    for k in (1, 3):
        _, a = _run_scaled_residual(tmp_path, impl, 1.0, k=k, seed=3)
        _, b = _run_scaled_residual(tmp_path, impl, None, k=k, seed=3)
        assert np.array_equal(a.view(np.uint16), b.view(np.uint16)), k


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("scale", ["n", "s", "m", "l"])
def test_yolov6_engine_vs_oracle_and_batch_invariance(scale, impl):
    path, sd, _ = cached_plan("yolov6", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=3, conv_impl=impl)
    x = yolo_blob([synth.frame(s) for s in (0, 1, 2)])
    raw = eng.infer(x)[0]
    with torch.no_grad():
        ref = o6.build(sd, scale)(torch.from_numpy(x[:2])).numpy()
    assert raw.shape == (3, 8400, 85)
    assert np.all(raw[..., 4] == 1.0)
    e_prob = float(np.abs(raw[:2, :, 5:] - ref[..., 5:]).max())
    e_box = float(np.abs(raw[:2, :, :4] - ref[..., :4]).max())
    print(f"[parity] yolov6-{scale} impl{impl}: prob {e_prob:.2e}, box {e_box:.3f} px")
    assert e_prob < 1e-3
    assert e_box < 0.5
    raw1 = eng.infer(x[1:2])[0]
    assert np.array_equal(raw1[0], raw[1]), "batch-1 frame differs from the same frame in a batch of 3"
    eng.close()


@pytest.mark.parametrize("scale", ["n", "m"])
def test_yolov6_fused_detect_matches_reference_postprocessing(scale):
    """The device decode + candidate selection + NMS equals the reference's v5/v6/v7 host post-processing of the engine's own output."""
    path, _, _ = cached_plan("yolov6", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=2)
    frames = np.stack([synth.frame(s) for s in (4, 5)])
    for score in (0.4, 0.05):
        boxes, scores, cls, idx, counts, ncand = eng.yolo_detect(frames, score, 0.45, max_det=8400)
        raw = eng.infer(_capi.yolo_preprocess(frames, (640, 640)))[0]
        geom = post.letterbox_geom(720, 1280, 640, 640)
        for b in range(2):
            r = post.yolo_postprocess(raw[b], "v5", geom, score, 0.45)
            n = int(counts[b])
            assert ncand[b] == r["n_cand"] and np.array_equal(idx[b, :n], r["idx"]) and np.array_equal(boxes[b, :n], r["boxes"])
            assert np.array_equal(scores[b, :n], r["scores"]) and np.array_equal(cls[b, :n], r["cls"])
        print(f"[detect] yolov6-{scale} score {score}: candidates {ncand.tolist()}, detections {counts.tolist()}")
    eng.close()


@pytest.mark.parametrize("scale", ["n", "s", "m", "l"])
def test_yolov6_candidate_sets_follow_the_margin_rule(scale):
    """Candidates (max class probability > 0.4) agree with the fp32 oracle's wherever the oracle's score is more than 1e-3 from the
    threshold, and few of them sit inside that margin."""
    path, sd, _ = cached_plan("yolov6", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=4)
    x = yolo_blob([synth.frame(s) for s in (4, 5, 6, 7)])
    raw = eng.infer(x)[0]
    eng.close()
    with torch.no_grad():
        ref = o6.build(sd, scale)(torch.from_numpy(x)).numpy()
    n_cand = n_margin = 0
    for b in range(4):
        mx_ref, mx_gpu = (ref[b, :, 5:] * ref[b, :, 4:5]).max(1), (raw[b, :, 5:] * raw[b, :, 4:5]).max(1)
        sure = np.abs(mx_ref - 0.4) > 1e-3
        cand = mx_ref > 0.4
        assert np.array_equal(cand[sure], (mx_gpu > 0.4)[sure])
        assert np.abs(mx_ref[cand] - mx_gpu[cand]).max(initial=0.0) < 1e-3
        n_cand += int(cand.sum())
        n_margin += int((~sure & (cand | (mx_gpu > 0.4))).sum())
    print(f"[margin] yolov6-{scale}: {n_cand} candidates over 4 frames, {n_margin} inside the 1e-3 margin")
    # ~100 candidates per frame (plan.SYNTH_PROFILES["yolov6"]).  The share inside the margin measures how densely the synthetic scores
    # crowd the threshold, not the error: a random head's per-anchor max-class logits spread by only 0.13-0.24 (L least), and widening
    # them with the head gain widens the fp16 error in proportion.  Measured on the H100: N 27 %, S 6 %, M 29 %, L 57 %.
    assert 200 <= n_cand <= 800 and n_margin <= {"n": 0.35, "s": 0.10, "m": 0.35, "l": 0.65}[scale] * n_cand


def test_yolo_detector_runs_a_yolov6_onnx_file(tmp_path):
    """YoloDetector(ObjectModelType.YOLOV6) on an exported YOLOv6-N .onnx file: recognised, converted, loaded and decoded."""
    import test_onnx_import as toi
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    W = plan.synth_weights("yolov6", 0, variant="n")
    plan.build_yolov6(W, "n")
    onnx_path = str(tmp_path / "yolov6n.onnx")
    toi._export(o6.build(W.state_dict, "n").fuse(), (1, 3, 640, 640), onnx_path)
    os.environ["ADAS_B200_PLAN_CACHE"] = str(tmp_path / "cache")
    try:
        YoloDetector.set_defaults({"model_path": onnx_path, "model_type": ObjectModelType.YOLOV6, "classes_path": None, "box_score": 0.4,
                                   "box_nms_iou": 0.45})
        det = YoloDetector(logger=None, max_batch=2)
    finally:
        os.environ.pop("ADAS_B200_PLAN_CACHE", None)
    assert det.engine.handle.model_kind == plan.MODEL_YOLOV6
    out = det.engine.engine_inference(yolo_blob([synth.frame(3)]))
    assert out[0].shape == (1, 8400, 85)
    fr = [synth.frame(3), synth.frame(4)]
    det.DetectFrame(fr[0])
    single = [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in det.object_info]
    both = det.DetectFrames(fr)
    assert len(single) > 0 and single == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]


def test_model_type_pairing_for_yolov6_plans(tmp_path):
    """The detector's existing pairing rule: a kind-5 plan runs as YOLOV5 / YOLOV6 / YOLOV7 and is refused for YOLOV5_LITE and the v8 layout."""
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    path, _, _ = cached_plan("yolov6", scale="n")
    for mt, ok in ((ObjectModelType.YOLOV6, True), (ObjectModelType.YOLOV5, True), (ObjectModelType.YOLOV7, True),
                   (ObjectModelType.YOLOV5_LITE, False), (ObjectModelType.YOLOV8, False), (ObjectModelType.YOLOV10, False)):
        YoloDetector.set_defaults({"model_path": path, "model_type": mt, "classes_path": None, "box_score": 0.4, "box_nms_iou": 0.45})
        if ok:
            det = YoloDetector(logger=None)
            det.DetectFrame(synth.frame(3))
            assert det.engine.handle.model_kind == plan.MODEL_YOLOV6
        else:
            with pytest.raises(Exception):
                YoloDetector(logger=None)
