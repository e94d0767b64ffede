"""GPU: YOLOv9 on the device -- the 2x2 stride-1 average pool (OP_AVGPOOL2), the ADown / AConv blocks built on it, and YOLOv9-T/S/M/C
end to end against the fp32 oracle (tests/yolov9_oracle.py) through YOLOv8's head decode, candidate selection and NMS."""
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
import yolov9_oracle as o9

pytestmark = pytest.mark.gpu
torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))


def _fp16_ulp(a: np.ndarray) -> np.ndarray:
    return np.spacing(np.abs(a).astype(np.float16)).astype(np.float32)


@pytest.mark.parametrize("H,W", [(20, 20), (13, 13), (10, 26), (7, 4)])
@pytest.mark.parametrize("fill", [0, 1])
def test_avgpool2_matches_torch_on_concat_slices(tmp_path, H, W, fill):
    """Channels [16, 16 + C) of a 64-channel input pooled into channels [8, 8 + C) of a 48-channel output; row H-1 / column W-1 hold the
    fill, every other channel and the halo stay zero."""
    B, C, ci, co = 2, 24, 16, 8
    rng = np.random.default_rng(H * 100 + W + fill)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    xin = pb.new_padded(H, W, 64)
    out = pb.new_padded(H, W, 48)
    pb.avgpool2(pb.sub(xin, ci, C), fill, out=pb.sub(out, co, C))
    path = str(tmp_path / f"ap_{H}_{W}_{fill}.b200w")
    pb.write(path)
    x = (rng.standard_normal((B, 64, H, W)) * 4).astype(np.float32)
    for impl in (0, 1):
        eng = _capi.Engine(path, device=0, max_batch=B, conv_impl=impl)
        eng.write_buffer(xin.buf, to_padded(x, 64))
        eng.run(B)
        buf = eng.read_buffer(out.buf, B).copy()
        eng.close()
        got = from_padded(buf, B, H, W, co, C)
        ref = F.avg_pool2d(torch.from_numpy(x[:, ci:ci + C]).half().float(), 2, 1, 0).numpy()
        assert np.all(np.abs(got[..., :H - 1, :W - 1] - ref) <= _fp16_ulp(ref)), (H, W, fill)
        edge = np.concatenate([got[..., H - 1, :].ravel(), got[..., :, W - 1].ravel()])
        assert np.all(edge == (-np.inf if fill else 0.0)), (H, W, fill)
        assert halo_is_zero(buf, B, H, W), "avgpool2 wrote into the zero halo"
        v = buf.reshape(B, H + 2, W + 2, -1).astype(np.float32)
        assert not v[..., :co].any() and not v[..., co + C:].any(), "avgpool2 wrote outside its channel slice"


def _block(block):
    """the oracle block in eval mode with randomised BatchNorm statistics"""
    for m in block.modules():
        if isinstance(m, o9.Conv):
            with torch.no_grad():
                m.bn.running_mean.uniform_(-0.1, 0.1)
                m.bn.running_var.uniform_(0.8, 1.2)
                m.bn.weight.uniform_(0.8, 1.2)
                m.bn.bias.uniform_(-0.1, 0.1)
    return block.eval()


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("kind,c1,c2,H,W", [("adown", 256, 256, 40, 40), ("adown", 128, 256, 20, 36), ("aconv", 64, 96, 40, 40),
                                            ("aconv", 240, 360, 20, 20), ("aconv", 32, 64, 32, 48)])
def test_adown_aconv_blocks_match_torch(tmp_path, impl, kind, c1, c2, H, W):
    """The packer's ADown / AConv (build_yolov9) against the oracle's modules, including the last output row and column."""
    torch.manual_seed(c1 + c2 + H)
    block = _block(o9.ADown(c1, c2) if kind == "adown" else o9.AConv(c1, c2))
    sd = {f"model.3.{k}": v.numpy() for k, v in block.state_dict().items()}
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    xin = pb.new_padded(H, W, c1)
    out = plan.Yolov9Packer(pb, plan.Weights(sd), kind).down("model.3", (xin, ((0, c1),)), c2)
    path = str(tmp_path / f"{kind}_{c1}_{c2}_{impl}.b200w")
    pb.write(path)
    B = 2
    x = np.random.default_rng(c1).standard_normal((B, c1, H, W)).astype(np.float32)
    eng = _capi.Engine(path, device=0, max_batch=B, conv_impl=impl)
    eng.write_buffer(xin.buf, to_padded(x, c1))
    eng.run(B)
    buf = eng.read_buffer(out[0].buf, B).copy()
    eng.close()
    got = from_padded(buf, B, H // 2, W // 2, out[0].coff, c2)
    with torch.no_grad():
        ref = block(torch.from_numpy(x).half().float()).numpy()
    assert ref.shape == got.shape
    err = np.abs(got - ref) / max(1.0, float(np.abs(ref).max()))
    assert err.max() < 3e-3, (kind, impl, float(err.max()))
    assert err[..., -1, :].max() < 3e-3 and err[..., :, -1].max() < 3e-3


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("scale", ["t", "s", "m", "c"])
def test_yolov9_engine_vs_oracle_and_batch_invariance(scale, impl):
    path, sd, _ = cached_plan("yolov9", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=3, conv_impl=impl)
    x = yolo_blob([synth.frame(s) for s in (0, 1, 2)])
    raw = eng.infer(x)[0]
    with torch.no_grad():
        ref = o9.build(sd, scale)(torch.from_numpy(x[:2])).numpy()
    assert raw.shape == (3, 84, 8400)
    e_prob = float(np.abs(raw[:2, 4:] - ref[:, 4:]).max())
    e_box = float(np.abs(raw[:2, :4] - ref[:, :4]).max())
    print(f"[parity] yolov9-{scale} impl{impl}: prob {e_prob:.2e}, box {e_box:.3f} px")
    assert e_prob < 1e-3
    assert e_box < 0.5
    raw1 = eng.infer(x[1:2])[0]
    assert np.array_equal(raw1[0], raw[1]), "batch-1 frame differs from the same frame in a batch of 3"
    eng.close()


@pytest.mark.parametrize("scale", ["t", "m"])
def test_yolov9_fused_detect_matches_reference_postprocessing(scale):
    """The device decode + candidate selection + NMS equals the reference's v8 host post-processing of the engine's own output."""
    path, _, _ = cached_plan("yolov9", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=2)
    frames = np.stack([synth.frame(s) for s in (4, 5)])
    total = 0
    for score in (0.4, 0.05):
        boxes, scores, cls, idx, counts, ncand = eng.yolo_detect(frames, score, 0.45, max_det=8400)
        raw = eng.infer(_capi.yolo_preprocess(frames, (640, 640)))[0]
        geom = post.letterbox_geom(720, 1280, 640, 640)
        for b in range(2):
            r = post.yolo_postprocess(raw[b], "v8", geom, score, 0.45)
            n = int(counts[b])
            total += n
            assert ncand[b] == r["n_cand"] and np.array_equal(idx[b, :n], r["idx"]) and np.array_equal(boxes[b, :n], r["boxes"])
            assert np.array_equal(scores[b, :n], r["scores"]) and np.array_equal(cls[b, :n], r["cls"])
        print(f"[detect] yolov9-{scale} score {score}: candidates {ncand.tolist()}, detections {counts.tolist()}")
    assert total > 0
    eng.close()


@pytest.mark.parametrize("scale", ["t", "s", "m", "c"])
def test_yolov9_candidate_sets_follow_the_margin_rule(scale):
    """Candidates (max class probability > 0.4) agree with the fp32 oracle's wherever the oracle's score is more than 1e-3 from the
    threshold, and few of them sit inside that margin."""
    path, sd, _ = cached_plan("yolov9", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=4)
    x = yolo_blob([synth.frame(s) for s in (4, 5, 6, 7)])
    raw = eng.infer(x)[0]
    eng.close()
    with torch.no_grad():
        ref = o9.build(sd, scale)(torch.from_numpy(x)).numpy()
    n_cand = n_margin = 0
    for b in range(4):
        mx_ref, mx_gpu = ref[b, 4:].max(0), raw[b, 4:].max(0)
        sure = np.abs(mx_ref - 0.4) > 1e-3
        cand = mx_ref > 0.4
        assert np.array_equal(cand[sure], (mx_gpu > 0.4)[sure])
        assert np.abs(mx_ref[cand] - mx_gpu[cand]).max(initial=0.0) < 1e-3
        n_cand += int(cand.sum())
        n_margin += int((~sure & (cand | (mx_gpu > 0.4))).sum())
    print(f"[margin] yolov9-{scale}: {n_cand} candidates over 4 frames, {n_margin} inside the 1e-3 margin")
    assert 200 <= n_cand <= 800 and n_margin <= 0.5 * n_cand


def test_yolo_detector_runs_a_yolov9_onnx_file(tmp_path):
    """YoloDetector(ObjectModelType.YOLOV9) on an exported YOLOv9-T .onnx file: recognised, converted, loaded and decoded."""
    import test_onnx_import as toi
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    W = plan.synth_weights("yolov9", 0, variant="t")
    plan.build_yolov9(W, "t")
    onnx_path = str(tmp_path / "yolov9-t.onnx")
    toi._export(o9.build(W.state_dict, "t").fuse(), (1, 3, 640, 640), onnx_path)
    os.environ["ADAS_B200_PLAN_CACHE"] = str(tmp_path / "cache")
    try:
        YoloDetector.set_defaults({"model_path": onnx_path, "model_type": ObjectModelType.YOLOV9, "classes_path": None, "box_score": 0.4,
                                   "box_nms_iou": 0.45})
        det = YoloDetector(logger=None, max_batch=2)
    finally:
        os.environ.pop("ADAS_B200_PLAN_CACHE", None)
    assert det.engine.handle.model_kind == plan.MODEL_YOLOV8
    out = det.engine.engine_inference(yolo_blob([synth.frame(3)]))
    assert out[0].shape == (1, 84, 8400)
    fr = [synth.frame(3), synth.frame(4)]
    det.DetectFrame(fr[0])
    single = [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in det.object_info]
    both = det.DetectFrames(fr)
    assert len(single) > 0 and single == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]
