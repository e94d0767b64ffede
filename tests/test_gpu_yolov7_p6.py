"""GPU: YOLOv7 P6 models (W6 / E6 / D6 / E6E) on the device -- the 80 / 96-channel direct stem, the four-level YOLOv5-layout decode, and the
networks end to end against the fp32 oracle (tests/yolov7_p6_oracle.py) with the plan-carried 4-level anchor table."""
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
import yolov7_p6_oracle as o6

pytestmark = pytest.mark.gpu
torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))


@pytest.mark.parametrize("cout", [80, 96])
def test_stem_conv_6x6_s2_wide(tmp_path, cout):
    """stem_conv.cu at 80 / 96 output channels (6x6 stride 2 pad 2, SiLU): against torch on the fp16-rounded operands at 1280 and at an
    odd size, and frame 1 of a batch of 3 equal to the same frame alone, bit for bit."""
    rng = np.random.default_rng(300 + cout)
    for (B, H, W) in ((1, 1280, 1280), (3, 70, 94)):
        pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
        w = (rng.standard_normal((cout, 3, 6, 6)) * np.sqrt(2.0 / 108)).astype(np.float32)
        b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
        out = pb.conv(pb.image, w, b, 6, 2, plan.ACT_SILU, pad=2, wide_stem=True)
        assert [op[0] for op in pb.ops] == [plan.OP_STEMCONV]
        path = str(tmp_path / f"stem{cout}_{H}.b200w")
        pb.write(path)
        eng = _capi.Engine(path, 0, max_batch=B)
        x = rng.standard_normal((B, 3, H, W)).astype(np.float32)
        eng.write_buffer(pb.image.buf, to_padded(x, 4))
        for _ in range(3):          # eager, graph capture, graph replay
            eng.run(B)
        Ho, Wo = H // 2, W // 2
        got_buf = eng.read_buffer(out.buf, B).copy()
        got = from_padded(got_buf, B, Ho, Wo, 0, cout)
        ref = F.silu(F.conv2d(torch.from_numpy(x).half().float(), torch.from_numpy(w).half().float(), torch.from_numpy(b), stride=2, padding=2))
        ref = ref.numpy()
        err = float(np.abs(got - ref).max()) / max(1.0, float(np.abs(ref).max()))
        print(f"[stem] cout {cout} {B}x{H}x{W}: relative error {err:.2e}")
        assert err < 2e-3, (cout, H, err)
        assert halo_is_zero(got_buf, B, Ho, Wo)
        if B > 1:
            eng1 = _capi.Engine(path, 0, max_batch=1)
            eng1.write_buffer(pb.image.buf, to_padded(x[1:2], 4))
            eng1.run(1)
            per = got_buf.shape[0] // B
            assert np.array_equal(eng1.read_buffer(out.buf, 1), got_buf[per:2 * per])
            eng1.close()
        eng.close()


def _host_v5_decode(heads, anchors, nc):
    """The YOLOv5-layout decode in numpy float32 from the raw head levels [(grid [B, H, W, C], stride)] and the plan's [L, 3, 2] anchors."""
    no, out = 5 + nc, []
    for li, (g, st) in enumerate(heads):
        B, H, W, _ = g.shape
        p = g[..., :3 * no].reshape(B, H, W, 3, no).transpose(0, 3, 1, 2, 4).astype(np.float32)
        s = (np.float32(1) / (np.float32(1) + np.exp(-p))).astype(np.float32)
        yv, xv = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
        o = s.copy()
        o[..., 0] = (s[..., 0] * np.float32(2) - np.float32(0.5) + xv) * np.float32(st)
        o[..., 1] = (s[..., 1] * np.float32(2) - np.float32(0.5) + yv) * np.float32(st)
        o[..., 2] = (s[..., 2] * np.float32(2)) * (s[..., 2] * np.float32(2)) * anchors[li, :, 0][None, :, None, None]
        o[..., 3] = (s[..., 3] * np.float32(2)) * (s[..., 3] * np.float32(2)) * anchors[li, :, 1][None, :, None, None]
        out.append(o.reshape(B, -1, no))
    return np.concatenate(out, 1)


def test_four_level_decode_matches_host_decode():
    """The engine's [B, A, 85] output against the host decode of its own head levels with the plan's 4 x 3 x 2 anchor table: the same rows
    in the same order (level -> anchor -> y -> x).  The sigmoid's expf is the only non-numpy operation (a few ulp)."""
    path, _, pb = cached_plan("yolov7", scale="w6", in_h=256, in_w=256)
    eng = _capi.Engine(path, 0, max_batch=2)
    x = np.stack([post.yolo_prepare_input(synth.frame(s), 256, 256)[0][0] for s in (0, 1)])
    raw = eng.infer(x)[0]
    heads = []
    for buf, _, C, st in pb.outputs:
        H, W = pb.buffers[buf][3], pb.buffers[buf][4]
        g = eng.read_buffer(buf, 2).reshape(2, H + 2, W + 2, C)[:, 1:-1, 1:-1]
        heads.append((g, st))
    ref = _host_v5_decode(heads, plan.read_anchors(path), 80)
    assert raw.shape == ref.shape == (2, 3 * (32 * 32 + 16 * 16 + 8 * 8 + 4 * 4), 85)
    # a sigmoid a few ulp off moves a box coordinate by at most ~1e-7 * (2 * stride or 4 * anchor) pixels; a wrong level, anchor or row
    # order moves it by whole cells
    e_box = float((np.abs(raw[..., :4] - ref[..., :4]) / np.maximum(np.abs(ref[..., :4]), 1000.0)).max())
    e_prob = float(np.abs(raw[..., 4:] - ref[..., 4:]).max())
    print(f"[decode] box {e_box:.1e} of max(|v|, 1000 px), probabilities {e_prob:.1e}")
    assert e_box < 1e-6 and e_prob < 5e-7
    eng.close()


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("scale,size", [("w6", 640), ("e6", 640), ("d6", 640), ("e6e", 640), ("w6", 1280)])
def test_p6_engine_vs_oracle_and_batch_invariance(scale, size, impl):
    path, sd, _ = cached_plan("yolov7", scale=scale, in_h=size, in_w=size)
    eng = _capi.Engine(path, 0, max_batch=3, conv_impl=impl)
    x = yolo_blob([synth.frame(s) for s in (0, 1, 2)], size, size)
    raw = eng.infer(x)[0]
    with torch.no_grad():
        ref = o6.build(sd, scale)(torch.from_numpy(x[:2])).numpy()
    assert raw.shape == (3, 3 * sum((size // s) ** 2 for s in (8, 16, 32, 64)), 85)
    e_prob = float(np.abs(raw[:2, :, 4:] - ref[..., 4:]).max())
    e_box = float(np.abs(raw[:2, :, :4] - ref[..., :4]).max())
    print(f"[parity] yolov7-{scale} {size} impl{impl}: prob {e_prob:.2e}, box {e_box:.3f} px")
    assert e_prob < 1e-3
    assert e_box < 0.5
    raw1 = eng.infer(x[1:2])[0]
    assert np.array_equal(raw1[0], raw[1]), "batch-1 frame differs from the same frame in a batch of 3"
    eng.close()


def test_w6_fused_detect_at_1280_matches_host_postprocessing():
    """A 1280x720 frame letterboxed to 1280x1280 (the resized image is 1280x721: the reference's +1) through the fused detect."""
    path, sd, _ = cached_plan("yolov7", scale="w6", in_h=1280, in_w=1280)
    eng = _capi.Engine(path, 0, max_batch=2)
    frames = np.stack([synth.frame(s) for s in (4, 5)])
    geom = post.letterbox_geom(720, 1280, 1280, 1280)
    assert tuple(geom["new"]) == (721, 1280)
    boxes, scores, cls, idx, counts, ncand = eng.yolo_detect(frames, 0.4, 0.45, max_det=1024)
    x = _capi.yolo_preprocess(frames, (1280, 1280))
    raw = eng.infer(x)[0]
    for b in range(2):
        r = post.yolo_postprocess(raw[b], "v5", geom, 0.4, 0.45)
        n = int(counts[b])
        assert ncand[b] == r["n_cand"] and np.array_equal(idx[b, :n], r["idx"]) and np.array_equal(boxes[b, :n], r["boxes"])
        assert np.array_equal(scores[b, :n], r["scores"]) and np.array_equal(cls[b, :n], r["cls"])
    with torch.no_grad():
        ref = o6.build(sd, "w6")(torch.from_numpy(x)).numpy()
    n_cand = n_margin = 0
    for b in range(2):
        mx_ref, mx_gpu = (ref[b, :, 5:] * ref[b, :, 4:5]).max(1), (raw[b, :, 5:] * raw[b, :, 4:5]).max(1)
        sure = np.abs(mx_ref - 0.4) > 1e-3
        cand = mx_ref > 0.4
        assert np.array_equal(cand[sure], (mx_gpu > 0.4)[sure])
        assert np.abs(mx_ref[cand] - mx_gpu[cand]).max(initial=0.0) < 1e-3
        n_cand += int(cand.sum())
        n_margin += int((~sure & (cand | (mx_gpu > 0.4))).sum())
    print(f"[parity] yolov7-w6 1280 candidates: {n_cand} over 2 frames, {n_margin} inside the 1e-3 margin, detections {counts.tolist()}")
    assert n_cand > 50 and n_margin <= 0.05 * n_cand
    eng.close()


def test_yolo_detector_runs_a_yolov7_w6_onnx_file(tmp_path):
    """YoloDetector(ObjectModelType.YOLOV7) on an exported W6 .onnx file (640x640): recognised, converted, decoded with 4 levels."""
    import test_onnx_import as toi
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    W = plan.synth_weights("yolov7", 0)
    plan.build_yolov7(W, "w6", in_h=640, in_w=640)
    onnx_path = str(tmp_path / "yolov7-w6.onnx")
    toi._export(o6.build(W.state_dict, "w6").fuse(), (1, 3, 640, 640), onnx_path)
    os.environ["ADAS_B200_PLAN_CACHE"] = str(tmp_path / "cache")
    try:
        YoloDetector.set_defaults({"model_path": onnx_path, "model_type": ObjectModelType.YOLOV7, "classes_path": None, "box_score": 0.4,
                                   "box_nms_iou": 0.45})
        det = YoloDetector(logger=None, max_batch=2)
    finally:
        os.environ.pop("ADAS_B200_PLAN_CACHE", None)
    out = det.engine.engine_inference(yolo_blob([synth.frame(3)], 640, 640))
    assert out[0].shape == (1, 3 * (80 * 80 + 40 * 40 + 20 * 20 + 10 * 10), 85)
    fr = [synth.frame(3), synth.frame(4)]
    det.DetectFrame(fr[0])
    single = [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in det.object_info]
    both = det.DetectFrames(fr)
    assert single == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]
    boxes, scores, cls, idx, counts, _ = det.engine.handle.yolo_detect(np.stack(fr), 0.4, 0.45, 1024)
    n = int(counts[0])
    assert [(r.conf, r.label) for r in det.object_info] == [(float(scores[0, i]), f"class{int(cls[0, i])}") for i in range(n)]
