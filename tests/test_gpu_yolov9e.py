"""GPU: YOLOv9-E on the device -- OP_CBFUSE against float64 element by element, the CBLinear -> CBFuse block against torch, YOLOv9-E end
to end against the fp32 oracle (tests/yolov9e_oracle.py), every op of the E plan against plan_interp's float64 references over
consecutive batches, the fused detect against host post-processing, and YoloDetector on an exported E file."""
import os

import numpy as np
import pytest
import torch

import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
from gpu_util import cached_plan, from_padded, halo_is_zero, yolo_blob
from oracle import post
import plan_interp as pi
import yolov9_oracle as o9
import yolov9e_oracle as oe

pytestmark = pytest.mark.gpu
torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))

SENTINEL = np.float16(-1234.0)

# (shifts of the sources in summation order, output H, W, in place); every source count 1-5 and every shift 0-4, non-square maps,
# a 1 x 2 source at shift 4
FUSE_CASES = [((0,), 8, 12, True), ((4,), 16, 32, False), ((1, 3), 24, 40, True), ((0, 2, 4), 32, 48, False),
              ((4, 3, 2, 1), 16, 16, True), ((0, 1, 2, 3, 4), 32, 64, True), ((4, 4, 0, 2, 1), 48, 16, False)]


def _fuse_plan(shifts, H, W, in_place, C=24):
    """CBFuse of C channels at offset 16 of a 48-channel output; base (out of place) at offset 8 of a 40-channel buffer; sources at
    offset 8 of 40-channel buffers."""
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    out = pb.new_padded(H, W, 48)
    base = pb.sub(out, 16, C) if in_place else pb.sub(pb.new_padded(H, W, 40), 8, C)
    srcs = [(pb.sub(pb.new_padded(H >> s, W >> s, 40), 8, C), s) for s in shifts]
    pb.cbfuse(base, srcs, out=pb.sub(out, 16, C))
    return pb, out


def _fill(pb, out, B, mb, seed):
    """Host buffers: random fp16 interiors in every operand slice of images < B, NaN in the neighbouring channels and in images >= B
    of every input, the sentinel around the output slice and in images >= B of the output; zero halos."""
    rng = np.random.default_rng(seed)
    bufs = {}
    _, p, _ = pb.ops[0]
    for i, (rows, Cb, _, H, W, _) in enumerate(pb.buffers):
        if i == pb.image.buf:
            bufs[i] = np.zeros((mb * rows, Cb), np.float16)
            continue
        v = np.zeros((mb, H + 2, W + 2, Cb), np.float16)
        inner = v[:, 1:-1, 1:-1]
        inner[:] = SENTINEL if i == out.buf else np.float16(np.nan)
        lo = 16 if i == out.buf else 8
        if i != out.buf or p.base_buf == p.out_buf:               # the output slice holds the base when in place
            inner[:B, :, :, lo:lo + p.C] = (rng.standard_normal((B, H, W, p.C)) * 3).astype(np.float16)
        bufs[i] = v.reshape(mb * rows, Cb)
    return bufs


@pytest.mark.parametrize("shifts,H,W,in_place", FUSE_CASES)
def test_cbfuse_matches_float64(tmp_path, shifts, H, W, in_place):
    B, mb = 2, 3
    pb, out = _fuse_plan(shifts, H, W, in_place)
    path = str(tmp_path / "cbf.b200w")
    pb.write(path)
    eng = _capi.Engine(path, device=0, max_batch=mb)
    results = []
    for r in range(3):                                            # eager, capture, replay; in place needs its base rewritten each time
        host = _fill(pb, out, B, mb, seed=H * 100 + W + len(shifts))
        for i, a in host.items():
            eng.write_buffer(i, a)
        eng.run(B)
        got_buf = eng.read_buffer(out.buf, mb)
        results.append(got_buf.copy())
        ref, bnd = pi.op_ref(pb, 0, host, B)
        got = pi.read_out(pb, 0, {out.buf: got_buf}, B)
        ratio, nbad = pi.excess(got, ref, bnd)
        assert nbad == 0, (r, shifts, ratio)
        assert halo_is_zero(got_buf, mb, H, W), "cbfuse wrote into the zero halo"
        v = got_buf.reshape(mb, H + 2, W + 2, -1)[:, 1:-1, 1:-1]
        assert np.all(v[:B, :, :, :16] == SENTINEL) and np.all(v[:B, :, :, 40:] == SENTINEL), "cbfuse wrote outside its channel slice"
        assert np.all(v[B:] == SENTINEL), "cbfuse wrote an image past the batch"
    assert all(np.array_equal(results[0].view(np.uint16), x.view(np.uint16)) for x in results[1:]), "eager / capture / replay differ"
    host = _fill(pb, out, B, mb, seed=H * 100 + W + len(shifts))
    for i, a in host.items():
        eng.write_buffer(i, a)
    eng.run(1)
    one = eng.read_buffer(out.buf, 1)
    eng.close()
    rows = pb.buffers[out.buf][0]
    assert np.array_equal(one.view(np.uint16), results[0][:rows].view(np.uint16)), "run(1) differs from image 0 of the batch"


def _block(block):
    for m in block.modules():
        if isinstance(m, o9.Conv):
            with torch.no_grad():
                m.bn.running_mean.uniform_(-0.1, 0.1)
                m.bn.running_var.uniform_(0.8, 1.2)
                m.bn.weight.uniform_(0.8, 1.2)
                m.bn.bias.uniform_(-0.1, 0.1)
    return block.eval()


@pytest.mark.parametrize("impl", [0, 1])
def test_cblinear_cbfuse_block_matches_torch(tmp_path, impl):
    """Two CBLinears (1x1 + bias, groups [64, 128] at 20 x 24 and [64, 128, 256] at 10 x 12) fused into the output of a 3x3 stride-2
    conv at 40 x 48 (group 0 of each, shifts 1 and 2), in place, against the oracle's modules."""
    torch.manual_seed(impl)
    conv = _block(o9.Conv(64, 64, 3, 2))
    l1, l2 = oe.CBLinear(128, (64, 128)).eval(), oe.CBLinear(256, (64, 128, 256)).eval()
    fuse = oe.CBFuse([0, 0])
    sd = {**{f"model.15.{k}": v.numpy() for k, v in conv.state_dict().items()},
          **{f"model.11.{k}": v.numpy() for k, v in l1.state_dict().items()}, **{f"model.12.{k}": v.numpy() for k, v in l2.state_dict().items()}}
    W8 = plan.Weights(sd)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 80, 96)
    x0 = pb.new_padded(80, 96, 64)
    x1 = pb.new_padded(20, 24, 128)
    x2 = pb.new_padded(10, 12, 256)
    g = plan.Yolov9Packer(pb, W8, "adown")
    y = g.cbs("model.15", g.feat(x0), 64, 3, 2)[0]
    lin = [pb.conv(x, *W8.conv_bias(f"model.{i}.conv", n, x.C, 1), 1, 1, plan.ACT_NONE) for i, x, n in ((11, x1, 192), (12, x2, 448))]
    pb.cbfuse(y, [(pb.sub(lin[0], 0, 64), 1), (pb.sub(lin[1], 0, 64), 2)])
    path = str(tmp_path / f"blk{impl}.b200w")
    pb.write(path)
    B = 2
    rng = np.random.default_rng(impl)
    xs = [rng.standard_normal((B, v.C, v.H, v.W)).astype(np.float16).astype(np.float32) for v in (x0, x1, x2)]
    eng = _capi.Engine(path, device=0, max_batch=B, conv_impl=impl)
    from gpu_util import to_padded
    for v, x in zip((x0, x1, x2), xs):
        eng.write_buffer(v.buf, to_padded(x, v.C))
    eng.run(B)
    got = from_padded(eng.read_buffer(y.buf, B), B, 40, 48, y.coff, 64)
    eng.close()
    with torch.no_grad():
        t = [torch.from_numpy(a) for a in xs]
        ref = fuse([l1(t[1]), l2(t[2]), conv(t[0])]).numpy()
    err = np.abs(got - ref) / max(1.0, float(np.abs(ref).max()))
    assert err.max() < 3e-3, (impl, float(err.max()))


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("h,w", [(640, 640), pytest.param(384, 640, marks=pytest.mark.slow)])
def test_yolov9e_engine_vs_oracle_and_batch_invariance(h, w, impl):
    path, sd, _ = cached_plan("yolov9", scale="e", in_h=h, in_w=w)
    eng = _capi.Engine(path, 0, max_batch=3, conv_impl=impl)
    x = yolo_blob([synth.frame(s) for s in (0, 1, 2)], h, w)
    raw = eng.infer(x)[0]
    with torch.no_grad():
        ref = oe.build(sd)(torch.from_numpy(x[:2])).numpy()
    A = (h // 8) * (w // 8) + (h // 16) * (w // 16) + (h // 32) * (w // 32)
    assert raw.shape == (3, 84, A)
    e_prob = float(np.abs(raw[:2, 4:] - ref[:, 4:]).max())
    e_box = float(np.abs(raw[:2, :4] - ref[:, :4]).max())
    print(f"[parity] yolov9-e {h}x{w} impl{impl}: prob {e_prob:.2e}, box {e_box:.3f} px, "
          f"candidates {[(int((ref[b, 4:].max(0) > 0.4).sum())) for b in range(2)]}")
    assert e_prob < 1e-3
    assert e_box < 0.5
    raw1 = eng.infer(x[1:2])[0]
    assert np.array_equal(raw1[0], raw[1]), "batch-1 frame differs from the same frame in a batch of 3"
    eng.close()


@pytest.mark.slow
def test_every_op_of_the_e_plan_matches_float64(tmp_path):
    """test_gpu_plan_conformance's batch A / B / A check on the E plan with CBFuse out of place (so that every op's inputs survive the
    run and every op is checked, CBFuse included), then the in-place plan gives the same head outputs bit for bit."""
    import test_gpu_plan_conformance as gpc
    W = plan.synth_weights("yolov9", 0, variant="e")
    apart = plan.build_yolov9e(W, cbfuse_in_place=False)
    assert not pi.stale_reads(apart) and not pi.overwritten(apart)
    kinds, steps = gpc.run_aba(apart, "yolov9", {}, 2, 2, str(tmp_path / "e_apart.b200w"))
    gpc.check_steps(kinds, steps)
    assert kinds.count("cbfuse") == 5
    assert all(d.startswith("cbfuse ") for k, (_, d) in zip(kinds, steps) if k == "cbfuse")
    x = gpc.frames_in(apart, "yolov9", {}, range(2))
    eng = _capi.Engine(str(tmp_path / "e_apart.b200w"), 0, max_batch=2)
    a = eng.infer(x)[0]
    eng.close()
    path, _, _ = cached_plan("yolov9", scale="e")
    eng = _capi.Engine(path, 0, max_batch=2)
    b = eng.infer(x)[0]
    steps = [eng.time_step(2, i, 1)[2] for i in range(eng.num_steps(2))]
    eng.close()
    assert sum(d.endswith(" in place") for d in steps) == 5
    assert np.array_equal(a, b), "in-place and out-of-place CBFuse plans differ"


def test_yolov9e_fused_detect_matches_reference_postprocessing():
    path, _, _ = cached_plan("yolov9", scale="e")
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
        print(f"[detect] yolov9-e score {score}: candidates {ncand.tolist()}, detections {counts.tolist()}")
    assert total > 0
    eng.close()


@pytest.mark.slow
def test_yolo_detector_runs_a_yolov9e_onnx_file(tmp_path):
    """YoloDetector(ObjectModelType.YOLOV9) on an exported YOLOv9-E .onnx file: recognised, converted, loaded and decoded."""
    import test_onnx_import as toi
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    W = plan.synth_weights("yolov9", 0, variant="e")
    plan.build_yolov9(W, "e")
    onnx_path = str(tmp_path / "yolov9-e.onnx")
    toi._export(oe.build(W.state_dict).fuse(), (1, 3, 640, 640), onnx_path)
    os.environ["ADAS_B200_PLAN_CACHE"] = str(tmp_path / "cache")
    try:
        YoloDetector.set_defaults({"model_path": onnx_path, "model_type": ObjectModelType.YOLOV9, "classes_path": None, "box_score": 0.4,
                                   "box_nms_iou": 0.45})
        det = YoloDetector(logger=None, max_batch=2)
    finally:
        os.environ.pop("ADAS_B200_PLAN_CACHE", None)
    assert det.engine.handle.model_kind == plan.MODEL_YOLOV8
    out = det.engine.engine_inference(yolo_blob([synth.frame(0)]))
    assert out[0].shape == (1, 84, 8400)
    fr = [synth.frame(0), synth.frame(2)]
    det.DetectFrame(fr[0])
    single = [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in det.object_info]
    both = det.DetectFrames(fr)
    assert len(single) > 0 and single == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]
