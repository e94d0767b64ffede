"""GPU: YOLOv6-Lite on the device -- Hardswish on every GEMM route and every tile the autotuner can pick, the stem conv and the 3x3 / 5x5
depthwise convs with Hardswish, OP_SE and OP_SHUFFLE2 element by element against float64 (channel slices, ragged batches, NaN in every
unread channel and image, sentinels around every output), YOLOv6-Lite-S/M/L end to end against the fp32 oracle
(tests/yolov6_lite_oracle.py) at 320 x 320 and 224 x 128 with batch invariance, every op of the S/M/L plans against float64 over
consecutive batches, the fused detect against host post-processing, and YoloDetector on a Lite plan file and on an exported Lite
.onnx file."""
import functools
import os

import numpy as np
import pytest
import torch

import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
from gpu_util import cached_plan, halo_is_zero, yolo_blob
from oracle import post
import op_conformance_cases as oc
import plan_interp as pi
import tile_space_cases as ts
import yolov6_lite_oracle as ol

pytestmark = pytest.mark.gpu
torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))

SENTINEL = np.float16(-1234.0)
HS = plan.ACT_HSWISH


# ---------------------------------------------------------------------------------------------------------------------------
# Hardswish on every GEMM route and tile
# ---------------------------------------------------------------------------------------------------------------------------
def _hs_case(case):
    return case[:10] + (HS,) + case[11:]


def _up2_hs(sweep_case, case, seed=0):
    """The transposed-conv sweep (`sweep_case`: tile_space_cases.sweep_case) with its epilogue switched to Hardswish."""
    sw = sweep_case(case, seed)
    a = sw.ref
    for i, _, _ in sw.ops:
        sw.pb.ops[i][1].act = HS
    name, _, B, H, W, cin, in_off, cout = case[:8]
    x = sw.ins[0][2]
    w = sw.pb.tensors[sw.pb.ops[sw.ops[0][0]][1].w_tensor].astype(np.float64)     # [4 Cout, Cin] in (dy, dx, c) order
    S = np.zeros_like(a)
    for q in range(4):
        S[:, :, q // 2::2, q % 2::2] = np.einsum("nk,bkhw->bnhw", np.abs(w[q * cout:(q + 1) * cout]), np.abs(x))
    S += np.abs(sw.pb.tensors[sw.pb.ops[sw.ops[0][0]][1].bias_tensor][:cout].astype(np.float64))[None, :, None, None]
    sw.ref = oc.act64(a, HS)
    sw.bound = oc.gemm_bound(sw.ref, S, oc.r8(cin), HS, a)
    return sw


@pytest.mark.parametrize("case", [_hs_case(c) for c in ts.SWEEP_CASES], ids=[c[0] for c in ts.SWEEP_CASES])
def test_hardswish_every_route_and_tile(tmp_path, monkeypatch, case):
    """test_gpu_tile_space's sweep (every tile configuration of the route, bit-identical across them, against float64) with the
    epilogue's activation set to Hardswish."""
    import test_gpu_tile_space as tgt
    if case[1] == "up2":
        monkeypatch.setattr(ts, "sweep_case", functools.partial(_up2_hs, ts.sweep_case))
    tgt.test_tile_sweep(tmp_path, case)


@pytest.mark.parametrize("route", ["tr", "stream"])
def test_hardswish_fully_connected(tmp_path, monkeypatch, route):
    """The swap-AB tensor-core FC (transposed store) and fc_stream with Hardswish, across batch classes."""
    import test_gpu_tile_space as tgt
    monkeypatch.setattr(ts, "fc_sweep", functools.partial(ts.fc_sweep, act=HS))
    K, N = ts.FC_TR if route == "tr" else ts.FC_STREAM
    batches = (1, 16, 17, 48) if route == "tr" else ts.FC_STREAM_BATCHES
    tgt._fc_batches(tmp_path, K, N, max(batches), [1, 2], batches, route).close()


# ---------------------------------------------------------------------------------------------------------------------------
# single ops against float64 with poisoned neighbours
# ---------------------------------------------------------------------------------------------------------------------------
def _host(pb, B, mb, seed, scale=3.0, zero=()):
    """Host buffers for op 0: random fp16 values in every region it reads for images < B, NaN everywhere else of its inputs (other
    channels, images >= B), the sentinel in its output buffer outside what it reads; zero halos.  `zero`: (buffer, lo, hi) regions
    that hold structural zeros (padded channels)."""
    rng = np.random.default_rng(seed)
    writes, reads = pi.op_regions(pb, 0)
    out_buf = writes[0].buf
    bufs = {}
    for i, (rows, C, _, H, W, _) in enumerate(pb.buffers):
        v = np.zeros((mb, H + 2, W + 2, C), np.float16)
        inner = v[:, 1:-1, 1:-1]
        inner[:] = SENTINEL if i == out_buf else np.float16(np.nan)
        if i == pb.image.buf:
            inner[:B, :, :, 3] = 0                                   # the image's structural fourth channel
        for r in reads:
            if r.buf == i:
                hi = min(r.hi, 3) if i == pb.image.buf else r.hi
                inner[:B, :, :, r.lo:hi] = (rng.standard_normal((B, H, W, hi - r.lo)) * scale).astype(np.float16)
        for zb, lo, hi in zero:
            if zb == i:
                inner[:B, :, :, lo:hi] = 0
        bufs[i] = v.reshape(mb * rows, C)
    return bufs


def _check_op(tmp_path, pb, B=2, mb=3, seed=0, scale=3.0, zero=(), name="op"):
    """Run op 0 eagerly, captured and replayed (inputs rewritten before each run: it may be in place); each run against float64
    within its bound (bit exact without one), nothing written outside its slice, images < B, or the interior; run(1) equals image 0."""
    path = str(tmp_path / f"{name}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, device=0, max_batch=mb)
    w = pi.out_region(pb, 0)
    rows, C, _, H, W = pi.geom(pb, w.buf)
    results = []
    for r in range(3):
        host = _host(pb, B, mb, seed, scale, zero)
        for i, a in host.items():
            eng.write_buffer(i, a)
        eng.run(B)
        got_buf = eng.read_buffer(w.buf, mb).copy()
        results.append(got_buf)
        ref, bnd = pi.op_ref(pb, 0, host, B)
        got = pi.read_out(pb, 0, {w.buf: got_buf}, B)
        ratio, nbad = pi.excess(got, ref, bnd)
        assert nbad == 0, (name, r, ratio)
        assert halo_is_zero(got_buf, mb, H, W), f"{name} wrote into the zero halo"
        v = got_buf.reshape(mb, H + 2, W + 2, C)[:, 1:-1, 1:-1]
        hv = host[w.buf].reshape(mb, H + 2, W + 2, C)[:, 1:-1, 1:-1]
        outside = np.ones(v.shape, bool)
        outside[:B, :, :, w.lo:w.hi] = False
        assert np.array_equal(v[outside].view(np.uint16), hv[outside].view(np.uint16)), f"{name} wrote outside its slice or batch"
        for zb, lo, hi in zero:
            if zb == w.buf:
                assert not v[:B, :, :, lo:hi].any(), f"{name}: padded channels are not zero"
    assert all(np.array_equal(results[0].view(np.uint16), x.view(np.uint16)) for x in results[1:]), "eager / capture / replay differ"
    host = _host(pb, B, mb, seed, scale, zero)
    for i, a in host.items():
        eng.write_buffer(i, a)
    eng.run(1)
    one = eng.read_buffer(w.buf, 1)
    eng.close()
    assert np.array_equal(one.view(np.uint16), results[0][:rows].view(np.uint16)), "run(1) differs from image 0 of the batch"


# (k, stride, H, W, C real, act): odd sizes (7 -> 4 at stride 2), C not a multiple of 8 carried padded
DW_CASES = [(3, 1, 7, 9, 24, HS), (3, 2, 7, 9, 12, 0), (5, 1, 7, 5, 40, HS), (5, 2, 7, 7, 44, HS), (5, 2, 16, 24, 96, HS),
            (5, 1, 40, 40, 96, 0), (5, 2, 1, 3, 8, HS)]


@pytest.mark.parametrize("k,s,H,W,c,act", DW_CASES)
def test_dwconv_matches_float64(tmp_path, k, s, H, W, c, act):
    rng = np.random.default_rng(k * 100 + H)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    C = oc.r8(c)
    x = pb.sub(pb.new_padded(H, W, C + 16), 8, C)
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    out = pb.sub(pb.new_padded(Ho, Wo, C + 24), 16, C)
    w = (rng.standard_normal((c, 1, k, k)) / k).astype(np.float32)
    b = (rng.standard_normal(c) * 0.1).astype(np.float32)
    pb.dwconv(x, w, b, k, s, act, out=out)
    _check_op(tmp_path, pb, name=f"dw{k}s{s}")


@pytest.mark.parametrize("H,W,s", [(320, 320, 2), (224, 128, 2), (37, 21, 2), (30, 18, 1)])
def test_stem_conv_24_channels_hardswish(tmp_path, H, W, s):
    """YOLOv6-Lite's stem: 3x3 stride 2, 3 -> 24 channels, Hardswish, in stem_conv.cu, into a channel slice."""
    rng = np.random.default_rng(H + W)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    out = pb.sub(pb.new_padded(Ho, Wo, 48), 16, 24)
    w = (rng.standard_normal((24, 4, 3, 3)) * 0.3).astype(np.float32)
    w[:, 3] = 0
    pb.conv(pb.image, w, (rng.standard_normal(24) * 0.1).astype(np.float32), 3, s, HS, out=out)
    assert pb.ops[0][0] == plan.OP_STEMCONV and len(pb.ops) == 1
    _check_op(tmp_path, pb, scale=1.0, name="stem24")


# (C real, H, W, in place): hidden = C // 4 is 2, 3, 6, 11, 22, 48; C not a multiple of 8 carried padded with zero channels
SE_CASES = [(8, 80, 80, True), (12, 40, 40, True), (24, 9, 7, False), (44, 10, 10, True), (88, 10, 10, False), (192, 5, 3, True),
            (1024, 4, 4, False)]


@pytest.mark.parametrize("c,H,W,in_place", SE_CASES)
def test_se_matches_float64(tmp_path, c, H, W, in_place):
    rng = np.random.default_rng(c + H)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    C, hid = oc.r8(c), c // 4
    xb = pb.new_padded(H, W, C + 24)
    x = pb.sub(xb, 8, C)
    out = None if in_place else pb.sub(pb.new_padded(H, W, C + 16), 8, C)
    w1 = (rng.standard_normal((hid, c, 1, 1)) / np.sqrt(c)).astype(np.float32)
    w2 = (rng.standard_normal((c, hid, 1, 1)) / np.sqrt(hid) * 3).astype(np.float32)
    pb.se(x, w1, (rng.standard_normal(hid) * 0.5).astype(np.float32), w2, rng.standard_normal(c).astype(np.float32), out=out)
    zero = [(xb.buf, 8 + c, 8 + C)] if C != c else []
    _check_op(tmp_path, pb, scale=2.0, zero=zero, name="se")


@pytest.mark.parametrize("n,H,W,same_buf", [(8, 9, 7, False), (16, 80, 80, True), (88, 10, 10, False), (144, 3, 5, True)])
def test_shuffle2_bit_exact(tmp_path, n, H, W, same_buf):
    """a and b slices of one buffer (an S1 block's x1 and a neighbour) or of two; the output slice sits inside a wider buffer."""
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    src = pb.new_padded(H, W, 3 * n + 8)
    a = pb.sub(src, 8, n)
    b = pb.sub(src, 8 + 2 * n, n) if same_buf else pb.sub(pb.new_padded(H, W, n + 8), 0, n)
    pb.shuffle2(a, b, out=pb.sub(pb.new_padded(H, W, 2 * n + 16), 8, 2 * n))
    _check_op(tmp_path, pb, name="shuffle2")


# ---------------------------------------------------------------------------------------------------------------------------
# whole networks
# ---------------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("scale,h,w", [("s", 320, 320), ("m", 320, 320), ("l", 320, 320), ("l", 224, 128), ("s", 320, 192)])
def test_yolov6_lite_engine_vs_oracle_and_batch_invariance(scale, h, w, impl):
    path, sd, _ = cached_plan("yolov6_lite", scale=scale, in_h=h, in_w=w)
    x = yolo_blob([synth.frame(s) for s in range(3)], h, w)
    xb = np.concatenate([x] * 11)[:32]                           # frame k of a 32-image batch
    eng = _capi.Engine(path, 0, max_batch=32, conv_impl=impl)
    raw = eng.infer(x)[0]
    with torch.no_grad():
        ref = ol.build(sd, scale)(torch.from_numpy(x)).numpy()
    A = sum(-(-h // s) * -(-w // s) for s in (8, 16, 32, 64))
    assert raw.shape == ref.shape == (3, A, 85)
    e_prob = float(np.abs(raw[..., 5:] - ref[..., 5:]).max())
    e_box = float(np.abs(raw[..., :4] - ref[..., :4]).max())
    print(f"[parity] yolov6lite-{scale} {h}x{w} impl{impl}: prob {e_prob:.2e}, box {e_box:.3f} px, "
          f"candidates {[int((ref[b, :, 5:].max(1) > 0.4).sum()) for b in range(3)]}")
    assert np.all(raw[..., 4] == 1.0)
    assert e_prob < 1e-3
    assert e_box < 0.5
    big = eng.infer(xb)[0]
    one = eng.infer(x[1:2])[0]
    eng.close()
    assert np.array_equal(one[0], raw[1]), "batch-1 frame differs from the same frame in a batch of 3"
    for k in (0, 1, 2, 31):
        assert np.array_equal(big[k], raw[k % 3]), f"frame {k} of a batch of 32 differs from the same frame at batch 3"


@pytest.mark.parametrize("scale", ["s", pytest.param("m", marks=pytest.mark.slow), pytest.param("l", marks=pytest.mark.slow)])
def test_every_op_of_the_lite_plan_matches_float64(tmp_path, scale):
    """test_gpu_plan_conformance's batch A / B / A check on the plan with SE out of place (so that every op's inputs survive the run
    and every op is checked), then the in-place plan gives the same head outputs bit for bit."""
    import test_gpu_plan_conformance as gpc
    W = plan.synth_weights("yolov6lite", 0, variant=scale)
    apart = plan.build_yolov6_lite(W, scale, se_in_place=False)
    assert not pi.stale_reads(apart) and not pi.overwritten(apart) and not pi.dataflow_violations(apart)
    kinds, steps = gpc.run_aba(apart, "yolov6", {}, 2, 2, str(tmp_path / f"lite_{scale}_apart.b200w"))
    gpc.check_steps(kinds, steps)
    n_s1 = sum(n - 1 for n in plan.YOLOV6_LITE_BLOCKS)
    assert kinds.count("se") == n_s1 + 4 and kinds.count("shuffle2") == n_s1
    x = gpc.frames_in(apart, "yolov6", {}, range(2))
    eng = _capi.Engine(str(tmp_path / f"lite_{scale}_apart.b200w"), 0, max_batch=2)
    a = eng.infer(x)[0]
    eng.close()
    path, _, _ = cached_plan("yolov6_lite", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=2)
    b = eng.infer(x)[0]
    descs = [eng.time_step(2, i, 1)[2] for i in range(eng.num_steps(2))]
    eng.close()
    assert sum(d.startswith("se ") and d.endswith(" in place") for d in descs) == n_s1 + 4
    assert np.array_equal(a, b), "in-place and out-of-place SE plans differ"


@pytest.mark.parametrize("scale", ["s", "l"])
def test_yolov6_lite_fused_detect_matches_reference_postprocessing(scale):
    path, _, _ = cached_plan("yolov6_lite", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=2)
    frames = np.stack([synth.frame(s) for s in (4, 5)])
    total = 0
    for score in (0.4, 0.05):
        boxes, scores, cls, idx, counts, ncand = eng.yolo_detect(frames, score, 0.45, max_det=2125)
        raw = eng.infer(_capi.yolo_preprocess(frames, (320, 320)))[0]
        geom = post.letterbox_geom(720, 1280, 320, 320)
        for b in range(2):
            r = post.yolo_postprocess(raw[b], "v5", geom, score, 0.45)
            n = int(counts[b])
            total += n
            assert ncand[b] == r["n_cand"] and np.array_equal(idx[b, :n], r["idx"]) and np.array_equal(boxes[b, :n], r["boxes"])
            assert np.array_equal(scores[b, :n], r["scores"]) and np.array_equal(cls[b, :n], r["cls"])
        print(f"[detect] yolov6lite-{scale} score {score}: candidates {ncand.tolist()}, detections {counts.tolist()}")
    assert total > 0
    eng.close()


def test_yolo_detector_runs_a_yolov6_lite_plan(tmp_path):
    """YoloDetector(ObjectModelType.YOLOV6) on a YOLOv6-Lite-S .b200w plan: loaded, run and decoded like any YOLOv6 model."""
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    path, _, _ = cached_plan("yolov6_lite", scale="s")
    YoloDetector.set_defaults({"model_path": path, "model_type": ObjectModelType.YOLOV6, "classes_path": None, "box_score": 0.4,
                               "box_nms_iou": 0.45})
    det = YoloDetector(logger=None, max_batch=2)
    assert det.engine.handle.model_kind == plan.MODEL_YOLOV6
    out = det.engine.engine_inference(yolo_blob([synth.frame(0)], 320, 320))
    assert out[0].shape == (1, 2125, 85)
    fr = [synth.frame(0), synth.frame(2)]
    det.DetectFrame(fr[0])
    single = [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in det.object_info]
    both = det.DetectFrames(fr)
    assert len(single) > 0 and single == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]


def test_yolo_detector_runs_a_yolov6_lite_onnx_file(tmp_path):
    """YoloDetector(ObjectModelType.YOLOV6) on an exported YOLOv6-Lite-M .onnx file (opset 14): recognised, converted, loaded and decoded,
    and its network output equal to the plan built from the same state_dict."""
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    import test_yolov6_lite_cpu as tlc
    path, sd, _ = cached_plan("yolov6_lite", scale="m")
    onnx_path = str(tmp_path / "yolov6lite_m.onnx")
    tlc._export(ol.build(sd, "m").fuse(), (1, 3, 320, 320), onnx_path, 14)
    os.environ["ADAS_B200_PLAN_CACHE"] = str(tmp_path / "cache")
    try:
        YoloDetector.set_defaults({"model_path": onnx_path, "model_type": ObjectModelType.YOLOV6, "classes_path": None, "box_score": 0.4,
                                   "box_nms_iou": 0.45})
        det = YoloDetector(logger=None, max_batch=2)
    finally:
        os.environ.pop("ADAS_B200_PLAN_CACHE", None)
    assert det.engine.handle.model_kind == plan.MODEL_YOLOV6
    x = yolo_blob([synth.frame(0)], 320, 320)
    out = det.engine.engine_inference(x)
    assert out[0].shape == (1, 2125, 85)
    eng = _capi.Engine(path, 0, max_batch=1)
    ref = eng.infer(x)[0]
    eng.close()
    assert np.abs(out[0][..., 5:] - ref[..., 5:]).max() < 1e-3 and np.abs(out[0][..., :4] - ref[..., :4]).max() < 0.5
    fr = [synth.frame(0), synth.frame(2)]
    det.DetectFrame(fr[0])
    single = [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in det.object_info]
    both = det.DetectFrames(fr)
    assert len(single) > 0 and single == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]
