"""GPU: whole networks and the reference-facing API through the C ABI.

Network parity is against the fp32 torch-CPU oracle sharing the seeded weights.  The product computes fp16 x fp16
-> fp32 (the reference's own `_fp16` engines do the same, coreEngine.py:168, onnxQuantization.py:38); the tolerance
on probabilities / lane logits is written next to each assert.  Everything downstream of the raw head tensor is
bit-exact and is checked as such (fused path == reference post-processing applied to the device's own raw tensor).
"""
import os

import numpy as np
import pytest
import torch

import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
from adas_b200.coreEngine import B200Engine
from gpu_util import cached_plan, yolo_blob
from oracle import nets, post

pytestmark = pytest.mark.gpu
torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))   # oneDNN collapses under 100+ threads


def _report(name, got, ref):
    d = np.abs(got - ref)
    print(f"[parity] {name}: max_abs={d.max():.3e} mean_abs={d.mean():.3e} ref_absmax={np.abs(ref).max():.3e}")
    return float(d.max())


@pytest.mark.parametrize("impl", [1, 0])
def test_yolov5n_engine_vs_oracle(impl):
    path, sd, _ = cached_plan("yolov5", scale="n")
    eng = _capi.Engine(path, 0, max_batch=2, conv_impl=impl)
    frames = [synth.frame(s) for s in (0, 1)]
    x = yolo_blob(frames)
    raw = eng.infer(x)[0]
    model = nets.build("yolov5", sd, scale="n")
    with torch.no_grad():
        ref = model(torch.from_numpy(x)).numpy()
    assert raw.shape == ref.shape == (2, 25200, 85)
    e_prob = _report(f"v5n impl{impl} obj/cls prob", raw[..., 4:], ref[..., 4:])
    e_box = _report(f"v5n impl{impl} box px", raw[..., :4], ref[..., :4])
    assert e_prob < 1e-3          # north_star: float scores within 1e-3 (fp16 operands through 60 convs vs the fp32 oracle)
    assert e_box < 0.5            # boxes within half a pixel of the 640-px input
    eng.close()


def test_yolov8l_batch8_and_batch32_equal_batch1():
    """BASELINE configs[1] / configs[3] batch sizes: frame k of a batch-32 and of a batch-8 run equals the batch-1 result bit for bit
    (the autotuner picks different tiles per (layer, batch); every tile shape accumulates in the same K order)."""
    path, sd, _ = cached_plan("yolov8", scale="l")
    eng = _capi.Engine(path, 0, max_batch=32)
    frames = [synth.frame(s % 8) if s < 24 else synth.frame(100 + s) for s in range(32)]
    x = yolo_blob(frames)
    raw32 = eng.infer(x)[0]
    raw8 = eng.infer(x[8:16])[0]
    assert np.array_equal(raw8, raw32[8:16])
    for k in (0, 5, 13, 31):
        raw1 = eng.infer(x[k:k + 1])[0]
        assert np.array_equal(raw1[0], raw32[k]), f"frame {k}: batch-1 differs from batch-32"
    assert np.array_equal(raw32[3], raw32[11])          # the same frame at two batch positions
    # fused detect at batch 32 == batch 1
    fr = np.stack(frames)
    d32 = eng.yolo_detect(fr, 0.4, 0.45, max_det=1024)
    for k in (2, 9, 30):
        d1 = eng.yolo_detect(fr[k:k + 1], 0.4, 0.45, max_det=1024)
        n = int(d1[4][0])
        assert n == int(d32[4][k])
        for j in range(4):
            assert np.array_equal(d1[j][0, :n], d32[j][k, :n])
    eng.close()


def test_yolov8l_engine_vs_oracle_and_batch_invariance():
    path, sd, _ = cached_plan("yolov8", scale="l")
    eng = _capi.Engine(path, 0, max_batch=4)
    frames = [synth.frame(s) for s in (0, 1, 2, 3)]
    x = yolo_blob(frames)
    raw4 = eng.infer(x)[0]
    model = nets.build("yolov8", sd, scale="l")
    with torch.no_grad():
        ref = model(torch.from_numpy(x[:2])).numpy()
    assert raw4.shape == (4, 84, 8400)
    e_prob = _report("v8l cls prob", raw4[:2, 4:], ref[:, 4:])
    e_box = _report("v8l box px", raw4[:2, :4], ref[:, :4])
    assert e_prob < 1e-3          # north_star: float scores within 1e-3 of the fp32 CPU path
    assert e_box < 1.0
    # per-frame results are independent of the batch they ran in (deterministic tiles, no split-K)
    raw1 = eng.infer(x[2:3])[0]
    assert np.array_equal(raw1[0], raw4[2])
    # SIMT validation kernels agree with the tensor-core path to accumulation-order noise
    eng_s = _capi.Engine(path, 0, max_batch=1, conv_impl=1)
    raw_s = eng_s.infer(x[:1])[0]
    # (two fp16-operand paths with different accumulation order and SiLU evaluation: rounding noise, bounded below the oracle tolerance)
    assert _report("v8l tc vs simt prob", raw4[:1, 4:], raw_s[:, 4:]) < 3e-3
    eng.close()
    eng_s.close()


def test_yolov8l_fused_detect_matches_reference_postprocessing():
    path, sd, _ = cached_plan("yolov8", scale="l")
    eng = _capi.Engine(path, 0, max_batch=4)
    frames = np.stack([synth.frame(s) for s in (4, 5, 6, 7)])
    boxes, scores, cls, idx, counts, ncand = eng.yolo_detect(frames, 0.4, 0.45, max_det=1024)
    # (a) pre-processing inside the fused path is the bit-exact blob, so engine_inference on it gives the same raw tensor
    x = _capi.yolo_preprocess(frames, (640, 640))
    assert np.array_equal(x, yolo_blob(frames))
    raw = eng.infer(x)[0]
    geom = post.letterbox_geom(720, 1280, 640, 640)
    total = 0
    for b in range(4):
        r = post.yolo_postprocess(raw[b], "v8", geom, 0.4, 0.45)     # the reference's host post-processing, restated
        n = int(counts[b])
        total += n
        assert ncand[b] == r["n_cand"]
        assert np.array_equal(idx[b, :n], r["idx"])
        assert np.array_equal(boxes[b, :n], r["boxes"])
        assert np.array_equal(scores[b, :n], r["scores"])
        assert np.array_equal(cls[b, :n], r["cls"])
    assert total > 0, "synthetic operating point produced no detections"
    print("[parity] v8l fused detect: per-frame detections", counts.tolist(), "candidates", ncand.tolist())
    # (b) against the fp32 oracle end to end: every candidate whose oracle score is further than the contract tolerance (1e-3) from
    # box_score must be selected identically, with the same class and a score within 1e-3; the calibrated synthetic operating point
    # (plan.SYNTH_PROFILES_CALIB) keeps the margin cases below 5 % of the candidates
    model = nets.build("yolov8", sd, scale="l")
    with torch.no_grad():
        ref = model(torch.from_numpy(x)).numpy()
    n_cand = n_margin = 0
    for b in range(4):
        mx_ref, mx_gpu = ref[b, 4:].max(0), raw[b, 4:].max(0)
        margin = 1e-3
        sure = np.abs(mx_ref - 0.4) > margin
        cand = mx_ref > 0.4
        assert np.array_equal(cand[sure], (mx_gpu > 0.4)[sure])
        assert np.array_equal(ref[b, 4:].argmax(0)[sure & cand], raw[b, 4:].argmax(0)[sure & cand])
        assert np.abs(mx_ref[cand] - mx_gpu[cand]).max(initial=0.0) < 1e-3
        n_cand += int(cand.sum())
        n_margin += int((~sure & (cand | (mx_gpu > 0.4))).sum())
    print(f"[parity] v8l candidate set: {n_cand} oracle candidates over 4 frames, {n_margin} inside the 1e-3 margin")
    assert n_cand > 50 and n_margin <= 0.05 * n_cand
    eng.close()


@pytest.mark.parametrize("backbone,dataset", [("18", "culane"), ("34", "culane"), ("18", "tusimple")])
def test_ufldv2_engine_vs_oracle(backbone, dataset):
    """CULane (320x1600, LayerNorm before the FC) and TuSimple (320x800, no LayerNorm, 56/41 anchors, crop 0.8) geometries of
    ModelConfig (ultrafastLaneDetectorV2.py:31-55); the plan header names the dataset and the library derives crop / anchors from it."""
    cfg = plan.UFLD_DATASETS[dataset]
    path, sd, _ = cached_plan("ufldv2", backbone=backbone, cfg=dataset)
    eng = _capi.Engine(path, 0, max_batch=2)
    assert eng.meta[6] == cfg["dataset"]
    frames = np.stack([synth.frame(s) for s in (0, 1)])
    x = _capi.ufld_preprocess(frames, (cfg["in_h"], cfg["in_w"]), cfg["crop_ratio"])
    outs = eng.infer(x)
    model = nets.build("ufldv2", sd, backbone=backbone, **{k: v for k, v in cfg.items() if k not in ("dataset", "crop_ratio")})
    row_anchor, col_anchor = post.UFLD_ANCHORS[dataset]
    with torch.no_grad():
        ref = [o.numpy() for o in model(torch.from_numpy(x))]
    worst = 0.0
    for name, got, r in zip(("loc_row", "loc_col", "exist_row", "exist_col"), outs, ref):
        assert got.shape == r.shape
        worst = max(worst, _report(f"ufld{backbone} {name}", got, r) / max(1.0, float(np.abs(r).max())))
    assert worst < 5e-3           # raw logits within 5e-3 of their dynamic range (diagnostic; the contract is on lane coordinates, below)
    # lane coordinates against the fp32 CPU path: decode of the ORACLE's heads vs the device result, per anchor.  north_star: lane
    # coordinates within 1e-3 (of the image extent they are a fraction of, ultrafastLaneDetectorV2.py:152,170).  An anchor is only
    # compared when the oracle's own decisions are decisive: existence logits and the two largest location logits further apart
    # than the logit tolerance (otherwise argmax may legitimately flip); the skipped fraction is printed and bounded.
    pts, npts, status, coords = eng.ufld_detect(frames, want_coords=True)
    n_cmp = n_skip = 0
    for b in range(2):
        for name, li, lanes, ext in (("row", 0, (1, 2), 1280.0), ("col", 1, (0, 3), 720.0)):
            loc_r, ex_r = ref[li][b], ref[2 + li][b]                     # [grid, cls, lane], [2, cls, lane]
            loc_g, ex_g = outs[li][b], outs[2 + li][b]
            ncls = loc_r.shape[1]
            for lane in lanes:
                valid_r, valid_g = ex_r[:, :, lane].argmax(0), ex_g[:, :, lane].argmax(0)
                thr = ncls / 2 if name == "row" else ncls / 4
                if abs(valid_r.sum() - thr) < 1.5 or (valid_r.sum() > thr) != (valid_g.sum() > thr):
                    n_skip += ncls
                    continue
                if not valid_r.sum() > thr:
                    continue
                out_l = {1: 1, 2: 2, 0: 0, 3: 3}[lane]
                got = {}                                                 # device points are emitted in anchor order over valid anchors
                ks = [k for k in range(ncls) if valid_g[k]]
                assert len(ks) == int(npts[b, out_l])
                for j, k in enumerate(ks):
                    got[k] = coords[b, out_l, j]
                for k in range(ncls):
                    top = np.sort(loc_r[:, k, lane])[-2:]
                    decisive = abs(ex_r[1, k, lane] - ex_r[0, k, lane]) > 2e-2 and (top[1] - top[0]) > 2e-2
                    if not decisive:
                        n_skip += 1
                        continue
                    assert bool(valid_r[k]) == (k in got)
                    if valid_r[k]:
                        m = int(loc_r[:, k, lane].argmax())
                        ind = list(range(max(0, m - 1), min(loc_r.shape[0] - 1, m + 1) + 1))
                        z = loc_r[ind, k, lane].astype(np.float32)
                        e = np.exp(z - z.max())
                        c = float((e / e.sum() * np.array(ind, np.float32)).sum() + 0.5) / (loc_r.shape[0] - 1) * ext
                        assert abs(got[k] - c) <= 1e-3 * ext, (b, name, lane, k, got[k], c)
                        n_cmp += 1
    print(f"[parity] ufld{backbone} {dataset} lane coordinates: {n_cmp} anchors within 1e-3 of the extent, {n_skip} skipped as indecisive")
    if dataset == "culane":
        assert n_cmp > 100 and n_skip < 0.3 * (n_cmp + n_skip)
    # fused lane detect == reference decode applied to the device's own head tensors
    for b in range(2):
        opts, ost, ocrd = post.ufld_decode([o[b:b + 1] for o in outs], 1280, 720, row_anchor, col_anchor)
        for l in range(4):
            n = int(npts[b, l])
            assert n == len(opts[l])
            assert np.allclose(coords[b, l, :n], np.array(ocrd[l]), rtol=0, atol=1e-3)
            diff = pts[b, l, :n] - np.array(opts[l], np.int32).reshape(-1, 2)
            for j in np.nonzero(diff.any(axis=1))[0]:
                assert np.abs(diff[j]).max() == 1 and abs(coords[b, l, j] - round(coords[b, l, j])) < 1e-3
        assert [bool(v) for v in status[b]] == ost
    eng.close()


def test_engine_protocol_and_detector_api(tmp_path):
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    from adas_b200.TrafficLaneDetector import UltrafastLaneDetectorV2, LaneModelType
    path, sd, _ = cached_plan("yolov5", scale="n")
    e = B200Engine(path)
    assert e.framework_type == "b200" and e.get_engine_input_shape() == [1, 3, 640, 640]
    shapes, names = e.get_engine_output_shape()
    assert shapes == [[1, 25200, 85]] and names == ["output0"]
    out = e.engine_inference(np.zeros((1, 3, 640, 640), np.float32))
    assert out[0].shape == (1, 25200, 85)
    with pytest.raises(Exception):
        B200Engine(str(tmp_path / "missing.b200w"))
    YoloDetector.set_defaults({"model_path": path, "model_type": ObjectModelType.YOLOV5, "classes_path": None, "box_score": 0.4,
                               "box_nms_iou": 0.45})
    det = YoloDetector(logger=None, max_batch=2)
    fr = synth.frame(3)
    det.DetectFrame(fr)
    single = det.object_info
    both = det.DetectFrames([fr, synth.frame(4)])
    assert [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in single] == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]
    for r in single:
        assert isinstance(r.tolist()[0], int)
    upath, usd, _ = cached_plan("ufldv2", backbone="18")
    lane = UltrafastLaneDetectorV2(upath, LaneModelType.UFLDV2_CULANE, None)
    lane.DetectFrame(fr)
    assert len(lane.lane_info.lanes_points) == 4 and len(lane.lane_info.lanes_status) == 4
    with pytest.raises(Exception):
        UltrafastLaneDetectorV2(upath, LaneModelType.UFLDV2_CURVELANES, None)


def test_yolov5_lite_plan_matches_decoded_plan():
    """ObjectModelType.YOLOV5_LITE end to end: a lite plan (sigmoid-only head + device lite_postprocess) gives the detections of the
    plan whose Detect layer decodes in the graph, bit for bit; engine_inference on the lite plan returns the UNdecoded tensor whose host
    lite_postprocess (oracle restatement of yoloDetector.py:36-50) reproduces the fused call; the model_type / plan pairing is enforced."""
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    path, sd, _ = cached_plan("yolov5", scale="n")
    lpath, _, _ = cached_plan("yolov5", scale="n", lite=True)
    cfg = {"classes_path": None, "box_score": 0.4, "box_nms_iou": 0.45}
    YoloDetector.set_defaults({"model_path": path, "model_type": ObjectModelType.YOLOV5, **cfg})
    det = YoloDetector(logger=None, max_batch=2)
    YoloDetector.set_defaults({"model_path": lpath, "model_type": ObjectModelType.YOLOV5_LITE, **cfg})
    det_l = YoloDetector(logger=None, max_batch=2)
    frames = [synth.frame(3), synth.frame(4)]
    a, b = det.DetectFrames(frames), det_l.DetectFrames(frames)
    key = lambda rs: [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in rs]
    assert sum(len(x) for x in a) > 0
    for ra, rb in zip(a, b):
        assert key(ra) == key(rb)
    # raw tensors: same logits, decoded vs sigmoid-only boxes
    x = yolo_blob(frames)
    raw, raw_l = det.engine.engine_inference(x)[0], det_l.engine.engine_inference(x)[0]
    assert np.array_equal(raw[..., 4:], raw_l[..., 4:]) and raw_l[..., :4].max() <= 1.0 and raw[..., :4].max() > 1.0
    for i in range(2):
        assert np.array_equal(post.yolo_lite_postprocess(raw_l[i]), raw[i])
        r = post.yolo_postprocess(raw_l[i], "v5lite", post.letterbox_geom(720, 1280, 640, 640), 0.4, 0.45)
        assert np.array_equal(np.array([[q.x, q.y, q.width, q.height] for q in b[i]], np.float32).reshape(-1, 4), r["boxes"])
    YoloDetector.set_defaults({"model_path": path, "model_type": ObjectModelType.YOLOV5_LITE, **cfg})
    with pytest.raises(Exception):
        YoloDetector(logger=None)            # lite model_type on a decoded plan
    YoloDetector.set_defaults({"model_path": lpath, "model_type": ObjectModelType.YOLOV5, **cfg})
    with pytest.raises(Exception):
        YoloDetector(logger=None)


@pytest.mark.parametrize("impl", ["native", "python"])
def test_bytetracker_matches_reference_golden(golden_dir, impl):
    from adas_b200.ObjectTracker import BYTETracker
    from bytetrack_py import BYTETrackerPy
    g = np.load(os.path.join(golden_dir, "track.npz"))
    cls_ = BYTETracker if impl == "native" else BYTETrackerPy
    for seed, nobj in ((0, 8), (1, 14), (2, 4), (3, 25)):
        trk = cls_(names=[])
        trk.reset()
        rows = []
        for f, (boxes, scores, labels) in enumerate(synth.track_sequence(seed, frames=45, objects=nobj)):
            trk.update(boxes, scores, labels, np.zeros((720, 1280, 3), np.uint8))
            for t in trk.tracked_stracks:
                tl = t.tlwh
                rows.append([f, t.track_id, int(t.is_activated), t.state, tl[0], tl[1], tl[2], tl[3], float(t.score), int(str(t.class_id)[5:])])
            for t in trk.lost_stracks:
                rows.append([f, t.track_id, -1, t.state, 0, 0, 0, 0, 0, -1])
        got, gold = np.array(rows, np.float64), g[f"seq{seed}"]
        assert got.shape == gold.shape, (seed, got.shape, gold.shape)
        assert np.array_equal(got[:, [0, 1, 2, 3, 9]], gold[:, [0, 1, 2, 3, 9]])      # frame, track id, activation, state, class: exact
        assert np.allclose(got[:, 4:9], gold[:, 4:9], rtol=0, atol=1e-6)              # Kalman boxes (fp64) and scores


def test_detect_pair_concurrent_streams_equal_separate_calls():
    """adas_detect_pair enqueues both networks on their own streams before waiting for either; the results must be bit-identical
    to the two stand-alone calls (host frames, and frames already resident on the device), over repeated graph replays."""
    ypath, _, _ = cached_plan("yolov8", scale="l")
    upath, _, _ = cached_plan("ufldv2", backbone="18")
    ye = _capi.Engine(ypath, 0, max_batch=3)
    ue = _capi.Engine(upath, 0, max_batch=3)
    frames = np.stack([synth.frame(s) for s in (21, 22, 23)])
    y_ref = ye.yolo_detect(frames, 0.4, 0.45)
    u_ref = ue.ufld_detect(frames)
    dev = torch.from_numpy(frames).cuda()
    torch.cuda.synchronize()
    for rep in range(4):         # eager -> capture -> replay -> replay
        on_dev = rep % 2 == 1
        y, u = _capi.detect_pair(ye, ue, dev.data_ptr() if on_dev else frames, 0.4, 0.45, 1024, on_dev, (3, 720, 1280))
        n = y[4]
        assert np.array_equal(n, y_ref[4]) and np.array_equal(y[5], y_ref[5])
        for b in range(3):
            for k in range(4):
                assert np.array_equal(y[k][b, :n[b]], y_ref[k][b, :n[b]])
        assert np.array_equal(u[1], u_ref[1]) and np.array_equal(u[2], u_ref[2])
        for b in range(3):
            for l in range(4):
                assert np.array_equal(u[0][b, l, :u[1][b, l]], u_ref[0][b, l, :u[1][b, l]])
    assert int(y_ref[4].sum()) > 0
    ye.close()
    ue.close()


def test_pipeline_overlapped_equals_synchronous():
    """AdasPipeline.step_pipelined (two engine pairs in flight, tracker one batch behind) returns, batch for batch, exactly what the
    synchronous step() does: detections, lane points and track ids."""
    from adas_b200.pipeline import AdasPipeline
    ypath, _, _ = cached_plan("yolov8", scale="l")
    upath, _, _ = cached_plan("ufldv2", backbone="18")
    batches = [np.stack([synth.frame(40 + 2 * i + j) for j in range(2)]) for i in range(5)]

    def run(pipelined: bool):
        pipe = AdasPipeline(ypath, upath, device=0, batch=2, sets=2 if pipelined else 1, depth=3)
        out = []
        if pipelined:
            for fr in batches:
                r = pipe.step_pipelined(fr)
                if r is not None:
                    out.append(r)
            out += pipe.flush()
        else:
            out = [pipe.step(fr) for fr in batches]
        pipe.close()
        return out

    a, b = run(False), run(True)
    assert len(a) == len(b) == len(batches)
    dets = 0
    for ra, rb in zip(a, b):
        assert np.array_equal(ra.counts, rb.counts)
        for i, n in enumerate(ra.counts):
            dets += int(n)
            assert np.array_equal(ra.boxes[i, :n], rb.boxes[i, :n]) and np.array_equal(ra.scores[i, :n], rb.scores[i, :n])
            assert np.array_equal(ra.class_ids[i, :n], rb.class_ids[i, :n])
        assert np.array_equal(ra.lane_npts, rb.lane_npts) and np.array_equal(ra.lane_status, rb.lane_status)
        for i in range(ra.lane_pts.shape[0]):
            for l in range(4):
                assert np.array_equal(ra.lane_pts[i, l, :ra.lane_npts[i, l]], rb.lane_pts[i, l, :rb.lane_npts[i, l]])
        assert len(ra.tracks) == len(rb.tracks)
        for ta, tb in zip(ra.tracks, rb.tracks):                          # TRACK_DTYPE record arrays, one per frame
            assert ta.tobytes() == tb.tobytes()
    assert dets > 0


def test_frames_to_detections_lanes_tracks_vs_cpu_reference_path():
    """End to end from FRAMES: AdasPipeline (device) against bench.CpuReferencePath (reference pre/post/tracker semantics + fp32
    torch-CPU nets with the same weights) on 16 consecutive frames of the bench's synthetic stream.
    Per frame: the candidate sets (anchors clearing box_score) must be equal except for anchors whose ORACLE score lies within the
    1e-3 contract tolerance of the threshold ("margin frame", counted and printed); on every other frame class ids, NMS emission
    (candidate indices incl. duplicates) are EXACTLY equal, scores within 1e-3, boxes within 0.5 source pixel; track ids / activation
    flags are compared exactly over the prefix of the stream before the first margin frame; lane status equal and lane points within
    one pixel wherever the lane-level decisions are decisive."""
    import bench
    from adas_b200.pipeline import AdasPipeline
    from oracle import track as otrack
    plans = {"yolov8": cached_plan("yolov8", scale="l"), "ufldv2": cached_plan("ufldv2", backbone="34")}
    cpu = bench.CpuReferencePath(plans)
    frames = bench.synth_stream(7, 16)
    # the parity weights' scores lie in [0.4, 0.5]: detector threshold 0.44, tracker births at det_thresh = track_thresh + 0.1 = 0.44
    score_thr, iou_thr, track_thr = 0.44, 0.45, 0.34
    cpu.trk = otrack.Tracker(track_thresh=track_thr)
    cpu.trk.reset()
    pipe = AdasPipeline(plans["yolov8"][0], plans["ufldv2"][0], device=0, batch=8, box_score=score_thr, box_nms_iou=iou_thr, sets=1,
                        track_thresh=track_thr)
    res = [pipe.step(frames[i:i + 8]) for i in (0, 8)]
    geom = post.letterbox_geom(720, 1280, 640, 640)
    exact, margin_frames, prefix_ok, n_det, n_tracks_cmp, n_lane_pts = 0, 0, True, 0, 0, 0
    for f in range(16):
        r, b = res[f // 8], f % 8
        blob, _ = post.yolo_prepare_input(frames[f], 640, 640)
        with torch.no_grad():
            raw = cpu.yolo(torch.from_numpy(blob)).numpy()[0]
        raw_dev = pipe.yolo.infer(blob)[0][0]
        det = post.yolo_postprocess(raw, "v8", geom, score_thr, iou_thr)
        mx, mx_dev = raw[4:].max(0), raw_dev[4:].max(0)
        cand, cand_dev = mx > score_thr, mx_dev > score_thr
        assert np.abs(mx - mx_dev)[cand | cand_dev].max(initial=0.0) < 1e-3, f      # float scores within the contract
        n = int(r.counts[b])
        if not np.array_equal(cand, cand_dev):
            diff = cand != cand_dev
            assert np.all(np.abs(mx[diff] - score_thr) < 1e-3), f                   # only margin anchors may flip
            margin_frames += 1
            ok = False
        elif not (n == len(det["idx"]) and np.array_equal(r.cand_index[b, :n], det["idx"])):
            # same candidates, different NMS emission: the reference NMS visits candidates by score and suppresses on IoU > thr, so a
            # legitimate flip needs two candidate scores closer than twice the score tolerance or an IoU within 2e-3 of the threshold
            cs = np.sort(mx[cand])
            close_scores = len(cs) > 1 and np.diff(cs).min() < 2e-3
            bx, _, _ = post.yolo_process_output(raw, "v8", score_thr)
            wb = post.convert_boxes(bx, geom).astype(np.float64)
            x1, y1, x2, y2 = wb[:, 0], wb[:, 1], wb[:, 0] + wb[:, 2], wb[:, 1] + wb[:, 3]
            ar = (x2 - x1 + 1) * (y2 - y1 + 1)
            iw = np.maximum(0, np.minimum(x2[:, None], x2[None]) - np.maximum(x1[:, None], x1[None]) + 1)
            ih = np.maximum(0, np.minimum(y2[:, None], y2[None]) - np.maximum(y1[:, None], y1[None]) + 1)
            iou = iw * ih / (ar[:, None] + ar[None] - iw * ih)
            close_iou = bool(np.any(np.abs(iou[np.triu_indices(len(ar), 1)] - iou_thr) < 2e-3))
            assert close_scores or close_iou, (f, r.cand_index[b, :n], det["idx"])
            dev = post.yolo_postprocess(raw_dev, "v8", geom, score_thr, iou_thr)        # and the device applies the reference semantics to ITS values
            assert np.array_equal(r.cand_index[b, :n], dev["idx"]), f
            margin_frames += 1
            ok = False
        else:
            ok = True
            assert int(r.n_candidates[b]) == det["n_cand"], f
            assert np.array_equal(r.class_ids[b, :n], det["cls"]), f
            assert np.abs(r.scores[b, :n] - det["scores"]).max(initial=0.0) < 1e-3, f
            assert np.abs(r.boxes[b, :n] - det["boxes"]).max(initial=0.0) < 0.5, f
            exact += 1
            n_det += n
        # lanes: decoded from the oracle's heads; status equal and points within a pixel when no existence flag sits on a near-tie
        x = post.ufld_prepare_input(frames[f], 320, 1600, 0.6)
        with torch.no_grad():
            heads = [o.numpy() for o in cpu.ufld(torch.from_numpy(x))]
        opts, ost, _ = post.ufld_decode(heads, 1280, 720, post.CULANE_ROW_ANCHOR, post.CULANE_COL_ANCHOR)
        for l in range(4):
            is_row = l in (1, 2)
            loc, ex = heads[0 if is_row else 1][0, :, :, l], heads[2 if is_row else 3][0, :, :, l]      # [grid, cls], [2, cls]
            ncls = loc.shape[1]
            valid_o = ex.argmax(0)
            thr = ncls / 2 if is_row else ncls / 4
            if abs(int(valid_o.sum()) - thr) < 3:
                continue                                        # the lane-level decision itself sits on the threshold
            assert bool(r.lane_status[b][l]) == ost[l], (f, l)
            if not valid_o.sum() > thr:
                continue                                        # lane not detected: no points on either side
            # points are matched by their anchor coordinate (y of a row anchor / x of a column anchor: unique per anchor)
            key = 1 if is_row else 0
            got = {int(p[key]): int(p[1 - key]) for p in r.lane_pts[b, l, :int(r.lane_npts[b, l])]}
            want = {int(p[key]): int(p[1 - key]) for p in opts[l]}
            anchors = (post.CULANE_ROW_ANCHOR * 720 if is_row else post.CULANE_COL_ANCHOR * 1280).astype(int)
            for k in range(ncls):
                top = np.sort(loc[:, k])[-2:]
                if abs(float(ex[1, k] - ex[0, k])) <= 2e-2 or float(top[1] - top[0]) <= 2e-2:
                    continue                                    # existence or argmax of this anchor is a near-tie in the oracle itself
                a = int(anchors[k])
                assert (a in got) == (a in want) == bool(valid_o[k]), (f, l, k)
                if valid_o[k]:
                    assert abs(got[a] - want[a]) <= 1, (f, l, k, got[a], want[a])
                    n_lane_pts += 1
        # tracker: both sides see the same detections while every frame so far was exact
        prefix_ok = prefix_ok and ok
        bxr = det["boxes"]
        xyxy = np.stack([bxr[:, 0], bxr[:, 1], bxr[:, 0] + bxr[:, 2], bxr[:, 1] + bxr[:, 3]], 1).astype(int) if len(bxr) else np.zeros((0, 4), int)
        trk = cpu.trk.update(xyxy, det["scores"], det["cls"])
        if prefix_ok:
            want = sorted((int(t.tid), bool(t.activated)) for t in trk)
            got = sorted((int(t["track_id"]), bool(t["is_activated"])) for t in r.tracks[b])
            assert got == want, (f, got, want)
            n_tracks_cmp += len(want)
    pipe.close()
    print(f"[parity] frames -> detections / lanes / tracks vs the CPU reference path: {exact}/16 frames exact ({margin_frames} margin frames), "
          f"{n_det} detections, {n_tracks_cmp} track records and {n_lane_pts} lane points compared")
    assert exact >= 6 and n_det > 0 and n_tracks_cmp > 0 and n_lane_pts > 1000


def test_two_devices_in_one_process():
    """Function attributes (the > 48 KB dynamic shared memory opt-in of the GEMM / NMS kernels) and the SM count are per device:
    a second engine on another GPU of the same process must work and give the same bits (runs where two GPUs are visible)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    path, _, _ = cached_plan("yolov8", scale="l")
    upath, _, _ = cached_plan("ufldv2", backbone="18", cfg="tusimple")
    frames = np.stack([synth.frame(70 + s) for s in range(2)])
    x = yolo_blob(list(frames))
    res = []
    for dev in (0, 1):
        eng = _capi.Engine(path, dev, max_batch=2)
        ufl = _capi.Engine(upath, dev, max_batch=2)
        raw = eng.infer(x)[0]
        det = eng.yolo_detect(frames, 0.44, 0.45)
        lanes = ufl.ufld_detect(frames)
        trk = _capi.NativeTracker(device=dev, track_thresh=0.34)
        trk.reset()                      # the id counter is process-global, as BaseTrack._count in the reference
        n = int(det[4][0])
        rec = trk.update(det[0][0, :n], det[1][0, :n], det[2][0, :n])
        res.append((raw, det, lanes, rec))
        eng.close(); ufl.close()
    assert np.array_equal(res[0][0], res[1][0])
    d0, d1 = res[0][1], res[1][1]               # (boxes, scores, class ids, candidate indices, counts, n_candidates): rows beyond counts are unset
    assert np.array_equal(d0[4], d1[4]) and np.array_equal(d0[5], d1[5])
    for b in range(2):
        n = int(d0[4][b])
        for k in range(4):
            assert np.array_equal(d0[k][b, :n], d1[k][b, :n]), (b, k)
    (p0, n0, s0, _), (p1, n1, s1, _) = res[0][2], res[1][2]      # lane points: entries beyond npts are unset
    assert np.array_equal(n0, n1) and np.array_equal(s0, s1)
    for b in range(2):
        for l in range(4):
            assert np.array_equal(p0[b, l, :n0[b, l]], p1[b, l, :n1[b, l]]), (b, l)
    for name in res[0][3].dtype.names:
        assert np.array_equal(res[0][3][name], res[1][3][name]), name


def test_engine_from_onnx_file_matches_state_dict_plan(tmp_path):
    """SURVEY 8f rank 2 on the device: `B200Engine("model.onnx")` (a file written by torch's exporter from the oracle network, BatchNorm
    fused the way ultralytics exports it) against the engine built from the state_dict plan and against the fp32 oracle.  The two
    plans' packed weights differ by at most one fp16 ulp (BN folded in fp32 by the exporter, in fp64 by plan.Weights), so the outputs
    agree to the fp16 noise floor rather than bit for bit; both stay within the 1e-3 contract of the oracle."""
    import test_onnx_import as toi
    W = plan.synth_weights("yolov5", 0)
    plan.build_yolov5(W, "n")                      # the seeded state_dict is generated as the builder asks for each tensor
    model = nets.build("yolov5", W.state_dict, scale="n")
    onnx_path = str(tmp_path / "yolov5n.onnx")
    toi._export(toi._fuse_conv_bn(nets.build("yolov5", W.state_dict, scale="n")), (1, 3, 640, 640), onnx_path)
    os.environ["ADAS_B200_PLAN_CACHE"] = str(tmp_path / "cache")
    try:
        e_onnx = B200Engine(onnx_path, device=0, max_batch=2)
    finally:
        os.environ.pop("ADAS_B200_PLAN_CACHE", None)
    path, _, _ = cached_plan("yolov5", scale="n")
    e_sd = B200Engine(path, device=0, max_batch=2)
    assert e_onnx.get_engine_input_shape() == e_sd.get_engine_input_shape() == [1, 3, 640, 640]
    assert e_onnx.get_engine_output_shape() == e_sd.get_engine_output_shape()
    x = yolo_blob([synth.frame(s) for s in (0, 1)])
    a, b = e_onnx.engine_inference(x)[0], e_sd.engine_inference(x)[0]
    with torch.no_grad():
        ref = model(torch.from_numpy(x)).numpy()
    d_ab = _report("v5n onnx-plan vs state_dict-plan prob", a[..., 4:], b[..., 4:])
    d_ref = _report("v5n onnx-plan vs fp32 oracle prob", a[..., 4:], ref[..., 4:])
    assert d_ab < 1e-3 and d_ref < 1e-3
    assert _report("v5n onnx-plan box px", a[..., :4], ref[..., :4]) < 0.5


def test_lane_geometry_from_resident_points_equals_standalone_call():
    """adas_ufld_lane_geometry works on the lane points the last lane detect left on the device: same results as uploading the
    points adas_ufld_detect returned (polygon, bird-view points, curvature / offset), with and without the polyfit resampling."""
    from adas_b200.TrafficLaneDetector.ufldDetector.perspectiveTransformation import PerspectiveTransformation
    path, _, _ = cached_plan("ufldv2", backbone="18", cfg="culane")
    eng = _capi.Engine(path, 0, max_batch=4)
    frames = np.stack([synth.frame(s) for s in range(4)])
    pts, npts, status, _ = eng.ufld_detect(frames)
    M = PerspectiveTransformation((1280, 720)).M
    for adjust in (False, True):
        a = eng.lane_geometry(4, (1280, 720), adjust_lanes=adjust, M=M)
        b = _capi.lane_geometry(pts, npts, status, (1280, 720), adjust_lanes=adjust, M=M)
        for ra, rb in zip(a, b):
            assert ra["area_status"] == rb["area_status"] and np.array_equal(ra["area"], rb["area"])
            assert all(np.array_equal(x, y) for x, y in zip(ra["bird"], rb["bird"]))
            assert ra["direction"] == rb["direction"] and ra["curvature"] == rb["curvature"] and ra["offset"] == rb["offset"]
    print("[lane geometry] area_status", [r["area_status"] for r in a], "directions", [r["direction"] for r in a])
    with pytest.raises(Exception):
        _capi.Engine(path, 0, max_batch=1).lane_geometry(1, (1280, 720))       # no lane detect has run on that engine
    eng.close()


def test_bird_view_of_resident_frames_equals_standalone_warp():
    """adas_engine_warp_perspective warps the frames the last detect call left on the device (no second upload)."""
    from adas_b200.TrafficLaneDetector.ufldDetector.perspectiveTransformation import PerspectiveTransformation
    path, _, _ = cached_plan("ufldv2", backbone="18", cfg="culane")
    eng = _capi.Engine(path, 0, max_batch=2)
    frames = np.stack([synth.frame(s) for s in (5, 6)])
    eng.ufld_detect(frames)
    M = PerspectiveTransformation((1280, 720)).M
    assert np.array_equal(eng.warp_perspective(2, M, (1280, 720)), _capi.warp_perspective(frames, M, (1280, 720)))
    eng.close()


@pytest.mark.parametrize("ds", ["tusimple", "culane"])
def test_ufld_v1_engine_vs_oracle(ds):
    """UFLD v1 (ultrafastLaneDetector.py + exportLib/ultrafastLane/model.py) end to end: pre-processing blob bit-exact, head tensor
    vs the fp32 oracle (pinned to the reference's own parsingNet, tests/golden/ufld_net_pin.json), fused lane detect == the
    reference decode applied to the device's own head, lane x-coordinates vs the oracle within 1e-3 of the source width on decisive
    rows, and the UltrafastLaneDetector wrapper."""
    from adas_b200.TrafficLaneDetector import UltrafastLaneDetector
    from adas_b200.TrafficLaneDetector.ufldDetector.utils import LaneModelType
    cfg = post.UFLD_V1[ds]
    G, R = cfg["griding_num"], cfg["cls_num_per_lane"]
    path, sd, _ = cached_plan("ufldv1", backbone="18", cfg=ds)
    eng = _capi.Engine(path, 0, max_batch=2)
    assert eng.model_kind == 4 and eng.output_shapes == [[1, G + 1, R, 4]]
    frames = np.stack([synth.frame(s) for s in (0, 1)])
    x = _capi.ufld_preprocess(frames, (288, 800), 1.0)
    for b in range(2):
        assert np.array_equal(x[b], post.ufld_prepare_input(frames[b], 288, 800, 1.0)[0])
    out = eng.infer(x)[0]
    model = nets.build("ufldv1", sd, backbone="18", griding_num=G, cls_num_per_lane=R)
    with torch.no_grad():
        ref = model(torch.from_numpy(x)).numpy()
    assert out.shape == ref.shape == (2, G + 1, R, 4)
    assert _report(f"ufld v1 {ds} head", out, ref) / max(1.0, float(np.abs(ref).max())) < 5e-3
    pts, npts, status, coords = eng.ufld_detect(frames, want_coords=True)
    n_cmp = n_skip = 0
    for b in range(2):
        # fused detect == reference decode applied to the device's own head
        opts, ost, _ = post.ufld_v1_decode(out[b], cfg, 800, 288, 1280, 720)
        assert [bool(v) for v in status[b]] == ost
        for l in range(4):
            n = int(npts[b, l])
            assert n == len(opts[l])
            diff = pts[b, l, :n] - np.array(opts[l], np.int32).reshape(-1, 2)
            for j in np.nonzero(diff.any(axis=1))[0]:
                assert np.abs(diff[j]).max() == 1 and abs(coords[b, l, j] - round(coords[b, l, j])) < 1e-3
        # against the fp32 oracle: rows whose "no lane" decision and grid argmax are decisive
        rpts, rst, rloc = post.ufld_v1_decode(ref[b], cfg, 800, 288, 1280, 720)
        _, _, gloc = post.ufld_v1_decode(out[b], cfg, 800, 288, 1280, 720)
        rr = ref[b][:, ::-1, :]
        for l in range(4):
            for p in range(R):
                top = np.sort(rr[:G, p, l])[-2:]
                decisive = abs(float(rr[G, p, l] - top[1])) > 5e-2 and float(top[1] - top[0]) > 5e-2
                if not decisive:
                    n_skip += 1
                    continue
                assert (rloc[p, l] == 0) == (gloc[p, l] == 0), (b, l, p)
                if rloc[p, l] != 0:
                    # loc is in grid cells; x = loc * (799 / (G - 1)) * img_w / 800 source pixels
                    scale = (799.0 / (G - 1)) * cfg["img_w"] / 800.0 * (1280 / cfg["img_w"])
                    assert abs(rloc[p, l] - gloc[p, l]) * scale <= 1e-3 * 1280, (b, l, p, rloc[p, l], gloc[p, l])
                    n_cmp += 1
    print(f"[parity] ufld v1 {ds}: {n_cmp} row anchors within 1e-3 of the width, {n_skip} skipped as indecisive; status {status.tolist()}")
    assert n_cmp > 50
    eng.close()
    det = UltrafastLaneDetector(path, LaneModelType.UFLD_TUSIMPLE if ds == "tusimple" else LaneModelType.UFLD_CULANE, None, device=0)
    det.DetectFrame(frames[0], adjust_lanes=False)
    for l in range(4):
        assert np.array_equal(np.array(det.lane_info.lanes_points[l], np.int32).reshape(-1, 2), pts[0, l, :int(npts[0, l])])
    assert det.lane_info.lanes_status == [bool(v) for v in status[0]]
    with pytest.raises(Exception):
        UltrafastLaneDetector(path, LaneModelType.UFLD_CULANE if ds == "tusimple" else LaneModelType.UFLD_TUSIMPLE, None, device=0)
