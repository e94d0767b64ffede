"""GPU: pre/post-processing kernels through the C ABI against the oracle and the reference-generated goldens.
Bit-exact: pre-processing blobs, candidate sets, boxes (float32), scores, class ids, NMS emission order, lane points."""
import os

import numpy as np
import pytest

import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi
from oracle import post

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("hw", [(720, 1280), (480, 640), (1080, 1920), (333, 517), (600, 600), (900, 500)])
def test_yolo_preprocess_bit_exact(hw):
    fr = np.stack([synth.frame(s, *hw) for s in (0, 1)])
    blob = _capi.yolo_preprocess(fr, (640, 640))
    for b in range(2):
        ref, _ = post.yolo_prepare_input(fr[b], 640, 640)
        assert np.array_equal(blob[b], ref[0]), hw


@pytest.mark.parametrize("hw", [(720, 1280), (480, 640), (1080, 1920)])
@pytest.mark.parametrize("geom", [(320, 1600, 0.6), (320, 800, 0.8)])       # CULane / TuSimple ModelConfig
def test_ufld_preprocess_bit_exact(hw, geom):
    in_h, in_w, crop = geom
    fr = np.stack([synth.frame(s, *hw) for s in (2, 3)])
    blob = _capi.ufld_preprocess(fr, (in_h, in_w), crop)
    for b in range(2):
        ref = post.ufld_prepare_input(fr[b], in_h, in_w, crop)
        assert np.array_equal(blob[b], ref[0]), hw


@pytest.mark.parametrize("hw", [(720, 1280), (480, 640)])
def test_ufld_tusimple_post_matches_reference_golden(golden_dir, hw):
    """UFLDV2_TUSIMPLE geometry (56 row anchors linspace(160,710,56)/720, 41 column anchors, 100-cell grids) against the reference's
    own detector output (tests/golden/make_golden.py gen_ufld_tusimple)."""
    g = np.load(os.path.join(golden_dir, "ufld_post_tusimple.npz"))
    cases = ((0, ()), (1, (2,)), (2, (0, 3))) if hw == (720, 1280) else ((0, ()),)
    dims = dict(ngr=100, ncr=56, ngc=100, ncc=41)
    heads = np.stack([np.concatenate([h.ravel() for h in synth.ufld_heads(s, invalid_lanes=iv, **dims)]) for s, iv in cases])
    pts, npts, status, coords = _capi.ufld_postprocess(heads, (100, 56, 100, 41, 4), (hw[1], hw[0]), post.TUSIMPLE_ROW_ANCHOR, post.TUSIMPLE_COL_ANCHOR)
    for b, (s, iv) in enumerate(cases):
        key = f"s{s}_{hw[0]}x{hw[1]}"
        _, _, ocrd = post.ufld_decode(synth.ufld_heads(s, invalid_lanes=iv, **dims), hw[1], hw[0], post.TUSIMPLE_ROW_ANCHOR, post.TUSIMPLE_COL_ANCHOR)
        for l in range(4):
            gold = g[f"{key}_lane{l}"]
            n = int(npts[b, l])
            assert n == len(gold), (key, l)
            c = coords[b, l, :n]
            # 1e-3 px is an observed tolerance on these seeded heads, tighter than the worst case (lane_conformance_cases.v2_coord_bound:
            # 2.9e-3 px at 1280 px); tests/test_gpu_lane_conformance.py holds crafted heads to the derived bound
            assert np.allclose(c, np.array(ocrd[l]), rtol=0, atol=1e-3), (key, l)
            diff = pts[b, l, :n] - gold
            for j in np.nonzero(diff.any(axis=1))[0]:
                assert np.abs(diff[j]).max() == 1 and abs(c[j] - round(c[j])) < 1e-3, (key, l, j)
        assert np.array_equal(status[b], g[key + "_status"])


def _check_yolo(res, b, gold_box, gold_conf, gold_cls):
    boxes, scores, cls, idx, counts, ncand = res
    n = int(counts[b])
    assert n == len(gold_conf)
    assert np.array_equal(boxes[b, :n], gold_box)
    assert np.array_equal(scores[b, :n].astype(np.float64), gold_conf)
    assert np.array_equal(cls[b, :n], gold_cls)


def test_yolo_post_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "yolo_post.npz"))
    seeds = (0, 1, 2, 3)
    raw = np.stack([synth.yolo_v8_head(s) for s in seeds])            # batched: per-frame results must equal batch-1
    res = _capi.yolo_postprocess(raw, 0, 80, (640, 640), (720, 1280), 0.4, 0.45)
    for b, s in enumerate(seeds):
        k = f"v8_s{s}_720x1280"
        _check_yolo(res, b, g[k + "_box"], g[k + "_conf"], g[k + "_cls"])
    res = _capi.yolo_postprocess(raw[:1], 0, 80, (640, 640), (480, 640), 0.4, 0.45)
    _check_yolo(res, 0, g["v8_s0_480x640_box"], g["v8_s0_480x640_conf"], g["v8_s0_480x640_cls"])
    raw5 = np.stack([synth.yolo_v5_head(s) for s in (10, 11)])
    res = _capi.yolo_postprocess(raw5, 1, 80, (640, 640), (720, 1280), 0.4, 0.45)
    for b, s in enumerate((10, 11)):
        k = f"v5_s{s}_720x1280"
        _check_yolo(res, b, g[k + "_box"], g[k + "_conf"], g[k + "_cls"])


def test_yolo_lite_post_matches_reference_golden(golden_dir):
    """SURVEY 8a row D: ObjectModelType.YOLOV5_LITE.  The device lite_postprocess + select + NMS on the sigmoid-only head equals the
    reference's own YoloDetector(model_type=YOLOV5_LITE) bit for bit (golden vectors made by tests/golden/make_golden.py lite)."""
    g = np.load(os.path.join(golden_dir, "yolo_lite.npz"))
    seeds = (20, 21, 22)
    raw = np.stack([synth.yolo_v5_lite_head(s) for s in seeds])
    res = _capi.yolo_postprocess(raw, 3, 80, (640, 640), (720, 1280), 0.4, 0.45)          # 3 = ADAS_MODEL_YOLOV5_LITE
    for b, s in enumerate(seeds):
        k = f"v5lite_s{s}_720x1280"
        _check_yolo(res, b, g[k + "_box"], g[k + "_conf"], g[k + "_cls"])
    res = _capi.yolo_postprocess(raw[:1], 3, 80, (640, 640), (480, 640), 0.4, 0.45)
    _check_yolo(res, 0, g["v5lite_s20_480x640_box"], g["v5lite_s20_480x640_conf"], g["v5lite_s20_480x640_cls"])
    # the same tensor through the non-lite kind must NOT match (the decode really happens on the device)
    res5 = _capi.yolo_postprocess(raw[:1], 1, 80, (640, 640), (720, 1280), 0.4, 0.45)
    assert int(res5[4][0]) != len(g["v5lite_s20_720x1280_box"]) or not np.array_equal(res5[0][0, :int(res5[4][0])], g["v5lite_s20_720x1280_box"])


@pytest.mark.parametrize("n_hot,thr,iou", [(0, 0.4, 0.45), (1, 0.4, 0.45), (2, 0.4, 0.5), (300, 0.4, 0.45), (900, 0.25, 0.3), (120, 0.6, 0.7)])
def test_yolo_post_vs_oracle_edge_cases(n_hot, thr, iou):
    raw = np.stack([synth.yolo_v8_head(50 + s, n_hot=n_hot) for s in range(3)])
    boxes, scores, cls, idx, counts, ncand = _capi.yolo_postprocess(raw, 0, 80, (640, 640), (720, 1280), thr, iou, max_det=1024)
    geom = post.letterbox_geom(720, 1280, 640, 640)
    dup = 0
    for b in range(3):
        r = post.yolo_postprocess(raw[b], "v8", geom, thr, iou)
        n = int(counts[b])
        assert ncand[b] == r["n_cand"]
        assert n == len(r["idx"])
        assert np.array_equal(idx[b, :n], r["idx"])                 # indices incl. the reference's duplicates
        assert np.array_equal(boxes[b, :n], r["boxes"])
        assert np.array_equal(scores[b, :n], r["scores"])
        assert np.array_equal(cls[b, :n], r["cls"])
        dup += n != len(set(idx[b, :n].tolist()))
    if n_hot in (120, 300):
        assert dup > 0      # the reference's duplicate-emitting swap path is exercised


@pytest.mark.parametrize("hw", [(720, 1280), (480, 640)])
def test_ufld_post_matches_reference_golden(golden_dir, hw):
    g = np.load(os.path.join(golden_dir, "ufld_post.npz"))
    cases = ((0, ()), (1, (1,)), (2, (0, 3)), (3, ())) if hw == (720, 1280) else ((0, ()),)
    heads = np.stack([np.concatenate([h.ravel() for h in synth.ufld_heads(s, invalid_lanes=iv)]) for s, iv in cases])
    pts, npts, status, coords = _capi.ufld_postprocess(heads, (200, 72, 100, 81, 4), (hw[1], hw[0]), post.CULANE_ROW_ANCHOR,
                                                        post.CULANE_COL_ANCHOR)
    for b, (s, iv) in enumerate(cases):
        key = f"s{s}_{hw[0]}x{hw[1]}"
        _, _, ocrd = post.ufld_decode(synth.ufld_heads(s, invalid_lanes=iv), hw[1], hw[0], post.CULANE_ROW_ANCHOR, post.CULANE_COL_ANCHOR)
        for l in range(4):
            gold = g[f"{key}_lane{l}"]
            n = int(npts[b, l])
            assert n == len(gold), (key, l)
            got = pts[b, l, :n]
            # expectation coordinates: float32 exp may differ in the last ulp between numpy and CUDA ->
            # compare the float64 pre-truncation coordinate to 1e-3 px and allow +-1 px only within 1e-3 of an integer (an observed
            # tolerance, tighter than the worst case lane_conformance_cases.v2_coord_bound derives: 2.9e-3 px at 1280 px)
            c = coords[b, l, :n]
            assert np.allclose(c, np.array(ocrd[l]), rtol=0, atol=1e-3), (key, l)
            diff = got - gold
            bad = np.nonzero(diff.any(axis=1))[0]
            for j in bad:
                assert np.abs(diff[j]).max() == 1 and abs(c[j] - round(c[j])) < 1e-3, (key, l, j, got[j], gold[j], c[j])
        assert np.array_equal(status[b], g[key + "_status"])


# ---- lane geometry on the device (SURVEY rows K + 8f-1; csrc/lane_geom.cu) ------------------------------------------------------
def _lanes_to_arrays(lanes_per_frame, status_per_frame, mp=81):
    B = len(lanes_per_frame)
    pts = np.zeros((B, 4, mp, 2), np.int32)
    npts = np.zeros((B, 4), np.int32)
    for b, lanes in enumerate(lanes_per_frame):
        for l in range(4):
            a = np.asarray(lanes[l], np.int32).reshape(-1, 2)
            pts[b, l, :len(a)] = a
            npts[b, l] = len(a)
    return pts, npts, np.asarray(status_per_frame, np.uint8).reshape(B, 4)


def _assert_points(got, want, what):
    """integer points must match; a +-1 step is tolerated only where the device's float64 least-squares solution may sit on the other
    side of an integer than LAPACK's (rare: the two solutions agree to ~1e-12 relative)"""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    d = np.abs(got.astype(np.int64) - want.astype(np.int64))
    assert d.max(initial=0) <= 1, (what, int(d.max()))
    assert (d > 0).sum() <= max(1, got.shape[0] // 200), (what, int((d > 0).sum()))


@pytest.mark.parametrize("adjust", [False, True])
def test_lane_area_on_device_matches_reference_golden(golden_dir, adjust):
    """ego-lane polygon and the degree-2 polyfit resampling (core.py:102-158) for a batch of frames in one launch, against the
    UNMODIFIED reference class's `_area` / `_area_adj` / `_area_status` (tests/golden/ufld_post.npz)."""
    g = np.load(os.path.join(golden_dir, "ufld_post.npz"))
    keys = ["s0_720x1280", "s1_720x1280", "s2_720x1280", "s3_720x1280"]
    lanes = [[g[f"{k}_lane{l}"] for l in range(4)] for k in keys]
    pts, npts, status = _lanes_to_arrays(lanes, [g[k + "_status"] for k in keys])
    res = _capi.lane_geometry(pts, npts, status, (1280, 720), adjust_lanes=adjust)
    for k, r in zip(keys, res):
        assert r["area_status"] == bool(g[k + "_area_status"][0]), k
        want = g[k + ("_area_adj" if adjust else "_area")].astype(np.int32).reshape(-1, 2)
        _assert_points(r["area"], want, (k, adjust))
        if not adjust:
            assert np.array_equal(r["area"], want)
    # another image height (480x640 golden case): its own launch
    k = "s0_480x640"
    pts, npts, status = _lanes_to_arrays([[g[f"{k}_lane{l}"] for l in range(4)]], [g[k + "_status"]])
    r = _capi.lane_geometry(pts, npts, status, (640, 480), adjust_lanes=adjust)[0]
    _assert_points(r["area"], g[k + ("_area_adj" if adjust else "_area")].astype(np.int32).reshape(-1, 2), (k, adjust))


def test_birdview_points_and_curvature_on_device_match_reference_golden(golden_dir):
    """transformToBirdViewPoints + calcCurveAndOffset (perspectiveTransformation.py:120-208) for 32 cases (8 lane pairs x the matrices
    after each updateTransformParams type), against the reference class's own results (tests/golden/birdview.npz)."""
    g = np.load(os.path.join(golden_dir, "birdview.npz"))
    cases = [(s, k) for s in range(8) for k in ("Default", "Top", "Bottom", None)]
    lanes, Ms = [], []
    for case, (seed, kind) in enumerate(cases):
        left, right = synth.ego_lanes(100 + seed)
        lanes.append([[], left, right, []])
        Ms.append(g[f"c{case}_M"])
    pts, npts, status = _lanes_to_arrays(lanes, [[0, 1, 1, 0]] * len(cases))
    res = _capi.lane_geometry(pts, npts, status, (1280, 720), adjust_lanes=False, M=np.stack(Ms), bird_wh=(1280, 720))
    worst_c = worst_o = 0.0
    for case, r in enumerate(res):
        _assert_points(r["bird"][1], g[f"c{case}_bl"].astype(np.int32).reshape(-1, 2), (case, "left"))
        _assert_points(r["bird"][2], g[f"c{case}_br"].astype(np.int32).reshape(-1, 2), (case, "right"))
        d, curv, off = g[f"c{case}_curve"]
        if np.array_equal(r["bird"][1], g[f"c{case}_bl"]) and np.array_equal(r["bird"][2], g[f"c{case}_br"]):
            assert {"L": -1.0, "F": 0.0, "R": 1.0}[r["direction"]] == d, case
            worst_c = max(worst_c, abs(r["curvature"] - curv) / abs(curv))
            worst_o = max(worst_o, abs(r["offset"] - off) / max(1e-6, abs(off)))
    print(f"[parity] bird-view curvature rel err {worst_c:.2e}, offset rel err {worst_o:.2e} over {len(cases)} cases")
    assert worst_c < 1e-8 and worst_o < 1e-8
    # a missing ego lane -> (None, None), None
    pts, npts, status = _lanes_to_arrays([[[], synth.ego_lanes(100)[0], [], []]], [[0, 1, 0, 0]])
    r = _capi.lane_geometry(pts, npts, status, (1280, 720), M=Ms[0])[0]
    assert r["direction"] is None and r["curvature"] is None and r["offset"] is None and not r["area_status"] and len(r["area"]) == 0


def test_warp_perspective_bit_exact_vs_reference_golden_and_cv2(golden_dir):
    """transformToBirdView / transformToFrontalView on the device (csrc/warp.cu): every pixel equals cv2.warpPerspective's -- checked
    against the hashes of the frames the reference class warped (tests/golden/birdview.npz, `_warp_sha`) and, where cv2 is importable,
    against cv2 directly for other matrices, the inverse direction and a smaller frame."""
    import hashlib
    g = np.load(os.path.join(golden_dir, "birdview.npz"))
    cases = [(s, k) for s in range(8) for k in ("Default", "Top", "Bottom", None)]
    frames = np.stack([synth.frame(seed) for seed, _ in cases])
    Ms = np.stack([g[f"c{c}_M"] for c in range(len(cases))])
    out = _capi.warp_perspective(frames, Ms, (1280, 720))
    for c in range(len(cases)):
        sha = np.frombuffer(hashlib.sha256(np.ascontiguousarray(out[c]).tobytes()).digest(), np.uint8)
        assert np.array_equal(sha, g[f"c{c}_warp_sha"]), c
    try:
        import cv2
    except Exception:
        return
    fr = np.stack([synth.frame(40 + i, 480, 640) for i in range(3)])
    Ms = np.stack([g["c3_Minv"], g["c5_M"], np.array([[1.0, 0.1, -30.0], [0.02, 0.9, 12.5], [1e-4, -2e-4, 1.0]])])
    for dsize in ((640, 480), (333, 97)):
        got = _capi.warp_perspective(fr, Ms, dsize)
        for b in range(3):
            assert np.array_equal(got[b], cv2.warpPerspective(fr[b], Ms[b], dsize, flags=cv2.INTER_LINEAR)), (dsize, b)
    with pytest.raises(Exception):
        _capi.warp_perspective(fr[:1], np.zeros((3, 3)), (64, 64))          # singular matrix


def test_tracker_batch_call_with_empty_and_ragged_frames_equals_per_frame_updates():
    """adas_tracker_update_batch over ragged frames (0 detections, only low-score detections, many detections) == the same frames fed
    one by one to adas_tracker_update: identical records; the global id counter is reset between the two runs."""
    def frames_of(seed):
        seq = []
        for f, (boxes, scores, labels) in enumerate(synth.track_sequence(seed, frames=24, objects=10)):
            b = np.asarray(boxes, np.float64).reshape(-1, 4)
            s = np.asarray(scores, np.float64)
            c = np.asarray([int(str(l)[5:]) for l in labels], np.int32)
            if f in (0, 5, 6, 17):                        # empty frames (also the very first one)
                b, s, c = b[:0], s[:0], c[:0]
            elif f == 9:                                  # only low-score detections: stage 2 alone
                s = np.minimum(s, 0.3)
            seq.append((b, s, c))
        return seq
    seq = frames_of(4)
    one = _capi.NativeTracker(0)
    one.reset()
    per_frame = [one.update(b, s, c) for b, s, c in seq]
    bat = _capi.NativeTracker(0)
    bat.reset()
    got = []
    for i in range(0, len(seq), 8):
        chunk = seq[i:i + 8]
        counts = [len(s) for _, s, _ in chunk]
        recs = bat.update_batch(counts, np.concatenate([b for b, _, _ in chunk]), np.concatenate([s for _, s, _ in chunk]),
                                np.concatenate([c for _, _, c in chunk]))
        got.extend(recs)
    assert len(got) == len(per_frame)
    n_tracks = 0
    for f, (a, b) in enumerate(zip(per_frame, got)):
        assert len(a) == len(b), f
        for name in a.dtype.names:
            if name not in ("pad", "pad2"):
                assert np.array_equal(a[name], b[name]), (f, name)
        n_tracks += len(a)
    assert n_tracks > 50


@pytest.mark.parametrize("ds,G,R", [("tusimple", 100, 56), ("culane", 200, 18)])
def test_ufld_v1_post_matches_reference_golden(golden_dir, ds, G, R):
    """UFLD v1 decode on the device (ufld_v1_post_kernel) against the reference detector's own points / status
    (tests/golden/ufld_v1_post.npz), both dataset geometries, two frame sizes."""
    g = np.load(os.path.join(golden_dir, "ufld_v1_post.npz"))
    cfg = post.UFLD_V1[ds]
    for (h, w), cases in (((720, 1280), ((0, ()), (1, (2,)), (2, (0, 3)))), ((480, 640), ((0, ()),))):
        head = np.concatenate([synth.ufld_v1_head(s, G, R, invalid_lanes=iv) for s, iv in cases])
        pts, npts, status, coords = _capi.ufld_v1_postprocess(head, G, R, (800, 288), (cfg["img_w"], cfg["img_h"]), (w, h), np.asarray(cfg["row_anchor"], np.float64))
        for b, (s, iv) in enumerate(cases):
            key = f"{ds}_s{s}_{h}x{w}"
            assert np.array_equal(status[b], g[key + "_status"]), key
            for l in range(4):
                gold = g[f"{key}_lane{l}"]
                n = int(npts[b, l])
                assert n == len(gold), (key, l)
                diff = pts[b, l, :n] - gold
                # numpy's float32 exp vs CUDA expf may differ in the last ulp: +-1 px only where the float64 x sits on an integer
                for j in np.nonzero(diff.any(axis=1))[0]:
                    assert np.abs(diff[j]).max() == 1 and abs(coords[b, l, j] - round(coords[b, l, j])) < 1e-3, (key, l, j)
