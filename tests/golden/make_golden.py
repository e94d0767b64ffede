"""tests/golden/make_golden.py -- generates the committed golden vectors by running the UNMODIFIED reference
(/root/reference, imported through oracle/ref_shims.py) on seeded synthetic inputs (tests/synth.py).

Run in the build container only:   python tests/golden/make_golden.py
Outputs (small, committed):        tests/golden/*.npz, tests/golden/ufld_net_pin.json
The inputs are NOT stored: tests regenerate them from the seeds (numpy Generator streams are version-stable).
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth  # noqa: E402
from oracle import ref_shims  # noqa: E402

ref_shims.install()
OUT = os.path.dirname(os.path.abspath(__file__))

import ObjectDetector.yoloDetector as ymod  # noqa: E402
from ObjectDetector.utils import NMS, ObjectModelType, Scaler  # noqa: E402
import TrafficLaneDetector.ufldDetector.ultrafastLaneDetectorV2 as umod  # noqa: E402
from TrafficLaneDetector.ufldDetector.utils import LaneModelType  # noqa: E402
from ObjectTracker.byteTrack.byteTracker import BYTETracker  # noqa: E402
from ObjectTracker.byteTrack import matching as rmatching  # noqa: E402


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def gen_nms():
    res = {}
    cases = [(s, n) for s, n in zip(range(100, 124), [2, 3, 5, 8, 13, 21, 34, 55, 89, 120, 144, 200, 233, 300, 377, 500, 2, 4, 6, 10, 40, 80, 160, 320])]
    for s, n in cases:
        b, c = synth.nms_case(s, n)
        for thr in (0.45, 0.5):
            keep = NMS.fast_soft_nms(b, list(c), thr, dets_type="xywh")
            res[f"s{s}_n{n}_t{thr}"] = np.asarray(keep, np.int32)
    # N = 0 / 1
    res["n0"] = np.asarray(NMS.fast_soft_nms(np.zeros((0, 4), np.float32), [], 0.45, dets_type="xywh"), np.int32)
    res["n1"] = np.asarray(NMS.fast_soft_nms(np.array([[1, 2, 3, 4]], np.float32), [0.9], 0.45, dets_type="xywh"), np.int32)
    np.savez_compressed(os.path.join(OUT, "nms.npz"), **res)
    ndup = sum(len(v) != len(set(v.tolist())) for v in res.values())
    print("nms cases", len(res), "with duplicate indices", ndup)


def make_yolo(model_type, raw_holder, in_hw=(640, 640)):
    shape = [1, 3, in_hw[0], in_hw[1]]
    ymod.OnnxEngine = lambda p: ref_shims.FakeEngine(shape, [[1, 1, 1]], ["output0"], lambda x: [raw_holder[0][None]])
    cfg = {"model_path": "fake.onnx", "model_type": model_type, "classes_path": os.path.join(ref_shims.REFERENCE_ROOT, "ObjectDetector/models/coco_label.txt"),
           "box_score": 0.4, "box_nms_iou": 0.45}
    ymod.YoloDetector.set_defaults(cfg)
    return ymod.YoloDetector(logger=None)


def gen_yolo():
    res = {}
    holder = [None]
    det = make_yolo(ObjectModelType.YOLOV8, holder)
    names = det.class_names
    for seed in (0, 1, 2, 3):
        for (h, w) in ((720, 1280), (480, 640)) if seed == 0 else ((720, 1280),):
            holder[0] = synth.yolo_v8_head(seed)
            fr = synth.frame(seed, h, w)
            det.DetectFrame(fr)
            info = det._object_info
            key = f"v8_s{seed}_{h}x{w}"
            res[key + "_box"] = np.array([[i.x, i.y, i.width, i.height] for i in info], np.float32).reshape(-1, 4)
            res[key + "_conf"] = np.array([i.conf for i in info], np.float64)
            res[key + "_cls"] = np.array([names.index(i.label) for i in info], np.int32)
            res[key + "_blob_sha"] = np.frombuffer(bytes.fromhex(sha(det.engine.last_input)), np.uint8)
            res[key + "_blob_sample"] = det.engine.last_input[0, :, ::37, ::41].copy()
    det5 = make_yolo(ObjectModelType.YOLOV5, holder)
    for seed in (10, 11):
        holder[0] = synth.yolo_v5_head(seed)
        fr = synth.frame(seed)
        det5.DetectFrame(fr)
        info = det5._object_info
        key = f"v5_s{seed}_720x1280"
        res[key + "_box"] = np.array([[i.x, i.y, i.width, i.height] for i in info], np.float32).reshape(-1, 4)
        res[key + "_conf"] = np.array([i.conf for i in info], np.float64)
        res[key + "_cls"] = np.array([names.index(i.label) for i in info], np.int32)
    np.savez_compressed(os.path.join(OUT, "yolo_post.npz"), **res)
    print("yolo cases", [(k, v.shape) for k, v in res.items() if k.endswith("_box")])


def gen_yolo_lite():
    """ObjectModelType.YOLOV5_LITE: the reference's own lite_postprocess + __process_output + NMS on a sigmoid-only head."""
    res = {}
    holder = [None]
    det = make_yolo(ObjectModelType.YOLOV5_LITE, holder)
    names = det.class_names
    for seed in (20, 21, 22):
        for (h, w) in ((720, 1280), (480, 640)) if seed == 20 else ((720, 1280),):
            holder[0] = synth.yolo_v5_lite_head(seed)          # DetectFrame decodes in place: fresh tensor per call
            fr = synth.frame(seed, h, w)
            det.DetectFrame(fr)
            info = det._object_info
            key = f"v5lite_s{seed}_{h}x{w}"
            res[key + "_box"] = np.array([[i.x, i.y, i.width, i.height] for i in info], np.float32).reshape(-1, 4)
            res[key + "_conf"] = np.array([i.conf for i in info], np.float64)
            res[key + "_cls"] = np.array([names.index(i.label) for i in info], np.int32)
    # the decoded tensor itself (lite_postprocess alone), sampled
    lite = ymod.YoloLiteParameters(ObjectModelType.YOLOV5_LITE, [1, 3, 640, 640], 80)
    dec = lite.lite_postprocess(synth.yolo_v5_lite_head(20).copy())
    res["decoded_s20_sha"] = np.frombuffer(bytes.fromhex(sha(dec)), np.uint8)
    res["decoded_s20_sample"] = dec[::97, :6].copy()
    np.savez_compressed(os.path.join(OUT, "yolo_lite.npz"), **res)
    print("yolo lite cases", [(k, v.shape) for k, v in res.items() if k.endswith("_box")])


def gen_ufld():
    res = {}
    holder = [None]
    shapes = [[1, 200, 72, 4], [1, 100, 81, 4], [1, 2, 72, 4], [1, 2, 81, 4]]
    umod.OnnxEngine = lambda p: ref_shims.FakeEngine([1, 3, 320, 1600], shapes, ["loc_row", "loc_col", "exist_row", "exist_col"],
                                                    lambda x: holder[0])
    det = umod.UltrafastLaneDetectorV2("fake.onnx", LaneModelType.UFLDV2_CULANE, None)
    for seed, inval in ((0, ()), (1, (1,)), (2, (0, 3)), (3, ())):
        holder[0] = synth.ufld_heads(seed, invalid_lanes=inval)
        for (h, w) in ((720, 1280), (480, 640)) if seed == 0 else ((720, 1280),):
            fr = synth.frame(seed, h, w)
            det.DetectFrame(fr, adjust_lanes=False)
            key = f"s{seed}_{h}x{w}"
            for l in range(4):
                res[f"{key}_lane{l}"] = np.array(det.lane_info.lanes_points[l], np.int32).reshape(-1, 2)
            res[key + "_status"] = np.array(det.lane_info.lanes_status, np.uint8)
            res[key + "_area_status"] = np.array([det.lane_info.area_status], np.uint8)
            res[key + "_area"] = np.array(det.lane_info.area_points, np.int32).reshape(-1, 2) if det.lane_info.area_status else np.zeros((0, 2), np.int32)
            res[key + "_blob_sha"] = np.frombuffer(bytes.fromhex(sha(det.engine.last_input)), np.uint8)
            res[key + "_blob_sample"] = det.engine.last_input[0, :, ::29, ::53].copy()
            det.DetectFrame(fr, adjust_lanes=True)
            res[key + "_area_adj"] = np.array(det.lane_info.area_points, np.int32).reshape(-1, 2) if det.lane_info.area_status else np.zeros((0, 2), np.int32)
    np.savez_compressed(os.path.join(OUT, "ufld_post.npz"), **res)
    print("ufld cases", [(k, v.shape) for k, v in res.items() if "lane" in k][:8])


def gen_ufld_tusimple():
    """UFLDV2_TUSIMPLE through the reference's detector: ModelConfig.init_tusimple_config (320x800, crop 0.8, 56 row anchors
    linspace(160,710,56)/720, 41 column anchors), heads [100,56,4] / [100,41,4]."""
    res = {}
    holder = [None]
    shapes = [[1, 100, 56, 4], [1, 100, 41, 4], [1, 2, 56, 4], [1, 2, 41, 4]]
    umod.OnnxEngine = lambda p: ref_shims.FakeEngine([1, 3, 320, 800], shapes, ["loc_row", "loc_col", "exist_row", "exist_col"],
                                                    lambda x: holder[0])
    det = umod.UltrafastLaneDetectorV2("fake.onnx", LaneModelType.UFLDV2_TUSIMPLE, None)
    for seed, inval in ((0, ()), (1, (2,)), (2, (0, 3))):
        holder[0] = synth.ufld_heads(seed, ngr=100, ncr=56, ngc=100, ncc=41, invalid_lanes=inval)
        for (h, w) in ((720, 1280), (480, 640)) if seed == 0 else ((720, 1280),):
            fr = synth.frame(seed, h, w)
            det.DetectFrame(fr, adjust_lanes=False)
            key = f"s{seed}_{h}x{w}"
            for l in range(4):
                res[f"{key}_lane{l}"] = np.array(det.lane_info.lanes_points[l], np.int32).reshape(-1, 2)
            res[key + "_status"] = np.array(det.lane_info.lanes_status, np.uint8)
            res[key + "_blob_sha"] = np.frombuffer(bytes.fromhex(sha(det.engine.last_input)), np.uint8)
            res[key + "_blob_sample"] = det.engine.last_input[0, :, ::29, ::53].copy()
    np.savez_compressed(os.path.join(OUT, "ufld_post_tusimple.npz"), **res)
    print("ufld tusimple cases", [(k, v.shape) for k, v in res.items() if "lane" in k][:8])


def gen_ufld_v1():
    """UFLD v1 (ultrafastLaneDetector.py) through the reference's detector, TuSimple and CULane configs, canned head tensors."""
    import TrafficLaneDetector.ufldDetector.ultrafastLaneDetector as v1mod
    res = {}
    holder = [None]
    for name, mt, (G, R) in (("tusimple", LaneModelType.UFLD_TUSIMPLE, (100, 56)), ("culane", LaneModelType.UFLD_CULANE, (200, 18))):
        v1mod.OnnxEngine = lambda p, G=G, R=R: ref_shims.FakeEngine([1, 3, 288, 800], [[1, G + 1, R, 4]], ["output"], lambda x: [holder[0]])
        det = v1mod.UltrafastLaneDetector("fake.onnx", mt, None)
        for seed, inval in ((0, ()), (1, (2,)), (2, (0, 3))):
            holder[0] = synth.ufld_v1_head(seed, G, R, invalid_lanes=inval)
            for (h, w) in ((720, 1280), (480, 640)) if seed == 0 else ((720, 1280),):
                fr = synth.frame(seed, h, w)
                # DetectFrame itself cannot run under numpy 2: it hands the object-array `lanes_detected` to
                # LaneDetectBase.__update_lanes_status, whose `lanes_status != []` no longer broadcasts (core.py:145) -- the two
                # stages under test are called directly (ultrafastLaneDetector.py:139-145 does exactly this sequence)
                blob = det._UltrafastLaneDetector__prepare_input(fr)
                out = det.engine.engine_inference(blob)
                lanes, status = det._UltrafastLaneDetector__process_output(out, det.cfg)
                key = f"{name}_s{seed}_{h}x{w}"
                for l in range(4):
                    res[f"{key}_lane{l}"] = np.array(lanes[l], np.int32).reshape(-1, 2)
                res[key + "_status"] = np.array([bool(v) for v in status], np.uint8)
                res[key + "_blob_sha"] = np.frombuffer(bytes.fromhex(sha(blob)), np.uint8)
    np.savez_compressed(os.path.join(OUT, "ufld_v1_post.npz"), **res)
    print("ufld v1 cases", [(k, v.shape) for k, v in res.items() if "lane" in k][:6])


def gen_track():
    res = {}
    for seed, nobj in ((0, 8), (1, 14), (2, 4), (3, 25)):
        trk = BYTETracker(names=[])
        trk.reset()
        seq = synth.track_sequence(seed, frames=45, objects=nobj)
        rows = []
        for f, (boxes, scores, labels) in enumerate(seq):
            fr = np.zeros((720, 1280, 3), np.uint8)
            trk.update(boxes, scores, labels, fr)
            for t in trk.tracked_stracks:
                tl = t.tlwh
                rows.append([f, t.track_id, int(t.is_activated), t.state, tl[0], tl[1], tl[2], tl[3], float(t.score), int(str(t.class_id)[5:])])
            for t in trk.lost_stracks:
                rows.append([f, t.track_id, -1, t.state, 0, 0, 0, 0, 0, -1])
        res[f"seq{seed}"] = np.array(rows, np.float64)
        res[f"seq{seed}_count"] = np.array([type(trk.tracked_stracks[0])._count if trk.tracked_stracks else 0], np.int64)
    # association cases (cost matrix + lapjv through the reference's linear_assignment)
    rng = np.random.default_rng(77)
    for k, (T, D) in enumerate(((1, 1), (3, 5), (7, 4), (12, 12), (30, 22), (1, 9), (40, 55))):
        a = rng.uniform(0, 900, (T, 2)); a = np.concatenate([a, a + rng.uniform(30, 150, (T, 2))], 1)
        idx = rng.integers(0, T, D)
        b = a[idx] + rng.normal(0, 12, (D, 4))
        sc = rng.uniform(0.3, 0.95, D)
        cost = rmatching.iou_distance(list(a), list(b))
        fused = 1 - (1 - cost) * sc[None, :]
        for nm, c, th in (("iou", cost, 0.5), ("fuse", fused, 0.8), ("fuse7", fused, 0.7)):
            m, ua, ub = rmatching.linear_assignment(c, thresh=th)
            x = np.full(T, -1, np.int32)
            for i, j in np.asarray(m).reshape(-1, 2):
                x[i] = j
            res[f"assoc{k}_{nm}_x"] = x
        res[f"assoc{k}_a"], res[f"assoc{k}_b"], res[f"assoc{k}_sc"] = a, b, sc
        res[f"assoc{k}_cost"], res[f"assoc{k}_fused"] = cost, fused
    np.savez_compressed(os.path.join(OUT, "track.npz"), **res)
    print("track rows", {k: v.shape for k, v in res.items() if k.startswith("seq") and not k.endswith("count")})


def gen_ufld_net_pin():
    """The oracle's restated UFLDv2 vs the reference's own parsingNet (shared weights, random input)."""
    import torch
    sys.path.insert(0, os.path.join(ref_shims.REFERENCE_ROOT, "TrafficLaneDetector/ufldDetector/exportLib"))
    from ultrafastLaneV2.model_culane import parsingNet
    import adas_b200  # noqa: F401
    from adas_b200 import plan
    from oracle import nets
    out = {}
    for bb in ("18", "34"):
        W = plan.synth_weights("ufldv2", 0)
        plan.build_ufldv2(W, bb)
        ref = parsingNet(pretrained=False, backbone=bb, num_grid_row=200, num_cls_row=72, num_grid_col=100, num_cls_col=81,
                         num_lane_on_row=4, num_lane_on_col=4, use_aux=False, input_height=320, input_width=1600, fc_norm=True).eval()
        nets.load_numpy_state_dict(ref, W.state_dict)
        mine = nets.build("ufldv2", W.state_dict, backbone=bb)
        x = torch.from_numpy(np.random.default_rng(5).standard_normal((1, 3, 320, 1600)).astype(np.float32))
        with torch.no_grad():
            r = ref(x)
            m = mine(x)
        d = [float((r[k] - v).abs().max()) for k, v in zip(("loc_row", "loc_col", "exist_row", "exist_col"), m)]
        out[f"res{bb}"] = {"max_abs_diff": d, "ref_abs_max": float(r["loc_row"].abs().max())}
        print("ufld net pin", bb, d)
    # UFLD v1: the oracle's restated net vs the reference's own v1 parsingNet (exportLib/ultrafastLane/model.py)
    from ultrafastLane.model import parsingNet as parsingNetV1
    for ds, (G, R) in (("tusimple", (100, 56)), ("culane", (200, 18))):
        W = plan.synth_weights("ufldv2", 0)
        plan.build_ufldv1(W, "18", ds)
        ref = parsingNetV1(size=(288, 800), pretrained=False, backbone="18", cls_dim=(G + 1, R, 4), use_aux=False).eval()
        nets.load_numpy_state_dict(ref, W.state_dict)
        mine = nets.build("ufldv1", W.state_dict, backbone="18", griding_num=G, cls_num_per_lane=R)
        x = torch.from_numpy(np.random.default_rng(5).standard_normal((1, 3, 288, 800)).astype(np.float32))
        with torch.no_grad():
            d = float((ref(x) - mine(x)).abs().max())
        out[f"v1_res18_{ds}"] = {"max_abs_diff": [d], "ref_abs_max": float(ref(x).abs().max())}
        print("ufld v1 net pin", ds, d)
    json.dump(out, open(os.path.join(OUT, "ufld_net_pin.json"), "w"), indent=1)


def gen_birdview():
    """perspectiveTransformation.py: matrices after each update type, bird-view points, curvature / offset."""
    from TrafficLaneDetector.ufldDetector.perspectiveTransformation import PerspectiveTransformation
    out = {}
    for case, (seed, kind) in enumerate([(s, k) for s in range(8) for k in ("Default", "Top", "Bottom", None)]):
        left, right = synth.ego_lanes(100 + seed)
        t = PerspectiveTransformation((1280, 720))
        if kind is not None:
            t.updateTransformParams(left, right, kind)
        bl, br = t.transformToBirdViewPoints(left), t.transformToBirdViewPoints(right)
        img = np.zeros((720, 1280, 3), np.uint8)
        (direction, curv), off = t.calcCurveAndOffset(img, bl, br)
        out[f"c{case}_src"], out[f"c{case}_M"], out[f"c{case}_Minv"] = t.src, t.M, t.M_inv
        out[f"c{case}_bl"], out[f"c{case}_br"] = np.asarray(bl), np.asarray(br)
        out[f"c{case}_curve"] = np.array([{"L": -1.0, "F": 0.0, "R": 1.0}[direction], curv, off])
        out[f"c{case}_draw_sha"] = np.frombuffer(bytes.fromhex(sha(img)), np.uint8)
        warped = t.transformToBirdView(synth.frame(seed))
        out[f"c{case}_warp_sha"] = np.frombuffer(bytes.fromhex(sha(warped)), np.uint8)
    t = PerspectiveTransformation((1280, 720))
    assert t.transformToBirdViewPoints([]) == [] and t.calcCurveAndOffset(np.zeros((720, 1280, 3), np.uint8), [], []) == ((None, None), None)
    np.savez_compressed(os.path.join(OUT, "birdview.npz"), **out)
    print("birdview.npz:", len(out), "arrays")


def gen_lane_conformance():
    """The reference's own __process_output (v2 and v1), __adjust_lanes_points, transformToBirdViewPoints and calcCurveAndOffset on the
    crafted heads and lanes of tests/lane_conformance_cases.py -> lane_conformance.npz."""
    import lane_conformance_cases as lc
    import TrafficLaneDetector.ufldDetector.ultrafastLaneDetector as v1mod
    from TrafficLaneDetector.ufldDetector.core import LaneDetectBase
    from TrafficLaneDetector.ufldDetector.perspectiveTransformation import PerspectiveTransformation
    res = {}
    for ds, mt in (("culane", LaneModelType.UFLDV2_CULANE), ("tusimple", LaneModelType.UFLDV2_TUSIMPLE)):
        ngr, ncr, ngc, ncc = lc.V2_GOLDEN_DIMS[ds]
        shapes = [[1, ngr, ncr, 4], [1, ngc, ncc, 4], [1, 2, ncr, 4], [1, 2, ncc, 4]]
        umod.OnnxEngine = lambda p, shapes=shapes: ref_shims.FakeEngine([1, 3, 320, 800], shapes, ["loc_row", "loc_col", "exist_row", "exist_col"],
                                                                      lambda x: None)
        det = umod.UltrafastLaneDetectorV2("fake.onnx", mt, None)
        for i, heads in enumerate(lc.v2_golden_heads(ds)):
            for w, h in lc.FRAME_SIZES:
                det.img_width, det.img_height = w, h
                lanes, status = det._UltrafastLaneDetectorV2__process_output(heads, det.cfg)
                key = f"v2_{ds}_{i}_{w}x{h}"
                for l in range(4):
                    res[f"{key}_lane{l}"] = np.array(lanes[l], np.int32).reshape(-1, 2)
                res[key + "_status"] = np.array(status, np.uint8)
    for ds, G, R in lc.V1_GOLDEN:
        mt = LaneModelType.UFLD_TUSIMPLE if ds == "tusimple" else LaneModelType.UFLD_CULANE
        v1mod.OnnxEngine = lambda p, G=G, R=R: ref_shims.FakeEngine([1, 3, 288, 800], [[1, G + 1, R, 4]], ["output"], lambda x: None)
        det = v1mod.UltrafastLaneDetector("fake.onnx", mt, None)
        for i, head in enumerate(lc.v1_golden_heads(G, R)):
            for w, h in lc.FRAME_SIZES:
                det.img_height, det.img_width = h, w
                det.h_ratio, det.w_ratio = h / det.cfg.img_h, w / det.cfg.img_w
                lanes, status = det._UltrafastLaneDetector__process_output([head], det.cfg)
                key = f"v1_{ds}_{i}_{w}x{h}"
                for l in range(4):
                    res[f"{key}_lane{l}"] = np.array(lanes[l], np.int32).reshape(-1, 2)
                res[key + "_status"] = np.array([bool(v) for v in status], np.uint8)
    res["M_default"] = PerspectiveTransformation((1280, 720)).M
    for c in lc.geom_cases():
        key = "geom_" + c["name"]
        left, right = [tuple(p) for p in c["left"]], [tuple(p) for p in c["right"]]
        if len(left) > 10 and len(right) > 10:
            al, ar = LaneDetectBase._LaneDetectBase__adjust_lanes_points(left, right, c["img_wh"][1])
            res[key + "_area_adj"] = np.vstack((al, np.flipud(ar))).astype(np.int32)
        if c["M"] is not None:
            t = PerspectiveTransformation((1280, 720))
            if c["M"] == "identity":
                t.M = np.eye(3)
            bl, br = t.transformToBirdViewPoints(left), t.transformToBirdViewPoints(right)
            res[key + "_bl"], res[key + "_br"] = np.asarray(bl, np.int64), np.asarray(br, np.int64)
            bw, bh = c["bird_wh"]
            try:
                (d, curv), off = t.calcCurveAndOffset(np.zeros((bh, bw, 3), np.uint8), bl, br)
                res[key + "_curve"] = np.array([{"L": -1.0, "F": 0.0, "R": 1.0}[d], curv, off])
            except IndexError:
                res[key + "_curve"] = np.array([np.nan, np.nan, np.nan])          # leftx[719] past a bird view under 720 rows
    np.savez_compressed(os.path.join(OUT, "lane_conformance.npz"), **res)
    print("lane_conformance.npz:", len(res), "arrays")


def gen_warp_edges():
    """cv2.warpPerspective (the library the reference calls in transformToBirdView) on the edge cases of
    tests/lane_conformance_cases.py: sha256 of every output -> warp_edges.npz."""
    import cv2
    import lane_conformance_cases as lc
    res = {}
    for name, seed, (h, w), mname, dsize in lc.warp_cases():
        res[name] = lc.sha(cv2.warpPerspective(lc.warp_source(seed, h, w), lc.WARP_MATRICES[mname], dsize, flags=cv2.INTER_LINEAR))
    Ms = lc.warp_batch_matrices()
    for b in range(len(Ms)):
        res[f"batch_{b}"] = lc.sha(cv2.warpPerspective(lc.warp_source(100 + b, 480, 640), Ms[b], (333, 97), flags=cv2.INTER_LINEAR))
    np.savez_compressed(os.path.join(OUT, "warp_edges.npz"), **res)
    print("warp_edges.npz:", len(res), "hashes")


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "lanes":
        gen_lane_conformance()
        gen_warp_edges()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "birdview":
        gen_birdview()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "lite":
        gen_yolo_lite()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "ufldv1":
        gen_ufld_v1()
        gen_ufld_net_pin()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "tusimple":
        gen_ufld_tusimple()
        sys.exit(0)
    gen_nms()
    gen_yolo()
    gen_yolo_lite()
    gen_ufld()
    gen_ufld_tusimple()
    gen_ufld_v1()
    gen_track()
    gen_ufld_net_pin()
    gen_birdview()
    gen_lane_conformance()
    gen_warp_edges()
