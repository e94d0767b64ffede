"""oracle/post.py -- TEST INFRASTRUCTURE ONLY: CPU (numpy) restatement of the reference's pre/post-processing.

Never imported by the product path (`vehicle-cv-adas_b200/`); only `tests/`, `__graft_entry__.smoke()` and
`bench.py`'s cpu_baseline / `--impl reference` leg use it.  Every function cites the reference lines it follows.
Pinned against the reference's own Python (run with the import shims of oracle/ref_shims.py in the build
container) by tests/golden/make_golden.py -> tests/golden/*.npz, and re-checked on every test run by
tests/test_oracle_golden.py.
"""
from __future__ import annotations

import numpy as np


# ---------------------------------------------------------------------------------------------
# pre-processing
# ---------------------------------------------------------------------------------------------
def resize_linear_u8(src: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """cv2.resize(src, (dw, dh), INTER_LINEAR) for uint8 HxWxC, restated: 11-bit fixed-point coefficients,
    x index clamped with zeroed fraction, y rows clipped, vertical pass ((b0*(r0>>4))>>16 + (b1*(r1>>4))>>16 + 2)>>2.
    (Used by Scaler.process_image, ObjectDetector/utils.py:53,58 and ultrafastLaneDetectorV2.py:102.)"""
    sh, sw = src.shape[:2]

    def coef(ssize, dsize, clamp):
        scale = 1.0 / (np.float64(dsize) / np.float64(ssize))
        d = np.arange(dsize)
        f = ((d + 0.5) * scale - 0.5).astype(np.float32)
        s = np.floor(f).astype(np.int32)
        f = (f - s.astype(np.float32)).astype(np.float32)
        if clamp:
            lo = s < 0
            f[lo] = 0
            s[lo] = 0
            hi = s >= ssize - 1
            f[hi] = 0
            s[hi] = ssize - 1
        a0 = np.rint((np.float32(1.0) - f) * np.float32(2048)).astype(np.int32)
        a1 = np.rint(f * np.float32(2048)).astype(np.int32)
        s1 = np.clip(s + 1, 0, ssize - 1)
        s0 = np.clip(s, 0, ssize - 1)
        return s0, s1, a0, a1

    sx, sx1, ax0, ax1 = coef(sw, dw, True)
    sy, sy1, by0, by1 = coef(sh, dh, False)
    S = src.astype(np.int32)
    hrow = S[:, sx, :] * ax0[None, :, None] + S[:, sx1, :] * ax1[None, :, None]
    r0, r1 = hrow[sy], hrow[sy1]
    out = (((by0[:, None, None] * (r0 >> 4)) >> 16) + ((by1[:, None, None] * (r1 >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def letterbox_geom(src_h, src_w, in_h, in_w):
    """Scaler.process_image bookkeeping, ObjectDetector/utils.py:42-62 -> dict(new, pad, old)."""
    padh = padw = 0
    newh, neww = in_h, in_w
    if src_h != src_w:
        hw = src_h / src_w
        if hw > 1:
            newh, neww = in_h, int(in_w / hw)
            padw = int((in_w - neww) * 0.5)
        else:
            newh, neww = int(in_h * hw) + 1, in_w
            padh = int((in_h - newh) * 0.5)
    return dict(old=(src_h, src_w), new=(newh, neww), pad=(padh, padw), target=(in_h, in_w))


def yolo_prepare_input(img_bgr: np.ndarray, in_h: int, in_w: int):
    """Scaler.process_image (utils.py:42-63) + cv2.dnn.blobFromImage(1/255, swapRB) (yoloDetector.py:96-102)."""
    g = letterbox_geom(img_bgr.shape[0], img_bgr.shape[1], in_h, in_w)
    (newh, neww), (padh, padw) = g["new"], g["pad"]
    if img_bgr.shape[0] != img_bgr.shape[1]:
        canvas = np.full((in_h, in_w, 3), 114, np.uint8)
        canvas[padh:padh + newh, padw:padw + neww] = resize_linear_u8(img_bgr, neww, newh)
    else:
        canvas = resize_linear_u8(img_bgr, in_w, in_h)
    blob = canvas[:, :, ::-1].astype(np.float32) * np.float32(1.0 / 255.0)       # float32 multiply like blobFromImage
    return np.ascontiguousarray(blob.transpose(2, 0, 1)[None]), g


def ufld_prepare_input(img_bgr: np.ndarray, in_h: int, in_w: int, crop_ratio: float) -> np.ndarray:
    """UltrafastLaneDetectorV2.__prepare_input, ultrafastLaneDetectorV2.py:96-112 (float64 normalisation, then float32)."""
    rgb = img_bgr[:, :, ::-1]
    r = resize_linear_u8(rgb, in_w, int(in_h / crop_ratio)).astype(np.float32)
    r = r[-in_h:, :, :]
    mean = [0.485, 0.456, 0.406]
    std = [0.229, 0.224, 0.225]
    x = (r / 255.0 - mean) / std
    return np.ascontiguousarray(x.transpose(2, 0, 1)[None]).astype(np.float32)


# ---------------------------------------------------------------------------------------------
# YOLO post-processing
# ---------------------------------------------------------------------------------------------
V5_ANCHORS = np.asarray([[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]], np.float32).reshape(3, -1, 2)


def yolo_lite_postprocess(outs: np.ndarray, in_hw=(640, 640)) -> np.ndarray:
    """YoloLiteParameters.lite_postprocess, yoloDetector.py:36-50 (model_type == YOLOV5_LITE): grid / anchor decode of a
    sigmoid-only head [A, 5+nc], float32, one rounding per numpy op.  grid = __make_grid(w, h) -> row r is (r % h, r // h)
    (np.meshgrid(arange(ny=h), arange(nx=w)), :31-33).  Returns a decoded copy (the reference works in place)."""
    outs = np.array(outs, np.float32)
    row = 0
    for i, stride in enumerate((8, 16, 32)):
        h, w = int(in_hw[0] / stride), int(in_hw[1] / stride)
        n = 3 * h * w
        r = np.arange(w * h)
        grid = np.stack((r % h, r // h), 1).astype(np.float32)
        xy = outs[row:row + n, 0:2]
        outs[row:row + n, 0:2] = (xy * np.float32(2.0) - np.float32(0.5) + np.tile(grid, (3, 1))) * np.float32(stride)
        wh = outs[row:row + n, 2:4] * np.float32(2.0)
        outs[row:row + n, 2:4] = wh * wh * np.repeat(V5_ANCHORS[i], h * w, axis=0)
        row += n
    return outs


def yolo_process_output(raw: np.ndarray, kind: str, box_score: float):
    """YoloDetector.__process_output, yoloDetector.py:104-133, vectorised.  raw: [4+nc, A] (v8) or [A, 5+nc] (v5, v5lite).
    Returns boxes xyxy float32 [N,4], class ids int [N], confs list[float] in ascending anchor order."""
    out = raw.T if kind == "v8" else raw
    out = np.asarray(out, np.float32)
    if kind == "v5lite":
        out = yolo_lite_postprocess(out)
    probs = out[:, 4:] if kind == "v8" else out[:, 5:] * out[:, 4:5]
    cls = np.argmax(probs, axis=1)
    conf = probs[np.arange(out.shape[0]), cls]
    keep = conf.astype(np.float64) > box_score               # float(classConf) > self.box_score, strict
    x, y, w, h = out[keep, 0], out[keep, 1], out[keep, 2], out[keep, 3]
    half = np.float32(0.5)
    boxes = np.stack([x - half * w, y - half * h, x + half * w, y + half * h], axis=-1).astype(np.float32)
    return boxes, cls[keep], [float(c) for c in conf[keep]]


def convert_boxes(boxes_xyxy: np.ndarray, g: dict) -> np.ndarray:
    """Scaler.convert_boxes_coordinate(in xyxy -> out xywh), utils.py:70-87 (float32 arithmetic)."""
    b = np.array(boxes_xyxy, np.float32)
    if b.size == 0:
        return b
    ratioh, ratiow = g["old"][0] / g["new"][0], g["old"][1] / g["new"][1]
    padh, padw = g["pad"]
    b[:, [0, 2]] = (b[:, [0, 2]] - padw) * ratiow
    b[:, [1, 3]] = (b[:, [1, 3]] - padh) * ratioh
    b[:, 2:4] = b[:, 2:4] - b[:, 0:2]
    return b


def soft_nms(boxes_xywh: np.ndarray, confs, iou_thr: float, score_thr: float = 0.001) -> np.ndarray:
    """NMS.fast_soft_nms as it actually behaves (utils.py:161-256): `method` is a str, so the hard-suppression
    branch runs; areas use the +1 convention; the "swap" overwrites row i with row maxpos and leaves row maxpos
    unchanged (tBD is a view, :214,226) while scores and areas are truly swapped (:227-228); returns
    dets[:,4][scores > 0.001] as int32 (duplicates possible)."""
    d = np.array(boxes_xywh, np.float32).copy()
    n = d.shape[0]
    if n == 0:
        return np.zeros(0, np.int32)
    if n == 1:
        return np.zeros(1, np.int32)
    d[:, 2:4] = d[:, 0:2] + d[:, 2:4]                       # xywh -> xyxy in float32 (:186-187)
    det = np.concatenate([d.astype(np.float64), np.arange(n, dtype=np.float64)[:, None]], axis=1)
    sc = np.array(confs, np.float64)
    ar = (det[:, 3] - det[:, 1] + 1) * (det[:, 2] - det[:, 0] + 1)
    for i in range(n):
        pos = i + 1
        if i != n - 1:
            mp = int(np.argmax(sc[pos:])) + pos
            ms = sc[mp]
        else:
            ms, mp = sc[-1], 0
        if sc[i] < ms:
            det[i, :] = det[mp, :]
            sc[i], sc[mp] = sc[mp], sc[i]
            ar[i], ar[mp] = ar[mp], ar[i]
        xx1 = np.maximum(det[i, 1], det[pos:, 1])
        yy1 = np.maximum(det[i, 0], det[pos:, 0])
        xx2 = np.minimum(det[i, 3], det[pos:, 3])
        yy2 = np.minimum(det[i, 2], det[pos:, 2])
        w = np.maximum(0.0, xx2 - xx1 + 1)
        h = np.maximum(0.0, yy2 - yy1 + 1)
        inter = w * h
        ovr = inter / (ar[i] + ar[pos:] - inter)
        wgt = np.ones(ovr.shape)
        wgt[ovr > iou_thr] = 0
        sc[pos:] = wgt * sc[pos:]
    return det[:, 4][sc > score_thr].astype(np.int32)


def yolo_postprocess(raw: np.ndarray, kind: str, g: dict, box_score: float, nms_iou: float):
    """DetectFrame after the network (yoloDetector.py:164-168): -> dict(boxes xywh f32 [K,4], scores f32, cls, idx, n_cand)."""
    boxes, cls, confs = yolo_process_output(raw, kind, box_score)
    xywh = convert_boxes(boxes, g)
    keep = soft_nms(xywh, confs, nms_iou)
    confs = np.array(confs, np.float64)
    return dict(boxes=xywh[keep].reshape(-1, 4), scores=confs[keep].astype(np.float32), cls=np.asarray(cls)[keep].astype(np.int32),
                idx=keep, n_cand=len(confs))


# ---------------------------------------------------------------------------------------------
# UFLDv2 decode
# ---------------------------------------------------------------------------------------------
def _softmax(x):
    x = x - np.max(x, axis=-1, keepdims=True)
    e = np.exp(x)
    return e / np.sum(e, axis=-1, keepdims=True)


def ufld_decode(outs, img_w: int, img_h: int, row_anchor, col_anchor, local_width: int = 1):
    """UltrafastLaneDetectorV2.__process_output, ultrafastLaneDetectorV2.py:114-181 for batch entry 0 of each tensor.
    Returns (points: 4 lists of (x,y) ints in order left-side, left-ego, right-ego, right-side; status: 4 bools;
    coords: 4 lists of the float64 pre-truncation expectation coordinate)."""
    loc_row, loc_col, ex_row, ex_col = [np.asarray(o, np.float32) for o in outs]
    ngr, ncr = loc_row.shape[1], loc_row.shape[2]
    ngc, ncc = loc_col.shape[1], loc_col.shape[2]
    mi_row, v_row = loc_row.argmax(1), ex_row.argmax(1)
    mi_col, v_col = loc_col.argmax(1), ex_col.argmax(1)
    pts = {k: [] for k in range(4)}
    crd = {k: [] for k in range(4)}
    for i in (1, 2):
        if v_row[0, :, i].sum() > ncr / 2:
            for k in range(ncr):
                if v_row[0, k, i]:
                    m = int(mi_row[0, k, i])
                    ind = list(range(max(0, m - local_width), min(ngr - 1, m + local_width) + 1))
                    c = (_softmax(loc_row[0, ind, k, i]) * list(map(float, ind))).sum() + 0.5
                    c = c / (ngr - 1) * img_w
                    pts[i].append((int(c), int(row_anchor[k] * img_h)))
                    crd[i].append(float(c))
    for i in (0, 3):
        if v_col[0, :, i].sum() > ncc / 4:
            for k in range(ncc):
                if v_col[0, k, i]:
                    m = int(mi_col[0, k, i])
                    ind = list(range(max(0, m - local_width), min(ngc - 1, m + local_width) + 1))
                    c = (_softmax(loc_col[0, ind, k, i]) * list(map(float, ind))).sum() + 0.5
                    c = c / (ngc - 1) * img_h
                    pts[i].append((int(col_anchor[k] * img_w), int(c)))
                    crd[i].append(float(c))
    order = (0, 1, 2, 3)
    return [pts[k] for k in order], [len(pts[k]) > 2 for k in order], [crd[k] for k in order]


CULANE_ROW_ANCHOR = np.linspace(0.42, 1, 72)      # ModelConfig.init_culane_config, ultrafastLaneDetectorV2.py:47-55
CULANE_COL_ANCHOR = np.linspace(0, 1, 81)
TUSIMPLE_ROW_ANCHOR = np.linspace(160, 710, 56) / 720   # ModelConfig.init_tusimple_config, ultrafastLaneDetectorV2.py:31-37
TUSIMPLE_COL_ANCHOR = np.linspace(0, 1, 41)
UFLD_ANCHORS = {"culane": (CULANE_ROW_ANCHOR, CULANE_COL_ANCHOR), "tusimple": (TUSIMPLE_ROW_ANCHOR, TUSIMPLE_COL_ANCHOR)}


# ---------------------------------------------------------------------------------------------
# UFLD v1 decode
# ---------------------------------------------------------------------------------------------
# ModelConfig of ultrafastLaneDetector.py:15-37: source geometry, grid cells, row anchors (in 288-row input coordinates)
UFLD_V1 = {
    "tusimple": dict(img_w=1280, img_h=720, griding_num=100, cls_num_per_lane=56, row_anchor=np.linspace(64, 284, 56)),
    "culane": dict(img_w=1640, img_h=590, griding_num=200, cls_num_per_lane=18, row_anchor=[round(v) for v in np.linspace(121, 287, 18)]),
}


def ufld_v1_decode(output: np.ndarray, cfg: dict, input_w: int, input_h: int, image_w: int, image_h: int):
    """UltrafastLaneDetector.__process_output (ultrafastLaneDetector.py:97-136) for one frame: `output` [griding_num+1, rows, 4]
    float32.  Rows are reversed, softmax (float32, as scipy.special.softmax computes it) over the grid cells without the last
    "no lane" bin, expectation with 1-based cell indices (float64), 0 where the argmax is the "no lane" bin; a lane is detected when
    more than two rows are non-zero.  Returns (points: 4 lists of [x, y] ints, status: 4 bools, loc: [rows, 4] float64)."""
    out = np.asarray(output, np.float32)
    out = out[:, ::-1, :]
    x = out[:-1]
    e = np.exp(x - np.amax(x, axis=0, keepdims=True))
    prob = e / np.sum(e, axis=0, keepdims=True)
    idx = (np.arange(cfg["griding_num"]) + 1).reshape(-1, 1, 1)
    loc = np.sum(prob * idx, axis=0)
    loc[np.argmax(out, axis=0) == cfg["griding_num"]] = 0
    col_sample = np.linspace(0, input_w - 1, cfg["griding_num"])
    col_sample_w = col_sample[1] - col_sample[0]
    h_ratio, w_ratio = image_h / cfg["img_h"], image_w / cfg["img_w"]
    pts, status = [], []
    R = cfg["cls_num_per_lane"]
    for lane in range(loc.shape[1]):
        lp = []
        if np.sum(loc[:, lane] != 0) > 2:
            status.append(True)
            for p in range(loc.shape[0]):
                if loc[p, lane] > 0:
                    px = loc[p, lane] * col_sample_w * cfg["img_w"] / input_w - 1
                    py = cfg["img_h"] * (cfg["row_anchor"][R - 1 - p] / input_h) - 1
                    lp.append([int(px * w_ratio), int(py * h_ratio)])
        else:
            status.append(False)
        pts.append(lp)
    return pts, status, loc


# ---------------------------------------------------------------------------------------------
# ByteTrack association
# ---------------------------------------------------------------------------------------------
def ious(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """matching.ious, matching.py:34-53 (no +1 convention), float64."""
    a = np.asarray(a, float).reshape(-1, 4)[:, None, :]
    b = np.asarray(b, float).reshape(-1, 4)[None, :, :]
    xx1, yy1 = np.maximum(a[..., 0], b[..., 0]), np.maximum(a[..., 1], b[..., 1])
    xx2, yy2 = np.minimum(a[..., 2], b[..., 2]), np.minimum(a[..., 3], b[..., 3])
    wh = np.maximum(0.0, xx2 - xx1) * np.maximum(0.0, yy2 - yy1)
    return wh / ((a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1]) + (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1]) - wh)


def iou_cost(a, b, det_scores=None) -> np.ndarray:
    """iou_distance (matching.py:55-80) and, with det_scores, fuse_score (matching.py:108-116)."""
    c = 1 - ious(a, b)
    if det_scores is not None and c.size:
        c = 1 - (1 - c) * np.asarray(det_scores, float)[None, :]
    return c


def lapjv_extended(cost: np.ndarray, thresh: float):
    """lap.lapjv(cost, extend_cost=True, cost_limit=thresh) as used by matching.linear_assignment (matching.py:20-31).
    `lap` (requirements.txt:4, unpinned, not vendored) is absent; its documented behaviour is restated: pad to
    (T+D)x(T+D) with cost_limit/2 in the off blocks and 0 in the dummy block, solve exactly, drop dummy matches.
    Exact for unique optima; tie-breaking of the real library is unpinned.
    A NaN cost (the IoU 0/0 of two zero-area boxes) never matches: `lap` documents nothing for NaN, so the pair is forbidden, as in
    the device solver (csrc/track.cu), and the rest of the problem is solved as if it were absent."""
    from scipy.optimize import linear_sum_assignment
    cost = np.asarray(cost, float)
    nr, nc = cost.shape
    n = nr + nc
    ext = np.full((n, n), thresh / 2.0)
    ext[nr:, nc:] = 0
    ext[:nr, :nc] = np.where(np.isnan(cost), np.inf, cost)
    r, c = linear_sum_assignment(ext)
    x = np.full(n, -1)
    y = np.full(n, -1)
    x[r] = c
    y[c] = r
    x[x >= nc] = -1
    y[y >= nr] = -1
    x, y = x[:nr], y[:nc]
    total = cost[np.nonzero(x != -1)[0], x[x != -1]].sum() + thresh / 2.0 * ((x < 0).sum() + (y < 0).sum())
    return x.astype(np.int32), y.astype(np.int32), float(total)
