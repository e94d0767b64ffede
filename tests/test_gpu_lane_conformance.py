"""GPU: lane decode (UFLD v2 / v1), lane geometry, bird-view warp and frame pre-processing at their edges, against the reference's own
results (tests/golden/lane_conformance.npz, warp_edges.npz) and float64 references with derived bounds (tests/lane_conformance_cases.py)."""
import os

import numpy as np
import pytest

import lane_conformance_cases as lc
import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi
from gpu_util import cached_plan
from oracle import post

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLD, "lane_conformance.npz"))


def _check_v2(pts, npts, status, coords, b, heads, w, h, ra, ca, gold_pts=None, gold_status=None):
    rpts, rst, rcrd, his = lc.v2_reference(heads, w, h, ra, ca)
    assert [bool(v) for v in status[b]] == rst
    if gold_status is not None:
        assert np.array_equal(status[b], gold_status)
    for lane in range(4):
        n = int(npts[b, lane])
        want = np.array(rpts[lane], np.int32).reshape(-1, 2)
        assert n == len(want), (lane, n, len(want))
        if gold_pts is not None:
            assert n == len(gold_pts[lane])
        if n == 0:
            continue
        ng, size, axis = (heads[0].shape[1], w, 0) if lane in (1, 2) else (heads[1].shape[1], h, 1)
        bound = lc.v2_coord_bound(ng, his[lane], size)
        c = coords[b, lane, :n]
        assert np.all(np.abs(c - np.array(rcrd[lane])) <= bound), (lane, float(np.abs(c - rcrd[lane]).max()))
        lc.int_points_agree(pts[b, lane, :n], want, c, bound, axis)
        if gold_pts is not None:
            lc.int_points_agree(pts[b, lane, :n], gold_pts[lane], c, bound, axis)


# ---- 1. UFLD v2 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ds", ["culane", "tusimple"])
def test_v2_decode_matches_reference_golden_at_every_frame_size(gold, ds):
    ngr, ncr, ngc, ncc = lc.V2_GOLDEN_DIMS[ds]
    ra, ca = post.UFLD_ANCHORS[ds]
    hs = lc.v2_golden_heads(ds)
    flat = np.stack([lc.flat_v2(x) for x in hs])
    for w, h in lc.FRAME_SIZES:
        pts, npts, status, coords = _capi.ufld_postprocess(flat, (ngr, ncr, ngc, ncc, 4), (w, h), ra, ca)
        for i, heads in enumerate(hs):
            key = f"v2_{ds}_{i}_{w}x{h}"
            _check_v2(pts, npts, status, coords, i, heads, w, h, ra, ca, [gold[f"{key}_lane{l}"] for l in range(4)], gold[key + "_status"])


@pytest.mark.parametrize("dims", [(200, 72, 100, 81), (100, 56, 100, 41), (50, 18, 50, 41), (2, 128, 2, 128), (5, 3, 4, 3),
                                  (200, 128, 100, 128)], ids=lambda d: "x".join(map(str, d)))
def test_v2_decode_vs_oracle_at_edge_dims_and_batches(dims):
    """Ties, 2-bin windows, p = 1/3 windows, underflowing exp, exist ties, keep counts on the threshold, ncr / ncc = 128 (strided
    thread loop), ngr = 2, 2 vs 3 points (ncr = 3); batches of 1, 3 and 133 (more CTAs than SMs): run(1) of frame k == frame k."""
    ngr, ncr, ngc, ncc = dims
    ra, ca = np.linspace(0.42, 1, ncr), np.linspace(0, 1, ncc)
    B = 133 if ncr in (72, 128) else 3
    keeps = lc.keep_threshold_counts(ncr, ncc)
    if ncr == 3:
        keeps = [(1, 2, 3, 2), (3, 3, 2, 0)]                         # kept with 2 points (status 0) / 3 points (status 1)
    hs = [lc.v2_heads(500 + k, ngr, ncr, ngc, ncc, keep=keeps[k % 2] if k < 4 else None)[0] for k in range(B)]
    flat = np.stack([lc.flat_v2(x) for x in hs])
    w, h = lc.FRAME_SIZES[B % len(lc.FRAME_SIZES)]
    pts, npts, status, coords = _capi.ufld_postprocess(flat, dims + (4,), (w, h), ra, ca)
    for b, heads in enumerate(hs):
        _check_v2(pts, npts, status, coords, b, heads, w, h, ra, ca)
    if ncr == 3:
        assert status[0].tolist() == [0, 0, 1, 0] and npts[0].tolist() == [1, 2, 3, 2]
    for k in (0, B // 2, B - 1):
        one = _capi.ufld_postprocess(flat[k:k + 1], dims + (4,), (w, h), ra, ca)
        for a, full in zip(one, (pts, npts, status, coords)):
            n = npts[k]
            if a.ndim >= 3:
                for lane in range(4):
                    assert np.array_equal(a[0, lane, :n[lane]], full[k, lane, :n[lane]])
            else:
                assert np.array_equal(a[0], full[k])


@pytest.mark.parametrize("dims", [(200, 129, 100, 81), (200, 72, 100, 129), (1, 72, 100, 81), (200, 72, 1, 81)])
def test_v2_decode_refuses_bad_dims(dims):
    heads = np.zeros((1, dims[0] * dims[1] * 4 + dims[2] * dims[3] * 4 + 8 * dims[1] + 8 * dims[3]), np.float32)
    with pytest.raises(Exception):
        _capi.ufld_postprocess(heads, dims + (4,), (1280, 720), np.linspace(0, 1, dims[1]), np.linspace(0, 1, dims[3]))


# ---- 2. UFLD v1 -------------------------------------------------------------------------------------------------------------------
def _check_v1(pts, npts, status, coords, b, head, cfg, w, h, gold_pts=None, gold_status=None):
    rpts, rst, _ = post.ufld_v1_decode(head[0], cfg, 800, 288, w, h)
    assert [bool(v) for v in status[b]] == rst
    if gold_status is not None:
        assert np.array_equal(status[b], gold_status)
    w_ratio = w / cfg["img_w"]
    for lane in range(4):
        n = int(npts[b, lane])
        want = np.array(rpts[lane], np.int32).reshape(-1, 2)
        assert n == len(want)
        if n:
            x = coords[b, lane, :n]
            bound = lc.v1_x_bound(cfg["griding_num"], x, w_ratio)
            lc.int_points_agree(pts[b, lane, :n], want, x, bound, 0)
            if gold_pts is not None:
                lc.int_points_agree(pts[b, lane, :n], gold_pts[lane], x, bound, 0)


def test_v1_decode_matches_reference_golden_at_every_frame_size(gold):
    for ds, G, R in lc.V1_GOLDEN:
        cfg = post.UFLD_V1[ds]
        hs = lc.v1_golden_heads(G, R)
        head = np.concatenate(hs)
        for w, h in lc.FRAME_SIZES:
            pts, npts, status, coords = _capi.ufld_v1_postprocess(head, G, R, (800, 288), (cfg["img_w"], cfg["img_h"]), (w, h),
                                                                  np.asarray(cfg["row_anchor"], np.float64))
            for i, hd in enumerate(hs):
                key = f"v1_{ds}_{i}_{w}x{h}"
                _check_v1(pts, npts, status, coords, i, hd, cfg, w, h, [gold[f"{key}_lane{l}"] for l in range(4)], gold[key + "_status"])


@pytest.mark.parametrize("G,R,B", [(3, 18, 3), (100, 56, 133), (200, 128, 3), (3, 128, 133)])
def test_v1_decode_vs_oracle_at_edge_dims_and_batches(G, R, B):
    cfg = dict(img_w=1280, img_h=720, griding_num=G, cls_num_per_lane=R, row_anchor=np.linspace(64, 284, R))
    hs = [lc.v1_head(600 + k, G, R, nonzero=((2, 3, None, 2) if k % 3 == 1 else None))[0] for k in range(B)]
    head = np.concatenate(hs)
    w, h = lc.FRAME_SIZES[B % len(lc.FRAME_SIZES)]
    out = _capi.ufld_v1_postprocess(head, G, R, (800, 288), (1280, 720), (w, h), cfg["row_anchor"])
    for b in range(B):
        _check_v1(*out, b, hs[b], cfg, w, h)
    one = _capi.ufld_v1_postprocess(head[B - 1:], G, R, (800, 288), (1280, 720), (w, h), cfg["row_anchor"])
    assert np.array_equal(one[1][0], out[1][B - 1]) and np.array_equal(one[2][0], out[2][B - 1])
    for lane in range(4):
        n = out[1][B - 1, lane]
        assert np.array_equal(one[0][0, lane, :n], out[0][B - 1, lane, :n])


@pytest.mark.parametrize("G,R", [(2, 18), (100, 129)])
def test_v1_decode_refuses_bad_dims(G, R):
    with pytest.raises(Exception):
        _capi.ufld_v1_postprocess(np.zeros((1, G + 1, R, 4), np.float32), G, R, (800, 288), (1280, 720), (1280, 720), np.linspace(64, 284, R))


# ---- 3. lane geometry -------------------------------------------------------------------------------------------------------------
def _geom_inputs(gold, c):
    pts, npts, status = lc.lanes_to_arrays([[[], c["left"], c["right"], []]], [[0, 1, 1, 0]], lc.GEOM_MP)
    M = None if c["M"] is None else (gold["M_default"] if c["M"] == "default" else np.eye(3))
    return pts, npts, status, M


@pytest.mark.parametrize("adjust", [False, True])
def test_lane_geometry_matches_reference_golden(gold, adjust):
    """Polygon, bird-view points, direction, curvature and offset of every crafted case.  Curvature and offset are compared with the
    reference's numbers when the device's bird-view points equal the reference's; where one point lies on the other side of an integer
    (allowed by the point bound), the fits see different data, so they are compared with the float64 restatement on the device's own
    points instead.  Both comparisons use the derived bounds; at least 15 of the 19 curvature cases must be the golden one."""
    n_golden = n_own = 0
    for c in lc.geom_cases():
        key = "geom_" + c["name"]
        pts, npts, status, M = _geom_inputs(gold, c)
        r = _capi.lane_geometry(pts, npts, status, c["img_wh"], adjust_lanes=adjust, M=M, bird_wh=c["bird_wh"])[0]
        assert r["area_status"]
        if adjust and key + "_area_adj" in gold.files:
            lc.check_adjusted_area(r["area"], gold[key + "_area_adj"], lc.adjust_reference(c["left"], c["right"], c["img_wh"][1]))
        else:
            assert np.array_equal(r["area"], np.vstack([np.asarray(c["left"]), np.asarray(c["right"])[::-1]])), key
        if M is None:
            assert r["bird"] is None
            continue
        for side, lane in (("_bl", c["left"]), ("_br", c["right"])):
            want, f, bn = lc.bird_points_reference(M, lane)
            got = r["bird"][1 if side == "_bl" else 2].astype(np.int64)
            gw = gold[key + side]
            d = np.abs(got - gw)
            assert d.max() <= 1 and np.all((d == 0) | (np.abs(f - np.round(f)) <= bn)), key
        want = gold[key + "_curve"]
        if np.isnan(want[0]):
            assert r["direction"] is None and r["curvature"] is None, key          # bird_h < 720: no curvature
            continue
        bl, br = gold[key + "_bl"], gold[key + "_br"]
        if np.array_equal(r["bird"][1], bl) and np.array_equal(r["bird"][2], br):
            d, curv, off, bc, bo, _ = lc.curve_reference(bl, br, c["bird_wh"][1], c["bird_wh"][0])
            assert {"L": -1.0, "F": 0.0, "R": 1.0}[r["direction"]] == want[0], key
            assert abs(r["curvature"] - want[1]) <= bc + abs(curv - want[1]), (key, r["curvature"], want[1], bc)
            assert abs(r["offset"] - want[2]) <= bo + abs(off - want[2]), (key, r["offset"], want[2], bo)
            n_golden += 1
        else:
            d, curv, off, bc, bo, _ = lc.curve_reference(r["bird"][1], r["bird"][2], c["bird_wh"][1], c["bird_wh"][0])
            assert r["direction"] == d, key
            assert abs(r["curvature"] - curv) <= bc and abs(r["offset"] - off) <= bo, (key, r["curvature"] - curv, bc, r["offset"] - off, bo)
            n_own += 1
    print(f"[lane geometry] curvature cases vs the reference {n_golden}, vs the restatement on the device's points {n_own}")
    assert n_golden >= 15 and n_golden + n_own == 19


def test_lane_geometry_two_points_and_bird_view_limits(gold):
    """2 points per ego lane: no curvature (the reference's rank-deficient fit is not reproduced); a 2160-row bird view computes one; a
    2161-row bird view is refused."""
    c = [c for c in lc.geom_cases() if c["name"] == "three_points"][0]
    pts, npts, status, M = _geom_inputs(gold, c)
    npts[0, 1] = 2
    r = _capi.lane_geometry(pts, npts, status, (1280, 720), M=M)[0]
    assert r["direction"] is None and len(r["bird"][1]) == 2
    c = [c for c in lc.geom_cases() if c["name"] == "bird_h2160"][0]
    pts, npts, status, M = _geom_inputs(gold, c)
    assert _capi.lane_geometry(pts, npts, status, (1280, 720), M=M, bird_wh=(1280, 2160))[0]["direction"] is not None
    with pytest.raises(Exception):
        _capi.lane_geometry(pts, npts, status, (1280, 720), M=M, bird_wh=(1280, 2161))


def test_lane_geometry_ragged_batch_of_133_equals_single_frames(gold):
    cases = lc.geom_cases()
    lanes, st, Ms = [], [], []
    for f in range(133):
        c = cases[f % len(cases)]
        n = (0, 2, 3, 11, lc.GEOM_MP)[f % 5]
        left = c["left"][:n] if n < len(c["left"]) else c["left"]
        lanes.append([[], left, c["right"], c["right"][:2]])
        st.append([0, int(len(left) > 2), 1, 0])
        Ms.append(gold["M_default"])
    pts, npts, status = lc.lanes_to_arrays(lanes, st, lc.GEOM_MP)
    for adjust in (False, True):
        res = _capi.lane_geometry(pts, npts, status, (1280, 720), adjust_lanes=adjust, M=np.stack(Ms))
        for f in (0, 1, 2, 3, 4, 66, 131, 132):
            one = _capi.lane_geometry(pts[f:f + 1], npts[f:f + 1], status[f:f + 1], (1280, 720), adjust_lanes=adjust, M=Ms[f])[0]
            r = res[f]
            assert r["area_status"] == one["area_status"] and np.array_equal(r["area"], one["area"])
            assert all(np.array_equal(a, b) for a, b in zip(r["bird"], one["bird"]))
            assert (r["direction"], r["curvature"], r["offset"]) == (one["direction"], one["curvature"], one["offset"])


def test_engine_warp_and_lane_geometry_interleaved_equal_standalone_calls():
    """The per-frame order detect -> bird-view warp -> lane geometry -> warp ...: the geometry call allocating (or growing) its buffers
    must leave the warp scratch alone, and every result equals the standalone call."""
    path, _, _ = cached_plan("ufldv2", backbone="18", cfg="culane")
    eng = _capi.Engine(path, 0, max_batch=2)
    frames = np.stack([synth.frame(s) for s in (5, 6)])
    pts, npts, status, _ = eng.ufld_detect(frames)
    M = np.load(os.path.join(GOLD, "lane_conformance.npz"))["M_default"]
    want_warp = _capi.warp_perspective(frames, M, (1280, 720))
    assert np.array_equal(eng.warp_perspective(2, M, (1280, 720)), want_warp)
    for adjust in (False, True):                                         # adjust grows cap_area: a second allocation
        a = eng.lane_geometry(2, (1280, 720), adjust_lanes=adjust, M=M)
        b = _capi.lane_geometry(pts, npts, status, (1280, 720), adjust_lanes=adjust, M=M)
        for ra, rb in zip(a, b):
            assert ra["area_status"] == rb["area_status"] and np.array_equal(ra["area"], rb["area"])
            assert all(np.array_equal(x, y) for x, y in zip(ra["bird"], rb["bird"]))
            assert (ra["direction"], ra["curvature"], ra["offset"]) == (rb["direction"], rb["curvature"], rb["offset"])
        assert np.array_equal(eng.warp_perspective(2, M, (1280, 720)), want_warp)
    # the resident frames at the block-width edges and the edge matrices; the growing sizes reallocate the warp scratch
    for mname, dsize, batch in (("identity", (1, 1), 1), ("past_int16", (7, 3), 2), ("persp", (2000, 5), 2), ("horizon", (4096, 16), 1),
                                ("behind", (333, 720), 2), ("huge_scale", (1280, 1440), 2), ("half_step", (64, 15), 2)):
        Mw = lc.WARP_MATRICES[mname]
        got = eng.warp_perspective(batch, Mw, dsize)
        assert np.array_equal(got, _capi.warp_perspective(frames[:batch], Mw, dsize)), (mname, dsize)
    eng.close()


# ---- 4. bird-view warp ------------------------------------------------------------------------------------------------------------
def test_warp_matches_cv2_hashes_at_block_width_edges():
    g = np.load(os.path.join(GOLD, "warp_edges.npz"))
    try:
        import cv2
    except Exception:
        cv2 = None
    bad = []
    for name, seed, (h, w), mname, dsize in lc.warp_cases():
        src = lc.warp_source(seed, h, w)
        out = _capi.warp_perspective(src[None], lc.WARP_MATRICES[mname], dsize)[0]
        if not np.array_equal(lc.sha(out), g[name]):
            bad.append(name)
        if cv2 is not None and dsize[0] * dsize[1] < 100000:
            assert np.array_equal(out, cv2.warpPerspective(src, lc.WARP_MATRICES[mname], dsize, flags=cv2.INTER_LINEAR)), name
    assert not bad, bad
    Ms = lc.warp_batch_matrices()
    frames = np.stack([lc.warp_source(100 + b, 480, 640) for b in range(len(Ms))])
    out = _capi.warp_perspective(frames, Ms, (333, 97))
    assert [b for b in range(len(Ms)) if not np.array_equal(lc.sha(out[b]), g[f"batch_{b}"])] == []


# ---- 5. pre-processing ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,ih,iw", lc.YOLO_PRE_CASES)
def test_yolo_preprocess_bit_exact_at_edges(h, w, ih, iw):
    fr = np.stack([lc.warp_source(h + s, h, w) for s in (0, 1)])
    blob = _capi.yolo_preprocess(fr, (ih, iw))
    for b in range(2):
        assert np.array_equal(blob[b], post.yolo_prepare_input(fr[b], ih, iw)[0][0])


@pytest.mark.parametrize("h,w,ih,iw,crop", lc.UFLD_PRE_CASES)
def test_ufld_preprocess_bit_exact_at_edges(h, w, ih, iw, crop):
    fr = lc.warp_source(w, h, w)[None]
    assert np.array_equal(_capi.ufld_preprocess(fr, (ih, iw), crop)[0], post.ufld_prepare_input(fr[0], ih, iw, crop)[0])


def test_yolo_preprocess_refuses_an_empty_letterbox():
    with pytest.raises(Exception):
        _capi.yolo_preprocess(np.zeros((1, 700, 1, 3), np.uint8), (640, 640))
    assert _capi.yolo_preprocess(np.zeros((1, 600, 1, 3), np.uint8), (640, 640)).shape == (1, 3, 640, 640)


def _check_image_buffer(eng, blobs, batch, sentinel):
    """Plan buffer 0 after a detect call at batch < max_batch: channels 0-2 = fp16(blob), the rest 0, the one-pixel halo 0, the images
    past the batch untouched."""
    bi = eng.buffer_info(0)
    H, W, C = bi["H"], bi["W"], bi["C"]
    buf = eng.read_buffer(0, eng.max_batch).reshape(eng.max_batch, H + 2, W + 2, C)
    for b in range(batch):
        want = blobs[b].transpose(1, 2, 0).astype(np.float16)
        assert np.array_equal(buf[b, 1:-1, 1:-1, :3].view(np.uint16), want.view(np.uint16)), b
        assert not buf[b, 1:-1, 1:-1, 3:].any()
        assert not (buf[b, 0].any() or buf[b, -1].any() or buf[b, :, 0].any() or buf[b, :, -1].any())
    assert np.array_equal(buf[batch:].view(np.uint16), sentinel[batch:].view(np.uint16))


def _poison(eng):
    bi = eng.buffer_info(0)
    H, W, C = bi["H"], bi["W"], bi["C"]
    s = np.zeros((eng.max_batch, H + 2, W + 2, C), np.float16)
    c = min(C, 4)                                    # the channels the pre-processing kernels write
    s[:, 1:-1, 1:-1, :c] = np.random.default_rng(3).uniform(-9, 9, (eng.max_batch, H, W, c)).astype(np.float16)
    eng.write_buffer(0, s.reshape(-1, C))
    return s


@pytest.mark.parametrize("hw", [(720, 1280), (900, 500)])
def test_engine_resident_fp16_image_of_every_detect_call(hw):
    ypath, _, _ = cached_plan("yolov5", scale="n")
    upath, _, _ = cached_plan("ufldv2", backbone="18", cfg="culane")
    yolo = _capi.Engine(ypath, 0, max_batch=3)
    ufld = _capi.Engine(upath, 0, max_batch=3)
    frames = np.stack([synth.frame(s, *hw) for s in (1, 2)])
    yb = [post.yolo_prepare_input(f, 640, 640)[0][0] for f in frames]
    ub = [post.ufld_prepare_input(f, 320, 1600, 0.6)[0] for f in frames]
    s = _poison(yolo)
    yolo.yolo_detect(frames, 0.4, 0.45)
    _check_image_buffer(yolo, yb, 2, s)
    s = _poison(ufld)
    ufld.ufld_detect(frames)
    _check_image_buffer(ufld, ub, 2, s)
    sy, su = _poison(yolo), _poison(ufld)
    _capi.detect_pair(yolo, ufld, frames, 0.4, 0.45)
    _check_image_buffer(yolo, yb, 2, sy)
    _check_image_buffer(ufld, ub, 2, su)
    yolo.close()
    ufld.close()
