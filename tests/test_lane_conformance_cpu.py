"""CPU side of the lane conformance suite (tests/lane_conformance_cases.py): the generators hit their cases, the references agree with
the committed reference goldens, and the bounds and hashes reject deliberately wrong emulations."""
import os

import numpy as np
import pytest

import lane_conformance_cases as lc
from oracle import post

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cv2():
    try:
        import cv2
        return cv2
    except Exception:
        pytest.skip("cv2 not importable")


# ---- 1. UFLD v2 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [(200, 72, 100, 81), (100, 56, 100, 41), (5, 18, 4, 41), (2, 128, 2, 128)])
def test_v2_generator_hits_its_cases(dims):
    ngr, ncr, ngc, ncc = dims
    heads, meta = lc.v2_heads(1, ngr, ncr, ngc, ncc)
    loc_row, loc_col, ex_row, ex_col = heads
    seen = set()
    for (lane, a), m in meta["argmax"].items():
        loc, ex = (loc_row, ex_row) if lane in (1, 2) else (loc_col, ex_col)
        col = loc[0, :, a, lane]
        assert int(col.argmax()) == m, (lane, a, meta["loc_case"][(lane, a)])
        assert bool(ex[0, 1, a, lane] > ex[0, 0, a, lane]) == meta["valid"][(lane, a)]
        seen.add(meta["loc_case"][(lane, a)])
        seen.add(meta["exist_case"][(lane, a)])
        case = meta["loc_case"][(lane, a)]
        if case == "equal_window" and 0 < m < len(col) - 1:
            e = np.exp(col[m - 1:m + 2] - col[m])
            assert np.all(e == np.float32(1.0))                         # p = 1/3 exactly as the kernel sees it
        if case == "sharp_zero" and len(col) > 2:
            assert np.exp(np.float32(-120.0)) == 0
        if case == "sharp_subnormal":
            assert 0 < np.exp(np.float32(-95.0)) < lc.F32_MIN_NORMAL
        if case in ("edge0", "edge_last"):
            assert m in (0, len(col) - 1)
    if ncr >= 18:
        assert seen >= set(lc.LOC_CASES) | set(lc.EXIST_VALID) | set(lc.EXIST_INVALID), seen


@pytest.mark.parametrize("ncr,ncc", [(72, 81), (56, 41), (18, 41)])
def test_v2_keep_threshold_counts_sit_on_the_threshold(ncr, ncc):
    for keep in lc.keep_threshold_counts(ncr, ncc):
        heads, _ = lc.v2_heads(2, 50, ncr, 50, ncc, keep=keep)
        pts, status, _ = post.ufld_decode(heads, 1280, 720, np.linspace(0.4, 1, ncr), np.linspace(0, 1, ncc))
        for lane in range(4):
            n, thr = keep[lane], (ncr / 2 if lane in (1, 2) else ncc / 4)
            assert (len(pts[lane]) > 0) == (n > thr) and abs(n - thr) <= 1, (lane, n, thr)


def test_v2_oracle_matches_reference_golden():
    g = np.load(os.path.join(GOLD, "lane_conformance.npz"))
    for ds in ("culane", "tusimple"):
        ra, ca = post.UFLD_ANCHORS[ds]
        for i, heads in enumerate(lc.v2_golden_heads(ds)):
            for w, h in lc.FRAME_SIZES:
                pts, status, _ = post.ufld_decode(heads, w, h, ra, ca)
                key = f"v2_{ds}_{i}_{w}x{h}"
                for l in range(4):
                    assert np.array_equal(np.array(pts[l], np.int32).reshape(-1, 2), g[f"{key}_lane{l}"]), (key, l)
                assert np.array_equal(np.array(status, np.uint8), g[key + "_status"])


def _f32_decode(heads, img_w, img_h, ra, ca, off=0, ge=False, swap=False):
    """A float32 emulation of the kernel, optionally wrong: softmax window shifted by `off`, a >= keep test, lanes 1 / 2 swapped."""
    loc_row, loc_col, ex_row, ex_col = heads
    res = {}
    for lane in range(4):
        part = 0 if lane in (1, 2) else 1
        src = (3 - lane if lane in (1, 2) else lane) if swap else lane
        loc, ex = (loc_row, ex_row) if part == 0 else (loc_col, ex_col)
        ng, nc = loc.shape[1], loc.shape[2]
        valid = ex[0, 1, :, src] > ex[0, 0, :, src]
        thr = nc / 2 if part == 0 else nc / 4
        keep = valid.sum() >= thr if ge else valid.sum() > thr
        c = []
        if keep:
            for k in np.nonzero(valid)[0]:
                col = loc[0, :, k, src]
                m = int(col.argmax()) + off
                lo, hi = max(0, m - 1), min(ng - 1, m + 1)
                e = np.exp(col[lo:hi + 1] - col.max())
                p = e / np.float32(e.sum(dtype=np.float32))
                c.append(((p.astype(np.float64) * np.arange(lo, hi + 1)).sum() + 0.5) / (ng - 1) * (img_w if part == 0 else img_h))
        res[lane] = np.array(c)
    return res


def test_v2_coordinate_bound_has_teeth():
    """A float32 emulation passes the coordinate bound; a window off by one, a >= keep test and swapped ego lanes fail it (or the
    point counts)."""
    heads, _ = lc.v2_heads(5, 200, 72, 100, 81, keep=lc.keep_threshold_counts(72, 81)[0])
    ra, ca = post.UFLD_ANCHORS["culane"]
    w, h = 3840, 2160
    _, _, crd, his = lc.v2_reference(heads, w, h, ra, ca)

    def ok(emu):
        for lane in range(4):
            size, ng = (w, 200) if lane in (1, 2) else (h, 100)
            if len(emu[lane]) != len(crd[lane]):
                return False
            if len(crd[lane]) and np.any(np.abs(emu[lane] - np.array(crd[lane])) > lc.v2_coord_bound(ng, his[lane], size)):
                return False
        return True
    assert ok(_f32_decode(heads, w, h, ra, ca))
    assert not ok(_f32_decode(heads, w, h, ra, ca, off=1))
    assert not ok(_f32_decode(heads, w, h, ra, ca, ge=True))
    assert not ok(_f32_decode(heads, w, h, ra, ca, swap=True))
    # the derived bound, not 1e-3 px, is what holds at 4K
    assert lc.v2_coord_bound(200, 199, 3840) > 1e-3 > lc.v2_coord_bound(200, 199, 320)


# ---- 2. UFLD v1 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G,R", [(3, 18), (100, 56), (200, 128)])
def test_v1_generator_hits_its_cases(G, R):
    head, cases = lc.v1_head(3, G, R)
    cfg = dict(img_w=1280, img_h=720, griding_num=G, cls_num_per_lane=R, row_anchor=np.linspace(64, 284, R))
    _, _, loc = post.ufld_v1_decode(head[0], cfg, 800, 288, 1280, 720)
    for (lane, r), case in cases.items():
        p = R - 1 - r                                              # the decode reverses the rows
        if case in ("none", "none_ulp_above"):
            assert loc[p, lane] == 0, (lane, r, case)
        else:
            assert loc[p, lane] > 0, (lane, r, case)
    assert set(cases.values()) == set(lc.V1_CASES)
    head, _ = lc.v1_head(4, G, R, nonzero=(2, 3, None, 2))
    _, status, loc = post.ufld_v1_decode(head[0], cfg, 800, 288, 1280, 720)
    assert (loc[:, 0] != 0).sum() == 2 and (loc[:, 1] != 0).sum() == 3 and status[:2] == [False, True]


def test_v1_oracle_matches_reference_golden():
    g = np.load(os.path.join(GOLD, "lane_conformance.npz"))
    for ds, G, R in lc.V1_GOLDEN:
        cfg = post.UFLD_V1[ds]
        for i, head in enumerate(lc.v1_golden_heads(G, R)):
            for w, h in lc.FRAME_SIZES:
                pts, status, _ = post.ufld_v1_decode(head[0], cfg, 800, 288, w, h)
                key = f"v1_{ds}_{i}_{w}x{h}"
                assert np.array_equal(np.array(status, np.uint8), g[key + "_status"]), key
                for l in range(4):
                    assert np.array_equal(np.array(pts[l], np.int32).reshape(-1, 2), g[f"{key}_lane{l}"]), (key, l)


# ---- 3. lane geometry -------------------------------------------------------------------------------------------------------------
def test_geometry_references_match_reference_golden_and_bounds_have_teeth():
    """The float64 restatements agree with the reference's own results within the derived bounds; the adjusted-polygon check rejects a
    fit with one point dropped on either side."""
    g = np.load(os.path.join(GOLD, "lane_conformance.npz"))
    n_adj = n_curve = 0
    for c in lc.geom_cases():
        key = "geom_" + c["name"]
        if key + "_area_adj" in g.files:
            ref = lc.adjust_reference(c["left"], c["right"], c["img_wh"][1])
            want = g[key + "_area_adj"]
            lc.check_adjusted_area(np.concatenate([np.stack([r["x"][r["keep"]].astype(np.int64), r["y"][r["keep"]].astype(np.int64)], 1)
                                                   [::1 if s == 0 else -1] for s, r in enumerate(ref)]), want, ref)
            n_adj += 1
        if key + "_curve" in g.files:
            M = g["M_default"] if c["M"] == "default" else np.eye(3)
            bl, fl, bnl = lc.bird_points_reference(M, c["left"])
            br, fr, bnr = lc.bird_points_reference(M, c["right"])
            for got, f, bn, want in ((bl, fl, bnl, g[key + "_bl"]), (br, fr, bnr, g[key + "_br"])):
                d = np.abs(got - want)
                assert d.max() <= 1 and np.all((d == 0) | (np.abs(f - np.round(f)) <= bn)), key
            bl, br = g[key + "_bl"], g[key + "_br"]
            want = g[key + "_curve"]
            if np.isnan(want[0]):
                assert c["bird_wh"][1] < 720
                continue
            d, curv, off, bc, bo, _ = lc.curve_reference(bl, br, c["bird_wh"][1], c["bird_wh"][0])
            assert {"L": -1.0, "F": 0.0, "R": 1.0}[d] == want[0], key
            assert abs(curv - want[1]) <= bc and abs(off - want[2]) <= bo, (key, curv - want[1], bc, off - want[2], bo)
            n_curve += 1
    assert n_adj >= 8 and n_curve >= 15
    # teeth: the adjusted polygon of a lane fitted without its last point, or with x and y swapped, fails the check
    c = [c for c in lc.geom_cases() if c["name"] == "adj_72_72"][0]
    ref = lc.adjust_reference(c["left"], c["right"], 720)
    want = g["geom_adj_72_72_area_adj"]
    for wrong in (lc.adjust_reference(c["left"][:-1], c["right"], 720), lc.adjust_reference(c["left"], c["right"][::-1][:-1], 720)):
        got = np.concatenate([np.stack([r["x"][r["keep"]].astype(np.int64), r["y"][r["keep"]].astype(np.int64)], 1)[::1 if s == 0 else -1]
                              for s, r in enumerate(wrong)])
        with pytest.raises(AssertionError):
            lc.check_adjusted_area(got, want, ref)


def _pixel_fits():
    """(name, y, x) of every pixel fit x(y) the geometry cases hand the kernel (the adjust fits; with M = identity the bird-view fits
    see the same points)."""
    for c in lc.geom_cases():
        for side, lane in (("left", c["left"]), ("right", c["right"])):
            p = np.asarray(lane, np.float64)
            if len(p) >= 3:
                yield f"{c['name']}/{side}", p[:, 1], p[:, 0]


def test_polyfit_bound_rejects_polyfit_without_its_column_scaling():
    """np.polyfit divides the Vandermonde columns [y^2, y, 1] by their norms before its SVD solve (lstsq, rcond = len(x) eps).  The
    same solve without that scaling is accurate only to about kappa(unscaled) U: on the 5-point direction lanes (y = 0 .. 40000,
    singular-value ratio 5.6e-10 unscaled) it lands 2 to 36 times outside the bound on a coefficient."""
    eps = np.finfo(np.float64).eps
    outside = []
    for name, y, x in _pixel_fits():
        dc, fit = lc.polyfit_perturbation(y, x)
        assert np.all(np.abs(np.polyfit(y, x, 2) - fit) <= dc), name
        A = np.stack([y * y, y, np.ones_like(y)], 1)
        unscaled = np.linalg.lstsq(A, x, rcond=len(y) * eps)[0]
        if np.any(np.abs(unscaled - fit) > dc):
            outside.append(name)
    # only the widely spread direction lanes are conditioned badly enough unscaled; the frontal lanes (y < 1101) are not
    assert {"dir_L/right", "dir_R/left", "dir_R/right"} <= set(outside) and all(n.startswith("dir_") for n in outside), outside


def test_polyfit_bound_does_not_separate_backward_stable_unscaled_solvers():
    """The limit of the bound, pinned: Householder QR (the kernel's method) is invariant to column scaling up to rounding, and the float64
    normal equations on these exactly quadratic or near-quadratic lanes stay accurate too, so at every conditioning these cases reach an
    unscaled QR or normal-equation solve lands inside the bound.  A kernel that dropped its column scaling would pass; the bound only
    rejects solvers whose error grows with the unscaled condition number, like the SVD solve above."""
    worst = 0.0
    for name, y, x in _pixel_fits():
        dc, fit = lc.polyfit_perturbation(y, x)
        A = np.stack([y * y, y, np.ones_like(y)], 1)
        q, r = np.linalg.qr(A)
        for z in (np.linalg.solve(r, q.T @ x), np.linalg.solve(A.T @ A, A.T @ x)):
            worst = max(worst, float(np.max(np.abs(z - fit) / dc)))
    assert worst <= 1.0, worst


def test_geometry_generators_hit_their_cases(golden_dir):
    cs = {c["name"]: c for c in lc.geom_cases()}
    # negative_fit: the fitted x of the resampled rows goes below 0, and those rows are dropped
    left, _ = lc.adjust_reference(cs["negative_fit"]["left"], cs["negative_fit"]["right"], 720)
    assert ((left["x"] < 0) & (left["y"] >= min(p[1] for p in cs["negative_fit"]["left"]))).sum() > 100
    # top_row: min(lefty) < H // 3, so the first resampled row is exactly min(lefty), and it is kept
    left, _ = lc.adjust_reference(cs["top_row"]["left"], cs["top_row"]["right"], 720)
    ymin = min(p[1] for p in cs["top_row"]["left"])
    assert ymin < 720 // 3 and left["y"][0] == ymin and left["keep"][0]
    # above_trapezoid: the default matrix's w is <= 0 for many of the points (behind the bird view's horizon)
    M = np.load(os.path.join(golden_dir, "lane_conformance.npz"))["M_default"]
    for lane in (cs["above_trapezoid"]["left"], cs["above_trapezoid"]["right"]):
        p = np.asarray(lane, np.float64)
        assert (M[2, 0] * p[:, 0] + M[2, 1] * p[:, 1] + M[2, 2] <= 0).sum() > 20
    # adjust switch: 10 / 11 points on each side; the largest lanes
    for name in ("adj_10_10", "adj_10_11", "adj_11_10", "adj_11_11", "adj_72_72", "adj_128_128"):
        nl, nr = map(int, name.split("_")[1:])
        assert (len(cs[name]["left"]), len(cs[name]["right"])) == (nl, nr)
    # direction lanes: the pixel fit's leading coefficient sits 1e-7 past or short of +-0.00015
    for name, a in (("dir_L", -0.0001501), ("dir_F_short_L", -0.0001499), ("dir_R", 0.0001501), ("dir_F_short_R", 0.0001499)):
        lane = cs[name]["left" if a < 0 else "right"]
        p = np.asarray(lane, np.float64)
        assert abs(np.polyfit(p[:, 1], p[:, 0], 2)[0] - a) < 1e-12
    # resampled-row counts that are not multiples of the kernel's 128-row chunks
    assert any(c["img_wh"][1] % 128 for c in cs.values()) and {480, 720, 1080, 1100, 1101} <= {c["img_wh"][1] for c in cs.values()}


# ---- 4. warp ------------------------------------------------------------------------------------------------------------------------
def test_warp_restatement_equals_cv2_and_the_goldens():
    cv2 = _cv2()
    g = np.load(os.path.join(GOLD, "warp_edges.npz"))
    n = 0
    for name, seed, (h, w), mname, dsize in lc.warp_cases():
        if dsize[1] == 720 and dsize[0] > 333:
            continue                                              # the large outputs are checked on the device against the hashes
        src = lc.warp_source(seed, h, w)
        got = lc.warp_emulate(src, lc.WARP_MATRICES[mname], dsize)
        assert np.array_equal(got, cv2.warpPerspective(src, lc.WARP_MATRICES[mname], dsize, flags=cv2.INTER_LINEAR)), name
        assert np.array_equal(lc.sha(got), g[name]), name
        n += 1
    assert n > 200


@pytest.mark.parametrize("mutation", [dict(bw0_fixed=64), dict(half_away=True), dict(wrap_int16=True), dict(clamp_taps=True)])
def test_warp_hashes_catch_each_mutation(mutation):
    g = np.load(os.path.join(GOLD, "warp_edges.npz"))
    changed = []
    for name, seed, (h, w), mname, dsize in lc.warp_cases():
        if dsize[1] == 720 and dsize[0] > 333:
            continue
        got = lc.warp_emulate(lc.warp_source(seed, h, w), lc.WARP_MATRICES[mname], dsize, **mutation)
        if not np.array_equal(lc.sha(got), g[name]):
            changed.append(name)
    assert changed, mutation


# ---- 5. pre-processing --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sh,sw,dh,dw", lc.RESIZE_SIZES + [(1280, 1280, 640, 640), (1920, 1920, 640, 640), (48, 32, 640, 427)])
def test_resize_restatement_equals_cv2(sh, sw, dh, dw):
    """oracle.post.resize_linear_u8 == cv2.resize(INTER_LINEAR) bit for bit, including exact 2x and 3x square downscales, where cv2
    takes its INTER_AREA route for INTER_LINEAR: the fixed-point bilinear weights are 1/2 and 1/2 there, so the results coincide."""
    cv2 = _cv2()
    src = np.random.default_rng(sh * 7 + sw).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    assert np.array_equal(post.resize_linear_u8(src, dw, dh), cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR))


def test_letterbox_geometry_edges():
    """Portrait frames letterbox left / right, landscape frames top / bottom (with the reference's + 1); a frame more than in_w times
    taller than wide letterboxes to 0 columns (refused by the device)."""
    g = post.letterbox_geom(900, 500, 640, 640)
    assert g["new"] == (640, 355) and g["pad"] == (0, 142)
    g = post.letterbox_geom(500, 900, 640, 640)
    assert g["new"] == (356, 640) and g["pad"] == (142, 0)
    assert post.letterbox_geom(700, 1, 640, 640)["new"][1] == 0
    assert all(post.letterbox_geom(h, w, ih, iw)["new"][1] >= 1 for h, w, ih, iw in lc.YOLO_PRE_CASES)
