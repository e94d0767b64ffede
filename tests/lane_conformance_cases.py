"""Generators, float64 references and per-element bounds for the lane side: UFLD v2 / v1 decode, lane geometry, bird-view warp and
frame pre-processing (tests/test_gpu_lane_conformance.py runs them on the device, tests/test_lane_conformance_cpu.py shows that
the generators hit their cases and that the bounds have teeth).

Units: u = 2**-24, the unit roundoff of float32; U = 2**-53, that of float64.  An ulp of a float32 in [2^k, 2^(k+1)) is 2u * 2^(k+1)
at most, i.e. at most 2u relative.
"""
import hashlib

import numpy as np

from oracle import post

u = 2.0 ** -24
U = 2.0 ** -53
F32_MIN_NORMAL = float(np.finfo(np.float32).tiny)


def f32_next(x, direction):
    return np.nextafter(np.float32(x), np.float32(direction), dtype=np.float32)


# =================================================================================================================================
# 1. UFLD v2 decode
# =================================================================================================================================
# loc cases, applied to one (anchor, lane) column of the grid axis; each names the edge of the decode it reaches
LOC_CASES = ("ridge", "edge0", "edge_last", "tie", "flat", "equal_window", "sharp_zero", "sharp_subnormal")
# exist cases: (exist[0], exist[1]) of one anchor; valid iff exist[1] > exist[0]
EXIST_VALID = ("clear", "ulp_above")
EXIST_INVALID = ("clear_low", "tie", "ulp_below")


def _loc_column(rng, ng, case):
    """One column of the grid axis (float32) and the grid index the kernel's first-maximum argmax must return."""
    v = rng.normal(-4.0, 1.0, ng).astype(np.float32)
    m = int(rng.integers(1, ng - 1)) if ng > 2 else 0
    if case == "ridge":
        v[m] = np.float32(6.0 + rng.random())
    elif case == "edge0":
        m = 0
        v[0] = np.float32(7.0)                        # 2-bin window {0, 1}
    elif case == "edge_last":
        m = ng - 1
        v[m] = np.float32(7.0)                        # 2-bin window {ng-2, ng-1}
    elif case == "tie":
        b = min(ng - 1, m + 1 + int(rng.integers(0, max(1, ng - m - 1))))
        if b == m:
            m, b = 0, ng - 1
        v[m] = v[b] = np.float32(5.5)                 # equal maxima: the first wins
    elif case == "flat":
        v[:] = np.float32(0.25)                       # every bin the maximum: argmax 0, window {0, 1}, p = 1/2
        m = 0
    elif case == "equal_window":
        if ng < 3:
            m = 0
            v[:] = np.float32(1e-3)
        else:
            m = max(1, min(m, ng - 2))
            v[m] = np.float32(1e-3)
            v[m - 1] = v[m + 1] = f32_next(v[m], -1.0)    # exp(-1 ulp of 1e-3) rounds to 1.0f: p = 1/3 each
    elif case == "sharp_zero":
        v[m] = np.float32(50.0)
        v[max(m - 1, 0):m] = np.float32(-70.0)        # exp(-120) = 0 in float32
        v[m + 1:m + 2] = np.float32(-70.0)
    elif case == "sharp_subnormal":
        v[m] = np.float32(50.0)
        v[max(m - 1, 0):m] = np.float32(-45.0)        # exp(-95) = 5.5e-42: a float32 subnormal
        v[m + 1:m + 2] = np.float32(-46.5)
    return v, m


def _exist_pair(rng, case):
    a = np.float32(rng.normal(0, 1))
    if case == "clear":
        return a, np.float32(a + 2.0)
    if case == "ulp_above":
        return a, f32_next(a, np.inf)
    if case == "clear_low":
        return a, np.float32(a - 2.0)
    if case == "tie":
        return a, a
    return a, f32_next(a, -np.inf)                     # ulp_below


def v2_heads(seed, ngr, ncr, ngc, ncc, keep=None):
    """Crafted UFLD v2 heads [loc_row [1,ngr,ncr,4], loc_col [1,ngc,ncc,4], ex_row [1,2,ncr,4], ex_col [1,2,ncc,4]] (float32).
    keep: valid-anchor count per output lane (lanes 1, 2 are row lanes, 0, 3 column lanes); default random.  Every loc case and
    every exist case is cycled through the columns.  Returns (heads, meta) with meta the intended argmax / validity per column."""
    rng = np.random.default_rng(seed)
    heads = [np.zeros((1, ngr, ncr, 4), np.float32), np.zeros((1, ngc, ncc, 4), np.float32),
             np.zeros((1, 2, ncr, 4), np.float32), np.zeros((1, 2, ncc, 4), np.float32)]
    meta = {"argmax": {}, "valid": {}, "loc_case": {}, "exist_case": {}}
    ci = int(rng.integers(0, len(LOC_CASES)))
    for lane in range(4):
        part = 0 if lane in (1, 2) else 1
        ng, nc = (ngr, ncr) if part == 0 else (ngc, ncc)
        loc, ex = heads[part], heads[2 + part]
        k = int(rng.integers(0, nc + 1)) if keep is None else int(keep[lane])
        valid = np.zeros(nc, bool)
        valid[rng.choice(nc, k, replace=False)] = True
        for a in range(nc):
            case = LOC_CASES[ci % len(LOC_CASES)]
            ci += 1
            col, m = _loc_column(rng, ng, case)
            loc[0, :, a, lane] = col
            ecase = (EXIST_VALID if valid[a] else EXIST_INVALID)[int(rng.integers(0, 2 if valid[a] else 3))]
            ex[0, 0, a, lane], ex[0, 1, a, lane] = _exist_pair(rng, ecase)
            key = (lane, a)
            meta["argmax"][key], meta["valid"][key], meta["loc_case"][key], meta["exist_case"][key] = m, bool(valid[a]), case, ecase
    return heads, meta


def keep_threshold_counts(ncr, ncc):
    """Valid-anchor counts exactly at and one past each keep threshold: row lanes need sum > ncr/2, column lanes sum > ncc/4."""
    r0, c0 = ncr // 2, ncc // 4
    return [(c0, r0, r0 + 1, c0 + 1), (c0 + 1, r0 + 1, r0, c0)]


def flat_v2(heads):
    return np.concatenate([h.ravel() for h in heads])


def v2_coord_bound(ng, hi, size):
    """Bound on |device - oracle| of the float64 expectation coordinate c = (sum_g p_g g + 0.5) / (ng - 1) * size.

    Both sides compute p_g = e_g / S in float32 over the <= 3 window bins with the same rounded x - max (an exact IEEE subtract on both
    sides), so they differ only through exp: CUDA's expf is within 2 ulp, numpy's float32 exp within 4 ulp (SVML's documented bound;
    its own loops are tighter), i.e. |de/e| <= 8u each.  The sum of <= 3 terms adds 2 roundings, the divide one: |dp/p| <= 8u + (8u +
    2u) + u = 19u per side, 38u between them (first order).  Summed against the indices, |d sum p_g g| <= 38u * sum p_g g <= 38u * hi
    with hi the window's last index.  The float64 tail (3 multiply-adds, a divide, a multiply) adds 6 U relative.  Where exp lands in
    the float32 subnormal range its error is absolute (2 ulp = 2**-148), times g <= hi: negligible next to 38u but kept.
    So the bound is (38u * hi + hi * 2**-148 * 2) / (ng - 1) * size + 6U * |c|: 2.2e-6 * size at hi = ng - 1, i.e. 2.9e-3 px at
    1280 px and 8.7e-3 px at 3840 px -- the fixed 1e-3 px used for the seeded heads is not a bound at 4K."""
    hi = np.asarray(hi, np.float64)
    c_max = (hi + 0.5) / (ng - 1) * size
    return (38 * u * hi + 4 * 2.0 ** -148 * hi) / (ng - 1) * size + 6 * U * c_max


def v2_reference(heads, img_w, img_h, row_anchor, col_anchor):
    """oracle.post.ufld_decode plus, per emitted point, the window's last index (for the bound)."""
    pts, status, crd = post.ufld_decode(heads, img_w, img_h, row_anchor, col_anchor)
    loc_row, loc_col, ex_row, ex_col = heads
    his = []
    for lane in range(4):
        loc, ex = (loc_row, ex_row) if lane in (1, 2) else (loc_col, ex_col)
        ng = loc.shape[1]
        v = ex[0].argmax(0)[:, lane]
        m = loc[0].argmax(0)[:, lane]
        his.append(np.minimum(ng - 1, m[v.astype(bool)] + 1) if v.sum() > (loc.shape[2] / 2 if lane in (1, 2) else loc.shape[2] / 4)
                   else np.zeros(0, int))
    return pts, status, crd, his


def int_points_agree(got_pts, want_pts, got_c, bound, coord_axis):
    """Truncated integer points agree except where the float64 coordinate lies within `bound` of an integer (where either side of the
    truncation is correct).  Returns the indices that were allowed to differ."""
    got_pts, want_pts = np.asarray(got_pts).reshape(-1, 2), np.asarray(want_pts).reshape(-1, 2)
    assert got_pts.shape == want_pts.shape, (got_pts.shape, want_pts.shape)
    d = got_pts - want_pts
    bad = np.nonzero(d.any(axis=1))[0]
    for j in bad:
        other = 1 - coord_axis
        assert d[j, other] == 0 and abs(int(d[j, coord_axis])) == 1, (j, got_pts[j], want_pts[j])
        c = float(got_c[j])
        assert abs(c - round(c)) <= float(np.broadcast_to(bound, got_c.shape)[j]), (j, c, bound)
    return bad


# =================================================================================================================================
# 2. UFLD v1 decode
# =================================================================================================================================
V1_CASES = ("ridge", "none_tie", "none_ulp_above", "sharp", "none")


def v1_head(seed, G, R, nonzero=None):
    """Crafted UFLD v1 head [1, G+1, R, 4] (float32).  Row cases cycle through V1_CASES: the "no lane" bin equal to the maximum (not
    none: the first maximum wins), one ulp above it (none), sharp logits (exp underflows to 0), plain "none" rows.  nonzero: per lane,
    force exactly that many rows to decode non-zero (the others "none"), e.g. 2 vs 3 for the detection threshold."""
    rng = np.random.default_rng(seed)
    out = rng.normal(-3, 1, (1, G + 1, R, 4)).astype(np.float32)
    cases = {}
    ci = int(rng.integers(0, len(V1_CASES)))
    for lane in range(4):
        force = None
        if nonzero is not None and nonzero[lane] is not None:
            force = np.zeros(R, bool)
            force[rng.choice(R, nonzero[lane], replace=False)] = True
        for r in range(R):
            case = V1_CASES[ci % len(V1_CASES)]
            ci += 1
            if force is not None:
                case = ("ridge", "none_tie", "sharp")[r % 3] if force[r] else "none"
            g = int(rng.integers(0, G))
            col = out[0, :, r, lane]
            if case == "ridge":
                col[g] = np.float32(6 + rng.random())
                col[G] = np.float32(-10)
            elif case == "none_tie":
                col[g] = np.float32(4.25)
                col[G] = col[:G].max()
            elif case == "none_ulp_above":
                col[g] = np.float32(4.25)
                col[G] = f32_next(col[:G].max(), np.inf)
            elif case == "sharp":
                col[:G] = np.float32(-100.0)
                col[g] = np.float32(30.0)                    # every other cell: exp(-130) = 0
                col[G] = np.float32(-200.0)
            else:
                col[G] = np.float32(40.0)
            cases[(lane, r)] = case
    return out, cases


V1_GOLDEN = (("tusimple", 100, 56), ("culane", 200, 18))
V2_GOLDEN_DIMS = {"culane": (200, 72, 100, 81), "tusimple": (100, 56, 100, 41)}
FRAME_SIZES = ((1280, 720), (640, 480), (333, 517), (1920, 1080), (3840, 2160))        # (w, h)


def v2_golden_heads(ds):
    """The crafted heads whose reference decode is committed: the keep counts at / past the thresholds (two ways round) and one
    random set of counts."""
    ngr, ncr, ngc, ncc = V2_GOLDEN_DIMS[ds]
    ks = keep_threshold_counts(ncr, ncc) + [None]
    return [v2_heads(300 + i, ngr, ncr, ngc, ncc, keep=k)[0] for i, k in enumerate(ks)]


def v1_golden_heads(G, R):
    """Crafted v1 heads: a cycled-case head, and heads with exactly 2 / 3 non-zero rows on alternating lanes."""
    return [v1_head(400, G, R)[0], v1_head(401, G, R, nonzero=(2, 3, None, 2))[0], v1_head(402, G, R, nonzero=(3, 2, 3, None))[0]]


def v1_x_bound(G, x_px, w_ratio):
    """Bound on |device - oracle| of the float64 x before truncation, x = (loc * csw * cfg_w / in_w - 1) * w_ratio.

    loc = sum_g p_g (g + 1) with p_g = e_g / S over all G cells: e_g within 8u of exact on each side (expf 2 ulp, numpy exp 4 ulp), S
    a sequential float32 sum of G terms in the same order on both sides (numpy reduces the outer axis row by row), so |dS/S| <= 8u +
    (G - 1)u, and the divide rounds once: |dp/p| <= (G + 16)u per side, 2(G + 16)u between them.  The float64 tail adds about
    (G + 6) U relative.  So |dx| <= (2(G + 16)u + (G + 6)U) * |x + w_ratio|: 4.3e-4 px at G = 200 and x = 1280."""
    return (2 * (G + 16) * u + (G + 6) * U) * np.abs(np.asarray(x_px, np.float64) + w_ratio)


# =================================================================================================================================
# 3. Lane geometry
# =================================================================================================================================
def polyfit_perturbation(x, y):
    """Bound on how far two backward-stable float64 least-squares solvers may land apart on np.polyfit(x, y, 2), per coefficient
    (highest power first), and the fit itself.

    Both numpy (SVD, LAPACK gelsd) and the kernel (Householder QR) solve the column-scaled Vandermonde system A_s z = y, c = z / scale.
    Each is backward stable: its answer solves a problem perturbed by ||dA|| <= eps ||A_s||, ||dy|| <= eps ||y|| with eps = 3 m sqrt(3)
    * 2U for m rows and 3 columns (Higham, Accuracy and Stability, Thm 19.5 / 20.3, the constant taken as 2).  The least-squares
    perturbation theorem (Higham Thm 20.1) then bounds each side's distance from the exact z:
        ||dz|| <= kappa eps / (1 - kappa eps) * (2 + (kappa + 1) ||r|| / (||A_s|| ||z||)) * ||z||
    with kappa the 2-norm condition number of A_s and r the residual.  The two answers differ by at most twice that, per coefficient
    after dividing by the column scale."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    A = np.stack([x * x, x, np.ones_like(x)], 1)
    scale = np.sqrt((A * A).sum(0))
    As = A / scale
    z, *_ = np.linalg.lstsq(As, y, rcond=None)
    r = y - As @ z
    sv = np.linalg.svd(As, compute_uv=False)
    kappa = sv[0] / sv[-1]
    m = len(x)
    eps = 3 * m * np.sqrt(3) * 2 * U
    ke = kappa * eps
    assert ke < 0.5, "ill-conditioned fit"
    nz = np.linalg.norm(z)
    dz = ke / (1 - ke) * (2 + (kappa + 1) * np.linalg.norm(r) / (sv[0] * max(nz, 1e-300))) * nz
    return 2 * dz / scale, np.polyfit(x, y, 2)


def resample_bound(dc, ys):
    """|dx| at the resampled rows y from the coefficient bound dc (the caller adds the 4 roundings of a y^2 + b y + c)."""
    ys = np.asarray(ys, np.float64)
    return dc[0] * ys * ys + dc[1] * np.abs(ys) + dc[2]


def adjust_reference(left, right, img_h):
    """LaneDetectBase.__adjust_lanes_points in float64 (numpy's polyfit): the kept (x_float, y_float) rows per side, the
    integer points, and a per-row bound on x."""
    out = []
    left, right = np.asarray(left, np.int64), np.asarray(right, np.int64)
    maxy = max(img_h - 1, left[:, 1].max(), right[:, 1].max())
    miny = min(img_h // 3, left[:, 1].min(), right[:, 1].min())
    both = np.linspace(miny, maxy, img_h)
    for lane in (left, right):
        ys_fit, xs_fit = lane[:, 1].astype(np.float64), lane[:, 0].astype(np.float64)
        dc, fit = polyfit_perturbation(ys_fit, xs_fit)
        fx = fit[0] * both ** 2 + fit[1] * both + fit[2]
        b = resample_bound(dc, both) + 4 * U * (np.abs(fit[0]) * both ** 2 + np.abs(fit[1] * both) + abs(fit[2]))
        keep = (both >= ys_fit.min()) & (fx >= 0)
        out.append(dict(x=fx, y=both, bound=b, keep=keep, near_zero=(np.abs(fx) <= b) & (both >= ys_fit.min())))
    return out


def check_adjusted_area(area, want, ref):
    """The device's resampled polygon against the reference's, row by row: left rows in order then right rows reversed; an integer may
    differ by one only where x is within the bound of an integer.  A row whose x is within the bound of 0 could be kept by one side
    only, which would shift every later row: the crafted cases have none (asserted), so the rows align one to one."""
    left, right = ref
    assert not (left["near_zero"].any() or right["near_zero"].any()), "a resampled row with x within the bound of 0"
    assert area.shape == want.shape, (area.shape, want.shape)
    xs = np.concatenate([left["x"][left["keep"]], right["x"][right["keep"]][::-1]])
    bs = np.concatenate([left["bound"][left["keep"]], right["bound"][right["keep"]][::-1]])
    assert len(xs) == len(want)
    d = area - want
    for j in np.nonzero(d.any(axis=1))[0]:
        assert d[j, 1] == 0 and abs(int(d[j, 0])) == 1 and abs(xs[j] - round(xs[j])) <= bs[j], (j, area[j], want[j], xs[j], bs[j])


def bird_points_reference(M, pts):
    """transformToBirdViewPoints in float64: p' = M [x y 1] as (M0 x + M1 y) + M2, (x'/w, y'/w) truncated.  Returns (int points, float
    values, bound): numpy's einsum may sum in another order than the kernel, and each of the 3 products, 2 sums and the divide rounds
    once, so two evaluations differ by at most 6 U (sum |terms of x'| / |w| + |x'/w| sum |terms of w| / |w|) per coordinate."""
    P = np.asarray(pts, np.float64).reshape(-1, 2)
    M = np.asarray(M, np.float64)
    x, y = P[:, 0], P[:, 1]
    t = [(M[r, 0] * x, M[r, 1] * y, np.full_like(x, M[r, 2])) for r in range(3)]
    h = [(a + b) + c for a, b, c in t]
    f = np.stack([h[0] / h[2], h[1] / h[2]], 1)
    aw = np.abs(t[2][0]) + np.abs(t[2][1]) + np.abs(t[2][2])
    bound = np.stack([6 * U * ((np.abs(t[k][0]) + np.abs(t[k][1]) + np.abs(t[k][2])) + np.abs(f[:, k]) * aw) / np.abs(h[2])
                      for k in range(2)], 1)
    return f.astype(np.int64), f, bound


def curve_reference(bl, br, bird_h, bird_w):
    """calcCurveAndOffset's numbers in float64 with numpy (direction, curvature, offset) and first-order bounds on curvature / offset:
    the coefficient bounds of the two pixel fits (polyfit_perturbation) and of the two metre refits are pushed through the formulas
    one coefficient at a time (a finite difference of the size of the bound), and summed."""
    ym, xm = 30 / 720, 3.7 / 700
    bl, br = np.asarray(bl, np.float64), np.asarray(br, np.float64)
    dl, lf = polyfit_perturbation(bl[:, 1], bl[:, 0])
    dr, rf = polyfit_perturbation(br[:, 1], br[:, 0])
    ploty = np.linspace(0, bird_h - 1, bird_h)

    def numbers(lf, rf, dlc=None, drc=None):
        leftx = lf[0] * ploty ** 2 + lf[1] * ploty + lf[2]
        rightx = rf[0] * ploty ** 2 + rf[1] * ploty + rf[2]
        lc = np.polyfit(ploty * ym, leftx * xm, 2) + (0 if dlc is None else dlc)
        rc = np.polyfit(ploty * ym, rightx * xm, 2) + (0 if drc is None else drc)
        y_eval = ploty.max()
        lrad = (1 + (2 * lc[0] * y_eval * ym + lc[1]) ** 2) ** 1.5 / abs(2 * lc[0])
        rrad = (1 + (2 * rc[0] * y_eval * ym + rc[1]) ** 2) ** 1.5 / abs(2 * rc[0])
        lane_w = abs(leftx[719] - rightx[719])
        off = ((leftx[719] + rightx[719]) / 2 - bird_w / 2) * (3.7 / lane_w)
        return (lrad + rrad) / 2, off

    curv, off = numbers(lf, rf)
    side = lf[0] if abs(lf[0]) > abs(rf[0]) else rf[0]
    if side < -0.00015 and bl[0, 0] <= bl[int(len(bl) / 2), 0]:
        d = "L"
    elif side > 0.00015 and br[0, 0] >= br[int(len(br) / 2), 0]:
        d = "R"
    else:
        d = "F"
    bc = bo = 0.0
    for which in range(2):
        base = (lf, rf)[which]
        dd = (dl, dr)[which]
        for k in range(3):
            c2 = base.copy()
            c2[k] += dd[k]
            args = (c2, rf) if which == 0 else (lf, c2)
            c, o = numbers(*args)
            bc, bo = bc + abs(c - curv), bo + abs(o - off)
    # the metre refits: exact quadratic data on bird_h rows, residual ~ 0; their own solver spread
    leftx = lf[0] * ploty ** 2 + lf[1] * ploty + lf[2]
    dlc, _ = polyfit_perturbation(ploty * ym, leftx * xm)
    rightx = rf[0] * ploty ** 2 + rf[1] * ploty + rf[2]
    drc, _ = polyfit_perturbation(ploty * ym, rightx * xm)
    for k in range(3):
        e = np.zeros(3)
        e[k] = dlc[k]
        c, _ = numbers(lf, rf, dlc=e)
        bc += abs(c - curv)
        e = np.zeros(3)
        e[k] = drc[k]
        c, _ = numbers(lf, rf, drc=e)
        bc += abs(c - curv)
    # the closing arithmetic (pow, a handful of multiplies / divides): 16 U relative
    return d, curv, off, bc + 16 * U * abs(curv), bo + 16 * U * abs(off), side


def exact_parabola_lane(a, c, n, step, descending=False):
    """Integer points x = c + a y^2 on y = 0, step, ... with a * step^2 an integer: the pixel fit recovers a to within its solver
    spread, so a leading coefficient set just past +-0.00015 is decided the same way by every backward-stable solver."""
    k = round(a * step * step)
    assert abs(a * step * step - k) < 1e-9, "a * step^2 must be an integer"
    p = np.stack([c + k * np.arange(n) ** 2, np.arange(n) * step], 1).astype(np.int64)
    return p[::-1] if descending else p


def lanes_to_arrays(lanes_per_frame, status_per_frame, mp):
    B = len(lanes_per_frame)
    pts = np.zeros((B, 4, mp, 2), np.int32)
    npts = np.zeros((B, 4), np.int32)
    for b, lanes in enumerate(lanes_per_frame):
        for l in range(4):
            a = np.asarray(lanes[l], np.int32).reshape(-1, 2)
            pts[b, l, :len(a)] = a
            npts[b, l] = len(a)
    return pts, npts, np.asarray(status_per_frame, np.uint8).reshape(B, 4)


def frontal_lane(seed, n, img_w, img_h, side, x_shift=0.0, y_top=None):
    """Seeded frontal-view ego lane of n integer points, rows ascending from y_top to the bottom of the frame."""
    rng = np.random.default_rng(seed)
    y0 = img_h * 0.45 if y_top is None else y_top
    ys = np.linspace(y0, img_h - 1, n)
    t = (ys - ys[0]) / max(1.0, ys[-1] - ys[0])
    centre = img_w * 0.5 + rng.uniform(-80, 80) * (1 - t) ** 2
    half = img_w * (0.03 + 0.2 * t)
    xs = centre + (-half if side == 0 else half) + x_shift + rng.normal(0, 1.2, n)
    return [(int(x), int(y)) for x, y in zip(xs, ys)]


GEOM_MP = 128          # points per lane of the geometry cases (the decode's largest: 128 anchors)


def geom_cases():
    """Crafted ego-lane pairs: dict(name, left, right, img_wh, M: None / "default" / "identity", bird_wh).  "default" is the
    reference PerspectiveTransformation((1280, 720)).M, stored with the goldens."""
    cs = []
    for nl, nr in ((10, 10), (10, 11), (11, 10), (11, 11), (72, 72), (128, 128)):          # the adjust switch and the largest lanes
        cs.append(dict(name=f"adj_{nl}_{nr}", left=frontal_lane(nl, nl, 1280, 720, 0), right=frontal_lane(100 + nr, nr, 1280, 720, 1),
                       img_wh=(1280, 720), M="default", bird_wh=(1280, 720)))
    for h in (480, 720, 1080, 1100, 1101):                                                    # resampled rows vs the 128-row chunks
        w = int(h * 16 / 9)
        cs.append(dict(name=f"img_h{h}", left=frontal_lane(h, 30, w, h, 0), right=frontal_lane(h + 1, 30, w, h, 1), img_wh=(w, h),
                       M=None, bird_wh=(1280, 720)))
    # the first lane row above h // 3: the first resampled row is exactly min(lefty), kept by y >= min(lefty)
    cs.append(dict(name="top_row", left=frontal_lane(5, 40, 1280, 720, 0, y_top=150), right=frontal_lane(6, 40, 1280, 720, 1, y_top=170),
                   img_wh=(1280, 720), M="default", bird_wh=(1280, 720)))
    # a steep left lane ending at 0.8 H: its fit goes negative below, rows dropped by x >= 0
    ys = np.linspace(360, 576, 20)
    left = [(int(400 - (y - 360) * 380 / 216 + 0.3 * np.sin(y)), int(y)) for y in ys]
    cs.append(dict(name="negative_fit", left=left, right=frontal_lane(7, 20, 1280, 720, 1), img_wh=(1280, 720), M=None,
                   bird_wh=(1280, 720)))
    # lanes reaching above the default trapezoid (the bird-view w shrinks towards the horizon, then turns negative)
    cs.append(dict(name="above_trapezoid", left=frontal_lane(8, 60, 1280, 720, 0, y_top=60), right=frontal_lane(9, 60, 1280, 720, 1, y_top=40),
                   img_wh=(1280, 720), M="default", bird_wh=(1280, 720)))
    # direction thresholds: leading coefficients just past and just short of +-0.00015, both orders of the left / right points
    for a_l, a_r, desc, tag in ((-0.0001501, 1e-5, True, "L"), (-0.0001501, 1e-5, False, "L_wrong_order"), (-0.0001499, 1e-5, True, "F_short_L"),
                                (1e-5, 0.0001501, True, "R"), (1e-5, 0.0001501, False, "R_wrong_order"), (1e-5, 0.0001499, True, "F_short_R")):
        cs.append(dict(name=f"dir_{tag}", left=exact_parabola_lane(a_l, 300, 5, 10000, desc).tolist(),
                       right=exact_parabola_lane(a_r, 900, 5, 10000, desc).tolist(), img_wh=(1280, 720), M="identity", bird_wh=(1280, 720)))
    # 3 points per ego lane (an exactly determined fit); bird-view heights around the 720-row and 2160-row limits
    cs.append(dict(name="three_points", left=frontal_lane(10, 3, 1280, 720, 0), right=frontal_lane(11, 3, 1280, 720, 1), img_wh=(1280, 720),
                   M="default", bird_wh=(1280, 720)))
    for bh in (480, 719, 720, 1100, 1101, 2160):
        cs.append(dict(name=f"bird_h{bh}", left=frontal_lane(12, 40, 1280, 720, 0), right=frontal_lane(13, 40, 1280, 720, 1),
                       img_wh=(1280, 720), M="default", bird_wh=(1280, bh)))
    return cs


# =================================================================================================================================
# 4. Bird-view warp
# =================================================================================================================================
def inv3(s):
    """cv::invert of a 3x3 float64 matrix: the adjugate over the first-row determinant expansion, OpenCV's operation order."""
    S = lambda r, c: s[r, c]  # noqa: E731
    d = S(0, 0) * (S(1, 1) * S(2, 2) - S(1, 2) * S(2, 1)) - S(0, 1) * (S(1, 0) * S(2, 2) - S(1, 2) * S(2, 0)) + \
        S(0, 2) * (S(1, 0) * S(2, 1) - S(1, 1) * S(2, 0))
    d = 1.0 / d
    t = np.empty(9)
    t[0] = (S(1, 1) * S(2, 2) - S(1, 2) * S(2, 1)) * d
    t[1] = (S(0, 2) * S(2, 1) - S(0, 1) * S(2, 2)) * d
    t[2] = (S(0, 1) * S(1, 2) - S(0, 2) * S(1, 1)) * d
    t[3] = (S(1, 2) * S(2, 0) - S(1, 0) * S(2, 2)) * d
    t[4] = (S(0, 0) * S(2, 2) - S(0, 2) * S(2, 0)) * d
    t[5] = (S(0, 2) * S(1, 0) - S(0, 0) * S(1, 2)) * d
    t[6] = (S(1, 0) * S(2, 1) - S(1, 1) * S(2, 0)) * d
    t[7] = (S(0, 1) * S(2, 0) - S(0, 0) * S(2, 1)) * d
    t[8] = (S(0, 0) * S(1, 1) - S(0, 1) * S(1, 0)) * d
    return t


def warp_emulate(src, Mf, dsize, bw0_fixed=None, half_away=False, wrap_int16=False, clamp_taps=False):
    """cv2.warpPerspective(src, Mf, dsize, INTER_LINEAR, BORDER_CONSTANT 0) restated in float64 numpy, the arithmetic of csrc/warp.cu.
    The keyword arguments are deliberate mutations (for the tests that show the hashes have teeth): a fixed block width, rounding
    half away from zero, int16 wrap-around instead of saturation, out-of-range taps read from clamped coordinates instead of 0."""
    ow, oh = dsize
    H, W = src.shape[:2]
    M = inv3(np.asarray(Mf, np.float64))
    bw0 = min(1024 // min(oh, 16), ow) if bw0_fixed is None else bw0_fixed
    x = np.arange(ow)
    xb = ((x // bw0) * bw0).astype(np.float64)[None, :]
    x1 = (x - (x // bw0) * bw0).astype(np.float64)[None, :]
    y = np.arange(oh, dtype=np.float64)[:, None]
    X0 = M[0] * xb + M[1] * y + M[2]
    Y0 = M[3] * xb + M[4] * y + M[5]
    W0 = M[6] * xb + M[7] * y + M[8]
    Wv = W0 + M[6] * x1
    with np.errstate(divide="ignore", invalid="ignore"):
        Wv = np.where(Wv != 0, 32.0 / np.where(Wv != 0, Wv, 1.0), 0.0)
    fX = np.clip((X0 + M[0] * x1) * Wv, -2.0 ** 31, 2.0 ** 31 - 1)
    fY = np.clip((Y0 + M[3] * x1) * Wv, -2.0 ** 31, 2.0 ** 31 - 1)
    rnd = (lambda v: np.sign(v) * np.floor(np.abs(v) + 0.5)) if half_away else np.rint
    X, Y = rnd(fX).astype(np.int64), rnd(fY).astype(np.int64)
    if wrap_int16:
        sx, sy = ((X >> 5) + 32768) % 65536 - 32768, ((Y >> 5) + 32768) % 65536 - 32768
    else:
        sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    ax, ay = X & 31, Y & 31
    wts = [(32 - ay) * (32 - ax), (32 - ay) * ax, ay * (32 - ax), ay * ax]
    acc = np.zeros((oh, ow, 3), np.int64)
    S = src.astype(np.int64)
    for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        yy, xx = sy + dy, sx + dx
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        if clamp_taps:
            p = S[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        else:
            p = np.where(ok[..., None], S[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], 0)
        acc += p * wts[k][..., None]
    return np.clip((acc * 32 + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


WARP_MATRICES = {
    "identity": np.eye(3),
    "half_px": np.array([[1.0, 0.0, 0.5], [0.0, 1.0, 0.5], [0.0, 0.0, 1.0]]),
    "half_step": np.array([[1.0, 0.0, 1 / 64], [0.0, 1.0, -1 / 64], [0.0, 0.0, 1.0]]),      # X lands on .5 of a 1/32-px step
    "mirror": np.array([[-1.0, 0.0, 639.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]),
    "persp": np.array([[1.0, 0.1, -30.0], [0.02, 0.9, 12.5], [1e-4, -2e-4, 1.0]]),
    "horizon": np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, -1 / 240.0, 1.0]]),       # W = 0 on row 240
    "behind": np.array([[1.0, 0.2, 0.0], [0.0, 1.0, 0.0], [1e-3, 2e-3, -0.5]]),            # W < 0 over most of the frame
    "past_int16": np.array([[1.0, 0.0, -65556.0], [0.0, 1.0, 65540.0], [0.0, 0.0, 1.0]]),  # source x = x + 65556: saturates to 32767
    "huge_scale": np.array([[1e-6, 0.0, 0.0], [0.0, 1e-6, 0.0], [0.0, 0.0, 1.0]]),         # X = 32e6 x: past INT_MAX from x = 68
    "tiny_scale": np.array([[1e4, 0.0, 3.0], [0.0, 1e4, 5.0], [0.0, 0.0, 1.0]]),           # the whole output samples 1 source pixel
}
WARP_HEIGHTS = (1, 3, 5, 15, 16, 720)
WARP_WIDTHS = (1, 7, 333, 2000, 4096)


def warp_source(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def warp_cases():
    """(name, source seed, source (h, w), matrix name, dsize) of the committed warp hashes (tests/golden/warp_edges.npz)."""
    cases = []
    for mname in WARP_MATRICES:
        for oh in WARP_HEIGHTS:
            for ow in WARP_WIDTHS:
                if oh == 720 and ow == 4096 and mname not in ("persp", "horizon"):
                    continue                                  # the largest output for two matrices only
                cases.append((f"{mname}_{ow}x{oh}", 7, (480, 640), mname, (ow, oh)))
    for mname in ("identity", "half_px", "tiny_scale", "mirror"):
        for dsize in ((1, 1), (3, 2), (64, 16)):
            cases.append((f"src1x1_{mname}_{dsize[0]}x{dsize[1]}", 8, (1, 1), mname, dsize))
            cases.append((f"src2x3_{mname}_{dsize[0]}x{dsize[1]}", 9, (2, 3), mname, dsize))
    return cases


def warp_batch_matrices(n=40):
    """A different matrix per frame for the batched warp: scaled / rotated / perspective mixtures of the named matrices."""
    rng = np.random.default_rng(11)
    names = list(WARP_MATRICES)
    Ms = []
    for i in range(n):
        M = WARP_MATRICES[names[i % len(names)]].copy()
        if i >= len(names):
            M = M @ np.array([[1 + rng.uniform(-0.2, 0.2), rng.uniform(-0.1, 0.1), rng.uniform(-40, 40)],
                              [rng.uniform(-0.1, 0.1), 1 + rng.uniform(-0.2, 0.2), rng.uniform(-40, 40)],
                              [rng.uniform(-3e-4, 3e-4), rng.uniform(-3e-4, 3e-4), 1.0]])
        Ms.append(M)
    return np.stack(Ms)


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


# =================================================================================================================================
# 5. Pre-processing
# =================================================================================================================================
# (frame h, w, network in_h, in_w): portrait, small upscaled, exact 2x / 3x square downscale, odd sizes, 1280 and 320 inputs
YOLO_PRE_CASES = [(900, 500, 640, 640), (1920, 1080, 640, 640), (48, 32, 640, 640), (32, 48, 640, 640), (1280, 1280, 640, 640),
                  (1920, 1920, 640, 640), (333, 517, 640, 640), (517, 333, 640, 640), (721, 1279, 1280, 1280), (720, 1280, 320, 320),
                  (2160, 3840, 1280, 1280), (101, 99, 320, 320)]
# (frame h, w, in_h, in_w, crop): v2 CULane / TuSimple, v1 (crop 1.0, resize_h == in_h), upscaling from small frames
UFLD_PRE_CASES = [(720, 1280, 320, 1600, 0.6), (333, 517, 320, 800, 0.8), (720, 1280, 288, 800, 1.0), (100, 160, 288, 800, 1.0),
                  (120, 200, 320, 1600, 0.6), (2160, 3840, 320, 800, 0.8)]
# cv2.resize sizes (src h, w, dst h, w) for the restated fixed-point resize, incl. widths where 3 w is not a multiple of the SIMD width
RESIZE_SIZES = [(720, 1280, 361, 640), (900, 500, 640, 355), (333, 517, 412, 640), (1080, 1920, 361, 640), (600, 600, 640, 640),
                (720, 1280, 533, 1600), (480, 640, 481, 640), (100, 37, 640, 236), (640, 640, 640, 640), (50, 50, 640, 640),
                (1000, 999, 641, 640), (720, 1280, 7, 13), (3, 5, 640, 640), (720, 1280, 640, 1), (1, 1280, 1, 640)]
