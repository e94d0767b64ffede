"""Tie-heavy ByteTrack inputs and an exact optimality certificate for the association solver.  Used by tests/test_gpu_track_edges.py
and tests/test_track_edges_cpu.py.

The product feeds the tracker INTEGER boxes (AdasPipeline._track truncates xyxy like demo.py does), so exact cost ties are common:
equal IoUs, duplicate boxes, costs exactly on a stage threshold, zero-width or zero-height boxes.  On such inputs the optimum of an
association stage is usually not unique, and oracle.post.lapjv_extended pins no tie-break.  So instead of comparing assignments, the
certificate here checks that an assignment is OPTIMAL, exactly:

  An extended assignment (lap.lapjv(extend_cost=True, cost_limit=thresh)) is a partial matching of rows to columns; its value is
  the sum of the matched costs plus thresh/2 for every unmatched row and every unmatched column.  `certify` evaluates that value in
  exact rational arithmetic over the float64 cost values, and compares it with the exact minimum over ALL partial matchings
  (dynamic programming over the column subsets of the smaller side) when that side has at most EXHAUSTIVE_MAX entries, and otherwise
  with the exact value of scipy's linear_sum_assignment answer on the extended matrix (the assignment must be no worse).
  A NaN cost (IoU 0/0 of two zero-area boxes) is a forbidden pair: it must never be matched, and the optimum is taken without it.
"""
from __future__ import annotations

import itertools
from fractions import Fraction

import numpy as np

from oracle import post, track

EXHAUSTIVE_MAX = 8           # smaller side of the problems whose optimum is computed over every partial matching
MATCH_THRESHS = (0.5, 0.8, 0.95)
TRACK_THRESHS = (0.2, 0.5, 0.7)


# ---------------------------------------------------------------------------------------------------------------------------------
# exact optimality certificate
# ---------------------------------------------------------------------------------------------------------------------------------
def _as_ints(cost, thresh):
    """cost entries (None for NaN) and thresh / 2 as integers over one common power-of-two denominator -> (rows, half, denominator)"""
    vals = [float(v) for v in cost.ravel() if not np.isnan(v)] + [thresh / 2.0]
    den = max(Fraction(v).denominator for v in vals)
    conv = lambda v: int(Fraction(v) * den)
    rows = [[None if np.isnan(v) else conv(float(v)) for v in r] for r in cost]
    return rows, conv(thresh / 2.0), den


def extended_value(cost, thresh, x) -> Fraction:
    """exact value of the partial matching x (x[i] = column of row i or -1)"""
    cost = np.asarray(cost, np.float64)
    T, D = cost.shape
    matched = [(i, int(j)) for i, j in enumerate(x) if j >= 0]
    return sum((Fraction(float(cost[i, j])) for i, j in matched), Fraction(0)) + Fraction(thresh) / 2 * (T + D - 2 * len(matched))


def exact_optimum(cost, thresh) -> Fraction:
    """exact minimum of the extended value over every partial matching without NaN pairs (DP over subsets of the smaller side)"""
    c = np.asarray(cost, np.float64)
    if c.shape[1] > c.shape[0]:
        c = c.T
    R, K = c.shape
    rows, half, den = _as_ints(c, thresh)
    best = {0: 0}
    for i in range(R):
        nb = {}
        for mask, v in best.items():
            w = v + half
            if mask not in nb or w < nb[mask]:
                nb[mask] = w
            for j in range(K):
                cij = rows[i][j]
                if cij is not None and not (mask >> j) & 1:
                    m2, w = mask | (1 << j), v + cij
                    if m2 not in nb or w < nb[m2]:
                        nb[m2] = w
        best = nb
    return Fraction(min(v + half * (K - bin(m).count("1")) for m, v in best.items()), den)


def scipy_value(cost, thresh) -> Fraction:
    """exact value of scipy's answer on the extended matrix (NaN pairs forbidden)"""
    x, _, _ = post.lapjv_extended(cost, thresh)
    return extended_value(cost, thresh, x)


class CertStats:
    """what the certificates of one test run covered"""

    def __init__(self):
        self.problems = self.exhaustive = self.bounded = self.tied = self.at_thresh = 0
        self.largest_exhaustive = (0, 0)

    def __str__(self):
        return (f"{self.problems} problems certified ({self.exhaustive} exhaustively, largest {self.largest_exhaustive[0]}x"
                f"{self.largest_exhaustive[1]}; {self.bounded} against scipy), {self.tied} with tied costs, {self.at_thresh} with a cost "
                f"exactly on the threshold")


def has_tie(cost, thresh) -> bool:
    """two equal costs of overlapping pairs (cost < 1), or a cost exactly on the threshold"""
    v = np.asarray(cost, np.float64).ravel()
    v = v[v < 1.0]
    return bool(len(np.unique(v)) < len(v) or (v == thresh).any())


def certify(cost, thresh, x, y=None, stats: CertStats = None) -> Fraction:
    """assert that (x, y) is a consistent partial matching, matches no NaN pair and no pair above thresh, and is an exact optimum
    of the extended problem; returns its exact value"""
    cost = np.asarray(cost, np.float64)
    T, D = cost.shape
    x = np.asarray(x).astype(np.int64)
    assert x.shape == (T,), (x.shape, T)
    cols = x[x >= 0]
    assert ((x >= -1) & (x < D)).all() and len(set(cols.tolist())) == len(cols), f"not a partial matching: {x}"
    if y is not None:
        y = np.asarray(y).astype(np.int64)
        want_y = np.full(D, -1)
        want_y[cols] = np.nonzero(x >= 0)[0]
        assert np.array_equal(y, want_y), f"y {y} is not the inverse of x {x}"
    for i in np.nonzero(x >= 0)[0]:
        c = cost[i, x[i]]
        assert not np.isnan(c), f"row {i} matched to column {x[i]} at a NaN cost"
        assert c <= thresh, f"row {i} matched to column {x[i]} at cost {c!r} > thresh {thresh!r}"
    val = extended_value(cost, thresh, x)
    if stats is not None:
        stats.problems += 1
        stats.tied += has_tie(cost, thresh)
        stats.at_thresh += bool((cost == thresh).any())
    if min(T, D) <= EXHAUSTIVE_MAX:
        opt = exact_optimum(cost, thresh)
        assert val == opt, f"assignment value {float(val)!r} exceeds the exact optimum {float(opt)!r} by {float(val - opt)!r} ({T}x{D})"
        if stats is not None:
            stats.exhaustive += 1
            if T * D > stats.largest_exhaustive[0] * stats.largest_exhaustive[1]:
                stats.largest_exhaustive = (T, D)
    else:
        ref = scipy_value(cost, thresh)
        assert val <= ref, f"assignment value {float(val)!r} exceeds scipy's {float(ref)!r} ({T}x{D})"
        if stats is not None:
            stats.bounded += 1
    return val


# ---------------------------------------------------------------------------------------------------------------------------------
# boxes the Kalman filter reproduces exactly
# ---------------------------------------------------------------------------------------------------------------------------------
def kalman_box(tlbr):
    """tlbr of a track initiated from `tlbr` (and of a stationary track re-measured at it), as oracle.track computes it"""
    b = np.asarray(tlbr, np.float64)
    t = track.Track(np.r_[b[:2], b[2:] - b[:2]], 0.9, 0)
    t.mean, t.cov = track.kf_initiate(track.Track.xyah(t.tlwh0))
    return t.tlbr()


def kalman_exact(tlbr) -> bool:
    return bool(np.array_equal(kalman_box(tlbr), np.asarray(tlbr, np.float64)))


# ---------------------------------------------------------------------------------------------------------------------------------
# crafted single-stage problems
# ---------------------------------------------------------------------------------------------------------------------------------
def _nudge(x, k):
    """x moved k float64 ulps (k < 0: down)"""
    for _ in range(abs(k)):
        x = np.nextafter(x, np.inf if k > 0 else -np.inf)
    return float(x)


def _problem(name, stage, tracks, dets, scores, thresh, kind):
    tracks, dets = np.asarray(tracks, np.float64).reshape(-1, 4), np.asarray(dets, np.float64).reshape(-1, 4)
    fuse = stage != 2
    sc = None if not fuse else np.asarray(scores, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        cost = post.iou_cost(tracks, dets, sc)
    return dict(name=name, stage=stage, tracks=tracks, dets=dets, scores=sc, thresh=float(thresh), cost=cost, kind=kind,
                tracker=all(kalman_exact(b) for b in tracks))


def _stage_problem_at(stage, thresh):
    """(track box, det box, score) of one pair whose float64 cost is exactly `thresh`: an IoU that is a power of two (exact), and for
    the fused stages the score (1 - thresh) / IoU, exact because the division is by a power of two"""
    if stage == 2:
        t, d, s = [0, 0, 10, 10], [0, 0, 10, 5], None                     # IoU 50 / 100
        assert thresh == 0.5
    else:
        for den, t, d in ((1, [0, 0, 8, 8], [0, 0, 8, 8]), (2, [0, 0, 8, 8], [0, 0, 8, 4]), (4, [0, 0, 8, 8], [0, 0, 8, 2]),
                          (16, [0, 0, 16, 16], [0, 0, 16, 1])):
            s = (1.0 - thresh) * den
            if 0.5 < s <= 1.0:                                             # a high-score detection at the default track_thresh
                break
        else:
            raise AssertionError(thresh)
    return t, d, s


def threshold_problems():
    """single-stage problems with a cost EXACTLY on the stage threshold (stage 1 at each match_thresh, stage 2 at 0.5, stage 3 at
    0.7), alone and among ties, plus the same problems with that cost nudged to the nearest reachable value either side"""
    out = []
    stages = [(1, m) for m in MATCH_THRESHS] + [(2, 0.5), (3, 0.7)]
    for stage, th in stages:
        t, d, s = _stage_problem_at(stage, th)
        sc = [s]
        p = _problem(f"s{stage}@{th} 1x1", stage, [t], [d], sc, th, "at")
        assert p["cost"][0, 0] == th, (stage, th, p["cost"])
        out.append(p)
        # two identical tracks x two identical detections: every partial matching has the same value
        out.append(_problem(f"s{stage}@{th} 2x2 all at thresh", stage, [t, t], [d, d], sc * 2, th, "at"))
        # an at-thresh pair next to a strictly better pair competing for the same detection, and a far detection
        sh = np.array([40, 40, 40, 40], np.float64)
        better_t = list(np.asarray(d) + 0)                                # a track equal to the detection: IoU 1
        out.append(_problem(f"s{stage}@{th} 2x3 compete", stage, [t, better_t, list(np.asarray(t) + sh)], [d, list(np.asarray(d) + sh)],
                            sc * 2, th, "at"))
        # nudged to the nearest cost either side that the arithmetic can produce
        for side in (-1, 1):
            for k in range(1, 200):
                if stage == 2:   # move the detection's bottom edge: a taller box overlaps more (lower cost)
                    dd = list(d)
                    dd[3] = _nudge(d[3], -side * k)
                    q = _problem(f"s{stage}@{th} nudged {side:+d}", stage, [t], [dd], None, th, "nudged")
                else:            # move the score: a higher score lowers the fused cost
                    q = _problem(f"s{stage}@{th} nudged {side:+d}", stage, [t], [d], [_nudge(s, -side * k)], th, "nudged")
                c = q["cost"][0, 0]
                if c != th:
                    assert (c > th) == (side > 0) and abs(c - th) < 1e-12, (stage, th, side, c)
                    out.append(q)
                    break
            else:
                raise AssertionError(f"no nudge reaches past {th} on side {side}")
    # one track between two equal detections, each exactly on the stage-2 threshold: IoU (12 - 4) / (12 + 4) = 1/2
    p = _problem("s2 symmetric at 0.5", 2, [[0, 0, 12, 12]], [[-4, 0, 8, 12], [4, 0, 16, 12]], None, 0.5, "at")
    assert (p["cost"] == 0.5).all()
    out.append(p)
    return out


def tie_problems(seed=0):
    """crafted problems with exactly tied costs below the threshold: one track between two mirror-image detections, duplicate
    detections (the same box twice), duplicate tracks, zero-width and zero-height detections (cost 1 against a real track), and
    integer-lattice boxes on a small grid, where many IoUs coincide"""
    rng = np.random.default_rng(seed)
    out = []
    for stage, th in ((1, 0.8), (2, 0.5), (3, 0.7), (1, 0.95)):
        sc = lambda n: None if stage == 2 else [0.9] * n
        out.append(_problem(f"s{stage} symmetric", stage, [[10, 0, 20, 10], [100, 0, 110, 10]],
                            [[5, 0, 15, 10], [15, 0, 25, 10], [100, 0, 110, 10]], sc(3), th, "tie"))
        out.append(_problem(f"s{stage} duplicate dets", stage, [[0, 0, 16, 16], [4, 0, 20, 16]],
                            [[2, 0, 18, 16], [2, 0, 18, 16], [2, 0, 18, 16]], sc(3), th, "tie"))
        out.append(_problem(f"s{stage} duplicate tracks", stage, [[0, 0, 16, 16]] * 3, [[0, 0, 16, 16], [1, 0, 17, 16]], sc(2), th, "tie"))
        out.append(_problem(f"s{stage} zero-area dets", stage, [[0, 0, 16, 16], [32, 0, 48, 16]],
                            [[8, 0, 8, 16], [32, 8, 48, 8], [0, 0, 16, 16], [0, 0, 16, 16], [33, 0, 49, 16]], sc(5), th, "tie"))
        for k in range(6):
            T, D = int(rng.integers(2, 8)), int(rng.integers(2, 8))
            if k == 5:
                T, D = 7, 7
            sz = [4, 8] if stage != 2 else [4, 8, 16]
            tr = [_lattice_box(rng, 6, sz) for _ in range(T)]
            de = [_lattice_box(rng, 6, sz) for _ in range(D)]
            s = None if stage == 2 else rng.choice([0.75, 0.875, 1.0], D).tolist()
            out.append(_problem(f"s{stage} lattice {T}x{D} #{k}", stage, tr, de, s, th, "lattice"))
        for k in range(2):                                                   # beyond the exhaustive size: checked against scipy
            T, D = 14 + 3 * k, 12 + 4 * k
            tr = [_lattice_box(rng, 10, [4, 8]) for _ in range(T)]
            de = [_lattice_box(rng, 10, [4, 8]) for _ in range(D)]
            s = None if stage == 2 else rng.choice([0.75, 0.875, 1.0], D).tolist()
            out.append(_problem(f"s{stage} lattice {T}x{D} large #{k}", stage, tr, de, s, th, "lattice"))
    return out


def _lattice_box(rng, span, sizes):
    x, y = rng.integers(0, span, 2)
    w = int(rng.choice(sizes))
    return [int(x), int(y), int(x) + w, int(y) + w]


def nan_problems(seed=1):
    """(cost, thresh) with whole NaN rows and columns and scattered NaN pairs among finite, partly tied, costs"""
    rng = np.random.default_rng(seed)
    out = []
    for T, D in ((1, 1), (1, 3), (3, 1), (3, 3), (4, 6), (6, 4), (7, 7), (12, 15)):
        c = rng.choice([0.25, 0.5, 0.625, 0.75, 0.8, 1.0], (T, D))
        c[rng.integers(0, T)] = np.nan
        c[:, rng.integers(0, D)] = np.nan
        if T * D > 4:
            c[rng.random((T, D)) < 0.2] = np.nan
        out.append((c, 0.8))
    out.append((np.full((3, 4), np.nan), 0.8))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# score boundaries
# ---------------------------------------------------------------------------------------------------------------------------------
def score_boundaries(track_thresh):
    """scores on and around the three score boundaries of BYTETracker.update, as the tracker compares them (float64): for each of
    0.1, track_thresh and det_thresh = track_thresh + 0.1 the boundary itself, its shortest decimal (0.3 for 0.2 + 0.1 =
    0.30000000000000004), and the float32 value nearest to it with its two float32 neighbours (the detector's scores are float32)"""
    out = []
    for b in (0.1, track_thresh, track_thresh + 0.1):
        f = np.float32(b)
        out += [b, round(b, 12), float(np.nextafter(f, np.float32(0))), float(f), float(np.nextafter(f, np.float32(1)))]
    return sorted(set(out))


def score_class(s, track_thresh):
    """'high' (stage 1 / 3, birth candidate), 'low' (stage 2) or 'dropped', and whether an unmatched high detection is born"""
    det_thresh = track_thresh + 0.1
    if s > track_thresh:
        return "high", not (s < det_thresh)
    if s > 0.1 and s < track_thresh:
        return "low", False
    return "dropped", False


# ---------------------------------------------------------------------------------------------------------------------------------
# integer-lattice sequences
# ---------------------------------------------------------------------------------------------------------------------------------
def max_time_lost(frame_rate, track_buffer):
    return int(frame_rate / 30.0 * track_buffer)


def lattice_sequence(seed, max_lost, track_thresh=0.5, frames=None):
    """per-frame (boxes xyxy float64 integers [n, 4], scores float64 [n], classes int32 [n]) of a small scene on the integer lattice:

      moving objects     whole-pixel velocities, occluded now and then;
      stationary pairs   a stationary object whose detection is, on some frames, replaced by two mirror-image detections (equal IoU);
      duplicates         one object detected twice per frame with the same box and score and two classes (born as two tracks with
                         identical rows from then on);
      gap objects        stationary, seen on frames 0..3, then missing for max_lost, max_lost + 1 and max_lost + 2 frames, then back;
      scores             every value of score_boundaries(track_thresh), cycled over a few detections, and low-score frames;
      zero-area          zero-width and zero-height detections with high scores now and then (born with a degenerate Kalman box);
      empty frames       two frames without detections.

    Returns (seq, info) with info["gaps"] = [(class, last frame seen, first frame back)]."""
    rng = np.random.default_rng(seed)
    n = frames or max(30, max_lost + 12)
    sb = score_boundaries(track_thresh)
    hi = float(np.float32(max(0.9, track_thresh + 0.25)))
    lo = float(np.float32((track_thresh + 0.1) / 2 + 0.05))
    seq = [([], [], []) for _ in range(n)]

    def add(f, box, s, c):
        seq[f][0].append([float(v) for v in box])
        seq[f][1].append(float(s))
        seq[f][2].append(int(c))

    # moving objects
    for o in range(4):
        p = rng.integers(0, 300, 2).astype(np.int64) + 400 * o
        v = rng.integers(-3, 4, 2)
        w = int(rng.choice([16, 24, 32]))
        for f in range(n):
            if rng.random() < 0.12:
                continue
            q = p + v * f
            add(f, [q[0], q[1], q[0] + w, q[1] + w], lo if rng.random() < 0.15 else hi, 10 + o)
    # stationary objects with mirror-image detection pairs (track between two equal detections)
    for o in range(2):
        x, y, w = 2000 + 300 * o, 100, 24
        for f in range(n):
            if f > 2 and f % 4 == 1:
                for dx in (-6, 6):
                    add(f, [x + dx, y, x + dx + w, y + w], hi, 20 + o)
            else:
                add(f, [x, y, x + w, y + w], hi, 20 + o)
    # duplicates: the same box twice, two classes
    for f in range(n):
        for c in (30, 31):
            add(f, [3000, 50 + 2 * f, 3032, 82 + 2 * f], hi, c)
    # gap objects
    gaps = []
    for k, g in enumerate((max_lost, max_lost + 1, max_lost + 2)):
        x = 4000 + 200 * k
        back = 4 + g
        for f in list(range(0, 4)) + list(range(back, n)):
            add(f, [x, 0, x + 32, 32], hi, 40 + k)
        gaps.append((40 + k, 3, back))
    # score boundaries: one stationary object per boundary value, plus a cycling detection next to a moving one
    for k, s in enumerate(sb):
        x = 6000 + 100 * k
        for f in range(1, n, 3):
            add(f, [x, 500, x + 16, 516], s, 50)
    for f in range(n):
        add(f, [7000, 0, 7016, 16], sb[f % len(sb)], 51)
    # zero-area detections
    for f in range(2, n, 5):
        add(f, [8000, 0, 8000, 16], hi, 60)              # zero width
        add(f, [8100, 0, 8116, 0], hi, 61)               # zero height
        add(f, [8200, 8, 8200, 8], hi, 62)               # a point
    out = []
    empty = {n - 4, n - 3} if n > 8 else set()                  # after every gap object's return
    for f, (b, s, c) in enumerate(seq):
        if f in empty:
            b, s, c = [], [], []
        out.append((np.asarray(b, np.float64).reshape(-1, 4), np.asarray(s, np.float64), np.asarray(c, np.int32)))
    return out, dict(gaps=gaps, empty=sorted(empty))


def truncate_xyxy(xywh_f32):
    """AdasPipeline._track's integer boxes: xyxy computed in float32 from xywh, truncated toward zero"""
    bx = np.asarray(xywh_f32, np.float32)
    xyxy = np.stack([bx[:, 0], bx[:, 1], bx[:, 0] + bx[:, 2], bx[:, 1] + bx[:, 3]], 1)
    return np.trunc(xyxy).astype(np.float64)


def all_partial_matchings(T, D):
    """every partial matching of a T x D problem as x arrays (brute force, for checking exact_optimum on tiny problems)"""
    for k in range(min(T, D) + 1):
        for rows in itertools.combinations(range(T), k):
            for cols in itertools.permutations(range(D), k):
                x = np.full(T, -1)
                x[list(rows)] = cols
                yield x
