"""CPU: the tie-heavy tracker inputs of track_edge_cases.py produce the equalities and ties they claim, the exact optimality certificate
accepts optimal assignments and rejects every other kind, and the oracle tracker with an injected solver is the oracle tracker."""
import numpy as np
import pytest

import post_conformance_cases as pc
import track_edge_cases as te
from oracle import post, track

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")        # numpy's 0/0 IoU of zero-area boxes


def test_threshold_problems_sit_exactly_on_and_next_to_each_threshold():
    probs = te.threshold_problems()
    at = [p for p in probs if p["kind"] == "at"]
    seen = set()
    for p in at:
        assert (p["cost"] == p["thresh"]).any(), p["name"]
        seen.add((p["stage"], p["thresh"]))
    assert seen == {(1, 0.5), (1, 0.8), (1, 0.95), (2, 0.5), (3, 0.7)}
    nudged = [p for p in probs if p["kind"] == "nudged"]
    assert len(nudged) == 10
    for p in nudged:
        c, th = p["cost"][0, 0], p["thresh"]
        assert c != th and abs(c - th) < 1e-12, p["name"]
        assert (c > th) == p["name"].endswith("+1"), p["name"]
    for p in probs + te.tie_problems():                 # the tracks' Kalman boxes are exactly the crafted boxes
        assert p["tracker"], p["name"]
        assert p["stage"] == 2 or all(te.score_class(s, 0.5)[0] == "high" for s in p["scores"]), p["name"]


def test_tie_problems_are_tied():
    probs = te.tie_problems()
    assert all(te.has_tie(p["cost"], p["thresh"]) for p in probs if p["kind"] == "tie")
    assert sum(te.has_tie(p["cost"], p["thresh"]) for p in probs) >= 0.8 * len(probs)
    sym = [p for p in probs if "symmetric" in p["name"]]
    assert sym and all(p["cost"][0, 0] == p["cost"][0, 1] < 1 for p in sym)
    zero = [p for p in probs if "zero-area" in p["name"]]
    assert zero and all((p["cost"][:, :2] == 1.0).all() for p in zero)       # a zero-area detection against a real track: IoU 0
    assert max(min(p["cost"].shape) for p in probs) > te.EXHAUSTIVE_MAX       # some are certified against scipy instead


def test_score_boundaries_fall_where_the_tracker_compares():
    # track_thresh 0.2: det_thresh is 0.30000000000000004, so float32(0.3) is born and 0.3 is not
    s = te.score_boundaries(0.2)
    assert 0.2 + 0.1 == 0.30000000000000004 and 0.3 in s and float(np.float32(0.3)) in s
    assert te.score_class(0.3, 0.2) == ("high", False)
    assert te.score_class(float(np.float32(0.3)), 0.2) == ("high", True)
    for tt in te.TRACK_THRESHS:
        s = te.score_boundaries(tt)
        assert te.score_class(0.1, tt)[0] == "dropped" and te.score_class(tt, tt)[0] == "dropped"
        assert te.score_class(tt + 0.1, tt) == ("high", True)
        for b in (0.1, tt, tt + 0.1):
            f = np.float32(b)
            for v in (np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1))):
                assert float(v) in s
        classes = {te.score_class(v, tt) for v in s}
        assert classes == {("dropped", False), ("low", False), ("high", False), ("high", True)}, tt


def test_lattice_sequence_has_what_it_claims():
    seq, info = te.lattice_sequence(5, 3, 0.5)
    boxes = np.concatenate([b for b, _, _ in seq])
    assert (boxes == np.round(boxes)).all()                                             # integer lattice
    assert [f for f, (b, _, _) in enumerate(seq) if len(b) == 0] == info["empty"] and len(info["empty"]) == 2
    wh = boxes[:, 2:] - boxes[:, :2]
    assert (wh[:, 0] == 0).any() and (wh[:, 1] == 0).any() and ((wh == 0).all(1)).any()   # zero width, zero height, points
    dup = 0
    for b, s, c in seq:
        for i in range(len(b)):
            for j in range(i + 1, len(b)):
                if np.array_equal(b[i], b[j]) and s[i] == s[j] and c[i] != c[j]:
                    dup += 1
    assert dup >= len(seq) - 2                                                          # same box twice, two classes
    f = 5                                                                               # mirror-image pair around a stationary box
    b, _, c = seq[f]
    pair = b[c == 20]
    assert len(pair) == 2
    iou = post.ious(np.array([[2000, 100, 2024, 124]], np.float64), pair)
    assert iou[0, 0] == iou[0, 1] < 1
    for cls, last, back in info["gaps"]:
        assert all((c == cls).any() == (f <= last or f >= back) for f, (_, _, c) in enumerate(seq) if f not in info["empty"])
    scores = np.concatenate([s for _, s, _ in seq])
    assert set(te.score_boundaries(0.5)) <= set(scores.tolist())


def test_exact_optimum_is_the_minimum_over_every_partial_matching():
    rng = np.random.default_rng(3)
    for _ in range(60):
        T, D = rng.integers(1, 5, 2)
        c = rng.choice([0.25, 0.5, 0.8, np.nextafter(0.8, 1), 1.0, np.nan], (T, D))
        vals = [te.extended_value(c, 0.8, x) for x in te.all_partial_matchings(T, D)
                if not any(np.isnan(c[i, j]) for i, j in enumerate(x) if j >= 0)]
        assert te.exact_optimum(c, 0.8) == min(vals)


def test_certificate_accepts_optimal_assignments():
    stats = te.CertStats()
    for p in te.threshold_problems() + te.tie_problems():
        x, y, _ = post.lapjv_extended(p["cost"], p["thresh"])
        te.certify(p["cost"], p["thresh"], x, y, stats)
    for c, th in te.nan_problems():
        x, y, _ = post.lapjv_extended(c, th)
        assert not np.isnan(c[np.nonzero(x >= 0)[0], x[x >= 0]]).any()
        te.certify(c, th, x, y, stats)
    assert stats.exhaustive and stats.bounded and stats.at_thresh
    # a tie swapped for an assignment of the same value is just as optimal: duplicate detections
    p = next(q for q in te.tie_problems() if "duplicate dets" in q["name"] and q["stage"] == 1)
    x, y, _ = post.lapjv_extended(p["cost"], p["thresh"])
    free = [j for j in range(3) if j not in x]
    xs = np.where(x == x[0], free[0], x) if free else x[::-1].copy()
    assert not np.array_equal(xs, x)
    te.certify(p["cost"], p["thresh"], xs)


def test_certificate_rejects_every_other_kind_of_assignment():
    th = 0.8
    # deliberately suboptimal: leave a cheap pair unmatched
    c = np.array([[0.25, 1.0], [1.0, 0.5]])
    te.certify(c, th, [0, 1])
    with pytest.raises(AssertionError, match="exceeds the exact optimum"):
        te.certify(c, th, [0, -1])
    # a swapped tie that costs more -- by one ulp of a single entry, which only an exact comparison sees
    c = np.array([[0.5, 0.5], [0.25, np.nextafter(0.25, 0)]])
    te.certify(c, th, [0, 1])
    with pytest.raises(AssertionError, match="exceeds the exact optimum"):
        te.certify(c, th, [1, 0])
    assert float(te.extended_value(c, th, [1, 0])) == float(te.extended_value(c, th, [0, 1]))   # float64 cannot tell them apart
    # a match above the threshold, by one ulp
    up = np.nextafter(th, 1)
    te.certify(np.array([[th]]), th, [0])
    te.certify(np.array([[up]]), th, [-1])
    with pytest.raises(AssertionError, match="> thresh"):
        te.certify(np.array([[up]]), th, [0])
    # a NaN pair matched, and inconsistent or non-matching outputs
    with pytest.raises(AssertionError, match="NaN"):
        te.certify(np.array([[np.nan, 0.3]]), th, [0])
    with pytest.raises(AssertionError, match="partial matching"):
        te.certify(np.array([[0.1, 0.3], [0.2, 0.1]]), th, [0, 0])
    with pytest.raises(AssertionError, match="inverse"):
        te.certify(np.array([[0.1, 0.3], [0.2, 0.1]]), th, [0, 1], [1, 0])
    # beyond the exhaustive size the bound is scipy's answer: a worse assignment is still caught
    rng = np.random.default_rng(0)
    c = rng.choice([0.25, 0.5, 0.75, 1.0], (12, 12))
    x, _, _ = post.lapjv_extended(c, th)
    te.certify(c, th, x)
    worse = x.copy()
    worse[np.argmax(x >= 0)] = -1
    with pytest.raises(AssertionError, match="exceeds scipy"):
        te.certify(c, th, worse)


def test_oracle_nan_costs_are_forbidden_pairs():
    c = np.array([[np.nan, 0.5], [0.2, np.nan], [np.nan, np.nan]])
    x, y, tot = post.lapjv_extended(c, 0.8)
    assert x.tolist() == [1, 0, -1] and y.tolist() == [1, 0] and tot == 0.5 + 0.2 + 0.4


def test_oracle_with_injected_solver_equals_the_oracle():
    """the solver hook changes nothing by itself: the oracle driven by lapjv_extended through the hook (every answer certified) equals
    the oracle on a crowded float-box sequence"""
    seq = pc.crowd_sequence(3, objects=40, frames=16, clutter=10)
    stats = te.CertStats()

    def certified(cost, thresh):
        x, y, tot = post.lapjv_extended(cost, thresh)
        te.certify(cost, thresh, x, y, stats)
        return x, y, tot
    a, b = track.Tracker(), track.Tracker(solver=certified)
    a.reset()
    want = [pc.track_rows(a.update(*f)) for f in seq]
    b.reset()
    got = [pc.track_rows(b.update(*f)) for f in seq]
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    assert stats.problems >= 2 * len(seq) - 2
