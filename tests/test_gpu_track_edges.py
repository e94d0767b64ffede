"""GPU: ByteTrack association and the native tracker on integer-pixel boxes, exact cost ties, threshold boundaries, NaN costs and
non-default tracker settings.  Every device assignment is checked with the exact optimality certificate of track_edge_cases.py; the
native tracker is compared frame by frame with oracle.track.Tracker driven by the device solver (so both break ties alike) whose
every answer is certified."""
import types

import numpy as np
import pytest

import post_conformance_cases as pc
import track_edge_cases as te
import adas_b200  # noqa: F401
from adas_b200 import _capi
from oracle import post, track

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]   # numpy's 0/0 IoU of zero-area boxes


def _dev_lap(cost, thresh):
    (x, y), = _capi.lap([cost], [thresh])
    return x, y


def _following(stats):
    """oracle solver: the device's answer on the oracle's own cost matrix, certified optimal"""
    def solve(cost, thresh):
        x, y = _dev_lap(cost, thresh)
        te.certify(cost, thresh, x, y, stats)
        return x, y
    return solve


# ---- one association stage through every entry point --------------------------------------------------------------------------
def _tracker_assignment(p):
    """x of problem p as the native tracker's fused association solves it in one frame: the tracks are born (class 1000 + i) on the
    frame before, the detections (class j) arrive on the next; a matched track takes its detection's class (vote 2 against 1)"""
    T, D = len(p["tracks"]), len(p["dets"])
    stage, th = p["stage"], p["thresh"]
    nt = _capi.NativeTracker(0, track_thresh=0.5, match_thresh=th if stage == 1 else 0.8)
    nt.reset()
    if stage == 3:
        nt.update(np.zeros((0, 4)), np.zeros(0), np.zeros(0, np.int32))       # births after frame 1 stay unconfirmed
    nt.update(p["tracks"], np.full(T, 0.9), 1000 + np.arange(T, dtype=np.int32))
    sc = np.full(D, 0.3) if stage == 2 else p["scores"]                      # stage 2: low-score detections
    assert stage != 2 or all(te.score_class(s, 0.5)[0] == "low" for s in sc)
    assert stage == 2 or all(te.score_class(s, 0.5)[0] == "high" for s in sc)
    recs = nt.update(p["dets"], sc, np.arange(D, dtype=np.int32))
    frame = 3 if stage == 3 else 2
    x = np.full(T, -1, np.int32)
    for r in recs:
        i = int(r["track_id"]) - 1
        if i < T and int(r["frame_id"]) == frame:
            x[i] = int(r["class_id"])
    nt.close()
    return x


def _y_of(x, D):
    y = np.full(D, -1, np.int32)
    y[x[x >= 0]] = np.nonzero(x >= 0)[0]
    return y


def test_crafted_problems_agree_on_every_entry_point():
    """every crafted problem through lap, associate, iou_cost + lap and a one-frame native tracker update: the device cost matrices
    equal numpy's float64 cost bit for bit, the four assignments are identical, and the assignment is certified optimal"""
    stats = te.CertStats()
    probs = te.threshold_problems() + te.tie_problems()
    n_tracker = 0
    for p in probs:
        cost, th, D = p["cost"], p["thresh"], len(p["dets"])
        dev_cost, = _capi.iou_cost([p["tracks"]], [p["dets"]], None if p["scores"] is None else [p["scores"]])
        assert np.array_equal(dev_cost, cost, equal_nan=True), p["name"]
        x1, y1 = _dev_lap(cost, th)
        x2, y2 = _dev_lap(dev_cost, th)
        x3, y3, c3 = _capi.associate(p["tracks"], p["dets"], p["scores"], th, want_cost=True)
        assert np.array_equal(c3, cost, equal_nan=True), p["name"]
        assert np.array_equal(x1, x2) and np.array_equal(y1, y2), p["name"]
        assert np.array_equal(x1, x3) and np.array_equal(y1, y3), (p["name"], x1, x3)
        if p["tracker"]:
            x4 = _tracker_assignment(p)
            assert np.array_equal(x1, x4), (p["name"], x1, x4)
            n_tracker += 1
        te.certify(cost, th, x1, y1, stats)
        assert np.array_equal(y1, _y_of(x1, D))
    print(f"[edges] crafted: {stats}; {n_tracker} also through the native tracker")
    assert n_tracker == len(probs)


def test_threshold_rule_cost_equal_to_thresh_matches():
    """the rule csrc/track.cu documents: a 1x1 problem at cost exactly thresh matches, one ulp above does not, one ulp below does;
    the same on the crafted box problems of every stage through lap, associate and the native tracker"""
    for th in (0.5, 0.7, 0.8, 0.95, 0.3, 1.0 / 3.0, 0.1, 0.6000000000000001):
        up, down = np.nextafter(th, 2.0), np.nextafter(th, -1.0)
        got = _capi.lap([np.array([[th]]), np.array([[up]]), np.array([[down]])], [th] * 3)
        assert [int(x[0]) for x, _ in got] == [0, -1, 0], th
    n = 0
    for p in te.threshold_problems():
        if len(p["tracks"]) != 1 or len(p["dets"]) != 1:
            continue
        c = p["cost"][0, 0]
        want = 0 if c <= p["thresh"] else -1
        assert p["kind"] == "nudged" or c == p["thresh"]
        x, _, _ = _capi.associate(p["tracks"], p["dets"], p["scores"], p["thresh"])
        assert int(x[0]) == want == int(_tracker_assignment(p)[0]), (p["name"], c, x)
        n += 1
    assert n == 15           # 5 stage thresholds x (on, one reachable step below, one above)


def test_batched_lap_ties_mixed_with_other_problems():
    """one batched lap launch over tied, threshold, NaN and continuous problems in shuffled order: every answer equals the same
    problem solved alone"""
    rng = np.random.default_rng(5)
    probs = [(p["cost"], p["thresh"]) for p in te.threshold_problems() + te.tie_problems()] + te.nan_problems()
    probs += [(pc.lap_cost(k, int(rng.integers(1, 40)), int(rng.integers(1, 40)), k % 2 == 0), 0.8) for k in range(12)]
    order = rng.permutation(len(probs))
    probs = [probs[i] for i in order]
    batched = _capi.lap([c for c, _ in probs], [t for _, t in probs])
    for (c, t), (x, y) in zip(probs, batched):
        xs, ys = _dev_lap(c, t)
        assert np.array_equal(x, xs) and np.array_equal(y, ys)


def test_nan_costs_never_match_and_the_rest_is_optimal():
    """NaN rows, columns and pairs among finite, tied costs: no NaN pair is matched and the assignment is the exact optimum of the
    problem without those pairs; zero-area boxes give the NaN through associate / iou_cost the same way"""
    stats = te.CertStats()
    for c, th in te.nan_problems():
        x, y = _dev_lap(c, th)
        te.certify(c, th, x, y, stats)
    tr = np.array([[0, 0, 0, 10], [5, 5, 5, 5], [0, 0, 10, 10], [20, 0, 30, 0]], np.float64)
    de = np.array([[0, 0, 0, 10], [3, 3, 3, 3], [0, 0, 10, 10], [0, 0, 10, 5], [20, 0, 30, 0]], np.float64)
    for sc in (None, np.full(5, 0.9)):
        for th in (0.5, 0.8):
            x, y, cost = _capi.associate(tr, de, sc, th, want_cost=True)
            with np.errstate(invalid="ignore"):
                want = post.iou_cost(tr, de, sc)
            assert np.array_equal(cost, want, equal_nan=True) and np.isnan(want).sum() == 9
            te.certify(cost, th, x, y, stats)
            xs, ys = _dev_lap(want, th)
            assert np.array_equal(x, xs) and np.array_equal(y, ys)
    print(f"[edges] NaN: {stats}")


# ---- the native tracker against the tie-following oracle --------------------------------------------------------------------------
def _run_oracle(seq, solver, **kw):
    t = track.Tracker(solver=solver, **kw)
    t.reset()
    out = []
    for b, s, c in seq:
        tr = t.update(b, s, c)
        out.append((pc.track_rows(tr), sorted((x.tid, x.state) for x in t.lost), {x.tid for x in t.removed}))
    return out


def _check(recs, want, f, lost=None):
    rows = want[0]
    got = pc.native_rows(recs)
    assert got.shape == rows.shape, (f, got.shape, rows.shape)
    assert np.array_equal(got[:, :4], rows[:, :4]), f                                 # id, state, activation, class: exact
    assert np.allclose(got[:, 4:], rows[:, 4:], rtol=0, atol=1e-6, equal_nan=True), f   # Kalman boxes (NaN for zero height), score
    if lost is not None:
        assert sorted(zip(lost["track_id"].tolist(), lost["state"].tolist())) == want[1], f


def _chunks(n):
    sizes, k, f = (3, 1, 5, 2, 8, 4), 0, 0
    while f < n:
        yield f, min(sizes[k % len(sizes)], n - f)
        f += sizes[k % len(sizes)]
        k += 1


def _track_id_of(rows, cls):
    ids = rows[rows[:, 3] == cls][:, 0]
    return int(ids[0]) if len(ids) else None


def _check_ageing(want, info, max_lost):
    """the gap objects, last matched on frame L and missing for g = max_time_lost, + 1, + 2 frames.  A lost track is aged out on the
    first frame F > L + 1 with F - L > max_time_lost, after that frame's association; the reference keeps it in its lost list for one
    more frame, so a detection returning on the very next frame re-finds it with its old id.  Hence: removed before the detection
    returns iff g >= max(2, max_time_lost + 1), and back with a new id iff g >= max(3, max_time_lost + 2)."""
    for k, (cls, last, back) in enumerate(info["gaps"]):
        g = max_lost + k
        assert back == last + g + 1
        tid = _track_id_of(want[last][0], cls)
        assert tid is not None
        removed = tid in want[back - 1][2]
        assert removed == (g >= max(2, max_lost + 1)), (k, g, max_lost)
        if removed:                      # on its removal frame it is still listed as lost, in state Removed
            r = last + max(2, max_lost + 1)
            assert tid not in want[r - 1][2] and tid in want[r][2] and (tid, track.REMOVED) in want[r][1]
        assert (_track_id_of(want[back][0], cls) == tid) == (g < max(3, max_lost + 2)), (k, g, max_lost)


@pytest.mark.parametrize("frame_rate", [10, 25, 30, 60])
@pytest.mark.parametrize("track_buffer", [1, 3, 30, 90])
def test_native_tracker_matches_tie_following_oracle_settings_grid(frame_rate, track_buffer):
    """integer-box sequences with duplicates, mirror-image detection pairs, score-boundary values, zero-area detections, empty frames
    and lost gaps of max_time_lost, + 1 and + 2 frames, for every match_thresh x track_thresh: `update` and `update_batch` (ragged
    chunks) equal the oracle driven by the certified device solver frame by frame"""
    max_lost = te.max_time_lost(frame_rate, track_buffer)
    stats = te.CertStats()
    for mt in te.MATCH_THRESHS:
        for tt in te.TRACK_THRESHS:
            kw = dict(track_thresh=tt, track_buffer=track_buffer, match_thresh=mt, frame_rate=frame_rate)
            seq, info = te.lattice_sequence(frame_rate * 1000 + track_buffer, max_lost, tt)
            want = _run_oracle(seq, _following(stats), **kw)
            _check_ageing(want, info, max_lost)
            nt = _capi.NativeTracker(0, **kw)
            nt.reset()
            for f, (b, s, c) in enumerate(seq):
                _check(nt.update(b, s, c), want[f], (mt, tt, f), nt.get(1))
                if f in [back - 1 for _, _, back in info["gaps"]]:
                    assert {int(i) for i in nt.get(2)["track_id"]} == want[f][2], (mt, tt, f)
            nt.close()
            nt = _capi.NativeTracker(0, **kw)
            nt.reset()
            for f0, k in _chunks(len(seq)):
                chunk = seq[f0:f0 + k]
                recs = nt.update_batch([len(s) for _, s, _ in chunk], np.concatenate([b for b, _, _ in chunk]).reshape(-1, 4),
                                       np.concatenate([s for _, s, _ in chunk]), np.concatenate([c for _, _, c in chunk]))
                for j, r in enumerate(recs):
                    _check(r, want[f0 + j], (mt, tt, f0 + j))
                _check(recs[-1], want[f0 + k - 1], (mt, tt, f0 + k - 1), nt.get(1))
            nt.close()
    print(f"[edges] frame_rate {frame_rate} track_buffer {track_buffer} (max_time_lost {max_lost}): {stats}")


def test_zero_area_detections_never_match_and_leave_other_tracks_alone():
    """zero-width, zero-height and point detections (high scores, so they are born, with a zero-width or NaN Kalman box) among real
    objects: they never match anything, and the real objects' tracks equal those of the same sequence without them"""
    rng = np.random.default_rng(11)
    real, degen = [], []
    for f in range(16):
        b = [[100 * o + f * (o % 3), 50, 100 * o + f * (o % 3) + 32, 82] for o in range(5)]
        real.append((np.array(b, np.float64), np.full(5, 0.9), np.arange(5, dtype=np.int32)))
        d = [[110, 50, 110, 82], [200, 60, 232, 60], [350, 60, 350, 60], [0, 0, 0, 0]] if f % 2 == 0 else [[110, 50, 110, 82]]
        degen.append((np.array(d, np.float64), np.full(len(d), float(rng.choice([0.9, 0.3]))), np.full(len(d), 9, np.int32)))
    mixed = [(np.concatenate([a[0], d[0]]), np.concatenate([a[1], d[1]]), np.concatenate([a[2], d[2]])) for a, d in zip(real, degen)]
    stats = te.CertStats()
    want = _run_oracle(mixed, _following(stats))
    alone = _run_oracle(real, _following(stats))
    nt = _capi.NativeTracker(0)
    nt.reset()
    born = set()
    for f, (b, s, c) in enumerate(mixed):
        recs = nt.update(b, s, c)
        _check(recs, want[f], f, nt.get(1))
        deg = recs[recs["class_id"] == 9]
        assert (deg["frame_id"] == deg["start_frame"]).all(), f          # a degenerate track is never matched after its birth
        born |= set(deg["track_id"].tolist())
        got = pc.native_rows(recs[recs["class_id"] != 9])
        ref = alone[f][0]
        assert np.array_equal(got[:, 1:4], ref[:, 1:4]) and np.allclose(got[:, 4:], ref[:, 4:], rtol=0, atol=1e-6), f
    assert len(born) > 8
    nt.close()


def test_pipeline_tracker_stage_truncates_float_boxes_like_the_oracle():
    """the product path: AdasPipeline._track turns float32 xywh detections into integer xyxy (truncation toward zero, also for
    corners in (-1, 0)) and feeds BYTETracker.update_batch_arrays; every frame's records equal the tie-following oracle's on the
    same integer boxes"""
    from adas_b200.ObjectTracker import BYTETracker
    from adas_b200.pipeline import AdasPipeline, StepResult
    rng = np.random.default_rng(3)
    seq, _ = te.lattice_sequence(77, 3, 0.5, frames=24)
    B, max_det = 4, 64
    stub = types.SimpleNamespace(tracker=BYTETracker(names=[]), class_names=None)
    stub.tracker.reset()
    ints, got = [], []
    for step in range(len(seq) // B):
        boxes = np.zeros((B, max_det, 4), np.float32)
        scores = np.zeros((B, max_det), np.float32)
        ids = np.zeros((B, max_det), np.int32)
        counts = np.zeros(B, np.int32)
        for f in range(B):
            b, s, c = seq[step * B + f]
            n = len(s)
            xy = b[:, :2] + rng.uniform(0, 0.999, (n, 2))
            xy[::5] -= b[::5, :2] + 0.5                                     # corners in (-1, 0): truncation gives 0, not -1
            wh = (b[:, 2:] - b[:, :2]) + rng.uniform(0, 0.999, (n, 2))
            boxes[f, :n] = np.concatenate([xy, wh], 1).astype(np.float32)
            scores[f, :n], ids[f, :n], counts[f] = s.astype(np.float32), c, n
            xyxy = te.truncate_xyxy(boxes[f, :n])
            assert (xyxy[::5, :2] == 0).all() and (xyxy == np.round(xyxy)).all()
            ints.append((xyxy, scores[f, :n].astype(np.float64), ids[f, :n].copy()))
        r = StepResult((boxes, scores, ids, np.zeros((B, max_det), np.int32), counts, counts.copy()),
                       (np.zeros((B, 4, 1, 2), np.int32), np.zeros((B, 4), np.int32), np.zeros((B, 4), np.uint8), None))
        AdasPipeline._track(stub, r)
        got += list(r.tracks)
    stats = te.CertStats()
    want = _run_oracle(ints, _following(stats))
    labels = stub.tracker._label_list
    for f, recs in enumerate(got):
        rows = pc.native_rows(recs)
        rows[:, 3] = [labels[int(c)] for c in rows[:, 3]]
        assert rows.shape == want[f][0].shape, f
        assert np.array_equal(rows[:, :4], want[f][0][:, :4]), f
        assert np.allclose(rows[:, 4:], want[f][0][:, 4:], rtol=0, atol=1e-6, equal_nan=True), f
    print(f"[edges] pipeline: {stats}")
