"""GPU: several cameras through one association launch per frame.  adas_tracker_update_multi against K single trackers updated one
after another frame by frame (camera 0 frame f, camera 1 frame f, ..., then frame f + 1), every record compared byte for byte
(track ids and the process-global track count included); the launch count; the refused arguments; and AdasPipeline(cameras=K)
against K single-camera pipelines fed the same streams."""
import ctypes as C

import numpy as np
import pytest
import torch

import synth
import track_edge_cases as te
import adas_b200  # noqa: F401
from adas_b200 import _capi
from gpu_util import cached_plan

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

N_FRAMES = 48
CHUNKS = (3, 1, 5, 2, 8, 4, 7)


def _empty():
    return np.zeros((0, 4), np.float64), np.zeros(0, np.float64), np.zeros(0, np.int32)


def _golden_stream(seed, nobj, offset):
    """a sequence of tests/golden/track.npz (synth.track_sequence) from frame `offset` on, after `offset % 3` empty frames"""
    seq = synth.track_sequence(seed, frames=45, objects=nobj)[offset:]
    out = [_empty() for _ in range(offset % 3)]
    for b, s, l in seq:
        out.append((np.asarray(b, np.float64).reshape(-1, 4), np.asarray(s, np.float64), np.array([int(x[5:]) for x in l], np.int32)))
    return out


def _crowded_stream(n_obj=150, seed=4):
    """more tracks than the association's shared-memory route holds (ASSOC_SMEM_ROWS = 120 rows): a moving grid of objects"""
    rng = np.random.default_rng(seed)
    base = np.array([[40 * (i % 15), 40 * (i // 15)] for i in range(n_obj)], np.float64)
    out = []
    for f in range(N_FRAMES):
        keep = rng.random(n_obj) > 0.1
        xy = base[keep] + f
        b = np.concatenate([xy, xy + 24], 1)
        s = np.where(rng.random(len(b)) < 0.85, 0.9, 0.3)
        out.append((b, s, np.arange(n_obj, dtype=np.int32)[keep] % 7))
    return out


def _crafted_stream(match_thresh):
    """the crafted threshold and tie problems of track_edge_cases as (tracks frame, detections frame, two empty frames)"""
    out = []
    for p in te.threshold_problems() + te.tie_problems():
        if p["stage"] == 1 and p["thresh"] != match_thresh:
            continue
        T, D = len(p["tracks"]), len(p["dets"])
        sc = np.full(D, 0.3) if p["stage"] == 2 else np.asarray(p["scores"], np.float64)
        out.append((p["tracks"], np.full(T, 0.9), 1000 + np.arange(T, dtype=np.int32)))
        out.append((p["dets"], sc, np.arange(D, dtype=np.int32)))
        out += [_empty(), _empty()]
    return out


def _cameras():
    """(tracker settings, per-frame detections) of eight cameras of different content and settings"""
    lat_a, _ = te.lattice_sequence(11, te.max_time_lost(30, 30), 0.5)
    lat_b, _ = te.lattice_sequence(12, te.max_time_lost(10, 3), 0.2)
    return [
        (dict(), lat_a),
        (dict(), _golden_stream(0, 8, 0)),
        (dict(), _crowded_stream()),
        (dict(), []),                                                             # no detections at all
        (dict(match_thresh=0.5, track_buffer=1), _crafted_stream(0.5)),
        (dict(match_thresh=0.95, track_buffer=1), _crafted_stream(0.95)),
        (dict(), _golden_stream(3, 25, 9)),
        (dict(track_thresh=0.2, frame_rate=10, track_buffer=3), lat_b),
    ]


SUBSETS = {1: [2], 2: [0, 3], 3: [4, 2, 1], 8: list(range(8))}


def _streams(cams, n):
    return [(kw, [seq[f] if f < len(seq) else _empty() for f in range(n)]) for kw, seq in cams]


def _snapshot(nt):
    return tuple(nt.get(w).tobytes() for w in (0, 1, 2))


def _run_single(streams, n):
    ts = [_capi.NativeTracker(0, **kw) for kw, _ in streams]
    for t in ts:
        t.reset()
    recs = [[None] * n for _ in ts]
    for f in range(n):
        for c, (t, (_, seq)) in enumerate(zip(ts, streams)):
            recs[c][f] = t.update(*seq[f])
    return ts, recs


def _run_multi(streams, n):
    ts = [_capi.NativeTracker(0, **kw) for kw, _ in streams]
    for t in ts:
        t.reset()
    recs = [[] for _ in ts]
    f0, k = 0, 0
    while f0 < n:
        m = min(CHUNKS[k % len(CHUNKS)], n - f0)
        frames = [[seq[f] for _, seq in streams] for f in range(f0, f0 + m)]                    # [frame][camera]
        counts = np.array([[len(d[1]) for d in fr] for fr in frames], np.int32)
        flat = [d for fr in frames for d in fr]
        out = _capi.NativeTracker.update_multi(ts, counts, np.concatenate([d[0] for d in flat]).reshape(-1, 4),
                                               np.concatenate([d[1] for d in flat]), np.concatenate([d[2] for d in flat]))
        for c in range(len(ts)):
            recs[c] += out[c]
        f0 += m
        k += 1
    return ts, recs


@pytest.mark.parametrize("k", sorted(SUBSETS))
def test_multi_tracker_equals_interleaved_single_trackers(k):
    """K cameras with different settings and content (golden sequences at different offsets, tie / threshold lattices, crafted
    at-threshold problems, a camera past the shared-memory route, a camera without detections) through adas_tracker_update_multi in
    ragged chunks: every record of every frame, and the tracked / lost / removed lists afterwards, equal byte for byte those of K
    single trackers updated frame by frame in camera order"""
    cams = [_cameras()[i] for i in SUBSETS[k]]
    n = max(N_FRAMES, max(len(s) for _, s in cams))
    streams = _streams(cams, n)
    single, want = _run_single(streams, n)
    want_lists = [_snapshot(t) for t in single]
    want_launches = [t.stats()["launches"] for t in single]
    count_single = _capi.NativeTracker.count()
    multi, got = _run_multi(streams, n)
    assert _capi.NativeTracker.count() == count_single
    n_rec, crowded = 0, 0
    for c in range(k):
        assert len(got[c]) == n
        for f in range(n):
            assert got[c][f].tobytes() == want[c][f].tobytes(), (k, c, f)
            n_rec += len(got[c][f])
        assert _snapshot(multi[c]) == want_lists[c], (k, c)
        st = multi[c].stats()
        assert st["frames"] == n and st["launches"] == want_launches[c], (c, st, want_launches[c])
        crowded = max(crowded, max(len(r) for r in got[c]))
    assert n_rec > 0
    if 2 in SUBSETS[k]:
        assert crowded > 120                      # the crowded camera's tracks are past the shared-memory route
    for t in single + multi:
        t.close()


def test_eight_cameras_make_one_association_launch_per_frame():
    """adas_launch_count: eight cameras that all associate on every frame after the first take one launch per frame together,
    eight single trackers take eight; each tracker counts the shared launch once"""
    streams = _streams([(dict(), _crowded_stream(6, seed=c)) for c in range(8)], 24)
    for kw, seq in streams:                                            # every camera has detections on every frame
        assert all(len(s) > 0 for _, s, _ in seq) and (seq[0][1] > 0.6).any()
    n0 = _capi.launch_count()
    single, _ = _run_single(streams, 24)
    n_single = _capi.launch_count() - n0
    n0 = _capi.launch_count()
    multi, _ = _run_multi(streams, 24)
    n_multi = _capi.launch_count() - n0
    assert n_multi == 23 and n_single == 8 * 23, (n_multi, n_single)
    assert all(t.stats()["launches"] == 23 for t in single + multi)
    for t in single + multi:
        t.close()


def test_refused_arguments_leave_every_tracker_unchanged():
    """k < 1, a null or repeated tracker, trackers on different devices and negative counts are refused with an error, and no
    tracker (nor the global track count) moves"""
    streams = _streams([(dict(), _golden_stream(1, 14, 0)), (dict(), _golden_stream(2, 4, 3))], 6)
    ts, _ = _run_multi(streams, 6)
    other = _capi.NativeTracker(1)                     # device 1: the handle is only created, it never touches a device
    before = [_snapshot(t) for t in ts] + [_capi.NativeTracker.count()] + [tuple(t.stats().values()) for t in ts]
    b, s, c = streams[0][1][0]
    n = len(s)
    lib = _capi.lib()

    def call(handles, k, counts):
        hs = (C.c_void_p * max(1, len(handles)))(*[h for h in handles])
        cnt = np.asarray(counts, np.int32)
        bb = np.ascontiguousarray(np.concatenate([b] * 2), np.float64)
        ss = np.ascontiguousarray(np.concatenate([s] * 2), np.float64)
        cc = np.ascontiguousarray(np.concatenate([c] * 2), np.int32)
        out = np.zeros(4 * 256, _capi.TRACK_DTYPE)
        n_out = np.zeros(4, np.int32)
        rc = lib.adas_tracker_update_multi(hs, k, 1, cnt.ctypes.data_as(C.c_void_p), bb.ctypes.data_as(C.c_void_p), ss.ctypes.data_as(C.c_void_p),
                                           cc.ctypes.data_as(C.c_void_p), 256, out.ctypes.data_as(C.c_void_p), n_out.ctypes.data_as(C.c_void_p))
        return rc, lib.adas_last_error().decode()

    h0, h1 = ts[0]._h.value, ts[1]._h.value
    bad = {
        "k = 0": ([h0, h1], 0, [n, n]),
        "k = -1": ([h0, h1], -1, [n, n]),
        "null tracker": ([h0, None], 2, [n, n]),
        "repeated tracker": ([h0, h1, h0], 3, [n, n, 0]),
        "other device": ([h0, other._h.value], 2, [n, n]),
        "negative count": ([h0, h1], 2, [2 * n + 1, -1]),
    }
    for name, (hs, k, counts) in bad.items():
        rc, msg = call(hs, k, counts)
        assert rc != 0 and msg, name
        after = [_snapshot(t) for t in ts] + [_capi.NativeTracker.count()] + [tuple(t.stats().values()) for t in ts]
        assert after == before, name
    with pytest.raises(Exception):
        _capi.NativeTracker.update_multi([ts[0], ts[0]], [[n, n]], np.concatenate([b, b]), np.concatenate([s, s]), np.concatenate([c, c]))
    assert [_snapshot(t) for t in ts] + [_capi.NativeTracker.count()] + [tuple(t.stats().values()) for t in ts] == before
    rc, msg = call([h0, h1], 2, [n, n])                                    # the same trackers still advance
    assert rc == 0, msg
    for t in ts + [other]:
        t.close()


# ---- the pipeline ------------------------------------------------------------------------------------------------------------------
def _same_result(a, b, where):
    assert np.array_equal(a.counts, b.counts) and np.array_equal(a.n_candidates, b.n_candidates), where
    for i, n in enumerate(a.counts):
        for x, y in ((a.boxes, b.boxes), (a.scores, b.scores), (a.class_ids, b.class_ids), (a.cand_index, b.cand_index)):
            assert np.array_equal(x[i, :n], y[i, :n]), where
    assert np.array_equal(a.lane_npts, b.lane_npts) and np.array_equal(a.lane_status, b.lane_status), where
    for i in range(a.lane_pts.shape[0]):
        for l in range(4):
            assert np.array_equal(a.lane_pts[i, l, :a.lane_npts[i, l]], b.lane_pts[i, l, :b.lane_npts[i, l]]), where
    assert len(a.tracks) == len(b.tracks), where
    for x, y in zip(a.tracks, b.tracks):
        assert x.tobytes() == y.tobytes(), where


def _one_frame(r, i):
    """frame i of a StepResult as a one-frame StepResult"""
    from adas_b200.pipeline import StepResult
    s = StepResult((r.boxes[i:i + 1], r.scores[i:i + 1], r.class_ids[i:i + 1], r.cand_index[i:i + 1], r.counts[i:i + 1], r.n_candidates[i:i + 1]),
                   (r.lane_pts[i:i + 1], r.lane_npts[i:i + 1], r.lane_status[i:i + 1], None))
    s.tracks = [r.tracks[i]]
    return s


def test_pipeline_cameras_equal_single_camera_pipelines():
    """AdasPipeline(cameras=3): one detect call for the frames of all cameras and one tracker call per step give, per camera and
    frame, the detections, lane points / status and track records of three single-camera pipelines updated frame by frame in camera
    order -- through step and through step_pipelined + flush, on host and on device frames; a mismatched frame size is refused"""
    from adas_b200.pipeline import AdasPipeline
    ypath, _, _ = cached_plan("yolov8", scale="l")
    upath, _, _ = cached_plan("ufldv2", backbone="18")
    K, F, S = 3, 4, 3
    frames = np.stack([np.stack([np.roll(synth.frame(60 + 7 * c + f), 16 * c, axis=1) for f in range(S * F)]) for c in range(K)])
    kw = dict(device=0, track_thresh=0.3)          # the seeded weights score objects in [0.4, 0.5]: births at det_thresh 0.4
    singles = [AdasPipeline(ypath, upath, batch=1, sets=1, **kw) for _ in range(K)]
    for p in singles:
        p.tracker.reset()
    want = [[None] * (S * F) for _ in range(K)]
    for f in range(S * F):
        for c in range(K):
            want[c][f] = singles[c].step(frames[c, f:f + 1])
    for p in singles:
        p.close()
    dets = sum(int(w.counts.sum()) for row in want for w in row)
    tracks = sum(len(w.tracks[0]) for row in want for w in row)
    assert dets > 0 and tracks > 0

    multi = AdasPipeline(ypath, upath, batch=F, sets=2, depth=2, cameras=K, **kw)
    assert len(multi.trackers) == K and multi.tracker is multi.trackers[0]
    dev = torch.from_numpy(frames).cuda()
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        multi.step([frames[0, :F], frames[1, :F], frames[2, :F, :360]])
    with pytest.raises(ValueError):
        multi.step(frames[:2, :F])
    for pipelined in (False, True):
        for t in multi.trackers:
            t.reset()
        got, keep = [], []
        for s in range(S):
            on_dev = (s + pipelined) % 2 == 1
            x = dev[:, s * F:(s + 1) * F].contiguous() if on_dev else frames[:, s * F:(s + 1) * F]
            args = (x.data_ptr(), True, tuple(x.shape[:4])) if on_dev else (x if s != 1 else list(x),)
            if pipelined:
                r = multi.step_pipelined(*args)
                if r is not None:
                    got.append(r)
                keep.append(x)                                                 # frames stay valid until their batch returns
            else:
                got.append(multi.step(*args))
        if pipelined:
            got += multi.flush()
        assert len(got) == S
        for s, rs in enumerate(got):
            assert len(rs) == K
            for c in range(K):
                assert len(rs[c].counts) == F
                for i in range(F):
                    _same_result(_one_frame(rs[c], i), want[c][s * F + i], (pipelined, s, c, i))
    multi.close()
