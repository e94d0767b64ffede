"""GPU: the multi-camera rig at its real sizes.  AdasPipeline(cameras=8, batch=8) runs YOLOv8l and UFLDv2-r34 (CULane) on 64 frames
per engine call, and 40 on a step of 5 frames per camera.

- Whole plans: each rig network in one engine of max_batch 64 runs batch 64 on frames A, batch 40 on frames B, batch 64 on A again
  (its graph capture) and once more (its replay).  After each of the first three runs every op of the sampled images is within its
  float64 bound (plan_interp.op_ref from its own inputs as the device left them; bit-exact where the op must be); after every run
  every halo of every image is zero; the capture and the replay equal the first run bit for bit in every buffer of every image.  A
  batch-1 engine then runs every frame alone: its network outputs equal the batch-64 / batch-40 outputs of that frame, and every
  buffer of each sampled image equals its batch-1 buffers bit for bit.  The step descriptions at 64 show a GEMM of more tiles than
  SMs, UFLD's weight-stream FC at M = 64 and its tensor-core FC at BN = 64.  The other plan families run at batch 32 (YOLOv7-W6 at
  1280: 16): every image's network outputs equal batch 1, and every op of the last image is within its bound.
- The rig pipeline at 8 x 8: steps of 8, 8, 5 and 8 frames per camera, on host and device frames, through step and through
  step_pipelined + flush, equal one batch-1 engine pair and eight single trackers updated frame by frame in camera order.
- Regrouped multi-tracker calls (rig_scale_cases.SCHEDULE) equal eight trackers updated one at a time in the same order.

Buffers are read one at a time (rig_scale_cases.stream_read): YOLOv8l's at batch 64 are about 10 GB.  One engine is open at a time
in the plan checks.  Each test prints the device memory in use at its peak."""
import re

import numpy as np
import pytest
import torch

import plan_interp as pi
import rig_scale_cases as rc
import synth
import test_gpu_multicam as tgm
import test_gpu_plan_conformance as tpc
from adas_b200 import _capi
from gpu_util import cached_plan

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

RIG = [("yolov8", "l", {}), ("ufldv2", "34", dict(cfg="culane"))]
SAMPLE = {64: [0, 1, 31, 62, 63], 40: [0, 38, 39]}
FAMILIES = [(f, s, kw, 16 if (f, s) == ("yolov7", "w6") else 32) for f, s, kw, _, _ in tpc.PLANS if (f, s, kw) not in RIG]


def _device_in_use():
    free, total = torch.cuda.mem_get_info(0)
    return total - free


class Peak:
    def __init__(self):
        self.v = _device_in_use()

    def note(self):
        self.v = max(self.v, _device_in_use())


def _readback(eng, pb, B, images):
    return rc.stream_read(pb, lambda i: eng.read_buffer(i, B), B, images)


def _op_fails(pb, rb, images, skip, worst, tag):
    return [f"{tag}: op {i} ({kind}) image {b}: {n} elements out of bound (max err / bound {r:.3g})"
            for i, kind, b, n, r in rc.check_images(pb, rb.sampled, images, skip, worst, device="cuda")]


def _worst(w):
    return ", ".join(f"{k} {v:.3g}" for k, v in sorted(w.items()))


def _equal_batch1(pb, path, runs, fails):
    """Every frame of each (frames, outputs, readback, sampled images) run alone in a batch-1 engine: its outputs, and every buffer of
    the sampled images, equal the batched run's."""
    eng = _capi.Engine(path, 0, max_batch=1)
    for x, out, rb, images in runs:
        for j in range(len(x)):
            o1 = eng.infer(x[j:j + 1])
            bad = [k for k in range(len(o1)) if not np.array_equal(o1[k][0], out[k][j])]
            if bad:
                fails.append(f"batch {len(x)} image {j}: outputs {bad} differ from batch 1")
            if j in images:
                r1 = _readback(eng, pb, 1, [])
                diff = [i for i, _ in rc.digest_diff(rb.digests, r1.digests, [j], [0])]
                if diff:
                    fails.append(f"batch {len(x)} image {j}: buffers {diff} differ from batch 1")
    eng.close()


@pytest.mark.slow
@pytest.mark.parametrize("family,scale,kw", RIG, ids=[f"{f}-{s}" for f, s, _ in RIG])
def test_rig_plan_at_batch_64(tmp_path, family, scale, kw):
    peak = Peak()
    pb = tpc.build(family, scale, **kw)
    path = str(tmp_path / f"{family}_{scale}.b200w")
    pb.write(path)
    xa = tpc.frames_in(pb, family, kw, range(64))
    xb = tpc.frames_in(pb, family, kw, range(100, 140))          # 8 cameras x 5 frames
    skip = set(pi.stale_reads(pb))
    eng = _capi.Engine(path, 0, max_batch=64)
    fails, worst, first = [], {64: {}, 40: {}}, {}
    for tag, x in (("eager A", xa), ("eager B", xb), ("capture A", xa), ("replay A", xa)):
        B = len(x)
        out = eng.infer(x)
        peak.note()
        rb = _readback(eng, pb, B, SAMPLE[B] if tag != "replay A" else [])
        if tag != "replay A":
            fails += _op_fails(pb, rb, SAMPLE[B], skip, worst[B], f"{tag} (batch {B})")
        if rb.halo:
            fails.append(f"{tag}: nonzero halo in buffers {rb.halo}")
        if tag in ("eager A", "eager B"):
            first[tag[-1]] = (x, out, rb._replace(sampled=None), SAMPLE[B])
        else:
            diff = sorted({i for i, _ in rc.digest_diff(first["A"][2].digests, rb.digests)})
            if diff:
                fails.append(f"{tag} differs from eager A in buffers {diff}")
            if not all(np.array_equal(a, b) for a, b in zip(out, first["A"][1])):
                fails.append(f"{tag}: network outputs differ from eager A")
        del rb
    steps = [eng.time_step(64, i, 1)[1:] for i in range(eng.num_steps(64))]
    eng.close()
    _equal_batch1(pb, path, [first["A"], first["B"]], fails)
    peak.note()

    kinds = [pi.op_kind(pb, i) for i in range(len(pb.ops))]
    tpc.check_steps(kinds, steps)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = max(int(m.group(1)) for _, d in steps for m in [re.search(r"tiles=(\d+)", d)] if m)
    fcs = [d for k, (_, d) in zip(kinds, steps) if k in ("gemm-tr", "gemm-fc_stream")]
    for B in (64, 40):
        print(f"[rig] {family}-{scale} batch {B}: sampled images {SAMPLE[B]}; worst err / bound: {_worst(worst[B])}")
    print(f"[rig] {family}-{scale} routes at 64: largest GEMM {tiles} tiles on {sms} SMs; FCs {fcs}; "
          f"peak device memory in use {peak.v / 2**30:.1f} GiB")
    assert not fails, "\n".join(fails[:20])
    assert tiles > sms
    if family == "ufldv2":
        assert any(d.startswith("M=64 ") and d.endswith(" fc_stream") for d in fcs), fcs
        if "gemm-tr" in kinds:
            assert any("tr=1" in d and " BN=64 " in d for d in fcs), fcs


@pytest.mark.parametrize("family,scale,kw,B", [pytest.param(*c, marks=[pytest.mark.slow] if c[3] == 16 else [],
                                                            id=f"{c[0]}-{c[1]}-b{c[3]}") for c in FAMILIES])
def test_family_batch_equals_batch1(tmp_path, family, scale, kw, B):
    peak = Peak()
    pb = tpc.build(family, scale, **kw)
    path = str(tmp_path / f"{family}_{scale}.b200w")
    pb.write(path)
    x = tpc.frames_in(pb, family, kw, range(200, 200 + B))
    eng = _capi.Engine(path, 0, max_batch=B)
    out = eng.infer(x)
    peak.note()
    rb = _readback(eng, pb, B, [B - 1])
    eng.close()
    worst, fails = {}, []
    fails += _op_fails(pb, rb, [B - 1], set(pi.stale_reads(pb)), worst, f"batch {B}")
    if rb.halo:
        fails.append(f"nonzero halo in buffers {rb.halo}")
    _equal_batch1(pb, path, [(x, out, rb._replace(sampled=None), [B - 1])], fails)
    print(f"[rig] {family}-{scale} batch {B}: sampled image {B - 1}; worst err / bound: {_worst(worst)}; "
          f"peak device memory in use {peak.v / 2**30:.1f} GiB")
    assert not fails, "\n".join(fails[:20])


# ---- the rig pipeline ----------------------------------------------------------------------------------------------------------------
@pytest.mark.slow
def test_rig_pipeline_8x8_equals_batch1_pair_and_single_trackers():
    """AdasPipeline(cameras=8, batch=8): steps of 8, 8, 5 and 8 frames per camera (the 5-frame step runs the engines at batch 40, a
    batch the pipeline has not built yet) equal, per camera and frame, one batch-1 engine pair with eight trackers updated frame by
    frame in camera order -- detections, lane points and status and track records byte for byte, through step and step_pipelined +
    flush, on host and device frames"""
    from adas_b200.ObjectTracker import BYTETracker
    from adas_b200.pipeline import AdasPipeline
    peak = Peak()
    ypath, _, _ = cached_plan("yolov8", scale="l")
    upath, _, _ = cached_plan("ufldv2", backbone="34", cfg="culane")
    K, F, STEPS = 8, 8, (8, 8, 5, 8)
    n = sum(STEPS)
    frames = np.stack([np.stack([np.roll(synth.frame(300 + 37 * c + f), 16 * c, axis=1) for f in range(n)]) for c in range(K)])
    kw = dict(device=0, track_thresh=0.3)          # the seeded weights score objects in [0.4, 0.5]: births at det_thresh 0.4

    ref = AdasPipeline(ypath, upath, batch=1, sets=1, **kw)
    trackers = [BYTETracker(track_thresh=0.3, names=[], device=0) for _ in range(K)]
    for t in trackers:
        t.reset()
    want = [[None] * n for _ in range(K)]
    for f in range(n):
        for c in range(K):
            ref.tracker = trackers[c]
            want[c][f] = ref.step(frames[c, f:f + 1])
    ref.close()
    assert sum(int(w.counts.sum()) for row in want for w in row) > 0 and sum(len(w.tracks[0]) for row in want for w in row) > 0

    multi = AdasPipeline(ypath, upath, batch=F, sets=1, cameras=K, **kw)
    dev = torch.from_numpy(frames).cuda()
    torch.cuda.synchronize()
    peak.note()
    for pipelined in (False, True):
        for t in multi.trackers:
            t.reset()
        got, keep, o = [], [], 0
        for s, m in enumerate(STEPS):
            on_dev = (s + pipelined) % 2 == 1
            x = dev[:, o:o + m].contiguous() if on_dev else frames[:, o:o + m]
            args = (x.data_ptr(), True, tuple(x.shape[:4])) if on_dev else (x,)
            if pipelined:
                r = multi.step_pipelined(*args)
                if r is not None:
                    got.append(r)
                keep.append(x)                                                 # frames stay valid until their batch returns
            else:
                got.append(multi.step(*args))
            o += m
            peak.note()
        if pipelined:
            got += multi.flush()
        assert len(got) == len(STEPS)
        o = 0
        for s, (rs, m) in enumerate(zip(got, STEPS)):
            assert len(rs) == K
            for c in range(K):
                assert len(rs[c].counts) == m
                for i in range(m):
                    tgm._same_result(tgm._one_frame(rs[c], i), want[c][o + i], (pipelined, s, c, i))
            o += m
    multi.close()
    print(f"[rig] pipeline 8 x 8: peak device memory in use {peak.v / 2**30:.1f} GiB")


# ---- regrouped multi-tracker calls ---------------------------------------------------------------------------------------------------
def _cat(dets):
    return (np.concatenate([d[0] for d in dets]).reshape(-1, 4), np.concatenate([d[1] for d in dets]),
            np.concatenate([d[2] for d in dets]).astype(np.int32))


def _run_schedule(cams, one_at_a_time):
    """Every call of rc.SCHEDULE on eight fresh trackers -> (trackers, records per tracker and frame, association launches, launches
    expected of the multi-tracker calls).  one_at_a_time: each call as plain updates, frame by frame in the call's tracker order; the
    expected count is then one launch per call and frame where any of the call's trackers launched."""
    ts = [_capi.NativeTracker(0, **kw) for kw, _ in cams]
    for t in ts:
        t.reset()
    recs = [[] for _ in ts]
    n0, expected = _capi.launch_count(), 0
    for (kind, g, m), w in zip(rc.SCHEDULE, rc.windows(rc.SCHEDULE)):
        frames = [[rc.stream_frame(cams, c, w[c][k]) for c in g] for k in range(m)]          # [frame][tracker of the call]
        if one_at_a_time:
            for fr in frames:
                l0 = _capi.launch_count()
                for c, d in zip(g, fr):
                    recs[c].append(ts[c].update(*d))
                expected += _capi.launch_count() > l0
        elif kind == "multi":
            counts = np.array([[len(d[1]) for d in fr] for fr in frames], np.int32)
            out = _capi.NativeTracker.update_multi([ts[c] for c in g], counts, *_cat([d for fr in frames for d in fr]))
            for c, r in zip(g, out):
                recs[c] += r
        elif kind == "update":
            recs[g[0]].append(ts[g[0]].update(*frames[0][0]))
        else:
            dets = [fr[0] for fr in frames]
            recs[g[0]] += ts[g[0]].update_batch(np.array([len(d[1]) for d in dets], np.int32), *_cat(dets))
    return ts, recs, _capi.launch_count() - n0, expected


def test_regrouped_multi_tracker_calls_equal_single_trackers():
    """rig_scale_cases.SCHEDULE: update_multi on all eight, in reversed order, with K = 1, with a fresh lead in front of a crowd of
    150, with a lead whose staging grows from a small first call to two crowds, mixed with plain update and update_batch on trackers
    that lead other groups.  Every record, the tracked / lost / removed lists, the process-global track count, each tracker's launch
    count and the number of association launches equal those of eight trackers updated one at a time in the same order."""
    cams = rc.rig_cameras()
    single, want, single_launches, expected = _run_schedule(cams, True)
    want_lists = [tgm._snapshot(t) for t in single]
    want_stats = [t.stats()["launches"] for t in single]
    count_single = _capi.NativeTracker.count()
    multi, got, launches, _ = _run_schedule(cams, False)
    assert _capi.NativeTracker.count() == count_single
    for c in range(8):
        assert len(got[c]) == len(want[c]), c
        for f, (a, b) in enumerate(zip(got[c], want[c])):
            assert a.tobytes() == b.tobytes(), (c, f)
        assert tgm._snapshot(multi[c]) == want_lists[c], c
        assert multi[c].stats()["launches"] == want_stats[c], (c, multi[c].stats(), want_stats[c])
    assert launches == expected < single_launches, (launches, expected, single_launches)
    assert max(len(r) for r in got[2]) > 120                       # the crowds are past the association's 120 shared-memory rows
    assert max(len(r) for r in got[6]) > 300
    print(f"[rig] schedule: {len(rc.SCHEDULE)} calls, {launches} association launches ({single_launches} one tracker at a time), "
          f"largest frame {max(len(r) for rs in got for r in rs)} tracks")
    for t in single + multi:
        t.close()
