"""GPU: a rig of cameras of different frame sizes through one adas_detect_pair_rig call.  Per camera, the boxes, scores, classes,
candidate indices and counts, the lane points and status, and both networks' input images equal those of adas_detect_pair on that
camera's frames alone, byte for byte (YOLOv8l + UFLDv2 and YOLOv5 + UFLD v1, host and device frames); a rig of one size equals
adas_detect_pair on the stacked frames; the 16-camera limit, every refusal, the follow-up calls that need frames of one size, and
AdasPipeline(frame_sizes=...) against single-camera pipelines."""
import ctypes as C

import numpy as np
import pytest
import torch

import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi
from gpu_util import cached_plan

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

# (H, W): no YOLO letterbox (640 x 640), the pad_w path (taller than wide), upscaling (500 x 333) and 64-bit offsets (3840 x 2160)
RIG = [(1080, 1920), (720, 1280), (640, 640), (1280, 720), (500, 333), (2160, 3840)]
F = 3
MAX_BATCH = len(RIG) * F
NMS_IOU = 0.45


@pytest.fixture(scope="module")
def pairs():
    out = {}
    for name, (yk, ykw), (uk, ukw) in (("v8_v2", ("yolov8", dict(scale="l")), ("ufldv2", dict(backbone="18"))),
                                       ("v5_v1", ("yolov5", dict(scale="n")), ("ufldv1", dict(backbone="18")))):
        y = _capi.Engine(cached_plan(yk, **ykw)[0], 0, max_batch=MAX_BATCH)
        u = _capi.Engine(cached_plan(uk, **ukw)[0], 0, max_batch=MAX_BATCH)
        out[name] = (y, u)
    yield out
    for y, u in out.values():
        y.close()
        u.close()


def _frames(sizes, f=F, seed=0):
    return [np.stack([synth.frame(seed + 31 * c + i, h, w) for i in range(f)]) for c, (h, w) in enumerate(sizes)]


def _frame(r, i):
    """the valid part of frame i of a detect_pair result"""
    (bx, sc, cl, ix, cnt, nc), (pts, npts, st, _) = r
    n = int(cnt[i])
    return (bx[i, :n].tobytes(), sc[i, :n].tobytes(), cl[i, :n].tobytes(), ix[i, :n].tobytes(), n, int(nc[i]), npts[i].tobytes(),
            st[i].tobytes(), tuple(pts[i, l, :npts[i, l]].tobytes() for l in range(4)))


def _net_input(e, batch):
    """buffer 0 (the padded fp16 network input, halo and letterbox border included) as [batch, rows, C]"""
    b = e.read_buffer(0, batch)
    return b.reshape(batch, -1, b.shape[1])


def _box_score(y, u, cams):
    """the highest of a few thresholds at which the seeded weights detect objects in the largest cameras"""
    for bs in (0.4, 0.3, 0.2, 0.1, 0.05, 0.02):
        (_, _, _, _, cnt, _), _ = _capi.detect_pair_rig(y, u, cams, bs, NMS_IOU)
        cnt = cnt.reshape(len(cams), -1)
        if cnt[0].sum() > 0 and cnt[-1].sum() > 0:
            return bs
    raise AssertionError("no detections in the largest cameras at any threshold")


@pytest.mark.parametrize("pair", ["v8_v2", "v5_v1"])
def test_rig_equals_detect_pair_per_camera(pairs, pair):
    y, u = pairs[pair]
    cams = _frames(RIG)
    bs = _box_score(y, u, cams)
    dev = [torch.from_numpy(a).cuda() for a in cams]
    torch.cuda.synchronize()
    for on_device in (False, True):
        arg = [(t.data_ptr(), tuple(t.shape[:3])) for t in dev] if on_device else cams
        rig = _capi.detect_pair_rig(y, u, arg, bs, NMS_IOU, on_device=on_device)
        yin, uin = _net_input(y, MAX_BATCH), _net_input(u, MAX_BATCH)
        (_, _, _, _, cnt, _), (_, npts, status, _) = rig
        assert cnt.shape == (MAX_BATCH,)
        assert cnt[:F].sum() > 0 and cnt[-F:].sum() > 0, cnt                      # not a vacuous comparison
        assert npts[:F].sum() > 0 and npts[-F:].sum() > 0 and status.any(), npts
        for c, (h, w) in enumerate(RIG):
            if on_device:
                want = _capi.detect_pair(y, u, dev[c].data_ptr(), bs, NMS_IOU, on_device=True, shape=(F, h, w))
            else:
                want = _capi.detect_pair(y, u, cams[c], bs, NMS_IOU)
            for i in range(F):
                assert _frame(rig, c * F + i) == _frame(want, i), (pair, on_device, c, i)
            assert np.array_equal(yin[c * F:(c + 1) * F], _net_input(y, F)), (pair, on_device, c)
            assert np.array_equal(uin[c * F:(c + 1) * F], _net_input(u, F)), (pair, on_device, c)


def test_rig_of_one_size_equals_detect_pair(pairs):
    y, u = pairs["v8_v2"]
    cams = _frames([(720, 1280)] * 3, seed=100)
    rig = _capi.detect_pair_rig(y, u, cams, 0.4, NMS_IOU)
    want = _capi.detect_pair(y, u, np.concatenate(cams), 0.4, NMS_IOU)
    assert rig[0][4].sum() > 0
    for i in range(3 * F):
        assert _frame(rig, i) == _frame(want, i), i


def test_sixteen_cameras_run_and_seventeen_are_refused(pairs):
    y, u = pairs["v8_v2"]
    sizes = [RIG[c % 5] for c in range(16)]                     # every size but 4K, one frame each
    cams = _frames(sizes, f=1, seed=200)
    rig = _capi.detect_pair_rig(y, u, cams, 0.4, NMS_IOU)
    for c in (0, 7, 15):
        want = _capi.detect_pair(y, u, cams[c], 0.4, NMS_IOU)
        assert _frame(rig, c) == _frame(want, 0), c
    with pytest.raises(Exception, match="17 cameras"):
        _capi.detect_pair_rig(y, u, cams + [cams[0]], 0.4, NMS_IOU)


def _raw(y, u, table, k, f, max_det=64, null_out=None):
    """adas_detect_pair_rig through ctypes with every argument under the caller's control: (rc, message)"""
    B = max(1, k * f)
    mp = 128                                                    # at least any lane engine's points per lane
    outs = [np.empty((B, max_det, 4), np.float32), np.empty((B, max_det), np.float32), np.empty((B, max_det), np.int32),
            np.empty((B, max_det), np.int32), np.empty(B, np.int32), np.empty(B, np.int32), np.empty((B, 4, mp, 2), np.int32),
            np.empty((B, 4), np.int32), np.empty((B, 4), np.uint8)]
    ptrs = [None if i == null_out else a.ctypes.data_as(C.c_void_p) for i, a in enumerate(outs)]
    rc = _capi.lib().adas_detect_pair_rig(y._h, u._h, table, k, f, 0, C.c_double(0.4), C.c_double(NMS_IOU), max_det, *ptrs)
    return rc, _capi.lib().adas_last_error().decode()


def test_refusals_leave_the_engines_working(pairs):
    y, u = pairs["v8_v2"]
    y5, u1 = pairs["v5_v1"]
    sizes = RIG[:3]
    cams = _frames(sizes, f=2, seed=300)
    before = _capi.detect_pair_rig(y, u, cams, 0.4, NMS_IOU)

    def table(entries):
        return (_capi.RigCamera * max(1, len(entries)))(*[_capi.RigCamera(p, h, w) for p, h, w in entries])

    ok = [(a.ctypes.data, a.shape[1], a.shape[2]) for a in cams]
    big = [ok[c % 3] for c in range(17)]
    cases = {
        "k = 0": (y, u, table(ok), 0, 2, None),
        "k = 17": (y, u, table(big), 17, 1, None),
        "F = 0": (y, u, table(ok), 3, 0, None),
        "k * F above max_batch": (y, u, table(ok), 3, MAX_BATCH // 3 + 1, None),
        "null camera table": (y, u, None, 3, 2, None),
        "null frame pointer": (y, u, table([ok[0], (None, 720, 1280), ok[2]]), 3, 2, "camera 1"),
        "zero rows": (y, u, table([ok[0], ok[1], (ok[2][0], 0, 640)]), 3, 2, "camera 2"),
        "zero columns": (y, u, table([(ok[0][0], 1080, 0), ok[1], ok[2]]), 3, 2, "camera 0"),
        "empty letterbox": (y, u, table([ok[0], (ok[1][0], 5000, 1), ok[2]]), 3, 2, "camera 1"),
        "two detectors": (y, y5, table(ok), 3, 2, None),
        "two lane engines": (u1, u, table(ok), 3, 2, None),
        "swapped pair": (u, y, table(ok), 3, 2, None),
    }
    for name, (ye, ue, tab, k, f, names) in cases.items():
        rc, msg = _raw(ye, ue, tab, k, f)
        assert rc != 0 and msg, name
        if names:
            assert names in msg, (name, msg)
    for i in range(9):                                          # every output pointer; n_candidates (5) may be null
        rc, msg = _raw(y, u, table(ok), 3, 2, null_out=i)
        assert (rc == 0) if i == 5 else (rc != 0 and "null output" in msg), (i, msg)
    if torch.cuda.device_count() > 1:
        u_other = _capi.Engine(cached_plan("ufldv2", backbone="18")[0], 1, max_batch=MAX_BATCH)
        rc, msg = _raw(y, u_other, table(ok), 3, 2)
        assert rc != 0 and "device" in msg
        u_other.close()
    after = _capi.detect_pair_rig(y, u, cams, 0.4, NMS_IOU)
    for i in range(3 * 2):
        assert _frame(after, i) == _frame(before, i), i


def test_follow_up_calls_need_frames_of_one_size(pairs):
    y, u = pairs["v8_v2"]
    cams = _frames(RIG[:2], f=1, seed=400)
    M = np.eye(3)
    _capi.detect_pair_rig(y, u, cams, 0.4, NMS_IOU)
    for call in (lambda: y.warp_perspective(1, M, (64, 32)), lambda: u.warp_perspective(1, M, (64, 32)),
                 lambda: u.lane_geometry(1, (1280, 720))):
        with pytest.raises(Exception, match="camera rig"):
            call()
    _capi.detect_pair(y, u, cams[1], 0.4, NMS_IOU)
    assert y.warp_perspective(1, M, (64, 32)).shape == (1, 32, 64, 3)
    assert u.warp_perspective(1, M, (64, 32)).shape == (1, 32, 64, 3)
    u.lane_geometry(1, (1280, 720))


# ---- the pipeline ------------------------------------------------------------------------------------------------------------------
def test_pipeline_frame_sizes_equal_single_camera_pipelines():
    """AdasPipeline(cameras=3, frame_sizes=...) gives, per camera and frame, the detections, lane points / status and track records of
    three single-camera pipelines updated frame by frame in camera order -- through step and through step_pipelined + flush, on
    host and on device frames; a camera at another size than declared is refused"""
    from adas_b200.pipeline import AdasPipeline
    from test_gpu_multicam import _one_frame, _same_result
    ypath, _, _ = cached_plan("yolov8", scale="l")
    upath, _, _ = cached_plan("ufldv2", backbone="18")
    sizes = [(1080, 1920), (720, 1280), (800, 1280)]
    K, Fp, S = 3, 4, 3
    frames = [np.stack([np.roll(synth.frame(60 + 7 * c + f, h, w), 16 * c, axis=1) for f in range(S * Fp)]) for c, (h, w) in enumerate(sizes)]
    kw = dict(device=0, track_thresh=0.3)
    singles = [AdasPipeline(ypath, upath, batch=1, sets=1, **kw) for _ in range(K)]
    want = [[None] * (S * Fp) for _ in range(K)]
    for f in range(S * Fp):
        for c in range(K):
            want[c][f] = singles[c].step(frames[c][f:f + 1])
    for p in singles:
        p.close()
    assert sum(int(w.counts.sum()) for row in want for w in row) > 0
    assert sum(len(w.tracks[0]) for row in want for w in row) > 0

    multi = AdasPipeline(ypath, upath, batch=Fp, sets=2, depth=2, cameras=K, frame_sizes=sizes, **kw)
    dev = [torch.from_numpy(a).cuda() for a in frames]
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        multi.step([frames[0][:Fp], frames[1][:Fp], frames[2][:Fp, :720]])
    with pytest.raises(ValueError):
        multi.step([(dev[0].data_ptr(), (Fp, 1080, 1920)), (dev[1].data_ptr(), (Fp, 720, 1280)), (dev[2].data_ptr(), (Fp, 720, 1280))],
                   on_device=True)
    for pipelined in (False, True):
        for t in multi.trackers:
            t.reset()
        got, keep = [], []
        for s in range(S):
            on_dev = (s + pipelined) % 2 == 1
            if on_dev:
                xs = [d[s * Fp:(s + 1) * Fp].contiguous() for d in dev]
                args = ([(x.data_ptr(), tuple(x.shape[:3])) for x in xs], True)
            else:
                xs = [a[s * Fp:(s + 1) * Fp] for a in frames]
                args = (xs,)
            if pipelined:
                r = multi.step_pipelined(*args)
                if r is not None:
                    got.append(r)
                keep.append(xs)                                                # frames stay valid until their batch returns
            else:
                got.append(multi.step(*args))
        if pipelined:
            got += multi.flush()
        assert len(got) == S
        for s, rs in enumerate(got):
            assert len(rs) == K
            for c in range(K):
                assert len(rs[c].counts) == Fp
                for i in range(Fp):
                    _same_result(_one_frame(rs[c], i), want[c][s * Fp + i], (pipelined, s, c, i))
    multi.close()
