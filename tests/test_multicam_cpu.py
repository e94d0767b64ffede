"""CPU: the multi-camera entry points refuse malformed input before touching a device -- adas_tracker_update_multi's argument checks
on fresh trackers, and AdasPipeline(cameras=K)'s frame checks (the pipeline stage alone, on a stand-in object)."""
import ctypes as C
import types

import numpy as np
import pytest

import adas_b200  # noqa: F401
from adas_b200 import _capi
from adas_b200.pipeline import AdasPipeline


def _update_multi(handles, k, counts):
    lib = _capi.lib()
    hs = (C.c_void_p * max(1, len(handles)))(*handles)
    cnt = np.ascontiguousarray(counts, np.int32)
    n = max(1, int(np.clip(cnt, 0, None).sum()))
    b, s, c = np.zeros((n, 4)), np.full(n, 0.9), np.zeros(n, np.int32)
    out, n_out = np.zeros(64, _capi.TRACK_DTYPE), np.zeros(8, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.adas_tracker_update_multi(hs, k, 1, p(cnt), p(b), p(s), p(c), 8, p(out), p(n_out))
    return rc, lib.adas_last_error().decode()


def test_update_multi_refuses_bad_arguments_before_any_device_work():
    a, b = _capi.NativeTracker(0), _capi.NativeTracker(0)
    other = _capi.NativeTracker(1)
    ha, hb = a._h.value, b._h.value
    cases = {
        "bad arguments": [([ha, hb], 0, [1, 1]), ([ha, hb], -3, [1, 1])],
        "is null": [([ha, None], 2, [1, 1]), ([None], 1, [1])],
        "is also tracker": [([ha, hb, ha], 3, [1, 1, 1]), ([hb, hb], 2, [0, 0])],
        "on device 1": [([ha, other._h.value], 2, [1, 1])],
        "negative detection count": [([ha, hb], 2, [3, -1]), ([ha], 1, [-2])],
    }
    for what, calls in cases.items():
        for args in calls:
            rc, msg = _update_multi(*args)
            assert rc != 0 and what in msg, (args, msg)
    for t in (a, b, other):
        assert t.get(0).size == 0 and t.get(1).size == 0 and t.stats() == {"frames": 0, "total_ms": 0.0, "wait_ms": 0.0, "launches": 0}
        t.close()


def test_pipeline_refuses_frames_it_cannot_batch_across_cameras():
    stub = types.SimpleNamespace(cameras=3, batch=4)
    f = np.zeros((3, 4, 48, 64, 3), np.uint8)
    frames, on_dev, shape = AdasPipeline._frames(stub, f, False, None)
    assert frames.shape == (12, 48, 64, 3) and not on_dev and shape is None
    frames, _, _ = AdasPipeline._frames(stub, [f[0], f[1], f[2]], False, None)
    assert np.array_equal(frames, f.reshape(12, 48, 64, 3))
    assert AdasPipeline._frames(stub, 1234, True, (3, 2, 720, 1280)) == (1234, True, (6, 720, 1280))
    bad = [
        ([f[0], f[1], f[2, :, :32]], False, None),                  # one camera of another frame size
        ([f[0], f[1], f[2, :3]], False, None),                      # one camera with fewer frames
        ([f[0], f[1]], False, None),                                # two cameras for three
        (f[:2], False, None),
        (np.zeros((3, 5, 48, 64, 3), np.uint8), False, None),       # more frames than the batch
        (f[..., :1], False, None),
        (1234, True, (3, 720, 1280)),                               # device frames without the camera dimension
        (1234, True, (2, 4, 720, 1280)),
        (1234, True, (3, 0, 720, 1280)),
    ]
    for frames, on_dev, shape in bad:
        with pytest.raises(ValueError):
            AdasPipeline._frames(stub, frames, on_dev, shape)
    one = types.SimpleNamespace(cameras=1, batch=4)                  # one camera: frames pass through unchanged
    x = f[0]
    assert AdasPipeline._frames(one, x, False, None) == (x, False, None)
