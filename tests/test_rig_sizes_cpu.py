"""CPU: AdasPipeline(frame_sizes=...) refuses malformed rigs before touching a device -- the per-step frame checks (on a stand-in object
with `cameras`, `batch` and `frame_sizes`) and the constructor's size checks -- and its letterbox arithmetic matches the oracle's."""
import types

import numpy as np
import pytest

import adas_b200  # noqa: F401
from adas_b200.pipeline import AdasPipeline, letterbox_hw
from oracle import post

SIZES = [(1080, 1920), (720, 1280), (800, 1280)]


def _stub(batch=4):
    return types.SimpleNamespace(cameras=len(SIZES), batch=batch, frame_sizes=list(SIZES))


def _host(F=2, sizes=SIZES):
    return [np.zeros((F, h, w, 3), np.uint8) for h, w in sizes]


def test_rig_frames_accept_matching_per_camera_lists():
    stub = _stub()
    cams = _host()
    out, on_dev, shape = AdasPipeline._rig_frames(stub, cams, False, None)
    assert not on_dev and shape is None and len(out) == 3 and all(a is b for a, b in zip(out, cams))
    dev = [(1000 + c, (4, h, w)) for c, (h, w) in enumerate(SIZES)]
    out, on_dev, _ = AdasPipeline._rig_frames(stub, dev, True, None)
    assert on_dev and out == dev
    out, _, _ = AdasPipeline._rig_frames(stub, tuple(_host(F=1)), False, None)      # any sequence of K arrays, F = 1
    assert [a.shape for a in out] == [(1, h, w, 3) for h, w in SIZES]
    out, on_dev, _ = AdasPipeline._frames(stub, cams, False, None)                  # _frames routes declared sizes to the rig check
    assert not on_dev and len(out) == 3 and all(a is b for a, b in zip(out, cams))


def test_rig_frames_refuse_what_does_not_match_the_declared_rig():
    stub = _stub(batch=4)
    cams = _host()
    bad_host = [
        cams[:2] + [np.zeros((2, 720, 1280, 3), np.uint8)],          # camera 2 at another size than declared
        [cams[0], cams[1][:, :, :640], cams[2]],                     # camera 1 narrower
        [cams[0], cams[1][:1], cams[2]],                             # camera 1 with fewer frames
        cams[:2],                                                    # K - 1 cameras
        cams + [cams[2]],                                            # K + 1 cameras
        _host(F=0),                                                  # F = 0
        _host(F=5),                                                  # F > batch
        [cams[0].astype(np.float32), cams[1], cams[2]],              # not uint8
        [cams[0][..., :1], cams[1], cams[2]],                        # one channel
        [cams[0][0], cams[1], cams[2]],                              # no frame dimension
        [list(cams[0]), cams[1], cams[2]],                           # not an array
        1234,
    ]
    for frames in bad_host:
        with pytest.raises(ValueError):
            AdasPipeline._rig_frames(stub, frames, False, None)
    dev = [(1000 + c, (2, h, w)) for c, (h, w) in enumerate(SIZES)]
    bad_dev = [
        dev[:2] + [(1002, (2, 720, 1280))],                          # wrong size
        [dev[0], (1001, (1, 720, 1280)), dev[2]],                    # fewer frames
        dev[:2],
        dev + [dev[0]],
        [(p, (0, h, w)) for p, (_, h, w) in dev],                    # F = 0
        [(p, (5, h, w)) for p, (_, h, w) in dev],                    # F > batch
        [dev[0], 1001, dev[2]],                                      # a device entry without its (F, H, W)
        [dev[0], (1001, (720, 1280)), dev[2]],
        [dev[0], (1001,), dev[2]],
    ]
    for frames in bad_dev:
        with pytest.raises(ValueError):
            AdasPipeline._rig_frames(stub, frames, True, None)


def test_frames_without_declared_sizes_is_unchanged():
    """a stand-in with only `cameras` and `batch` still takes the one-size path, which refuses mixed sizes"""
    stub = types.SimpleNamespace(cameras=2, batch=4)
    f = np.zeros((2, 3, 48, 64, 3), np.uint8)
    frames, _, _ = AdasPipeline._frames(stub, [f[0], f[1]], False, None)
    assert frames.shape == (6, 48, 64, 3)
    with pytest.raises(ValueError):
        AdasPipeline._frames(stub, [f[0], f[1, :, :32]], False, None)


def test_constructor_size_checks():
    assert AdasPipeline._check_frame_sizes(3, SIZES, (640, 640)) == SIZES
    assert AdasPipeline._check_frame_sizes(16, [(720, 1280)] * 16, (640, 640)) == [(720, 1280)] * 16
    bad = [
        (3, SIZES[:2], (640, 640)),                                  # K != len(frame_sizes)
        (2, SIZES, (640, 640)),
        (3, [(0, 1280)] + SIZES[1:], (640, 640)),                    # 0 x N
        (3, [(720, 0)] + SIZES[1:], (640, 640)),
        (17, [(720, 1280)] * 17, (640, 640)),                        # 17 cameras
        (3, SIZES[:2] + [(5000, 1)], (640, 640)),                    # 1 wide, 5000 tall: the letterbox has no columns
        (1, [(720,)], (640, 640)),
        (1, 7, (640, 640)),
    ]
    for k, sizes, in_hw in bad:
        with pytest.raises(ValueError):
            AdasPipeline._check_frame_sizes(k, sizes, in_hw)
    # without the network's input size only the count and the 1 x 1 minimum are checked (before any engine exists)
    assert AdasPipeline._check_frame_sizes(1, [(5000, 1)]) == [(5000, 1)]
    with pytest.raises(ValueError):
        AdasPipeline(__file__, __file__, cameras=3, frame_sizes=SIZES[:2])           # refused before a plan is read


@pytest.mark.parametrize("hw", [(1080, 1920), (720, 1280), (640, 640), (1280, 720), (500, 333), (2160, 3840), (1, 5000), (5000, 7), (639, 640)])
def test_letterbox_matches_the_oracle(hw):
    """the constructor's empty-letterbox check computes the letterbox as the oracle (and the device) do"""
    assert letterbox_hw(*hw, 640, 640) == tuple(post.letterbox_geom(*hw, 640, 640)["new"])
