"""Helpers of the rig-size tests (test_rig_scale_cpu.py, test_gpu_rig_scale.py).

A multi-camera rig of 8 cameras x 8 frames runs its networks at batch 64.  Every buffer of YOLOv8l at batch 64 together is on the
order of 10 GB, so the checks never hold a whole run on the host:
- `stream_read` reads one buffer at a time and keeps a sha256 digest of every image's rows of it, the rows of a few sampled images,
  and whether its halo is zero;
- `subset` keeps the listed images of every buffer, so `plan_interp.op_ref(pb, i, sub, len(images))` checks images 61-63 of a
  batch-64 run for the cost of a batch-3 check, and `check_images` names the op and the image of every element out of its bound.

`SCHEDULE` is a list of multi-tracker calls over eight trackers whose groups change from call to call: the first tracker of an
`adas_tracker_update_multi` call (its lead) owns the call's staging, stream and completion word, so the schedule makes fresh leads,
leads whose staging must grow, reversed groups and single-tracker calls on trackers other groups lead."""
import hashlib
from typing import Dict, List, NamedTuple, Sequence, Tuple

import numpy as np

import plan_interp as pi
from adas_b200 import plan


def subset(pb, bufs: Dict[int, np.ndarray], images: Sequence[int]) -> Dict[int, np.ndarray]:
    """The listed images of every buffer (pb.buffers[i][0] rows per image, dense buffers included), in the listed order."""
    out = {}
    for i, a in bufs.items():
        rows = pb.buffers[i][0]
        out[i] = np.concatenate([a[b * rows:(b + 1) * rows] for b in images])
    return out


def halo_is_zero(pb, i: int, a: np.ndarray, B: int) -> bool:
    """The zero border of padded buffer i over B images (the stem re-layout's output owns its top halo row); dense buffers have none."""
    _, C, _, H, W, _ = pb.buffers[i]
    if H == 0:
        return True
    v = a[:B * (H + 2) * (W + 2)].reshape(B, H + 2, W + 2, C)
    stem = any(t == plan.OP_STEMPACK and p[1] == i for t, p, _ in pb.ops)
    edges = [v[:, -1], v[:, :, 0], v[:, :, -1]] + ([] if stem else [v[:, 0]])
    return not any(np.any(e != 0) for e in edges)


class Readback(NamedTuple):
    digests: Dict[int, List[str]]       # buffer -> sha256 of each image's rows
    sampled: Dict[int, np.ndarray]      # subset(pb, buffers, images)
    halo: List[int]                     # buffers with a nonzero halo


def stream_read(pb, read, B: int, images: Sequence[int]) -> Readback:
    """Every buffer of a B-image run through `read(i)` (an array of at least B images' rows), one buffer at a time."""
    digests, sampled, halo = {}, {}, []
    for i in range(len(pb.buffers)):
        rows = pb.buffers[i][0]
        a = read(i)
        digests[i] = [hashlib.sha256(np.ascontiguousarray(a[b * rows:(b + 1) * rows])).hexdigest() for b in range(B)]
        sampled[i] = np.concatenate([a[b * rows:(b + 1) * rows] for b in images] or [a[:0]])
        if not halo_is_zero(pb, i, a, B):
            halo.append(i)
        del a
    return Readback(digests, sampled, halo)


def digest_diff(a: Dict[int, List[str]], b: Dict[int, List[str]], images_a=None, images_b=None) -> List[Tuple[int, int]]:
    """(buffer, image of a) whose rows differ between two readbacks; images_a[k] of a is compared with images_b[k] of b (default:
    every image of a with the same image of b)."""
    out = []
    for i in sorted(a):
        ia = range(len(a[i])) if images_a is None else images_a
        ib = ia if images_b is None else images_b
        out += [(i, x) for x, y in zip(ia, ib) if a[i][x] != b[i][y]]
    return out


def check_images(pb, sub: Dict[int, np.ndarray], images: Sequence[int], skip, worst: Dict[str, float], device: str = "cpu"):
    """Every op of the images of `sub` (subset(pb, buffers, images)) against plan_interp.op_ref, as test_gpu_plan_conformance.check_ops
    does it (ops in `skip` are not checked; of an output a later op overwrites in part, the rest is checked).  Returns (op, kind,
    image, elements out of bound, max error / bound) of every op and image with an element out of its bound; worst[kind] is the
    largest error / bound seen."""
    fails = []
    clobbered = pi.overwritten(pb)
    n = len(images)
    for i in range(len(pb.ops)):
        if i in skip:
            continue
        ref, bnd = pi.op_ref(pb, i, sub, n, device=device)
        got = pi.read_out(pb, i, sub, n)
        if i in clobbered:
            keep = ~clobbered[i]
            ref, got = ref[:, keep], got[:, keep]
            bnd = None if bnd is None else bnd[:, keep]
        kind = pi.op_kind(pb, i)
        for k, b in enumerate(images):
            ratio, nbad = pi.excess(got[k:k + 1], ref[k:k + 1], None if bnd is None else bnd[k:k + 1])
            worst[kind] = max(worst.get(kind, 0.0), ratio)
            if nbad:
                fails.append((i, kind, b, nbad, ratio))
    return fails


# ---- regrouped multi-tracker calls --------------------------------------------------------------------------------------------------
ALL = tuple(range(8))
REV = tuple(reversed(ALL))
# (call, trackers, frames): "multi" = NativeTracker.update_multi over the trackers (the first leads), "update" = one plain update,
# "batch" = update_batch.  Trackers are the cameras of rig_cameras(): 2 and 6 are crowds of 150 and 400 objects, 3 never sees a
# detection, so on its own it never touches the device.
SCHEDULE = [
    ("multi", (1,), 3),            # K = 1, and tracker 1's first call: a few objects, so its staging starts at the minimum size
    ("multi", (3, 2), 3),          # a fresh lead without staging in front of the crowd of 150 (past the 120 shared-memory rows)
    ("multi", ALL, 4),             # all eight, led by tracker 0 on its first call
    ("update", (1,), 1),           # plain update on a tracker that leads other groups
    ("multi", (1, 6, 2), 3),       # lead 1 again, now with both crowds: its staging grows
    ("multi", REV, 3),             # the same trackers in reversed order
    ("batch", (7,), 3),            # update_batch on the lead of the reversed group
    ("update", (0,), 1),
    ("multi", (5, 0), 2),
    ("batch", (3,), 2),
    ("multi", (2,), 2),            # K = 1 on the crowd
    ("update", (7,), 1),
    ("multi", ALL, 6),
    ("batch", (1,), 4),
    ("multi", REV, 4),
    ("multi", (6, 4, 2, 0), 5),
    ("multi", ALL, 8),
]


def windows(schedule) -> List[Dict[int, range]]:
    """For each call, the frames of each of its trackers' streams it consumes (every tracker walks its own stream in order)."""
    pos: Dict[int, int] = {}
    out = []
    for _, group, n in schedule:
        w = {}
        for c in group:
            w[c] = range(pos.get(c, 0), pos.get(c, 0) + n)
            pos[c] = w[c].stop
        out.append(w)
    return out


def frames_used(schedule) -> int:
    return max(w.stop for ws in windows(schedule) for w in ws.values())


def rig_cameras():
    """(tracker settings, per-frame detections) of eight cameras: test_gpu_multicam._cameras(), with camera 6 a crowd of 400 objects
    (more rows than the association's minimum staging and scratch hold)."""
    import test_gpu_multicam as mc
    cams = mc._cameras()
    cams[6] = (dict(), mc._crowded_stream(400, seed=9))
    return cams


def stream_frame(cams, c: int, f: int):
    seq = cams[c][1]
    return seq[f] if f < len(seq) else (np.zeros((0, 4), np.float64), np.zeros(0, np.float64), np.zeros(0, np.int32))


def high_dets(cams, c: int, f: int) -> int:
    """detections of camera c's frame f above its track threshold (the rows of the association's stage 1)"""
    return int((np.asarray(stream_frame(cams, c, f)[1]) > cams[c][0].get("track_thresh", 0.5)).sum())
