"""pipeline.py -- the per-frame loop of the reference's demo.py (261-316) as a batched, overlapped stream runner.

demo.py does, per frame and strictly in sequence: `objectDetector.DetectFrame` (269) -> `objectTracker.update` (272-277)
-> `laneDetector.DetectFrame` (280) -> analytics/drawing.  Here one step takes a batch of consecutive frames of one
stream:  a worker thread makes ONE library call (`adas_detect_pair`) that enqueues the object network and the lane network
on their own CUDA streams before waiting for either -- the tail waves of one network's persistent conv kernels are
back-filled by the other's (driving the two streams from two Python threads
instead was slower, the interpreter lock serialises the launches) -- while the host thread runs the ByteTrack updates of
the PREVIOUS batch; consecutive batches alternate between two engine pairs so the device never waits for the host:
the tracker is sequential in time per stream (SURVEY 8e), so it pipelines one batch behind the detectors.  Per-frame
results are identical to calling the three detectors frame by frame.

A rig of several cameras runs through ONE pipeline (`cameras=K`): the engines hold K * batch frames, each step makes one
`adas_detect_pair` call for the frames of all cameras, and the K trackers (one per camera) advance in one library call with one
association launch per frame for all of them (`adas_tracker_update_multi`).  Results equal K single-camera pipelines whose
trackers are updated frame by frame in camera order.

Cameras of different frame sizes (`frame_sizes=[(H, W), ...]`, one per camera) run through the same single call
(`adas_detect_pair_rig`): every frame is letterboxed / resized from its own camera's size into the one network batch, and each
camera's boxes and lane points come back in that camera's pixels.
"""
from __future__ import annotations

import sys
import threading
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from typing import List, Optional

import numpy as np

from . import _capi
from .ObjectTracker import BYTETracker, update_trackers


class StepResult:
    __slots__ = ("boxes", "scores", "class_ids", "cand_index", "counts", "n_candidates", "lane_pts", "lane_npts", "lane_status", "tracks")

    def __init__(self, y, u):
        self.boxes, self.scores, self.class_ids, self.cand_index, self.counts, self.n_candidates = y
        self.lane_pts, self.lane_npts, self.lane_status, _ = u
        self.tracks: Optional[List[list]] = None


def letterbox_hw(src_h: int, src_w: int, in_h: int, in_w: int):
    """(rows, columns) an src_h x src_w frame is resized to inside an in_h x in_w network input (Scaler.process_image's letterbox,
    the arithmetic of the device's letterbox_geom)"""
    if src_h == src_w:
        return in_h, in_w
    hw_scale = src_h / src_w
    if hw_scale > 1.0:
        return in_h, int(in_w / hw_scale)
    return int(in_h * hw_scale) + 1, in_w


MAX_RIG_CAMERAS = 16          # ADAS_MAX_RIG_CAMERAS


class AdasPipeline:
    def __init__(self, yolo_plan: str, ufld_plan: str, device: int = 0, batch: int = 8, box_score: float = 0.4, box_nms_iou: float = 0.45,
                 max_det: int = 1024, class_names: Optional[List[str]] = None, depth: int = 3, sets: int = 2, track_thresh: float = 0.5,
                 cameras: int = 1, frame_sizes=None):
        """`cameras` = K streams of one frame size through one pipeline: with K > 1, step / step_pipelined take [K, F, H, W, 3] frames
        (F <= batch; a host array, a sequence of K [F, H, W, 3] host arrays, or a device pointer with shape (K, F, H, W)) and
        return one StepResult per camera.

        `frame_sizes` = K (H, W) pairs: the cameras may differ in frame size.  step / step_pipelined then take a list of K host arrays
        [F, H_c, W_c, 3] uint8 (on_device=False) or of K (device pointer, (F, H_c, W_c)) pairs (on_device=True), each camera at its
        declared size and all with the same F <= batch, and return one StepResult per camera in that camera's pixels."""
        if cameras < 1:
            raise ValueError(f"cameras must be at least 1, got {cameras}")
        if frame_sizes is not None:
            frame_sizes = AdasPipeline._check_frame_sizes(cameras, frame_sizes)
        self.batch, self.box_score, self.box_nms_iou, self.max_det = batch, box_score, box_nms_iou, max_det
        self.cameras = cameras
        self.frame_sizes = frame_sizes
        nb = cameras * batch
        # `sets` independent (object engine, lane engine) pairs: consecutive batches alternate between them so the next batch's
        # kernels are already queued on the device (own streams, own activation buffers) while the previous batch drains --
        # no idle gap between library calls, and four streams' worth of kernels to back-fill partial waves.
        self.sets = []
        for _ in range(max(1, sets)):
            self.sets.append((_capi.Engine(yolo_plan, device, max_batch=nb), _capi.Engine(ufld_plan, device, max_batch=nb), threading.Lock()))
        self.yolo, self.ufld = self.sets[0][0], self.sets[0][1]
        # build every launch program here, one engine at a time: the per-layer tile autotune times candidates on the device and
        # must not run while another engine is busy (with two pairs the first two batches would otherwise tune concurrently);
        # the second pass captures the CUDA graphs.
        for y, u, _ in self.sets:
            for e in (y, u):
                e.run(nb)
                e.run(nb)
        if frame_sizes is not None:
            try:
                AdasPipeline._check_frame_sizes(cameras, frame_sizes, tuple(self.yolo.input_shape[2:4]))
                # one rig call per engine pair: the resize tables of every camera and the staging arena exist before the first step
                zeros = [np.zeros((batch, h, w, 3), np.uint8) for h, w in frame_sizes]
                for y, u, _ in self.sets:
                    _capi.detect_pair_rig(y, u, zeros, box_score, box_nms_iou, max_det)
            except Exception:
                for y, u, _ in self.sets:
                    y.close()
                    u.close()
                raise
        self._next_set = 0
        self.trackers = [BYTETracker(track_thresh=track_thresh, names=class_names or [], device=device) for _ in range(cameras)]
        for t in self.trackers:
            t.reset()
        self.tracker = self.trackers[0]
        self.class_names = class_names
        self._pool = ThreadPoolExecutor(max_workers=len(self.sets))
        sys.setswitchinterval(2e-4)       # the detector thread only needs the interpreter between two library calls
        self.depth = max(1, depth)                     # batches in flight in the detector thread
        self._queue = deque()

    def close(self):
        self._pool.shutdown(wait=True)
        for y, u, _ in self.sets:
            y.close()
            u.close()

    # -- stages -------------------------------------------------------------------------------------------
    def _detect_both(self, frames, on_device: bool, shape, k: int = 0):
        y, u, lock = self.sets[k]
        with lock:                        # one batch at a time per engine pair
            if self.frame_sizes is not None:
                return _capi.detect_pair_rig(y, u, frames, self.box_score, self.box_nms_iou, self.max_det, on_device)
            return _capi.detect_pair(y, u, frames, self.box_score, self.box_nms_iou, self.max_det, on_device, shape)

    def _detect(self, frames, on_device: bool, shape):
        k = self._next_set
        self._next_set = (k + 1) % len(self.sets)
        return self._pool.submit(self._detect_both, frames, on_device, shape, k)

    def _track(self, r: StepResult) -> None:
        """ByteTrack for the frames of one batch, in time order, in ONE library call (adas_tracker_update_batch): r.tracks[i] is the
        TRACK_DTYPE record array of frame i (`self.tracker.messages(r.tracks[i])` gives the reference's track messages)."""
        import time
        t0 = time.perf_counter()
        counts = np.asarray(r.counts, np.int32)
        keep = np.arange(r.boxes.shape[1])[None, :] < counts[:, None]            # [B, max_det] valid detections, frame-major
        bx = r.boxes[keep]
        # demo.py:272-275 feeds RectInfo.tolist("xyxy") -> ints (truncation), and the label as class id
        xyxy = np.stack([bx[:, 0], bx[:, 1], bx[:, 0] + bx[:, 2], bx[:, 1] + bx[:, 3]], 1).astype(np.int64).astype(np.float64)
        if self.class_names is None:
            r.tracks = self.tracker.update_batch_arrays(counts, xyxy, r.scores[keep].astype(np.float64), r.class_ids[keep])
        else:
            cls, o, dets = r.class_ids[keep], 0, []
            for n in counts.tolist():
                dets.append((xyxy[o:o + n], r.scores[keep][o:o + n], [self.class_names[c] for c in cls[o:o + n]]))
                o += n
            r.tracks = self.tracker.update_batch(dets)
        self.track_seconds = getattr(self, "track_seconds", 0.0) + (time.perf_counter() - t0)
        self.track_batches = getattr(self, "track_batches", 0) + 1

    @staticmethod
    def _check_frame_sizes(cameras: int, frame_sizes, in_hw=None):
        """the declared (H, W) of every camera as a list of int pairs; refuses (ValueError) a count other than `cameras`, more than
        MAX_RIG_CAMERAS cameras, a size below 1 x 1, and -- given the YOLO input size in_hw -- a size whose letterbox is empty"""
        try:
            sizes = [(int(h), int(w)) for h, w in frame_sizes]
        except (TypeError, ValueError):
            raise ValueError(f"frame_sizes must be {cameras} (H, W) pairs, got {frame_sizes!r}") from None
        if len(sizes) != cameras:
            raise ValueError(f"{len(sizes)} frame sizes for {cameras} cameras")
        if cameras > MAX_RIG_CAMERAS:
            raise ValueError(f"{cameras} cameras of declared sizes; a rig has at most {MAX_RIG_CAMERAS}")
        for c, (h, w) in enumerate(sizes):
            if h < 1 or w < 1:
                raise ValueError(f"camera {c}: frame size {h} x {w}")
            if in_hw is not None and min(letterbox_hw(h, w, *in_hw)) < 1:
                raise ValueError(f"camera {c}: a {h} x {w} frame letterboxes to {letterbox_hw(h, w, *in_hw)} inside {tuple(in_hw)}: nothing to detect in")
        return sizes

    def _rig_frames(self, frames, on_device: bool, shape):
        """the frames of one step of a pipeline with declared frame sizes, as adas_detect_pair_rig takes them: K host arrays
        [F, H_c, W_c, 3] uint8 or K (device pointer, (F, H_c, W_c)) pairs, each camera at its declared size, one F in 1..batch"""
        K = self.cameras
        try:
            cams = list(frames)
        except TypeError:
            raise ValueError(f"frames of {K} cameras of declared sizes must be a list of {K} entries, got {type(frames).__name__}") from None
        if len(cams) != K:
            raise ValueError(f"frames of {len(cams)} cameras for a pipeline of {K}")
        out, F = [], None
        for c, (a, (h, w)) in enumerate(zip(cams, self.frame_sizes)):
            if on_device:
                if not (isinstance(a, (tuple, list)) and len(a) == 2 and isinstance(a[1], (tuple, list)) and len(a[1]) == 3):
                    raise ValueError(f"camera {c}: device frames are (pointer, (frames, H, W)), got {a!r}")
                f, fh, fw = (int(v) for v in a[1])
                out.append((int(a[0]), (f, fh, fw)))
            else:
                if not (isinstance(a, np.ndarray) and a.dtype == np.uint8 and a.ndim == 4 and a.shape[3] == 3):
                    what = f"{a.dtype} {a.shape}" if isinstance(a, np.ndarray) else type(a).__name__
                    raise ValueError(f"camera {c}: frames must be a uint8 [frames, H, W, 3] array, got {what}")
                f, fh, fw = a.shape[:3]
                out.append(a)
            if (fh, fw) != (h, w):
                raise ValueError(f"camera {c} sends {fh} x {fw} frames; its declared size is {h} x {w}")
            if F is None:
                F = f
            elif f != F:
                raise ValueError(f"every camera must send the same number of frames: camera {c} sends {f}, camera 0 {F}")
        if not 1 <= F <= self.batch:
            raise ValueError(f"{F} frames per camera; this pipeline takes 1 to {self.batch}")
        return out, on_device, None

    def _frames(self, frames, on_device: bool, shape):
        """the frames of one step as adas_detect_pair takes them: with K > 1 cameras, camera-major [K * F, H, W, 3]"""
        if getattr(self, "frame_sizes", None) is not None:
            return AdasPipeline._rig_frames(self, frames, on_device, shape)
        K = self.cameras
        if K == 1:
            return frames, on_device, shape
        if on_device:
            if shape is None or len(shape) != 4 or int(shape[0]) != K:
                raise ValueError(f"device frames of {K} cameras need shape (cameras={K}, frames, H, W), got {shape}")
            F, H, W = (int(v) for v in shape[1:])
            if not 1 <= F <= self.batch:
                raise ValueError(f"{F} frames per camera; this pipeline takes 1 to {self.batch}")
            return frames, True, (K * F, H, W)
        if not (isinstance(frames, np.ndarray) and frames.ndim == 5):
            cams = [np.asarray(f) for f in frames]
            if len(cams) != K:
                raise ValueError(f"frames of {len(cams)} cameras for a pipeline of {K}")
            for c, a in enumerate(cams):
                if a.shape != cams[0].shape:
                    raise ValueError(f"all cameras must send the same number of frames of one size: camera {c} sends {a.shape}, "
                                     f"camera 0 {cams[0].shape}")
            frames = np.stack(cams)
        if frames.ndim != 5 or frames.shape[0] != K or frames.shape[4] != 3:
            raise ValueError(f"frames of {K} cameras must be [cameras={K}, frames, H, W, 3], got {frames.shape}")
        if not 1 <= frames.shape[1] <= self.batch:
            raise ValueError(f"{frames.shape[1]} frames per camera; this pipeline takes 1 to {self.batch}")
        return frames.reshape((-1,) + frames.shape[2:]), False, None

    def _track_cameras(self, y, rs: List[StepResult]) -> None:
        """ByteTrack for the frames of one batch of every camera in ONE library call (adas_tracker_update_multi): rs[c].tracks[i] is
        the TRACK_DTYPE record array of camera c's frame i, as _track gives it for one camera."""
        import time
        t0 = time.perf_counter()
        boxes, scores, cls, _, counts, _ = y                                     # [K * F, ...], camera-major
        K = self.cameras
        F = len(counts) // K
        cnt = np.asarray(counts, np.int32).reshape(K, F).T                       # [F, K]
        order = lambda a: a.reshape((K, F) + a.shape[1:]).swapaxes(0, 1)         # frame-major, then camera
        keep = np.arange(boxes.shape[1])[None, None, :] < cnt[:, :, None]
        bx = order(boxes)[keep]
        xyxy = np.stack([bx[:, 0], bx[:, 1], bx[:, 0] + bx[:, 2], bx[:, 1] + bx[:, 3]], 1).astype(np.int64).astype(np.float64)
        labels = order(cls)[keep]
        if self.class_names is not None:
            labels = np.asarray(self.class_names, dtype=object)[labels]
        recs = update_trackers(self.trackers, cnt, xyxy, order(scores)[keep].astype(np.float64), labels)
        for r, tr in zip(rs, recs):
            r.tracks = tr
        self.track_seconds = getattr(self, "track_seconds", 0.0) + (time.perf_counter() - t0)
        self.track_batches = getattr(self, "track_batches", 0) + 1

    def _result(self, yu):
        y, u = yu
        if self.cameras == 1 and self.frame_sizes is None:
            r = StepResult(y, u)
            self._track(r)
            return r
        F = len(y[4]) // self.cameras
        cam = lambda t, c: tuple(None if a is None else a[c * F:(c + 1) * F] for a in t)
        rs = [StepResult(cam(y, c), cam(u, c)) for c in range(self.cameras)]
        self._track_cameras(y, rs)
        return rs

    # -- public ---------------------------------------------------------------------------------------------
    def step(self, frames, on_device: bool = False, shape=None):
        """Synchronous: detectors (concurrently), then the tracker for this batch.  One StepResult, or with K > 1 cameras a list of
        K (one per camera)."""
        return self._result(self._detect_both(*self._frames(frames, on_device, shape)))

    def step_pipelined(self, frames, on_device: bool = False, shape=None):
        """Queue this batch for the detector thread (up to `depth` batches in flight, so the GPU never waits for Python) and
        return the oldest finished batch with its tracks (None while the pipeline fills); call flush() at the end.
        Frame buffers must stay valid until their batch has been returned."""
        self._queue.append(self._detect(*self._frames(frames, on_device, shape)))
        if len(self._queue) <= self.depth:
            return None
        return self._result(self._queue.popleft().result())

    def flush(self) -> list:
        out = []
        while self._queue:
            out.append(self._result(self._queue.popleft().result()))
        return out
