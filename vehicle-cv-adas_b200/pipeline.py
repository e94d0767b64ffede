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
"""
from __future__ import annotations

import sys
import threading
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from typing import List, Optional

import numpy as np

from . import _capi
from .ObjectTracker import BYTETracker


class StepResult:
    __slots__ = ("boxes", "scores", "class_ids", "cand_index", "counts", "n_candidates", "lane_pts", "lane_npts", "lane_status", "tracks")

    def __init__(self, y, u):
        self.boxes, self.scores, self.class_ids, self.cand_index, self.counts, self.n_candidates = y
        self.lane_pts, self.lane_npts, self.lane_status, _ = u
        self.tracks: Optional[List[list]] = None


class AdasPipeline:
    def __init__(self, yolo_plan: str, ufld_plan: str, device: int = 0, batch: int = 8, box_score: float = 0.4, box_nms_iou: float = 0.45,
                 max_det: int = 1024, class_names: Optional[List[str]] = None, depth: int = 3, sets: int = 2, track_thresh: float = 0.5):
        self.batch, self.box_score, self.box_nms_iou, self.max_det = batch, box_score, box_nms_iou, max_det
        # `sets` independent (object engine, lane engine) pairs: consecutive batches alternate between them so the next batch's
        # kernels are already queued on the device (own streams, own activation buffers) while the previous batch drains --
        # no idle gap between library calls, and four streams' worth of kernels to back-fill partial waves.
        self.sets = []
        for _ in range(max(1, sets)):
            self.sets.append((_capi.Engine(yolo_plan, device, max_batch=batch), _capi.Engine(ufld_plan, device, max_batch=batch), threading.Lock()))
        self.yolo, self.ufld = self.sets[0][0], self.sets[0][1]
        # build every launch program here, one engine at a time: the per-layer tile autotune times candidates on the device and
        # must not run while another engine is busy (with two pairs the first two batches would otherwise tune concurrently);
        # the second pass captures the CUDA graphs.
        for y, u, _ in self.sets:
            for e in (y, u):
                e.run(batch)
                e.run(batch)
        self._next_set = 0
        self.tracker = BYTETracker(track_thresh=track_thresh, names=class_names or [], device=device)
        self.tracker.reset()
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

    # -- public ---------------------------------------------------------------------------------------------
    def step(self, frames, on_device: bool = False, shape=None) -> StepResult:
        """Synchronous: detectors (concurrently), then the tracker for this batch."""
        r = StepResult(*self._detect_both(frames, on_device, shape))
        self._track(r)
        return r

    def step_pipelined(self, frames, on_device: bool = False, shape=None) -> Optional[StepResult]:
        """Queue this batch for the detector thread (up to `depth` batches in flight, so the GPU never waits for Python) and
        return the oldest finished batch with its tracks (None while the pipeline fills); call flush() at the end.
        Frame buffers must stay valid until their batch has been returned."""
        self._queue.append(self._detect(frames, on_device, shape))
        if len(self._queue) <= self.depth:
            return None
        r = StepResult(*self._queue.popleft().result())
        self._track(r)
        return r

    def flush(self) -> List[StepResult]:
        out = []
        while self._queue:
            r = StepResult(*self._queue.popleft().result())
            self._track(r)
            out.append(r)
        return out
