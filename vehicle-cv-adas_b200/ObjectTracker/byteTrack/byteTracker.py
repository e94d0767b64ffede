"""BYTETracker with the reference's API (ObjectTracker/byteTrack/byteTracker.py:12-215).

`update(bboxes_xyxy, scores, class_ids, frame)` follows the reference's three association stages (62-185):
thresholds 0.5 / 0.1 / det 0.6 (48,73-75), match 0.8 (fused) / 0.5 (plain IoU) / 0.7 (fused) (108,130,152),
30-frame lost buffer (49), duplicate removal at IoU-distance < 0.15 (utils.py:54-69).  The whole update runs in the
native tracker (csrc/tracker.cu: Kalman and list bookkeeping in host C++ because they are sequential per stream, the
three association stages of a frame as ONE device launch); this module is the API-compatible view of it.
"""
import numpy as np

from ..core import ObjectTrackBase
from .strack import BaseTrack, LimitedList, TrackState, tlwh_to_xyah


class TrackView:
    """Read-only view of one native track with the attribute surface of the reference's STrack (strack.py:33-215)."""
    __slots__ = ("track_id", "is_activated", "state", "score", "class_id", "start_frame", "frame_id", "tracklet_len", "mean", "_tlwh",
                 "trajectories", "crops", "time_since_update", "location")

    def __init__(self):
        self.trajectories = LimitedList(30)
        self.crops = []
        self.time_since_update = 0
        self.location = (np.inf, np.inf)

    @property
    def tlwh(self):
        return self._tlwh.copy()

    @property
    def tlbr(self):
        r = self._tlwh.copy()
        r[2:] += r[:2]
        return r

    @property
    def xyah(self):
        return tlwh_to_xyah(self._tlwh)

    @property
    def end_frame(self):
        return self.frame_id

    def filter_trajectories(self, frame, pad=(0, 0)):
        ph, pw = pad
        return [b for b in list(self.trajectories)
                if b[0] >= pw and b[1] >= ph and b[2] <= frame.shape[1] - pw and b[3] <= frame.shape[0] - ph]

    def get_track_message(self, count):
        return {"track_id": self.track_id, "count": count, "is_activated": self.is_activated, "state": self.state, "score": self.score,
                "start_frame_number": self.start_frame, "curr_frame_number": self.frame_id, "time_since_update": self.time_since_update,
                "location": str(self.location), "crops": self.crops, "class_id": self.class_id}

    def __repr__(self):
        return f"OT_{self.track_id}_({self.start_frame}-{self.end_frame})"


class BYTETracker(ObjectTrackBase):
    """The reference's BYTETracker API (byteTracker.py:12-215) over the native tracker (csrc/tracker.cu): `update` is one
    library call per frame -- Kalman + bookkeeping in host C++, the three association stages on the device."""

    def __init__(self, track_thresh=0.5, track_buffer=30, match_thresh=0.8, frame_rate=30, min_box_area=10, device=0, **kwargs):
        super().__init__(**kwargs)
        from ... import _capi
        self._capi = _capi
        self._nt = _capi.NativeTracker(device, track_thresh, track_buffer, match_thresh, frame_rate)
        self.track_thresh, self.match_thresh, self.min_box_area = track_thresh, match_thresh, min_box_area
        self.det_thresh = track_thresh + 0.1
        self.buffer_size = int(frame_rate / 30.0 * track_buffer)
        self.max_time_lost = self.buffer_size
        self.frame_id = 0
        self._labels, self._label_list = {}, []
        self._views = {}
        self.tracked_stracks = []
        self.removed_stracks = []

    def _cid(self, label):
        k = label.item() if hasattr(label, "item") else label
        i = self._labels.get(k)
        if i is None:
            i = self._labels[k] = len(self._label_list)
            self._label_list.append(k)
        return i

    def _view(self, rec, frame=None):
        tid = int(rec["track_id"])
        v = self._views.get(tid)
        if v is None:
            v = self._views[tid] = TrackView()
            if frame is not None:                      # STrack.update_crops at birth (strack.py:131-143, byteTracker.py:167)
                tx1, ty1, tw, th = rec["tlwh"].astype(int)
                x1, y1 = max(0, tx1), max(0, ty1)
                x2, y2 = min(frame.shape[1], tx1 + tw), min(frame.shape[0], ty1 + th)
                v.crops.append(frame[y1:y2, x1:x2, :].copy())
        v.track_id, v.is_activated, v.state = tid, bool(rec["is_activated"]), int(rec["state"])
        v.score, v.class_id = float(rec["score"]), self._label_list[int(rec["class_id"])]
        v.start_frame, v.frame_id, v.tracklet_len = int(rec["start_frame"]), int(rec["frame_id"]), int(rec["tracklet_len"])
        v.mean, v._tlwh = rec["mean"].copy(), rec["tlwh"].copy()
        if int(rec["traj_frame"]) == self.frame_id:
            v.trajectories.append(rec["det_tlbr"].copy())
        return v

    def update(self, bboxes, scores, class_ids, frame=None):
        self.frame_id += 1
        ids = np.fromiter((self._cid(c) for c in class_ids), dtype=np.int32, count=len(class_ids)) if len(class_ids) else np.zeros(0, np.int32)
        recs = self._nt.update(np.asarray(bboxes, dtype=np.float64).reshape(-1, 4), np.asarray(scores, dtype=np.float64), ids)
        self.tracked_stracks = [self._view(r, frame) for r in recs]
        if len(self._views) > 4 * max(64, len(recs)):                 # forget views of long-gone tracks
            alive = {int(r["track_id"]) for r in recs} | {int(r["track_id"]) for r in self._nt.get(1)}
            self._views = {k: v for k, v in self._views.items() if k in alive}
        cnt = self._capi.NativeTracker.count()
        return [t.get_track_message(cnt) for t in self.tracked_stracks]

    def update_batch(self, frames_dets):
        """All frames of a pipeline step in ONE library call (no interpreter work between frames).
        frames_dets: sequence of (bboxes xyxy [n,4], scores [n], class_ids [n]) per frame, in time order.
        Returns one TRACK_DTYPE record array per frame (the tracked_stracks of that frame); `messages(recs)` turns a record array into
        the reference's track messages (strack.py:207-215).  `tracked_stracks` afterwards reflects the last frame."""
        counts = np.fromiter((len(d[1]) for d in frames_dets), dtype=np.int32, count=len(frames_dets))
        tot = int(counts.sum())
        boxes = np.zeros((tot, 4), np.float64)
        scores = np.zeros(tot, np.float64)
        ids = np.zeros(tot, np.int32)
        o = 0
        for (bb, sc, cl), n in zip(frames_dets, counts):
            if n:
                boxes[o:o + n] = np.asarray(bb, dtype=np.float64).reshape(-1, 4)
                scores[o:o + n] = np.asarray(sc, dtype=np.float64)
                ids[o:o + n] = [self._cid(c) for c in (cl.tolist() if hasattr(cl, "tolist") else cl)]
            o += n
        recs = self._nt.update_batch(counts, boxes, scores, ids)
        self.frame_id += len(frames_dets)
        if recs:
            self.tracked_stracks = [self._view(r, None) for r in recs[-1]]
        return recs

    def update_batch_arrays(self, counts, xyxy, scores, class_ids):
        """update_batch on already concatenated arrays (the pipeline's hot path): counts [F] int, xyxy [sum, 4], scores [sum],
        class_ids [sum] integer labels.  Labels are mapped to the tracker's class slots in first-seen order like `update` does."""
        return self._advanced(self._nt.update_batch(counts, xyxy, scores, self._class_slots(class_ids)))

    def _class_slots(self, class_ids):
        """class slots of a label array, registering unseen labels in order of first appearance"""
        cl = np.asarray(class_ids)
        if not cl.size:
            return np.zeros(0, np.int32)
        uniq, first = np.unique(cl, return_index=True)
        for u in uniq[np.argsort(first)].tolist():
            self._cid(u)
        lut = np.array([self._labels[u] for u in uniq.tolist()], np.int32)
        return lut[np.searchsorted(uniq, cl)]

    def _advanced(self, recs):
        """bookkeeping after the native tracker advanced len(recs) frames"""
        self.frame_id += len(recs)
        if recs:
            self.tracked_stracks = [self._view(r, None) for r in recs[-1]]
        return recs

    def messages(self, recs):
        """Track messages (STrack.get_track_message, strack.py:207-215) of one frame's record array."""
        return [{"track_id": int(r["track_id"]), "count": int(r["pad"]), "is_activated": bool(r["is_activated"]), "state": int(r["state"]),
                 "score": float(r["score"]), "start_frame_number": int(r["start_frame"]), "curr_frame_number": int(r["frame_id"]),
                 "time_since_update": 0, "location": str((np.inf, np.inf)), "crops": [], "class_id": self._label_list[int(r["class_id"])]}
                for r in recs]

    @property
    def lost_stracks(self):
        out = []
        for r in self._nt.get(1):
            v = self._views.get(int(r["track_id"])) or TrackView()
            v.track_id, v.is_activated, v.state = int(r["track_id"]), bool(r["is_activated"]), int(r["state"])
            v.score, v.class_id = float(r["score"]), self._label_list[int(r["class_id"])]
            v.start_frame, v.frame_id, v.tracklet_len = int(r["start_frame"]), int(r["frame_id"]), int(r["tracklet_len"])
            v.mean, v._tlwh = r["mean"].copy(), r["tlwh"].copy()
            out.append(v)
        return out

    def reset(self):
        self.frame_id = 0
        self.tracked_stracks, self.removed_stracks, self._views = [], [], {}
        self._nt.reset()

    def DrawTrackedOnFrame(self, frame, show_box=True, show_traject=True):
        for t in [t for t in self.tracked_stracks if t.is_activated]:
            tlwh = t.tlwh
            if tlwh[2] * tlwh[3] > self.min_box_area:
                if show_box:
                    self.plot_bbox(frame, tlwh, t.class_id, t.track_id)
                if show_traject:
                    self.plot_trajectories(frame, t.trajectories, t.class_id, t.track_id)
                    self.plot_directions(frame, t.xyah, t.filter_trajectories(frame, (10, 10)), t.class_id)


def update_trackers(trackers, counts, xyxy, scores, class_ids):
    """Advance K BYTETrackers (one per camera) over F frames in ONE library call, with one association launch per frame for all
    cameras.  counts [F, K]; xyxy [sum, 4], scores [sum] and class_ids [sum] concatenated frame-major, then in camera order.  Each
    tracker maps labels to its own class slots as update_batch_arrays does.  Returns, per camera, the list (per frame) of
    TRACK_DTYPE record arrays: exactly what the K trackers' update_batch_arrays would return when driven one frame at a time in
    camera order.  Each tracker's tracked_stracks afterwards reflects its last frame."""
    from ... import _capi
    K = len(trackers)
    cnt = np.asarray(counts, np.int32).reshape(-1, K)
    cl = np.asarray(class_ids)
    cam = np.repeat(np.tile(np.arange(K), cnt.shape[0]), cnt.ravel())         # camera of each detection
    ids = np.zeros(len(cl), np.int32)
    for k, t in enumerate(trackers):
        sel = cam == k
        ids[sel] = t._class_slots(cl[sel])
    recs = _capi.NativeTracker.update_multi([t._nt for t in trackers], cnt, xyxy, scores, ids)
    for t, r in zip(trackers, recs):
        t._advanced(r)
    return recs
