"""oracle/track.py -- TEST INFRASTRUCTURE ONLY: CPU restatement of the reference's ByteTrack.

Follows ObjectTracker/byteTrack/byteTracker.py:62-185 (three association stages, births, ageing, list maintenance),
dtypes/strack.py (state, class vote, conversions), dtypes/kalman_filter.py:55-226 (constant-velocity filter) and
utils.py:9-69 (joint / sub / duplicate removal), with matching.py's IoU cost and `lap.lapjv` restated in
oracle/post.py.  Pinned against the unmodified reference by tests/golden/track.npz (tests/test_oracle_track.py).
Never imported by the product path.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

from . import post

NEW, TRACKED, LOST, REMOVED = 0, 1, 2, 3
_F = np.eye(8)
for _i in range(4):
    _F[_i, 4 + _i] = 1.0
_H = np.eye(4, 8)
_WP, _WV = 1.0 / 20, 1.0 / 160


class _Counter:
    n = 0


class Track:
    def __init__(self, tlwh, score, cls):
        self.tlwh0 = np.asarray(tlwh, dtype=float)
        self.mean = None
        self.cov = None
        self.activated = False
        self.state = NEW
        self.tid = 0
        self.frame = 0
        self.start = 0
        self.score = score
        self.cls = cls
        self.votes = {cls: 1}

    def tlwh(self):
        if self.mean is None:
            return self.tlwh0.copy()
        r = self.mean[:4].copy()
        r[2] *= r[3]
        r[:2] -= r[2:] / 2
        return r

    def tlbr(self):
        r = self.tlwh()
        r[2:] += r[:2]
        return r

    @staticmethod
    def xyah(tlwh):
        r = np.asarray(tlwh).copy()
        r[:2] += r[2:] / 2
        r[2] /= r[3]
        return r

    def vote(self, cls):
        self.votes[cls] = self.votes.get(cls, 1) + 1            # strack.py:128 (a new class starts at 2)
        self.cls = max(self.votes, key=self.votes.get)


def kf_initiate(m):
    mean = np.r_[m, np.zeros_like(m)]
    std = [2 * _WP * m[3], 2 * _WP * m[3], 1e-2, 2 * _WP * m[3], 10 * _WV * m[3], 10 * _WV * m[3], 1e-5, 10 * _WV * m[3]]
    return mean, np.diag(np.square(std))


def kf_multi_predict(mean, cov):
    sp = [_WP * mean[:, 3], _WP * mean[:, 3], 1e-2 * np.ones_like(mean[:, 3]), _WP * mean[:, 3]]
    sv = [_WV * mean[:, 3], _WV * mean[:, 3], 1e-5 * np.ones_like(mean[:, 3]), _WV * mean[:, 3]]
    sqr = np.square(np.r_[sp, sv]).T
    q = np.asarray([np.diag(sqr[i]) for i in range(len(mean))])
    mean = np.dot(mean, _F.T)
    left = np.dot(_F, cov).transpose((1, 0, 2))
    return mean, np.dot(left, _F.T) + q


def kf_update(mean, cov, z):
    std = [_WP * mean[3], _WP * mean[3], 1e-1, _WP * mean[3]]
    pm = np.dot(_H, mean)
    pc = np.linalg.multi_dot((_H, cov, _H.T)) + np.diag(np.square(std))
    cf, low = scipy.linalg.cho_factor(pc, lower=True, check_finite=False)
    k = scipy.linalg.cho_solve((cf, low), np.dot(cov, _H.T).T, check_finite=False).T
    return mean + np.dot(z - pm, k.T), cov - np.linalg.multi_dot((k, pc, k.T))


def _assign(tracks, dets, thresh, fuse, solver=None):
    """one association stage; `solver(cost, thresh) -> (x, y, ...)` is post.lapjv_extended unless given (a test may pass one that
    follows another solver's tie-breaking)"""
    if not tracks or not dets:
        return [], list(range(len(tracks))), list(range(len(dets)))
    a = np.array([t.tlbr() for t in tracks])
    b = np.array([d.tlbr() for d in dets])
    cost = post.iou_cost(a, b, [d.score for d in dets] if fuse else None)
    x, y = (solver or post.lapjv_extended)(cost, thresh)[:2]
    return [(i, int(j)) for i, j in enumerate(x) if j >= 0], [i for i, j in enumerate(x) if j < 0], [j for j, i in enumerate(y) if i < 0]


def _joint(a, b):
    seen, out = set(), []
    for t in a + b:
        if t.tid not in seen:
            seen.add(t.tid)
            out.append(t)
    return out


def _sub(a, b):
    d = {t.tid: t for t in a}
    for t in b:
        d.pop(t.tid, None)
    return list(d.values())


class Tracker:
    def __init__(self, track_thresh=0.5, track_buffer=30, match_thresh=0.8, frame_rate=30, solver=None):
        self.tracked, self.lost, self.removed = [], [], []
        self.track_thresh, self.match_thresh = track_thresh, match_thresh
        self.solver = solver
        self.det_thresh = track_thresh + 0.1
        self.max_lost = int(frame_rate / 30.0 * track_buffer)
        self.frame = 0

    def reset(self):
        self.tracked, self.lost, self.removed = [], [], []
        self.frame = 0
        _Counter.n = 0

    def _hit(self, t, d, activated, refind):
        z = Track.xyah(d.tlwh())
        if t.state == TRACKED:
            t.frame = self.frame
            t.mean, t.cov = kf_update(t.mean, t.cov, z)
            t.state, t.activated, t.score = TRACKED, True, d.score
            t.vote(d.cls)
            activated.append(t)
        else:
            t.mean, t.cov = kf_update(t.mean, t.cov, z)
            t.state, t.activated, t.frame, t.score = TRACKED, True, self.frame, d.score
            t.vote(d.cls)
            refind.append(t)

    def update(self, boxes, scores, classes):
        self.frame += 1
        activated, refind, lost, removed = [], [], [], []
        boxes, scores, classes = np.array(boxes), np.array(scores), np.array(classes)
        hi = scores > self.track_thresh
        lo = np.logical_and(scores > 0.1, scores < self.track_thresh)

        def mk(mask):
            out = []
            for bb, s, c in zip(boxes[mask], scores[mask], classes[mask]):
                r = np.asarray(bb).copy()
                r[2:] -= r[:2]
                out.append(Track(r, s, c))
            return out

        dets, dets2 = mk(hi), mk(lo)
        unconf = [t for t in self.tracked if not t.activated]
        conf = [t for t in self.tracked if t.activated]
        pool = _joint(conf, self.lost)
        if pool:
            mm = np.asarray([t.mean.copy() for t in pool])
            cc = np.asarray([t.cov for t in pool])
            for i, t in enumerate(pool):
                if t.state != TRACKED:
                    mm[i][7] = 0
            mm, cc = kf_multi_predict(mm, cc)
            for t, m, c in zip(pool, mm, cc):
                t.mean, t.cov = m, c
        m1, ut, ud = _assign(pool, dets, self.match_thresh, True, self.solver)
        for i, j in m1:
            self._hit(pool[i], dets[j], activated, refind)
        rem = [pool[i] for i in ut if pool[i].state == TRACKED]
        m2, ut2, _ = _assign(rem, dets2, 0.5, False, self.solver)
        for i, j in m2:
            self._hit(rem[i], dets2[j], activated, refind)
        for i in ut2:
            if rem[i].state != LOST:
                rem[i].state = LOST
                lost.append(rem[i])
        dets = [dets[i] for i in ud]
        m3, uu, ud3 = _assign(unconf, dets, 0.7, True, self.solver)
        for i, j in m3:
            self._hit(unconf[i], dets[j], activated, refind)
        for i in uu:
            unconf[i].state = REMOVED
            removed.append(unconf[i])
        for j in ud3:
            t = dets[j]
            if t.score < self.det_thresh:
                continue
            _Counter.n += 1
            t.tid = _Counter.n
            t.mean, t.cov = kf_initiate(Track.xyah(t.tlwh0))
            t.state = TRACKED
            t.activated = self.frame == 1
            t.frame = t.start = self.frame
            activated.append(t)
        for t in self.lost:
            if self.frame - t.frame > self.max_lost:
                t.state = REMOVED
                removed.append(t)
        self.tracked = [t for t in self.tracked if t.state == TRACKED]
        self.tracked = _joint(self.tracked, activated)
        self.tracked = _joint(self.tracked, refind)
        self.lost = _sub(self.lost, self.tracked)
        self.lost.extend(lost)
        self.lost = _sub(self.lost, self.removed)
        self.removed.extend(removed)
        if self.tracked and self.lost:
            d = post.iou_cost(np.array([t.tlbr() for t in self.tracked]), np.array([t.tlbr() for t in self.lost]))
            da, db = set(), set()
            for ia, ib in zip(*np.where(d < 0.15)):
                if self.tracked[ia].frame - self.tracked[ia].start > self.lost[ib].frame - self.lost[ib].start:
                    db.add(ib)
                else:
                    da.add(ia)
            self.tracked = [t for i, t in enumerate(self.tracked) if i not in da]
            self.lost = [t for i, t in enumerate(self.lost) if i not in db]
        return self.tracked
