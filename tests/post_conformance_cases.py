"""Generators, float64 references and error bounds of the post-processing conformance suite (head decode, candidate selection and
NMS, association and tracking at crowd scale).  Used by tests/test_gpu_post_conformance.py and tests/test_post_conformance_cpu.py.

Decode bounds.  The decode kernels (csrc/yolo_post.cu) are compiled with -fmad=false and without fast-math, so every float32 operation
rounds once, to nearest: a result v carries an error of at most U |v|, U = 2^-24.  CUDA documents `expf` to within 2 ulp, i.e. a
relative error of at most 4U.  The reference below decodes the SAME float32 head values in float64; the bounds sum the float32
roundings of the kernel's own operation chain:

  sigmoid 1 / (1 + expf(-z)):  expf 4U (scaled by e / (1 + e) <= 1), the add U, the division U  ->  6U * s  (+ FLT_MIN absolute for the
                                values expf flushes to 0 or inf).
  DFL expectation over nb bins (16 for v8, 17 for v6 reg_max 16):  m = max is exact, p - m rounds by U |p - m| which expf turns into a
                                relative error of U |p - m|, expf adds 4U: eps = 4U + U max|p - m|.  Numerator and denominator are
                                sequential float32 sums of nb terms (nb U each, plus U for k * e), the division adds U:
                                |d' - d| <= d (2 eps + 2 nb U + U) + U d   (weights all perturbed by at most eps + nb U, relative).
                                An expf result in the subnormal range (p - m < -87) is off by up to 2 ulp of the subnormal spacing,
                                2^-148, absolutely; summed with weights k < nb over a denominator >= 1 (the max bin's term is 1),
                                that adds nb^2 2^-148.
  box  x1 = ax - d0, x2 = ax + d2 (U each), (x1 + x2) (U), * 0.5 (exact), * stride (U);  w = (x2 - x1) * stride likewise.
  v5   (s * 2 - 0.5 + x) * stride: 2 err_s + U |t1| + U |t2| before the stride, U after;  (2 s)^2 * anchor: 2 * 6U + 2U relative.
Second-order terms are covered by a factor (1 + 1e-3).
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24
FLT_MIN = float(np.finfo(np.float32).tiny)
SECOND_ORDER = 1.0 + 1e-3


# ---------------------------------------------------------------------------------------------------------------------------------
# head decode: float64 reference and per-element bound
# ---------------------------------------------------------------------------------------------------------------------------------
def _sigmoid(z):
    with np.errstate(over="ignore"):
        s = 1.0 / (1.0 + np.exp(-z))
    return s, 6 * U * s * SECOND_ORDER + FLT_MIN


def _dfl(p, nb):
    """p [..., 4 * nb] float64 (side-major) -> distances [..., 4] and their bound"""
    p = p.reshape(p.shape[:-1] + (4, nb))
    dl = p - p.max(-1, keepdims=True)
    e = np.exp(dl)
    k = np.arange(nb, dtype=np.float64)
    d = (e * k).sum(-1) / e.sum(-1)
    eps = 4 * U + U * (-dl).max(-1)
    return d, (d * (2 * eps + 2 * nb * U + U) + U * d + nb * nb * 2.0 ** -148) * SECOND_ORDER


def _box_from_dist(d, ed, x, y, st):
    """cx, cy, w, h (float64) and bounds of the v8 / v6 box arithmetic from distances d [..., 4] with bounds ed"""
    ax, ay = x + 0.5, y + 0.5
    x1, y1, x2, y2 = ax - d[..., 0], ay - d[..., 1], ax + d[..., 2], ay + d[..., 3]
    out = [(x1 + x2) * 0.5 * st, (y1 + y2) * 0.5 * st, (x2 - x1) * st, (y2 - y1) * st]
    ec = lambda ea, eb, a, b, s: (st * 0.5 * (ea + eb + U * (abs(a) + abs(b)) + U * abs(a + b)) + U * abs(s)) * SECOND_ORDER
    ew = lambda ea, eb, a, b, s: (st * (ea + eb + U * (abs(a) + abs(b)) + U * abs(b - a)) + U * abs(s)) * SECOND_ORDER
    bnd = [ec(ed[..., 0], ed[..., 2], x1, x2, out[0]), ec(ed[..., 1], ed[..., 3], y1, y2, out[1]),
           ew(ed[..., 0], ed[..., 2], x1, x2, out[2]), ew(ed[..., 1], ed[..., 3], y1, y2, out[3])]
    return np.stack(out, -1), np.stack(bnd, -1)


def _grid(H, W):
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    return x.ravel(), y.ravel()


def decode_reference(kind, levels, nc, reg_max=16, anchors=None):
    """float64 decode of head levels [(grid [B, H, W, C] float32, stride)] -> (ref, bound) in the engine's raw layout:
    kind "v8": [B, 4 + nc, A];  "v6": [B, A, 5 + nc] (reg_max 0 or 16);  "v5": [B, A, 5 + nc] with anchors [L, 3, 2]."""
    refs, bnds = [], []
    for li, (g, st) in enumerate(levels):
        B, H, W, C = g.shape
        p = g.astype(np.float64)
        x, y = _grid(H, W)
        if kind in ("v8", "v6"):
            p = p.reshape(B, H * W, C)
            nb = 16 if kind == "v8" else reg_max + 1
            if kind == "v6" and reg_max == 0:
                d, ed = p[..., :4], np.zeros(p.shape[:-1] + (4,))
            else:
                d, ed = _dfl(p[..., :4 * nb], nb)
            box, eb = _box_from_dist(d, ed, x, y, float(st))
            cc = 64 if kind == "v8" else (4 * (reg_max + 1) + 7) // 8 * 8
            s, es = _sigmoid(p[..., cc:cc + nc])
            if kind == "v8":
                refs.append(np.concatenate([box, s], -1))
                bnds.append(np.concatenate([eb, es], -1))
            else:
                one = np.ones(box.shape[:-1] + (1,))
                refs.append(np.concatenate([box, one, s], -1))
                bnds.append(np.concatenate([eb, np.zeros_like(one), es], -1))
        else:
            no = 5 + nc
            p = p[..., :3 * no].reshape(B, H * W, 3, no).transpose(0, 2, 1, 3)          # [B, anchor, cell, no]
            s, es = _sigmoid(p)
            o, eo = s.copy(), es.copy()
            for c, grid in ((0, x), (1, y)):
                t1 = s[..., c] * 2 - 0.5
                t2 = t1 + grid
                o[..., c] = t2 * st
                eo[..., c] = (st * (2 * es[..., c] + U * abs(t1) + U * abs(t2)) + U * abs(o[..., c])) * SECOND_ORDER
            for c in (2, 3):
                a = np.asarray(anchors[li], np.float64)[:, c - 2][None, :, None]
                o[..., c] = (s[..., c] * 2) ** 2 * a
                eo[..., c] = (8 * s[..., c] * es[..., c] * a + 2 * U * abs(o[..., c])) * SECOND_ORDER
            refs.append(o.reshape(B, 3 * H * W, no))
            bnds.append(eo.reshape(B, 3 * H * W, no))
    ref, bnd = np.concatenate(refs, 1), np.concatenate(bnds, 1)
    if kind == "v8":
        ref, bnd = ref.transpose(0, 2, 1), bnd.transpose(0, 2, 1)
    return ref, bnd


def decode_excess(got, ref, bnd):
    """max over elements of |got - ref| / bound (<= 1 passes) and the worst absolute error"""
    err = np.abs(got.astype(np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bnd > 0, err / bnd, np.where(err > 0, np.inf, 0.0))        # a zero bound (an exact value) demands equality
    return float(r.max()), float(err.max())


# ---------------------------------------------------------------------------------------------------------------------------------
# numpy float32 emulation of the decode kernels (CPU teeth checks): the kernel's operation order, or deliberately wrong variants
# ---------------------------------------------------------------------------------------------------------------------------------
def emulate_decode(kind, levels, nc, reg_max=16, anchors=None, mutation=None, reverse_sums=False):
    f = np.float32
    outs = []
    strides = [st for _, st in levels]
    for li, (g, st) in enumerate(levels):
        B, H, W, C = g.shape
        if mutation == "stride_off_by_one_level":
            st = strides[min(li + 1, len(strides) - 1)] if li == 0 else st
        p = g.astype(np.float32)
        y, x = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
        x, y = x.ravel(), y.ravel()
        if mutation == "xy_swapped":
            x, y = y, x
        off = f(0.0) if mutation == "anchor_offset_0" else f(0.5)
        if kind in ("v8", "v6"):
            p = p.reshape(B, H * W, C)
            nb = 16 if kind == "v8" else reg_max + 1
            d = np.empty((B, H * W, 4), np.float32)
            for s in range(4):
                if kind == "v6" and reg_max == 0:
                    d[..., s] = p[..., s]
                    continue
                nbk = 15 if mutation == "dfl_15_bins" else nb
                bins = p[..., s * nb:s * nb + nbk]
                m = bins.max(-1, keepdims=True)
                e = np.exp((bins - m).astype(np.float32)).astype(np.float32)
                order = range(nbk - 1, -1, -1) if reverse_sums else range(nbk)
                den = np.zeros((B, H * W), np.float32)
                num = np.zeros((B, H * W), np.float32)
                for k in order:
                    den = (den + e[..., k]).astype(np.float32)
                    num = (num + e[..., k] * f(k)).astype(np.float32)
                d[..., s] = num / den
            ax, ay = x + off, y + off
            x1, y1, x2, y2 = ax - d[..., 0], ay - d[..., 1], ax + d[..., 2], ay + d[..., 3]
            stf = f(st)
            box = np.stack([(x1 + x2) * f(0.5) * stf, (y1 + y2) * f(0.5) * stf, (x2 - x1) * stf, (y2 - y1) * stf], -1)
            cc = 64 if kind == "v8" else (4 * (reg_max + 1) + 7) // 8 * 8
            with np.errstate(over="ignore"):
                sg = (f(1) / (f(1) + np.exp(-p[..., cc:cc + nc]))).astype(np.float32)
            if kind == "v8":
                outs.append(np.concatenate([box, sg], -1))
            else:
                outs.append(np.concatenate([box, np.ones(box.shape[:-1] + (1,), np.float32), sg], -1))
        else:
            no = 5 + nc
            q = p[..., :3 * no].reshape(B, H * W, 3, no).transpose(0, 2, 1, 3)
            with np.errstate(over="ignore"):
                s = (f(1) / (f(1) + np.exp(-q))).astype(np.float32)
            o = s.copy()
            stf = f(st)
            o[..., 0] = (s[..., 0] * f(2) - f(0.5) + x) * stf
            o[..., 1] = (s[..., 1] * f(2) - f(0.5) + y) * stf
            a = np.asarray(anchors[li], np.float32)
            if mutation == "anchor_wh_swapped":
                a = a[:, ::-1]
            o[..., 2] = (s[..., 2] * f(2)) * (s[..., 2] * f(2)) * a[:, 0][None, :, None]
            o[..., 3] = (s[..., 3] * f(2)) * (s[..., 3] * f(2)) * a[:, 1][None, :, None]
            outs.append(o.reshape(B, 3 * H * W, no))
    out = np.concatenate(outs, 1)
    return out.transpose(0, 2, 1) if kind == "v8" else out


def random_levels(seed, kind, in_hw=(256, 384), nc=80, reg_max=16, strides=(8, 16, 32)):
    """seeded head levels shaped like a plan's f32 head buffers' interiors: [(grid [1, H, W, C], stride)]"""
    rng = np.random.default_rng(seed)
    levels = []
    for st in strides:
        H, W = in_hw[0] // st, in_hw[1] // st
        if kind == "v8":
            C = 64 + nc
            g = np.concatenate([rng.normal(0, 3, (1, H, W, 64)), rng.normal(-3, 3, (1, H, W, nc))], -1)
        elif kind == "v6":
            cc = (4 * (reg_max + 1) + 7) // 8 * 8
            C = cc + nc
            g = rng.normal(-3, 3, (1, H, W, C))
            g[..., :4 * (reg_max + 1)] = rng.uniform(0, 8, (1, H, W, 4)) if reg_max == 0 else rng.normal(0, 3, (1, H, W, 4 * (reg_max + 1)))
        else:
            C = 3 * (5 + nc)
            g = rng.normal(-1, 2, (1, H, W, C))
        levels.append((g.astype(np.float32), st))
    return levels


# ---------------------------------------------------------------------------------------------------------------------------------
# crafted head logits: the values seeded weights never produce
# ---------------------------------------------------------------------------------------------------------------------------------
CLASS_LOGITS = [30.0, -30.0, 17.0, -17.0, 88.0, -88.0, 88.5, -88.5, 89.0, -89.0, 104.0, -104.0, 0.0, 3.5, -3.5, 1e4, -1e4, 16.5, -0.25]


def dfl_patterns(nb, rng):
    """side logits [n, nb] with the DFL edge cases: all bins equal (small and large), one dominant bin at 0 or at nb - 1 over -30 or over
    bins whose expf after the max subtraction underflows (-88 .. -104: subnormal or 0), bins near the fp16 range (60000 over 59904), a
    ramp from -100 to 0, and ordinary N(0, 3) logits"""
    pats = [np.zeros(nb), np.full(nb, 50.0)]
    for k in (0, nb - 1):
        for low in (-30.0, -88.0, -104.0):
            v = np.full(nb, low)
            v[k] = 0.0
            pats.append(v)
        v = np.full(nb, 59904.0)
        v[k] = 60000.0
        pats.append(v)
    pats.append(np.linspace(-100.0, 0.0, nb))
    pats.append(np.linspace(0.0, -100.0, nb))
    pats.append(rng.normal(0, 3, nb))
    return np.array(pats)


def crafted_head(seed, kind, H, W, C, nc, reg_max=16, B=2):
    """head logits [B, H, W, C] (float16-exact, so a 1x1 identity conv reproduces them in f32 exactly): every cell's four DFL sides
    and class logits cycle through dfl_patterns / CLASS_LOGITS with a per-image, per-cell offset"""
    rng = np.random.default_rng(seed)
    nb = 16 if kind == "v8" else reg_max + 1
    cc = 64 if kind == "v8" else (4 * (reg_max + 1) + 7) // 8 * 8
    pats = dfl_patterns(nb, rng)
    g = np.zeros((B, H * W, C), np.float32)
    cl = np.array(CLASS_LOGITS)
    for b in range(B):
        for a in range(H * W):
            for s in range(4):
                g[b, a, s * nb:(s + 1) * nb] = pats[(a * 4 + s + 7 * b) % len(pats)]
            g[b, a, cc:cc + nc] = cl[(a + np.arange(nc) + 3 * b) % len(cl)]
    return g.astype(np.float16).astype(np.float32).reshape(B, H, W, C)


# ---------------------------------------------------------------------------------------------------------------------------------
# candidate selection + NMS inputs
# ---------------------------------------------------------------------------------------------------------------------------------
def v8_selection_raw(seed, hits, A=8400, nc=80, in_hw=(640, 640)):
    """raw [4 + nc, A] float32 whose candidate count at box_score 0.4 is exactly `hits`: every other anchor's best class prob is below
    0.35.  Boxes (input pixels) sit in clusters so the NMS suppresses and swaps."""
    rng = np.random.default_rng(seed)
    raw = np.empty((4 + nc, A), np.float32)
    raw[4:] = rng.uniform(0, 0.35, (nc, A))
    k = max(hits // 6, 1)
    centres = rng.uniform(30, min(in_hw) - 30, (k, 2))
    c = centres[np.arange(A) % k] + rng.normal(0, 10, (A, 2))
    raw[0], raw[1] = c[:, 0], c[:, 1]
    raw[2:4] = rng.uniform(12, 90, (2, A))
    hot = rng.permutation(A)[:hits]
    raw[4 + rng.integers(0, nc, hits), hot] = rng.uniform(0.45, 0.99, hits)
    return raw


def v5_selection_raw(seed, hits, A=25200, nc=80, in_hw=(640, 640)):
    """raw [A, 5 + nc] float32 (YOLOv5 layout, conf = cls * obj) with exactly `hits` candidates at box_score 0.4"""
    rng = np.random.default_rng(seed)
    raw = np.empty((A, 5 + nc), np.float32)
    raw[:, 4] = rng.uniform(0, 1, A)
    raw[:, 5:] = rng.uniform(0, 0.35, (A, nc))
    k = max(hits // 6, 1)
    centres = rng.uniform(30, min(in_hw) - 30, (k, 2))
    raw[:, 0:2] = centres[np.arange(A) % k] + rng.normal(0, 10, (A, 2))
    raw[:, 2:4] = rng.uniform(12, 90, (A, 2))
    hot = rng.permutation(A)[:hits]
    raw[hot, 4] = rng.uniform(0.8, 1.0, hits)
    raw[hot, 5 + rng.integers(0, nc, hits)] = rng.uniform(0.6, 0.99, hits)
    return raw


def v8_tie_raw(seed, box_score, A=8400, nc=80):
    """raw [4 + nc, A] with the ties of the selection and NMS rules: 600 anchors at conf exactly 1.0f in 100 groups of identical
    boxes; 60 anchors whose two best classes tie (first class wins); confs at box_score and one float32 ulp either side (the compare is
    strict); 30 zero-area and 30 sub-pixel boxes.  Returns (raw, expected candidate count)."""
    rng = np.random.default_rng(seed)
    raw = np.empty((4 + nc, A), np.float32)
    raw[4:] = rng.uniform(0, 0.3, (nc, A))
    raw[0:2] = rng.uniform(20, 620, (2, A))
    raw[2:4] = rng.uniform(10, 60, (2, A))
    perm = rng.permutation(A)
    sat, tie, edge, zero, sub = perm[:600], perm[600:660], perm[660:663], perm[663:693], perm[693:723]
    grp = rng.uniform(20, 620, (100, 4)).astype(np.float32)
    grp[:, 2:] = rng.uniform(15, 80, (100, 2))
    raw[0:4, sat] = grp[np.arange(600) % 100].T
    raw[4 + rng.integers(0, nc, 600), sat] = np.float32(1.0)
    c1 = rng.integers(0, nc - 1, 60)
    c2 = c1 + 1 + rng.integers(0, nc - 1 - c1)
    v = rng.uniform(0.5, 0.95, 60).astype(np.float32)
    raw[4 + c1, tie] = v
    raw[4 + c2, tie] = v
    t = np.float32(box_score)
    assert float(t) == box_score
    raw[4 + 7, edge] = [np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1))]
    raw[4 + 3, zero] = rng.uniform(0.5, 0.9, 30)
    raw[2, zero[:15]] = 0.0
    raw[3, zero[15:]] = 0.0
    raw[4 + 4, sub] = rng.uniform(0.5, 0.9, 30)
    raw[2:4, sub] = rng.uniform(0.05, 0.9, (2, 30))
    return raw, 600 + 60 + 1 + 30 + 30


# ---------------------------------------------------------------------------------------------------------------------------------
# association problems and crowded tracking sequences
# ---------------------------------------------------------------------------------------------------------------------------------
def lap_cost(seed, T, D, sparse):
    """T x D cost: uniform (0, 1), or IoU-like -- mostly exactly 1.0 (no overlap) with ~3 overlaps per row in (0, 1)"""
    rng = np.random.default_rng(seed)
    if not sparse:
        return rng.uniform(0, 1, (T, D))
    c = np.ones((T, D))
    for i in range(T):
        j = rng.integers(0, D, 3)
        c[i, j] = rng.uniform(0.05, 0.95, 3)
    return c


def crowd_sequence(seed, objects=300, frames=64, clutter=150):
    """Per-frame (boxes xyxy float64 [n, 4], scores float64 [n], class ids int32 [n]) of a crowded scene: linear motion, staggered births,
    drop-outs, low-score detections (stage 2), and `clutter` one-frame high-score detections per frame that are born unconfirmed and
    removed on the next frame (stage 3, and the removed list grows by ~clutter per frame).  Float boxes: exact cost ties have measure 0."""
    rng = np.random.default_rng(seed)
    pos = rng.uniform(0, 4000, (objects, 2))
    vel = rng.uniform(-6, 6, (objects, 2))
    size = rng.uniform(30, 90, (objects, 2))
    cls = rng.integers(0, 4, objects)
    born = np.where(rng.random(objects) < 0.6, 0, rng.integers(1, frames // 2, objects))
    gone = np.where(rng.random(objects) < 0.2, rng.integers(frames // 2, frames, objects), frames)
    seq = []
    for f in range(frames):
        b, s, c = [], [], []
        for o in range(objects):
            if f < born[o] or f >= gone[o] or rng.random() < 0.08:
                continue
            p = pos[o] + vel[o] * f + rng.normal(0, 1.0, 2)
            wh = size[o] + rng.normal(0, 1.0, 2)
            b.append([p[0] - wh[0] / 2, p[1] - wh[1] / 2, p[0] + wh[0] / 2, p[1] + wh[1] / 2])
            s.append(rng.uniform(0.65, 0.95) if rng.random() > 0.15 else rng.uniform(0.15, 0.45))
            c.append(cls[o] if rng.random() > 0.05 else 9)
        for _ in range(clutter if f > 0 else 0):
            x, y = rng.uniform(0, 4000, 2)
            w, h = rng.uniform(20, 50, 2)
            b.append([x, y, x + w, y + h])
            s.append(rng.uniform(0.62, 0.9))
            c.append(5)
        seq.append((np.asarray(b, np.float64).reshape(-1, 4), np.asarray(s, np.float64), np.asarray(c, np.int32)))
    return seq


def grid_boxes(n, x0=0.0, y0=0.0, cell=60.0, size=40.0, cols=64):
    """n non-overlapping boxes xyxy on a grid (no two of them overlap, so every association is unique)"""
    i = np.arange(n)
    x, y = x0 + (i % cols) * cell, y0 + (i // cols) * cell
    return np.stack([x, y, x + size, y + size], 1).astype(np.float64)


def track_rows(tracks):
    """[n, 9] float64 rows (track id, state, activated, class, tlwh, score) of a list of oracle.track.Track"""
    return np.array([[t.tid, t.state, int(t.activated), t.cls, *t.tlwh(), t.score] for t in tracks], np.float64).reshape(-1, 9)


def native_rows(recs):
    """the same rows from native TRACK_DTYPE records"""
    return np.column_stack([recs["track_id"], recs["state"], recs["is_activated"], recs["class_id"], recs["tlwh"],
                            recs["score"]]).astype(np.float64).reshape(-1, 9)


def run_oracle(tracker_cls, seq, **kw):
    """oracle.track.Tracker over seq -> (per-frame (tracked rows, lost ids)), max pool (confirmed + lost) and max unconfirmed the
    association saw, and the final length of the removed list"""
    t = tracker_cls(**kw)
    t.reset()
    out, pmax, umax = [], 0, 0
    for b, s, c in seq:
        conf = [x for x in t.tracked if x.activated]
        ids = {x.tid for x in conf}
        pmax = max(pmax, len(conf) + len([x for x in t.lost if x.tid not in ids]))
        umax = max(umax, len(t.tracked) - len(conf))
        tracked = t.update(b, s, c)
        out.append((track_rows(tracked), [x.tid for x in t.lost]))
    return out, pmax, umax, len(t.removed)
