"""GPU: plans at the edges the loader allows, and the footprint model of tests/plan_footprint.py against the device.

Only plans that adas_plan_validate accepts and that the footprint model finds in bounds are ever run here.

1. Tightest legal heads: YOLOv8 and YOLOv5-layout levels exactly 64 + nc and 3 (5 + nc) columns wide at a nonzero channel offset of
   a wider fp32 buffer, and a UFLD v2 head exactly total_dim wide at an offset of a dense buffer, every neighbouring column and the
   halo NaN; decoded on the device and compared with the float64 references.
2. Every byte of every buffer that the model says no op, staging kernel or head decode touches at batch 2 of max_batch 3 (channels
   past all claimed slices, the third image, the allocation slack) is poisoned; one inference must leave the poison unchanged (no
   stray writes) and give bit for bit the outputs and buffer contents of a run where those bytes held zeros (no stray reads)."""
import ctypes as C

import numpy as np
import pytest

import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
import lane_conformance_cases as lc
import plan_footprint as fp
import post_conformance_cases as pc
import synth
from oracle import post
from test_gpu_lane_conformance import _check_v2
from test_plan_validation_cpu import FAMILIES

pytestmark = pytest.mark.gpu


def _accepted_in_bounds(path, max_batch):
    _capi.plan_validate(path)
    pl = fp.parse(open(path, "rb").read())
    assert fp.out_of_bounds(pl, max_batch) == []
    return pl


def _level_buffer(g, off, width, total):
    """[B, H, W, c] head values -> [B * (H + 2) * (W + 2), total] fp32 with the values in columns [off, off + width) of the interior
    and NaN everywhere else (halo ring and neighbouring columns)"""
    B, H, W, _ = g.shape
    out = np.full((B, H + 2, W + 2, total), np.nan, np.float32)
    out[:, 1:-1, 1:-1, off:off + width] = g[..., :width]
    return out.reshape(-1, total)


def _head_plan(tmp_path, kind, in_h, in_w, nc, strides, off, anchors=None):
    width = 64 + nc if kind == "v8" else 3 * (5 + nc)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8 if kind == "v8" else plan.MODEL_YOLOV5, 3, in_h, in_w)
    levels, A = [], 0
    for st in strides:
        H, W = in_h // st, in_w // st
        head = pb.new_padded(H, W, (off + width + 4) // 4 * 4, f32=True)      # at least one NaN column after the level
        pb.outputs.append((head.buf, off, width, st))
        levels.append((head, st))
        A += (1 if kind == "v8" else 3) * H * W
    pb.meta[0], pb.meta[1] = nc, A
    if anchors is not None:
        pb.meta[3] = 1 + pb.tensor(np.asarray(anchors, np.float32))
    path = str(tmp_path / f"tight_{kind}_{len(strides)}.b200w")
    pb.write(path)
    return path, levels, width


@pytest.mark.parametrize("kind,in_hw,nc,strides", [("v8", (64, 96), 13, (8, 16, 32)), ("v5", (128, 192), 2, (8, 16, 32, 64))],
                         ids=["v8-3-levels", "v5-4-levels"])
def test_tightest_legal_yolo_head_matches_float64(tmp_path, kind, in_hw, nc, strides):
    rng = np.random.default_rng(7)
    anchors = None if kind == "v8" else rng.uniform(4, 200, (len(strides), 3, 2)).astype(np.float32)
    off = 5
    path, levels, width = _head_plan(tmp_path, kind, *in_hw, nc, strides, off, anchors)
    _accepted_in_bounds(path, 2)
    eng = _capi.Engine(path, 0, max_batch=2)
    grids = []
    for li, (head, st) in enumerate(levels):
        if kind == "v8":
            g = pc.crafted_head(60 + li, "v8", head.H, head.W, width, nc).astype(np.float32)
        else:
            g = rng.normal(0, 3, (2, head.H, head.W, width)).astype(np.float32)
        eng.write_buffer(head.buf, _level_buffer(g, off, width, head.C))
        grids.append((g, st))
    raw = eng.infer(np.zeros((2, 3) + in_hw, np.float32))[0]
    ref, bnd = pc.decode_reference(kind, grids, nc, 16, anchors)
    assert raw.shape == ref.shape, (raw.shape, ref.shape)
    assert np.isfinite(raw).all(), "a NaN neighbour of the head columns reached the decode"
    ex, worst = pc.decode_excess(raw, ref, bnd)
    print(f"[tight head] {kind} {len(strides)} levels, {width} columns at offset {off}: max err {worst:.2e}, max err / bound {ex:.3f}")
    assert ex <= 1.0
    eng.close()


def test_tightest_legal_ufld_head_matches_oracle(tmp_path):
    """A UFLD v2 TuSimple head written by the test exactly total_dim wide at offset 3 of a dense fp32 buffer, NaN on both sides"""
    cfg = plan.UFLD_TUSIMPLE
    ngr, ncr, ngc, ncc = cfg["num_grid_row"], cfg["num_cls_row"], cfg["num_grid_col"], cfg["num_cls_col"]
    total = ngr * ncr * 4 + ngc * ncc * 4 + 2 * ncr * 4 + 2 * ncc * 4
    off = 3
    pb = plan.PlanBuilder(plan.MODEL_UFLDV2, 3, cfg["in_h"], cfg["in_w"])
    hb = pb.new_dense(1, off + total + 5, f32=True)
    pb.outputs.append((hb, off, total, 0))
    pb.meta[0:7] = [ngr, ncr, ngc, ncc, 4, total, 1]
    path = str(tmp_path / "tight_ufld.b200w")
    pb.write(path)
    _accepted_in_bounds(path, 2)
    ra, ca = post.UFLD_ANCHORS["tusimple"]
    keeps = lc.keep_threshold_counts(ncr, ncc)
    hs = [lc.v2_heads(700 + b, ngr, ncr, ngc, ncc, keep=keeps[b])[0] for b in range(2)]
    buf = np.full((2, off + total + 5), np.nan, np.float32)
    for b, heads in enumerate(hs):
        buf[b, off:off + total] = lc.flat_v2(heads)
    eng = _capi.Engine(path, 0, max_batch=2)
    eng.write_buffer(hb, buf)
    h, w = 720, 1280
    frames = np.stack([synth.frame(s, h, w) for s in (0, 1)])
    pts, npts, status, coords = eng.ufld_detect(frames, want_coords=True)
    for b, heads in enumerate(hs):
        _check_v2(pts, npts, status, coords, b, heads, w, h, ra, ca)
    assert np.array_equal(eng.read_buffer(hb, 2).view(np.uint32), buf.view(np.uint32))       # the head was only read
    eng.close()


# ---- 2. the footprint model against the device -----------------------------------------------------------------------------------
def _claimed_bytes(pl, batch, max_batch):
    """per buffer: bool mask over its whole allocation (logical extent + 256 bytes of slack) of the bytes the model says are touched"""
    masks = []
    for rpi, Cb, dtype, *_ in pl.bufs:
        masks.append(np.zeros(max_batch * rpi * Cb * (4 if dtype == 1 else 2) + 256, bool))
    regions, _, faults = fp.footprint(pl, batch)
    assert not faults
    for r in regions:
        m = masks[r.buf]
        row = r.ld * r.esize
        span = r.rows * row
        grid = np.zeros(max(span, m.size), bool)
        grid[:span].reshape(r.rows, row)[:, r.c0 * r.esize:r.c1 * r.esize] = True
        m |= grid[:m.size]
    return masks


def _read_all(eng, i, nbytes):
    out = np.empty(nbytes, np.uint8)
    _capi.check(_capi.lib().adas_engine_read_buffer(eng._h, i, out.ctypes.data_as(C.c_void_p), C.c_int64(nbytes)))
    return out


@pytest.mark.parametrize("name", [n for n, _ in FAMILIES])
def test_footprint_model_covers_what_the_kernels_touch(tmp_path, monkeypatch, name):
    monkeypatch.setenv("ADAS_B200_AUTOTUNE", "0")       # one tile choice per op: the two runs below share one program
    path = str(tmp_path / f"{name}.b200w")
    dict(FAMILIES)[name]().write(path)
    batch, max_batch = 2, 3
    pl = _accepted_in_bounds(path, max_batch)
    masks = _claimed_bytes(pl, batch, max_batch)
    eng = _capi.Engine(path, 0, max_batch=max_batch)
    in_h, in_w = pl.in_hw
    x = np.random.default_rng(3).uniform(-1, 1, (batch, 3, in_h, in_w)).astype(np.float32)
    # run 1: every byte zero (as allocated)
    clean = [o.copy() for o in eng.infer(x)]
    after_clean = [_read_all(eng, i, m.size) for i, m in enumerate(masks)]
    # run 2: the same zeros where the model claims a byte, 0xFF (NaN in fp16 and fp32) everywhere else
    for i, m in enumerate(masks):
        fill = np.where(m, 0, 0xFF).astype(np.uint8)
        eng.write_buffer(i, fill)
    poisoned = eng.infer(x)
    n_poison = 0
    for i, m in enumerate(masks):
        got = _read_all(eng, i, m.size)
        assert (got[~m] == 0xFF).all(), f"buffer {i}: {int((got[~m] != 0xFF).sum())} unclaimed bytes were written"
        assert np.array_equal(got[m], after_clean[i][m]), f"buffer {i}: claimed bytes differ from the zero-filled run"
        n_poison += int((~m).sum())
    for a, b in zip(poisoned, clean):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    print(f"[footprint] {name}: {len(masks)} buffers, {n_poison} poisoned bytes untouched, outputs bit-identical")
    eng.close()
