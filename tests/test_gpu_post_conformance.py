"""GPU: head decode, candidate selection + NMS, and ByteTrack association at crowd-scale sizes, past the shared-memory routes of their
kernels, against float64 / oracle references (tests/post_conformance_cases.py holds the generators and the decode bounds)."""
import numpy as np
import pytest

import post_conformance_cases as pc
import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
from gpu_util import cached_plan
from oracle import post, track

pytestmark = pytest.mark.gpu


# ---- 1. head decode element by element ------------------------------------------------------------------------------------------
def _plan(tmp_path, kind, scale, **kw):
    W = plan.synth_weights(kind, 0, variant=scale)
    pb = getattr(plan, "build_" + kind)(W, scale, **kw)
    path = str(tmp_path / f"{kind}_{scale}.b200w")
    pb.write(path)
    return path, pb


DECODE_CASES = [("yolov8", "n", dict(in_h=256, in_w=384), "v8"), ("yolov10", "n", dict(nc=70, in_h=256, in_w=384), "v8"),
                ("yolov6", "n", {}, "v6"), ("yolov6", "m", {}, "v6"), ("yolov5", "n", {}, "v5"), ("yolov7", "tiny", {}, "v5"),
                ("yolov7", "w6", dict(in_h=256, in_w=256), "v5")]


@pytest.mark.parametrize("kind,scale,kw,layout", DECODE_CASES, ids=[f"{c[0]}-{c[1]}" for c in DECODE_CASES])
def test_head_decode_matches_float64_reference(tmp_path, kind, scale, kw, layout):
    """The engine's raw output against a float64 decode of its own f32 head buffers, per element, within the bound derived from the
    kernel's float32 arithmetic (post_conformance_cases.py).  Also: run(1) after a batch-2 run gives frame 0's bits."""
    path, pb = _plan(tmp_path, kind, scale, **kw)
    eng = _capi.Engine(path, 0, max_batch=2)
    nc, reg_max = pb.meta[0], (pb.meta[2] if layout == "v6" else 16)
    in_h, in_w = eng.input_shape[2], eng.input_shape[3]
    x = np.concatenate([post.yolo_prepare_input(synth.frame(s), in_h, in_w)[0] for s in (0, 1)])
    raw = eng.infer(x)[0]
    levels = []
    for buf, _, C, st in pb.outputs:
        H, W = pb.buffers[buf][3], pb.buffers[buf][4]
        levels.append((eng.read_buffer(buf, 2).reshape(2, H + 2, W + 2, C)[:, 1:-1, 1:-1].copy(), st))
    anchors = plan.read_anchors(path) if layout == "v5" else None
    ref, bnd = pc.decode_reference(layout, levels, nc, reg_max, anchors)
    assert raw.shape == ref.shape, (raw.shape, ref.shape)
    ex, worst = pc.decode_excess(raw, ref, bnd)
    print(f"[decode] {kind}-{scale} {in_h}x{in_w} {layout} reg_max {reg_max} levels {len(levels)}: max err {worst:.2e}, "
          f"max err / bound {ex:.3f}")
    assert ex <= 1.0
    one = eng.infer(x[:1])[0]
    assert np.array_equal(one[0], raw[0])
    eng.close()


def _check_frame(res, b, r):
    boxes, scores, cls, idx, counts, ncand = res
    n = int(counts[b])
    assert int(ncand[b]) == r["n_cand"], (b, int(ncand[b]), r["n_cand"])
    assert n == len(r["idx"]), b
    assert np.array_equal(idx[b, :n], r["idx"]), b
    assert np.array_equal(boxes[b, :n], r["boxes"]), b
    assert np.array_equal(scores[b, :n], r["scores"]), b
    assert np.array_equal(cls[b, :n], r["cls"]), b


def _identity_head_plan(tmp_path, kind, in_h=64, in_w=96, nc=16, reg_max=16):
    """A plan whose three head levels are 1 x 1 identity convs (fp16 in, f32 out, zero bias: exact) of fp16 buffers the test writes,
    so the decode sees exactly the logits the test chooses.  -> (path, [(input view, head view, stride)])"""
    cc = 64 if kind == "v8" else (4 * (reg_max + 1) + 7) // 8 * 8
    C = (cc + nc + 7) // 8 * 8
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8 if kind == "v8" else plan.MODEL_YOLOV6, 3, in_h, in_w)
    levels, A = [], 0
    for st in (8, 16, 32):
        H, W = in_h // st, in_w // st
        x = pb.new_padded(H, W, C)
        head = pb.new_padded(H, W, C, f32=True)
        pb.conv(x, np.eye(C, dtype=np.float32).reshape(C, C, 1, 1), np.zeros(C, np.float32), 1, 1, plan.ACT_NONE, out=head, out_f32=True)
        pb.outputs.append((head.buf, 0, C, st))
        levels.append((x, head, st))
        A += H * W
    pb.meta[0], pb.meta[1], pb.meta[2] = nc, A, (0 if kind == "v8" else reg_max)
    path = str(tmp_path / f"identity_head_{kind}.b200w")
    pb.write(path)
    return path, levels, C


def _padded(g, fill=0.0):
    """[B, H, W, C] -> [B * (H + 2) * (W + 2), C] fp16 with the halo ring set to `fill`"""
    B, H, W, C = g.shape
    out = np.full((B, H + 2, W + 2, C), fill, np.float16)
    out[:, 1:-1, 1:-1] = g.astype(np.float16)
    return out.reshape(-1, C)


@pytest.mark.parametrize("kind", ["v8", "v6"])
def test_head_decode_crafted_logits_and_nan_halo(tmp_path, kind):
    """Logits the seeded weights never produce -- class logits of +-30, +-88 .. +-104 (the sigmoid saturates to exactly 1.0f, or expf(-z)
    overflows and the probability underflows), all-equal DFL bins, one dominant bin at 0 or at the last bin, bins whose expf after the
    max subtraction is subnormal or 0, bins near the fp16 range -- decoded on the device and compared per element with the float64
    reference under the same bounds.  Then NaN in the halo ring of every head level (and of the conv inputs) must not reach the raw
    output: it stays finite and bit-identical to the clean run."""
    nc, reg_max = 16, 16
    path, levels, C = _identity_head_plan(tmp_path, kind, nc=nc, reg_max=reg_max)
    eng = _capi.Engine(path, 0, max_batch=2)
    grids = []
    for li, (x, head, st) in enumerate(levels):
        g = pc.crafted_head(40 + li, kind, x.H, x.W, C, nc, reg_max)
        eng.write_buffer(x.buf, _padded(g))
        grids.append((g, st))
    img = np.zeros((2, 3, 64, 96), np.float32)
    raw = eng.infer(img)[0]
    ref, bnd = pc.decode_reference(kind, grids, nc, reg_max)
    assert raw.shape == ref.shape, (raw.shape, ref.shape)
    ex, worst = pc.decode_excess(raw, ref, bnd)
    probs = raw[:, 4:] if kind == "v8" else raw[..., 5:]
    print(f"[decode] crafted {kind}: max err {worst:.2e}, max err / bound {ex:.3f}, probabilities == 1.0f: {int((probs == 1).sum())}, "
          f"== 0: {int((probs == 0).sum())}")
    assert ex <= 1.0
    assert (probs == 1.0).any() and (probs == 0.0).any() and (probs[probs > 0] < pc.FLT_MIN).any()
    # NaN halo: poison the ring of the conv inputs and of the head buffers, run again
    for (x, head, st), (g, _) in zip(levels, grids):
        eng.write_buffer(x.buf, _padded(g, np.nan))
        hb = eng.read_buffer(head.buf, 2).reshape(2, x.H + 2, x.W + 2, C)
        hb[:, 0], hb[:, -1], hb[:, :, 0], hb[:, :, -1] = np.nan, np.nan, np.nan, np.nan
        eng.write_buffer(head.buf, hb.reshape(-1, C))
    again = eng.infer(img)[0]
    for x, head, st in levels:
        hb = eng.read_buffer(head.buf, 2).reshape(2, x.H + 2, x.W + 2, C)
        assert np.isnan(hb[:, 0]).all() and np.isnan(hb[:, :, -1]).all()        # the decode really ran next to a NaN halo
        assert not np.isnan(hb[:, 1:-1, 1:-1]).any()
    assert np.isfinite(again).all() and np.array_equal(again.view(np.uint32), raw.view(np.uint32))
    eng.close()


def test_lite_post_non_square_bit_exact():
    """lite_postprocess on the device at a non-square input (the reference's `r % h` grid) equals the oracle bit for bit"""
    rng = np.random.default_rng(5)
    in_hw = (256, 384)
    A = 3 * sum((in_hw[0] // s) * (in_hw[1] // s) for s in (8, 16, 32))
    raw = rng.uniform(0, 1, (2, A, 85)).astype(np.float32)
    raw[:, :, 4] = rng.uniform(0.8, 1.0, (2, A))
    raw[:, :, 5:] = rng.uniform(0, 0.45, (2, A, 80))
    res = _capi.yolo_postprocess(raw, 3, 80, in_hw, in_hw, 0.4, 0.45, max_det=A)
    g = post.letterbox_geom(in_hw[0], in_hw[1], *in_hw)
    for b in range(2):
        r = post.yolo_postprocess(post.yolo_lite_postprocess(raw[b], in_hw), "v5", g, 0.4, 0.45)
        assert r["n_cand"] > 0
        _check_frame(res, b, r)


# ---- 2. selection + NMS at every size -------------------------------------------------------------------------------------------
def test_v8_selection_and_nms_both_routes_in_one_launch():
    """Candidate totals 2047 / 2048 (shared-memory NMS working set) and 2049 / 5000 / 8400 (global working set) in ONE batch, so one
    launch runs both routes; every frame equals the oracle bit for bit."""
    hits = (2047, 2048, 2049, 5000, 8400)
    raw = np.stack([pc.v8_selection_raw(h, h) for h in hits])
    res = _capi.yolo_postprocess(raw, 0, 80, (640, 640), (720, 1280), 0.4, 0.45, max_det=8400)
    g = post.letterbox_geom(720, 1280, 640, 640)
    print(f"[nms] candidates per frame {res[5].tolist()}, survivors {res[4].tolist()}")
    assert res[5].min() <= 2048 < res[5].max()
    for b in range(len(hits)):
        _check_frame(res, b, post.yolo_postprocess(raw[b], "v8", g, 0.4, 0.45))


def test_v5_layout_selection_and_nms_25200_and_102000_anchors():
    g = post.letterbox_geom(720, 1280, 640, 640)
    raw = np.stack([pc.v5_selection_raw(s, h) for s, h in ((1, 2600), (2, 1500))])
    res = _capi.yolo_postprocess(raw, 1, 80, (640, 640), (720, 1280), 0.4, 0.45, max_det=4096)
    assert res[5][0] > 2048 >= res[5][1]
    for b in range(2):
        _check_frame(res, b, post.yolo_postprocess(raw[b], "v5", g, 0.4, 0.45))
    raw6 = pc.v5_selection_raw(3, 3000, A=102000, in_hw=(1280, 1280))[None]
    g6 = post.letterbox_geom(720, 1280, 1280, 1280)
    res6 = _capi.yolo_postprocess(raw6, 1, 80, (1280, 1280), (720, 1280), 0.4, 0.45, max_det=4096)
    assert res6[5][0] == 3000
    _check_frame(res6, 0, post.yolo_postprocess(raw6[0], "v5", g6, 0.4, 0.45))


def test_selection_and_nms_ties_and_degenerate_boxes():
    """confs of exactly 1.0f (first-maximum argmax and the swap), identical boxes, class ties inside an anchor, confs at box_score and
    one ulp either side (strict compare), zero-area and sub-pixel boxes (the +1 area convention)"""
    bs = float(np.float32(0.45))
    raw, n = pc.v8_tie_raw(3, bs)
    raw2, n2 = pc.v8_tie_raw(4, bs)
    res = _capi.yolo_postprocess(np.stack([raw, raw2]), 0, 80, (640, 640), (640, 640), bs, 0.5, max_det=4096)
    g = post.letterbox_geom(640, 640, 640, 640)
    assert res[5].tolist() == [n, n2]
    for b, r in enumerate((raw, raw2)):
        _check_frame(res, b, post.yolo_postprocess(r, "v8", g, bs, 0.5))


def test_more_survivors_than_max_det_raises_and_engine_recovers():
    path, _, _ = cached_plan("yolov5", scale="n")
    eng = _capi.Engine(path, 0, max_batch=2)
    frames = np.stack([synth.frame(s) for s in (0, 1)])
    want = eng.yolo_detect(frames, 0.4, 0.45)
    assert want[4].max() >= 2
    with pytest.raises(Exception, match=r"detections survive the NMS but the output arrays hold 1 \(raise max_det\)"):
        eng.yolo_detect(frames, 0.4, 0.45, max_det=1)
    got = eng.yolo_detect(frames, 0.4, 0.45)
    assert np.array_equal(got[4], want[4]) and np.array_equal(got[5], want[5])          # counts, candidate totals
    for b in range(2):
        n = int(want[4][b])
        for k in range(4):                                                                 # boxes, scores, classes, indices
            assert np.array_equal(got[k][b, :n], want[k][b, :n]), (b, k)
    eng.close()


# ---- 3. association and tracker at crowd scale ----------------------------------------------------------------------------------
@pytest.mark.parametrize("T,D", [(121, 121), (500, 700), (1024, 1024), (1, 2047)])
@pytest.mark.parametrize("sparse", [False, True])
def test_lap_large_problems_match_exact_optimum(T, D, sparse):
    cost = pc.lap_cost(T * 7 + D, T, D, sparse)
    (x, y), = _capi.lap([cost], [0.8])
    ox, oy, tot = post.lapjv_extended(cost, 0.8)
    m = x >= 0
    got = cost[np.nonzero(m)[0], x[m]].sum() + 0.4 * ((x < 0).sum() + (y < 0).sum())
    assert abs(got - tot) <= 1e-9
    assert np.array_equal(x, ox) and np.array_equal(y, oy)           # continuous costs: the optimum is unique


def test_lap_refuses_problems_beyond_its_limits():
    with pytest.raises(Exception, match="too large"):
        _capi.lap([np.ones((1025, 1))], [0.8])
    with pytest.raises(Exception, match="too large"):
        _capi.lap([np.ones((1000, 1049))], [0.8])


def _compare_frame(recs, lost, want, want_lost, f):
    got = pc.native_rows(recs)
    assert got.shape == want.shape, (f, got.shape, want.shape)
    assert np.array_equal(got[:, :4], want[:, :4]), f                       # id, state, activation, class: exact
    assert np.allclose(got[:, 4:], want[:, 4:], rtol=0, atol=1e-6), f      # Kalman boxes (fp64) and scores
    assert sorted(lost["track_id"].tolist()) == sorted(want_lost), f


def test_native_tracker_crowd_matches_oracle_past_shared_memory_routes():
    seq = pc.crowd_sequence(7, objects=300, frames=64, clutter=150)
    want, pmax, umax, nrem = pc.run_oracle(track.Tracker, seq)
    print(f"[track] max pool {pmax}, max unconfirmed {umax}, removed {nrem}")
    assert pmax > 120 and umax > 120 and nrem > 4096
    nt = _capi.NativeTracker(0)
    nt.reset()
    for f, (b, s, c) in enumerate(seq):
        recs = nt.update(b, s, c)
        _compare_frame(recs, nt.get(1), *want[f], f)
    nt.close()


def test_native_tracker_update_batch_ragged_at_crowd_scale():
    seq = pc.crowd_sequence(8, objects=250, frames=40, clutter=130)
    e = (np.zeros((0, 4)), np.zeros(0), np.zeros(0, np.int32))
    seq = seq[:5] + [e] + seq[5:20] + [e, e] + seq[20:]
    want, pmax, umax, _ = pc.run_oracle(track.Tracker, seq)
    assert pmax > 120 and umax > 120
    nt = _capi.NativeTracker(0)
    nt.reset()
    f = 0
    for i, k in enumerate((3, 8, 1, 8, 8, 8, 7)):
        chunk = seq[f:f + k]
        recs = nt.update_batch([len(s) for _, s, _ in chunk], np.concatenate([b for b, _, _ in chunk]).reshape(-1, 4),
                               np.concatenate([s for _, s, _ in chunk]), np.concatenate([c for _, _, c in chunk]))
        for j, r in enumerate(recs):
            got, w = pc.native_rows(r), want[f + j][0]
            assert got.shape == w.shape and np.array_equal(got[:, :4], w[:, :4]), f + j
            assert np.allclose(got[:, 4:], w[:, 4:], rtol=0, atol=1e-6), f + j
        f += k
    assert f == len(seq)
    nt.close()


def test_native_tracker_pool_past_1024_keeps_working_on_empty_frames():
    """1100 confirmed tracks (first frame), an association of 1100 tracks x 1400 detections, then 35 empty frames: the tracks go lost,
    age out and are removed, and the tracker keeps matching the oracle -- before, a pool over 1024 refused every later frame."""
    a = pc.grid_boxes(1100)
    new = pc.grid_boxes(300, y0=5000.0)
    e = (np.zeros((0, 4)), np.zeros(0), np.zeros(0, np.int32))
    seq = [(a, np.full(1100, 0.9), np.zeros(1100, np.int32)),
           (np.concatenate([a + 1.5, new]), np.full(1400, 0.9), np.zeros(1400, np.int32))] + [e] * 35 + \
          [(new + 3.0, np.full(300, 0.8), np.ones(300, np.int32))]
    want, pmax, _, _ = pc.run_oracle(track.Tracker, seq)
    assert pmax > 1024
    nt = _capi.NativeTracker(0)
    nt.reset()
    for f, (b, s, c) in enumerate(seq):
        recs = nt.update(b, s, c)
        _compare_frame(recs, nt.get(1), *want[f], f)
    assert len(nt.get(1)) == 0 and len(nt.get(0)) == 300
    nt.close()


def test_native_tracker_removed_trim_keeps_tracks_removed_this_frame():
    """2100 confirmed tracks go lost together and age out in ONE frame, while the removed list already holds 2000 unconfirmed tracks:
    4100 > 4096 entries, so the removed list is trimmed on that frame.  The trim must not drop the 2100 tracks removed on that frame --
    the next frame's sub(lost, removed) is what takes them out of the lost list; the lost lists must equal the oracle's throughout."""
    a = pc.grid_boxes(2100)
    e = (np.zeros((0, 4)), np.zeros(0), np.zeros(0, np.int32))
    seq = [(a, np.full(2100, 0.9), np.zeros(2100, np.int32))]
    for k in range(4):                                   # 4 x 500 one-frame births, each removed unconfirmed on the next frame
        seq.append((pc.grid_boxes(500, y0=10000.0 + 3000.0 * k), np.full(500, 0.9), np.ones(500, np.int32)))
    seq += [e] * 30
    want, _, _, nrem = pc.run_oracle(track.Tracker, seq)
    assert nrem == 6200           # 2000 unconfirmed + 2100 aged out, which the reference lists again on the next frame
    nt = _capi.NativeTracker(0)
    nt.reset()
    for f, (b, s, c) in enumerate(seq):
        recs = nt.update(b, s, c)
        _compare_frame(recs, nt.get(1), *want[f], f)
    assert len(want[-1][1]) == 0 and len(nt.get(1)) == 0
    nt.close()


def _oracle_rows(seq):
    """oracle tracked rows per frame (the class column holds the label the frames carry)"""
    return [w for w, _ in pc.run_oracle(track.Tracker, seq)[0]]


def _assert_records(recs, want, labels, f):
    got = pc.native_rows(recs)
    got[:, 3] = [labels[int(c)] for c in got[:, 3]]
    assert got.shape == want.shape, (f, got.shape, want.shape)
    assert np.array_equal(got[:, :4], want[:, :4]), f
    assert np.allclose(got[:, 4:], want[:, 4:], rtol=0, atol=1e-6), f


def test_bytetracker_update_batch_more_than_256_live_tracks():
    """BYTETracker.update_batch / update_batch_arrays (the pipeline's path) return every record with 300+ live tracks, and frame_id
    stays in step with the native tracker -- before, more than 256 tracks raised after the native tracker had advanced."""
    from adas_b200.ObjectTracker import BYTETracker
    trk = BYTETracker(names=[])
    trk.reset()
    a = pc.grid_boxes(300)
    cls = np.arange(300) % 3 + 7                                  # labels 7, 8, 9 -> the tracker's class slots 0, 1, 2
    seq = [(a + f, np.full(300, 0.9), cls) for f in range(4)] + [(a + 4, np.full(300, 0.9), cls), (np.zeros((0, 4)), np.zeros(0), cls[:0]),
                                                                 (a + 6, np.full(300, 0.9), cls)]
    want = _oracle_rows(seq)
    recs = trk.update_batch(seq[:4])
    assert [len(r) for r in recs] == [300] * 4 and trk.frame_id == 4 == int(recs[-1]["frame_id"].max())
    counts = np.array([300, 0, 300], np.int32)
    recs += trk.update_batch_arrays(counts, np.concatenate([seq[4][0], seq[6][0]]), np.full(600, 0.9), np.concatenate([cls, cls]))
    assert [len(r) for r in recs] == [300, 300, 300, 300, 300, 0, 300] and trk.frame_id == 7 == int(recs[-1]["frame_id"].max())
    for f, r in enumerate(recs):
        _assert_records(r, want[f], trk._label_list, f)
    assert len(trk.tracked_stracks) == 300


def test_pipeline_tracker_stage_more_than_256_live_tracks():
    """AdasPipeline's tracker stage on steps whose frames carry 300 detections: every frame's records equal the oracle's on the same
    (integer-truncated) boxes, and the tracker's frame_id follows the frames fed -- before, the step raised once more than 256 tracks
    were live, after the native tracker had advanced."""
    from adas_b200.pipeline import AdasPipeline, StepResult
    ypath, _, _ = cached_plan("yolov8", scale="n")
    upath, _, _ = cached_plan("ufldv2", backbone="18")
    pipe = AdasPipeline(ypath, upath, batch=4, sets=1, depth=1)
    B, max_det, n = 4, 1024, 300
    a = pc.grid_boxes(n) + 0.4                                     # fractional corners: the pipeline truncates xyxy to integers
    cls = (np.arange(n) % 2).astype(np.int32)
    seq, k = [], 0
    for step in range(2):
        boxes = np.zeros((B, max_det, 4), np.float32)
        scores = np.zeros((B, max_det), np.float32)
        ids = np.zeros((B, max_det), np.int32)
        counts = np.array([n, n, 0, n] if step == 1 else [n] * B, np.int32)
        for f in range(B):
            c = int(counts[f])
            xy = (a[:c] + 2.0 * k).astype(np.float32)
            boxes[f, :c, :2], boxes[f, :c, 2:] = xy[:, :2], xy[:, 2:] - xy[:, :2]
            scores[f, :c] = np.float32(0.9)
            ids[f, :c] = cls[:c]
            bx = boxes[f, :c]
            xyxy = np.stack([bx[:, 0], bx[:, 1], bx[:, 0] + bx[:, 2], bx[:, 1] + bx[:, 3]], 1).astype(np.int64).astype(np.float64)
            seq.append((xyxy, scores[f, :c].astype(np.float64), ids[f, :c]))
            k += 1
        r = StepResult((boxes, scores, ids, np.zeros((B, max_det), np.int32), counts, counts.copy()),
                       (np.zeros((B, 4, 1, 2), np.int32), np.zeros((B, 4), np.int32), np.zeros((B, 4), np.uint8), None))
        pipe._track(r)
        assert len(r.tracks) == B and pipe.tracker.frame_id == B * (step + 1)
        want = _oracle_rows(seq)
        for f in range(B):
            _assert_records(r.tracks[f], want[B * step + f], pipe.tracker._label_list, B * step + f)
    assert max(len(t) for t in r.tracks) == n
    pipe.close()
