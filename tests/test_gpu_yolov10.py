"""GPU: YOLOv10 on the device -- the depthwise conv (OP_DWCONV) and PSA attention (OP_ATTN) kernels against torch, the v10 blocks
against the oracle's modules, and YOLOv10-N/S/M/B/L/X end to end against the fp32 oracle (tests/yolov10_oracle.py) through YOLOv8's head
decode, candidate selection and NMS."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import synth
import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
from gpu_util import cached_plan, from_padded, halo_is_zero, to_padded, yolo_blob
from oracle import post
import yolov10_oracle as o10

pytestmark = pytest.mark.gpu
torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))


def _h(a: np.ndarray) -> np.ndarray:
    return a.astype(np.float16).astype(np.float32)


@pytest.mark.parametrize("H,W", [(20, 20), (13, 13), (10, 26), (7, 4)])
@pytest.mark.parametrize("k,s", [(3, 1), (3, 2), (7, 1)])
@pytest.mark.parametrize("act,with_res", [(plan.ACT_NONE, False), (plan.ACT_SILU, True), (plan.ACT_SILU, False)])
def test_dwconv_matches_torch_on_concat_slices(tmp_path, H, W, k, s, act, with_res):
    """Channels [16, 16 + C) of a 64-channel input into channels [8, 8 + C) of a 48-channel output (+ channels [24, 24 + C) of a residual
    buffer); every other channel and the halo stay zero."""
    B, C, ci, co, cr = 2, 24, 16, 8, 24
    rng = np.random.default_rng(H * 100 + W + 7 * k + s + act)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    xin = pb.new_padded(H, W, 64)
    out = pb.new_padded(Ho, Wo, 48)
    rb = pb.new_padded(Ho, Wo, 56) if with_res else None
    w = (rng.standard_normal((C, 1, k, k)) / k).astype(np.float32)
    b = (rng.standard_normal(C) * 0.1).astype(np.float32)
    pb.dwconv(pb.sub(xin, ci, C), w, b, k, s, act, out=pb.sub(out, co, C), res=pb.sub(rb, cr, C) if with_res else None)
    path = str(tmp_path / "dw.b200w")
    pb.write(path)
    x = (rng.standard_normal((B, 64, H, W)) * 2).astype(np.float32)
    r = rng.standard_normal((B, 56, Ho, Wo)).astype(np.float32)
    eng = _capi.Engine(path, device=0, max_batch=B)
    eng.write_buffer(xin.buf, to_padded(x, 64))
    if with_res:
        eng.write_buffer(rb.buf, to_padded(r, 56))
    eng.run(B)
    buf = eng.read_buffer(out.buf, B).copy()
    eng.close()
    got = from_padded(buf, B, Ho, Wo, co, C)
    with torch.no_grad():
        ref = F.conv2d(torch.from_numpy(_h(x[:, ci:ci + C])), torch.from_numpy(_h(w)), torch.from_numpy(b), s, k // 2, groups=C)
        ref = F.silu(ref) if act == plan.ACT_SILU else ref
        ref = (ref + torch.from_numpy(_h(r[:, cr:cr + C]))) if with_res else ref
    ref = ref.numpy()
    assert got.shape == ref.shape
    tol = np.spacing(np.abs(ref).astype(np.float16)).astype(np.float32) + 1e-4 * max(1.0, float(np.abs(ref).max()))
    assert np.all(np.abs(got - ref) <= tol), float(np.abs(got - ref).max())
    assert halo_is_zero(buf, B, Ho, Wo), "dwconv wrote into the zero halo"
    v = buf.reshape(B, Ho + 2, Wo + 2, -1).astype(np.float32)
    assert not v[..., :co].any() and not v[..., co + C:].any(), "dwconv wrote outside its channel slice"


def _attn_ref(q, k, v, scale):
    """q, k [B, nh, kd, N], v [B, nh, hd, N] fp32 -> [B, nh * hd, N] (upstream's (v @ attn^T) order)"""
    a = ((q.transpose(-2, -1) @ k) * scale).softmax(-1)
    return (v @ a.transpose(-2, -1)).reshape(q.shape[0], -1, q.shape[-1])


@pytest.mark.parametrize("HW", [(20, 20), (15, 20), (40, 40), (9, 7)])
@pytest.mark.parametrize("nh,kd,hd", [(2, 32, 64), (4, 36, 72), (5, 32, 64)])
def test_attention_matches_torch(tmp_path, HW, nh, kd, hd):
    """N = 400, 300, 1600 and 63 (not a multiple of the 64-key tile); 2e-3 of max |ref|; repeatable and batch-invariant."""
    H, W = HW
    N, B = H * W, 3
    kdp = (kd + 15) // 16 * 16
    cin, coff = nh * (2 * kdp + hd), 8
    rng = np.random.default_rng(N + nh)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    xin = pb.new_padded(H, W, cin + 16)
    out = pb.new_padded(H, W, nh * hd + 8)
    pb.attention(pb.sub(xin, coff, cin), nh, kdp, hd, kd ** -0.5, out=pb.sub(out, 8, nh * hd))
    path = str(tmp_path / "at.b200w")
    pb.write(path)
    q = _h(rng.standard_normal((B, nh, kd, N)) * 1.5)
    k = _h(rng.standard_normal((B, nh, kd, N)) * 1.5)
    v = _h(rng.standard_normal((B, nh, hd, N)))
    x = np.zeros((B, cin + 16, N), np.float32)
    for h in range(nh):
        x[:, coff + h * kdp:coff + h * kdp + kd] = q[:, h]
        x[:, coff + (nh + h) * kdp:coff + (nh + h) * kdp + kd] = k[:, h]
    x[:, coff + 2 * nh * kdp:coff + cin] = v.reshape(B, nh * hd, N)
    x[:, coff + cin:] = 7.0                                           # channels past the slice are not read
    eng = _capi.Engine(path, device=0, max_batch=B)
    eng.write_buffer(xin.buf, to_padded(x.reshape(B, -1, H, W), cin + 16))
    eng.run(B)
    buf = eng.read_buffer(out.buf, B).copy()
    eng.run(B)
    again = eng.read_buffer(out.buf, B).copy()
    eng.write_buffer(xin.buf, to_padded(x[1:2].reshape(1, -1, H, W), cin + 16))
    eng.run(1)
    one = eng.read_buffer(out.buf, 1).copy()
    eng.close()
    got = from_padded(buf, B, H, W, 8, nh * hd).reshape(B, nh * hd, N)
    with torch.no_grad():
        ref = _attn_ref(torch.from_numpy(q), torch.from_numpy(k), torch.from_numpy(v), kd ** -0.5).numpy()
    err = float(np.abs(got - ref).max()) / float(np.abs(ref).max())
    print(f"[attn] N={N} nh={nh} kd={kd} hd={hd}: err {err:.2e} of max |ref|")
    assert err <= 2e-3
    assert np.array_equal(buf, again), "two runs differ"
    rows = (H + 2) * (W + 2)
    assert np.array_equal(one[:rows], buf[rows:2 * rows]), "batch-1 result differs from the same image in a batch of 3"
    assert halo_is_zero(buf, B, H, W)
    vv = buf.reshape(B, H + 2, W + 2, -1)
    assert not vv[..., :8].astype(np.float32).any()


def _block(block):
    """the oracle block in eval mode with randomised BatchNorm statistics"""
    for m in block.modules():
        if isinstance(m, o10.Conv):
            with torch.no_grad():
                m.bn.running_mean.uniform_(-0.1, 0.1)
                m.bn.running_var.uniform_(0.8, 1.2)
                m.bn.weight.uniform_(0.8, 1.2)
                m.bn.bias.uniform_(-0.1, 0.1)
    return block.eval()


BLOCKS = [("scdown", 64, 128, 40, 40), ("scdown", 128, 128, 13, 10), ("cib", 64, 64, 20, 20), ("cib_lk", 64, 64, 20, 20),
          ("c2fcib", 128, 128, 20, 20), ("c2fcib_lk", 256, 256, 20, 14), ("psa", 256, 256, 20, 20), ("psa", 576, 576, 20, 20),
          ("psa", 640, 640, 15, 20)]


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("kind,c1,c2,H,W", BLOCKS)
def test_v10_blocks_match_the_oracle(tmp_path, impl, kind, c1, c2, H, W):
    torch.manual_seed(c1 + c2 + H)
    mk = {"scdown": lambda: o10.SCDown(c1, c2), "cib": lambda: o10.CIB(c1, True, False), "cib_lk": lambda: o10.CIB(c1, True, True),
          "c2fcib": lambda: o10.C2f(c1, c2, 2, True, False), "c2fcib_lk": lambda: o10.C2f(c1, c2, 1, True, True),
          "psa": lambda: o10.PSA(c1)}[kind]
    block = _block(mk())
    sd = {f"model.5.{k}": v.numpy() for k, v in block.state_dict().items()}
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    g = plan.Yolov10Packer(pb, plan.Weights(sd))
    xin = pb.new_padded(H, W, c1)
    if kind == "scdown":
        out = g.scdown(xin, "model.5", c2)
    elif kind.startswith("cib"):
        out = g.cib(xin, "model.5", c1, True, kind.endswith("lk"))
    elif kind.startswith("c2fcib"):
        out = g.c2f(xin, "model.5", c2, 2 if kind == "c2fcib" else 1, True, kind.endswith("lk"))
    else:
        out = g.psa(xin, "model.5")
    path = str(tmp_path / f"{kind}.b200w")
    pb.write(path)
    B = 2
    x = np.random.default_rng(c1).standard_normal((B, c1, H, W)).astype(np.float32)
    eng = _capi.Engine(path, device=0, max_batch=B, conv_impl=impl)
    eng.write_buffer(xin.buf, to_padded(x, c1))
    eng.run(B)
    buf = eng.read_buffer(out.buf, B).copy()
    eng.close()
    got = from_padded(buf, B, out.H, out.W, out.coff, c2)
    with torch.no_grad():
        ref = block(torch.from_numpy(_h(x))).numpy()
    assert ref.shape == got.shape
    err = np.abs(got - ref) / max(1.0, float(np.abs(ref).max()))
    print(f"[block] {kind} {c1} {H}x{W} impl{impl}: {err.max():.2e}")
    assert err.max() < 3e-3, (kind, impl, float(err.max()))


@pytest.mark.parametrize("nc", [80, 70])
def test_v10_head_matches_the_oracle(tmp_path, nc):
    """The one-to-one head (box branch, depthwise class branch) on three 64 / 128 / 256-channel maps.  With nc = 70 the class branch
    is c3 = 70 channels wide, stored as 72 with zero channels behind it."""
    torch.manual_seed(nc)
    det = _block(o10.V10Detect(nc, (64, 128, 256)))
    sd = {f"model.23.{k}": v.numpy() for k, v in det.state_dict().items()}
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 320, 320)
    feats = [pb.new_padded(320 // s, 320 // s, c) for s, c in ((8, 64), (16, 128), (32, 256))]
    A = plan.v10_detect(pb, plan.Yolov10Packer(pb, plan.Weights(sd)), "model.23", feats, nc)
    pb.meta[0], pb.meta[1] = nc, A
    path = str(tmp_path / "head.b200w")
    pb.write(path)
    rng = np.random.default_rng(1)
    xs = [rng.standard_normal((2, f.C, f.H, f.W)).astype(np.float32) for f in feats]
    eng = _capi.Engine(path, device=0, max_batch=2)
    for f, x in zip(feats, xs):
        eng.write_buffer(f.buf, to_padded(x, f.C))
    eng.run(2)
    heads = [eng.read_buffer(o[0], 2).copy() for o in pb.outputs]
    eng.close()
    with torch.no_grad():
        for li, (f, x) in enumerate(zip(feats, xs)):
            t = torch.from_numpy(_h(x))
            ref = torch.cat((det.one2one_cv2[li](t), det.one2one_cv3[li](t)), 1).numpy()
            got = from_padded(heads[li], 2, f.H, f.W, 0, 64 + nc)
            err = np.abs(got - ref).max() / max(1.0, float(np.abs(ref).max()))
            assert err < 3e-3, (li, float(err))


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("scale", ["n", "s", "m", "b", "l", "x"])
def test_yolov10_engine_vs_oracle_and_batch_invariance(scale, impl):
    path, sd, _ = cached_plan("yolov10", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=3, conv_impl=impl)
    x = yolo_blob([synth.frame(s) for s in (0, 1, 2)])
    raw = eng.infer(x)[0]
    with torch.no_grad():
        ref = o10.build(sd, scale)(torch.from_numpy(x[:2])).numpy()
    assert raw.shape == (3, 84, 8400)
    e_prob = float(np.abs(raw[:2, 4:] - ref[:, 4:]).max())
    e_box = float(np.abs(raw[:2, :4] - ref[:, :4]).max())
    print(f"[parity] yolov10-{scale} impl{impl}: prob {e_prob:.2e}, box {e_box:.3f} px")
    assert e_prob < 1e-3
    assert e_box < 0.5
    raw1 = eng.infer(x[1:2])[0]
    assert np.array_equal(raw1[0], raw[1]), "batch-1 frame differs from the same frame in a batch of 3"
    eng.close()


@pytest.mark.parametrize("in_h,in_w", [(1280, 1280), (480, 640)])
def test_yolov10n_at_other_input_sizes(in_h, in_w):
    """1600 attention tokens at 1280x1280; a non-square 640x480 letterbox."""
    path, sd, _ = cached_plan("yolov10", scale="n", in_h=in_h, in_w=in_w)
    eng = _capi.Engine(path, 0, max_batch=2)
    x = yolo_blob([synth.frame(s) for s in (0, 1)], in_h, in_w)
    raw = eng.infer(x)[0]
    eng.close()
    with torch.no_grad():
        ref = o10.build(sd, "n")(torch.from_numpy(x)).numpy()
    A = sum((in_h // s) * (in_w // s) for s in (8, 16, 32))
    assert raw.shape == (2, 84, A) == ref.shape
    e_prob = float(np.abs(raw[:, 4:] - ref[:, 4:]).max())
    e_box = float(np.abs(raw[:, :4] - ref[:, :4]).max())
    print(f"[parity] yolov10-n {in_h}x{in_w}: prob {e_prob:.2e}, box {e_box:.3f} px")
    assert e_prob < 1e-3 and e_box < 0.5


@pytest.mark.parametrize("scale", ["n", "m"])
def test_yolov10_fused_detect_matches_reference_postprocessing(scale):
    """The device decode + candidate selection + NMS equals the reference's v8 host post-processing of the engine's own output."""
    path, _, _ = cached_plan("yolov10", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=2)
    frames = np.stack([synth.frame(s) for s in (4, 5)])
    total = 0
    for score in (0.4, 0.05):
        boxes, scores, cls, idx, counts, ncand = eng.yolo_detect(frames, score, 0.45, max_det=8400)
        raw = eng.infer(_capi.yolo_preprocess(frames, (640, 640)))[0]
        geom = post.letterbox_geom(720, 1280, 640, 640)
        for b in range(2):
            r = post.yolo_postprocess(raw[b], "v8", geom, score, 0.45)
            n = int(counts[b])
            total += n
            assert ncand[b] == r["n_cand"] and np.array_equal(idx[b, :n], r["idx"]) and np.array_equal(boxes[b, :n], r["boxes"])
            assert np.array_equal(scores[b, :n], r["scores"]) and np.array_equal(cls[b, :n], r["cls"])
        print(f"[detect] yolov10-{scale} score {score}: candidates {ncand.tolist()}, detections {counts.tolist()}")
    assert total > 0
    eng.close()


@pytest.mark.parametrize("scale", ["n", "s", "m", "b", "l", "x"])
def test_yolov10_candidate_sets_follow_the_margin_rule(scale):
    """Candidates (max class probability > 0.4) agree with the fp32 oracle's wherever the oracle's score is more than 1e-3 from the
    threshold, and within 1e-3 of it where they do not."""
    path, sd, _ = cached_plan("yolov10", scale=scale)
    eng = _capi.Engine(path, 0, max_batch=4)
    x = yolo_blob([synth.frame(s) for s in (4, 5, 6, 7)])
    raw = eng.infer(x)[0]
    eng.close()
    with torch.no_grad():
        ref = o10.build(sd, scale)(torch.from_numpy(x)).numpy()
    n_cand = n_margin = 0
    for b in range(4):
        mx_ref, mx_gpu = ref[b, 4:].max(0), raw[b, 4:].max(0)
        sure = np.abs(mx_ref - 0.4) > 1e-3
        cand = mx_ref > 0.4
        assert np.array_equal(cand[sure], (mx_gpu > 0.4)[sure])
        assert np.abs(mx_ref[cand] - mx_gpu[cand]).max(initial=0.0) < 1e-3
        n_cand += int(cand.sum())
        n_margin += int((~sure & (cand | (mx_gpu > 0.4))).sum())
    print(f"[margin] yolov10-{scale}: {n_cand} candidates over 4 frames, {n_margin} inside the 1e-3 margin")
    assert 100 <= n_cand <= 1600


def test_yolo_detector_runs_a_yolov10_onnx_file(tmp_path):
    """YoloDetector(ObjectModelType.YOLOV10) on an exported YOLOv10-N .onnx file: recognised, converted, loaded and decoded."""
    import test_onnx_import as toi
    from adas_b200.ObjectDetector import YoloDetector, ObjectModelType
    W = plan.synth_weights("yolov10", 0, variant="n")
    plan.build_yolov10(W, "n")
    onnx_path = str(tmp_path / "yolov10n.onnx")
    toi._export(o10.build(W.state_dict, "n").fuse(), (1, 3, 640, 640), onnx_path)
    os.environ["ADAS_B200_PLAN_CACHE"] = str(tmp_path / "cache")
    try:
        YoloDetector.set_defaults({"model_path": onnx_path, "model_type": ObjectModelType.YOLOV10, "classes_path": None, "box_score": 0.4,
                                   "box_nms_iou": 0.45})
        det = YoloDetector(logger=None, max_batch=2)
    finally:
        os.environ.pop("ADAS_B200_PLAN_CACHE", None)
    assert det.engine.handle.model_kind == plan.MODEL_YOLOV8
    out = det.engine.engine_inference(yolo_blob([synth.frame(3)]))
    assert out[0].shape == (1, 84, 8400)
    fr = [synth.frame(3), synth.frame(4)]
    det.DetectFrame(fr[0])
    single = [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in det.object_info]
    both = det.DetectFrames(fr)
    assert len(single) > 0 and single == [(r.x, r.y, r.width, r.height, r.conf, r.label) for r in both[0]]
