"""CPU: YOLOv6-Lite-S/M/L -- widths and parameter counts against the published figures, the oracle's fuse, the packer's folds against
the oracle, training-form and fused checkpoints packing one plan, the float64 plan interpreter against the oracle at 320 x 320 and at
inputs that are not multiples of 64, the plans' dataflow, the OP_SE / OP_SHUFFLE2 / activation / four-level head validators, and the
seeded plans of every other family staying byte-identical.

The graph restates upstream's configs (release 0.4.0); with no upstream file available, the published parameter counts are its anchor:
0.55 / 0.79 / 1.09 M for S / M / L.  The restatement has 0.558 / 0.791 / 1.099 M (DPBlock's convs carry a bias, as nn.Conv2d does by
default); the published figures are these truncated to two decimals (without the DPBlock biases M would have 0.788 M)."""
import hashlib

import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import plan
import plan_footprint as fp
import plan_interp as pi
import synth
import yolov6_lite_oracle as ol
from gpu_util import to_padded
from oracle import post

def _weights(scale, seed=0, **kw):
    W = plan.synth_weights("yolov6lite", seed, variant=scale)
    return W, plan.build_yolov6_lite(W, scale, **kw)


def test_widths_follow_the_upstream_rounding():
    out, mid, neck = plan.yolov6_lite_widths("s")
    assert out == [24, 32, 48, 96, 176] and mid[1:] == [16, 24, 48, 88] and neck == [176, 96, 48]
    halves = {sc: [m // 2 for m in plan.yolov6_lite_widths(sc)[1][1:]] for sc in "sml"}
    assert halves == {"s": [8, 12, 24, 44], "m": [8, 16, 36, 72], "l": [12, 24, 48, 96]}
    with pytest.raises(AssertionError, match="'s', 'm' or 'l'"):
        plan.yolov6_lite_widths("n")


@pytest.mark.parametrize("scale,params", [("s", 0.557942), ("m", 0.791381), ("l", 1.098789)])
def test_parameter_counts_match_the_published_figures(scale, params):
    n = sum(p.numel() for p in ol.YOLOv6Lite(scale).parameters())
    assert n == round(params * 1e6)
    assert int(n / 1e4) / 100 == plan.YOLOV6_LITE_PARAMS[scale] / 1e6          # published: truncated to two decimals


def test_plan_shape():
    W, pb = _weights("s")
    assert pb.model_kind == plan.MODEL_YOLOV6 and pb.meta[:3] == [80, 2125, 0]
    assert [s for _, _, _, s in pb.outputs] == [8, 16, 32, 64]
    kinds = [t for t, _, _ in pb.ops]
    n_s1 = sum(n - 1 for n in plan.YOLOV6_LITE_BLOCKS)
    assert kinds.count(plan.OP_SE) == n_s1 + 4 and kinds.count(plan.OP_SHUFFLE2) == n_s1
    assert kinds[0] == plan.OP_STEMCONV and pb.ops[0][1].Cout == 24 and pb.ops[0][1].act == plan.ACT_HSWISH
    dws = [p for t, p, _ in pb.ops if t == plan.OP_DWCONV]
    assert {(p.k, p.stride) for p in dws} == {(3, 1), (3, 2), (5, 1), (5, 2)}
    assert plan.OP_IM2COL not in kinds                                          # every conv is a 1x1 GEMM, a depthwise or the stem
    # SE hidden widths: C // 4 of the real (unpadded) widths, C padded to 8
    assert sorted({(p.C, p.hid) for t, p, _ in pb.ops if t == plan.OP_SE}) == [(8, 2), (16, 3), (24, 6), (48, 11), (48, 12), (88, 22)]


def test_oracle_fused_equals_training_form():
    W, _ = _weights("m", 1)
    x = torch.rand(2, 3, 320, 320)
    with torch.no_grad():
        a = ol.build(W.state_dict, "m")(x).numpy()
        b = ol.build(W.state_dict, "m").fuse()(x).numpy()
    assert a.shape == (2, 2125, 85)
    assert np.abs(a[..., 5:] - b[..., 5:]).max() < 1e-5
    assert np.abs(a[..., :4] - b[..., :4]).max() < 1e-3


def test_packer_folds_equal_oracle_fuse():
    """Every conv of the plan (GEMM, depthwise, stem) carries the oracle's fused conv: fp16 weights within half an fp16 ulp of it, fp32
    biases within 1e-6 relative."""
    W, pb = _weights("s", 2)
    fused = ol.build(W.state_dict, "s").fuse()
    convs = [m for m in fused.modules() if isinstance(m, torch.nn.Conv2d)]
    packed = []
    for t, p, _ in pb.ops:
        if t == plan.OP_DWCONV:
            C, k = p.C, p.k
            packed.append(("dw", pb.tensors[p.w_tensor].astype(np.float64).T.reshape(C, k, k), pb.tensors[p.bias_tensor]))
        elif t == plan.OP_STEMCONV:
            packed.append(("stem", pb.tensors[p.w_tensor][:, :, :12].astype(np.float64).reshape(24, 3, 3, 4)[..., :3].transpose(0, 3, 1, 2),
                           pb.tensors[p.bias_tensor]))
        elif t == plan.OP_GEMM:
            packed.append(("gemm", pb.tensors[p.w_tensor].astype(np.float64), pb.tensors[p.bias_tensor]))
    se = [m for m in fused.modules() if isinstance(m, ol.SEBlock)]
    assert len(packed) + 2 * len(se) == len(convs)
    # match each packed conv to the oracle conv of its bias (the head's box / class convs share a filled bias: then also by weights)
    by_bias = {}
    for c in convs:
        by_bias.setdefault(round(float(c.bias.detach()[0]), 6), []).append(c)

    def layout(kind, w, c):
        cw = c.weight.detach().numpy().astype(np.float64)
        n = c.out_channels
        if kind == "dw":
            return w[:n], cw[:, 0]
        if kind == "gemm":                                   # [Cout, Cin] 1x1; padded outputs / inputs carry zeros past the real ones
            return w[:n, :c.in_channels], cw.reshape(n, -1)
        return w, cw

    for kind, w, b in packed:
        cands = [layout(kind, w, c) + (c,) for c in by_bias[round(float(b[0]), 6)]]
        w, cw, c = min((x for x in cands if x[0].shape == x[1].shape), key=lambda x: np.abs(x[0] - x[1]).max())
        assert np.all(np.abs(w - cw) <= 2.0 ** -11 * np.abs(cw) + 2.0 ** -24), kind
        assert np.allclose(b[:c.out_channels], c.bias.detach().numpy(), rtol=1e-6, atol=1e-7), kind


def _same_plan(a, b):
    assert [(t, p, f) for t, p, f in a.ops] == [(t, p, f) for t, p, f in b.ops]
    assert a.buffers == b.buffers and a.outputs == b.outputs and a.meta == b.meta
    for x, y in zip(a.tensors, b.tensors):
        assert x.shape == y.shape and x.dtype == y.dtype
        assert np.abs(x.astype(np.float64) - y.astype(np.float64)).max() <= 2e-3 * max(1.0, float(np.abs(x).max()))


@pytest.mark.parametrize("scale", ["s", "l"])
def test_training_and_fused_checkpoints_pack_one_plan(scale):
    """Training-form keys (BatchNorms apart, as the seeded weights are) and the keys of a fused (deployed) model give the same plan; the
    training form read back as a real state_dict gives the seeded plan bit for bit."""
    W, ref = _weights(scale, 3)
    real = plan.build_yolov6_lite(plan.Weights(dict(W.state_dict)), scale)
    assert [(t, p) for t, p, _ in ref.ops] == [(t, p) for t, p, _ in real.ops]
    assert all(np.array_equal(a, b) for a, b in zip(ref.tensors, real.tensors))
    sd = ol.fused_state_dict(ol.build(W.state_dict, scale))
    assert not any(".bn" in k for k in sd)
    _same_plan(ref, plan.build_yolov6_lite(plan.Weights(sd), scale))


def test_input_must_be_a_multiple_of_32():
    with pytest.raises(AssertionError, match="multiple of 32"):
        _weights("s", in_h=320, in_w=336)


def _decode(pb, bufs):
    """The device decode (yolo_post.cu, reg_max 0) of plan_interp's head buffers for image 0: [A, 4 + nc]."""
    outs = []
    for buf, _, _, stride in pb.outputs:
        rows, C, _, H, W = pi.geom(pb, buf)
        v = bufs[buf][:rows].reshape(H + 2, W + 2, C)[1:-1, 1:-1]
        d = v[..., :4]
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        x1, y1, x2, y2 = xx + 0.5 - d[..., 0], yy + 0.5 - d[..., 1], xx + 0.5 + d[..., 2], yy + 0.5 + d[..., 3]
        box = np.stack([(x1 + x2) / 2, (y1 + y2) / 2, x2 - x1, y2 - y1], -1) * stride
        outs.append(np.concatenate([box, 1 / (1 + np.exp(-v[..., 8:8 + pb.meta[0]]))], -1).reshape(-1, 4 + pb.meta[0]))
    return np.concatenate(outs)


@pytest.mark.parametrize("scale,h,w", [("s", 320, 320), ("m", 320, 320), ("l", 320, 320), ("l", 224, 128), ("m", 320, 192)])
def test_interpreter_reproduces_the_oracle(scale, h, w):
    """plan_interp (float64, every op of the plan) against the fp32 oracle, including the ceil(H / 64) x ceil(W / 64) P6 level of inputs
    that are not multiples of 64; rounded to the plan's dtypes (the device's storage) it stays inside the 1e-3 probability contract."""
    W, pb = _weights(scale, 0, in_h=h, in_w=w)
    assert [(pi.geom(pb, b)[3], pi.geom(pb, b)[4]) for b, _, _, _ in pb.outputs] == [(-(-h // s), -(-w // s)) for s in (8, 16, 32, 64)]
    blob = post.yolo_prepare_input(synth.frame(0), h, w)[0]
    with torch.no_grad():
        ref = ol.build(W.state_dict, scale)(torch.from_numpy(blob)).numpy()[0]
    for rnd, tol_p, tol_b in ((False, 3e-4, 0.02), (True, 1e-3, 0.1)):
        got = _decode(pb, pi.interpret(pb, to_padded(blob, 4), 1, round_to_plan=rnd))
        assert np.abs(got[:, 4:] - ref[:, 5:]).max() < tol_p, (rnd, np.abs(got[:, 4:] - ref[:, 5:]).max())
        assert np.abs(got[:, :4] - ref[:, :4]).max() < tol_b, (rnd, np.abs(got[:, :4] - ref[:, :4]).max())


def test_dataflow():
    """With SE out of place no op writes over another's region and every read was written before; in place (the default) the only
    overlaps are the SE ops writing the slice they read."""
    W = plan.synth_weights("yolov6lite", 0, variant="m")
    apart = plan.build_yolov6_lite(W, "m", se_in_place=False)
    assert not pi.dataflow_violations(apart) and not pi.stale_reads(apart) and not pi.overwritten(apart)
    inplace = plan.build_yolov6_lite(W, "m")
    v = pi.dataflow_violations(inplace)
    assert v and all("(se) writes" in m for m in v)
    assert all(inplace.ops[i][0] == plan.OP_SE for i in pi.stale_reads(inplace))


def test_se_and_shuffle_references():
    """OP_SE's reference is upstream's SEBlock and OP_SHUFFLE2's is cat + channel_shuffle(2), on random slices."""
    rng = np.random.default_rng(0)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 5, 7)
    x = pb.sub(pb.new_padded(5, 7, 32), 8, 16)
    blk = ol.SEBlock(12).eval()
    sd = {k: v.numpy() for k, v in blk.state_dict().items()}
    pb.se(x, sd["conv1.weight"], sd["conv1.bias"], sd["conv2.weight"], sd["conv2.bias"])
    a, b = pb.sub(pb.new_padded(5, 7, 16), 0, 16), pb.sub(x.__class__(x.buf, 16, 16, 5, 7), 0, 16)
    pb.shuffle2(a, b)
    bufs = pi.new_buffers(pb, 1, np.float64)
    xv = rng.standard_normal((1, 12, 5, 7))
    bufs[x.buf].reshape(7, 9, 32)[1:-1, 1:-1, 8:20] = xv[0].transpose(1, 2, 0)
    bufs[a.buf].reshape(7, 9, 16)[1:-1, 1:-1] = rng.standard_normal((5, 7, 16))
    ref, bnd = pi.op_ref(pb, 0, bufs, 1)
    with torch.no_grad():
        want = blk(torch.from_numpy(xv).float()).numpy()
    assert np.abs(ref[:, :12] - want).max() < 1e-5 and not ref[:, 12:].any() and np.all(bnd > 0)
    sh, none = pi.op_ref(pb, 1, bufs, 1)
    av = pi.image_view(pb, bufs, a.buf, 0, 0, 16, "cpu")
    bv = pi.image_view(pb, bufs, b.buf, 0, b.coff, b.coff + 16, "cpu")
    assert none is None and np.array_equal(sh, ol.channel_shuffle(torch.cat([av, bv], 1)).numpy())


# ---------------------------------------------------------------------------------------------------------------------------
# the validators
# ---------------------------------------------------------------------------------------------------------------------------


def _op_field(raw, i, name):
    return fp.parse(raw).field_off(i, name)


def _check(tmp_path, raw, cases):
    for name, data, msg in cases:
        bad = tmp_path / "bad.b200w"
        bad.write_bytes(data)
        err = fp.engine_error(bad)
        assert err is not None and "plan" in err and msg in err, (name, err)


no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="load-time validation is observed through the missing-device error")


@no_gpu
def test_plan_validator_rejects_bad_se_ops(tmp_path):
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 8, 8)
    x = pb.new_padded(8, 8, 40)
    other = pb.new_padded(4, 4, 40)
    f32 = pb.new_padded(8, 8, 40, f32=True)
    out = pb.new_padded(8, 8, 40)
    rng = np.random.default_rng(0)
    pb.se(pb.sub(x, 8, 24), rng.standard_normal((5, 22)), rng.standard_normal(5), rng.standard_normal((22, 5)), rng.standard_normal(22))
    f16 = pb.tensor(np.zeros(24 * 5, np.float16))
    good = tmp_path / "se.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    p = lambda name: _op_field(raw, 0, name)
    _check(tmp_path, raw, [
        ("input index", fp.corrupt(raw, p("in_buf"), "<i", 99), "index out of range"),
        ("output index", fp.corrupt(raw, p("out_buf"), "<i", -1), "index out of range"),
        ("fp32 input", fp.corrupt(fp.corrupt(raw, p("in_buf"), "<i", f32.buf), p("out_buf"), "<i", f32.buf), "fp16"),
        ("geometry", fp.corrupt(raw, p("out_buf"), "<i", other.buf), "H x W"),
        ("channels", fp.corrupt(raw, p("C"), "<i", 12), "channels"),
        ("too many channels", fp.corrupt(raw, p("C"), "<i", 1032), "channels"),
        ("no hidden", fp.corrupt(raw, p("hid"), "<i", 0), "hidden"),
        ("hidden 257", fp.corrupt(raw, p("hid"), "<i", 257), "hidden"),
        ("offset", fp.corrupt(fp.corrupt(raw, p("in_coff"), "<i", 4), p("out_coff"), "<i", 4), "multiples of 8"),
        ("w1 size", fp.corrupt(raw, p("w1"), "<i", 1), "se tensor 0"),
        ("w2 is b2", fp.corrupt(raw, p("w2"), "<i", 3), "se tensor 2"),
        ("fp16 tensor", fp.corrupt(raw, p("b1"), "<i", f16), "se tensor 1"),
        ("tensor index", fp.corrupt(raw, p("b2"), "<i", 99), "se tensor 3"),
        ("slice", fp.corrupt(fp.corrupt(raw, p("in_coff"), "<i", 24), p("out_coff"), "<i", 24), "exceeds"),
        ("partial overlap", fp.corrupt(raw, p("out_coff"), "<i", 16), "overlaps"),
    ])
    ok = tmp_path / "ok.b200w"
    ok.write_bytes(fp.corrupt(raw, p("out_buf"), "<i", out.buf))                                   # out of place
    assert "no CUDA device" in fp.engine_error(ok)


@no_gpu
def test_plan_validator_rejects_bad_shuffle2_ops(tmp_path):
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 8, 8)
    src = pb.new_padded(8, 8, 48)
    other = pb.new_padded(4, 4, 48)
    f32 = pb.new_padded(8, 8, 48, f32=True)
    pb.shuffle2(pb.sub(src, 0, 16), pb.sub(src, 32, 16), out=pb.sub(pb.new_padded(8, 8, 40), 8, 32))
    good = tmp_path / "sh.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    p = lambda name: _op_field(raw, 0, name)
    _check(tmp_path, raw, [
        ("a index", fp.corrupt(raw, p("a_buf"), "<i", 99), "index out of range"),
        ("b index", fp.corrupt(raw, p("b_buf"), "<i", -1), "index out of range"),
        ("out index", fp.corrupt(raw, p("out_buf"), "<i", 99), "index out of range"),
        ("fp32 source", fp.corrupt(raw, p("b_buf"), "<i", f32.buf), "fp16"),
        ("geometry", fp.corrupt(raw, p("a_buf"), "<i", other.buf), "H x W"),
        ("channels", fp.corrupt(raw, p("n"), "<i", 12), "multiples of 8"),
        ("no channels", fp.corrupt(raw, p("n"), "<i", 0), "multiples of 8"),
        ("offset", fp.corrupt(raw, p("a_coff"), "<i", 4), "multiples of 8"),
        ("source slice", fp.corrupt(raw, p("b_coff"), "<i", 40), "exceeds"),
        ("output slice", fp.corrupt(raw, p("out_coff"), "<i", 16), "exceeds"),
        ("output over a source", fp.corrupt(fp.corrupt(raw, p("out_buf"), "<i", src.buf), p("out_coff"), "<i", 16), "overlaps"),
    ])


@no_gpu
@pytest.mark.parametrize("op", ["gemm", "stem", "dwconv"])
def test_activation_codes(tmp_path, op):
    """5 (Hardswish) is accepted wherever an activation is; 4 (unused) and 6 are not."""
    rng = np.random.default_rng(0)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 16, 16)
    x = pb.new_padded(16, 16, 32)
    if op == "gemm":
        pb.conv(x, rng.standard_normal((32, 32, 1, 1)).astype(np.float32), np.zeros(32, np.float32), 1, 1, plan.ACT_HSWISH)
    elif op == "stem":
        pb.conv(pb.image, rng.standard_normal((24, 3, 3, 3)).astype(np.float32), np.zeros(24, np.float32), 3, 2, plan.ACT_HSWISH)
    else:
        pb.dwconv(x, rng.standard_normal((32, 1, 5, 5)).astype(np.float32), np.zeros(32, np.float32), 5, 2, plan.ACT_HSWISH)
    assert pb.ops[-1][0] == {"gemm": plan.OP_GEMM, "stem": plan.OP_STEMCONV, "dwconv": plan.OP_DWCONV}[op]
    good = tmp_path / f"{op}.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    f = _op_field(raw, len(pb.ops) - 1, "act")
    msg = "dwconv act" if op == "dwconv" else "unknown activation"
    _check(tmp_path, raw, [(f"act {a}", fp.corrupt(raw, f, "<i", a), f"{msg} {a}") for a in (4, 6, -1)])
    if op == "dwconv":
        _check(tmp_path, raw, [("k 5 stride 3", fp.corrupt(raw, _op_field(raw, 0, "stride"), "<i", 3), "dwconv k 5 stride 3"),
                               ("k 9", fp.corrupt(raw, _op_field(raw, 0, "k"), "<i", 9), "dwconv k 9")])


@no_gpu
def test_four_level_head_validation(tmp_path):
    """A YOLOv6 plan with a stride-64 level of ceil(H / 64) x ceil(W / 64) cells loads; a fourth level of the wrong grid or stride, or a
    fifth, is refused naming the rule."""
    _, pb = _weights("s", in_h=224, in_w=128)
    good = tmp_path / "lite.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    out = lambda i, k: fp.parse(raw).out_off(i) + 4 * k
    _check(tmp_path, raw, [
        ("P6 grid of the P5 level", fp.corrupt(raw, out(3, 0), "<i", pb.outputs[2][0]), "YOLOv6 head has 3 levels"),
        ("P6 stride 32", fp.corrupt(raw, out(3, 3), "<i", 32), "YOLOv6 head has 3 levels"),
        ("P5 grid on level 2", fp.corrupt(raw, out(2, 0), "<i", pb.outputs[1][0]), "YOLOv6 level 2"),
    ])


# ---------------------------------------------------------------------------------------------------------------------------
# every other family packs exactly as before
# ---------------------------------------------------------------------------------------------------------------------------
SEEDED = [("yolov8", "n", lambda W: plan.build_yolov8(W, "n", in_h=320, in_w=320), "67ba130fc759bd0a"),
          ("yolov5", "s", lambda W: plan.build_yolov5(W, "s", in_h=320, in_w=320), "7c6fa47adabde5f7"),
          ("yolov5", "lite", lambda W: plan.build_yolov5(W, "n", in_h=320, in_w=320, lite=True), "61b3502b641b3ec4"),
          ("yolov7", "tiny", lambda W: plan.build_yolov7(W, "tiny", in_h=320, in_w=320), "ab7341e3f3a28a1c"),
          ("yolov6", "n", lambda W: plan.build_yolov6(W, "n", in_h=320, in_w=320), "af23e2d4f66fdbfc"),
          ("yolov6", "m", lambda W: plan.build_yolov6(W, "m", in_h=320, in_w=320), "a937daf4b787a5e2"),
          ("yolov9", "t", lambda W: plan.build_yolov9(W, "t", in_h=320, in_w=320), "e7c144cea6e9440b"),
          ("yolov10", "n", lambda W: plan.build_yolov10(W, "n", in_h=320, in_w=320), "2cf48ea975042851"),
          ("ufldv2", "18", lambda W: plan.build_ufldv2(W, "18", plan.UFLD_TUSIMPLE), "6ddff2da68bc6032")]


@pytest.mark.parametrize("kind,scale,build,digest", SEEDED, ids=[f"{k}-{s}" for k, s, _, _ in SEEDED])
def test_seeded_plans_of_other_families_are_unchanged(tmp_path, kind, scale, build, digest):
    """SHA-256 prefixes of the seeded plans as the packer wrote them before YOLOv6-Lite (the 24-channel stem route and the new ops
    must not move any other network)."""
    path = tmp_path / "p.b200w"
    build(plan.synth_weights(kind, 0, variant=scale)).write(str(path))
    assert hashlib.sha256(path.read_bytes()).hexdigest()[:16] == digest


@pytest.mark.parametrize("form", ["training", "fused"])
def test_checkpoint_conversion(tmp_path, form):
    from adas_b200 import convert
    W, ref = _weights("m", 4)
    sd = W.state_dict if form == "training" else ol.fused_state_dict(ol.build(W.state_dict, "m"))
    ckpt = str(tmp_path / f"lite_{form}.pth")
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, ckpt)
    got = convert.plan_from_state_dict(convert.load_checkpoint_state_dict(ckpt), "yolov6-lite", scale="m")
    _same_plan(ref, got)
    out = tmp_path / "lite_m.b200w"
    assert convert.main([ckpt, "--kind", "yolov6-lite", "--scale", "m", "--out", str(out)]) == 0 and out.stat().st_size > 0


# ---------------------------------------------------------------------------------------------------------------------------
# ONNX import
# ---------------------------------------------------------------------------------------------------------------------------
def _export(model, shape, path, opset):
    """tests/test_onnx_import._export at a chosen opset: Hardswish is a HardSwish node from opset 14 on, HardSigmoid + Mul before."""
    import warnings
    from torch.onnx._internal.torchscript_exporter import onnx_proto_utils
    onnx_proto_utils._add_onnxscript_fn = lambda model_bytes, custom_opsets: model_bytes
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        torch.onnx.export(model.eval(), torch.zeros(*shape), path, opset_version=opset, dynamo=False, input_names=["images"])


@pytest.mark.parametrize("opset", [12, 14])
@pytest.mark.parametrize("scale", ["s", "m", "l"])
def test_onnx_export_is_recognised_and_packs_the_state_dict_plan(tmp_path, scale, opset):
    from adas_b200 import onnx_import
    import test_onnx_import as toi
    W, ref = _weights(scale, 5)
    path = str(tmp_path / f"lite_{scale}_{opset}.onnx")
    _export(ol.build(W.state_dict, scale).fuse(), (1, 3, 320, 320), path, opset)
    m = onnx_import.read_onnx(path)
    assert ("HardSwish" in {n.op_type for n in m.nodes}) == (opset >= 14)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.nc, spec.in_h, spec.in_w) == ("yolov6-lite", scale, 80, 320, 320)
    toi._assert_same_plan(ref, onnx_import.build_plan(m, spec), f"yolov6lite-{scale} opset {opset}")


def test_onnx_training_form_export_and_other_inputs(tmp_path):
    """A training-form export (BatchNorms apart) at 224 x 128 with 20 classes packs the plan of its state_dict."""
    from adas_b200 import onnx_import
    import test_onnx_import as toi
    W = plan.synth_weights("yolov6lite", 6, variant="l")
    ref = plan.build_yolov6_lite(W, "l", nc=20, in_h=224, in_w=128)
    path = str(tmp_path / "lite_l.onnx")
    _export(ol.build(W.state_dict, "l", nc=20), (1, 3, 224, 128), path, 14)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.nc, spec.in_h, spec.in_w) == ("yolov6-lite", "l", 20, 224, 128)
    toi._assert_same_plan(ref, onnx_import.build_plan(m, spec), "yolov6lite-l training form")


class _LiteLike(torch.nn.Module):
    """Depthwise convs, an SE-style HardSigmoid gate and `levels` named detect.cls_preds / reg_preds, stage width `width`."""
    def __init__(self, width=64, levels=4, names=True):
        super().__init__()
        self.stem = torch.nn.Conv2d(3, width, 3, 2, 1)
        self.dw = torch.nn.Conv2d(width, width, 3, 1, 1, groups=width)
        head = torch.nn.Module()
        head.cls_preds = torch.nn.ModuleList(torch.nn.Conv2d(width, 80, 1) for _ in range(levels))
        head.reg_preds = torch.nn.ModuleList(torch.nn.Conv2d(width, 4, 1) for _ in range(levels))
        if names:
            self.detect = head
        else:
            self.h = head

    def forward(self, x):
        y = self.dw(torch.nn.functional.hardswish(self.stem(x)))
        y = y * torch.nn.functional.hardsigmoid(y.mean((2, 3), keepdim=True))
        head = self.detect if hasattr(self, "detect") else self.h
        return torch.cat([c(y).flatten(2) for c in head.cls_preds] + [r(y).flatten(2) for r in head.reg_preds], 1)


@pytest.mark.parametrize("kw,shape,what", [
    (dict(), (1, 3, 64, 64), "stage-4 width of 64"),
    (dict(width=176, levels=3), (1, 3, 64, 64), "3 detection levels"),
    (dict(width=176), (1, 3, 64, 80), "multiple of 32"),
    (dict(width=176, names=False), (1, 3, 64, 64), "module names"),
])
def test_out_of_scope_lite_files_name_the_supported_variants(tmp_path, kw, shape, what):
    from adas_b200 import onnx_import
    path = str(tmp_path / "bad.onnx")
    _export(_LiteLike(**kw), shape, path, 12)
    with pytest.raises(Exception, match="YOLOv6-Lite-S / M / L") as e:
        onnx_import.recognise(onnx_import.read_onnx(path))
    assert what in str(e.value) and "YOLOv6-N / S / M / L" in str(e.value)
