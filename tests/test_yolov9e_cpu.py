"""CPU: YOLOv9-E (GELAN-E) -- counts against the published figures, the oracle's fuse, the packer's folds, ONNX recognition and
checkpoint conversion, the OP_CBFUSE validator, the float64 plan interpreter against the oracle, the plan's dataflow, and the teeth of
the per-element CBFuse bound of plan_interp.

The graph restates upstream's `models/detect/gelan-e.yaml` (v0.1); with no upstream file available, the published counts are its
anchor: 57.3 M parameters and 189.0 GFLOP (YOLOv9-E, fused) and 58.1 M parameters (GELAN-E, training form)."""

import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import onnx_import, plan
import plan_footprint as fp
import plan_interp as pi
import post_conformance_cases as pc
import synth
import test_onnx_import as toi
import yolov9_oracle as o9
import yolov9e_oracle as oe
from gpu_util import to_padded
from oracle import post


def _weights(seed):
    W = plan.synth_weights("yolov9", seed, variant="e")
    return W, plan.build_yolov9(W, "e", in_h=320, in_w=320)


def test_yolov9e_counts_match_the_published_figures():
    W = plan.synth_weights("yolov9", 0, variant="e")
    pb = plan.build_yolov9(W, "e")
    assert abs(pb.flops_per_img / 1e9 - 188.95) < 0.005, pb.flops_per_img / 1e9
    train = oe.build(W.state_dict)
    assert abs(sum(p.numel() for p in train.parameters()) / 1e6 - 58.11) < 0.005
    n_train = sum(isinstance(m, torch.nn.Conv2d) for m in train.modules())
    fused = oe.build(W.state_dict).fuse()
    assert abs(o9.fused_params(fused) / 1e6 - 57.346) < 0.0005, o9.fused_params(fused) / 1e6
    assert o9.flops(fused) == pb.flops_per_img
    n_fused = sum(isinstance(m, torch.nn.Conv2d) for m in fused.modules())
    assert (n_fused, n_train) == (261, 309) == (plan.yolov9_conv_count("e"), 261 + plan.yolov9_repconvn_count("e"))
    assert pb.model_kind == plan.MODEL_YOLOV8 and pb.meta[:2] == [80, 8400] and len(pb.outputs) == 3
    fuses = [op for op in pb.ops if op[0] == plan.OP_CBFUSE]
    assert [p.n_src for _, p, _ in fuses] == [5, 4, 3, 2, 1]
    assert all(p.out_buf == p.base_buf and p.out_coff == p.base_coff for _, p, _ in fuses)    # in place
    assert [p.C for _, p, _ in fuses] == [64, 128, 256, 512, 1024]
    # the two image convs run in stem_conv.cu
    assert sum(1 for t, p, _ in pb.ops if t == plan.OP_STEMCONV and p.Cout == 64) == 2


def test_oracle_fused_equals_training_form():
    W, _ = _weights(1)
    x = torch.rand(1, 3, 320, 320)
    with torch.no_grad():
        a = oe.build(W.state_dict)(x).numpy()
        b = oe.build(W.state_dict).fuse()(x).numpy()
    assert a.shape == (1, 84, 2100)
    assert np.abs(a[:, 4:] - b[:, 4:]).max() < 1e-4
    assert np.abs(a[:, :4] - b[:, :4]).max() < 1e-4 * max(1.0, float(np.abs(a[:, :4]).max()))


def test_packer_folds_equal_oracle_fuse():
    """RepConvN and Conv + BN folded by the packer equal the oracle's fuse() to 1e-5; the CBLinear GEMMs carry `model.{10..14}.conv`
    as it is (all groups of one CBLinear in one GEMM)."""
    W, pb = _weights(2)
    fused = oe.build(W.state_dict).fuse()
    n_rep = n_conv = 0
    for name, m in fused.named_modules():
        if isinstance(m, o9.RepConvN):
            c = m.conv
            w, b = W.repconvn(name, c.out_channels, c.in_channels, plan.BN_EPS_YOLO)
            n_rep += 1
        elif isinstance(m, o9.Conv):
            c = m.conv
            w, b = W.conv_bn(name, c.out_channels, c.in_channels // c.groups, c.kernel_size[0], plan.BN_EPS_YOLO)
            n_conv += 1
        else:
            continue
        assert np.abs(w - c.weight.detach().numpy()).max() < 1e-5 and np.abs(b - c.bias.detach().numpy()).max() < 1e-5, name
    assert n_rep == 48 and n_conv > 0
    gemms = {pb.tensors[p.w_tensor].shape: p for t, p, _ in pb.ops             # the head's final 1x1 convs store fp32
             if t == plan.OP_GEMM and p.act == plan.ACT_NONE and pb.buffers[p.out_buf][2] == 0}
    assert len(gemms) == 5
    for i, (cin, cout) in enumerate(((64, 64), (256, 192), (512, 448), (1024, 960), (1024, 1984))):
        p = gemms[(cout, cin)]
        w = fused.model[10 + i].conv.weight.detach().numpy()[:, :, 0, 0]
        assert np.array_equal(pb.tensors[p.w_tensor], w.astype(np.float16))
        assert np.array_equal(pb.tensors[p.bias_tensor], fused.model[10 + i].conv.bias.detach().numpy())


def test_fused_checkpoint_packs_the_training_form_plan():
    W, ref = _weights(6)
    sd = {k: v.detach().numpy() for k, v in oe.build(W.state_dict).fuse().state_dict().items()}
    assert not any(".conv1." in k or ".bn." in k for k in sd)
    got = plan.build_yolov9(plan.Weights(sd), "e", in_h=320, in_w=320)
    assert [(t, p) for t, p, _ in ref.ops] == [(t, p) for t, p, _ in got.ops]
    for a, b in zip(ref.tensors, got.tensors):
        assert a.shape == b.shape and np.abs(a.astype(np.float32) - b.astype(np.float32)).max() <= 2e-3 * max(1.0, float(np.abs(a).max()))


@pytest.mark.parametrize("names", ["kept", "lost"])
def test_export_is_recognised_and_packs_the_state_dict_plan(tmp_path, names):
    W, ref = _weights(3)
    model = oe.build(W.state_dict)
    path = str(tmp_path / f"v9e_{names}.onnx")
    toi._export(model.fuse() if names == "kept" else model, (1, 3, 320, 320), path)
    m = onnx_import.read_onnx(path)
    spec = onnx_import.recognise(m)
    assert (spec.kind, spec.scale, spec.nc, spec.in_h, spec.in_w) == ("yolov9", "e", 80, 320, 320)
    w = onnx_import.OnnxWeights(m)
    got = plan.build_yolov9(w, "e", in_h=320, in_w=320)
    assert (w.used_anonymous > 200) == (names == "lost")
    toi._assert_same_plan(ref, got, f"yolov9-e names {names}")


def test_yolov9c_file_is_still_c(tmp_path):
    W = plan.synth_weights("yolov9", 4, variant="c")
    plan.build_yolov9(W, "c", in_h=320, in_w=320)
    path = str(tmp_path / "v9c.onnx")
    toi._export(o9.build(W.state_dict, "c").fuse(), (1, 3, 320, 320), path)
    spec = onnx_import.recognise(onnx_import.read_onnx(path))
    assert (spec.kind, spec.scale) == ("yolov9", "c")


class _TwoOutputs(torch.nn.Module):
    """An E file with a second output (as an auxiliary-branch training file has)."""
    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        y = self.net(x)
        return y, y[:, :4]


def test_two_output_yolov9e_file_is_refused(tmp_path):
    W, _ = _weights(5)
    path = str(tmp_path / "v9e_two.onnx")
    toi._export(_TwoOutputs(oe.build(W.state_dict).fuse()), (1, 3, 320, 320), path)
    with pytest.raises(Exception, match="YOLOv9-T / S / M / C / E") as e:
        onnx_import.recognise(onnx_import.read_onnx(path))
    assert "outputs" in str(e.value)


@pytest.mark.parametrize("form", ["training", "fused"])
def test_checkpoint_conversion(tmp_path, form):
    from adas_b200 import convert
    W, ref = _weights(6)
    ref = plan.build_yolov9(W, "e")
    sd = W.state_dict if form == "training" else {k: v.numpy() for k, v in oe.build(W.state_dict).fuse().state_dict().items()}
    ckpt = str(tmp_path / f"v9e_{form}.pth")
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, ckpt)
    got = convert.plan_from_state_dict(convert.load_checkpoint_state_dict(ckpt), "yolov9", scale="e")
    toi._assert_same_plan(ref, got, f"yolov9-e {form} checkpoint")
    assert convert.main([ckpt, "--kind", "yolov9", "--scale", "e", "--out", str(tmp_path / "v9e.b200w")]) == 0


def test_input_must_be_a_multiple_of_32():
    with pytest.raises(AssertionError, match="multiple of 32"):
        plan.build_yolov9(plan.synth_weights("yolov9", 0, variant="e"), "e", in_h=320, in_w=336)


# ---------------------------------------------------------------------------------------------------------------------------
# the OP_CBFUSE validator
# ---------------------------------------------------------------------------------------------------------------------------


@pytest.mark.skipif(torch.cuda.is_available(), reason="load-time validation is observed through the missing-device error")
def test_plan_validator_rejects_bad_cbfuse_ops(tmp_path):
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 16, 16)
    out = pb.new_padded(16, 16, 48)
    s0 = pb.new_padded(16, 16, 32)
    s1 = pb.new_padded(8, 8, 24)
    s2 = pb.new_padded(4, 4, 16)
    f32 = pb.new_padded(16, 16, 32, f32=True)
    other = pb.new_padded(8, 8, 48)
    pb.cbfuse(pb.sub(out, 8, 16), [(pb.sub(s0, 8, 16), 0), (pb.sub(s1, 0, 16), 1), (pb.sub(s2, 0, 16), 2)])
    good = tmp_path / "cbf.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    p = lambda name: fp.parse(raw).field_off(0, name)
    cases = [
        ("output index", fp.corrupt(raw, p("out_buf"), "<i", 99), "index out of range"),
        ("base index", fp.corrupt(raw, p("base_buf"), "<i", -1), "index out of range"),
        ("source index", fp.corrupt(raw, p("src1.buf"), "<i", 99), "index out of range"),
        ("fp32 source", fp.corrupt(raw, p("src0.buf"), "<i", f32.buf), "fp16"),
        ("fp32 output", fp.corrupt(fp.corrupt(raw, p("out_buf"), "<i", f32.buf), p("base_buf"), "<i", f32.buf), "fp16"),
        ("no sources", fp.corrupt(raw, p("n_src"), "<i", 0), "sources"),
        ("six sources", fp.corrupt(raw, p("n_src"), "<i", 6), "sources"),
        ("shift 5", fp.corrupt(raw, p("src1.shift"), "<i", 5), "shift"),
        ("negative shift", fp.corrupt(raw, p("src0.shift"), "<i", -1), "shift"),
        ("shift + 1", fp.corrupt(raw, p("src1.shift"), "<i", 2), "geometry"),
        ("shift - 1", fp.corrupt(raw, p("src2.shift"), "<i", 1), "geometry"),
        ("base geometry", fp.corrupt(raw, p("base_buf"), "<i", other.buf), "output's H x W"),
        ("channels", fp.corrupt(raw, p("C"), "<i", 12), "multiples of 8"),
        ("output offset", fp.corrupt(fp.corrupt(raw, p("out_coff"), "<i", 4), p("base_coff"), "<i", 4), "multiples of 8"),
        ("source offset", fp.corrupt(raw, p("src0.coff"), "<i", 4), "multiples of 8"),
        ("output slice", fp.corrupt(fp.corrupt(raw, p("out_coff"), "<i", 40), p("base_coff"), "<i", 40), "exceeds"),
        ("source slice", fp.corrupt(raw, p("src0.coff"), "<i", 24), "exceeds"),
        ("source is the output", fp.corrupt(fp.corrupt(raw, p("src0.buf"), "<i", out.buf), p("src0.coff"), "<i", 16), "overlaps"),
        ("base overlaps the output", fp.corrupt(raw, p("base_coff"), "<i", 16), "overlaps"),
    ]
    for name, data, msg in cases:
        bad = tmp_path / "bad.b200w"
        bad.write_bytes(data)
        err = fp.engine_error(bad)
        assert err is not None and "plan" in err and msg in err, (name, err)
    # out of place (base in another buffer) is valid
    ok = tmp_path / "ok.b200w"
    ok.write_bytes(fp.corrupt(raw, p("base_buf"), "<i", s0.buf))
    assert "no CUDA device" in fp.engine_error(ok)


# ---------------------------------------------------------------------------------------------------------------------------
# the plan: dataflow and the float64 interpreter against the oracle
# ---------------------------------------------------------------------------------------------------------------------------
def test_dataflow():
    """Out of place, no op writes over another's region, every read was written before, nothing is overwritten later.  In place (the
    default), the only overlaps are each CBFuse writing the slice its base producers (conv 15 / 17, ADown 20 / 23 / 26's two convs)
    wrote just before it, and the only stale reads are the CBFuse ops' own base reads."""
    W = plan.synth_weights("yolov9", 0, variant="e")
    apart = plan.build_yolov9e(W, cbfuse_in_place=False)
    assert not pi.dataflow_violations(apart) and not pi.stale_reads(apart) and not pi.overwritten(apart)
    pb = plan.build_yolov9(W, "e")
    fuses = [i for i, op in enumerate(pb.ops) if op[0] == plan.OP_CBFUSE]
    for m in pi.dataflow_violations(pb):
        i, j = int(m.split()[1]), int(m.split(" over op ")[1].split("'")[0])
        assert i in fuses and i - 3 <= j < i and " writes " in m, m           # ADown: cv1, max pool, cv2
    assert sorted(pi.stale_reads(pb)) == fuses and all(v == [i] for i, v in pi.stale_reads(pb).items())
    clobbered = pi.overwritten(pb)
    assert len(clobbered) == 8 and all(clobbered[j].all() for j in clobbered)
    assert all(any(0 < i - j <= 3 for i in fuses) for j in clobbered)
    # the same ops and weights either way; only the CBFuse outputs (and the readers of them) move
    assert len(apart.ops) == len(pb.ops) and [t for t, _, _ in apart.ops] == [t for t, _, _ in pb.ops]
    assert all(np.array_equal(a, b) for a, b in zip(apart.tensors, pb.tensors))


def test_interpreter_reproduces_network():
    W = plan.synth_weights("yolov9", 0, variant="e")
    pb = plan.build_yolov9(W, "e", in_h=128, in_w=160)
    x = post.yolo_prepare_input(synth.frame(0), pb.in_h, pb.in_w)[0].astype(np.float16).astype(np.float32)
    bufs = pi.interpret(pb, to_padded(x, 4).astype(np.float64), 1)
    levels = []
    for buf, _, C, st in pb.outputs:
        H, Wd = pb.buffers[buf][3], pb.buffers[buf][4]
        levels.append((bufs[buf].reshape(1, H + 2, Wd + 2, -1)[:, 1:-1, 1:-1, :C], st))
    got, _ = pc.decode_reference("v8", levels, 80, 16, None)
    with torch.no_grad():
        ref = oe.build(W.state_dict)(torch.from_numpy(x)).numpy()
    e = np.abs(got - ref)
    print(f"[chain] yolov9-e: box error {e[:, :4].max():.3f} px, probability error {e[:, 4:].max():.2e}")
    assert e[:, :4].max() < 0.5 and e[:, 4:].max() < 1e-3


# ---------------------------------------------------------------------------------------------------------------------------
# teeth of the CBFuse bound
# ---------------------------------------------------------------------------------------------------------------------------
HT, WT, C, NB = 16, 24, 16, 2


def _teeth_plan():
    """CBFuse of channels [8, 24) of a 32-channel output, in place, with 4 sources (shifts 0, 1, 2, 3) at channel offset 8 of 32-channel
    buffers (so a read at the wrong offset meets real data)."""
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, HT, WT)
    out = pb.new_padded(HT, WT, 32)
    srcs = [(pb.sub(pb.new_padded(HT >> s, WT >> s, 32), 8, C), s) for s in range(4)]
    pb.cbfuse(pb.sub(out, 8, C), srcs)
    rng = np.random.default_rng(7)
    bufs = pi.new_buffers(pb, NB)
    for b, (_, _, _, H, W, _) in enumerate(pb.buffers):
        if b != pb.image.buf:
            v = bufs[b].reshape(NB, H + 2, W + 2, -1)
            v[:, 1:-1, 1:-1] = (rng.standard_normal(v[:, 1:-1, 1:-1].shape) * 4).astype(np.float16)
    return pb, bufs


def _emulate(pb, bufs, drop=None, shift_delta=(None, 0), coff_delta=(None, 0), base_twice=False, f16_acc=False):
    """The kernel in numpy: fp32 sum (base, then the sources in order), one rounding -- or one of the faults."""
    _, p, _ = pb.ops[0]
    def view(buf, coff, s):
        H, W = pb.buffers[buf][3], pb.buffers[buf][4]
        v = bufs[buf].reshape(NB, H + 2, W + 2, -1)[:, 1:-1, 1:-1, coff:coff + C].astype(np.float32)
        ys, xs = np.minimum(np.arange(HT) >> s, H - 1), np.minimum(np.arange(WT) >> s, W - 1)
        return v[:, ys][:, :, xs]
    dt = np.float16 if f16_acc else np.float32
    base = view(p.base_buf, p.base_coff, 0).astype(dt)
    acc = base + base if base_twice else base
    for k, (buf, coff, s) in enumerate(plan.cbfuse_sources(p)):
        if k == drop:
            continue
        s = s + (shift_delta[1] if shift_delta[0] == k else 0)
        coff = coff + (coff_delta[1] if coff_delta[0] == k else 0)
        acc = (acc + view(buf, coff, max(s, 0)).astype(dt)).astype(dt)
    return acc.astype(np.float16).astype(np.float64).transpose(0, 3, 1, 2)


def _ratio(pb, bufs, got):
    ref, bnd = pi.op_ref(pb, 0, bufs, NB)
    return pi.excess(got, ref, bnd)[0]


def test_cbfuse_bound_accepts_fp32_and_rejects_faults():
    pb, bufs = _teeth_plan()
    assert _ratio(pb, bufs, _emulate(pb, bufs)) <= 1.0
    faults = {f"drop source {k}": dict(drop=k) for k in range(4)}
    faults.update({f"source {k} shift {d:+d}": dict(shift_delta=(k, d)) for k in range(4) for d in (-1, 1) if k + d >= 0})
    faults.update({f"source {k} channel offset {d:+d}": dict(coff_delta=(k, d)) for k in range(4) for d in (-8, 8)})
    faults.update({"base added twice": dict(base_twice=True), "fp16 accumulation": dict(f16_acc=True)})
    for name, kw in faults.items():
        assert _ratio(pb, bufs, _emulate(pb, bufs, **kw)) > 1.0, name

