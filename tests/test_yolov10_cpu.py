"""CPU: YOLOv10-N/S/M/B/L/X packer -- published counts, the RepVGGDW / BN folds, PSA's qkv permutation, checkpoint forms and the
validation of the depthwise-conv and attention ops.

The graphs restate ultralytics 8.2.41's yolov10{n,s,m,b,l,x}.yaml with the one-to-one head; the published counts are their anchor:
parameters of the fused graph (the 16 fixed DFL weights included) and 2 * MAC of the convolutions at 640x640."""

import numpy as np
import pytest
import torch

import adas_b200  # noqa: F401
from adas_b200 import plan
import plan_footprint as fp
import yolov10_oracle as o10

PUBLISHED = [("n", 2.299, 6.69), ("s", 7.249, 21.58), ("m", 15.359, 59.10), ("b", 19.066, 91.95), ("l", 24.371, 120.34),
             ("x", 29.474, 160.38)]


@pytest.mark.parametrize("scale,mparams,gflop", PUBLISHED)
def test_yolov10_counts_match_the_published_figures(scale, mparams, gflop):
    W = plan.synth_weights("yolov10", 0, variant=scale)
    pb = plan.build_yolov10(W, scale)
    assert abs(pb.flops_per_img / 1e9 - gflop) < 0.005, pb.flops_per_img / 1e9
    fused = o10.build(W.state_dict, scale).fuse()
    assert abs(o10.fused_params(fused) / 1e6 - mparams) < 0.0005, o10.fused_params(fused) / 1e6
    assert o10.flops(fused) == pb.flops_per_img
    assert pb.model_kind == plan.MODEL_YOLOV8 and pb.meta[:2] == [80, 8400] and len(pb.outputs) == 3
    assert sum(1 for op in pb.ops if op[0] == plan.OP_ATTN) == 1
    dw = [op for op in pb.ops if op[0] == plan.OP_DWCONV]
    n_lk = sum(1 for op in dw if op[1].k == 7)
    lk_blocks = [li for li, lk in plan.YOLOV10_CIB[scale].items() if lk]
    assert n_lk == len(lk_blocks) * plan._v8_n(3, plan.YOLOV10_SCALES[scale][0])
    assert sum(1 for op in dw if op[1].stride == 2) == 3                          # the three SCDowns
    assert 0 < pb.dw_flops_per_img < pb.flops_per_img


@pytest.mark.parametrize("scale", ["n", "m"])
def test_packer_folds_equal_oracle_fuse(scale):
    """Conv + BN and RepVGGDW (7x7 + 3x3 on the centre taps) folded by the packer equal the oracle's fuse() to 1e-5."""
    W = plan.synth_weights("yolov10", 2, variant=scale)
    pb = plan.build_yolov10(W, scale, in_h=320, in_w=320)
    g = plan.Yolov10Packer(pb, W)
    fused = o10.build(W.state_dict, scale).fuse()
    n_rep = n_dw = 0
    for name, m in fused.named_modules():
        if isinstance(m, o10.RepVGGDW):
            c = m.conv
            v = g.repvggdw(plan.View(0, 0, (c.out_channels + 7) // 8 * 8, 8, 8), name, c.out_channels)
            op = pb.ops[-1]
            wk = pb.tensors[op[1].w_tensor].astype(np.float32)[:, :c.out_channels]
            ref = c.weight.detach().numpy().reshape(c.out_channels, 49).T
            assert np.abs(wk - ref).max() <= 1e-3 * max(1.0, float(np.abs(ref).max())) and v.C % 8 == 0
            assert np.abs(pb.tensors[op[1].bias_tensor][:c.out_channels] - c.bias.detach().numpy()).max() < 1e-5
            n_rep += 1
        elif isinstance(m, o10.Conv):
            c = m.conv
            w, b = g.conv_bn(name, c.out_channels, c.in_channels // c.groups, c.kernel_size[0])
            assert np.abs(w - c.weight.detach().numpy()).max() < 1e-5 and np.abs(b - c.bias.detach().numpy()).max() < 1e-5, name
            n_dw += c.groups > 1
    assert n_rep == (1 if scale == "n" else 0) and n_dw > 0


@pytest.mark.parametrize("scale", ["n", "s", "m"])
def test_oracle_fused_equals_training_form(scale):
    W = plan.synth_weights("yolov10", 1, variant=scale)
    plan.build_yolov10(W, scale, in_h=320, in_w=256)
    x = torch.rand(1, 3, 320, 256)
    with torch.no_grad():
        a = o10.build(W.state_dict, scale)(x).numpy()
        b = o10.build(W.state_dict, scale).fuse()(x).numpy()
    assert a.shape == (1, 84, 10 * 8 * 21)
    assert np.abs(a[:, 4:] - b[:, 4:]).max() < 1e-4
    assert np.abs(a[:, :4] - b[:, :4]).max() < 1e-4 * max(1.0, float(np.abs(a[:, :4]).max()))


@pytest.mark.parametrize("nh,kd,hd", [(2, 32, 64), (4, 36, 72), (5, 32, 64)])
def test_qkv_permutation_gives_the_oracle_q_k_v(nh, kd, hd):
    """The packed qkv weights applied in numpy give the oracle Attention's q, k and v, with zero padding rows past kd."""
    c = nh * hd
    torch.manual_seed(nh)
    att = o10.Attention(c).eval()
    assert (att.nh, att.kd, att.hd) == (nh, kd, hd)
    att.qkv.fuse()
    x = torch.randn(1, c, 5, 7)
    with torch.no_grad():
        q, k, v = att.qkv_split(x)
    w = att.qkv.conv.weight.detach().numpy()
    b = att.qkv.conv.bias.detach().numpy()
    wp, bp = plan.qkv_permute(w, b, nh, kd, hd)
    kdp = (kd + 15) // 16 * 16
    assert wp.shape == (nh * (2 * kdp + hd), c, 1, 1)
    y = np.einsum("oc,cn->on", wp[:, :, 0, 0], x.numpy().reshape(c, 35)) + bp[:, None]
    for h in range(nh):
        qp, kp = y[h * kdp:(h + 1) * kdp], y[(nh + h) * kdp:(nh + h + 1) * kdp]
        assert np.allclose(qp[:kd], q[0, h].numpy(), atol=1e-4) and not qp[kd:].any()
        assert np.allclose(kp[:kd], k[0, h].numpy(), atol=1e-4) and not kp[kd:].any()
        assert np.allclose(y[2 * nh * kdp + h * hd:2 * nh * kdp + (h + 1) * hd], v[0, h].numpy(), atol=1e-4)


def test_fused_checkpoint_with_one_to_many_keys_packs_the_training_form_plan():
    """A state_dict after upstream's fuse (Conv with a bias, RepVGGDW as one 7x7 `conv`) with the one-to-many head's keys present packs
    the same network as the training-form weights; the extra keys are never read."""
    W = plan.synth_weights("yolov10", 6, variant="s")
    ref = plan.build_yolov10(W, "s", in_h=320, in_w=320)
    sd = {k: v.detach().numpy() for k, v in o10.build(W.state_dict, "s").fuse().state_dict().items()}
    assert not any(".conv1." in k or ".bn." in k for k in sd)
    for k in [k for k in sd if ".one2one_cv" in k]:
        sd[k.replace(".one2one_cv", ".cv")] = -sd[k]
    sd["model.23.dfl.conv.weight"] = np.arange(16, dtype=np.float32).reshape(1, 16, 1, 1)
    got = plan.build_yolov10(plan.Weights(sd), "s", in_h=320, in_w=320)
    assert [(t, p) for t, p, _ in ref.ops] == [(t, p) for t, p, _ in got.ops]
    for a, b in zip(ref.tensors, got.tensors):
        assert a.shape == b.shape and np.abs(a.astype(np.float32) - b.astype(np.float32)).max() <= 2e-3 * max(1.0, float(np.abs(a).max()))


def test_build_yolov10_refuses_bad_inputs():
    W = plan.synth_weights("yolov10", 0, variant="n")
    with pytest.raises(AssertionError, match="multiple of 32"):
        plan.build_yolov10(W, "n", in_h=600, in_w=640)
    with pytest.raises(AssertionError, match="scale"):
        plan.build_yolov10(W, "e")
    pb = plan.build_yolov10(W, "n", in_h=480, in_w=640)
    assert pb.meta[1] == 60 * 80 + 30 * 40 + 15 * 20


def _check_cases(tmp_path, raw, cases):
    for name, data, msg in cases:
        bad = tmp_path / "bad.b200w"
        bad.write_bytes(data)
        err = fp.engine_error(bad)
        assert err is not None and "plan" in err and msg in err, (name, err)


@pytest.mark.skipif(torch.cuda.is_available(), reason="load-time validation is observed through the missing-device error")
def test_plan_validator_rejects_bad_dwconv_ops(tmp_path):
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 16, 16)
    xin = pb.new_padded(16, 16, 64)
    out = pb.new_padded(16, 16, 32)
    half = pb.new_padded(8, 8, 32)
    f32 = pb.new_padded(16, 16, 32, f32=True)
    res = pb.new_padded(16, 16, 32)
    w = np.ones((16, 1, 3, 3), np.float32)
    pb.dwconv(pb.sub(xin, 8, 16), w, np.zeros(16, np.float32), 3, 1, plan.ACT_SILU, out=pb.sub(out, 8, 16), res=pb.sub(res, 16, 16))
    w7 = pb.tensor(np.zeros((49, 16), np.float16))
    good = tmp_path / "dw.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    off = lambda name: fp.parse(raw).field_off(0, name)
    c = lambda name, v, r=raw: fp.corrupt(r, off(name), "<i", v)
    _check_cases(tmp_path, raw, [
        ("input index", c("in_buf", 99), "index out of range"),
        ("output index", c("out_buf", -1), "index out of range"),
        ("residual index", c("res_buf", 77), "index out of range"),
        ("fp32 output", c("out_buf", f32.buf), "fp16"),
        ("fp32 residual", c("res_buf", f32.buf), "fp16"),
        ("kernel", c("k", 5), "dwconv k"),
        ("stride", c("stride", 3), "dwconv k"),
        ("7x7 stride 2", c("stride", 2, c("k", 7, c("w_tensor", w7))), "dwconv k"),
        ("act", c("act", 2), "act"),
        ("geometry", c("out_buf", half.buf), "output geometry"),
        ("channels", c("C", 12), "multiples of 8"),
        ("input offset", c("in_coff", 4), "multiples of 8"),
        ("output offset", c("out_coff", 12), "multiples of 8"),
        ("residual offset", c("res_coff", 4), "multiples of 8"),
        ("weight size", c("k", 7), "weight tensor"),
        ("bias tensor", c("bias_tensor", 0), "bias tensor"),
        ("residual geometry", c("res_buf", half.buf), "residual"),
        ("residual slice", c("res_coff", 24), "residual"),
        ("input slice", c("in_coff", 56), "exceeds"),
        ("output slice", c("out_coff", 24), "exceeds"),
        ("in place", c("out_coff", 16, c("out_buf", xin.buf)), "overlaps"),
    ])


@pytest.mark.skipif(torch.cuda.is_available(), reason="load-time validation is observed through the missing-device error")
def test_plan_validator_rejects_bad_attention_ops(tmp_path):
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 8, 8)
    qkv = pb.new_padded(8, 8, 2 * (2 * 32 + 64))
    out = pb.new_padded(8, 8, 128)
    half = pb.new_padded(4, 4, 128)
    f32 = pb.new_padded(8, 8, 128, f32=True)
    pb.attention(qkv, 2, 32, 64, 32 ** -0.5, out=out)
    good = tmp_path / "at.b200w"
    pb.write(str(good))
    assert "no CUDA device" in fp.engine_error(good)
    raw = good.read_bytes()
    off = lambda name: fp.parse(raw).field_off(0, name)
    c = lambda name, v, r=raw: fp.corrupt(r, off(name), "<i", v)
    _check_cases(tmp_path, raw, [
        ("input index", c("in_buf", 99), "index out of range"),
        ("output index", c("out_buf", -1), "index out of range"),
        ("fp32 output", c("out_buf", f32.buf), "fp16"),
        ("geometry", c("out_buf", half.buf), "H x W"),
        ("heads", c("nh", 0), "attention heads"),
        ("kdp", c("kdp", 24), "attention heads"),
        ("hd", c("hd", 60), "attention heads"),
        ("input offset", c("in_coff", 4), "multiples of 8"),
        ("output offset", c("out_coff", 12), "multiples of 8"),
        ("qkv slice", c("nh", 3), "exceeds"),
        ("output slice", c("out_coff", 8), "exceeds"),
        ("in place", c("out_buf", qkv.buf), "overlaps"),
        ("scale", fp.corrupt(raw, off("scale"), "<f", float("nan")), "scale"),
        ("negative scale", fp.corrupt(raw, off("scale"), "<f", -1.0), "scale"),
    ])


def test_convert_packs_a_yolov10_checkpoint(tmp_path):
    """`convert --kind yolov10` on a saved training-form state_dict with the one-to-many head's keys writes the state_dict's plan."""
    from adas_b200 import convert
    W = plan.synth_weights("yolov10", 4, variant="n")
    ref = plan.build_yolov10(W, "n")
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in W.state_dict.items()}
    sd.update({k.replace(".one2one_cv", ".cv"): v.clone() for k, v in sd.items() if ".one2one_cv" in k})
    src = tmp_path / "yolov10n.state_dict.pth"
    torch.save({"model": sd}, str(src))
    out = convert.convert(str(src), str(tmp_path / "n.b200w"), kind="yolov10", scale="n")
    ref.write(str(tmp_path / "ref.b200w"))
    assert (tmp_path / "ref.b200w").read_bytes() == open(out, "rb").read()
