"""CPU: the dataflow of every plan builder, the float64 plan interpreter (plan_interp.py) against the networks' fp32 oracles, and the
faults the per-op check of test_gpu_plan_conformance.py must reject.

- Dataflow: no two ops write overlapping regions and every op reads only regions an earlier op (or pre-processing, for the image)
  wrote.  The GPU check compares each op with a reference computed from its input buffers as read back after the run; that holds
  only if nothing overwrote them later.  The one exception, YOLOv10's PSA block, is allowed below with its reason, and the GPU check
  skips the two ops that read the overwritten half.
- The interpreter, chained from the image through every op, reproduces each family's fp32 oracle within the whole-network
  tolerances (1e-3 on probabilities, 0.5 px on boxes, 5e-3 of the range on lane logits): the difference is the plan's fp16 weights.
- Teeth: on a conv -> swap-AB FC plan run for batch A then batch B, an fp32 accumulation in shuffled order passes the check, and each
  of these fails it: the FC's first 384 K entries from batch A, one 128-row M tile of the conv computed from batch A, one M tile left
  at batch A's value, and the conv reading its neighbour's channel slice."""
import numpy as np
import pytest
import torch

import plan_interp as pi
import post_conformance_cases as pc
import synth
from adas_b200 import plan
from gpu_util import to_padded
from oracle import nets, post

# (family, scale, builder kwargs) of every builder the dataflow check covers
DATAFLOW = [("yolov5", "n", {}), ("yolov5", "s", {}), ("yolov8", "n", {}), ("yolov8", "l", {}), ("yolov7", "base", {}),
            ("yolov7", "tiny", {}), ("yolov7", "w6", {}), ("yolov7", "e6e", {}), ("yolov6", "n", {}), ("yolov6", "l", {}),
            ("yolov9", "t", {}), ("yolov9", "c", {}), ("yolov10", "n", {}), ("yolov10", "x", {}),
            ("ufldv2", "18", dict(cfg="culane")), ("ufldv2", "34", dict(cfg="culane")), ("ufldv2", "18", dict(cfg="tusimple")),
            ("ufldv2", "34", dict(cfg="tusimple")), ("ufldv1", "18", dict(cfg="culane")), ("ufldv1", "18", dict(cfg="tusimple"))]

# The plans test_gpu_plan_conformance.py runs: (family, scale, builder kwargs, max_batch, batch)
GPU_PLANS = [("yolov8", "l", {}, 8, 8), ("ufldv2", "34", dict(cfg="culane"), 8, 8),
             ("yolov5", "n", {}, 4, 3), ("yolov6", "n", {}, 4, 3), ("yolov7", "tiny", {}, 4, 3), ("yolov9", "t", {}, 4, 3),
             ("yolov10", "n", {}, 4, 3), ("ufldv2", "18", dict(cfg="tusimple"), 4, 3), ("ufldv1", "18", dict(cfg="culane"), 4, 3),
             ("yolov7", "w6", dict(in_h=1280, in_w=1280), 2, 2)]


def build(family, scale, **kw):
    """Seeded synthetic weights and the plan builder of one network."""
    W = plan.synth_weights("ufldv2" if family == "ufldv1" else family, 0, variant=scale)
    return W, getattr(plan, "build_" + family)(W, scale, **kw)


def psa_in_place(pb, msg):
    """YOLOv10 PSA: `b += ffn(b)` stores ffn.1's output over the b half of cv1's output, so that cv2 reads cat(a, b) as one slice.
    Only the qkv conv and the proj residual read that half, and both run before ffn.1; plan_interp.stale_reads names them."""
    i = int(msg.split()[1])
    t, p, _ = pb.ops[i]
    j = int(msg.split(" over op ")[1].split("'")[0])
    tj, pj, _ = pb.ops[j]
    return (t == tj == plan.OP_GEMM and p.res_buf >= 0 and p.ntaps == pj.ntaps == 1
            and p.out_buf == pj.out_buf and p.out_coff == pj.out_coff + p.N and pj.N == 2 * p.N)


@pytest.mark.parametrize("family,scale,kw", DATAFLOW, ids=[f"{f}-{s}" + ("-" + kw["cfg"] if "cfg" in kw else "") for f, s, kw in DATAFLOW])
def test_dataflow(family, scale, kw):
    _, pb = build(family, scale, **kw)
    bad = [m for m in pi.dataflow_violations(pb) if not (family == "yolov10" and " writes " in m and psa_in_place(pb, m))]
    assert not bad, "\n".join(bad[:10])
    stale = pi.stale_reads(pb)
    if family == "yolov10":
        assert len(stale) == 2 and all(pb.ops[i][0] == plan.OP_GEMM for i in stale), stale
        assert len(pi.overwritten(pb)) == 1                       # cv1, whose b half ffn.1 overwrites
    else:
        assert not stale and not pi.overwritten(pb), stale


def test_gpu_plans_reach_every_route():
    """The plans of the GPU check contain every op type and GEMM route the builders emit, and at least one FC on tensor cores."""
    import test_gpu_plan_conformance
    assert test_gpu_plan_conformance.PLANS == GPU_PLANS
    kinds = set()
    for family, scale, kw, _, _ in GPU_PLANS:
        kinds |= {pi.op_kind(pb, i) for pb in [build(family, scale, **kw)[1]] for i in range(len(pb.ops))}
    everything = set()
    for family, scale, kw in DATAFLOW:
        _, pb = build(family, scale, **kw)
        everything |= {pi.op_kind(pb, i) for i in range(len(pb.ops))}
    assert everything <= kinds, everything - kinds
    assert {"gemm-1x1", "gemm-9tap", "gemm-s2", "gemm-up2", "gemm-tr", "gemm-fc_stream", "gemm-stem7x7s2", "im2col", "stempack",
            "stemconv", "maxpool", "upsample", "avgpool2", "dwconv", "attention", "layernorm"} <= kinds, kinds


# ---------------------------------------------------------------------------------------------------------------------------
# the interpreter against the oracles
# ---------------------------------------------------------------------------------------------------------------------------
def _oracle(family, scale, sd, **kw):
    if family in ("yolov5", "yolov8"):
        return nets.build(family, sd, scale=scale)
    if family == "ufldv2":
        cfg = plan.UFLD_DATASETS[kw["cfg"]]
        return nets.build("ufldv2", sd, backbone=scale, **{k: v for k, v in cfg.items() if k not in ("dataset", "crop_ratio")})
    if family == "ufldv1":
        cfg = post.UFLD_V1[kw["cfg"]]
        return nets.build("ufldv1", sd, backbone=scale, griding_num=cfg["griding_num"], cls_num_per_lane=cfg["cls_num_per_lane"])
    mod = __import__({"yolov7": "yolov7_oracle", "yolov6": "yolov6_oracle", "yolov9": "yolov9_oracle", "yolov10": "yolov10_oracle"}[family])
    return mod.build(sd, scale)


CHAIN = [("yolov5", "n", {}), ("yolov8", "n", {}), ("yolov7", "tiny", {}), ("yolov6", "n", {}), ("yolov9", "t", {}),
         ("yolov10", "n", {}), ("ufldv2", "18", dict(cfg="tusimple")), ("ufldv1", "18", dict(cfg="culane"))]


@pytest.mark.parametrize("family,scale,kw", CHAIN, ids=[f"{f}-{s}" for f, s, _ in CHAIN])
def test_interpreter_reproduces_network(tmp_path, family, scale, kw):
    ufld = family.startswith("ufld")
    if not ufld:
        kw = dict(kw, in_h=128, in_w=160)
    W, pb = build(family, scale, **kw)
    if ufld:
        cfg = plan.UFLD_DATASETS[kw["cfg"]] if family == "ufldv2" else post.UFLD_V1[kw["cfg"]]
        x = post.ufld_prepare_input(synth.frame(0), pb.in_h, pb.in_w, cfg["crop_ratio"] if family == "ufldv2" else 1.0)
    else:
        x = post.yolo_prepare_input(synth.frame(0), pb.in_h, pb.in_w)[0]
    x = x.astype(np.float16).astype(np.float32)                    # the engine's image buffer is fp16
    bufs = pi.interpret(pb, to_padded(x, 4).astype(np.float64), 1)
    with torch.no_grad():
        ref = _oracle(family, scale, W.state_dict, **kw)(torch.from_numpy(x))
    if ufld:
        ob, _, n, _ = pb.outputs[0]
        got = bufs[ob].reshape(1, -1)[:, :n]
        r = np.concatenate([t.numpy().reshape(1, -1) for t in (ref if isinstance(ref, list) else [ref])], 1)
        err = float(np.abs(got - r).max()) / max(1.0, float(np.abs(r).max()))
        print(f"[chain] {family}-{scale}: head error {err:.2e} of its range")
        assert err < 5e-3
        return
    levels = []
    for buf, _, C, st in pb.outputs:
        H, Wd = pb.buffers[buf][3], pb.buffers[buf][4]
        levels.append((bufs[buf].reshape(1, H + 2, Wd + 2, -1)[:, 1:-1, 1:-1, :C], st))
    layout = {"yolov5": "v5", "yolov7": "v5", "yolov6": "v6"}.get(family, "v8")
    anchors = None
    if layout == "v5":
        path = str(tmp_path / "p.b200w")
        pb.write(path)
        anchors = plan.read_anchors(path)
    got, _ = pc.decode_reference(layout, levels, pb.meta[0], pb.meta[2] if layout == "v6" else 16, anchors)
    ref = ref.numpy() if not isinstance(ref, (list, tuple)) else ref[0].numpy()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if layout == "v8":
        box, prob = np.abs(got - ref)[:, :4], np.abs(got - ref)[:, 4:]
    else:
        box, prob = np.abs(got - ref)[..., :4], np.abs(got - ref)[..., 4:]
    print(f"[chain] {family}-{scale}: box error {box.max():.3f} px, probability error {prob.max():.2e}")
    assert box.max() < 0.5 and prob.max() < 1e-3


# ---------------------------------------------------------------------------------------------------------------------------
# teeth
# ---------------------------------------------------------------------------------------------------------------------------
H, W_, CIN, COUT, NFC, B = 14, 14, 64, 8, 64, 2


def _teeth_plan():
    """A 3x3 conv of channels [64, 128) of a 192-channel buffer into an 8-channel padded map, whose whole per-image slab (16 x 16 x 8 =
    2048 entries, the first 384 of them the top halo row and 12 pixels of image row 0) feeds a swap-AB FC."""
    rng = np.random.default_rng(3)
    pb = plan.PlanBuilder(plan.MODEL_UFLDV2, 3, H, W_)
    xbuf = pb.new_padded(H, W_, 3 * CIN)
    w = oc_f16(rng, (COUT, CIN, 3, 3), np.sqrt(2.0 / (9 * CIN)))
    b = oc_f16(rng, COUT, 0.1)
    y = pb.conv(pb.sub(xbuf, CIN, CIN), w.astype(np.float32), b.astype(np.float32), 3, 1, plan.ACT_SILU)
    K = pb.buffers[y.buf][0] * pb.buffers[y.buf][1]
    out = pb.new_dense(1, NFC, f32=True)
    pb.fc(y.buf, K, (rng.standard_normal((NFC, K)) / np.sqrt(K)).astype(np.float16), oc_f16(rng, NFC, 0.1).astype(np.float32),
          plan.ACT_NONE, out)
    return pb, xbuf.buf


def oc_f16(rng, shape, scale=1.0):
    return (scale * rng.standard_normal(shape)).astype(np.float16).astype(np.float64)


def _emulate(pb, i, bufs, rng):
    """Op i as an fp32 kernel with a shuffled accumulation order: exact fp16 products, fp32 sums in a random K order, fp32 bias and
    activation, stored in the buffer's dtype."""
    t, p, _ = pb.ops[i]
    w = pb.tensors[p.w_tensor].astype(np.float32)
    bias = pb.tensors[p.bias_tensor].astype(np.float32)
    if p.transposed:
        rows, C = pb.buffers[p.a_buf][:2]
        x = bufs[p.a_buf][:B * rows].reshape(B, rows * C)[:, :p.Kc].astype(np.float32)
        cols = [x[:, k:k + 1] * w[:, k][None, :] for k in range(p.Kc)]                # [B, N] per k
    else:
        rows, C, _, Hh, Ww = pb.buffers[p.a_buf][:5]
        xp = bufs[p.a_buf][:B * rows].reshape(B, Hh + 2, Ww + 2, C)[..., p.a_coff:p.a_coff + p.Kc].astype(np.float32)
        wk = w.reshape(p.N, 3, 3, p.Kc)
        cols = [xp[:, dy:dy + Hh, dx:dx + Ww, c:c + 1] * wk[:, dy, dx, c] for dy in range(3) for dx in range(3) for c in range(p.Kc)]
    acc = np.zeros_like(cols[0])
    for k in rng.permutation(len(cols)):
        acc = acc + cols[k]
    a = acc + bias
    y = a / (np.float32(1) + np.exp(-a)) if p.act == 1 else a
    if p.transposed:
        return y.astype(np.float64)
    return y.transpose(0, 3, 1, 2).astype(np.float16).astype(np.float64)


def _teeth_runs():
    pb, xbuf = _teeth_plan()
    rng = np.random.default_rng(5)
    runs = []
    for seed in (11, 12):                                         # batch A, then batch B
        bufs = pi.new_buffers(pb, B) if not runs else {k: v.copy() for k, v in runs[-1].items()}
        r = np.random.default_rng(seed)
        v = bufs[xbuf].reshape(B, H + 2, W_ + 2, -1)
        v[:, 1:-1, 1:-1] = r.standard_normal((B, H, W_, 3 * CIN)).astype(np.float16)
        for i in range(len(pb.ops)):
            pi.write_out(pb, i, bufs, B, _emulate(pb, i, bufs, rng))
        runs.append(bufs)
    return pb, runs


@pytest.fixture(scope="module")
def teeth():
    return _teeth_runs()


def _worst(pb, bufs):
    out = []
    for i in range(len(pb.ops)):
        ref, bnd = pi.op_ref(pb, i, bufs, B)
        out.append(pi.excess(pi.read_out(pb, i, bufs, B), ref, bnd)[0])
    return out


def test_teeth_accepts_shuffled_fp32(teeth):
    pb, (A, Bb) = teeth
    assert pi.op_kind(pb, 0) == "gemm-9tap" and pi.op_kind(pb, 1) == "gemm-fc_stream"
    for bufs in (A, Bb):
        worst = _worst(pb, bufs)
        assert max(worst) <= 1.0, worst


def test_teeth_rejects_fc_prefetch_from_previous_batch(teeth):
    pb, (A, Bb) = teeth
    t, p, _ = pb.ops[1]
    rows, C = pb.buffers[p.a_buf][:2]
    x = Bb[p.a_buf][:B * rows].reshape(B, rows * C).astype(np.float64).copy()
    x[:, :384] = A[p.a_buf][:B * rows].reshape(B, rows * C)[:, :384]
    assert (x != Bb[p.a_buf][:B * rows].reshape(B, rows * C)).any()
    w = pb.tensors[p.w_tensor].astype(np.float64)
    got = x @ w.T + pb.tensors[p.bias_tensor]
    ref, bnd = pi.op_ref(pb, 1, Bb, B)
    assert pi.excess(got, ref, bnd)[0] > 1.0


def _tile_fault(pb, A, Bb, from_a_inputs):
    """The conv's padded-row M tile [128, 256) of batch B: computed from batch A's input, or left at batch A's output."""
    conv = pb.ops[0][1]
    out = Bb[conv.out_buf].copy()
    if from_a_inputs:
        redo = {k: v.copy() for k, v in Bb.items()}
        redo[conv.a_buf] = A[conv.a_buf]
        pi.write_out(pb, 0, redo, B, pi.op_ref(pb, 0, redo, B, want_bound=False)[0])
        src = redo[conv.out_buf]
    else:
        src = A[conv.out_buf]
    rows = np.arange(out.shape[0])
    hp = (rows % ((H + 2) * (W_ + 2))) // (W_ + 2)
    wp = rows % (W_ + 2)
    sel = (rows >= 128) & (rows < 256) & (hp >= 1) & (hp <= H) & (wp >= 1) & (wp <= W_)
    out[sel] = src[sel].astype(out.dtype)
    bufs = dict(Bb)
    bufs[conv.out_buf] = out
    ref, bnd = pi.op_ref(pb, 0, bufs, B)
    return pi.excess(pi.read_out(pb, 0, bufs, B), ref, bnd)


def test_teeth_rejects_tile_from_previous_batch(teeth):
    pb, (A, Bb) = teeth
    ratio, n = _tile_fault(pb, A, Bb, True)
    assert ratio > 1.0 and n > 0


def test_teeth_rejects_stale_tile(teeth):
    pb, (A, Bb) = teeth
    ratio, n = _tile_fault(pb, A, Bb, False)
    assert ratio > 1.0 and n > 0


def test_teeth_rejects_neighbour_slice(teeth):
    pb, (A, Bb) = teeth
    moved = {k: v.copy() for k, v in Bb.items()}
    t, p, f = pb.ops[0]
    pb2 = plan.PlanBuilder(pb.model_kind, 3, H, W_)
    pb2.buffers, pb2.tensors = pb.buffers, pb.tensors
    q = p.copy()
    q.a_coff += 64                                                   # the conv reads channels [128, 192)
    pb2.ops = [(t, q, f)] + pb.ops[1:]
    pi.write_out(pb, 0, moved, B, pi.op_ref(pb2, 0, Bb, B, want_bound=False)[0].astype(np.float16).astype(np.float64))
    ref, bnd = pi.op_ref(pb, 0, Bb, B)
    assert pi.excess(pi.read_out(pb, 0, moved, B), ref, bnd)[0] > 1.0
