"""CPU half of the op conformance suite: every case of op_conformance_cases packs onto its intended route, and the per-element
bounds accept an emulated kernel (fp32 accumulation in a shuffled order, fp16 store) while rejecting the faults they exist to catch."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import op_conformance_cases as oc
from adas_b200 import plan


@pytest.mark.parametrize("family,case,make", oc.ALL, ids=[oc.case_id(f, c) for f, c, _ in oc.ALL])
def test_case_packs_onto_its_route(family, case, make):
    spec = make(case)
    assert oc.plan_route(spec) == spec.route, (family, case, [(t, p[:20]) for t, p, _ in spec.pb.ops])
    gemms = [p for t, p, _ in spec.pb.ops if t == plan.OP_GEMM]
    if spec.route == "s2":
        assert gemms[0][16] == 1
    if spec.route == "up2":
        assert gemms[0][19] == 1
    if spec.route in ("tr", "fc_stream"):
        assert gemms[0][14] == 1 and (gemms[0][6] * gemms[0][2] * 2 <= oc.FC_STREAM_MAX_BYTES) == (spec.route == "fc_stream")
    if spec.route == "im2col4":
        assert [p for t, p, _ in spec.pb.ops if t == plan.OP_IM2COL][0][2] % 8 == 4
    assert np.isfinite(spec.ref).all() or spec.route == "avgpool2"
    if spec.bound is not None:
        assert spec.bound.shape == spec.ref.shape and (spec.bound > 0).all()


# ---- the bounds have teeth -------------------------------------------------------------------------------------------------
def _acc(terms: np.ndarray, rng, dtype=np.float32) -> np.ndarray:
    """Sum terms [..., K] in `dtype`, one element after another, in a random order (the kernels' orders are some permutation)."""
    t = terms[..., rng.permutation(terms.shape[-1])].astype(dtype)
    return np.add.accumulate(t, axis=-1, dtype=dtype)[..., -1]


def _conv_terms(x, w, s, pad):
    """[B, Cout, Ho, Wo, K] products of a conv (K = taps * Cin) in float64 (exact for fp16 operands)."""
    B, cin, H, W = x.shape
    cout, _, k, _ = w.shape
    cols = F.unfold(torch.from_numpy(x), k, padding=pad, stride=s).numpy()       # [B, cin*k*k, L]
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    prod = cols[:, None, :, :] * w.reshape(cout, -1)[None, :, :, None]           # [B, Cout, K, L]
    return prod.transpose(0, 1, 3, 2).reshape(B, cout, Ho, Wo, -1)


def _emulate(x, w, b, s, pad, act, r=None, res="none", slope=oc.LEAKY, dtype=np.float32, drop=None, seed=0):
    rng = np.random.default_rng(seed)
    w = w.copy()
    if drop is not None:
        drop(w)
    acc = _acc(_conv_terms(x, w, s, pad), rng, dtype).astype(np.float32)
    a = acc + b.astype(np.float32)[None, :, None, None]
    if res == "pre":
        a = a + r.astype(np.float32)
    y = oc.act64(a.astype(np.float64), act, slope).astype(np.float32)
    if res == "post":
        y = y + r.astype(np.float32)
    return y.astype(np.float16).astype(np.float64)


def _problem(seed=1, cin=128, cout=16, H=6, W=7, k=3):
    rng = np.random.default_rng(seed)
    x = oc.f16(rng, (2, cin, H, W))
    w = oc.f16(rng, (cout, cin, k, k), np.sqrt(2.0 / (cin * k * k)))
    b = oc.f16(rng, cout, 0.5)
    r = oc.f16(rng, (2, cout, H, W))
    return x, w, b, r


def _violations(got, ref, bound):
    return int((np.abs(got - ref) > bound).sum())


@pytest.mark.parametrize("act,res", [(0, "none"), (1, "post"), (2, "pre"), (3, "post")])
def test_bound_accepts_emulated_kernel(act, res):
    x, w, b, r = _problem()
    ref, S, a, rp = oc.conv_ref(x, w, b, 1, 1, act, r, res)
    bound = oc.gemm_bound(ref, S, 9 * x.shape[1], act, a, rp)
    for seed in range(2):
        got = _emulate(x, w, b, 1, 1, act, r, res, seed=seed)
        assert _violations(got, ref, bound) == 0


def _drop_tap(w):
    w[:, :, 2, 0] = 0


def _drop_kblock(w):
    w[:, 64:128] = 0


CORRUPTIONS = {
    "tap dropped": dict(drop=_drop_tap),
    "k-block dropped": dict(drop=_drop_kblock),
    "fp16 accumulation": dict(dtype=np.float16),
    "leaky slope 0.125": dict(slope=0.125),
}


@pytest.mark.parametrize("name", sorted(CORRUPTIONS))
def test_bound_rejects_kernel_faults(name):
    x, w, b, r = _problem()
    act = 3 if "leaky" in name else 1
    ref, S, a, rp = oc.conv_ref(x, w, b, 1, 1, act)
    bound = oc.gemm_bound(ref, S, 9 * x.shape[1], act, a, rp)
    got = _emulate(x, w, b, 1, 1, act, **CORRUPTIONS[name])
    assert _violations(got, ref, bound) > 0, name


def test_bound_rejects_missing_bias_on_one_channel():
    x, w, b, r = _problem()
    ref, S, a, _ = oc.conv_ref(x, w, b, 1, 1, 1)
    bound = oc.gemm_bound(ref, S, 9 * x.shape[1], 1, a)
    b2 = b.copy(); b2[5] = 0
    assert _violations(_emulate(x, w, b2, 1, 1, 1), ref, bound) > 0


def test_bound_rejects_shifted_border_column():
    x, w, b, r = _problem()
    ref, S, a, _ = oc.conv_ref(x, w, b, 1, 1, 0)
    bound = oc.gemm_bound(ref, S, 9 * x.shape[1], 0, a)
    got = _emulate(x, w, b, 1, 1, 0)
    got[..., -1] = got[..., -2]
    assert _violations(got, ref, bound) > 0


def test_bound_rejects_residual_added_twice():
    x, w, b, r = _problem()
    ref, S, a, rp = oc.conv_ref(x, w, b, 1, 1, 1, r, "post")
    bound = oc.gemm_bound(ref, S, 9 * x.shape[1], 1, a, rp)
    assert _violations(_emulate(x, w, b, 1, 1, 1, 2 * r, "post"), ref, bound) > 0


def _attention_emulate(q, k, v, scale, pv_dtype):
    """The kernel's arithmetic for one head: fp32 logits, fp32 softmax weights rounded to fp16, P V summed in pv_dtype."""
    s = (q.astype(np.float32) @ k.astype(np.float32).T) * np.float32(scale)
    p = np.exp(s - s.max(1, keepdims=True)).astype(np.float32)
    l = p.sum(1, keepdims=True, dtype=np.float32)
    ph = p.astype(np.float16)
    terms = ph[:, :, None].astype(pv_dtype) * v[None, :, :].astype(pv_dtype)   # [N, M, hd]
    o = np.add.accumulate(terms, axis=1, dtype=pv_dtype)[:, -1].astype(np.float32)
    return (o / l).astype(np.float16).astype(np.float64)


@pytest.mark.parametrize("pv_dtype,ok", [(np.float32, True), (np.float16, False)])
def test_attention_bound(pv_dtype, ok):
    rng = np.random.default_rng(4)
    N, kdp, hd = 65, 64, 128
    q, k = oc.f16(rng, (N, kdp)), oc.f16(rng, (N, kdp))
    v = oc.f16(rng, (N, hd), 1.0, 3.0)
    scale = 0.125
    s = q @ k.T * scale
    P = np.exp(s - s.max(1, keepdims=True)); P /= P.sum(1, keepdims=True)
    ref = P @ v
    bound = oc.attention_bound(q, k, v, scale, ref)
    got = _attention_emulate(q, k, v, scale, pv_dtype)
    assert (_violations(got, ref, bound) == 0) == ok


def _layernorm_emulate(x, gamma, beta, d_norm, eps, two_pass):
    """fp32 row statistics with 256 per-thread strided runs and a tree over them, then the fp32 affine map and the fp16 store."""
    xf = x.astype(np.float32)
    D = x.shape[1]
    pad = (-D) % 256
    runs = np.concatenate([xf, np.zeros((x.shape[0], pad), np.float32)], 1).reshape(x.shape[0], -1, 256)   # [rows, steps, thread]

    def tree(v):        # v [rows, steps, 256]: sequential per thread, then pairwise
        t = np.add.accumulate(v, axis=1, dtype=np.float32)[:, -1]
        while t.shape[1] > 1:
            t = (t[:, 0::2] + t[:, 1::2]).astype(np.float32)
        return t[:, 0]

    mean = (tree(runs) / np.float32(d_norm))[:, None]
    if two_pass:
        dev = np.where(np.arange(runs.shape[1] * 256).reshape(runs.shape[1], 256)[None] < d_norm, runs - mean[:, :, None], 0).astype(np.float32)
        var = (tree(dev * dev) / np.float32(d_norm))[:, None]
    else:
        var = np.maximum(tree(runs * runs)[:, None] / np.float32(d_norm) - mean * mean, 0).astype(np.float32)
    rstd = (1 / np.sqrt(var + np.float32(eps))).astype(np.float32)
    y = (xf - mean) * rstd * gamma.astype(np.float32) + beta.astype(np.float32)
    return y.astype(np.float16).astype(np.float64)


@pytest.mark.parametrize("two_pass,ok", [(True, True), (False, False)])
def test_layernorm_bound_at_mean_over_std_200(two_pass, ok):
    spec = oc.layernorm_spec((4, 4992, 4000, 200.0))
    x = spec.ins[0][2]
    g = spec.pb.tensors[spec.pb.ops[0][1].gamma_tensor]
    bt = spec.pb.tensors[spec.pb.ops[0][1].beta_tensor]
    got = _layernorm_emulate(x, g, bt, 4000, 1e-5, two_pass)
    assert (_violations(got, spec.ref, spec.bound) == 0) == ok


def test_references_know_every_plan_op_and_activation():
    """plan_interp and the bounds know Hardswish and every op type of the plan format with no setup; activation code 4 (which the
    format leaves unused and the engine's validator refuses) and an unknown op type raise instead of passing as the identity."""
    import plan_interp as pi
    assert oc.act64(np.array([-1.0]), plan.ACT_HSWISH)[0] == -1.0 / 3.0
    rng = np.random.default_rng(0)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 8, 8)
    x = pb.new_padded(8, 8, 32)
    pb.cbfuse(pb.sub(x, 0, 16), [(pb.sub(pb.new_padded(4, 4, 16), 0, 16), 1)])
    pb.se(pb.sub(x, 16, 16), rng.standard_normal((4, 16)), rng.standard_normal(4), rng.standard_normal((16, 4)), rng.standard_normal(16))
    pb.shuffle2(pb.sub(x, 0, 8), pb.sub(x, 8, 8))
    assert [pi.op_kind(pb, i) for i in range(len(pb.ops))] == ["cbfuse", "se", "shuffle2"]
    a = np.array([-1.0, 2.0])
    for f in (lambda: pi._act(torch.from_numpy(a), 4), lambda: oc.act64(a, 4), lambda: oc.gemm_bound(a, a, 1, 4, a)):
        with pytest.raises(ValueError, match="unknown activation code 4"):
            f()
    _, p, fl = pb.ops[0]
    pb.ops[0] = (99, p, fl)
    with pytest.raises(ValueError, match="unknown type 99"):
        pi.op_regions(pb, 0)
    with pytest.raises(ValueError, match="unknown type 99"):
        pi.op_ref(pb, 0, pi.new_buffers(pb, 1, np.float64), 1)
