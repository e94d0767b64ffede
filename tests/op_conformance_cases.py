"""One-op plans for the op conformance suite: the case table, float64 references and per-element error bounds.

Shared by test_gpu_op_conformance.py (runs every case on the GPU) and test_op_conformance_cpu.py (checks on the CPU that each case
packs onto its intended route and that the bounds reject the kernel faults they exist to catch).

Every operand is a channel slice of a wider buffer; `Spec.ins` lists what the op may read, `Spec.out` the slice it must write.
References are float64 computations on the fp16-rounded operands; bounds follow the arithmetic of the kernels (docstrings below), so
an element-wise comparison `|got - ref| <= bound` holds for any fp32 accumulation order and fails for a dropped tap, a dropped k-block,
a missing bias, a shifted border column, a doubled residual, a wrong activation slope or fp16 accumulation."""
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

import adas_b200  # noqa: F401
from adas_b200 import plan

U16, U32 = 2.0 ** -11, 2.0 ** -24          # unit roundoff of fp16 / fp32
NAN16, INF16 = 0x7E00, 0x7C00              # poison bit patterns: NaN for sum-type ops, +inf for max pooling
FC_STREAM_MAX_BYTES = 25 << 20             # FC weight matrices up to this size run on fc_stream (engine.cu)
LEAKY = 0.1


@dataclass
class Spec:
    pb: plan.PlanBuilder
    B: int
    ins: List[Tuple[int, int, np.ndarray]]   # (buffer, channel offset, float64 data [B, c, H, W] padded or [B, c] dense)
    out: Tuple[int, int, int]                # (buffer, channel offset, channels written)
    ref: np.ndarray                          # float64, same layout as the data
    bound: Optional[np.ndarray]              # per-element bound; None = bit-exact
    route: str
    poison: int = NAN16
    simt: bool = False                       # the op has a SIMT twin (conv_impl = 1)


def r8(c: int) -> int:
    return (c + 7) // 8 * 8


def f16(rng, shape, scale=1.0, loc=0.0) -> np.ndarray:
    """fp16-representable float64 values."""
    return (loc + scale * rng.standard_normal(shape)).astype(np.float16).astype(np.float64)


def view(pb, H, W, C, off, f32=False):
    """A C-channel view at channel `off` of a buffer that extends 16 channels past it (off None: a whole buffer of its own)."""
    if off is None:
        return pb.new_padded(H, W, r8(C) if C % 4 == 0 and C >= 8 else C, f32=f32)
    return pb.sub(pb.new_padded(H, W, off + r8(C) + 16, f32=f32), off, C)


def act64(a: np.ndarray, act: int, slope: float = LEAKY) -> np.ndarray:
    if act == plan.ACT_NONE:
        return a
    if act == 1:
        return a / (1.0 + np.exp(-a))
    if act == 2:
        return np.maximum(a, 0.0)
    if act == 3:
        return np.where(a >= 0, a, slope * a)
    if act == plan.ACT_HSWISH:
        return a * np.clip(a + 3.0, 0.0, 6.0) / 6.0
    raise ValueError(f"unknown activation code {act}")


# ---------------------------------------------------------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------------------------------------------------------
def gemm_bound(ref, S, K, act, a, res_post=None, out_f32=False):
    """Bound of one GEMM / conv / FC / depthwise output element.

    S = sum |x_i w_i| + |bias| (+ |r| for a residual added before the activation), K = taps * padded K per tap.  Any fp32 summation
    order of K products (exact: fp16 x fp16 fits fp32) and the bias has error <= gamma_K * S <= K * 2^-24 * S; 2^-23 doubles it for
    the bias / pre-activation residual adds and for tensor-core accumulators that truncate instead of rounding.  The activation has
    Lipschitz constant 1 (none, ReLU, LeakyReLU) or 1.1 (SiLU) and SiLU's fp32 evaluation (exp, divide) adds 2^-20 |a|; LeakyReLU's
    fp32 slope adds 2^-22 |a|.  Hardswish has Lipschitz constant 1.5 (slope (2x + 3) / 6 on [-3, 3], 0 or 1 outside); its fp32
    evaluation -- x + 3, the clamp (exact), the product with x and the product with fp32(1/6) -- adds four roundings of at most
    |x| (|x| + 3) / 6 each (which bounds |x + 3| |x| / 6 and every intermediate): 2^-21 |a| (|a| + 3) / 6.  A residual added after the
    activation costs one product and one add: 2^-24 |alpha r| + 2^-24 |ref|.  The fp16 store rounds to nearest: 2^-11 |ref| relative
    plus 2^-24 absolute below the normal range."""
    E = K * 2.0 ** -23 * S
    if act == 1:
        E = 1.1 * E + 2.0 ** -20 * np.abs(a)
    elif act == 3:
        E = E + 2.0 ** -22 * np.abs(a)
    elif act == plan.ACT_HSWISH:
        a = np.abs(a)
        E = 1.5 * E + 2.0 ** -21 * a * (a + 3.0) / 6.0
    elif act not in (plan.ACT_NONE, plan.ACT_RELU):
        raise ValueError(f"unknown activation code {act}")
    if res_post is not None:
        E = E + U32 * np.abs(res_post) + U32 * np.abs(ref)
    if out_f32:
        return E + U32 * np.abs(ref) + 2.0 ** -60
    return U16 * np.abs(ref) + (1 + U16) * E + U32


def attention_bound(q, k, v, scale, ref):
    """Bound of softmax(q k^T * scale) v for one head: q [N, kdp], k [N, kdp], v [N, hd], ref [N, hd] (float64).

    Logits: s_nm = sum_d q_nd k_md in fp32 from exact fp16 products: |ds| <= kdp 2^-23 sum_d |q_nd k_md|; scaling by scale*log2(e)
    (one fp32 constant, one product) adds 2^-22 |s|; exp2f adds 2^-22 relative.  Writing delta_nm for the resulting log-domain error of
    p_nm, the normalised weights move by at most (e^(2 max_m delta_nm) - 1) <= 2.01 max_m delta_nm relative, so the output moves by
    <= 2.01 max_m delta_nm * sum_m P_nm |v_m| (P the exact softmax).  The kernel then rounds p = exp2(s - running max) <= 1 to fp16
    before P V: 2^-11 relative, or 2^-25 absolute where p is subnormal in fp16 (a sharp softmax); the fp32 row sum l >= 1 uses the
    unrounded p, so after dividing by l this is <= 2^-11 sum_m P_nm |v_m| + 2^-25 sum_m |v_m|.  P V accumulates N products in fp32:
    N 2^-23 sum_m P_nm |v_m|.  The final 1/l and product: 2^-23 |ref|; the fp16 store: 2^-11 |ref| + 2^-24."""
    N = q.shape[0]
    qk = np.abs(q) @ np.abs(k).T                               # [N, N] sum_d |q_nd k_md|
    s = (q @ k.T) * scale
    delta = scale * kdp_term(q.shape[1]) * qk + 2.0 ** -22 * np.abs(s) + 2.0 ** -22
    P = np.exp(s - s.max(1, keepdims=True))
    P /= P.sum(1, keepdims=True)
    mag = P @ np.abs(v)                                        # [N, hd] sum_m P_nm |v_m|
    vsum = np.abs(v).sum(0)[None, :]
    E = (2.01 * delta.max(1, keepdims=True) + U16 + N * 2.0 ** -23) * mag + 2.0 ** -25 * vsum
    return U16 * np.abs(ref) + (1 + U16) * (E + 2.0 ** -23 * np.abs(ref)) + U32


def kdp_term(kdp: int) -> float:
    return kdp * 2.0 ** -23


LN_C = 4.0


def layernorm_bound(x, gamma, beta, d_norm, ref):
    """Bound of (x - mu) / sqrt(var + eps) * gamma + beta, statistics over the first d_norm entries of each row.

    A numerically stable fp32 evaluation (the mean first, then sum (x - mu)^2, each summed in short per-thread runs and a fixed tree)
    computes (x - mu) / sigma with error <= c D 2^-24 (1 + |x - mu| / sigma): the mean's error is relative to sigma times
    (run length + tree depth) 2^-24 |mu| / sigma, which for the rows of this suite (|mu| / sigma <= 200, D ~ 4000 over 256 threads,
    24 + 8 additions) stays below 2 D 2^-24, and the second pass sums non-negative terms, so sigma is relative-accurate to the same
    order.  c = 4.  There is no (mu / sigma)^2 term: that is what a one-pass E[x^2] - mu^2 variance would add.  The affine part adds
    2^-23 (|gamma y| + |beta|), the fp16 store 2^-11 |ref| + 2^-24."""
    D = d_norm
    xs = x[:, :d_norm]
    mu = xs.mean(1, keepdims=True)
    sig = np.sqrt(((xs - mu) ** 2).mean(1, keepdims=True))
    y = (x - mu) / sig
    E = np.abs(gamma) * LN_C * D * U32 * (1 + np.abs(y)) + 2.0 ** -23 * (np.abs(gamma * y) + np.abs(beta))
    return U16 * np.abs(ref) + (1 + U16) * E + U32


# ---------------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------------
def conv_ref(x, w, b, s, pad, act, r=None, res="none", alpha=1.0, slope=LEAKY):
    """float64 conv + bias (+ residual before / after the activation); returns (ref, S, pre-activation, alpha * r)."""
    xt, wt = torch.from_numpy(x), torch.from_numpy(w)
    acc = F.conv2d(xt, wt, None, stride=s, padding=pad).numpy()
    S = F.conv2d(xt.abs(), wt.abs(), None, stride=s, padding=pad).numpy() + np.abs(b)[None, :, None, None]
    a = acc + b[None, :, None, None]
    if res == "pre":
        a = a + r
        S = S + np.abs(r)
    y = act64(a, act, slope)
    rp = None
    if res == "post":
        rp = alpha * r
        y = y + rp
    return y, S, a, rp


# ---------------------------------------------------------------------------------------------------------------------------
# case table
# ---------------------------------------------------------------------------------------------------------------------------
# res: None, "pre" (before the activation), "post" (after it) or a float alpha (after it, scaled).  *_off: channel offset of the
# operand in a wider buffer (None: a buffer of its own).  route: 1x1 | slab | tap (per-tap loads, no_slab) | s2 | im2col8 | im2col4
GEMM_CASES = [
    # B  Cin Cout H   W  k  s act res    f32    in_off out_off res_off route
    (3, 64, 80, 9, 15, 1, 1, 1, None, False, 24, 40, None, "1x1"),       # Kc = 64, ragged M, N = 80
    (2, 72, 24, 7, 13, 1, 1, 2, "pre", False, 40, 24, 64, "1x1"),        # Kc % 64 = 8, residual before ReLU, N = 24
    (2, 104, 8, 5, 11, 1, 1, 3, "post", False, 0, 24, 40, "1x1"),        # Kc % 64 = 40, LeakyReLU, N = 8
    (2, 128, 320, 6, 9, 1, 1, 0, 0.7, False, 24, 0, 24, "1x1"),          # N = 320, scaled residual alpha = 0.7
    (1, 64, 24, 10, 10, 1, 1, 0, None, True, 40, 8, None, "1x1"),        # fp32 output slice
    (3, 64, 64, 3, 5, 3, 1, 1, "post", False, 64, 24, 40, "slab"),       # input coff 64 * 1, B 3 of 5
    (3, 128, 48, 1, 7, 3, 1, 2, "pre", False, 24, 0, 24, "tap"),         # H = 1, input coff 8 * 3, per-tap loads
    (3, 64, 32, 2, 2, 3, 1, 3, None, False, 40, 8, None, "slab"),        # 2 x 2 map
    (2, 64, 48, 10, 14, 3, 2, 3, None, False, 24, None, None, "s2"),     # stride 2, odd output W (7)
    (2, 128, 64, 8, 6, 1, 2, 3, "post", False, 40, 24, 8, "s2"),         # 1x1 stride 2, output W 3
    (2, 16, 32, 9, 11, 3, 2, 1, None, False, 24, 8, None, "im2col8"),    # 8-channel gather, k 3 s 2
    (2, 24, 16, 7, 9, 5, 1, 2, None, False, 8, None, None, "im2col8"),   # k 5 s 1
    (1, 40, 24, 8, 8, 3, 2, 0, "post", False, 40, 24, 8, "im2col8"),     # Cin 40, residual
    (2, 4, 24, 9, 10, 3, 2, 1, None, False, 24, None, None, "im2col4"),  # 4-channel gather (Cout 24: not a stem shape)
    (2, 12, 24, 7, 7, 3, 1, 2, None, False, 8, 8, None, "im2col4"),      # Cin 12
]

NSTORE_CASES = [(False,), (True,)]       # Cout 70 (n_store 72) at channel 24 of a 112-channel buffer, without / with a residual

UP2_CASES = [
    # B Cin Cout H  W out_off
    (2, 16, 8, 3, 5, 24),
    (3, 64, 136, 5, 3, 8),
]

FC_CASES = [
    # B   K     N     act f32
    (17, 4096, 3203, 1, True),       # swap-AB on tensor cores (26 MB of weights), BN 32
    (33, 4096, 3203, 3, False),      # BN 48
    (9, 4992, 1003, 2, False),       # fc_stream, two blockIdx.y rows of 8 images
    (16, 4992, 1003, 1, True),
    (31, 4992, 1003, 0, False),
]

MAXPOOL_CASES = [
    # B C    H  W  k s p in_off out_off
    (2, 8, 7, 9, 2, 2, 0, 24, 40),
    (3, 264, 5, 7, 3, 2, 1, 8, 24),
    (2, 8, 9, 11, 5, 1, 2, 40, 0),
    (2, 264, 6, 5, 3, 1, 1, None, 24),
]

UPSAMPLE_CASES = [
    # B C H W in_off out_off
    (2, 8, 1, 7, 24, 40),
    (3, 8, 7, 1, None, 8),
    (2, 8, 7, 7, 40, None),
]

AVGPOOL_CASES = [(3, 16, 6, 8, 24, 40, 0), (2, 8, 4, 6, 8, None, 1)]          # B C H W in_off out_off fill

DWCONV_CASES = [
    # B C  H W k s act in_off out_off res_off
    (2, 24, 7, 9, 3, 1, 1, 24, 8, 40),
    (3, 16, 8, 6, 3, 2, 0, 40, None, None),
    (2, 8, 9, 9, 7, 1, 1, 8, 24, None),
]

ATTN_CASES = [
    # B nh kdp hd  H W scale in_off out_off
    (2, 1, 64, 128, 5, 13, 0.125, 24, 8),      # N = 65: a second key tile with one key
    (2, 2, 16, 32, 1, 1, 0.25, 8, None),       # N = 1
    (3, 1, 32, 64, 1, 5, 0.18, 40, 24),        # N = 5
    (2, 2, 64, 128, 4, 4, 0.125, None, 40),    # N = 16
    (2, 1, 16, 16, 3, 3, None, 24, 8),         # sharp softmax: scale chosen so that max logit - next >= 20
]

STEM_CASES = [
    # kind   B H   W   k s pad cout act out_off
    ("stemconv", 2, 18, 26, 3, 2, 1, 32, 1, 24),
    ("stemconv", 3, 16, 20, 6, 2, 2, 16, 2, None),
    ("stem7x7s2", 2, 16, 24, 7, 2, 3, 64, 2, None),
]

LN_CASES = [
    # B  d_len d_norm mean/std
    (1, 4992, 4000, 0.0),
    (3, 4992, 4000, 10.0),
    (32, 4992, 4000, 200.0),
    (3, 1000, 1000, 200.0),
]


# ---------------------------------------------------------------------------------------------------------------------------
# builders: case tuple -> Spec
# ---------------------------------------------------------------------------------------------------------------------------
def gemm_spec(case, seed=0) -> Spec:
    B, cin, cout, H, W, k, s, act, res, f32, in_off, out_off, res_off, route = case
    rng = np.random.default_rng(seed)
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
    xv = view(pb, H, W, cin, in_off)
    ov = None if out_off is None else view(pb, Ho, Wo, cout, out_off, f32=f32)
    rv = None if res is None else view(pb, Ho, Wo, cout, res_off)
    x = f16(rng, (B, cin, H, W))
    w = f16(rng, (cout, cin, k, k), np.sqrt(2.0 / (cin * k * k)))
    b = f16(rng, cout, 0.1).astype(np.float32).astype(np.float64)
    r = f16(rng, (B, cout, Ho, Wo)) if res is not None else None
    alpha = float(np.float32(res)) if isinstance(res, float) else 1.0
    kind = "none" if res is None else ("pre" if res == "pre" else "post")
    o = pb.conv(xv, w.astype(np.float32), b.astype(np.float32), k, s, act, out=ov, res=rv, res_pre_act=(kind == "pre"), out_f32=f32,
                res_scale=res if isinstance(res, float) else None, tile=(64, 2) if route == "slab" else None, no_slab=(route == "tap"))
    ref, S, a, rp = conv_ref(x, w, b, s, pad, act, r, kind, alpha)
    K = k * k * r8(xv.C)
    ins = [(xv.buf, xv.coff, x)] + ([(rv.buf, rv.coff, r)] if rv is not None else [])
    return Spec(pb, B, ins, (o.buf, o.coff, cout), ref, gemm_bound(ref, S, K, act, a, rp, f32), route, simt=True)


def nstore_spec(case, seed=0) -> Spec:
    """Cout = 70 (n_store 72) at channel 24 of a 112-channel buffer: the conv owns channels [24, 96), channels [94, 96) hold exact
    zeros and everything else stays untouched.  The residual owns 72 channels too, zero past 70 (as a conv of Cout 70 leaves them);
    the channels past its 72 are poisoned."""
    (with_res,) = case
    rng = np.random.default_rng(seed)
    B, cin, cout, H, W = 2, 64, 70, 5, 9
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
    xv = view(pb, H, W, cin, 8)
    ov = pb.sub(pb.new_padded(H, W, 112), 24, cout)
    rv = pb.sub(pb.new_padded(H, W, 120), 40, cout) if with_res else None
    x = f16(rng, (B, cin, H, W))
    w = f16(rng, (cout, cin, 1, 1), np.sqrt(2.0 / cin))
    b = f16(rng, cout, 0.1)
    r = f16(rng, (B, cout, H, W)) if with_res else None
    o = pb.conv(xv, w.astype(np.float32), b.astype(np.float32), 1, 1, 1, out=ov, res=rv)
    ref, S, a, rp = conv_ref(x, w, b, 1, 0, 1, r, "post" if with_res else "none")
    zeros = np.zeros((B, r8(cout) - cout, H, W))
    ref, S, a = (np.concatenate([t, zeros], 1) for t in (ref, S, a))
    ins = [(xv.buf, xv.coff, x)]
    if with_res:
        rp = np.concatenate([rp, zeros], 1)
        ins.append((rv.buf, rv.coff, np.concatenate([r, zeros], 1)))
    return Spec(pb, B, ins, (o.buf, o.coff, r8(cout)), ref, gemm_bound(ref, S, r8(cin), 1, a, rp), "1x1", simt=True)


def up2_spec(case, seed=0) -> Spec:
    B, cin, cout, H, W, out_off = case
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV6, 3, H, W)
    xv = view(pb, H, W, cin, 0)
    ov = view(pb, 2 * H, 2 * W, cout, out_off)
    x = f16(rng, (B, cin, H, W))
    w = f16(rng, (cin, cout, 2, 2), np.sqrt(1.0 / cin))
    b = f16(rng, cout, 0.1)
    o = pb.conv_transpose2x2(xv, w.astype(np.float32), b.astype(np.float32), ov)
    xt, wt = torch.from_numpy(x), torch.from_numpy(w)
    ref = F.conv_transpose2d(xt, wt, torch.from_numpy(b), stride=2).numpy()
    S = F.conv_transpose2d(xt.abs(), wt.abs(), torch.from_numpy(np.abs(b)), stride=2).numpy()
    return Spec(pb, B, [(xv.buf, xv.coff, x)], (o.buf, o.coff, cout), ref, gemm_bound(ref, S, r8(cin), 0, ref), "up2", simt=True)


def fc_route(K: int, N: int) -> str:
    return "fc_stream" if N * K * 2 <= FC_STREAM_MAX_BYTES else "tr"


def fc_spec(case, seed=0) -> Spec:
    B, K, N, act, f32 = case
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_UFLDV2, 3, 8, 8)
    xin = pb.new_dense(1, K + 16)                       # the 16 entries past K must not be read
    out = pb.new_dense(1, r8(N) + 16, f32=f32)          # nor anything past N written
    x = f16(rng, (B, K))
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float16)
    b = f16(rng, N, 0.1)
    pb.fc(xin, K, w, b.astype(np.float32), act, out)
    w64 = w.astype(np.float64)
    a = x @ w64.T + b
    S = np.abs(x) @ np.abs(w64).T + np.abs(b)
    ref = act64(a, act)
    return Spec(pb, B, [(xin, 0, x)], (out, 0, N), ref, gemm_bound(ref, S, K, act, a, None, f32), fc_route(K, N), simt=True)


def maxpool_spec(case, seed=0) -> Spec:
    B, C, H, W, k, s, p, in_off, out_off = case
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
    xv = view(pb, H, W, C, in_off)
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    ov = None if out_off is None else view(pb, Ho, Wo, C, out_off)
    o = pb.maxpool(xv, k, s, p, out=ov)
    x = f16(rng, (B, C, H, W))
    ref = F.max_pool2d(torch.from_numpy(x), k, s, p).numpy()
    return Spec(pb, B, [(xv.buf, xv.coff, x)], (o.buf, o.coff, C), ref, None, "maxpool", poison=INF16)


def upsample_spec(case, seed=0) -> Spec:
    B, C, H, W, in_off, out_off = case
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
    xv = view(pb, H, W, C, in_off)
    ov = view(pb, 2 * H, 2 * W, C, out_off)
    o = pb.upsample2x(xv, ov)
    x = f16(rng, (B, C, H, W))
    ref = x.repeat(2, 2).repeat(2, 3)
    return Spec(pb, B, [(xv.buf, xv.coff, x)], (o.buf, o.coff, C), ref, None, "upsample")


def avgpool_spec(case, seed=0) -> Spec:
    B, C, H, W, in_off, out_off, fill = case
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    xv = view(pb, H, W, C, in_off)
    ov = None if out_off is None else view(pb, H, W, C, out_off)
    o = pb.avgpool2(xv, fill, out=ov)
    x = f16(rng, (B, C, H, W))
    xf = x.astype(np.float32)                                 # the kernel's fp32 order: ((a + b) + (c + d)) * 0.25, one rounding
    m = (((xf[:, :, :-1, :-1] + xf[:, :, :-1, 1:]) + (xf[:, :, 1:, :-1] + xf[:, :, 1:, 1:])) * np.float32(0.25)).astype(np.float16)
    ref = np.full((B, C, H, W), -np.inf if fill else 0.0)
    ref[:, :, :-1, :-1] = m
    return Spec(pb, B, [(xv.buf, xv.coff, x)], (o.buf, o.coff, C), ref, None, "avgpool2")


def dwconv_spec(case, seed=0) -> Spec:
    B, C, H, W, k, s, act, in_off, out_off, res_off = case
    rng = np.random.default_rng(seed)
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    xv = view(pb, H, W, C, in_off)
    ov = None if out_off is None else view(pb, Ho, Wo, C, out_off)
    rv = None if res_off is None else view(pb, Ho, Wo, C, res_off)
    x = f16(rng, (B, C, H, W))
    w = f16(rng, (C, 1, k, k), np.sqrt(2.0 / (k * k)))
    b = f16(rng, C, 0.1)
    r = f16(rng, (B, C, Ho, Wo)) if rv is not None else None
    o = pb.dwconv(xv, w.astype(np.float32), b.astype(np.float32), k, s, act, out=ov, res=rv)
    xt, wt = torch.from_numpy(x), torch.from_numpy(w)
    a = F.conv2d(xt, wt, torch.from_numpy(b), stride=s, padding=pad, groups=C).numpy()
    S = F.conv2d(xt.abs(), wt.abs(), torch.from_numpy(np.abs(b)), stride=s, padding=pad, groups=C).numpy()
    ref = act64(a, act) + (r if r is not None else 0.0)
    ins = [(xv.buf, xv.coff, x)] + ([(rv.buf, rv.coff, r)] if rv is not None else [])
    return Spec(pb, B, ins, (o.buf, o.coff, C), ref, gemm_bound(ref, S, k * k, act, a, r), "dwconv")


def attention_ref(qkv, nh, kdp, hd, scale):
    """qkv [B, nh*(2kdp+hd), H, W] float64 -> (ref [B, nh*hd, H, W], bound)."""
    B, _, H, W = qkv.shape
    t = qkv.reshape(B, -1, H * W).transpose(0, 2, 1)             # [B, N, C]
    ref = np.zeros((B, H * W, nh * hd))
    bnd = np.zeros_like(ref)
    for bi in range(B):
        for h in range(nh):
            q = t[bi, :, h * kdp:(h + 1) * kdp]
            k = t[bi, :, (nh + h) * kdp:(nh + h + 1) * kdp]
            v = t[bi, :, 2 * nh * kdp + h * hd:2 * nh * kdp + (h + 1) * hd]
            s = q @ k.T * scale
            P = np.exp(s - s.max(1, keepdims=True))
            P /= P.sum(1, keepdims=True)
            o = P @ v
            ref[bi, :, h * hd:(h + 1) * hd] = o
            bnd[bi, :, h * hd:(h + 1) * hd] = attention_bound(q, k, v, scale, o)
    back = lambda a: a.transpose(0, 2, 1).reshape(B, nh * hd, H, W)
    return back(ref), back(bnd)


def sharp_scale(qkv, nh, kdp):
    """The smallest scale at which every query's largest logit leads the next by >= 20."""
    B, _, H, W = qkv.shape
    t = qkv.reshape(B, -1, H * W).transpose(0, 2, 1)
    gap = np.inf
    for bi in range(B):
        for h in range(nh):
            s = t[bi, :, h * kdp:(h + 1) * kdp] @ t[bi, :, (nh + h) * kdp:(nh + h + 1) * kdp].T
            s.sort(1)
            gap = min(gap, float((s[:, -1] - s[:, -2]).min()))
    return 20.0 / gap


def attention_spec(case, seed=0) -> Spec:
    B, nh, kdp, hd, H, W, scale, in_off, out_off = case
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, H, W)
    cin = nh * (2 * kdp + hd)
    xv = view(pb, H, W, cin, in_off)
    ov = None if out_off is None else view(pb, H, W, nh * hd, out_off)
    qkv = f16(rng, (B, cin, H, W))
    if scale is None:
        scale = float(np.float32(sharp_scale(qkv, nh, kdp)))
    o = pb.attention(xv, nh, kdp, hd, scale, out=ov)
    ref, bnd = attention_ref(qkv, nh, kdp, hd, float(np.float32(scale)))
    return Spec(pb, B, [(xv.buf, xv.coff, qkv)], (o.buf, o.coff, nh * hd), ref, bnd, "attention")


def stem_spec(case, seed=0) -> Spec:
    kind, B, H, W, k, s, pad, cout, act, out_off = case
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8 if kind == "stemconv" else plan.MODEL_UFLDV2, 3, H, W)
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    x = np.zeros((B, 4, H, W))
    x[:, :3] = f16(rng, (B, 3, H, W))                          # the image's 4th channel is a structural zero
    w = f16(rng, (cout, 3, k, k), np.sqrt(2.0 / (3 * k * k)))
    b = f16(rng, cout, 0.1)
    if kind == "stemconv":
        ov = None if out_off is None else view(pb, Ho, Wo, cout, out_off)
        o = pb.conv(pb.image, w.astype(np.float32), b.astype(np.float32), k, s, act, pad=pad, out=ov)
    else:
        o = pb.stem7x7s2(pb.image, w.astype(np.float32), b.astype(np.float32), act)
    ref, S, a, _ = conv_ref(x[:, :3], w, b, s, pad, act)
    return Spec(pb, B, [(pb.image.buf, 0, x)], (o.buf, o.coff, cout), ref, gemm_bound(ref, S, k * k * 4, act, a), kind,
                simt=(kind == "stem7x7s2"))


def layernorm_spec(case, seed=0) -> Spec:
    B, d_len, d_norm, ratio = case
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_UFLDV2, 3, 8, 8)
    xin = pb.new_dense(1, d_len + 8)
    out = pb.new_dense(1, d_len + 8)
    x = np.zeros((B, d_len))
    x[:, :d_norm] = f16(rng, (B, d_norm), 1.0, ratio)           # std 1, mean `ratio`; entries past d_norm are structural zeros
    gamma = np.zeros(d_len); beta = np.zeros(d_len)
    gamma[:d_norm] = (1.0 + 0.1 * rng.standard_normal(d_norm)).astype(np.float32)
    beta[:d_norm] = (0.1 * rng.standard_normal(d_norm)).astype(np.float32)
    eps = 1e-5
    pb.layernorm(xin, d_len, d_norm, gamma, beta, eps, out)
    xs = x[:, :d_norm]
    mu = xs.mean(1, keepdims=True)
    var = ((xs - mu) ** 2).mean(1, keepdims=True)
    ref = (x - mu) / np.sqrt(var + float(np.float32(eps))) * gamma + beta
    return Spec(pb, B, [(xin, 0, x)], (out, 0, d_len), ref, layernorm_bound(x, gamma, beta, d_norm, ref), "layernorm")


ALL = ([("gemm", c, gemm_spec) for c in GEMM_CASES] + [("nstore", c, nstore_spec) for c in NSTORE_CASES]
       + [("up2", c, up2_spec) for c in UP2_CASES] + [("fc", c, fc_spec) for c in FC_CASES]
       + [("maxpool", c, maxpool_spec) for c in MAXPOOL_CASES] + [("upsample", c, upsample_spec) for c in UPSAMPLE_CASES]
       + [("avgpool2", c, avgpool_spec) for c in AVGPOOL_CASES] + [("dwconv", c, dwconv_spec) for c in DWCONV_CASES]
       + [("attention", c, attention_spec) for c in ATTN_CASES] + [("stem", c, stem_spec) for c in STEM_CASES]
       + [("layernorm", c, layernorm_spec) for c in LN_CASES])


def case_id(family, case) -> str:
    return family + "-" + "-".join(str(v) for v in case)


def plan_route(spec: Spec) -> Optional[str]:
    """The route the packed op list takes, read from the plan alone (None: no recognised route)."""
    ops = spec.pb.ops
    types = [t for t, _, _ in ops]
    gemms = [p for t, p, _ in ops if t == plan.OP_GEMM]
    if plan.OP_IM2COL in types:
        cin = [p for t, p, _ in ops if t == plan.OP_IM2COL][0].Cin
        return "im2col4" if cin % 8 == 4 else "im2col8"
    if plan.OP_STEMCONV in types:
        return "stemconv"
    if plan.OP_STEMPACK in types:
        return "stem7x7s2" if len(gemms) == 1 and gemms[0].ntaps == 4 else None
    if len(gemms) == 1:
        p = gemms[0]
        if p.transposed:
            return fc_route(p.Kc, p.N)
        if p.up2:
            return "up2"
        if p.s2:
            return "s2"
        if p.ntaps == 9:
            return "tap" if p.no_slab else "slab"
        if p.ntaps == 1:
            return "1x1"
        return None
    single = (plan.OP_MAXPOOL, plan.OP_UPSAMPLE2X, plan.OP_AVGPOOL2, plan.OP_DWCONV, plan.OP_ATTN, plan.OP_LAYERNORM)
    return plan.OP_NAMES[types[0]] if len(types) == 1 and types[0] in single else None
