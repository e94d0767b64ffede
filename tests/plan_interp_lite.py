"""plan_interp.py with YOLOv6-Lite's ops: Hardswish (activation code 5) in the GEMM, stem-conv and depthwise references and their error
bounds, OP_SE (squeeze-excite) and OP_SHUFFLE2 (concat + channel shuffle): their regions, float64 references with per-element bounds,
and every plan_interp function that walks a plan, so YOLOv6-Lite plans go through the same dataflow, interpreter and per-op checks as
every other network.

`extended()` is a context in which plan_interp itself knows them (plan_interp._act treats an unknown code as the identity, so Hardswish
has to be supplied here), and so do op_conformance_cases.act64 / gemm_bound (the single-layer sweeps of tile_space_cases); outside it both
modules are unchanged, as with plan_interp_cbfuse."""
import contextlib

import numpy as np
import torch

import op_conformance_cases as oc
import plan_interp as pi
from adas_b200 import plan

U16, U32 = oc.U16, oc.U32
_base_gemm_bound = oc.gemm_bound


def hardswish(a):
    """x * clamp(x + 3, 0, 6) / 6 (torch.nn.Hardswish), on tensors or arrays."""
    if isinstance(a, torch.Tensor):
        return a * torch.clamp(a + 3.0, 0.0, 6.0) / 6.0
    return a * np.clip(a + 3.0, 0.0, 6.0) / 6.0


def hardswish_bound(ref, S, K, a, res_post=None, out_f32=False):
    """oc.gemm_bound for Hardswish.  Its Lipschitz constant is 1.5 (slope (2x + 3) / 6 on [-3, 3], 0 or 1 outside), so the accumulation
    error (K 2^-23 S) grows by 1.5; the fp32 evaluation -- x + 3, the clamp (exact), the product with x and the product with fp32(1/6)
    -- adds four roundings of at most |x| (|x| + 3) / 6 each (which bounds |x + 3| |x| / 6 and every intermediate): 2^-21 |x| (|x| + 3) / 6.
    Expressed through gemm_bound's activation-free form with S scaled to carry both terms."""
    a = np.abs(a)
    E = 1.5 * K * 2.0 ** -23 * S + 2.0 ** -21 * a * (a + 3.0) / 6.0
    return _base_gemm_bound(ref, E / (K * 2.0 ** -23), K, 0, a, res_post, out_f32)


def _se_regions(p):
    C = p[2]
    return [pi.Region(p[8], p[9], p[9] + C)], [pi.Region(p[0], p[1], p[1] + C)]


def _se_ref(pb, p, bufs, B, dev, want_bound):
    """x * hardsigmoid(W2 relu(W1 mean(x) + b1) + b2) per image, and its bound.  The kernel (lite_ops.cu): the mean is an fp32 sum of HW
    terms and a division, within (HW + 1) 2^-24 mean|x|; each FC is an fp32 dot product with a bias, within n 2^-24 (|b| + sum |w| |v|)
    of its fp32 inputs plus the propagated input error (ReLU: Lipschitz 1); hardsigmoid (Lipschitz 1/6, then + 3 and / 6 in fp32) adds
    2^-23; the product x * g adds 2^-24 |x g|; the fp16 store 2^-11 |ref| + 2^-24.  Each 2^-24 is doubled below for margin."""
    in_buf, coff, C, hid = p[:4]
    w1, b1, w2, b2 = (pb.tensors[t].astype(np.float64) for t in p[4:8])
    w1, w2 = w1.reshape(hid, C), w2.reshape(C, hid)
    refs, bnds = [], []
    for b in range(B):
        x = pi._np(pi.image_view(pb, bufs, in_buf, b, coff, coff + C, dev))[0]        # [C, H, W]
        HW = x.shape[1] * x.shape[2]
        m = x.reshape(C, HW).mean(1)
        pre_h = b1 + w1 @ m
        h = np.maximum(pre_h, 0.0)
        pre_g = b2 + w2 @ h
        g = np.clip(pre_g + 3.0, 0.0, 6.0) / 6.0
        y = x * g[:, None, None]
        refs.append(y[None])
        if want_bound:
            u = 2.0 ** -23
            dm = (HW + 1) * u * np.abs(x).reshape(C, HW).mean(1)
            dh = np.abs(w1) @ dm + C * u * (np.abs(b1) + np.abs(w1) @ np.abs(m))
            dg = (np.abs(w2) @ dh + hid * u * (np.abs(b2) + np.abs(w2) @ np.abs(h))) / 6.0 + u
            E = np.abs(x) * dg[:, None, None] + u * np.abs(y)
            bnds.append((U16 * np.abs(y) + (1 + U16) * E + U32)[None])
    return np.concatenate(refs), (np.concatenate(bnds) if want_bound else None)


def _shuffle2_regions(p):
    n = p[4]
    return [pi.Region(p[5], p[6], p[6] + 2 * n)], [pi.Region(p[0], p[1], p[1] + n), pi.Region(p[2], p[3], p[3] + n)]


def _shuffle2_ref(pb, p, bufs, B, dev):
    n = p[4]
    res = []
    for b in range(B):
        a = pi.image_view(pb, bufs, p[0], b, p[1], p[1] + n, dev)
        c = pi.image_view(pb, bufs, p[2], b, p[3], p[3] + n, dev)
        res.append(pi._np(torch.stack([a, c], 2).reshape(1, 2 * n, a.shape[2], a.shape[3])))
    return np.concatenate(res)


@contextlib.contextmanager
def extended():
    base_regions, base_ref, base_act, base_bound, base_act64 = pi.op_regions, pi.op_ref, pi._act, oc.gemm_bound, oc.act64
    names = {plan.OP_SE: "se", plan.OP_SHUFFLE2: "shuffle2"}
    had = {t: t in pi.OP_NAMES for t in names}

    def op_regions(pb, i):
        t, p, _ = pb.ops[i]
        if t == plan.OP_SE:
            return _se_regions(p)
        if t == plan.OP_SHUFFLE2:
            return _shuffle2_regions(p)
        return base_regions(pb, i)

    def op_ref(pb, i, bufs, B, device="cpu", want_bound=True):
        t, p, _ = pb.ops[i]
        if t not in names:
            return base_ref(pb, i, bufs, B, device=device, want_bound=want_bound)
        with torch.no_grad():
            if t == plan.OP_SE:
                return _se_ref(pb, p, bufs, B, torch.device(device), want_bound)
            return _shuffle2_ref(pb, p, bufs, B, torch.device(device)), None

    def act(a, code):
        return hardswish(a) if code == plan.ACT_HSWISH else base_act(a, code)

    def act64(a, code, *args, **kw):
        return hardswish(a) if code == plan.ACT_HSWISH else base_act64(a, code, *args, **kw)

    def gemm_bound(ref, S, K, code, a, res_post=None, out_f32=False):
        if code == plan.ACT_HSWISH:
            return hardswish_bound(ref, S, K, a, res_post, out_f32)
        return base_bound(ref, S, K, code, a, res_post, out_f32)

    pi.op_regions, pi.op_ref, pi._act, oc.gemm_bound, oc.act64 = op_regions, op_ref, act, gemm_bound, act64
    pi.OP_NAMES.update(names)
    try:
        yield pi
    finally:
        pi.op_regions, pi.op_ref, pi._act, oc.gemm_bound, oc.act64 = base_regions, base_ref, base_act, base_bound, base_act64
        for t, h in had.items():
            if not h:
                del pi.OP_NAMES[t]


def _within(name):
    f = getattr(pi, name)

    def g(*a, **kw):
        with extended():
            return getattr(pi, name)(*a, **kw)
    g.__name__, g.__doc__ = name, f.__doc__
    return g


op_regions, op_ref, op_kind, out_region, read_out, write_out = map(_within, ("op_regions", "op_ref", "op_kind", "out_region", "read_out", "write_out"))
dataflow_violations, stale_reads, overwritten, interpret = map(_within, ("dataflow_violations", "stale_reads", "overwritten", "interpret"))
excess, new_buffers, geom = pi.excess, pi.new_buffers, pi.geom
