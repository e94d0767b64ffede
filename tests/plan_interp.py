"""A float64 reference of every packed plan op, and the dataflow of a plan (which op writes and reads which buffer region).

`op_ref(pb, i, bufs, B)` computes what op i of a `PlanBuilder` must write, from that op's own input buffers as the device left them
(`bufs[buf]`: the [mb * rows_per_img, C] array read back after a run, mb >= B), so each op is checked on its own and bounds do not
compound through the network.  It returns the reference and the per-element bound of op_conformance_cases (None: the op must be
bit-exact), in the layout `read_out(pb, i, bufs, B)` extracts from the buffers.  References are torch float64 convolutions and matrix
products, one image at a time, on `device`.

`op_regions(pb, i)` gives op i's write and read regions: (buffer, lo, hi) channel ranges of every row of a padded buffer, or element
ranges of the per-image slab of a dense one.  A GEMM reads the same channels at every tap, so the region is the same for every
route.  `dataflow_violations(pb)` lists overlapping writes and reads of regions no earlier op wrote; a read-back buffer equals what its
consumer saw only if the plan has neither.

`interpret(pb, image, B)` chains op_ref from the image through the whole plan (the CPU check that the interpreter reads the packed
layouts the way the networks mean them)."""
from typing import Dict, List, NamedTuple, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

import op_conformance_cases as oc
from adas_b200 import plan


class Region(NamedTuple):
    buf: int
    lo: int
    hi: int


def geom(pb, buf):
    rows, C, dtype, H, W, _ = pb.buffers[buf]
    return rows, C, dtype, H, W


def _flat(pb, buf, lo, hi) -> Region:
    """A read of per-image slab elements [lo, hi): on a padded buffer, every channel (an FC or LayerNorm reads the whole slab; the halo
    entries are zero by contract)."""
    rows, C, _, H, _ = geom(pb, buf)
    return Region(buf, 0, C) if H > 0 else Region(buf, lo, hi)


def gemm_route(p) -> str:
    """The GEMM route of a packed op (the names of op_conformance_cases.plan_route)."""
    if p.transposed:
        return oc.fc_route(p.Kc, p.N)
    if p.up2:
        return "up2"
    if p.s2:
        return "s2"
    if p.ntaps == 9:
        return "9tap"
    if p.ntaps == 4:
        return "stem7x7s2"
    return "1x1"


def op_kind(pb, i) -> str:
    """A name for the op's type and route: "gemm-1x1", "gemm-9tap", ..., "maxpool", ..."""
    t, p, _ = pb.ops[i]
    if t == plan.OP_GEMM:
        return "gemm-" + gemm_route(p)
    return plan.OP_NAMES[t]


def op_regions(pb, i) -> Tuple[List[Region], List[Region]]:
    """(writes, reads) of op i.  An in-place CBFuse or SE reads its own write region."""
    t, p, _ = pb.ops[i]
    if t == plan.OP_GEMM:
        a, acoff, Kc, N, out, ocoff = p.a_buf, p.a_coff, p.Kc, p.N, p.out_buf, p.out_coff
        if p.transposed:
            return [Region(out, ocoff, ocoff + N)], [_flat(pb, a, 0, Kc)]
        reads = [Region(a, acoff, acoff + Kc)] + ([Region(p.res_buf, p.res_coff, p.res_coff + N)] if p.res_buf >= 0 else [])
        return [Region(out, ocoff, ocoff + (N // 4 if p.up2 else N))], reads
    if t == plan.OP_IM2COL:      # owns its whole patch buffer: columns past kh * kw * Cin stay zero, and meet zero weights
        return [Region(p.out_buf, 0, geom(pb, p.out_buf)[1])], [Region(p.in_buf, p.in_coff, p.in_coff + p.Cin)]
    if t in (plan.OP_MAXPOOL, plan.OP_UPSAMPLE2X, plan.OP_AVGPOOL2):
        return [Region(p.out_buf, p.out_coff, p.out_coff + p.C)], [Region(p.in_buf, p.in_coff, p.in_coff + p.C)]
    if t == plan.OP_STEMPACK:
        return [Region(p.out_buf, 0, 64)], [Region(p.in_buf, 0, 4)]
    if t == plan.OP_STEMCONV:
        return [Region(p.out_buf, p.out_coff, p.out_coff + p.Cout)], [Region(p.in_buf, 0, 4)]
    if t == plan.OP_LAYERNORM:
        return [Region(p.out_buf, 0, p.d_len)], [_flat(pb, p.in_buf, 0, p.d_len)]
    if t == plan.OP_DWCONV:
        C = p.C
        return ([Region(p.out_buf, p.out_coff, p.out_coff + C)],
                [Region(p.in_buf, p.in_coff, p.in_coff + C)] + ([Region(p.res_buf, p.res_coff, p.res_coff + C)] if p.res_buf >= 0 else []))
    if t == plan.OP_ATTN:
        nh, kdp, hd = p.nh, p.kdp, p.hd
        return [Region(p.out_buf, p.out_coff, p.out_coff + nh * hd)], [Region(p.in_buf, p.in_coff, p.in_coff + nh * (2 * kdp + hd))]
    if t == plan.OP_CBFUSE:
        C = p.C
        return ([Region(p.out_buf, p.out_coff, p.out_coff + C)],
                [Region(p.base_buf, p.base_coff, p.base_coff + C)] + [Region(q[0], q[1], q[1] + C) for q in plan.cbfuse_sources(p)])
    if t == plan.OP_SE:
        return [Region(p.out_buf, p.out_coff, p.out_coff + p.C)], [Region(p.in_buf, p.in_coff, p.in_coff + p.C)]
    if t == plan.OP_SHUFFLE2:
        n = p.n
        return [Region(p.out_buf, p.out_coff, p.out_coff + 2 * n)], [Region(p.a_buf, p.a_coff, p.a_coff + n), Region(p.b_buf, p.b_coff, p.b_coff + n)]
    raise ValueError(f"op {i}: unknown type {t}")


def _overlap(a: Region, b: Region) -> bool:
    return a.buf == b.buf and a.lo < b.hi and b.lo < a.hi


def dataflow_violations(pb) -> List[str]:
    """Overlapping writes and reads of regions not written before, as messages."""
    out = []
    written: Dict[int, np.ndarray] = {}
    writers: List[Tuple[int, Region]] = []

    def mask(buf):
        if buf not in written:
            rows, C, _, H, _ = geom(pb, buf)
            written[buf] = np.zeros(C if H > 0 else rows * C, bool)
        return written[buf]

    mask(pb.image.buf)[:4] = True                   # the image: written by pre-processing
    for i in range(len(pb.ops)):
        w, r = op_regions(pb, i)
        msgs = []
        for reg in r:
            m = mask(reg.buf)
            if not m[reg.lo:reg.hi].all():
                miss = np.nonzero(~m[reg.lo:reg.hi])[0] + reg.lo
                msgs.append(f"op {i} ({op_kind(pb, i)}) reads unwritten {reg} (first {int(miss[0])}, {len(miss)} missing)")
        for reg in w:
            for j, o in writers:
                if _overlap(reg, o):
                    msgs.append(f"op {i} ({op_kind(pb, i)}) writes {reg} over op {j}'s {o}")
            mask(reg.buf)[reg.lo:reg.hi] = True
            writers.append((i, reg))
        out += msgs
    return out


def stale_reads(pb) -> Dict[int, List[int]]:
    """op -> later ops that overwrite a region it reads: its inputs can no longer be read back after the run."""
    out: Dict[int, List[int]] = {}
    regs = [op_regions(pb, i) for i in range(len(pb.ops))]
    for i, (_, r) in enumerate(regs):
        later = [j for j in range(i, len(pb.ops)) for w in regs[j][0] if any(_overlap(w, x) for x in r)]
        if later:
            out[i] = later
    return out


def overwritten(pb) -> Dict[int, np.ndarray]:
    """op -> boolean mask over its output region (channels, or dense elements) of the part later ops overwrite."""
    out: Dict[int, np.ndarray] = {}
    regs = [op_regions(pb, i)[0] for i in range(len(pb.ops))]
    for i, (w, *_) in enumerate(regs):
        m = np.zeros(w.hi - w.lo, bool)
        for j in range(i + 1, len(pb.ops)):
            for o in regs[j]:
                if _overlap(w, o):
                    m[max(o.lo, w.lo) - w.lo:min(o.hi, w.hi) - w.lo] = True
        if m.any():
            out[i] = m
    return out


def out_region(pb, i) -> Region:
    return op_regions(pb, i)[0][0]


# ---------------------------------------------------------------------------------------------------------------------------
# buffer access
# ---------------------------------------------------------------------------------------------------------------------------
def _t(a, device) -> torch.Tensor:
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=torch.float64)
    return torch.from_numpy(np.ascontiguousarray(a).astype(np.float64)).to(device)


def image_view(pb, bufs, buf, b, lo, hi, device, halo=False) -> torch.Tensor:
    """Channels [lo, hi) of image b of a padded buffer as [1, c, H(+2), W(+2)] float64."""
    rows, C, _, H, W = geom(pb, buf)
    a = bufs[buf][b * rows:(b + 1) * rows].reshape(H + 2, W + 2, C)
    a = a if halo else a[1:-1, 1:-1]
    return _t(a[:, :, lo:hi], device).permute(2, 0, 1)[None]


def read_out(pb, i, bufs, B) -> np.ndarray:
    """What op i wrote, as float64: [B, c, H, W] interior of a padded output ([B, 64, H + 2, W + 2] for the stem re-layout, which owns
    the top halo row), [B, n] of a dense one."""
    reg = out_region(pb, i)
    rows, C, _, H, W = geom(pb, reg.buf)
    a = bufs[reg.buf][:B * rows]
    if H == 0:
        return a.reshape(B, rows * C)[:, reg.lo:reg.hi].astype(np.float64)
    v = a.reshape(B, H + 2, W + 2, C)
    if pb.ops[i][0] != plan.OP_STEMPACK:
        v = v[:, 1:-1, 1:-1]
    return v[..., reg.lo:reg.hi].astype(np.float64).transpose(0, 3, 1, 2)


def write_out(pb, i, bufs, B, val: np.ndarray) -> None:
    """Store `val` (read_out's layout) into op i's region of bufs, in the buffer's dtype."""
    reg = out_region(pb, i)
    rows, C, _, H, W = geom(pb, reg.buf)
    a = bufs[reg.buf]
    if H == 0:
        a[:B * rows].reshape(B, rows * C)[:, reg.lo:reg.hi] = val
        return
    v = a[:B * rows].reshape(B, H + 2, W + 2, C)
    if pb.ops[i][0] != plan.OP_STEMPACK:
        v = v[:, 1:-1, 1:-1]
    v[..., reg.lo:reg.hi] = val.transpose(0, 2, 3, 1)


def new_buffers(pb, mb, dtype=None) -> Dict[int, np.ndarray]:
    """Zeroed buffers for mb images in their plan dtypes (or all in `dtype`)."""
    return {i: np.zeros((mb * b[0], b[1]), dtype or (np.float32 if b[2] == 1 else np.float16)) for i, b in enumerate(pb.buffers)}


# ---------------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------------
def _act(a: torch.Tensor, act: int) -> torch.Tensor:
    if act == plan.ACT_NONE:
        return a
    if act == 1:
        return a * torch.sigmoid(a)
    if act == 2:
        return torch.clamp_min(a, 0.0)
    if act == 3:
        return torch.where(a >= 0, a, oc.LEAKY * a)
    if act == plan.ACT_HSWISH:
        return a * torch.clamp(a + 3.0, 0.0, 6.0) / 6.0
    raise ValueError(f"unknown activation code {act}")


def _np(t: torch.Tensor) -> np.ndarray:
    return t.detach().cpu().numpy()


def _gemm_conv(pb, p, bufs, b, dev, absval=False):
    """Accumulator [1, N, Ho, Wo] of a non-FC GEMM for image b (the kernel's operand addressing), or of |x| |w| with absval."""
    a, acoff, Kc, ntaps, N = p.a_buf, p.a_coff, p.Kc, p.ntaps, p.N
    w = torch.from_numpy(pb.tensors[p.w_tensor].astype(np.float64)).to(dev)
    f = (lambda t: t.abs()) if absval else (lambda t: t)
    w = f(w)
    if p.up2:                                                     # 2x2 transposed conv: a 1x1 GEMM with columns (dy, dx, c)
        x = f(image_view(pb, bufs, a, b, acoff, acoff + Kc, dev))
        acc = torch.einsum("nk,bkhw->bnhw", w, x)
        co = N // 4
        _, _, H, W = acc.shape
        out = acc.new_zeros((1, co, 2 * H, 2 * W))
        for q in range(4):
            out[:, :, q // 2::2, q % 2::2] = acc[:, q * co:(q + 1) * co]
        return out
    if ntaps == 4:                                                # 7x7 stem: 4 vertical taps over the re-laid-out image rows
        x = f(image_view(pb, bufs, a, b, 0, Kc, dev, halo=True))   # [1, 64, Ho + 2, Wo + 2]
        x = F.pad(x[:, :, :, 1:-1], (0, 0, 1, 0))                  # row -1: the previous image's zero halo / the matrix start
        wk = w.reshape(N, 4, Kc).permute(0, 2, 1)[..., None]       # [N, 64, 4, 1]
        return F.conv2d(x, wk)
    k = 3 if ntaps == 9 else 1
    wk = w.reshape(N, k, k, Kc).permute(0, 3, 1, 2)
    s = 2 if p.s2 else 1
    if k == 3:                                                    # the halo supplies the padding
        return F.conv2d(f(image_view(pb, bufs, a, b, acoff, acoff + Kc, dev, halo=True)), wk, stride=s)
    return F.conv2d(f(image_view(pb, bufs, a, b, acoff, acoff + Kc, dev)), wk, stride=s)


def _gemm_ref(pb, i, bufs, B, dev, want_bound):
    t, p, fl = pb.ops[i]
    N, act = p.N, p.act
    out_f32 = geom(pb, p.out_buf)[2] == 1
    bias = torch.from_numpy(pb.tensors[p.bias_tensor].astype(np.float64)).to(dev) if p.bias_tensor >= 0 else None
    if p.transposed:                                              # FC: one K-vector per image, the whole per-image slab
        rows, C, _, _, _ = geom(pb, p.a_buf)
        x = _t(bufs[p.a_buf][:B * rows].reshape(B, rows * C)[:, :p.Kc], dev)
        w = torch.from_numpy(pb.tensors[p.w_tensor].astype(np.float64)).to(dev)
        a = x @ w.T + (bias if bias is not None else 0.0)
        ref = _act(a, act)
        if not want_bound:
            return _np(ref), None
        S = x.abs() @ w.abs().T + (bias.abs() if bias is not None else 0.0)
        return _np(ref), oc.gemm_bound(_np(ref), _np(S), p.Kc, act, _np(a), None, out_f32)
    refs, bnds = [], []
    alpha = float(np.float32(fl[0])) if fl[0] != 0.0 else 1.0       # f[0] = res_scale
    K = p.ntaps * p.Kc
    for b in range(B):
        acc = _gemm_conv(pb, p, bufs, b, dev)
        bb = bias[None, :, None, None] if bias is not None else 0.0
        if p.up2 and bias is not None:
            bb = bias[:N // 4][None, :, None, None]
        a = acc + bb
        r = None
        if p.res_buf >= 0:
            r = image_view(pb, bufs, p.res_buf, b, p.res_coff, p.res_coff + N, dev)
            if p.res_pre_act:
                a = a + r
        y = _act(a, act)
        rp = None
        if r is not None and not p.res_pre_act:
            rp = alpha * r
            y = y + rp
        refs.append(_np(y))
        if want_bound:
            S = _gemm_conv(pb, p, bufs, b, dev, absval=True) + (bb.abs() if bias is not None else 0.0)
            if r is not None and p.res_pre_act:
                S = S + r.abs()
            bnds.append(oc.gemm_bound(refs[-1], _np(S), p.Kc if p.up2 else K, act, _np(a), None if rp is None else _np(rp), out_f32))
    return np.concatenate(refs), (np.concatenate(bnds) if want_bound else None)


def _im2col_ref(pb, p, bufs, B, dev):
    in_buf, coff, Cin, kh, kw, s, pad = p.in_buf, p.in_coff, p.Cin, p.kh, p.kw, p.stride, p.pad
    _, Kpad, _, Ho, Wo = geom(pb, p.out_buf)
    res = []
    for b in range(B):
        x = F.pad(image_view(pb, bufs, in_buf, b, coff, coff + Cin, dev), (pad, pad + kw, pad, pad + kh))
        cols = [x[:, :, ky:ky + s * (Ho - 1) + 1:s, kx:kx + s * (Wo - 1) + 1:s] for ky in range(kh) for kx in range(kw)]
        y = torch.cat(cols, 1)
        res.append(_np(F.pad(y, (0, 0, 0, 0, 0, Kpad - y.shape[1]))))
    return np.concatenate(res)


def _stempack_ref(pb, p, bufs, B, dev):
    img = p.in_buf
    _, _, _, H, W = geom(pb, img)
    Ho, Wo = H // 2, W // 2
    res = []
    for b in range(B):
        x = F.pad(image_view(pb, bufs, img, b, 0, 4, dev), (3, 4, 1, 1))   # image row y at y + 1, column x at x + 3
        out = x.new_zeros((1, 64, Ho + 2, Wo + 2))
        for pp in range(2):
            for kx in range(7):
                # Q row j, column xo + 1, channels pp*32 + kx*4 + c = img[2j - 1 + pp][2xo + kx - 3][c]
                out[:, pp * 32 + kx * 4:pp * 32 + kx * 4 + 4, :Ho + 1, 1:Wo + 1] = x[:, :, pp:pp + 2 * Ho + 1:2, kx:kx + 2 * Wo - 1:2]
        res.append(_np(out))
    return np.concatenate(res)


def _stemconv_ref(pb, p, bufs, B, dev, want_bound):
    img, wt, bt, cout, k, pad, act = p.in_buf, p.w_tensor, p.bias_tensor, p.Cout, p.k, p.pad, p.act
    s = 2 if p.stride == 0 else p.stride
    KR = (4 * k + 15) // 16 * 16
    wq = pb.tensors[wt].astype(np.float64).reshape(cout, k, KR)[:, :, :4 * k].reshape(cout, k, k, 4)
    w = torch.from_numpy(wq).permute(0, 3, 1, 2).contiguous().to(dev)
    bias = torch.from_numpy(pb.tensors[bt].astype(np.float64)).to(dev) if bt >= 0 else torch.zeros(cout, dtype=torch.float64, device=dev)
    refs, bnds = [], []
    for b in range(B):
        x = image_view(pb, bufs, img, b, 0, 4, dev)
        a = F.conv2d(x, w, stride=s, padding=pad) + bias[None, :, None, None]
        refs.append(_np(_act(a, act)))
        if want_bound:
            S = F.conv2d(x.abs(), w.abs(), stride=s, padding=pad) + bias.abs()[None, :, None, None]
            bnds.append(oc.gemm_bound(refs[-1], _np(S), k * k * 4, act, _np(a)))
    return np.concatenate(refs), (np.concatenate(bnds) if want_bound else None)


def _dwconv_ref(pb, p, bufs, B, dev, want_bound):
    in_buf, coff, C, k, s, act, wt, bt, rb, rcoff = p.in_buf, p.in_coff, p.C, p.k, p.stride, p.act, p.w_tensor, p.bias_tensor, p.res_buf, p.res_coff
    w = torch.from_numpy(pb.tensors[wt].astype(np.float64).T.reshape(C, 1, k, k).copy()).to(dev)
    bias = torch.from_numpy(pb.tensors[bt].astype(np.float64)).to(dev)
    refs, bnds = [], []
    for b in range(B):
        x = image_view(pb, bufs, in_buf, b, coff, coff + C, dev)
        a = F.conv2d(x, w, stride=s, padding=k // 2, groups=C) + bias[None, :, None, None]
        y = _act(a, act)
        r = image_view(pb, bufs, rb, b, rcoff, rcoff + C, dev) if rb >= 0 else None
        if r is not None:
            y = y + r
        refs.append(_np(y))
        if want_bound:
            S = F.conv2d(x.abs(), w.abs(), stride=s, padding=k // 2, groups=C) + bias.abs()[None, :, None, None]
            bnds.append(oc.gemm_bound(refs[-1], _np(S), k * k, act, _np(a), None if r is None else _np(r)))
    return np.concatenate(refs), (np.concatenate(bnds) if want_bound else None)


def _layernorm_ref(pb, p, fl, bufs, B, want_bound):
    """Statistics over the d_norm entries the plan gives a nonzero gamma or beta (the rest are structural zeros, as the kernel counts
    them: mean = sum / d_norm, variance = (sum of (x - mean)^2 - (d_len - d_norm) mean^2) / d_norm)."""
    in_buf, d_len, gt, bt, d_norm = p.in_buf, p.d_len, p.gamma_tensor, p.beta_tensor, p.d_norm
    rows, C, _, _, _ = geom(pb, in_buf)
    x = bufs[in_buf][:B * rows].reshape(B, rows * C)[:, :d_len].astype(np.float64)
    g = pb.tensors[gt].astype(np.float64)[:d_len]
    be = pb.tensors[bt].astype(np.float64)[:d_len]
    real = (g != 0) | (be != 0)
    if real.sum() != d_norm:
        real = np.arange(d_len) < d_norm
    order = np.concatenate([np.nonzero(real)[0], np.nonzero(~real)[0]])
    mu = x.sum(1, keepdims=True) / d_norm
    var = (((x - mu) ** 2).sum(1, keepdims=True) - (d_len - d_norm) * mu ** 2) / d_norm
    ref = (x - mu) / np.sqrt(var + float(np.float32(fl[0]))) * g + be          # f[0] = eps
    if not want_bound:
        return ref, None
    inv = np.argsort(order)
    bnd = oc.layernorm_bound(x[:, order], g[order], be[order], d_norm, ref[:, order])[:, inv]
    return ref, bnd


def _cbfuse_ref(pb, p, bufs, B, dev, want_bound):
    """base + sum of the sources, each repeated 2^shift times along H and W.  The kernel sums in fp32 (base first, then the sources
    in order) and rounds once: within n_src * 2^-24 * (|base| + sum |src|) of the exact sum, then half an fp16 ulp."""
    C = p.C
    refs, bnds = [], []
    for b in range(B):
        acc = image_view(pb, bufs, p.base_buf, b, p.base_coff, p.base_coff + C, dev)
        S = acc.abs()
        for buf, coff, s in plan.cbfuse_sources(p):
            v = image_view(pb, bufs, buf, b, coff, coff + C, dev).repeat_interleave(1 << s, 2).repeat_interleave(1 << s, 3)
            acc = acc + v
            S = S + v.abs()
        refs.append(_np(acc))
        if want_bound:
            e32 = p.n_src * 2.0 ** -24 * _np(S)
            bnds.append(e32 + 0.5 * np.spacing((np.abs(refs[-1]) + e32).astype(np.float16)).astype(np.float64))
    return np.concatenate(refs), (np.concatenate(bnds) if want_bound else None)


def _se_ref(pb, p, bufs, B, dev, want_bound):
    """x * hardsigmoid(W2 relu(W1 mean(x) + b1) + b2) per image, and its bound.  The kernel (lite_ops.cu): the mean is an fp32 sum of HW
    terms and a division, within (HW + 1) 2^-24 mean|x|; each FC is an fp32 dot product with a bias, within n 2^-24 (|b| + sum |w| |v|)
    of its fp32 inputs plus the propagated input error (ReLU: Lipschitz 1); hardsigmoid (Lipschitz 1/6, then + 3 and / 6 in fp32) adds
    2^-23; the product x * g adds 2^-24 |x g|; the fp16 store 2^-11 |ref| + 2^-24.  Each 2^-24 is doubled below for margin."""
    in_buf, coff, C, hid = p.in_buf, p.in_coff, p.C, p.hid
    w1, b1, w2, b2 = (pb.tensors[t].astype(np.float64) for t in (p.w1, p.b1, p.w2, p.b2))
    w1, w2 = w1.reshape(hid, C), w2.reshape(C, hid)
    refs, bnds = [], []
    for b in range(B):
        x = _np(image_view(pb, bufs, in_buf, b, coff, coff + C, dev))[0]              # [C, H, W]
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
            bnds.append((oc.U16 * np.abs(y) + (1 + oc.U16) * E + oc.U32)[None])
    return np.concatenate(refs), (np.concatenate(bnds) if want_bound else None)


def _shuffle2_ref(pb, p, bufs, B, dev):
    """cat(a, b) with the channels interleaved (a0, b0, a1, b1, ...): ShuffleNetV2's channel_shuffle of two groups."""
    n = p.n
    res = []
    for b in range(B):
        a = image_view(pb, bufs, p.a_buf, b, p.a_coff, p.a_coff + n, dev)
        c = image_view(pb, bufs, p.b_buf, b, p.b_coff, p.b_coff + n, dev)
        res.append(_np(torch.stack([a, c], 2).reshape(1, 2 * n, a.shape[2], a.shape[3])))
    return np.concatenate(res)


def op_ref(pb, i, bufs, B, device="cpu", want_bound=True) -> Tuple[np.ndarray, Optional[np.ndarray]]:
    """(reference, bound) of op i for images < B from `bufs`, in read_out's layout.  bound None: bit-exact."""
    t, p, fl = pb.ops[i]
    dev = torch.device(device)
    with torch.no_grad():
        if t == plan.OP_GEMM:
            return _gemm_ref(pb, i, bufs, B, dev, want_bound)
        if t == plan.OP_IM2COL:
            return _im2col_ref(pb, p, bufs, B, dev), None
        if t == plan.OP_STEMPACK:
            return _stempack_ref(pb, p, bufs, B, dev), None
        if t == plan.OP_STEMCONV:
            return _stemconv_ref(pb, p, bufs, B, dev, want_bound)
        if t == plan.OP_DWCONV:
            return _dwconv_ref(pb, p, bufs, B, dev, want_bound)
        if t == plan.OP_LAYERNORM:
            return _layernorm_ref(pb, p, fl, bufs, B, want_bound)
        if t == plan.OP_MAXPOOL:
            in_buf, coff, C, k, s, pad = p.in_buf, p.in_coff, p.C, p.k, p.stride, p.pad
            return np.concatenate([_np(F.max_pool2d(image_view(pb, bufs, in_buf, b, coff, coff + C, dev), k, s, pad)) for b in range(B)]), None
        if t == plan.OP_UPSAMPLE2X:
            in_buf, coff, C = p.in_buf, p.in_coff, p.C
            return np.concatenate([_np(image_view(pb, bufs, in_buf, b, coff, coff + C, dev).repeat_interleave(2, 2).repeat_interleave(2, 3))
                                   for b in range(B)]), None
        if t == plan.OP_AVGPOOL2:
            in_buf, coff, C, fill = p.in_buf, p.in_coff, p.C, p.fill
            res = []
            for b in range(B):
                x = _np(image_view(pb, bufs, in_buf, b, coff, coff + C, dev)).astype(np.float32)    # the kernel's fp32 order, one rounding
                m = (((x[:, :, :-1, :-1] + x[:, :, :-1, 1:]) + (x[:, :, 1:, :-1] + x[:, :, 1:, 1:])) * np.float32(0.25)).astype(np.float16)
                r = np.full(x.shape, -np.inf if fill else 0.0)
                r[:, :, :-1, :-1] = m
                res.append(r)
            return np.concatenate(res), None
        if t == plan.OP_ATTN:
            in_buf, coff, nh, kdp, hd = p.in_buf, p.in_coff, p.nh, p.kdp, p.hd
            refs, bnds = [], []
            for b in range(B):
                qkv = _np(image_view(pb, bufs, in_buf, b, coff, coff + nh * (2 * kdp + hd), dev))
                r, bd = oc.attention_ref(qkv, nh, kdp, hd, float(np.float32(fl[0])))     # f[0] = softmax scale
                refs.append(r)
                bnds.append(bd)
            return np.concatenate(refs), (np.concatenate(bnds) if want_bound else None)
        if t == plan.OP_CBFUSE:
            return _cbfuse_ref(pb, p, bufs, B, dev, want_bound)
        if t == plan.OP_SE:
            return _se_ref(pb, p, bufs, B, dev, want_bound)
        if t == plan.OP_SHUFFLE2:
            return _shuffle2_ref(pb, p, bufs, B, dev), None
    raise ValueError(f"op {i}: unknown type {t}")


def excess(got: np.ndarray, ref: np.ndarray, bound: Optional[np.ndarray]) -> Tuple[float, int]:
    """(max |got - ref| / bound, elements over the bound); a bit-exact op gives 0 or inf and the count of differing elements."""
    if bound is None:
        dt = np.float16 if got.dtype != np.float32 else np.float32
        g, r = got.astype(dt), ref.astype(dt)
        bad = int((g.view(np.uint16 if dt == np.float16 else np.uint32) != r.view(np.uint16 if dt == np.float16 else np.uint32)).sum())
        return (np.inf if bad else 0.0), bad
    err = np.abs(got - ref)
    ratio = np.where(np.isfinite(err), err / bound, np.inf)
    return float(ratio.max(initial=0.0)), int((~(err <= bound)).sum())


def interpret(pb, image: np.ndarray, B: int, round_to_plan: bool = False) -> Dict[int, np.ndarray]:
    """Every op's reference in plan order, from the padded image ([B * rows, 4]).  Buffers hold float64 (round_to_plan: each op's
    result is rounded to its buffer's dtype, as the device stores it)."""
    bufs = new_buffers(pb, B, np.float64)
    bufs[pb.image.buf][:] = image
    for i in range(len(pb.ops)):
        ref, _ = op_ref(pb, i, bufs, B, want_bound=False)
        if round_to_plan:
            ref = ref.astype(np.float32 if geom(pb, out_region(pb, i).buf)[2] == 1 else np.float16).astype(np.float64)
        write_out(pb, i, bufs, B, ref)
    return bufs
