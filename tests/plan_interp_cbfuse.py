"""plan_interp.py with OP_CBFUSE (YOLOv9-E's CBFuse): its regions, its float64 reference with a per-element bound, and every
plan_interp function that walks a plan, so YOLOv9-E plans go through the same dataflow, interpreter and per-op checks as every other
network.

`extended()` is a context in which plan_interp itself knows the op (its OP_NAMES, op_regions and op_ref see OP_CBFUSE, every other op
as before); the module-level functions here run inside it, and a caller wraps code that uses plan_interp indirectly (the batch A / B / A
check of test_gpu_plan_conformance) in it.  Outside the context plan_interp is unchanged."""
import contextlib
from typing import List, Tuple

import numpy as np

import plan_interp as pi
from adas_b200 import plan


def cbfuse_sources(p) -> List[Tuple[int, int, int]]:
    """(buffer, channel offset, shift) of each source of an OP_CBFUSE op, in summation order."""
    return [tuple(p[6 + 3 * s:9 + 3 * s]) for s in range(p[5])]


def _cbfuse_regions(p):
    """In place, the base read is the write region itself."""
    C = p[2]
    return [pi.Region(p[0], p[1], p[1] + C)], [pi.Region(p[3], p[4], p[4] + C)] + [pi.Region(q[0], q[1], q[1] + C) for q in cbfuse_sources(p)]


def _cbfuse_ref(pb, p, bufs, B, dev, want_bound):
    """base + sum of the sources, each repeated 2^shift times along H and W.  The kernel sums in fp32 (base first, then the sources
    in order) and rounds once: within n_src * 2^-24 * (|base| + sum |src|) of the exact sum, then half an fp16 ulp."""
    C = p[2]
    refs, bnds = [], []
    for b in range(B):
        acc = pi.image_view(pb, bufs, p[3], b, p[4], p[4] + C, dev)
        S = acc.abs()
        for buf, coff, s in cbfuse_sources(p):
            v = pi.image_view(pb, bufs, buf, b, coff, coff + C, dev).repeat_interleave(1 << s, 2).repeat_interleave(1 << s, 3)
            acc = acc + v
            S = S + v.abs()
        refs.append(pi._np(acc))
        if want_bound:
            e32 = p[5] * 2.0 ** -24 * pi._np(S)
            bnds.append(e32 + 0.5 * np.spacing((np.abs(refs[-1]) + e32).astype(np.float16)).astype(np.float64))
    return np.concatenate(refs), (np.concatenate(bnds) if want_bound else None)


@contextlib.contextmanager
def extended():
    base_regions, base_ref, had_name = pi.op_regions, pi.op_ref, plan.OP_CBFUSE in pi.OP_NAMES

    def op_regions(pb, i):
        t, p, _ = pb.ops[i]
        return _cbfuse_regions(p) if t == plan.OP_CBFUSE else base_regions(pb, i)

    def op_ref(pb, i, bufs, B, device="cpu", want_bound=True):
        t, p, _ = pb.ops[i]
        if t != plan.OP_CBFUSE:
            return base_ref(pb, i, bufs, B, device=device, want_bound=want_bound)
        import torch
        with torch.no_grad():
            return _cbfuse_ref(pb, p, bufs, B, torch.device(device), want_bound)

    pi.op_regions, pi.op_ref = op_regions, op_ref
    pi.OP_NAMES[plan.OP_CBFUSE] = "cbfuse"
    try:
        yield pi
    finally:
        pi.op_regions, pi.op_ref = base_regions, base_ref
        if not had_name:
            del pi.OP_NAMES[plan.OP_CBFUSE]


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
