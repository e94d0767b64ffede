"""GPU: every plan op on channel slices, ragged batches and poisoned neighbours against the float64 references and per-element
bounds of op_conformance_cases.

Each case is a one-op plan run through the engine with max_batch = B + 2:
- input buffers hold the operand slice for images < B; every other channel and every image >= B holds a poison (fp16 NaN, +inf for
  max pooling) that changes the result if read; halos stay zero (the layout contract);
- the output buffer holds a finite random sentinel; after the run everything outside the op's slice of images < B is unchanged bit
  for bit and the halo is zero;
- eager, graph-capture and replay runs give the same bits, and run(1) gives image 0 the bits of the batch-B run;
- the product path (conv_impl 0) and the SIMT twin (conv_impl 1, where the op has one) both meet the bound, and differ by at most
  twice the bound;
- the step descriptions prove the intended route was taken."""
import numpy as np
import pytest

import op_conformance_cases as oc
from adas_b200 import _capi, plan

pytestmark = pytest.mark.gpu

TOKENS = {   # route -> (op types that must appear, substrings of the GEMM / op step description)
    "1x1": ({plan.OP_GEMM}, ["taps=1 ", "s2=0", "tr=0", "up2=0"]),
    "slab": ({plan.OP_GEMM}, ["taps=9 ", "s2=0", "slab=1"]),
    "tap": ({plan.OP_GEMM}, ["taps=9 ", "s2=0", "slab=0"]),
    "s2": ({plan.OP_GEMM}, ["s2=1"]),
    "im2col8": ({plan.OP_IM2COL, plan.OP_GEMM}, ["taps=1 ", "s2=0"]),
    "im2col4": ({plan.OP_IM2COL, plan.OP_GEMM}, ["taps=1 ", "s2=0"]),
    "up2": ({plan.OP_GEMM}, ["up2=1"]),
    "tr": ({plan.OP_GEMM}, ["tr=1"]),
    "fc_stream": ({plan.OP_GEMM}, ["fc_stream"]),
    "stemconv": ({plan.OP_STEMCONV}, ["stem "]),
    "stem7x7s2": ({plan.OP_STEMPACK, plan.OP_GEMM}, ["taps=4 "]),
    "maxpool": ({plan.OP_MAXPOOL}, []),
    "upsample": ({plan.OP_UPSAMPLE2X}, []),
    "avgpool2": ({plan.OP_AVGPOOL2}, []),
    "dwconv": ({plan.OP_DWCONV}, ["dwconv "]),
    "attention": ({plan.OP_ATTN}, ["attention "]),
    "layernorm": ({plan.OP_LAYERNORM}, []),
}


def _geom(pb, buf):
    rows, C, dtype, H, W, _ = pb.buffers[buf]
    return rows, C, np.float32 if dtype == 1 else np.float16, H, W


def _fill(pb, buf, mb, fill, rng=None):
    """Whole buffer for mb images: interior = `fill` bits (or a random finite sentinel when rng is given), halo zero."""
    rows, C, dt, H, W = _geom(pb, buf)
    if rng is not None:
        a = rng.standard_normal((mb * rows, C)).astype(dt)
    else:
        assert dt == np.float16
        a = np.full((mb * rows, C), fill, np.uint16).view(np.float16)
    if H > 0:
        v = a.reshape(mb, H + 2, W + 2, C)
        v[:, 0] = 0; v[:, -1] = 0; v[:, :, 0] = 0; v[:, :, -1] = 0
    return a


def _region(pb, buf, mb, B, coff, c):
    """Boolean mask of the elements an op writing channels [coff, coff + c) of images < B may change."""
    rows, C, dt, H, W = _geom(pb, buf)
    m = np.zeros((mb * rows, C), bool)
    if H > 0:
        m.reshape(mb, H + 2, W + 2, C)[:B, 1:-1, 1:-1, coff:coff + c] = True
    else:
        m.reshape(mb, rows * C)[:B, coff:coff + c] = True
    return m


def _write_slice(a, pb, buf, B, coff, data):
    rows, C, dt, H, W = _geom(pb, buf)
    if H > 0:
        a.reshape(-1, H + 2, W + 2, C)[:B, 1:-1, 1:-1, coff:coff + data.shape[1]] = data.transpose(0, 2, 3, 1)
    else:
        a.reshape(-1, rows * C)[:B, coff:coff + data.shape[1]] = data


def _read_slice(a, pb, buf, B, coff, c):
    rows, C, dt, H, W = _geom(pb, buf)
    if H > 0:
        return a.reshape(-1, H + 2, W + 2, C)[:B, 1:-1, 1:-1, coff:coff + c].astype(np.float64).transpose(0, 3, 1, 2)
    return a.reshape(-1, rows * C)[:B, coff:coff + c].astype(np.float64)


def _bits(a):
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _run(tmp_path, spec, impl, tag):
    pb, B = spec.pb, spec.B
    mb = B + 2
    path = str(tmp_path / f"{tag}_{impl}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, 0, max_batch=mb, conv_impl=impl)
    in_bufs = {}
    for buf, coff, data in spec.ins:
        a = in_bufs.setdefault(buf, _fill(pb, buf, mb, spec.poison))
        _write_slice(a, pb, buf, B, coff, data)
    for buf, a in in_bufs.items():
        eng.write_buffer(buf, a)
    obuf, ocoff, oc_ = spec.out
    assert obuf not in in_bufs
    sentinel = _fill(pb, obuf, mb, 0, np.random.default_rng(7))
    eng.write_buffer(obuf, sentinel)
    runs = []
    for _ in range(3):                     # eager, graph capture, graph replay
        eng.run(B)
        runs.append(eng.read_buffer(obuf, mb).copy())
    assert np.array_equal(_bits(runs[0]), _bits(runs[2])), "eager and graph-replay runs differ"
    out = runs[2]
    keep = ~_region(pb, obuf, mb, B, ocoff, oc_)
    changed = np.argwhere(_bits(out)[keep] != _bits(sentinel)[keep])
    assert changed.size == 0, f"{len(changed)} elements outside the output slice / images >= {B} changed"
    got = _read_slice(out, pb, obuf, B, ocoff, oc_)
    # batch invariance: image 0 alone gives the same bits
    eng.run(1)
    one = eng.read_buffer(obuf, mb)
    assert np.array_equal(_bits(_read_slice(one, pb, obuf, 1, ocoff, oc_).astype(out.dtype)),
                          _bits(_read_slice(out, pb, obuf, 1, ocoff, oc_).astype(out.dtype))), "run(1) differs from image 0 of run(B)"
    steps = [eng.time_step(B, i, 1) for i in range(eng.num_steps(B))]
    eng.close()
    rows, C, dt, H, W = _geom(pb, obuf)
    if H > 0:
        v = out.reshape(mb, H + 2, W + 2, C).astype(np.float32)
        assert not (v[:, 0].any() or v[:, -1].any() or v[:, :, 0].any() or v[:, :, -1].any()), "the op wrote into the zero halo"
    return got, [(t, d) for _, t, d in steps]


def _check_route(spec, steps):
    types, toks = TOKENS[spec.route]
    assert types <= {t for t, _ in steps}, (spec.route, steps)
    main = [d for t, d in steps if t in (plan.OP_GEMM, plan.OP_STEMCONV, plan.OP_DWCONV, plan.OP_ATTN)]
    for tok in toks:
        assert any(tok in d for d in main), (spec.route, tok, steps)


def _check_value(spec, got, impl):
    if spec.bound is None:
        assert np.array_equal(got.astype(np.float16).view(np.uint16), spec.ref.astype(np.float16).view(np.uint16)), f"impl {impl}: not bit-exact"
        return
    err = np.abs(got - spec.ref)
    bad = ~(err <= spec.bound)
    ratio = float(np.max(np.where(np.isfinite(err), err / spec.bound, np.inf)))
    assert not bad.any(), f"impl {impl}: {int(bad.sum())} of {bad.size} elements exceed the bound (max err / bound {ratio:.3g})"


@pytest.mark.parametrize("family,case,make", oc.ALL, ids=[oc.case_id(f, c) for f, c, _ in oc.ALL])
def test_op_conformance(tmp_path, family, case, make):
    spec = make(case)
    got0, steps = _run(tmp_path, spec, 0, family)
    _check_route(spec, steps)
    _check_value(spec, got0, 0)
    if spec.simt:
        got1, _ = _run(tmp_path, spec, 1, family)
        _check_value(spec, got1, 1)
        assert (np.abs(got0 - got1) <= 2 * spec.bound).all(), "product path and SIMT twin differ by more than twice the bound"
