"""CPU: the plan loader refuses every plan its kernels cannot run in bounds.

A .b200w plan is input data, and the kernels index with its strides, offsets and counts without checking them.  The sweep below
corrupts one field at a time of small plans of every model family (and of single-op plans) and asserts that each result is either
refused by the loader (adas_plan_validate: the same parse and checks as adas_engine_create, no device) or in bounds by the
footprint model of tests/plan_footprint.py for every max_batch up to 4.  The named cases pin holes the loader once had."""
import struct

import pytest

import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
import op_conformance_cases as oc
import plan_footprint as fp

INT32_MAX = 2 ** 31 - 1
REFUSALS = ("plan ", "truncated ", "Parameters must be a .b200w plan file")

FAMILIES = [
    ("v5n", lambda: plan.build_yolov5(plan.synth_weights("yolov5", 0, variant="n"), "n", in_h=256, in_w=256)),
    ("v7-tiny", lambda: plan.build_yolov7(plan.synth_weights("yolov7", 0, variant="tiny"), "tiny", in_h=256, in_w=256)),
    ("v7-w6", lambda: plan.build_yolov7(plan.synth_weights("yolov7", 0, variant="w6"), "w6", in_h=256, in_w=256)),
    ("v8n", lambda: plan.build_yolov8(plan.synth_weights("yolov8", 0, variant="n"), "n", in_h=256, in_w=256)),
    ("v9-t", lambda: plan.build_yolov9(plan.synth_weights("yolov9", 0, variant="t"), "t", in_h=256, in_w=256)),
    ("v9-e", lambda: plan.build_yolov9e(plan.synth_weights("yolov9", 0, variant="e"), in_h=256, in_w=256)),
    ("v10n", lambda: plan.build_yolov10(plan.synth_weights("yolov10", 0, variant="n"), "n", in_h=256, in_w=256)),
    ("v6n", lambda: plan.build_yolov6(plan.synth_weights("yolov6", 0, variant="n"), "n", in_h=256, in_w=256)),
    ("v6-lite", lambda: plan.build_yolov6_lite(plan.synth_weights("yolov6lite", 0, variant="s"), "s", in_h=256, in_w=256)),
    ("ufld2-culane", lambda: plan.build_ufldv2(plan.synth_weights("ufldv2", 0), "18", "culane")),
    ("ufld2-tusimple", lambda: plan.build_ufldv2(plan.synth_weights("ufldv2", 0), "18", "tusimple")),
    ("ufld1", lambda: plan.build_ufldv1(plan.synth_weights("ufldv2", 0), "18", "tusimple")),
]
SINGLE_OPS = ["gemm", "up2", "fc", "maxpool", "avgpool2", "dwconv", "attention", "stem", "layernorm"]

_cache = {}


def _write(tmp_path_factory, name, build):
    if name not in _cache:
        path = str(tmp_path_factory.mktemp("plans") / f"{name}.b200w")
        build().write(path)
        _cache[name] = path
    return _cache[name]


def _single_op(family):
    return next(oc_case for oc_case in oc.ALL if oc_case[0] == family)


def _refused(path):
    try:
        _capi.plan_validate(path)
    except Exception as e:
        return str(e)
    return None


def _values(v, neighbour, nb):
    vals = {0, -1, 1, v - 1, v + 1, v - 8, v + 8, INT32_MAX}
    if neighbour is not None:
        vals.add(neighbour)
    if 0 <= v < nb:
        vals.add((v + 1) % nb)
    return sorted(x for x in vals if x != v)


def _op_fields(typ, p):
    """Names of the fields the loader reads of an op, in slot order: its plan.OP_FIELDS, then the sources of a CBFUSE"""
    names = plan.OP_FIELDS[typ]
    if typ == plan.OP_CBFUSE:
        names += tuple(f"src{s}.{n}" for s in range(max(0, min(p.n_src, plan.CBFUSE_MAX_SRC))) for n in plan.CBFUSE_SRC_FIELDS)
    return names


def _mutations(pl):
    """(description, byte offset, value) of every single-field corruption of the sweep"""
    nb = len(pl.bufs)
    out = []
    # header: version .. meta[15] (uint32), then blob offset / size (uint64)
    for i, name in enumerate(fp.HEADER_FIELDS):
        v = pl.header[1 + i]
        for x in _values(v, None, nb):
            out.append((f"header {name} {v} -> {x}", 8 + 4 * i, "<I", x & 0xFFFFFFFF))
    for j, name in enumerate(("blob_offset", "blob_bytes")):
        v = pl.header[26 + j]
        for x in (0, 1, v - 8, v + 8, v + 1, v - 1, 2 ** 63 - 1):
            if x != v and x >= 0:
                out.append((f"header {name} {v} -> {x}", 8 + 4 * len(fp.HEADER_FIELDS) + 8 * j, "<Q", x))
    seen = set()
    for i, b in enumerate(pl.bufs):
        for f in range(6):
            key = ("buf", tuple(b), f)
            if key in seen:            # identical records get the same corruptions once
                continue
            seen.add(key)
            nbr = pl.bufs[i - 1][f] if i else None
            vals = _values(b[f], nbr, nb)
            if f == 2:
                vals = sorted(set(vals) | {1 - b[f]})
            for x in vals:
                out.append((f"buffer {i} field {f} {b[f]} -> {x}", pl.buf_off(i) + 4 * f, "<I", x & 0xFFFFFFFF))
    for i, o in enumerate(pl.outs):
        for f in range(4):
            nbr = pl.outs[i - 1][f] if i else None
            for x in _values(o[f], nbr, nb):
                out.append((f"output {i} field {f} {o[f]} -> {x}", pl.out_off(i) + 4 * f, "<I", x & 0xFFFFFFFF))
    # ops: the first of each (type, route) in the plan, every field it reads
    picked, routes = [], set()
    for oi, (typ, p, _) in enumerate(pl.ops):
        route = (typ, p.ntaps, p.res_buf >= 0, p.transposed, p.s2, p.up2) if typ == plan.OP_GEMM else (typ,)
        if route not in routes:
            routes.add(route)
            picked.append(oi)
    for oi in picked:
        typ, p, _ = pl.ops[oi]
        for f, name in enumerate(_op_fields(typ, p)):
            nbr = pl.ops[oi - 1][1][f] if oi else None
            for x in _values(p[f], nbr, nb):
                if -2 ** 31 <= x <= INT32_MAX:
                    out.append((f"op {oi} (type {typ}) p[{f}] {name} {p[f]} -> {x}", pl.op_off(oi) + 4 + 4 * f, "<i", x))
    return out


def _sweep(path):
    raw = open(path, "rb").read()
    pl = fp.parse(raw)
    assert _refused(path) is None
    assert fp.out_of_bounds(pl, 4) == [], "the unmodified plan must be in bounds"
    holes, n_acc = [], 0
    muts = _mutations(pl)
    # an accepted plan's records end before its blob (blob_offset corruptions move it by at most 8 bytes): parse only those
    records = raw[:pl.header[26] + 4096]
    with open(path, "r+b") as f:
        for desc, off, fmt, x in muts:
            orig = raw[off:off + struct.calcsize(fmt)]
            f.seek(off); f.write(struct.pack(fmt, x)); f.flush()
            try:
                msg = _refused(path)
                if msg is not None:
                    assert msg.startswith(REFUSALS), (desc, msg)
                    continue
                n_acc += 1
                mut = bytearray(records)
                struct.pack_into(fmt, mut, off, x)
                try:
                    mpl = fp.parse(bytes(mut))
                    bad = [b for mb in (1, 2, 3, 4) for b in fp.out_of_bounds(mpl, mb)]
                except Exception as e:          # the model could not even follow the plan's indices
                    bad = [f"footprint model: {type(e).__name__}: {e}"]
                if bad:
                    holes.append(f"{desc}: {bad[0]}")
            finally:
                f.seek(off); f.write(orig); f.flush()
    return len(muts), n_acc, holes


@pytest.mark.parametrize("name", [n for n, _ in FAMILIES])
def test_mutated_family_plans_are_refused_or_in_bounds(tmp_path_factory, name):
    path = _write(tmp_path_factory, name, dict(FAMILIES)[name])
    n, n_acc, holes = _sweep(path)
    print(f"[sweep] {name}: {n} corruptions, {n_acc} accepted and in bounds")
    assert not holes, f"{len(holes)} accepted plans leave their buffers, e.g.\n" + "\n".join(holes[:10])


@pytest.mark.parametrize("family", SINGLE_OPS)
def test_mutated_single_op_plans_are_refused_or_in_bounds(tmp_path_factory, family):
    fam, case, spec_fn = _single_op(family)
    path = _write(tmp_path_factory, oc.case_id(fam, case), lambda: spec_fn(case).pb)
    n, n_acc, holes = _sweep(path)
    print(f"[sweep] {oc.case_id(fam, case)}: {n} corruptions, {n_acc} accepted and in bounds")
    assert not holes, f"{len(holes)} accepted plans leave their buffers, e.g.\n" + "\n".join(holes[:10])


# ---- the holes the loader had, each on the smallest plan that shows it ---------------------------------------------------------
def _expect_refused(src, tmp_path, name, off, fmt, value, phrase):
    raw = fp.corrupt(open(src, "rb").read(), off, fmt, value)
    bad = tmp_path / f"{name}.b200w"
    bad.write_bytes(raw)
    msg = _refused(str(bad))
    assert msg is not None, f"{name}: the corrupted plan loads"
    assert msg.startswith("plan ") and phrase in msg, (name, msg)
    return fp.parse(raw)


def test_yolov8_head_corruptions_are_refused(tmp_path_factory, tmp_path):
    path = _write(tmp_path_factory, "v8n", dict(FAMILIES)["v8n"])
    pl = fp.parse(open(path, "rb").read())
    o0 = pl.outs[0]
    meta1 = 8 + 4 * fp.HEADER_FIELDS.index("meta1")
    # (name, offset, value, message phrase, whether the decode then leaves its buffer: a narrowed record or a wrong stride
    # still lies inside it, but the decode reads 64 + nc columns and places boxes by the stride)
    cases = [("v8-narrow", pl.out_off(0) + 8, 8, "columns wide", False),
             ("v8-stride", pl.out_off(0) + 12, 99, "stride", False),
             ("v8-anchors", meta1, pl.meta[1] + 1000, "anchors", True),
             ("v8-fp16", pl.buf_off(o0[0]) + 8, 0, "fp16 columns wide", True)]
    for name, off, value, phrase, leaves in cases:
        bad = _expect_refused(path, tmp_path, name, off, "<I", value, phrase)
        assert bool(fp.out_of_bounds(bad, 1)) == leaves, name


def test_yolov5_head_corruptions_are_refused(tmp_path_factory, tmp_path):
    path = _write(tmp_path_factory, "v5n", dict(FAMILIES)["v5n"])
    pl = fp.parse(open(path, "rb").read())
    ob, coff, C, _ = pl.outs[0]
    need = 3 * (5 + pl.meta[0])
    bufC = pl.bufs[ob][1]
    # one column short: the record ends at its buffer's edge, the decode reads one column past it
    raw = bytearray(open(path, "rb").read())
    struct.pack_into("<II", raw, pl.out_off(0) + 4, bufC - (need - 1), need - 1)
    short = tmp_path / "v5-short.b200w"
    short.write_bytes(bytes(raw))
    msg = _refused(str(short))
    assert msg is not None and "columns wide" in msg, msg
    assert fp.out_of_bounds(fp.parse(bytes(raw)), 1)
    bad = _expect_refused(path, tmp_path, "v5-fp16", pl.buf_off(ob) + 8, "<I", 0, "columns wide")
    assert fp.out_of_bounds(bad, 1)


@pytest.mark.parametrize("name", ["ufld2-culane", "ufld1"])
def test_ufld_head_corruptions_are_refused(tmp_path_factory, tmp_path, name):
    path = _write(tmp_path_factory, name, dict(FAMILIES)[name])
    pl = fp.parse(open(path, "rb").read())
    ob = pl.outs[0][0]
    phrase = "UFLD head is one output"
    _expect_refused(path, tmp_path, "ufld-narrow", pl.out_off(0) + 8, "<I", 8, phrase)
    bad = _expect_refused(path, tmp_path, "ufld-fp16", pl.buf_off(ob) + 8, "<I", 0, phrase)
    assert fp.out_of_bounds(bad, 1)
    # a padded 1 x 1 grid of 9 rows per image: the decode would read image b at row b, not at row 9 b
    raw = bytearray(open(path, "rb").read())
    struct.pack_into("<I", raw, pl.buf_off(ob), 9)
    struct.pack_into("<II", raw, pl.buf_off(ob) + 12, 1, 1)
    padded = tmp_path / "ufld-padded.b200w"
    padded.write_bytes(bytes(raw))
    msg = _refused(str(padded))
    assert msg is not None and phrase in msg, msg
    assert fp.out_of_bounds(fp.parse(bytes(raw)), 2)


def test_ufld_plan_without_outputs_needs_a_known_dataset(tmp_path_factory, tmp_path):
    path = _write(tmp_path_factory, "ufld2-culane", dict(FAMILIES)["ufld2-culane"])
    raw = bytearray(open(path, "rb").read())
    struct.pack_into("<I", raw, 8 + 4 * fp.HEADER_FIELDS.index("n_outputs"), 0)
    ok = tmp_path / "ufld-no-outputs.b200w"
    ok.write_bytes(bytes(raw))
    assert _refused(str(ok)) is None          # a plan without outputs (single-op test plans) still loads
    struct.pack_into("<I", raw, 8 + 4 * fp.HEADER_FIELDS.index("meta6"), 7)
    bad = tmp_path / "ufld-no-outputs-dataset7.b200w"
    bad.write_bytes(bytes(raw))
    msg = _refused(str(bad))
    assert msg is not None and "unknown UFLD dataset id 7" in msg, msg


def test_gemm_residual_must_have_the_output_geometry(tmp_path_factory, tmp_path):
    path = _write(tmp_path_factory, "v8n", dict(FAMILIES)["v8n"])
    pl = fp.parse(open(path, "rb").read())
    oi = next(i for i, (t, p, _) in enumerate(pl.ops)
              if t == plan.OP_GEMM and p.res_buf >= 0 and pl.bufs[p.out_buf][3] == 64 and pl.bufs[p.out_buf][4] == 64)
    p = pl.ops[oi][1]
    small = next(i for i, b in enumerate(pl.bufs) if b[3] == 16 and b[4] == 16 and b[2] == 0 and b[1] >= p.res_coff + p.N)
    bad = _expect_refused(path, tmp_path, "v8-residual", pl.field_off(oi, "res_buf"), "<i", small, "residual")
    assert fp.out_of_bounds(bad, 1)


def test_validate_hook_reports_missing_and_malformed_files(tmp_path):
    missing = str(tmp_path / "absent.b200w")
    msg = _refused(missing)
    assert "can't not found" in msg and missing in msg
    junk = tmp_path / "junk.b200w"
    junk.write_bytes(b"B200PLAN" + b"\0" * 300)
    assert _refused(str(junk)).startswith("Parameters must be a .b200w plan file")
