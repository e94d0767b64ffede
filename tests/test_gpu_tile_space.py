"""GPU: every GEMM tile configuration the autotuner can pick, on every route, against the float64 references of op_conformance_cases
and bit for bit against each other.

The autotuner times candidates on the device and keeps the fastest, so which tile a layer runs differs between cards and runs; the
other GPU tests only reach the configurations that won on the card they ran on.  Here:
- sweep: one plan per case holding one op per configuration of tile_space_cases.tile_space (all read the same input slice, each
  writes its own output slice), with the discipline of test_gpu_op_conformance (NaN-poisoned neighbours and images >= B, sentinels
  around every output slice, zero halos, eager = graph replay, run(1) = image 0).  Every op's step description must report the
  configuration asked for; every output must be within its per-element bound; all configurations must agree bit for bit;
- FC batch sweep: the swap-AB tensor-core FC, whose BN follows the batch, at both ends of every 16-image class, and fc_stream across
  its 8-image rows: image k has the same bits at every batch and MT;
- whole networks: every autotune candidate of every GEMM of each plan of test_gpu_plan_conformance, forced one variant at a time,
  must reproduce the autotuned run bit for bit in every buffer."""
import copy
import hashlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import op_conformance_cases as oc  # noqa: E402
import plan_interp as pi  # noqa: E402
import test_gpu_plan_conformance as gpc  # noqa: E402
import tile_space_cases as ts  # noqa: E402
from adas_b200 import _capi, plan  # noqa: E402
from test_gpu_op_conformance import _bits, _fill, _geom, _read_slice, _region, _write_slice  # noqa: E402

pytestmark = pytest.mark.gpu

DESC_RE = re.compile(r"BN=(\d+) MT=(\d+) slab=(\d+) stages=(\d+)")
STAGES_SEEN = {}   # sweep case -> stage counts its descriptions reported


def _ran(desc):
    m = DESC_RE.search(desc)
    assert m, desc
    return tuple(int(v) for v in m.groups())          # (BN, MT, slab, stages)


# ---------------------------------------------------------------------------------------------------------------------------
# sweep
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ts.SWEEP_CASES, ids=[c[0] for c in ts.SWEEP_CASES])
def test_tile_sweep(tmp_path, case):
    sw = ts.sweep_case(case)
    pb, B = sw.pb, sw.B
    mb = B + 2
    path = str(tmp_path / f"{sw.name}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, 0, max_batch=mb)
    in_bufs = {}
    for buf, coff, data in sw.ins:
        a = in_bufs.setdefault(buf, _fill(pb, buf, mb, oc.NAN16))
        _write_slice(a, pb, buf, B, coff, data)
    for buf, a in in_bufs.items():
        eng.write_buffer(buf, a)
    out_bufs = sorted({ob for _, _, (ob, _) in sw.ops})
    assert not set(out_bufs) & set(in_bufs) and len(out_bufs) == len(sw.ops)
    sentinel = {ob: _fill(pb, ob, mb, 0, np.random.default_rng(7 + ob)) for ob in out_bufs}
    for ob, a in sentinel.items():
        eng.write_buffer(ob, a)
    runs = []
    for _ in range(3):                     # eager, graph capture, graph replay
        eng.run(B)
        runs.append({ob: eng.read_buffer(ob, mb).copy() for ob in out_bufs})
    eng.run(1)
    one = {ob: eng.read_buffer(ob, mb) for ob in out_bufs}
    descs = [eng.time_step(B, i, 1)[2] for i in range(eng.num_steps(B))]
    eng.close()

    fails, worst, first, stages_seen = [], 0.0, None, set()
    for i, c, (ob, coff) in sw.ops:
        tag = c.name()
        out = runs[2][ob]
        ran = _ran(descs[i])
        stages_seen.add(ran[3])
        if ran != (c.BN, c.MT, c.slab, c.stages):
            fails.append(f"{tag}: asked for it, ran BN={ran[0]} MT={ran[1]} slab={ran[2]} stages={ran[3]} ({descs[i]})")
            continue
        if not np.array_equal(_bits(runs[0][ob]), _bits(out)):
            fails.append(f"{tag}: eager and graph-replay runs differ")
        keep = ~_region(pb, ob, mb, B, coff, sw.C)
        nchg = int((_bits(out)[keep] != _bits(sentinel[ob])[keep]).sum())
        if nchg:
            fails.append(f"{tag}: {nchg} elements outside the output slice / images >= {B} changed")
        rows, C, dt, H, W = _geom(pb, ob)
        v = out.reshape(mb, H + 2, W + 2, C).astype(np.float32)
        if v[:, 0].any() or v[:, -1].any() or v[:, :, 0].any() or v[:, :, -1].any():
            fails.append(f"{tag}: wrote into the zero halo")
        got = _read_slice(out, pb, ob, B, coff, sw.C)
        err = np.abs(got - sw.ref)
        bad = ~(err <= sw.bound)
        ratio = float(np.max(np.where(np.isfinite(err), err / sw.bound, np.inf)))
        worst = max(worst, ratio)
        if bad.any():
            fails.append(f"{tag}: {int(bad.sum())} of {bad.size} out of bound, max err/bound {ratio:.3g}")
        bits = _bits(_read_slice(out, pb, ob, B, coff, sw.C).astype(out.dtype))
        if first is None:
            first = (tag, bits)
        elif not np.array_equal(bits, first[1]):
            fails.append(f"{tag}: {int((bits != first[1]).sum())} elements differ in bits from {first[0]}")
        if not np.array_equal(_bits(_read_slice(one[ob], pb, ob, 1, coff, sw.C).astype(out.dtype)), bits[:1]):
            fails.append(f"{tag}: run(1) differs from image 0 of run({B})")
    STAGES_SEEN[sw.name] = stages_seen
    print(f"[sweep] {sw.name} ({sw.route}): {len(sw.ops)} configurations, stages {sorted(stages_seen)}, "
          f"worst err/bound {worst:.3g}")
    assert not fails, "\n".join(fails[:40])


def test_sweep_reaches_every_stage_count():
    """The sweep's descriptions reach every pipeline depth from 2 to 8 stages."""
    if len(STAGES_SEEN) != len(ts.SWEEP_CASES):
        pytest.skip("needs every sweep case of this module in the same session")
    seen = set().union(*STAGES_SEEN.values())
    assert seen >= set(range(2, ts.MAX_STAGES + 1)), sorted(seen)


# ---------------------------------------------------------------------------------------------------------------------------
# FC batch sweep
# ---------------------------------------------------------------------------------------------------------------------------
def _fc_batches(tmp_path, K, N, mb, mts, batches, route):
    """Run the FC plan of ts.fc_sweep (one op per MT hint) at every batch of `batches`; returns the engine, still open."""
    nimg = max(batches)
    pb, ops, (xin, x), ref, bound = ts.fc_sweep(K, N, nimg, mts)
    path = str(tmp_path / f"fc_{route}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, 0, max_batch=mb)
    sentinel = {ob: _fill(pb, ob, mb, 0, np.random.default_rng(7 + ob)) for _, _, ob in ops}
    canon = None                                  # bits of every image from the first batch that holds it
    have = 0
    fails, worst, classes = [], 0.0, set()
    for b in batches:
        a = _fill(pb, xin, mb, oc.NAN16)          # images >= b and the 16 entries past K: NaN
        a.reshape(mb, -1)[:b, :K] = x[:b]
        eng.write_buffer(xin, a)
        for ob, s in sentinel.items():
            eng.write_buffer(ob, s)
        eng.run(b)
        outs = {ob: eng.read_buffer(ob, mb) for _, _, ob in ops}
        descs = [eng.time_step(b, i, 1)[2] for i in range(eng.num_steps(b))]
        for i, mt, ob in ops:
            d = descs[i]
            tag = f"batch {b} MT hint {mt}"
            if route == "tr":
                BN, MT, _, _ = _ran(d)
                want = (ts.r16(b), min(mt, ts.mt_max(ts.r16(b))))
                classes.add(BN)
                if "tr=1" not in d or (BN, MT) != want:
                    fails.append(f"{tag}: wanted BN={want[0]} MT={want[1]}, ran {d}")
            elif "fc_stream" not in d:
                fails.append(f"{tag}: not on fc_stream: {d}")
            out = outs[ob]
            keep = ~_region(pb, ob, mb, b, 0, N)
            nchg = int((_bits(out)[keep] != _bits(sentinel[ob])[keep]).sum())
            if nchg:
                fails.append(f"{tag}: {nchg} elements outside the output / images >= {b} changed")
            got = out.reshape(mb, -1)[:b, :N]
            err = np.abs(got.astype(np.float64) - ref[:b])
            bad = ~(err <= bound[:b])
            ratio = float(np.max(np.where(np.isfinite(err), err / bound[:b], np.inf)))
            worst = max(worst, ratio)
            if bad.any():
                fails.append(f"{tag}: {int(bad.sum())} of {bad.size} out of bound, max err/bound {ratio:.3g}")
            bits = _bits(np.ascontiguousarray(got))
            if canon is None:
                canon = np.zeros((nimg, N), bits.dtype)
            if b > have:                              # images seen for the first time: their bits become the reference
                canon[have:b] = bits[have:]
                have = b
            if not np.array_equal(bits, canon[:b]):
                rows = np.unique(np.argwhere(bits != canon[:b])[:, 0])
                fails.append(f"{tag}: images {rows[:8].tolist()} differ in bits from their first run")
    print(f"[fc] {route}: K {K} N {N}, batches {list(batches)}, BN classes {sorted(classes)}, worst err/bound {worst:.3g}")
    assert not fails, "\n".join(fails[:40])
    return eng


def test_fc_tensor_core_batch_sweep(tmp_path):
    """Both ends of every 16-image class (BN 16 .. 256) and every MT; batch 257 is refused before anything launches."""
    K, N = ts.FC_TR
    assert N * K * 2 > oc.FC_STREAM_MAX_BYTES
    eng = _fc_batches(tmp_path, K, N, 257, [1, 2, 3, 4], ts.FC_TR_BATCHES, "tr")
    n0 = _capi.launch_count()
    with pytest.raises(Exception, match="at most 256 images"):
        eng.run(257)
    assert _capi.launch_count() == n0
    eng.close()


def test_fc_stream_batch_invariance(tmp_path):
    K, N = ts.FC_STREAM
    assert N * K * 2 <= oc.FC_STREAM_MAX_BYTES
    _fc_batches(tmp_path, K, N, 256, [0], ts.FC_STREAM_BATCHES, "fc_stream").close()


# ---------------------------------------------------------------------------------------------------------------------------
# whole networks under every autotune candidate
# ---------------------------------------------------------------------------------------------------------------------------
NET_PLANS = [c for c in gpc.PLANS if c[4] in (3, 8)]
AT_RE = re.compile(r"\[autotune\] op (\d+) .* BN=(\d+) mt=(\d+) no_slab=(\d+) :")


def _autotune_candidates(family, scale, kw, mb, B):
    """{op: [(BN, MT, no_slab), ...]}: the candidates autotune timed for each GEMM op at batch B.  ADAS_B200_AT_LOG is read once per
    process, so the plan is built and run in a subprocess."""
    env = dict(os.environ, ADAS_B200_AT_LOG="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "autotune-log", json.dumps([family, scale, kw, mb, B])], env=env,
                       cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    cands = {}
    for m in AT_RE.finditer(r.stderr):
        cands.setdefault(int(m.group(1)), []).append(tuple(int(v) for v in m.groups()[1:]))
    return cands


def _digests(bufs, pb, one_image=False):
    return {i: hashlib.sha256(a[:pb.buffers[i][0]].tobytes() if one_image else a.tobytes()).hexdigest() for i, a in bufs.items()}


@pytest.mark.parametrize("family,scale,kw,mb,B", [pytest.param(*c, marks=[pytest.mark.slow] if c[4] == 8 else [], id=gpc.plan_id(*c))
                                                   for c in NET_PLANS])
def test_network_every_candidate(tmp_path, family, scale, kw, mb, B):
    pb = gpc.build(family, scale, **kw)
    cands = _autotune_candidates(family, scale, kw, mb, B)
    x = gpc.frames_in(pb, family, kw, range(B))
    path = str(tmp_path / "auto.b200w")
    pb.write(path)
    eng = _capi.Engine(path, 0, max_batch=mb)
    eng.infer(x)
    bufs = gpc.read_all(eng, pb, mb)
    want, want0 = _digests(bufs, pb), _digests(bufs, pb, one_image=True)
    del bufs
    descs = [eng.time_step(B, i, 1)[2] for i in range(eng.num_steps(B))]
    eng.close()
    # every GEMM the autotuner chooses for: its timed candidates, or the one configuration it ran without timing
    tuned = {}
    for i, (t, p, _) in enumerate(pb.ops):
        if t != plan.OP_GEMM or p.transposed or p.BN > 0:
            continue
        if i in cands:
            tuned[i] = cands[i]
        else:
            BN, MT, slab, _ = _ran(descs[i])
            tuned[i] = [(BN, MT, p.no_slab)]
    assert set(cands) <= set(tuned), sorted(set(cands) - set(tuned))
    V = max(len(c) for c in tuned.values())
    fails = []
    for v in range(V):
        pv = copy.copy(pb)
        pv.ops = [(t, p.copy(), list(f)) for t, p, f in pb.ops]
        for i, cl in tuned.items():
            ts.force_tile(pv, i, *cl[v % len(cl)])
        path = str(tmp_path / f"variant{v}.b200w")
        pv.write(path)
        eng = _capi.Engine(path, 0, max_batch=mb)
        eng.infer(x)
        got = _digests(gpc.read_all(eng, pv, mb), pv)
        bad = [i for i in got if got[i] != want[i]]
        eng.infer(x[:1])
        got0 = _digests({i: eng.read_buffer(i, 1) for i in range(len(pv.buffers))}, pv, one_image=True)
        bad0 = [i for i in got0 if got0[i] != want0[i]]
        eng.close()
        os.remove(path)
        if bad or bad0:
            forced = {i: cl[v % len(cl)] for i, cl in tuned.items()}
            suspects = sorted({i for i, (t, p, _) in enumerate(pb.ops) if t == plan.OP_GEMM and p.out_buf in bad})
            fails.append(f"variant {v}: buffers {bad} differ from the autotuned run, image 0 of run(1) differs in {bad0}; "
                         f"GEMMs writing them ran (BN, MT, no_slab) {[(i, forced.get(i)) for i in suspects]}")
    kinds = {}
    for i, cl in tuned.items():
        kinds.setdefault(pi.op_kind(pb, i), set()).update(cl)
    print(f"[net] {gpc.plan_id(family, scale, kw, mb, B)}: {len(tuned)} tuned GEMMs, {V} variants; distinct candidates per op kind: "
          + ", ".join(f"{k} {len(s)}" for k, s in sorted(kinds.items())))
    assert not fails, "\n".join(fails[:20])


if __name__ == "__main__" and sys.argv[1:2] == ["autotune-log"]:
    import tempfile
    family, scale, kw, mb, B = json.loads(sys.argv[2])
    pb = gpc.build(family, scale, **kw)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "plan.b200w")
        pb.write(path)
        eng = _capi.Engine(path, 0, max_batch=mb)
        eng.infer(gpc.frames_in(pb, family, kw, range(B)))
        eng.close()
    print("ok")
