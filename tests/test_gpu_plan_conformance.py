"""GPU: every op of whole network plans against the float64 reference of plan_interp.py, computed from that op's own input buffers as
the device left them, across consecutive batches.

Each plan runs batch A, then batch B, then A again (eager, graph capture, graph replay; A and B are different frames through the
library's pre-processing).  After each run every buffer is read back and
- every op's output is within its bound of op_conformance_cases (bit-exact for pooling, upsample, gathers and re-layouts);
- every padded buffer's halo is zero (the stem re-layout owns its top halo row);
- the third run equals the first bit for bit in every buffer.
A kernel that reads the previous launch's or the previous batch's data fails the check of the run after the data changed.

The plans cover the shapes users run (the bench.py workload at batch 8, ten families at batch 3 of 4, YOLOv7-W6 at 1280), so the
persistent GEMM runs many tiles per CTA with its producer running ahead.  The step descriptions must show every route the plans reach,
GEMMs of more than 4 tiles per SM, and no swap-AB FC fetching its B operand (the activation) before its programmatic-dependent-launch
wait (`wpre=0`).  A two-op plan (a short, deep conv feeding a tensor-core FC) and UFLDv2-r18 TuSimple with ADAS_B200_FC_STREAM=0 (its
first FC then runs on tensor cores straight after the pool conv) check that case deterministically."""
import hashlib
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

import plan_interp as pi  # noqa: E402
import synth  # noqa: E402
from adas_b200 import _capi, plan  # noqa: E402
from test_gpu_op_conformance import TOKENS  # noqa: E402

pytestmark = pytest.mark.gpu

# (family, scale, builder kwargs, max_batch, batch); the same list as test_plan_conformance_cpu.GPU_PLANS
PLANS = [("yolov8", "l", {}, 8, 8), ("ufldv2", "34", dict(cfg="culane"), 8, 8),
         ("yolov5", "n", {}, 4, 3), ("yolov6", "n", {}, 4, 3), ("yolov7", "tiny", {}, 4, 3), ("yolov9", "t", {}, 4, 3),
         ("yolov10", "n", {}, 4, 3), ("ufldv2", "18", dict(cfg="tusimple"), 4, 3), ("ufldv1", "18", dict(cfg="culane"), 4, 3),
         ("yolov7", "w6", dict(in_h=1280, in_w=1280), 2, 2)]
SLOW = {0, 1, 9}   # 90-150 s each on an H100 (three batches of float64 references at 640 / 1280 / 320x1600)

ROUTE_TOKENS = {   # plan_interp.op_kind -> route of test_gpu_op_conformance.TOKENS (9-tap: slab or per-tap, as autotune timed them)
    "gemm-1x1": "1x1", "gemm-s2": "s2", "gemm-up2": "up2", "gemm-tr": "tr", "gemm-fc_stream": "fc_stream",
    "gemm-stem7x7s2": "stem7x7s2", "stemconv": "stemconv", "maxpool": "maxpool", "upsample": "upsample", "avgpool2": "avgpool2",
    "dwconv": "dwconv", "attention": "attention", "layernorm": "layernorm"}

RESULTS = {}       # plan id -> (op kinds, step descriptions), for the coverage test at the end of the module


def plan_id(family, scale, kw, mb, B):
    return f"{family}-{scale}" + "".join(f"-{v}" for v in kw.values()) + f"-b{B}"


def build(family, scale, **kw):
    W = plan.synth_weights("ufldv2" if family == "ufldv1" else family, 0, variant=scale)
    return getattr(plan, "build_" + family)(W, scale, **kw)


def frames_in(pb, family, kw, seeds):
    """The network input of synthetic frames through the library's pre-processing."""
    f = np.stack([synth.frame(s) for s in seeds])
    if family == "ufldv2":
        return _capi.ufld_preprocess(f, (pb.in_h, pb.in_w), plan.UFLD_DATASETS[kw["cfg"]]["crop_ratio"])
    if family == "ufldv1":
        return _capi.ufld_preprocess(f, (pb.in_h, pb.in_w), 1.0)
    return _capi.yolo_preprocess(f, (pb.in_h, pb.in_w))


def read_all(eng, pb, mb):
    return {i: eng.read_buffer(i, mb) for i in range(len(pb.buffers))}


def halo_errors(pb, bufs, mb):
    stem_q = {p.out_buf for t, p, _ in pb.ops if t == plan.OP_STEMPACK}
    bad = []
    for i, (rows, C, _, H, W, _) in enumerate(pb.buffers):
        if H == 0:
            continue
        v = bufs[i].reshape(mb, H + 2, W + 2, C)
        edges = [v[:, -1], v[:, :, 0], v[:, :, -1]] + ([] if i in stem_q else [v[:, 0]])
        if any(np.any(e != 0) for e in edges):
            bad.append(i)
    return bad


def check_ops(pb, bufs, B, skip, worst, tag):
    """Every op against plan_interp; returns failure messages and updates worst[kind] = max error / bound.  Ops in `skip` read a
    region a later op overwrites; of an output a later op overwrites in part (YOLOv10 PSA's cv1), the rest is checked."""
    fails = []
    clobbered = pi.overwritten(pb)
    for i in range(len(pb.ops)):
        if i in skip:
            continue
        ref, bnd = pi.op_ref(pb, i, bufs, B, device="cuda")
        got = pi.read_out(pb, i, bufs, B)
        if i in clobbered:
            keep = ~clobbered[i]
            ref, got = ref[:, keep], got[:, keep]
            bnd = None if bnd is None else bnd[:, keep]
        ratio, nbad = pi.excess(got, ref, bnd)
        kind = pi.op_kind(pb, i)
        worst[kind] = max(worst.get(kind, 0.0), ratio)
        if nbad:
            fails.append(f"{tag}: op {i} ({kind}): {nbad} of {ref.size} elements out of bound (max err / bound {ratio:.3g})")
    return fails


def run_aba(pb, family, kw, mb, B, path):
    """Batch A, B, A through the engine; every op checked after every run.  Returns (op kinds, step descriptions, worst ratios)."""
    pb.write(path)
    eng = _capi.Engine(path, 0, max_batch=mb)
    xa = frames_in(pb, family, kw, range(B))
    xb = frames_in(pb, family, kw, range(100, 100 + B))
    assert not np.array_equal(xa, xb)
    skip = set(pi.stale_reads(pb))
    worst, fails, first = {}, [], None
    for r, x in enumerate((xa, xb, xa)):
        eng.infer(x)
        bufs = read_all(eng, pb, mb)
        fails += check_ops(pb, bufs, B, skip, worst, ("eager A", "capture B", "replay A")[r])
        halo = halo_errors(pb, bufs, mb)
        if halo:
            fails.append(f"run {r}: nonzero halo in buffers {halo}")
        digest = {i: hashlib.sha256(a.tobytes()).hexdigest() for i, a in bufs.items()}
        if r == 0:
            first = digest
        elif r == 2 and digest != first:
            fails.append(f"replay of batch A differs from its eager run in buffers {[i for i in digest if digest[i] != first[i]]}")
        del bufs
    steps = [eng.time_step(B, i, 1) for i in range(eng.num_steps(B))]
    eng.close()
    print(f"[plan] {os.path.basename(path)}: {len(pb.ops)} ops, skipped {sorted(skip)}; worst err / bound: "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))
    assert not fails, "\n".join(fails[:20])
    kinds = [pi.op_kind(pb, i) for i in range(len(pb.ops))]
    return kinds, [(t, d) for _, t, d in steps]


def check_steps(kinds, steps):
    assert len(steps) == len(kinds)
    for kind, (t, d) in zip(kinds, steps):
        if kind == "gemm-9tap":
            assert "taps=9 " in d and "s2=0" in d, d
        elif kind in ROUTE_TOKENS:
            for tok in TOKENS[ROUTE_TOKENS[kind]][1]:
                assert tok in d, (kind, tok, d)
        if "tr=1" in d:
            assert d.endswith("wpre=0"), d


@pytest.mark.parametrize("family,scale,kw,mb,B", [pytest.param(*c, marks=[pytest.mark.slow] if k in SLOW else [], id=plan_id(*c))
                                                   for k, c in enumerate(PLANS)])
def test_plan_aba(tmp_path, family, scale, kw, mb, B):
    pb = build(family, scale, **kw)
    kinds, steps = run_aba(pb, family, kw, mb, B, str(tmp_path / f"{family}_{scale}.b200w"))
    check_steps(kinds, steps)
    RESULTS[plan_id(family, scale, kw, mb, B)] = (kinds, steps)


def test_pdl_conv_then_tensor_core_fc(tmp_path):
    """A short, deep 3x3 conv (7 CTAs, K = 18432) feeding a swap-AB FC on tensor cores (4200 x 3200 fp16 weights, past fc_stream's
    25 MB).  The FC's first stages x 64 K entries include interior pixels of the conv output, so an FC that fetched them before the
    conv finished reads batch A's values in the batch-B run."""
    rng = np.random.default_rng(0)
    Bn, H, W, cin, cout, N = 4, 8, 38, 2048, 8, 4200
    pb = plan.PlanBuilder(plan.MODEL_UFLDV2, 3, H, W)
    xbuf = pb.new_padded(H, W, cin)
    w = (rng.standard_normal((cout, cin, 3, 3)) * np.sqrt(2.0 / (9 * cin))).astype(np.float16).astype(np.float32)
    y = pb.conv(xbuf, w, (0.1 * rng.standard_normal(cout)).astype(np.float32), 3, 1, plan.ACT_SILU)
    K = pb.buffers[y.buf][0] * pb.buffers[y.buf][1]
    out = pb.new_dense(1, N, f32=True)
    pb.fc(y.buf, K, (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float16), (0.1 * rng.standard_normal(N)).astype(np.float32),
          plan.ACT_NONE, out)
    assert N * K * 2 > (25 << 20) and pi.op_kind(pb, 1) == "gemm-tr"
    path = str(tmp_path / "pdl.b200w")
    pb.write(path)
    eng = _capi.Engine(path, 0, max_batch=Bn)
    rows = pb.buffers[xbuf.buf][0]
    for seed in (1, 2):                                       # batch A, then batch B
        a = np.zeros((Bn, H + 2, W + 2, cin), np.float16)
        a[:, 1:-1, 1:-1] = np.random.default_rng(seed).standard_normal((Bn, H, W, cin)).astype(np.float16)
        eng.write_buffer(xbuf.buf, a.reshape(Bn * rows, cin))
        eng.run(Bn)
    bufs = read_all(eng, pb, Bn)
    steps = [eng.time_step(Bn, i, 1)[2] for i in range(2)]
    eng.close()
    worst = {}
    fails = check_ops(pb, bufs, Bn, set(), worst, "batch B")
    print(f"[pdl] {steps}; worst err / bound {worst}")
    assert not fails, fails
    tiles = int(re.search(r"tiles=(\d+)", steps[0]).group(1))
    stages = int(re.search(r"stages=(\d+)", steps[1]).group(1))
    assert tiles < 20 and "tr=1" in steps[1] and steps[1].endswith("wpre=0")
    assert stages * 64 > (W + 3) * 8                          # the first stages x 64 K entries reach interior pixels of image row 0


def test_ufld_first_fc_on_tensor_cores():
    """UFLDv2-r18 TuSimple with ADAS_B200_FC_STREAM=0 (read once per process, so in a subprocess): the first FC runs on tensor cores
    directly after the pool conv, whose grid is a few CTAs that trigger their dependents at their start."""
    env = dict(os.environ, ADAS_B200_FC_STREAM="0")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "ufld-fc-tr"], env=env, cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


def test_route_coverage():
    """Every route of the plans shows in their step descriptions; 1x1, 9-tap and stride-2 GEMMs each reach > 4 tiles per SM."""
    if len(RESULTS) != len(PLANS):
        pytest.skip("needs every plan of this module in the same session")
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kinds = set()
    big = {}
    for ks, steps in RESULTS.values():
        kinds |= set(ks)
        for k, (_, d) in zip(ks, steps):
            m = re.search(r"tiles=(\d+)", d)
            if m:
                big[k] = max(big.get(k, 0), int(m.group(1)))
    assert {k for k in kinds if k in ROUTE_TOKENS} == set(ROUTE_TOKENS), set(ROUTE_TOKENS) - kinds
    assert "gemm-9tap" in kinds and "im2col" in kinds
    for k in ("gemm-1x1", "gemm-9tap", "gemm-s2"):
        assert big.get(k, 0) > 4 * sms, (k, big.get(k), sms)
    print(f"[coverage] largest tile counts {big}, {sms} SMs")


if __name__ == "__main__" and sys.argv[1:] == ["ufld-fc-tr"]:
    assert os.environ.get("ADAS_B200_FC_STREAM") == "0"
    import tempfile
    pb = build("ufldv2", "18", cfg="tusimple")
    with tempfile.TemporaryDirectory() as d:
        kinds, steps = run_aba(pb, "ufldv2", dict(cfg="tusimple"), 4, 3, os.path.join(d, "ufldv2_r18_tusimple_fc_tr.b200w"))
    fcs = [d for k, (t, d) in zip(kinds, steps) if k in ("gemm-tr", "gemm-fc_stream")]
    print("[fc]", fcs)
    assert len(fcs) == 2 and all("tr=1" in d and d.endswith("wpre=0") for d in fcs), fcs
    check_steps([k if k != "gemm-fc_stream" else "gemm-tr" for k in kinds], steps)
    print("ok")
