"""CPU half of the tile-space suite: the configurations tile_space_cases lists, the packing of the sweep cases, and bounds that accept
an emulated kernel while rejecting the faults a single tile configuration could have."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import op_conformance_cases as oc
import tile_space_cases as ts
from adas_b200 import plan


# ---- the space ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route,N,count", [("1x1", 248, 33), ("im2col", 256, 33), ("s2", 300, 33), ("slab", 248, 65),
                                           ("up2", 544, 7), ("stem7x7s2", 64, 16), ("1x1", 40, 12)])
def test_tile_space_size(route, N, count):
    space = ts.tile_space(route, N)
    assert len(space) == len(set(space)) == count
    for c in space:
        assert c.BN % 16 == 0 and 16 <= c.BN <= min(256, ts.r16(N)) and 1 <= c.MT <= min(4, 256 // c.BN)
        assert c.MT * c.BN <= ts.V3_ACC_COLS and 2 <= c.stages <= 8
        assert c.slab == (route == "slab" and not c.no_slab)
    if route == "slab":
        assert {(c.BN, c.MT) for c in space if not c.slab} == {(c.BN, c.MT) for c in ts.tile_space("1x1", N)}
        assert {(c.BN, c.MT) for c in space if c.slab} == {(c.BN, c.MT) for c in ts.tile_space("1x1", N)} - {(256, 1)}


def test_fc_tile_space_follows_the_batch():
    assert [(c.BN, c.MT) for c in ts.tile_space("tr", 1)] == [(16, m) for m in (1, 2, 3, 4)]
    assert [(c.BN, c.MT) for c in ts.tile_space("tr", 65)] == [(80, 1), (80, 2), (80, 3)]
    assert [(c.BN, c.MT) for c in ts.tile_space("tr", 256)] == [(256, 1)]
    assert {ts.r16(b) for b in ts.FC_TR_BATCHES} == set(range(16, 257, 16))
    assert all(b - 1 in ts.FC_TR_BATCHES or b == 1 for b in ts.FC_TR_BATCHES if b % 16 == 1)


def test_sweep_reaches_every_stage_count():
    stages = {c.stages for case in ts.SWEEP_CASES for _, c, _ in ts.sweep_case(case).ops}
    assert stages == set(range(2, 9)), sorted(stages)


@pytest.mark.parametrize("case", ts.SWEEP_CASES, ids=[c[0] for c in ts.SWEEP_CASES])
def test_sweep_case_packs_onto_its_route(case):
    sw = ts.sweep_case(case)
    N = sw.pb.ops[sw.ops[0][0]][1].N
    assert [c for _, c, _ in sw.ops] == ts.tile_space(sw.route, N)
    want = {"slab": ("slab", "tap"), "im2col": ("im2col8", "im2col4")}.get(sw.route, (sw.route,))
    outs = set()
    for i, c, (ob, coff) in sw.ops:
        p = sw.pb.ops[i][1]
        route = ts.op_route(sw.pb, i)
        assert route in want and (route == "tap") == bool(c.no_slab), (sw.name, i, route)
        assert (p.BN, p.MT, p.no_slab) == (c.BN, c.MT, c.no_slab)
        assert (p.out_buf, p.out_coff) == (ob, coff) and coff == ts.OUT_OFF
        outs.add(ob)
    assert len(outs) == len(sw.ops)
    assert sw.bound.shape == sw.ref.shape and (sw.bound > 0).all() and np.isfinite(sw.ref).all()


def test_force_tile_on_fc_sets_only_the_mt_hint():
    pb, ops, _, _, _ = ts.fc_sweep(64, 40, 2, [1, 3])
    for i, mt, out in ops:
        p = pb.ops[i][1]
        assert p.transposed == 1 and p.BN == 0 and p.MT == mt and p.out_buf == out
    assert pb.ops[0][1].w_tensor == pb.ops[1][1].w_tensor     # one weight tensor


# ---- the bounds have teeth -----------------------------------------------------------------------------------------------------
def _emulate(x, w, b, act, fault=None, BN=240):
    """The kernel's arithmetic for a stride-1 1x1 / 3x3 conv on the padded row layout: per tap an fp32 product sum (BLAS order) of
    fp16 operands, taps added in fp32, fp32 bias and activation, fp16 store.  `fault` plants one tile-specific error."""
    B, cin, H, W = x.shape
    cout, _, k, _ = w.shape
    Wp = W + 2
    w = w.copy()
    if fault == "k-tail block dropped":
        w[:, cin // 64 * 64:] = 0
    xp = np.zeros((B, H + 2, Wp, cin), np.float32)
    xp[:, 1:-1, 1:-1] = x.transpose(0, 2, 3, 1)
    X = xp.reshape(-1, cin)
    M = X.shape[0]
    acc = np.zeros((M, cout), np.float32)
    for dy in range(k):
        for dx in range(k):
            sh = (dy - 1) * Wp + dx - 1 if k == 3 else 0
            if fault == "slab tap one row off" and dx == 2:
                sh += 1
            Xs = np.zeros_like(X)
            Xs[max(0, -sh):min(M, M - sh)] = X[max(0, sh):min(M, M + sh)]
            acc = (acc + Xs @ w[:, :, dy, dx].T.astype(np.float32)).astype(np.float32)
    written = np.ones(cout, bool)
    if fault == "last partial N tile dropped":
        written[cout // BN * BN:] = False
    if fault == "16-column wgmma at the offset of the 8 columns before it":
        assert BN == 240                                       # pieces 128 + 64 + 32 + 16: the last starts at column 224
        a2 = acc.copy()
        a2[:, 216:232] = acc[:, 224:240]
        a2[:, 232:240] = 0
        acc = a2
    y = oc.act64((acc + b.astype(np.float32)).astype(np.float64), act).astype(np.float32)
    y[:, ~written] = 0
    if fault == "sub-tile stored at the rows of the one before":
        BMT = 2 * ts.BM                                        # MT = 2
        y2 = y.copy()
        for m0 in range(0, M, BMT):
            hi = min(M, m0 + BMT)
            if hi > m0 + ts.BM:
                y2[m0:hi - ts.BM] = y[m0 + ts.BM:hi]
                y2[m0 + ts.BM:hi] = 0
        y = y2
    out = y.astype(np.float16).astype(np.float64).reshape(B, H + 2, Wp, cout)[:, 1:-1, 1:-1]
    return out.transpose(0, 3, 1, 2)


def _problem(k, cin, cout, B=1, H=14, W=14, seed=3):
    rng = np.random.default_rng(seed)
    x = oc.f16(rng, (B, cin, H, W))
    w = oc.f16(rng, (cout, cin, k, k), np.sqrt(2.0 / (cin * k * k)))
    b = oc.f16(rng, cout, 0.1)
    ref, S, a, _ = oc.conv_ref(x, w, b, 1, k // 2, 1)
    return x, w, b, ref, oc.gemm_bound(ref, S, k * k * oc.r8(cin), 1, a)


def _violations(got, ref, bound):
    return int((np.abs(got - ref) > bound).sum())


@pytest.mark.parametrize("k,cin,cout,H,W", [(1, 200, 248, 14, 14), (3, 64, 40, 6, 130), (3, 192, 248, 6, 9)])
def test_bound_accepts_emulated_kernel(k, cin, cout, H, W):
    x, w, b, ref, bound = _problem(k, cin, cout, H=H, W=W)
    assert _violations(_emulate(x, w, b, 1), ref, bound) == 0


@pytest.mark.parametrize("fault,k,cin,cout,H,W,BN", [
    ("last partial N tile dropped", 1, 200, 248, 14, 14, 160),
    ("16-column wgmma at the offset of the 8 columns before it", 1, 200, 248, 14, 14, 240),
    ("sub-tile stored at the rows of the one before", 1, 200, 248, 14, 14, 240),
    ("k-tail block dropped", 1, 200, 248, 14, 14, 240),
    ("slab tap one row off", 3, 64, 40, 6, 130, 48),
])
def test_bound_rejects_tile_fault(fault, k, cin, cout, H, W, BN):
    x, w, b, ref, bound = _problem(k, cin, cout, H=H, W=W)
    assert _violations(_emulate(x, w, b, 1), ref, bound) == 0
    assert _violations(_emulate(x, w, b, 1, fault, BN), ref, bound) > 0, fault


def _emulate_s2(x, w, b, act, stale_rows=False):
    """A stride-2 3x3 conv in fp32 (torch's order), fp16 store; with stale_rows, each 13 x 9 output patch (117 of the 128 MMA rows)
    also stores rows 117..127, which land on the first 11 pixels of the next patch's top row with whatever the A sub-tile held."""
    y = F.conv2d(torch.from_numpy(x.astype(np.float32)), torch.from_numpy(w.astype(np.float32)), torch.from_numpy(b.astype(np.float32)),
                 stride=2, padding=1)
    y = oc.act64(y.numpy().astype(np.float64), act).astype(np.float32)
    if stale_rows:
        Ho, Wo = y.shape[2:]
        bw, bh = 13, 9
        assert Wo == bw
        for ty in range((Ho + bh - 1) // bh):
            yo = ty * bh + bh
            if yo < Ho:
                y[:, :, yo, :128 - bw * bh] = y[:, :, ty * bh, :128 - bw * bh]   # stale rows: another pixel's values
    return y.astype(np.float16).astype(np.float64)


def test_bound_rejects_stride2_rows_past_the_patch():
    rng = np.random.default_rng(5)
    x = oc.f16(rng, (1, 128, 40, 26))
    w = oc.f16(rng, (248, 128, 3, 3), np.sqrt(2.0 / (128 * 9)))
    b = oc.f16(rng, 248, 0.1)
    ref, S, a, _ = oc.conv_ref(x, w, b, 2, 1, 1)
    bound = oc.gemm_bound(ref, S, 9 * 128, 1, a)
    assert ref.shape[2:] == (20, 13)
    assert _violations(_emulate_s2(x, w, b, 1), ref, bound) == 0
    assert _violations(_emulate_s2(x, w, b, 1, stale_rows=True), ref, bound) > 0


def test_sweep_bounds_accept_their_own_reference_in_fp16():
    """Rounding the float64 reference to the output type stays inside every sweep case's bound."""
    for case in ts.SWEEP_CASES:
        sw = ts.sweep_case(case)
        f32 = case[-1]
        got = sw.ref.astype(np.float32 if f32 else np.float16).astype(np.float64)
        assert _violations(got, sw.ref, sw.bound) == 0, sw.name
        assert sw.ref.shape[1] == sw.C and plan.OP_GEMM in {t for t, _, _ in sw.pb.ops}
