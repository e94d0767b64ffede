"""The GEMM tile space: every (BN, MT, slab) configuration the product kernel accepts on each route, a way to force one onto a packed
plan op, and sweep cases that run one op per configuration in one plan.

Shared by test_gpu_tile_space.py (runs every configuration on the GPU) and test_tile_space_cpu.py (checks the space, the packing and
the bounds on the CPU).

The autotuner (engine.cu build_program) times the cost model's best candidates (gemm_v3.cu gemm_v3_candidates) on the device and
keeps the fastest for each (op, batch), so which tile a layer runs depends on the card, its clocks and its load.  Every configuration
must therefore be correct, and all of them must give the same bits (the K order is (dy, k-block, dx) for every tile shape).

The rules below restate gemm_v3_config (gemm_v3.cu) and the constants of gemm_v3.h / tc_common.cuh; a change there makes the GPU
test's description check fail instead of silently shrinking what the sweep covers."""
from dataclasses import dataclass, field
from types import SimpleNamespace
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

import op_conformance_cases as oc
from adas_b200 import plan

# gemm_v3.h / tc_common.cuh
BM, BK = 128, 64
V3_ACC_COLS = 256                              # MT * BN <= 256 accumulator columns per consumer thread
V3_DYN_SMEM_MAX = 227 * 1024 - 1024
A_STAGE_BYTES = BM * BK * 2
SLAB_BYTES = (BM + 8) * BK * 2
MAX_STAGES = 8                                 # full_bar[8] / empty_bar[8]
UP2_BN = (64, 128, 256)                        # gemm_v3.cu v3_up2_tile: the transposed-conv store is compiled for these only


def r16(n: int) -> int:
    return (n + 15) // 16 * 16


def mt_max(BN: int) -> int:
    """gemm_v3.cu:368: a taller tile than the accumulator registers hold runs as the tallest that fits."""
    return min(4, V3_ACC_COLS // BN)


def b_bytes(BN: int) -> int:
    return (BN * BK * 2 + 1023) & ~1023        # gemm_v3.cu:370


def slab_fits(BN: int, MT: int) -> bool:
    """gemm_v3.cu:375-376: slab mode needs two stages of MT slabs + three weight tiles."""
    return 2 * (MT * SLAB_BYTES + 3 * b_bytes(BN)) <= V3_DYN_SMEM_MAX - 1024


def stages(BN: int, MT: int, slab: bool) -> int:
    """gemm_v3.cu:377-381: as many pipeline stages as fit in shared memory, at most 8 (0: the tile does not fit)."""
    stage = MT * SLAB_BYTES + 3 * b_bytes(BN) if slab else MT * A_STAGE_BYTES + b_bytes(BN)
    n = min(MAX_STAGES, (V3_DYN_SMEM_MAX - 1024) // stage)
    return n if n >= 2 else 0


@dataclass(frozen=True)
class Config:
    BN: int
    MT: int
    no_slab: int = 0          # the GEMM plan field no_slab
    slab: int = 0             # what the kernel runs: slab mode only for 3x3 stride-1 convs that fit
    stages: int = 0

    def name(self) -> str:
        return f"BN={self.BN} MT={self.MT} slab={self.slab} stages={self.stages}"


def _cfg(BN, MT, no_slab, slab):
    return Config(BN, MT, no_slab, int(slab), stages(BN, MT, slab))


def tile_space(route: str, N: int) -> List[Config]:
    """Every configuration the kernel runs for a GEMM of N output columns on `route`.

    1x1 / im2col / s2: (BN, MT) for every multiple of 16 up to round_up(N, 16) (all the tuner can return: gemm_v3_candidates rounds a
    wider candidate down to it) and MT 1 .. mt_max(BN).  slab (3x3 stride-1): the same shapes, each run in slab mode where two slab
    stages fit and with per-tap loads (no_slab).  up2: BN 64 / 128 / 256.  stem7x7s2 (taps = 4): as 1x1 (N = Cout <= 64).
    tr (the swap-AB FC on tensor cores): N is the batch; BN = round_up(batch, 16) is fixed (engine.cu:195), MT runs 1 .. mt_max."""
    if route == "tr":
        BN = r16(N)
        return [_cfg(BN, mt, 0, False) for mt in range(1, mt_max(BN) + 1)]
    bns = UP2_BN if route == "up2" else range(16, min(256, r16(N)) + 1, 16)
    out = []
    for BN in bns:
        for mt in range(1, mt_max(BN) + 1):
            if route == "slab":
                if slab_fits(BN, mt):
                    out.append(_cfg(BN, mt, 0, True))
                out.append(_cfg(BN, mt, 1, False))
            else:
                assert route in ("1x1", "im2col", "s2", "up2", "stem7x7s2"), route
                out.append(_cfg(BN, mt, 0, False))
    return out


def force_tile(pb, op_index: int, BN: int, MT: int, no_slab: int = 0) -> None:
    """Write the tile fields of a packed GEMM op: BN, the MT hint and no_slab (per-tap loads).  The swap-AB FC takes only MT: its BN
    follows the batch."""
    t, p, _ = pb.ops[op_index]
    assert t == plan.OP_GEMM, t
    if not p.transposed:
        p.BN = BN
        p.no_slab = no_slab
    p.MT = MT


def clone_gemm(pb, op_index: int, out) -> int:
    """Append a copy of GEMM op `op_index` that writes `out` (anything with .buf and .coff) instead; weights, bias and inputs are
    shared."""
    t, p, f = pb.ops[op_index]
    assert t == plan.OP_GEMM
    q = p.copy()
    q.out_buf, q.out_coff = out.buf, out.coff
    pb.ops.append((t, q, list(f)))
    return len(pb.ops) - 1


def op_route(pb, i: int) -> Optional[str]:
    """oc.plan_route of GEMM op i alone, with the op that feeds it (IM2COL / STEMPACK) when there is one."""
    t, p, _ = pb.ops[i]
    pre = [op for op in pb.ops if op[0] in (plan.OP_IM2COL, plan.OP_STEMPACK) and op[1].out_buf == p.a_buf]
    return oc.plan_route(SimpleNamespace(pb=SimpleNamespace(ops=pre[:1] + [pb.ops[i]])))


# ---------------------------------------------------------------------------------------------------------------------------
# sweep cases
# ---------------------------------------------------------------------------------------------------------------------------
@dataclass
class Sweep:
    name: str
    route: str                                  # a route of tile_space
    pb: plan.PlanBuilder
    B: int
    ins: List[Tuple[int, int, np.ndarray]]      # as oc.Spec.ins
    ref: np.ndarray
    bound: np.ndarray
    C: int                                      # channels each op writes
    ops: List[Tuple[int, Config, Tuple[int, int]]] = field(default_factory=list)   # (op index, config, (out buffer, channel offset))


# name, route, B, H, W, Cin, in_off, Cout, k, s, act, res ("pre" / "post" / None), f32 output
SWEEP_CASES = [
    ("1x1-k200-res-post", "1x1", 3, 40, 40, 200, 24, 248, 1, 1, 1, "post", False),   # K tail 8; N ragged for nearly every BN
    ("1x1-k1032-res-pre", "1x1", 2, 16, 20, 1032, 8, 248, 1, 1, 2, "pre", False),     # 17 k-blocks: the stage ring wraps
    ("1x1-n40-f32", "1x1", 2, 9, 15, 64, 40, 40, 1, 1, 0, None, True),                # BN 16 / 32 / 48 with MT up to 4
    ("3x3-c192-res-pre", "slab", 2, 24, 40, 192, 64, 248, 3, 1, 2, "pre", False),     # 27 pipeline steps per tile; 2-stage slab rings
    ("3x3-w130-res-post", "slab", 3, 6, 130, 64, 0, 40, 3, 1, 1, "post", False),      # wide rows, narrow BN
    ("s2-3x3", "s2", 2, 40, 26, 128, 64, 248, 3, 2, 3, None, False),                  # 13 x 9 = 117-row patches
    ("s2-1x1", "s2", 2, 40, 26, 128, 0, 248, 1, 2, 1, "post", False),
    ("im2col-k5", "im2col", 2, 12, 14, 24, 8, 248, 5, 1, 1, None, False),              # Kpad 600: K tail 24 through the patch matrix
    ("up2", "up2", 2, 9, 11, 64, 8, 136, 2, 2, 0, None, False),                        # N = 4 * 136 = 544 into a concat slice
    ("stem7x7s2", "stem7x7s2", 2, 64, 96, 3, 0, 64, 7, 2, 2, None, False),            # taps = 4
]
OUT_OFF = 8                                     # every output is the channel slice [8, 8 + C) of a buffer 16 channels wider


def sweep_case(case, seed=0) -> Sweep:
    name, route, B, H, W, cin, in_off, cout, k, s, act, res, f32 = case
    rng = np.random.default_rng(seed)
    if route == "up2":
        return _up2_sweep(name, B, H, W, cin, in_off, cout, rng)
    if route == "stem7x7s2":
        return _stem_sweep(name, B, H, W, cout, act, rng)
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
    xv = oc.view(pb, H, W, cin, in_off)
    rv = None if res is None else oc.view(pb, Ho, Wo, cout, 24)
    x = oc.f16(rng, (B, cin, H, W))
    w = oc.f16(rng, (cout, cin, k, k), np.sqrt(2.0 / (cin * k * k)))
    b = oc.f16(rng, cout, 0.1)
    r = oc.f16(rng, (B, cout, Ho, Wo)) if res is not None else None
    pb.conv(xv, w.astype(np.float32), b.astype(np.float32), k, s, act, out=oc.view(pb, Ho, Wo, cout, OUT_OFF, f32=f32), res=rv, res_pre_act=(res == "pre"), out_f32=f32)
    ref, S, a, rp = oc.conv_ref(x, w, b, s, pad, act, r, res or "none")
    K = k * k * oc.r8(xv.C) if route != "im2col" else oc.r8(k * k * cin)
    ins = [(xv.buf, xv.coff, x)] + ([(rv.buf, rv.coff, r)] if rv is not None else [])
    sw = Sweep(name, route, pb, B, ins, ref, oc.gemm_bound(ref, S, K, act, a, rp, f32), cout)
    _fan_out(sw, lambda: oc.view(pb, Ho, Wo, cout, OUT_OFF, f32=f32), tile_space(route, cout))
    return sw


def _fan_out(sw, new_out, configs):
    """One GEMM op per configuration: the builder's op takes the first, clones writing fresh outputs take the rest."""
    first = max(i for i, (t, _, _) in enumerate(sw.pb.ops) if t == plan.OP_GEMM)
    for j, c in enumerate(configs):
        i = first if j == 0 else clone_gemm(sw.pb, first, new_out())
        force_tile(sw.pb, i, c.BN, c.MT, c.no_slab)
        p = sw.pb.ops[i][1]
        sw.ops.append((i, c, (p.out_buf, p.out_coff)))


def _up2_sweep(name, B, H, W, cin, in_off, cout, rng) -> Sweep:
    pb = plan.PlanBuilder(plan.MODEL_YOLOV6, 3, H, W)
    xv = oc.view(pb, H, W, cin, in_off)
    x = oc.f16(rng, (B, cin, H, W))
    w = oc.f16(rng, (cin, cout, 2, 2), np.sqrt(1.0 / cin))
    b = oc.f16(rng, cout, 0.1)
    pb.conv_transpose2x2(xv, w.astype(np.float32), b.astype(np.float32), oc.view(pb, 2 * H, 2 * W, cout, OUT_OFF))
    xt, wt = torch.from_numpy(x), torch.from_numpy(w)
    ref = F.conv_transpose2d(xt, wt, torch.from_numpy(b), stride=2).numpy()
    S = F.conv_transpose2d(xt.abs(), wt.abs(), torch.from_numpy(np.abs(b)), stride=2).numpy()
    sw = Sweep(name, "up2", pb, B, [(xv.buf, xv.coff, x)], ref, oc.gemm_bound(ref, S, oc.r8(cin), 0, ref), cout)
    _fan_out(sw, lambda: oc.view(pb, 2 * H, 2 * W, cout, OUT_OFF), tile_space("up2", 4 * cout))
    return sw


def _stem_sweep(name, B, H, W, cout, act, rng) -> Sweep:
    pb = plan.PlanBuilder(plan.MODEL_UFLDV2, 3, H, W)
    x = np.zeros((B, 4, H, W))
    x[:, :3] = oc.f16(rng, (B, 3, H, W))                       # the image's 4th channel is a structural zero
    w = oc.f16(rng, (cout, 3, 7, 7), np.sqrt(2.0 / (3 * 49)))
    b = oc.f16(rng, cout, 0.1)
    o = pb.stem7x7s2(pb.image, w.astype(np.float32), b.astype(np.float32), act)
    ref, S, a, _ = oc.conv_ref(x[:, :3], w, b, 2, 3, act)
    sw = Sweep(name, "stem7x7s2", pb, B, [(pb.image.buf, 0, x)], ref, oc.gemm_bound(ref, S, 49 * 4, act, a), cout)
    # the builder's output is a buffer of its own: move every op (the first included) to a slice of a wider buffer
    first = max(i for i, (t, _, _) in enumerate(pb.ops) if t == plan.OP_GEMM)
    ov = oc.view(pb, o.H, o.W, cout, OUT_OFF)
    pb.ops[first][1].out_buf, pb.ops[first][1].out_coff = ov.buf, ov.coff
    _fan_out(sw, lambda: oc.view(pb, o.H, o.W, cout, OUT_OFF), tile_space("stem7x7s2", cout))
    return sw


# ---------------------------------------------------------------------------------------------------------------------------
# FC batch sweep
# ---------------------------------------------------------------------------------------------------------------------------
FC_TR = (4096, 3203)              # K, N: 26 MB of weights, past fc_stream's 25 MB: the swap-AB GEMM on tensor cores
FC_STREAM = (4992, 1003)
FC_TR_BATCHES = sorted({1} | {b for k in range(1, 17) for b in (16 * k, 16 * k + 1) if b <= 256})
FC_STREAM_BATCHES = (1, 7, 8, 9, 255, 256)     # fc_stream works in rows of 8 images


def fc_sweep(K, N, mb, mts, act=1, f32=True, seed=0):
    """One plan holding one FC per MT hint (all share one weight tensor and read one input); returns (pb, ops, x, ref, bound)."""
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_UFLDV2, 3, 8, 8)
    xin = pb.new_dense(1, K + 16)
    x = oc.f16(rng, (mb, K))
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float16)
    b = oc.f16(rng, N, 0.1)
    ops = []
    for mt in mts:
        out = pb.new_dense(1, oc.r8(N) + 16, f32=f32)
        if not ops:
            pb.fc(xin, K, w, b.astype(np.float32), act, out)
        else:
            clone_gemm(pb, ops[0][0], SimpleNamespace(buf=out, coff=0))
        force_tile(pb, len(pb.ops) - 1, 0, mt)
        ops.append((len(pb.ops) - 1, mt, out))
    w64 = w.astype(np.float64)
    a = x @ w64.T + b
    S = np.abs(x) @ np.abs(w64).T + np.abs(b)
    ref = oc.act64(a, act)
    return pb, ops, (xin, x), ref, oc.gemm_bound(ref, S, K, act, a, None, f32)
