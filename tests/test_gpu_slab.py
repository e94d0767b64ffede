"""GPU: 3x3 stride-1 convs in slab mode (one activation slab per (dy, k-block) feeds the three dx taps) against the fp32 torch
reference and, bit for bit, against the same layer with one activation tile per tap (plan hook no_slab)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import adas_b200  # noqa: F401
from adas_b200 import _capi, plan
from gpu_util import from_padded, halo_is_zero, to_padded

pytestmark = pytest.mark.gpu


def _conv3x3(tmp_path, B, cin, cout, H, W, act, residual, tile, no_slab, out_slice=None, seed=0):
    """Runs one 3x3 stride-1 conv; returns (whole output buffer, [B,cout,H,W] result, torch reference, step description)."""
    rng = np.random.default_rng(seed)
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
    xin = pb.new_padded(H, W, cin)
    w = (rng.standard_normal((cout, cin, 3, 3)) * np.sqrt(2.0 / (cin * 9))).astype(np.float32)
    b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    res_view = pb.new_padded(H, W, cout) if residual else None
    out_view = pb.sub(pb.new_padded(H, W, out_slice[0]), out_slice[1], cout) if out_slice else None
    out = pb.conv(xin, w, b, 3, 1, act, res=res_view, res_pre_act=(residual == "pre"), out=out_view, tile=tile, no_slab=no_slab)
    path = str(tmp_path / f"slab_{seed}_{int(no_slab)}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, device=0, max_batch=B)
    x = rng.standard_normal((B, cin, H, W)).astype(np.float32)
    eng.write_buffer(xin.buf, to_padded(x, cin))
    r = None
    if residual:
        r = rng.standard_normal((B, cout, H, W)).astype(np.float32)
        eng.write_buffer(res_view.buf, to_padded(r, cout))
    if out_slice:
        eng.write_buffer(out.buf, to_padded(rng.standard_normal((B, out_slice[0], H, W)).astype(np.float32), out_slice[0]))
    eng.run(B)
    buf = eng.read_buffer(out.buf, B).copy()
    descs = [eng.time_step(B, i, 1)[2] for i in range(eng.num_steps(B))]
    eng.close()
    desc = [d for d in descs if "v3" in d]
    assert len(desc) == 1, descs
    ref = F.conv2d(torch.from_numpy(x).half().float(), torch.from_numpy(w).half().float(), torch.from_numpy(b), padding=1)
    if residual == "pre":
        ref = ref + torch.from_numpy(r).half().float()
    ref = {0: lambda t: t, 1: F.silu, 2: F.relu}[act](ref)
    if residual == "post":
        ref = ref + torch.from_numpy(r).half().float()
    return buf, from_padded(buf, B, H, W, out.coff, cout), ref.numpy(), desc[0]


SLAB_CASES = [
    # B cin cout H  W   act residual  (BN, MT)   out_slice
    (2, 64, 64, 20, 24, 1, None, (64, 4), None),            # four sub-tiles, one k-block, ragged last M tile
    (2, 128, 64, 30, 34, 2, "pre", (64, 3), None),          # three sub-tiles, residual before ReLU, ragged M
    (1, 64, 64, 160, 96, 1, None, (64, 4), None),           # many tiles per CTA: the slab ring carries across tiles
    (2, 64, 64, 20, 24, 1, "post", (64, 2), None),          # two 64-wide sub-tiles, residual after SiLU
    (1, 192, 128, 40, 40, 1, "post", (128, 2), None),       # three k-blocks
    (1, 64, 320, 20, 20, 1, None, (128, 1), None),          # N = 320: last N tile half outside the tensor
    (1, 128, 320, 20, 20, 0, None, (192, 1), None),         # 192-wide tiles, last one partly outside N
    (2, 256, 160, 16, 16, 1, "post", (160, 1), None),       # BN = 160 (128 + 32 column wgmmas)
    (1, 128, 128, 40, 40, 1, "post", (128, 2), (384, 128)),  # output into a channel slice of a concat buffer
]


@pytest.mark.parametrize("case", SLAB_CASES)
def test_conv_slab_parity(tmp_path, case):
    B, cin, cout, H, W, act, residual, tile, out_slice = case
    seed = cin + cout + tile[0] + tile[1]
    buf, got, ref, desc = _conv3x3(tmp_path, B, cin, cout, H, W, act, residual, tile, False, out_slice, seed)
    assert "slab=1" in desc, desc
    err = float(np.abs(got - ref).max()) / max(1.0, float(np.abs(ref).max()))
    assert err < 4e-3, f"case {case}: relative error {err}"
    assert halo_is_zero(buf, B, H, W), "conv wrote into the zero halo"
    buf0, _, _, desc0 = _conv3x3(tmp_path, B, cin, cout, H, W, act, residual, tile, True, out_slice, seed)
    assert "slab=0" in desc0, desc0
    assert np.array_equal(buf.view(np.uint16), buf0.view(np.uint16)), f"case {case}: slab and per-tap outputs differ"


def test_conv_slab_bitwise_autotuned(tmp_path):
    """The tile chosen by the cost model and autotune, with and without slab loads: the same bits."""
    outs = [_conv3x3(tmp_path, 2, 128, 128, 40, 40, 1, None, None, ns, seed=9)[0] for ns in (False, True)]
    assert np.array_equal(outs[0].view(np.uint16), outs[1].view(np.uint16))


def test_conv_slab_not_used_when_two_stages_do_not_fit(tmp_path):
    # MT = 1, BN = 256: one slab stage (17 KiB + 3 x 32 KiB) is more than half the shared memory -> per-tap loads
    _, got, ref, desc = _conv3x3(tmp_path, 1, 128, 256, 20, 20, 1, None, (256, 1), False, seed=3)
    assert "slab=0" in desc, desc
    assert float(np.abs(got - ref).max()) / max(1.0, float(np.abs(ref).max())) < 4e-3
