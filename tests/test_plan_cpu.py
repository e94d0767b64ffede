"""CPU: host logic of the packer (adas_b200.plan): graph restatements reproduce the published FLOP / parameter counts,
BN folding and weight layout are right, the UFLD FC1 scatter matches view(-1, input_dim), the .b200w header parses."""
import os
import re
import struct

import numpy as np
import torch

import adas_b200  # noqa: F401
from adas_b200 import plan
import plan_footprint as fp


def _params(W):
    return sum(v.size for k, v in W.state_dict.items() if "num_batches" not in k and "running" not in k)


def test_yolov8l_graph_matches_published_counts():
    W = plan.synth_weights("yolov8", 0)
    pb = plan.build_yolov8(W, "l")
    assert abs(pb.flops_per_img / 1e9 - 165.1) < 0.3            # ultralytics: 165.2 GFLOP
    assert abs(_params(W) / 1e6 - 43.7) < 0.15                  # 43.7 M
    assert pb.meta[:2] == [80, 8400] and len(pb.outputs) == 3


def test_yolov5n_graph_matches_published_counts():
    W = plan.synth_weights("yolov5", 0)
    pb = plan.build_yolov5(W, "n")
    assert abs(pb.flops_per_img / 1e9 - 4.5) < 0.15              # yolov5n: 4.5 GFLOP
    assert abs(_params(W) / 1e6 - 1.87) < 0.03
    assert pb.meta[:2] == [80, 25200]


def test_bn_folding_and_layout():
    W = plan.Weights(seed=3)
    wf, bf = W.conv_bn("m", 6, 5, 3, 1e-3)
    conv = torch.nn.Conv2d(5, 6, 3, 1, 1, bias=False)
    bn = torch.nn.BatchNorm2d(6, eps=1e-3).eval()
    sd = W.state_dict
    conv.weight.data = torch.from_numpy(sd["m.conv.weight"])
    bn.weight.data = torch.from_numpy(sd["m.bn.weight"])
    bn.bias.data = torch.from_numpy(sd["m.bn.bias"])
    bn.running_mean.data = torch.from_numpy(sd["m.bn.running_mean"])
    bn.running_var.data = torch.from_numpy(sd["m.bn.running_var"])
    x = torch.randn(2, 5, 7, 9)
    with torch.no_grad():
        ref = bn(conv(x))
        got = torch.nn.functional.conv2d(x, torch.from_numpy(wf), torch.from_numpy(bf), padding=1)
    assert torch.allclose(ref, got, atol=1e-5)
    # K-major packing: [Cout, kh, kw, Cin]
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, 8, 8)
    xin = pb.new_padded(8, 8, 64)
    w = np.arange(16 * 64 * 9, dtype=np.float32).reshape(16, 64, 3, 3) / 1e4
    pb.conv(xin, w, None, 3, 1, 0)
    packed = pb.tensors[-1].astype(np.float32).reshape(16, 3, 3, 64)
    assert np.allclose(packed, w.transpose(0, 2, 3, 1), atol=2e-3)


def test_ufld_fc1_scatter_equals_flatten():
    W = plan.synth_weights("ufldv2", 1)
    pb = plan.build_ufldv2(W, "18")
    assert abs(pb.flops_per_img / 1e9 - (75.15 - 2 * (37.58 - 0.195 - 18.9))) < 60   # res18 is lighter; sanity only
    fc1 = [op for op in pb.ops if op[0] == plan.OP_GEMM and op[1].transposed == 1][0]
    w1p = pb.tensors[fc1[1].w_tensor].astype(np.float32)            # [2048, slab]
    fh, fw = 10, 50
    fea = np.random.default_rng(0).standard_normal((8, fh, fw)).astype(np.float32)
    slab = np.zeros(((fh + 2), (fw + 2), 8), np.float32)
    slab[1:-1, 1:-1, :] = fea.transpose(1, 2, 0)
    got = w1p @ slab.ravel()
    ref = W.state_dict["cls.1.weight"].astype(np.float16).astype(np.float32) @ fea.ravel()
    assert np.allclose(got, ref, atol=1e-3)
    ln = [op for op in pb.ops if op[0] == plan.OP_LAYERNORM][0]
    assert ln[1].d_len == (fh + 2) * (fw + 2) * 8 and ln[1].d_norm == 4000


def test_plan_file_header(tmp_path):
    W = plan.synth_weights("yolov5", 0)
    pb = plan.build_yolov5(W, "n")
    path = tmp_path / "v5n.b200w"
    pb.write(str(path))
    raw = path.read_bytes()
    h = struct.unpack_from(plan.HDR_FMT, raw)
    assert h[0] == b"B200PLAN" and h[1] == plan.PLAN_VERSION and h[2] == plan.MODEL_YOLOV5
    assert h[3:6] == (3, 640, 640)
    n_buf, n_ops, n_t, n_out = h[6:10]
    assert (n_buf, n_ops, n_t, n_out) == (len(pb.buffers), len(pb.ops), len(pb.tensors), 3)
    blob_off, blob_bytes = h[-2:]
    assert blob_off % 256 == 0 and blob_off + blob_bytes == len(raw)
    assert plan.HDR_SIZE + n_buf * plan.BUF_SIZE + n_ops * plan.OP_SIZE + n_t * plan.TEN_SIZE + n_out * plan.OUT_SIZE <= blob_off


def test_tusimple_plan_geometry():
    """UFLDV2_TUSIMPLE (ModelConfig.init_tusimple_config + configs/tusimple_res18.py): 320x800, 100x56 / 100x41 heads, no LayerNorm."""
    W = plan.synth_weights("ufldv2", 0)
    pb = plan.build_ufldv2(W, "18", "tusimple")
    assert pb.meta[:7] == [100, 56, 100, 41, 4, 100 * 56 * 4 + 100 * 41 * 4 + 2 * 56 * 4 + 2 * 41 * 4, 1]
    assert (pb.in_h, pb.in_w) == (320, 800)
    assert not any(op[0] == plan.OP_LAYERNORM for op in pb.ops)                 # fc_norm = False: cls.0 is Identity
    assert "cls.0.weight" not in W.state_dict
    fc1 = [op for op in pb.ops if op[0] == plan.OP_GEMM and op[1].transposed == 1][0]
    assert fc1[1].Kc == (10 + 2) * (25 + 2) * 8                                  # reads the padded 10x25x8 pool slab directly
    assert plan.build_ufldv2(plan.synth_weights("ufldv2", 0), "34").meta[6] == 0  # CULane


def test_ufld_v1_plan_geometry():
    """UFLD v1 (exportLib/ultrafastLane/model.py): 288x800 input, Linear(1800, 2048), head [griding_num + 1, rows, 4], keys cls.0 / cls.2."""
    for ds, G, R in (("tusimple", 100, 56), ("culane", 200, 18)):
        W = plan.synth_weights("ufldv2", 0)
        pb = plan.build_ufldv1(W, "18", ds)
        assert pb.model_kind == plan.MODEL_UFLDV1 and (pb.in_h, pb.in_w) == (288, 800)
        assert pb.meta[:7] == [G, R, 0, 0, 4, (G + 1) * R * 4, 1 if ds == "tusimple" else 0]
        assert "cls.0.weight" in W.state_dict and W.state_dict["cls.0.weight"].shape == (2048, 1800) and "cls.1.weight" not in W.state_dict
        assert W.state_dict["cls.2.weight"].shape == ((G + 1) * R * 4, 2048)
        assert not any(op[0] == plan.OP_LAYERNORM for op in pb.ops)


def test_engine_rejects_inconsistent_plans(tmp_path):
    """Every index / offset / size of a plan is validated when it is loaded (before any device work, so this runs without a GPU):
    a corrupt or hostile plan must produce an error naming the plan, never an out-of-bounds access."""
    from adas_b200 import _capi
    W = plan.synth_weights("ufldv2", 0)
    pb = plan.build_ufldv2(W, "18", "tusimple")
    good = tmp_path / "good.b200w"
    pb.write(str(good))
    raw = good.read_bytes()
    pl = fp.parse(raw)
    n_buf = len(pb.buffers)
    first_gemm = next(i for i, op in enumerate(pb.ops) if op[0] == plan.OP_GEMM)
    cases = {
        "buffer index": fp.corrupt(raw, pl.field_off(first_gemm, "out_buf"), "<i", n_buf + 7),
        "weight tensor index": fp.corrupt(raw, pl.field_off(first_gemm, "w_tensor"), "<i", 100000),
        "channel slice": fp.corrupt(raw, pl.field_off(first_gemm, "out_coff"), "<i", 1 << 20),
        "tensor offset": fp.corrupt(raw, pl.ten_off(0), "<Q", 1 << 40),
        "dataset id": fp.corrupt(raw, 8 + 4 * 2 + 4 * 3 + 4 * 4 + 4 * 6, "<I", 7),
        "dataset geometry": fp.corrupt(raw, 8 + 4 * 2 + 4 * 3 + 4 * 4 + 4 * 6, "<I", 0),                 # TuSimple heads labelled CULane
        "op type": fp.corrupt(raw, pl.op_off(1), "<I", 99),
        "truncated blob": raw[:len(raw) - 4096],
    }
    for name, data in cases.items():
        p = tmp_path / "bad.b200w"
        p.write_bytes(data)
        try:
            _capi.Engine(str(p))
        except Exception as e:
            assert "plan" in str(e), (name, str(e))
        else:
            raise AssertionError(f"{name}: corrupt plan was accepted")
    # the untouched file passes validation: without a GPU the only complaint left is the missing device
    import torch
    if not torch.cuda.is_available():
        try:
            _capi.Engine(str(good))
        except Exception as e:
            assert "no CUDA device" in str(e), str(e)


def _plan_h_op_layout():
    """PlanOpType's enumerators {name: value} and the op structs {name: (int32 fields, nested arrays [(name, fields, count)])} of
    csrc/plan.h, in declaration order."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = re.sub(r"//[^\n]*", "", open(os.path.join(root, "vehicle-cv-adas_b200", "csrc", "plan.h")).read())
    src = src[src.index("enum PlanOpType"):]                  # the op structs follow the enum (PlanOp itself precedes it)
    enum = re.search(r"enum PlanOpType : uint32_t \{(.*?)\};", src, re.S).group(1)
    values = {n: int(v) for n, v in re.findall(r"(OP_\w+)\s*=\s*(\d+)", enum)}
    fields = lambda body: [n.strip() for decl in re.findall(r"int32_t ([^;]+);", body) for n in decl.split(",")]
    structs = {}
    for name, body in re.findall(r"struct (\w+Op) \{(.*?)\};", src, re.S):
        nested = [(m[2], fields(m[1]), int(m[3])) for m in re.findall(r"struct (\w+) \{([^}]*)\} (\w+)\[(\d+)\];", body)]
        structs[name] = (fields(re.sub(r"struct \w+ \{[^}]*\}[^;]*;", "", body)), nested)
    return values, structs


def test_plan_h_op_structs_match_op_fields():
    """plan.h's op structs (what the loader reads) and plan.OP_FIELDS (what the packer and the tests write and read) name the same
    fields in the same order; the op codes and record sizes agree."""
    values, structs = _plan_h_op_layout()
    assert len(values) == len(plan.OP_FIELDS) == len(plan.OP_NAMES) == 13
    assert {getattr(plan, n) for n in values} == set(plan.OP_FIELDS) == set(plan.OP_NAMES)
    assert sorted(structs) == sorted(n[3:].capitalize() + "Op" for n in values)          # OP_GEMM: GemmOp, OP_IM2COL: Im2colOp, ...
    for n, v in values.items():
        assert getattr(plan, n) == v, n
        flat, nested = structs[n[3:].capitalize() + "Op"]
        assert tuple(flat) == plan.OP_FIELDS[v], n
        assert nested == ([("src", list(plan.CBFUSE_SRC_FIELDS), plan.CBFUSE_MAX_SRC)] if v == plan.OP_CBFUSE else []), n
        assert len(flat) + sum(len(f) * c for _, f, c in nested) <= plan.OP_NP, n
    assert (plan.HDR_SIZE, plan.BUF_SIZE, plan.OP_SIZE, plan.TEN_SIZE, plan.OUT_SIZE) == (124, 24, 112, 24, 16)


def test_op_params_read_and_write_by_name():
    p = plan.OpParams(plan.OP_SHUFFLE2, [1, 2, 3, 4, 8, 5, 16])
    assert p == [1, 2, 3, 4, 8, 5, 16] + [0] * 16 and (p.b_buf, p.n, p.out_coff) == (3, 8, 16)
    p.out_coff = 24
    assert p == [1, 2, 3, 4, 8, 5, 24] + [0] * 16 and p.copy() == p and p.copy().typ == plan.OP_SHUFFLE2
    for bad in (lambda: p.BN, lambda: setattr(p, "BN", 64)):
        try:
            bad()
        except AttributeError as e:
            assert "shuffle2 op has no field 'BN'" in str(e)
        else:
            raise AssertionError("a field of another op type was accepted")
    pb = plan.PlanBuilder(plan.MODEL_YOLOV8, 3, 8, 8)
    try:
        pb._op(plan.OP_MAXPOOL, in_buf=0, out_coff=8, fill=1)
    except AttributeError as e:
        assert "maxpool op has no field 'fill'" in str(e)
    else:
        raise AssertionError("_op accepted a field the op does not have")


def test_plan_cache_is_private(tmp_path, monkeypatch):
    import os
    d = tmp_path / "cache"
    monkeypatch.setenv("ADAS_B200_PLAN_CACHE", str(d))
    assert plan.cache_dir() == str(d) and (os.stat(d).st_mode & 0o777) == 0o700
    os.chmod(d, 0o777)
    try:
        plan.cache_dir()
    except Exception as e:
        assert "private" in str(e)
    else:
        raise AssertionError("a world-writable plan cache must be refused")


def test_cached_plan_file_is_the_fresh_build(tmp_path, monkeypatch):
    """gpu_util.cached_plan writes the plan it has just built even when the cache already holds a file of the same name from an older
    builder: the engine must never load a plan other than the one whose weights and PlanBuilder the test compares against."""
    from gpu_util import cached_plan
    monkeypatch.setenv("ADAS_B200_PLAN_CACHE", str(tmp_path / "cache"))
    path, _, _ = cached_plan("yolov5", scale="n", in_h=64, in_w=64)
    old = open(path, "rb").read()
    get = plan.Weights.get
    monkeypatch.setattr(plan.Weights, "get", lambda self, name, shape, kind:
                        get(self, name, shape, kind) * np.float32(2.0 if name == "model.0.conv.weight" else 1.0))
    again, _, pb = cached_plan("yolov5", scale="n", in_h=64, in_w=64)
    fresh = tmp_path / "fresh.b200w"
    pb.write(str(fresh))
    assert again == path and open(path, "rb").read() == fresh.read_bytes() != old
