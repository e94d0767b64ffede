"""onnx_import.py -- ingest the reference's model files: `.onnx` -> packed sm_90a plan (`.b200w`).

The reference hands `.onnx` / `.trt` files to ONNXRuntime / TensorRT (coreEngine.py:54-55,164-166); its models come from
ultralytics / yolov5 exports (README.md:53-58) and from `TrafficLaneDetector/convertPytorchToONNX.py:60-87` (UFLD).  This module
is the H100 replacement of that ingestion step (SURVEY 8f rank 2): it reads the ONNX protobuf directly (the `onnx` package is
not a dependency -- the wire format is parsed here), recovers the convolution / linear / LayerNorm parameters, recognises the
architecture (YOLOv8 / YOLOv5 / YOLOv6 / YOLOv7 / YOLOv9 / YOLOv10 / UFLDv2, scale, class count, input size) and drives the same `plan.build_*` builders that the
state_dict path uses.  Nothing here runs the network: the graph is only a parameter container plus a shape oracle.

How parameters are matched to layers:
  * by NAME when the exporter kept module names.  ultralytics / yolov5 fuse Conv+BN in PyTorch before exporting, so their
    files carry `model.N...conv.weight` / `.conv.bias` (already folded) -- taken as they are;
  * by ORDER for convolutions whose names were lost: `torch.onnx.export` folds eval-mode BatchNorm into the preceding Conv and
    the folded tensors get anonymous names (`onnx::Conv_123`).  These are consumed in graph order, which is the module
    execution order the plan builders follow, and every shape is checked;
  * un-fused exports (Conv followed by BatchNormalization with named parameters) fold through the normal `Weights.conv_bn`.
"""
from __future__ import annotations

import hashlib
import os
import re
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import plan


# ---------------------------------------------------------------------------------------------------------------
# protobuf wire format (only what ONNX uses: varint, 64-bit, length-delimited, 32-bit)
# ---------------------------------------------------------------------------------------------------------------
def _varint(buf: memoryview, pos: int) -> Tuple[int, int]:
    result = 0
    shift = 0
    while True:
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            return result, pos
        shift += 7
        if shift > 70:
            raise ValueError("malformed varint")


def _fields(buf: memoryview):
    """Yield (field_number, wire_type, value) for one message; length-delimited values are memoryviews."""
    pos, n = 0, len(buf)
    while pos < n:
        key, pos = _varint(buf, pos)
        fno, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v = bytes(buf[pos:pos + 8]); pos += 8
        elif wt == 2:
            ln, pos = _varint(buf, pos)
            v = buf[pos:pos + ln]; pos += ln
        elif wt == 5:
            v = bytes(buf[pos:pos + 4]); pos += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt}")
        yield fno, wt, v


def _sint64(v: int) -> int:          # int64 fields are plain two's-complement varints
    return v - (1 << 64) if v >= (1 << 63) else v


def _packed_ints(wt: int, v) -> List[int]:
    if wt == 0:
        return [_sint64(v)]
    out, pos = [], 0
    while pos < len(v):
        x, pos = _varint(v, pos)
        out.append(_sint64(x))
    return out


_DTYPES = {1: np.float32, 2: np.uint8, 3: np.int8, 5: np.int16, 6: np.int32, 7: np.int64, 9: np.bool_, 10: np.float16, 11: np.float64}


def _tensor(buf: memoryview) -> Tuple[str, np.ndarray]:
    """TensorProto: dims=1, data_type=2, float_data=4, int32_data=5, int64_data=7, name=8, raw_data=9, double_data=10."""
    dims: List[int] = []
    dtype, name, raw = 1, "", None
    floats: List[float] = []
    ints: List[int] = []
    external = False
    for fno, wt, v in _fields(buf):
        if fno == 1:
            dims += _packed_ints(wt, v)
        elif fno == 2:
            dtype = v
        elif fno == 4:
            floats += list(np.frombuffer(v, "<f4")) if wt == 2 else [struct.unpack("<f", v)[0]]
        elif fno in (5, 7):
            ints += _packed_ints(wt, v)
        elif fno == 8:
            name = bytes(v).decode()
        elif fno == 9:
            raw = bytes(v)
        elif fno == 10:
            floats += list(np.frombuffer(v, "<f8")) if wt == 2 else [struct.unpack("<d", v)[0]]
        elif fno == 13 or (fno == 14 and v == 1):
            external = True
    if external:
        raise Exception(f"initializer {name}: external tensor data is not supported (re-export with a single .onnx file)")
    if dtype not in _DTYPES:
        raise Exception(f"initializer {name}: unsupported ONNX data type {dtype}")
    np_t = _DTYPES[dtype]
    if raw is not None:
        a = np.frombuffer(raw, dtype=np.dtype(np_t).newbyteorder("<")).astype(np_t)
    elif floats:
        a = np.asarray(floats, dtype=np_t)
    elif dtype == 10 and ints:           # fp16 stored as uint16 bit patterns in int32_data
        a = np.asarray(ints, dtype=np.uint16).view(np.float16)
    else:
        a = np.asarray(ints, dtype=np_t)
    return name, a.reshape(dims) if dims else a.reshape(())


@dataclass
class OnnxNode:
    op_type: str
    name: str
    inputs: List[str]
    outputs: List[str]
    attrs: Dict[str, object] = field(default_factory=dict)


def _attribute(buf: memoryview):
    """AttributeProto: name=1, f=2, i=3, s=4, t=5, floats=7, ints=8."""
    name, val = "", None
    floats: List[float] = []
    ints: List[int] = []
    has_list = False
    for fno, wt, v in _fields(buf):
        if fno == 1:
            name = bytes(v).decode()
        elif fno == 2:
            val = struct.unpack("<f", v)[0]
        elif fno == 3:
            val = _sint64(v)
        elif fno == 4:
            val = bytes(v)
        elif fno == 5:
            val = _tensor(v)[1]
        elif fno == 7:
            has_list = True
            floats += list(np.frombuffer(v, "<f4")) if wt == 2 else [struct.unpack("<f", v)[0]]
        elif fno == 8:
            has_list = True
            ints += _packed_ints(wt, v)
    if has_list:
        val = ints if ints else floats
    return name, val


def _node(buf: memoryview) -> OnnxNode:
    """NodeProto: input=1, output=2, name=3, op_type=4, attribute=5."""
    n = OnnxNode("", "", [], [])
    for fno, wt, v in _fields(buf):
        if fno == 1:
            n.inputs.append(bytes(v).decode())
        elif fno == 2:
            n.outputs.append(bytes(v).decode())
        elif fno == 3:
            n.name = bytes(v).decode()
        elif fno == 4:
            n.op_type = bytes(v).decode()
        elif fno == 5:
            k, a = _attribute(v)
            n.attrs[k] = a
    return n


def _value_info(buf: memoryview) -> Tuple[str, List[Optional[int]]]:
    """ValueInfoProto: name=1, type=2 -> TypeProto.tensor_type=1 -> shape=2 -> dim=1 -> dim_value=1 / dim_param=2."""
    name, shape = "", []
    for fno, wt, v in _fields(buf):
        if fno == 1:
            name = bytes(v).decode()
        elif fno == 2:
            for f2, _, v2 in _fields(v):
                if f2 != 1:
                    continue
                for f3, _, v3 in _fields(v2):
                    if f3 != 2:
                        continue
                    for f4, _, v4 in _fields(v3):
                        if f4 != 1:
                            continue
                        d = None
                        for f5, w5, v5 in _fields(v4):
                            if f5 == 1:
                                d = _sint64(v5)
                        shape.append(d)
    return name, shape


@dataclass
class OnnxModel:
    nodes: List[OnnxNode]
    initializers: Dict[str, np.ndarray]
    inputs: List[Tuple[str, List[Optional[int]]]]
    outputs: List[Tuple[str, List[Optional[int]]]]
    opset: int
    producer: str


def read_onnx(path: str) -> OnnxModel:
    """ModelProto: producer_name=2, graph=7, opset_import=8;  GraphProto: node=1, initializer=5, input=11, output=12."""
    if not os.path.isfile(path):
        raise Exception("The model path [%s] can't not found!" % path)
    with open(path, "rb") as f:
        data = memoryview(f.read())
    try:
        return _read_model(data, path)
    except (IndexError, ValueError, struct.error, UnicodeDecodeError) as e:
        raise Exception("The model path [%s] is not a readable ONNX file (%s: %s)" % (path, type(e).__name__, e)) from e


def _read_model(data: memoryview, path: str) -> OnnxModel:
    graph, opset, producer = None, 0, ""
    for fno, wt, v in _fields(data):
        if fno == 7:
            graph = v
        elif fno == 2:
            producer = bytes(v).decode()
        elif fno == 8:
            dom, ver = "", 0
            for f2, _, v2 in _fields(v):
                if f2 == 1:
                    dom = bytes(v2).decode()
                elif f2 == 2:
                    ver = v2
            if dom in ("", "ai.onnx"):
                opset = max(opset, ver)
    if graph is None:
        raise Exception("The model path [%s] is not an ONNX ModelProto (no graph)" % path)
    m = OnnxModel([], {}, [], [], opset, producer)
    for fno, wt, v in _fields(graph):
        if fno == 1:
            m.nodes.append(_node(v))
        elif fno == 5:
            name, a = _tensor(v)
            m.initializers[name] = a
        elif fno == 11:
            m.inputs.append(_value_info(v))
        elif fno == 12:
            m.outputs.append(_value_info(v))
    for n in m.nodes:                   # Constant nodes are parameters too (some exporters emit weights this way); identical
        if n.op_type == "Constant" and "value" in n.attrs and n.outputs:      # initializers are stored once and aliased by Identity
            m.initializers.setdefault(n.outputs[0], np.asarray(n.attrs["value"]))
        elif n.op_type == "Identity" and n.inputs and n.inputs[0] in m.initializers and n.outputs:
            m.initializers.setdefault(n.outputs[0], m.initializers[n.inputs[0]])
    m.inputs = [(k, s) for k, s in m.inputs if k not in m.initializers]      # old exporters list initializers as inputs
    return m


# ---------------------------------------------------------------------------------------------------------------
# parameters -> plan.Weights
# ---------------------------------------------------------------------------------------------------------------
class OnnxWeights(plan.Weights):
    """`plan.Weights` whose parameters come from an ONNX graph (see the module docstring for the matching rules)."""

    def __init__(self, model: OnnxModel):
        named = {k: v for k, v in model.initializers.items() if v.dtype.kind == "f" and v.ndim >= 1}
        super().__init__({k: v.astype(np.float32) for k, v in named.items()})
        # convolutions in graph order: (weight name, weight, bias or None)
        self.convs: List[Tuple[str, np.ndarray, Optional[np.ndarray]]] = []
        for n in model.nodes:
            if n.op_type != "Conv" or len(n.inputs) < 2 or n.inputs[1] not in model.initializers:
                continue
            w = model.initializers[n.inputs[1]].astype(np.float32)
            b = model.initializers[n.inputs[2]].astype(np.float32) if len(n.inputs) > 2 and n.inputs[2] in model.initializers else None
            self.convs.append((n.inputs[1], w, b))
        # the bias a named convolution actually uses is the one its node references (exporters share identical initializers, so
        # `x.bias` may be stored once under another module's name)
        self._node_bias = {name: b for name, _, b in self.convs}
        self._anon = [c for c in self.convs if not _is_module_name(c[0])]
        self._anon_used = set()
        self.used_anonymous = 0

    def conv_bn(self, prefix: str, cout: int, cin: int, k: int, eps: float, conv_key="conv", bn_key="bn", res_branch=False):
        wkey = f"{prefix}.{conv_key}.weight" if conv_key else f"{prefix}.weight"
        bkey = wkey[:-len("weight")] + "bias"
        sd = self.state_dict
        if wkey in sd and f"{prefix}.{bn_key}.running_var" in sd:                # un-fused export: fold here
            return super().conv_bn(prefix, cout, cin, k, eps, conv_key, bn_key, res_branch)
        if wkey in sd:                                                            # fused before export, names kept
            w = sd[wkey]
            assert tuple(w.shape) == (cout, cin, k, k), f"{wkey}: expected {(cout, cin, k, k)}, file has {tuple(w.shape)}"
            b = self._node_bias.get(wkey)
            if b is None:
                b = sd[bkey] if bkey in sd else np.zeros(cout, np.float32)
            return w.astype(np.float32), b.astype(np.float32)
        # BN folded by the exporter: anonymous tensors, consumed in graph (= execution) order.  A residual block's 1x1 shortcut may
        # be traced before or after its two 3x3 convolutions (torchvision runs it after bn2), so the first unconsumed tensor of the
        # expected shape among the next three is taken.
        pending = [i for i in range(len(self._anon)) if i not in self._anon_used][:3]
        if not pending:
            raise Exception(f"ONNX file has no parameters left for {prefix} (architecture mismatch?)")
        for i in pending:
            name, w, b = self._anon[i]
            if tuple(w.shape) == (cout, cin, k, k):
                self._anon_used.add(i)
                self.used_anonymous += 1
                return w, (b if b is not None else np.zeros(cout, np.float32))
        name, w, _ = self._anon[pending[0]]
        raise Exception(f"{prefix}: expected a {(cout, cin, k, k)} convolution, the next unnamed Conv in the file ({name}) is {tuple(w.shape)}; "
                        "export with the module names kept (fuse Conv+BN in PyTorch before torch.onnx.export, as ultralytics does)")

    def conv_bias(self, prefix: str, cout: int, cin: int, k: int):
        return self.conv_bn(prefix, cout, cin, k, 0.0, conv_key="", bn_key="__no_bn__")

    def repconvn(self, prefix: str, cout: int, cin: int, eps: float):
        """Fused (`conv.weight`) or named un-fused RepConvN as in plan.Weights; exporter-folded, its 3x3 and 1x1 branches are two
        anonymous convolutions in graph order, summed here in fp64."""
        if f"{prefix}.conv.weight" in self.state_dict or f"{prefix}.conv1.bn.running_var" in self.state_dict:
            return super().repconvn(prefix, cout, cin, eps)
        w3, b3 = self.conv_bn(f"{prefix}.conv1", cout, cin, 3, eps)
        w1, b1 = self.conv_bn(f"{prefix}.conv2", cout, cin, 1, eps)
        w = w3.astype(np.float64)
        w[:, :, 1, 1] += w1[:, :, 0, 0]
        return w.astype(np.float32), (b3.astype(np.float64) + b1).astype(np.float32)

    def repvggdw(self, prefix: str, c: int, eps: float):
        """Fused (`conv.weight`) or named un-fused RepVGGDW as in plan.Weights; exporter-folded, its 7x7 and 3x3 depthwise branches are
        two anonymous convolutions in graph order (a file fused upstream has the 7x7 alone), summed here in fp64."""
        if f"{prefix}.conv.weight" in self.state_dict or f"{prefix}.conv.bn.running_var" in self.state_dict:
            return super().repvggdw(prefix, c, eps)
        w7, b7 = self.conv_bn(f"{prefix}.conv", c, 1, 7, eps)
        nxt = next((i for i in range(len(self._anon)) if i not in self._anon_used), None)
        if nxt is None or tuple(self._anon[nxt][1].shape) != (c, 1, 3, 3):
            return w7, b7
        w3, b3 = self.conv_bn(f"{prefix}.conv1", c, 1, 3, eps)
        w = w7.astype(np.float64)
        w[:, :, 2:5, 2:5] += w3
        return w.astype(np.float32), (b7.astype(np.float64) + b3).astype(np.float32)


def _is_module_name(name: str) -> bool:
    """True for exporter-kept parameter names (`model.0.conv.weight`, `pool.weight`), False for `onnx::Conv_123` and friends."""
    return name.endswith(".weight") and "::" not in name and not name.split(".")[0].isdigit()


# ---------------------------------------------------------------------------------------------------------------
# architecture recognition
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class ModelSpec:
    kind: str                 # "yolov8" | "yolov5" | "yolov7" | "yolov6" | "yolov6-lite" | "yolov9" | "yolov10" | "ufldv2"
    scale: str                # YOLO scale letter ("tiny" / "base" for YOLOv7) or ResNet depth ("18" / "34")
    nc: int = 80
    in_h: int = 640
    in_w: int = 640
    act: Optional[str] = None            # YOLOv7: "silu" | "leaky"
    anchors: Optional[Tuple[float, ...]] = None     # YOLOv7: 18 anchor sizes in pixels when the file carries them
    reg_max: int = 0                     # YOLOv6: 0 (raw l, t, r, b) or 16 (17-bin DFL)
    acts: Optional[Tuple[str, str, str]] = None     # YOLOv6: activations of the body / neck / head roles, read from the graph


_V8_WIDTH = {16: "n", 32: "s", 48: "m", 64: "l", 80: "x"}


def recognise(model: OnnxModel) -> ModelSpec:
    w = OnnxWeights(model)
    if not w.convs:
        raise Exception("no convolutions found in the ONNX graph")
    in_shape = model.inputs[0][1] if model.inputs else []
    in_h = int(in_shape[2]) if len(in_shape) == 4 and in_shape[2] else 0
    in_w = int(in_shape[3]) if len(in_shape) == 4 and in_shape[3] else 0
    first = w.convs[0][1]
    shapes = [tuple(c[1].shape) for c in w.convs]
    if first.shape[1:] == (3, 7, 7):                                          # torchvision ResNet stem -> UFLDv2
        n3 = sum(1 for s in shapes if s[2:] == (3, 3))
        depth = {16: "18", 32: "34"}.get(n3)
        if depth is None:
            raise Exception(f"UFLD backbone with {n3} 3x3 convolutions is not supported (ResNet-18/34 only)")
        return ModelSpec("ufldv2", depth, 0, in_h or 320, in_w or 1600)
    if _is_yolov9(model):                                            # ADown / AConv's 2x2 stride-1 average pool; no other family pools so
        return _recognise_yolov9(model, w, in_h, in_w)
    if any(n.op_type == "ConvTranspose" for n in model.nodes):       # YOLOv6's BiFusion; v5 / v7 / v8 upsample with Resize
        return _recognise_yolov6(model, w, in_h, in_w)
    if _is_yolov6_lite(model):                                       # depthwise convs + SEBlock's HardSigmoid, no transposed conv
        return _recognise_yolov6_lite(model, w, in_h, in_w)
    if _is_yolov7(model, w):
        return _recognise_yolov7(model, w, in_h, in_w)
    if _is_yolov10(model):                                           # depthwise convs + PSA's softmax; v6-Lite is taken above
        return _recognise_yolov10(model, w, in_h, in_w)
    cout0, k0 = first.shape[0], first.shape[2]
    if cout0 not in _V8_WIDTH:
        raise Exception(f"unrecognised YOLO width: first convolution has {cout0} output channels")
    scale = _V8_WIDTH[cout0]
    named_nc = None                     # the class count is read from the head's own tensors when their names survived
    for name, cw, _ in w.convs:
        if re.fullmatch(r"model\.\d+\.cv3\.\d+\.2\.weight", name):      # YOLOv8 Detect.cv3[i][2]: Conv2d(c3, nc, 1)
            named_nc = cw.shape[0]
        elif re.fullmatch(r"model\.\d+\.m\.\d+\.weight", name) and cw.shape[2:] == (1, 1) and cw.shape[0] % 3 == 0:
            named_nc = cw.shape[0] // 3 - 5                                     # YOLOv5 Detect.m[i]: Conv2d(c, 3 * (nc + 5), 1)
    if k0 == 6:                                                               # yolov5 v6.x stem Conv(3, c, 6, 2, 2)
        if named_nc is not None:
            return ModelSpec("yolov5", scale, named_nc, in_h or 640, in_w or 640)
        no = [s[0] for s in shapes if s[2:] == (1, 1)][-1]                    # Detect.m[i]: 3 * (nc + 5)
        assert no % 3 == 0, f"YOLOv5 head with {no} outputs"
        return ModelSpec("yolov5", scale, no // 3 - 5, in_h or 640, in_w or 640)
    if k0 == 3:
        if named_nc is not None:
            return ModelSpec("yolov8", scale, named_nc, in_h or 640, in_w or 640)
        # Detect.cv3[i][2]: Conv2d(c3, nc, 1) -- the last 1x1 convolutions before the (optional) fixed DFL conv
        ones = [s for s in shapes if s[2:] == (1, 1) and s[0] != 1]
        return ModelSpec("yolov8", scale, ones[-1][0], in_h or 640, in_w or 640)
    raise Exception(f"unrecognised first convolution {first.shape}")


_V7_SUPPORTED = "YOLOv7 and YOLOv7-tiny (P5, 3 detection levels), YOLOv7-W6 / E6 / D6 / E6E (P6, 4 levels; YOLOv7-X is not supported)"


def _is_yolov7(model: OnnxModel, w: OnnxWeights) -> bool:
    """YOLOv7 family: RepConv / IDetect names where they survive, else the 2x2 stride-2 max pool of its MP blocks (YOLOv5 / v8 pool
    5x5 only) or the ReOrg space-to-depth stem of the P6 models (first convolution on 12 channels)."""
    if any("rbr_reparam" in n or "rbr_dense" in n or n.endswith(".implicit") for n in model.initializers):
        return True
    if any(n.op_type == "MaxPool" and list(n.attrs.get("kernel_shape", [])) == [2, 2] for n in model.nodes):
        return True
    return w.convs[0][1].shape[1] == 12


def _recognise_yolov7(model: OnnxModel, w: OnnxWeights, in_h: int, in_w: int) -> ModelSpec:
    first = w.convs[0][1]
    stem = next(n for n in model.nodes if n.op_type == "Conv" and n.inputs[1] == w.convs[0][0])
    stride0 = list(stem.attrs.get("strides", [1, 1]))[0]
    heads = [(name, cw) for name, cw, _ in w.convs if re.fullmatch(r"model\.\d+\.m\.\d+\.weight", name)]
    if not heads:                               # names lost: the detection convs are the trailing 1x1 convs with 3 * (nc + 5) outputs
        tail = w.convs[::-1]
        no = tail[0][1].shape[0]
        n = 0
        while n < len(tail) and tail[n][1].shape[0] == no and tail[n][1].shape[2:] == (1, 1):
            n += 1
        heads = [(name, cw) for name, cw, _ in tail[:n][::-1]]
    no = heads[-1][1].shape[0]
    if first.shape[1] == 12:
        return _recognise_yolov7_p6(model, w, stem, heads, in_h, in_w)
    if first.shape != (32, 3, 3, 3) or stride0 not in (1, 2) or len(heads) != 3 or no % 3 != 0 or (in_h and in_h > 1024):
        raise Exception(f"YOLOv7-family file outside the supported models: first convolution {tuple(first.shape)} stride {stride0}, "
                        f"{len(heads)} detection levels, input {in_h}x{in_w}; supported: {_V7_SUPPORTED}")
    scale = "base" if stride0 == 1 else "tiny"
    named = re.fullmatch(r"model\.(\d+)\.m\.\d+\.weight", heads[-1][0])
    if named and int(named.group(1)) != {"base": 105, "tiny": 77}[scale]:
        raise Exception(f"YOLOv7 head at layer {named.group(1)} does not match the {scale} graph; supported: {_V7_SUPPORTED}")
    act = "leaky" if any(n.op_type == "LeakyRelu" for n in model.nodes) else "silu"
    return ModelSpec("yolov7", scale, no // 3 - 5, in_h or 640, in_w or 640, act, _v7_anchors(model, 3))


def _v7_anchors(model: OnnxModel, levels: int) -> Optional[Tuple[float, ...]]:
    """IDetect's `anchor_grid` ([levels, 1, 3, 1, 1, 2]) or, in constant-folded exports, one [1, 3, 1, 1, 2] tensor per level in graph order."""
    grids = [v for k, v in model.initializers.items() if k.endswith("anchor_grid") and v.size == 6 * levels]
    if not grids:
        per_level = [v for k, v in model.initializers.items() if tuple(v.shape) == (1, 3, 1, 1, 2) and v.dtype.kind == "f"]
        if len(per_level) == levels:
            grids = [np.concatenate([g.reshape(6) for g in per_level])]
    return tuple(float(v) for v in np.asarray(grids[0], np.float32).reshape(6 * levels)) if grids else None


def reorg_slices(model: OnnxModel, stem) -> Optional[List[Tuple[int, int]]]:
    """(row, column) offsets of the four stride-2 slices of the image that the stem convolution's input concatenates, in concat order
    (upstream ReOrg: x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]); None if that input is not such a
    Concat of Slice chains on the network input."""
    image = model.inputs[0][0] if model.inputs else None
    prod = {o: n for n in model.nodes for o in n.outputs}
    cat = prod.get(stem.inputs[0])
    if cat is None or cat.op_type != "Concat" or len(cat.inputs) != 4 or int(cat.attrs.get("axis", 1)) % 4 != 1:
        return None
    order = []
    for t in cat.inputs:
        off: Dict[int, int] = {}
        while t != image:
            n = prod.get(t)
            if n is None or n.op_type != "Slice" or len(n.inputs) < 5 or any(i not in model.initializers for i in n.inputs[1:5]):
                return None
            starts, _, axes, steps = (np.asarray(model.initializers[i]).reshape(-1) for i in n.inputs[1:5])
            for s, a, st in zip(starts, axes, steps):
                a = int(a) % 4
                if a not in (2, 3) or int(st) != 2 or a in off:
                    return None
                off[a] = int(s)
            t = n.inputs[0]
        if set(off) != {2, 3}:
            return None
        order.append((off[2], off[3]))
    return order


# convolutions of each P6 file (tells E6 from E6E when the module names are gone); stem width -> scales
_P6_CONVS = {"w6": 107, "e6": 145, "d6": 167, "e6e": 244}
_P6_STEM = {64: ("w6",), 80: ("e6", "e6e"), 96: ("d6",)}


def _recognise_yolov7_p6(model: OnnxModel, w: OnnxWeights, stem, heads, in_h: int, in_w: int) -> ModelSpec:
    """YOLOv7 P6 (W6 / E6 / D6 / E6E): a ReOrg stem (the image's four stride-2 slices, concatenated in upstream's order) feeding Conv(12, c, 3),
    4 detection convs, an input that is a multiple of 64."""
    first = w.convs[0][1]
    cands = _P6_STEM.get(int(first.shape[0]), ()) if tuple(first.shape[1:]) == (12, 3, 3) else ()
    if not cands:
        raise Exception(f"YOLOv7 P6 stem {tuple(first.shape)}: 64 (W6), 80 (E6 / E6E) or 96 (D6) channels from a 12-channel ReOrg; supported: {_V7_SUPPORTED}")
    order = reorg_slices(model, stem)
    if order != [tuple(s) for s in plan.REORG_SLICES]:
        raise Exception(f"YOLOv7 P6 stem input is not upstream's ReOrg of the image (slice offsets {order}, expected "
                        f"{[tuple(s) for s in plan.REORG_SLICES]}); supported: {_V7_SUPPORTED}")
    no = heads[-1][1].shape[0]
    if len(heads) != 4 or no % 3 != 0:
        raise Exception(f"YOLOv7 file with a ReOrg stem and {len(heads)} detection levels (a P6 model has 4); supported: {_V7_SUPPORTED}")
    if (in_h and in_h % 64) or (in_w and in_w % 64):
        raise Exception(f"YOLOv7 P6 file with a {in_h}x{in_w} input: a multiple of 64 (stride-64 head); supported: {_V7_SUPPORTED}")
    named = re.fullmatch(r"model\.(\d+)\.m\.\d+\.weight", heads[-1][0])
    if named:
        scales = [s for s in cands if plan.YOLOV7_P6[s]["det"] == int(named.group(1))]
    else:
        scales = [s for s in cands if _P6_CONVS[s] == len(w.convs)]
    if len(scales) != 1:
        raise Exception(f"YOLOv7 P6 file with a {first.shape[0]}-channel stem and {len(w.convs)} convolutions"
                        f"{f', head at layer {named.group(1)}' if named else ''} matches none of {', '.join(cands)}; supported: {_V7_SUPPORTED}")
    act = "leaky" if any(n.op_type == "LeakyRelu" for n in model.nodes) else "silu"
    return ModelSpec("yolov7", scales[0], no // 3 - 5, in_h or 1280, in_w or 1280, act, _v7_anchors(model, 4))


_V6_SUPPORTED = ("YOLOv6-N / S / M / L (release 0.4.0, P5, 3 detection levels, BiFusion's transposed convs) and YOLOv6-Lite-S / M / L "
                 "(4 detection levels, depthwise convs and SEBlock, no transposed conv, input a multiple of 32); the P6 models and the 2.x "
                 "models are not supported")
_V6_WIDTH = {16: "n", 32: "s", 48: "m", 64: "l"}


def conv_activations(model: OnnxModel) -> Dict[str, str]:
    """weight name -> activation applied to that Conv's output: "relu" (Relu), "silu" (Sigmoid and a Mul of the conv output with it),
    "sigmoid" (a Sigmoid alone) or "none"."""
    users: Dict[str, List] = {}
    for n in model.nodes:
        for i in n.inputs:
            users.setdefault(i, []).append(n)
    acts = {}
    for n in model.nodes:
        if n.op_type != "Conv" or len(n.inputs) < 2 or not n.outputs:
            continue
        y = n.outputs[0]
        us = users.get(y, [])
        act = "none"
        if any(u.op_type == "Relu" for u in us):
            act = "relu"
        else:
            sig = [u for u in us if u.op_type == "Sigmoid"]
            if sig:
                act = "silu" if any(u.op_type == "Mul" and sig[0].outputs[0] in u.inputs for u in us) else "sigmoid"
        acts[n.inputs[1]] = act
    return acts


def _v6_role(name: str) -> Optional[str]:
    """activation role of a YOLOv6 conv by its module name (plan.build_yolov6): None for the prediction / DFL-projection convs."""
    if re.match(r"detect\.(stems|cls_convs|reg_convs)\.", name):
        return "head"
    if name.startswith("detect."):
        return None
    if re.match(r"neck\.(reduce_layer\d|Bifusion\d|downsample\d)\.", name):
        return "neck"
    return "body"


def _recognise_yolov6(model: OnnxModel, w: OnnxWeights, in_h: int, in_w: int) -> ModelSpec:
    grouped = [n.inputs[1] for n in model.nodes if n.op_type == "Conv" and int(n.attrs.get("group", 1)) > 1]
    if grouped:
        raise Exception(f"YOLOv6 file with grouped / depthwise convolutions ({grouped[0]}) and transposed convolutions: neither "
                        f"YOLOv6-N / S / M / L nor YOLOv6-Lite; supported: {_V6_SUPPORTED}")
    named = {k for k in model.initializers if _is_module_name(k)}
    cls = sorted((k for k in named if re.fullmatch(r"detect\.cls_preds\.\d+\.weight", k)), key=lambda k: int(k.split(".")[2]))
    reg = sorted((k for k in named if re.fullmatch(r"detect\.reg_preds\.\d+\.weight", k)), key=lambda k: int(k.split(".")[2]))
    if not cls or len(cls) != len(reg):
        raise Exception("YOLOv6 file without its module names (detect.cls_preds.*): export the fused model with torch.onnx.export, which "
                        f"keeps them; supported: {_V6_SUPPORTED}")
    if len(cls) != 3 or (in_h and in_h > 1024) or (in_w and in_w > 1024):
        raise Exception(f"YOLOv6 file with {len(cls)} detection levels at {in_h}x{in_w} (a P6 model?); supported: {_V6_SUPPORTED}")
    cout0 = w.convs[0][1].shape[0]
    if w.convs[0][1].shape[1:] != (3, 3, 3) or cout0 not in _V6_WIDTH:
        raise Exception(f"YOLOv6 stem {tuple(w.convs[0][1].shape)} is not one of N / S / M / L; supported: {_V6_SUPPORTED}")
    scale = _V6_WIDTH[cout0]
    nc = int(model.initializers[cls[0]].shape[0])
    nbox = int(model.initializers[reg[0]].shape[0])
    if nbox not in (4, 68):
        raise Exception(f"YOLOv6 box head with {nbox} outputs (4: raw distances, 68: 17-bin DFL); supported: {_V6_SUPPORTED}")
    acts = conv_activations(model)
    roles: Dict[str, str] = {}
    for name, _, _ in w.convs:                          # graph order: each role's activation is its first conv's
        role = _v6_role(name)
        if role is None:
            continue
        a = acts.get(name, "none")
        if a not in ("relu", "silu"):
            raise Exception(f"YOLOv6 conv {name} has activation {a!r}; the {role} convolutions take ReLU or SiLU")
        if roles.setdefault(role, a) != a:
            raise Exception(f"YOLOv6 conv {name} has activation {a!r}, the other {role} convolutions {roles[role]!r}: "
                            "a graph the packer cannot represent")
    return ModelSpec("yolov6", scale, nc, in_h or 640, in_w or 640, reg_max=0 if nbox == 4 else 16,
                     acts=(roles.get("body", "relu"), roles.get("neck", "relu"), roles.get("head", "silu")))


_V6_LITE_WIDTH = {176: "s", 288: "m", 384: "l"}      # stage-4 output width (plan.yolov6_lite_widths)


def _depthwise(model: OnnxModel) -> bool:
    """Any depthwise convolution: group = Cin = Cout > 1."""
    return any(n.op_type == "Conv" and int(n.attrs.get("group", 1)) > 1 and len(n.inputs) > 1 and n.inputs[1] in model.initializers
               and model.initializers[n.inputs[1]].shape[1] == 1 and model.initializers[n.inputs[1]].shape[0] == int(n.attrs["group"])
               for n in model.nodes)


def _is_yolov6_lite(model: OnnxModel) -> bool:
    """Depthwise convolutions together with SEBlock's HardSigmoid gate (Hardswish itself exports as HardSwish at opset >= 14, as
    HardSigmoid + Mul at opset 12).  YOLOv10 files have depthwise convs but no HardSigmoid; no other supported family has one."""
    return _depthwise(model) and any(n.op_type == "HardSigmoid" for n in model.nodes)


def _recognise_yolov6_lite(model: OnnxModel, w: OnnxWeights, in_h: int, in_w: int) -> ModelSpec:
    """YOLOv6-Lite-S / M / L: the scale comes from the stage-4 output width (the widest convolution outside the class predictions:
    176 / 288 / 384), the class count from `detect.cls_preds.0`, which must have kept its module name."""
    named = {k for k in model.initializers if _is_module_name(k)}
    cls = sorted((k for k in named if re.fullmatch(r"detect\.cls_preds\.\d+\.weight", k)), key=lambda k: int(k.split(".")[2]))
    if not cls:
        raise Exception("YOLOv6-Lite file without its module names (detect.cls_preds.*): export the model with torch.onnx.export, which "
                        f"keeps them; supported: {_V6_SUPPORTED}")
    if len(cls) != 4:
        raise Exception(f"YOLOv6-Lite file with {len(cls)} detection levels (4: strides 8 / 16 / 32 / 64); supported: {_V6_SUPPORTED}")
    if len(model.outputs) != 1:
        raise Exception(f"YOLOv6-Lite file with {len(model.outputs)} outputs; supported: {_V6_SUPPORTED}")
    if (in_h and in_h % 32) or (in_w and in_w % 32):
        raise Exception(f"YOLOv6-Lite file with a {in_h}x{in_w} input: a multiple of 32; supported: {_V6_SUPPORTED}")
    width = max(int(cw.shape[0]) for name, cw, _ in w.convs if not name.startswith("detect.cls_preds."))
    if width not in _V6_LITE_WIDTH:
        raise Exception(f"YOLOv6-Lite file with a stage-4 width of {width} channels (176: S, 288: M, 384: L); supported: {_V6_SUPPORTED}")
    return ModelSpec("yolov6-lite", _V6_LITE_WIDTH[width], int(model.initializers[cls[0]].shape[0]), in_h or 320, in_w or 320)


_V9_SUPPORTED = ("YOLOv9-T / S / M / C / E (WongKinYiu/yolov9 v0.1, the converted GELAN graphs with a DDetect head, exported with one "
                 "output; files with the auxiliary branch and ultralytics' YOLOv9 are not supported)")
_V9_STEM = {16: ("t",), 32: ("s", "m"), 64: ("c",)}
_V9_DOWN3 = {128: "s", 240: "m"}            # layer 3 (AConv) width tells S from M


def _is_yolov9(model: OnnxModel) -> bool:
    return any(n.op_type == "AveragePool" and list(n.attrs.get("kernel_shape", [])) == [2, 2] and list(n.attrs.get("strides", [1, 1])) == [1, 1]
               for n in model.nodes)


def _recognise_yolov9(model: OnnxModel, w: OnnxWeights, in_h: int, in_w: int) -> ModelSpec:
    """YOLOv9-T / S / M / C: the stem width gives the scale (32: S or M by layer 3's width), the head must have DDetect's grouped box
    convolutions, and the convolution count must be the scale's (fused, or with RepConvN's two branches apart).  YOLOv9-E: two
    [64, 3, 3, 3] convolutions read the image (its two backbones, model.1 and model.15); the same head and count checks follow."""
    if len(model.outputs) != 1:
        raise Exception(f"YOLOv9 file with {len(model.outputs)} outputs (an auxiliary-branch training file?); supported: {_V9_SUPPORTED}")
    first = w.convs[0][1]
    image = model.inputs[0][0] if model.inputs else None
    image_convs = [model.initializers.get(n.inputs[1]) for n in model.nodes if n.op_type == "Conv" and n.inputs and n.inputs[0] == image]
    if len(image_convs) == 2 and all(c is not None and tuple(c.shape) == (64, 3, 3, 3) for c in image_convs):
        cands = ("e",)
    else:
        cands = _V9_STEM.get(int(first.shape[0]), ()) if tuple(first.shape[1:]) == (3, 3, 3) else ()
    if not cands:
        raise Exception(f"YOLOv9 stem {tuple(first.shape)}: 16 (T), 32 (S / M) or 64 (C) channels, or two 64-channel image convolutions (E); "
                        f"supported: {_V9_SUPPORTED}")
    grouped = [n for n in model.nodes if n.op_type == "Conv" and int(n.attrs.get("group", 1)) == 4]
    if len(grouped) != 6:
        raise Exception(f"YOLOv9 file with {len(grouped)} group-4 convolutions: a head without DDetect's grouped box convolutions "
                        f"(6); supported: {_V9_SUPPORTED}")
    if (in_h and in_h % 32) or (in_w and in_w % 32):
        raise Exception(f"YOLOv9 file with a {in_h}x{in_w} input: a multiple of 32; supported: {_V9_SUPPORTED}")
    scale = cands[0]
    if len(cands) > 1:
        named = model.initializers.get("model.3.cv1.conv.weight")
        if named is not None:
            width = int(named.shape[0])
        else:                                                    # the conv reading the first 2x2 average pool (AConv's cv1)
            pool = next(n for n in model.nodes if n.op_type == "AveragePool")
            conv = next((n for n in model.nodes if n.op_type == "Conv" and n.inputs[0] == pool.outputs[0]), None)
            width = int(model.initializers[conv.inputs[1]].shape[0]) if conv is not None and conv.inputs[1] in model.initializers else 0
        if width not in _V9_DOWN3:
            raise Exception(f"YOLOv9 file with a 32-channel stem and a {width}-channel layer 3 (128: S, 240: M); supported: {_V9_SUPPORTED}")
        scale = _V9_DOWN3[width]
    n = sum(1 for _, cw, _ in w.convs if tuple(cw.shape) != (1, 16, 1, 1))       # upstream's fixed DFL conv is not counted
    fused = plan.yolov9_conv_count(scale)
    if n not in (fused, fused + plan.yolov9_repconvn_count(scale)):
        raise Exception(f"YOLOv9 file with {n} convolutions, YOLOv9-{scale.upper()} has {fused} ({fused + plan.yolov9_repconvn_count(scale)} with "
                        f"RepConvN's branches apart); supported: {_V9_SUPPORTED}")
    nc = None
    head = "model.42" if scale == "e" else "model.22"
    for name, cw, _ in w.convs:
        if re.fullmatch(re.escape(head) + r"\.cv3\.\d+\.2\.weight", name):      # DDetect.cv3[i][2]: Conv2d(c3, nc, 1)
            nc = int(cw.shape[0])
    if nc is None:                                               # names lost: the last 1x1 conv before the (optional) DFL conv
        nc = int([cw.shape[0] for _, cw, _ in w.convs if cw.shape[2:] == (1, 1) and cw.shape[0] != 1][-1])
    return ModelSpec("yolov9", scale, nc, in_h or 640, in_w or 640)


_V10_SUPPORTED = ("YOLOv10-N / S / M / B / L / X (ultralytics 8.2.41) with the one-to-one head, one output ([1, 4 + nc, A] or the "
                  "top-k [1, 300, 6] tail), input a multiple of 32")
_V10_STEM = {16: ("n",), 32: ("s",), 48: ("m",), 64: ("b", "l"), 80: ("x",)}


def _is_yolov10(model: OnnxModel) -> bool:
    """Depthwise convolutions (group = Cin = Cout > 1: SCDown, CIB, PSA's pe, the v10 class branch) together with a Softmax outside
    the DFL decode (PSA's attention).  YOLOv8 files have the DFL softmax but no depthwise conv; YOLOv9's grouped convs have 4 groups."""
    return _depthwise(model) and any(n.op_type == "Softmax" for n in model.nodes)


def _recognise_yolov10(model: OnnxModel, w: OnnxWeights, in_h: int, in_w: int) -> ModelSpec:
    """YOLOv10-N / S / M / B / L / X: the stem width gives the scale (64: B or L by `model.2.m.2.*`, else by the convolution count).
    Without module names the convolution count must be the scale's (fused, or with RepVGGDW's two branches apart): a file that also
    carries the one-to-many head cannot be matched by order and is refused.  The class count comes from `model.23.one2one_cv3.*.2`."""
    if len(model.outputs) != 1:
        raise Exception(f"YOLOv10 file with {len(model.outputs)} outputs; supported: {_V10_SUPPORTED}")
    if (in_h and in_h % 32) or (in_w and in_w % 32):
        raise Exception(f"YOLOv10 file with a {in_h}x{in_w} input: a multiple of 32; supported: {_V10_SUPPORTED}")
    first = w.convs[0][1]
    cands = _V10_STEM.get(int(first.shape[0]), ()) if tuple(first.shape[1:]) == (3, 3, 3) else ()
    if not cands:
        raise Exception(f"YOLOv10 stem {tuple(first.shape)}: 16 (N), 32 (S), 48 (M), 64 (B / L) or 80 (X) channels; supported: {_V10_SUPPORTED}")
    named = any(re.fullmatch(r"model\.23\.one2one_cv3\.\d+\.2\.weight", k) for k in model.initializers) and \
        any(k.startswith("model.2.") for k in model.initializers)
    n = sum(1 for _, cw, _ in w.convs if tuple(cw.shape) != (1, 16, 1, 1))        # upstream's fixed DFL conv is not counted
    counts = {sc: (plan.yolov10_conv_count(sc), plan.yolov10_conv_count(sc) + plan.yolov10_repvggdw_count(sc)) for sc in cands}
    if named:
        scale = ("l" if any(k.startswith("model.2.m.2.") for k in model.initializers) else "b") if len(cands) > 1 else cands[0]
    else:
        fits = [sc for sc in cands if n in counts[sc]]
        if not fits:
            o2m = [sc for sc in cands if n - 24 in counts[sc]]
            if o2m:
                raise Exception(f"YOLOv10-{o2m[0].upper()} file without module names that also carries the one-to-many head ({n} "
                                f"convolutions): its convolutions cannot be matched in order; export the model after upstream's fuse() "
                                f"(which drops that head) or keep the module names; supported: {_V10_SUPPORTED}")
            raise Exception(f"YOLOv10 file with {n} convolutions, " + ", ".join(f"YOLOv10-{sc.upper()} has {c[0]} ({c[1]} with RepVGGDW's "
                            f"branches apart)" for sc, c in counts.items()) + f"; supported: {_V10_SUPPORTED}")
        scale = fits[0]
    nc = None
    for name, cw, _ in w.convs:
        if re.fullmatch(r"model\.23\.one2one_cv3\.\d+\.2\.weight", name):      # v10Detect.one2one_cv3[i][2]: Conv2d(c3, nc, 1)
            nc = int(cw.shape[0])
    if nc is None:                                               # names lost: the last 1x1 conv before the (optional) DFL conv
        nc = int([cw.shape[0] for _, cw, _ in w.convs if cw.shape[2:] == (1, 1) and cw.shape[0] != 1][-1])
    return ModelSpec("yolov10", scale, nc, in_h or 640, in_w or 640)


def build_plan(model: OnnxModel, spec: Optional[ModelSpec] = None) -> "plan.PlanBuilder":
    spec = spec or recognise(model)
    w = OnnxWeights(model)
    if spec.kind == "yolov8":
        return plan.build_yolov8(w, spec.scale, nc=spec.nc, in_h=spec.in_h, in_w=spec.in_w)
    if spec.kind == "yolov5":
        return plan.build_yolov5(w, spec.scale, nc=spec.nc, in_h=spec.in_h, in_w=spec.in_w)
    if spec.kind == "yolov7":
        return plan.build_yolov7(w, spec.scale, nc=spec.nc, in_h=spec.in_h, in_w=spec.in_w, act=spec.act, anchors=spec.anchors)
    if spec.kind == "yolov9":
        return plan.build_yolov9(w, spec.scale, nc=spec.nc, in_h=spec.in_h, in_w=spec.in_w)
    if spec.kind == "yolov10":
        return plan.build_yolov10(w, spec.scale, nc=spec.nc, in_h=spec.in_h, in_w=spec.in_w)
    if spec.kind == "yolov6":
        body, neck, head = spec.acts or (None, "relu", "silu")
        return plan.build_yolov6(w, spec.scale, nc=spec.nc, in_h=spec.in_h, in_w=spec.in_w, act_body=body, act_neck=neck, act_head=head,
                                 reg_max=spec.reg_max)
    if spec.kind == "yolov6-lite":
        return plan.build_yolov6_lite(w, spec.scale, nc=spec.nc, in_h=spec.in_h, in_w=spec.in_w)
    if spec.kind == "ufldv2":
        # the dataset follows from the input binding (ModelConfig: CULane 320x1600, TuSimple 320x800); the engine rejects any other
        cfg = dict(plan.UFLD_TUSIMPLE if (spec.in_h, spec.in_w) == (320, 800) else plan.UFLD_CULANE)
        cfg["in_h"], cfg["in_w"] = spec.in_h, spec.in_w
        return plan.build_ufldv2(w, spec.scale, cfg)
    raise Exception(f"unsupported model kind {spec.kind}")


def plan_from_onnx(onnx_path: str, out_path: Optional[str] = None) -> str:
    """Convert once and cache: returns the path of the `.b200w` plan for `onnx_path` (the counterpart of the reference's
    convertOnnxToTensorRT.py, which writes a `.trt` next to the `.onnx`)."""
    if not os.path.isfile(onnx_path):
        raise Exception("The model path [%s] can't not found!" % onnx_path)
    st = os.stat(onnx_path)
    if out_path is None:
        tag = hashlib.sha1(f"{os.path.abspath(onnx_path)}:{st.st_size}:{st.st_mtime_ns}:{plan.PLAN_VERSION}".encode()).hexdigest()[:16]
        cache = plan.cache_dir()
        out_path = os.path.join(cache, f"{os.path.splitext(os.path.basename(onnx_path))[0]}-{tag}.b200w")
    if os.path.isfile(out_path) and os.path.getmtime(out_path) >= st.st_mtime:
        return out_path
    pb = build_plan(read_onnx(onnx_path))
    tmp = out_path + f".tmp{os.getpid()}"
    pb.write(tmp)
    os.replace(tmp, out_path)
    return out_path
