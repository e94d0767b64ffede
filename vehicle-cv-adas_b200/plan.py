"""plan.py -- the packer: turns a network state_dict into a `.b200w` plan for libadas_b200.

Replaces the reference's offline model tooling for this runtime (convertOnnxToTensorRT.py,
onnxQuantization.py, TrafficLaneDetector/convertPytorchToONNX.py:50-96): instead of exporting to
ONNX and building a TensorRT engine, the weights are BN-folded, cast to fp16, laid out K-major
([Cout, kh, kw, Cin]) for the sm_90a implicit-GEMM kernel, and written next to the op list the
C++ runtime replays (csrc/plan.h documents the binary layout).

Network graphs
  * YOLOv8 (ultralytics 8.1 `yolov8.yaml`, README.md:56 of the reference), YOLOv5 v6.2
    (`yolov5{n,s,...}.yaml`, README.md:53) and YOLOv7 / YOLOv7-tiny (`cfg/training/yolov7{,-tiny}.yaml`):
    not shipped by the reference; restated from the public architecture (SURVEY.md Appendix A),
    state_dict keys follow the upstream naming so real checkpoints can be packed.
  * UFLDv2: TrafficLaneDetector/ufldDetector/exportLib/ultrafastLaneV2/model_culane.py:7-63 and
    backbone.py:14-58 (torchvision ResNet18/34 trunk -> 1x1 pool conv -> LayerNorm -> MLP).

Activation layout: "padded NHWC" -- a [B*(H+2)*(W+2), C] fp16 matrix with a zero halo, so every
3x3 stride-1 conv is 9 row-shifted GEMMs over one 2-D TMA-addressable matrix; concats are channel
slices of a shared buffer (producers write their slice), so Concat/Split cost nothing.
"""
from __future__ import annotations

import math
import os
import re
import struct
import zlib
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

MODEL_YOLOV8, MODEL_YOLOV5, MODEL_UFLDV2, MODEL_UFLDV1 = 0, 1, 2, 4      # 3 = ADAS_MODEL_YOLOV5_LITE (post-processing kind only)
MODEL_YOLOV6 = 5                                                         # anchor-free head, [B, 8400, 5 + nc] output; meta[2] = reg_max
ACT_NONE, ACT_SILU, ACT_RELU, ACT_LEAKY = 0, 1, 2, 3          # ACT_LEAKY: LeakyReLU(0.1)
ACT_HSWISH = 5                                                # Hardswish x * clamp(x + 3, 0, 6) / 6; code 4 is unused
PLAN_VERSION = 1

# ---------------------------------------------------------------------------------------------
# record layout (csrc/plan.h)
# ---------------------------------------------------------------------------------------------
HDR_FMT, BUF_FMT, OP_FMT, TEN_FMT, OUT_FMT = "<8sII3I4I16IQQ", "<6I", "<I23i4f", "<QQII", "<4I"
HDR_SIZE, BUF_SIZE, OP_SIZE, TEN_SIZE, OUT_SIZE = (struct.calcsize(f) for f in (HDR_FMT, BUF_FMT, OP_FMT, TEN_FMT, OUT_FMT))
OP_NP, OP_NF = 23, 4                                          # PlanOp: type, int32 p[23], float f[4]

OP_GEMM, OP_IM2COL, OP_MAXPOOL, OP_UPSAMPLE2X, OP_LAYERNORM, OP_STEMPACK, OP_STEMCONV = 1, 2, 3, 4, 5, 6, 7
OP_AVGPOOL2, OP_DWCONV, OP_ATTN, OP_CBFUSE, OP_SE, OP_SHUFFLE2 = 8, 9, 10, 11, 12, 13
OP_NAMES = {OP_GEMM: "gemm", OP_IM2COL: "im2col", OP_MAXPOOL: "maxpool", OP_UPSAMPLE2X: "upsample", OP_LAYERNORM: "layernorm",
            OP_STEMPACK: "stempack", OP_STEMCONV: "stemconv", OP_AVGPOOL2: "avgpool2", OP_DWCONV: "dwconv", OP_ATTN: "attention",
            OP_CBFUSE: "cbfuse", OP_SE: "se", OP_SHUFFLE2: "shuffle2"}
# The fields of PlanOp.p per op type, in slot order: the members of plan.h's op structs (OP_GEMM: GemmOp, ...).  What each field
# means is documented there.
OP_FIELDS = {
    OP_GEMM: ("a_buf", "a_coff", "Kc", "ntaps", "w_tensor", "bias_tensor", "N", "act", "res_buf", "res_coff", "res_pre_act", "out_buf",
              "out_coff", "masked", "transposed", "BN", "s2", "MT", "no_slab", "up2"),
    OP_IM2COL: ("in_buf", "in_coff", "Cin", "kh", "kw", "stride", "pad", "out_buf"),
    OP_MAXPOOL: ("in_buf", "in_coff", "C", "k", "stride", "pad", "out_buf", "out_coff"),
    OP_UPSAMPLE2X: ("in_buf", "in_coff", "C", "out_buf", "out_coff"),
    OP_LAYERNORM: ("in_buf", "d_len", "gamma_tensor", "beta_tensor", "out_buf", "d_norm"),
    OP_STEMPACK: ("in_buf", "out_buf"),
    OP_STEMCONV: ("in_buf", "w_tensor", "bias_tensor", "Cout", "k", "pad", "act", "out_buf", "out_coff", "stride"),
    OP_AVGPOOL2: ("in_buf", "in_coff", "C", "out_buf", "out_coff", "fill"),
    OP_DWCONV: ("in_buf", "in_coff", "C", "k", "stride", "act", "w_tensor", "bias_tensor", "out_buf", "out_coff", "res_buf", "res_coff"),
    OP_ATTN: ("in_buf", "in_coff", "nh", "kdp", "hd", "out_buf", "out_coff"),
    OP_CBFUSE: ("out_buf", "out_coff", "C", "base_buf", "base_coff", "n_src"),     # then CBFUSE_MAX_SRC x CBFUSE_SRC_FIELDS
    OP_SE: ("in_buf", "in_coff", "C", "hid", "w1", "b1", "w2", "b2", "out_buf", "out_coff"),
    OP_SHUFFLE2: ("a_buf", "a_coff", "b_buf", "b_coff", "n", "out_buf", "out_coff"),
}
CBFUSE_SRC_FIELDS, CBFUSE_MAX_SRC = ("buf", "coff", "shift"), 5
OP_FLOATS = {OP_GEMM: ("res_scale",), OP_LAYERNORM: ("eps",), OP_ATTN: ("scale",)}      # the named entries of PlanOp.f
_FIELD_SLOT = {t: {n: i for i, n in enumerate(names)} for t, names in OP_FIELDS.items()}


class OpParams(list):
    """PlanOp.p of one op: the 23 int32 slots as a list (so it packs, indexes and compares as one), whose fields of OP_FIELDS[typ]
    also read and write by name (`p.out_buf`, `p.BN = 64`).  A name the op type does not have is an error."""
    __slots__ = ("typ",)

    def __init__(self, typ: int, values=()):
        values = list(values)
        assert len(values) <= OP_NP, (typ, values)
        super().__init__(values + [0] * (OP_NP - len(values)))
        object.__setattr__(self, "typ", typ)

    def __getattr__(self, name: str) -> int:
        return self[field_slot(self.typ, name)]

    def __setattr__(self, name: str, value: int) -> None:
        self[field_slot(self.typ, name)] = value

    def copy(self) -> "OpParams":
        return OpParams(self.typ, self)

    def __reduce__(self):                                     # copy.copy / deepcopy / pickle rebuild through __init__
        return OpParams, (self.typ, list(self))


def field_slot(typ: int, name: str) -> int:
    """Slot of field `name` of op type `typ` in PlanOp.p."""
    try:
        return _FIELD_SLOT[typ][name]
    except KeyError:
        raise AttributeError(f"{OP_NAMES.get(typ, typ)} op has no field {name!r}") from None


def cbfuse_src_slot(s: int) -> int:
    """Slot of the first field of source s of an OP_CBFUSE op in PlanOp.p."""
    return len(OP_FIELDS[OP_CBFUSE]) + len(CBFUSE_SRC_FIELDS) * s


def cbfuse_sources(p: OpParams) -> List[Tuple[int, int, int]]:
    """(buffer, channel offset, shift) of each source of an OP_CBFUSE op, in summation order."""
    return [tuple(p[cbfuse_src_slot(s):cbfuse_src_slot(s + 1)]) for s in range(p.n_src)]


def cache_dir() -> str:
    """Directory for converted / synthetic plan files: $ADAS_B200_PLAN_CACHE, else ~/.cache/adas_b200 -- created 0700 and refused if it
    belongs to another user or is writable by others (a plan is trusted input to the engine; the reference writes its .trt next to
    the .onnx the user named, convertOnnxToTensorRT.py)."""
    d = os.environ.get("ADAS_B200_PLAN_CACHE") or os.path.join(os.path.expanduser("~"), ".cache", "adas_b200")
    os.makedirs(d, mode=0o700, exist_ok=True)
    st = os.stat(d)
    if hasattr(os, "getuid") and (st.st_uid != os.getuid() or (st.st_mode & 0o022)):
        raise Exception(f"plan cache {d} is not a private directory of this user (owner {st.st_uid}, mode {oct(st.st_mode & 0o777)})")
    return d



# ---------------------------------------------------------------------------------------------
# weights: real state_dict or seeded synthetic
# ---------------------------------------------------------------------------------------------
class Weights:
    """Source of raw (un-folded) parameters by upstream key name.

    `sd` may be a real state_dict (numpy arrays or torch tensors).  With `sd=None` parameters are
    generated on first use from a seed (He-normal convs, mildly randomised BatchNorm statistics)
    and recorded in `self.state_dict`, which the CPU oracle loads to share the exact weights.
    """

    def __init__(self, sd: Optional[Dict[str, object]] = None, seed: int = 0, profile: Optional[dict] = None):
        self.real = sd is not None
        self.state_dict: Dict[str, np.ndarray] = {}
        if sd is not None:
            for k, v in sd.items():
                self.state_dict[k] = np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v)
        self.seed = seed
        self.profile = profile or {}

    def _rng(self, name: str) -> np.random.Generator:
        return np.random.default_rng([self.seed, zlib.crc32(name.encode())])

    def get(self, name: str, shape: Tuple[int, ...], kind: str) -> np.ndarray:
        if name in self.state_dict:
            a = self.state_dict[name]
            assert tuple(a.shape) == tuple(shape), f"{name}: expected {shape}, state_dict has {a.shape}"
            return a.astype(np.float32)
        assert not self.real, f"state_dict is missing {name}"
        r = self._rng(name)
        for pat, val in self.profile.get("fill", ()):       # e.g. detection-head biases that set the score operating point
            if re.fullmatch(pat, name):
                a = np.full(shape, val[1] if isinstance(val, tuple) else val, np.float32)
                if isinstance(val, tuple):                  # (xywh, objectness + classes) of each of the 3 anchors of a YOLOv5-layout head
                    a.reshape(3, -1)[:, :4] = val[0]
                self.state_dict[name] = a
                return a
        if kind == "conv":
            fan_in = int(np.prod(shape[1:]))
            gain = self.profile.get("conv_gain", 1.0)
            for pat, g in self.profile.get("gains", ()):
                if re.fullmatch(pat, name):
                    gain = g
            a = r.standard_normal(shape, dtype=np.float32) * np.float32(gain * math.sqrt(2.0 / fan_in))
        elif kind == "linear":
            a = r.standard_normal(shape, dtype=np.float32) * np.float32(math.sqrt(1.0 / shape[1]))
        elif kind == "bn_gamma":
            lo, hi = self.profile.get("gamma", (0.9, 1.1))
            a = r.uniform(lo, hi, shape).astype(np.float32)
        elif kind == "bn_gamma_res":      # last BN of a residual branch: damped so depth does not blow up
            a = r.uniform(0.25, 0.4, shape).astype(np.float32)
        elif kind == "bn_beta":
            a = (r.standard_normal(shape) * 0.05).astype(np.float32)
        elif kind == "bn_mean":
            a = (r.standard_normal(shape) * 0.05).astype(np.float32)
        elif kind == "bn_var":
            a = r.uniform(0.9, 1.1, shape).astype(np.float32)
        elif kind == "bias":
            a = (r.standard_normal(shape) * 0.02).astype(np.float32)
        elif kind == "ln_gamma":
            a = r.uniform(0.9, 1.1, shape).astype(np.float32)
        elif kind == "ln_beta":
            a = (r.standard_normal(shape) * 0.02).astype(np.float32)
        elif kind == "implicit_a":          # YOLOv7 ImplicitA: nn.init.normal_(mean=0, std=0.02)
            a = (r.standard_normal(shape) * 0.02).astype(np.float32)
        elif kind == "implicit_m":          # YOLOv7 ImplicitM: nn.init.normal_(mean=1, std=0.02)
            a = (1.0 + r.standard_normal(shape) * 0.02).astype(np.float32)
        elif kind == "alpha":               # YOLOv6 BottleRep shortcut scale (initialised to 1, learned)
            a = r.uniform(0.7, 1.3, shape).astype(np.float32)
        else:
            raise ValueError(kind)
        self.state_dict[name] = a
        return a

    def override(self, name: str, value: np.ndarray) -> None:
        self.state_dict[name] = np.asarray(value, dtype=np.float32)

    # folded conv+BN: returns (w [Cout,Cin,kh,kw] fp32, b [Cout] fp32)
    def conv_bn(self, prefix: str, cout: int, cin: int, k: int, eps: float, conv_key="conv", bn_key="bn", res_branch=False):
        wf, bf = self._conv_bn64(prefix, cout, cin, k, eps, conv_key, bn_key, res_branch)
        return wf.astype(np.float32), bf.astype(np.float32)

    def _conv_bn64(self, prefix: str, cout: int, cin: int, k: int, eps: float, conv_key="conv", bn_key="bn", res_branch=False):
        w = self.get(f"{prefix}.{conv_key}.weight" if conv_key else f"{prefix}.weight", (cout, cin, k, k), "conv")
        bn = f"{prefix}.{bn_key}"
        g = self.get(f"{bn}.weight", (cout,), "bn_gamma_res" if res_branch else "bn_gamma")
        b = self.get(f"{bn}.bias", (cout,), "bn_beta")
        m = self.get(f"{bn}.running_mean", (cout,), "bn_mean")
        v = self.get(f"{bn}.running_var", (cout,), "bn_var")
        if not self.real and f"{bn}.num_batches_tracked" not in self.state_dict:
            self.state_dict[f"{bn}.num_batches_tracked"] = np.zeros((), dtype=np.int64)
        scale = (g.astype(np.float64) / np.sqrt(v.astype(np.float64) + eps))
        return w.astype(np.float64) * scale[:, None, None, None], b.astype(np.float64) - m.astype(np.float64) * scale

    def repconv(self, prefix: str, cout: int, cin: int, eps: float, keys: Tuple[str, str] = ("0", "1"), identity: bool = False):
        """RepVGG-style block (YOLOv7 RepConv, YOLOv6 RepVGGBlock) as one folded 3x3 conv, summed in fp64: BN-folded rbr_dense + BN-folded
        rbr_1x1 on the centre tap (+ with `identity`, the rbr_identity BatchNorm as a scaled identity on the centre tap, cin == cout at
        stride 1).  `keys` names the conv / BN inside each branch: ("0", "1") for YOLOv7's Sequential, ("conv", "bn") for YOLOv6.  A
        checkpoint that was re-parameterised upstream carries `rbr_reparam` instead.  With `identity`, all three synthetic BNs are damped
        like the last BN of a residual branch (a chain of undamped identity blocks grows its activations geometrically)."""
        ck, bk = keys
        if f"{prefix}.rbr_reparam.weight" in self.state_dict or (self.real and f"{prefix}.rbr_dense.{ck}.weight" not in self.state_dict):
            return self.conv_bias(f"{prefix}.rbr_reparam", cout, cin, 3)
        if not identity:
            assert f"{prefix}.rbr_identity.running_var" not in self.state_dict, f"{prefix}: RepConv with an identity branch"
        wd, bd = self._conv_bn64(f"{prefix}.rbr_dense", cout, cin, 3, eps, conv_key=ck, bn_key=bk, res_branch=identity)
        w1, b1 = self._conv_bn64(f"{prefix}.rbr_1x1", cout, cin, 1, eps, conv_key=ck, bn_key=bk, res_branch=identity)
        wd[:, :, 1, 1] += w1[:, :, 0, 0]
        bd += b1
        if identity:
            assert cin == cout, f"{prefix}: identity branch needs cin == cout"
            bn = f"{prefix}.rbr_identity"
            g = self.get(f"{bn}.weight", (cout,), "bn_gamma_res").astype(np.float64)
            be = self.get(f"{bn}.bias", (cout,), "bn_beta").astype(np.float64)
            m = self.get(f"{bn}.running_mean", (cout,), "bn_mean").astype(np.float64)
            v = self.get(f"{bn}.running_var", (cout,), "bn_var").astype(np.float64)
            if not self.real and f"{bn}.num_batches_tracked" not in self.state_dict:
                self.state_dict[f"{bn}.num_batches_tracked"] = np.zeros((), dtype=np.int64)
            s = g / np.sqrt(v + eps)
            wd[np.arange(cout), np.arange(cout), 1, 1] += s
            bd += be - m * s
        return wd.astype(np.float32), bd.astype(np.float32)

    def repconvn(self, prefix: str, cout: int, cin: int, eps: float):
        """YOLOv9 RepConvN (3x3 `conv1` + 1x1 `conv2`, each Conv2d + BatchNorm, no identity branch) as one folded 3x3 conv, summed in
        fp64 with the 1x1 on the centre tap.  A file fused upstream carries `conv.weight` + `conv.bias` instead."""
        if f"{prefix}.conv.weight" in self.state_dict:
            return self.conv_bias(f"{prefix}.conv", cout, cin, 3)
        w3, b3 = self._conv_bn64(f"{prefix}.conv1", cout, cin, 3, eps)
        w1, b1 = self._conv_bn64(f"{prefix}.conv2", cout, cin, 1, eps)
        w3[:, :, 1, 1] += w1[:, :, 0, 0]
        return w3.astype(np.float32), (b3 + b1).astype(np.float32)

    def repvggdw(self, prefix: str, c: int, eps: float):
        """YOLOv10 RepVGGDW: dw7x7+BN (`conv`) + dw3x3+BN (`conv1`), folded in fp64 into one depthwise 7x7 (the 3x3 on the centre taps).
        A file fused upstream carries `conv.weight` + `conv.bias` instead."""
        if f"{prefix}.conv.weight" in self.state_dict:
            return self.conv_bias(f"{prefix}.conv", c, 1, 7)
        w7, b7 = self._conv_bn64(f"{prefix}.conv", c, 1, 7, eps)
        w3, b3 = self._conv_bn64(f"{prefix}.conv1", c, 1, 3, eps)
        w7[:, :, 2:5, 2:5] += w3
        return w7.astype(np.float32), (b7 + b3).astype(np.float32)

    def implicit_head(self, prefix: str, li: int, no: int, cin: int):
        """YOLOv7 IDetect level li: im * (m(x + ia)) folded into the 1x1 conv, w' = im * w, b' = im * (b + w @ ia) in fp64.  Files
        fused upstream (IDetect.fuse) carry the folded m.li conv and no implicit tensors."""
        w, b = self.conv_bias(f"{prefix}.m.{li}", no, cin, 1)
        ka, km = f"{prefix}.ia.{li}.implicit", f"{prefix}.im.{li}.implicit"
        if self.real and ka not in self.state_dict:
            return w, b
        ia = self.get(ka, (1, cin, 1, 1), "implicit_a").astype(np.float64).reshape(cin)
        im = self.get(km, (1, no, 1, 1), "implicit_m").astype(np.float64).reshape(no)
        w64 = w.astype(np.float64)
        return (w64 * im[:, None, None, None]).astype(np.float32), (im * (b.astype(np.float64) + w64[:, :, 0, 0] @ ia)).astype(np.float32)

    def anchor_grid(self, prefix: str, levels: int = 3) -> Optional[np.ndarray]:
        """Anchors in input pixels from an upstream Detect / IDetect `anchor_grid` buffer ([levels, 1, 3, 1, 1, 2]), when the source has one."""
        a = self.state_dict.get(f"{prefix}.anchor_grid")
        return None if a is None or a.size != 6 * levels else np.asarray(a, np.float32).reshape(6 * levels)

    def conv_bias(self, prefix: str, cout: int, cin: int, k: int):
        w = self.get(f"{prefix}.weight", (cout, cin, k, k), "conv")
        b = self.get(f"{prefix}.bias", (cout,), "bias")
        return w, b


# Synthetic-weight operating points (calibrated against the fp32 oracle on synthetic frames, tools/synth_operating_point.py).
# Random He-init heads give logits ~ N(0, 0.07^2), i.e. every score ~0.5; the profiles widen the final 1x1 head convs and shift
# their biases so that O(100) of the 8400 / 25200 anchors clear box_score = 0.4 and the DFL boxes vary in size.
# The head gain sets BOTH the spread of the per-anchor scores and the size of the fp16-vs-fp32 score error (both scale with it):
# a random network has a fixed noise-to-signal ratio (~1 % of the per-anchor logit spread after ~100 fp16 layers), so the gains
# below are the largest that keep the probability error under the 1e-3 contract (v8l: 16 -> 8e-4 on the device, 5.5e-4 in the CPU fp16 emulation; v5n: 20 -> 8.6e-4; at gain 45 the v8l device error is 1.5e-3)
# and ~2-4 % of the candidates then sit within 1e-3 of the threshold.  (Tried and dropped: BatchNorm statistics measured on
# calibration frames -- activations standardised like a trained net's -- spread the scores 14x but amplified the fp16 error 10x
# further: max probability error 0.15, 73 px on DFL boxes.)
SYNTH_PROFILES = {
    "yolov8": {"gains": [(r"model\.22\.cv3\.\d\.2\.weight", 16.0), (r"model\.22\.cv2\.\d\.2\.weight", 25.0)],
               "fill": [(r"model\.22\.cv3\.\d\.2\.bias", -3.5)]},
    "yolov5": {"gains": [(r"model\.24\.m\.\d\.weight", 20.0)],
               "fill": [(r"model\.24\.m\.\d\.bias", -2.7)]},
    # lane existence: random heads give P(valid) = 0.5 per anchor, i.e. no lane passes the "more than half / a quarter of the anchors
    # valid" test and nothing downstream of the decode is exercised; +1.0 on the "valid" logits makes ~88 % of the anchors valid
    "ufldv2": {"ufld_exist_bias": 1.0},
    # YOLOv9 T/S/M/C: YOLOv8's head gains (CPU fp16 emulation: probability error 2-4e-4, box error 0.1 px on 8 frames); the class bias
    # of each scale puts ~100 of the 8400 anchors per frame above box_score = 0.4 (fp32 oracle, synthetic frames 0-3: at bias -3.5 the
    # 100th-highest max-class logit sits 0.53 (T), -0.31 (S), 0.04 (M), 0.05 (C) from logit(0.4); per-anchor spread 0.16-0.47).
    # YOLOv9-E (head model.42): at YOLOv8's gains the CPU fp16 emulation (plan_interp.interpret, every op rounded to fp16) was 5.9e-3
    # off in probability on frame 0 (4: 1.3e-3) and 0.42 px on boxes: its 261-conv graph and the CBFuse sums leave large per-frame
    # offsets on the class logits.  Class gain 2 and box gain 12 gave 7.6e-4 / 3.3e-4 and 0.22 / 0.13 px on frames 0 / 1, but 1.0e-3 on
    # the device at 384x640 (H100), so the class gain is 1.5: device 7.1e-4 / 0.26 px at 640x640 and 6.9e-4 / 0.26 px at 384x640 on
    # frames 0 / 1; `tools/synth_operating_point.py yolov9 e 1.5,-1.25` gives 5.6e-4 / 2.2e-4 there and up to 1.02e-3 on frame 2.  Class
    # bias -1.25 puts 183, 9, 274, 53 anchors of synthetic frames 0-3 above box_score = 0.4 (fp32 oracle, 640x640); the per-frame spread
    # is wide, and frames 4, 6, 7 have none.
    "yolov9": {"gains": [(r"model\.22\.cv3\.\d\.2\.weight", 16.0), (r"model\.22\.cv2\.\d\.2\.weight", 25.0),
                         (r"model\.42\.cv3\.\d\.2\.weight", 1.5), (r"model\.42\.cv2\.\d\.2\.weight", 12.0)],
               "fill": [(r"model\.22\.cv3\.\d\.2\.bias", -3.5)],
               "variants": {**{sc: {"fill": [(r"model\.22\.cv3\.\d\.2\.bias", -3.5 - d)]}
                               for sc, d in (("t", 0.53), ("s", -0.31), ("m", 0.04), ("c", 0.05))},
                            "e": {"fill": [(r"model\.42\.cv3\.\d\.2\.bias", -1.25)]}}},
    # YOLOv10 N/S/M/B/L/X: YOLOv8's head gains on the one-to-one head (CPU fp16 emulation, q / k / v and the attention output rounded
    # too: probability error 2.5-3.7e-4, box error 0.13-0.23 px on 4 frames).  The class bias of each scale puts ~100 of the 8400
    # anchors per frame above box_score = 0.4 (fp32 oracle, synthetic frames 0-3: at bias -3.5 the 100th-highest max-class logit sits
    # -0.80 (N), 0.05 (S), 0.11 (M), 0.10 (B), 0.49 (L), 0.53 (X) from logit(0.4)).  The seeded PSA attention is not peaky (mean
    # largest softmax weight 0.003 over 400 tokens), so its qkv weights are not damped.
    "yolov10": {"gains": [(r"model\.23\.one2one_cv3\.\d\.2\.weight", 16.0), (r"model\.23\.one2one_cv2\.\d\.2\.weight", 25.0)],
                "fill": [(r"model\.23\.one2one_cv3\.\d\.2\.bias", -3.5)],
                "variants": {sc: {"fill": [(r"model\.23\.one2one_cv3\.\d\.2\.bias", -3.5 - d)]}
                             for sc, d in (("n", -0.804), ("s", 0.054), ("m", 0.112), ("b", 0.099), ("l", 0.485), ("x", 0.534))}},
    # YOLOv7 base (model.105, SiLU) and tiny (model.77, LeakyReLU).  The tiny net's activations are not damped layer by layer as with
    # SiLU: its fp16 noise at the head is ~50x larger, so its head gain is 0.3, its objectness / class biases (-0.2) set the operating
    # point and its box biases sit at -3, where the xywh sigmoids are flat (box noise 0.4 px -> 0.01 px).  CPU fp16 emulation on
    # 4 frames: base 6.1e-4 / 0.10 px / ~280 candidates per frame, tiny 5.9e-4 / 0.01 px / ~100 candidates per frame.
    # The P6 heads W6 (model.118), E6 (140) and D6 (162) take base's head gain.  W6's bias (-1.75) puts ~230 of the 102000 anchors
    # of a letterboxed 1280x720 frame above box_score = 0.4 (fp32 oracle, frames 4 and 5; at -2.0 there are ~120 but half sit within 1e-3 of it).  E6E (261)
    # runs every ELAN twice and sums the pair: at gain 16 its device error was 1.4e-3 / 0.99 px at 640, so its head gain is 6 and its box
    # biases sit at -4, where the xywh sigmoids are flat.
    "yolov7": {"gains": [(r"model\.105\.m\.\d\.weight", 16.0), (r"model\.77\.m\.\d\.weight", 0.3),
                         (r"model\.(118|140|162)\.m\.\d\.weight", 16.0), (r"model\.261\.m\.\d\.weight", 6.0)],
               "fill": [(r"model\.105\.m\.\d\.bias", -3.0), (r"model\.77\.m\.\d\.bias", (-3.0, -0.2)),
                        (r"model\.118\.m\.\d\.bias", -1.75), (r"model\.(140|162)\.m\.\d\.bias", -3.0), (r"model\.261\.m\.\d\.bias", (-4.0, -3.0))]},
    # YOLOv6 N/S/M/L: convs damped (0.85, and 0.6 on the BepC3 / SPPF / BiFusion 1x1 convs) so that the ReLU bodies of M do not grow
    # their activations layer by layer; class logits widened (gain 12: at 16 the M device error is 1.04e-3); box biases of 2 grid cells
    # keep the raw l, t, r, b distances of N/S positive (a constant bias cancels in the DFL softmax of M/L).  The class bias of each
    # scale (`variants`) puts ~100 of the 8400 anchors per frame above box_score = 0.4, measured on the fp32 oracle over synthetic
    # frames 0-3: the 100th-highest max-class logit sits 0.135 (N), 0.177 (S), 0.30 (M) above and 0.595 (L) below logit(0.4) at
    # bias -3.  The per-anchor max-class logit spread is small (std 0.13-0.24), so the scores crowd the threshold.
    "yolov6": {"conv_gain": 0.85,
               "gains": [(r"(backbone|neck)\..*\.cv\d\.block\.conv\.weight", 0.6), (r"detect\.cls_preds\.\d\.weight", 12.0),
                         (r"detect\.reg_preds\.\d\.weight", 1.0)],
               "fill": [(r"detect\.reg_preds\.\d\.bias", 2.0)],
               "variants": {sc: {"fill": [(r"detect\.cls_preds\.\d\.bias", -3.0 + d)]}
                            for sc, d in (("n", -0.135), ("s", -0.177), ("m", -0.30), ("l", 0.595))}},
    # YOLOv6-Lite S/M/L: Hardswish halves small activations (slope 1/2 at 0) and grows large ones quadratically, so a random net either
    # forgets its input or blows up: at conv gain 1.0 the neck outputs of two synthetic frames differ by 0.1-5 %, at 1.2 S's neck
    # reaches |x| ~ 10 and L's ~ 100, at 1.3 ~ 1e5 (fp32 oracle, frames 0-3).  Near that edge the net also amplifies rounding: at gain
    # 1.15 the CPU fp16 emulation (plan_interp.interpret, every op rounded to its buffer dtype) was up to 8.5e-3 off in probability with
    # YOLOv6's class gain 12.  Gain 1.1 (neck maps differ by 1-22 % between frames) with class gain 8 gives 3.3e-4 (S) to 7.0e-4 (L) on
    # frames 0-3.  Box biases of 2 grid cells keep the raw l, t, r, b distances positive.  The class bias of each scale puts ~50 of the
    # 2125 anchors (320 x 320) per frame above box_score = 0.4: at bias 0 the 50th-highest max-class logit sits 1.65 (S), 1.60 (M), 1.62
    # (L) above 0, so the bias is -0.405 minus that; the per-anchor spread of the max-class logit is small (std 0.12).
    "yolov6lite": {"conv_gain": 1.1,
                   "gains": [(r"detect\.cls_preds\.\d\.weight", 8.0)],
                   "fill": [(r"detect\.reg_preds\.\d\.bias", 2.0)],
                   "variants": {sc: {"fill": [(r"detect\.cls_preds\.\d\.bias", -0.405 - d)]} for sc, d in (("s", 1.65), ("m", 1.60), ("l", 1.62))}},
}


# "workload" head for throughput runs (bench.py): a wider score distribution (scores up to ~0.9, so ByteTrack sees high- and
# low-score detections and keeps tracks alive) at the price of a ~1.5e-3 fp16-vs-fp32 probability error; the parity tests use
# SYNTH_PROFILES, whose scores all lie in [0.4, 0.5].
SYNTH_PROFILES_WORKLOAD = {
    "yolov8": {"gains": [(r"model\.22\.cv3\.\d\.2\.weight", 45.0), (r"model\.22\.cv2\.\d\.2\.weight", 25.0)],
               "fill": [(r"model\.22\.cv3\.\d\.2\.bias", -9.0)]},
}


def synth_weights(kind: str, seed: int = 0, variant: Optional[str] = None, workload: bool = False) -> "Weights":
    """Seeded synthetic weights.  A profile's `variants` entry (YOLOv6, YOLOv6-Lite, YOLOv9, YOLOv10) adds per-variant `fill` rules ahead of the shared ones; other
    kinds ignore `variant`."""
    prof = SYNTH_PROFILES_WORKLOAD.get(kind, SYNTH_PROFILES[kind]) if workload else SYNTH_PROFILES[kind]
    extra = prof.get("variants", {}).get(variant)
    if extra:
        prof = {**prof, "fill": list(extra.get("fill", ())) + list(prof.get("fill", ()))}
    return Weights(None, seed=seed, profile=prof)


# ---------------------------------------------------------------------------------------------
# plan builder
# ---------------------------------------------------------------------------------------------
@dataclass
class View:
    buf: int
    coff: int
    C: int
    H: int
    W: int


class PlanBuilder:
    def __init__(self, model_kind: int, in_c: int, in_h: int, in_w: int):
        self.model_kind, self.in_c, self.in_h, self.in_w = model_kind, in_c, in_h, in_w
        self.buffers: List[Tuple[int, int, int, int, int, int]] = []   # rows_per_img, C, dtype, H, W, flags
        self.ops: List[Tuple[int, OpParams, List[float]]] = []
        self.tensors: List[np.ndarray] = []
        self.outputs: List[Tuple[int, int, int, int]] = []
        self.meta = [0] * 16
        self.flops_per_img = 0   # 2*MAC of the convs/FCs as mathematically defined (no padding waste)
        self.stem_flops_per_img = 0   # the part of flops_per_img that runs in stem_conv.cu (mma.sync) rather than in the wgmma GEMM launches
        self.dw_flops_per_img = 0     # the part of flops_per_img that runs in dwconv.cu (depthwise convs) rather than in the GEMM launches
        self.stem_direct = os.environ.get("ADAS_B200_STEMCONV", "1") != "0"
        self.strided_tma = os.environ.get("ADAS_B200_STRIDED_TMA", "1") != "0"
        # buffer 0: the network input image, padded NHWC with C=4 (R,G,B,0)
        self.image = self.new_padded(in_h, in_w, 4)

    # -- buffers ------------------------------------------------------------------------------
    def new_padded(self, H: int, W: int, C: int, f32: bool = False) -> View:
        assert C % 4 == 0
        self.buffers.append(((H + 2) * (W + 2), C, 1 if f32 else 0, H, W, 0))
        return View(len(self.buffers) - 1, 0, C, H, W)

    def new_dense(self, rows_per_img: int, C: int, f32: bool = False) -> int:
        self.buffers.append((rows_per_img, C, 1 if f32 else 0, 0, 0, 0))
        return len(self.buffers) - 1

    def tensor(self, a: np.ndarray) -> int:
        assert a.dtype in (np.float16, np.float32)
        self.tensors.append(np.ascontiguousarray(a))
        return len(self.tensors) - 1

    @staticmethod
    def sub(v: View, coff: int, C: int) -> View:
        assert coff + C <= v.C + 0 or True
        return View(v.buf, v.coff + coff, C, v.H, v.W)

    # -- ops ----------------------------------------------------------------------------------
    def _op(self, typ: int, f: Optional[List[float]] = None, **fields: int) -> OpParams:
        """Append an op of type `typ` with the named fields of OP_FIELDS[typ] (the others 0) and floats f (the others 0.0)."""
        p = OpParams(typ)
        for name, v in fields.items():
            setattr(p, name, v)
        self.ops.append((typ, p, list(f or []) + [0.0] * (OP_NF - len(f or []))))
        return p

    def conv(self, x: View, w: np.ndarray, b: Optional[np.ndarray], k: int, s: int, act: int, out: Optional[View] = None,
             res: Optional[View] = None, res_pre_act: bool = False, out_f32: bool = False, pad: Optional[int] = None,
             tile: Optional[Tuple[int, int]] = None, no_slab: bool = False, res_scale: Optional[float] = None,
             wide_stem: bool = False) -> View:
        """w: folded [Cout, Cin_real, k, k] fp32.  x.C may exceed Cin_real (zero-padded image channel).
        res_scale: out = act(conv) + res_scale * res (YOLOv6 BottleRep's alpha); None = a plain residual add (op f[0] = 0).
        no_slab (test hook): a 3x3 stride-1 conv loads one activation tile per tap instead of one slab per (dy, k-block).
        wide_stem: an 80 / 96-channel image conv also runs in stem_conv.cu (the YOLOv7 P6 stems); without it those widths keep the
        im2col + GEMM route, so the 80-channel stems of YOLOv5x / YOLOv8x pack as before.
        Cout % 8 != 0: the epilogue stores 8-channel vectors, so the conv owns n_store = round_up(Cout, 8) channels
        [out.coff, out.coff + n_store) of `out` (a concat neighbour starts at out.coff + n_store); channels [Cout, n_store) hold
        act(0) = 0 (zero weights and bias) plus the residual's channels [Cout, n_store).  A residual therefore owns n_store channels
        too, with zeros past Cout -- as every output of such a conv has, so a residual written by a conv of the same Cout (the
        YOLOv9 GELAN blocks) keeps the tail exactly zero."""
        assert res_scale is None or (res is not None and not res_pre_act and math.isfinite(res_scale) and res_scale != 0.0), res_scale
        cout, cin_real = int(w.shape[0]), int(w.shape[1])
        pad = k // 2 if pad is None else pad
        Ho = (x.H + 2 * pad - k) // s + 1
        Wo = (x.W + 2 * pad - k) // s + 1
        self.flops_per_img += 2 * Ho * Wo * cout * cin_real * k * k
        cin = x.C
        assert cin >= cin_real
        if cin > cin_real:
            wp = np.zeros((cout, cin, k, k), np.float32)
            wp[:, :cin_real] = w
            w = wp
        n_store = (cout + 7) // 8 * 8                      # the epilogue stores 8-channel vectors
        if out is None:
            out = self.new_padded(Ho, Wo, n_store, f32=out_f32)
        assert out.H == Ho and out.W == Wo, (out, Ho, Wo)
        stem_couts = (16, 24, 32, 48, 64, 80, 96) if wide_stem else (16, 24, 32, 48, 64)
        if (self.stem_direct and x.buf == self.image.buf and x.C == 4 and s in (1, 2) and 3 <= k <= 7 and cout in stem_couts and res is None
                and not out_f32 and tile is None and out.coff % 8 == 0):
            return self.stem_conv(x, w, b, k, s, pad, act, out)
        wk = np.transpose(w, (0, 2, 3, 1)).reshape(cout, k * k * cin)   # [Cout, kh, kw, Cin]
        if n_store != cout:
            wk = np.concatenate([wk, np.zeros((n_store - cout, wk.shape[1]), np.float32)], 0)
            if b is not None:
                b = np.concatenate([b, np.zeros(n_store - cout, np.float32)])
        bias_t = self.tensor(b.astype(np.float32)) if b is not None else -1
        res_buf, res_coff = (res.buf, res.coff) if res is not None else (-1, 0)
        s2 = 0
        if k == 1 and s == 1 and pad == 0 and cin % 8 == 0:
            a, ntaps, Kc = x, 1, cin
        elif k == 3 and s == 1 and pad == 1 and cin % 64 == 0:
            a, ntaps, Kc = x, 9, cin
        elif s == 2 and cin % 64 == 0 and ((k == 3 and pad == 1) or (k == 1 and pad == 0)) and x.H % 2 == 0 and x.W % 2 == 0 \
                and self.strided_tma:
            # stride-2 conv read straight from the padded input through a traversal-stride-2 TMA map (no patch matrix)
            a, ntaps, Kc, s2 = x, k * k, cin, 1
        else:
            # patch gather into a [rows_out_padded, Kpad] matrix, then a plain GEMM
            assert cin % 4 == 0
            Kpad = (k * k * cin + 7) // 8 * 8
            self.buffers.append(((Ho + 2) * (Wo + 2), Kpad, 0, Ho, Wo, 0))
            pb = len(self.buffers) - 1
            self._op(OP_IM2COL, in_buf=x.buf, in_coff=x.coff, Cin=cin, kh=k, kw=k, stride=s, pad=pad, out_buf=pb)
            a, ntaps, Kc = View(pb, 0, Kpad, Ho, Wo), 1, Kpad
            if Kpad != wk.shape[1]:
                wk = np.concatenate([wk, np.zeros((wk.shape[0], Kpad - wk.shape[1]), np.float32)], 1)
        w_t = self.tensor(wk.astype(np.float16))
        bn, mt = tile if tile is not None else (0, 0)          # (BN, MT) forced by tests; 0 = cost model + autotune
        self._op(OP_GEMM, [res_scale] if res_scale is not None else None, a_buf=a.buf, a_coff=a.coff, Kc=Kc, ntaps=ntaps, w_tensor=w_t,
                 bias_tensor=bias_t, N=n_store, act=act, res_buf=res_buf, res_coff=res_coff, res_pre_act=1 if res_pre_act else 0,
                 out_buf=out.buf, out_coff=out.coff, masked=1, BN=bn, s2=s2, MT=mt, no_slab=1 if no_slab else 0)
        return View(out.buf, out.coff, cout, Ho, Wo)

    def conv_transpose2x2(self, x: View, w: np.ndarray, b: Optional[np.ndarray], out: View, tile: Optional[Tuple[int, int]] = None) -> View:
        """ConvTranspose2d(k=2, s=2, p=0), w [Cin, Cout, 2, 2] as upstream stores it.  The 2x2 windows do not overlap, so it is a 1x1 GEMM
        with N = 4 * Cout, columns ordered (dy, dx, c); the epilogue stores column group (dy, dx) of input pixel (y, x) to output pixel
        (2y + dy, 2x + dx) of `out` (a 2H x 2W view, possibly a concat slice).  The bias is replicated for the 4 groups."""
        cin, cout = int(w.shape[0]), int(w.shape[1])
        assert w.shape[2:] == (2, 2) and cout % 8 == 0 and x.C == cin and cin % 8 == 0, (w.shape, x.C)
        assert out.H == 2 * x.H and out.W == 2 * x.W and out.C == cout, (out, x)
        self.flops_per_img += 2 * x.H * x.W * cin * cout * 4
        wk = np.transpose(w, (2, 3, 1, 0)).reshape(4 * cout, cin)             # [dy, dx, Cout, Cin]
        bias_t = self.tensor(np.tile(b.astype(np.float32), 4)) if b is not None else -1
        bn, mt = tile if tile is not None else (0, 0)
        self._op(OP_GEMM, a_buf=x.buf, a_coff=x.coff, Kc=cin, ntaps=1, w_tensor=self.tensor(wk.astype(np.float16)), bias_tensor=bias_t,
                 N=4 * cout, act=ACT_NONE, res_buf=-1, out_buf=out.buf, out_coff=out.coff, masked=1, BN=bn, MT=mt, up2=1)
        return View(out.buf, out.coff, cout, out.H, out.W)

    def stem_conv(self, x: View, w: np.ndarray, b: Optional[np.ndarray], k: int, s: int, pad: int, act: int, out: View) -> View:
        """k x k stride-1 or stride-2 conv of the C=4 image by stem_conv.cu (no patch matrix): weights packed [Cout][k][KR], KR = round_up(4k, 16),
        element [dy][dx*4 + c] -- one 16-wide k-step of the warp MMA is a run of consecutive bytes of one image row.
        `w` arrives zero-padded to 4 input channels."""
        cout = int(w.shape[0])
        KR = (4 * k + 15) // 16 * 16
        wq = np.zeros((cout, k, KR), np.float32)
        wq[:, :, :4 * k] = np.transpose(w, (0, 2, 3, 1)).reshape(cout, k, 4 * k)      # [Cout, dy, dx, c]
        w_t = self.tensor(wq.astype(np.float16))
        bias_t = self.tensor(b.astype(np.float32)) if b is not None else -1
        self.stem_flops_per_img += 2 * out.H * out.W * cout * 3 * k * k
        self._op(OP_STEMCONV, in_buf=x.buf, w_tensor=w_t, bias_tensor=bias_t, Cout=cout, k=k, pad=pad, act=act, out_buf=out.buf,
                 out_coff=out.coff, stride=0 if s == 2 else s)   # 0 = stride 2
        return View(out.buf, out.coff, cout, out.H, out.W)

    def stem7x7s2(self, x: View, w: np.ndarray, b: np.ndarray, act: int) -> View:
        """7x7 stride-2 pad-3 conv on the C=4 image without a patch matrix: the image is re-laid out once as
        Q[j][xo][p*32 + kx*4 + c] = img[2j-1+p][2xo+kx-3][c] (row PAIRS x the 7 horizontal taps = 64 channels) on the
        OUTPUT's padded grid, which turns the conv into 4 vertically shifted GEMM taps of K = 64 (rows yo-1 .. yo+2)."""
        cout, cin_real = int(w.shape[0]), int(w.shape[1])
        assert w.shape[2:] == (7, 7) and x.C == 4 and cin_real <= 4 and x.H % 2 == 0 and x.W % 2 == 0
        Ho, Wo = x.H // 2, x.W // 2
        self.flops_per_img += 2 * Ho * Wo * cout * cin_real * 49
        q = self.new_padded(Ho, Wo, 64)
        self._op(OP_STEMPACK, in_buf=x.buf, out_buf=q.buf)
        wq = np.zeros((cout, 4, 2, 8, 4), np.float32)             # [n][t][p][kx(7 used of 8)][c]
        for t in range(4):
            for pp in range(2):
                ky = 2 * t + pp
                if ky < 7:
                    wq[:, t, pp, :7, :cin_real] = np.transpose(w[:, :, ky, :], (0, 2, 1))
        out = self.new_padded(Ho, Wo, (cout + 7) // 8 * 8)
        w_t = self.tensor(wq.reshape(cout, 256).astype(np.float16))
        bias_t = self.tensor(b.astype(np.float32))
        # ntaps = 4 selects the vertical tap table (row shifts -2, -1, 0, +1 padded rows)
        self._op(OP_GEMM, a_buf=q.buf, Kc=64, ntaps=4, w_tensor=w_t, bias_tensor=bias_t, N=cout, act=act, res_buf=-1, out_buf=out.buf,
                 masked=1)
        return View(out.buf, 0, cout, Ho, Wo)

    def maxpool(self, x: View, k: int, s: int, p: int, out: Optional[View] = None) -> View:
        Ho = (x.H + 2 * p - k) // s + 1
        Wo = (x.W + 2 * p - k) // s + 1
        if out is None:
            out = self.new_padded(Ho, Wo, x.C)
        assert out.H == Ho and out.W == Wo and x.C % 8 == 0
        self._op(OP_MAXPOOL, in_buf=x.buf, in_coff=x.coff, C=x.C, k=k, stride=s, pad=p, out_buf=out.buf, out_coff=out.coff)
        return View(out.buf, out.coff, x.C, Ho, Wo)

    def avgpool2(self, x: View, fill: int, out: Optional[View] = None) -> View:
        """2x2 stride-1 average pool (upstream `avg_pool2d(x, 2, 1, 0)`, an (H-1) x (W-1) map) stored on x's H x W grid: row H-1 and
        column W-1 hold 0 (fill 0: a following 3x3 stride-2 pad-1 conv sees upstream's zero padding there) or -inf (fill 1: a following
        3x3 stride-2 pad-1 max pool ignores them)."""
        if out is None:
            out = self.new_padded(x.H, x.W, x.C)
        assert out.H == x.H and out.W == x.W and x.C % 8 == 0 and x.coff % 8 == 0 and out.coff % 8 == 0 and fill in (0, 1)
        self._op(OP_AVGPOOL2, in_buf=x.buf, in_coff=x.coff, C=x.C, out_buf=out.buf, out_coff=out.coff, fill=fill)
        return View(out.buf, out.coff, x.C, x.H, x.W)

    def dwconv(self, x: View, w: np.ndarray, b: np.ndarray, k: int, s: int, act: int, out: Optional[View] = None,
               res: Optional[View] = None) -> View:
        """Depthwise k x k conv (pad k/2; k 3 / 5 stride 1 / 2, k 7 stride 1) of x's channels: w [C_real, 1, k, k] fp32, b [C_real];
        x.C may exceed C_real (zero-padded channels get zero weights and bias).  out = act(conv + b) (+ res).  Weights are packed
        [k*k][C] fp16 so one tap of 8 channels is one 16-byte load (dwconv.cu)."""
        c_real = int(w.shape[0])
        assert w.shape[1:] == (1, k, k) and c_real <= x.C and x.C % 8 == 0 and x.coff % 8 == 0, (w.shape, x)
        assert (k in (3, 5) and s in (1, 2)) or (k == 7 and s == 1), (k, s)
        assert act in (ACT_NONE, ACT_SILU, ACT_HSWISH), act
        Ho = (x.H + 2 * (k // 2) - k) // s + 1
        Wo = (x.W + 2 * (k // 2) - k) // s + 1
        if out is None:
            out = self.new_padded(Ho, Wo, x.C)
        assert out.H == Ho and out.W == Wo and out.coff % 8 == 0, (out, Ho, Wo)
        assert res is None or (res.H == Ho and res.W == Wo and res.coff % 8 == 0), res
        wk = np.zeros((k * k, x.C), np.float32)
        wk[:, :c_real] = w.reshape(c_real, k * k).T
        bk = np.zeros(x.C, np.float32)
        bk[:c_real] = b
        f = 2 * Ho * Wo * c_real * k * k
        self.flops_per_img += f
        self.dw_flops_per_img += f
        self._op(OP_DWCONV, in_buf=x.buf, in_coff=x.coff, C=x.C, k=k, stride=s, act=act, w_tensor=self.tensor(wk.astype(np.float16)),
                 bias_tensor=self.tensor(bk), out_buf=out.buf, out_coff=out.coff, res_buf=res.buf if res is not None else -1,
                 res_coff=res.coff if res is not None else 0)
        return View(out.buf, out.coff, x.C, Ho, Wo)

    def attention(self, qkv: View, nh: int, kdp: int, hd: int, scale: float, out: Optional[View] = None) -> View:
        """Multi-head self-attention over the H*W pixels (attention.cu).  qkv holds [Q nh*kdp | K nh*kdp | V nh*hd] channels; the
        output holds nh*hd channels, head-major: softmax(Q K^T * scale) V of head h in channels [h*hd, (h+1)*hd)."""
        assert qkv.C == nh * (2 * kdp + hd) and kdp % 16 == 0 and hd % 8 == 0 and qkv.coff % 8 == 0 and math.isfinite(scale) and scale > 0
        if out is None:
            out = self.new_padded(qkv.H, qkv.W, nh * hd)
        assert out.H == qkv.H and out.W == qkv.W and out.coff % 8 == 0, out
        self._op(OP_ATTN, [scale], in_buf=qkv.buf, in_coff=qkv.coff, nh=nh, kdp=kdp, hd=hd, out_buf=out.buf, out_coff=out.coff)
        return View(out.buf, out.coff, nh * hd, qkv.H, qkv.W)

    def upsample2x(self, x: View, out: View) -> View:
        assert out.H == 2 * x.H and out.W == 2 * x.W and x.C % 8 == 0
        self._op(OP_UPSAMPLE2X, in_buf=x.buf, in_coff=x.coff, C=x.C, out_buf=out.buf, out_coff=out.coff)
        return View(out.buf, out.coff, x.C, out.H, out.W)

    def cbfuse(self, base: View, srcs: Sequence[Tuple[View, int]], out: Optional[View] = None) -> View:
        """YOLOv9-E CBFuse: out = base + sum of the nearest-upsampled source slices, source i read at (y >> shift_i, x >> shift_i)
        (fp32 sum in the listed order, one rounding).  out None: in place on `base`."""
        out = base if out is None else out
        assert 1 <= len(srcs) <= 5 and base.C == out.C and base.C % 8 == 0 and base.coff % 8 == 0 and out.coff % 8 == 0, (base, out)
        assert (base.H, base.W) == (out.H, out.W), (base, out)
        for v, shift in srcs:
            assert v.C == out.C and v.coff % 8 == 0 and 0 <= shift <= 4 and (v.H << shift, v.W << shift) == (out.H, out.W), (v, shift, out)
            assert v.buf != out.buf or v.coff >= out.coff + out.C or out.coff >= v.coff + v.C, (v, out)
        p = self._op(OP_CBFUSE, out_buf=out.buf, out_coff=out.coff, C=out.C, base_buf=base.buf, base_coff=base.coff, n_src=len(srcs))
        for s, (v, shift) in enumerate(srcs):
            p[cbfuse_src_slot(s):cbfuse_src_slot(s + 1)] = [v.buf, v.coff, shift]
        return View(out.buf, out.coff, out.C, out.H, out.W)

    def se(self, x: View, w1: np.ndarray, b1: np.ndarray, w2: np.ndarray, b2: np.ndarray, out: Optional[View] = None) -> View:
        """Squeeze-excite (YOLOv6-Lite SEBlock): out = x * hardsigmoid(w2 relu(w1 mean(x) + b1) + b2), mean over the H x W interior.
        w1 [hid, C_real(, 1, 1)], b1 [hid], w2 [C_real, hid(, 1, 1)], b2 [C_real] (1x1 convs with bias), kept fp32.  x.C may exceed
        C_real: the padded channels get zero FC weights, so they read as zero means and, being zero, stay zero.  out None: in place."""
        hid, c_real = int(w1.shape[0]), int(w1.shape[1])
        assert x.C % 8 == 0 and x.coff % 8 == 0 and c_real <= x.C and tuple(w2.shape[:2]) == (c_real, hid), (x, w1.shape, w2.shape)
        out = x if out is None else out
        assert (out.H, out.W, out.C) == (x.H, x.W, x.C) and out.coff % 8 == 0, (out, x)
        w1p = np.zeros((hid, x.C), np.float32)
        w1p[:, :c_real] = w1.reshape(hid, c_real)
        w2p = np.zeros((x.C, hid), np.float32)
        w2p[:c_real] = w2.reshape(c_real, hid)
        b2p = np.zeros(x.C, np.float32)
        b2p[:c_real] = b2
        self._op(OP_SE, in_buf=x.buf, in_coff=x.coff, C=x.C, hid=hid, w1=self.tensor(w1p), b1=self.tensor(np.asarray(b1, np.float32).reshape(hid)),
                 w2=self.tensor(w2p), b2=self.tensor(b2p), out_buf=out.buf, out_coff=out.coff)
        return View(out.buf, out.coff, x.C, x.H, x.W)

    def shuffle2(self, a: View, b: View, out: Optional[View] = None) -> View:
        """torch.cat([a, b], 1) then channel_shuffle(groups = 2): out(2j) = a(j), out(2j + 1) = b(j); a.C == b.C, a multiple of 8."""
        n = a.C
        assert b.C == n and n % 8 == 0 and a.coff % 8 == 0 and b.coff % 8 == 0 and (a.H, a.W) == (b.H, b.W), (a, b)
        if out is None:
            out = self.new_padded(a.H, a.W, 2 * n)
        assert out.C == 2 * n and (out.H, out.W) == (a.H, a.W) and out.coff % 8 == 0, out
        for v in (a, b):
            assert v.buf != out.buf or v.coff >= out.coff + 2 * n or out.coff >= v.coff + n, (v, out)
        self._op(OP_SHUFFLE2, a_buf=a.buf, a_coff=a.coff, b_buf=b.buf, b_coff=b.coff, n=n, out_buf=out.buf, out_coff=out.coff)
        return View(out.buf, out.coff, 2 * n, a.H, a.W)

    def layernorm(self, in_buf: int, d_len: int, d_norm: int, gamma: np.ndarray, beta: np.ndarray, eps: float, out_buf: int) -> None:
        self._op(OP_LAYERNORM, [eps], in_buf=in_buf, d_len=d_len, gamma_tensor=self.tensor(gamma.astype(np.float32)),
                 beta_tensor=self.tensor(beta.astype(np.float32)), out_buf=out_buf, d_norm=d_norm)

    def fc(self, in_buf: int, K: int, w: np.ndarray, b: np.ndarray, act: int, out_buf: int) -> None:
        """swap-AB GEMM: weights [Nout, K] stream through the A operand once per batch."""
        nout = int(w.shape[0])
        assert w.shape[1] == K and K % 8 == 0
        self._op(OP_GEMM, a_buf=in_buf, Kc=K, ntaps=1, w_tensor=self.tensor(w.astype(np.float16)), bias_tensor=self.tensor(b.astype(np.float32)),
                 N=nout, act=act, res_buf=-1, out_buf=out_buf, transposed=1)

    # -- serialisation ---------------------------------------------------------------------------
    def write(self, path: str) -> None:
        rec = bytearray()
        for b in self.buffers:
            rec += struct.pack(BUF_FMT, *b)
        for typ, p, f in self.ops:
            rec += struct.pack(OP_FMT, typ, *p, *f)
        offs = []
        off = 0
        for t in self.tensors:
            offs.append(off)
            off += (t.nbytes + 255) // 256 * 256
        for t, o in zip(self.tensors, offs):
            rec += struct.pack(TEN_FMT, o, t.nbytes, 1 if t.dtype == np.float32 else 0, 0)
        for o in self.outputs:
            rec += struct.pack(OUT_FMT, *o)
        blob_offset = (HDR_SIZE + len(rec) + 255) // 256 * 256
        hdr = struct.pack(HDR_FMT, b"B200PLAN", PLAN_VERSION, self.model_kind, self.in_c, self.in_h, self.in_w, len(self.buffers),
                          len(self.ops), len(self.tensors), len(self.outputs), *self.meta, blob_offset, off)
        with open(path, "wb") as f:
            f.write(hdr)
            f.write(rec)
            f.write(b"\0" * (blob_offset - HDR_SIZE - len(rec)))
            for t in self.tensors:
                f.write(t.tobytes())
                padn = (-t.nbytes) % 256
                if padn:
                    f.write(b"\0" * padn)


# ---------------------------------------------------------------------------------------------
# YOLOv8
# ---------------------------------------------------------------------------------------------
YOLOV8_SCALES = {  # depth, width, max_channels (ultralytics yolov8.yaml)
    "n": (0.33, 0.25, 1024), "s": (0.33, 0.50, 1024), "m": (0.67, 0.75, 768), "l": (1.00, 1.00, 512), "x": (1.00, 1.25, 512),
}
BN_EPS_YOLO = 1e-3


def _v8_ch(c: int, width: float, max_ch: int) -> int:
    return int(math.ceil(min(c, max_ch) * width / 8) * 8)


def _v8_n(n: int, depth: float) -> int:
    return max(round(n * depth), 1)


def build_yolov8(weights: Weights, scale: str = "l", nc: int = 80, in_h: int = 640, in_w: int = 640) -> PlanBuilder:
    depth, width, max_ch = YOLOV8_SCALES[scale]
    ch = lambda c: _v8_ch(c, width, max_ch)
    rep = lambda n: _v8_n(n, depth)
    pb = PlanBuilder(MODEL_YOLOV8, 3, in_h, in_w)
    W = weights

    def cbs(x: View, name: str, cout: int, k: int, s: int, out: Optional[View] = None, res: Optional[View] = None,
            cin: Optional[int] = None, res_branch: bool = False) -> View:
        w, b = W.conv_bn(name, cout, cin if cin is not None else x.C, k, BN_EPS_YOLO, res_branch=res_branch)
        return pb.conv(x, w, b, k, s, ACT_SILU, out=out, res=res)

    def c2f(x: View, name: str, c2: int, n: int, shortcut: bool, out: Optional[View] = None) -> View:
        c = c2 // 2
        cat = pb.new_padded(x.H, x.W, (2 + n) * c)
        cbs(x, f"{name}.cv1", 2 * c, 1, 1, out=pb.sub(cat, 0, 2 * c))
        for i in range(n):
            src = pb.sub(cat, (1 + i) * c, c)
            t = cbs(src, f"{name}.m.{i}.cv1", c, 3, 1)
            cbs(t, f"{name}.m.{i}.cv2", c, 3, 1, out=pb.sub(cat, (2 + i) * c, c), res=src if shortcut else None, res_branch=shortcut)
        return cbs(cat, f"{name}.cv2", c2, 1, 1, out=out)

    c1, c2_, c3, c4, c5 = ch(64), ch(128), ch(256), ch(512), ch(1024)
    H, Wd = in_h, in_w
    # head concat buffers are allocated up front so producers can write straight into their slices
    cat11 = pb.new_padded(H // 16, Wd // 16, c5 + c4)      # [up(9), 6]
    cat14 = pb.new_padded(H // 8, Wd // 8, c4 + c3)        # [up(12), 4]
    cat17 = pb.new_padded(H // 16, Wd // 16, c3 + c4)      # [16, 12]
    cat20 = pb.new_padded(H // 32, Wd // 32, c4 + c5)      # [19, 9]

    x = cbs(pb.image, "model.0", c1, 3, 2, cin=3)
    x = cbs(x, "model.1", c2_, 3, 2)
    x = c2f(x, "model.2", c2_, rep(3), True)
    x = cbs(x, "model.3", c3, 3, 2)
    p3 = c2f(x, "model.4", c3, rep(6), True, out=pb.sub(cat14, c4, c3))
    x = cbs(p3, "model.5", c4, 3, 2)
    p4 = c2f(x, "model.6", c4, rep(6), True, out=pb.sub(cat11, c5, c4))
    x = cbs(p4, "model.7", c5, 3, 2)
    x = c2f(x, "model.8", c5, rep(3), True)
    # SPPF
    ch_ = c5 // 2
    sp = pb.new_padded(x.H, x.W, 4 * ch_)
    y = cbs(x, "model.9.cv1", ch_, 1, 1, out=pb.sub(sp, 0, ch_))
    for i in range(3):
        y = pb.maxpool(y, 5, 1, 2, out=pb.sub(sp, (i + 1) * ch_, ch_))
    p5 = cbs(sp, "model.9.cv2", c5, 1, 1, out=pb.sub(cat20, c4, c5))
    # top-down
    pb.upsample2x(p5, pb.sub(cat11, 0, c5))
    h12 = c2f(cat11, "model.12", c4, rep(3), False, out=pb.sub(cat17, c3, c4))
    pb.upsample2x(h12, pb.sub(cat14, 0, c4))
    h15 = c2f(cat14, "model.15", c3, rep(3), False)
    cbs(h15, "model.16", c3, 3, 2, out=pb.sub(cat17, 0, c3))
    h18 = c2f(cat17, "model.18", c4, rep(3), False)
    cbs(h18, "model.19", c4, 3, 2, out=pb.sub(cat20, 0, c4))
    h21 = c2f(cat20, "model.21", c5, rep(3), False)
    A = v8_detect(pb, W, "model.22", (h15, h18, h21), nc)
    pb.meta[0], pb.meta[1] = nc, A
    return pb


def grouped_to_dense(w: np.ndarray, groups: int) -> np.ndarray:
    """Grouped conv weight [Cout, Cin / groups, k, k] as the equivalent dense [Cout, Cin, k, k] block-diagonal weight (exact)."""
    if groups == 1:
        return w
    cout, cg = int(w.shape[0]), int(w.shape[1])
    og = cout // groups
    d = np.zeros((cout, cg * groups) + tuple(w.shape[2:]), w.dtype)
    for g in range(groups):
        d[g * og:(g + 1) * og, g * cg:(g + 1) * cg] = w[g * og:(g + 1) * og]
    return d


def v8_detect(pb: PlanBuilder, W: Weights, name: str, feats, nc: int, box_groups: int = 1, conv_bn=None) -> int:
    """YOLOv8 Detect (and YOLOv9 DDetect: `box_groups` = 4 on the second and third box convs) on the P3 / P4 / P5 views; returns the
    anchor count.  Grouped convs are packed as dense block-diagonal weights; flops_per_img counts their grouped MACs.  `conv_bn(name,
    cout, cin, k)` replaces W.conv_bn for the Conv + BN layers (YOLOv9: upstream-fused files)."""
    conv_bn = conv_bn or (lambda n, co, ci, k: W.conv_bn(n, co, ci, k, BN_EPS_YOLO))
    reg_max = 16
    cb = max(16, feats[0].C // 4, reg_max * 4)
    cc = max(feats[0].C, min(nc, 100))
    A = 0
    for li, (feat, stride) in enumerate(zip(feats, (8, 16, 32))):
        cin = feat.C
        # first convs of the box and cls branches share their input: one GEMM with N = cb + cc
        wb, bb = conv_bn(f"{name}.cv2.{li}.0", cb, cin, 3)
        wc, bc = conv_bn(f"{name}.cv3.{li}.0", cc, cin, 3)
        t0 = pb.conv(feat, np.concatenate([wb, wc], 0), np.concatenate([bb, bc]), 3, 1, ACT_SILU)
        w1, b1 = conv_bn(f"{name}.cv2.{li}.1", cb, cb // box_groups, 3)
        tb = pb.conv(pb.sub(t0, 0, cb), grouped_to_dense(w1, box_groups), b1, 3, 1, ACT_SILU)
        w2, b2 = conv_bn(f"{name}.cv3.{li}.1", cc, cc, 3)
        tc = pb.conv(pb.sub(t0, cb, cc), w2, b2, 3, 1, ACT_SILU)
        head = pb.new_padded(feat.H, feat.W, 4 * reg_max + (nc + 7) // 8 * 8, f32=True)
        wbx, bbx = W.conv_bias(f"{name}.cv2.{li}.2", 4 * reg_max, cb // box_groups, 1)
        wcl, bcl = W.conv_bias(f"{name}.cv3.{li}.2", nc, cc, 1)
        pb.conv(tb, grouped_to_dense(wbx, box_groups), bbx, 1, 1, ACT_NONE, out=pb.sub(head, 0, 4 * reg_max), out_f32=True)
        pb.conv(tc, wcl, bcl, 1, 1, ACT_NONE, out=pb.sub(head, 4 * reg_max, (nc + 7) // 8 * 8), out_f32=True)
        # the dense packing of the two grouped convs does (groups - 1) / groups of their counted MACs as zeros
        pb.flops_per_img -= 2 * feat.H * feat.W * (cb * cb * 9 + 4 * reg_max * cb) * (box_groups - 1) // box_groups
        pb.outputs.append((head.buf, 0, head.C, stride))
        A += feat.H * feat.W
    return A


# ---------------------------------------------------------------------------------------------
# YOLOv5 (v6.2)
# ---------------------------------------------------------------------------------------------
YOLOV5_SCALES = {"n": (0.33, 0.25), "s": (0.33, 0.50), "m": (0.67, 0.75), "l": (1.0, 1.0), "x": (1.33, 1.25)}


def build_yolov5(weights: Weights, scale: str = "n", nc: int = 80, in_h: int = 640, in_w: int = 640, lite: bool = False) -> PlanBuilder:
    """lite=True packs a YOLOv5-lite style head: the engine output is the sigmoid-only tensor and the grid / anchor decode is
    `YoloLiteParameters.lite_postprocess` (reference yoloDetector.py:36-50, ObjectModelType.YOLOV5_LITE), run on the device by the
    fused detect calls.  Header meta[2] marks such plans."""
    depth, width = YOLOV5_SCALES[scale]
    ch = lambda c: int(math.ceil(c * width / 8) * 8)
    rep = lambda n: max(round(n * depth), 1)
    pb = PlanBuilder(MODEL_YOLOV5, 3, in_h, in_w)
    W = weights

    def cbs(x: View, name: str, cout: int, k: int, s: int, out=None, res=None, cin=None, pad=None, res_branch=False) -> View:
        w, b = W.conv_bn(name, cout, cin if cin is not None else x.C, k, BN_EPS_YOLO, res_branch=res_branch)
        return pb.conv(x, w, b, k, s, ACT_SILU, out=out, res=res, pad=pad)

    def c3(x: View, name: str, c2: int, n: int, shortcut: bool, out=None) -> View:
        c_ = c2 // 2
        cat = pb.new_padded(x.H, x.W, 2 * c_)
        y = cbs(x, f"{name}.cv1", c_, 1, 1)
        for i in range(n):
            t = cbs(y, f"{name}.m.{i}.cv1", c_, 1, 1)
            last = i == n - 1
            y = cbs(t, f"{name}.m.{i}.cv2", c_, 3, 1, out=pb.sub(cat, 0, c_) if last else None, res=y if shortcut else None,
                    res_branch=shortcut)
        cbs(x, f"{name}.cv2", c_, 1, 1, out=pb.sub(cat, c_, c_))
        return cbs(cat, f"{name}.cv3", c2, 1, 1, out=out)

    c64, c128, c256, c512, c1024 = ch(64), ch(128), ch(256), ch(512), ch(1024)
    H, Wd = in_h, in_w
    cat12 = pb.new_padded(H // 16, Wd // 16, c512 + c512)   # [up(10), 6]
    cat16 = pb.new_padded(H // 8, Wd // 8, c256 + c256)     # [up(14), 4]
    cat19 = pb.new_padded(H // 16, Wd // 16, c256 + c256)   # [18, 14]
    cat22 = pb.new_padded(H // 32, Wd // 32, c512 + c512)   # [21, 10]

    x = cbs(pb.image, "model.0", c64, 6, 2, cin=3, pad=2)
    x = cbs(x, "model.1", c128, 3, 2)
    x = c3(x, "model.2", c128, rep(3), True)
    x = cbs(x, "model.3", c256, 3, 2)
    p3 = c3(x, "model.4", c256, rep(6), True, out=pb.sub(cat16, c256, c256))
    x = cbs(p3, "model.5", c512, 3, 2)
    p4 = c3(x, "model.6", c512, rep(9), True, out=pb.sub(cat12, c512, c512))
    x = cbs(p4, "model.7", c1024, 3, 2)
    x = c3(x, "model.8", c1024, rep(3), True)
    ch_ = c1024 // 2
    sp = pb.new_padded(x.H, x.W, 4 * ch_)
    y = cbs(x, "model.9.cv1", ch_, 1, 1, out=pb.sub(sp, 0, ch_))
    for i in range(3):
        y = pb.maxpool(y, 5, 1, 2, out=pb.sub(sp, (i + 1) * ch_, ch_))
    x = cbs(sp, "model.9.cv2", c1024, 1, 1)
    h10 = cbs(x, "model.10", c512, 1, 1, out=pb.sub(cat22, c512, c512))
    pb.upsample2x(h10, pb.sub(cat12, 0, c512))
    x = c3(cat12, "model.13", c512, rep(3), False)
    h14 = cbs(x, "model.14", c256, 1, 1, out=pb.sub(cat19, c256, c256))
    pb.upsample2x(h14, pb.sub(cat16, 0, c256))
    h17 = c3(cat16, "model.17", c256, rep(3), False)
    cbs(h17, "model.18", c256, 3, 2, out=pb.sub(cat19, 0, c256))
    h20 = c3(cat19, "model.20", c512, rep(3), False)
    cbs(h20, "model.21", c512, 3, 2, out=pb.sub(cat22, 0, c512))
    h23 = c3(cat22, "model.23", c1024, rep(3), False)
    no = 3 * (nc + 5)
    A = 0
    for li, (feat, stride) in enumerate(((h17, 8), (h20, 16), (h23, 32))):
        w, b = W.conv_bias(f"model.24.m.{li}", no, feat.C, 1)
        head = pb.new_padded(feat.H, feat.W, (no + 7) // 8 * 8, f32=True)
        pb.conv(feat, w, b, 1, 1, ACT_NONE, out=head, out_f32=True)
        pb.outputs.append((head.buf, 0, head.C, stride))
        A += 3 * feat.H * feat.W
    pb.meta[0], pb.meta[1] = nc, A
    pb.meta[2] = 1 if lite else 0
    return pb


# ---------------------------------------------------------------------------------------------
# YOLOv7 / YOLOv7-tiny (cfg/training/yolov7.yaml, yolov7-tiny.yaml; P5 models only)
# ---------------------------------------------------------------------------------------------
YOLOV5_ANCHORS = ((10, 13, 16, 30, 33, 23), (30, 61, 62, 45, 59, 119), (116, 90, 156, 198, 373, 326))
YOLOV7_ANCHORS = ((12, 16, 19, 36, 40, 28), (36, 75, 76, 55, 72, 146), (142, 110, 192, 243, 459, 401))
YOLOV7_P6_ANCHORS = ((19, 27, 44, 40, 38, 94), (96, 68, 86, 152, 180, 137), (140, 301, 303, 264, 238, 542), (436, 615, 739, 380, 925, 792))
YOLOV7_ACTS = {"silu": ACT_SILU, "leaky": ACT_LEAKY}
# P6 models (cfg/deploy/yolov7-{w6,e6,d6,e6e}.yaml): ReOrg + Conv(12, stem, 3, 1) stem; five stride-2 stages, each a down-sampling layer
# (W6: Conv 3x3 s2, else DownC) to `cout` channels and an ELAN of width c with n3 chained 3x3 convs to `cout`; head output widths of the
# P3 .. P6 levels (SPPCSPC's width is the P6 one); E6E runs every ELAN twice on the same input and sums the pair (Shortcut).
# D6 as restated here (96-channel stem, 8-conv ELANs, E6's head widths) has 133.8 M parameters / 701.7 GFLOP against the published
# 154.7 M / 806.8 G: some width of the upstream graph is not reproduced.  A D6 checkpoint whose shapes differ is refused by name and shape
# (Weights.get), never packed wrongly.
YOLOV7_P6 = {
    "w6": dict(stem=64, downc=False, n3=4, stages=((128, 64), (256, 128), (512, 256), (768, 384), (1024, 512)), outs=(128, 256, 384, 512),
               pair=False, det=118),
    "e6": dict(stem=80, downc=True, n3=6, stages=((160, 64), (320, 128), (640, 256), (960, 384), (1280, 512)), outs=(160, 320, 480, 640),
               pair=False, det=140),
    "d6": dict(stem=96, downc=True, n3=8, stages=((192, 64), (384, 128), (768, 256), (1152, 384), (1536, 512)), outs=(192, 384, 576, 768),
               pair=False, det=162),
    "e6e": dict(stem=80, downc=True, n3=6, stages=((160, 64), (320, 128), (640, 256), (960, 384), (1280, 512)), outs=(160, 320, 480, 640),
                pair=True, det=261),
}
# head ELAN widths (c, c3): top-down P5, P4, P3, then bottom-up P4, P5, P6
YOLOV7_P6_HEAD = ((384, 192), (256, 128), (128, 64), (256, 128), (384, 192), (512, 256))
YOLOV7_SCALES = ("tiny", "base") + tuple(YOLOV7_P6)
# ReOrg's four strided slices in the order upstream concatenates them: (row, column) offsets of x[..., ::2, ::2], x[..., 1::2, ::2],
# x[..., ::2, 1::2], x[..., 1::2, 1::2]
REORG_SLICES = ((0, 0), (1, 0), (0, 1), (1, 1))


def reorg_stem_weights(w: np.ndarray) -> np.ndarray:
    """Conv(12, c, 3, s=1, p=1) after ReOrg as one Conv(3, c, 6, s=2, p=2) on the image: w6[o, c, 2ky + dy, 2kx + dx] =
    w[o, 3 * slice(dy, dx) + c, ky, kx].  A pure permutation (exact in any precision); ReOrg pixel -1 covers image rows / columns
    -2 and -1, so the zero padding matches too."""
    cout = w.shape[0]
    assert w.shape[1:] == (12, 3, 3), w.shape
    w6 = np.zeros((cout, 3, 6, 6), w.dtype)
    for sl, (dy, dx) in enumerate(REORG_SLICES):
        w6[:, :, dy::2, dx::2] = w[:, 3 * sl:3 * sl + 3]
    return w6


def yolov7_levels(scale: str) -> int:
    return 4 if scale in YOLOV7_P6 else 3


def build_yolov7(weights: Weights, scale: str = "tiny", nc: int = 80, in_h: Optional[int] = None, in_w: Optional[int] = None,
                 act: Optional[str] = None, anchors=None) -> PlanBuilder:
    """YOLOv7 ("base", SiLU), YOLOv7-tiny ("tiny", LeakyReLU(0.1); act="silu" gives the tiny-SiLU variant) or the P6 models "w6", "e6",
    "d6", "e6e" (SiLU, 4 levels, 1280x1280 by default, inputs a multiple of 64).  The head decodes like YOLOv5's ([B, 25200, 5 + nc] at
    640 for P5; [B, 102000, 5 + nc] at 1280 for P6; MODEL_YOLOV5 kind) with the anchor table carried by the plan (header meta[3]).
    RepConv (base head) and IDetect's implicit layers are folded here in fp64; an ELAN's two 1x1 convolutions on the same input run
    as one GEMM writing the last two slices of its concat.  Training-form P6 checkpoints (IAuxDetect four layers after the deploy
    IDetect, aux convs in between) pack from their main path: the deploy numbering is the same up to the head."""
    assert scale in YOLOV7_SCALES, f"YOLOv7 scale {scale!r}: one of {', '.join(YOLOV7_SCALES)} (YOLOv7-X is not supported)"
    p6 = YOLOV7_P6.get(scale)
    in_h = in_h or (1280 if p6 else 640)
    in_w = in_w or (1280 if p6 else 640)
    if p6:
        assert in_h % 64 == 0 and in_w % 64 == 0, f"YOLOv7-{scale.upper()} input {in_h}x{in_w}: a multiple of 64 (stride-64 head)"
    act_id = YOLOV7_ACTS[act or ("leaky" if scale == "tiny" else "silu")]
    pb = PlanBuilder(MODEL_YOLOV5, 3, in_h, in_w)
    W = weights
    eps = BN_EPS_YOLO

    def cbs(x: View, name: str, cout: int, k: int, s: int = 1, out: Optional[View] = None, cin: Optional[int] = None,
            res: Optional[View] = None) -> View:
        w, b = W.conv_bn(name, cout, cin if cin is not None else x.C, k, eps)
        return pb.conv(x, w, b, k, s, act_id, out=out, res=res)

    def elan(x: View, i: int, c: int, c3: int, n3: int, cout: int, out: Optional[View] = None, keep=None, res: Optional[View] = None) -> View:
        """a = model.i, b = model.i+1 (1x1 on x), n3 chained 3x3 convs from b (model.i+2 ..), concat model.i+2+n3 of the kept 3x3
        outputs in reverse order, then b, a; then the 1x1 model.i+3+n3 (+ `res` after its activation: E6E's Shortcut).  `keep`:
        0-based 3x3 positions in the concat (default all)."""
        keep = list(range(n3)) if keep is None else list(keep)
        cat = pb.new_padded(x.H, x.W, len(keep) * c3 + 2 * c)
        wa, ba = W.conv_bn(f"model.{i}", c, x.C, 1, eps)
        wb, bb = W.conv_bn(f"model.{i + 1}", c, x.C, 1, eps)
        ab = pb.conv(x, np.concatenate([wb, wa], 0), np.concatenate([bb, ba]), 1, 1, act_id, out=pb.sub(cat, len(keep) * c3, 2 * c))
        t = pb.sub(ab, 0, c)
        for j in range(n3):
            slot = keep[::-1].index(j) if j in keep else None
            t = cbs(t, f"model.{i + 2 + j}", c3, 3, out=pb.sub(cat, slot * c3, c3) if slot is not None else None)
        return cbs(cat, f"model.{i + 3 + n3}", cout, 1, out=out, res=res)

    def mp_block(x: View, i: int, c: int, out: View) -> View:
        """model.i MaxPool 2x2 s2; model.i+1 = 1x1 of the pool, model.i+2 = 1x1 of x, model.i+3 = 3x3 s2 of model.i+2;
        out = [model.i+3, model.i+1, ...] (channel slices 0 and 1 of `out`)."""
        p = pb.maxpool(x, 2, 2, 0)
        cbs(p, f"model.{i + 1}", c, 1, out=pb.sub(out, c, c))
        t = cbs(x, f"model.{i + 2}", c, 1)
        cbs(t, f"model.{i + 3}", c, 3, 2, out=pb.sub(out, 0, c))
        return out

    def pools(x: View, cat: View, slots: List[int]) -> None:
        """max pools 5, 9, 13 (stride 1, "same" padding) of x into the channel slots of `cat`: 9 and 13 as chained 5x5 pools (exact for
        max pooling whose padding never wins; the pool op takes k <= 7)."""
        y = x
        for sl in slots:
            y = pb.maxpool(y, 5, 1, 2, out=pb.sub(cat, sl * x.C, x.C))

    def sppcspc(x: View, i: int, c_: int, out: View) -> View:
        """model.i SPPCSPC(c_): cv7([cv6(cv5([x1, p5, p9, p13])), cv2(x)]), x1 = cv4(cv3(cv1(x)))."""
        cat7 = pb.new_padded(x.H, x.W, 2 * c_)               # cv7 input [y1, y2]
        sp = pb.new_padded(x.H, x.W, 4 * c_)                 # cv5 input [x1, p5, p9, p13]
        t = cbs(x, f"model.{i}.cv1", c_, 1)
        t = cbs(t, f"model.{i}.cv3", c_, 3)
        x1 = cbs(t, f"model.{i}.cv4", c_, 1, out=pb.sub(sp, 0, c_))
        pools(x1, sp, [1, 2, 3])
        t = cbs(sp, f"model.{i}.cv5", c_, 1)
        cbs(t, f"model.{i}.cv6", c_, 3, out=pb.sub(cat7, 0, c_))
        cbs(x, f"model.{i}.cv2", c_, 1, out=pb.sub(cat7, c_, c_))
        return cbs(cat7, f"model.{i}.cv7", c_, 1, out=out)

    def down_c(x: View, i: int, cout: int, out: View) -> View:
        """model.i DownC(cout): [cv2(cv1(x)) (3x3 s2), cv3(MaxPool 2x2 s2 (x))], cv1 keeping x's width."""
        h = cout // 2
        cbs(pb.maxpool(x, 2, 2, 0), f"model.{i}.cv3", h, 1, out=pb.sub(out, h, h))
        t = cbs(x, f"model.{i}.cv1", x.C, 1)
        cbs(t, f"model.{i}.cv2", h, 3, 2, out=pb.sub(out, 0, h))
        return out

    H, Wd = in_h, in_w
    det_levels = 3
    if p6:
        n3, pair = p6["n3"], p6["pair"]
        n_elan = 4 + n3                                      # layers of one ELAN
        blk = 2 * n_elan + 1 if pair else n_elan             # layers of an ELAN block (E6E: two ELANs + Shortcut)

        def elan_block(x: View, i: int, c: int, c3: int, cout: int, out: Optional[View] = None, keep=None) -> View:
            if not pair:
                return elan(x, i, c, c3, n3, cout, out=out, keep=keep)
            e1 = elan(x, i, c, c3, n3, cout, keep=keep)
            return elan(x, i + n_elan, c, c3, n3, cout, out=out, keep=keep, res=e1)

        def down(x: View, i: int, cout: int, out: Optional[View] = None) -> View:
            out = out if out is not None else pb.new_padded(x.H // 2, x.W // 2, cout)
            return down_c(x, i, cout, out) if p6["downc"] else cbs(x, f"model.{i}", cout, 3, 2, out=out)

        # model.0 ReOrg + model.1 Conv(12, stem, 3, 1) = one 6x6 stride-2 conv of the image (stem_conv.cu)
        w, b = W.conv_bn("model.1", p6["stem"], 12, 3, eps)
        x = pb.conv(pb.image, reorg_stem_weights(w), b, 6, 2, act_id, pad=2, wide_stem=True)
        bk = tuple(range(1, n3, 2))                          # backbone ELAN: cat[3x3 #n3, .., #4, #2, b, a]
        i, stages = 2, []
        for cout, c in p6["stages"]:
            x = elan_block(down(x, i, cout), i + 1, c, c, cout, keep=bk)
            i += 1 + blk
            stages.append(x)
        o3, o4, o5, o6 = p6["outs"]
        cat_n6 = pb.new_padded(H // 64, Wd // 64, 2 * o6)    # [down(n5), sppcspc]
        cat_n5 = pb.new_padded(H // 32, Wd // 32, 2 * o5)    # [down(n4), h5]
        cat_n4 = pb.new_padded(H // 16, Wd // 16, 2 * o4)    # [down(n3), h4]
        h = sppcspc(x, i, o6, pb.sub(cat_n6, o6, o6))
        i += 1
        # top-down: conv + upsample of the level above, route conv of the backbone level, ELAN (into the bottom-up concat's slice 1)
        hd = p6.get("head", YOLOV7_P6_HEAD)
        for src, (c, c3), cout, cat_n in ((stages[3], hd[0], o5, cat_n5), (stages[2], hd[1], o4, cat_n4), (stages[1], hd[2], o3, None)):
            cat = pb.new_padded(src.H, src.W, 2 * cout)      # [route conv, up(conv)]
            t = cbs(h, f"model.{i}", cout, 1)
            pb.upsample2x(t, pb.sub(cat, cout, cout))
            cbs(src, f"model.{i + 2}", cout, 1, out=pb.sub(cat, 0, cout))
            i += 4
            h = elan_block(cat, i, c, c3, cout, out=pb.sub(cat_n, cout, cout) if cat_n is not None else None)
            i += blk
        # bottom-up: down-sampling into slice 0 of the level's concat, ELAN
        feats = [h]
        for (c, c3), cout, cat_n in ((hd[3], o4, cat_n4), (hd[4], o5, cat_n5), (hd[5], o6, cat_n6)):
            down(feats[-1], i, cout, out=pb.sub(cat_n, 0, cout))
            i += 2
            feats.append(elan_block(cat_n, i, c, c3, cout))
            i += blk
        feats = [cbs(f, f"model.{i + li}", 2 * f.C, 3) for li, f in enumerate(feats)]
        det = i + 4
        assert det == p6["det"], (scale, det)
        det_levels = 4
        if W.real and f"model.{det + 4}.m.0.weight" in W.state_dict and f"model.{det}.m.0.weight" not in W.state_dict:
            det += 4                                         # training form: IAuxDetect after the four aux convs (not used here)
    elif scale == "base":
        x = cbs(pb.image, "model.0", 32, 3, 1, cin=3)
        x = cbs(x, "model.1", 64, 3, 2)
        x = cbs(x, "model.2", 64, 3, 1)
        x = cbs(x, "model.3", 128, 3, 2)
        bk = (1, 3)                                          # backbone ELAN: cat[3x3 #4, 3x3 #2, b, a]
        x = elan(x, 4, 64, 64, 4, 256, keep=bk)                                          # -> 11
        x = elan(mp_block(x, 12, 128, pb.new_padded(H // 8, Wd // 8, 256)), 17, 128, 128, 4, 512, keep=bk)          # 16, -> 24
        p3 = x
        x = elan(mp_block(x, 25, 256, pb.new_padded(H // 16, Wd // 16, 512)), 30, 256, 256, 4, 1024, keep=bk)       # 29, -> 37
        p4 = x
        x = elan(mp_block(x, 38, 512, pb.new_padded(H // 32, Wd // 32, 1024)), 43, 256, 256, 4, 1024, keep=bk)      # 42, -> 50
        cat93 = pb.new_padded(H // 32, Wd // 32, 1024)       # [92, 90, 51]
        cat80 = pb.new_padded(H // 16, Wd // 16, 512)        # [79, 77, 63]
        cat55 = pb.new_padded(H // 16, Wd // 16, 512)        # [54, up(52)]
        cat67 = pb.new_padded(H // 8, Wd // 8, 256)          # [66, up(64)]
        h51 = sppcspc(x, 51, 512, pb.sub(cat93, 512, 512))      # SPPCSPC(1024, 512)
        t = cbs(h51, "model.52", 256, 1)
        pb.upsample2x(t, pb.sub(cat55, 256, 256))
        cbs(p4, "model.54", 256, 1, out=pb.sub(cat55, 0, 256))
        h63 = elan(cat55, 56, 256, 128, 4, 256, out=pb.sub(cat80, 256, 256))
        t = cbs(h63, "model.64", 128, 1)
        pb.upsample2x(t, pb.sub(cat67, 128, 128))
        cbs(p3, "model.66", 128, 1, out=pb.sub(cat67, 0, 128))
        h75 = elan(cat67, 68, 128, 64, 4, 128)
        h88 = elan(mp_block(h75, 76, 128, cat80), 81, 256, 128, 4, 256)
        h101 = elan(mp_block(h88, 89, 256, cat93), 94, 512, 256, 4, 512)
        feats, det = [], 105
        for i, (f, c2) in enumerate(((h75, 256), (h88, 512), (h101, 1024))):
            w, b = W.repconv(f"model.{102 + i}", c2, f.C, eps)
            feats.append(pb.conv(f, w, b, 3, 1, act_id))
    else:
        x = cbs(pb.image, "model.0", 32, 3, 2, cin=3)
        x = cbs(x, "model.1", 64, 3, 2)
        x = elan(x, 2, 32, 32, 2, 64)                                                    # -> 7
        x = elan(pb.maxpool(x, 2, 2, 0), 9, 64, 64, 2, 128)                              # 8, -> 14
        p3 = x
        x = elan(pb.maxpool(x, 2, 2, 0), 16, 128, 128, 2, 256)                           # 15, -> 21
        p4 = x
        x = elan(pb.maxpool(x, 2, 2, 0), 23, 256, 256, 2, 512)                           # 22, -> 28
        cat67 = pb.new_padded(H // 32, Wd // 32, 512)        # [66, 37]
        cat59 = pb.new_padded(H // 16, Wd // 16, 256)        # [58, 47]
        cat36 = pb.new_padded(H // 32, Wd // 32, 512)        # [35, 29]
        cat34 = pb.new_padded(H // 32, Wd // 32, 1024)       # [p13, p9, p5, 30]
        cat41 = pb.new_padded(H // 16, Wd // 16, 256)        # [40, up(38)]
        cat51 = pb.new_padded(H // 8, Wd // 8, 128)          # [50, up(48)]
        cbs(x, "model.29", 256, 1, out=pb.sub(cat36, 256, 256))
        h30 = cbs(x, "model.30", 256, 1, out=pb.sub(cat34, 768, 256))
        pools(h30, cat34, [2, 1, 0])
        cbs(cat34, "model.35", 256, 1, out=pb.sub(cat36, 0, 256))
        h37 = cbs(cat36, "model.37", 256, 1, out=pb.sub(cat67, 256, 256))
        t = cbs(h37, "model.38", 128, 1)
        pb.upsample2x(t, pb.sub(cat41, 128, 128))
        cbs(p4, "model.40", 128, 1, out=pb.sub(cat41, 0, 128))
        h47 = elan(cat41, 42, 64, 64, 2, 128, out=pb.sub(cat59, 128, 128))
        t = cbs(h47, "model.48", 64, 1)
        pb.upsample2x(t, pb.sub(cat51, 64, 64))
        cbs(p3, "model.50", 64, 1, out=pb.sub(cat51, 0, 64))
        h57 = elan(cat51, 52, 32, 32, 2, 64)
        cbs(h57, "model.58", 128, 3, 2, out=pb.sub(cat59, 0, 128))
        h65 = elan(cat59, 60, 64, 64, 2, 128)
        cbs(h65, "model.66", 256, 3, 2, out=pb.sub(cat67, 0, 256))
        h73 = elan(cat67, 68, 128, 128, 2, 256)
        feats = [cbs(f, f"model.{74 + i}", c2, 3) for i, (f, c2) in enumerate(((h57, 128), (h65, 256), (h73, 512)))]
        det = 77
    # IDetect: m[i](ia[i](x)) * im[i], folded into the 1x1 head convolutions
    no = 3 * (nc + 5)
    A = 0
    for li, (feat, stride) in enumerate(zip(feats, (8, 16, 32, 64)[:det_levels])):
        w, b = W.implicit_head(f"model.{det}", li, no, feat.C)
        head = pb.new_padded(feat.H, feat.W, (no + 7) // 8 * 8, f32=True)
        pb.conv(feat, w, b, 1, 1, ACT_NONE, out=head, out_f32=True)
        pb.outputs.append((head.buf, 0, head.C, stride))
        A += 3 * feat.H * feat.W
    if anchors is None:
        anchors = W.anchor_grid(f"model.{det}", det_levels)
    if anchors is None:
        anchors = YOLOV7_P6_ANCHORS if p6 else YOLOV7_ANCHORS if scale == "base" else YOLOV5_ANCHORS
    anc = np.asarray(anchors, np.float32).reshape(6 * det_levels)
    assert np.all(np.isfinite(anc)) and np.all(anc > 0), f"anchors must be finite and positive: {anc}"
    pb.meta[0], pb.meta[1] = nc, A
    pb.meta[3] = pb.tensor(anc) + 1                          # 1 + tensor index; 0 = the YOLOv5 table (plans without the field)
    return pb


def read_anchors(path: str) -> np.ndarray:
    """Anchor table [L levels, 3 anchors, 2] a YOLOv5-layout plan decodes with: its own (header meta[3], L = its output count) or the
    YOLOv5 table (L = 3)."""
    with open(path, "rb") as f:
        raw = f.read()
    h = struct.unpack_from(HDR_FMT, raw)
    n_buf, n_ops, n_t, n_out, meta, blob = h[6], h[7], h[8], h[9], h[10:26], h[26]
    if meta[3] == 0:
        return np.asarray(YOLOV5_ANCHORS, np.float32).reshape(3, 3, 2)
    rec = HDR_SIZE + n_buf * BUF_SIZE + n_ops * OP_SIZE + (meta[3] - 1) * TEN_SIZE
    off, nbytes, _, _ = struct.unpack_from(TEN_FMT, raw, rec)
    assert meta[3] <= n_t and nbytes == 24 * n_out
    return np.frombuffer(raw, np.float32, 6 * n_out, blob + off).reshape(n_out, 3, 2).copy()


# ---------------------------------------------------------------------------------------------
# YOLOv6 3.0 (meituan/YOLOv6 release 0.4.0, configs/yolov6{n,s,m,l}.py; P5 models only)
# ---------------------------------------------------------------------------------------------
YOLOV6_SCALES = {"n": (0.33, 0.25), "s": (0.33, 0.50), "m": (0.60, 0.75), "l": (1.0, 1.0)}     # depth, width
YOLOV6_CSP_E = {"m": 2 / 3, "l": 1 / 2}
YOLOV6_ACTS = {"relu": ACT_RELU, "silu": ACT_SILU}


def yolov6_reg_max(scale: str) -> int:
    """0 for N/S (the head regresses l, t, r, b directly), 16 for M/L (17-bin DFL)."""
    return 16 if scale in ("m", "l") else 0


def build_yolov6(weights: Weights, scale: str = "n", nc: int = 80, in_h: int = 640, in_w: int = 640, act_body: Optional[str] = None,
                 act_neck: str = "relu", act_head: str = "silu", reg_max: Optional[int] = None) -> PlanBuilder:
    """YOLOv6-N/S (EfficientRep + RepBiFPANNeck) or -M/L (CSPBepBackbone + CSPRepBiFPANNeck), EffiDeHead, under upstream module names
    (`backbone.*`, `neck.*`, `detect.*`).  Output [B, 8400, 5 + nc] (MODEL_YOLOV6, header meta[2] = reg_max).

    Activations by conv role (defaults as upstream builds them):
      act_body  stem, backbone / neck blocks, the BepC3 1x1 convs and the SPPF convs: "relu" for N/S/M (RepVGG blocks), "silu" for L
                (training_mode "conv_silu": Conv-BN-SiLU blocks, BepC3 / SPPF in their SiLU form)
      act_neck  the neck's reduce layers, BiFusion cv1 / cv2 / cv3 / downsample and the PAN downsamples (ConvBNReLU upstream): "relu"
      act_head  the head's stem, cls_conv and reg_conv (ConvBNSiLU upstream): "silu"
    RepVGG blocks (3x3 + 1x1 + identity BN) are folded into one 3x3 conv here in fp64 (Weights.repconv); BottleRep's learned `alpha`
    scales the shortcut in the GEMM epilogue; BiFusion's ConvTranspose2d(k=2, s=2) is a 1x1 GEMM storing 2x2 pixel groups.  Each level
    of the head holds 4 * (reg_max + 1) box columns, then the class logits from the next multiple of 8 on (the anchor-aided `_ab`
    branch of training checkpoints is not used at inference and is ignored)."""
    assert scale in YOLOV6_SCALES, f"YOLOv6 scale {scale!r}: 'n', 's', 'm' or 'l' (Lite, P6 and the 2.x models are not supported)"
    depth, width = YOLOV6_SCALES[scale]
    ch = [int(math.ceil(c * width / 8) * 8) for c in (64, 128, 256, 512, 1024, 256, 128, 128, 256, 256, 512)]
    rep = [max(round(n * depth), 1) if n > 1 else n for n in (1, 6, 12, 18, 6, 12, 12, 12, 12)]
    csp = scale in YOLOV6_CSP_E
    repvgg = scale != "l"                                  # L trains Conv-BN-SiLU blocks
    a_body = YOLOV6_ACTS[act_body or ("silu" if scale == "l" else "relu")]
    a_neck, a_head = YOLOV6_ACTS[act_neck], YOLOV6_ACTS[act_head]
    reg_max = yolov6_reg_max(scale) if reg_max is None else reg_max
    assert reg_max in (0, 16)
    pb = PlanBuilder(MODEL_YOLOV6, 3, in_h, in_w)
    W = weights
    eps = BN_EPS_YOLO

    def fused_or_bn(name: str, cout: int, cin: int, k: int, res_branch: bool = False):
        """ConvModule (`name.conv` + `name.bn`) or its deployed form (`name.conv` with a bias)."""
        if W.real and f"{name}.conv.bias" in W.state_dict and f"{name}.bn.weight" not in W.state_dict:
            return W.conv_bias(f"{name}.conv", cout, cin, k)
        return W.conv_bn(name, cout, cin, k, eps, res_branch=res_branch)

    def cin_of(x: View) -> int:
        return 3 if x.buf == pb.image.buf else x.C          # the image buffer carries a zero fourth channel

    def cbr(x: View, name: str, cout: int, k: int, s: int, act: int, out: Optional[View] = None, **kw) -> View:
        """ConvBNReLU / ConvBNSiLU: `name.block.conv`, `name.block.bn`."""
        w, b = fused_or_bn(f"{name}.block", cout, cin_of(x), k, res_branch=kw.get("res") is not None)
        return pb.conv(x, w, b, k, s, act, out=out, **kw)

    def blk(x: View, name: str, cout: int, s: int = 1, out: Optional[View] = None, **kw) -> View:
        """the body block: RepVGGBlock (folded) or, for L, ConvBNSiLU 3x3."""
        if not repvgg:
            return cbr(x, name, cout, 3, s, a_body, out=out, **kw)
        cin = cin_of(x)
        w, b = W.repconv(name, cout, cin, eps, keys=("conv", "bn"), identity=(cin == cout and s == 1))
        return pb.conv(x, w, b, 3, s, a_body, out=out, **kw)

    def rep_block(x: View, name: str, cout: int, n: int, out: Optional[View] = None) -> View:
        """RepBlock of RepVGG blocks: conv1, then block.0 .. block.n-2."""
        names = [f"{name}.conv1"] + [f"{name}.block.{i}" for i in range(n - 1)]
        for i, nm in enumerate(names):
            x = blk(x, nm, cout, out=out if i == len(names) - 1 else None)
        return x

    def bottle_rep(x: View, name: str, out: Optional[View] = None) -> View:
        """BottleRep(c, c, weight=True): conv2(conv1(x)) + alpha * x."""
        t = blk(x, f"{name}.conv1", x.C)
        alpha = float(W.get(f"{name}.alpha", (1,), "alpha")[0])
        if alpha == 0.0:                                    # op f[0] = 0 stands for a scale of 1: a zero alpha drops the shortcut
            return blk(t, f"{name}.conv2", x.C, out=out)
        return blk(t, f"{name}.conv2", x.C, out=out, res=x, res_scale=alpha)

    def bepc3(x: View, name: str, cout: int, n: int, out: Optional[View] = None) -> View:
        """BepC3: cv3(cat(m(cv1(x)), cv2(x))), m = RepBlock of n // 2 BottleReps (at least one)."""
        c_ = int(cout * YOLOV6_CSP_E[scale])
        cat = pb.new_padded(x.H, x.W, 2 * c_)
        y = cbr(x, f"{name}.cv1", c_, 1, 1, a_body)
        names = [f"{name}.m.conv1"] + [f"{name}.m.block.{i}" for i in range(max(n // 2, 1) - 1)]
        for i, nm in enumerate(names):
            y = bottle_rep(y, nm, out=pb.sub(cat, 0, c_) if i == len(names) - 1 else None)
        cbr(x, f"{name}.cv2", c_, 1, 1, a_body, out=pb.sub(cat, c_, c_))
        return cbr(cat, f"{name}.cv3", cout, 1, 1, a_body, out=out)

    stage = (lambda x, name, c, n, out=None: bepc3(x, name, c, n, out)) if csp else rep_block

    def sppf(x: View, name: str, out: Optional[View] = None) -> View:
        """N/S: SimCSPSPPF (`.cspsppf`); M/L: SimSPPF / SPPF (`.sppf`).  The 5x5 pools are chained."""
        c = x.C
        if not csp:
            c_ = c // 2
            cat7 = pb.new_padded(x.H, x.W, 2 * c_)          # cv7 input [y0 = cv2(x), y3]
            sp = pb.new_padded(x.H, x.W, 4 * c_)            # cv5 input [x1, m(x1), m(m(x1)), m(m(m(x1)))]
            nm = f"{name}.cspsppf"
            t = cbr(x, f"{nm}.cv1", c_, 1, 1, a_body)
            t = cbr(t, f"{nm}.cv3", c_, 3, 1, a_body)
            y = cbr(t, f"{nm}.cv4", c_, 1, 1, a_body, out=pb.sub(sp, 0, c_))
            for i in range(3):
                y = pb.maxpool(y, 5, 1, 2, out=pb.sub(sp, (i + 1) * c_, c_))
            cbr(x, f"{nm}.cv2", c_, 1, 1, a_body, out=pb.sub(cat7, 0, c_))
            t = cbr(sp, f"{nm}.cv5", c_, 1, 1, a_body)
            cbr(t, f"{nm}.cv6", c_, 3, 1, a_body, out=pb.sub(cat7, c_, c_))
            return cbr(cat7, f"{nm}.cv7", c, 1, 1, a_body, out=out)
        c_ = c // 2
        sp = pb.new_padded(x.H, x.W, 4 * c_)
        nm = f"{name}.sppf"
        y = cbr(x, f"{nm}.cv1", c_, 1, 1, a_body, out=pb.sub(sp, 0, c_))
        for i in range(3):
            y = pb.maxpool(y, 5, 1, 2, out=pb.sub(sp, (i + 1) * c_, c_))
        return cbr(sp, f"{nm}.cv2", c, 1, 1, a_body, out=out)

    def transpose(x: View, name: str, out: View) -> View:
        c = x.C
        w = W.get(f"{name}.upsample_transpose.weight", (c, c, 2, 2), "conv")
        b = W.get(f"{name}.upsample_transpose.bias", (c,), "bias")
        return pb.conv_transpose2x2(x, w, b, out)

    def bifusion(x0: View, x1: View, x2: View, name: str, c: int) -> View:
        """cv3(cat(Transpose(x0), cv1(x1), downsample(cv2(x2)))) at x1's resolution."""
        cat = pb.new_padded(x1.H, x1.W, 3 * c)
        transpose(x0, f"{name}.upsample", pb.sub(cat, 0, c))
        cbr(x1, f"{name}.cv1", c, 1, 1, a_neck, out=pb.sub(cat, c, c))
        t = cbr(x2, f"{name}.cv2", c, 1, 1, a_neck)
        cbr(t, f"{name}.downsample", c, 3, 2, a_neck, out=pb.sub(cat, 2 * c, c))
        return cbr(cat, f"{name}.cv3", c, 1, 1, a_neck)

    H, Wd = in_h, in_w
    # backbone (stem -> ERBlock_2 .. ERBlock_5); P2 feeds the neck (fuse_P2)
    x = blk(pb.image, "backbone.stem", ch[0], 2)
    feats = []
    for i in range(1, 5):
        x = blk(x, f"backbone.ERBlock_{i + 1}.0", ch[i], 2)
        x = stage(x, f"backbone.ERBlock_{i + 1}.1", ch[i], rep[i])
        feats.append(x)
    p2, p3, p4, _ = feats
    p5 = sppf(x, "backbone.ERBlock_5.2")
    # neck (RepBiFPANNeck / CSPRepBiFPANNeck); PAN concats allocated up front, producers write their slices
    cat_n4 = pb.new_padded(H // 32, Wd // 32, ch[9] + ch[5])      # [down_feat0, fpn_out0]
    cat_n3 = pb.new_padded(H // 16, Wd // 16, ch[7] + ch[6])      # [down_feat1, fpn_out1]
    fpn0 = cbr(p5, "neck.reduce_layer0", ch[5], 1, 1, a_neck, out=pb.sub(cat_n4, ch[9], ch[5]))
    f_out0 = stage(bifusion(fpn0, p4, p3, "neck.Bifusion0", ch[5]), "neck.Rep_p4", ch[5], rep[5])
    fpn1 = cbr(f_out0, "neck.reduce_layer1", ch[6], 1, 1, a_neck, out=pb.sub(cat_n3, ch[7], ch[6]))
    pan2 = stage(bifusion(fpn1, p3, p2, "neck.Bifusion1", ch[6]), "neck.Rep_p3", ch[6], rep[6])
    cbr(pan2, "neck.downsample2", ch[7], 3, 2, a_neck, out=pb.sub(cat_n3, 0, ch[7]))
    pan1 = stage(cat_n3, "neck.Rep_n3", ch[8], rep[7])
    cbr(pan1, "neck.downsample1", ch[9], 3, 2, a_neck, out=pb.sub(cat_n4, 0, ch[9]))
    pan0 = stage(cat_n4, "neck.Rep_n4", ch[10], rep[8])
    # EffiDeHead
    nb = 4 * (reg_max + 1)
    cls_col = (nb + 7) // 8 * 8
    A = 0
    for li, (feat, stride) in enumerate(((pan2, 8), (pan1, 16), (pan0, 32))):
        c = feat.C
        t = cbr(feat, f"detect.stems.{li}", c, 1, 1, a_head)
        # cls_conv and reg_conv share their input: one GEMM with N = 2c, [cls | reg]
        wc, bc = fused_or_bn(f"detect.cls_convs.{li}.block", c, c, 3)
        wr, br = fused_or_bn(f"detect.reg_convs.{li}.block", c, c, 3)
        t2 = pb.conv(t, np.concatenate([wc, wr], 0), np.concatenate([bc, br]), 3, 1, a_head)
        head = pb.new_padded(feat.H, feat.W, cls_col + (nc + 7) // 8 * 8, f32=True)
        wrp, brp = W.conv_bias(f"detect.reg_preds.{li}", nb, c, 1)
        wcp, bcp = W.conv_bias(f"detect.cls_preds.{li}", nc, c, 1)
        pb.conv(pb.sub(t2, c, c), wrp, brp, 1, 1, ACT_NONE, out=pb.sub(head, 0, cls_col), out_f32=True)
        pb.conv(pb.sub(t2, 0, c), wcp, bcp, 1, 1, ACT_NONE, out=pb.sub(head, cls_col, (nc + 7) // 8 * 8), out_f32=True)
        pb.outputs.append((head.buf, 0, head.C, stride))
        A += feat.H * feat.W
    pb.meta[0], pb.meta[1], pb.meta[2] = nc, A, reg_max
    return pb


# ---------------------------------------------------------------------------------------------
# YOLOv6-Lite (meituan/YOLOv6 release 0.4.0, configs/yolov6_lite/yolov6_lite_{s,m,l}.py: Lite_EffiBackbone, Lite_EffiNeck,
# Lite_EffideHead).  Restated from the upstream configs; no upstream file is available here, so the widths are pinned by the published
# parameter counts (tests/test_yolov6_lite_cpu.py).
# ---------------------------------------------------------------------------------------------
YOLOV6_LITE_SCALES = {"s": 0.7, "m": 1.1, "l": 1.5}      # width_multiple
YOLOV6_LITE_BLOCKS = (1, 3, 7, 3)                          # Lite_EffiBlockS2 + (n - 1) x Lite_EffiBlockS1 per stage
YOLOV6_LITE_NECK = 96                                      # unified neck / head width
YOLOV6_LITE_PARAMS = {"s": 0.55e6, "m": 0.79e6, "l": 1.09e6}   # published (README of release 0.4.0)


def _make_divisible_mobile(v: float, d: int) -> int:
    """Upstream `make_divisible` of the Lite models (MobileNet rounding): nearest multiple of d, at least d, and not below 0.9 v."""
    n = max(d, int(v + d / 2) // d * d)
    return n + d if n < 0.9 * v else n


def yolov6_lite_widths(scale: str) -> Tuple[List[int], List[int], List[int]]:
    """(backbone out_channels [stem, stage 1-4], mid_channels [stem slot unused, stage 1-4], neck inputs [P5, P4, P3])."""
    assert scale in YOLOV6_LITE_SCALES, f"YOLOv6-Lite scale {scale!r}: 's', 'm' or 'l'"
    w = YOLOV6_LITE_SCALES[scale]
    out = [_make_divisible_mobile(c * w, 16) for c in (24, 32, 64, 128, 256)]
    mid = [_make_divisible_mobile(int(c * 0.5), 8) for c in out]
    out[0] = 24                                            # the stem is fixed at 24 channels
    neck_in = [_make_divisible_mobile(c * w, 16) for c in (256, 128, 64)]
    return out, mid, neck_in


def _r8(v: View) -> View:
    """The view widened to the 8-channel-aligned width its producer owns (a conv of Cout % 8 != 0 stores zero channels up to it)."""
    return View(v.buf, v.coff, (v.C + 7) // 8 * 8, v.H, v.W)


def build_yolov6_lite(weights: Weights, scale: str = "s", nc: int = 80, in_h: int = 320, in_w: int = 320, se_in_place: bool = True) -> PlanBuilder:
    """YOLOv6-Lite-S/M/L under upstream module names (`backbone.conv_0`, `backbone.lite_effiblock_{1..4}.{j}`, `neck.reduce_layer{0,1,2}`,
    `neck.Csp_{p4,p3,n3,n4}`, `neck.downsample{2,1}`, `neck.p6_conv_{1,2}`, `detect.{stems,cls_convs,reg_convs,cls_preds,reg_preds}.{0..3}`).
    Output [B, A, 5 + nc] (MODEL_YOLOV6, reg_max 0) over four levels, strides 8 / 16 / 32 / 64; level i has ceil(H / s) x ceil(W / s) cells.

    Every activation is Hardswish (ACT_HSWISH).  ConvBNHS / ConvBN (`name.block.conv` + `name.block.bn`) and DPBlock (`conv_dw_1` + `bn_1`,
    `conv_pw_1` + `bn_2`, convs with bias) are folded in fp64; a deployed file carries the fused convs with a bias and no BatchNorm.
    Depthwise convs run in dwconv.cu, SEBlock as OP_SE (in place), the concat + channel shuffle of Lite_EffiBlockS1 as OP_SHUFFLE2; the
    split is a channel slice.  Channel widths that are not multiples of 8 (the S2 blocks' mid / 2 branch) are carried zero-padded.
    se_in_place False: every SE writes a buffer of its own (same results; every op's inputs then survive the run, for per-op checks)."""
    out_c, mid_c, neck_in = yolov6_lite_widths(scale)
    assert in_h % 32 == 0 and in_w % 32 == 0, f"YOLOv6-Lite input {in_h}x{in_w}: a multiple of 32 in each dimension"
    pb = PlanBuilder(MODEL_YOLOV6, 3, in_h, in_w)
    W = weights
    eps = BN_EPS_YOLO
    U = YOLOV6_LITE_NECK
    HS = ACT_HSWISH

    def fold(name: str, conv: str, bn: str, cout: int, cin: int, k: int, conv_bias: bool):
        """conv (+ its bias) then BatchNorm, folded in fp64; the fused form is `conv` with a bias and no `bn`."""
        if W.real and f"{name}.{bn}.weight" not in W.state_dict:
            return W.conv_bias(f"{name}.{conv}", cout, cin, k)
        w = W.get(f"{name}.{conv}.weight", (cout, cin, k, k), "conv").astype(np.float64)
        cb = np.zeros(cout)
        if conv_bias and (not W.real or f"{name}.{conv}.bias" in W.state_dict):
            cb = W.get(f"{name}.{conv}.bias", (cout,), "bias").astype(np.float64)
        g = W.get(f"{name}.{bn}.weight", (cout,), "bn_gamma").astype(np.float64)
        be = W.get(f"{name}.{bn}.bias", (cout,), "bn_beta").astype(np.float64)
        m = W.get(f"{name}.{bn}.running_mean", (cout,), "bn_mean").astype(np.float64)
        v = W.get(f"{name}.{bn}.running_var", (cout,), "bn_var").astype(np.float64)
        if not W.real and f"{name}.{bn}.num_batches_tracked" not in W.state_dict:
            W.state_dict[f"{name}.{bn}.num_batches_tracked"] = np.zeros((), dtype=np.int64)
        sc = g / np.sqrt(v + eps)
        return (w * sc[:, None, None, None]).astype(np.float32), ((cb - m) * sc + be).astype(np.float32)

    def cbn(x: View, name: str, cout: int, k: int, s: int = 1, act: int = HS, dw: bool = False, out: Optional[View] = None,
            cin: Optional[int] = None) -> View:
        """ConvBNHS (act) / ConvBN (act none): `name.block.conv` + `name.block.bn`, no conv bias."""
        cin = cout if dw else (cin if cin is not None else x.C)
        w, b = fold(f"{name}.block", "conv", "bn", cout, 1 if dw else cin, k, False)
        xa = x if x.buf == pb.image.buf else _r8(x)         # the image buffer carries a zero fourth channel
        if dw:
            return pb.dwconv(xa, w, b, k, s, act, out=out)
        return pb.conv(xa, w, b, k, s, act, out=out)

    def dp(x: View, name: str, c: int, k: int = 5, s: int = 1, out: Optional[View] = None, res: Optional[View] = None) -> View:
        """DPBlock: depthwise k x k (stride s) + BN + Hardswish, then 1x1 + BN + Hardswish (+ res after the activation)."""
        wd, bd = fold(name, "conv_dw_1", "bn_1", c, 1, k, True)
        t = pb.dwconv(x, wd, bd, k, s, HS)
        wp, bp = fold(name, "conv_pw_1", "bn_2", c, c, 1, True)
        return pb.conv(t, wp, bp, 1, 1, HS, out=out, res=res)

    def se(x: View, name: str, c: int) -> View:
        hid = c // 4
        w1, b1 = W.conv_bias(f"{name}.conv1", hid, c, 1)
        w2, b2 = W.conv_bias(f"{name}.conv2", c, hid, 1)
        x = _r8(x)
        return pb.se(x, w1, b1, w2, b2, out=None if se_in_place else pb.new_padded(x.H, x.W, x.C))

    def block_s1(x: View, name: str, mid: int, cout: int) -> View:
        h = cout // 2
        t = cbn(pb.sub(x, h, h), f"{name}.conv_pw_1", mid, 1)
        t = cbn(t, f"{name}.conv_dw_1", mid, 3, act=ACT_NONE, dw=True)
        t = se(t, f"{name}.se", mid)
        t = cbn(t, f"{name}.conv_1", h, 1, cin=mid)
        return pb.shuffle2(pb.sub(x, 0, h), t)

    def block_s2(x: View, name: str, cin: int, mid: int, cout: int) -> View:
        h, m2 = cout // 2, mid // 2
        Ho, Wo = (x.H - 1) // 2 + 1, (x.W - 1) // 2 + 1
        cat = pb.new_padded(Ho, Wo, cout)
        t = cbn(x, f"{name}.conv_dw_1", cin, 3, 2, act=ACT_NONE, dw=True)
        cbn(t, f"{name}.conv_1", h, 1, cin=cin, out=pb.sub(cat, 0, h))
        t = cbn(x, f"{name}.conv_pw_2", m2, 1, cin=cin)
        t = cbn(t, f"{name}.conv_dw_2", m2, 3, 2, act=ACT_NONE, dw=True)
        t = se(t, f"{name}.se", m2)
        cbn(t, f"{name}.conv_2", h, 1, cin=m2, out=pb.sub(cat, h, h))
        t = cbn(cat, f"{name}.conv_dw_3", cout, 3, dw=True)
        return cbn(t, f"{name}.conv_pw_3", cout, 1)

    def csp(x: View, name: str, out: Optional[View] = None) -> View:
        """CSPBlock(2U, U, k=5): conv_3(cat(blocks(conv_1(x)), conv_2(x))), blocks = DarknetBlock (1x1 HS, then DPBlock k=5)."""
        m = U // 2
        cat = pb.new_padded(x.H, x.W, 2 * m)
        t = cbn(x, f"{name}.conv_1", m, 1)
        t = cbn(t, f"{name}.blocks.conv_1", m, 1)
        dp(t, f"{name}.blocks.conv_2", m, out=pb.sub(cat, 0, m))
        cbn(x, f"{name}.conv_2", m, 1, out=pb.sub(cat, m, m))
        return cbn(cat, f"{name}.conv_3", U, 1, out=out)

    # backbone
    x = cbn(pb.image, "backbone.conv_0", out_c[0], 3, 2, cin=3)
    feats = []
    for i, n in enumerate(YOLOV6_LITE_BLOCKS):
        nm = f"backbone.lite_effiblock_{i + 1}"
        x = block_s2(x, f"{nm}.0", out_c[i], mid_c[i + 1], out_c[i + 1])
        for j in range(1, n):
            x = block_s1(x, f"{nm}.{j}", mid_c[i + 1], out_c[i + 1])
        if i:
            feats.append(x)
    x2, x1, x0 = feats
    assert (x0.C, x1.C, x2.C) == tuple(neck_in), ((x0.C, x1.C, x2.C), neck_in)
    # neck; the PAN concats are allocated up front and their producers write their slices
    cat_p4 = pb.new_padded(x1.H, x1.W, 2 * U)          # [upsample(fpn_out0), reduce_layer1(x1)]
    cat_p3 = pb.new_padded(x2.H, x2.W, 2 * U)          # [upsample(f_out1), reduce_layer2(x2)]
    cat_n3 = pb.new_padded(x1.H, x1.W, 2 * U)          # [downsample2(pan_out3), f_out1]
    cat_n4 = pb.new_padded(x0.H, x0.W, 2 * U)          # [downsample1(pan_out2), fpn_out0]
    fpn0 = cbn(x0, "neck.reduce_layer0", U, 1, out=pb.sub(cat_n4, U, U))
    pb.upsample2x(fpn0, pb.sub(cat_p4, 0, U))
    cbn(x1, "neck.reduce_layer1", U, 1, out=pb.sub(cat_p4, U, U))
    f_out1 = csp(cat_p4, "neck.Csp_p4", out=pb.sub(cat_n3, U, U))
    pb.upsample2x(f_out1, pb.sub(cat_p3, 0, U))
    cbn(x2, "neck.reduce_layer2", U, 1, out=pb.sub(cat_p3, U, U))
    pan3 = csp(cat_p3, "neck.Csp_p3")
    dp(pan3, "neck.downsample2", U, s=2, out=pb.sub(cat_n3, 0, U))
    pan2 = csp(cat_n3, "neck.Csp_n3")
    dp(pan2, "neck.downsample1", U, s=2, out=pb.sub(cat_n4, 0, U))
    pan1 = csp(cat_n4, "neck.Csp_n4")
    top = dp(fpn0, "neck.p6_conv_1", U, s=2)
    pan0 = dp(pan1, "neck.p6_conv_2", U, s=2, res=top)     # p6_conv_1(fpn_out0) + p6_conv_2(pan_out1), after both activations
    # Lite_EffideHead: reg_max 0, box distances in columns 0-3, class logits from column 8
    cls_col = 8
    A = 0
    for li, (feat, stride) in enumerate(((pan3, 8), (pan2, 16), (pan1, 32), (pan0, 64))):
        assert (feat.H, feat.W) == (-(-in_h // stride), -(-in_w // stride)), (li, feat)
        t = dp(feat, f"detect.stems.{li}", U)
        tc = dp(t, f"detect.cls_convs.{li}", U)
        tr = dp(t, f"detect.reg_convs.{li}", U)
        head = pb.new_padded(feat.H, feat.W, cls_col + (nc + 7) // 8 * 8, f32=True)
        wrp, brp = W.conv_bias(f"detect.reg_preds.{li}", 4, U, 1)
        wcp, bcp = W.conv_bias(f"detect.cls_preds.{li}", nc, U, 1)
        pb.conv(tr, wrp, brp, 1, 1, ACT_NONE, out=pb.sub(head, 0, cls_col), out_f32=True)
        pb.conv(tc, wcp, bcp, 1, 1, ACT_NONE, out=pb.sub(head, cls_col, (nc + 7) // 8 * 8), out_f32=True)
        pb.outputs.append((head.buf, 0, head.C, stride))
        A += feat.H * feat.W
    pb.meta[0], pb.meta[1], pb.meta[2] = nc, A, 0
    return pb


# ---------------------------------------------------------------------------------------------
# YOLOv9 (WongKinYiu/yolov9 release v0.1: the converted / GELAN yolov9-t, -s, -m, -c; P5 models only)
# ---------------------------------------------------------------------------------------------
# Per scale: stem convs (model.0, model.1); model.2 (ELAN1 (c2, c3, c4) for T / S, RepNCSPELAN4 (c2, c3, c4, n) for M / C); the down
# block (AConv or ADown) and output widths of layers 3, 5, 7, 16, 19; RepNCSPELAN4 (c2, c3, c4, n) of layers 4, 6, 8, 12, 15, 18, 21;
# SPPELAN (c2, c3) of layer 9.  The head is DDetect (model.22).  Not checked against any upstream file (none is available here): the
# restatement reproduces the published parameter / FLOP counts (tests/test_yolov9_cpu.py).
YOLOV9 = {
    "t": dict(stem=(16, 32), l2=(32, 32, 16, None), down="aconv", downs=(64, 96, 128, 48, 64), spp=(128, 64),
              r4=((64, 64, 32, 3), (96, 96, 48, 3), (128, 128, 64, 3), (96, 96, 48, 3), (64, 64, 32, 3), (96, 96, 48, 3), (128, 128, 64, 3))),
    "s": dict(stem=(32, 64), l2=(64, 64, 32, None), down="aconv", downs=(128, 192, 256, 96, 128), spp=(256, 128),
              r4=((128, 128, 64, 3), (192, 192, 96, 3), (256, 256, 128, 3), (192, 192, 96, 3), (128, 128, 64, 3), (192, 192, 96, 3),
                  (256, 256, 128, 3))),
    "m": dict(stem=(32, 64), l2=(128, 128, 64, 1), down="aconv", downs=(240, 360, 480, 184, 240), spp=(480, 240),
              r4=((240, 240, 120, 1), (360, 360, 180, 1), (480, 480, 240, 1), (360, 360, 180, 1), (240, 240, 120, 1), (360, 360, 180, 1),
                  (480, 480, 240, 1))),
    "c": dict(stem=(64, 128), l2=(256, 128, 64, 1), down="adown", downs=(256, 512, 512, 256, 512), spp=(512, 256),
              r4=((512, 256, 128, 1), (512, 512, 256, 1), (512, 512, 256, 1), (512, 512, 256, 1), (256, 256, 128, 1), (512, 512, 256, 1),
                  (512, 512, 256, 1))),
}


# YOLOv9-E (GELAN-E, upstream `models/detect/gelan-e.yaml`): two backbones.  model.0 is Silence (the image passes through), so
# model.1 and model.15 both read the image.  `elan`: RepNCSPELAN4 (c2, c3, c4, n) of layers 3, 5, 7, 9 (again as 19, 22, 25, 28 in the
# second backbone); `downs`: ADown widths of layers 4, 6, 8 (20, 23, 26); `cbl`: CBLinear groups of layers 10-14, which read layers 1,
# 3, 5, 7, 9; `spp`: SPPELAN (c2, c3) of layer 29; `head`: RepNCSPELAN4 of layers 32, 35, 38, 41; `head_downs`: ADown widths of layers
# 36, 39.  CBFuse (16, 18, 21, 24, 27) adds group `level` of every CBLinear from layer 10 + level on, nearest-upsampled, to the output
# of layer 15, 17, 20, 23 or 26.  The head is DDetect (model.42) on layers 35, 38, 41.
YOLOV9_E = dict(stem=(64, 128), elan=((256, 128, 64, 2), (512, 256, 128, 2), (1024, 512, 256, 2), (1024, 512, 256, 2)),
                downs=(256, 512, 1024), cbl=((64,), (64, 128), (64, 128, 256), (64, 128, 256, 512), (64, 128, 256, 512, 1024)),
                spp=(512, 256), head=((512, 512, 256, 2), (256, 256, 128, 2), (512, 512, 256, 2), (512, 1024, 512, 2)), head_downs=(256, 512))


def yolov9_conv_count(scale: str) -> int:
    """Convolutions of the fused graph (RepConvN as one conv; the fixed DFL conv not counted).  A training-form file has one more per
    RepConvN (its 1x1 branch): yolov9_repconvn_count(scale)."""
    n_r4 = lambda n: 10 + 4 * n                        # cv1, 2 x (RepNCSP: cv1, cv2, cv3, n x (RepConvN, Conv) + Conv 3x3), cv4
    if scale == "e":                                   # 4 stem convs, 12 ELANs, 8 ADowns, 5 CBLinears, SPPELAN, DDetect
        e = YOLOV9_E
        return 4 + 2 * sum(n_r4(r[3]) for r in e["elan"]) + sum(n_r4(r[3]) for r in e["head"]) + 2 * 8 + len(e["cbl"]) + 2 + 3 * 6
    cfg = YOLOV9[scale]
    l2 = 4 if cfg["l2"][3] is None else n_r4(cfg["l2"][3])
    down = 1 if cfg["down"] == "aconv" else 2
    return 2 + l2 + 5 * down + sum(n_r4(r[3]) for r in cfg["r4"]) + 2 + 3 * 6


def yolov9_repconvn_count(scale: str) -> int:
    if scale == "e":
        return 2 * (2 * sum(r[3] for r in YOLOV9_E["elan"]) + sum(r[3] for r in YOLOV9_E["head"]))
    cfg = YOLOV9[scale]
    return 2 * ((cfg["l2"][3] or 0) + sum(r[3] for r in cfg["r4"]))


class Yolov9Packer:
    """The GELAN blocks of YOLOv9 on a PlanBuilder.  A feature is (stored view, real channel segments ((offset in the view, count), ...)):
    every concat member and chunk starts at a multiple of 8 channels (the GEMM's alignment).  A producer stores round_up(cout, 8)
    channels, zero past cout; consumers' weights are scattered around those zero columns, and the first 1x1 conv of a RepNCSPELAN4 writes
    its two chunks as two aligned row blocks of one GEMM.  Only YOLOv9-M has widths (180, 90, 60) that need it.  flops_per_img counts
    the real channels only."""

    def __init__(self, pb: PlanBuilder, W: Weights, down: str):
        self.pb, self.W, self.down_kind, self.eps = pb, W, down, BN_EPS_YOLO

    @staticmethod
    def r8(c: int) -> int:
        return (c + 7) // 8 * 8

    @staticmethod
    def feat(v: View, c: Optional[int] = None):
        return (v, ((0, v.C if c is None else c),))

    @staticmethod
    def real(x) -> int:
        return sum(n for _, n in x[1])

    def conv(self, x, w: np.ndarray, b: np.ndarray, k: int, s: int = 1, out: Optional[View] = None, res: Optional[View] = None,
             real_cout: Optional[int] = None):
        """w [cout, real input channels, k, k] on x's segments (SiLU); returns the output feature."""
        v, segs = x
        cout = int(w.shape[0])
        cin_real = int(w.shape[1])
        if segs != ((0, v.C),):
            wx = np.zeros((cout, v.C, k, k), np.float32)
            j = 0
            for off, n in segs:
                wx[:, off:off + n] = w[:, j:j + n]
                j += n
            assert j == cin_real, (segs, w.shape)
            w = wx
        f0 = self.pb.flops_per_img
        y = self.pb.conv(v, w, b, k, s, ACT_SILU, out=out, res=res)
        self.pb.flops_per_img = f0 + 2 * y.H * y.W * (real_cout or cout) * cin_real * k * k
        return self.feat(View(y.buf, y.coff, self.r8(cout), y.H, y.W), cout)

    def conv_bn(self, name: str, cout: int, cin: int, k: int, res_branch: bool = False):
        """Conv + BatchNorm, or its upstream-fused form (`conv.weight` + `conv.bias`, no `bn`)."""
        W = self.W
        if W.real and f"{name}.conv.bias" in W.state_dict and f"{name}.bn.weight" not in W.state_dict:
            return W.conv_bias(f"{name}.conv", cout, cin, k)
        return W.conv_bn(name, cout, cin, k, self.eps, res_branch=res_branch)

    def cbs(self, name: str, x, cout: int, k: int, s: int = 1, out: Optional[View] = None, res: Optional[View] = None):
        w, b = self.conv_bn(name, cout, self.real(x), k, res_branch=res is not None)
        return self.conv(x, w, b, k, s, out=out, res=res)

    def rep_ncsp(self, name: str, x, c2: int, n: int, out: Optional[View] = None):
        """RepNCSP: cv3(cat(m(cv1(x)), cv2(x))), m = n x RepNBottleneck (RepConvN 3x3, Conv 3x3, residual add)."""
        pb, r8 = self.pb, self.r8
        c_ = c2 // 2
        cat = pb.new_padded(x[0].H, x[0].W, 2 * r8(c_))
        a = self.cbs(f"{name}.cv1", x, c_, 1)
        for j in range(n):
            w, b = self.W.repconvn(f"{name}.m.{j}.cv1", c_, c_, self.eps)
            t = self.conv(a, w, b, 3)
            a = self.cbs(f"{name}.m.{j}.cv2", t, c_, 3, out=pb.sub(cat, 0, r8(c_)) if j == n - 1 else None, res=a[0])
        self.cbs(f"{name}.cv2", x, c_, 1, out=pb.sub(cat, r8(c_), r8(c_)))
        return self.cbs(f"{name}.cv3", (cat, ((0, c_), (r8(c_), c_))), c2, 1, out=out)

    def elan(self, name: str, x, c2: int, c3: int, c4: int, n: Optional[int], out: Optional[View] = None):
        """RepNCSPELAN4 (n = RepNCSP depth) or ELAN1 (n None): cv4(cat(chunk0, chunk1, cv2(chunk1), cv3(cv2(...))))."""
        pb, r8 = self.pb, self.r8
        h = c3 // 2
        o = (0, r8(h), 2 * r8(h), 2 * r8(h) + r8(c4))
        cat = pb.new_padded(x[0].H, x[0].W, o[3] + r8(c4))
        w, b = self.conv_bn(f"{name}.cv1", c3, self.real(x), 1)
        if r8(h) != h:                                   # the two chunks as aligned row blocks of one GEMM
            wz = np.zeros((2 * r8(h),) + w.shape[1:], np.float32)
            bz = np.zeros(2 * r8(h), np.float32)
            wz[:h], wz[r8(h):r8(h) + h], bz[:h], bz[r8(h):r8(h) + h] = w[:h], w[h:], b[:h], b[h:]
            w, b = wz, bz
        self.conv(x, w, b, 1, out=pb.sub(cat, 0, 2 * r8(h)), real_cout=c3)
        t = (pb.sub(cat, o[1], r8(h)), ((0, h),))
        for i, slot in ((2, o[2]), (3, o[3])):
            if n is None:
                t = self.cbs(f"{name}.cv{i}", t, c4, 3, out=pb.sub(cat, slot, r8(c4)))
            else:
                t = self.rep_ncsp(f"{name}.cv{i}.0", t, c4, n)
                t = self.cbs(f"{name}.cv{i}.1", t, c4, 3, out=pb.sub(cat, slot, r8(c4)))
        return self.cbs(f"{name}.cv4", (cat, ((0, h), (o[1], h), (o[2], c4), (o[3], c4))), c2, 1, out=out)

    def down(self, name: str, x, c2: int, out: Optional[View] = None):
        """AConv: cv1 (3x3 s2) of the 2x2 stride-1 average pool.  ADown: the pool's first half through cv1 (3x3 s2), its second half
        through a 3x3 stride-2 max pool and cv2 (1x1), concatenated.  The pool is stored on the input's even H x W grid with a zero
        (AConv, ADown's first half) or -inf (ADown's second half) last row and column (PlanBuilder.avgpool2)."""
        pb = self.pb
        v = x[0]
        out = out if out is not None else pb.new_padded(v.H // 2, v.W // 2, self.r8(c2))
        if self.down_kind == "aconv":
            return self.cbs(f"{name}.cv1", (pb.avgpool2(v, 0), x[1]), c2, 3, 2, out=out)
        half, c = self.real(x) // 2, c2 // 2
        assert x[1] == ((0, v.C),) and half % 8 == 0 and c % 8 == 0, (name, x[1], c2)
        p = pb.new_padded(v.H, v.W, v.C)
        pb.avgpool2(pb.sub(v, 0, half), 0, out=pb.sub(p, 0, half))
        pb.avgpool2(pb.sub(v, half, half), 1, out=pb.sub(p, half, half))
        self.cbs(f"{name}.cv1", self.feat(pb.sub(p, 0, half)), c, 3, 2, out=pb.sub(out, 0, c))
        self.cbs(f"{name}.cv2", self.feat(pb.maxpool(pb.sub(p, half, half), 3, 2, 1)), c, 1, out=pb.sub(out, c, c))
        return self.feat(View(out.buf, out.coff, c2, out.H, out.W))

    def sppelan(self, name: str, x, c2: int, c3: int, out: Optional[View] = None):
        """SPPELAN: cv5(cat(y, p(y), p(p(y)), p(p(p(y))))), y = cv1(x), p = 5x5 stride-1 max pool."""
        pb, r8 = self.pb, self.r8
        sp = pb.new_padded(x[0].H, x[0].W, 4 * r8(c3))
        y = self.cbs(f"{name}.cv1", x, c3, 1, out=pb.sub(sp, 0, r8(c3)))[0]
        for i in range(1, 4):
            y = pb.maxpool(y, 5, 1, 2, out=pb.sub(sp, i * r8(c3), r8(c3)))
        return self.cbs(f"{name}.cv5", (sp, tuple((i * r8(c3), c3) for i in range(4))), c2, 1, out=out)


def build_yolov9(weights: Weights, scale: str = "c", nc: int = 80, in_h: int = 640, in_w: int = 640) -> PlanBuilder:
    """YOLOv9-T / S / M / C (GELAN graphs, upstream `model.<i>` names; Conv = Conv2d + BatchNorm + SiLU) with the DDetect head (model.22).
    The output and its decode are YOLOv8's ([B, 4 + nc, A], MODEL_YOLOV8 kind).  Inputs are multiples of 32.

    RepConvN is folded here in fp64 (training-form `conv1` / `conv2` keys) or taken fused (`conv.weight` + `conv.bias`); a Conv fused
    upstream (`conv.bias`, no `bn`) is taken as it is.  ADown / AConv's 2x2 stride-1 average pool runs as OP_AVGPOOL2 on the input's grid,
    so their stride-2 convs see even maps.  DDetect's grouped box convs pack as dense block-diagonal weights.  Channel layout: Yolov9Packer.
    YOLOv9-E: build_yolov9e."""
    assert scale in YOLOV9 or scale == "e", f"YOLOv9 scale {scale!r}: 't', 's', 'm', 'c' or 'e'"
    assert in_h % 32 == 0 and in_w % 32 == 0, f"YOLOv9 input {in_h}x{in_w}: a multiple of 32"
    if scale == "e":
        return build_yolov9e(weights, nc, in_h, in_w)
    cfg = YOLOV9[scale]
    pb = PlanBuilder(MODEL_YOLOV8, 3, in_h, in_w)
    g = Yolov9Packer(pb, weights, cfg["down"])
    H, Wd = in_h, in_w
    d, r, (s2, s3) = cfg["downs"], cfg["r4"], cfg["spp"]
    assert all(c % 8 == 0 for c in d + (s2,) + tuple(x[0] for x in r)), scale     # the head's concat members are aligned as they are
    cat11 = pb.new_padded(H // 16, Wd // 16, s2 + r[1][0])     # [up(9), 6]
    cat14 = pb.new_padded(H // 8, Wd // 8, r[3][0] + r[0][0])  # [up(12), 4]
    cat17 = pb.new_padded(H // 16, Wd // 16, d[3] + r[3][0])   # [16, 12]
    cat20 = pb.new_padded(H // 32, Wd // 32, d[4] + s2)        # [19, 9]

    x = g.cbs("model.0", (pb.image, ((0, 3),)), cfg["stem"][0], 3, 2)
    x = g.cbs("model.1", x, cfg["stem"][1], 3, 2)
    x = g.elan("model.2", x, *cfg["l2"])
    x = g.down("model.3", x, d[0])
    p3 = g.elan("model.4", x, *r[0], out=pb.sub(cat14, r[3][0], r[0][0]))
    x = g.down("model.5", p3, d[1])
    p4 = g.elan("model.6", x, *r[1], out=pb.sub(cat11, s2, r[1][0]))
    x = g.down("model.7", p4, d[2])
    x = g.elan("model.8", x, *r[2])
    p5 = g.sppelan("model.9", x, s2, s3, out=pb.sub(cat20, d[4], s2))
    pb.upsample2x(p5[0], pb.sub(cat11, 0, s2))
    h12 = g.elan("model.12", g.feat(cat11), *r[3], out=pb.sub(cat17, d[3], r[3][0]))
    pb.upsample2x(h12[0], pb.sub(cat14, 0, r[3][0]))
    h15 = g.elan("model.15", g.feat(cat14), *r[4])
    g.down("model.16", h15, d[3], out=pb.sub(cat17, 0, d[3]))
    h18 = g.elan("model.18", g.feat(cat17), *r[5])
    g.down("model.19", h18, d[4], out=pb.sub(cat20, 0, d[4]))
    h21 = g.elan("model.21", g.feat(cat20), *r[6])
    A = v8_detect(pb, weights, "model.22", (h15[0], h18[0], h21[0]), nc, box_groups=4, conv_bn=g.conv_bn)
    pb.meta[0], pb.meta[1] = nc, A
    return pb


def build_yolov9e(weights: Weights, nc: int = 80, in_h: int = 640, in_w: int = 640, cbfuse_in_place: bool = True) -> PlanBuilder:
    """YOLOv9-E (GELAN-E, YOLOV9_E), ops emitted and weights requested in upstream's execution order (1-9, 10-14, 15, ...), so files
    whose names were lost are consumed in graph order.  Each CBLinear (`model.{10..14}.conv`, biased 1x1, no BN, no activation) is one
    GEMM writing all its groups into one buffer; each CBFuse is one OP_CBFUSE on the slice that conv 15 / 17 or ADown 20 / 23 / 26 has
    just written (cbfuse_in_place False: into a buffer of its own, so that every op's inputs survive the run).  The two image convs
    run in stem_conv.cu.  Inputs are multiples of 32, so every source's nearest-upsampling factor is an exact power of two."""
    assert in_h % 32 == 0 and in_w % 32 == 0, f"YOLOv9 input {in_h}x{in_w}: a multiple of 32"
    cfg = YOLOV9_E
    pb = PlanBuilder(MODEL_YOLOV8, 3, in_h, in_w)
    g = Yolov9Packer(pb, weights, "adown")
    H, Wd = in_h, in_w
    el, (h32, h35, h38, h41), (s2, s3), (d36, d39) = cfg["elan"], cfg["head"], cfg["spp"], cfg["head_downs"]
    cat31 = pb.new_padded(H // 16, Wd // 16, s2 + el[2][0])     # [up(29), 25]
    cat34 = pb.new_padded(H // 8, Wd // 8, h32[0] + el[1][0])   # [up(32), 22]
    cat37 = pb.new_padded(H // 16, Wd // 16, d36 + h32[0])      # [36, 32]
    cat40 = pb.new_padded(H // 32, Wd // 32, d39 + s2)          # [39, 29]
    image = (pb.image, ((0, 3),))

    # first backbone (1-9) and the CBLinear projections of layers 1, 3, 5, 7, 9 (10-14)
    x1 = g.cbs("model.1", image, cfg["stem"][0], 3, 2)
    x3 = g.elan("model.3", g.cbs("model.2", x1, cfg["stem"][1], 3, 2), *el[0])
    x5 = g.elan("model.5", g.down("model.4", x3, cfg["downs"][0]), *el[1])
    x7 = g.elan("model.7", g.down("model.6", x5, cfg["downs"][1]), *el[2])
    x9 = g.elan("model.9", g.down("model.8", x7, cfg["downs"][2]), *el[3])
    lin = []
    for i, (x, groups) in enumerate(zip((x1, x3, x5, x7, x9), cfg["cbl"])):
        assert all(c % 8 == 0 for c in groups) and x[1] == ((0, x[0].C),)
        w, b = weights.conv_bias(f"model.{10 + i}.conv", sum(groups), x[0].C, 1)
        lin.append(pb.conv(x[0], w, b, 1, 1, ACT_NONE))

    def cbfuse(y, level):
        """CBFuse of level `level` (output stride 2 << level): group `level` of CBLinear 10 + k, k >= level, upsampled by 2^(k - level)."""
        w = cfg["cbl"][level][level]
        srcs = [(pb.sub(lin[k], sum(cfg["cbl"][k][:level]), w), k - level) for k in range(level, len(lin))]
        v = y[0]
        assert y[1] == ((0, v.C),) and v.C == w, (y, w)
        return g.feat(pb.cbfuse(v, srcs, out=None if cbfuse_in_place else pb.new_padded(v.H, v.W, v.C)))

    # second backbone (15-28): its five stages each fused with the CBLinear groups of their resolution
    y = cbfuse(g.cbs("model.15", image, cfg["stem"][0], 3, 2), 0)                 # 16
    y = cbfuse(g.cbs("model.17", y, cfg["stem"][1], 3, 2), 1)                     # 18
    y = cbfuse(g.down("model.20", g.elan("model.19", y, *el[0]), cfg["downs"][0]), 2)       # 21
    y22 = g.elan("model.22", y, *el[1], out=pb.sub(cat34, h32[0], el[1][0]))
    y = cbfuse(g.down("model.23", y22, cfg["downs"][1]), 3)                       # 24
    y25 = g.elan("model.25", y, *el[2], out=pb.sub(cat31, s2, el[2][0]))
    y = cbfuse(g.down("model.26", y25, cfg["downs"][2]), 4)                       # 27
    y28 = g.elan("model.28", y, *el[3])

    # head (29-41)
    p29 = g.sppelan("model.29", y28, s2, s3, out=pb.sub(cat40, d39, s2))
    pb.upsample2x(p29[0], pb.sub(cat31, 0, s2))                                   # 30, 31
    p32 = g.elan("model.32", g.feat(cat31), *h32, out=pb.sub(cat37, d36, h32[0]))
    pb.upsample2x(p32[0], pb.sub(cat34, 0, h32[0]))                               # 33, 34
    p35 = g.elan("model.35", g.feat(cat34), *h35)
    g.down("model.36", p35, d36, out=pb.sub(cat37, 0, d36))                       # 36, 37
    p38 = g.elan("model.38", g.feat(cat37), *h38)
    g.down("model.39", p38, d39, out=pb.sub(cat40, 0, d39))                       # 39, 40
    p41 = g.elan("model.41", g.feat(cat40), *h41)
    A = v8_detect(pb, weights, "model.42", (p35[0], p38[0], p41[0]), nc, box_groups=4, conv_bn=g.conv_bn)
    pb.meta[0], pb.meta[1] = nc, A
    return pb


# ---------------------------------------------------------------------------------------------
# YOLOv10 (ultralytics 8.2.41 `yolov10{n,s,m,b,l,x}.yaml`; the one-to-one head)
# ---------------------------------------------------------------------------------------------
# depth, width, max_channels; the C2f layers that are C2fCIB, mapped to lk (the 7x7 RepVGGDW in the CIB's middle conv)
YOLOV10_SCALES = {"n": (0.33, 0.25, 1024), "s": (0.33, 0.50, 1024), "m": (0.67, 0.75, 768), "b": (0.67, 1.00, 512),
                  "l": (1.00, 1.00, 512), "x": (1.00, 1.25, 512)}
YOLOV10_CIB = {"n": {22: True}, "s": {8: True, 22: True}, "m": {8: False, 19: False, 22: False},
               "b": {8: False, 13: False, 19: False, 22: False}, "l": {8: False, 13: False, 19: False, 22: False},
               "x": {6: False, 8: False, 13: False, 19: False, 22: False}}


def yolov10_conv_count(scale: str) -> int:
    """Convolutions of the fused one-to-one graph (RepVGGDW as one conv; the fixed DFL conv not counted): stem and layers 1, 3, 17;
    three SCDowns; SPPF; PSA (cv1, qkv, pe, proj, two ffn convs, cv2); the C2f / C2fCIB layers (cv1, cv2 and 2 convs per Bottleneck,
    5 per CIB); the head (3 box and 5 class convs per level).  A training-form file has one more per RepVGGDW
    (yolov10_repvggdw_count), one with the one-to-many head 24 more."""
    depth = YOLOV10_SCALES[scale][0]
    cibs = YOLOV10_CIB[scale]
    reps = {2: 3, 4: 6, 6: 6, 8: 3, 13: 3, 16: 3, 19: 3, 22: 3}
    c2f = sum(2 + _v8_n(n, depth) * (5 if li in cibs else 2) for li, n in reps.items())
    return 4 + 3 * 2 + 2 + 7 + c2f + 3 * 8


def yolov10_repvggdw_count(scale: str) -> int:
    depth = YOLOV10_SCALES[scale][0]
    return sum(_v8_n(3, depth) for lk in YOLOV10_CIB[scale].values() if lk)     # every C2fCIB layer repeats 3 (x depth) blocks


def yolov10_attention_dims(c: int) -> Tuple[int, int, int, int]:
    """PSA Attention(dim = c): (heads, key dim, head dim, key dim padded to 16) -- nh = c // 64, hd = c // nh, kd = hd // 2."""
    nh = c // 64
    hd = c // nh
    kd = hd // 2
    return nh, kd, hd, (kd + 15) // 16 * 16


class Yolov10Packer:
    """The YOLOv10 blocks on a PlanBuilder.  Conv = Conv2d + BatchNorm (eps 1e-3) folded in fp64, or a Conv fused upstream (`conv.bias`,
    no `bn`) taken as it is.  Depthwise convs run as OP_DWCONV, PSA's attention as OP_ATTN; everything else is the GEMM."""

    def __init__(self, pb: PlanBuilder, W: Weights):
        self.pb, self.W = pb, W

    def conv_bn(self, name: str, cout: int, cin: int, k: int, res_branch: bool = False):
        W = self.W
        if W.real and f"{name}.conv.bias" in W.state_dict and f"{name}.bn.weight" not in W.state_dict:
            return W.conv_bias(f"{name}.conv", cout, cin, k)
        return W.conv_bn(name, cout, cin, k, BN_EPS_YOLO, res_branch=res_branch)

    def cbs(self, x: View, name: str, cout: int, k: int, s: int = 1, act: int = ACT_SILU, out: Optional[View] = None,
            res: Optional[View] = None, cin: Optional[int] = None) -> View:
        w, b = self.conv_bn(name, cout, cin if cin is not None else x.C, k, res_branch=res is not None)
        return self.pb.conv(x, w, b, k, s, act, out=out, res=res)

    def dw(self, x: View, name: str, c: int, k: int, s: int = 1, act: int = ACT_SILU, out: Optional[View] = None,
           res: Optional[View] = None) -> View:
        w, b = self.conv_bn(name, c, 1, k, res_branch=res is not None)
        return self.pb.dwconv(x, w, b, k, s, act, out=out, res=res)

    def repvggdw(self, x: View, name: str, c: int) -> View:
        """RepVGGDW as one folded depthwise 7x7 with SiLU (Weights.repvggdw)."""
        w, b = self.W.repvggdw(name, c, BN_EPS_YOLO)
        return self.pb.dwconv(x, w, b, 7, 1, ACT_SILU)

    def scdown(self, x: View, name: str, c2: int, out: Optional[View] = None) -> View:
        """SCDown: 1x1 Conv (c1 -> c2), then a 3x3 stride-2 depthwise Conv without activation."""
        t = self.cbs(x, f"{name}.cv1", c2, 1)
        return self.dw(t, f"{name}.cv2", c2, 3, 2, act=ACT_NONE, out=out)

    def cib(self, x: View, name: str, c: int, shortcut: bool, lk: bool, out: Optional[View] = None) -> View:
        """CIB(c, c, e=1): x (+) [dw3x3, 1x1 c->2c, (RepVGGDW 7x7 | dw3x3), 1x1 2c->c, dw3x3], every conv SiLU."""
        t = self.dw(x, f"{name}.cv1.0", c, 3)
        t = self.cbs(t, f"{name}.cv1.1", 2 * c, 1)
        t = self.repvggdw(t, f"{name}.cv1.2", 2 * c) if lk else self.dw(t, f"{name}.cv1.2", 2 * c, 3)
        t = self.cbs(t, f"{name}.cv1.3", c, 1)
        return self.dw(t, f"{name}.cv1.4", c, 3, out=out, res=x if shortcut else None)

    def c2f(self, x: View, name: str, c2: int, n: int, shortcut: bool, cib: Optional[bool] = None, out: Optional[View] = None) -> View:
        """C2f (cib None) or C2fCIB (cib = lk): cv2(cat(chunk0, chunk1, m0(chunk1), m1(m0(...)), ...))."""
        pb = self.pb
        c = c2 // 2
        cat = pb.new_padded(x.H, x.W, (2 + n) * c)
        self.cbs(x, f"{name}.cv1", 2 * c, 1, out=pb.sub(cat, 0, 2 * c))
        for i in range(n):
            src, dst = pb.sub(cat, (1 + i) * c, c), pb.sub(cat, (2 + i) * c, c)
            if cib is None:
                t = self.cbs(src, f"{name}.m.{i}.cv1", c, 3)
                self.cbs(t, f"{name}.m.{i}.cv2", c, 3, out=dst, res=src if shortcut else None)
            else:
                self.cib(src, f"{name}.m.{i}", c, shortcut, cib, out=dst)
        return self.cbs(cat, f"{name}.cv2", c2, 1, out=out)

    def psa(self, x: View, name: str, out: Optional[View] = None) -> View:
        """PSA(c1): a, b = cv1(x).split(c); b += attn(b); b += ffn(b); cv2(cat(a, b)).  attn(b) = proj(attention(q, k, v) + pe(v)):
        the qkv conv's rows are permuted from upstream's per-head [q kd | k kd | v hd] into [Q all heads | K all heads | V all heads],
        each q / k padded to kdp rows with zero weights and biases; V then is the c-channel tensor upstream's pe conv reads."""
        pb, c1 = self.pb, x.C
        c = c1 // 2
        nh, kd, hd, kdp = yolov10_attention_dims(c)
        ab = pb.new_padded(x.H, x.W, 2 * c)
        self.cbs(x, f"{name}.cv1", 2 * c, 1, out=ab)
        b = pb.sub(ab, c, c)
        w, bias = self.conv_bn(f"{name}.attn.qkv", c + 2 * nh * kd, c, 1)
        wq, bq = qkv_permute(w, bias, nh, kd, hd)
        f0 = pb.flops_per_img
        qkv = pb.conv(b, wq, bq, 1, 1, ACT_NONE)
        pb.flops_per_img = f0 + 2 * x.H * x.W * (c + 2 * nh * kd) * c           # the kdp - kd zero rows are not counted
        att = pb.attention(qkv, nh, kdp, hd, float(kd) ** -0.5)
        u = self.dw(pb.sub(qkv, 2 * nh * kdp, c), f"{name}.attn.pe", c, 3, act=ACT_NONE, res=att)
        b2 = self.cbs(u, f"{name}.attn.proj", c, 1, act=ACT_NONE, res=b)
        f = self.cbs(b2, f"{name}.ffn.0", 2 * c, 1)
        self.cbs(f, f"{name}.ffn.1", c, 1, act=ACT_NONE, out=b, res=b2)
        return self.cbs(ab, f"{name}.cv2", c1, 1, out=out)


def qkv_permute(w: np.ndarray, b: np.ndarray, nh: int, kd: int, hd: int) -> Tuple[np.ndarray, np.ndarray]:
    """Rows of PSA's qkv conv from upstream's per-head [q kd | k kd | v hd] order into [Q | K | V], all heads each, q / k padded to
    kdp = round_up(kd, 16) rows per head with zero weights and biases (zeros change no q . k product)."""
    kdp = (kd + 15) // 16 * 16
    per = 2 * kd + hd
    assert w.shape[0] == nh * per, (w.shape, nh, kd, hd)
    wo = np.zeros((nh * (2 * kdp + hd),) + w.shape[1:], np.float32)
    bo = np.zeros(nh * (2 * kdp + hd), np.float32)
    for h in range(nh):
        src = h * per
        for part, (s0, n, d0) in enumerate(((0, kd, h * kdp), (kd, kd, nh * kdp + h * kdp), (2 * kd, hd, 2 * nh * kdp + h * hd))):
            wo[d0:d0 + n] = w[src + s0:src + s0 + n]
            bo[d0:d0 + n] = b[src + s0:src + s0 + n]
    return wo, bo


def v10_detect(pb: PlanBuilder, g: Yolov10Packer, name: str, feats, nc: int) -> int:
    """YOLOv10 v10Detect, the one-to-one branch (`one2one_cv2` / `one2one_cv3`) on the P3 / P4 / P5 views; returns the anchor count.
    Writes YOLOv8's f32 head buffers and outputs ([64 DFL logits | nc class logits] per pixel), so the kind-0 decode reads them.  The box
    branch is YOLOv8's; the class branch is [dw3x3, 1x1 -> c3], [dw3x3, 1x1 c3 -> c3], 1x1 -> nc, c3 = max(ch0, min(nc, 100))."""
    reg_max = 16
    cb = max(16, feats[0].C // 4, reg_max * 4)
    c3 = max(feats[0].C, min(nc, 100))
    A = 0
    for li, (feat, stride) in enumerate(zip(feats, (8, 16, 32))):
        cin = feat.C
        b2, b3 = f"{name}.one2one_cv2.{li}", f"{name}.one2one_cv3.{li}"
        head = pb.new_padded(feat.H, feat.W, 4 * reg_max + (nc + 7) // 8 * 8, f32=True)
        tb = g.cbs(g.cbs(feat, f"{b2}.0", cb, 3), f"{b2}.1", cb, 3)
        wbx, bbx = g.W.conv_bias(f"{b2}.2", 4 * reg_max, cb, 1)
        pb.conv(tb, wbx, bbx, 1, 1, ACT_NONE, out=pb.sub(head, 0, 4 * reg_max), out_f32=True)
        r8 = lambda v: View(v.buf, v.coff, (v.C + 7) // 8 * 8, v.H, v.W)     # c3 may not be a multiple of 8: zero channels follow
        t = r8(g.cbs(g.dw(feat, f"{b3}.0.0", cin, 3), f"{b3}.0.1", c3, 1))
        t = r8(g.cbs(g.dw(t, f"{b3}.1.0", c3, 3), f"{b3}.1.1", c3, 1, cin=c3))
        wcl, bcl = g.W.conv_bias(f"{b3}.2", nc, c3, 1)
        pb.conv(t, wcl, bcl, 1, 1, ACT_NONE, out=pb.sub(head, 4 * reg_max, (nc + 7) // 8 * 8), out_f32=True)
        pb.outputs.append((head.buf, 0, head.C, stride))
        A += feat.H * feat.W
    return A


def build_yolov10(weights: Weights, scale: str = "n", nc: int = 80, in_h: int = 640, in_w: int = 640) -> PlanBuilder:
    """YOLOv10-N / S / M / B / L / X (upstream `model.<i>` names, head `model.23`) with the one-to-one head; the one-to-many head's
    keys are never read.  The output and its decode are YOLOv8's ([B, 4 + nc, A], MODEL_YOLOV8 kind), not upstream's top-k tail.
    Inputs are multiples of 32."""
    assert scale in YOLOV10_SCALES, f"YOLOv10 scale {scale!r}: one of {sorted(YOLOV10_SCALES)}"
    assert in_h % 32 == 0 and in_w % 32 == 0, f"YOLOv10 input {in_h}x{in_w}: a multiple of 32"
    depth, width, max_ch = YOLOV10_SCALES[scale]
    cibs = YOLOV10_CIB[scale]
    ch = lambda c: _v8_ch(c, width, max_ch)
    rep = lambda n: _v8_n(n, depth)
    pb = PlanBuilder(MODEL_YOLOV8, 3, in_h, in_w)
    g = Yolov10Packer(pb, weights)

    def c2f(x, li, c2, n, shortcut, out=None):
        return g.c2f(x, f"model.{li}", c2, n, shortcut or li in cibs, cibs.get(li), out=out)

    c1, c2_, c3, c4, c5 = ch(64), ch(128), ch(256), ch(512), ch(1024)
    H, Wd = in_h, in_w
    cat12 = pb.new_padded(H // 16, Wd // 16, c5 + c4)      # [up(10), 6]
    cat15 = pb.new_padded(H // 8, Wd // 8, c4 + c3)        # [up(13), 4]
    cat18 = pb.new_padded(H // 16, Wd // 16, c3 + c4)      # [17, 13]
    cat21 = pb.new_padded(H // 32, Wd // 32, c4 + c5)      # [20, 10]

    x = g.cbs(pb.image, "model.0", c1, 3, 2, cin=3)
    x = g.cbs(x, "model.1", c2_, 3, 2)
    x = c2f(x, 2, c2_, rep(3), True)
    x = g.cbs(x, "model.3", c3, 3, 2)
    p3 = c2f(x, 4, c3, rep(6), True, out=pb.sub(cat15, c4, c3))
    x = g.scdown(p3, "model.5", c4)
    p4 = c2f(x, 6, c4, rep(6), True, out=pb.sub(cat12, c5, c4))
    x = g.scdown(p4, "model.7", c5)
    x = c2f(x, 8, c5, rep(3), True)
    ch_ = c5 // 2                                           # SPPF
    sp = pb.new_padded(x.H, x.W, 4 * ch_)
    y = g.cbs(x, "model.9.cv1", ch_, 1, out=pb.sub(sp, 0, ch_))
    for i in range(3):
        y = pb.maxpool(y, 5, 1, 2, out=pb.sub(sp, (i + 1) * ch_, ch_))
    x = g.cbs(sp, "model.9.cv2", c5, 1)
    p5 = g.psa(x, "model.10", out=pb.sub(cat21, c4, c5))
    pb.upsample2x(p5, pb.sub(cat12, 0, c5))
    h13 = c2f(cat12, 13, c4, rep(3), False, out=pb.sub(cat18, c3, c4))
    pb.upsample2x(h13, pb.sub(cat15, 0, c4))
    h16 = c2f(cat15, 16, c3, rep(3), False)
    g.cbs(h16, "model.17", c3, 3, 2, out=pb.sub(cat18, 0, c3))
    h19 = c2f(cat18, 19, c4, rep(3), False)
    g.scdown(h19, "model.20", c4, out=pb.sub(cat21, 0, c4))
    h22 = c2f(cat21, 22, c5, rep(3), False)
    A = v10_detect(pb, g, "model.23", (h16, h19, h22), nc)
    pb.meta[0], pb.meta[1] = nc, A
    return pb


# ---------------------------------------------------------------------------------------------
# UFLDv2 (model_culane.parsingNet, backbone.resnet 18/34)
# ---------------------------------------------------------------------------------------------
# dataset geometries: ModelConfig (ultrafastLaneDetectorV2.py:31-55) + exportLib/ultrafastLaneV2/configs/{culane,tusimple}_res*.py
# (`dataset` is the id stored in the plan header, meta[6]; the engine derives crop ratio and anchors from it)
UFLD_CULANE = dict(num_grid_row=200, num_cls_row=72, num_grid_col=100, num_cls_col=81, num_lanes=4, in_h=320, in_w=1600, fc_norm=True,
                   dataset=0, crop_ratio=0.6)
UFLD_TUSIMPLE = dict(num_grid_row=100, num_cls_row=56, num_grid_col=100, num_cls_col=41, num_lanes=4, in_h=320, in_w=800, fc_norm=False,
                     dataset=1, crop_ratio=0.8)
UFLD_DATASETS = {"culane": UFLD_CULANE, "tusimple": UFLD_TUSIMPLE}
# UFLD v1 (ultrafastLaneDetector.py:15-37 ModelConfig; exportLib/ultrafastLane/model.py): 288x800 input, one output tensor
UFLD_V1_TUSIMPLE = dict(v1=True, griding_num=100, cls_num_per_lane=56, num_lanes=4, in_h=288, in_w=800, fc_norm=False, dataset=1, crop_ratio=1.0)
UFLD_V1_CULANE = dict(v1=True, griding_num=200, cls_num_per_lane=18, num_lanes=4, in_h=288, in_w=800, fc_norm=False, dataset=0, crop_ratio=1.0)
UFLD_V1_DATASETS = {"culane": UFLD_V1_CULANE, "tusimple": UFLD_V1_TUSIMPLE}
BN_EPS_TV = 1e-5
UFLD_STEM_DEFAULT = "pack"


def build_ufldv1(weights: Weights, backbone: str = "18", cfg="tusimple") -> PlanBuilder:
    """UFLD v1: the same ResNet trunk, pool conv and two FC layers as v2 without LayerNorm; head = [griding_num + 1, rows, 4]."""
    return build_ufldv2(weights, backbone, UFLD_V1_DATASETS[cfg] if isinstance(cfg, str) else cfg)


def build_ufldv2(weights: Weights, backbone: str = "34", cfg=UFLD_CULANE) -> PlanBuilder:
    if isinstance(cfg, str):
        cfg = UFLD_DATASETS[cfg]
    blocks = {"18": [2, 2, 2, 2], "34": [3, 4, 6, 3]}[backbone]
    in_h, in_w = cfg["in_h"], cfg["in_w"]
    v1 = bool(cfg.get("v1"))
    pb = PlanBuilder(MODEL_UFLDV1 if v1 else MODEL_UFLDV2, 3, in_h, in_w)
    W = weights
    w, b = W.conv_bn("model", 64, 3, 7, BN_EPS_TV, conv_key="conv1", bn_key="bn1")
    # stem: "pack" = re-layout pass + a 4-tap wgmma GEMM (stem7x7s2), "direct" = stem_conv.cu straight from the image
    if os.environ.get("ADAS_B200_UFLD_STEM", UFLD_STEM_DEFAULT) == "pack":
        x = pb.stem7x7s2(pb.image, w, b, ACT_RELU)
    else:
        x = pb.conv(pb.image, w, b, 7, 2, ACT_RELU, pad=3)
    x = pb.maxpool(x, 3, 2, 1)
    cin = 64
    for li, (n, cout) in enumerate(zip(blocks, (64, 128, 256, 512)), start=1):
        for bi in range(n):
            s = 2 if (bi == 0 and li > 1) else 1
            name = f"model.layer{li}.{bi}"
            w1, b1 = W.conv_bn(name, cout, cin, 3, BN_EPS_TV, conv_key="conv1", bn_key="bn1")
            w2, b2 = W.conv_bn(name, cout, cout, 3, BN_EPS_TV, conv_key="conv2", bn_key="bn2", res_branch=True)
            if s != 1 or cin != cout:
                wd, bd = W.conv_bn(f"{name}.downsample", cout, cin, 1, BN_EPS_TV, conv_key="0", bn_key="1")
                idt = pb.conv(x, wd, bd, 1, s, ACT_NONE, pad=0)
            else:
                idt = x
            t = pb.conv(x, w1, b1, 3, s, ACT_RELU)
            x = pb.conv(t, w2, b2, 3, 1, ACT_RELU, res=idt, res_pre_act=True)
            cin = cout
    # pool: Conv2d(512, 8, 1) with bias, no BN/activation (model_culane.py:39,48)
    wp, bp = W.conv_bias("pool", 8, 512, 1)
    pool = pb.conv(x, wp, bp, 1, 1, ACT_NONE)
    fh, fw = pool.H, pool.W
    input_dim = fh * fw * 8                     # model_culane.py:23
    if v1:       # UFLD v1 head (exportLib/ultrafastLane/model.py:20-66): one tensor [griding_num + 1, cls_num_per_lane, 4]
        ngr, ncr, ngc, ncc, nl = cfg["griding_num"], cfg["cls_num_per_lane"], 0, 0, cfg["num_lanes"]
        total_dim = (ngr + 1) * ncr * nl
        assert input_dim == 1800, "UFLD v1 hard-codes Linear(1800, 2048) (model.py:62): 288x800 input"
    else:
        ngr, ncr, ngc, ncc, nl = cfg["num_grid_row"], cfg["num_cls_row"], cfg["num_grid_col"], cfg["num_cls_col"], cfg["num_lanes"]
        total_dim = ngr * ncr * nl + ngc * ncc * nl + 2 * ncr * nl + 2 * ncc * nl
    mid = 2048
    # the flattened NCHW feature f = c*fh*fw + h*fw + w lives at j = ((h+1)*(fw+2) + (w+1))*8 + c of the padded slab
    slab = (fh + 2) * (fw + 2) * 8
    cidx, hidx, widx = np.meshgrid(np.arange(8), np.arange(fh), np.arange(fw), indexing="ij")
    f_idx = (cidx * fh * fw + hidx * fw + widx).ravel()
    j_idx = (((hidx + 1) * (fw + 2) + (widx + 1)) * 8 + cidx).ravel()
    if cfg.get("fc_norm", True):
        g = W.get("cls.0.weight", (input_dim,), "ln_gamma")
        be = W.get("cls.0.bias", (input_dim,), "ln_beta")
    else:
        g, be = None, None
    # v2: cls = Sequential(LayerNorm | Identity, Linear, ReLU, Linear) -> cls.1 / cls.3; v1: Sequential(Linear, ReLU, Linear) -> cls.0 / cls.2
    k1, k2 = ("cls.0", "cls.2") if v1 else ("cls.1", "cls.3")
    w1 = W.get(k1 + ".weight", (mid, input_dim), "linear")
    b1 = W.get(k1 + ".bias", (mid,), "bias")
    w2 = W.get(k2 + ".weight", (total_dim, mid), "linear")
    b2 = W.get(k2 + ".bias", (total_dim,), "bias")
    exist_bias = None if (W.real or v1) else W.profile.get("ufld_exist_bias")
    if v1 and not W.real and not getattr(W, "_ufld_v1_applied", False):
        # synthetic operating point for v1: the "no lane" bin (last grid index) loses on most rows, so lanes are detected, and the
        # head gain is halved -- the v1 coordinate is an expectation over ALL grid cells, so its fp16-vs-fp32 error scales with the
        # logit scale of a random head (CPU fp16 emulation, tools/synth_operating_point.py style: gain 1 -> 8e-4 of the width,
        # 0.5 -> 3e-4; trained heads are peaked and far less sensitive)
        b2 = b2.copy()
        b2.reshape(ngr + 1, ncr, nl)[ngr] -= np.float32(2.0)
        w2 = (w2 * np.float32(0.5)).astype(np.float32)
        W.state_dict[k2 + ".bias"] = b2
        W.state_dict[k2 + ".weight"] = w2
        W._ufld_v1_applied = True
    if exist_bias and not getattr(W, "_ufld_exist_applied", False):
        # synthetic operating point (see SYNTH_PROFILES): shift the "valid" planes of exist_row / exist_col, in the shared state_dict
        b2 = b2.copy()
        d12 = ngr * ncr * nl + ngc * ncc * nl
        b2[d12 + ncr * nl:d12 + 2 * ncr * nl] += np.float32(exist_bias)
        b2[total_dim - ncc * nl:] += np.float32(exist_bias)
        W.state_dict["cls.3.bias"] = b2
        W._ufld_exist_applied = True
    pb.flops_per_img += 2 * (mid * input_dim + total_dim * mid)
    w1p = np.zeros((mid, slab), np.float32)
    w1p[:, j_idx] = w1[:, f_idx]
    feat_buf = pool.buf
    if g is not None:
        gp = np.zeros(slab, np.float32); gp[j_idx] = g[f_idx]
        bpad = np.zeros(slab, np.float32); bpad[j_idx] = be[f_idx]
        ln_buf = pb.new_dense(1, slab)
        pb.layernorm(pool.buf, slab, input_dim, gp, bpad, 1e-5, ln_buf)
        feat_buf = ln_buf
        fc_in_K = slab
    else:
        # fc_norm=False (TuSimple configs): cls.0 is Identity; the FC reads the pool conv's padded slab directly, one row per image
        # (its halo entries are structural zeros and meet zero weight columns)
        fc_in_K = slab
    h_buf = pb.new_dense(1, mid)
    pb.fc(feat_buf, fc_in_K, w1p, b1, ACT_RELU, h_buf)
    o_buf = pb.new_dense(1, total_dim, f32=True)
    pb.fc(h_buf, mid, w2, b2, ACT_NONE, o_buf)
    pb.outputs.append((o_buf, 0, total_dim, 0))
    pb.meta[0:6] = [ngr, ncr, ngc, ncc, nl, total_dim]
    pb.meta[6] = int(cfg.get("dataset", 0))
    return pb
