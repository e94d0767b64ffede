"""Helpers for the GPU parity tests: padded-NHWC packing, cached plan files and network inputs."""
import os

import numpy as np

import adas_b200  # noqa: F401
from adas_b200 import plan
from oracle import post


def to_padded(x_nchw: np.ndarray, C: int) -> np.ndarray:
    """[B,c,H,W] float -> [B*(H+2)*(W+2), C] fp16 with zero halo / zero extra channels."""
    B, c, H, W = x_nchw.shape
    out = np.zeros((B, H + 2, W + 2, C), np.float16)
    out[:, 1:-1, 1:-1, :c] = x_nchw.transpose(0, 2, 3, 1).astype(np.float16)
    return out.reshape(-1, C)


def from_padded(buf: np.ndarray, B: int, H: int, W: int, coff: int, c: int) -> np.ndarray:
    """[B*(H+2)*(W+2), ld] -> [B,c,H,W] float32 interior."""
    v = buf.reshape(B, H + 2, W + 2, -1)[:, 1:-1, 1:-1, coff:coff + c]
    return v.astype(np.float32).transpose(0, 3, 1, 2)


def halo_is_zero(buf: np.ndarray, B: int, H: int, W: int) -> bool:
    v = buf.reshape(B, H + 2, W + 2, -1).astype(np.float32)
    return not (v[:, 0].any() or v[:, -1].any() or v[:, :, 0].any() or v[:, :, -1].any())


def cached_plan(kind: str, seed: int = 0, **kw):
    """Build the seeded synthetic plan of one network and write it to the plan cache: (path, state_dict, PlanBuilder).

    `kind` names the builder (`plan.build_<kind>`: "yolov5", "yolov6", "yolov6_lite", "yolov7", "yolov8", "yolov9", "yolov10", "ufldv1",
    "ufldv2"; YOLOv9-E is "yolov9" with scale "e") and `kw` are its arguments.  The file is rewritten from this build on every call,
    through a temporary name of this process, so it never holds a plan an older builder wrote, nor a mix of two processes' writes."""
    import zlib
    synth = {"ufldv1": "ufldv2", "yolov6_lite": "yolov6lite"}.get(kind, kind)
    prof = zlib.crc32(repr((plan.SYNTH_PROFILES[synth], plan.PLAN_VERSION)).encode()) & 0xffff      # a changed operating point is a new plan
    tag = kind + "_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items())) + f"_s{seed}_{prof:04x}"
    path = os.path.join(plan.cache_dir(), tag + ".b200w")
    variant = kw.get("scale", kw.get("backbone"))             # calibrated BatchNorm statistics exist for the tested variants
    W = plan.synth_weights(synth, seed, variant=variant)
    pb = getattr(plan, "build_" + kind)(W, **kw)
    tmp = f"{path}.{os.getpid()}.tmp"
    pb.write(tmp)
    os.replace(tmp, path)
    return path, W.state_dict, pb


def yolo_blob(frames, h: int = 640, w: int = 640) -> np.ndarray:
    """The letterboxed [B, 3, h, w] float32 network input of a list of frames (the oracle's pre-processing)."""
    return np.concatenate([post.yolo_prepare_input(f, h, w)[0] for f in frames])
