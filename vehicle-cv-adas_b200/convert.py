"""convert.py -- model files -> packed `.b200w` plans (command line + functions).

Counterpart of the reference's conversion scripts: `convertOnnxToTensorRT.py` (ONNX -> .trt engine written next to the model)
and `TrafficLaneDetector/convertPytorchToONNX.py:77-87` (UFLD `.pth` checkpoint -> ONNX: `torch.load(...)['model']`, the
`module.` prefix of DataParallel checkpoints stripped).  Here both sources go straight to the plan the sm_90a engine loads:

    python -m adas_b200.convert yolov8l.onnx                       # architecture recognised from the graph
    python -m adas_b200.convert culane_res34.pth --kind ufldv2 --backbone 34
    python -m adas_b200.convert yolov5n.pt.state_dict.pth --kind yolov5 --scale n
    python -m adas_b200.convert yolov7-tiny.state_dict.pth --kind yolov7 --scale tiny
    python -m adas_b200.convert yolov7-w6.state_dict.pth --kind yolov7 --scale w6     # P6: w6 | e6 | d6 | e6e, 1280x1280
    python -m adas_b200.convert yolov6s.state_dict.pth --kind yolov6 --scale s
    python -m adas_b200.convert yolov6lite_s.state_dict.pth --kind yolov6-lite --scale s    # s | m | l, 320x320
    python -m adas_b200.convert yolov9-c.state_dict.pth --kind yolov9 --scale c     # t | s | m | c | e
    python -m adas_b200.convert yolov10s.state_dict.pth --kind yolov10 --scale s    # n | s | m | b | l | x
    python -m adas_b200.convert yolov10s.onnx                                         # recognised, also with the top-k tail

Upstream YOLOv6 checkpoints pickle the whole model; extract its parameters once, in the YOLOv6 repository:
    torch.save(torch.load("yolov6s.pt", map_location="cpu", weights_only=False)["model"].float().state_dict(), "yolov6s.state_dict.pth")
Training-form (rbr_dense / rbr_1x1 / rbr_identity + BatchNorm) and deployed (rbr_reparam, fused conv biases) keys are both accepted.
YOLOv6-Lite checkpoints are extracted the same way; training-form (ConvBNHS / DPBlock with their BatchNorms) and fused keys are both
accepted.  YOLOv6-Lite .onnx files are recognised like the other families.
YOLOv9 checkpoints (WongKinYiu/yolov9) pickle the whole model too; extract the parameters once, in the YOLOv9 repository:
    torch.save(torch.load("yolov9-c-converted.pt", map_location="cpu", weights_only=False)["model"].float().state_dict(), "yolov9-c.state_dict.pth")
Training-form (RepConvN conv1 / conv2 + BatchNorm) and fused (conv weight + bias) keys are both accepted; only the converted (GELAN)
graphs are supported, not the training files with the auxiliary branch.
YOLOv10 checkpoints (ultralytics 8.2.41) pickle the whole model; extract the parameters once, in an ultralytics checkout:
    torch.save(torch.load("yolov10s.pt", map_location="cpu", weights_only=False)["model"].float().state_dict(), "yolov10s.state_dict.pth")
Training-form (Conv + BatchNorm, RepVGGDW conv / conv1) and fused keys are both accepted.  Only the one-to-one head
(`model.23.one2one_cv2` / `one2one_cv3`) is packed; the one-to-many head's keys are ignored.  The plan emits YOLOv8's [B, 4 + nc, A]
output, decoded by the YOLOv8 path, not upstream's top-k [1, 300, 6] tail.

Checkpoints hold un-fused Conv/BatchNorm parameters under the upstream key names (the names `plan.build_*` ask for), so BatchNorm
is folded here in float64 exactly as for the seeded weights.  Only the parameter dictionary is read: pickled model objects
(ultralytics `.pt`) need their own package to unpickle and are out of scope -- export those to ONNX or save a state_dict.
"""
from __future__ import annotations

import argparse
import os
from typing import Dict, Optional

import numpy as np

from . import plan
from .onnx_import import build_plan, read_onnx, recognise


def load_checkpoint_state_dict(path: str) -> Dict[str, np.ndarray]:
    """`.pth` / `.pt` holding a state_dict, or a dict with it under 'model' / 'state_dict' (convertPytorchToONNX.py:77-84)."""
    import torch
    obj = torch.load(path, map_location="cpu", weights_only=True)
    for key in ("model", "state_dict", "net"):
        if isinstance(obj, dict) and key in obj and isinstance(obj[key], dict):
            obj = obj[key]
            break
    if not isinstance(obj, dict):
        raise Exception("The model path [%s] does not hold a parameter dictionary" % path)
    sd = {}
    for k, v in obj.items():
        if not hasattr(v, "shape"):
            continue
        k = k[7:] if k.startswith("module.") else k
        sd[k] = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)
    return sd


def plan_from_state_dict(sd: Dict[str, np.ndarray], kind: str, scale: str = "l", backbone: str = "34", nc: int = 80) -> "plan.PlanBuilder":
    w = plan.Weights(sd)
    if kind == "yolov8":
        return plan.build_yolov8(w, scale, nc=nc)
    if kind == "yolov5":
        return plan.build_yolov5(w, scale, nc=nc)
    if kind == "yolov7":
        return plan.build_yolov7(w, scale, nc=nc)
    if kind == "yolov6":
        return plan.build_yolov6(w, scale, nc=nc)
    if kind == "yolov6-lite":
        return plan.build_yolov6_lite(w, scale, nc=nc)
    if kind == "yolov9":
        return plan.build_yolov9(w, scale, nc=nc)
    if kind == "yolov10":
        return plan.build_yolov10(w, scale, nc=nc)
    if kind == "ufldv2":
        return plan.build_ufldv2(w, backbone)
    raise Exception(f"unsupported model kind {kind}")


def convert(path: str, out: Optional[str] = None, kind: Optional[str] = None, scale: str = "l", backbone: str = "34", nc: int = 80) -> str:
    if not os.path.isfile(path):
        raise Exception("The model path [%s] can't not found!" % path)
    out = out or os.path.splitext(path)[0] + ".b200w"
    if path.endswith(".onnx"):
        model = read_onnx(path)
        pb = build_plan(model, recognise(model))
    else:
        if kind is None:
            raise Exception("--kind is required for checkpoint files (yolov8 | yolov5 | yolov7 | yolov6 | yolov6-lite | yolov9 | yolov10 | ufldv2)")
        pb = plan_from_state_dict(load_checkpoint_state_dict(path), kind, scale, backbone, nc)
    pb.write(out)
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="convert an .onnx model or a state_dict checkpoint to a .b200w plan")
    ap.add_argument("model")
    ap.add_argument("--out", default=None)
    ap.add_argument("--kind", default=None, choices=["yolov8", "yolov5", "yolov7", "yolov6", "yolov6-lite", "yolov9", "yolov10", "ufldv2"])
    ap.add_argument("--scale", default="l", help="YOLO scale letter (n | s | m | l for yolov6, s | m | l for yolov6-lite, t | s | m | c | e for yolov9, n | s | m | b | l | x for yolov10), or tiny | base | w6 | e6 | d6 | e6e for yolov7 (checkpoints only; ONNX files are recognised)")
    ap.add_argument("--backbone", default="34", choices=["18", "34"], help="UFLDv2 ResNet depth (checkpoints only)")
    ap.add_argument("--nc", type=int, default=80)
    a = ap.parse_args(argv)
    out = convert(a.model, a.out, a.kind, a.scale, a.backbone, a.nc)
    print("plan written to:\n\t%s (%.1f MB)" % (out, os.path.getsize(out) / 1e6))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
