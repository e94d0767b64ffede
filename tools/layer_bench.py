"""Time single conv layers (GEMM op only) through the engine: python tools/layer_bench.py [substring of the layer name]"""
import os, sys, tempfile
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
import numpy as np
import adas_b200
from adas_b200 import _capi, plan
LAYERS = [
    ("P3 1x1 1024->256 80x80", 8, 1024, 256, 80, 80, 1),
    ("P4 1x1 2048->512 40x40", 8, 2048, 512, 40, 40, 1),  # name, B, cin, cout, H, W, k
    ("P3 3x3 128->128 80x80", 8, 128, 128, 80, 80, 3),
    ("P4 3x3 256->256 40x40", 8, 256, 256, 40, 40, 3),
    ("P5 3x3 256->256 20x20", 8, 256, 256, 20, 20, 3),
    ("P2 3x3 64->64 160x160", 8, 64, 64, 160, 160, 3),
    ("P3 1x1 768->256 80x80", 8, 768, 256, 80, 80, 1),
    ("P3 3x3 128->128 80x80 B32", 32, 128, 128, 80, 80, 3),
    ("P4 3x3 256->256 40x40 B32", 32, 256, 256, 40, 40, 3),
]
rng = np.random.default_rng(0)
FILTER = sys.argv[1] if len(sys.argv) > 1 else ""
for name, B, cin, cout, H, W, k in LAYERS:
    if FILTER not in name:
        continue
    pb = plan.PlanBuilder(plan.MODEL_YOLOV5, 3, H, W)
    xin = pb.new_padded(H, W, cin)
    w = (rng.standard_normal((cout, cin, k, k)) * 0.05).astype(np.float32)
    out = pb.conv(xin, w, np.zeros(cout, np.float32), k, 1, 1)
    path = os.path.join(tempfile.gettempdir(), f"lb_{cin}_{cout}_{H}_{k}.b200w")
    pb.write(path)
    eng = _capi.Engine(path, 0, max_batch=B)
    ms, n = eng.time_ops(B, 1 << 1, 20)
    macs = B * (H + 2) * (W + 2) * cout * cin * k * k
    print(f"bn={os.environ.get('ADAS_B200_BN','-')} mt={os.environ.get('ADAS_B200_MT','-')} {name:28s} {ms*1e3:8.1f} us  {2*macs/ms/1e9:7.1f} TFLOP/s(incl halo)", flush=True)
    eng.close()
