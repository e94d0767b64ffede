"""multicam_bench.py -- K cameras through ONE AdasPipeline(cameras=K) against K single-camera AdasPipelines stepped in turn in one
process: YOLOv8l + UFLDv2-r34 + ByteTrack (bench.py's workload and seeded weights), F frames per camera per step, synthetic 1280x720
streams (a different one per camera) resident on the device, every arm driven through step_pipelined as bench.py drives it.

Per (K, arm): frames/s over `--repeats` timed windows of `--steps` steps (each window ends with flush + device synchronise), the
tracker's wall time and association launches per step from adas_tracker_stats, and the device memory the arm's pipelines hold
after warm-up.  The two arms cannot be alive together at K = 8 without crowding an 80 GB card, so each arm is built, measured and
closed in turn.  K = 1 is one arm (one camera through one pipeline is both).  Prints one JSON line per (K, arm) and the card, its
power limit and the SM clocks sampled during the timed windows.  Needs a GPU; there is no CPU fallback.

With `--sizes WxH,WxH,...` the cameras differ in frame size (K = the number of sizes): one AdasPipeline(cameras=K,
frame_sizes=...) against K single-camera pipelines stepped in turn, on device-resident synthetic frames of each camera's size
(tests/synth.py's frame(seed, h, w)), measured as above.

    python tools/multicam_bench.py --cameras 1,2,4,8 --frames 8 --steps 30 --warmup 4 --repeats 3
    python tools/multicam_bench.py --sizes 1920x1080,1280x800,1280x800,1280x720 --frames 8
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402


def used_mib() -> float:
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2 ** 20


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except Exception as e:                     # the numbers are still printed, without their card
        out = f"nvidia-smi failed: {e}"
    return {"nvidia_smi": out, "query": q}


def run_arm(plans, K: int, F: int, multi: bool, pool, args, clocks, sizes=None):
    """pool: [batches, K, F, H, W, 3] on the device, or with `sizes` a list of K [batches, F, H_c, W_c, 3] device tensors"""
    from adas_b200.pipeline import AdasPipeline
    H, W = bench.FRAME_H, bench.FRAME_W
    kw = dict(device=0, batch=F, box_score=bench.BOX_SCORE, box_nms_iou=bench.NMS_IOU, max_det=bench.MAX_DET)
    torch.cuda.synchronize()
    base = used_mib()
    t_build = time.time()
    y, u = plans["yolov8"][0], plans["ufldv2"][0]
    pipes = [AdasPipeline(y, u, cameras=K, frame_sizes=sizes, **kw)] if multi else [AdasPipeline(y, u, **kw) for _ in range(K)]
    t_build = time.time() - t_build
    nb = pool[0].shape[0] if sizes is not None else pool.shape[0]

    def step(i):
        if sizes is not None:
            xs = [p[i % nb] for p in pool]                        # K x [F, H_c, W_c, 3], contiguous
            if multi:
                pipes[0].step_pipelined([(x.data_ptr(), tuple(x.shape[:3])) for x in xs], True)
            else:
                for x, p in zip(xs, pipes):
                    p.step_pipelined(x.data_ptr(), True, tuple(x.shape[:3]))
            return
        x = pool[i % nb]                                          # [K, F, H, W, 3], contiguous
        if multi:
            pipes[0].step_pipelined(x.data_ptr(), True, (K, F, H, W) if K > 1 else (F, H, W))
        else:
            for c, p in enumerate(pipes):
                p.step_pipelined(x[c].data_ptr(), True, (F, H, W))

    def drain():
        for p in pipes:
            p.flush()
        torch.cuda.synchronize()

    for i in range(args.warmup):
        step(i)
    drain()
    mem = used_mib() - base
    trackers = [t._nt for p in pipes for t in p.trackers]
    fps, trk_ms, launches, wait_ms, sm = [], [], [], [], []
    for r in range(args.repeats):
        s0 = [t.stats() for t in trackers]
        t0 = time.time()
        for i in range(args.steps):
            step(i)
        drain()
        t1 = time.time()
        s1 = [t.stats() for t in trackers]
        d = [{k: b[k] - a[k] for k in a} for a, b in zip(s0, s1)]
        fps.append(K * F * args.steps / (t1 - t0))
        # one K-camera call advances every tracker: its wall time and round trips are counted once per tracker, so take the lead's;
        # separate pipelines add up.  A shared launch counts once for each tracker in it: the most any camera took part in.
        trk_ms.append((d[0]["total_ms"] if multi else sum(x["total_ms"] for x in d)) / args.steps)
        wait_ms.append((d[0]["wait_ms"] if multi else sum(x["wait_ms"] for x in d)) / args.steps)
        launches.append((max(x["launches"] for x in d) if multi else sum(x["launches"] for x in d)) / args.steps)
        sm.append(clocks.window(t0, t1))
    for p in pipes:
        p.close()
    del pipes, trackers
    torch.cuda.synchronize()
    return {"cameras": K, "frames_per_step": F, "arm": "one pipeline" if multi else f"{K} pipelines",
            "sizes_wh": None if sizes is None else [f"{w}x{h}" for h, w in sizes],
            "frames_per_s": [round(v, 1) for v in fps], "tracker_ms_per_step": [round(v, 3) for v in trk_ms],
            "assoc_round_trip_ms_per_step": [round(v, 3) for v in wait_ms], "assoc_launches_per_step": [round(v, 2) for v in launches],
            "device_mib_after_warmup": round(mem, 0), "build_s": round(t_build, 1),
            "sm_mhz": [c["sm_mhz"] for c in sm], "clock_reasons": sorted({x for c in sm for x in c["reasons"]})}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--cameras", default="1,2,4,8")
    ap.add_argument("--frames", type=int, default=8, help="frames per camera per step")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sizes", default=None, help="WxH,WxH,...: one camera per size, of different frame sizes (replaces --cameras)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multicam_bench.py needs a GPU")
    F = args.frames
    plans = bench.build_plans()
    clocks = bench.ClockSampler(0)
    clocks.start()
    lines = [json.dumps({"card": card()})]
    print(lines[0], flush=True)
    try:
        if args.sizes:
            sys.path.insert(0, os.path.join(ROOT, "tests"))
            import synth
            sizes = [(int(h), int(w)) for w, h in (s.lower().split("x") for s in args.sizes.split(","))]
            K = len(sizes)
            pool = [torch.from_numpy(np.stack([np.stack([synth.frame(500 + 37 * c + b * F + f, h, w) for f in range(F)]) for b in range(4)])).cuda()
                    for c, (h, w) in enumerate(sizes)]                                                 # K x [4 batches, F, H_c, W_c, 3]
            for multi in [True, False]:
                res = run_arm(plans, K, F, multi, pool, args, clocks, sizes=sizes)
                lines.append(json.dumps(res))
                print(lines[-1], flush=True)
            del pool
            torch.cuda.empty_cache()
        for K in ([] if args.sizes else [int(k) for k in args.cameras.split(",")]):
            streams = [bench.synth_stream(500 + c, 4 * F) for c in range(K)]
            host = np.stack([np.stack([s[b * F:(b + 1) * F] for s in streams]) for b in range(4)])     # [4 batches, K, F, H, W, 3]
            pool = torch.from_numpy(host).cuda()
            del streams, host
            for multi in ([True] if K == 1 else [True, False]):
                res = run_arm(plans, K, F, multi, pool, args, clocks)
                lines.append(json.dumps(res))
                print(lines[-1], flush=True)
            del pool
            torch.cuda.empty_cache()
    finally:
        clocks.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
