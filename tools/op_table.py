"""Per-layer table of a plan at real clocks: every launch replayed alone (CUDA events, L2-warm), GEMM shapes and tile choices.
usage: python tools/op_table.py yolov8|ufldv2|yolov5|yolov7|yolov7-tiny|yolov7-w6|yolov7-e6|yolov7-d6|yolov7-e6e|yolov6n|yolov6s|yolov6m|yolov6l|yolov6lite-s|yolov6lite-m|yolov6lite-l|yolov9-t|yolov9-s|yolov9-m|yolov9-c|yolov9-e|yolov10n|yolov10s|yolov10m|yolov10b|yolov10l|yolov10x [batch] [iters]
(the YOLOv7 P6 models run at 1280x1280, YOLOv6-Lite at 320x320)   (env switches of the library apply)"""
import os, re, sys, tempfile
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
import adas_b200
from adas_b200 import _capi, plan
from gpu_util import cached_plan
kind = sys.argv[1]; B = int(sys.argv[2]) if len(sys.argv) > 2 else 8; iters = int(sys.argv[3]) if len(sys.argv) > 3 else 20
if kind.startswith("yolov7"):        # built fresh: ADAS_B200_STEMCONV decides at pack time where the stem runs
    pb = plan.build_yolov7(plan.synth_weights("yolov7", 0), {"yolov7": "base", "yolov7-tiny": "tiny"}.get(kind, kind[7:]))
    path = os.path.join(tempfile.mkdtemp(), kind + ".b200w")
    pb.write(path)
elif kind.startswith("yolov6lite"):
    pb = plan.build_yolov6_lite(plan.synth_weights("yolov6lite", 0, variant=kind[-1]), kind[-1])
    path = os.path.join(tempfile.mkdtemp(), kind + ".b200w")
    pb.write(path)
elif kind.startswith("yolov6"):
    pb = plan.build_yolov6(plan.synth_weights("yolov6", 0, variant=kind[-1]), kind[-1])
    path = os.path.join(tempfile.mkdtemp(), kind + ".b200w")
    pb.write(path)
elif kind.startswith("yolov10"):
    pb = plan.build_yolov10(plan.synth_weights("yolov10", 0, variant=kind[-1]), kind[-1])
    path = os.path.join(tempfile.mkdtemp(), kind + ".b200w")
    pb.write(path)
elif kind.startswith("yolov9"):
    pb = plan.build_yolov9(plan.synth_weights("yolov9", 0, variant=kind[-1]), kind[-1])
    path = os.path.join(tempfile.mkdtemp(), kind + ".b200w")
    pb.write(path)
else:
    kw = {"yolov8": dict(scale="l"), "ufldv2": dict(backbone="34"), "yolov5": dict(scale="n")}[kind]
    path, sd, pb = cached_plan(kind, **kw)
eng = _capi.Engine(path, 0, max_batch=B)
eng.run(B)
n = eng.num_steps(B)
names = {**plan.OP_NAMES, 31: "(folded)"}
tot = 0.0; tot_g = 0.0; rows = []
for i in range(n):
    ms, t, d = eng.time_step(B, i, iters)
    tot += ms
    tf = ""
    if t == 1:
        tot_g += ms
        m = re.match(r"M=(\d+) N=(\d+) K=(\d+)", d)
        if m:
            M, N, K = map(int, m.groups())
            tf = f"{2.0 * M * N * K / ms / 1e9:7.1f} TF(incl halo)"
    rows.append((ms, i, names.get(t, str(t)), d, tf))
    print(f"{i:3d} {names.get(t, str(t)):9s} {ms * 1e3:8.1f} us {tf} {d}", flush=True)
flops = (pb.flops_per_img - pb.stem_flops_per_img - pb.dw_flops_per_img) * B      # the stem and depthwise convs are not GEMM launches
print(f"TOTAL {kind} b{B}: sum of isolated launches {tot * 1e3:.1f} us (gemm {tot_g * 1e3:.1f} us) -> {flops / tot_g / 1e9:.1f} TFLOP/s algorithmic over GEMM time")
ms_all, nl = eng.time_ops(B, 0xFFFFFFFF, 10)
ms_g, ng = eng.time_ops(B, 1 << 1, 10)
print(f"back-to-back: all {ms_all * 1e3:.1f} us ({nl} launches), gemm only {ms_g * 1e3:.1f} us ({ng}) -> {flops / ms_g / 1e9:.1f} TFLOP/s, "
      f"plan only {B / ms_all * 1e3:.0f} images/s")
ms_ap = sum(r[0] for r in rows if r[2] == "avgpool2")
ms_ic = sum(r[0] for r in rows if r[2] == "im2col" and pb.ops[r[1]][1].Cin < 64)        # one launch per plan op
print(f"share of the sum of isolated launches: avgpool2 {100 * ms_ap / tot:.1f} %, im2col of convs with < 64 input channels {100 * ms_ic / tot:.1f} %")
dw_rows = [r for r in rows if r[2] == "dwconv"]
if dw_rows:
    ms_dw = sum(r[0] for r in dw_rows)
    ms_at = sum(r[0] for r in rows if r[2] == "attention")
    dw_bytes = 0                              # fp16 input + output (+ residual) of every depthwise launch, weights once: computed from shapes
    for r in dw_rows:
        p = pb.ops[r[1]][1]
        bi, bo = pb.buffers[p.in_buf], pb.buffers[p.out_buf]
        C, k = p.C, p.k
        dw_bytes += 2 * B * C * (bi[3] * bi[4] + bo[3] * bo[4] * (2 if p.res_buf >= 0 else 1)) + C * (2 * k * k + 4)
    print(f"share of the sum of isolated launches: dwconv {100 * ms_dw / tot:.1f} %, attention {100 * ms_at / tot:.1f} %; "
          f"dwconv {dw_bytes / 1e6:.1f} MB in {ms_dw * 1e3:.1f} us -> {dw_bytes / ms_dw / 1e6:.0f} GB/s (HBM3 data sheet: 3350 GB/s)")
cb_rows = [r for r in rows if r[2] == "cbfuse"]
if cb_rows:
    ms_cb = sum(r[0] for r in cb_rows)
    cb_bytes = 0                              # fp16: the target read and written once, each source read once at its own resolution
    for r in cb_rows:
        p = pb.ops[r[1]][1]
        ob = pb.buffers[p.out_buf]
        cb_bytes += 2 * B * p.C * ob[3] * ob[4] * 2 + sum(2 * B * p.C * pb.buffers[sb][3] * pb.buffers[sb][4] for sb, _, _ in plan.cbfuse_sources(p))
    print(f"share of the sum of isolated launches: cbfuse {100 * ms_cb / tot:.1f} %; cbfuse {cb_bytes / 1e6:.1f} MB in {ms_cb * 1e3:.1f} us -> "
          f"{cb_bytes / ms_cb / 1e6:.0f} GB/s (HBM3 data sheet: 3350 GB/s)")
se_rows = [r for r in rows if r[2] in ("se", "shuffle2")]
if se_rows:
    share = {k: sum(r[0] for r in rows if r[2] == k) for k in ("se", "shuffle2", "dwconv", "gemm")}
    print("share of the sum of isolated launches: " + ", ".join(f"{k} {100 * v / tot:.1f} %" for k, v in share.items()))
    for k in ("se", "shuffle2"):              # bytes from shapes: SE reads its fp16 slice twice (mean, then scale), writes it once and reads
        nbytes = 0                            # its fp32 FC weights once per image; SHUFFLE2 reads two n-channel slices and writes 2n channels
        for r in (r for r in rows if r[2] == k):
            p = pb.ops[r[1]][1]
            if k == "se":
                b = pb.buffers[p.in_buf]
                nbytes += 2 * B * b[3] * b[4] * 3 * p.C + B * 4 * (2 * p.C * p.hid + p.C + p.hid)
            else:
                b = pb.buffers[p.a_buf]
                nbytes += 2 * B * b[3] * b[4] * 4 * p.n
        print(f"{k}: {nbytes / 1e6:.2f} MB in {share[k] * 1e3:.1f} us -> {nbytes / share[k] / 1e6:.0f} GB/s (HBM3 data sheet: 3350 GB/s)")
    act = sum(B * rows_ * C * (4 if f32 else 2) for rows_, C, f32, _, _, _ in pb.buffers)
    wts = sum(t.nbytes for t in pb.tensors)
    print(f"device memory of the plan at batch {B}: activations {act / 1e6:.1f} MB, weights {wts / 1e6:.2f} MB")
eng.close()
