"""Scan synthetic head operating points (gain, bias) on the CPU: fp32 oracle vs its fp16-storage emulation (oracle.nets.forward_fp16_emulated).
Prints the probability / box error the device path will show, the candidates per frame at box_score 0.4 and how many sit within 1e-3 / 2e-3
of the threshold.  Test infrastructure (uses oracle/):  python tools/synth_operating_point.py yolov8 l 45,-9 40,-8.2
(yolov9 t|s|m|c|e, yolov10 n|s|m|b|l|x: the scale's class bias; the head gains of plan.SYNTH_PROFILES[kind] are kept)
(yolov6lite s|m|l: 320x320, gain = the class-logit gain, bias = the scale's class bias; the fp16 emulation is plan_interp's rounded run of
the plan itself, tests/plan_interp.py)
"""
import sys, os
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, 'tests'))
import numpy as np, torch
torch.set_num_threads(8)
import adas_b200
from adas_b200 import plan
from oracle import nets, post
import synth
kind, variant = sys.argv[1], sys.argv[2]
builder = {"yolov8": plan.build_yolov8, "yolov9": plan.build_yolov9, "yolov10": plan.build_yolov10}.get(kind, plan.build_yolov5)
size = 320 if kind == "yolov6lite" else 640
x = torch.from_numpy(np.concatenate([post.yolo_prepare_input(synth.frame(s), size, size)[0] for s in (0,1,2,3,4,5,6,7)]))
for a in sys.argv[3:]:
    g,b = map(float,a.split(','))
    if kind=="yolov6lite":
        import yolov6_lite_oracle, plan_interp, test_yolov6_lite_cpu
        from gpu_util import to_padded
        plan.SYNTH_PROFILES["yolov6lite"]={**plan.SYNTH_PROFILES["yolov6lite"], "gains":[(r"detect\.cls_preds\.\d\.weight", g)],
                                       "variants": {variant: {"fill": [(r"detect\.cls_preds\.\d\.bias", b)]}}}
        W = plan.synth_weights(kind, 0, variant=variant); pb = plan.build_yolov6_lite(W, variant)
        with torch.no_grad():
            ref = yolov6_lite_oracle.build(W.state_dict, variant)(x).numpy()
        emu = np.stack([test_yolov6_lite_cpu._decode(pb, plan_interp.interpret(pb, to_padded(x[i:i + 1].numpy(), 4), 1, round_to_plan=True))
                        for i in range(len(x))])
        ref = np.concatenate([ref[..., :4], ref[..., 5:]], -1)
        e=np.abs(ref[...,4:]-emu[...,4:]); mx=ref[...,4:].max(2); mg=emu[...,4:].max(2); eb=np.abs(ref[...,:4]-emu[...,:4]).max()
        cand=mx>0.4
        print(f"g={g} b={b}: max prob err {e.max():.2e} box err {eb:.3f} | cands {cand.sum(1).tolist()} within1e-3 {(np.abs(mx-0.4)<1e-3).sum(1).tolist()} flips {int((cand!=(mg>0.4)).sum())}", flush=True)
        print("   per-frame max prob err", [f"{v:.2e}" for v in e.reshape(e.shape[0],-1).max(1)])
        continue
    if kind=="yolov8":
        plan.SYNTH_PROFILES["yolov8"]={"gains":[(r"model\.22\.cv3\.\d\.2\.weight", g), (r"model\.22\.cv2\.\d\.2\.weight", 25.0)],"fill":[(r"model\.22\.cv3\.\d\.2\.bias", b)]}
    elif kind=="yolov9":
        hd, bg = ("model\\.42", 12.0) if variant == "e" else ("model\\.22", 25.0)      # YOLOv9-E's head is model.42 (box gain 12)
        plan.SYNTH_PROFILES["yolov9"]={**plan.SYNTH_PROFILES["yolov9"], "gains":[(hd + r"\.cv3\.\d\.2\.weight", g), (hd + r"\.cv2\.\d\.2\.weight", bg)],
                                   "variants": {variant: {"fill": [(hd + r"\.cv3\.\d\.2\.bias", b)]}}}
    elif kind=="yolov10":
        plan.SYNTH_PROFILES["yolov10"]={**plan.SYNTH_PROFILES["yolov10"], "gains":[(r"model\.23\.one2one_cv3\.\d\.2\.weight", g), (r"model\.23\.one2one_cv2\.\d\.2\.weight", 25.0)],
                                    "variants": {variant: {"fill": [(r"model\.23\.one2one_cv3\.\d\.2\.bias", b)]}}}
    else:
        plan.SYNTH_PROFILES["yolov5"]={"gains":[(r"model\.24\.m\.\d\.weight", g)],"fill":[(r"model\.24\.m\.\d\.bias", b)]}
    W = plan.synth_weights(kind, 0, variant=variant); builder(W, variant)
    if kind=="yolov9":
        import yolov9_oracle, yolov9e_oracle
        md = yolov9e_oracle.build(W.state_dict) if variant == "e" else yolov9_oracle.build(W.state_dict, variant)
    elif kind=="yolov10":
        import yolov10_oracle
        md = yolov10_oracle.build(W.state_dict, variant)
    else:
        md = nets.build(kind, W.state_dict, scale=variant)
    with torch.no_grad():
        ref = md(x).numpy()
        emu = (yolov10_oracle.forward_fp16_emulated if kind == "yolov10" else nets.forward_fp16_emulated)(md, x).numpy()
    if kind in ("yolov8", "yolov9", "yolov10"):
        e=np.abs(ref[:,4:]-emu[:,4:]); mx=ref[:,4:].max(1); mg=emu[:,4:].max(1); eb=np.abs(ref[:,:4]-emu[:,:4]).max()
    else:
        e=np.abs(ref[...,4:]-emu[...,4:]); mx=(ref[...,5:]*ref[...,4:5]).max(2); mg=(emu[...,5:]*emu[...,4:5]).max(2); eb=np.abs(ref[...,:4]-emu[...,:4]).max()
    cand=mx>0.4
    print(f"g={g} b={b}: max prob err {e.max():.2e} box err {eb:.3f} | cands {cand.sum(1).tolist()} within1e-3 {(np.abs(mx-0.4)<1e-3).sum(1).tolist()} within2e-3 {int((np.abs(mx-0.4)<2e-3).sum())} flips {int((cand!=(mg>0.4)).sum())}", flush=True)
    if kind in ("yolov8", "yolov9", "yolov10"): print("   per-frame max prob err", [f"{v:.2e}" for v in e.max(axis=(1,2))])
    else: print("   per-frame max prob err", [f"{v:.2e}" for v in e.reshape(e.shape[0],-1).max(1)])
