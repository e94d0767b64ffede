"""fp32 torch-CPU restatement of the YOLOv7 P6 models W6, E6, D6 and E6E (cfg/deploy/yolov7-{w6,e6,d6,e6e}.yaml) -- ReOrg, DownC, Shortcut and a
4-level IDetect with ImplicitA / ImplicitM -- reusing the building blocks and the upstream-style `fuse()` of tests/yolov7_oracle.py.  Test
infrastructure only.  The graph is written as the upstream yaml (from-index, module, arguments), so state_dict keys are upstream's and
the packer's seeded weights load with strict=True.  Not pinned by any upstream file (none can be obtained here): the anchors of the
graph are the published parameter / FLOP counts (tests/test_yolov7_p6_cpu.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

import yolov7_oracle as o7

P6_ANCHORS = ((19, 27, 44, 40, 38, 94), (96, 68, 86, 152, 180, 137), (140, 301, 303, 264, 238, 542), (436, 615, 739, 380, 925, 792))

# stem width, down-sampling module, 3x3 convs per ELAN, backbone stages (out, ELAN width), head level widths P3..P6, ELAN pairs
P6_CFG = {
    "w6": (64, "Conv", 4, ((128, 64), (256, 128), (512, 256), (768, 384), (1024, 512)), (128, 256, 384, 512), False),
    "e6": (80, "DownC", 6, ((160, 64), (320, 128), (640, 256), (960, 384), (1280, 512)), (160, 320, 480, 640), False),
    "d6": (96, "DownC", 8, ((192, 64), (384, 128), (768, 256), (1152, 384), (1536, 512)), (192, 384, 576, 768), False),
    "e6e": (80, "DownC", 6, ((160, 64), (320, 128), (640, 256), (960, 384), (1280, 512)), (160, 320, 480, 640), True),
}


class ReOrg(nn.Module):
    def forward(self, x):
        return torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1)


class DownC(nn.Module):
    def __init__(self, c1, c2, act=None):
        super().__init__()
        self.cv1 = o7.Conv(c1, c1, 1, 1, act)
        self.cv2 = o7.Conv(c1, c2 // 2, 3, 2, act)
        self.cv3 = o7.Conv(c1, c2 // 2, 1, 1, act)

    def forward(self, x):
        return torch.cat((self.cv2(self.cv1(x)), self.cv3(nn.functional.max_pool2d(x, 2, 2))), 1)


class Shortcut(o7.Concat):           # a Concat subclass so that the model's forward hands it the list of its inputs
    def forward(self, xs):
        return xs[0] + xs[1]


class IDetect4(o7.IDetect):
    """IDetect with 4 levels (strides 8 / 16 / 32 / 64)."""
    def __init__(self, nc, ch, anchors):
        super().__init__(nc, ch, anchors[:3])
        self.register_buffer("anchor_grid", torch.tensor(anchors, dtype=torch.float32).view(len(ch), 1, 3, 1, 1, 2), persistent=False)


def p6_cfg(scale):
    stem, down, n3, stages, outs, pair = P6_CFG[scale]
    bk, allk = tuple(range(1, n3, 2)), tuple(range(n3))

    def block(c, c3, cout, keep):
        layers = o7._elan(0, c, c3, n3, cout, keep)
        if pair:
            layers += o7._elan(0, c, c3, n3, cout, keep, src=-len(layers) - 1) + [([-1, -len(layers) - 1], "Shortcut", ())]
        return layers

    def dn(c):
        return [(-1, "Conv", (c, 3, 2))] if down == "Conv" else [(-1, "DownC", (c,))]

    L = [(-1, "ReOrg", ()), (-1, "Conv", (stem, 3, 1))]
    routes = []
    for cout, c in stages:
        L += dn(cout) + block(c, c, cout, bk)
        routes.append(len(L) - 1)
    o3, o4, o5, o6 = outs
    L.append((-1, "SPPCSPC", (o6,)))
    n6 = len(L) - 1
    tops = []
    for lat, route, (c, c3) in ((o5, routes[3], (384, 192)), (o4, routes[2], (256, 128)), (o3, routes[1], (128, 64))):
        L += [(-1, "Conv", (lat, 1, 1)), (-1, "Up", ()), (route, "Conv", (lat, 1, 1)), ([-1, -2], "Concat", ())] + block(c, c3, lat, allk)
        tops.append(len(L) - 1)
    feats = [tops[2]]
    for cout, other, (c, c3) in ((o4, tops[1], (256, 128)), (o5, tops[0], (384, 192)), (o6, n6, (512, 256))):
        L += dn(cout) + [([-1, other], "Concat", ())] + block(c, c3, cout, allk)
        feats.append(len(L) - 1)
    n0 = len(L)
    L += [(f, "Conv", (2 * w, 3, 1)) for f, w in zip(feats, outs)]
    L.append(([n0, n0 + 1, n0 + 2, n0 + 3], "IDetect4", ()))
    return L


class YOLOv7P6(o7.YOLOv7):
    def __init__(self, scale="w6", nc=80, anchors=None):
        nn.Module.__init__(self)
        anchors = anchors or P6_ANCHORS
        ch, mods, self.froms = [3], [], []
        for i, (f, kind, a) in enumerate(p6_cfg(scale)):
            f = [i + j if j < 0 else j for j in (f if isinstance(f, list) else [f])]
            cin = [ch[j + 1] for j in f]
            if kind == "Conv":
                m, c = o7.Conv(cin[0], a[0], a[1], a[2]), a[0]
            elif kind == "DownC":
                m, c = DownC(cin[0], a[0]), a[0]
            elif kind == "SPPCSPC":
                m, c = o7.SPPCSPC(cin[0], a[0]), a[0]
            elif kind == "IDetect4":
                m, c = IDetect4(nc, cin, anchors), 0
            elif kind == "Concat":
                m, c = o7.Concat(), sum(cin)
            elif kind == "Shortcut":
                m, c = Shortcut(), cin[0]
            elif kind == "ReOrg":
                m, c = ReOrg(), 4 * cin[0]
            else:
                m, c = {"Up": o7.Up}[kind](), cin[0]
            mods.append(m)
            ch.append(c)
            self.froms.append(f)
        self.model = nn.ModuleList(mods)


def build(sd: dict, scale="w6", nc=80, anchors=None) -> YOLOv7P6:
    model = YOLOv7P6(scale, nc, anchors)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)).clone() for k, v in sd.items()}, strict=True)
    return model.eval()
