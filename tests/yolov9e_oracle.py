"""fp32 torch-CPU restatement of YOLOv9-E (the converted GELAN-E graph, upstream `models/detect/gelan-e.yaml`, release v0.1) in training
form, built from the blocks of yolov9_oracle.py.  CBLinear and CBFuse are written as upstream writes them (a biased 1x1 conv split
into groups; `F.interpolate(size=...)` nearest, summed, plus the target), and `fuse()` re-parameterises RepConvN and folds Conv + BN as
upstream does.  Module names are upstream's (`model.<i>.…`, model.0 the Silence layer, head `model.42`), so the packer's seeded
weights load here with strict=True.  Test infrastructure only; the anchors of the graph are the published parameter / FLOP counts
(tests/test_yolov9e_cpu.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

import yolov9_oracle as o9
from adas_b200 import plan


class Silence(nn.Module):
    def forward(self, x):
        return x


class CBLinear(nn.Module):
    def __init__(self, c1, c2s):
        super().__init__()
        self.c2s = list(c2s)
        self.conv = nn.Conv2d(c1, sum(c2s), 1, 1, 0, bias=True)

    def forward(self, x):
        return self.conv(x).split(self.c2s, dim=1)


class CBFuse(nn.Module):
    def __init__(self, idx):
        super().__init__()
        self.idx = list(idx)

    def forward(self, xs):
        target_size = xs[-1].shape[2:]
        res = [F.interpolate(x[self.idx[i]], size=target_size, mode="nearest") for i, x in enumerate(xs[:-1])]
        return torch.sum(torch.stack(res + xs[-1:]), dim=0)


class Upsample(nn.Module):
    def forward(self, x):
        return F.interpolate(x, scale_factor=2.0, mode="nearest")


class YOLOv9E(nn.Module):
    def __init__(self, nc=80):
        super().__init__()
        c = plan.YOLOV9_E
        el, (h32, h35, h38, h41), (s2, s3), (d36, d39) = c["elan"], c["head"], c["spp"], c["head_downs"]
        (c0, c1), d, cbl = c["stem"], c["downs"], c["cbl"]
        self.model = nn.ModuleList([
            Silence(),                                                                     # 0
            o9.Conv(3, c0, 3, 2), o9.Conv(c0, c1, 3, 2), o9.ELAN(c1, *el[0]),               # 1, 2, 3
            o9.ADown(el[0][0], d[0]), o9.ELAN(d[0], *el[1]),                               # 4, 5
            o9.ADown(el[1][0], d[1]), o9.ELAN(d[1], *el[2]),                               # 6, 7
            o9.ADown(el[2][0], d[2]), o9.ELAN(d[2], *el[3]),                               # 8, 9
            CBLinear(c0, cbl[0]), CBLinear(el[0][0], cbl[1]), CBLinear(el[1][0], cbl[2]),  # 10, 11, 12
            CBLinear(el[2][0], cbl[3]), CBLinear(el[3][0], cbl[4]),                        # 13, 14
            o9.Conv(3, c0, 3, 2), CBFuse([0, 0, 0, 0, 0]),                                 # 15, 16
            o9.Conv(c0, c1, 3, 2), CBFuse([1, 1, 1, 1]),                                   # 17, 18
            o9.ELAN(c1, *el[0]), o9.ADown(el[0][0], d[0]), CBFuse([2, 2, 2]),              # 19, 20, 21
            o9.ELAN(d[0], *el[1]), o9.ADown(el[1][0], d[1]), CBFuse([3, 3]),               # 22, 23, 24
            o9.ELAN(d[1], *el[2]), o9.ADown(el[2][0], d[2]), CBFuse([4]),                  # 25, 26, 27
            o9.ELAN(d[2], *el[3]),                                                         # 28
            o9.SPPELAN(el[3][0], s2, s3), Upsample(), nn.Identity(),                       # 29, 30, 31 (Concat)
            o9.ELAN(s2 + el[2][0], *h32), Upsample(), nn.Identity(),                       # 32, 33, 34
            o9.ELAN(h32[0] + el[1][0], *h35), o9.ADown(h35[0], d36), nn.Identity(),        # 35, 36, 37
            o9.ELAN(d36 + h32[0], *h38), o9.ADown(h38[0], d39), nn.Identity(),             # 38, 39, 40
            o9.ELAN(d39 + s2, *h41),                                                       # 41
            o9.DDetect(nc, (h35[0], h38[0], h41[0])),                                      # 42
        ])

    def forward(self, x):
        m = self.model
        x0 = m[0](x)
        x1 = m[1](x0)
        x3 = m[3](m[2](x1))
        x5 = m[5](m[4](x3))
        x7 = m[7](m[6](x5))
        x9 = m[9](m[8](x7))
        l10, l11, l12, l13, l14 = m[10](x1), m[11](x3), m[12](x5), m[13](x7), m[14](x9)
        y = m[16]([l10, l11, l12, l13, l14, m[15](x0)])
        y = m[18]([l11, l12, l13, l14, m[17](y)])
        y = m[21]([l12, l13, l14, m[20](m[19](y))])
        y22 = m[22](y)
        y = m[24]([l13, l14, m[23](y22)])
        y25 = m[25](y)
        y = m[27]([l14, m[26](y25)])
        y28 = m[28](y)
        p29 = m[29](y28)
        p32 = m[32](torch.cat((m[30](p29), y25), 1))
        p35 = m[35](torch.cat((m[33](p32), y22), 1))
        p38 = m[38](torch.cat((m[36](p35), p32), 1))
        p41 = m[41](torch.cat((m[39](p38), p29), 1))
        return m[42]([p35, p38, p41])

    def fuse(self):
        for mod in list(self.modules()):
            if isinstance(mod, o9.RepConvN):
                mod.fuse()
        for mod in list(self.modules()):
            if isinstance(mod, o9.Conv) and hasattr(mod, "bn"):
                mod.fuse()
        return self


def build(sd, nc=80) -> YOLOv9E:
    """The training-form network with the seeded (or checkpoint) state_dict loaded strictly."""
    m = YOLOv9E(nc)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)).clone() for k, v in sd.items()}, strict=True)
    return m.eval()
