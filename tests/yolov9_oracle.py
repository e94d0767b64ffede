"""fp32 torch-CPU restatement of YOLOv9-T / S / M / C (WongKinYiu/yolov9 release v0.1, the converted GELAN graphs) in training form --
RepConvN with both branches, DDetect with real `groups=4` box convs -- and an upstream-style `fuse()` (RepConvN re-parameterisation,
Conv-BN fuse) for export.  Test infrastructure only.  Module names are upstream's (`model.<i>.…`, head `model.22`), so the packer's
seeded weights load here with strict=True.  Not pinned by any upstream file (none can be obtained here): the anchors of the graph are
the published parameter / FLOP counts (tests/test_yolov9_cpu.py)."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import nets  # noqa: E402

from adas_b200 import plan  # noqa: E402


class Conv(nn.Module):
    """Conv2d (no bias) + BatchNorm2d (eps 1e-3) + SiLU (or no activation); after fuse(), `conv` carries the bias and `bn` is gone."""
    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, act=True):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, k // 2 if p is None else p, groups=g, bias=False)
        self.bn = nn.BatchNorm2d(c2, eps=1e-3, momentum=0.03)
        self.act = nn.SiLU() if act else nn.Identity()

    def forward(self, x):
        return self.act(self.bn(self.conv(x)) if hasattr(self, "bn") else self.conv(x))

    def fuse(self):
        c, bn = self.conv, self.bn
        s = bn.weight.detach().double() / torch.sqrt(bn.running_var.double() + bn.eps)
        f = nn.Conv2d(c.in_channels, c.out_channels, c.kernel_size, c.stride, c.padding, groups=c.groups, bias=True)
        f.weight.data = (c.weight.detach().double() * s.view(-1, 1, 1, 1)).float()
        f.bias.data = (bn.bias.detach().double() - bn.running_mean.double() * s).float()
        self.conv = f
        del self.bn


class RepConvN(nn.Module):
    """act(conv1(x) + conv2(x)): 3x3 and 1x1 Conv + BN without activation, no identity branch.  fuse(): one 3x3 `conv` with a bias."""
    def __init__(self, c1, c2):
        super().__init__()
        self.conv1 = Conv(c1, c2, 3, act=False)
        self.conv2 = Conv(c1, c2, 1, act=False)
        self.act = nn.SiLU()

    def forward(self, x):
        if hasattr(self, "conv"):
            return self.act(self.conv(x))
        return self.act(self.conv1(x) + self.conv2(x))

    def fuse(self):
        self.conv1.fuse()
        self.conv2.fuse()
        c = nn.Conv2d(self.conv1.conv.in_channels, self.conv1.conv.out_channels, 3, 1, 1, bias=True)
        w = self.conv1.conv.weight.detach().clone()
        w[:, :, 1, 1] += self.conv2.conv.weight.detach()[:, :, 0, 0]
        c.weight.data, c.bias.data = w, self.conv1.conv.bias.detach() + self.conv2.conv.bias.detach()
        self.conv = c
        del self.conv1, self.conv2


class RepNBottleneck(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.cv1, self.cv2 = RepConvN(c, c), Conv(c, c, 3)

    def forward(self, x):
        return x + self.cv2(self.cv1(x))


class RepNCSP(nn.Module):
    def __init__(self, c1, c2, n):
        super().__init__()
        c_ = c2 // 2
        self.cv1, self.cv2, self.cv3 = Conv(c1, c_, 1), Conv(c1, c_, 1), Conv(2 * c_, c2, 1)
        self.m = nn.Sequential(*(RepNBottleneck(c_) for _ in range(n)))

    def forward(self, x):
        return self.cv3(torch.cat((self.m(self.cv1(x)), self.cv2(x)), 1))


class ELAN(nn.Module):
    """RepNCSPELAN4(c1, c2, c3, c4, n) or, with n None, ELAN1(c1, c2, c3, c4)."""
    def __init__(self, c1, c2, c3, c4, n):
        super().__init__()
        self.c = c3 // 2
        self.cv1 = Conv(c1, c3, 1)
        if n is None:
            self.cv2, self.cv3 = Conv(c3 // 2, c4, 3), Conv(c4, c4, 3)
        else:
            self.cv2 = nn.Sequential(RepNCSP(c3 // 2, c4, n), Conv(c4, c4, 3))
            self.cv3 = nn.Sequential(RepNCSP(c4, c4, n), Conv(c4, c4, 3))
        self.cv4 = Conv(c3 + 2 * c4, c2, 1)

    def forward(self, x):
        y = list(self.cv1(x).chunk(2, 1))
        y.extend(m(y[-1]) for m in (self.cv2, self.cv3))
        return self.cv4(torch.cat(y, 1))


class AConv(nn.Module):
    def __init__(self, c1, c2):
        super().__init__()
        self.cv1 = Conv(c1, c2, 3, 2, 1)

    def forward(self, x):
        return self.cv1(F.avg_pool2d(x, 2, 1, 0, False, True))


class ADown(nn.Module):
    def __init__(self, c1, c2):
        super().__init__()
        self.c = c2 // 2
        self.cv1 = Conv(c1 // 2, self.c, 3, 2, 1)
        self.cv2 = Conv(c1 // 2, self.c, 1, 1, 0)

    def forward(self, x):
        x1, x2 = F.avg_pool2d(x, 2, 1, 0, False, True).chunk(2, 1)
        return torch.cat((self.cv1(x1), self.cv2(F.max_pool2d(x2, 3, 2, 1))), 1)


class SPPELAN(nn.Module):
    def __init__(self, c1, c2, c3):
        super().__init__()
        self.cv1, self.cv5 = Conv(c1, c3, 1), Conv(4 * c3, c2, 1)

    def forward(self, x):
        y = [self.cv1(x)]
        for _ in range(3):
            y.append(F.max_pool2d(y[-1], 5, 1, 2))
        return self.cv5(torch.cat(y, 1))


class DDetect(nets.DetectV8):
    """YOLOv8's Detect with grouped (g = 4) second and third box convs; decode (16-bin DFL, xywh, sigmoid scores) unchanged."""
    def __init__(self, nc, ch):
        nn.Module.__init__(self)
        self.nc, self.reg_max = nc, 16
        c2, c3 = max(16, ch[0] // 4, 64), max(ch[0], min(nc, 100))
        self.cv2 = nn.ModuleList(nn.Sequential(Conv(x, c2, 3), Conv(c2, c2, 3, g=4), nn.Conv2d(c2, 64, 1, groups=4)) for x in ch)
        self.cv3 = nn.ModuleList(nn.Sequential(Conv(x, c3, 3), Conv(c3, c3, 3), nn.Conv2d(c3, nc, 1)) for x in ch)
        self.strides = (8.0, 16.0, 32.0)


class YOLOv9(nn.Module):
    def __init__(self, scale="c", nc=80):
        super().__init__()
        cfg = plan.YOLOV9[scale]
        d, r, (s2, s3) = cfg["downs"], cfg["r4"], cfg["spp"]
        dn = AConv if cfg["down"] == "aconv" else ADown
        c0, c1 = cfg["stem"]
        l2 = cfg["l2"]
        self.model = nn.ModuleList([
            Conv(3, c0, 3, 2), Conv(c0, c1, 3, 2), ELAN(c1, *l2), dn(l2[0], d[0]), ELAN(d[0], *r[0]),
            dn(r[0][0], d[1]), ELAN(d[1], *r[1]), dn(r[1][0], d[2]), ELAN(d[2], *r[2]), SPPELAN(r[2][0], s2, s3),
            nn.Identity(), nn.Identity(), ELAN(s2 + r[1][0], *r[3]), nn.Identity(), nn.Identity(), ELAN(r[3][0] + r[0][0], *r[4]),
            dn(r[4][0], d[3]), nn.Identity(), ELAN(d[3] + r[3][0], *r[5]), dn(r[5][0], d[4]), nn.Identity(),
            ELAN(d[4] + s2, *r[6]), DDetect(nc, (r[4][0], r[5][0], r[6][0])),
        ])

    def forward(self, x):
        m = self.model
        up = lambda t: F.interpolate(t, scale_factor=2.0, mode="nearest")
        x = m[2](m[1](m[0](x)))
        p3 = m[4](m[3](x))
        p4 = m[6](m[5](p3))
        p5 = m[9](m[8](m[7](p4)))
        h12 = m[12](torch.cat((up(p5), p4), 1))
        h15 = m[15](torch.cat((up(h12), p3), 1))
        h18 = m[18](torch.cat((m[16](h15), h12), 1))
        h21 = m[21](torch.cat((m[19](h18), p5), 1))
        return m[22]([h15, h18, h21])

    def fuse(self):
        for mod in list(self.modules()):
            if isinstance(mod, RepConvN):
                mod.fuse()
        for mod in list(self.modules()):
            if isinstance(mod, Conv) and hasattr(mod, "bn"):
                mod.fuse()
        return self


def build(sd, scale="c", nc=80) -> YOLOv9:
    """The training-form network with the seeded (or checkpoint) state_dict loaded strictly."""
    m = YOLOv9(scale, nc)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)).clone() for k, v in sd.items()}, strict=True)
    return m.eval()


def fused_params(model: nn.Module) -> int:
    """Parameters of the fused graph plus the 16 weights of upstream's fixed DFL conv."""
    return sum(p.numel() for p in model.parameters()) + 16


def flops(model: nn.Module, h=640, w=640) -> int:
    """2 * MAC of every conv at h x w (grouped convs at their grouped MACs), from forward hooks."""
    total = [0]

    def hook(mod, inp, out):
        total[0] += 2 * out.numel() * (mod.in_channels // mod.groups) * mod.kernel_size[0] * mod.kernel_size[1]

    hs = [mm.register_forward_hook(hook) for mm in model.modules() if isinstance(mm, nn.Conv2d)]
    with torch.no_grad():
        model(torch.zeros(1, 3, h, w))
    for hh in hs:
        hh.remove()
    return total[0]
