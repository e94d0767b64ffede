"""fp32 torch-CPU restatement of YOLOv10-N / S / M / B / L / X (ultralytics 8.2.41 `yolov10{n,s,m,b,l,x}.yaml`) in training form --
Conv + BN, RepVGGDW with both branches -- with the one-to-one head only, and an upstream-style `fuse()` (Conv-BN fuse, RepVGGDW folded
to one 7x7) for export.  Test infrastructure only.  Module names are upstream's (`model.<i>.…`, head `model.23.one2one_cv2/3`), so the
packer's seeded weights load here with strict=True.  Written from the architecture; the anchors of the graph are the published
parameter / FLOP counts (tests/test_yolov10_cpu.py)."""
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
from yolov9_oracle import Conv  # noqa: E402  (Conv2d + BN eps 1e-3 + SiLU, groups, fuse())


class RepVGGDW(nn.Module):
    """SiLU(dw7x7+BN (x) + dw3x3+BN (x)); fuse(): one 7x7 `conv` with a bias."""
    def __init__(self, c):
        super().__init__()
        self.conv = Conv(c, c, 7, g=c, act=False)
        self.conv1 = Conv(c, c, 3, g=c, act=False)
        self.act = nn.SiLU()

    def forward(self, x):
        if hasattr(self, "conv1"):
            return self.act(self.conv(x) + self.conv1(x))
        return self.act(self.conv(x))

    def fuse(self):
        self.conv.fuse()
        self.conv1.fuse()
        c = self.conv.conv
        w = c.weight.detach().clone()
        w[:, :, 2:5, 2:5] += self.conv1.conv.weight.detach()
        f = nn.Conv2d(c.in_channels, c.out_channels, 7, 1, 3, groups=c.groups, bias=True)
        f.weight.data, f.bias.data = w, c.bias.detach() + self.conv1.conv.bias.detach()
        self.conv = f
        del self.conv1


class CIB(nn.Module):
    def __init__(self, c, shortcut, lk):
        super().__init__()
        self.cv1 = nn.Sequential(Conv(c, c, 3, g=c), Conv(c, 2 * c, 1), RepVGGDW(2 * c) if lk else Conv(2 * c, 2 * c, 3, g=2 * c),
                                 Conv(2 * c, c, 1), Conv(c, c, 3, g=c))
        self.add = shortcut

    def forward(self, x):
        return x + self.cv1(x) if self.add else self.cv1(x)


class C2f(nn.Module):
    """C2f (cib None) or C2fCIB (cib = lk)."""
    def __init__(self, c1, c2, n, shortcut, cib=None):
        super().__init__()
        self.c = c2 // 2
        self.cv1 = Conv(c1, 2 * self.c, 1)
        self.cv2 = Conv((2 + n) * self.c, c2, 1)
        if cib is None:
            self.m = nn.ModuleList(Bottleneck(self.c, shortcut) for _ in range(n))
        else:
            self.m = nn.ModuleList(CIB(self.c, shortcut, cib) for _ in range(n))

    def forward(self, x):
        y = list(self.cv1(x).chunk(2, 1))
        y.extend(m(y[-1]) for m in self.m)
        return self.cv2(torch.cat(y, 1))


class Bottleneck(nn.Module):
    def __init__(self, c, shortcut):
        super().__init__()
        self.cv1, self.cv2 = Conv(c, c, 3), Conv(c, c, 3)
        self.add = shortcut

    def forward(self, x):
        y = self.cv2(self.cv1(x))
        return x + y if self.add else y


class SCDown(nn.Module):
    def __init__(self, c1, c2):
        super().__init__()
        self.cv1 = Conv(c1, c2, 1)
        self.cv2 = Conv(c2, c2, 3, 2, g=c2, act=False)

    def forward(self, x):
        return self.cv2(self.cv1(x))


class SPPF(nn.Module):
    def __init__(self, c1, c2):
        super().__init__()
        c_ = c1 // 2
        self.cv1, self.cv2 = Conv(c1, c_, 1), Conv(4 * c_, c2, 1)

    def forward(self, x):
        y = [self.cv1(x)]
        for _ in range(3):
            y.append(F.max_pool2d(y[-1], 5, 1, 2))
        return self.cv2(torch.cat(y, 1))


class Attention(nn.Module):
    """nh = dim // 64 heads, hd = dim // nh, kd = hd // 2; qkv channels per head [q kd | k kd | v hd]."""
    def __init__(self, dim):
        super().__init__()
        self.nh, self.kd, self.hd, _ = plan.yolov10_attention_dims(dim)
        self.scale = self.kd ** -0.5
        self.qkv = Conv(dim, dim + 2 * self.nh * self.kd, 1, act=False)
        self.proj = Conv(dim, dim, 1, act=False)
        self.pe = Conv(dim, dim, 3, g=dim, act=False)
        self.round = lambda t: t                  # fp16 emulation hook (forward_fp16_emulated)

    def qkv_split(self, x):
        B, C, H, W = x.shape
        qkv = self.round(self.qkv(x)).view(B, self.nh, 2 * self.kd + self.hd, H * W)
        return qkv.split([self.kd, self.kd, self.hd], dim=2)

    def forward(self, x):
        B, C, H, W = x.shape
        q, k, v = self.qkv_split(x)
        attn = ((q.transpose(-2, -1) @ k) * self.scale).softmax(dim=-1)
        a = self.round((v @ attn.transpose(-2, -1)).view(B, C, H, W))
        return self.proj(a + self.pe(v.reshape(B, C, H, W)))


class PSA(nn.Module):
    def __init__(self, c1):
        super().__init__()
        self.c = c1 // 2
        self.cv1, self.cv2 = Conv(c1, 2 * self.c, 1), Conv(2 * self.c, c1, 1)
        self.attn = Attention(self.c)
        self.ffn = nn.Sequential(Conv(self.c, 2 * self.c, 1), Conv(2 * self.c, self.c, 1, act=False))

    def forward(self, x):
        a, b = self.cv1(x).split((self.c, self.c), dim=1)
        b = b + self.attn(b)
        b = b + self.ffn(b)
        return self.cv2(torch.cat((a, b), 1))


class V10Detect(nets.DetectV8):
    """The one-to-one branch of v10Detect; YOLOv8's decode (16-bin DFL, xywh, sigmoid scores)."""
    def __init__(self, nc, ch):
        nn.Module.__init__(self)
        self.nc, self.reg_max = nc, 16
        c2, c3 = max(16, ch[0] // 4, 64), max(ch[0], min(nc, 100))
        self.one2one_cv2 = nn.ModuleList(nn.Sequential(Conv(x, c2, 3), Conv(c2, c2, 3), nn.Conv2d(c2, 64, 1)) for x in ch)
        self.one2one_cv3 = nn.ModuleList(nn.Sequential(nn.Sequential(Conv(x, x, 3, g=x), Conv(x, c3, 1)),
                                                       nn.Sequential(Conv(c3, c3, 3, g=c3), Conv(c3, c3, 1)), nn.Conv2d(c3, nc, 1)) for x in ch)
        self.strides = (8.0, 16.0, 32.0)

    @property
    def cv2(self):
        return self.one2one_cv2

    @property
    def cv3(self):
        return self.one2one_cv3


class YOLOv10(nn.Module):
    def __init__(self, scale="n", nc=80):
        super().__init__()
        d, w, mc = plan.YOLOV10_SCALES[scale]
        cibs = plan.YOLOV10_CIB[scale]
        ch = lambda c: plan._v8_ch(c, w, mc)
        n = lambda k: plan._v8_n(k, d)
        c1, c2, c3, c4, c5 = ch(64), ch(128), ch(256), ch(512), ch(1024)
        f = lambda li, ci, co, k, sc: C2f(ci, co, n(k), sc or li in cibs, cibs.get(li))
        I = nn.Identity
        self.model = nn.ModuleList([
            Conv(3, c1, 3, 2), Conv(c1, c2, 3, 2), f(2, c2, c2, 3, True), Conv(c2, c3, 3, 2), f(4, c3, c3, 6, True), SCDown(c3, c4),
            f(6, c4, c4, 6, True), SCDown(c4, c5), f(8, c5, c5, 3, True), SPPF(c5, c5), PSA(c5), I(), I(), f(13, c5 + c4, c4, 3, False),
            I(), I(), f(16, c4 + c3, c3, 3, False), Conv(c3, c3, 3, 2), I(), f(19, c3 + c4, c4, 3, False), SCDown(c4, c4), I(),
            f(22, c4 + c5, c5, 3, False), V10Detect(nc, (c3, c4, c5)),
        ])

    def forward(self, x):
        m = self.model
        up = lambda t: F.interpolate(t, scale_factor=2.0, mode="nearest")
        x = m[2](m[1](m[0](x)))
        p3 = m[4](m[3](x))
        p4 = m[6](m[5](p3))
        p5 = m[10](m[9](m[8](m[7](p4))))
        h13 = m[13](torch.cat((up(p5), p4), 1))
        h16 = m[16](torch.cat((up(h13), p3), 1))
        h19 = m[19](torch.cat((m[17](h16), h13), 1))
        h22 = m[22](torch.cat((m[20](h19), p5), 1))
        return m[23]([h16, h19, h22])

    def fuse(self):
        for mod in list(self.modules()):
            if isinstance(mod, RepVGGDW):
                mod.fuse()
        for mod in list(self.modules()):
            if isinstance(mod, Conv) and hasattr(mod, "bn"):
                mod.fuse()
        return self


def build(sd, scale="n", nc=80) -> YOLOv10:
    """The training-form network with the seeded (or checkpoint) state_dict loaded strictly."""
    m = YOLOv10(scale, nc)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)).clone() for k, v in sd.items()}, strict=True)
    return m.eval()


def fused_params(model: nn.Module) -> int:
    """Parameters of the fused one-to-one graph plus the 16 weights of upstream's fixed DFL conv."""
    return sum(p.numel() for p in model.parameters()) + 16


def flops(model: nn.Module, h=640, w=640) -> int:
    """2 * MAC of every conv at h x w (depthwise convs at their grouped MACs), from forward hooks."""
    total = [0]

    def hook(mod, inp, out):
        total[0] += 2 * out.numel() * (mod.in_channels // mod.groups) * mod.kernel_size[0] * mod.kernel_size[1]

    hs = [mm.register_forward_hook(hook) for mm in model.modules() if isinstance(mm, nn.Conv2d)]
    with torch.no_grad():
        model(torch.zeros(1, 3, h, w))
    for hh in hs:
        hh.remove()
    return total[0]


def forward_fp16_emulated(model: YOLOv10, x: torch.Tensor) -> torch.Tensor:
    """The engine's fp16 storage points on the CPU: every conv's input rounded to fp16 (oracle.nets.forward_fp16_emulated) and, in
    PSA, the qkv conv's output (q, k, v) and the attention output as well."""
    rnd = lambda t: t.half().float()
    atts = [m for m in model.modules() if isinstance(m, Attention)]
    for a in atts:
        a.round = rnd
    try:
        return nets.forward_fp16_emulated(model, x)
    finally:
        for a in atts:
            a.round = lambda t: t
