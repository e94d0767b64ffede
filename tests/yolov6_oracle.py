"""fp32 torch-CPU restatement of YOLOv6 3.0 N/S/M/L (meituan/YOLOv6 release 0.4.0, configs/yolov6{n,s,m,l}.py) in training form --
RepVGG blocks with their three branches, BottleRep with its learned `alpha`, BiFusion with ConvTranspose2d, EffiDeHead with and without
DFL plus the anchor-aided `_ab` branch of training checkpoints -- and an upstream-style `fuse()` (RepVGG re-parameterisation, Conv-BN
fuse) for export.  Test infrastructure only.  Module names are upstream's (`backbone.*`, `neck.*`, `detect.*`), so the packer's seeded
weights load here.  Not pinned by any upstream file (none can be obtained here): the anchors of the graph are the published parameter /
FLOP counts (tests/test_yolov6_cpu.py)."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

SCALES = {"n": (0.33, 0.25), "s": (0.33, 0.50), "m": (0.60, 0.75), "l": (1.0, 1.0)}
CSP_E = {"m": 2 / 3, "l": 1 / 2}


def _bn(c):
    return nn.BatchNorm2d(c, eps=1e-3, momentum=0.03)           # upstream initialize_weights sets eps = 1e-3


class ConvModule(nn.Module):
    def __init__(self, c1, c2, k, s, act):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, k // 2, bias=False)
        self.bn = _bn(c2)
        self.act = act

    def forward(self, x):
        x = self.conv(x) if self.bn is None else self.bn(self.conv(x))
        return x if self.act is None else self.act(x)


class ConvBNAct(nn.Module):
    """ConvBNReLU / ConvBNSiLU: `block` = ConvModule."""
    def __init__(self, c1, c2, k=3, s=1, act="relu"):
        super().__init__()
        self.block = ConvModule(c1, c2, k, s, nn.ReLU() if act == "relu" else nn.SiLU())

    def forward(self, x):
        return self.block(x)


class RepVGGBlock(nn.Module):
    def __init__(self, c1, c2, k=3, s=1, act="relu"):
        super().__init__()
        self.nonlinearity = nn.ReLU() if act == "relu" else nn.SiLU()
        self.rbr_identity = _bn(c1) if c1 == c2 and s == 1 else None
        self.rbr_dense = ConvModule(c1, c2, 3, s, None)
        self.rbr_1x1 = ConvModule(c1, c2, 1, s, None)
        self.rbr_1x1.conv.padding = (0, 0)

    def forward(self, x):
        if hasattr(self, "rbr_reparam"):
            return self.nonlinearity(self.rbr_reparam(x))
        idt = 0 if self.rbr_identity is None else self.rbr_identity(x)
        return self.nonlinearity(self.rbr_dense(x) + self.rbr_1x1(x) + idt)


class BottleRep(nn.Module):
    def __init__(self, c1, c2, basic):
        super().__init__()
        self.conv1, self.conv2 = basic(c1, c2), basic(c2, c2)
        self.alpha = nn.Parameter(torch.ones(1))

    def forward(self, x):
        return self.conv2(self.conv1(x)) + self.alpha * x


class RepBlock(nn.Module):
    def __init__(self, c1, c2, n, basic, bottle=False):
        super().__init__()
        if bottle:
            n = n // 2
            self.conv1 = BottleRep(c1, c2, basic)
            self.block = nn.Sequential(*(BottleRep(c2, c2, basic) for _ in range(n - 1))) if n > 1 else None
        else:
            self.conv1 = basic(c1, c2)
            self.block = nn.Sequential(*(basic(c2, c2) for _ in range(n - 1))) if n > 1 else None

    def forward(self, x):
        x = self.conv1(x)
        return x if self.block is None else self.block(x)


class BepC3(nn.Module):
    def __init__(self, c1, c2, n, e, basic, act):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1, self.cv2 = ConvBNAct(c1, c_, 1, 1, act), ConvBNAct(c1, c_, 1, 1, act)
        self.cv3 = ConvBNAct(2 * c_, c2, 1, 1, act)
        self.m = RepBlock(c_, c_, n, basic, bottle=True)

    def forward(self, x):
        return self.cv3(torch.cat((self.m(self.cv1(x)), self.cv2(x)), 1))


def _pool(x):
    return F.max_pool2d(x, 5, 1, 2)


class CSPSPPFModule(nn.Module):
    def __init__(self, c1, c2, act):
        super().__init__()
        c_ = c2 // 2
        self.cv1, self.cv2 = ConvBNAct(c1, c_, 1, 1, act), ConvBNAct(c1, c_, 1, 1, act)
        self.cv3, self.cv4 = ConvBNAct(c_, c_, 3, 1, act), ConvBNAct(c_, c_, 1, 1, act)
        self.cv5, self.cv6 = ConvBNAct(4 * c_, c_, 1, 1, act), ConvBNAct(c_, c_, 3, 1, act)
        self.cv7 = ConvBNAct(2 * c_, c2, 1, 1, act)

    def forward(self, x):
        x1 = self.cv4(self.cv3(self.cv1(x)))
        y0 = self.cv2(x)
        y1 = _pool(x1)
        y2 = _pool(y1)
        y3 = self.cv6(self.cv5(torch.cat([x1, y1, y2, _pool(y2)], 1)))
        return self.cv7(torch.cat((y0, y3), 1))


class SPPFModule(nn.Module):
    def __init__(self, c1, c2, act):
        super().__init__()
        c_ = c1 // 2
        self.cv1, self.cv2 = ConvBNAct(c1, c_, 1, 1, act), ConvBNAct(4 * c_, c2, 1, 1, act)

    def forward(self, x):
        x = self.cv1(x)
        y1 = _pool(x)
        y2 = _pool(y1)
        return self.cv2(torch.cat([x, y1, y2, _pool(y2)], 1))


class SimCSPSPPF(nn.Module):
    def __init__(self, c1, c2, act):
        super().__init__()
        self.cspsppf = CSPSPPFModule(c1, c2, act)

    def forward(self, x):
        return self.cspsppf(x)


class SimSPPF(nn.Module):
    def __init__(self, c1, c2, act):
        super().__init__()
        self.sppf = SPPFModule(c1, c2, act)

    def forward(self, x):
        return self.sppf(x)


class Transpose(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.upsample_transpose = nn.ConvTranspose2d(c, c, 2, 2, bias=True)

    def forward(self, x):
        return self.upsample_transpose(x)


class BiFusion(nn.Module):
    def __init__(self, cin, c, act):
        super().__init__()
        self.cv1, self.cv2 = ConvBNAct(cin[0], c, 1, 1, act), ConvBNAct(cin[1], c, 1, 1, act)
        self.cv3 = ConvBNAct(3 * c, c, 1, 1, act)
        self.upsample = Transpose(c)
        self.downsample = ConvBNAct(c, c, 3, 2, act)

    def forward(self, x):
        return self.cv3(torch.cat((self.upsample(x[0]), self.cv1(x[1]), self.downsample(self.cv2(x[2]))), 1))


class Backbone(nn.Module):
    def __init__(self, ch, rep, blk, stage, sppf):
        super().__init__()
        self.stem = blk(3, ch[0], 3, 2)
        for i in range(1, 5):
            mods = [blk(ch[i - 1], ch[i], 3, 2), stage(ch[i], ch[i], rep[i])]
            if i == 4:
                mods.append(sppf(ch[4], ch[4]))
            setattr(self, f"ERBlock_{i + 1}", nn.Sequential(*mods))

    def forward(self, x):
        x = self.ERBlock_2(self.stem(x))
        out = [x]
        for i in (3, 4, 5):
            x = getattr(self, f"ERBlock_{i}")(x)
            out.append(x)
        return out


class Neck(nn.Module):
    def __init__(self, ch, rep, stage, act):
        super().__init__()
        self.reduce_layer0 = ConvBNAct(ch[4], ch[5], 1, 1, act)
        self.Bifusion0 = BiFusion([ch[3], ch[2]], ch[5], act)
        self.Rep_p4 = stage(ch[5], ch[5], rep[5])
        self.reduce_layer1 = ConvBNAct(ch[5], ch[6], 1, 1, act)
        self.Bifusion1 = BiFusion([ch[2], ch[1]], ch[6], act)
        self.Rep_p3 = stage(ch[6], ch[6], rep[6])
        self.downsample2 = ConvBNAct(ch[6], ch[7], 3, 2, act)
        self.Rep_n3 = stage(ch[6] + ch[7], ch[8], rep[7])
        self.downsample1 = ConvBNAct(ch[8], ch[9], 3, 2, act)
        self.Rep_n4 = stage(ch[5] + ch[9], ch[10], rep[8])

    def forward(self, xs):
        x3, x2, x1, x0 = xs
        fpn0 = self.reduce_layer0(x0)
        f_out0 = self.Rep_p4(self.Bifusion0([fpn0, x1, x2]))
        fpn1 = self.reduce_layer1(f_out0)
        pan2 = self.Rep_p3(self.Bifusion1([fpn1, x2, x3]))
        pan1 = self.Rep_n3(torch.cat([self.downsample2(pan2), fpn1], 1))
        pan0 = self.Rep_n4(torch.cat([self.downsample1(pan1), fpn0], 1))
        return [pan2, pan1, pan0]


class Detect(nn.Module):
    """EffiDeHead with the anchor-aided branch of training (cls_preds_ab / reg_preds_ab, 3 anchors), unused at inference."""
    def __init__(self, nc, chs, reg_max, act):
        super().__init__()
        self.nc, self.reg_max = nc, reg_max
        self.stems = nn.ModuleList(ConvBNAct(c, c, 1, 1, act) for c in chs)
        self.cls_convs = nn.ModuleList(ConvBNAct(c, c, 3, 1, act) for c in chs)
        self.reg_convs = nn.ModuleList(ConvBNAct(c, c, 3, 1, act) for c in chs)
        self.cls_preds = nn.ModuleList(nn.Conv2d(c, nc, 1) for c in chs)
        self.reg_preds = nn.ModuleList(nn.Conv2d(c, 4 * (reg_max + 1), 1) for c in chs)
        self.cls_preds_ab = nn.ModuleList(nn.Conv2d(c, nc * 3, 1) for c in chs)
        self.reg_preds_ab = nn.ModuleList(nn.Conv2d(c, 4 * 3, 1) for c in chs)
        self.proj_conv = nn.Conv2d(reg_max + 1, 1, 1, bias=False)
        self.proj = nn.Parameter(torch.linspace(0, reg_max, reg_max + 1), requires_grad=False)
        self.proj_conv.weight = nn.Parameter(self.proj.view(1, reg_max + 1, 1, 1).clone(), requires_grad=False)

    def forward(self, xs):
        cls, reg, anchors, strides = [], [], [], []
        for i, x in enumerate(xs):
            b, _, h, w = x.shape
            t = self.stems[i](x)
            c = torch.sigmoid(self.cls_preds[i](self.cls_convs[i](t)))
            r = self.reg_preds[i](self.reg_convs[i](t))
            if self.reg_max > 0:
                r = r.reshape(b, 4, self.reg_max + 1, h * w).permute(0, 2, 1, 3)
                r = self.proj_conv(F.softmax(r, dim=1))
            cls.append(c.reshape(b, self.nc, h * w))
            reg.append(r.reshape(b, 4, h * w))
            yv, xv = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
            anchors.append(torch.stack((xv, yv), -1).view(-1, 2) + 0.5)
            strides.append(torch.full((h * w, 1), float(8 << i)))
        cls = torch.cat(cls, -1).permute(0, 2, 1)
        reg = torch.cat(reg, -1).permute(0, 2, 1)
        a, st = torch.cat(anchors), torch.cat(strides)
        x1y1, x2y2 = a - reg[..., :2], a + reg[..., 2:]
        box = torch.cat(((x1y1 + x2y2) / 2, x2y2 - x1y1), -1) * st
        return torch.cat((box, torch.ones_like(box[..., :1]), cls), -1)            # [b, 8400, 5 + nc]


class YOLOv6(nn.Module):
    def __init__(self, scale="n", nc=80, act_body=None, act_neck="relu", act_head="silu", reg_max=None):
        super().__init__()
        depth, width = SCALES[scale]
        ch = [int(math.ceil(c * width / 8) * 8) for c in (64, 128, 256, 512, 1024, 256, 128, 128, 256, 256, 512)]
        rep = [max(round(n * depth), 1) if n > 1 else n for n in (1, 6, 12, 18, 6, 12, 12, 12, 12)]
        ab = act_body or ("silu" if scale == "l" else "relu")
        reg_max = (16 if scale in CSP_E else 0) if reg_max is None else reg_max
        if scale == "l":
            blk = lambda c1, c2, k=3, s=1: ConvBNAct(c1, c2, k, s, ab)                 # noqa: E731
        else:
            blk = lambda c1, c2, k=3, s=1: RepVGGBlock(c1, c2, k, s, ab)               # noqa: E731
        if scale in CSP_E:
            stage = lambda c1, c2, n: BepC3(c1, c2, n, CSP_E[scale], blk, ab)          # noqa: E731
            sppf = lambda c1, c2: SimSPPF(c1, c2, ab)                                  # noqa: E731
        else:
            stage = lambda c1, c2, n: RepBlock(c1, c2, n, blk)                         # noqa: E731
            sppf = lambda c1, c2: SimCSPSPPF(c1, c2, ab)                               # noqa: E731
        self.backbone = Backbone(ch, rep, blk, stage, sppf)
        self.neck = Neck(ch, rep, stage, act_neck)
        self.detect = Detect(nc, (ch[6], ch[8], ch[10]), reg_max, act_head)

    def forward(self, x):
        return self.detect(self.neck(self.backbone(x)))

    @torch.no_grad()
    def fuse(self):
        """As upstream before export: RepVGG -> rbr_reparam (3x3 + 1x1 + identity in fp64), ConvModule conv + BN -> conv with bias."""
        def fold(conv, bn):
            w, s = conv.weight.double(), bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
            return w * s[:, None, None, None], bn.bias.double() - bn.running_mean.double() * s
        for m in list(self.modules()):
            if isinstance(m, RepVGGBlock) and not hasattr(m, "rbr_reparam"):
                wd, bd = fold(m.rbr_dense.conv, m.rbr_dense.bn)
                w1, b1 = fold(m.rbr_1x1.conv, m.rbr_1x1.bn)
                wd[:, :, 1, 1] += w1[:, :, 0, 0]
                bd += b1
                if m.rbr_identity is not None:
                    bn = m.rbr_identity
                    s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
                    idx = torch.arange(wd.shape[0])
                    wd[idx, idx, 1, 1] += s
                    bd += bn.bias.double() - bn.running_mean.double() * s
                d = m.rbr_dense.conv
                r = nn.Conv2d(d.in_channels, d.out_channels, 3, d.stride, 1, bias=True)
                r.weight.data, r.bias.data = wd.float(), bd.float()
                m.rbr_reparam = r
                del m.rbr_dense, m.rbr_1x1, m.rbr_identity
        for m in self.modules():
            if isinstance(m, ConvModule) and m.bn is not None:
                w, b = fold(m.conv, m.bn)
                c = m.conv
                f = nn.Conv2d(c.in_channels, c.out_channels, c.kernel_size, c.stride, c.padding, bias=True)
                f.weight.data, f.bias.data = w.float(), b.float()
                m.conv, m.bn = f, None
        return self


AB_KEYS = (".cls_preds_ab.", ".reg_preds_ab.", "detect.proj")


def build(sd: dict, scale="n", nc=80, **kw) -> YOLOv6:
    """The oracle with `sd` loaded.  The packer's seeded state_dict holds what inference reads; the anchor-aided branch and the fixed DFL
    projection (which inference does not read) keep the oracle's own values, every other key must be present."""
    model = YOLOv6(scale, nc, **kw)
    full = model.state_dict()
    missing = [k for k in full if k not in sd]
    assert all(any(a in k for a in AB_KEYS) for k in missing), [k for k in missing if not any(a in k for a in AB_KEYS)][:5]
    sd = {**{k: full[k] for k in missing}, **{k: torch.from_numpy(np.asarray(v)).clone() for k, v in sd.items()}}
    model.load_state_dict(sd, strict=True)
    return model.eval()
