"""fp32 torch-CPU restatement of YOLOv6-Lite-S/M/L (meituan/YOLOv6 release 0.4.0, configs/yolov6_lite/yolov6_lite_{s,m,l}.py:
Lite_EffiBackbone, Lite_EffiNeck, Lite_EffideHead) in training form -- ConvBNHS / ConvBN with their BatchNorms, DPBlock with conv biases
and BatchNorms, SEBlock, channel shuffle -- and an upstream-style `fuse()` (conv + BN -> conv with bias) for export.  Test infrastructure
only.  Module names are upstream's, so the packer's seeded weights load here.  Not pinned by any upstream file (none can be obtained
here): the anchors of the graph are the published parameter counts (tests/test_yolov6_lite_cpu.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

import adas_b200  # noqa: F401
from adas_b200 import plan


def _bn(c):
    return nn.BatchNorm2d(c, eps=1e-3, momentum=0.03)           # upstream initialize_weights sets eps = 1e-3


class ConvModule(nn.Module):
    def __init__(self, c1, c2, k, s, groups=1, act=True):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, k // 2, groups=groups, bias=False)
        self.bn = _bn(c2)
        self.act = nn.Hardswish() if act else None

    def forward(self, x):
        x = self.conv(x) if self.bn is None else self.bn(self.conv(x))
        return x if self.act is None else self.act(x)


class ConvBN(nn.Module):
    """ConvBNHS (act) / ConvBN (no act): `block` = ConvModule."""
    def __init__(self, c1, c2, k=1, s=1, groups=1, act=True):
        super().__init__()
        self.block = ConvModule(c1, c2, k, s, groups, act)

    def forward(self, x):
        return self.block(x)


class SEBlock(nn.Module):
    def __init__(self, c, reduction=4):
        super().__init__()
        self.conv1 = nn.Conv2d(c, c // reduction, 1)
        self.conv2 = nn.Conv2d(c // reduction, c, 1)

    def forward(self, x):
        g = F.hardsigmoid(self.conv2(F.relu(self.conv1(x.mean((2, 3), keepdim=True)))))
        return x * g


def channel_shuffle(x, groups=2):
    b, c, h, w = x.shape
    return x.view(b, groups, c // groups, h, w).transpose(1, 2).reshape(b, c, h, w)


class BlockS1(nn.Module):
    def __init__(self, cin, mid, cout):
        super().__init__()
        self.conv_pw_1 = ConvBN(cin // 2, mid, 1)
        self.conv_dw_1 = ConvBN(mid, mid, 3, 1, mid, act=False)
        self.se = SEBlock(mid)
        self.conv_1 = ConvBN(mid, cout // 2, 1)

    def forward(self, x):
        x1, x2 = x.chunk(2, 1)
        return channel_shuffle(torch.cat([x1, self.conv_1(self.se(self.conv_dw_1(self.conv_pw_1(x2))))], 1))


class BlockS2(nn.Module):
    def __init__(self, cin, mid, cout):
        super().__init__()
        self.conv_dw_1 = ConvBN(cin, cin, 3, 2, cin, act=False)
        self.conv_1 = ConvBN(cin, cout // 2, 1)
        self.conv_pw_2 = ConvBN(cin, mid // 2, 1)
        self.conv_dw_2 = ConvBN(mid // 2, mid // 2, 3, 2, mid // 2, act=False)
        self.se = SEBlock(mid // 2)
        self.conv_2 = ConvBN(mid // 2, cout // 2, 1)
        self.conv_dw_3 = ConvBN(cout, cout, 3, 1, cout)
        self.conv_pw_3 = ConvBN(cout, cout, 1)

    def forward(self, x):
        a = self.conv_1(self.conv_dw_1(x))
        b = self.conv_2(self.se(self.conv_dw_2(self.conv_pw_2(x))))
        return self.conv_pw_3(self.conv_dw_3(torch.cat([a, b], 1)))


class DPBlock(nn.Module):
    def __init__(self, c, k=5, s=1):
        super().__init__()
        self.conv_dw_1 = nn.Conv2d(c, c, k, s, (k - 1) // 2, groups=c)
        self.bn_1 = _bn(c)
        self.conv_pw_1 = nn.Conv2d(c, c, 1)
        self.bn_2 = _bn(c)

    def forward(self, x):
        x = self.conv_dw_1(x) if self.bn_1 is None else self.bn_1(self.conv_dw_1(x))
        x = F.hardswish(x)
        x = self.conv_pw_1(x) if self.bn_2 is None else self.bn_2(self.conv_pw_1(x))
        return F.hardswish(x)


class DarknetBlock(nn.Module):
    def __init__(self, c, k):
        super().__init__()
        self.conv_1 = ConvBN(c, c, 1)
        self.conv_2 = DPBlock(c, k)

    def forward(self, x):
        return self.conv_2(self.conv_1(x))


class CSPBlock(nn.Module):
    def __init__(self, cin, cout, k=5):
        super().__init__()
        m = cout // 2
        self.conv_1 = ConvBN(cin, m, 1)
        self.conv_2 = ConvBN(cin, m, 1)
        self.conv_3 = ConvBN(2 * m, cout, 1)
        self.blocks = DarknetBlock(m, k)

    def forward(self, x):
        return self.conv_3(torch.cat([self.blocks(self.conv_1(x)), self.conv_2(x)], 1))


class Backbone(nn.Module):
    def __init__(self, out, mid):
        super().__init__()
        self.conv_0 = ConvBN(3, out[0], 3, 2)
        for i, n in enumerate(plan.YOLOV6_LITE_BLOCKS):
            blocks = [BlockS2(out[i], mid[i + 1], out[i + 1])] + [BlockS1(out[i + 1], mid[i + 1], out[i + 1]) for _ in range(n - 1)]
            setattr(self, f"lite_effiblock_{i + 1}", nn.Sequential(*blocks))

    def forward(self, x):
        x = self.conv_0(x)
        feats = []
        for i in range(4):
            x = getattr(self, f"lite_effiblock_{i + 1}")(x)
            if i:
                feats.append(x)
        return feats


class Neck(nn.Module):
    def __init__(self, neck_in, u):
        super().__init__()
        self.reduce_layer0 = ConvBN(neck_in[0], u, 1)
        self.reduce_layer1 = ConvBN(neck_in[1], u, 1)
        self.reduce_layer2 = ConvBN(neck_in[2], u, 1)
        self.Csp_p4, self.Csp_p3, self.Csp_n3, self.Csp_n4 = (CSPBlock(2 * u, u, 5) for _ in range(4))
        self.downsample2, self.downsample1 = DPBlock(u, 5, 2), DPBlock(u, 5, 2)
        self.p6_conv_1, self.p6_conv_2 = DPBlock(u, 5, 2), DPBlock(u, 5, 2)

    def forward(self, xs):
        x2, x1, x0 = xs
        up = lambda t: F.interpolate(t, scale_factor=2.0, mode="nearest")         # noqa: E731
        fpn_out0 = self.reduce_layer0(x0)
        f_out1 = self.Csp_p4(torch.cat([up(fpn_out0), self.reduce_layer1(x1)], 1))
        pan_out3 = self.Csp_p3(torch.cat([up(f_out1), self.reduce_layer2(x2)], 1))
        pan_out2 = self.Csp_n3(torch.cat([self.downsample2(pan_out3), f_out1], 1))
        pan_out1 = self.Csp_n4(torch.cat([self.downsample1(pan_out2), fpn_out0], 1))
        pan_out0 = self.p6_conv_1(fpn_out0) + self.p6_conv_2(pan_out1)
        return [pan_out3, pan_out2, pan_out1, pan_out0]


class Detect(nn.Module):
    def __init__(self, nc, u):
        super().__init__()
        self.nc = nc
        self.stems = nn.ModuleList(DPBlock(u, 5) for _ in range(4))
        self.cls_convs = nn.ModuleList(DPBlock(u, 5) for _ in range(4))
        self.reg_convs = nn.ModuleList(DPBlock(u, 5) for _ in range(4))
        self.cls_preds = nn.ModuleList(nn.Conv2d(u, nc, 1) for _ in range(4))
        self.reg_preds = nn.ModuleList(nn.Conv2d(u, 4, 1) for _ in range(4))

    def forward(self, xs):
        cls, reg, anchors, strides = [], [], [], []
        for i, x in enumerate(xs):
            b, _, h, w = x.shape
            t = self.stems[i](x)
            cls.append(torch.sigmoid(self.cls_preds[i](self.cls_convs[i](t))).reshape(b, self.nc, h * w))
            reg.append(self.reg_preds[i](self.reg_convs[i](t)).reshape(b, 4, h * w))
            yv, xv = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
            anchors.append(torch.stack((xv, yv), -1).view(-1, 2) + 0.5)
            strides.append(torch.full((h * w, 1), float(8 << i)))
        cls = torch.cat(cls, -1).permute(0, 2, 1)
        reg = torch.cat(reg, -1).permute(0, 2, 1)
        a, st = torch.cat(anchors), torch.cat(strides)
        x1y1, x2y2 = a - reg[..., :2], a + reg[..., 2:]
        box = torch.cat(((x1y1 + x2y2) / 2, x2y2 - x1y1), -1) * st
        return torch.cat((box, torch.ones_like(box[..., :1]), cls), -1)            # [b, A, 5 + nc]


class YOLOv6Lite(nn.Module):
    def __init__(self, scale="s", nc=80):
        super().__init__()
        out, mid, neck_in = plan.yolov6_lite_widths(scale)
        self.backbone = Backbone(out, mid)
        self.neck = Neck(neck_in, plan.YOLOV6_LITE_NECK)
        self.detect = Detect(nc, plan.YOLOV6_LITE_NECK)

    def forward(self, x):
        return self.detect(self.neck(self.backbone(x)))

    @torch.no_grad()
    def fuse(self):
        """As upstream before export: every conv + BatchNorm becomes one conv with a bias (folded in fp64)."""
        def fold(conv, bn):
            s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
            cb = conv.bias.double() if conv.bias is not None else torch.zeros_like(s)
            f = nn.Conv2d(conv.in_channels, conv.out_channels, conv.kernel_size, conv.stride, conv.padding, groups=conv.groups, bias=True)
            f.weight.data = (conv.weight.double() * s[:, None, None, None]).float()
            f.bias.data = ((cb - bn.running_mean.double()) * s + bn.bias.double()).float()
            return f
        for m in self.modules():
            if isinstance(m, ConvModule) and m.bn is not None:
                m.conv, m.bn = fold(m.conv, m.bn), None
            elif isinstance(m, DPBlock) and m.bn_1 is not None:
                m.conv_dw_1, m.bn_1 = fold(m.conv_dw_1, m.bn_1), None
                m.conv_pw_1, m.bn_2 = fold(m.conv_pw_1, m.bn_2), None
        return self


def build(sd: dict, scale="s", nc=80) -> YOLOv6Lite:
    """The oracle with `sd` loaded (every key present: strict)."""
    model = YOLOv6Lite(scale, nc)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)).clone() for k, v in sd.items()}, strict=True)
    return model.eval()


def fused_state_dict(model: YOLOv6Lite) -> dict:
    return {k: v.numpy().copy() for k, v in model.fuse().state_dict().items()}
