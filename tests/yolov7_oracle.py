"""fp32 torch-CPU restatement of YOLOv7 and YOLOv7-tiny (P5, cfg/training/yolov7.yaml and yolov7-tiny.yaml) in training form --
RepConv with its three branches, IDetect with ImplicitA / ImplicitM -- plus `fuse()` as upstream does it before exporting.  Test
infrastructure only.  The graph is written as the upstream yaml (from-index, module, arguments), so state_dict keys are upstream's
and the packer's seeded weights load with strict=True.  Not pinned by any upstream file (none can be obtained here): the anchors of
the graph are the published parameter / FLOP counts (tests/test_yolov7_cpu.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

V5_ANCHORS = ((10, 13, 16, 30, 33, 23), (30, 61, 62, 45, 59, 119), (116, 90, 156, 198, 373, 326))
V7_ANCHORS = ((12, 16, 19, 36, 40, 28), (36, 75, 76, 55, 72, 146), (142, 110, 192, 243, 459, 401))


class Conv(nn.Module):
    def __init__(self, c1, c2, k=1, s=1, act=None):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, k // 2, bias=False)
        self.bn = nn.BatchNorm2d(c2, eps=1e-3, momentum=0.03)       # upstream initialize_weights sets eps = 1e-3
        self.act = act() if act is not None else nn.SiLU()

    def forward(self, x):
        return self.act(self.bn(self.conv(x)))


class MP(nn.Module):
    def forward(self, x):
        return nn.functional.max_pool2d(x, 2, 2)


class SP(nn.Module):
    def __init__(self, k):
        super().__init__()
        self.k = k

    def forward(self, x):
        return nn.functional.max_pool2d(x, self.k, 1, self.k // 2)


class Up(nn.Module):
    def forward(self, x):
        return nn.functional.interpolate(x, scale_factor=2, mode="nearest")


class Concat(nn.Module):
    def forward(self, xs):
        return torch.cat(xs, 1)


class SPPCSPC(nn.Module):
    def __init__(self, c1, c2, act=None):
        super().__init__()
        c_ = c2
        self.cv1, self.cv2 = Conv(c1, c_, 1, 1, act), Conv(c1, c_, 1, 1, act)
        self.cv3, self.cv4 = Conv(c_, c_, 3, 1, act), Conv(c_, c_, 1, 1, act)
        self.m = nn.ModuleList(SP(k) for k in (5, 9, 13))
        self.cv5, self.cv6 = Conv(4 * c_, c_, 1, 1, act), Conv(c_, c_, 3, 1, act)
        self.cv7 = Conv(2 * c_, c2, 1, 1, act)

    def forward(self, x):
        x1 = self.cv4(self.cv3(self.cv1(x)))
        y1 = self.cv6(self.cv5(torch.cat([x1] + [m(x1) for m in self.m], 1)))
        return self.cv7(torch.cat((y1, self.cv2(x)), 1))


class RepConv(nn.Module):
    def __init__(self, c1, c2):
        super().__init__()
        self.act = nn.SiLU()
        self.rbr_dense = nn.Sequential(nn.Conv2d(c1, c2, 3, 1, 1, bias=False), nn.BatchNorm2d(c2, eps=1e-3, momentum=0.03))
        self.rbr_1x1 = nn.Sequential(nn.Conv2d(c1, c2, 1, 1, 0, bias=False), nn.BatchNorm2d(c2, eps=1e-3, momentum=0.03))

    def forward(self, x):
        if hasattr(self, "rbr_reparam"):
            return self.act(self.rbr_reparam(x))
        return self.act(self.rbr_dense(x) + self.rbr_1x1(x))


class Implicit(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.implicit = nn.Parameter(torch.zeros(1, c, 1, 1))


class IDetect(nn.Module):
    def __init__(self, nc, ch, anchors):
        super().__init__()
        self.nc, self.no, self.na = nc, nc + 5, 3
        self.m = nn.ModuleList(nn.Conv2d(c, self.no * self.na, 1) for c in ch)
        self.ia = nn.ModuleList(Implicit(c) for c in ch)
        self.im = nn.ModuleList(Implicit(self.no * self.na) for _ in ch)
        self.register_buffer("anchor_grid", torch.tensor(anchors, dtype=torch.float32).view(3, 1, 3, 1, 1, 2), persistent=False)
        self.fused = False

    def forward(self, feats):
        z = []
        for i, x in enumerate(feats):
            x = self.m[i](x) if self.fused else self.m[i](x + self.ia[i].implicit) * self.im[i].implicit
            b, _, ny, nx = x.shape
            y = x.view(b, self.na, self.no, ny, nx).permute(0, 1, 3, 4, 2).contiguous().sigmoid()
            yv, xv = torch.meshgrid(torch.arange(ny, dtype=torch.float32), torch.arange(nx, dtype=torch.float32), indexing="ij")
            grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2)
            xy = (y[..., 0:2] * 2 - 0.5 + grid) * float(8 << i)
            wh = (y[..., 2:4] * 2) ** 2 * self.anchor_grid[i]
            z.append(torch.cat((xy, wh, y[..., 4:]), -1).view(b, -1, self.no))
        return torch.cat(z, 1)                                   # [b, 25200, 5 + nc]


def _elan(i, c, c3, n3, cout, keep, src=-1):
    """a, b 1x1 on the input; n3 chained 3x3 from b; concat of the kept 3x3 outputs (last first), b, a; 1x1 to cout."""
    layers = [(src, "Conv", (c, 1, 1)), (src - 1 if src < 0 else src, "Conv", (c, 1, 1))]
    layers += [(-1, "Conv", (c3, 3, 1)) for _ in range(n3)]
    layers.append(([-1 - (n3 - 1 - j) for j in sorted(keep, reverse=True)] + [-1 - n3, -2 - n3], "Concat", ()))
    layers.append((-1, "Conv", (cout, 1, 1)))
    return layers


def _mp(c, extra=()):
    return [(-1, "MP", ()), (-1, "Conv", (c, 1, 1)), (-3, "Conv", (c, 1, 1)), (-1, "Conv", (c, 3, 2)), ([-1, -3] + list(extra), "Concat", ())]


def yolov7_cfg():
    bk = (1, 3)
    L = [(-1, "Conv", (32, 3, 1)), (-1, "Conv", (64, 3, 2)), (-1, "Conv", (64, 3, 1)), (-1, "Conv", (128, 3, 2))]
    L += _elan(4, 64, 64, 4, 256, bk) + _mp(128) + _elan(17, 128, 128, 4, 512, bk) + _mp(256) + _elan(30, 256, 256, 4, 1024, bk)
    L += _mp(512) + _elan(43, 256, 256, 4, 1024, bk)
    L += [(-1, "SPPCSPC", (512,)), (-1, "Conv", (256, 1, 1)), (-1, "Up", ()), (37, "Conv", (256, 1, 1)), ([-1, -2], "Concat", ())]
    L += _elan(56, 256, 128, 4, 256, range(4))
    L += [(-1, "Conv", (128, 1, 1)), (-1, "Up", ()), (24, "Conv", (128, 1, 1)), ([-1, -2], "Concat", ())]
    L += _elan(68, 128, 64, 4, 128, range(4)) + _mp(128, (63,)) + _elan(81, 256, 128, 4, 256, range(4))
    L += _mp(256, (51,)) + _elan(94, 512, 256, 4, 512, range(4))
    L += [(75, "RepConv", (256,)), (88, "RepConv", (512,)), (101, "RepConv", (1024,)), ([102, 103, 104], "IDetect", ())]
    assert len(L) == 106
    return L


def yolov7_tiny_cfg():
    L = [(-1, "Conv", (32, 3, 2)), (-1, "Conv", (64, 3, 2))]
    L += _elan(2, 32, 32, 2, 64, range(2)) + [(-1, "MP", ())] + _elan(9, 64, 64, 2, 128, range(2)) + [(-1, "MP", ())]
    L += _elan(16, 128, 128, 2, 256, range(2)) + [(-1, "MP", ())] + _elan(23, 256, 256, 2, 512, range(2))
    L += [(-1, "Conv", (256, 1, 1)), (-2, "Conv", (256, 1, 1)), (-1, "SP", (5,)), (-2, "SP", (9,)), (-3, "SP", (13,)),
          ([-1, -2, -3, -4], "Concat", ()), (-1, "Conv", (256, 1, 1)), ([-1, -7], "Concat", ()), (-1, "Conv", (256, 1, 1))]
    L += [(-1, "Conv", (128, 1, 1)), (-1, "Up", ()), (21, "Conv", (128, 1, 1)), ([-1, -2], "Concat", ())] + _elan(42, 64, 64, 2, 128, range(2))
    L += [(-1, "Conv", (64, 1, 1)), (-1, "Up", ()), (14, "Conv", (64, 1, 1)), ([-1, -2], "Concat", ())] + _elan(52, 32, 32, 2, 64, range(2))
    L += [(-1, "Conv", (128, 3, 2)), ([-1, 47], "Concat", ())] + _elan(60, 64, 64, 2, 128, range(2))
    L += [(-1, "Conv", (256, 3, 2)), ([-1, 37], "Concat", ())] + _elan(68, 128, 128, 2, 256, range(2))
    L += [(57, "Conv", (128, 3, 1)), (65, "Conv", (256, 3, 1)), (73, "Conv", (512, 3, 1)), ([74, 75, 76], "IDetect", ())]
    assert len(L) == 78
    return L


class YOLOv7(nn.Module):
    def __init__(self, scale="tiny", nc=80, act=None, anchors=None):
        super().__init__()
        act = act or ("leaky" if scale == "tiny" else "silu")
        actf = (lambda: nn.LeakyReLU(0.1)) if act == "leaky" else nn.SiLU
        cfg = yolov7_tiny_cfg() if scale == "tiny" else yolov7_cfg()
        anchors = anchors or (V5_ANCHORS if scale == "tiny" else V7_ANCHORS)
        ch, mods, self.froms = [3], [], []
        for i, (f, kind, a) in enumerate(cfg):
            f = [i + j if j < 0 else j for j in (f if isinstance(f, list) else [f])]
            cin = [ch[j + 1] for j in f]
            if kind == "Conv":
                m, c = Conv(cin[0], a[0], a[1], a[2], actf), a[0]
            elif kind == "SPPCSPC":
                m, c = SPPCSPC(cin[0], a[0], actf), a[0]
            elif kind == "RepConv":
                m, c = RepConv(cin[0], a[0]), a[0]
            elif kind == "IDetect":
                m, c = IDetect(nc, cin, anchors), 0
            elif kind == "Concat":
                m, c = Concat(), sum(cin)
            else:
                m, c = {"MP": MP, "Up": Up}.get(kind, lambda: SP(a[0]))(), cin[0]
            mods.append(m)
            ch.append(c)
            self.froms.append(f)
        self.model = nn.ModuleList(mods)

    def forward(self, x):
        y = []
        for i, m in enumerate(self.model):
            f = self.froms[i]
            inp = x if i == 0 else (y[f[0]] if len(f) == 1 and not isinstance(m, (Concat, IDetect)) else [y[j] for j in f])
            y.append(m(inp))
        return y[-1]

    @torch.no_grad()
    def fuse(self):
        """As upstream before export: RepConv -> rbr_reparam, implicit layers into IDetect.m, Conv + BN -> conv with bias (names kept)."""
        def fold(conv, bn):
            w, s = conv.weight.double(), bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
            f = nn.Conv2d(conv.in_channels, conv.out_channels, conv.kernel_size, conv.stride, conv.padding, bias=True)
            f.weight.data = (w * s[:, None, None, None]).float()
            f.bias.data = (bn.bias.double() - bn.running_mean.double() * s).float()
            return f
        for m in self.modules():
            if isinstance(m, RepConv):
                d, o = fold(*m.rbr_dense), fold(*m.rbr_1x1)
                d.weight.data[:, :, 1, 1] += o.weight.data[:, :, 0, 0]
                d.bias.data += o.bias.data
                m.rbr_reparam = d
                del m.rbr_dense, m.rbr_1x1
            elif isinstance(m, Conv) and isinstance(m.bn, nn.BatchNorm2d):
                m.conv, m.bn = fold(m.conv, m.bn), nn.Identity()
            elif isinstance(m, IDetect):
                for i, conv in enumerate(m.m):
                    ia, im = m.ia[i].implicit.reshape(-1), m.im[i].implicit.reshape(-1)
                    conv.bias.data = (conv.bias + conv.weight[:, :, 0, 0] @ ia) * im
                    conv.weight.data = conv.weight * im[:, None, None, None]
                del m.ia, m.im
                m.fused = True
        return self


def build(sd: dict, scale="tiny", nc=80, act=None, anchors=None) -> YOLOv7:
    model = YOLOv7(scale, nc, act, anchors)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)).clone() for k, v in sd.items()}, strict=True)
    return model.eval()
