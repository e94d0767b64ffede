"""Footprint model of a .b200w plan: what every op, head decode and output copy of the engine reads and writes.

Written from the index arithmetic of csrc/engine.cu (build_program, head_decode, infer_common, ufld_post_dispatch) and the kernels
it launches.  `parse` reads the plan file itself (the records of csrc/plan.h), not the PlanBuilder that wrote it, so a corrupted
file is modelled as the loader would see it.

A region is a strided block of one buffer: `rows` rows of `ld` elements, of which columns [c0, c1) are touched, each element
`esize` bytes as the kernel reads it.  The row count follows the geometry the kernel walks (the buffer whose H x W it was given),
which need not be the buffer's own.  A plan is in bounds at a batch when every region lies inside its buffer's logical extent
(max_batch * rows_per_img * C elements of the buffer's dtype; the allocation slack does not count) and every tensor read fits
its tensor.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass
from typing import List, Optional, Tuple

import adas_b200  # noqa: F401
from adas_b200 import plan
from adas_b200.plan import (BUF_FMT, BUF_SIZE, HDR_FMT, HDR_SIZE, MODEL_UFLDV1, MODEL_UFLDV2, MODEL_YOLOV6, MODEL_YOLOV8, OP_ATTN,
                            OP_AVGPOOL2, OP_CBFUSE, OP_DWCONV, OP_FMT, OP_GEMM, OP_IM2COL, OP_LAYERNORM, OP_MAXPOOL, OP_NP, OP_SE,
                            OP_SHUFFLE2, OP_SIZE, OP_STEMCONV, OP_STEMPACK, OP_UPSAMPLE2X, OUT_FMT, OUT_SIZE, TEN_FMT, TEN_SIZE)

HEADER_FIELDS = ["version", "model_kind", "in_c", "in_h", "in_w", "n_buffers", "n_ops", "n_tensors", "n_outputs"] + \
                [f"meta{i}" for i in range(16)]


@dataclass
class Plan:
    header: list            # unpacked HDR_FMT fields: magic, version, model_kind, in_c, in_h, in_w, n_buffers, n_ops, n_tensors, n_outputs, meta*16, blob_offset, blob_bytes
    bufs: List[list]        # rows_per_img, C, dtype, H, W, flags
    ops: List[Tuple[int, plan.OpParams, list]]
    tensors: List[list]     # offset, bytes, dtype, pad
    outs: List[list]        # buffer, coff, C, stride

    @property
    def model_kind(self): return self.header[2]
    @property
    def in_hw(self): return self.header[4], self.header[5]
    @property
    def meta(self): return self.header[10:26]

    # byte offsets of each record, for corrupting the file in place
    def buf_off(self, i): return HDR_SIZE + i * BUF_SIZE
    def op_off(self, i): return HDR_SIZE + len(self.bufs) * BUF_SIZE + i * OP_SIZE
    def ten_off(self, i): return self.op_off(len(self.ops)) + i * TEN_SIZE
    def out_off(self, i): return self.ten_off(len(self.tensors)) + i * OUT_SIZE

    def field_off(self, i, name):
        """Byte offset of field `name` of op i: a field of plan.OP_FIELDS, "src<s>.<field>" of a CBFUSE source (plan.CBFUSE_SRC_FIELDS)
        or a float of plan.OP_FLOATS."""
        typ = self.ops[i][0]
        if name in plan.OP_FLOATS.get(typ, ()):
            slot = OP_NP + plan.OP_FLOATS[typ].index(name)
        elif typ == OP_CBFUSE and name.startswith("src"):
            s, field = name[3:].split(".")
            slot = plan.cbfuse_src_slot(int(s)) + plan.CBFUSE_SRC_FIELDS.index(field)
        else:
            slot = plan.field_slot(typ, name)
        return self.op_off(i) + 4 + 4 * slot


def corrupt(raw: bytes, off: int, fmt: str, value) -> bytes:
    """`raw` with `value` packed in struct format `fmt` at byte `off` (a record field: Plan.buf_off / op_off / ten_off / out_off)."""
    b = bytearray(raw)
    struct.pack_into(fmt, b, off, value)
    return bytes(b)


def engine_error(path) -> Optional[str]:
    """The error loading the plan file at `path` raises, None if it loads.  The loader validates the whole plan before any device work,
    so without a GPU a valid plan fails only for the missing device."""
    from adas_b200 import _capi
    try:
        _capi.Engine(str(path))
    except Exception as e:
        return str(e)
    return None


def parse(raw: bytes) -> Plan:
    h = list(struct.unpack_from(HDR_FMT, raw, 0))
    nb, no, nt, nout = h[6:10]
    off = HDR_SIZE
    bufs = [list(struct.unpack_from(BUF_FMT, raw, off + i * BUF_SIZE)) for i in range(nb)]
    off += nb * BUF_SIZE
    ops = []
    for i in range(no):
        r = struct.unpack_from(OP_FMT, raw, off + i * OP_SIZE)
        ops.append((r[0], plan.OpParams(r[0], r[1:1 + OP_NP]), list(r[1 + OP_NP:])))
    off += no * OP_SIZE
    tensors = [list(struct.unpack_from(TEN_FMT, raw, off + i * TEN_SIZE)) for i in range(nt)]
    off += nt * TEN_SIZE
    outs = [list(struct.unpack_from(OUT_FMT, raw, off + i * OUT_SIZE)) for i in range(nout)]
    return Plan(h, bufs, ops, tensors, outs)


@dataclass
class Region:
    buf: int
    write: bool
    rows: int
    ld: int
    c0: int
    c1: int
    esize: int
    what: str


def _esize(dtype: int) -> int:
    return 4 if dtype == 1 else 2


def _rows(B: int, H: int, W: int) -> int:
    """rows of B padded H x W images"""
    return B * (H + 2) * (W + 2)


class _Model:
    def __init__(self, pl: Plan, batch: int):
        self.pl, self.B = pl, batch
        self.regions: List[Region] = []
        self.tensor_reads: List[Tuple[int, int, Optional[int], str]] = []   # tensor, bytes, dtype required (None: any), what
        self.faults: List[str] = []          # arithmetic the kernels cannot do (division by a zero grid width, ...)

    def buf(self, i):
        return self.pl.bufs[i]

    def region(self, b, write, rows, ld, c0, c1, esize, what):
        self.regions.append(Region(b, write, rows, ld, c0, c1, esize, what))

    def slice(self, b, write, rows, c0, n, what, esize=2):
        self.region(b, write, rows, self.buf(b)[1], c0, c0 + n, esize, what)

    def padded_rows(self, b):
        rb = self.buf(b)
        return self.B * rb[0]

    def tensor(self, t, nbytes, dtype, what):
        self.tensor_reads.append((t, nbytes, dtype, what))

    # ---- ops ----
    def op(self, oi, typ, p):
        B, buf = self.B, self.buf
        w = f"op {oi}"
        if typ == OP_GEMM:
            self.tensor(p.w_tensor, p.N * p.Kc * p.ntaps * 2, 0, w + " weights")
            if p.bias_tensor >= 0:
                self.tensor(p.bias_tensor, p.N * 4, 1, w + " bias")
            ob, N = p.out_buf, p.N
            oes = _esize(buf(ob)[2])
            if p.transposed:
                # one input vector per image: the whole per-image slab read flat (FC tensor-core and fc_stream routes alike)
                self.region(p.a_buf, False, B, buf(p.a_buf)[0] * buf(p.a_buf)[1], 0, p.Kc, 2, w + " FC input")
                self.region(ob, True, B, buf(ob)[0] * buf(ob)[1], 0, N, oes, w + " FC output")
                return
            # the operand tensor map spans the input's batch rows (taps past it read zeros); output rows follow the M walk
            self.slice(p.a_buf, False, self.padded_rows(p.a_buf), p.a_coff, p.Kc, w + " input")
            if p.s2:
                out_rows = self.padded_rows(ob)
            elif p.up2:
                A_ = buf(p.a_buf)
                out_rows = _rows(B, 2 * A_[3], 2 * A_[4])
            else:
                out_rows = self.padded_rows(p.a_buf)
            self.slice(ob, True, out_rows, p.out_coff, N // 4 if p.up2 else N, w + " output", oes)
            if p.res_buf >= 0:
                # the epilogue reads the residual at the output row index
                self.slice(p.res_buf, False, out_rows, p.res_coff, N, w + " residual")
        elif typ == OP_IM2COL:
            o = p.out_buf
            self.slice(p.in_buf, False, self.padded_rows(p.in_buf), p.in_coff, p.Cin, w + " input")
            self.region(o, True, _rows(B, buf(o)[3], buf(o)[4]), buf(o)[1], 0, p.kh * p.kw * p.Cin, 2, w + " patches")
        elif typ == OP_MAXPOOL:
            o = p.out_buf
            self.slice(p.in_buf, False, self.padded_rows(p.in_buf), p.in_coff, p.C, w + " input")
            self.slice(o, True, _rows(B, buf(o)[3], buf(o)[4]), p.out_coff, p.C, w + " output")
        elif typ == OP_UPSAMPLE2X:
            H, W = buf(p.in_buf)[3], buf(p.in_buf)[4]
            self.slice(p.in_buf, False, _rows(B, H, W), p.in_coff, p.C, w + " input")
            self.slice(p.out_buf, True, _rows(B, 2 * H, 2 * W), p.out_coff, p.C, w + " output")
        elif typ == OP_AVGPOOL2:
            rows = _rows(B, buf(p.in_buf)[3], buf(p.in_buf)[4])
            self.slice(p.in_buf, False, rows, p.in_coff, p.C, w + " input")
            self.slice(p.out_buf, True, rows, p.out_coff, p.C, w + " output")
        elif typ == OP_DWCONV:
            C, k = p.C, p.k
            self.tensor(p.w_tensor, C * k * k * 2, 0, w + " weights")
            self.tensor(p.bias_tensor, C * 4, 1, w + " bias")
            self.slice(p.in_buf, False, _rows(B, buf(p.in_buf)[3], buf(p.in_buf)[4]), p.in_coff, C, w + " input")
            orows = _rows(B, buf(p.out_buf)[3], buf(p.out_buf)[4])
            self.slice(p.out_buf, True, orows, p.out_coff, C, w + " output")
            if p.res_buf >= 0:
                self.slice(p.res_buf, False, orows, p.res_coff, C, w + " residual")
        elif typ == OP_ATTN:
            nh, kdp, hd = p.nh, p.kdp, p.hd
            rows = _rows(B, buf(p.in_buf)[3], buf(p.in_buf)[4])
            self.slice(p.in_buf, False, rows, p.in_coff, nh * (2 * kdp + hd), w + " qkv")
            self.slice(p.out_buf, True, rows, p.out_coff, nh * hd, w + " output")
        elif typ == OP_CBFUSE:
            C = p.C
            H, W = buf(p.out_buf)[3], buf(p.out_buf)[4]
            self.slice(p.out_buf, True, _rows(B, H, W), p.out_coff, C, w + " output")
            self.slice(p.base_buf, False, _rows(B, H, W), p.base_coff, C, w + " base")
            for s, (sb, scoff, sh) in enumerate(plan.cbfuse_sources(p)):
                self.slice(sb, False, _rows(B, H >> sh, W >> sh), scoff, C, w + f" source {s}")
        elif typ == OP_SE:
            C, hid = p.C, p.hid
            for t, n in zip((p.w1, p.b1, p.w2, p.b2), (hid * C, hid, C * hid, C)):
                self.tensor(t, n * 4, 1, w + " se tensor")
            rows = _rows(B, buf(p.in_buf)[3], buf(p.in_buf)[4])
            self.slice(p.in_buf, False, rows, p.in_coff, C, w + " input")
            self.slice(p.out_buf, True, rows, p.out_coff, C, w + " output")
        elif typ == OP_SHUFFLE2:
            n = p.n
            rows = _rows(B, buf(p.out_buf)[3], buf(p.out_buf)[4])
            self.slice(p.a_buf, False, rows, p.a_coff, n, w + " a")
            self.slice(p.b_buf, False, rows, p.b_coff, n, w + " b")
            self.slice(p.out_buf, True, rows, p.out_coff, 2 * n, w + " output")
        elif typ == OP_STEMPACK:
            H, W = buf(p.in_buf)[3], buf(p.in_buf)[4]
            self.region(p.in_buf, False, _rows(B, H, W), 4, 0, 4, 2, w + " image")       # the kernel's image row stride is 4 channels
            self.region(p.out_buf, True, _rows(B, H >> 1, W >> 1), 64, 0, 64, 2, w + " packed")
        elif typ == OP_STEMCONV:
            Cout, k = p.Cout, p.k
            self.tensor(p.w_tensor, Cout * k * ((4 * k + 15) // 16 * 16) * 2, None, w + " weights")
            if p.bias_tensor >= 0:
                self.tensor(p.bias_tensor, Cout * 4, None, w + " bias")
            H, W = buf(p.in_buf)[3], buf(p.in_buf)[4]
            self.region(p.in_buf, False, _rows(B, H, W), 4, 0, 4, 2, w + " image")
            self.slice(p.out_buf, True, _rows(B, buf(p.out_buf)[3], buf(p.out_buf)[4]), p.out_coff, Cout, w + " output")
        elif typ == OP_LAYERNORM:
            d_len = p.d_len
            self.tensor(p.gamma_tensor, d_len * 4, None, w + " gamma")
            self.tensor(p.beta_tensor, d_len * 4, None, w + " beta")
            self.region(p.in_buf, False, B, buf(p.in_buf)[0] * buf(p.in_buf)[1], 0, d_len, 2, w + " input")
            self.region(p.out_buf, True, B, buf(p.out_buf)[0] * buf(p.out_buf)[1], 0, d_len, 2, w + " output")
        else:
            self.faults.append(f"{w}: unknown op type {typ}")

    # ---- input staging, head decodes and output copies ----
    def staging(self):
        in_h, in_w = self.pl.in_hw
        C0 = self.buf(0)[1]
        # nchw_to_padded writes every channel of buffer 0's row; the frame pre-processing writes 4
        self.region(0, True, _rows(self.B, in_h, in_w), C0, 0, C0, 2, "input staging")

    def yolo_levels(self, cells_per_anchor_row: int, ncols, what: str):
        """The decode walks meta[1] anchors through the levels in order; anchors past a level's cells spill into the next, and
        those past the last level's cells index past its grid."""
        pl, B = self.pl, self.B
        A = pl.meta[1]
        a = A
        n = len(pl.outs)
        for li, (ob, coff, oC, stride) in enumerate(pl.outs):
            b = self.buf(ob)
            H, W = b[3], b[4]
            hw = cells_per_anchor_row * H * W
            cnt = a if li == n - 1 else min(a, hw)
            a -= cnt
            if cnt <= 0:
                continue
            if W == 0 or H == 0:
                self.faults.append(f"{what} level {li}: a {H}x{W} grid")
                continue
            if cells_per_anchor_row == 1:          # v8 / v6: anchor = cell
                an, cell = 0, cnt - 1
            else:                                   # v5: anchor = an * H * W + cell
                an, cell = (cnt - 1) // (H * W), min(cnt, H * W) - 1
            y, x = divmod(cell, W)
            row = (y + 1) * (W + 2) + (x + 1)
            rows = (B - 1) * b[0] + row + 1
            c1 = coff + ncols(an)
            self.region(ob, False, rows, b[1], coff, c1, 4, f"{what} level {li}")

    def heads(self):
        pl = self.pl
        kind, meta = pl.model_kind, pl.meta
        if not pl.outs:
            return
        if kind in (MODEL_UFLDV1, MODEL_UFLDV2):
            ob, coff, oC, _ = pl.outs[0]
            b = self.buf(ob)
            # ufld_post_dispatch and the infer_common copies read image i at row i of the head buffer
            if b[0] != 1:
                self.faults.append(f"UFLD head buffer has {b[0]} rows per image; the decode reads image b at row b")
            self.region(ob, False, self.B, b[1], coff, coff + meta[5], 4, "UFLD head")
            return
        nc = meta[0]
        if kind == MODEL_YOLOV8:
            if len(pl.outs) != 3:
                self.faults.append("v8 decode takes 3 levels")
            self.yolo_levels(1, lambda an: 64 + nc, "v8 decode")
        elif kind == MODEL_YOLOV6:
            rm = meta[2]
            cls_col = (4 * (rm + 1) + 7) // 8 * 8
            self.yolo_levels(1, lambda an: cls_col + nc, "v6 decode")
        else:
            self.yolo_levels(3, lambda an: (an + 1) * (5 + nc), "v5 decode")


def footprint(pl: Plan, batch: int):
    """(regions, tensor reads, faults) of one run of the plan at `batch` images: input staging, every op, the head decode."""
    m = _Model(pl, batch)
    m.staging()
    for oi, (typ, p, f) in enumerate(pl.ops):
        m.op(oi, typ, p)
    m.heads()
    return m.regions, m.tensor_reads, m.faults


def out_of_bounds(pl: Plan, max_batch: int) -> List[str]:
    """Every region or tensor read of a run at max_batch images that leaves its buffer's logical extent or its tensor."""
    bad = []
    regions, treads, faults = footprint(pl, max_batch)
    bad += faults
    nb, nt = len(pl.bufs), len(pl.tensors)
    for r in regions:
        if not 0 <= r.buf < nb:
            bad.append(f"{r.what}: buffer {r.buf} does not exist")
            continue
        rpi, C, dtype = pl.bufs[r.buf][:3]
        extent = max_batch * rpi * C * _esize(dtype)
        if r.rows <= 0 or r.c1 <= r.c0:
            continue
        if r.c0 < 0 or r.c1 > r.ld or r.esize != _esize(dtype):
            bad.append(f"{r.what}: columns [{r.c0}, {r.c1}) of {r.esize}-byte elements on a row of {r.ld} "
                       f"{_esize(dtype)}-byte elements (buffer {r.buf})")
            continue
        end = ((r.rows - 1) * r.ld + r.c1) * r.esize
        if end > extent:
            bad.append(f"{r.what}: ends at byte {end} of buffer {r.buf}, which holds {extent}")
    for t, nbytes, dtype, what in treads:
        if not 0 <= t < nt:
            bad.append(f"{what}: tensor {t} does not exist")
        elif pl.tensors[t][1] < nbytes or (dtype is not None and pl.tensors[t][2] != dtype):
            bad.append(f"{what}: tensor {t} holds {pl.tensors[t][1]} bytes of dtype {pl.tensors[t][2]}, the op reads {nbytes}")
    return bad
