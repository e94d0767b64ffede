// plan.h -- on-disk layout of a .b200w plan (the serialized network: op list + packed weights).
// Written by vehicle-cv-adas_b200/plan.py, read by engine.cu.  Plays the role of the reference's
// serialized TensorRT engine / ONNX file (coreEngine.py:54-55,164-166); the packer replaces
// convertOnnxToTensorRT.py / onnxQuantization.py for this runtime.
#pragma once
#include <stdint.h>
#include <string.h>

namespace adas {

static const char kPlanMagic[8] = {'B', '2', '0', '0', 'P', 'L', 'A', 'N'};
static const uint32_t kPlanVersion = 1;

#pragma pack(push, 1)
struct PlanHeader {
    char magic[8];
    uint32_t version;
    uint32_t model_kind;          // ADAS_MODEL_*
    uint32_t in_c, in_h, in_w;    // network input binding (NCHW semantic)
    uint32_t n_buffers, n_ops, n_tensors, n_outputs;
    uint32_t meta[16];            // YOLO: [0]=nc [1]=n_anchors(total) [2]=lite (YOLOv6: reg_max) [3]=1+anchor tensor (0: YOLOv5 table)
                                  // UFLD: [0]=ngr [1]=ncr [2]=ngc [3]=ncc [4]=nl [5]=total_dim
    uint64_t blob_offset, blob_bytes;
};
struct PlanBuffer {               // activation buffer: [batch * rows_per_img, C] elements
    uint32_t rows_per_img;
    uint32_t C;                   // row stride in elements
    uint32_t dtype;               // 0 = fp16, 1 = fp32
    uint32_t H, W;                // > 0: padded-NHWC geometry, rows_per_img == (H+2)*(W+2)
    uint32_t flags;
};
struct PlanOp {
    uint32_t type;                // PlanOpType
    int32_t p[23];
    float f[4];
};
struct PlanTensor {
    uint64_t offset, bytes;       // relative to blob_offset
    uint32_t dtype;               // 0 = fp16, 1 = fp32
    uint32_t pad;
};
struct PlanOutput {
    uint32_t buffer, coff, C, stride;   // stride: YOLO level stride (8/16/32)
};
#pragma pack(pop)

enum PlanOpType : uint32_t {
    OP_GEMM = 1,
    OP_IM2COL = 2,
    OP_MAXPOOL = 3,
    OP_UPSAMPLE2X = 4,
    OP_LAYERNORM = 5,
    OP_STEMPACK = 6,
    OP_STEMCONV = 7,
    OP_AVGPOOL2 = 8,
    OP_DWCONV = 9,
    OP_ATTN = 10,
    OP_CBFUSE = 11,
    OP_SE = 12,
    OP_SHUFFLE2 = 13,
};

// The fields of PlanOp::p for each op type, in slot order: op type OP_XXX reads struct XxxOp (op_fields below); the packer writes
// zero past the last field.  plan.py's OP_FIELDS names the same fields in the same order (tests/test_plan_cpu.py checks both).
// A buffer field indexes PlanBuffer records, a tensor field PlanTensor records (-1: none where allowed); a coff is the first
// channel of a slice of its buffer's rows.

// Implicit-GEMM conv / FC.  f[0] = res_scale (0 = 1): out = act(acc + bias) + res_scale * res
struct GemmOp {
    int32_t a_buf, a_coff;
    int32_t Kc;                   // channels per tap
    int32_t ntaps;                // 1, 9 (3x3 stride 1, or 3x3 stride 2 with s2) or 4 (stem7x7s2's vertical taps)
    int32_t w_tensor, bias_tensor;
    int32_t N;                    // output columns
    int32_t act;                  // 0 none, 1 SiLU, 2 ReLU, 3 LeakyReLU(0.1), 5 Hardswish x * clamp(x + 3, 0, 6) / 6 (4 is unused and rejected)
    int32_t res_buf, res_coff;    // res_buf -1: no residual
    int32_t res_pre_act;          // 1: the residual is added before the activation
    int32_t out_buf, out_coff;
    int32_t masked;               // 1: store only the interior of the output's padded grid
    int32_t transposed;           // 1: swap-AB FC, one input vector per image (the whole per-image slab)
    int32_t BN;                   // test hook: > 0 forces the tile width (0 = cost model + autotune)
    int32_t s2;                   // 1: stride-2 conv read from the padded input through a traversal-stride-2 TMA map
    int32_t MT;                   // test hook: > 0 forces the sub-tile count
    int32_t no_slab;              // test hook: 1 = one activation tile per 3x3 tap
    int32_t up2;                  // 1: 2x2 stride-2 transposed conv, N = 4 * Cout in (dy, dx, c) order stored to pixel (2y+dy, 2x+dx)
                                  //    of a 2H x 2W output (Cout % 8 == 0; out_coff / the output slice hold Cout channels)
};
// Patch gather of a k x k conv into a [rows_out_padded, Kpad] matrix (Kpad = out_buf's C)
struct Im2colOp { int32_t in_buf, in_coff, Cin, kh, kw, stride, pad, out_buf; };
struct MaxpoolOp { int32_t in_buf, in_coff, C, k, stride, pad, out_buf, out_coff; };
struct Upsample2xOp { int32_t in_buf, in_coff, C, out_buf, out_coff; };
// 7x7 stride-2 stem re-layout of the image (in_buf, C = 4), see elementwise.cu stempack_kernel
struct StempackOp { int32_t in_buf, out_buf; };
// k x k stem conv of the image (in_buf, C = 4), stem_conv.cu; weights packed [Cout][k][round_up(4k,16)]
struct StemconvOp {
    int32_t in_buf, w_tensor, bias_tensor, Cout, k, pad, act, out_buf, out_coff;
    int32_t stride;               // 1 or 2; 0 = 2
};
// f[0] = eps.  Statistics over d_norm entries; the other d_len - d_norm slab entries are structural zeros with gamma = beta = 0
struct LayernormOp { int32_t in_buf, d_len, gamma_tensor, beta_tensor, out_buf, d_norm; };
// 2x2 stride-1 mean into a buffer of the input's H x W geometry; row H-1 and column W-1 hold 0 (fill 0) or -inf (fill 1),
// see elementwise.cu avgpool2_kernel
struct Avgpool2Op { int32_t in_buf, in_coff, C, out_buf, out_coff, fill; };
// Depthwise k x k conv (k 3, 5 or 7, pad k/2, stride 1 or 2 with k 3 / 5), weights fp16 [k*k][C], bias fp32 [C],
// act 0 none / 1 SiLU / 5 Hardswish; out = act(acc + bias) (+ res, res_buf -1: none), see dwconv.cu
struct DwconvOp { int32_t in_buf, in_coff, C, k, stride, act, w_tensor, bias_tensor, out_buf, out_coff, res_buf, res_coff; };
// f[0] = softmax scale.  Multi-head self-attention over the H*W pixels; input channels [Q nh*kdp | K nh*kdp | V nh*hd], output nh*hd
// channels head-major, see attention.cu
struct AttnOp { int32_t in_buf, in_coff, nh, kdp, hd, out_buf, out_coff; };
// YOLOv9-E CBFuse: out(y, x, c) = base(y, x, c) + sum_i src_i(y >> shift_i, x >> shift_i, src_coff_i + c) over the output's
// interior (n_src 1..5, shift 0..4, src H x W << shift == out H x W); fp32 sum in the listed order, one rounding; base may be the
// output slice itself (in place), see elementwise.cu cbfuse_kernel
struct CbfuseOp {
    int32_t out_buf, out_coff, C, base_buf, base_coff, n_src;
    struct Src { int32_t buf, coff, shift; } src[5];      // the first n_src are read
};
// YOLOv6-Lite SEBlock over the interior of a C-channel slice, gate = hardsigmoid(w2 relu(w1 mean(x) + b1) + b2), out = x * gate
// (one fp16 rounding); w1 .. b2 are fp32 tensors w1 [hid][C], b1 [hid], w2 [C][hid], b2 [C]; C % 8 == 0, C <= 1024, 1 <= hid <= 256;
// out == in slice (in place) or disjoint from it, see lite_ops.cu se_kernel
struct SeOp { int32_t in_buf, in_coff, C, hid, w1, b1, w2, b2, out_buf, out_coff; };
// concat + channel_shuffle(2) of two n-channel slices, out(y, x, 2j) = a(y, x, j), out(y, x, 2j + 1) = b(y, x, j) over the interior
// (n % 8 == 0; all three on one H x W grid; the 2n-channel output slice overlaps neither source), see lite_ops.cu shuffle2_kernel
struct Shuffle2Op { int32_t a_buf, a_coff, b_buf, b_coff, n, out_buf, out_coff; };

// The fields of `op` as op type T (a copy: the record's bytes are not reinterpreted in place).
template <class T>
T op_fields(const PlanOp& op) {
    static_assert(sizeof(T) <= sizeof(PlanOp::p), "an op's fields must fit PlanOp::p");
    T t;
    memcpy(&t, op.p, sizeof(T));
    return t;
}

}  // namespace adas
