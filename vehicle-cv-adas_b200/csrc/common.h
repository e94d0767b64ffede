// common.h -- shared declarations for libadas_b200 (sm_90a: H100).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include <atomic>

struct adas_lane_geom;      // include/adas_b200.h

#include <nvtx3/nvToolsExt.h>     // header-only NVTX v3: ranges cost a few ns unless a tool (nsys / ncu) is attached

namespace adas {

// NVTX range for the host-side phases of the C-ABI calls (per-frame path: detect calls, plan replay, tracker update): they show up as
// named spans in nsys / ncu timelines next to the kernels they enqueue.
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
    NvtxRange(const NvtxRange&) = delete;
    NvtxRange& operator=(const NvtxRange&) = delete;
};


// ---- error plumbing -----------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define ADAS_CUDA(call)                                                                     \
    do {                                                                                    \
        cudaError_t _e = (call);                                                            \
        if (_e != cudaSuccess) {                                                            \
            adas::set_error("%s:%d CUDA error %d (%s) in %s", __FILE__, __LINE__, (int)_e, \
                            cudaGetErrorString(_e), #call);                                 \
            return 1;                                                                       \
        }                                                                                   \
    } while (0)

#define ADAS_CHECK(cond, ...)                                                               \
    do {                                                                                    \
        if (!(cond)) {                                                                      \
            adas::set_error(__VA_ARGS__);                                                   \
            return 1;                                                                       \
        }                                                                                   \
    } while (0)

// ---- GEMM / implicit-GEMM conv parameters ---------------------------------------------------
// out[row, n] = act( sum_{tap, c} A[row + shift(tap), c] * Wt[n, tap*Kc + c] + bias[n] ) (+ res)
// Activations live in "padded NHWC": a [B*(H+2)*(W+2), C] matrix with an all-zero 1-pixel halo,
// so a 3x3 stride-1 conv is 9 row-shifted GEMMs over the same 2-D matrix (shift =
// dy*(W+2)+dx) and every operand tile is one 2-D TMA box.
struct GemmParams {
    int M;          // rows of A / rows of out
    int N;          // output features
    int Kc;         // K extent per tap (multiple of 8; multiple of 64 when ntaps == 9)
    int ntaps;      // 1 or 9
    int Wp;         // padded width (W+2) of the A geometry, used for the tap shifts
    int kpt;        // k-blocks (of 64) per tap = ceil(Kc/64)
    int BN;         // tile width (multiple of 16, <= 256)
    int stages;     // smem pipeline depth
    int act;        // 0 none, 1 SiLU, 2 ReLU, 3 LeakyReLU(0.1), 5 Hardswish
    int out_f32;    // 0: fp16 out, 1: fp32 out
    int out_ld;     // row stride of out, elements
    int res_ld;     // row stride of res, elements; NEGATIVE = add the residual before the activation (ResNet)
    int mask_H, mask_W;  // > 0: only rows in the interior of the padded (H+2)x(W+2) grid are stored
    int mt_hint;    // number of 128-row sub-tiles per CTA tile (1..4; they share each weight tile), 0 = auto
    int no_slab;    // 1: 3x3 stride-1 convs load one activation tile per tap instead of one slab per (dy, k-block) (A/B hook)
    // stride-2 convs (3x3 pad 1, or 1x1) read the input through a 4-D TMA map with traversal stride 2: an M tile is a
    // bw x bh patch of output pixels of one image; s2_* describe the output grid and the input's padded height
    int s2, s2_bw, s2_bh, s2_tw, s2_th, s2_Ho, s2_Wo, s2_Hp_in;
    int transposed; // 1: out[n * out_ld + row] (swap-AB FC: rows = features, cols = batch), bias per row
    // 1: 2x2 stride-2 transposed conv (ConvTranspose2d k=2 s=2 p=0) as a 1x1 GEMM with N = 4 * Cout, columns (dy, dx, c): input pixel
    // (y, x) stores column group (dy, dx) to pixel (2y + dy, 2x + dx) of the (2H+2) x (2W+2) padded output (masked rows only)
    int up2;
    float res_scale;     // out = act(acc + bias) + res_scale * res (1 for a plain residual add)
    const float* bias;   // [N] ([M] when transposed) or nullptr
    const __half* res;   // residual, same row indexing as out, or nullptr
    void* out;
    // SIMT validation path only: raw operand pointers
    const __half* A; int a_ld;
    const __half* Wt; int w_ld;
};

int  gemm_simt_launch(const GemmParams& p, cudaStream_t st);
int  make_tmap_4d_s2(CUtensorMap* tm, const void* base, uint64_t C, uint64_t Wp, uint64_t Hp, uint64_t B, uint64_t ld_elems,
                     uint32_t box_w_src, uint32_t box_h_src);
// v3 kernel (gemm_v3.cu): the product path
int  gemm_v3_prepare(const GemmParams& p, const void* a_base, uint64_t a_inner, uint64_t a_rows, uint64_t a_stride_bytes,
                     const void* b_base, uint64_t b_inner, uint64_t b_rows, uint64_t b_stride_bytes, void** opaque);
int  gemm_v3_prepare_s2(const GemmParams& p, const void* a_base, uint64_t a_C, uint64_t a_Wp, uint64_t a_Hp, uint64_t a_B, uint64_t a_ld,
                        const void* b_base, uint64_t b_inner, uint64_t b_rows, uint64_t b_stride_bytes, void** opaque);
int  gemm_v3_run(void* opaque, cudaStream_t st);
void gemm_v3_free(void* opaque);
void gemm_v3_describe(const void* opaque, char* out, int cap);
int  gemm_v3_candidates(const GemmParams& base, int max_out, int* BN_out, int* mt_out, int* no_slab_out);
int  make_tmap_2d(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t rows, uint64_t row_stride_bytes,
                  uint32_t box_inner, uint32_t box_rows);

// ---- element-wise / data movement kernels (elementwise.cu) -----------------------------------
int launch_im2col(const __half* in, int in_ld, int in_coff, int B, int H, int W, int Cin, int kh, int kw,
                  int stride, int pad, int Ho, int Wo, __half* out, int Kpad, cudaStream_t st);
int launch_maxpool(const __half* in, int in_ld, int B, int H, int W, int C, int k, int s, int p,
                   __half* out, int out_ld, int Ho, int Wo, cudaStream_t st);
int launch_avgpool2(const __half* in, int in_ld, int B, int H, int W, int C, __half* out, int out_ld, int fill, cudaStream_t st);
int launch_upsample2x(const __half* in, int in_ld, int B, int H, int W, int C, __half* out, int out_ld,
                      cudaStream_t st);
// CBFuse (YOLOv9-E): out = base + sum of nearest-upsampled channel slices of n_src sources, each on an (H >> shift) x (W >> shift)
// padded grid; fp32 sum in the listed order, one rounding, interior pixels only.  base may be out (in place).
static const int kCbfuseMaxSrc = 5;
struct CbfuseSrc { const __half* ptr; int ld; int shift; };
struct CbfuseParams {
    __half* out; int out_ld;
    const __half* base; int base_ld;
    int B, H, W, C, n_src;
    CbfuseSrc src[kCbfuseMaxSrc];
};
int launch_cbfuse(const CbfuseParams& p, cudaStream_t st);
int launch_layernorm(const __half* in, int in_ld, int rows, int d_len, int d_norm, const float* gamma,
                     const float* beta, float eps, __half* out, int out_ld, cudaStream_t st);
int launch_fc_stream(const __half* x, int x_ld, int batch, const __half* W, int K, int N, const float* bias, int act, void* out, int out_ld,
                     int out_f32, cudaStream_t st);
int launch_nchw_to_padded(const float* in, int B, int C, int H, int W, __half* out, int out_ld, cudaStream_t st);
int launch_stempack(const __half* img, int B, int H, int W, __half* q, cudaStream_t st);
// lane_geom.cu: ego-lane polygon / polyfit resampling / bird-view points / curvature + offset, one block per frame
int launch_lane_geom(const int32_t* pts, const int32_t* npts, const uint8_t* status, const double* M, int batch, int max_pts, int img_w, int img_h,
                     int adjust, int bird_w, int bird_h, int32_t* area, int cap_area, int32_t* bird, ::adas_lane_geom* out, cudaStream_t st);
// warp.cu: cv2.warpPerspective (INTER_LINEAR, constant black border) of device-resident BGR frames
int launch_warp_perspective(const uint8_t* d_src, int B, int H, int W, const double* M_host, double* d_Minv, uint8_t* d_dst, int oh, int ow, cudaStream_t st);
// stem_conv.cu: k x k stride-1 or stride-2 conv of the padded C=4 image (warp-level MMA, no patch matrix)
int stem_conv_supported(int Cout, int k, int pad);
int launch_stem_conv(const __half* img, int B, int H, int W, const __half* wq, const float* bias, int Cout, int k, int pad, int stride, int act,
                     __half* out, int out_ld, int Ho, int Wo, cudaStream_t st);
int launch_zero_rows(__half* buf, int ld, int C, int row0, int nrows, cudaStream_t st);
// dwconv.cu: depthwise k x k conv (k 3 / 7, stride 1 / 2) of a channel slice, out = act(acc + bias) (+ res)
int launch_dwconv(const __half* in, int in_ld, int B, int H, int W, int C, int k, int stride, const __half* w, const float* bias, int act,
                  const __half* res, int res_ld, __half* out, int out_ld, int Ho, int Wo, cudaStream_t st);
// lite_ops.cu: squeeze-excite of a channel slice (YOLOv6-Lite SEBlock), gate = hardsigmoid(W2 relu(W1 mean + b1) + b2), one CTA per
// image; W1 fp32 [hid][C], W2 fp32 [C][hid].  out may be in (in place).
static const int kSeMaxC = 1024;
struct SeParams {
    const __half* in; int in_ld;
    __half* out; int out_ld;
    const float *w1, *b1, *w2, *b2;
    int B, H, W, C, hid;
};
int se_supported(int C, int hid);
int launch_se(const SeParams& p, cudaStream_t st);
// lite_ops.cu: out(2j) = a(j), out(2j + 1) = b(j), j < n (concat + channel_shuffle(2)), interior pixels of an H x W padded grid
int launch_shuffle2(const __half* a, int a_ld, const __half* b, int b_ld, __half* out, int out_ld, int B, int H, int W, int n, cudaStream_t st);
// attention.cu: multi-head self-attention over the H*W pixels of each image (YOLOv10 PSA)
int attention_supported(int nh, int kdp, int hd);
int launch_attention(const __half* qkv, int in_ld, int B, int H, int W, int nh, int kdp, int hd, float scale, __half* out, int out_ld,
                     cudaStream_t st);

// ---- pre-processing (preprocess.cu) -----------------------------------------------------------
struct LetterboxGeom {
    int src_h, src_w, in_h, in_w, new_h, new_w, pad_h, pad_w;
};
LetterboxGeom letterbox_geom(int src_h, int src_w, int in_h, int in_w);
// writes fp16 padded NHWC (C=4: R,G,B,0) and/or fp32 NCHW blob
int launch_yolo_pre(const uint8_t* frames, int B, const LetterboxGeom& g, __half* img_padded, int img_ld,
                    float* blob_nchw, cudaStream_t st);
int launch_ufld_pre(const uint8_t* frames, int B, int H, int W, int in_h, int in_w, int resize_h,
                    const float* lut /*3*256 dev*/, __half* img_padded, int img_ld, float* blob_nchw,
                    cudaStream_t st);

// ---- YOLO post-processing (yolo_post.cu) --------------------------------------------------------
struct YoloLevel { const float* ptr; int ld; int H, W; int stride; int rows_per_img; };
static const int kYoloMaxLevels = 4;      // P6 heads (strides 8 / 16 / 32 / 64); every other head has 3 levels
int launch_yolov8_head_decode(const YoloLevel* lv /*3*/, int B, int nc, float* raw /*[B,4+nc,A]*/, int A,
                              cudaStream_t st);
int launch_yolov5_head_decode(const YoloLevel* lv /*n_levels*/, int n_levels /*3, or 4 with anchors*/, int B, int nc, float* raw /*[B,A,5+nc]*/,
                              int A, int lite, const float* anchors /*device [n_levels][3][2], nullptr = YOLOv5 table*/, cudaStream_t st);
int launch_yolov5_lite_post(float* raw /*[B,A,5+nc], in place*/, int B, int A, int nc, int in_h, int in_w, cudaStream_t st);
// YOLOv6 level columns: 4 * (reg_max + 1) box columns (stored as 8-column groups), the nc class logits from the next multiple of 8 on
__host__ __device__ inline unsigned yolov6_cls_col(unsigned reg_max) { return (4u * (reg_max + 1u) + 7u) / 8u * 8u; }
int launch_yolov6_head_decode(const YoloLevel* lv /*n_levels*/, int n_levels /*3, or 4 (YOLOv6-Lite)*/, int B, int nc, int reg_max, float* raw /*[B,A,5+nc]*/, int A, cudaStream_t st);
struct YoloPostBufs {
    // device scratch, sized for max_batch
    int32_t* flags;      // [B, A] candidate flag
    int32_t* cls;        // [B, A]
    float*   conf;       // [B, A]
    int32_t* n_cand;     // [B]
    float*   cand_box;   // [B, cap, 4] xywh (source pixels)
    float*   cand_conf;  // [B, cap]
    int32_t* cand_cls;   // [B, cap]
    double*  nms_work;   // [B, cap, 7]
    int cap;             // max candidates kept per frame
    // outputs (device)
    float* out_box; float* out_score; int32_t* out_cls; int32_t* out_idx; int32_t* out_count;
};
int launch_yolo_post(const float* raw, int kind, int B, int A, int nc, const LetterboxGeom& g, double box_score,
                     double nms_iou, int max_det, YoloPostBufs& w, cudaStream_t st);

// ---- UFLD post-processing (ufld_post.cu) -----------------------------------------------------------
struct UfldDims { int ngr, ncr, ngc, ncc, nl; };
int launch_ufld_v1_post(const float* head, int ld, int B, int G, int R, int in_w, int in_h, int cfg_w, int cfg_h, int img_w, int img_h,
                        const double* row_anchor, int32_t* pts, int32_t* npts, uint8_t* status, double* coords, int max_pts, cudaStream_t st);
int launch_ufld_post(const float* heads, int ld, int B, UfldDims d, int img_w, int img_h, const double* row_anchor,
                     const double* col_anchor, int32_t* pts, int32_t* npts, uint8_t* status, double* coords,
                     int max_pts, cudaStream_t st);

}  // namespace adas
