// yolo_post.cu -- YOLO head decode, candidate selection and the reference-exact NMS on the device.
// Compiled with -fmad=false: every float op below must round exactly like numpy's (no FMA contraction).
//
// Replaces (reference file:line):
//   head decode            the Detect layer baked into the exported ONNX (ultralytics 8.1 / yolov5 v6.2; SURVEY App. A)
//   lite_postprocess       ObjectDetector/yoloDetector.py:36-50 (same grid/anchor arithmetic as the v5 Detect layer)
//   __process_output       ObjectDetector/yoloDetector.py:104-133  per-anchor argmax, strict threshold, xywh->xyxy
//   convert_boxes_coordinate ObjectDetector/utils.py:70-87         undo letterbox, ->xywh (float32 arithmetic)
//   NMS.fast_soft_nms      ObjectDetector/utils.py:161-256         class-agnostic; `method` is a str so the hard branch
//                                                                  runs; +1 areas; row i overwritten by row maxpos
//                                                                  (view aliasing), scores/areas really swapped;
//                                                                  emits dets[:,4][scores > 0.001] (duplicates possible)
#include "common.h"
#include <mutex>

namespace adas {

// ------------------------------------------------------------------------------------------------
// YOLOv8 Detect: per level fp32 [rows, ld>=64+nc] in padded-grid row order: cols 0..63 DFL logits
// (4 sides x 16 bins), 64.. class logits.  raw[b][ch][a], a = level offset + y*W + x.
__global__ void yolov8_decode_kernel(YoloLevel l0, YoloLevel l1, YoloLevel l2, int B, int nc, float* __restrict__ raw, int A) {
    const long long total = (long long)B * A;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / A);
        int a = (int)(i % A);
        YoloLevel lv = l0;
        if (a >= l0.H * l0.W) { a -= l0.H * l0.W; lv = l1; if (a >= l1.H * l1.W) { a -= l1.H * l1.W; lv = l2; } }
        const int y = a / lv.W, x = a % lv.W;
        const float* p = lv.ptr + ((size_t)b * lv.rows_per_img + (size_t)(y + 1) * (lv.W + 2) + (x + 1)) * lv.ld;
        float d[4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            float m = p[s * 16];
            for (int k = 1; k < 16; ++k) m = fmaxf(m, p[s * 16 + k]);
            float den = 0.f, num = 0.f;
            for (int k = 0; k < 16; ++k) {
                const float e = expf(p[s * 16 + k] - m);
                den += e;
                num += e * (float)k;
            }
            d[s] = num / den;
        }
        const float ax = (float)x + 0.5f, ay = (float)y + 0.5f;
        const float x1 = ax - d[0], y1 = ay - d[1], x2 = ax + d[2], y2 = ay + d[3];
        const float st = (float)lv.stride;
        float* o = raw + (size_t)b * (4 + nc) * A + (i % A);
        o[0] = (x1 + x2) * 0.5f * st;
        o[(size_t)A] = (y1 + y2) * 0.5f * st;
        o[(size_t)2 * A] = (x2 - x1) * st;
        o[(size_t)3 * A] = (y2 - y1) * st;
        for (int c = 0; c < nc; ++c) o[(size_t)(4 + c) * A] = 1.f / (1.f + expf(-p[64 + c]));
    }
}

int launch_yolov8_head_decode(const YoloLevel* lv, int B, int nc, float* raw, int A, cudaStream_t st) {
    const long long total = (long long)B * A;
    int blocks = (int)((total + 127) / 128);
    yolov8_decode_kernel<<<blocks, 128, 0, st>>>(lv[0], lv[1], lv[2], B, nc, raw, A);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

// YOLOv6 EffiDeHead (anchor-free): per level fp32 [rows, ld] in padded-grid row order: cols 0 .. 4(R+1)-1 the box (side-major: l, t, r, b
// x R+1 bins; R = reg_max), class logits from yolov6_cls_col(R).  R = 0: the four columns are the distances; R = 16: softmax over the 17
// bins projected on 0..16 (the fixed proj_conv).  raw[b][a][5+nc], a = level offset + y*W + x: cx, cy, w, h (input pixels), 1.0, the class
// sigmoids -- the YOLOv5 layout, so `conf = cls * obj` of the v5 post-processing is exactly the class probability.
// Up to four head levels by value (strides 8 / 16 / 32 / 64 of the P6 models), n of them in use.
struct YoloLevels { YoloLevel l[kYoloMaxLevels]; int n; };

// 3 levels, or 4 with a stride-64 level (YOLOv6-Lite); the per-anchor arithmetic does not depend on the level count.
__global__ void yolov6_decode_kernel(const YoloLevels L, int B, int nc, int reg_max, float* __restrict__ raw, int A) {
    const long long total = (long long)B * A;
    const int nb = reg_max + 1, cc = (int)yolov6_cls_col((unsigned)reg_max);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / A);
        int a = (int)(i % A);
        YoloLevel lv = L.l[0];
#pragma unroll
        for (int j = 1; j < kYoloMaxLevels; ++j)
            if (j < L.n && a >= lv.H * lv.W) { a -= lv.H * lv.W; lv = L.l[j]; }
        const int y = a / lv.W, x = a % lv.W;
        const float* p = lv.ptr + ((size_t)b * lv.rows_per_img + (size_t)(y + 1) * (lv.W + 2) + (x + 1)) * lv.ld;
        float d[4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            if (reg_max == 0) { d[s] = p[s]; continue; }
            float m = p[s * nb];
            for (int k = 1; k < nb; ++k) m = fmaxf(m, p[s * nb + k]);
            float den = 0.f, num = 0.f;
            for (int k = 0; k < nb; ++k) {
                const float e = expf(p[s * nb + k] - m);
                den += e;
                num += e * (float)k;
            }
            d[s] = num / den;
        }
        const float ax = (float)x + 0.5f, ay = (float)y + 0.5f;
        const float x1 = ax - d[0], y1 = ay - d[1], x2 = ax + d[2], y2 = ay + d[3];
        const float st = (float)lv.stride;
        float* o = raw + (size_t)i * (5 + nc);
        o[0] = (x1 + x2) * 0.5f * st;
        o[1] = (y1 + y2) * 0.5f * st;
        o[2] = (x2 - x1) * st;
        o[3] = (y2 - y1) * st;
        o[4] = 1.f;
        for (int c = 0; c < nc; ++c) o[5 + c] = 1.f / (1.f + expf(-p[cc + c]));
    }
}

int launch_yolov6_head_decode(const YoloLevel* lv, int n_levels, int B, int nc, int reg_max, float* raw, int A, cudaStream_t st) {
    ADAS_CHECK(n_levels == 3 || n_levels == kYoloMaxLevels, "YOLOv6 decode: %d levels (3 or 4)", n_levels);
    YoloLevels L;
    for (int j = 0; j < kYoloMaxLevels; ++j) L.l[j] = lv[j < n_levels ? j : 0];
    L.n = n_levels;
    const long long total = (long long)B * A;
    int blocks = (int)((total + 127) / 128);
    yolov6_decode_kernel<<<blocks, 128, 0, st>>>(L, B, nc, reg_max, raw, A);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

// YOLOv5 Detect: per level fp32 [rows, ld>=3*(5+nc)], channel = anchor*(5+nc) + k.
// raw[b][idx][5+nc], idx = level offset + anchor*H*W + y*W + x  (yoloDetector.py:45-48 ordering).
// Anchor (w, h) pairs [level][anchor]: the plan's own table (YOLOv7; 3 or 4 levels) or, without one, the YOLOv5 table below (3 levels).
__constant__ float c_v5_anchors[18] = {10, 13, 16, 30, 33, 23, 30, 61, 62, 45, 59, 119, 116, 90, 156, 198, 373, 326};

// lite != 0: the head of a YOLOv5-lite export -- sigmoid only, grid/anchor decode left to lite_postprocess (yoloDetector.py:36-50).
__global__ void yolov5_decode_kernel(const YoloLevels L, int B, int nc, float* __restrict__ raw, int A, int lite, const float* __restrict__ anchors) {
    const long long total = (long long)B * A;
    const int no = 5 + nc;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / A);
        int a = (int)(i % A);
        YoloLevel lv = L.l[0];
        int li = 0;
        // level of row a: unrolled with constant indices so the levels stay in registers / parameter space
#pragma unroll
        for (int j = 1; j < kYoloMaxLevels; ++j)
            if (j < L.n && a >= 3 * lv.H * lv.W) { a -= 3 * lv.H * lv.W; lv = L.l[j]; li = j; }
        const int hw = lv.H * lv.W;
        const int an = a / hw;
        const int r = a % hw;
        const int y = r / lv.W, x = r % lv.W;
        const float* p = lv.ptr + ((size_t)b * lv.rows_per_img + (size_t)(y + 1) * (lv.W + 2) + (x + 1)) * lv.ld + an * no;
        float* o = raw + ((size_t)b * A + (i % A)) * no;
        const float st = (float)lv.stride;
        const float sx = 1.f / (1.f + expf(-p[0])), sy = 1.f / (1.f + expf(-p[1]));
        const float sw = 1.f / (1.f + expf(-p[2])), sh = 1.f / (1.f + expf(-p[3]));
        if (lite) { o[0] = sx; o[1] = sy; o[2] = sw; o[3] = sh; }
        else {
            o[0] = (sx * 2.f - 0.5f + (float)x) * st;
            o[1] = (sy * 2.f - 0.5f + (float)y) * st;
            const float aw = anchors ? anchors[li * 6 + an * 2] : c_v5_anchors[li * 6 + an * 2];
            const float ah = anchors ? anchors[li * 6 + an * 2 + 1] : c_v5_anchors[li * 6 + an * 2 + 1];
            o[2] = (sw * 2.f) * (sw * 2.f) * aw;
            o[3] = (sh * 2.f) * (sh * 2.f) * ah;
        }
        for (int k = 4; k < no; ++k) o[k] = 1.f / (1.f + expf(-p[k]));
    }
}

int launch_yolov5_head_decode(const YoloLevel* lv, int n_levels, int B, int nc, float* raw, int A, int lite, const float* anchors, cudaStream_t st) {
    ADAS_CHECK(n_levels == 3 || (n_levels == kYoloMaxLevels && !lite && anchors != nullptr),
               "YOLOv5-layout decode: %d levels (3, or 4 with the plan's anchor table)", n_levels);
    YoloLevels L;
    for (int j = 0; j < kYoloMaxLevels; ++j) L.l[j] = lv[j < n_levels ? j : 0];
    L.n = n_levels;
    const long long total = (long long)B * A;
    int blocks = (int)((total + 127) / 128);
    yolov5_decode_kernel<<<blocks, 128, 0, st>>>(L, B, nc, raw, A, lite, anchors);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

// YoloLiteParameters.lite_postprocess (yoloDetector.py:36-50), in place on raw[b][idx][5+nc] like the reference: rows are ordered
// level -> anchor -> grid cell; per level h = int(in_h / stride), w = int(in_w / stride), grid = __make_grid(w, h) whose row r is
// (r % h, r // h) (np.meshgrid(arange(ny = h), arange(nx = w)) -- identical to (x, y) only for square inputs; kept as the reference
// computes it).  float32 arithmetic, one rounding per numpy op: xy = ((v * 2) - 0.5 + g) * stride ; wh = ((v * 2) ** 2) * anchor.
__global__ void yolov5_lite_post_kernel(float* __restrict__ raw, int B, int A, int nc, int in_h, int in_w) {
    const long long total = (long long)B * A;
    const int no = 5 + nc;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int a = (int)(i % A);
        int li = 0, h = 0, w = 0, stride = 8;
        for (li = 0; li < 3; ++li) {
            stride = 8 << li;
            h = in_h / stride; w = in_w / stride;
            if (a < 3 * h * w) break;
            a -= 3 * h * w;
        }
        if (li == 3) continue;              // rows past the three levels (never produced by a v5 head)
        const int hw = h * w;
        const int an = a / hw;
        const int r = a - an * hw;
        const float gx = (float)(r % h), gy = (float)(r / h);
        float* o = raw + (size_t)i * no;
        const float st = (float)stride;
        o[0] = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(o[0], 2.f), 0.5f), gx), st);
        o[1] = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(o[1], 2.f), 0.5f), gy), st);
        const float tw = __fmul_rn(o[2], 2.f), th = __fmul_rn(o[3], 2.f);
        o[2] = __fmul_rn(__fmul_rn(tw, tw), c_v5_anchors[li * 6 + an * 2]);
        o[3] = __fmul_rn(__fmul_rn(th, th), c_v5_anchors[li * 6 + an * 2 + 1]);
    }
}

int launch_yolov5_lite_post(float* raw, int B, int A, int nc, int in_h, int in_w, cudaStream_t st) {
    const long long total = (long long)B * A;
    int blocks = (int)((total + 127) / 128);
    yolov5_lite_post_kernel<<<blocks, 128, 0, st>>>(raw, B, A, nc, in_h, in_w);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Candidate selection: one thread per anchor (yoloDetector.py:120-128).
//   v8: probs = row[4:];  v5: probs = row[5:] * row[4] (float32 product);  first max wins ties;
//   keep iff float(conf) > box_score (float64 compare).
__global__ void yolo_select_kernel(const float* __restrict__ raw, int kind, int B, int A, int nc, double box_score,
                                   int32_t* __restrict__ flags, int32_t* __restrict__ cls, float* __restrict__ conf) {
    const long long total = (long long)B * A;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / A);
        const int a = (int)(i % A);
        float best = 0.f;
        int bi = 0;
        if (kind == 0) {
            const float* p = raw + (size_t)b * (4 + nc) * A + a;
            best = p[(size_t)4 * A];
            for (int c = 1; c < nc; ++c) {
                const float v = p[(size_t)(4 + c) * A];
                if (v > best) { best = v; bi = c; }
            }
        } else {
            const float* p = raw + ((size_t)b * A + a) * (5 + nc);
            const float obj = p[4];
            best = __fmul_rn(p[5], obj);
            for (int c = 1; c < nc; ++c) {
                const float v = __fmul_rn(p[5 + c], obj);
                if (v > best) { best = v; bi = c; }
            }
        }
        flags[i] = ((double)best > box_score) ? 1 : 0;
        cls[i] = bi;
        conf[i] = best;
    }
}

// ------------------------------------------------------------------------------------------------
// One CTA per frame: ordered compaction of the flagged anchors (ascending anchor index), box
// conversion to source-image xywh, then warp 0 runs the sequential NMS out of shared memory.
static constexpr int NMS_THREADS = 1024;

struct NmsSmem {   // dynamic smem carve-up, cap entries each
    double* x1; double* y1; double* x2; double* y2; double* idx; double* sc; double* ar;
};

__global__ void __launch_bounds__(NMS_THREADS)
yolo_compact_nms_kernel(const float* __restrict__ raw, int kind, int A, int nc, LetterboxGeom g, double nms_iou,
                        int max_det, int cap, int scap, double* __restrict__ work, const int32_t* __restrict__ flags, const int32_t* __restrict__ cls,
                        const float* __restrict__ conf, int32_t* __restrict__ n_cand, float* __restrict__ cand_box,
                        float* __restrict__ cand_conf, int32_t* __restrict__ cand_cls, float* __restrict__ out_box,
                        float* __restrict__ out_score, int32_t* __restrict__ out_cls, int32_t* __restrict__ out_idx,
                        int32_t* __restrict__ out_count) {
    extern __shared__ double nms_sm[];
    __shared__ int warp_tot[32];
    __shared__ int s_total;
    const int b = blockIdx.x;
    const int tid = threadIdx.x;
    const int lane = tid & 31, wid = tid >> 5;
    const int per = (A + NMS_THREADS - 1) / NMS_THREADS;   // consecutive anchors per thread
    const int a0 = tid * per;
    const int a1 = min(A, a0 + per);
    const int32_t* fl = flags + (size_t)b * A;

    int mine = 0;
    for (int a = a0; a < a1; ++a) mine += fl[a];
    // block exclusive scan of `mine`
    int incl = mine;
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int v = warp_tot[lane];
        int inc2 = v;
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc2, o);
            if (lane >= o) inc2 += t;
        }
        warp_tot[lane] = inc2 - v;
        if (lane == 31) s_total = inc2;
    }
    __syncthreads();
    int pos = warp_tot[wid] + incl - mine;
    const int total = s_total;
    const int N = min(total, cap);

    // float32 letterbox undo: (x - pad) * ratio, ratio = float32(old/new)  (utils.py:65-68,82-83)
    const float ratioh = (float)((double)g.src_h / (double)g.new_h);
    const float ratiow = (float)((double)g.src_w / (double)g.new_w);
    const float padw = (float)g.pad_w, padh = (float)g.pad_h;

    // NMS working set (7 doubles per candidate): shared memory while it fits (`scap` candidates), else this frame's slice of a
    // global scratch sized for every anchor -- the reference has no candidate limit (yoloDetector.py:104-133 keeps them all)
    double* base = (total <= scap) ? nms_sm : work + (size_t)b * cap * 7;
    const int cs = (total <= scap) ? scap : cap;
    double* X1 = base; double* Y1 = X1 + cs; double* X2 = Y1 + cs; double* Y2 = X2 + cs;
    double* ID = Y2 + cs; double* SC = ID + cs; double* AR = SC + cs;

    for (int a = a0; a < a1; ++a) {
        if (!fl[a]) continue;
        if (pos < cap) {
            float cx, cy, w, h;
            if (kind == 0) {
                const float* p = raw + (size_t)b * (4 + nc) * A + a;
                cx = p[0]; cy = p[(size_t)A]; w = p[(size_t)2 * A]; h = p[(size_t)3 * A];
            } else {
                const float* p = raw + ((size_t)b * A + a) * (5 + nc);
                cx = p[0]; cy = p[1]; w = p[2]; h = p[3];
            }
            const float hw = __fmul_rn(0.5f, w), hh = __fmul_rn(0.5f, h);
            float bx1 = __fsub_rn(cx, hw), by1 = __fsub_rn(cy, hh), bx2 = __fadd_rn(cx, hw), by2 = __fadd_rn(cy, hh);
            bx1 = __fmul_rn(__fsub_rn(bx1, padw), ratiow);
            bx2 = __fmul_rn(__fsub_rn(bx2, padw), ratiow);
            by1 = __fmul_rn(__fsub_rn(by1, padh), ratioh);
            by2 = __fmul_rn(__fsub_rn(by2, padh), ratioh);
            const float bw = __fsub_rn(bx2, bx1), bh = __fsub_rn(by2, by1);
            float* cb = cand_box + ((size_t)b * cap + pos) * 4;
            cb[0] = bx1; cb[1] = by1; cb[2] = bw; cb[3] = bh;
            const float cf = conf[(size_t)b * A + a];
            cand_conf[(size_t)b * cap + pos] = cf;
            cand_cls[(size_t)b * cap + pos] = cls[(size_t)b * A + a];
            // NMS working copy: xywh -> xyxy in float32 (utils.py:186-187), then float64
            X1[pos] = (double)bx1; Y1[pos] = (double)by1;
            X2[pos] = (double)__fadd_rn(bx1, bw); Y2[pos] = (double)__fadd_rn(by1, bh);
            ID[pos] = (double)pos; SC[pos] = (double)cf;
        }
        ++pos;
    }
    if (tid == 0) n_cand[b] = total;
    __syncthreads();
    if (wid != 0) return;

    // ---------------- sequential NMS, one warp ----------------
    for (int j = lane; j < N; j += 32) AR[j] = __dmul_rn(__dadd_rn(__dsub_rn(X2[j], X1[j]), 1.0), __dadd_rn(__dsub_rn(Y2[j], Y1[j]), 1.0));
    __syncwarp();
    for (int i = 0; i + 1 < N; ++i) {
        const int p0 = i + 1;
        // argmax of SC[p0:], first maximum
        double bv = -1.0; int bj = 0x7fffffff;
        for (int j = p0 + lane; j < N; j += 32) {
            const double v = SC[j];
            if (v > bv) { bv = v; bj = j; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
            if (ov > bv || (ov == bv && oj < bj)) { bv = ov; bj = oj; }
        }
        // Once every remaining score is 0 nothing can change any more (no swap: 0 < 0 is false; suppression only
        // writes zeros), so the remaining iterations of the reference loop are no-ops: stop here.
        if (!(bv > 0.0)) break;
        if (lane == 0 && SC[i] < bv) {
            // dets[i,:] <- dets[maxpos,:]; dets[maxpos,:] keeps its values (tBD is a view of row i)
            X1[i] = X1[bj]; Y1[i] = Y1[bj]; X2[i] = X2[bj]; Y2[i] = Y2[bj]; ID[i] = ID[bj];
            const double ts = SC[i]; SC[i] = SC[bj]; SC[bj] = ts;
            const double ta = AR[i]; AR[i] = AR[bj]; AR[bj] = ta;
        }
        __syncwarp();
        const double ix1 = X1[i], iy1 = Y1[i], ix2 = X2[i], iy2 = Y2[i], ia = AR[i];
        for (int j = p0 + lane; j < N; j += 32) {
            if (SC[j] == 0.0) continue;                  // already suppressed: weight * 0 stays 0
            const double xx1 = fmax(ix1, X1[j]), yy1 = fmax(iy1, Y1[j]);
            const double xx2 = fmin(ix2, X2[j]), yy2 = fmin(iy2, Y2[j]);
            const double w = fmax(0.0, __dadd_rn(__dsub_rn(xx2, xx1), 1.0));
            const double h = fmax(0.0, __dadd_rn(__dsub_rn(yy2, yy1), 1.0));
            const double inter = __dmul_rn(w, h);
            const double ovr = __ddiv_rn(inter, __dsub_rn(__dadd_rn(ia, AR[j]), inter));
            if (ovr > nms_iou) SC[j] = 0.0;   // weight 0; weight 1 leaves the score unchanged
        }
        __syncwarp();
    }
    // keep = dets[:,4][scores > 0.001], in row order
    int outn = 0;
    for (int base = 0; base < N; base += 32) {
        const int j = base + lane;
        const bool keep = (j < N) && (SC[j] > 0.001);
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            const int o = outn + __popc(m & ((1u << lane) - 1u));
            if (o < max_det) {
                const int ci = (int)ID[j];
                const float* cb = cand_box + ((size_t)b * cap + ci) * 4;
                float* ob = out_box + ((size_t)b * max_det + o) * 4;
                ob[0] = cb[0]; ob[1] = cb[1]; ob[2] = cb[2]; ob[3] = cb[3];
                out_score[(size_t)b * max_det + o] = cand_conf[(size_t)b * cap + ci];
                out_cls[(size_t)b * max_det + o] = cand_cls[(size_t)b * cap + ci];
                out_idx[(size_t)b * max_det + o] = ci;
            }
        }
        outn += __popc(m);
    }
    if (lane == 0) out_count[b] = outn;
}

int launch_yolo_post(const float* raw, int kind, int B, int A, int nc, const LetterboxGeom& g, double box_score,
                     double nms_iou, int max_det, YoloPostBufs& w, cudaStream_t st) {
    const long long total = (long long)B * A;
    int blocks = (int)((total + 127) / 128);
    yolo_select_kernel<<<blocks, 128, 0, st>>>(raw, kind, B, A, nc, box_score, w.flags, w.cls, w.conf);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    const int scap = w.cap < 2048 ? w.cap : 2048;            // candidates whose working set lives in shared memory (112 KiB)
    const int smem = scap * 7 * (int)sizeof(double);
    {   // the >48 KiB opt-in is a per-device attribute: set it once per device (advisor finding, r01)
        static std::mutex mu;
        static bool attr_set[64] = {false};
        int dev = 0;
        ADAS_CUDA(cudaGetDevice(&dev));
        std::lock_guard<std::mutex> lk(mu);
        if (dev >= 0 && dev < 64 && !attr_set[dev]) {
            ADAS_CUDA(cudaFuncSetAttribute(yolo_compact_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            attr_set[dev] = true;
        }
    }
    yolo_compact_nms_kernel<<<B, NMS_THREADS, smem, st>>>(raw, kind, A, nc, g, nms_iou, max_det, w.cap, scap, w.nms_work, w.flags, w.cls, w.conf,
                                                          w.n_cand, w.cand_box, w.cand_conf, w.cand_cls, w.out_box,
                                                          w.out_score, w.out_cls, w.out_idx, w.out_count);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace adas
