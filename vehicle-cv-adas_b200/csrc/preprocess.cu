// preprocess.cu -- frame pre-processing on the device, bit-exact with the reference's OpenCV path.
//
// Replaces:
//   Scaler.process_image            ObjectDetector/utils.py:42-63   (letterbox, cv2.resize INTER_LINEAR on uint8, pad 114)
//   YoloDetector.__prepare_input    ObjectDetector/yoloDetector.py:96-102 (blobFromImage: swapRB, *1/255, NCHW)
//   UltrafastLaneDetectorV2.__prepare_input  TrafficLaneDetector/ufldDetector/ultrafastLaneDetectorV2.py:96-112
//                                   (BGR->RGB, resize to (W, int(H/crop)), keep bottom rows, (x/255-mean)/std in float64)
//
// cv2.resize(INTER_LINEAR) on 8-bit data is fixed point: 11-bit coefficients per axis
// (x: source index clamped to [0, w-1] with the fraction zeroed at the borders; y: fraction kept,
// row indices clipped), horizontal pass in int32, vertical pass
//   ((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2.
// The coefficient tables are built on the host in the same float/double arithmetic OpenCV uses,
// so the kernel is integer-only and reproduces cv2's bytes exactly (verified against cv2 4.13).
#include "common.h"
#include <math.h>
#include <map>
#include <mutex>

namespace adas {

LetterboxGeom letterbox_geom(int src_h, int src_w, int in_h, int in_w) {
    // Scaler.process_image, utils.py:45-56 (note the "+ 1" on the short side and int() truncation)
    LetterboxGeom g;
    g.src_h = src_h; g.src_w = src_w; g.in_h = in_h; g.in_w = in_w;
    g.new_h = in_h; g.new_w = in_w; g.pad_h = 0; g.pad_w = 0;
    if (src_h != src_w) {
        const double hw_scale = (double)src_h / (double)src_w;
        if (hw_scale > 1.0) {
            g.new_h = in_h;
            g.new_w = (int)((double)in_w / hw_scale);
            g.pad_w = (int)((double)(in_w - g.new_w) * 0.5);
        } else {
            g.new_h = (int)((double)in_h * hw_scale) + 1;
            g.new_w = in_w;
            g.pad_h = (int)((double)(in_h - g.new_h) * 0.5);
        }
    }
    return g;
}

struct ResizeTab {
    int* xofs = nullptr;     // [dw]   left source column
    int* xofs1 = nullptr;    // [dw]   right source column
    short* xa = nullptr;     // [dw*2] coefficients
    int* yofs = nullptr;     // [dh]   upper source row (clipped)
    int* yofs1 = nullptr;    // [dh]   lower source row (clipped)
    short* yb = nullptr;     // [dh*2]
};

static short sat_short_round(float v) {
    long r = lrintf(v);   // round half to even, like cvRound
    if (r > 32767) r = 32767;
    if (r < -32768) r = -32768;
    return (short)r;
}

// One table set per (device, src w/h, dst w/h); tiny, cached for the process lifetime.
static int get_resize_tab(int sw, int sh, int dw, int dh, ResizeTab* out) {
    static std::mutex mu;
    static std::map<std::vector<int>, ResizeTab> cache;
    int dev = 0;
    ADAS_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(mu);
    std::vector<int> key = {dev, sw, sh, dw, dh};
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return 0; }
    std::vector<int> xo(dw), xo1(dw), yo(dh), yo1(dh);
    std::vector<short> xa(dw * 2), yb(dh * 2);
    const double scale_x = 1.0 / ((double)dw / (double)sw);
    const double scale_y = 1.0 / ((double)dh / (double)sh);
    for (int dx = 0; dx < dw; ++dx) {
        float fx = (float)((dx + 0.5) * scale_x - 0.5);
        int sx = (int)floorf(fx);
        fx -= (float)sx;
        if (sx < 0) { fx = 0.f; sx = 0; }
        if (sx >= sw - 1) { fx = 0.f; sx = sw - 1; }
        xo[dx] = sx;
        xo1[dx] = sx + 1 < sw ? sx + 1 : sw - 1;
        xa[dx * 2] = sat_short_round((1.f - fx) * 2048.f);
        xa[dx * 2 + 1] = sat_short_round(fx * 2048.f);
    }
    for (int dy = 0; dy < dh; ++dy) {
        float fy = (float)((dy + 0.5) * scale_y - 0.5);
        int sy = (int)floorf(fy);
        fy -= (float)sy;
        int s0 = sy, s1 = sy + 1;
        if (s0 < 0) s0 = 0; if (s0 > sh - 1) s0 = sh - 1;
        if (s1 < 0) s1 = 0; if (s1 > sh - 1) s1 = sh - 1;
        yo[dy] = s0; yo1[dy] = s1;
        yb[dy * 2] = sat_short_round((1.f - fy) * 2048.f);
        yb[dy * 2 + 1] = sat_short_round(fy * 2048.f);
    }
    ResizeTab t;
    ADAS_CUDA(cudaMalloc(&t.xofs, dw * sizeof(int)));
    ADAS_CUDA(cudaMalloc(&t.xofs1, dw * sizeof(int)));
    ADAS_CUDA(cudaMalloc(&t.xa, dw * 2 * sizeof(short)));
    ADAS_CUDA(cudaMalloc(&t.yofs, dh * sizeof(int)));
    ADAS_CUDA(cudaMalloc(&t.yofs1, dh * sizeof(int)));
    ADAS_CUDA(cudaMalloc(&t.yb, dh * 2 * sizeof(short)));
    ADAS_CUDA(cudaMemcpy(t.xofs, xo.data(), dw * sizeof(int), cudaMemcpyHostToDevice));
    ADAS_CUDA(cudaMemcpy(t.xofs1, xo1.data(), dw * sizeof(int), cudaMemcpyHostToDevice));
    ADAS_CUDA(cudaMemcpy(t.xa, xa.data(), dw * 2 * sizeof(short), cudaMemcpyHostToDevice));
    ADAS_CUDA(cudaMemcpy(t.yofs, yo.data(), dh * sizeof(int), cudaMemcpyHostToDevice));
    ADAS_CUDA(cudaMemcpy(t.yofs1, yo1.data(), dh * sizeof(int), cudaMemcpyHostToDevice));
    ADAS_CUDA(cudaMemcpy(t.yb, yb.data(), dh * 2 * sizeof(short), cudaMemcpyHostToDevice));
    cache[key] = t;
    *out = t;
    return 0;
}

// bilinear sample of all three channels of resized pixel (dy, dx); returns BGR bytes
__device__ __forceinline__ void resize_px(const uint8_t* __restrict__ src, int sw, const ResizeTab& t, int dy, int dx,
                                          int (&bgr)[3]) {
    const int x0 = t.xofs[dx], x1 = t.xofs1[dx];
    const int a0 = t.xa[dx * 2], a1 = t.xa[dx * 2 + 1];
    const int y0 = t.yofs[dy], y1 = t.yofs1[dy];
    const int b0 = t.yb[dy * 2], b1 = t.yb[dy * 2 + 1];
    const uint8_t* r0 = src + (size_t)y0 * sw * 3;
    const uint8_t* r1 = src + (size_t)y1 * sw * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int h0 = (int)r0[x0 * 3 + c] * a0 + (int)r0[x1 * 3 + c] * a1;
        const int h1 = (int)r1[x0 * 3 + c] * a0 + (int)r1[x1 * 3 + c] * a1;
        int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
        v = v < 0 ? 0 : (v > 255 ? 255 : v);
        bgr[c] = v;
    }
}

// YOLO letterbox + blob. One thread per network-input pixel.
__global__ void yolo_pre_kernel(const uint8_t* __restrict__ frames, int B, LetterboxGeom g, ResizeTab t,
                                __half* __restrict__ img, int img_ld, float* __restrict__ blob) {
    const long long total = (long long)B * g.in_h * g.in_w;
    const float inv255 = (float)(1.0 / 255.0);   // blobFromImage multiplies in float32
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % g.in_w);
        long long r = i / g.in_w;
        const int y = (int)(r % g.in_h);
        const int b = (int)(r / g.in_h);
        int bgr[3] = {114, 114, 114};
        const int ry = y - g.pad_h, rx = x - g.pad_w;
        if (ry >= 0 && ry < g.new_h && rx >= 0 && rx < g.new_w)
            resize_px(frames + (size_t)b * g.src_h * g.src_w * 3, g.src_w, t, ry, rx, bgr);
        const float rf = __fmul_rn((float)bgr[2], inv255);
        const float gf = __fmul_rn((float)bgr[1], inv255);
        const float bf = __fmul_rn((float)bgr[0], inv255);
        if (img != nullptr) {
            const size_t row = ((size_t)b * (g.in_h + 2) + (y + 1)) * (g.in_w + 2) + (x + 1);
            __half2 lo = __floats2half2_rn(rf, gf);
            __half2 hi = __floats2half2_rn(bf, 0.f);
            uint2 v;
            v.x = *reinterpret_cast<uint32_t*>(&lo);
            v.y = *reinterpret_cast<uint32_t*>(&hi);
            *reinterpret_cast<uint2*>(img + row * img_ld) = v;
        }
        if (blob != nullptr) {
            const size_t plane = (size_t)g.in_h * g.in_w;
            float* o = blob + (size_t)b * 3 * plane + (size_t)y * g.in_w + x;
            o[0] = rf; o[plane] = gf; o[2 * plane] = bf;
        }
    }
}

int launch_yolo_pre(const uint8_t* frames, int B, const LetterboxGeom& g, __half* img_padded, int img_ld,
                    float* blob_nchw, cudaStream_t st) {
    ResizeTab t;
    if (get_resize_tab(g.src_w, g.src_h, g.new_w, g.new_h, &t)) return 1;
    const long long total = (long long)B * g.in_h * g.in_w;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    yolo_pre_kernel<<<blocks, 256, 0, st>>>(frames, B, g, t, img_padded, img_ld, blob_nchw);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

// UFLD: resize to (in_w, resize_h), keep the bottom in_h rows, per-channel LUT (float64 math done on host).
__global__ void ufld_pre_kernel(const uint8_t* __restrict__ frames, int B, int H, int W, int in_h, int in_w, int row0,
                                ResizeTab t, const float* __restrict__ lut, __half* __restrict__ img, int img_ld,
                                float* __restrict__ blob) {
    const long long total = (long long)B * in_h * in_w;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % in_w);
        long long r = i / in_w;
        const int y = (int)(r % in_h);
        const int b = (int)(r / in_h);
        int bgr[3];
        resize_px(frames + (size_t)b * H * W * 3, W, t, y + row0, x, bgr);
        const float rf = lut[bgr[2]];
        const float gf = lut[256 + bgr[1]];
        const float bf = lut[512 + bgr[0]];
        if (img != nullptr) {
            const size_t row = ((size_t)b * (in_h + 2) + (y + 1)) * (in_w + 2) + (x + 1);
            __half2 lo = __floats2half2_rn(rf, gf);
            __half2 hi = __floats2half2_rn(bf, 0.f);
            uint2 v;
            v.x = *reinterpret_cast<uint32_t*>(&lo);
            v.y = *reinterpret_cast<uint32_t*>(&hi);
            *reinterpret_cast<uint2*>(img + row * img_ld) = v;
        }
        if (blob != nullptr) {
            const size_t plane = (size_t)in_h * in_w;
            float* o = blob + (size_t)b * 3 * plane + (size_t)y * in_w + x;
            o[0] = rf; o[plane] = gf; o[2 * plane] = bf;
        }
    }
}

int launch_ufld_pre(const uint8_t* frames, int B, int H, int W, int in_h, int in_w, int resize_h, const float* lut,
                    __half* img_padded, int img_ld, float* blob_nchw, cudaStream_t st) {
    ResizeTab t;
    if (get_resize_tab(W, H, in_w, resize_h, &t)) return 1;
    ADAS_CHECK(resize_h >= in_h, "ufld_pre: resized height %d smaller than network height %d", resize_h, in_h);
    const long long total = (long long)B * in_h * in_w;
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    ufld_pre_kernel<<<blocks, 256, 0, st>>>(frames, B, H, W, in_h, in_w, resize_h - in_h, t, lut, img_padded, img_ld,
                                            blob_nchw);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace adas
