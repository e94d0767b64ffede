// dwconv.cu -- depthwise k x k convolution (k = 3 or 5, stride 1 or 2; k = 7, stride 1) of a channel slice of a padded-NHWC fp16 buffer
// (OP_DWCONV).
//
// YOLOv10's SCDown, CIB, RepVGGDW (folded to one 7x7), PSA's positional conv and the v10 classification head; YOLOv6-Lite's 3x3 and 5x5
// (DPBlock) depthwise convs.  Packing these as dense
// block-diagonal GEMMs would do C times the work and read C times the weight bytes, so they run here instead:
//   one thread = 8 channels (one 16-byte vector) x DW_TX consecutive output pixels of one output row;
//   per filter row the (DW_TX - 1) * S + K input pixels that the DW_TX windows cover are loaded once into registers and shared by all
//   DW_TX outputs; the K input rows a thread reads are also read by the K - 1 neighbouring output rows, which run in the same or the
//   next few CTAs, so those re-reads are served by L1 / L2 rather than HBM;
//   weights are packed [k*k][C] fp16 (one tap of 8 channels = one 16-byte load), bias fp32, accumulation fp32 in a fixed tap order;
//   epilogue: out = act(acc + bias) (+ res), rounded to fp16 once (act 0 none, 1 SiLU, 5 Hardswish).
// Taps are bound-checked against the H x W interior: the buffer's halo is one pixel wide and a 5x5 / 7x7 window reaches two / three pixels
// out, so
// an unchecked tap would read the neighbouring row of the padded matrix (or the next image) instead of zero.  Only interior pixels of
// the output slice are written; its halo stays zero.
#include "common.h"
#include "tc_common.cuh"

namespace adas {

static constexpr int DW_THREADS = 256;
static constexpr int DW_TX = 4;                 // output pixels per thread along x

struct DwParams {
    const __half* in;   int in_ld;              // channel slice start, row stride (elements)
    const __half* w;                            // [k*k][C]
    const float* bias;                          // [C]
    const __half* res;  int res_ld;             // residual slice (Ho x Wo padded geometry) or nullptr
    __half* out;        int out_ld;
    int B, H, W, C, Ho, Wo, act, xblocks;
};

__device__ __forceinline__ void dw_fma8(float (&acc)[8], const uint4& x, const uint4& w) {
    const __half2* xh = reinterpret_cast<const __half2*>(&x);
    const __half2* wh = reinterpret_cast<const __half2*>(&w);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 xf = __half22float2(xh[j]), wf = __half22float2(wh[j]);
        acc[2 * j] = fmaf(xf.x, wf.x, acc[2 * j]);
        acc[2 * j + 1] = fmaf(xf.y, wf.y, acc[2 * j + 1]);
    }
}

template <int K, int S>
__global__ void __launch_bounds__(DW_THREADS) dwconv_kernel(const DwParams p) {
    constexpr int NX = (DW_TX - 1) * S + K;     // input pixels of one filter row covered by the DW_TX windows
    const int c8 = p.C >> 3;
    const long long total = (long long)p.B * p.Ho * p.xblocks * c8;
    const int Wp = p.W + 2, Wpo = p.Wo + 2;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(i % c8);
        long long t = i / c8;
        const int xb = (int)(t % p.xblocks); t /= p.xblocks;
        const int y = (int)(t % p.Ho);
        const int b = (int)(t / p.Ho);
        const int x0 = xb * DW_TX;
        const int ix0 = x0 * S - K / 2, iy0 = y * S - K / 2;
        float acc[DW_TX][8];
#pragma unroll
        for (int tx = 0; tx < DW_TX; ++tx)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[tx][j] = 0.f;
        const __half* wc = p.w + cg * 8;
#pragma unroll 1
        for (int dy = 0; dy < K; ++dy) {
            const int iy = iy0 + dy;
            if (iy < 0 || iy >= p.H) continue;                  // zero padding rows (the halo holds only one of them)
            const __half* row = p.in + (((size_t)b * (p.H + 2) + iy + 1) * Wp + 1) * p.in_ld + cg * 8;
            uint4 v[NX];
#pragma unroll
            for (int j = 0; j < NX; ++j) {
                const int ix = ix0 + j;
                v[j] = (ix >= 0 && ix < p.W) ? __ldg(reinterpret_cast<const uint4*>(row + (size_t)ix * p.in_ld)) : make_uint4(0u, 0u, 0u, 0u);
            }
#pragma unroll
            for (int dx = 0; dx < K; ++dx) {
                const uint4 wv = __ldg(reinterpret_cast<const uint4*>(wc + (size_t)(dy * K + dx) * p.C));
#pragma unroll
                for (int tx = 0; tx < DW_TX; ++tx) dw_fma8(acc[tx], v[tx * S + dx], wv);
            }
        }
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + cg * 8));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bias + cg * 8 + 4));
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        const size_t orow = ((size_t)b * (p.Ho + 2) + y + 1) * Wpo + x0 + 1;
#pragma unroll
        for (int tx = 0; tx < DW_TX; ++tx) {
            if (x0 + tx >= p.Wo) break;
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = act_apply(acc[tx][j] + bb[j], p.act);
            if (p.res) {
                const uint4 r = *reinterpret_cast<const uint4*>(p.res + (orow + tx) * p.res_ld + cg * 8);
                const __half2* rh = reinterpret_cast<const __half2*>(&r);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 rf = __half22float2(rh[j]);
                    o[2 * j] += rf.x;
                    o[2 * j + 1] += rf.y;
                }
            }
            uint4 ov;
            __half2* oh = reinterpret_cast<__half2*>(&ov);
#pragma unroll
            for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(o[2 * j], o[2 * j + 1]);
            *reinterpret_cast<uint4*>(p.out + (orow + tx) * p.out_ld + cg * 8) = ov;
        }
    }
}

int launch_dwconv(const __half* in, int in_ld, int B, int H, int W, int C, int k, int stride, const __half* w, const float* bias, int act,
                  const __half* res, int res_ld, __half* out, int out_ld, int Ho, int Wo, cudaStream_t st) {
    ADAS_CHECK(C % 8 == 0 && in_ld % 8 == 0 && out_ld % 8 == 0 && (res == nullptr || res_ld % 8 == 0), "dwconv: channel alignment");
    ADAS_CHECK(((k == 3 || k == 5) && (stride == 1 || stride == 2)) || (k == 7 && stride == 1), "dwconv: k %d stride %d (3 / 5 s1 / s2, 7 s1)", k, stride);
    ADAS_CHECK(Ho == (H + 2 * (k / 2) - k) / stride + 1 && Wo == (W + 2 * (k / 2) - k) / stride + 1, "dwconv: output geometry %dx%d of %dx%d", Ho, Wo, H, W);
    DwParams p;
    p.in = in; p.in_ld = in_ld; p.w = w; p.bias = bias; p.res = res; p.res_ld = res_ld; p.out = out; p.out_ld = out_ld;
    p.B = B; p.H = H; p.W = W; p.C = C; p.Ho = Ho; p.Wo = Wo; p.act = act; p.xblocks = (Wo + DW_TX - 1) / DW_TX;
    const long long total = (long long)B * Ho * p.xblocks * (C / 8);
    long long blocks = (total + DW_THREADS - 1) / DW_THREADS;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (k == 7) dwconv_kernel<7, 1><<<(int)blocks, DW_THREADS, 0, st>>>(p);
    else if (k == 5 && stride == 2) dwconv_kernel<5, 2><<<(int)blocks, DW_THREADS, 0, st>>>(p);
    else if (k == 5) dwconv_kernel<5, 1><<<(int)blocks, DW_THREADS, 0, st>>>(p);
    else if (stride == 2) dwconv_kernel<3, 2><<<(int)blocks, DW_THREADS, 0, st>>>(p);
    else dwconv_kernel<3, 1><<<(int)blocks, DW_THREADS, 0, st>>>(p);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace adas
