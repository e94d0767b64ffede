// lite_ops.cu -- the two mobile-network ops of YOLOv6-Lite: squeeze-excite (OP_SE) and the concat + channel shuffle of two channel
// slices (OP_SHUFFLE2).  Both read and write padded-NHWC fp16 channel slices, interior pixels only (halos stay zero).
//
// OP_SE: out(y, x, c) = x(y, x, c) * gate[c],  gate = hardsigmoid(W2 relu(W1 mean(x) + b1) + b2)   (upstream SEBlock, 1x1 convs with bias)
//   One CTA per image.  The per-image input of every SE of the Lite nets is small (at most 80 x 80 x 16 or 40 x 40 x 96 halves at
//   320 x 320, ~200 KB), so one CTA reads it twice (the second pass mostly from L2) in a few microseconds, and the whole op -- mean,
//   both FCs and the scaling -- is one launch with no cross-CTA partials, no atomics and no second kernel.  Splitting an image over
//   several CTAs would need either a grid-wide barrier or a separate gate kernel; at these sizes launch latency dominates either way.
//   The mean is deterministic and batch-invariant: thread (pixel slot s, channel group g) sums pixels s, s + S, s + 2S, ... in that
//   order (S = pixel slots of the CTA, fixed by C alone), then channel c sums the S slot partials in ascending slot order and divides
//   by H * W.  The FCs are fp32 dot products in ascending index order (weights fp32).  The product x * gate is rounded to fp16 once.
//   In place (out == in) is allowed: every element is read (pass 1) before the barrier and then read and written by one thread.
//
// OP_SHUFFLE2: out(y, x, 2j) = a(y, x, j), out(y, x, 2j + 1) = b(y, x, j) for j < n -- torch.cat([a, b], 1) followed by
//   channel_shuffle(groups = 2).  Pure data movement (bit exact): one thread moves 8 channels of each source (two 16-byte loads) to 16
//   interleaved output channels (two 16-byte stores).
#include "common.h"
#include "tc_common.cuh"

namespace adas {

static constexpr int SE_THREADS = 512;

__global__ void __launch_bounds__(SE_THREADS) se_kernel(const SeParams p) {
    __shared__ float part[SE_THREADS * 8];             // [slot][C] slot partial sums (slots * C <= SE_THREADS * 8)
    __shared__ float mean[kSeMaxC];
    __shared__ float hid[kSeMaxC / 4];
    __shared__ float gate[kSeMaxC];
    const int b = blockIdx.x, c8 = p.C >> 3, slots = SE_THREADS / c8, HW = p.H * p.W, Wp = p.W + 2;
    const int cg = threadIdx.x % c8, slot = threadIdx.x / c8;
    const size_t img_row0 = (size_t)b * (p.H + 2) * Wp;
    auto row_of = [&](int px) { const int y = px / p.W; return img_row0 + (size_t)(y + 1) * Wp + (px - y * p.W) + 1; };
    // pass 1: per-slot channel sums
    if (slot < slots) {
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int px = slot; px < HW; px += slots) {
            const uint4 v = *reinterpret_cast<const uint4*>(p.in + row_of(px) * p.in_ld + cg * 8);
            const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(h[j]);
                acc[2 * j] += f.x;
                acc[2 * j + 1] += f.y;
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) part[slot * p.C + cg * 8 + j] = acc[j];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < p.C; c += SE_THREADS) {
        float s = 0.f;
        for (int k = 0; k < slots; ++k) s += part[k * p.C + c];
        mean[c] = s / (float)HW;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < p.hid; j += SE_THREADS) {
        const float* w = p.w1 + (size_t)j * p.C;
        float s = p.b1[j];
        for (int c = 0; c < p.C; ++c) s = fmaf(w[c], mean[c], s);
        hid[j] = fmaxf(s, 0.f);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < p.C; c += SE_THREADS) {
        const float* w = p.w2 + (size_t)c * p.hid;
        float s = p.b2[c];
        for (int j = 0; j < p.hid; ++j) s = fmaf(w[j], hid[j], s);
        gate[c] = fminf(fmaxf(s + 3.f, 0.f), 6.f) / 6.f;          // hardsigmoid
    }
    __syncthreads();
    // pass 2: scale
    if (slot < slots) {
        float g[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] = gate[cg * 8 + j];
        for (int px = slot; px < HW; px += slots) {
            const size_t r = row_of(px);
            const uint4 v = *reinterpret_cast<const uint4*>(p.in + r * p.in_ld + cg * 8);
            const __half2* h = reinterpret_cast<const __half2*>(&v);
            uint4 o;
            __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(h[j]);
                oh[j] = __floats2half2_rn(f.x * g[2 * j], f.y * g[2 * j + 1]);
            }
            *reinterpret_cast<uint4*>(p.out + r * p.out_ld + cg * 8) = o;
        }
    }
}

int se_supported(int C, int hid) { return C >= 8 && C % 8 == 0 && C <= kSeMaxC && hid >= 1 && hid <= kSeMaxC / 4; }

int launch_se(const SeParams& p, cudaStream_t st) {
    ADAS_CHECK(se_supported(p.C, p.hid), "se: %d channels, %d hidden (C a multiple of 8 up to %d, 1 to %d hidden)", p.C, p.hid, kSeMaxC, kSeMaxC / 4);
    ADAS_CHECK(p.in_ld % 8 == 0 && p.out_ld % 8 == 0 && p.B >= 1 && p.H >= 1 && p.W >= 1, "se: channel alignment / geometry");
    se_kernel<<<p.B, SE_THREADS, 0, st>>>(p);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

__global__ void shuffle2_kernel(const __half* __restrict__ a, int a_ld, const __half* __restrict__ b, int b_ld, __half* __restrict__ out,
                                int out_ld, int B, int H, int W, int n8) {
    const long long total = (long long)B * H * W * n8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(i % n8);
        long long t = i / n8;
        const int x = (int)(t % W); t /= W;
        const int y = (int)(t % H);
        const int im = (int)(t / H);
        const size_t r = ((size_t)im * (H + 2) + y + 1) * (W + 2) + x + 1;
        const uint4 va = __ldg(reinterpret_cast<const uint4*>(a + r * a_ld + cg * 8));
        const uint4 vb = __ldg(reinterpret_cast<const uint4*>(b + r * b_ld + cg * 8));
        const uint32_t* ua = reinterpret_cast<const uint32_t*>(&va);
        const uint32_t* ub = reinterpret_cast<const uint32_t*>(&vb);
        uint32_t o[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {                          // halves (a 2k, a 2k+1) and (b 2k, b 2k+1) -> a 2k, b 2k, a 2k+1, b 2k+1
            o[2 * k] = __byte_perm(ua[k], ub[k], 0x5410);
            o[2 * k + 1] = __byte_perm(ua[k], ub[k], 0x7632);
        }
        uint4* dst = reinterpret_cast<uint4*>(out + r * out_ld + cg * 16);
        dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
        dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
    }
}

int launch_shuffle2(const __half* a, int a_ld, const __half* b, int b_ld, __half* out, int out_ld, int B, int H, int W, int n, cudaStream_t st) {
    ADAS_CHECK(n >= 8 && n % 8 == 0 && a_ld % 8 == 0 && b_ld % 8 == 0 && out_ld % 8 == 0, "shuffle2: %d channels per source (a multiple of 8)", n);
    const long long total = (long long)B * H * W * (n / 8);
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    shuffle2_kernel<<<(int)blocks, 256, 0, st>>>(a, a_ld, b, b_ld, out, out_ld, B, H, W, n / 8);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace adas
