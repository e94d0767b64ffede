// stem_conv.cu -- the first convolution of a network (k x k, stride 1 or 2, 3 input channels) read straight from the padded NHWC image.
//
// Replaces, for the stem only, the patch-matrix route (im2col_kernel / stempack_kernel + a GEMM launch): the image has C = 4
// (R, G, B, 0) per pixel, so the k pixels one output needs from one input row are k*4 CONTIGUOUS halves.  The reduction index is laid
// out as  K = k rows x KR,  KR = round_up(4k, 16):  element [dy][dx*4 + c]  (zero weights in the padding), which makes every
// 16-wide k-step of a warp-level mma.m16n8k16 a run of consecutive bytes of one image row -- no gather, no patch matrix in memory.
// The stem has 3 input channels: the GEMM kernel's 64-channel k-blocks would be > 50 % zeros behind an im2col pass, and the layer
// is bound by writing its 64-channel output anyway.
//
// One warp owns 16 consecutive output pixels of one output row (the M of m16n8k16) and all Cout channels (NT n-tiles of 8):
//   k-slot permutation: a thread of the warp MMA holds k-slots {2t, 2t+1, 2t+8, 2t+9} of a 16-wide step.  Mapping those four slots to
//                the four CONTIGUOUS halves 4t .. 4t+3 of the 32-byte row chunk (one pixel) for BOTH operands leaves the dot product
//                unchanged and turns the fragment loads into one 8-byte load per operand row (instead of two 4-byte loads);
//   A fragments: 8-byte global loads = one pixel (coalesced: 4 lanes x 8 B per output pixel), predicated at the image border (the padded
//                layout only has a one-pixel halo; k = 6 / 7 stems reach further out);
//   B fragments: folded weights in shared memory in plain [dy][dx*4 + c] order, row stride = 16 (mod 64) halves so that the 8-byte
//                fragment loads of a half-warp hit distinct banks;
//   epilogue:    + bias -> activation -> fp16 -> per-warp staging in shared memory -> 16-byte coalesced stores of interior pixels.
// Accumulation is fp32 in a fixed order, independent of the batch size and of the grid: frame k of a batch equals the batch-1 result.
//
// Reference: the conv stacks behind coreEngine.py:150-157 / 184-186 (first Conv of YOLOv8 [3x3 s2], YOLOv5 [6x6 s2 p2], ResNet [7x7 s2 p3],
// YOLOv7 [3x3 s1 at full input resolution], YOLOv7-tiny [3x3 s2], YOLOv7-W6 / E6 / E6E [ReOrg + 3x3 folded into 6x6 s2 p2, 64 / 80
// channels; 96 for D6]).
#include "common.h"
#include "tc_common.cuh"
#include "gemm_v3.h"

namespace adas {

static constexpr int STEM_THREADS = 256;
static constexpr int STEM_WARPS = STEM_THREADS / 32;
// halves per staged pixel row (16-byte aligned, bank-shifted): 64 + 8 up to 64 channels, Cout + 8 for the 80 / 96-channel P6 stems
__host__ __device__ constexpr int stem_stg_ld(int nt) { return nt <= 8 ? 64 + 8 : nt * 8 + 8; }

__device__ __forceinline__ void mma_m16n8k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

struct StemParams {
    const __half* img;      // [B, Hp, Wp, 4] padded image
    const __half* wq;       // [Cout][k][KR] packed folded weights
    const float* bias;      // [Cout]
    __half* out;            // padded NHWC output (+ channel offset), row stride out_ld
    int B, Hp, Wp;          // padded input geometry (H + 2, W + 2)
    int Ho, Wo, out_ld;
    int k, pad, stride, KR, K;   // K = k * KR
    int w_ld;               // shared-memory row stride of the weights (halves)
    int act, tiles_per_row, total_tiles;
};

template <int NT>
__global__ void __launch_bounds__(STEM_THREADS) stem_conv_kernel(const StemParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr int STEM_STG_LD = stem_stg_ld(NT);
    const int w_ld = p.w_ld;                                          // halves
    __half* ws = reinterpret_cast<__half*>(smem);
    __half* stg_all = ws + (size_t)NT * 8 * w_ld;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    // folded weights -> shared memory (4-byte copies; K is a multiple of 16)
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(p.wq);
        const int k2 = p.K >> 1, w_ld2 = w_ld >> 1;
        for (int i = threadIdx.x; i < NT * 8 * k2; i += STEM_THREADS) {
            const int n = i / k2, kk = i - n * k2;
            reinterpret_cast<uint32_t*>(ws)[n * w_ld2 + kk] = src[i];
        }
    }
    __syncthreads();
    __half* stg = stg_all + warp * 16 * STEM_STG_LD;
    const int ksteps_row = p.KR >> 4;
    const uint2* img64 = reinterpret_cast<const uint2*>(p.img);         // one uint2 = one pixel (4 halves)
    for (int tile = blockIdx.x * STEM_WARPS + warp; tile < p.total_tiles; tile += gridDim.x * STEM_WARPS) {
        const int b = tile / (p.Ho * p.tiles_per_row);
        const int r = tile - b * (p.Ho * p.tiles_per_row);
        const int y = r / p.tiles_per_row, x0 = (r - y * p.tiles_per_row) * 16;
        float acc[NT][4];
#pragma unroll
        for (int j = 0; j < NT; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
        // padded input coordinates of tap (dy = 0, dx = 0) for output pixel (y, x): row s*y + 1 - pad, column s*x + 1 - pad
        const int col_g = p.stride * (x0 + g) + 1 - p.pad, col_g8 = col_g + 8 * p.stride;
        for (int dy = 0; dy < p.k; ++dy) {
            const int row = p.stride * y + 1 - p.pad + dy;
            const bool row_ok = row >= 0 && row < p.Hp;
            const size_t row_base = ((size_t)b * p.Hp + (row_ok ? row : 0)) * p.Wp;
            for (int ks = 0; ks < ksteps_row; ++ks) {
                // lane t of a pixel group holds pixel dx = ks*4 + t of this filter row: halves (dx*4 .. dx*4+3) = k-slots {2t, 2t+1, 2t+8, 2t+9}
                const int dx = ks * 4 + t;
                auto ld = [&](int col) -> uint2 {
                    return (row_ok && col >= 0 && col < p.Wp) ? __ldg(img64 + row_base + col) : make_uint2(0u, 0u);
                };
                const uint2 lo = ld(col_g + dx), hi = ld(col_g8 + dx);
                const uint32_t a[4] = {lo.x, hi.x, lo.y, hi.y};
                const __half* wrow = ws + (size_t)g * w_ld + dy * p.KR + ks * 16 + 4 * t;
#pragma unroll
                for (int j = 0; j < NT; ++j) {
                    const uint2 bw = *reinterpret_cast<const uint2*>(wrow + (size_t)j * 8 * w_ld);
                    mma_m16n8k16(acc[j], a, bw.x, bw.y);
                }
            }
        }
        // epilogue: c0,c1 -> pixel g, channels j*8 + 2t, +1 ; c2,c3 -> pixel g + 8
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const int n = j * 8 + 2 * t;
            const float b0 = p.bias ? p.bias[n] : 0.f, b1 = p.bias ? p.bias[n + 1] : 0.f;
            const __half2 lo = __floats2half2_rn(act_apply(acc[j][0] + b0, p.act), act_apply(acc[j][1] + b1, p.act));
            const __half2 hi = __floats2half2_rn(act_apply(acc[j][2] + b0, p.act), act_apply(acc[j][3] + b1, p.act));
            *reinterpret_cast<__half2*>(stg + g * STEM_STG_LD + n) = lo;
            *reinterpret_cast<__half2*>(stg + (g + 8) * STEM_STG_LD + n) = hi;
        }
        __syncwarp();
        const size_t out_row0 = ((size_t)b * (p.Ho + 2) + (y + 1)) * (p.Wo + 2) + (x0 + 1);
#pragma unroll
        for (int i = lane; i < 16 * NT; i += 32) {
            const int px = i / NT, v = i - px * NT;
            if (x0 + px < p.Wo) {
                const uint4 val = *reinterpret_cast<const uint4*>(stg + px * STEM_STG_LD + v * 8);
                *reinterpret_cast<uint4*>(p.out + (out_row0 + px) * p.out_ld + v * 8) = val;
            }
        }
        __syncwarp();
    }
}

int stem_conv_supported(int Cout, int k, int pad) {
    return (Cout == 16 || Cout == 24 || Cout == 32 || Cout == 48 || Cout == 64 || Cout == 80 || Cout == 96) && k >= 3 && k <= 7 && pad >= 0 && pad <= 3;
}

// The 80 / 96-channel stems (YOLOv7-E6 / E6E / D6, ReOrg + 3x3 folded into a 6x6 stride-2 conv) stage more than 48 KB: the kernel opts
// in on every launch (a host-side attribute, legal during graph capture).  k = 7 at 96 channels needs 77 KB.
static constexpr int STEM_WIDE_SMEM = 96 * 1024;

int launch_stem_conv(const __half* img, int B, int H, int W, const __half* wq, const float* bias, int Cout, int k, int pad, int stride, int act,
                     __half* out, int out_ld, int Ho, int Wo, cudaStream_t st) {
    ADAS_CHECK(stem_conv_supported(Cout, k, pad), "stem_conv: unsupported shape Cout=%d k=%d pad=%d", Cout, k, pad);
    ADAS_CHECK(stride == 1 || stride == 2, "stem_conv: stride %d (1 or 2)", stride);
    ADAS_CHECK(Ho == (H + 2 * pad - k) / stride + 1 && Wo == (W + 2 * pad - k) / stride + 1 && out_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
               "stem_conv: output geometry %dx%d (ld %d) does not match a %dx%d stride-%d conv of %dx%d", Ho, Wo, out_ld, k, k, stride, H, W);
    StemParams p;
    p.img = img; p.wq = wq; p.bias = bias; p.out = out;
    p.B = B; p.Hp = H + 2; p.Wp = W + 2; p.Ho = Ho; p.Wo = Wo; p.out_ld = out_ld;
    p.k = k; p.pad = pad; p.stride = stride; p.KR = (4 * k + 15) / 16 * 16; p.K = k * p.KR; p.act = act;
    p.tiles_per_row = (Wo + 15) / 16;
    p.total_tiles = B * Ho * p.tiles_per_row;
    // weight row stride = 16 (mod 64) halves: the 8-byte fragment loads of a half-warp (4 rows x 4 lanes) then cover all 32 banks once;
    // K + 8 (2-way conflicts) only where the conflict-free stride would not fit 48 KB
    // (the 80 / 96-channel stems opt in to more than 48 KB and keep the conflict-free stride)
    const int stg_bytes = STEM_WARPS * 16 * stem_stg_ld(Cout / 8) * 2;
    const int smem_cap = Cout > 64 ? STEM_WIDE_SMEM : 48 * 1024;
    p.w_ld = p.K + ((16 - p.K % 64) + 64) % 64;
    if (Cout * p.w_ld * 2 + stg_bytes > smem_cap) p.w_ld = p.K + 8;
    const int smem = Cout * p.w_ld * 2 + stg_bytes;
    ADAS_CHECK(smem <= smem_cap, "stem_conv: %d bytes of shared memory", smem);
    int blocks = (p.total_tiles + STEM_WARPS - 1) / STEM_WARPS;
    int n_sms = 132;
    if (v3_num_sms(&n_sms)) return 1;
    // resident blocks only (at most 3 per SM): the weight copy is per block, a warp walks ~20 tiles.  The 80 / 96-channel kernels hold
    // fewer blocks per SM (96 channels: 92 registers, 2 blocks), so their cap comes from the occupancy of the kernel as launched.
    int per_sm = 3;
    auto wide = [&](auto kernel) -> int {
        ADAS_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, STEM_WIDE_SMEM));
        int occ = 0;
        ADAS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, STEM_THREADS, smem));
        ADAS_CHECK(occ >= 1, "stem_conv: %d-channel kernel does not fit an SM (%d bytes of shared memory)", Cout, smem);
        if (occ < per_sm) per_sm = occ;
        return 0;
    };
    if (Cout == 80 && wide(stem_conv_kernel<10>)) return 1;
    if (Cout == 96 && wide(stem_conv_kernel<12>)) return 1;
    const int cap = n_sms * per_sm;
    if (blocks > cap) blocks = cap;
    switch (Cout / 8) {
        case 2: stem_conv_kernel<2><<<blocks, STEM_THREADS, smem, st>>>(p); break;
        case 3: stem_conv_kernel<3><<<blocks, STEM_THREADS, smem, st>>>(p); break;      // YOLOv6-Lite's 24-channel stem
        case 4: stem_conv_kernel<4><<<blocks, STEM_THREADS, smem, st>>>(p); break;
        case 6: stem_conv_kernel<6><<<blocks, STEM_THREADS, smem, st>>>(p); break;
        case 10: stem_conv_kernel<10><<<blocks, STEM_THREADS, smem, st>>>(p); break;
        case 12: stem_conv_kernel<12><<<blocks, STEM_THREADS, smem, st>>>(p); break;
        default: stem_conv_kernel<8><<<blocks, STEM_THREADS, smem, st>>>(p); break;
    }
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace adas
