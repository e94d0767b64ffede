// attention.cu -- multi-head self-attention over the pixels of a padded-NHWC map (YOLOv10 PSA, OP_ATTN).
//
// Input: the qkv conv's output slice, laid out by the packer as [Q all heads | K all heads | V all heads]; each head's q / k hold
// kdp = round_up(kd, 16) channels (zero weight and bias past kd, which change no dot product), each head's v holds hd channels in
// upstream's head-major order.  Output: nh * hd channels, channel h * hd + d = sum_m softmax_m(q_n . k_m * scale) v_m[d] -- the order of
// upstream's (v @ attn^T).view(B, C, H, W).
//
// One CTA = (image, head, 64 queries); 4 warps of 16 queries.  Q fragments stay in registers; K and V tiles of 64 keys stream through
// shared memory.  Q K^T and P V are mma.sync m16n8k16 (fp16 in, fp32 accumulate) with an fp32 online softmax in base 2.  Keys past N are
// zero-filled and masked to -inf; queries past N are computed and not stored.  Keys are never split across CTAs, so every query's sum
// runs in one fixed order: frame i of a batch equals the batch-1 result bit for bit.
#include "common.h"

namespace adas {

namespace {

constexpr int AT_THREADS = 128;
constexpr int AT_Q = 64;                 // queries per CTA (4 warps x 16)
constexpr int AT_KT = 64;                // keys per shared-memory tile
constexpr int AT_MAX_KS = 4;             // kdp <= 64 (upstream: kd = hd / 2 < 64)
constexpr int AT_MAX_DT = 16;            // hd <= 128

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

__device__ __forceinline__ uint32_t pack_h2(__half lo, __half hi) {
    const __half2 h = __halves2half2(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

struct AttnParams {
    const __half* qkv; int in_ld;        // slice start of the packed qkv channels, row stride
    __half* out; int out_ld;             // slice start of the output, row stride
    int H, W, N, nh, kdp, hd, qtiles;
    float scale_log2;                    // scale * log2(e)
};

__global__ void __launch_bounds__(AT_THREADS) attn_kernel(const AttnParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int kld = p.kdp + 8, vld = p.hd + 8;                       // +8 halves: rows shift by 4 banks
    __half* Ks = reinterpret_cast<__half*>(smem);                    // [AT_KT][kld]
    __half* Vs = Ks + AT_KT * kld;                                   // [AT_KT][vld]
    int blk = blockIdx.x;
    const int qt = blk % p.qtiles; blk /= p.qtiles;
    const int h = blk % p.nh, b = blk / p.nh;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int Wp = p.W + 2;
    auto row_of = [&](int n) -> size_t {
        const int y = n / p.W, x = n - y * p.W;
        return ((size_t)b * (p.H + 2) + y + 1) * Wp + x + 1;
    };
    const __half* Qg = p.qkv + h * p.kdp;
    const __half* Kg = p.qkv + (p.nh + h) * p.kdp;
    const __half* Vg = p.qkv + 2 * p.nh * p.kdp + h * p.hd;
    const int nks = p.kdp >> 4, ndt = p.hd >> 3;

    const int r0 = qt * AT_Q + warp * 16 + g, r1 = r0 + 8;
    const bool ok0 = r0 < p.N, ok1 = r1 < p.N;
    uint32_t qa[AT_MAX_KS][4];
    {
        const __half* q0 = Qg + row_of(ok0 ? r0 : 0) * p.in_ld + 2 * t;
        const __half* q1 = Qg + row_of(ok1 ? r1 : 0) * p.in_ld + 2 * t;
#pragma unroll
        for (int ks = 0; ks < AT_MAX_KS; ++ks) {
            if (ks < nks) {
                qa[ks][0] = ok0 ? *reinterpret_cast<const uint32_t*>(q0 + ks * 16) : 0u;
                qa[ks][1] = ok1 ? *reinterpret_cast<const uint32_t*>(q1 + ks * 16) : 0u;
                qa[ks][2] = ok0 ? *reinterpret_cast<const uint32_t*>(q0 + ks * 16 + 8) : 0u;
                qa[ks][3] = ok1 ? *reinterpret_cast<const uint32_t*>(q1 + ks * 16 + 8) : 0u;
            }
        }
    }
    float o[AT_MAX_DT][4];
#pragma unroll
    for (int j = 0; j < AT_MAX_DT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;     // running max (base-2 logits) and this thread's partial row sums

    for (int k0 = 0; k0 < p.N; k0 += AT_KT) {
        __syncthreads();                                              // the previous tile is no longer read
        const int kv8 = p.kdp >> 3, vv8 = p.hd >> 3;
        for (int i = threadIdx.x; i < AT_KT * kv8; i += AT_THREADS) {
            const int r = i / kv8, c = i - r * kv8, key = k0 + r;
            const uint4 v = key < p.N ? __ldg(reinterpret_cast<const uint4*>(Kg + row_of(key) * p.in_ld + c * 8)) : make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(Ks + r * kld + c * 8) = v;
        }
        for (int i = threadIdx.x; i < AT_KT * vv8; i += AT_THREADS) {
            const int r = i / vv8, c = i - r * vv8, key = k0 + r;
            const uint4 v = key < p.N ? __ldg(reinterpret_cast<const uint4*>(Vg + row_of(key) * p.in_ld + c * 8)) : make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(Vs + r * vld + c * 8) = v;
        }
        __syncthreads();
        // S = Q K^T for 8 n-tiles of 8 keys
        float s[AT_KT / 8][4];
#pragma unroll
        for (int j = 0; j < AT_KT / 8; ++j) {
            s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
            const __half* kr = Ks + (j * 8 + g) * kld + 2 * t;
#pragma unroll
            for (int ks = 0; ks < AT_MAX_KS; ++ks) {
                if (ks < nks) {
                    const uint32_t b0 = *reinterpret_cast<const uint32_t*>(kr + ks * 16);
                    const uint32_t b1 = *reinterpret_cast<const uint32_t*>(kr + ks * 16 + 8);
                    mma16816(s[j], qa[ks], b0, b1);
                }
            }
        }
        // online softmax: thread holds rows g (c0, c1) and g + 8 (c2, c3), keys j*8 + 2t, +1
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < AT_KT / 8; ++j) {
            const int key = k0 + j * 8 + 2 * t;
            const bool v0 = key < p.N, v1 = key + 1 < p.N;
            s[j][0] = v0 ? s[j][0] * p.scale_log2 : -INFINITY;
            s[j][1] = v1 ? s[j][1] * p.scale_log2 : -INFINITY;
            s[j][2] = v0 ? s[j][2] * p.scale_log2 : -INFINITY;
            s[j][3] = v1 ? s[j][3] * p.scale_log2 : -INFINITY;
            mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
            mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
        }
#pragma unroll
        for (int d = 1; d <= 2; d <<= 1) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, d));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, d));
        }
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);      // finite: key k0 < N is valid
        const float al0 = exp2f(m0 - mn0), al1 = exp2f(m1 - mn1);    // 0 on the first tile
        m0 = mn0; m1 = mn1;
        float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
        for (int j = 0; j < AT_KT / 8; ++j) {
            s[j][0] = exp2f(s[j][0] - mn0); s[j][1] = exp2f(s[j][1] - mn0);
            s[j][2] = exp2f(s[j][2] - mn1); s[j][3] = exp2f(s[j][3] - mn1);
            sum0 += s[j][0] + s[j][1];
            sum1 += s[j][2] + s[j][3];
        }
        l0 = l0 * al0 + sum0;
        l1 = l1 * al1 + sum1;
#pragma unroll
        for (int j = 0; j < AT_MAX_DT; ++j) { o[j][0] *= al0; o[j][1] *= al0; o[j][2] *= al1; o[j][3] *= al1; }
        // O += P V: the S accumulators of n-tiles 2kk, 2kk+1 are the A fragment of key step kk
#pragma unroll
        for (int kk = 0; kk < AT_KT / 16; ++kk) {
            const uint32_t a[4] = {pack_h2(s[2 * kk][0], s[2 * kk][1]), pack_h2(s[2 * kk][2], s[2 * kk][3]),
                                   pack_h2(s[2 * kk + 1][0], s[2 * kk + 1][1]), pack_h2(s[2 * kk + 1][2], s[2 * kk + 1][3])};
            const __half* vr = Vs + (kk * 16 + 2 * t) * vld + g;
#pragma unroll
            for (int j = 0; j < AT_MAX_DT; ++j) {
                if (j < ndt) {
                    const __half* v = vr + j * 8;
                    const uint32_t b0 = pack_h2(v[0], v[vld]);
                    const uint32_t b1 = pack_h2(v[8 * vld], v[9 * vld]);
                    mma16816(o[j], a, b0, b1);
                }
            }
        }
    }
#pragma unroll
    for (int d = 1; d <= 2; d <<= 1) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, d);
        l1 += __shfl_xor_sync(0xffffffffu, l1, d);
    }
    const float i0 = 1.f / l0, i1 = 1.f / l1;
    __half* o0 = p.out + row_of(ok0 ? r0 : 0) * p.out_ld + h * p.hd + 2 * t;
    __half* o1 = p.out + row_of(ok1 ? r1 : 0) * p.out_ld + h * p.hd + 2 * t;
#pragma unroll
    for (int j = 0; j < AT_MAX_DT; ++j) {
        if (j < ndt) {
            if (ok0) *reinterpret_cast<__half2*>(o0 + j * 8) = __floats2half2_rn(o[j][0] * i0, o[j][1] * i0);
            if (ok1) *reinterpret_cast<__half2*>(o1 + j * 8) = __floats2half2_rn(o[j][2] * i1, o[j][3] * i1);
        }
    }
}

}  // namespace

int attention_supported(int nh, int kdp, int hd) {
    return nh >= 1 && kdp >= 16 && kdp <= 16 * AT_MAX_KS && kdp % 16 == 0 && hd >= 8 && hd <= 8 * AT_MAX_DT && hd % 8 == 0;
}

int launch_attention(const __half* qkv, int in_ld, int B, int H, int W, int nh, int kdp, int hd, float scale, __half* out, int out_ld,
                     cudaStream_t st) {
    ADAS_CHECK(attention_supported(nh, kdp, hd) && in_ld % 8 == 0 && out_ld % 8 == 0, "attention: nh %d kdp %d hd %d", nh, kdp, hd);
    AttnParams p;
    p.qkv = qkv; p.in_ld = in_ld; p.out = out; p.out_ld = out_ld;
    p.H = H; p.W = W; p.N = H * W; p.nh = nh; p.kdp = kdp; p.hd = hd;
    p.qtiles = (p.N + AT_Q - 1) / AT_Q;
    p.scale_log2 = scale * 1.4426950408889634f;
    const int smem = AT_KT * ((kdp + 8) + (hd + 8)) * 2;
    const long long blocks = (long long)B * nh * p.qtiles;
    ADAS_CHECK(blocks <= 0x7fffffff, "attention: %lld CTAs", blocks);
    attn_kernel<<<(int)blocks, AT_THREADS, smem, st>>>(p);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace adas
