// gemm_v3.cu -- the product GEMM / implicit-GEMM conv kernel: fused conv(+folded BN)+bias+SiLU/ReLU(+residual) and the FC layers as a
// persistent, warp-specialised Hopper kernel (wgmma, fp16 x fp16 -> fp32 in registers) with TMA-staged operands.
//
// Replaces: the opaque conv stacks ONNXRuntime/TensorRT execute behind coreEngine.py:150-157 (TensorRTEngine.engine_inference) /
// :184-186 (OnnxEngine.engine_inference).
//
// Tile: BM = 128 output rows (pixels of the padded NHWC grid) x MT sub-tiles x BN output channels x BK = 64 channels per k-block.
// A 3x3 stride-1 conv runs 9 taps x (Cin/64) k-blocks, each A tile being the SAME 2-D activation matrix read at row offset
// m0 + dy*(W+2) + dx (the zero halo of the padded layout supplies the conv padding, TMA's out-of-bounds zero fill covers the matrix
// ends).  The three dx taps of one (dy, k-block) differ only by a one-row shift, so in slab mode one pipeline stage holds one
// (dy, k-block): per sub-tile one TMA box of SLAB_ROWS = 136 rows, read by the dx taps from rows 0, 1 and 2 on, plus the three dx
// weight tiles -- a third of the activation bytes of one box per tap.  Slab mode needs two such stages in shared memory (not
// MT = 1 x BN = 256); autotune times every slab tile against the same tile with one activation box per tap.  Stride-2 convs read
// 4-D boxes with traversal stride 2.  K order is (dy, k-block, dx) for every tile shape and both operand modes, so results are
// bit-identical whatever tile is chosen and whatever the batch size.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one elected thread; the group gives its registers up with setmaxnreg),
// warpgroups 1 and 2 = consumers: each issues the wgmmas of 64 rows of every sub-tile (m64nBNk16, BN split into instructions of
// 128/64/32/16 columns) and runs the epilogue of those rows straight from its accumulator registers: +bias -> activation ->
// (+residual) -> fp16/fp32 stores of interior rows (the zero halo of padded outputs is never written).  Persistent: grid =
// min(tiles, SMs); the producer runs ahead into the next tile while the consumers finish the epilogue of the current one.
// The consumers' tile loop is compiled once per (sub-tile count, taps per stage) and picked once per CTA, so a stage's wgmmas
// are issued as one unbroken chain with compile-time operand offsets (v3_mainloop).
//
// Function attributes and the SM count are per device (a process may hold engines on several GPUs).
#include "common.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include "tc_common.cuh"
#include "gemm_v3.h"

namespace adas {

// UP2: the 2x2 transposed-conv store (GemmParams::up2).  A separate instantiation (BN 64 / 128 / 256 only): its address arithmetic in the
// unrolled epilogue costs the other instantiations spill slots, so they are compiled without it.
// HS: the Hardswish epilogue (act 5), a separate instantiation for the same reason: one more activation branch in the shared epilogue
// cost the BN 128 / 256 kernels 4 to 8 bytes of spill loads and YOLOv8-L ~3 % of its end-to-end rate on the H100.
template <bool HS>
__device__ __forceinline__ float v3_act(float x, int act) {
    if constexpr (HS) return hardswish(x);
    else return act_apply_base(x, act);
}

// Layout of one pipeline stage, as gemm_v3_config computes it: MT activation tiles (slab mode: SLAB_BYTES each, else
// A_STAGE_BYTES), then the weight tiles of its taps, each padded to 1024 bytes.
__host__ __device__ constexpr int v3_b_bytes(int BN) { return ((BN * BK * 2) + 1023) & ~1023; }
__host__ __device__ constexpr int v3_mt_max(int BN) { return V3_ACC_COLS / BN < 4 ? V3_ACC_COLS / BN : 4; }
__host__ __device__ constexpr int v3_slab_stage_bytes(int BN, int MT) { return MT * SLAB_BYTES + 3 * v3_b_bytes(BN); }
// slab mode needs two stages in shared memory
__host__ __device__ constexpr bool v3_slab_fits(int BN, int MT) { return 2 * v3_slab_stage_bytes(BN, MT) <= V3_DYN_SMEM_MAX - 1024; }

// Consumer mainloop of one tile: nsteps pipeline stages of TPS taps each (3 in slab mode, else 1).  A stage is one wgmma chain:
// one fence, then all TPS x MT x BK/16 x pieces(BN) wgmmas of this warpgroup's 64 rows back to back, then one commit, so the
// tensor pipe does not drain between taps or sub-tiles.  Nothing else touches the accumulators inside the loop: the wgmmas'
// "+f" operands order them, and reg_fence after the last wait keeps the epilogue's reads behind it.  Per sub-tile the K order is
// (dy, k-block, dx, k16) in both modes -- slab tap t reads the slab from row t on and its own weight tile -- so every tile shape
// and mode gives the same bits.
template <int BN, int MT, int TPS>
__device__ __forceinline__ void v3_mainloop(float (&acc)[MT][BN / 2], uint32_t smem_base, uint32_t a_row_off, int nsteps, int stages,
                                            uint32_t& s, uint32_t& ph, uint64_t* full_bar, uint64_t* empty_bar, int lane) {
    constexpr uint32_t A_SUB = TPS == 3 ? SLAB_BYTES : A_STAGE_BYTES;
    constexpr uint32_t B_BYTES = v3_b_bytes(BN);
    constexpr uint32_t STAGE = MT * A_SUB + TPS * B_BYTES;
    uint32_t prev = 0;
    for (int ks = 0; ks < nsteps; ++ks) {
        mbar_wait(smem_u32(&full_bar[s]), ph);
        const uint32_t st = smem_base + s * STAGE;
        const uint64_t adesc = make_smem_desc(st + a_row_off);
        const uint64_t bdesc = make_smem_desc(st + MT * A_SUB);
        const uint32_t scale = ks != 0;                     // the first k-step of a tile overwrites the accumulators
        wgmma_fence();
#pragma unroll
        for (int t = 0; t < TPS; ++t)
#pragma unroll
            for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                for (int k = 0; k < BK / 16; ++k)           // descriptors count 16-byte units
                    WgmmaCols<0, BN>::run(acc[mt], adesc + (mt * A_SUB + t * 128) / 16 + 2 * k, bdesc + t * B_BYTES / 16 + 2 * k,
                                          (t | k) != 0 ? 1u : scale);
        wgmma_commit();
        wgmma_wait<1>();                                    // the wgmmas of the previous step are done: its stage can be refilled
        if (ks > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
        prev = s;
        if (++s == (uint32_t)stages) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) reg_fence(acc[mt][i]);
    if (lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
}

// The tiles of one consumer warpgroup (rows cw*64 .. cw*64+63 of every sub-tile): mainloop, then the epilogue straight from the
// accumulator registers.
template <int BN, bool UP2, bool HS, int MT, int TPS>
__device__ __forceinline__ void v3_tiles(const GemmV3& g, uint32_t smem_base, uint64_t* full_bar, uint64_t* empty_bar, int warp_idx, int lane) {
    const GemmParams& p = g.p;
    const int cw = (warp_idx - 4) >> 2;                 // consumer warpgroup
    const int wq = warp_idx & 3;                        // warp of the group: 16 of those rows
    const int nsteps = p.ntaps * p.kpt / TPS;           // pipeline stages per tile
    const int per_img = p.s2_tw * p.s2_th;
    const size_t res_ld = (size_t)(p.res_ld < 0 ? -p.res_ld : p.res_ld);
    float acc[MT][BN / 2];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[mt][i] = 0.f;
    uint32_t s = 0, ph = 0;
    for (int w = blockIdx.x; w < g.total_tiles; w += gridDim.x) {
        v3_mainloop<BN, MT, TPS>(acc, smem_base, (uint32_t)cw * (64u * 128u), nsteps, g.stages, s, ph, full_bar, empty_bar, lane);

        // ---- epilogue: thread holds rows r0 and r0 + 8 of each sub-tile, columns 8j + 2(lane%4) + {0,1} ----
        const int n_t = w % g.n_tiles, m_t = w / g.n_tiles;
        const int n0 = n_t * BN;
        const int m0 = m_t * (BM * MT);
        const int c0 = 2 * (lane & 3);
        const float neg_slope = p.act == 3 ? 0.1f : 0.f;     // ReLU and LeakyReLU(0.1) share one instruction sequence
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = cw * 64 + wq * 16 + (lane >> 2) + 8 * h;      // row inside the sub-tile
                int row = m0 + mt * BM + r;
                bool ok = row < p.M;
                if (p.s2) {
                    const int pi = m_t * MT + mt;
                    const int b = fast_div(pi, g.fd_per_img);
                    const int rem = pi - b * per_img;
                    const int ty = fast_div(rem, g.fd_tw), tx = rem - ty * p.s2_tw;
                    const int j = fast_div(r, g.fd_bw), i = r - j * p.s2_bw;
                    const int yo = ty * p.s2_bh + j, xo = tx * p.s2_bw + i;
                    ok = (pi < g.n_patches) && (r < p.s2_bw * p.s2_bh) && (yo < p.s2_Ho) && (xo < p.s2_Wo);
                    row = (b * (p.s2_Ho + 2) + yo + 1) * (p.s2_Wo + 2) + xo + 1;
                } else if (p.mask_H > 0 && ok) {
                    const int Wp = p.mask_W + 2;
                    const int pp = row - fast_div(row, g.fd_img) * g.fd_img.d;
                    const int yy = fast_div(pp, g.fd_wp);
                    const int xx = pp - yy * Wp;
                    ok = (yy >= 1) && (yy <= p.mask_H) && (xx >= 1) && (xx <= p.mask_W);
                }
                if (!ok) continue;
                if (p.transposed) {
                    // swap-AB FC: rows are output features, columns are batch entries
                    const float row_bias = p.bias != nullptr ? __ldg(p.bias + row) : 0.f;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = n0 + 8 * j + c0 + e;
                            if (col < p.N) {
                                const float x = v3_act<HS>(acc[mt][4 * j + 2 * h + e] + row_bias, p.act);
                                if (p.out_f32) reinterpret_cast<float*>(p.out)[(size_t)col * (size_t)p.out_ld + row] = x;
                                else reinterpret_cast<__half*>(p.out)[(size_t)col * (size_t)p.out_ld + row] = __float2half_rn(x);
                            }
                        }
                    }
                    continue;
                }
                if constexpr (UP2) {
                    // 2x2 stride-2 transposed conv (no residual): column n = (2 dy + dx) * Cout + c of input pixel (yy, xx) goes to
                    // output pixel (2 yy - 1 + dy, 2 xx - 1 + dx) of the (2H+2) x (2W+2) grid.  Cout % 8 == 0, so an 8-column
                    // group lies in one (dy, dx).
                    const int bi = fast_div(row, g.fd_img);
                    const int pp = row - bi * g.fd_img.d;
                    const int yy = fast_div(pp, g.fd_wp), xx = pp - yy * (p.mask_W + 2);
                    const int Wo2 = 2 * p.mask_W + 2, co = p.N >> 2;
                    const int up_row = (bi * (2 * p.mask_H + 2) + 2 * yy - 1) * Wo2 + 2 * xx - 1;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j) {
                        const int n = n0 + 8 * j + c0;
                        if (n0 + 8 * j >= p.N) break;
                        float x0 = acc[mt][4 * j + 2 * h], x1 = acc[mt][4 * j + 2 * h + 1];
                        if (p.bias != nullptr) { x0 += __ldg(p.bias + n); x1 += __ldg(p.bias + n + 1); }
                        x0 = v3_act<HS>(x0, p.act); x1 = v3_act<HS>(x1, p.act);
                        const int q = (n >= co) + (n >= 2 * co) + (n >= 3 * co);
                        const size_t o = (size_t)(up_row + (q >> 1) * Wo2 + (q & 1)) * (size_t)p.out_ld + (n - q * co);
                        if (p.out_f32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + o) = make_float2(x0, x1);
                        else *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.out) + o) = __floats2half2_rn(x0, x1);
                    }
                    continue;
                }
                const __half* rp = p.res != nullptr ? p.res + (size_t)row * res_ld : nullptr;
                // Bias and residual loads go out RB column groups at a time, ahead of their stores.  The stores may alias them as far
                // as the compiler knows, so a load inside the store loop waits for the previous store and each one pays its full
                // L1 / L2 / HBM latency in turn.
                constexpr int RB = BN / 8 < 8 ? BN / 8 : 8;
#pragma unroll
                for (int j0 = 0; j0 < BN / 8; j0 += RB) {
                    if (n0 + 8 * j0 >= p.N) break;
                    __half2 rq[RB];
                    float2 bq[RB];
#pragma unroll
                    for (int jj = 0; jj < RB; ++jj) {
                        const int j = j0 + jj;
                        const bool in = j < BN / 8 && n0 + 8 * j < p.N;
                        rq[jj] = __float2half2_rn(0.f);
                        bq[jj] = make_float2(0.f, 0.f);
                        if (rp != nullptr && in) rq[jj] = *reinterpret_cast<const __half2*>(rp + n0 + 8 * j + c0);
                        if (p.bias != nullptr && in) bq[jj] = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + c0));
                    }
#pragma unroll
                    for (int jj = 0; jj < RB; ++jj) {
                        const int j = j0 + jj;
                        if (j >= BN / 8) break;
                        const int n = n0 + 8 * j + c0;
                        if (n0 + 8 * j >= p.N) break;                  // N % 8 == 0: an 8-column group is all in or all out
                        float x0 = acc[mt][4 * j + 2 * h], x1 = acc[mt][4 * j + 2 * h + 1];
                        if (p.bias != nullptr) { x0 += bq[jj].x; x1 += bq[jj].y; }
                        const float2 rv = __half22float2(rq[jj]);
                        if (p.res_ld < 0) { x0 += rv.x; x1 += rv.y; }
                        if constexpr (HS) { x0 = hardswish(x0); x1 = hardswish(x1); }
                        else if (p.act == 1) silu2(x0, x1);
                        else if (p.act >= 2) { x0 = relu_leaky(x0, neg_slope); x1 = relu_leaky(x1, neg_slope); }
                        if (p.res_ld > 0) { x0 += p.res_scale * rv.x; x1 += p.res_scale * rv.y; }   // scale 1: the bits of a plain add
                        if (p.out_f32) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + (size_t)row * (size_t)p.out_ld + n) = make_float2(x0, x1);
                        else *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.out) + (size_t)row * (size_t)p.out_ld + n) = __floats2half2_rn(x0, x1);
                    }
                }
            }
        }
    }
}

// Picks the consumers' tile loop once per CTA: one instantiation per sub-tile count that fits the accumulator registers, each
// with a slab-mode twin where two slab stages fit.
template <int BN, bool UP2, bool HS, int MT>
__device__ __forceinline__ void v3_consumers(const GemmV3& g, uint32_t smem_base, uint64_t* full_bar, uint64_t* empty_bar, int warp_idx, int lane) {
    if constexpr (MT < v3_mt_max(BN)) {
        if (g.MT != MT) { v3_consumers<BN, UP2, HS, MT + 1>(g, smem_base, full_bar, empty_bar, warp_idx, lane); return; }
    }
    if constexpr (!UP2 && v3_slab_fits(BN, MT)) {          // the transposed-conv store runs 1x1 GEMMs only
        if (g.slab) { v3_tiles<BN, UP2, HS, MT, 3>(g, smem_base, full_bar, empty_bar, warp_idx, lane); return; }
    }
    v3_tiles<BN, UP2, HS, MT, 1>(g, smem_base, full_bar, empty_bar, warp_idx, lane);
}

template <int BN, bool UP2, bool HS>
__global__ void __launch_bounds__(V3_THREADS, 1)
conv_gemm_v3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmV3 g) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[8];
    __shared__ __align__(8) uint64_t empty_bar[8];

    const GemmParams& p = g.p;
    const int warp_idx = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int stages = g.stages;
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int BMT = BM * g.MT;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
        for (int s = 0; s < stages; ++s) {
            mbar_init(smem_u32(&full_bar[s]), 1);
            mbar_init(smem_u32(&empty_bar[s]), 4 * V3_CONSUMERS);     // one arrive per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    // ---- TMA producer pieces (thread 0) ----
    const int tps = g.slab ? 3 : 1;                       // taps per pipeline stage
    const uint32_t a_bytes = p.s2 ? (uint32_t)(p.s2_bw * p.s2_bh * BK * 2) : (uint32_t)g.a_sub_bytes;
    const uint32_t tx_bytes = (uint32_t)g.MT * a_bytes + (uint32_t)(tps * BN * BK * 2);
    const bool dx_inner = p.ntaps == 9;                   // 9-tap order is (dy, k-block, dx)
    const int o_cnt = dx_inner ? 3 : p.ntaps;            // outer loop: dy (9 taps) or tap
    const int i_cnt = dx_inner && !g.slab ? 3 : 1;       // inner loop: dx (9 taps, one tap per stage)
    const int per_img = p.s2_tw * p.s2_th;
    // weight (B operand) tiles of one pipeline step: taps grp .. grp + tps - 1
    auto load_b = [&](int grp, int kc, int n0, uint32_t stage, uint32_t fb) {
        const uint32_t b_dst = smem_base + stage * g.stage_bytes + g.MT * g.a_sub_bytes;
        for (int t = 0; t < tps; ++t) tma_load_2d(b_dst + t * g.b_bytes, &tmB, (grp + t) * p.Kc + kc * BK, n0, fb);
    };
    // activation (A operand) tiles of one pipeline step
    auto load_a = [&](int grp, int kc, int m_t, uint32_t stage, uint32_t fb) {
        const uint32_t a_dst = smem_base + stage * g.stage_bytes;
        const int m0 = m_t * BMT;
        if (p.s2) {
            // stride-2 conv: sub-tile = bw x bh output pixels of image b; input pixel of tap (dy,dx) is (2*yo+dy, 2*xo+dx)
            // in padded coordinates, fetched by one 4-D TMA box with traversal stride 2 in x and y
            const int dy = p.ntaps == 9 ? grp / 3 : 1, dx = p.ntaps == 9 ? grp % 3 : 1;
            for (int mt = 0; mt < g.MT; ++mt) {
                const int pi = m_t * g.MT + mt;
                const int b = pi / per_img;
                const int rem = pi - b * per_img;
                const int ty = rem / p.s2_tw, tx = rem - ty * p.s2_tw;
                tma_load_4d(a_dst + mt * g.a_sub_bytes, &tmA, kc * BK, 2 * tx * p.s2_bw + dx, 2 * ty * p.s2_bh + dy, b, fb);
            }
        } else {
            // slab mode: grp = 3 * dy, so the slab starts at the dx = 0 tap's first row; its box is SLAB_ROWS tall
            int shift = 0;
            if (p.ntaps == 9) shift = (grp / 3 - 1) * p.Wp + (grp % 3 - 1);
            else if (p.ntaps == 4) shift = (grp - 2) * p.Wp;          // stem: row pairs yo-1 .. yo+2 (plan.py stem7x7s2)
            for (int mt = 0; mt < g.MT; ++mt) tma_load_2d(a_dst + mt * g.a_sub_bytes, &tmA, kc * BK, m0 + shift + mt * BM, fb);
        }
    };
    // Programmatic dependent launch: everything above overlapped the tail of the previous kernel in the stream; its results may
    // only be touched after `griddepcontrol.wait`.  The B operand holds the weights for a conv (A = activations): the producer arms
    // the first pipeline stages and fetches their B tiles BEFORE the wait, so only the A tiles see the dependency.  In swap-AB mode
    // (p.transposed) B is the activation, so gemm_v3_config turns the prefetch off there.
    int pre = 0;                                          // pipeline steps whose weight tiles were fetched ahead of the wait
    if (threadIdx.x == 0 && g.pdl && g.prefetch_w && (int)blockIdx.x < g.total_tiles) {
        const int steps_tile = o_cnt * p.kpt * i_cnt;
        pre = steps_tile < stages ? steps_tile : stages;
        const int n0 = ((int)blockIdx.x % g.n_tiles) * BN;
        for (int j = 0; j < pre; ++j) {
            const int in = j % i_cnt, kc = (j / i_cnt) % p.kpt, o = j / (i_cnt * p.kpt);
            const uint32_t fb = smem_u32(&full_bar[j]);
            mbar_expect_tx(fb, tx_bytes);
            load_b(dx_inner ? o * 3 + in : o, kc, n0, (uint32_t)j, fb);
        }
    }
    if (g.pdl) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }

    if (warp_idx < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (threadIdx.x == 0) {
            // ================= TMA producer =================
            uint32_t s = 0, ph = 0;
            int step = 0;                                        // steps issued by this CTA (only compared against `pre`)
            for (int w = blockIdx.x; w < g.total_tiles; w += gridDim.x) {
                const int n_t = w % g.n_tiles, m_t = w / g.n_tiles;
                const int n0 = n_t * BN;
                for (int o = 0; o < o_cnt; ++o) {
                    for (int kc = 0; kc < p.kpt; ++kc) {
                        for (int in = 0; in < i_cnt; ++in) {
                            const int grp = dx_inner ? o * 3 + in : o;
                            const uint32_t fb = smem_u32(&full_bar[s]);
                            if (step < pre) {
                                load_a(grp, kc, m_t, s, fb);     // stage already armed, weights already in flight
                            } else {
                                mbar_wait(smem_u32(&empty_bar[s]), ph ^ 1u);
                                mbar_expect_tx(fb, tx_bytes);
                                load_a(grp, kc, m_t, s, fb);
                                load_b(grp, kc, n0, s, fb);
                            }
                            ++step;
                            if (++s == (uint32_t)stages) { s = 0; ph ^= 1u; }
                        }
                    }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
        // ================= consumers (MMA + epilogue) =================
        v3_consumers<BN, UP2, HS, 1>(g, smem_base, full_bar, empty_bar, warp_idx, lane);
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------------
// BN is a template parameter (the accumulator array and the wgmma widths are static): every multiple of 16 up to 256.
#define V3_FOR_EACH_BN(X) X(16) X(32) X(48) X(64) X(80) X(96) X(112) X(128) X(144) X(160) X(176) X(192) X(208) X(224) X(240) X(256)

template <bool HS>
static const void* v3_kernel_act(int BN, bool up2) {
    if (up2) {
        switch (BN) {
            case 64: return reinterpret_cast<const void*>(&conv_gemm_v3_kernel<64, true, HS>);
            case 128: return reinterpret_cast<const void*>(&conv_gemm_v3_kernel<128, true, HS>);
            case 256: return reinterpret_cast<const void*>(&conv_gemm_v3_kernel<256, true, HS>);
            default: return nullptr;
        }
    }
    switch (BN) {
#define V3_CASE(b) case b: return reinterpret_cast<const void*>(&conv_gemm_v3_kernel<b, false, HS>);
        V3_FOR_EACH_BN(V3_CASE)
#undef V3_CASE
        default: return nullptr;
    }
}
static const void* v3_kernel(int BN, bool up2 = false, bool hswish = false) {
    return hswish ? v3_kernel_act<true>(BN, up2) : v3_kernel_act<false>(BN, up2);
}
static bool v3_up2_tile(int BN) { return BN == 64 || BN == 128 || BN == 256; }

struct V3Device { bool attr_set = false; int num_sms = 0; };
static std::mutex g_v3_mu;
static V3Device g_v3_dev[64];

static int v3_device_state(int* num_sms) {
    int dev = 0;
    ADAS_CUDA(cudaGetDevice(&dev));
    ADAS_CHECK(dev >= 0 && dev < 64, "device index %d out of range", dev);
    std::lock_guard<std::mutex> lk(g_v3_mu);
    V3Device& d = g_v3_dev[dev];
    if (!d.attr_set) {
        // function attributes are per device: set them once for every device an engine runs on
        for (int hs = 0; hs < 2; ++hs) {
            for (int bn = 16; bn <= 256; bn += 16) ADAS_CUDA(cudaFuncSetAttribute(v3_kernel(bn, false, hs), cudaFuncAttributeMaxDynamicSharedMemorySize, V3_DYN_SMEM_MAX));
            for (int bn = 64; bn <= 256; bn *= 2) ADAS_CUDA(cudaFuncSetAttribute(v3_kernel(bn, true, hs), cudaFuncAttributeMaxDynamicSharedMemorySize, V3_DYN_SMEM_MAX));
        }
        ADAS_CUDA(cudaDeviceGetAttribute(&d.num_sms, cudaDevAttrMultiProcessorCount, dev));
        d.attr_set = true;
    }
    *num_sms = d.num_sms;
    return 0;
}

static FastDiv make_fastdiv(int d) {
    FastDiv f;
    f.d = d < 1 ? 1 : d;
    f.mul = 0; f.shr = 0;
    if (f.d > 1) {
        int lg = 0;
        while ((1u << lg) < (uint32_t)f.d) ++lg;          // ceil(log2(d))
        const int p = 31 + lg;
        f.mul = (uint32_t)((((uint64_t)1 << p) + (uint64_t)f.d - 1) / (uint64_t)f.d);
        f.shr = (uint32_t)(p - 32);
    }
    return f;
}

int v3_num_sms(int* num_sms) { return v3_device_state(num_sms); }

static int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
}

int gemm_v3_config(const GemmParams& p_in, GemmV3* g) {
    GemmParams p = p_in;
    static const int force_bn = env_int("ADAS_B200_BN", 0), force_mt = env_int("ADAS_B200_MT", 0);
    if (force_bn >= 16 && force_bn <= 256 && force_bn % 16 == 0 && force_bn <= ((p.N + 15) / 16) * 16 && !p.transposed && !p.up2) p.BN = force_bn;   // test hook
    if (p.BN % 16 != 0 || p.BN < 16 || p.BN > 256) return 1;
    if (p.up2 && !v3_up2_tile(p.BN)) return 1;                 // the transposed-conv store is compiled for BN 64 / 128 / 256
    g->p = p;
    g->MT = p.mt_hint >= 1 ? p.mt_hint : ((p.BN <= 128) ? 2 : 1);
    if (force_mt >= 1 && force_mt <= 4) g->MT = force_mt;     // test hook: exercise every sub-tile count
    if (g->MT > 4) return 1;
    // the accumulators of a CTA tile live in registers (MT * BN / 2 per consumer thread): a taller tile than fits runs as the
    // tallest one that does -- results do not depend on the tile shape
    if (g->MT > v3_mt_max(p.BN)) g->MT = v3_mt_max(p.BN);
    const int b_bytes = v3_b_bytes(p.BN);
    g->b_bytes = b_bytes;
    // 3x3 stride-1: the three dx taps of one (dy, k-block) read the same activation rows shifted by one, so one slab of
    // SLAB_ROWS rows per sub-tile feeds all three -- when two such stages fit (not at MT = 1, BN = 256)
    static const int no_slab_env = env_int("ADAS_B200_NOSLAB", 0);
    const int slab_stage = v3_slab_stage_bytes(p.BN, g->MT);
    g->slab = p.ntaps == 9 && !p.s2 && !p.up2 && !p.no_slab && !no_slab_env && v3_slab_fits(p.BN, g->MT);
    g->a_sub_bytes = g->slab ? SLAB_BYTES : A_STAGE_BYTES;
    g->stage_bytes = g->slab ? slab_stage : g->MT * g->a_sub_bytes + b_bytes;
    int stages = (V3_DYN_SMEM_MAX - 1024) / g->stage_bytes;
    if (stages > 8) stages = 8;
    if (stages < 2) return 1;
    g->stages = stages;
    g->p.stages = stages;
    const int BMT = BM * g->MT;
    g->n_tiles = (p.N + p.BN - 1) / p.BN;
    g->m_tiles = (p.M + BMT - 1) / BMT;
    g->total_tiles = g->n_tiles * g->m_tiles;
    g->n_patches = p.s2 ? p.M / BM : 0;
    g->fd_img = make_fastdiv((p.mask_H + 2) * (p.mask_W + 2));
    g->fd_wp = make_fastdiv(p.mask_W + 2);
    g->fd_per_img = make_fastdiv(p.s2 ? p.s2_tw * p.s2_th : 1);
    g->fd_tw = make_fastdiv(p.s2 ? p.s2_tw : 1);
    g->fd_bw = make_fastdiv(p.s2 ? p.s2_bw : 1);
    g->pdl = 0;
    static const int no_prefetch = env_int("ADAS_B200_NO_WPREFETCH", 0);
    g->prefetch_w = (no_prefetch || p.transposed) ? 0 : 1;     // swap-AB: B is the previous kernel's output, not the weights
    return 0;
}

static int v3_smem_bytes(const GemmV3& g) { return g.stages * g.stage_bytes + 1024; }

int gemm_v3_launch(const GemmV3Launch& L, cudaStream_t st) {
    int num_sms = 0;
    if (v3_device_state(&num_sms)) return 1;
    static const int pdl = env_int("ADAS_B200_PDL", 1);
    GemmV3 gp = L.g;
    gp.pdl = pdl ? 1 : 0;
    const void* fn = v3_kernel(gp.p.BN, gp.p.up2 != 0, gp.p.act == 5);
    ADAS_CHECK(fn != nullptr, "gemm_v3: no kernel for BN %d%s", gp.p.BN, gp.p.up2 ? " with the transposed-conv store" : "");
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(gp.total_tiles < num_sms ? gp.total_tiles : num_sms, 1, 1);
    cfg.blockDim = dim3(V3_THREADS, 1, 1);
    cfg.dynamicSmemBytes = v3_smem_bytes(gp);
    cfg.stream = st;
    cudaLaunchAttribute attr1;
    attr1.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr1.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr1;
    cfg.numAttrs = pdl ? 1 : 0;
    CUtensorMap tmA = L.tmA, tmB = L.tmB;
    void* args[] = {&tmA, &tmB, &gp};
    ADAS_CUDA(cudaLaunchKernelExC(&cfg, fn, args));
    count_launch();
    return 0;
}

// Tile candidates ranked by a rough cost model (the engine times the best few on the device once per (op, batch)): operand bytes
// delivered from L2 at ~32 B/clk/SM, wgmma time, an epilogue that does not overlap the main loop of the same CTA, waves of tiles
// over the SMs and a fixed launch cost.  A tile that can run in slab mode is handed out twice, slab first and then per tap
// (no_slab_out = 1): two slab stages hold only one stage of look-ahead, which measures slower than per-tap loads on some H100
// layers (80x80 N = 128, 40x40 N = 256), so the device timing decides.
int gemm_v3_candidates(const GemmParams& base, int max_out, int* BN_out, int* mt_out, int* no_slab_out) {
    int num_sms = 132;
    if (v3_num_sms(&num_sms)) return 0;
    const int cand[] = {256, 192, 128, 64, 160, 96, 80, 48, 32, 16};
    struct C { double t; int BN, mt, slab; } list[64];
    int n = 0;
    const int N = base.N, ntaps = base.ntaps;
    const int kpt = (base.Kc + 63) / 64;
    for (int ci = 0; ci < 10; ++ci) {
        int BN = cand[ci];
        if (BN > N) { if (BN - N >= 64 || (BN % 64 == 0 && BN - N >= 16 && N > 64)) continue; BN = (N + 15) / 16 * 16; }
        if (BN > 256) continue;
        if (BN < 64 && N >= 64) continue;                        // narrow tiles only ever win on narrow layers
        if (base.up2 && !v3_up2_tile(BN)) continue;
        const int n_tiles = (N + BN - 1) / BN;
        if ((double)n_tiles * BN > 1.35 * N) continue;           // too much padded-N work
        bool dup = false;
        for (int k = 0; k < n; ++k) dup = dup || (list[k].BN == BN);
        if (dup) continue;
        for (int mt = 1; mt <= 4; ++mt) {
            GemmParams p = base;
            p.BN = BN; p.mt_hint = mt;
            GemmV3 g;
            if (gemm_v3_config(p, &g)) continue;
            if (g.p.BN != BN || g.MT != mt) continue;            // clamped, or forced by a test hook
            const double tiles = (double)g.total_tiles;
            const int tps = g.slab ? 3 : 1;                      // taps per pipeline stage
            const double bytes = (double)ntaps * kpt / tps * (g.MT * (double)g.a_sub_bytes + tps * BN * 128.0);
            const double rate = BN >= 64 ? 1.0 : 0.7;                              // narrow wgmmas are bound by the A re-read
            const double mma = (double)g.MT * ntaps * kpt * 4.0 * BN / rate;
            const double epi = (double)g.MT * 128.0 * BN * 0.12;
            const double per_tile = fmax(bytes / 32.0, mma) + epi + 400.0;
            const double waves = ceil(tiles / (double)num_sms);
            const double t = waves * per_tile + 3500.0;
            if (n < 64) { list[n].t = t; list[n].BN = BN; list[n].mt = mt; list[n].slab = g.slab; ++n; }
        }
    }
    for (int i = 1; i < n; ++i) { C c = list[i]; int j = i - 1; while (j >= 0 && list[j].t > c.t) { list[j + 1] = list[j]; --j; } list[j + 1] = c; }
    if (n == 0) { list[0].BN = N <= 256 ? (N + 15) / 16 * 16 : 256; list[0].mt = 1; list[0].slab = 0; n = 1; }
    if (base.up2 && !v3_up2_tile(list[0].BN)) list[0].BN = N >= 256 ? 256 : N >= 128 ? 128 : 64;
    int out = 0;
    for (int i = 0; i < n && out < max_out; ++i) {
        for (int ns = 0; ns <= list[i].slab && out < max_out; ++ns) {
            BN_out[out] = list[i].BN; mt_out[out] = list[i].mt; no_slab_out[out] = ns; ++out;
        }
    }
    return out;
}

int gemm_v3_prepare(const GemmParams& p, const void* a_base, uint64_t a_inner, uint64_t a_rows, uint64_t a_stride_bytes,
                    const void* b_base, uint64_t b_inner, uint64_t b_rows, uint64_t b_stride_bytes, void** opaque) {
    ADAS_CHECK(p.BN % 16 == 0 && p.BN >= 16 && p.BN <= 256, "gemm_v3: bad BN %d", p.BN);
    ADAS_CHECK(p.N % 8 == 0 || p.transposed, "gemm_v3: N %d must be a multiple of 8", p.N);
    ADAS_CHECK(!p.s2, "gemm_v3_prepare: stride-2 ops go through gemm_v3_prepare_s2");
    GemmV3Launch* L = new GemmV3Launch();
    if (gemm_v3_config(p, &L->g)) { delete L; ADAS_CHECK(false, "gemm_v3: tile does not fit (BN %d, mt %d)", p.BN, p.mt_hint); }
    if (make_tmap_2d(&L->tmA, a_base, a_inner, a_rows, a_stride_bytes, 64, L->g.slab ? SLAB_ROWS : BM) ||
        make_tmap_2d(&L->tmB, b_base, b_inner, b_rows, b_stride_bytes, 64, (uint32_t)L->g.p.BN)) {
        delete L;
        return 1;
    }
    *opaque = L;
    return 0;
}

int gemm_v3_prepare_s2(const GemmParams& p, const void* a_base, uint64_t a_C, uint64_t a_Wp, uint64_t a_Hp, uint64_t a_B, uint64_t a_ld,
                       const void* b_base, uint64_t b_inner, uint64_t b_rows, uint64_t b_stride_bytes, void** opaque) {
    ADAS_CHECK(p.s2 && p.BN % 16 == 0 && p.BN >= 16 && p.BN <= 256 && p.N % 8 == 0, "gemm_v3_s2: bad tile (BN %d)", p.BN);
    GemmV3Launch* L = new GemmV3Launch();
    if (gemm_v3_config(p, &L->g)) { delete L; ADAS_CHECK(false, "gemm_v3_s2: tile does not fit (BN %d, mt %d)", p.BN, p.mt_hint); }
    if (make_tmap_4d_s2(&L->tmA, a_base, a_C, a_Wp, a_Hp, a_B, a_ld, 2u * (uint32_t)p.s2_bw, 2u * (uint32_t)p.s2_bh) ||
        make_tmap_2d(&L->tmB, b_base, b_inner, b_rows, b_stride_bytes, 64, (uint32_t)L->g.p.BN)) {
        delete L;
        return 1;
    }
    *opaque = L;
    return 0;
}

int gemm_v3_run(void* opaque, cudaStream_t st) { return gemm_v3_launch(*static_cast<GemmV3Launch*>(opaque), st); }
void gemm_v3_free(void* opaque) { delete static_cast<GemmV3Launch*>(opaque); }
void gemm_v3_describe(const void* opaque, char* out, int cap) {
    const GemmV3& g = static_cast<const GemmV3Launch*>(opaque)->g;
    snprintf(out, (size_t)cap, "M=%d N=%d K=%d taps=%d act=%d res=%d f32=%d s2=%d tr=%d up2=%d | v3 BN=%d MT=%d slab=%d stages=%d tiles=%d wpre=%d", g.p.M,
             g.p.N, g.p.Kc * g.p.ntaps, g.p.ntaps, g.p.act, g.p.res ? (g.p.res_ld < 0 ? -1 : 1) : 0, g.p.out_f32, g.p.s2, g.p.transposed, g.p.up2,
             g.p.BN, g.MT, g.slab, g.stages, g.total_tiles, g.prefetch_w);
}

}  // namespace adas
