// tc_common.cuh -- device helpers of the Hopper GEMM kernel (mbarrier, TMA, wgmma descriptors and instructions, epilogue math).
#pragma once
#include "common.h"

namespace adas {

static constexpr int BM = 128;
static constexpr int BK = 64;                       // fp16 elements per k-block = 128 bytes = one swizzle row
static constexpr int A_STAGE_BYTES = BM * BK * 2;   // 16 KiB
static constexpr int SLAB_ROWS = BM + 8;            // 3x3 stride-1 slab: BM rows + the 2 rows the dx = 1, 2 taps reach, to 8-row groups
static constexpr int SLAB_BYTES = SLAB_ROWS * BK * 2;   // 17 KiB: consecutive slabs stay 1024-byte aligned

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t smem_dst, const CUtensorMap* tm, int c0, int c1, int c2, int c3, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
        ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
        : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA, fp16 x fp16 -> fp32 in registers) ------------------------------------------------------
// Shared-memory matrix descriptor of a K-major, 128B-swizzled operand tile as TMA writes it: rows of 128 bytes, 8-row groups
// 1024 bytes apart; a k-step of 16 elements advances the start by 32 bytes.  The start may also lie whole rows into a swizzle atom
// (slab mode: dx = 1, 2 rows into a 1024-byte aligned box) with the base-offset field (bits 49-51) left at 0: the swizzle XOR follows
// the absolute shared-memory address, as TMA's does.  Setting it to (addr >> 7) & 7 is not needed; with 0 the slab path is bit-identical
// to one aligned box per tap (tests/test_gpu_slab.py).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);   // start address, 16-byte units
    d |= (uint64_t)1 << 16;                         // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;               // stride byte offset: 8 rows * 128 B
    d |= (uint64_t)1 << 62;                         // layout: SWIZZLE_128B
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across a wgmma.wait_group
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory; acc = 0 overwrites D.
template <int N>
__device__ __forceinline__ void wgmma_n(float* d, uint64_t ad, uint64_t bd, uint32_t acc);
template <> __device__ __forceinline__ void wgmma_n<16>(float* d, uint64_t ad, uint64_t bd, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(ad), "l"(bd), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_n<32>(float* d, uint64_t ad, uint64_t bd, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(ad), "l"(bd), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_n<64>(float* d, uint64_t ad, uint64_t bd, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(ad), "l"(bd), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_n<128>(float* d, uint64_t ad, uint64_t bd, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(ad), "l"(bd), "r"(acc));
}

// A tile of width BN issued as instructions of 128 / 64 / 32 / 16 columns (each reads the A operand once more; at N >= 32 per
// instruction the tensor cores, not shared-memory bandwidth, bound the rate).  OFF = first column of this piece.
template <int OFF, int REM>
struct WgmmaCols {
    static __device__ __forceinline__ void run(float* d, uint64_t ad, uint64_t bd, uint32_t acc) {
        constexpr int W = REM >= 128 ? 128 : REM >= 64 ? 64 : REM >= 32 ? 32 : 16;
        wgmma_n<W>(d + OFF / 2, ad, bd + (uint64_t)(OFF * 128 / 16), acc);   // B rows OFF.. start OFF * 128 bytes further
        WgmmaCols<OFF + W, REM - W>::run(d, ad, bd, acc);
    }
};
template <int OFF>
struct WgmmaCols<OFF, 0> {
    static __device__ __forceinline__ void run(float*, uint64_t, uint64_t, uint32_t) {}
};

// max(x, x * s) for 0 <= s < 1: ReLU at s = 0, torch.nn.LeakyReLU(s) otherwise (x if x >= 0 else x * s), in the same three
// instructions, so the unrolled GEMM epilogues carry one code path for both.  The + 0 turns the -0 that ReLU would give for x < 0
// (x * 0 = -0) into +0, the bits fmaxf(x, 0) gives.
__device__ __forceinline__ float relu_leaky(float x, float s) { return fmaxf(x, x * s) + 0.0f; }

// Hardswish (torch.nn.Hardswish): x * clamp(x + 3, 0, 6) / 6 in fp32, the division as a product with fp32(1/6) (within one fp32 ulp of
// the quotient; a true IEEE division inlines a slow-path subroutine).
__device__ __forceinline__ float hardswish(float x) { return x * fminf(fmaxf(x + 3.0f, 0.0f), 6.0f) * (1.0f / 6.0f); }

// Activation codes 0 none, 1 SiLU, 2 ReLU, 3 LeakyReLU(0.1); the GEMM kernel's instantiations without Hardswish use this alone.
__device__ __forceinline__ float act_apply_base(float x, int act) {
    if (act == 1) return __fdividef(x, 1.0f + __expf(-x));   // SiLU
    if (act >= 2) return relu_leaky(x, act == 3 ? 0.1f : 0.0f);   // ReLU, LeakyReLU(0.1)
    return x;
}

// Activation codes of plan.h: 0 none, 1 SiLU, 2 ReLU, 3 LeakyReLU(0.1), 5 Hardswish (4 is unused).
__device__ __forceinline__ float act_apply(float x, int act) { return act == 5 ? hardswish(x) : act_apply_base(x, act); }

__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// SiLU of two values with one reciprocal: 1/(1+t0) = (1+t1) / ((1+t0)(1+t1)).  Per element 1.5 SFU ops (ex2 + half a rcp) instead
// of 2.  Arguments are clamped at -40 so the product of two (1 + e^40) stays inside fp32 (SiLU(-40) = -1.7e-16 rounds to -0 in half
// precision either way).
__device__ __forceinline__ void silu2(float& x0, float& x1) {
    const float L = -1.4426950408889634f;
    const float a0 = 1.0f + ex2_approx(fmaxf(x0, -40.f) * L);
    const float a1 = 1.0f + ex2_approx(fmaxf(x1, -40.f) * L);
    const float r = rcp_approx(a0 * a1);
    x0 *= r * a1;
    x1 *= r * a0;
}

// n / d for 0 <= n < 2^31 without a hardware divide (the epilogue's row arithmetic).
struct FastDiv {
    uint32_t mul, shr;
    int d;
};
__device__ __forceinline__ int fast_div(int n, const FastDiv& f) { return f.d == 1 ? n : (int)(__umulhi((uint32_t)n, f.mul) >> f.shr); }
}  // namespace adas
