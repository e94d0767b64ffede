// tensor_map.cu -- TMA descriptors for the conv / FC GEMM kernel (gemm_v3.cu) and the CUDA-core validation kernel the
// tests compare the wgmma path against (conv_impl = 1; never the product path).
//
// Tensor maps: 2-D [rows, channels] views of padded-NHWC activations and of weight matrices (128-byte swizzle, out-of-bounds rows read
// as zero) and 4-D [C, W, H, B] views with traversal stride 2 for stride-2 convs.
#include "common.h"
#include "tc_common.cuh"
#include <stdlib.h>
#include <string.h>

namespace adas {

// ---- TMA descriptor (driver entry point fetched through the runtime; no libcuda link) ----------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
    return fn;
}

int make_tmap_2d(CUtensorMap* tm, const void* base, uint64_t inner, uint64_t rows, uint64_t row_stride_bytes,
                 uint32_t box_inner, uint32_t box_rows) {
    PFN_encodeTiled fn = get_encode_fn();
    ADAS_CHECK(fn != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
    ADAS_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base %p not 16-byte aligned", base);
    ADAS_CHECK((row_stride_bytes & 15) == 0, "TMA row stride %llu not a multiple of 16", (unsigned long long)row_stride_bytes);
    cuuint64_t dims[2] = {inner, rows};
    cuuint64_t strides[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_inner, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    ADAS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed: %d (inner=%llu rows=%llu stride=%llu box=%u,%u)", (int)r,
               (unsigned long long)inner, (unsigned long long)rows, (unsigned long long)row_stride_bytes, box_inner, box_rows);
    return 0;
}

int make_tmap_4d_s2(CUtensorMap* tm, const void* base, uint64_t C, uint64_t Wp, uint64_t Hp, uint64_t B, uint64_t ld_elems,
                    uint32_t box_w_src, uint32_t box_h_src) {
    PFN_encodeTiled fn = get_encode_fn();
    ADAS_CHECK(fn != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
    ADAS_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld_elems * 2) % 16 == 0, "TMA 4-D map alignment");
    ADAS_CHECK(box_w_src <= 256 && box_h_src <= 256, "TMA 4-D box too large (%u x %u)", box_w_src, box_h_src);
    cuuint64_t dims[4] = {C, Wp, Hp, B};
    cuuint64_t strides[3] = {ld_elems * 2, Wp * ld_elems * 2, Hp * Wp * ld_elems * 2};
    cuuint32_t box[4] = {64, box_w_src, box_h_src, 1};
    cuuint32_t estr[4] = {1, 2, 2, 1};          // traversal stride 2 in x and y: the box delivers ceil(box/2) pixels per axis
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    ADAS_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(4-D, stride 2) failed: %d", (int)r);
    return 0;
}

// ---- SIMT validation kernel: same contract, CUDA cores, fp32 accumulate ---------------------------
__global__ void gemm_simt_kernel(const GemmParams p) {
    const int row = blockIdx.x * 64 + (threadIdx.x >> 2);       // 64 rows per block
    const int ng = blockIdx.y * 4 + (threadIdx.x & 3);          // group of 8 output columns
    const int n = ng * 8;
    if (row >= p.M || n >= p.N) return;
    bool row_ok = true;
    long out_row = row;
    if (p.mask_H > 0) {
        const int Wp = p.mask_W + 2;
        const int img = (p.mask_H + 2) * Wp;
        const int pp = row % img;
        const int yy = pp / Wp;
        const int xx = pp - yy * Wp;
        row_ok = (yy >= 1) && (yy <= p.mask_H) && (xx >= 1) && (xx <= p.mask_W);
        if (p.up2) {
            // 2x2 stride-2 transposed conv: column group (dy, dx) of input pixel (yy, xx) -> output pixel (2yy - 1 + dy, 2xx - 1 + dx)
            const int co = p.N / 4, q = n / co;
            out_row = ((long)(row / img) * (2 * p.mask_H + 2) + 2 * yy - 1 + q / 2) * (2 * p.mask_W + 2) + 2 * xx - 1 + q % 2;
        }
    }
    if (!row_ok) return;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    const int ncols = (p.N - n) < 8 ? (p.N - n) : 8;
    for (int tap = 0; tap < p.ntaps; ++tap) {
        int shift = 0;
        if (p.ntaps == 9) shift = (tap / 3 - 1) * p.Wp + (tap % 3 - 1);
        else if (p.ntaps == 4) shift = (tap - 2) * p.Wp;
        long ar = (long)row + shift;
        if (p.s2) {
            // out row -> (b, yo, xo); input pixel (2*yo+dy, 2*xo+dx) in the input's padded grid
            const int Wop = p.mask_W + 2, img = (p.mask_H + 2) * Wop;
            const int b = row / img, pp = row - b * img;
            const int yo = pp / Wop - 1, xo = pp % Wop - 1;
            const int dy = p.ntaps == 9 ? tap / 3 : 1, dx = p.ntaps == 9 ? tap % 3 : 1;
            ar = ((long)b * p.s2_Hp_in + 2 * yo + dy) * p.Wp + 2 * xo + dx;
        } else if (ar < 0 || ar >= p.M) continue;
        if (ar < 0) continue;
        const __half* a = p.A + (size_t)ar * p.a_ld;
        for (int c = 0; c < p.Kc; ++c) {
            const float av = __half2float(a[c]);
            for (int j = 0; j < ncols; ++j)
                acc[j] = fmaf(av, __half2float(p.Wt[(size_t)(n + j) * p.w_ld + tap * p.Kc + c]), acc[j]);
        }
    }
    for (int j = 0; j < ncols; ++j) {
        float x = acc[j];
        if (p.bias) x += p.transposed ? p.bias[row] : p.bias[n + j];
        if (p.res != nullptr && p.res_ld < 0) x += __half2float(p.res[(size_t)row * (size_t)(-p.res_ld) + n + j]);
        x = act_apply(x, p.act);
        if (p.res != nullptr && p.res_ld > 0) x += p.res_scale * __half2float(p.res[(size_t)row * (size_t)p.res_ld + n + j]);
        const size_t o = p.transposed ? ((size_t)(n + j) * p.out_ld + row)
                                      : p.up2 ? ((size_t)out_row * p.out_ld + (n + j) % (p.N / 4)) : ((size_t)row * p.out_ld + n + j);
        if (p.out_f32) reinterpret_cast<float*>(p.out)[o] = x;
        else reinterpret_cast<__half*>(p.out)[o] = __float2half_rn(x);
    }
}

int gemm_simt_launch(const GemmParams& p, cudaStream_t st) {
    dim3 grid((p.M + 63) / 64, (p.N + 31) / 32, 1);
    gemm_simt_kernel<<<grid, 256, 0, st>>>(p);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace adas
