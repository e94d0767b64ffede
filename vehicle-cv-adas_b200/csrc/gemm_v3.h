// gemm_v3.h -- tile configuration / launch record of the product GEMM kernel (gemm_v3.cu).
#pragma once
#include "common.h"
#include "tc_common.cuh"

namespace adas {

static constexpr int V3_CONSUMERS = 2;                         // consumer warpgroups: rows 0..63 / 64..127 of every 128-row sub-tile
static constexpr int V3_THREADS = 128 * (1 + V3_CONSUMERS);     // 384: one producer warpgroup (one TMA thread) + the consumers
static constexpr int V3_ACC_COLS = 256;                         // MT * BN <= 256: MT * BN / 2 fp32 accumulator registers per thread
static constexpr int V3_DYN_SMEM_MAX = 227 * 1024 - 1024;

struct GemmV3 {
    GemmParams p;
    int MT;            // 1..4 sub-tiles of 128 rows (stride-2: output patches) per CTA tile; they share every weight tile
    int slab;          // 3x3 stride-1: a stage holds one (dy, k-block) -- MT slabs of SLAB_ROWS rows + the three dx weight tiles
    int a_sub_bytes, b_bytes, stage_bytes, stages;
    int n_tiles, m_tiles, total_tiles;
    int pdl;
    int prefetch_w;    // fetch the first stages' weight tiles before griddepcontrol.wait
    int n_patches;     // stride-2: batch * s2_tw * s2_th
    FastDiv fd_img, fd_wp, fd_per_img, fd_tw, fd_bw;   // divisors of the epilogue's row arithmetic
};

struct GemmV3Launch {
    CUtensorMap tmA, tmB;
    GemmV3 g;
};

int gemm_v3_config(const GemmParams& p_in, GemmV3* g);
int v3_num_sms(int* num_sms);

}  // namespace adas
