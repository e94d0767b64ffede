// track.cu -- ByteTrack association kernels (compiled with -fmad=false; float64 like the reference).
//
// Replaces (ObjectTracker/byteTrack/matching.py):
//   ious / iou_distance   :34-80    iou = wh / (a1 + a2 - wh), no "+1" convention; cost = 1 - iou
//   fuse_score            :108-116  cost = 1 - (1 - cost) * det_score[j]
//   linear_assignment     :20-31    lap.lapjv(cost, extend_cost=True, cost_limit=thresh): the exact optimum of the
//                                   (T+D)x(T+D) extended problem == min over partial matchings of
//                                   sum(cost[matched]) + thresh/2 * (#unmatched rows + #unmatched cols).
// `lap` is an un-vendored third-party C extension (requirements.txt:4, unpinned); the solver here is a
// shortest-augmenting-path (Jonker-Volgenant / Hungarian with potentials) on the equivalent rectangular
// problem: T rows x (D real + T private dummy) columns, real cost c - thresh, own dummy cost 0.
// One warp per problem; the column scan of each Dijkstra step is lane-parallel with a deterministic
// (lowest column) argmin.
// Ties (the real library's tie-breaking is unpinned): every entry point (lap, associate, the fused tracker stages) runs the same
// lap_solve on the same float64 costs, so all of them return the same assignment.  Threshold rule: a pair whose cost equals
// thresh exactly is matched when nothing else competes for it -- real columns precede the dummy ones, so the lowest-column argmin
// prefers the match (a 1x1 problem at cost == thresh matches; one ulp above it does not).
// NaN costs (IoU 0/0 of two zero-area boxes; the reference's behaviour is undefined): `cur < minv` is false for NaN, so the search
// never relaxes a NaN edge and a NaN pair is never matched; the result is the optimum of the problem without those pairs.  Every
// row still reaches its own finite dummy column, so the "no finite candidate" exit below is a guard, not a path.
#include "common.h"

namespace adas {

// cost[t][d] of one association stage (matching.py:34-80,108-116), float64, one rounding per numpy op
__device__ __forceinline__ double assoc_cost(const double* A, const double* Bx, const double* sc, int fuse, int t, int dd) {
    const double ax1 = A[t * 4], ay1 = A[t * 4 + 1], ax2 = A[t * 4 + 2], ay2 = A[t * 4 + 3];
    const double bx1 = Bx[dd * 4], by1 = Bx[dd * 4 + 1], bx2 = Bx[dd * 4 + 2], by2 = Bx[dd * 4 + 3];
    const double xx1 = fmax(ax1, bx1), yy1 = fmax(ay1, by1);
    const double xx2 = fmin(ax2, bx2), yy2 = fmin(ay2, by2);
    const double w = fmax(0.0, __dsub_rn(xx2, xx1));
    const double h = fmax(0.0, __dsub_rn(yy2, yy1));
    const double wh = __dmul_rn(w, h);
    const double aa = __dmul_rn(__dsub_rn(ax2, ax1), __dsub_rn(ay2, ay1));
    const double ab = __dmul_rn(__dsub_rn(bx2, bx1), __dsub_rn(by2, by1));
    const double iou = __ddiv_rn(wh, __dsub_rn(__dadd_rn(aa, ab), wh));
    double c = __dsub_rn(1.0, iou);
    if (fuse) {
        const double sim = __dsub_rn(1.0, c);
        c = __dsub_rn(1.0, __dmul_rn(sim, sc[dd]));
    }
    return c;
}

__global__ void iou_cost_kernel(const double* __restrict__ a, const int32_t* __restrict__ a_off, const double* __restrict__ bxs,
                                const int32_t* __restrict__ b_off, const double* __restrict__ det_scores, int fuse,
                                double* __restrict__ cost, const int64_t* __restrict__ cost_off) {
    const int pr = blockIdx.x;
    const int T = a_off[pr + 1] - a_off[pr];
    const int D = b_off[pr + 1] - b_off[pr];
    const double* A = a + (size_t)a_off[pr] * 4;
    const double* Bx = bxs + (size_t)b_off[pr] * 4;
    const double* sc = det_scores ? det_scores + b_off[pr] : nullptr;
    double* C = cost + cost_off[pr];
    for (int i = threadIdx.x; i < T * D; i += blockDim.x) C[i] = assoc_cost(A, Bx, sc, fuse, i / D, i % D);
}

int launch_iou_cost(int problems, const double* a, const int32_t* a_off, const double* b, const int32_t* b_off,
                    const double* det_scores, int fuse, double* cost, const int64_t* cost_off, cudaStream_t st) {
    iou_cost_kernel<<<problems, 256, 0, st>>>(a, a_off, b, b_off, det_scores, fuse, cost, cost_off);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------
static constexpr int LAP_MAX_COLS = 2048;   // D + T

__device__ __forceinline__ double lap_cost(const double* C, int D, int T, double thresh, int i, int j) {
    // i in [0,T), j in [0, D+T)
    if (j < D) return __dsub_rn(C[(size_t)i * D + j], thresh);
    return (j - D == i) ? 0.0 : 1e300;
}

// Exact assignment of one problem by ONE WARP (all 32 lanes call it together).  C: T x D cost matrix; X[T] / Y[D] receive the matched
// column / row or -1.  Scratch: v, minv (m + 1 doubles), p / way / used (3 x ws int32, ws >= m + 1), u (T + 1 doubles).
__device__ void lap_solve(const double* __restrict__ C, int T, int D, double thresh, int32_t* __restrict__ X, int32_t* __restrict__ Y,
                          double* __restrict__ v, double* __restrict__ minv, int32_t* __restrict__ p, int ws, double* u) {
    const int lane = threadIdx.x & 31;
    const int m = D + T;
    int32_t* way = p + ws;
    int32_t* used = way + ws;
    for (int j = lane; j <= m; j += 32) { v[j] = 0.0; p[j] = 0; way[j] = 0; }
    for (int i = lane; i <= T; i += 32) u[i] = 0.0;
    __syncwarp();
    // columns are 1-based internally (column 0 is the virtual start), rows 1-based
    for (int i = 1; i <= T; ++i) {
        if (lane == 0) p[0] = i;
        for (int j = lane; j <= m; j += 32) { minv[j] = 1e308; used[j] = 0; }
        __syncwarp();
        int j0 = 0;
        while (true) {
            if (lane == 0) used[j0] = 1;
            __syncwarp();
            const int i0 = p[j0];
            const double ui0 = u[i0];
            double bd = 1e308; int bj = 0x7fffffff;
            for (int j = 1 + lane; j <= m; j += 32) {
                if (!used[j]) {
                    const double cur = __dsub_rn(__dsub_rn(lap_cost(C, D, T, thresh, i0 - 1, j - 1), ui0), v[j]);
                    if (cur < minv[j]) { minv[j] = cur; way[j] = j0; }
                    const double mv = minv[j];
                    if (mv < bd) { bd = mv; bj = j; }
                }
            }
            for (int o = 16; o > 0; o >>= 1) {
                const double od = __shfl_xor_sync(0xffffffffu, bd, o);
                const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
                if (od < bd || (od == bd && oj < bj)) { bd = od; bj = oj; }
            }
            if (bj == 0x7fffffff) break;      // no finite candidate (NaN costs): leave the row unmatched instead of spinning
            __syncwarp();                     // the scan above wrote minv[j] / way[j] with a different lane -> column mapping than the update below
            const double delta = bd;
            const int j1 = bj;
            for (int j = lane; j <= m; j += 32) {
                if (used[j]) { u[p[j]] = __dadd_rn(u[p[j]], delta); v[j] = __dsub_rn(v[j], delta); }
                else minv[j] = __dsub_rn(minv[j], delta);
            }
            __syncwarp();
            j0 = j1;
            if (p[j0] == 0) break;
        }
        // augment along the alternating path
        if (lane == 0 && p[j0] == 0) {
            while (j0 != 0) {
                const int j1 = way[j0];
                p[j0] = p[j1];
                j0 = j1;
            }
        }
        __syncwarp();
    }
    for (int i = lane; i < T; i += 32) X[i] = -1;
    for (int j = lane; j < D; j += 32) Y[j] = -1;
    __syncwarp();
    for (int j = 1 + lane; j <= D; j += 32) {
        const int r = p[j];
        if (r != 0) { X[r - 1] = j - 1; Y[j - 1] = r - 1; }
    }
    __syncwarp();
}

__global__ void lap_kernel(const double* __restrict__ cost, const int64_t* __restrict__ cost_off, const int32_t* __restrict__ Ts,
                           const int32_t* __restrict__ Ds, const double* __restrict__ threshs, int32_t* __restrict__ x,
                           const int32_t* __restrict__ x_off, int32_t* __restrict__ y, const int32_t* __restrict__ y_off,
                           double* __restrict__ work_v, double* __restrict__ work_minv, int32_t* __restrict__ work_i) {
    // one warp per problem (blockDim = 32)
    const int pr = blockIdx.x;
    __shared__ double u[LAP_MAX_COLS / 2 + 1];   // row potentials (T <= 1024)
    lap_solve(cost + cost_off[pr], Ts[pr], Ds[pr], threshs[pr], x + x_off[pr], y + y_off[pr], work_v + (size_t)pr * (LAP_MAX_COLS + 1),
              work_minv + (size_t)pr * (LAP_MAX_COLS + 1), work_i + (size_t)pr * 3 * (LAP_MAX_COLS + 1), LAP_MAX_COLS + 1, u);
}

// ------------------------------------------------------------------------------------------------
// The three association stages of BYTETracker.update (byteTracker.py:100-160) in ONE launch by one warp:
//   stage 1  pool (confirmed + lost, already predicted) x high-score detections, fused cost, match_thresh
//   stage 2  unmatched pool tracks that are still `Tracked` x low-score detections, plain IoU cost, 0.5
//   stage 3  unconfirmed tracks x the high-score detections stage 1 left unmatched, fused cost, 0.7
// The lists stage 2 and 3 work on are index filters of stage 1's result (ascending order, as the reference builds them), so the
// host needs only this kernel's outputs to apply the Kalman updates -- one launch and one synchronisation per frame instead of
// three launch pairs and three round trips.
// in  (doubles): [P, U, D, D2, match_thresh] header (5) | pool tlbr P*4 | pool tracked flag P | unconf tlbr U*4 | det tlbr D*4 |
//                det score D | det2 tlbr D2*4
// out (int32):   m1[P] det index or -1 | m2[P] det2 index or -1 (only for stage-2 rows) | m3[U] ORIGINAL det index or -1 |
//                free3[D] 1 = high-score detection unmatched after stages 1 and 3 (a birth candidate)
// Host round trip: `in_host` / `out_host` / `done_host` are MAPPED pinned host buffers.  The warp pulls the inputs over the link with
// coalesced loads into device scratch, solves, pushes the results back and then (the last problem of the launch to finish) publishes
// `seq` in *done_host behind a system-scope fence -- the host spins on that word (tracker.cu) instead of paying two copy-engine
// transfers and a stream synchronisation per frame.
// Row potentials live in shared memory only up to ASSOC_SMEM_ROWS rows (1 KB): next to a conv CTA that holds ~224 KB of an SM's shared
// memory this block still fits, so it starts at once instead of waiting for a conv CTA to retire; larger problems use global scratch.
// The column scratch (v, minv: ws doubles; p / way / used: 3 x ws int32) is sized by the host for the largest stage of the problem
// (ws > max(P + D, P + D2, U + D)), so the fused association has no size limit of its own -- like the reference.
static constexpr int ASSOC_SMEM_ROWS = 120;

__device__ void assoc3_body(const double* __restrict__ in, int32_t* __restrict__ out, double* __restrict__ cost, double* __restrict__ work_v,
                            double* __restrict__ work_minv, int32_t* __restrict__ work_i, int ws, int32_t* __restrict__ lists, double* u) {
    const int lane = threadIdx.x;
    const int P = (int)in[0], U = (int)in[1], D = (int)in[2], D2 = (int)in[3];
    const double match_thresh = in[4];
    const double* pool = in + 5;
    const double* trk = pool + (size_t)P * 4;
    const double* unconf = trk + P;
    const double* det = unconf + (size_t)U * 4;
    const double* dsc = det + (size_t)D * 4;
    const double* det2 = dsc + D;
    int32_t* m1 = out; int32_t* m2 = m1 + P; int32_t* m3 = m2 + P; int32_t* free3 = m3 + U;
    int32_t* rem = lists;                 // [P]   stage-2 rows (pool indices)
    int32_t* left = rem + P;              // [D]   stage-3 columns (det indices)
    int32_t* xs = left + D;               // [max(P,U)] assignment scratch (rows)
    int32_t* ys = xs + (P > U ? P : U);   // [max(D,D2)] assignment scratch (columns)
    double* lsc = cost + (size_t)(P > U ? P : U) * (D > D2 ? D : D2);   // scores of `left` behind the cost matrix
    double* lbox = lsc + D;                                               // boxes of `left`
    double* rbox = lbox + (size_t)D * 4;                                  // boxes of `rem`
    // ---- stage 1 ----
    for (int i = lane; i < P; i += 32) { m1[i] = -1; m2[i] = -1; }
    for (int i = lane; i < U; i += 32) m3[i] = -1;
    for (int j = lane; j < D; j += 32) ys[j] = -1;
    __syncwarp();
    if (P > 0 && D > 0) {
        for (int i = lane; i < P * D; i += 32) cost[i] = assoc_cost(pool, det, dsc, 1, i / D, i % D);
        __syncwarp();
        lap_solve(cost, P, D, match_thresh, m1, ys, work_v, work_minv, work_i, ws, u);
    }
    // rem = unmatched pool rows that are Tracked; left = unmatched detections (both ascending)
    int R = 0, L = 0;
    if (lane == 0) {
        for (int i = 0; i < P; ++i) if (m1[i] < 0 && trk[i] != 0.0) rem[R++] = i;
        for (int j = 0; j < D; ++j) if (ys[j] < 0) left[L++] = j;
    }
    R = __shfl_sync(0xffffffffu, R, 0);
    L = __shfl_sync(0xffffffffu, L, 0);
    __syncwarp();
    // ---- stage 2 ----
    if (R > 0 && D2 > 0) {
        for (int i = lane; i < R * 4; i += 32) rbox[i] = pool[(size_t)rem[i >> 2] * 4 + (i & 3)];
        __syncwarp();
        for (int i = lane; i < R * D2; i += 32) cost[i] = assoc_cost(rbox, det2, nullptr, 0, i / D2, i % D2);
        __syncwarp();
        lap_solve(cost, R, D2, 0.5, xs, ys, work_v, work_minv, work_i, ws, u);
        for (int k = lane; k < R; k += 32) m2[rem[k]] = xs[k];
        __syncwarp();
    }
    // rows of stage 2 are flagged for the host: m2 == -1 on a stage-2 row means "mark lost"; rows that were not in stage 2 get -2
    for (int i = lane; i < P; i += 32) if (!(m1[i] < 0 && trk[i] != 0.0)) m2[i] = -2;
    // ---- stage 3 ----
    for (int j = lane; j < D; j += 32) free3[j] = 0;
    __syncwarp();
    if (U > 0 && L > 0) {
        for (int i = lane; i < L * 4; i += 32) lbox[i] = det[(size_t)left[i >> 2] * 4 + (i & 3)];
        for (int j = lane; j < L; j += 32) lsc[j] = dsc[left[j]];
        __syncwarp();
        for (int i = lane; i < U * L; i += 32) cost[i] = assoc_cost(unconf, lbox, lsc, 1, i / L, i % L);
        __syncwarp();
        lap_solve(cost, U, L, 0.7, xs, ys, work_v, work_minv, work_i, ws, u);
        for (int k = lane; k < U; k += 32) m3[k] = xs[k] >= 0 ? left[xs[k]] : -1;
        for (int j = lane; j < L; j += 32) if (ys[j] < 0) free3[left[j]] = 1;
    } else {
        for (int j = lane; j < L; j += 32) free3[left[j]] = 1;
    }
}

// One block (one warp) per problem: the cameras of a multi-camera rig are independent trackers, so a time step solves all of them in
// one launch.  Each problem has its own slices of every buffer (Assoc3Problem) and picks the shared-memory route on its own sizes, so
// one crowded camera does not move the others to global memory.  The completion word is per launch: every block pushes its result,
// fences and counts itself done; the last one publishes `seq`.
__global__ void assoc3_kernel(Assoc3Buffers b, int problems, int32_t seq) {
    __shared__ double u_s[ASSOC_SMEM_ROWS + 1];
    const int lane = threadIdx.x;
    const int64_t d = lane < 8 ? reinterpret_cast<const int64_t*>(b.probs + blockIdx.x)[lane] : 0;   // the descriptor: one 64-byte read
    const int64_t in_off = __shfl_sync(0xffffffffu, d, 0), n_in = __shfl_sync(0xffffffffu, d, 1);
    const int64_t out_off = __shfl_sync(0xffffffffu, d, 2), n_out = __shfl_sync(0xffffffffu, d, 3);
    const int64_t cost_off = __shfl_sync(0xffffffffu, d, 4), lists_off = __shfl_sync(0xffffffffu, d, 5);
    const int64_t ws_off = __shfl_sync(0xffffffffu, d, 6), ws = __shfl_sync(0xffffffffu, d, 7);
    double* in = b.in + in_off;
    for (int64_t i = lane; i < n_in; i += 32) in[i] = b.in_host[in_off + i];
    __syncwarp();
    const int P = (int)in[0], U = (int)in[1];
    int32_t* out = b.out + out_off;
    assoc3_body(in, out, b.cost + cost_off, b.v + ws_off, b.minv + ws_off, b.wi + 3 * ws_off, (int)ws, b.lists + lists_off,
                (P <= ASSOC_SMEM_ROWS && U <= ASSOC_SMEM_ROWS) ? u_s : b.u + ws_off);
    __syncwarp();
    for (int64_t i = lane; i < n_out; i += 32) b.out_host[out_off + i] = out[i];
    __threadfence_system();
    __syncwarp();
    if (lane == 0 && atomicAdd(b.finished, 1u) == (unsigned)problems - 1) {
        *b.finished = 0;                               // ready for the next launch (stream-ordered after this one)
        __threadfence_system();
        *(volatile int32_t*)b.done_host = seq;
    }
}

int launch_assoc3(int problems, const Assoc3Buffers& b, int32_t seq, cudaStream_t st) {
    assoc3_kernel<<<problems, 32, 0, st>>>(b, problems, seq);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

int launch_lap(int problems, const double* cost, const int64_t* cost_off, const int32_t* T, const int32_t* D,
               const double* thresh, int32_t* x, const int32_t* x_off, int32_t* y, const int32_t* y_off, double* work_v,
               double* work_minv, int32_t* work_i, cudaStream_t st) {
    lap_kernel<<<problems, 32, 0, st>>>(cost, cost_off, T, D, thresh, x, x_off, y, y_off, work_v, work_minv, work_i);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

int lap_max_cols() { return LAP_MAX_COLS; }

}  // namespace adas
