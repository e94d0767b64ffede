// ufld_post.cu -- UFLDv2 row/column-anchor decode on the device (compiled with -fmad=false).
//
// Replaces UltrafastLaneDetectorV2.__process_output + _softmax
//   TrafficLaneDetector/ufldDetector/ultrafastLaneDetectorV2.py:114-181, :15-19
//   - max_indices = loc.argmax(grid axis) (first maximum), valid = exist.argmax(axis=1) (tie -> 0)   :127-134
//   - row lanes {1,2}: lane kept iff sum(valid) > num_cls_row/2;  col lanes {0,3}: > num_cls_col/4    :148,166
//   - per valid anchor: float32 softmax over the <=3 bins around the argmax, float64 expectation
//     (sum p*ind + 0.5)/(num_grid-1)*image_size, int() truncation                                    :151-154,169-172
//   - lane order left-side(col 0), left-ego(row 1), right-ego(row 2), right-side(col 3); detected iff > 2 points
//
// One CTA per frame.  Thread t < ncr*nl scans the row head for (anchor k = t/nl, lane i = t%nl) so that
// consecutive threads read consecutive floats of loc_row[g][k][i]; the column head likewise.
#include "common.h"

namespace adas {

static constexpr int UFLD_THREADS = 384;
static constexpr int UFLD_MAX_ANCH = 128;

__global__ void __launch_bounds__(UFLD_THREADS)
ufld_post_kernel(const float* __restrict__ heads, int ld, UfldDims d, const RigTable t,
                 const double* __restrict__ row_anchor, const double* __restrict__ col_anchor, int32_t* __restrict__ pts,
                 int32_t* __restrict__ npts, uint8_t* __restrict__ status, double* __restrict__ coords, int max_pts) {
    __shared__ int s_valid[2][4][UFLD_MAX_ANCH];      // [row/col][lane][anchor]
    __shared__ double s_coord[2][4][UFLD_MAX_ANCH];   // expectation coordinate (float64, pre-truncation)
    const int b = blockIdx.x;
    const int tid = threadIdx.x;
    const int img_w = t.cam[b / t.F].W, img_h = t.cam[b / t.F].H;     // this frame's camera
    const float* loc_row = heads + (size_t)b * ld;
    const float* loc_col = loc_row + (size_t)d.ngr * d.ncr * d.nl;
    const float* ex_row = loc_col + (size_t)d.ngc * d.ncc * d.nl;
    const float* ex_col = ex_row + (size_t)2 * d.ncr * d.nl;

    for (int part = 0; part < 2; ++part) {
        const int ng = part == 0 ? d.ngr : d.ngc;
        const int ncls = part == 0 ? d.ncr : d.ncc;
        const float* loc = part == 0 ? loc_row : loc_col;
        const float* ex = part == 0 ? ex_row : ex_col;
        const double size = part == 0 ? (double)img_w : (double)img_h;
        for (int t = tid; t < ncls * d.nl; t += UFLD_THREADS) {
            const int k = t / d.nl, i = t % d.nl;
            const int stride = ncls * d.nl;
            float best = loc[t];
            int m = 0;
            for (int g = 1; g < ng; ++g) {
                const float v = loc[(size_t)g * stride + t];
                if (v > best) { best = v; m = g; }
            }
            const int valid = ex[stride + t] > ex[t] ? 1 : 0;
            const int lo = m - 1 < 0 ? 0 : m - 1;
            const int hi = m + 1 > ng - 1 ? ng - 1 : m + 1;
            // float32 softmax (x - max, exp, / sum), then float64 expectation
            float e[3];
            float sum = 0.f;
            for (int g = lo; g <= hi; ++g) {
                e[g - lo] = expf(__fsub_rn(loc[(size_t)g * stride + t], best));
                sum = __fadd_rn(sum, e[g - lo]);
            }
            double acc = 0.0;
            for (int g = lo; g <= hi; ++g) {
                const float pr = __fdiv_rn(e[g - lo], sum);
                acc = __dadd_rn(acc, __dmul_rn((double)pr, (double)g));
            }
            double c = __dadd_rn(acc, 0.5);
            c = __dmul_rn(__ddiv_rn(c, (double)(ng - 1)), size);
            s_valid[part][i][k] = valid;
            s_coord[part][i][k] = c;
        }
    }
    __syncthreads();
    if (tid < 4) {
        // output lane `tid`: 0 = col lane 0, 1 = row lane 1, 2 = row lane 2, 3 = col lane 3
        const int part = (tid == 1 || tid == 2) ? 0 : 1;
        const int lane = tid;   // head lane index equals the output slot for {0,1,2,3}
        const int ncls = part == 0 ? d.ncr : d.ncc;
        int cnt = 0;
        for (int k = 0; k < ncls; ++k) cnt += s_valid[part][lane][k];
        const bool keep = part == 0 ? ((double)cnt > (double)d.ncr / 2.0) : ((double)cnt > (double)d.ncc / 4.0);
        int n = 0;
        int32_t* o = pts + ((size_t)b * 4 + tid) * max_pts * 2;
        double* oc = coords ? coords + ((size_t)b * 4 + tid) * max_pts : nullptr;
        if (keep) {
            for (int k = 0; k < ncls; ++k) {
                if (!s_valid[part][lane][k]) continue;
                const double c = s_coord[part][lane][k];
                int px, py;
                if (part == 0) { px = (int)c; py = (int)__dmul_rn(row_anchor[k], (double)img_h); }
                else           { px = (int)__dmul_rn(col_anchor[k], (double)img_w); py = (int)c; }
                o[n * 2] = px; o[n * 2 + 1] = py;
                if (oc) oc[n] = c;
                ++n;
            }
        }
        npts[b * 4 + tid] = n;
        status[b * 4 + tid] = n > 2 ? 1 : 0;
    }
}

int launch_ufld_post_rig(const float* heads, int ld, const RigTable& t, UfldDims d, const double* row_anchor, const double* col_anchor,
                         int32_t* pts, int32_t* npts, uint8_t* status, double* coords, int max_pts, cudaStream_t st) {
    ADAS_CHECK(t.n >= 1 && t.n <= ADAS_MAX_RIG_CAMERAS && t.F >= 1, "ufld_post: %d cameras of %d frames", t.n, t.F);
    ADAS_CHECK(d.nl == 4, "ufld_post: num_lanes must be 4 (got %d)", d.nl);
    ADAS_CHECK(d.ncr <= UFLD_MAX_ANCH && d.ncc <= UFLD_MAX_ANCH, "ufld_post: too many anchors");
    // the expectation divides by num_grid - 1: a 1-cell grid has no coordinate (the reference's int() of the infinity raises)
    ADAS_CHECK(d.ngr >= 2 && d.ngc >= 2, "ufld_post: grids of %d x %d cells, need at least 2 each", d.ngr, d.ngc);
    ufld_post_kernel<<<t.n * t.F, UFLD_THREADS, 0, st>>>(heads, ld, d, t, row_anchor, col_anchor, pts, npts, status, coords, max_pts);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

int launch_ufld_post(const float* heads, int ld, int B, UfldDims d, int img_w, int img_h, const double* row_anchor,
                     const double* col_anchor, int32_t* pts, int32_t* npts, uint8_t* status, double* coords, int max_pts,
                     cudaStream_t st) {
    return launch_ufld_post_rig(heads, ld, rig_one(nullptr, B, img_h, img_w), d, row_anchor, col_anchor, pts, npts, status, coords, max_pts, st);
}

// ------------------------------------------------------------------------------------------------------------------------------
// UFLD v1 decode: UltrafastLaneDetector.__process_output, TrafficLaneDetector/ufldDetector/ultrafastLaneDetector.py:97-136
//   - rows reversed (`[:, ::-1, :]`); float32 softmax over the griding_num cells without the last "no lane" bin, computed the way
//     scipy.special.softmax does (x - max, exp, sequential float32 sum along the grid axis, divide)                       :102-103
//   - expectation sum(prob * (cell + 1)) in float64 (float32 prob x int64 index promotes), 0 where the argmax over all
//     griding_num + 1 bins (first maximum) is the "no lane" bin                                                            :104-109
//   - lane detected iff more than two rows are non-zero; points for rows with loc > 0:
//       x = loc * col_sample_w * cfg.img_w / input_width - 1,  y = cfg.img_h * (row_anchor[R-1-p] / input_height) - 1,
//       [int(x * w_ratio), int(y * h_ratio)]                                                                               :112-131
// One CTA per frame, one thread per (reversed row p, lane l); head layout [griding_num + 1][rows][4].
__global__ void __launch_bounds__(UFLD_THREADS)
ufld_v1_post_kernel(const float* __restrict__ head, int ld, int G, int R, int in_w, int in_h, int cfg_w, int cfg_h, const RigTable t,
                    const double* __restrict__ row_anchor, int32_t* __restrict__ pts, int32_t* __restrict__ npts, uint8_t* __restrict__ status,
                    double* __restrict__ coords, int max_pts) {
    __shared__ double s_loc[4][UFLD_MAX_ANCH];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int img_w = t.cam[b / t.F].W, img_h = t.cam[b / t.F].H;     // this frame's camera
    const float* out = head + (size_t)b * ld;
    const int stride = R * 4;
    for (int t = tid; t < R * 4; t += UFLD_THREADS) {
        const int p = t / 4, l = t % 4;
        const int r = R - 1 - p;                                   // reversed rows
        const float* col = out + (size_t)r * 4 + l;
        float mx = col[0];
        for (int g = 1; g < G; ++g) mx = fmaxf(mx, col[(size_t)g * stride]);
        const bool none = col[(size_t)G * stride] > mx;            // argmax over G + 1 bins is the last one only if it is strictly larger
        float sum = 0.f;
        for (int g = 0; g < G; ++g) sum = __fadd_rn(sum, expf(__fsub_rn(col[(size_t)g * stride], mx)));
        double acc = 0.0;
        for (int g = 0; g < G; ++g) {
            const float pr = __fdiv_rn(expf(__fsub_rn(col[(size_t)g * stride], mx)), sum);
            acc = __dadd_rn(acc, __dmul_rn((double)pr, (double)(g + 1)));
        }
        s_loc[l][p] = none ? 0.0 : acc;
    }
    __syncthreads();
    if (tid < 4) {
        const int l = tid;
        int nz = 0;
        for (int p = 0; p < R; ++p) nz += s_loc[l][p] != 0.0;
        int n = 0;
        int32_t* o = pts + ((size_t)b * 4 + l) * max_pts * 2;
        double* oc = coords ? coords + ((size_t)b * 4 + l) * max_pts : nullptr;
        if (nz > 2) {
            // col_sample = np.linspace(0, input_width - 1, griding_num): col_sample[1] - col_sample[0] = 1 * step + 0 - 0
            const double csw = __ddiv_rn((double)(in_w - 1), (double)(G - 1));
            const double w_ratio = __ddiv_rn((double)img_w, (double)cfg_w), h_ratio = __ddiv_rn((double)img_h, (double)cfg_h);
            for (int p = 0; p < R; ++p) {
                const double loc = s_loc[l][p];
                if (!(loc > 0.0)) continue;
                const double x = __dsub_rn(__ddiv_rn(__dmul_rn(__dmul_rn(loc, csw), (double)cfg_w), (double)in_w), 1.0);
                const double y = __dsub_rn(__dmul_rn((double)cfg_h, __ddiv_rn(row_anchor[R - 1 - p], (double)in_h)), 1.0);
                o[n * 2] = (int)__dmul_rn(x, w_ratio);
                o[n * 2 + 1] = (int)__dmul_rn(y, h_ratio);
                if (oc) oc[n] = __dmul_rn(x, w_ratio);
                ++n;
            }
        }
        npts[b * 4 + l] = n;
        status[b * 4 + l] = nz > 2 ? 1 : 0;
    }
}

int launch_ufld_v1_post_rig(const float* head, int ld, const RigTable& t, int G, int R, int in_w, int in_h, int cfg_w, int cfg_h,
                            const double* row_anchor, int32_t* pts, int32_t* npts, uint8_t* status, double* coords, int max_pts, cudaStream_t st) {
    ADAS_CHECK(t.n >= 1 && t.n <= ADAS_MAX_RIG_CAMERAS && t.F >= 1, "ufld_v1_post: %d cameras of %d frames", t.n, t.F);
    ADAS_CHECK(G >= 3 && R >= 1 && R <= UFLD_MAX_ANCH && max_pts >= R, "ufld_v1_post: bad head %d x %d", G, R);
    ufld_v1_post_kernel<<<t.n * t.F, UFLD_THREADS, 0, st>>>(head, ld, G, R, in_w, in_h, cfg_w, cfg_h, t, row_anchor, pts, npts, status, coords, max_pts);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

int launch_ufld_v1_post(const float* head, int ld, int B, int G, int R, int in_w, int in_h, int cfg_w, int cfg_h, int img_w, int img_h,
                        const double* row_anchor, int32_t* pts, int32_t* npts, uint8_t* status, double* coords, int max_pts, cudaStream_t st) {
    return launch_ufld_v1_post_rig(head, ld, rig_one(nullptr, B, img_h, img_w), G, R, in_w, in_h, cfg_w, cfg_h, row_anchor, pts, npts, status, coords,
                                   max_pts, st);
}

}  // namespace adas
