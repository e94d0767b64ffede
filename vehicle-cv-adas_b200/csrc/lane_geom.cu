// lane_geom.cu -- what the reference does with the decoded lane points on the host, as one block per frame on the device
// (SURVEY 8f rank 1: the per-frame numpy / LAPACK tail after the lane decode):
//
//   * LaneDetectBase.__update_lanes_status / __update_lanes_area / __adjust_lanes_points  (ufldDetector/core.py:102-158):
//       area_status = both ego lanes detected; the ego-lane polygon = left ++ flipud(right), each side optionally replaced by a
//       degree-2 np.polyfit of x over y resampled on np.linspace(miny, maxy, image_height);
//   * PerspectiveTransformation.transformToBirdViewPoints (perspectiveTransformation.py:120-142): p' = M [x y 1]^T, (x'/w, y'/w)
//       truncated to int;
//   * PerspectiveTransformation.calcCurveAndOffset (perspectiveTransformation.py:145-208, the arithmetic; the arrows / text drawn on
//       the bird-view image stay with the host drawing code): degree-2 fits of the two bird-view ego lanes, direction from the
//       larger leading coefficient, refits in metres over the image rows, radius of curvature, lateral offset.
//
// np.polyfit(x, y, 2) = least squares on the Vandermonde matrix [x^2, x, 1] with columns scaled to unit 2-norm (numpy/lib/
// polynomial.py: lhs /= scale; lstsq; c /= scale).  numpy solves the scaled system by SVD (LAPACK gelsd); here it is Householder QR in
// float64 on the same scaled matrix -- the same least-squares solution up to rounding: both are backward stable, so they differ by at
// most the conditioning bound of tests/lane_conformance_cases.py polyfit_perturbation, which the tests carry through to the integer
// points (exact away from integer boundaries) and to curvature / offset.  All float64
// arithmetic that feeds an int() truncation follows numpy's operation order with _rn intrinsics (this file is built with -fmad=false).
#include "common.h"
#include "../../include/adas_b200.h"
#include <math.h>
#include <mutex>

namespace adas {

static constexpr int LG_THREADS = 128;
// rows of the largest fit: the bird-view image height (720 in the reference's demo; 2160 covers a 4K-tall bird view).  Six such
// float64 columns are the block's dynamic shared memory: 101.25 KB, within sm_90's 227 KB opt-in.
static constexpr int LG_MAX_N = 2160;

// deterministic block-wide sum (fixed order: per-thread strided partials -> warp shuffle tree -> warps in order)
__device__ double block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < LG_THREADS / 32; ++w) s += red[w];
    return s;
}

// c[0..2] (highest power first) = np.polyfit(x, y, 2) for n >= 3 points; a0,a1,a2,b: n-element scratch columns in shared memory
__device__ void polyfit2(const double* x, const double* y, int n, double* a0, double* a1, double* a2, double* b, double* red, double* c) {
    const int t = threadIdx.x;
    double s0 = 0, s1 = 0, s2 = 0;
    for (int i = t; i < n; i += LG_THREADS) {
        const double xi = x[i], q = xi * xi;
        a0[i] = q; a1[i] = xi; a2[i] = 1.0; b[i] = y[i];
        s0 += q * q; s1 += q; s2 += 1.0;
    }
    double scale[3];
    scale[0] = sqrt(block_sum(s0, red)); scale[1] = sqrt(block_sum(s1, red)); scale[2] = sqrt(block_sum(s2, red));
    for (int i = t; i < n; i += LG_THREADS) { a0[i] /= scale[0]; a1[i] /= scale[1]; a2[i] /= scale[2]; }
    __syncthreads();
    double* col[4] = {a0, a1, a2, b};
    double R[3][4];
    for (int k = 0; k < 3; ++k) {
        // Householder vector of column k below (and including) row k
        double p = 0;
        for (int i = k + t; i < n; i += LG_THREADS) p += col[k][i] * col[k][i];
        const double nrm = sqrt(block_sum(p, red));
        const double akk = col[k][k];
        const double alpha = akk > 0 ? -nrm : nrm;
        __syncthreads();
        if (t == 0) col[k][k] = akk - alpha;          // v = a_k - alpha e_k  (stored in place)
        __syncthreads();
        const double vnorm2 = 2.0 * (nrm * nrm - akk * alpha);      // |v|^2 = |a|^2 - 2 alpha a_kk + alpha^2
        R[k][k] = alpha;
        for (int j = k + 1; j < 4; ++j) {
            double d = 0;
            for (int i = k + t; i < n; i += LG_THREADS) d += col[k][i] * col[j][i];
            const double tau = vnorm2 > 0 ? 2.0 * block_sum(d, red) / vnorm2 : 0.0;
            for (int i = k + t; i < n; i += LG_THREADS) col[j][i] -= tau * col[k][i];
            __syncthreads();
            R[k][j] = col[j][k];
        }
    }
    // back substitution on the 3x3 triangle; a (numerically) zero pivot drops that coefficient (numpy's rank-deficient answer is the
    // minimum-norm one -- not reproduced; it needs all abscissae equal, which decoded lanes cannot produce)
    double z[3];
    for (int k = 2; k >= 0; --k) {
        double s = R[k][3];
        for (int j = k + 1; j < 3; ++j) s -= R[k][j] * z[j];
        z[k] = fabs(R[k][k]) > 1e-300 ? s / R[k][k] : 0.0;
    }
    c[0] = z[0] / scale[0]; c[1] = z[1] / scale[1]; c[2] = z[2] / scale[2];
    __syncthreads();
}

struct LaneGeomParams {
    const int32_t* pts; const int32_t* npts; const uint8_t* status;     // [B,4,max_pts,2], [B,4], [B,4]
    const double* M;                                                    // [B,9] row-major or nullptr (no bird view)
    int32_t* area; int32_t* bird; adas_lane_geom* out;
    int max_pts, img_w, img_h, adjust, bird_w, bird_h, cap_area;
};

__global__ void __launch_bounds__(LG_THREADS) lane_geom_kernel(const LaneGeomParams p) {
    extern __shared__ double sm[];
    double* a0 = sm; double* a1 = a0 + LG_MAX_N; double* a2 = a1 + LG_MAX_N; double* bb = a2 + LG_MAX_N;
    double* xs = bb + LG_MAX_N; double* ys = xs + LG_MAX_N;
    __shared__ double red[LG_THREADS / 32];
    const int f = blockIdx.x, t = threadIdx.x;
    const int32_t* P = p.pts + (size_t)f * 4 * p.max_pts * 2;
    const int32_t* N = p.npts + (size_t)f * 4;
    adas_lane_geom* o = p.out + f;
    const bool area_ok = p.status[f * 4 + 1] != 0 && p.status[f * 4 + 2] != 0;      // __update_lanes_status: the two ego lanes
    int32_t* area = p.area + (size_t)f * p.cap_area * 2;
    int n_area = 0;
    if (area_ok) {
        const int nl = N[1], nr = N[2];
        const int32_t* L = P + (size_t)1 * p.max_pts * 2;
        const int32_t* Rr = P + (size_t)2 * p.max_pts * 2;
        if (p.adjust && nl > 10 && nr > 10) {
            // __adjust_lanes_points: x = polyfit(y) per side, resampled on linspace(miny, maxy, image_height)
            double cl[3], cr[3];
            for (int i = t; i < nl; i += LG_THREADS) { xs[i] = (double)L[2 * i + 1]; ys[i] = (double)L[2 * i]; }
            __syncthreads();
            polyfit2(xs, ys, nl, a0, a1, a2, bb, red, cl);
            for (int i = t; i < nr; i += LG_THREADS) { xs[i] = (double)Rr[2 * i + 1]; ys[i] = (double)Rr[2 * i]; }
            __syncthreads();
            polyfit2(xs, ys, nr, a0, a1, a2, bb, red, cr);
            int miny = p.img_h / 3, maxy = p.img_h - 1, minl = 0x7fffffff, minr = 0x7fffffff;
            for (int i = 0; i < nl; ++i) { const int y = L[2 * i + 1]; maxy = max(maxy, y); miny = min(miny, y); minl = min(minl, y); }
            for (int i = 0; i < nr; ++i) { const int y = Rr[2 * i + 1]; maxy = max(maxy, y); miny = min(miny, y); minr = min(minr, y); }
            // np.linspace(miny, maxy, H): arange(H) * step + start, last element = stop
            const int H = p.img_h;
            const double step = __ddiv_rn((double)(maxy - miny), (double)(H - 1));
            // left side in order, then the right side reversed (np.flipud): two ordered compactions by one thread each pass would be
            // serial; instead every thread decides its rows and a block-wide exclusive scan (in row order) places them
            for (int side = 0; side < 2; ++side) {
                const double* c = side == 0 ? cl : cr;
                const int ymin = side == 0 ? minl : minr;
                for (int base = 0; base < H; base += LG_THREADS) {
                    const int idx = base + t;                       // position in emission order
                    const int i = side == 0 ? idx : H - 1 - idx;     // row of the linspace
                    bool keep = false; int px = 0, py = 0;
                    if (idx < H) {
                        const double y = (i == H - 1 && H > 1) ? (double)maxy : __dadd_rn(__dmul_rn((double)i, step), (double)miny);
                        const double x = __dadd_rn(__dadd_rn(__dmul_rn(c[0], __dmul_rn(y, y)), __dmul_rn(c[1], y)), c[2]);
                        keep = y >= (double)ymin && x >= 0.0;
                        px = (int)x; py = (int)y;
                    }
                    // ordered compaction of this chunk
                    const unsigned m = __ballot_sync(0xffffffffu, keep);
                    __shared__ int wcount[LG_THREADS / 32];
                    if ((t & 31) == 0) wcount[t >> 5] = __popc(m);
                    __syncthreads();
                    int off = n_area;
                    for (int w = 0; w < (t >> 5); ++w) off += wcount[w];
                    off += __popc(m & ((1u << (t & 31)) - 1u));
                    if (keep && off < p.cap_area) { area[2 * off] = px; area[2 * off + 1] = py; }
                    int tot = 0;
                    for (int w = 0; w < LG_THREADS / 32; ++w) tot += wcount[w];
                    n_area += tot;
                    __syncthreads();
                }
            }
        } else {
            for (int i = t; i < nl; i += LG_THREADS) if (i < p.cap_area) { area[2 * i] = L[2 * i]; area[2 * i + 1] = L[2 * i + 1]; }
            for (int i = t; i < nr; i += LG_THREADS) {
                const int d = nl + i, s = nr - 1 - i;
                if (d < p.cap_area) { area[2 * d] = Rr[2 * s]; area[2 * d + 1] = Rr[2 * s + 1]; }
            }
            n_area = nl + nr;
        }
    }
    // ---- bird view ----
    int direction = 2;
    double curvature = 0.0, offset = 0.0;
    if (p.M != nullptr) {
        const double* M = p.M + (size_t)f * 9;
        int32_t* B = p.bird + (size_t)f * 4 * p.max_pts * 2;
        for (int l = 0; l < 4; ++l)
            for (int i = t; i < N[l]; i += LG_THREADS) {
                const double x = (double)P[((size_t)l * p.max_pts + i) * 2], y = (double)P[((size_t)l * p.max_pts + i) * 2 + 1];
                const double nx = __dadd_rn(__dadd_rn(__dmul_rn(M[0], x), __dmul_rn(M[1], y)), M[2]);
                const double ny = __dadd_rn(__dadd_rn(__dmul_rn(M[3], x), __dmul_rn(M[4], y)), M[5]);
                const double nw = __dadd_rn(__dadd_rn(__dmul_rn(M[6], x), __dmul_rn(M[7], y)), M[8]);
                B[((size_t)l * p.max_pts + i) * 2] = (int32_t)(long long)__ddiv_rn(nx, nw);
                B[((size_t)l * p.max_pts + i) * 2 + 1] = (int32_t)(long long)__ddiv_rn(ny, nw);
            }
        __syncthreads();
        const int nl = N[1], nr = N[2];
        // below 720 rows the reference's leftx[719] raises IndexError: no curvature / offset ("None"), like a missing lane.  Two
        // points make a rank-deficient fit (numpy's minimum-norm answer is not reproduced): also "None".
        if (nl >= 3 && nr >= 3 && p.bird_h >= 720) {
            const int32_t* L = B + (size_t)1 * p.max_pts * 2;
            const int32_t* Rr = B + (size_t)2 * p.max_pts * 2;
            double lf[3], rf[3], lc[3], rc[3];
            for (int i = t; i < nl; i += LG_THREADS) { xs[i] = (double)L[2 * i + 1]; ys[i] = (double)L[2 * i]; }
            __syncthreads();
            polyfit2(xs, ys, nl, a0, a1, a2, bb, red, lf);
            for (int i = t; i < nr; i += LG_THREADS) { xs[i] = (double)Rr[2 * i + 1]; ys[i] = (double)Rr[2 * i]; }
            __syncthreads();
            polyfit2(xs, ys, nr, a0, a1, a2, bb, red, rf);
            const double side = fabs(lf[0]) > fabs(rf[0]) ? lf[0] : rf[0];
            if (side < -0.00015 && L[0] <= L[2 * (nl / 2)]) direction = -1;
            else if (side > 0.00015 && Rr[0] >= Rr[2 * (nr / 2)]) direction = 1;
            else direction = 0;
            const int H = p.bird_h;
            const double ym = 30.0 / 720.0, xm = 3.7 / 700.0;
            // ploty = linspace(0, H-1, H) = 0, 1, ..., H-1 exactly; leftx = a y^2 + b y + c
            for (int pass = 0; pass < 2; ++pass) {
                const double* cf = pass == 0 ? lf : rf;
                for (int i = t; i < H; i += LG_THREADS) {
                    const double y = (double)i;
                    xs[i] = y * ym;
                    ys[i] = (cf[0] * (y * y) + cf[1] * y + cf[2]) * xm;
                }
                __syncthreads();
                polyfit2(xs, ys, H, a0, a1, a2, bb, red, pass == 0 ? lc : rc);
            }
            const double y_eval = (double)(H - 1);
            const double tl = 2.0 * lc[0] * y_eval * ym + lc[1], tr = 2.0 * rc[0] * y_eval * ym + rc[1];
            const double lrad = pow(1.0 + tl * tl, 1.5) / fabs(2.0 * lc[0]);
            const double rrad = pow(1.0 + tr * tr, 1.5) / fabs(2.0 * rc[0]);
            curvature = (lrad + rrad) / 2.0;
            const double y719 = 719.0;                                  // the reference indexes leftx[719] whatever the image height
            const double lx = lf[0] * (y719 * y719) + lf[1] * y719 + lf[2], rx = rf[0] * (y719 * y719) + rf[1] * y719 + rf[2];
            const double lane_w = fabs(lx - rx);
            offset = ((lx + rx) / 2.0 - (double)p.bird_w / 2.0) * (3.7 / lane_w);
        }
    }
    if (t == 0) {
        o->area_status = area_ok ? 1 : 0; o->n_area = n_area; o->direction = direction; o->pad = 0;
        for (int l = 0; l < 4; ++l) o->n_bird[l] = p.M != nullptr ? N[l] : 0;
        o->curvature = curvature; o->offset = offset;
    }
}

int launch_lane_geom(const int32_t* pts, const int32_t* npts, const uint8_t* status, const double* M, int batch, int max_pts, int img_w, int img_h,
                     int adjust, int bird_w, int bird_h, int32_t* area, int cap_area, int32_t* bird, adas_lane_geom* out, cudaStream_t st) {
    ADAS_CHECK(max_pts >= 1 && max_pts <= LG_MAX_N && img_h >= 2 && cap_area >= 2 * max_pts, "lane_geometry: bad sizes (max_pts %d, img_h %d, cap_area %d)", max_pts, img_h, cap_area);
    ADAS_CHECK(!adjust || cap_area >= 2 * img_h, "lane_geometry: adjust_lanes needs room for 2 x image_height area points (cap_area %d)", cap_area);
    ADAS_CHECK(M == nullptr || bird_h <= LG_MAX_N, "lane_geometry: bird view of %d rows, at most %d are supported", bird_h, LG_MAX_N);
    LaneGeomParams p;
    p.pts = pts; p.npts = npts; p.status = status; p.M = M; p.area = area; p.bird = bird; p.out = out;
    p.max_pts = max_pts; p.img_w = img_w; p.img_h = img_h; p.adjust = adjust; p.bird_w = bird_w; p.bird_h = bird_h; p.cap_area = cap_area;
    const int smem = 6 * LG_MAX_N * 8;                      // 101.25 KB: needs the opt-in
    static std::mutex mu;
    static bool set_for[64] = {};
    int dev = 0;
    ADAS_CUDA(cudaGetDevice(&dev));
    {
        std::lock_guard<std::mutex> lk(mu);
        if (dev >= 0 && dev < 64 && !set_for[dev]) {
            ADAS_CUDA(cudaFuncSetAttribute(lane_geom_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            set_for[dev] = true;
        }
    }
    lane_geom_kernel<<<batch, LG_THREADS, smem, st>>>(p);
    count_launch();
    ADAS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace adas

extern "C" int adas_lane_geometry(int device, const int32_t* pts, const int32_t* npts, const uint8_t* status, int batch, int max_pts, int img_w,
                                  int img_h, int adjust_lanes, const double* M, int bird_w, int bird_h, int32_t* area, int cap_area, int32_t* bird,
                                  adas_lane_geom* out) {
    using namespace adas;
    ADAS_CHECK(pts && npts && status && area && out && batch >= 1 && (M == nullptr || bird != nullptr), "adas_lane_geometry: null argument");
    for (int i = 0; i < batch * 4; ++i) ADAS_CHECK(npts[i] >= 0 && npts[i] <= max_pts, "adas_lane_geometry: npts[%d] = %d outside [0, %d]", i, npts[i], max_pts);
    ADAS_CUDA(cudaSetDevice(device));
    const size_t np_ = (size_t)batch * 4 * max_pts * 2;
    int32_t *d_p = nullptr, *d_n = nullptr, *d_a = nullptr, *d_b = nullptr; uint8_t* d_s = nullptr; double* d_M = nullptr; adas_lane_geom* d_o = nullptr;
    int rc = 0;
    auto fail = [&](cudaError_t e, const char* what) { if (e != cudaSuccess && !rc) { set_error("adas_lane_geometry %s: %s", what, cudaGetErrorString(e)); rc = 1; } };
    fail(cudaMalloc(&d_p, np_ * 4), "alloc"); fail(cudaMalloc(&d_n, (size_t)batch * 16), "alloc"); fail(cudaMalloc(&d_s, (size_t)batch * 4), "alloc");
    fail(cudaMalloc(&d_a, (size_t)batch * cap_area * 8), "alloc"); fail(cudaMalloc(&d_o, (size_t)batch * sizeof(adas_lane_geom)), "alloc");
    if (M) { fail(cudaMalloc(&d_M, (size_t)batch * 72), "alloc"); fail(cudaMalloc(&d_b, np_ * 4), "alloc"); }
    if (!rc) {
        fail(cudaMemcpy(d_p, pts, np_ * 4, cudaMemcpyHostToDevice), "H2D");
        fail(cudaMemcpy(d_n, npts, (size_t)batch * 16, cudaMemcpyHostToDevice), "H2D");
        fail(cudaMemcpy(d_s, status, (size_t)batch * 4, cudaMemcpyHostToDevice), "H2D");
        if (M) fail(cudaMemcpy(d_M, M, (size_t)batch * 72, cudaMemcpyHostToDevice), "H2D");
        fail(cudaMemset(d_a, 0, (size_t)batch * cap_area * 8), "memset");
    }
    if (!rc) rc = launch_lane_geom(d_p, d_n, d_s, d_M, batch, max_pts, img_w, img_h, adjust_lanes, bird_w, bird_h, d_a, cap_area, d_b, d_o, 0);
    if (!rc) {
        fail(cudaMemcpy(area, d_a, (size_t)batch * cap_area * 8, cudaMemcpyDeviceToHost), "D2H");
        fail(cudaMemcpy(out, d_o, (size_t)batch * sizeof(adas_lane_geom), cudaMemcpyDeviceToHost), "D2H");
        if (M) fail(cudaMemcpy(bird, d_b, np_ * 4, cudaMemcpyDeviceToHost), "D2H");
    }
    cudaFree(d_p); cudaFree(d_n); cudaFree(d_s); cudaFree(d_a); cudaFree(d_o); cudaFree(d_M); cudaFree(d_b);
    return rc;
}
