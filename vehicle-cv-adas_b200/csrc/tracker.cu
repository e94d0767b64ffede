// tracker.cu -- native ByteTrack state machine (host C++) driving the device association kernels of track.cu.
//
// Replaces the per-frame Python of ObjectTracker/byteTrack/byteTracker.py:62-185 (three association stages, births,
// ageing, list maintenance), dtypes/strack.py (track records, class vote, conversions), dtypes/kalman_filter.py:55-226
// (constant-velocity filter, float64) and utils.py:9-69 (joint / sub / duplicate removal).  The IoU cost matrices and
// the exact assignment of all three stages of a frame run on the device in ONE launch (track.cu assoc3_kernel: one upload, one
// launch, one download, one synchronisation per frame); the 8x8 float64 Kalman algebra and the list bookkeeping are sequential
// per stream and stay on the host.  adas_tracker_update_batch takes all frames of a pipeline step in one call.
#include "common.h"
#include "../../include/adas_b200.h"
#include <math.h>
#include <time.h>
#include <string.h>
#include <algorithm>
#include <memory>
#include <utility>

namespace adas {
static inline uint64_t now_ns() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec; }
int launch_iou_cost(int problems, const double* a, const int32_t* a_off, const double* b, const int32_t* b_off,
                    const double* det_scores, int fuse, double* cost, const int64_t* cost_off, cudaStream_t st);
int launch_lap(int problems, const double* cost, const int64_t* cost_off, const int32_t* T, const int32_t* D,
               const double* thresh, int32_t* x, const int32_t* x_off, int32_t* y, const int32_t* y_off, double* work_v,
               double* work_minv, int32_t* work_i, cudaStream_t st);
int lap_max_cols();
int launch_assoc3(const double* in_host, int n_in, double* in_dev, int32_t* out_host, int n_out, int32_t* out_dev, int32_t* done_host, int32_t seq,
                  double* cost, double* work_v, double* work_minv, int32_t* work_i, int ws, int32_t* lists, double* work_u, cudaStream_t st);

enum { ST_NEW = 0, ST_TRACKED = 1, ST_LOST = 2, ST_REMOVED = 3 };
static std::atomic<int> g_track_count{0};          // BaseTrack._count: process-global (base_track.py:12,33-36)

struct Track {
    double tlwh0[4];
    double mean[8];
    double cov[64];
    bool has_kf = false, activated = false;
    int state = ST_NEW, id = 0, frame = 0, start = 0, cls = 0, tracklet_len = 0;
    double score = 0.0;
    double det_tlbr[4] = {0, 0, 0, 0};
    int traj_frame = 0;
    std::vector<std::pair<int, int>> votes;     // class-id history in insertion order (dict semantics)

    void tlwh(double* o) const {
        if (!has_kf) { memcpy(o, tlwh0, 32); return; }
        o[2] = mean[2] * mean[3]; o[3] = mean[3];
        o[0] = mean[0] - o[2] / 2; o[1] = mean[1] - o[3] / 2;
    }
    void tlbr(double* o) const { tlwh(o); o[2] += o[0]; o[3] += o[1]; }
    void vote(int c) {                          // strack.py:122-129 (a class seen for the first time after birth starts at 2)
        bool found = false;
        for (auto& v : votes) if (v.first == c) { v.second += 1; found = true; break; }
        if (!found) votes.push_back({c, 2});
        int best = votes[0].second; cls = votes[0].first;
        for (auto& v : votes) if (v.second > best) { best = v.second; cls = v.first; }
    }
};
typedef std::shared_ptr<Track> TrackP;

static const double W_POS = 1.0 / 20, W_VEL = 1.0 / 160;

static void xyah_of_tlwh(const double* t, double* z) { z[0] = t[0] + t[2] / 2; z[1] = t[1] + t[3] / 2; z[2] = t[2] / t[3]; z[3] = t[3]; }

static void kf_initiate(Track& t) {                // kalman_filter.py:55-86
    double z[4];
    xyah_of_tlwh(t.tlwh0, z);
    for (int i = 0; i < 4; ++i) { t.mean[i] = z[i]; t.mean[4 + i] = 0.0; }
    const double h = z[3];
    const double std_[8] = {2 * W_POS * h, 2 * W_POS * h, 1e-2, 2 * W_POS * h, 10 * W_VEL * h, 10 * W_VEL * h, 1e-5, 10 * W_VEL * h};
    memset(t.cov, 0, sizeof(t.cov));
    for (int i = 0; i < 8; ++i) t.cov[i * 9] = std_[i] * std_[i];
    t.has_kf = true;
}

static void kf_predict(Track& t) {                 // kalman_filter.py:155-192 with F = [[I, I], [0, I]]
    if (t.state != ST_TRACKED) t.mean[7] = 0.0;   // strack.py:66-68
    const double h = t.mean[3];
    const double sp[4] = {W_POS * h, W_POS * h, 1e-2, W_POS * h}, sv[4] = {W_VEL * h, W_VEL * h, 1e-5, W_VEL * h};
    for (int i = 0; i < 4; ++i) t.mean[i] += t.mean[4 + i];
    double fc[64], out[64];
    for (int i = 0; i < 8; ++i)                   // F * cov : row i += row i+4 for i < 4
        for (int j = 0; j < 8; ++j) fc[i * 8 + j] = t.cov[i * 8 + j] + (i < 4 ? t.cov[(i + 4) * 8 + j] : 0.0);
    for (int i = 0; i < 8; ++i)                   // (F cov) * F^T : col j += col j+4 for j < 4
        for (int j = 0; j < 8; ++j) out[i * 8 + j] = fc[i * 8 + j] + (j < 4 ? fc[i * 8 + j + 4] : 0.0);
    for (int i = 0; i < 4; ++i) { out[i * 9] += sp[i] * sp[i]; out[(4 + i) * 9] += sv[i] * sv[i]; }
    memcpy(t.cov, out, sizeof(out));
}

static void kf_update(Track& t, const double* z) {  // kalman_filter.py:194-226 (project + Cholesky solve)
    const double h = t.mean[3];
    const double sd[4] = {W_POS * h, W_POS * h, 1e-1, W_POS * h};
    double pc[16], L[16];
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) pc[i * 4 + j] = t.cov[i * 8 + j] + (i == j ? sd[i] * sd[i] : 0.0);
    memset(L, 0, sizeof(L));
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j <= i; ++j) {
            double s = pc[i * 4 + j];
            for (int k = 0; k < j; ++k) s -= L[i * 4 + k] * L[j * 4 + k];
            L[i * 4 + j] = (i == j) ? sqrt(s) : s / L[j * 4 + j];
        }
    // gain[r][:] solves pc * g = cov[r][0:4]^T for every state row r  (K = cov H^T pc^-1)
    double K[32];
    for (int r = 0; r < 8; ++r) {
        double y[4], g[4];
        for (int i = 0; i < 4; ++i) { double s = t.cov[r * 8 + i]; for (int k = 0; k < i; ++k) s -= L[i * 4 + k] * y[k]; y[i] = s / L[i * 4 + i]; }
        for (int i = 3; i >= 0; --i) { double s = y[i]; for (int k = i + 1; k < 4; ++k) s -= L[k * 4 + i] * g[k]; g[i] = s / L[i * 4 + i]; }
        for (int i = 0; i < 4; ++i) K[r * 4 + i] = g[i];
    }
    double innov[4];
    for (int i = 0; i < 4; ++i) innov[i] = z[i] - t.mean[i];
    for (int r = 0; r < 8; ++r) { double s = 0; for (int i = 0; i < 4; ++i) s += innov[i] * K[r * 4 + i]; t.mean[r] += s; }
    double kp[32];                                 // K * pc
    for (int r = 0; r < 8; ++r) for (int j = 0; j < 4; ++j) { double s = 0; for (int i = 0; i < 4; ++i) s += K[r * 4 + i] * pc[i * 4 + j]; kp[r * 4 + j] = s; }
    for (int r = 0; r < 8; ++r) for (int c = 0; c < 8; ++c) { double s = 0; for (int j = 0; j < 4; ++j) s += kp[r * 4 + j] * K[c * 4 + j]; t.cov[r * 8 + c] -= s; }
}

static double iou_dist(const double* a, const double* b) {   // matching.py:34-53 on the host (duplicate removal only)
    const double xx1 = std::max(a[0], b[0]), yy1 = std::max(a[1], b[1]), xx2 = std::min(a[2], b[2]), yy2 = std::min(a[3], b[3]);
    const double w = std::max(0.0, xx2 - xx1), h = std::max(0.0, yy2 - yy1), wh = w * h;
    return 1.0 - wh / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - wh);
}

}  // namespace adas

using namespace adas;

struct adas_tracker {
    int device = 0;
    double track_thresh = 0.5, match_thresh = 0.8, det_thresh = 0.6;
    int max_time_lost = 30, frame_id = 0;
    std::vector<TrackP> tracked, lost, removed;
    // device scratch (persistent) for the association stages
    cudaStream_t st = nullptr;
    size_t cap_boxes = 0, cap_cost = 0;
    double *d_a = nullptr, *d_b = nullptr, *d_s = nullptr, *d_c = nullptr, *d_th = nullptr, *d_v = nullptr, *d_mv = nullptr;
    int32_t *d_meta = nullptr, *d_x = nullptr, *d_y = nullptr, *d_wi = nullptr;
    int64_t* d_co = nullptr;
    std::vector<double> ha, hb, hs;
    std::vector<int32_t> hx, hy;
    // fused three-stage association (one launch + one synchronisation per frame)
    double* h3_in = nullptr; int32_t* h3_out = nullptr;      // pinned + mapped: the association kernel reads / writes them over the link
    double* h3_in_dev = nullptr; int32_t* h3_out_dev = nullptr;   // their device-side addresses
    int32_t* h_done = nullptr; int32_t* h_done_dev = nullptr; int32_t seq = 0;   // completion word the host spins on
    double* d_u = nullptr;                                    // row potentials of problems beyond the kernel's shared-memory budget
    size_t cap_ws = 0;                                        // entries of d_v / d_mv / d_u and of each third of d_wi (column scratch)
    // wall-clock accounting of the update path (adas_tracker_stats): frames, total ns, ns between launch and result, launches
    uint64_t st_frames = 0, st_total_ns = 0, st_wait_ns = 0, st_launches = 0;
    double* d3_in = nullptr; int32_t* d3_out = nullptr; double* d3_cost = nullptr; int32_t* d3_lists = nullptr;
    size_t cap3_in = 0, cap3_out = 0, cap3_cost = 0, cap3_lists = 0;
};

namespace adas {

static int ensure_scratch(adas_tracker* t, size_t nb, size_t nc) {
    if (t->st == nullptr) {
        // the association kernels are tiny and on the host's critical path: highest priority, so they are scheduled as soon as any
        // CTA slot frees up between the detectors' persistent conv kernels
        int prio_lo = 0, prio_hi = 0;
        cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
        ADAS_CUDA(cudaStreamCreateWithPriority(&t->st, cudaStreamNonBlocking, prio_hi));
        const size_t wc = (size_t)lap_max_cols() + 1;
        ADAS_CUDA(cudaMalloc(&t->d_th, 8)); ADAS_CUDA(cudaMalloc(&t->d_v, wc * 8)); ADAS_CUDA(cudaMalloc(&t->d_mv, wc * 8));
        ADAS_CUDA(cudaMalloc(&t->d_wi, wc * 12)); ADAS_CUDA(cudaMalloc(&t->d_meta, 32)); ADAS_CUDA(cudaMalloc(&t->d_co, 16));
        ADAS_CUDA(cudaMalloc(&t->d_u, wc * 8));
        t->cap_ws = wc;
        ADAS_CUDA(cudaHostAlloc(&t->h_done, 64, cudaHostAllocMapped));
        *t->h_done = 0;
        ADAS_CUDA(cudaHostGetDevicePointer(&t->h_done_dev, t->h_done, 0));
    }
    if (nb > t->cap_boxes || nc > t->cap_cost) {
        cudaFree(t->d_a); cudaFree(t->d_b); cudaFree(t->d_s); cudaFree(t->d_c); cudaFree(t->d_x); cudaFree(t->d_y);
        t->cap_boxes = std::max<size_t>(256, nb * 2); t->cap_cost = std::max<size_t>(65536, nc * 2);
        ADAS_CUDA(cudaMalloc(&t->d_a, t->cap_boxes * 32)); ADAS_CUDA(cudaMalloc(&t->d_b, t->cap_boxes * 32)); ADAS_CUDA(cudaMalloc(&t->d_s, t->cap_boxes * 8));
        ADAS_CUDA(cudaMalloc(&t->d_c, t->cap_cost * 8)); ADAS_CUDA(cudaMalloc(&t->d_x, t->cap_boxes * 4)); ADAS_CUDA(cudaMalloc(&t->d_y, t->cap_boxes * 4));
    }
    return 0;
}

static void hit(adas_tracker* t, Track& tr, const Track& det, std::vector<TrackP>* activated, std::vector<TrackP>* refind, const TrackP& self) {
    double tl[4], z[4];
    det.tlwh(tl);
    xyah_of_tlwh(tl, z);
    const bool was_tracked = tr.state == ST_TRACKED;
    kf_update(tr, z);
    if (was_tracked) { tr.tracklet_len += 1; det.tlbr(tr.det_tlbr); tr.traj_frame = t->frame_id; } else tr.tracklet_len = 0;
    tr.frame = t->frame_id; tr.state = ST_TRACKED; tr.activated = true; tr.score = det.score;
    tr.vote(det.cls);
    (was_tracked ? activated : refind)->push_back(self);
}

static std::vector<TrackP> joint(const std::vector<TrackP>& a, const std::vector<TrackP>& b) {   // utils.py:9-30
    std::vector<TrackP> out;
    std::vector<int> seen;
    for (const auto* l : {&a, &b})
        for (const auto& x : *l)
            if (std::find(seen.begin(), seen.end(), x->id) == seen.end()) { seen.push_back(x->id); out.push_back(x); }
    return out;
}
static std::vector<TrackP> sub(const std::vector<TrackP>& a, const std::vector<TrackP>& b) {     // utils.py:33-51 (dict: last duplicate wins, first position kept)
    std::vector<TrackP> uniq;
    for (const auto& x : a) {
        bool rep = false;
        for (auto& u : uniq) if (u->id == x->id) { u = x; rep = true; break; }
        if (!rep) uniq.push_back(x);
    }
    std::vector<TrackP> out;
    for (const auto& x : uniq) {
        bool drop = false;
        for (const auto& y : b) if (y->id == x->id) { drop = true; break; }
        if (!drop) out.push_back(x);
    }
    return out;
}

static void fill_out(const Track& s, adas_track* o) {
    o->track_id = s.id; o->state = s.state; o->is_activated = s.activated ? 1 : 0; o->class_id = s.cls; o->score = s.score;
    o->start_frame = s.start; o->frame_id = s.frame; o->tracklet_len = s.tracklet_len;
    s.tlwh(o->tlwh);
    if (s.has_kf) memcpy(o->mean, s.mean, 64); else memset(o->mean, 0, 64);
    memcpy(o->det_tlbr, s.det_tlbr, 32); o->traj_frame = s.traj_frame; o->pad2 = 0;
    o->pad = g_track_count.load();          // BaseTrack._count when this record was written (the "count" of get_track_message)
}

}  // namespace adas

namespace adas {
// scratch of the fused association, sized for this frame (called before any tracker state is touched)
static int assoc3_prepare(adas_tracker* t, int P, int U, int D, int D2) {
    if (ensure_scratch(t, 1, 1)) return 1;
    // column scratch of the largest stage: stage 1 is P x (D + P), stage 2 R x (D2 + R) with R <= P, stage 3 U x (D + U)
    const size_t ws = (size_t)std::max({P + D, P + D2, U + D}) + 1;
    if (ws > t->cap_ws) {
        cudaFree(t->d_v); cudaFree(t->d_mv); cudaFree(t->d_wi); cudaFree(t->d_u);
        t->d_v = t->d_mv = t->d_u = nullptr; t->d_wi = nullptr; t->cap_ws = 0;
        const size_t wc = ws * 2;
        ADAS_CUDA(cudaMalloc(&t->d_v, wc * 8)); ADAS_CUDA(cudaMalloc(&t->d_mv, wc * 8));
        ADAS_CUDA(cudaMalloc(&t->d_wi, wc * 12)); ADAS_CUDA(cudaMalloc(&t->d_u, wc * 8));
        t->cap_ws = wc;
    }
    const size_t mr = (size_t)std::max(P, U), mc = (size_t)std::max(D, D2);
    const size_t n_in = 5 + (size_t)P * 5 + (size_t)U * 4 + (size_t)D * 5 + (size_t)D2 * 4, n_out = (size_t)2 * P + U + D + 4;
    const size_t n_cost = mr * mc + (size_t)D * 5 + (size_t)P * 4 + 8, n_lists = (size_t)P + D + mr + mc + 8;
    if (n_in > t->cap3_in) {
        if (t->h3_in) cudaFreeHost(t->h3_in);
        cudaFree(t->d3_in);
        t->cap3_in = std::max<size_t>(4096, n_in * 2);
        ADAS_CUDA(cudaHostAlloc(&t->h3_in, t->cap3_in * 8, cudaHostAllocMapped));
        ADAS_CUDA(cudaHostGetDevicePointer(&t->h3_in_dev, t->h3_in, 0));
        ADAS_CUDA(cudaMalloc(&t->d3_in, t->cap3_in * 8));
    }
    if (n_out > t->cap3_out) {
        if (t->h3_out) cudaFreeHost(t->h3_out);
        cudaFree(t->d3_out);
        t->cap3_out = std::max<size_t>(4096, n_out * 2);
        ADAS_CUDA(cudaHostAlloc(&t->h3_out, t->cap3_out * 4, cudaHostAllocMapped));
        ADAS_CUDA(cudaHostGetDevicePointer(&t->h3_out_dev, t->h3_out, 0));
        ADAS_CUDA(cudaMalloc(&t->d3_out, t->cap3_out * 4));
    }
    if (n_cost > t->cap3_cost) { cudaFree(t->d3_cost); t->cap3_cost = std::max<size_t>(65536, n_cost * 2); ADAS_CUDA(cudaMalloc(&t->d3_cost, t->cap3_cost * 8)); }
    if (n_lists > t->cap3_lists) { cudaFree(t->d3_lists); t->cap3_lists = std::max<size_t>(4096, n_lists * 2); ADAS_CUDA(cudaMalloc(&t->d3_lists, t->cap3_lists * 4)); }
    return 0;
}

// the three association stages of one frame: one launch (track.cu assoc3_kernel) that reads and writes mapped host memory
static int assoc3_run(adas_tracker* t, const std::vector<TrackP>& pool, const std::vector<TrackP>& unconf, const std::vector<TrackP>& dets,
                      const std::vector<TrackP>& dets2, bool need_dev, std::vector<int32_t>* m1, std::vector<int32_t>* m2, std::vector<int32_t>* m3,
                      std::vector<int32_t>* free3) {
    const int P = (int)pool.size(), U = (int)unconf.size(), D = (int)dets.size(), D2 = (int)dets2.size();
    m1->assign(P, -1); m2->assign(P, -2); m3->assign(U, -1); free3->assign(D, 1);
    if (!need_dev) {
        // nothing to match against (matching.py:21-22): every Tracked pool row goes through stage 2 unmatched, every detection stays free
        for (int i = 0; i < P; ++i) if (pool[i]->state == ST_TRACKED) (*m2)[i] = -1;
        return 0;
    }
    double* h = t->h3_in;
    h[0] = P; h[1] = U; h[2] = D; h[3] = D2; h[4] = t->match_thresh;
    double* q = h + 5;
    for (int i = 0; i < P; ++i, q += 4) pool[i]->tlbr(q);
    for (int i = 0; i < P; ++i) *q++ = pool[i]->state == ST_TRACKED ? 1.0 : 0.0;
    for (int i = 0; i < U; ++i, q += 4) unconf[i]->tlbr(q);
    for (int j = 0; j < D; ++j, q += 4) dets[j]->tlbr(q);
    for (int j = 0; j < D; ++j) *q++ = dets[j]->score;
    for (int j = 0; j < D2; ++j, q += 4) dets2[j]->tlbr(q);
    const size_t n_in = (size_t)(q - h), n_out = (size_t)2 * P + U + D;
    // one launch, no copies, no stream synchronisation: the kernel pulls `h` and pushes the result through mapped host memory and
    // publishes this frame's sequence number last; the host spins on it (and asks the stream now and then, so that a failed launch
    // or a device fault ends the wait with an error instead of a hang)
    const int32_t seq = ++t->seq;
    const uint64_t w0 = now_ns();
    if (launch_assoc3(t->h3_in_dev, (int)n_in, t->d3_in, t->h3_out_dev, (int)n_out, t->d3_out, t->h_done_dev, seq, t->d3_cost, t->d_v, t->d_mv, t->d_wi,
                      (int)t->cap_ws, t->d3_lists, t->d_u, t->st)) return 1;
    {
        volatile int32_t* done = t->h_done;
        uint32_t spins = 0;
        while (*done != seq) {
            if ((++spins & 0xfffu) == 0) {
                const cudaError_t q = cudaStreamQuery(t->st);
                if (q == cudaSuccess) { ADAS_CHECK(*done == seq, "association kernel finished without publishing its result"); break; }
                ADAS_CHECK(q == cudaErrorNotReady, "association kernel failed: %s", cudaGetErrorString(q));
            }
#if defined(__x86_64__) || defined(__i386__)
            __builtin_ia32_pause();
#endif
        }
        std::atomic_thread_fence(std::memory_order_acquire);
    }
    t->st_wait_ns += now_ns() - w0; t->st_launches += 1;
    const int32_t* o = t->h3_out;
    for (int i = 0; i < P; ++i) (*m1)[i] = o[i];
    for (int i = 0; i < P; ++i) (*m2)[i] = o[P + i];
    for (int k = 0; k < U; ++k) (*m3)[k] = o[2 * P + k];
    for (int j = 0; j < D; ++j) (*free3)[j] = o[2 * P + U + j];
    return 0;
}
}  // namespace adas

extern "C" {

int adas_tracker_create(int device, double track_thresh, int track_buffer, double match_thresh, int frame_rate, adas_tracker** out) {
    ADAS_CHECK(out != nullptr, "adas_tracker_create: null argument");
    adas_tracker* t = new adas_tracker();
    t->device = device; t->track_thresh = track_thresh; t->match_thresh = match_thresh; t->det_thresh = track_thresh + 0.1;
    t->max_time_lost = (int)((double)frame_rate / 30.0 * track_buffer);
    *out = t;
    return 0;
}

int adas_tracker_destroy(adas_tracker* t) {
    if (!t) return 0;
    cudaSetDevice(t->device);
    cudaFree(t->d_a); cudaFree(t->d_b); cudaFree(t->d_s); cudaFree(t->d_c); cudaFree(t->d_x); cudaFree(t->d_y); cudaFree(t->d_th); cudaFree(t->d_v);
    cudaFree(t->d_mv); cudaFree(t->d_wi); cudaFree(t->d_meta); cudaFree(t->d_co);
    if (t->h3_in) cudaFreeHost(t->h3_in);
    if (t->h3_out) cudaFreeHost(t->h3_out);
    if (t->h_done) cudaFreeHost(t->h_done);
    cudaFree(t->d_u);
    cudaFree(t->d3_in); cudaFree(t->d3_out); cudaFree(t->d3_cost); cudaFree(t->d3_lists);
    if (t->st) cudaStreamDestroy(t->st);
    delete t;
    return 0;
}

int adas_tracker_reset(adas_tracker* t) {          // BYTETracker.reset, byteTracker.py:187-200 (also BaseTrack.reset_counter)
    t->frame_id = 0; t->tracked.clear(); t->lost.clear(); t->removed.clear();
    g_track_count.store(0);
    return 0;
}

static int update_one(adas_tracker* t, int n, const double* boxes_xyxy, const double* scores, const int32_t* class_ids, int max_out,
                      adas_track* out, int* n_out) {
    std::vector<TrackP> activated, refind, lost_now, removed_now, dets, dets2;
    for (int i = 0; i < n; ++i) {
        const double s = scores[i];
        const bool hi = s > t->track_thresh, lo = (s > 0.1) && (s < t->track_thresh);
        if (!hi && !lo) continue;
        TrackP d = std::make_shared<Track>();
        d->tlwh0[0] = boxes_xyxy[i * 4]; d->tlwh0[1] = boxes_xyxy[i * 4 + 1];
        d->tlwh0[2] = boxes_xyxy[i * 4 + 2] - boxes_xyxy[i * 4]; d->tlwh0[3] = boxes_xyxy[i * 4 + 3] - boxes_xyxy[i * 4 + 1];
        d->score = s; d->cls = class_ids[i]; d->votes.push_back({class_ids[i], 1});
        (hi ? dets : dets2).push_back(d);
    }
    std::vector<TrackP> unconfirmed, confirmed;
    for (auto& x : t->tracked) (x->activated ? confirmed : unconfirmed).push_back(x);
    std::vector<TrackP> pool = joint(confirmed, t->lost);
    // the association has no size limit (its scratch grows with the frame, like the reference's); scratch is allocated BEFORE any
    // state is touched, so a failed frame leaves the tracker exactly as it was
    const int P = (int)pool.size(), U = (int)unconfirmed.size(), D = (int)dets.size(), D2 = (int)dets2.size();
    std::vector<int32_t> m1, m2, m3, free3;
    const bool need_dev = (P > 0 || U > 0) && (D > 0 || D2 > 0);
    if (need_dev && assoc3_prepare(t, P, U, D, D2)) return 1;
    t->frame_id += 1;
    for (auto& x : pool) kf_predict(*x);
    if (assoc3_run(t, pool, unconfirmed, dets, dets2, need_dev, &m1, &m2, &m3, &free3)) { t->frame_id -= 1; return 1; }
    // stage 1: confirmed + lost vs high-score detections, fused cost
    for (int i = 0; i < P; ++i) if (m1[i] >= 0) hit(t, *pool[i], *dets[m1[i]], &activated, &refind, pool[i]);
    // stage 2: still-tracked leftovers vs low-score detections, plain IoU (m2 == -2: the row was not part of stage 2)
    for (int i = 0; i < P; ++i) if (m2[i] >= 0) hit(t, *pool[i], *dets2[m2[i]], &activated, &refind, pool[i]);
    for (int i = 0; i < P; ++i) if (m2[i] == -1 && pool[i]->state != ST_LOST) { pool[i]->state = ST_LOST; lost_now.push_back(pool[i]); }
    // stage 3: unconfirmed vs leftover high detections, fused cost
    for (int k = 0; k < U; ++k) if (m3[k] >= 0) hit(t, *unconfirmed[k], *dets[m3[k]], &activated, &activated, unconfirmed[k]);
    for (int k = 0; k < U; ++k) if (m3[k] < 0) { unconfirmed[k]->state = ST_REMOVED; removed_now.push_back(unconfirmed[k]); }
    // births
    std::vector<TrackP>& left = dets;
    for (int j = 0; j < D; ++j) {
        if (!free3[j]) continue;
        Track& d = *left[j];
        if (d.score < t->det_thresh) continue;
        d.id = g_track_count.fetch_add(1) + 1;
        kf_initiate(d);
        d.tracklet_len = 0; d.state = ST_TRACKED; d.activated = (t->frame_id == 1);
        d.frame = d.start = t->frame_id;
        activated.push_back(left[j]);
    }
    // ageing and list maintenance (byteTracker.py:170-183)
    for (auto& x : t->lost) if (t->frame_id - x->frame > t->max_time_lost) { x->state = ST_REMOVED; removed_now.push_back(x); }
    std::vector<TrackP> keep;
    for (auto& x : t->tracked) if (x->state == ST_TRACKED) keep.push_back(x);
    t->tracked = joint(joint(keep, activated), refind);
    t->lost = sub(t->lost, t->tracked);
    t->lost.insert(t->lost.end(), lost_now.begin(), lost_now.end());
    t->lost = sub(t->lost, t->removed);
    t->removed.insert(t->removed.end(), removed_now.begin(), removed_now.end());
    {   // remove_duplicate_stracks, utils.py:54-69
        const size_t na = t->tracked.size(), nb = t->lost.size();
        std::vector<char> da(na, 0), db(nb, 0);
        std::vector<double> ba(na * 4), bb(nb * 4);
        for (size_t i = 0; i < na; ++i) t->tracked[i]->tlbr(&ba[i * 4]);
        for (size_t j = 0; j < nb; ++j) t->lost[j]->tlbr(&bb[j * 4]);
        for (size_t i = 0; i < na; ++i)
            for (size_t j = 0; j < nb; ++j)
                if (iou_dist(&ba[i * 4], &bb[j * 4]) < 0.15) {
                    const int ta = t->tracked[i]->frame - t->tracked[i]->start, tb = t->lost[j]->frame - t->lost[j]->start;
                    if (ta > tb) db[j] = 1; else da[i] = 1;
                }
        std::vector<TrackP> ra, rb;
        for (size_t i = 0; i < na; ++i) if (!da[i]) ra.push_back(t->tracked[i]);
        for (size_t j = 0; j < nb; ++j) if (!db[j]) rb.push_back(t->lost[j]);
        t->tracked.swap(ra); t->lost.swap(rb);
    }
    // keep `removed` bounded by trimming its oldest entries, but never this frame's: a lost track that aged out in this frame is still in
    // `lost` until the next frame's sub(lost, removed) drops it
    if (t->removed.size() > 4096)
        t->removed.erase(t->removed.begin(), t->removed.begin() + std::min<size_t>(2048, t->removed.size() - removed_now.size()));
    int k = 0;
    for (auto& x : t->tracked) { if (out && k < max_out) fill_out(*x, &out[k]); ++k; }
    if (n_out) *n_out = k;
    return 0;
}

int adas_tracker_update(adas_tracker* t, int n, const double* boxes_xyxy, const double* scores, const int32_t* class_ids, int max_out,
                        adas_track* out, int* n_out) {
    ADAS_CHECK(t != nullptr && n >= 0, "adas_tracker_update: bad arguments");
    ADAS_CUDA(cudaSetDevice(t->device));
    return update_one(t, n, boxes_xyxy, scores, class_ids, max_out, out, n_out);
}

int adas_tracker_update_batch(adas_tracker* t, int n_frames, const int32_t* counts, const double* boxes_xyxy, const double* scores,
                              const int32_t* class_ids, int max_out, adas_track* out, int32_t* n_out) {
    ADAS_CHECK(t != nullptr && n_frames >= 0 && counts != nullptr && n_out != nullptr, "adas_tracker_update_batch: bad arguments");
    ADAS_CUDA(cudaSetDevice(t->device));
    adas::NvtxRange nv("adas_tracker_update_batch");
    size_t off = 0;
    const uint64_t t0 = adas::now_ns();
    for (int f = 0; f < n_frames; ++f) {
        int k = 0;
        if (update_one(t, counts[f], boxes_xyxy + off * 4, scores + off, class_ids + off, max_out, out ? out + (size_t)f * max_out : nullptr, &k)) return 1;
        n_out[f] = k;
        off += (size_t)counts[f];
    }
    t->st_total_ns += adas::now_ns() - t0; t->st_frames += (uint64_t)n_frames;
    return 0;
}

int adas_tracker_stats(adas_tracker* t, double* out4) {
    ADAS_CHECK(t != nullptr && out4 != nullptr, "adas_tracker_stats: null argument");
    out4[0] = (double)t->st_frames; out4[1] = (double)t->st_total_ns * 1e-6; out4[2] = (double)t->st_wait_ns * 1e-6; out4[3] = (double)t->st_launches;
    return 0;
}

int adas_tracker_get(adas_tracker* t, int which, int max_out, adas_track* out, int* n_out) {
    const std::vector<TrackP>& l = which == 0 ? t->tracked : (which == 1 ? t->lost : t->removed);
    int k = 0;
    for (auto& x : l) { if (out && k < max_out) fill_out(*x, &out[k]); ++k; }
    if (n_out) *n_out = k;
    return 0;
}

int adas_tracker_count(void) { return g_track_count.load(); }

}  // extern "C"
