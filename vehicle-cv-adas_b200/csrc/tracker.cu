// tracker.cu -- native ByteTrack state machine (host C++) driving the device association kernels of track.cu.
//
// Replaces the per-frame Python of ObjectTracker/byteTrack/byteTracker.py:62-185 (three association stages, births,
// ageing, list maintenance), dtypes/strack.py (track records, class vote, conversions), dtypes/kalman_filter.py:55-226
// (constant-velocity filter, float64) and utils.py:9-69 (joint / sub / duplicate removal).  The IoU cost matrices and
// the exact assignment of all three stages of a frame run on the device in ONE launch (track.cu assoc3_kernel: one upload, one
// launch, one download, one synchronisation per frame); the 8x8 float64 Kalman algebra and the list bookkeeping are sequential
// per stream and stay on the host.  adas_tracker_update_batch takes all frames of a pipeline step in one call;
// adas_tracker_update_multi advances several trackers (one per camera) a frame at a time with ONE association launch per frame for
// all of them: each frame is split into prepare (detections, Kalman predict, packing the launch's input), the launch, and apply
// (matches, births, ageing, list maintenance) in tracker order.
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
    // the frame between prepare and apply: its detections by score, the association's rows, and this tracker's problem in the launch
    std::vector<TrackP> dets, dets2, unconfirmed, pool;
    bool need_dev = false;
    Assoc3Problem prob{};
    // fused three-stage association of the calls this tracker leads (alone, or first of adas_tracker_update_multi): one launch and
    // one synchronisation per frame for every tracker of the call.  Grown on demand, kept for reuse.
    cudaStream_t st = nullptr;
    Assoc3Problem* h_probs = nullptr; double* h_in = nullptr; int32_t* h_out = nullptr;   // pinned + mapped: the kernel reads / writes
    int32_t* h_done = nullptr; int32_t seq = 0;                                            // them over the link; h_done: completion word
    Assoc3Buffers dev{};                                      // device-side addresses of the above, device copies and scratch
    size_t cap_probs = 0, cap_in = 0, cap_out = 0, cap_cost = 0, cap_lists = 0, cap_ws = 0;
    // wall-clock accounting of the update path (adas_tracker_stats): frames, total ns, ns between launch and result, launches
    uint64_t st_frames = 0, st_total_ns = 0, st_wait_ns = 0, st_launches = 0;
};

namespace adas {

// mapped pinned host buffer (and, with `dev_copy`, a device buffer of the same size) of at least `need` elements
template <typename T>
static int grow_mapped(T** host, const T** host_dev, T** dev_copy, size_t* cap, size_t need, size_t min_cap) {
    if (need <= *cap) return 0;
    if (*host) cudaFreeHost(*host);
    if (dev_copy) cudaFree(*dev_copy);
    *host = nullptr; *cap = 0;
    const size_t c = std::max(min_cap, need * 2);
    ADAS_CUDA(cudaHostAlloc((void**)host, c * sizeof(T), cudaHostAllocMapped));
    ADAS_CUDA(cudaHostGetDevicePointer((void**)host_dev, *host, 0));
    if (dev_copy) ADAS_CUDA(cudaMalloc((void**)dev_copy, c * sizeof(T)));
    *cap = c;
    return 0;
}

// launch buffers of `problems` problems with the given total sizes; called before any tracker state is touched
static int assoc3_reserve(adas_tracker* t, size_t problems, size_t n_in, size_t n_out, size_t n_cost, size_t n_lists, size_t n_ws) {
    Assoc3Buffers& b = t->dev;
    if (t->st == nullptr) {
        // the association kernel is tiny and on the host's critical path: highest priority, so it is scheduled as soon as any
        // CTA slot frees up between the detectors' persistent conv kernels
        int prio_lo = 0, prio_hi = 0;
        cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
        ADAS_CUDA(cudaStreamCreateWithPriority(&t->st, cudaStreamNonBlocking, prio_hi));
        ADAS_CUDA(cudaHostAlloc(&t->h_done, 64, cudaHostAllocMapped));
        *t->h_done = 0;
        ADAS_CUDA(cudaHostGetDevicePointer((void**)&b.done_host, t->h_done, 0));
        ADAS_CUDA(cudaMalloc(&b.finished, sizeof(unsigned int)));
        ADAS_CUDA(cudaMemsetAsync(b.finished, 0, sizeof(unsigned int), t->st));
    }
    if (grow_mapped(&t->h_probs, &b.probs, (Assoc3Problem**)nullptr, &t->cap_probs, problems, 16)) return 1;
    if (grow_mapped(&t->h_in, &b.in_host, &b.in, &t->cap_in, n_in, 4096)) return 1;
    if (grow_mapped(&t->h_out, (const int32_t**)&b.out_host, &b.out, &t->cap_out, n_out, 4096)) return 1;
    if (n_cost > t->cap_cost) {
        cudaFree(b.cost); b.cost = nullptr; t->cap_cost = 0;
        const size_t c = std::max<size_t>(65536, n_cost * 2);
        ADAS_CUDA(cudaMalloc(&b.cost, c * 8));
        t->cap_cost = c;
    }
    if (n_lists > t->cap_lists) {
        cudaFree(b.lists); b.lists = nullptr; t->cap_lists = 0;
        const size_t c = std::max<size_t>(4096, n_lists * 2);
        ADAS_CUDA(cudaMalloc(&b.lists, c * 4));
        t->cap_lists = c;
    }
    if (n_ws > t->cap_ws) {
        cudaFree(b.v); cudaFree(b.minv); cudaFree(b.u); cudaFree(b.wi);
        b.v = b.minv = b.u = nullptr; b.wi = nullptr; t->cap_ws = 0;
        const size_t wc = std::max<size_t>(4096, n_ws * 2);
        ADAS_CUDA(cudaMalloc(&b.v, wc * 8)); ADAS_CUDA(cudaMalloc(&b.minv, wc * 8)); ADAS_CUDA(cudaMalloc(&b.u, wc * 8)); ADAS_CUDA(cudaMalloc(&b.wi, wc * 12));
        t->cap_ws = wc;
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
// sizes of one problem of the fused association; the column scratch covers the largest stage: stage 1 is P x (D + P), stage 2
// R x (D2 + R) with R <= P, stage 3 U x (D + U)
static void assoc3_sizes(Assoc3Problem* p, int P, int U, int D, int D2, size_t* n_cost, size_t* n_lists) {
    const size_t mr = (size_t)std::max(P, U), mc = (size_t)std::max(D, D2);
    p->n_in = 5 + (int64_t)P * 5 + (int64_t)U * 4 + (int64_t)D * 5 + (int64_t)D2 * 4;
    p->n_out = (int64_t)2 * P + U + D;
    p->ws = (int64_t)std::max({P + D, P + D2, U + D}) + 1;
    *n_cost = mr * mc + (size_t)D * 5 + (size_t)P * 4 + 8;
    *n_lists = (size_t)P + D + mr + mc + 8;
}

// first half of a frame, without touching the tracker's state: the detections by score, the association's rows and whether the
// frame needs the device (matching.py:21-22: no association when either side is empty)
static void frame_classify(adas_tracker* t, int n, const double* boxes_xyxy, const double* scores, const int32_t* class_ids) {
    t->dets.clear(); t->dets2.clear(); t->unconfirmed.clear(); t->pool.clear();
    for (int i = 0; i < n; ++i) {
        const double s = scores[i];
        const bool hi = s > t->track_thresh, lo = (s > 0.1) && (s < t->track_thresh);
        if (!hi && !lo) continue;
        TrackP d = std::make_shared<Track>();
        d->tlwh0[0] = boxes_xyxy[i * 4]; d->tlwh0[1] = boxes_xyxy[i * 4 + 1];
        d->tlwh0[2] = boxes_xyxy[i * 4 + 2] - boxes_xyxy[i * 4]; d->tlwh0[3] = boxes_xyxy[i * 4 + 3] - boxes_xyxy[i * 4 + 1];
        d->score = s; d->cls = class_ids[i]; d->votes.push_back({class_ids[i], 1});
        (hi ? t->dets : t->dets2).push_back(d);
    }
    std::vector<TrackP> confirmed;
    for (auto& x : t->tracked) (x->activated ? confirmed : t->unconfirmed).push_back(x);
    t->pool = joint(confirmed, t->lost);
    t->need_dev = (!t->pool.empty() || !t->unconfirmed.empty()) && (!t->dets.empty() || !t->dets2.empty());
}

// prepare: the frame starts, the pool is predicted and, when the frame needs the device, its problem is packed at prob.in_off
static void frame_prepare(adas_tracker* t, double* in) {
    t->frame_id += 1;
    for (auto& x : t->pool) kf_predict(*x);
    if (!t->need_dev) return;
    const int P = (int)t->pool.size(), U = (int)t->unconfirmed.size(), D = (int)t->dets.size(), D2 = (int)t->dets2.size();
    double* h = in + t->prob.in_off;
    h[0] = P; h[1] = U; h[2] = D; h[3] = D2; h[4] = t->match_thresh;
    double* q = h + 5;
    for (int i = 0; i < P; ++i, q += 4) t->pool[i]->tlbr(q);
    for (int i = 0; i < P; ++i) *q++ = t->pool[i]->state == ST_TRACKED ? 1.0 : 0.0;
    for (int i = 0; i < U; ++i, q += 4) t->unconfirmed[i]->tlbr(q);
    for (int j = 0; j < D; ++j, q += 4) t->dets[j]->tlbr(q);
    for (int j = 0; j < D; ++j) *q++ = t->dets[j]->score;
    for (int j = 0; j < D2; ++j, q += 4) t->dets2[j]->tlbr(q);
}

// apply: matches of the three stages (the kernel's output at prob.out_off), births, ageing and list maintenance
// (byteTracker.py:100-185), then the tracked list into out[0, max_out)
static void frame_apply(adas_tracker* t, const int32_t* out_all, int max_out, adas_track* out, int32_t* n_out) {
    std::vector<TrackP>& pool = t->pool;
    std::vector<TrackP>& unconfirmed = t->unconfirmed;
    std::vector<TrackP>& dets = t->dets;
    std::vector<TrackP>& dets2 = t->dets2;
    const int P = (int)pool.size(), U = (int)unconfirmed.size(), D = (int)dets.size();
    std::vector<int32_t> m1(P, -1), m2(P, -2), m3(U, -1), free3(D, 1);
    if (t->need_dev) {
        const int32_t* o = out_all + t->prob.out_off;
        for (int i = 0; i < P; ++i) m1[i] = o[i];
        for (int i = 0; i < P; ++i) m2[i] = o[P + i];
        for (int k = 0; k < U; ++k) m3[k] = o[2 * P + k];
        for (int j = 0; j < D; ++j) free3[j] = o[2 * P + U + j];
    } else {
        // nothing to match against (matching.py:21-22): every Tracked pool row goes through stage 2 unmatched, every detection stays free
        for (int i = 0; i < P; ++i) if (pool[i]->state == ST_TRACKED) m2[i] = -1;
    }
    std::vector<TrackP> activated, refind, lost_now, removed_now;
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
    t->dets.clear(); t->dets2.clear(); t->unconfirmed.clear(); t->pool.clear();
}

// one tracker's detections of one frame and where its records go
struct CamFrame {
    int n;
    const double* boxes_xyxy;
    const double* scores;
    const int32_t* class_ids;
    adas_track* out;
    int32_t* n_out;
};

// spin on the launch's completion word (asking the stream now and then, so that a failed launch or a device fault ends the wait with an
// error instead of a hang)
static int assoc3_wait(adas_tracker* t, int32_t seq) {
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
    return 0;
}

// One frame of k distinct trackers on one device: prepare every tracker, ONE association launch (on ts[0]'s stream and buffers) for
// all that need the device, one wait, then apply in tracker order -- births take track ids in that order, so the result is exactly
// that of updating the trackers one after another.  The launch's buffers are sized before any tracker state is touched, so a frame
// that fails there leaves every tracker exactly as it was.
static int step_frame(adas_tracker* const* ts, int k, const CamFrame* cf, int max_out) {
    adas_tracker* lead = ts[0];
    int problems = 0;
    size_t n_in = 0, n_out = 0, n_cost = 0, n_lists = 0, n_ws = 0;
    for (int c = 0; c < k; ++c) {
        adas_tracker* t = ts[c];
        frame_classify(t, cf[c].n, cf[c].boxes_xyxy, cf[c].scores, cf[c].class_ids);
        if (!t->need_dev) continue;
        Assoc3Problem& p = t->prob;
        size_t nc = 0, nl = 0;
        assoc3_sizes(&p, (int)t->pool.size(), (int)t->unconfirmed.size(), (int)t->dets.size(), (int)t->dets2.size(), &nc, &nl);
        p.in_off = (int64_t)n_in; p.out_off = (int64_t)n_out; p.cost_off = (int64_t)n_cost; p.lists_off = (int64_t)n_lists; p.ws_off = (int64_t)n_ws;
        n_in += (size_t)p.n_in; n_out += (size_t)p.n_out; n_cost += nc; n_lists += nl; n_ws += (size_t)p.ws;
        ++problems;
    }
    if (problems > 0 && assoc3_reserve(lead, (size_t)problems, n_in, n_out, n_cost, n_lists, n_ws)) return 1;
    for (int c = 0, q = 0; c < k; ++c) {
        frame_prepare(ts[c], lead->h_in);
        if (ts[c]->need_dev) lead->h_probs[q++] = ts[c]->prob;
    }
    if (problems > 0) {
        // one launch, no copies, no stream synchronisation: the kernel pulls the inputs and pushes the results through mapped host
        // memory and publishes this frame's sequence number last
        const int32_t seq = ++lead->seq;
        const uint64_t w0 = now_ns();
        if (launch_assoc3(problems, lead->dev, seq, lead->st) || assoc3_wait(lead, seq)) {
            for (int c = 0; c < k; ++c) ts[c]->frame_id -= 1;
            return 1;
        }
        const uint64_t w = now_ns() - w0;
        for (int c = 0; c < k; ++c) if (ts[c]->need_dev) { ts[c]->st_wait_ns += w; ts[c]->st_launches += 1; }
    }
    for (int c = 0; c < k; ++c) frame_apply(ts[c], lead->h_out, max_out, cf[c].out, cf[c].n_out);
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
    if (t->st) {                                   // the stream is created first: a tracker without one holds no device resource
        cudaSetDevice(t->device);
        const Assoc3Buffers& b = t->dev;
        cudaFree(b.in); cudaFree(b.out); cudaFree(b.cost); cudaFree(b.lists); cudaFree(b.v); cudaFree(b.minv); cudaFree(b.u); cudaFree(b.wi);
        cudaFree(b.finished);
        if (t->h_probs) cudaFreeHost(t->h_probs);
        if (t->h_in) cudaFreeHost(t->h_in);
        if (t->h_out) cudaFreeHost(t->h_out);
        if (t->h_done) cudaFreeHost(t->h_done);
        cudaStreamDestroy(t->st);
    }
    delete t;
    return 0;
}

int adas_tracker_reset(adas_tracker* t) {          // BYTETracker.reset, byteTracker.py:187-200 (also BaseTrack.reset_counter)
    t->frame_id = 0; t->tracked.clear(); t->lost.clear(); t->removed.clear();
    g_track_count.store(0);
    return 0;
}

int adas_tracker_update(adas_tracker* t, int n, const double* boxes_xyxy, const double* scores, const int32_t* class_ids, int max_out,
                        adas_track* out, int* n_out) {
    ADAS_CHECK(t != nullptr && n >= 0, "adas_tracker_update: bad arguments");
    ADAS_CUDA(cudaSetDevice(t->device));
    const adas::CamFrame cf{n, boxes_xyxy, scores, class_ids, out, n_out};
    return adas::step_frame(&t, 1, &cf, max_out);
}

int adas_tracker_update_batch(adas_tracker* t, int n_frames, const int32_t* counts, const double* boxes_xyxy, const double* scores,
                              const int32_t* class_ids, int max_out, adas_track* out, int32_t* n_out) {
    ADAS_CHECK(t != nullptr && n_frames >= 0 && counts != nullptr && n_out != nullptr, "adas_tracker_update_batch: bad arguments");
    ADAS_CUDA(cudaSetDevice(t->device));
    adas::NvtxRange nv("adas_tracker_update_batch");
    size_t off = 0;
    const uint64_t t0 = adas::now_ns();
    for (int f = 0; f < n_frames; ++f) {
        const adas::CamFrame cf{counts[f], boxes_xyxy + off * 4, scores + off, class_ids + off, out ? out + (size_t)f * max_out : nullptr, &n_out[f]};
        if (adas::step_frame(&t, 1, &cf, max_out)) return 1;
        off += (size_t)counts[f];
    }
    t->st_total_ns += adas::now_ns() - t0; t->st_frames += (uint64_t)n_frames;
    return 0;
}

int adas_tracker_update_multi(adas_tracker* const* trackers, int k, int n_frames, const int32_t* counts, const double* boxes_xyxy,
                              const double* scores, const int32_t* class_ids, int max_out, adas_track* out, int32_t* n_out) {
    ADAS_CHECK(trackers != nullptr && k >= 1 && n_frames >= 0, "adas_tracker_update_multi: bad arguments (k = %d, n_frames = %d)", k, n_frames);
    ADAS_CHECK(n_frames == 0 || (counts != nullptr && n_out != nullptr), "adas_tracker_update_multi: null counts or n_out");
    for (int c = 0; c < k; ++c) {
        ADAS_CHECK(trackers[c] != nullptr, "adas_tracker_update_multi: tracker %d is null", c);
        for (int c2 = 0; c2 < c; ++c2)
            ADAS_CHECK(trackers[c2] != trackers[c], "adas_tracker_update_multi: tracker %d is also tracker %d", c, c2);
        ADAS_CHECK(trackers[c]->device == trackers[0]->device, "adas_tracker_update_multi: tracker %d is on device %d, tracker 0 on device %d", c,
                   trackers[c]->device, trackers[0]->device);
    }
    size_t total = 0;
    for (size_t i = 0; i < (size_t)n_frames * k; ++i) {
        ADAS_CHECK(counts[i] >= 0, "adas_tracker_update_multi: negative detection count %d (frame %zu, tracker %zu)", counts[i], i / k, i % k);
        total += (size_t)counts[i];
    }
    ADAS_CHECK(total == 0 || (boxes_xyxy != nullptr && scores != nullptr && class_ids != nullptr), "adas_tracker_update_multi: null detections");
    ADAS_CUDA(cudaSetDevice(trackers[0]->device));
    adas::NvtxRange nv("adas_tracker_update_multi");
    std::vector<adas::CamFrame> cf(k);
    size_t off = 0;
    const uint64_t t0 = adas::now_ns();
    for (int f = 0; f < n_frames; ++f) {
        for (int c = 0; c < k; ++c) {
            const size_t i = (size_t)f * k + c;
            cf[c] = adas::CamFrame{counts[i], boxes_xyxy + off * 4, scores + off, class_ids + off, out ? out + i * max_out : nullptr, &n_out[i]};
            off += (size_t)counts[i];
        }
        if (adas::step_frame(trackers, k, cf.data(), max_out)) return 1;
    }
    const uint64_t dt = adas::now_ns() - t0;
    for (int c = 0; c < k; ++c) { trackers[c]->st_total_ns += dt; trackers[c]->st_frames += (uint64_t)n_frames; }
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
