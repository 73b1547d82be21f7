// vo_driver.cpp -- native (C++) lock-step tracking loop over the C ABI: the host side of BASELINE config C5.
//
// CALLER code in the shape of the reference's src/Module/VisualOdometry.cpp:38-107 (AddFrame), :281-302
// (TrackRefFrame), src/Module/LocalMapping.cpp:24-140 (TrackLocalMap: FindCandidates / ProjectMapPoints /
// OptimizeCurrent), VisualOdometry.cpp:182-218 + :304-321 (SetKeyframe / NeedNewKeyFrame) and LocalMapping.cpp:149-172
// (LocalBA -> ba::LocalBAG2O).  It is the same loop as ygz_slam_b200/vo.py (which the tests run against the CPU oracle
// backend for end-to-end parity); this file is that loop without the Python interpreter in the way, so that the
// measured tracked-frames/s reflect the device path and not numpy call overhead.  No image or optimisation
// arithmetic happens here: every numeric step is ONE batched C-ABI call over all streams (ygzb_frames_upload,
// ygzb_sparse_align, ygzb_project_align, ygzb_pose_only, ygzb_detect, ygzb_local_ba).
//
// Input-side simplifications are those of vo.py: ground-truth depth initialises the map points of a key-frame
// (test/test_feature_alignment.cpp:72-85 does the same with TUM depth), no BoW / loop closing.
//
// Build: host C++ only (g++), links libygz_b200.so; see ygz_slam_b200/build.py (libygz_vo.so).
#include <algorithm>
#include <array>
#include <atomic>
#include <bit>
#include <chrono>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/ygz_b200.h"
#include "../../include/ygz_vo.h"
#include "../csrc/se3.cuh"
#include "timed_threads.h"

namespace {

constexpr double FX = 520.9, FY = 521.0, CX = 325.1, CY = 249.7;   // config/default.yaml:32-35 (as Python floats in vo.py): the batch camera
constexpr int W = 640, H = 480;                                    // per-stage path (the resident engine takes the context's size)
constexpr int kLocalKeyframes = 3;                                 // LocalMapping.local_keyframes (default.yaml:68)
constexpr int kSlotsPerStream = kLocalKeyframes + 2;
constexpr int kMinInliers = 30;                                    // vo.keyframe.min_features (default.yaml:66)
constexpr int kSpeculativeFrames = 3;                              // engine: frames tracked ahead once a key-frame may trigger any time
static_assert(sizeof(ygzb_map_point) == 32 && offsetof(ygzb_map_point, pw) == 8, "a map point row is 32 bytes: id, pw[3]");
static_assert(sizeof(ygz_vo_map_update) == 432 && offsetof(ygz_vo_map_update, sequence) == 8 &&
                  offsetof(ygz_vo_map_update, local_frame) == 24 && offsetof(ygz_vo_map_update, n_moved) == 40 &&
                  offsetof(ygz_vo_map_update, T_cw) == 48,
              "ygz_vo_map_update is laid out as include/ygz_vo.h documents");

struct Mat34 {
    double m[12];
};
Mat34 identity() { return Mat34{{1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0}}; }
ygzb::SE3d to_se3(const Mat34& T) { return ygzb::se3_from_mat(T.m); }
Mat34 from_se3(const ygzb::SE3d& s) {
    Mat34 T;
    ygzb::se3_to_mat(s, T.m);
    return T;
}
Mat34 mul(const Mat34& A, const Mat34& B) {  // plain matrix product of [R|t] transforms
    Mat34 C;
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) C.m[4 * r + c] = A.m[4 * r] * B.m[c] + A.m[4 * r + 1] * B.m[4 + c] + A.m[4 * r + 2] * B.m[8 + c];
        C.m[4 * r + 3] = A.m[4 * r] * B.m[3] + A.m[4 * r + 1] * B.m[7] + A.m[4 * r + 2] * B.m[11] + A.m[4 * r + 3];
    }
    return C;
}
Mat34 inv(const Mat34& A) {
    Mat34 C;
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) C.m[4 * r + c] = A.m[4 * c + r];
        C.m[4 * r + 3] = -(A.m[r] * A.m[3] + A.m[4 + r] * A.m[7] + A.m[8 + r] * A.m[11]);
    }
    return C;
}
void se3_log(const Mat34& T, double out[6]) { ygzb::se3_log(to_se3(T), out); }  // [upsilon; omega]

struct Keyframe {
    int slot = 0, frame_id = 0;
    Mat34 T;
    std::vector<double> px;      // 2n full-res pixels of its features
    std::vector<int> level;
    std::vector<double> depth;   // n
    std::vector<double> pw;      // 3n world points
    long mp0 = 0;                // map point ids are [mp0, mp0 + n)
    std::vector<long> obs_id;    // older map points tracked into this frame ...
    std::vector<double> obs_px;  // ... and their measured pixels
    int n() const { return (int)depth.size(); }
};

// the counters of a stream that both loops keep (per-stage Stream, resident EStream)
struct Counters {
    long n_keyframes = 0, n_ba = 0, n_candidates = 0, n_projected = 0, n_inliers = 0;
    long ba_obs = 0, ba_pts = 0, ba_kfs = 0, ba_trials = 0, ba_iters = 0;
    double ba_flops = 0;   // SURVEY 8d model: per LM trial 300 n_obs + sum_j (216 k_j^2 + 108 k_j + 50) + dim^3 / 3
    long n_restarts = 0;   // resident engine: sequences started by ygz_vo_restart (the per-stage driver has none)
    // the 16 stats of the stream (ygz_vo_run, ygz_vo_stream_stats): lost, the counters, restarts, 0...
    void write_stats(bool lost, int64_t* o) const {
        for (int k = 0; k < 16; ++k) o[k] = 0;
        o[0] = lost; o[1] = n_keyframes; o[2] = n_ba; o[3] = n_candidates; o[4] = n_projected; o[5] = n_inliers;
        o[6] = ba_obs; o[7] = ba_pts; o[8] = ba_kfs; o[9] = ba_trials; o[10] = ba_iters; o[11] = (int64_t)ba_flops;
        o[12] = n_restarts;
    }
};

struct Stream : Counters {
    int slot0 = 0;
    std::deque<Keyframe> keyframes;   // at most kLocalKeyframes + 1, the newest is the reference key-frame
    Mat34 T = identity();
    bool has_pose = false, lost = false, has_ref = false, has_last = false;
    int frames_since_kf = 0;
    long next_mp = 0;
    std::vector<long> last_id;
    std::vector<double> last_px;
    int first_local() const { return std::max(0, (int)keyframes.size() - kLocalKeyframes); }
};

struct Params {
    int kf_min_frames;
    double kf_min_rot, kf_min_trans;
    int ref_mode = YGZB_TRACK_REF_KEYFRAME;   // resident engine: what a frame is aligned against (ygzb_tracker_set_reference_mode)
    int min_inliers = kMinInliers;            // resident engine: pose-only inliers below which a stream is lost
    double K[4] = {FX, FY, CX, CY};           // resident engine: the tracker's camera
};

// NeedNewKeyFrame (VisualOdometry.cpp:304-321) of a frame at T, frames_since_kf frames after the key-frame at T_kf
bool need_keyframe(const Params& p, int frames_since_kf, const Mat34& T, const Mat34& T_kf) {
    if (frames_since_kf < p.kf_min_frames) return false;
    double d[6];
    se3_log(mul(T, inv(T_kf)), d);
    const double rot = std::sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]), tr = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    return rot > p.kf_min_rot || tr > p.kf_min_trans;
}

#define CHK(call)                                     \
    do {                                              \
        int _rc = (call);                             \
        if (_rc != YGZB_OK) return _rc;               \
    } while (0)

// wall time per C-ABI stage (printed when YGZ_VO_TIMING is set): where a lock-step frame goes
enum { kTUpload, kTSparse, kTProject, kTPoseOnly, kTDetect, kTLocalBA, kTStages };
std::atomic<long long> g_stage_ns[kTStages];   // summed over the host threads
struct StageTimer {
    int stage;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    explicit StageTimer(int s) : stage(s) {}
    ~StageTimer() {
        g_stage_ns[stage].fetch_add(std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count(),
                                    std::memory_order_relaxed);
    }
};
#define TIMED(stage, call)        \
    do {                          \
        StageTimer _t(stage);     \
        CHK(call);                \
    } while (0)

class Driver {
  public:
    // slot layout: [0, S) = staging slots of the incoming frames (contiguous: one upload per lock-step frame), then a ring
    // of kSlotsPerStream - 1 key-frame slots per stream; a frame that becomes a key-frame is copied device-to-device
    Driver(ygzb_ctx* ctx, ygzb_frames* fr, int n_streams, const Params& p) : ctx_(ctx), fr_(fr), S_(n_streams), prm_(p), st_(n_streams) {
        for (int i = 0; i < S_; ++i) st_[i].slot0 = S_ + i * (kSlotsPerStream - 1);
        int rows = 0, cols = 0;
        ygzb_grid_dims(ctx, &rows, &cols);
        n_cells_ = rows * cols;
    }
    std::vector<Stream>& streams() { return st_; }
    // bytes this driver hands to / reads back from the C ABI (host buffers), counted from the arrays of every call
    long long h2d_image_bytes = 0, h2d_other_bytes = 0, d2h_bytes = 0;

    // one lock-step frame: images[i] = grey frame of stream i, depth[i] = its (static) ground-truth depth map
    int add_frames(const uint8_t* const* images, const double* const* depth, int frame_id) {
        cur_slot_.resize(S_);
        for (int i = 0; i < S_; ++i) cur_slot_[i] = i;
        // one strided copy when the caller's frames are equally spaced in host memory (a stacked [stream][frame] array)
        bool strided = S_ > 1;
        const ptrdiff_t stride = S_ > 1 ? images[1] - images[0] : 0;
        for (int i = 1; i + 1 < S_ && strided; ++i) strided = images[i + 1] - images[i] == stride;
        h2d_image_bytes += (long long)S_ * W * H;
        if (strided && stride >= (ptrdiff_t)W * H) {
            TIMED(kTUpload, ygzb_frames_upload(fr_, 0, S_, images[0], 1, (size_t)stride));
        } else {
            for (int i = 0; i < S_; ++i) TIMED(kTUpload, ygzb_frames_upload(fr_, i, 1, images[i], 1, (size_t)W * H));
        }
        std::vector<int> boot, track;
        for (int i = 0; i < S_; ++i) {
            if (st_[i].lost) continue;
            if (!st_[i].has_ref) boot.push_back(i);
            else track.push_back(i);
        }
        if (!boot.empty()) {
            for (int i : boot) {
                st_[i].T = identity();
                st_[i].has_pose = true;
            }
            CHK(make_keyframes(boot, depth, frame_id, true));
        }
        if (!track.empty()) CHK(track_frames(track, depth, frame_id));
        return YGZB_OK;
    }

  private:
    int next_slot(int i) const {
        const Stream& s = st_[i];
        for (int c = 0; c < kSlotsPerStream - 1; ++c) {
            const int slot = s.slot0 + c;
            bool used = false;
            for (int k = s.first_local(); k < (int)s.keyframes.size(); ++k) used |= s.keyframes[k].slot == slot;
            if (!used) return slot;
        }
        return s.slot0;  // cannot happen: the ring has kLocalKeyframes + 1 slots
    }

    // TrackRefFrame + TrackLocalMap + key-frame decision for the streams in idx
    int track_frames(std::vector<int> idx, const double* const* depth, int frame_id) {
        const int n = (int)idx.size();
        // -- Matcher::SparseImageAlignment(ref, cur) with cur._TCW = ref._TCW (VisualOdometry.cpp:281-302)
        std::vector<int32_t> ref_slot(n), cur_slot(n), offs(n + 1, 0), n_meas(n);
        std::vector<double> px, dep, T_ref(12 * (size_t)n), T_cur(12 * (size_t)n);
        for (int j = 0; j < n; ++j) {
            const Keyframe& kf = st_[idx[j]].keyframes.back();
            ref_slot[j] = kf.slot;
            cur_slot[j] = cur_slot_[idx[j]];
            offs[j + 1] = offs[j] + kf.n();
            px.insert(px.end(), kf.px.begin(), kf.px.end());
            dep.insert(dep.end(), kf.depth.begin(), kf.depth.end());
            std::memcpy(&T_ref[12 * (size_t)j], kf.T.m, sizeof(kf.T.m));
        }
        T_cur = T_ref;
        std::vector<uint8_t> has(px.size() / 2, 1);
        h2d_other_bytes += 8ll * n + 4ll * (n + 1) + 25ll * (long long)has.size() + 192ll * n;
        d2h_bytes += 100ll * n;
        TIMED(kTSparse, ygzb_sparse_align(fr_, n, ref_slot.data(), cur_slot.data(), offs.data(), px.data(), dep.data(), has.data(), T_ref.data(),
                              T_cur.data(), 2, 0, 30, 1e-6, n_meas.data(), nullptr));
        std::vector<int> alive;
        std::vector<Mat34> T_of(S_);
        for (int j = 0; j < n; ++j) {
            Mat34 Tc, Tr;
            std::memcpy(Tc.m, &T_cur[12 * (size_t)j], sizeof(Tc.m));
            std::memcpy(Tr.m, &T_ref[12 * (size_t)j], sizeof(Tr.m));
            double lg[6];
            se3_log(mul(Tc, inv(Tr)), lg);   // Matcher.cpp:482-488: motion norm check
            double nrm = 0;
            for (double v : lg) nrm += v * v;
            if (std::sqrt(nrm) <= 0.2) {
                T_of[idx[j]] = Tc;
                alive.push_back(idx[j]);
            } else {
                st_[idx[j]].lost = true;   // the reference keeps the last pose and reports VO_LOST
            }
        }
        idx = alive;
        if (idx.empty()) return YGZB_OK;

        // -- FindCandidates: project the points of the local key-frames, border 20 (LocalMapping.cpp:47-80), then
        //    ProjectMapPoints: Matcher::FindDirectProjection per candidate (:82-111) as ONE batch.  Poses go in relative
        //    to the reference key-frame (I, T_cur * T_ref^-1): GetWarpAffineMatrix is only correct for an identity
        //    reference pose (Matcher.cpp:425-430, quirk kept in the kernel).
        struct Cand { int stream, kf, n; };
        size_t bound = 0;   // every point of every local key-frame can become a candidate
        for (int i : idx)
            for (int k = st_[i].first_local(); k < (int)st_[i].keyframes.size(); ++k) bound += (size_t)st_[i].keyframes[k].n();
        std::vector<Cand> cand(bound);
        std::vector<int32_t> c_ref_slot(bound), c_cur_slot(bound), c_ref_pose(bound), c_cur_pose(bound);
        const Mat34 eye = identity();
        std::vector<double> poses(eye.m, eye.m + 12), c_ref_px(2 * bound), c_ref_depth(bound), c_cur_px(2 * bound);
        std::vector<uint8_t> c_level(bound);
        std::vector<int> job_begin;
        size_t nc_sz = 0;
        for (int i : idx) {
            Stream& s = st_[i];
            const Mat34& T = T_of[i];
            job_begin.push_back((int)nc_sz);
            const int pose_base = (int)(poses.size() / 12);
            for (int k = s.first_local(); k < (int)s.keyframes.size(); ++k) {
                const Mat34 rel = mul(T, inv(s.keyframes[k].T));
                poses.insert(poses.end(), rel.m, rel.m + 12);
            }
            for (int k = s.first_local(); k < (int)s.keyframes.size(); ++k) {
                const Keyframe& kf = s.keyframes[k];
                const int32_t cur = cur_slot_[i], pose_id = pose_base + (k - s.first_local());
                for (int g = 0; g < kf.n(); ++g) {
                    const double* X = &kf.pw[3 * (size_t)g];
                    const double x = T.m[0] * X[0] + T.m[1] * X[1] + T.m[2] * X[2] + T.m[3];
                    const double y = T.m[4] * X[0] + T.m[5] * X[1] + T.m[6] * X[2] + T.m[7];
                    const double z = T.m[8] * X[0] + T.m[9] * X[1] + T.m[10] * X[2] + T.m[11];
                    const double u = FX * x / z + CX, v = FY * y / z + CY;
                    if (!(z > 0 && u >= 20 && u < W - 20 && v >= 20 && v < H - 20)) continue;
                    const size_t c = nc_sz++;
                    cand[c] = {i, k, g};
                    c_ref_slot[c] = kf.slot;
                    c_cur_slot[c] = cur;
                    c_ref_pose[c] = 0;
                    c_cur_pose[c] = pose_id;
                    c_ref_px[2 * c] = kf.px[2 * (size_t)g];
                    c_ref_px[2 * c + 1] = kf.px[2 * (size_t)g + 1];
                    c_ref_depth[c] = kf.depth[g];
                    c_level[c] = (uint8_t)kf.level[g];
                    c_cur_px[2 * c] = u;
                    c_cur_px[2 * c + 1] = v;
                }
            }
            s.n_candidates += (long)nc_sz - job_begin.back();
        }
        job_begin.push_back((int)nc_sz);
        const int nc = (int)nc_sz;
        std::vector<uint8_t> search_level(nc ? nc : 1), ok(nc ? nc : 1);
        h2d_other_bytes += 57ll * nc + 8ll * (long long)poses.size();
        d2h_bytes += 18ll * nc;
        if (nc)
            TIMED(kTProject, ygzb_project_align(fr_, nc, c_ref_slot.data(), c_cur_slot.data(), (int)(poses.size() / 12), poses.data(), c_ref_pose.data(),
                                   c_cur_pose.data(), c_ref_px.data(), c_ref_depth.data(), c_level.data(), c_cur_px.data(),
                                   search_level.data(), ok.data()));

        // -- ba::OptimizeCurrentPoseOnly on the successfully projected points (LocalMapping.cpp:126; BA.cpp:188-264)
        const int m = (int)idx.size();
        std::vector<int32_t> po(m + 1, 0), n_inl(m);
        std::vector<double> pw(3 * (size_t)nc + 3), obs(2 * (size_t)nc + 2), Tp(12 * (size_t)m);
        std::vector<long> obs_id((size_t)nc + 1);
        size_t q_out = 0;
        for (int j = 0; j < m; ++j) {
            Stream& s = st_[idx[j]];
            int cnt = 0;
            for (int c = job_begin[j]; c < job_begin[j + 1]; ++c) {
                if (!ok[c]) continue;
                const Keyframe& kf = s.keyframes[cand[c].kf];
                std::memcpy(&pw[3 * q_out], &kf.pw[3 * (size_t)cand[c].n], 3 * sizeof(double));
                obs[2 * q_out] = c_cur_px[2 * (size_t)c];
                obs[2 * q_out + 1] = c_cur_px[2 * (size_t)c + 1];
                obs_id[q_out] = kf.mp0 + cand[c].n;
                ++q_out;
                ++cnt;
            }
            po[j + 1] = po[j] + cnt;
            s.n_projected += cnt;
            std::memcpy(&Tp[12 * (size_t)j], T_of[idx[j]].m, sizeof(Mat34));
        }
        const size_t tot = (size_t)po[m];
        std::vector<uint8_t> inl(tot ? tot : 1);
        std::vector<double> dep_out(tot ? tot : 1);
        h2d_other_bytes += 4ll * (m + 1) + 40ll * (long long)tot + 96ll * m;
        d2h_bytes += 96ll * m + 9ll * (long long)tot + 4ll * m;
        TIMED(kTPoseOnly, ygzb_pose_only(ctx_, m, po.data(), pw.data(), obs.data(), Tp.data(), inl.data(), dep_out.data(),
                           n_inl.data()));
        std::vector<int> need;
        for (int j = 0; j < m; ++j) {
            Stream& s = st_[idx[j]];
            if (n_inl[j] < kMinInliers) {
                s.lost = true;
                continue;
            }
            s.last_id.clear();
            s.last_px.clear();
            for (int q = po[j]; q < po[j + 1]; ++q)
                if (inl[q]) {
                    s.last_id.push_back(obs_id[q]);
                    s.last_px.push_back(obs[2 * (size_t)q]);
                    s.last_px.push_back(obs[2 * (size_t)q + 1]);
                }
            s.has_last = true;
            std::memcpy(s.T.m, &Tp[12 * (size_t)j], sizeof(Mat34));
            s.frames_since_kf += 1;
            s.n_inliers += n_inl[j];
            if (need_keyframe(prm_, s.frames_since_kf, s.T, s.keyframes.back().T)) need.push_back(idx[j]);
        }
        if (!need.empty()) CHK(make_keyframes(need, depth, frame_id, false));
        return YGZB_OK;
    }

    // SetKeyframe: Detect (grid FAST + ORB), depth-initialised map points, local BA (VisualOdometry.cpp:182-218)
    int make_keyframes(const std::vector<int>& idx, const double* const* depth, int frame_id, bool fresh) {
        const int n = (int)idx.size();
        std::vector<int32_t> slots(n), off(n + 1);
        for (int j = 0; j < n; ++j) slots[j] = cur_slot_[idx[j]];
        const size_t cap = (size_t)n * n_cells_;
        kx_.resize(cap); ky_.resize(cap); klevel_.resize(cap); kscore_.resize(cap); kangle_.resize(cap); kdesc_.resize(cap * 32);
        ygzb_keypoints kp{off.data(), kx_.data(), ky_.data(), klevel_.data(), kscore_.data(), kangle_.data(), kdesc_.data(), nullptr, (int)cap};
        TIMED(kTDetect, ygzb_detect(fr_, slots.data(), n, nullptr, &kp));
        h2d_other_bytes += 4ll * n;
        d2h_bytes += 4ll * (n + 1) + 49ll * off[n];
        std::vector<int> ba_jobs;
        for (int j = 0; j < n; ++j) {
            Stream& s = st_[idx[j]];
            Keyframe kf;
            kf.slot = next_slot(idx[j]);   // the frame leaves its staging slot: keep its pyramid in the stream's key-frame ring
            TIMED(kTDetect, ygzb_frames_copy(fr_, slots[j], kf.slot));
            kf.frame_id = frame_id;
            kf.T = s.T;
            const Mat34 Tin = inv(s.T);
            const int cnt = off[j + 1] - off[j];
            kf.px.resize(2 * (size_t)cnt); kf.level.resize(cnt); kf.depth.resize(cnt); kf.pw.resize(3 * (size_t)cnt);
            for (int g = 0; g < cnt; ++g) {
                const double x = kx_[off[j] + g], y = ky_[off[j] + g];
                const double d = depth[idx[j]][(size_t)(int)y * W + (int)x];
                kf.px[2 * (size_t)g] = x;
                kf.px[2 * (size_t)g + 1] = y;
                kf.level[g] = klevel_[off[j] + g];
                kf.depth[g] = d;
                const double pc[3] = {(x - CX) * d / FX, (y - CY) * d / FY, d};
                for (int r = 0; r < 3; ++r)
                    kf.pw[3 * (size_t)g + r] = Tin.m[4 * r] * pc[0] + Tin.m[4 * r + 1] * pc[1] + Tin.m[4 * r + 2] * pc[2] + Tin.m[4 * r + 3];
            }
            kf.mp0 = s.next_mp;
            s.next_mp += cnt;
            if (!fresh && s.has_last) {
                kf.obs_id = s.last_id;
                kf.obs_px = s.last_px;
            }
            s.keyframes.push_back(std::move(kf));
            while ((int)s.keyframes.size() > kLocalKeyframes + 1) s.keyframes.pop_front();
            s.has_ref = true;
            s.frames_since_kf = 0;
            s.n_keyframes += 1;
            if (!fresh && s.keyframes.size() >= 2) ba_jobs.push_back(idx[j]);
        }
        if (!ba_jobs.empty()) CHK(local_ba(ba_jobs));
        return YGZB_OK;
    }

    // LocalMapping::LocalBA -> ba::LocalBAG2O over the local key-frames and the points at least two of them observe
    int local_ba(const std::vector<int>& idx) {
        const int P = (int)idx.size();
        std::vector<int32_t> kf_off(P + 1, 0), pt_off(P + 1, 0), ob_off(P + 1, 0), kf_idx, pt_idx;
        std::vector<double> poses, pts, obs;
        std::vector<uint8_t> fixed;
        struct Ref { int kf, n; };
        std::vector<std::vector<Ref>> owners(P);
        for (int p = 0; p < P; ++p) {
            Stream& s = st_[idx[p]];
            const int k0 = s.first_local(), nk = (int)s.keyframes.size() - k0;
            for (int k = 0; k < nk; ++k) {
                double lg[6];
                se3_log(s.keyframes[k0 + k].T, lg);
                const double g2o[6] = {lg[3], lg[4], lg[5], lg[0], lg[1], lg[2]};   // VertexSE3Sophus: [omega; upsilon]
                poses.insert(poses.end(), g2o, g2o + 6);
                fixed.push_back(k == 0);   // the oldest local key-frame fixes the gauge (key-frame 0 in the reference)
            }
            // observations: a key-frame observes its own points (detected pixel) and the older points tracked into it
            struct Ob { long id; int kf; double u, v; };
            std::vector<Ob> all;
            auto in_local = [&](long id) {
                for (int k = 0; k < nk; ++k) {
                    const Keyframe& kf = s.keyframes[k0 + k];
                    if (id >= kf.mp0 && id < kf.mp0 + kf.n()) return true;
                }
                return false;
            };
            for (int k = 0; k < nk; ++k) {
                const Keyframe& kf = s.keyframes[k0 + k];
                for (int g = 0; g < kf.n(); ++g) all.push_back({kf.mp0 + g, k, kf.px[2 * (size_t)g], kf.px[2 * (size_t)g + 1]});
                for (size_t q = 0; q < kf.obs_id.size(); ++q)
                    if (in_local(kf.obs_id[q])) all.push_back({kf.obs_id[q], k, kf.obs_px[2 * q], kf.obs_px[2 * q + 1]});
            }
            // points seen by a single key-frame do not constrain anything: keep ids with >= 2 observations, numbered in
            // ascending id order (np.unique in vo.py)
            std::vector<long> ids;
            ids.reserve(all.size());
            for (const Ob& o : all) ids.push_back(o.id);
            std::sort(ids.begin(), ids.end());
            std::vector<long> multi;
            for (size_t a = 0; a < ids.size();) {
                size_t b = a;
                while (b < ids.size() && ids[b] == ids[a]) ++b;
                if (b - a >= 2) multi.push_back(ids[a]);
                a = b;
            }
            for (long id : multi) {
                for (int k = 0; k < nk; ++k) {
                    const Keyframe& kf = s.keyframes[k0 + k];
                    if (id >= kf.mp0 && id < kf.mp0 + kf.n()) {
                        const int g = (int)(id - kf.mp0);
                        owners[p].push_back({k0 + k, g});
                        pts.insert(pts.end(), &kf.pw[3 * (size_t)g], &kf.pw[3 * (size_t)g] + 3);
                        break;
                    }
                }
            }
            int n_ob = 0;
            for (const Ob& o : all) {
                const auto it = std::lower_bound(multi.begin(), multi.end(), o.id);
                if (it == multi.end() || *it != o.id) continue;
                kf_idx.push_back(o.kf);
                pt_idx.push_back((int32_t)(it - multi.begin()));
                obs.push_back(o.u);
                obs.push_back(o.v);
                ++n_ob;
            }
            kf_off[p + 1] = kf_off[p] + nk;
            pt_off[p + 1] = pt_off[p] + (int)multi.size();
            ob_off[p + 1] = ob_off[p] + n_ob;
        }
        ygzb_ba_params bp;
        ygzb_default_ba_params(&bp);
        std::vector<uint8_t> outl(obs.size() / 2 + 1);
        std::vector<ygzb_ba_stats> bst(P);
        h2d_other_bytes += 12ll * (P + 1) + 49ll * (long long)fixed.size() + 24ll * (long long)(pts.size() / 3) + 24ll * (long long)kf_idx.size();
        d2h_bytes += 48ll * (long long)fixed.size() + 24ll * (long long)(pts.size() / 3) + (long long)kf_idx.size();
        static const double zero3[3] = {0, 0, 0};
        static const int32_t zero_i = 0;
        TIMED(kTLocalBA, ygzb_local_ba(ctx_, P, kf_off.data(), pt_off.data(), ob_off.data(), poses.data(), fixed.data(), pts.empty() ? const_cast<double*>(zero3) : pts.data(),
                          kf_idx.empty() ? &zero_i : kf_idx.data(), pt_idx.empty() ? &zero_i : pt_idx.data(), obs.empty() ? zero3 : obs.data(), &bp,
                          outl.data(), bst.data()));
        for (int p = 0; p < P; ++p) {
            Stream& s = st_[idx[p]];
            const int k0 = s.first_local(), nk = (int)s.keyframes.size() - k0;
            {   // problem sizes and the FLOP model of SURVEY 8d (for the roofline of the BA kernel)
                const int no = ob_off[p + 1] - ob_off[p], npt = pt_off[p + 1] - pt_off[p];
                std::vector<int> deg(npt, 0);
                for (int o = ob_off[p]; o < ob_off[p + 1]; ++o) deg[pt_idx[o]]++;
                double per_trial = 300.0 * no;
                for (int d : deg) per_trial += 216.0 * d * d + 108.0 * d + 50.0;
                const double dim = 6.0 * (nk - 1);
                per_trial += dim * dim * dim / 3.0;
                s.ba_obs += no; s.ba_pts += npt; s.ba_kfs += nk; s.ba_trials += bst[p].lm_trials; s.ba_iters += bst[p].iters;
                s.ba_flops += per_trial * bst[p].lm_trials;
            }
            for (int k = 0; k < nk; ++k) {
                const double* g = &poses[6 * (size_t)(kf_off[p] + k)];
                const double v[6] = {g[3], g[4], g[5], g[0], g[1], g[2]};
                s.keyframes[k0 + k].T = from_se3(ygzb::se3_exp(v));
            }
            for (size_t q = 0; q < owners[p].size(); ++q) {
                Keyframe& kf = s.keyframes[owners[p][q].kf];
                std::memcpy(&kf.pw[3 * (size_t)owners[p][q].n], &pts[3 * ((size_t)pt_off[p] + q)], 3 * sizeof(double));
            }
            s.T = s.keyframes.back().T;
            s.n_ba += 1;
        }
        return YGZB_OK;
    }

    ygzb_ctx* ctx_;
    ygzb_frames* fr_;
    int S_, n_cells_ = 0;
    Params prm_;
    std::vector<Stream> st_;
    std::vector<int> cur_slot_;
    std::vector<float> kx_, ky_, kscore_, kangle_;
    std::vector<uint8_t> klevel_, kdesc_;
};


// ---- device-resident engine --------------------------------------------------------------------------------------------
// The same caller logic on ygzb_tracker_*: the local map lives on the device.  Frames come from a FIFO per stream
// (image, depth map, caller's tag); a ROUND enqueues for every stream a window of its queued frames -- up to and
// including the first frame that may become a key-frame (every frame is tracked against the newest key-frame, so the
// frames of a window are independent; the reference tracks against the previous frame, VisualOdometry.cpp:88-90, and
// key-frame tracking is this engine's batching choice) --
// as ONE fused chain (upload + pyramid, sparse alignment, candidate projection, direct projection, pose-only), reads one
// 128-byte record per frame back, takes the key-frame decisions, and inserts the key-frames (Detect, map points, local
// BA, all on the device) with the next round's enqueue.  Results are identical to frame-by-frame processing, whatever
// the window and however many frames are queued when a round starts.
struct KfInfo {
    int entry = 0, n = 0, frame_id = 0;
    Mat34 T;
    long mp0 = 0;
};
struct QFrame {
    const uint8_t* image;
    const double* depth;   // NULL: the stream's current depth map stays valid
    int64_t tag;
    bool stacked;          // image lies in the caller's stacked sequence of the stream (one allocation, batch entry points)
    bool restart = false;  // first frame of a new sequence (ygz_vo_restart): it becomes a first key-frame
};
using Camera = std::array<double, 4>;   // fx, fy, cx, cy
// bit for bit, as records compare cameras
bool same_camera(const Camera& a, const Camera& b) { return std::memcmp(a.data(), b.data(), sizeof a) == 0; }
// a lens (ygz_vo_set_lens): the raw camera K and its distortion dist = {k1, k2, p1, p2, k3}; on = false: none
struct Lens {
    bool on = false;
    Camera K{};
    std::array<double, 5> dist{};
    // bit for bit, as records compare cameras
    bool same(const Lens& o) const {
        return on == o.on && (!on || (same_camera(K, o.K) && std::memcmp(dist.data(), o.dist.data(), sizeof dist) == 0));
    }
};
// the frames a stream pushes (ygz_vo_set_frame_format): w x h pixels of `channels` bytes (1 grey, 3 BGR), rows packed
struct Format {
    int w = 0, h = 0, channels = 1;
    size_t bytes() const { return (size_t)w * h * channels; }
    bool operator==(const Format&) const = default;
};
// what a sequence of a stream is pushed under: its camera (ygz_vo_set_camera), its lens (ygz_vo_set_lens) and the format of
// its frames (ygz_vo_set_frame_format)
struct Source {
    Camera K{};
    Lens lens;
    Format fmt;
    // bit for bit, as records compare K and the lens
    bool operator==(const Source& o) const { return same_camera(K, o.K) && lens.same(o.lens) && fmt == o.fmt; }
    // frames of a size other than the context's W x H are only resampled by a lens
    bool pushable(int W, int H) const { return lens.on || (fmt.w == W && fmt.h == H); }
};
struct SeqStart {
    Mat34 T;                  // pose of the sequence's first key-frame
    Source src;               // camera, lens and frame format of the sequence
};
struct EStream : Counters {
    std::deque<KfInfo> kfs;   // at most YGZB_TRACK_RING, the newest is the reference key-frame; the last kLocalKeyframes are local
    std::deque<QFrame> queue; // frames without a final result, oldest first; the first one is frame next_frame
    Mat34 T = identity();
    Mat34 start = identity(); // pose of the next sequence's first key-frame (ygz_vo_restart)
    Source src;               // source of the current sequence, or of the next one while a restart is pending
    std::deque<SeqStart> starts;   // the queued frames that start a sequence (the stream's first, restarts), in order
    bool has_pose = false, lost = false, has_depth = false;
    bool restart_pending = false;   // the next push starts a new sequence at `start`
    int frames_since_kf = 0, next_frame = 0;
    long next_mp = 0;
};

// a page-locked buffer the tracker writes through its device mapping, `stride` elements per job, switched on and off
// through one of the tracker's setters (ygzb_tracker_set_observations, _information, _map_updates)
template <typename T>
struct PinnedOutput {
    T* h = nullptr;   // NULL: off
    size_t stride = 0;
    PinnedOutput() = default;
    PinnedOutput(const PinnedOutput&) = delete;
    PinnedOutput& operator=(const PinnedOutput&) = delete;
    ~PinnedOutput() {
        if (h) ygzb_host_free(h);
    }
    bool on() const { return h != nullptr; }
    // job j's elements of the batch that has just come back, or NULL when off
    const T* job(size_t j) const { return h ? h + j * stride : nullptr; }
    // on: room for `jobs` jobs of `per_job` elements, allocated and handed to the tracker; off: the tracker stops writing
    // and, once the device has caught up, the buffer is freed
    int set(ygzb_ctx* ctx, ygzb_tracker* tr, int (*attach)(ygzb_tracker*, T*, size_t), bool on_, size_t jobs, size_t per_job) {
        if (on_ == on()) return YGZB_OK;
        if (!on_) {
            CHK(attach(tr, nullptr, 0));
            CHK(ygzb_synchronize(ctx));
            ygzb_host_free(h);
            h = nullptr;
            return YGZB_OK;
        }
        void* p = nullptr;
        CHK(ygzb_host_alloc(&p, jobs * per_job * sizeof(T)));
        const int rc = attach(tr, static_cast<T*>(p), jobs * per_job);
        if (rc != YGZB_OK) {
            ygzb_host_free(p);
            return rc;
        }
        h = static_cast<T*>(p);
        stride = per_job;
        return YGZB_OK;
    }
};

// the part of a queue's buffer before `head` has been taken: clear the buffer when it is drained, erase that part once it
// passes half of it
template <typename T>
void compact(std::vector<T>& v, size_t& head) {
    if (head == v.size()) {
        v.clear();
        head = 0;
    } else if (head > v.size() / 2) {
        v.erase(v.begin(), v.begin() + (ptrdiff_t)head);
        head = 0;
    }
}

// records, oldest first, each with its run of rows: the records from `first` and the rows back to back from `head`, each
// in one buffer that keeps its capacity across rounds, so that a round neither allocates nor touches fresh pages once the
// buffers have grown
template <typename Rec, typename Row>
struct RowQueue {
    struct Entry {
        Rec rec;
        size_t n_rows;
    };
    std::vector<Entry> recs;
    std::vector<Row> rows;
    size_t first = 0, head = 0;

    size_t size() const { return recs.size() - first; }
    bool empty() const { return size() == 0; }
    const Entry& operator[](size_t i) const { return recs[first + i]; }
    const Row* front_rows() const { return rows.data() + head; }
    void push(const Rec& rec, const Row* r, size_t n_rows) {
        recs.push_back({rec, n_rows});
        rows.insert(rows.end(), r, r + n_rows);
    }
    void drop(size_t k) { take(k, nullptr, [](size_t, const Rec&) {}); }
    // the k oldest records leave: each to put(i, record), their rows to `out` (NULL: dropped); returns their row count
    template <typename Put>
    size_t take(size_t k, Row* out, Put put) {
        size_t n = 0;
        for (size_t i = 0; i < k; ++i) {
            put(i, (*this)[i].rec);
            n += (*this)[i].n_rows;
        }
        if (out && n) std::memcpy(out, front_rows(), n * sizeof(Row));
        first += k;
        head += n;
        compact(recs, first);
        compact(rows, head);
        return n;
    }
    // whole records, oldest first, while their rows fit: at most `capacity` records, their rows into out[row_capacity];
    // YGZB_ERR_CAPACITY with *n = 0 and *n_rows = its row count when the first one's rows do not fit (never for capacity 0)
    template <typename Put>
    int take_whole(int capacity, int* n, Row* out, size_t row_capacity, size_t* n_rows, Put put) {
        *n = 0;
        *n_rows = 0;
        if (capacity > 0 && !empty() && (*this)[0].n_rows > row_capacity) {
            *n_rows = (*this)[0].n_rows;
            return YGZB_ERR_CAPACITY;
        }
        for (size_t used = 0; *n < capacity && *n < (int)size() && used + (*this)[*n].n_rows <= row_capacity;) used += (*this)[(*n)++].n_rows;
        *n_rows = take(*n, out, put);
        return YGZB_OK;
    }
};

// what a frame's result carries besides its pose: its observation rows (observations on) and its information record
// (information on; NULL: zeros, as for a sequence's first key-frame and a LOST frame)
struct Attachments {
    const ygzb_observation* rows = nullptr;
    size_t n_rows = 0;
    const ygzb_pose_information* info = nullptr;
};

class Engine {
    struct Win { int stream, first, count, job0; };   // a window in flight: frames [first, first + count) of a stream (job0 < 0: first frame)
    struct KfFrame {   // the frame behind a pending key-frame job
        int frame, n_inliers;
        int64_t tag;
        const double* depth;
        ygzb_pose_information info;   // its tracking job's information record (information on; zeros for a first key-frame)
    };
    struct Result {   // a final result and its information record (zeros while information is off)
        ygz_vo_result r;
        ygzb_pose_information info;
    };
  public:
    Engine(ygzb_ctx* ctx, int n_streams, int window, const Params& p) : ctx_(ctx), S_(n_streams), F_(std::max(1, window)), prm_(p), st_(n_streams) {
        for (int i = 0; i < S_; ++i) order_.push_back(i);
        // YGZ_VO_BLOCKING_SYNC=1: sleep instead of spinning in the one synchronisation per round (hosts with fewer CPUs than
        // engine threads; bench.py sets it when the threads of all ranks outnumber the CPUs it may use)
        const char* e = std::getenv("YGZ_VO_BLOCKING_SYNC");
        blocking_sync_ = e && std::atoi(e) != 0;
    }
    ~Engine() {
        if (tr_) ygzb_tracker_destroy(tr_);
        if (fr_) ygzb_frames_destroy(fr_);
        if (h_res_) ygzb_host_free(h_res_);
        if (h_kres_) ygzb_host_free(h_kres_);
    }
    // order[i] = the caller's index of tracker stream i (images, depth maps, trajectory rows); identity unless set
    void set_order(const std::vector<int>& order) { order_ = order; }
    const std::vector<int>& order() const { return order_; }
    // depth (may be NULL): one map per caller stream that every key-frame of it uses unless a frame brings its own
    int init(const double* const* depth) {
        ygzb_params cp;
        CHK(ygzb_get_params(ctx_, &cp));
        W_ = cp.image_width;
        H_ = cp.image_height;
        // every stream starts with the tracker's camera, no lens and grey frames of the context's size
        const Source dflt{{prm_.K[0], prm_.K[1], prm_.K[2], prm_.K[3]}, {}, {W_, H_, 1}};
        for (EStream& s : st_) s.src = dflt;
        tr_src_.assign(S_, dflt);
        int rows = 0, cols = 0;
        CHK(ygzb_grid_dims(ctx_, &rows, &cols));
        ring_cells_ = (size_t)YGZB_TRACK_RING * rows * cols;
        // slots: S*F frame slots, S*RING key-frame slots, then (previous-frame reference) one reference slot per stream
        const bool prev = prm_.ref_mode == YGZB_TRACK_REF_PREVIOUS;
        CHK(ygzb_frames_create(ctx_, S_ * F_ + S_ * YGZB_TRACK_RING + (prev ? S_ : 0), &fr_));
        CHK(ygzb_tracker_create(fr_, S_, S_ * F_, prm_.K, &tr_));
        if (prev) {
            std::vector<int32_t> ref_slots(S_);
            for (int i = 0; i < S_; ++i) ref_slots[i] = S_ * F_ + S_ * YGZB_TRACK_RING + i;
            CHK(ygzb_tracker_set_reference_mode(tr_, YGZB_TRACK_REF_PREVIOUS, ref_slots.data()));
        }
        if (depth)
            for (int i = 0; i < S_; ++i) {
                CHK(ygzb_tracker_set_depth(tr_, i, depth[order_[i]]));
                st_[i].has_depth = true;
            }
        void* p = nullptr;
        CHK(ygzb_host_alloc(&p, sizeof(ygzb_track_result) * (size_t)S_ * F_));
        h_res_ = static_cast<ygzb_track_result*>(p);
        CHK(ygzb_host_alloc(&p, sizeof(ygzb_keyframe_result) * (size_t)S_));
        h_kres_ = static_cast<ygzb_keyframe_result*>(p);
        ygzb_default_ba_params(&ba_);
        return YGZB_OK;
    }
    std::vector<EStream>& streams() { return st_; }
    int width() const { return W_; }
    int height() const { return H_; }
    long long h2d_image_bytes = 0, h2d_other_bytes = 0, d2h_bytes = 0;

    // queues frame (image, depth, tag) of tracker stream i; the caller has checked the arguments.  The stream's first frame
    // and the first one after a restart queue the pose their key-frame starts at
    void push(int i, const uint8_t* image, const double* depth, int64_t tag, bool stacked = false) {
        EStream& s = st_[i];
        QFrame f{image, depth, tag, stacked};
        if (pushed(i) == 0 || s.restart_pending) {
            f.restart = s.restart_pending;
            s.starts.push_back({s.start, s.src});
            s.restart_pending = false;
        }
        s.queue.push_back(f);
        s.has_depth |= depth != nullptr;
    }
    // frames pushed to stream i so far (those with a final result or a pending key-frame insertion, then the queued ones)
    long pushed(int i) const { return st_[i].next_frame + (long)st_[i].queue.size(); }
    // the next frame pushed to stream i starts a new sequence at T (before the stream's first push: its first sequence
    // starts at T); the frames pushed before keep the results they would have had without the call.  The tracker checks
    // T (finite, a rotation) and keeps it; that does not reach an insertion of the old sequence, because step 1 of a round
    // sets every first key-frame's own pose right before its insertion
    int restart(int i, const Mat34& T) {
        CHK(ygzb_tracker_set_start_pose(tr_, i, T.m));
        EStream& s = st_[i];
        s.start = T;
        s.restart_pending = pushed(i) > 0;
        return YGZB_OK;
    }
    // the source of stream i's next sequence: only before its first push or while a restart is pending (the caller has
    // checked it); it reaches the tracker when that sequence's first frame is uploaded (use_source)
    int set_source(int i, const Source& src) {
        EStream& s = st_[i];
        if (pushed(i) > 0 && !s.restart_pending) return YGZB_ERR_INVALID;
        s.src = src;
        return YGZB_OK;
    }
    const Source& source(int i) const { return st_[i].src; }
    // final results go to `traj` (this group's [S][n_frames][12], rows in the caller's stream order; NULL: none) and, with
    // collect, to the result queue that pop_results drains
    void set_outputs(double* traj, int n_frames, bool collect) {
        traj_ = traj;
        traj_frames_ = n_frames;
        collect_ = collect;
    }
    // the oldest results, at most `capacity` of them (ygz_vo_poll: their rows and records are discarded)
    size_t pop_results(ygz_vo_result* out, size_t capacity) {
        const size_t n = std::min(capacity, results_.size());
        results_.take(n, nullptr, [&](size_t k, const Result& r) { out[k] = r.r; });
        return n;
    }
    // whole results, oldest first, with their information records (info; NULL: discarded) and, with observations on,
    // their observation rows while those fit; YGZB_ERR_CAPACITY with *n = 0 and *n_obs = its row count when the first
    // one's rows do not.  n_obs is only touched with observations on
    int pop_results(ygz_vo_result* out, int capacity, int* n, ygzb_pose_information* info, ygzb_observation* obs, size_t obs_capacity,
                    size_t* n_obs) {
        size_t no_rows;
        return results_.take_whole(capacity, n, obs, obs_capacity, observations() ? n_obs : &no_rows, [&](size_t k, const Result& r) {
            out[k] = r.r;
            if (info) info[k] = r.info;
        });
    }
    // nothing queued, no key-frame insertion pending, no result or map update waiting to be polled
    bool idle() const {
        for (const EStream& s : st_)
            if (!s.queue.empty()) return false;
        return kjobs_.empty() && results_.empty() && updates_.empty();
    }
    bool observations() const { return obs_.on(); }
    bool information() const { return info_.on(); }
    bool map_updates() const { return map_.on(); }
    // whole map updates with their rows, oldest first, while both fit; YGZB_ERR_CAPACITY with *n = 0 and *n_rows = its row
    // count when the first one's rows do not
    int pop_map_updates(ygz_vo_map_update* out, int capacity, int* n, ygzb_map_point* rows, size_t row_capacity, size_t* n_rows) {
        return updates_.take_whole(capacity, n, rows, row_capacity, n_rows, [&](size_t k, const ygz_vo_map_update& u) { out[k] = u; });
    }
    // on: every result from here on carries the observation rows of its frame (max_jobs * YGZB_TRACK_RING * cells rows
    // for the tracker); off: none.  Call only when idle()
    int set_observations(bool on) { return obs_.set(ctx_, tr_, ygzb_tracker_set_observations, on, (size_t)S_ * F_, ring_cells_); }
    // on: every result from here on carries the information record of its frame (max_jobs records for the tracker); off:
    // none.  Call only when idle()
    int set_information(bool on) { return info_.set(ctx_, tr_, ygzb_tracker_set_information, on, (size_t)S_ * F_, 1); }
    // on: every key-frame insertion from here on queues its map update (n_streams * YGZB_TRACK_RING * cells rows for the
    // tracker); off: none.  Call only when idle()
    int set_map_updates(bool on) { return map_.set(ctx_, tr_, ygzb_tracker_set_map_updates, on, (size_t)S_, ring_cells_); }

    // Batch feed: queues frames [queued, limit) of every stream from the stacked sequences images[caller stream] (with the
    // depth map of init) and runs until they all have their result and nothing is in flight.
    int run_until(const uint8_t* const* images, int limit) {
        for (int i = 0; i < S_; ++i) {
            EStream& s = st_[i];
            for (int k = s.next_frame + (int)s.queue.size(); k < limit; ++k) push(i, images[order_[i]] + (size_t)k * W_ * H_, nullptr, k, true);
        }
        return flush();
    }
    int flush() {
        for (bool idle = false; !idle;) CHK(round(&idle));
        return YGZB_OK;
    }

    // One round, software-pipelined around ONE host synchronisation:
    //   1. enqueue the key-frame insertions the previous round decided (the frame's depth map first, when it has one;
    //      Detect, map points, local BA) -- asynchronous,
    //   2. plan the next window of every stream from its queue, upload its frames and enqueue its tracking chain right
    //      behind; the tracker runs the uploads and the sparse alignment of that batch on a second CUDA stream, concurrently
    //      with the local BA of step 1 (the alignment works relative to the reference key-frame and needs its features, not
    //      its refined pose),
    //   3. synchronise, apply the key-frame results (poses after the BA, feature counts),
    //   4. take the decisions of the tracking batch that has just come back (lost streams, key-frame triggers).
    // *idle: nothing was queued or pending, nothing was enqueued.
    int round(bool* idle) {
        *idle = false;
        // ---- 1. key-frame insertions decided last round (asynchronous)
        if (!kjobs_.empty()) {
            StageTimer tm(kTLocalBA);
            for (size_t q = 0; q < kjobs_.size(); ++q) {   // bookkeeping that does not need the device's answer
                EStream& s = st_[kjobs_[q].stream];
                const KfFrame& f = kframes_[q].rec;
                KfInfo kf;
                kf.entry = kjobs_[q].entry;
                kf.frame_id = f.frame;
                kf.mp0 = kjobs_[q].mp0;
                kf.T = s.T;
                s.kfs.push_back(kf);
                while ((int)s.kfs.size() > YGZB_TRACK_RING) s.kfs.pop_front();
                s.frames_since_kf = 0;
                s.n_keyframes += 1;
                // the key-frame's own depth map: on the context stream like the insertion, so it lands just before it
                if (f.depth) {
                    CHK(ygzb_tracker_set_depth(tr_, kjobs_[q].stream, f.depth));
                    h2d_other_bytes += (long long)W_ * H_ * (long long)sizeof(double);
                }
                // a sequence's first key-frame starts at the pose its frame was pushed with
                if (kjobs_[q].track_job < 0) CHK(ygzb_tracker_set_start_pose(tr_, kjobs_[q].stream, s.T.m));
            }
            CHK(ygzb_tracker_make_keyframes(tr_, (int)kjobs_.size(), kjobs_.data(), &ba_, h_kres_));
            // per job: the job, its start pose (staged behind the jobs in the same copy) and its problem index
            h2d_other_bytes += (long long)(kjobs_.size() * (sizeof(ygzb_keyframe_job) + 12 * sizeof(double) + 4));
            d2h_bytes += (long long)(kjobs_.size() * sizeof(ygzb_keyframe_result));
        }
        // ---- 2. next window of every stream: uploads + tracking chain (asynchronous, right behind the key-frames)
        std::vector<ygzb_track_job> jobs;
        for (int i = 0; i < S_; ++i) {
            EStream& s = st_[i];
            if (s.lost)   // the reference keeps the last pose and reports VO_LOST, up to a restart
                while (!s.queue.empty() && !s.queue.front().restart) emit_front(i, YGZ_VO_LOST, 0);
            if (s.queue.empty()) continue;
            // window: up to and including the first frame that may become a key-frame; past that point every frame may, and a
            // few frames are tracked speculatively -- the ones behind a key-frame trigger are dropped and tracked again against
            // the new key-frame next round (results stay those of frame-by-frame processing); never more than is queued, and
            // never past a restart.  A sequence's first frame is a window of its own
            const bool first = s.kfs.empty() || s.queue.front().restart;
            int w = 1;
            if (!first) {
                const int sure = prm_.kf_min_frames - s.frames_since_kf;
                w = sure >= 1 ? std::min(F_, sure) : std::min(F_, kSpeculativeFrames);
                for (int t = 1; t < w && t < (int)s.queue.size(); ++t)
                    if (s.queue[t].restart) w = t;
            }
            w = std::min(w, (int)s.queue.size());
            // a sequence's source reaches the tracker right before its first frame's upload.  Every frame of the old sequence
            // has been uploaded by then (a window never crosses a restart), and the tracker orders the maps and the format
            // behind those uploads.  The old sequence is done with the camera too.  Its device readers are kf_fill_kernel,
            // track_prep_kernel and candidate projection (ba_build_kernel and kf_points_kernel read none, and a local BA
            // takes its cameras as kernel parameters when it is enqueued).  ygzb_tracker_set_camera waits on the front stream
            // for e_fill and e_main, which follow the old sequence's last such readers: its last insertion was enqueued in
            // step 1 of this round, and its last tracking chain ran in an earlier round.  The new sequence's first insertion
            // waits for e_up
            if (first) CHK(use_source(i, s.starts.front().src));
            CHK(upload(i, w));
            if (first) {
                wins_.push_back({i, s.next_frame, 1, -1});
                continue;
            }
            wins_.push_back({i, s.next_frame, w, (int)jobs.size()});
            const int nl = std::min(kLocalKeyframes, (int)s.kfs.size());
            for (int t = 0; t < w; ++t) {
                ygzb_track_job j{};
                j.stream = i;
                j.cur_slot = i * F_ + t;
                j.n_local = nl;
                for (int k = 0; k < nl; ++k) j.entry[k] = s.kfs[s.kfs.size() - nl + k].entry;
                jobs.push_back(j);
            }
        }
        if (!jobs.empty()) {
            StageTimer tm(kTSparse);
            CHK(ygzb_tracker_track(tr_, (int)jobs.size(), jobs.data(), h_res_));
            h2d_other_bytes += (long long)(jobs.size() * sizeof(ygzb_track_job));
            d2h_bytes += (long long)(jobs.size() * sizeof(ygzb_track_result));
        }
        if (kjobs_.empty() && wins_.empty()) {   // every queue is empty, nothing in flight
            *idle = true;
            return YGZB_OK;
        }
        // ---- 3. one synchronisation per round; key-frame results
        {
            StageTimer tm(kTPoseOnly);
            CHK(blocking_sync_ ? ygzb_synchronize_blocking(ctx_) : ygzb_synchronize(ctx_));
        }
        for (size_t q = 0; q < kjobs_.size(); ++q) {
            const ygzb_keyframe_job& kj = kjobs_[q];
            const ygzb_keyframe_result& r = h_kres_[q];
            EStream& s = st_[kj.stream];
            s.kfs.back().n = r.n_features;
            s.next_mp = kj.mp0 + r.n_features;
            for (int k = 0; k < kj.n_local; ++k) std::memcpy(s.kfs[s.kfs.size() - kj.n_local + k].T.m, r.T_cw[k], sizeof(Mat34));
            s.T = s.kfs.back().T;
            if (kj.run_ba && kj.n_local >= 2) {
                s.n_ba += 1;
                s.ba_obs += r.ba_observations; s.ba_pts += r.ba_points; s.ba_kfs += kj.n_local; s.ba_trials += r.ba_trials; s.ba_iters += r.ba_iters;
                const double kbar = r.ba_points ? (double)r.ba_observations / r.ba_points : 0.0, dim = 6.0 * (kj.n_local - 1);
                s.ba_flops += r.ba_trials * (300.0 * r.ba_observations + r.ba_points * (216.0 * kbar * kbar + 108.0 * kbar + 50.0) + dim * dim * dim / 3.0);
            }
            const auto& kf = kframes_[0];
            emit(kj.stream, kf.rec.frame, kf.rec.tag, YGZ_VO_KEYFRAME, kf.rec.n_inliers, {kframes_.front_rows(), kf.n_rows, &kf.rec.info});
            kframes_.drop(1);
            if (map_updates()) queue_map_update(kj, r, map_.job(q));
        }
        kjobs_.clear();
        // ---- 4. results of the tracking batch
        for (const Win& b : wins_) {
            EStream& s = st_[b.stream];
            if (b.job0 < 0) {   // first frame of a sequence: becomes its first key-frame (depth-initialised map)
                const QFrame& f = s.queue.front();
                if (f.restart) {   // the old sequence is final (its last insertion applied in step 3): start as a fresh stream
                    s.kfs.clear();
                    s.lost = false;
                    s.frames_since_kf = 0;
                    s.next_mp = 0;
                    s.n_restarts += 1;
                }
                s.T = s.starts.front().T;
                s.starts.pop_front();
                s.has_pose = true;
                pend_keyframe(b.stream, b.stream * F_, -1, 0);
                continue;
            }
            for (int t = 0; t < b.count; ++t) {
                const int j = b.job0 + t;
                const ygzb_track_result& r = h_res_[j];
                const Attachments a{obs_.job(j), obs_.on() ? (size_t)r.n_inliers : 0, info_.job(j)};   // (the tracker wrote r.n_inliers rows)
                if (!r.aligned) {   // Matcher::SparseImageAlignment returned false (Matcher.cpp:482-488)
                    s.lost = true;
                    emit_front(b.stream, YGZ_VO_LOST, 0);
                    break;
                }
                s.n_candidates += r.n_candidates;
                s.n_projected += r.n_projected;
                if (r.n_inliers < prm_.min_inliers) {
                    s.lost = true;
                    emit_front(b.stream, YGZ_VO_LOST, r.n_inliers, {a.rows, a.n_rows});
                    break;
                }
                std::memcpy(s.T.m, r.T_cw, sizeof(s.T.m));
                s.frames_since_kf += 1;
                s.n_inliers += r.n_inliers;
                if (need_keyframe(prm_, s.frames_since_kf, s.T, s.kfs.back().T)) {
                    pend_keyframe(b.stream, b.stream * F_ + t, j, r.n_inliers, a);
                    break;   // frames of the window behind the key-frame (speculative ones) stay queued: tracked again next round
                }
                emit_front(b.stream, YGZ_VO_TRACKED, r.n_inliers, a);
            }
        }
        wins_.clear();
        return YGZB_OK;
    }

    void stats(int i, int64_t* o) const { st_[i].write_stats(st_[i].lost, o); }

    // local map of stream i (every key-frame still in its ring, oldest first) into `rec`: asynchronous, valid after
    // ygzb_synchronize; call with nothing in flight (after run_until or flush)
    int export_map(int i, ygzb_map_record* rec) const {
        std::vector<int32_t> entries;
        for (const KfInfo& kf : st_[i].kfs) entries.push_back(kf.entry);
        return ygzb_tracker_export(tr_, i, (int)entries.size(), entries.data(), rec);
    }
    // previous-frame mode: whether stream i has a reference (its first key-frame has been inserted), and that reference
    // into `rec` (asynchronous like export_map)
    bool has_reference(int i) const { return prm_.ref_mode == YGZB_TRACK_REF_PREVIOUS && !st_[i].kfs.empty(); }
    int export_reference(int i, ygzb_reference_record* rec) const { return ygzb_tracker_export_reference(tr_, i, rec); }
    // stream i continues a stream of another engine: its map (exported by export_map) goes into the same ring entries, its
    // key-frame images into this engine's key-frame slots of stream i, in previous-frame mode its reference (exported by
    // export_reference; NULL if it has none) into stream i's reference slot, and its host bookkeeping is taken over as it is
    int adopt(int i, const EStream& s, const ygzb_map_record* rec, const ygzb_reference_record* ref) {
        std::vector<int32_t> entries, slots;
        for (const KfInfo& kf : s.kfs) {
            entries.push_back(kf.entry);
            slots.push_back(S_ * F_ + i * YGZB_TRACK_RING + kf.entry);
        }
        if (rec->n_keyframes != (int)entries.size()) return YGZB_ERR_INVALID;
        CHK(use_source(i, s.src));
        CHK(ygzb_tracker_import(tr_, i, entries.data(), slots.data(), rec));
        if (ref) CHK(ygzb_tracker_import_reference(tr_, i, ref));
        st_[i] = s;
        return YGZB_OK;
    }
    // stream i has no queued frame and no key-frame insertion pending: every frame pushed to it has its final result
    bool settled(int i) const {
        if (!st_[i].queue.empty()) return false;
        for (const ygzb_keyframe_job& kj : kjobs_)
            if (kj.stream == i) return false;
        return true;
    }
    // the depth map stream i's next key-frame takes when its frame brings none (asynchronous, like export_map), and back
    int get_depth(int i, double* out) const { return ygzb_tracker_get_depth(tr_, i, out); }
    int set_depth(int i, const double* depth) { return ygzb_tracker_set_depth(tr_, i, depth); }
    // the tracker's check of a start pose (finite, a rotation), which keeps it as restart() does; a round sets every first
    // key-frame's own pose before its insertion, so the kept pose reaches nothing else
    int check_start_pose(int i, const Mat34& T) { return ygzb_tracker_set_start_pose(tr_, i, T.m); }

  private:
    // the tracker's camera, undistortion maps and raw frame format of stream i become those of `src`, in that order, for
    // everything enqueued from here on; nothing is enqueued for a part the tracker has already.  The maps are those of the
    // lens seen through the camera (none without a lens)
    int use_source(int i, const Source& src) {
        Source& cur = tr_src_[i];
        const bool new_K = !same_camera(cur.K, src.K);
        if (new_K) CHK(ygzb_tracker_set_camera(tr_, i, src.K.data()));
        cur.K = src.K;
        if (!cur.lens.same(src.lens) || (src.lens.on && new_K)) {
            const Lens& L = src.lens;
            if (L.on) {
                const size_t n = (size_t)W_ * H_;
                if (!(maps_lens_.same(L) && same_camera(maps_K_, src.K))) {   // (streams of one lens and camera share the host maps)
                    map_xy_.resize(2 * n);
                    map_a_.resize(n);
                    maps_lens_ = {};
                    CHK(ygzb_undistort_map(W_, H_, L.K.data(), L.dist.data(), src.K.data(), map_xy_.data(), map_a_.data()));
                    maps_lens_ = L;
                    maps_K_ = src.K;
                }
                CHK(ygzb_tracker_set_undistort(tr_, i, map_xy_.data(), map_a_.data()));
                h2d_other_bytes += (long long)(n * 6);
            } else {
                CHK(ygzb_tracker_set_undistort(tr_, i, nullptr, nullptr));
            }
            cur.lens = L;
        }
        if (cur.fmt != src.fmt) CHK(ygzb_tracker_set_source(tr_, i, src.fmt.w, src.fmt.h, src.fmt.channels));
        cur.fmt = src.fmt;
        return YGZB_OK;
    }
    // the first w queued frames of stream i into its frame slots: one strided copy when they are equally spaced in one
    // stacked sequence, one copy per frame otherwise (frames pushed one by one may sit in separate allocations, which one
    // strided copy cannot span even when their addresses happen to be equally spaced).  The frames are in the tracker's
    // format of the stream (use_source), that of their sequence
    int upload(int i, int w) {
        const std::deque<QFrame>& q = st_[i].queue;
        const size_t fb = tr_src_[i].fmt.bytes();
        const ptrdiff_t stride = w > 1 ? q[1].image - q[0].image : (ptrdiff_t)fb;
        bool strided = stride >= (ptrdiff_t)fb;
        for (int t = 0; t < w && strided; ++t) strided = q[t].stacked && (t < 2 || q[t].image - q[t - 1].image == stride);
        h2d_image_bytes += (long long)w * (long long)fb;
        if (strided) return ygzb_tracker_upload_stream(tr_, i, i * F_, w, q[0].image, (size_t)stride);
        for (int t = 0; t < w; ++t) CHK(ygzb_tracker_upload_stream(tr_, i, i * F_ + t, 1, q[t].image, fb));
        return YGZB_OK;
    }
    // the map update of key-frame job kj, whose result r and rows (r.ba_points moved, then r.n_features new) have just come
    // back: the rows are copied here, since the next round's insertions reuse the buffer.  Step 3 has applied r to the
    // stream's key-frames, so the last kj.n_local of them are the local ones after the insertion
    void queue_map_update(const ygzb_keyframe_job& kj, const ygzb_keyframe_result& r, const ygzb_map_point* rows) {
        const EStream& s = st_[kj.stream];
        ygz_vo_map_update u{};
        u.stream = order_[kj.stream];
        u.frame = s.kfs.back().frame_id;
        u.sequence = s.n_restarts;
        u.n_local = kj.n_local;
        const size_t first = s.kfs.size() - (size_t)kj.n_local;
        u.retired_frame = first > 0 ? s.kfs[first - 1].frame_id : -1;   // (the ring keeps the key-frame that has just left)
        for (int k = 0; k < YGZB_TRACK_RING; ++k) u.local_frame[k] = k < kj.n_local ? s.kfs[first + k].frame_id : -1;
        for (int k = 0; k < kj.n_local; ++k) std::memcpy(u.T_cw[k], r.T_cw[k], sizeof(u.T_cw[k]));
        u.n_moved = r.ba_points;
        u.n_new = r.n_features;
        updates_.push(u, rows, (size_t)u.n_moved + (size_t)u.n_new);
    }
    // the stream's oldest queued frame becomes a key-frame: its insertion is enqueued at the start of the next round, its
    // result is emitted once the insertion's local BA has come back; its tracking job's attachments are held with it until
    // then, since the next round's batch reuses the buffers
    void pend_keyframe(int stream, int frame_slot, int track_job, int n_inliers, const Attachments& a = {}) {
        EStream& s = st_[stream];
        const QFrame f = s.queue.front();
        s.queue.pop_front();
        kjobs_.push_back(make_kf_job(stream, frame_slot, track_job));
        kframes_.push({s.next_frame++, n_inliers, f.tag, f.depth, a.info ? *a.info : ygzb_pose_information{}}, a.rows, a.n_rows);
    }
    // the stream's oldest queued frame is final with the stream's current pose
    void emit_front(int stream, int status, int n_inliers, const Attachments& a = {}) {
        EStream& s = st_[stream];
        const int64_t tag = s.queue.front().tag;
        s.queue.pop_front();
        emit(stream, s.next_frame++, tag, status, n_inliers, a);
    }
    void emit(int stream, int frame, int64_t tag, int status, int n_inliers, const Attachments& a) {
        const EStream& s = st_[stream];
        if (traj_) {
            double* out = traj_ + ((size_t)order_[stream] * traj_frames_ + frame) * 12;
            for (int c = 0; c < 12; ++c) out[c] = s.has_pose ? s.T.m[c] : NAN;
        }
        if (collect_) {
            Result res{};
            ygz_vo_result& r = res.r;
            r.stream = order_[stream];
            r.frame = frame;
            r.tag = tag;
            r.status = status;
            r.n_inliers = n_inliers;
            std::memcpy(r.T_cw, s.T.m, sizeof(r.T_cw));
            if (a.info) res.info = *a.info;
            results_.push(res, a.rows, a.n_rows);
        }
    }
    ygzb_keyframe_job make_kf_job(int stream, int frame_slot, int track_job) const {
        const EStream& s = st_[stream];
        ygzb_keyframe_job kj{};
        kj.stream = stream;
        kj.frame_slot = frame_slot;
        kj.track_job = track_job;
        // ring entry: one that none of the key-frames that stay local uses (the oldest of a full ring leaves the map)
        const int keep = std::min(kLocalKeyframes, (int)s.kfs.size());
        for (int e = 0; e < YGZB_TRACK_RING; ++e) {
            bool used = false;
            for (int k = 0; k < keep; ++k) used |= s.kfs[s.kfs.size() - 1 - k].entry == e;
            if (!used) {
                kj.entry = e;
                break;
            }
        }
        kj.kf_slot = S_ * F_ + stream * YGZB_TRACK_RING + kj.entry;
        const int nl = std::min(kLocalKeyframes, (int)s.kfs.size() + 1);
        kj.n_local = nl;
        for (int k = 0; k < nl - 1; ++k) kj.local_entry[k] = s.kfs[s.kfs.size() - (nl - 1) + k].entry;
        kj.local_entry[nl - 1] = kj.entry;
        kj.run_ba = (track_job >= 0 && nl >= 2) ? 1 : 0;
        kj.mp0 = s.next_mp;
        return kj;
    }

    ygzb_ctx* ctx_;
    ygzb_frames* fr_ = nullptr;
    ygzb_tracker* tr_ = nullptr;
    int S_, F_, W_ = 0, H_ = 0;
    Params prm_;
    std::vector<EStream> st_;
    ygzb_track_result* h_res_ = nullptr;
    ygzb_keyframe_result* h_kres_ = nullptr;
    ygzb_ba_params ba_;
    std::vector<Win> wins_;
    std::vector<ygzb_keyframe_job> kjobs_;   // key-frame insertions for the next round ...
    RowQueue<KfFrame, ygzb_observation> kframes_;   // ... and their frames, with their observation rows
    std::vector<int> order_;
    // the source the tracker has of every stream, as use_source last set it: its camera (ygzb_tracker_set_camera), the lens
    // its maps were built for with that camera (ygzb_tracker_set_undistort) and its raw frame format (ygzb_tracker_set_source)
    std::vector<Source> tr_src_;
    std::vector<int16_t> map_xy_;  // host maps of use_source, built for lens maps_lens_ seen through camera maps_K_ (lens off: none)
    std::vector<uint16_t> map_a_;
    Lens maps_lens_;
    Camera maps_K_{};
    double* traj_ = nullptr;
    int traj_frames_ = 0;
    bool collect_ = false;
    RowQueue<Result, ygzb_observation> results_;   // final results waiting to be polled, with their observation rows
    RowQueue<ygz_vo_map_update, ygzb_map_point> updates_;   // map updates waiting to be polled, with their rows
    // the tracker's page-locked outputs: observation rows (set_observations), information records (set_information) and
    // map rows (set_map_updates)
    size_t ring_cells_ = 0;   // YGZB_TRACK_RING * cells: the rows of a tracking job or a key-frame job
    PinnedOutput<ygzb_observation> obs_;
    PinnedOutput<ygzb_pose_information> info_;
    PinnedOutput<ygzb_map_point> map_;
    bool blocking_sync_ = false;
};

// host arrays behind a map record of up to YGZB_TRACK_RING key-frames (ygzb_map_record capacities)
struct MapBuf {
    std::vector<int32_t> entry, n_features, n_obs;
    std::vector<int64_t> mp0, obs_id;
    std::vector<double> T, px, depth, pw, obs_px;
    std::vector<uint8_t> level, image;
    ygzb_map_record rec{};
    MapBuf(int cells, int w, int h) {
        const size_t R = YGZB_TRACK_RING, F = R * cells, O = R * YGZB_MAP_OBS_PER_CELL * cells;
        entry.resize(R); n_features.resize(R); n_obs.resize(R); mp0.resize(R); T.resize(12 * R); image.resize(R * w * h);
        px.resize(2 * F); level.resize(F); depth.resize(F); pw.resize(3 * F); obs_id.resize(O); obs_px.resize(2 * O);
        rec.entry = entry.data(); rec.T_cw = T.data(); rec.mp0 = mp0.data(); rec.n_features = n_features.data(); rec.n_obs = n_obs.data();
        rec.image = image.data(); rec.px = px.data(); rec.level = level.data(); rec.depth = depth.data(); rec.pw = pw.data();
        rec.obs_id = obs_id.data(); rec.obs_px = obs_px.data();
    }
};

// host arrays behind a reference record (ygzb_reference_record capacity)
struct RefBuf {
    std::vector<double> px, depth;
    std::vector<uint8_t> image;
    ygzb_reference_record rec{};
    RefBuf(int cells, int w, int h) {
        const size_t cap = (size_t)YGZB_TRACK_REF_FEATURES_PER_CELL * cells;
        px.resize(2 * cap); depth.resize(cap); image.resize((size_t)w * h);
        rec.capacity = (int32_t)cap;
        rec.px = px.data(); rec.depth = depth.data(); rec.image = image.data();
    }
};

// ---- stream records (ygz_vo_save_stream / ygz_vo_load_stream; the layout is documented in include/ygz_vo.h) ------------
static_assert(std::endian::native == std::endian::little, "stream records are little-endian and copied field by field");
constexpr uint8_t kRecordMagic[4] = {'Y', 'G', 'Z', 'S'};

// what a record is made under and must be loaded under: the engine's image size, grid, pyramid and reference mode, and the
// stream's source
struct RecordGeom {
    int32_t width, height, cells, n_levels, ref_mode;
    Source src{};   // (save and load set it; read_record's is the record's)
    size_t wh() const { return (size_t)width * height; }
    Format default_fmt() const { return {width, height, 1}; }
};
constexpr size_t kRecordLensBytes = 9 * sizeof(double);   // version 2's lens block: K[4], dist[5]
constexpr size_t kRecordFormatBytes = 4 * sizeof(int32_t);   // version 3's format block: width, height, channels, has_lens

// the largest record of an engine whose streams are `st`: a full ring at capacity, a full reference, a depth map (the
// sections of write_record), with a lens block while some stream has a lens and a format block while some stream has a
// format other than the default, now or for its next sequence
size_t record_bound(const RecordGeom& g, const std::vector<EStream>& st) {
    bool lens = false, fmt = false;
    for (const EStream& s : st) {
        lens |= s.src.lens.on;
        fmt |= s.src.fmt != g.default_fmt();
    }
    const size_t R = YGZB_TRACK_RING, F = R * g.cells, O = R * YGZB_MAP_OBS_PER_CELL * g.cells;
    const size_t C = (size_t)YGZB_TRACK_REF_FEATURES_PER_CELL * g.cells, WH = g.wh();
    return 68 + (fmt ? kRecordFormatBytes : 0) + (lens ? kRecordLensBytes : 0)   // header, format, lens
           + (4 + R * 116 + 2 * 96 + 4 + 16 + 12 * 8)           // host state
           + (4 + R * (116 + WH) + F * 49 + O * 24)             // map
           + (4 + 96 + C * 24 + WH)                             // reference
           + WH * sizeof(double);                               // depth map
}

// appends fields to `out`; out == nullptr only counts the bytes
struct RecordWriter {
    uint8_t* out;
    size_t n = 0;
    void bytes(const void* src, size_t k) {
        if (out && k) std::memcpy(out + n, src, k);
        n += k;
    }
    template <typename T> void put(T v) { bytes(&v, sizeof v); }
};

// reads fields from in[0, size); a read past the end clears ok and reads nothing from then on
struct RecordReader {
    const uint8_t* in;
    size_t size, n = 0;
    bool ok = true;
    void bytes(void* dst, size_t k) {
        if (!ok || k > size - n) {
            ok = false;
            return;
        }
        if (k) std::memcpy(dst, in + n, k);
        n += k;
    }
    template <typename T> T get() {
        T v{};
        bytes(&v, sizeof v);
        return v;
    }
};

// the version of a record of the stream's source g.src: 3 with a format other than the default, else 2 with a lens, else 1
uint32_t record_version(const RecordGeom& g) {
    if (g.src.fmt != g.default_fmt()) return YGZ_VO_STREAM_RECORD_VERSION_FORMAT;
    return g.src.lens.on ? YGZ_VO_STREAM_RECORD_VERSION_LENS : YGZ_VO_STREAM_RECORD_VERSION;
}
// the header's blocks behind the reference mode: the format block (version 3), then the lens block (with a lens)
void write_source_blocks(RecordWriter& w, const RecordGeom& g) {
    const Source& s = g.src;
    if (record_version(g) == YGZ_VO_STREAM_RECORD_VERSION_FORMAT) {
        w.put<int32_t>(s.fmt.w); w.put<int32_t>(s.fmt.h); w.put<int32_t>(s.fmt.channels); w.put<int32_t>(s.lens.on);
    }
    if (s.lens.on) {
        w.bytes(s.lens.K.data(), sizeof s.lens.K);
        w.bytes(s.lens.dist.data(), sizeof s.lens.dist);
    }
}
// reads the blocks of a record of `version` into rg.src (whose camera is read already): false unless they are well formed
// and the record's version is that of the source they give (a default format is always written as version 1 or 2)
bool read_source_blocks(RecordReader& r, uint32_t version, RecordGeom& rg) {
    Source& s = rg.src;
    s.lens.on = version == YGZ_VO_STREAM_RECORD_VERSION_LENS;
    s.fmt = rg.default_fmt();
    if (version == YGZ_VO_STREAM_RECORD_VERSION_FORMAT) {
        s.fmt.w = r.get<int32_t>(); s.fmt.h = r.get<int32_t>(); s.fmt.channels = r.get<int32_t>();
        const int32_t has_lens = r.get<int32_t>();
        if (has_lens != 0 && has_lens != 1) return false;
        s.lens.on = has_lens;
    }
    if (s.lens.on) {
        r.bytes(s.lens.K.data(), sizeof s.lens.K);
        r.bytes(s.lens.dist.data(), sizeof s.lens.dist);
    }
    return r.ok && record_version(rg) == version;
}

// the record of stream `s` with its map `m` (exported from the ring entries of s.kfs), its reference `r` (previous-frame
// mode once it has a key-frame, else NULL) and its depth map (NULL unless s.has_depth)
void write_record(RecordWriter& w, const RecordGeom& g, const EStream& s, const ygzb_map_record& m, const ygzb_reference_record* r,
                  const double* depth) {
    const size_t WH = g.wh();
    // 1. header (the size is written last)
    w.bytes(kRecordMagic, 4);
    w.put<uint32_t>(record_version(g));
    const size_t size_at = w.n;
    w.put<uint64_t>(0);
    w.put<int32_t>(g.width); w.put<int32_t>(g.height); w.put<int32_t>(g.cells); w.put<int32_t>(g.n_levels);
    w.bytes(g.src.K.data(), sizeof g.src.K);
    w.put<int32_t>(g.ref_mode);
    write_source_blocks(w, g);
    // 2. host state
    w.put<int32_t>((int32_t)s.kfs.size());
    for (const KfInfo& kf : s.kfs) {
        w.put<int32_t>(kf.entry); w.put<int32_t>(kf.n); w.put<int32_t>(kf.frame_id); w.put<int64_t>(kf.mp0);
        w.bytes(kf.T.m, sizeof kf.T.m);
    }
    w.bytes(s.T.m, sizeof s.T.m);
    w.bytes(s.start.m, sizeof s.start.m);
    w.put<uint8_t>(s.restart_pending); w.put<uint8_t>(s.has_pose); w.put<uint8_t>(s.lost); w.put<uint8_t>(s.has_depth);
    w.put<int32_t>(s.frames_since_kf); w.put<int32_t>(s.next_frame); w.put<int64_t>(s.next_mp);
    for (long c : {s.n_keyframes, s.n_ba, s.n_candidates, s.n_projected, s.n_inliers, s.ba_obs, s.ba_pts, s.ba_kfs, s.ba_trials, s.ba_iters,
                   s.n_restarts})
        w.put<int64_t>(c);
    w.put<double>(s.ba_flops);
    // 3. map: per key-frame, then the live rows
    w.put<int32_t>(m.n_keyframes);
    size_t F = 0, O = 0;
    for (int k = 0; k < m.n_keyframes; ++k) {
        w.put<int32_t>(m.entry[k]); w.put<int32_t>(m.n_features[k]); w.put<int32_t>(m.n_obs[k]); w.put<int64_t>(m.mp0[k]);
        w.bytes(m.T_cw + 12 * (size_t)k, 12 * sizeof(double));
        w.bytes(m.image + k * WH, WH);
        F += (size_t)m.n_features[k];
        O += (size_t)m.n_obs[k];
    }
    w.bytes(m.px, F * 2 * sizeof(double)); w.bytes(m.level, F); w.bytes(m.depth, F * sizeof(double)); w.bytes(m.pw, F * 3 * sizeof(double));
    w.bytes(m.obs_id, O * sizeof(int64_t)); w.bytes(m.obs_px, O * 2 * sizeof(double));
    // 4. reference
    if (r) {
        w.put<int32_t>(r->n);
        w.bytes(r->T_cw, sizeof r->T_cw);
        w.bytes(r->px, (size_t)r->n * 2 * sizeof(double)); w.bytes(r->depth, (size_t)r->n * sizeof(double)); w.bytes(r->image, WH);
    }
    // 5. depth map
    if (depth) w.bytes(depth, WH * sizeof(double));
    if (w.out) {
        const uint64_t size = w.n;
        std::memcpy(w.out + size_at, &size, sizeof size);
    }
}

// a record unpacked into what Engine::adopt takes: the stream's bookkeeping, its map and reference records, its depth map
struct StreamRecord {
    EStream s;
    MapBuf map;
    RefBuf ref;
    bool has_ref = false;
    std::vector<double> depth;
    explicit StreamRecord(const RecordGeom& g) : map(g.cells, g.width, g.height), ref(g.cells, g.width, g.height) {}
};

// unpacks and checks the whole record in[0, size) against the engine's geometry `g`: YGZB_ERR_INVALID for anything but
// a well-formed record of that geometry whose counts, entries and levels are in range
int read_record(const uint8_t* in, size_t size, const RecordGeom& g, StreamRecord& out) {
    RecordReader r{in, size};
    const size_t WH = g.wh();
    // 1. header
    uint8_t magic[4];
    r.bytes(magic, 4);
    const uint32_t version = r.get<uint32_t>();
    const uint64_t total = r.get<uint64_t>();
    RecordGeom rg{};
    rg.width = r.get<int32_t>(); rg.height = r.get<int32_t>(); rg.cells = r.get<int32_t>(); rg.n_levels = r.get<int32_t>();
    r.bytes(rg.src.K.data(), sizeof rg.src.K);
    rg.ref_mode = r.get<int32_t>();
    if (!r.ok || std::memcmp(magic, kRecordMagic, 4) != 0 || total != size) return YGZB_ERR_INVALID;
    if (!read_source_blocks(r, version, rg)) return YGZB_ERR_INVALID;
    if (rg.width != g.width || rg.height != g.height || rg.cells != g.cells || rg.n_levels != g.n_levels || rg.ref_mode != g.ref_mode ||
        rg.src != g.src)   // K and the lens bit for bit
        return YGZB_ERR_INVALID;
    // 2. host state
    EStream& s = out.s;
    const int32_t n_kf = r.get<int32_t>();
    if (!r.ok || n_kf < 0 || n_kf > YGZB_TRACK_RING) return YGZB_ERR_INVALID;
    for (int k = 0; k < n_kf; ++k) {
        KfInfo kf;
        kf.entry = r.get<int32_t>(); kf.n = r.get<int32_t>(); kf.frame_id = r.get<int32_t>(); kf.mp0 = (long)r.get<int64_t>();
        r.bytes(kf.T.m, sizeof kf.T.m);
        if (kf.entry < 0 || kf.entry >= YGZB_TRACK_RING || kf.n < 0 || kf.n > g.cells || kf.frame_id < 0 || kf.mp0 < 0) return YGZB_ERR_INVALID;
        for (const KfInfo& o : s.kfs)
            if (o.entry == kf.entry) return YGZB_ERR_INVALID;
        if (!s.kfs.empty() && kf.frame_id <= s.kfs.back().frame_id) return YGZB_ERR_INVALID;   // oldest first
        s.kfs.push_back(kf);
    }
    r.bytes(s.T.m, sizeof s.T.m);
    r.bytes(s.start.m, sizeof s.start.m);
    uint8_t flags[4];
    r.bytes(flags, 4);
    for (uint8_t f : flags)
        if (f > 1) return YGZB_ERR_INVALID;
    s.restart_pending = flags[0]; s.has_pose = flags[1]; s.lost = flags[2]; s.has_depth = flags[3];
    s.frames_since_kf = r.get<int32_t>(); s.next_frame = r.get<int32_t>(); s.next_mp = (long)r.get<int64_t>();
    if (s.frames_since_kf < 0 || s.next_frame < 0 || s.next_mp < 0) return YGZB_ERR_INVALID;
    // a state a settled stream can have (the round and push rely on it: a stream's first push queues its start pose, and
    // a stream with key-frames tracks against them):
    //  - no key-frame: never pushed -- no frame, flag, depth map or map point yet (a restart before the first push only
    //    sets `start`);
    //  - key-frames: their frames lie before the next one, a pose and a depth map (the first frame brought one), frames
    //    tracked since the newest key-frame at most the frames after it, and the next map point id right behind its points
    if (s.kfs.empty()) {
        if (s.next_frame != 0 || s.frames_since_kf != 0 || s.next_mp != 0 || s.restart_pending || s.has_pose || s.lost || s.has_depth)
            return YGZB_ERR_INVALID;
    } else {
        const KfInfo& kf = s.kfs.back();
        if (s.next_frame <= kf.frame_id || !s.has_pose || !s.has_depth || s.frames_since_kf > s.next_frame - 1 - kf.frame_id ||
            s.next_mp != kf.mp0 + kf.n)
            return YGZB_ERR_INVALID;
    }
    for (long* c : {&s.n_keyframes, &s.n_ba, &s.n_candidates, &s.n_projected, &s.n_inliers, &s.ba_obs, &s.ba_pts, &s.ba_kfs, &s.ba_trials,
                    &s.ba_iters, &s.n_restarts})
        *c = (long)r.get<int64_t>();
    s.ba_flops = r.get<double>();
    // 3. map: the key-frames of the host state, in the same order
    ygzb_map_record& m = out.map.rec;
    m.width = g.width; m.height = g.height; m.cells = g.cells; m.n_levels = g.n_levels;
    std::memcpy(m.K, g.src.K.data(), sizeof m.K);
    m.n_keyframes = r.get<int32_t>();
    if (!r.ok || m.n_keyframes != n_kf) return YGZB_ERR_INVALID;
    size_t F = 0, O = 0;
    for (int k = 0; k < n_kf; ++k) {
        m.entry[k] = r.get<int32_t>(); m.n_features[k] = r.get<int32_t>(); m.n_obs[k] = r.get<int32_t>(); m.mp0[k] = r.get<int64_t>();
        r.bytes(m.T_cw + 12 * (size_t)k, 12 * sizeof(double));
        r.bytes(m.image + k * WH, WH);
        if (m.entry[k] != s.kfs[k].entry || m.n_features[k] != s.kfs[k].n || m.mp0[k] != s.kfs[k].mp0 || m.n_obs[k] < 0 ||
            m.n_obs[k] > YGZB_MAP_OBS_PER_CELL * g.cells)
            return YGZB_ERR_INVALID;
        F += (size_t)m.n_features[k];
        O += (size_t)m.n_obs[k];
    }
    r.bytes(m.px, F * 2 * sizeof(double)); r.bytes(m.level, F); r.bytes(m.depth, F * sizeof(double)); r.bytes(m.pw, F * 3 * sizeof(double));
    r.bytes(m.obs_id, O * sizeof(int64_t)); r.bytes(m.obs_px, O * 2 * sizeof(double));
    if (!r.ok) return YGZB_ERR_INVALID;
    for (size_t q = 0; q < F; ++q)
        if (m.level[q] >= g.n_levels) return YGZB_ERR_INVALID;
    // 4. reference: what a stream tracked against the previous frame aligns its next frame against, once it has one
    out.has_ref = g.ref_mode == YGZB_TRACK_REF_PREVIOUS && n_kf > 0;
    if (out.has_ref) {
        ygzb_reference_record& q = out.ref.rec;
        q.width = g.width; q.height = g.height; q.cells = g.cells; q.n_levels = g.n_levels;
        std::memcpy(q.K, g.src.K.data(), sizeof q.K);
        q.n = r.get<int32_t>();
        if (!r.ok || q.n < 0 || q.n > q.capacity) return YGZB_ERR_INVALID;
        r.bytes(q.T_cw, sizeof q.T_cw);
        r.bytes(q.px, (size_t)q.n * 2 * sizeof(double)); r.bytes(q.depth, (size_t)q.n * sizeof(double)); r.bytes(q.image, WH);
    }
    // 5. depth map
    if (s.has_depth) {
        out.depth.resize(WH);
        r.bytes(out.depth.data(), WH * sizeof(double));
    }
    return r.ok && r.n == size ? YGZB_OK : YGZB_ERR_INVALID;
}

// page-locked staging of ygz_vo_save_stream, allocated on its first call: a map record at full capacity, a reference
// record and a depth map in one ygzb_host_alloc, so that the exports copy straight into host memory
struct SaveStage {
    void* mem = nullptr;
    ygzb_map_record map{};
    ygzb_reference_record ref{};
    double* depth = nullptr;
    SaveStage() = default;
    SaveStage(const SaveStage&) = delete;
    SaveStage& operator=(const SaveStage&) = delete;
    ~SaveStage() {
        if (mem) ygzb_host_free(mem);
    }
    int init(const RecordGeom& g) {
        size_t bytes = carve(g, nullptr);
        CHK(ygzb_host_alloc(&mem, bytes));
        carve(g, static_cast<uint8_t*>(mem));
        return YGZB_OK;
    }

  private:
    // lays the arrays out from base (nullptr: only sizes them), 8-byte aligned; returns the bytes
    size_t carve(const RecordGeom& g, uint8_t* base) {
        const size_t R = YGZB_TRACK_RING, F = R * g.cells, O = R * YGZB_MAP_OBS_PER_CELL * g.cells;
        const size_t C = (size_t)YGZB_TRACK_REF_FEATURES_PER_CELL * g.cells, WH = g.wh();
        size_t off = 0;
        auto take = [&](auto*& p, size_t count) {
            off = (off + 7) & ~(size_t)7;
            p = base ? reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + off) : nullptr;
            off += count * sizeof(*p);
        };
        take(map.T_cw, 12 * R); take(map.mp0, R); take(map.px, 2 * F); take(map.depth, F); take(map.pw, 3 * F); take(map.obs_id, O);
        take(map.obs_px, 2 * O); take(map.entry, R); take(map.n_features, R); take(map.n_obs, R); take(map.level, F); take(map.image, R * WH);
        take(ref.px, 2 * C); take(ref.depth, C); take(ref.image, WH);
        take(depth, WH);
        ref.capacity = (int32_t)C;
        return off;
    }
};

// A batch of the resident engine (run_engine): what every host thread reads
struct EngineBatch {
    int device, n_frames, window, handoff;   // handoff < 0: no hand-over
    const ygzb_params* params;
    const uint8_t* const* images;
    const double* const* depth;
    ygzb_map_record* maps;
    ygzb_reference_record* refs;
    double* traj;
    Params prm;
};

// The streams [s0, s0 + ns) of a batch that one host thread tracks, on its own engine and context (a hand-over replaces both)
struct EngineGroup {
    const EngineBatch& b;
    const int s0, ns;
    std::array<long long, 4>& tot;   // the thread's totals of the timed region
    ygzb_ctx* ctx;
    bool own_ctx = false, handed = false;
    int rc = YGZB_OK;
    std::unique_ptr<Engine> eng;
    long long launch_base = 0;

    EngineGroup(const EngineBatch& batch, int first, int end, ygzb_ctx* caller, bool create, std::array<long long, 4>& totals)
        : b(batch), s0(first), ns(end - first), tot(totals), ctx(caller) {
        open(create);
    }
    ~EngineGroup() { close(); }
    // a new engine (with the stream order `order`, if given) on ctx, or on a context it creates first
    void open(bool create, const std::vector<int>* order = nullptr) {
        own_ctx = create;
        if (create) rc = ygzb_create(b.device, b.params, &ctx);
        eng = std::make_unique<Engine>(ctx, ns, b.window, b.prm);
        eng->set_outputs(b.traj + (size_t)s0 * b.n_frames * 12, b.n_frames, false);
        if (order) eng->set_order(*order);
        if (rc != YGZB_OK) return;
        launch_base = ygzb_launch_count(ctx);
        rc = eng->init(b.depth + s0);
    }
    void close() {
        eng.reset();   // the engine releases its tracker and frame slots before the context goes
        if (own_ctx && ctx) ygzb_destroy(ctx);
        ctx = nullptr;
    }
    // runs the streams to frame `limit`; the hand-over comes first when its frame lies before `limit` (or at the end)
    void advance(int limit) {
        if (rc == YGZB_OK && b.handoff >= 0 && !handed && (b.handoff < limit || limit == b.n_frames)) {
            handed = true;
            rc = hand_over();
        }
        if (rc == YGZB_OK) rc = eng->run_until(b.images + s0, limit);
    }
    // adds the launches and bytes of the current engine since the last count to tot, and counts from zero again
    void count() {
        tot[0] += ctx ? ygzb_launch_count(ctx) - launch_base : 0;
        tot[1] += eng->h2d_image_bytes; tot[2] += eng->h2d_other_bytes; tot[3] += eng->d2h_bytes;
        launch_base = ygzb_launch_count(ctx);
        eng->h2d_image_bytes = eng->h2d_other_bytes = eng->d2h_bytes = 0;
    }
    // run to frame `handoff`, export every stream's map (and in previous-frame mode its reference), tear the tracker, its
    // frame pool and (but for the caller's) the context down, and carry the streams over to a fresh engine on a new context
    // in reverse order
    int hand_over() {
        CHK(eng->run_until(b.images + s0, b.handoff));
        int cells_r = 0, cells_c = 0;
        ygzb_grid_dims(ctx, &cells_r, &cells_c);
        std::vector<MapBuf> own;
        std::vector<RefBuf> own_refs;
        std::vector<ygzb_map_record*> recs(ns);
        std::vector<ygzb_reference_record*> ref_recs(ns, nullptr);
        if (!b.maps) own.reserve(ns);
        if (!b.refs) own_refs.reserve(ns);
        for (int i = 0; i < ns; ++i) {
            if (b.maps) {
                recs[i] = b.maps + s0 + eng->order()[i];
            } else {
                own.emplace_back(cells_r * cells_c, eng->width(), eng->height());
                recs[i] = &own.back().rec;
            }
            CHK(eng->export_map(i, recs[i]));
            if (!eng->has_reference(i)) continue;
            if (b.refs) {
                ref_recs[i] = b.refs + s0 + eng->order()[i];
            } else {
                own_refs.emplace_back(cells_r * cells_c, eng->width(), eng->height());
                ref_recs[i] = &own_refs.back().rec;
            }
            CHK(eng->export_reference(i, ref_recs[i]));
        }
        CHK(ygzb_synchronize(ctx));
        const std::vector<EStream> carried = eng->streams();
        const std::vector<int> reversed(eng->order().rbegin(), eng->order().rend());
        count();
        close();
        open(true, &reversed);
        CHK(rc);
        for (int j = 0; j < ns; ++j) CHK(eng->adopt(j, carried[ns - 1 - j], recs[ns - 1 - j], ref_recs[ns - 1 - j]));
        return YGZB_OK;
    }
};

// Device-resident engine over the streams of each host thread; with handoff >= 0 the streams move to a new tracker at frame
// `handoff` (see ygz_vo_run_handoff_ex).  Shared by ygz_vo_run(_ex) (handoff < 0) and ygz_vo_run_handoff(_ex).
int run_engine(ygzb_ctx* ctx, int n_threads, int n_streams, int warm, EngineBatch b, int64_t* stats, double* seconds, double* device_ms,
               int64_t* totals) {
    if (b.prm.ref_mode != YGZB_TRACK_REF_KEYFRAME && b.prm.ref_mode != YGZB_TRACK_REF_PREVIOUS) return YGZB_ERR_INVALID;
    if (!ctx || !b.params || n_streams < 1 || b.n_frames < 1 || !b.images || !b.depth || !b.traj || !stats || !seconds) return YGZB_ERR_INVALID;
    n_threads = std::max(1, std::min(n_threads, n_streams));
    warm = std::max(0, std::min(warm, b.n_frames - 1));
    if (b.handoff >= 0) b.handoff = std::min(b.handoff, b.n_frames);
    TimedThreads threads(n_threads);
    const int rc = threads.run([&](int t) {
        EngineGroup g(b, (int)((long)n_streams * t / n_threads), (int)((long)n_streams * (t + 1) / n_threads), ctx, t > 0, threads.tot[t]);
        g.advance(warm);
        g.count();
        g.tot = {};   // the totals of the timed region start here
        threads.begin(t, g.rc, g.ctx, ctx);
        if (t == 0)
            for (auto& v : g_stage_ns) v.store(0);
        g.advance(b.n_frames);
        threads.end(t, g.rc, g.ctx, ctx, device_ms);
        g.count();
        for (int s = 0; s < g.ns; ++s) g.eng->stats(s, stats + 16 * (size_t)(g.s0 + g.eng->order()[s]));
        return g.rc;
    }, seconds, totals, 8);
    if (getenv("YGZ_VO_TIMING")) {
        const int timed = b.n_frames - warm;
        fprintf(stderr, "[ygz_vo engine] %d streams on %d host threads, window %d, %d timed frames: %.3f ms per frame index; track rounds %.3f ms, "
                        "key-frame rounds %.3f ms (host wall, summed over threads)\n",
                n_streams, n_threads, b.window, timed, 1e3 * *seconds / timed, 1e-6 * g_stage_ns[kTSparse].load(), 1e-6 * g_stage_ns[kTLocalBA].load());
    }
    return rc;
}

}  // namespace

// ---- streaming API (include/ygz_vo.h): the resident engine fed frame by frame --------------------------------------------
struct ygz_vo {
    ygzb_ctx* ctx;
    int n_streams, width, height;
    std::unique_ptr<Engine> eng;
    RecordGeom geom{};   // what this engine's stream records are made under
    SaveStage stage;     // staging of ygz_vo_save_stream (allocated on its first call)
};

extern "C" {

// PER-STAGE PATH: every numeric step is one blocking C-ABI call with host buffers (the reference's call granularity);
// kept as the cross-check of the device-resident engine below (tests/test_vo.py) and as a diagnostic of bench.py.
// Tracks n_streams independent 640x480 grey streams in lock step for n_frames frames.  The streams are split over
// n_threads host threads; thread 0 drives the caller's context, every further thread creates its own context (= its
// own CUDA stream) on the same device with the same parameters, so the kernels of one group overlap the host work and
// the kernels of the others.  The contexts must use the 3-level pyramid of the reference default.
//   images[s] : n_frames * 480 * 640 bytes, depth[s] : 480 * 640 doubles (static ground-truth depth of stream s)
//   traj      : n_streams * n_frames * 12 doubles out (T_cw after every frame; NaN while a stream has no pose)
//   stats     : n_streams * 16 out: lost, keyframes, local BAs, candidates, projected, inliers, BA observations, BA points,
//               BA key-frames, BA LM trials, BA iterations, BA model FLOP (SURVEY 8d), 0...
//   totals    : (may be NULL) 8 out, timed region only, summed over the host threads: kernel launches, image H2D bytes,
//               other H2D bytes, D2H bytes, 0...
//   seconds   : wall time of frames [warm, n_frames) including the final device synchronisation (all threads meet at a
//               barrier before frame `warm` and after the last frame)
//   device_ms : (may be NULL) the same region timed with CUDA events on the caller's context stream: first event after
//               the warm-up barrier, second one after every thread has synchronised its stream
int ygz_vo_run_stages(ygzb_ctx* ctx, int device, const ygzb_params* params, int n_threads, int n_streams, int n_frames,
               const uint8_t* const* images, const double* const* depth, int kf_min_frames, double kf_min_rot, double kf_min_trans,
               int warm, double* traj, int64_t* stats, double* seconds, double* device_ms, int64_t* totals) {
    if (!ctx || !params || n_streams < 1 || n_frames < 1 || !images || !depth || !traj || !stats || !seconds) return YGZB_ERR_INVALID;
    n_threads = std::max(1, std::min(n_threads, n_streams));
    warm = std::max(0, std::min(warm, n_frames - 1));
    TimedThreads threads(n_threads);
    const int rc = threads.run([&](int t) {
        const int s0 = (int)((long)n_streams * t / n_threads), s1 = (int)((long)n_streams * (t + 1) / n_threads), ns = s1 - s0;
        ygzb_ctx* my = ctx;
        int rc = YGZB_OK;
        if (t > 0) rc = ygzb_create(device, params, &my);
        ygzb_frames* fr = nullptr;
        if (rc == YGZB_OK) rc = ygzb_frames_create(my, ns * kSlotsPerStream, &fr);
        Driver drv(my, fr, ns, Params{kf_min_frames, kf_min_rot, kf_min_trans});
        std::vector<const uint8_t*> img(ns);
        for (int k = 0; k < n_frames; ++k) {
            if (k == warm) {
                threads.tot[t][0] = -ygzb_launch_count(my);
                drv.h2d_image_bytes = drv.h2d_other_bytes = drv.d2h_bytes = 0;
                threads.begin(t, rc, my, ctx);   // device time of the timed region: CUDA events on the caller's context stream
                if (t == 0)
                    for (auto& v : g_stage_ns) v.store(0);
            }
            if (rc != YGZB_OK) continue;   // keep meeting the barriers
            for (int s = 0; s < ns; ++s) img[s] = images[s0 + s] + (size_t)k * W * H;
            rc = drv.add_frames(img.data(), depth + s0, k);
            for (int s = 0; s < ns; ++s) {
                double* out = traj + ((size_t)(s0 + s) * n_frames + k) * 12;
                const Stream& st = drv.streams()[s];
                for (int c = 0; c < 12; ++c) out[c] = st.has_pose ? st.T.m[c] : NAN;
            }
        }
        threads.end(t, rc, my, ctx, device_ms);
        threads.tot[t] = {threads.tot[t][0] + ygzb_launch_count(my), drv.h2d_image_bytes, drv.h2d_other_bytes, drv.d2h_bytes};
        for (int s = 0; s < ns; ++s) drv.streams()[s].write_stats(drv.streams()[s].lost, stats + 16 * (size_t)(s0 + s));
        if (fr) ygzb_frames_destroy(fr);
        if (t > 0 && my) ygzb_destroy(my);
        return rc;
    }, seconds, totals, 8);
    if (getenv("YGZ_VO_TIMING")) {
        static const char* names[kTStages] = {"upload", "sparse_align", "project_align", "pose_only", "detect", "local_ba"};
        double sum = 0;
        for (int i = 0; i < kTStages; ++i) sum += 1e-9 * g_stage_ns[i].load();
        const int timed = n_frames - warm;
        fprintf(stderr, "[ygz_vo] %d streams on %d host threads x %d timed frames: %.3f ms per lock-step frame; C-ABI time summed over threads %.3f ms\n",
                n_streams, n_threads, timed, 1e3 * *seconds / timed, 1e3 * sum / timed);
        for (int i = 0; i < kTStages; ++i) fprintf(stderr, "[ygz_vo]   %-14s %.3f ms/frame\n", names[i], 1e-6 * g_stage_ns[i].load() / timed);
    }
    return rc;
}

// Device-resident engine (see Engine above).  Same arguments as ygz_vo_run_stages plus
//   window : frames of one stream that may be in flight in one round (1 = one frame at a time, the latency mode);
// frames [0, warm) are processed before the timed region starts (no window crosses frame `warm`).
int ygz_vo_run(ygzb_ctx* ctx, int device, const ygzb_params* params, int n_threads, int n_streams, int n_frames,
               const uint8_t* const* images, const double* const* depth, int kf_min_frames, double kf_min_rot, double kf_min_trans,
               int warm, int window, double* traj, int64_t* stats, double* seconds, double* device_ms, int64_t* totals) {
    return run_engine(ctx, n_threads, n_streams, warm, {device, n_frames, window, -1, params, images, depth, nullptr, nullptr, traj,
                      {kf_min_frames, kf_min_rot, kf_min_trans, YGZB_TRACK_REF_KEYFRAME}}, stats, seconds, device_ms, totals);
}

// ygz_vo_run with the tracker's reference mode: YGZB_TRACK_REF_KEYFRAME (= ygz_vo_run) or YGZB_TRACK_REF_PREVIOUS, the
// reference's rule of aligning each frame against the previous one (one extra frame slot per stream holds its pyramid).
// Windows are planned as in ygz_vo_run; the frames of a window then form a dependent chain on the device.
int ygz_vo_run_ex(ygzb_ctx* ctx, int device, const ygzb_params* params, int n_threads, int n_streams, int n_frames,
                  const uint8_t* const* images, const double* const* depth, int kf_min_frames, double kf_min_rot, double kf_min_trans,
                  int warm, int window, double* traj, int64_t* stats, double* seconds, double* device_ms, int64_t* totals, int ref_mode) {
    return run_engine(ctx, n_threads, n_streams, warm, {device, n_frames, window, -1, params, images, depth, nullptr, nullptr, traj,
                      {kf_min_frames, kf_min_rot, kf_min_trans, ref_mode}}, stats, seconds, device_ms, totals);
}

// The device-resident engine with a hand-over of every stream to a new tracker: ygz_vo_run_ex's arguments plus
//   handoff : every host thread runs its streams to frame `handoff` (nothing in flight), exports each stream's key-frames
//             (ygzb_tracker_export) and, in YGZB_TRACK_REF_PREVIOUS mode, then its reference (ygzb_tracker_export_reference),
//             destroys its tracker and frame pool, creates a fresh tracker on a new context of the same device with the
//             stream order reversed (a stream changes its index), imports the maps (ygzb_tracker_import) and then the
//             references (ygzb_tracker_import_reference), takes the host-side bookkeeping over and runs on to the last frame;
//   maps    : NULL, or n_streams records (one per stream, each sized for YGZB_TRACK_RING key-frames, images included) that
//             receive the exported maps and are what the new tracker imports;
//   refs    : (previous-frame mode; unused in key-frame mode) NULL, or n_streams reference records (each with capacity >=
//             YGZB_TRACK_REF_FEATURES_PER_CELL * grid cells, px, depth and image set) that receive the exported references
//             and are what the new tracker imports.  A stream without a key-frame at the hand-over has no reference yet and
//             leaves its record as it was.
// Results equal those of ygz_vo_run_ex with warm = handoff, which splits the run at the same frame.  The hand-over's own
// record copies are not counted in `totals`.
int ygz_vo_run_handoff_ex(ygzb_ctx* ctx, int device, const ygzb_params* params, int n_threads, int n_streams, int n_frames,
                          const uint8_t* const* images, const double* const* depth, int kf_min_frames, double kf_min_rot, double kf_min_trans,
                          int warm, int window, int handoff, ygzb_map_record* maps, ygzb_reference_record* refs, double* traj, int64_t* stats,
                          double* seconds, double* device_ms, int64_t* totals, int ref_mode) {
    if (handoff < 0) return YGZB_ERR_INVALID;
    return run_engine(ctx, n_threads, n_streams, warm, {device, n_frames, window, handoff, params, images, depth, maps,
                      ref_mode == YGZB_TRACK_REF_PREVIOUS ? refs : nullptr, traj, {kf_min_frames, kf_min_rot, kf_min_trans, ref_mode}},
                      stats, seconds, device_ms, totals);
}

// ygz_vo_run_handoff_ex in key-frame mode, without reference records
int ygz_vo_run_handoff(ygzb_ctx* ctx, int device, const ygzb_params* params, int n_threads, int n_streams, int n_frames,
                       const uint8_t* const* images, const double* const* depth, int kf_min_frames, double kf_min_rot, double kf_min_trans,
                       int warm, int window, int handoff, ygzb_map_record* maps, double* traj, int64_t* stats, double* seconds,
                       double* device_ms, int64_t* totals) {
    return ygz_vo_run_handoff_ex(ctx, device, params, n_threads, n_streams, n_frames, images, depth, kf_min_frames, kf_min_rot, kf_min_trans,
                                 warm, window, handoff, maps, nullptr, traj, stats, seconds, device_ms, totals, YGZB_TRACK_REF_KEYFRAME);
}

int ygz_vo_create(ygzb_ctx* ctx, const ygz_vo_config* cfg, ygz_vo** out) {
    if (!out) return YGZB_ERR_INVALID;
    *out = nullptr;
    ygzb_params cp;
    if (!ctx || !cfg || ygzb_get_params(ctx, &cp) != YGZB_OK) return YGZB_ERR_INVALID;
    if (cfg->n_streams < 1 || cfg->window < 1 || cfg->kf_min_frames < 0 || cfg->min_inliers < 0 || !(cfg->kf_min_rot >= 0) ||
        !(cfg->kf_min_trans >= 0) || (cfg->ref_mode != YGZB_TRACK_REF_KEYFRAME && cfg->ref_mode != YGZB_TRACK_REF_PREVIOUS))
        return YGZB_ERR_INVALID;
    // the context's camera is float (PinholeCamera); the tracker projects with the caller's doubles, which must be that camera
    const float ck[4] = {cp.fx, cp.fy, cp.cx, cp.cy};
    for (int k = 0; k < 4; ++k)
        if (!std::isfinite(cfg->K[k]) || (float)cfg->K[k] != ck[k]) return YGZB_ERR_INVALID;
    if (!(cfg->K[0] > 0 && cfg->K[1] > 0)) return YGZB_ERR_INVALID;
    Params prm{cfg->kf_min_frames, cfg->kf_min_rot, cfg->kf_min_trans, cfg->ref_mode, cfg->min_inliers, {cfg->K[0], cfg->K[1], cfg->K[2], cfg->K[3]}};
    std::unique_ptr<ygz_vo> vo(new (std::nothrow) ygz_vo{ctx, cfg->n_streams, cp.image_width, cp.image_height, nullptr});
    if (!vo) return YGZB_ERR_INVALID;
    int rows = 0, cols = 0;
    CHK(ygzb_grid_dims(ctx, &rows, &cols));
    vo->geom = RecordGeom{cp.image_width, cp.image_height, rows * cols, cp.n_levels, cfg->ref_mode};
    vo->eng = std::make_unique<Engine>(ctx, cfg->n_streams, cfg->window, prm);
    vo->eng->set_outputs(nullptr, 0, true);
    CHK(vo->eng->init(nullptr));
    *out = vo.release();
    return YGZB_OK;
}

int ygz_vo_push(ygz_vo* vo, int stream, const uint8_t* image, const double* depth, int64_t tag) {
    if (!vo || stream < 0 || stream >= vo->n_streams || !image) return YGZB_ERR_INVALID;
    const EStream& s = vo->eng->streams()[stream];
    if (!depth && (!s.has_depth || s.restart_pending)) return YGZB_ERR_INVALID;
    // a sequence's first frame fixes its source
    const bool starts = vo->eng->pushed(stream) == 0 || s.restart_pending;
    if (starts && !s.src.pushable(vo->eng->width(), vo->eng->height())) return YGZB_ERR_INVALID;
    vo->eng->push(stream, image, depth, tag);
    return YGZB_OK;
}

int ygz_vo_restart(ygz_vo* vo, int stream, const double T_cw[12]) {
    if (!vo || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    Mat34 T = identity();
    if (T_cw) std::memcpy(T.m, T_cw, sizeof(T.m));
    return vo->eng->restart(stream, T);
}

int ygz_vo_set_camera(ygz_vo* vo, int stream, const double K[4]) {
    if (!vo || !K || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    for (int c = 0; c < 4; ++c)
        if (!std::isfinite(K[c])) return YGZB_ERR_INVALID;
    if (!(K[0] > 0 && K[1] > 0)) return YGZB_ERR_INVALID;
    Source src = vo->eng->source(stream);
    src.K = Camera{K[0], K[1], K[2], K[3]};
    return vo->eng->set_source(stream, src);
}

int ygz_vo_set_lens(ygz_vo* vo, int stream, const double K[4], const double dist[5]) {
    if (!vo || stream < 0 || stream >= vo->n_streams || !K != !dist) return YGZB_ERR_INVALID;
    Lens L;
    if (K) {
        for (int c = 0; c < 4; ++c)
            if (!std::isfinite(K[c])) return YGZB_ERR_INVALID;
        for (int c = 0; c < 5; ++c)
            if (!std::isfinite(dist[c])) return YGZB_ERR_INVALID;
        if (!(K[0] > 0 && K[1] > 0)) return YGZB_ERR_INVALID;
        L.on = true;
        std::copy_n(K, 4, L.K.begin());
        std::copy_n(dist, 5, L.dist.begin());
    }
    Source src = vo->eng->source(stream);
    src.lens = L;
    return vo->eng->set_source(stream, src);
}

int ygz_vo_get_lens(const ygz_vo* vo, int stream, int* has_lens, double K[4], double dist[5]) {
    if (!vo || !has_lens || !K || !dist || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    const Lens& L = vo->eng->source(stream).lens;
    *has_lens = L.on ? 1 : 0;
    std::copy(L.K.begin(), L.K.end(), K);   // (zeros without a lens)
    std::copy(L.dist.begin(), L.dist.end(), dist);
    return YGZB_OK;
}

int ygz_vo_set_frame_format(ygz_vo* vo, int stream, int width, int height, int channels) {
    if (!vo || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    if (width < 1 || height < 1 || width > 32767 || height > 32767 || (channels != 1 && channels != 3)) return YGZB_ERR_INVALID;
    Source src = vo->eng->source(stream);
    src.fmt = Format{width, height, channels};
    return vo->eng->set_source(stream, src);
}

int ygz_vo_get_frame_format(const ygz_vo* vo, int stream, int* width, int* height, int* channels) {
    if (!vo || !width || !height || !channels || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    const Format& F = vo->eng->source(stream).fmt;
    *width = F.w;
    *height = F.h;
    *channels = F.channels;
    return YGZB_OK;
}

int ygz_vo_get_camera(const ygz_vo* vo, int stream, double K[4]) {
    if (!vo || !K || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    const Camera& c = vo->eng->source(stream).K;
    std::copy(c.begin(), c.end(), K);
    return YGZB_OK;
}

int ygz_vo_step(ygz_vo* vo) {
    if (!vo) return YGZB_ERR_INVALID;
    bool idle = false;
    return vo->eng->round(&idle);
}

int ygz_vo_flush(ygz_vo* vo) {
    if (!vo) return YGZB_ERR_INVALID;
    return vo->eng->flush();
}

int ygz_vo_poll(ygz_vo* vo, ygz_vo_result* out, int capacity, int* n) {
    if (!vo || !n || capacity < 0 || (capacity > 0 && !out)) return YGZB_ERR_INVALID;
    *n = (int)vo->eng->pop_results(out, (size_t)capacity);
    return YGZB_OK;
}

int ygz_vo_set_observations(ygz_vo* vo, int on) {
    if (!vo || !vo->eng->idle()) return YGZB_ERR_INVALID;
    return vo->eng->set_observations(on != 0);
}

int ygz_vo_poll_observations(ygz_vo* vo, ygz_vo_result* out, int capacity, int* n, ygzb_observation* obs, size_t obs_capacity, size_t* n_obs) {
    if (!vo || !n || !n_obs || capacity < 0 || (capacity > 0 && !out) || (obs_capacity > 0 && !obs) || !vo->eng->observations())
        return YGZB_ERR_INVALID;
    return vo->eng->pop_results(out, capacity, n, nullptr, obs, obs_capacity, n_obs);
}

int ygz_vo_set_information(ygz_vo* vo, int on) {
    if (!vo || !vo->eng->idle()) return YGZB_ERR_INVALID;
    return vo->eng->set_information(on != 0);
}

int ygz_vo_poll_ex(ygz_vo* vo, ygz_vo_result* out, int capacity, int* n, ygzb_pose_information* info, ygzb_observation* obs,
                   size_t obs_capacity, size_t* n_obs) {
    if (!vo || !n || capacity < 0 || (capacity > 0 && !out)) return YGZB_ERR_INVALID;
    Engine& e = *vo->eng;
    if (e.information() != (info != nullptr)) return YGZB_ERR_INVALID;
    if (e.observations() ? (!n_obs || (obs_capacity > 0 && !obs)) : (obs || obs_capacity > 0)) return YGZB_ERR_INVALID;
    if (!e.observations() && n_obs) *n_obs = 0;
    return e.pop_results(out, capacity, n, info, obs, obs_capacity, n_obs);
}

int ygz_vo_set_map_updates(ygz_vo* vo, int on) {
    if (!vo || !vo->eng->idle()) return YGZB_ERR_INVALID;
    return vo->eng->set_map_updates(on != 0);
}

int ygz_vo_poll_map_updates(ygz_vo* vo, ygz_vo_map_update* out, int capacity, int* n, ygzb_map_point* rows, size_t row_capacity,
                            size_t* n_rows) {
    if (!vo || !n || !n_rows || capacity < 0 || (capacity > 0 && !out) || (row_capacity > 0 && !rows) || !vo->eng->map_updates())
        return YGZB_ERR_INVALID;
    return vo->eng->pop_map_updates(out, capacity, n, rows, row_capacity, n_rows);
}

int ygz_vo_stream_stats(ygz_vo* vo, int stream, int64_t stats[16]) {
    if (!vo || !stats || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    vo->eng->stats(stream, stats);
    return YGZB_OK;
}

int ygz_vo_export_map(ygz_vo* vo, int stream, ygzb_map_record* out) {
    if (!vo || !out || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    return vo->eng->export_map(stream, out);
}

int ygz_vo_stream_record_bound(const ygz_vo* vo, size_t* bytes) {
    if (!vo || !bytes) return YGZB_ERR_INVALID;
    *bytes = record_bound(vo->geom, vo->eng->streams());
    return YGZB_OK;
}

// the stream's map, reference and depth map into the page-locked staging, one synchronisation, then the live rows into
// the caller's buffer
int ygz_vo_save_stream(ygz_vo* vo, int stream, void* buf, size_t capacity, size_t* size) {
    if (!vo || !size || (!buf && capacity) || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    Engine& e = *vo->eng;
    if (!e.settled(stream)) return YGZB_ERR_INVALID;
    if (!vo->stage.mem) CHK(vo->stage.init(vo->geom));
    const EStream& s = e.streams()[stream];
    RecordGeom g = vo->geom;
    g.src = s.src;
    SaveStage& st = vo->stage;
    CHK(e.export_map(stream, &st.map));
    const bool ref = e.has_reference(stream);
    if (ref) CHK(e.export_reference(stream, &st.ref));
    if (s.has_depth) CHK(e.get_depth(stream, st.depth));
    CHK(ygzb_synchronize(vo->ctx));
    RecordWriter count{nullptr};
    write_record(count, g, s, st.map, ref ? &st.ref : nullptr, s.has_depth ? st.depth : nullptr);
    *size = count.n;
    if (count.n > capacity) return YGZB_ERR_CAPACITY;
    RecordWriter w{static_cast<uint8_t*>(buf)};
    write_record(w, g, s, st.map, ref ? &st.ref : nullptr, s.has_depth ? st.depth : nullptr);
    return YGZB_OK;
}

// the whole record is unpacked and checked first (read_record, then the start pose), so a record that fails leaves the
// stream as it was; then Engine::adopt installs it as it installs a stream handed over by the batch entry points
int ygz_vo_load_stream(ygz_vo* vo, int stream, const void* buf, size_t size) {
    if (!vo || !buf || stream < 0 || stream >= vo->n_streams) return YGZB_ERR_INVALID;
    Engine& e = *vo->eng;
    if (!e.settled(stream)) return YGZB_ERR_INVALID;
    RecordGeom g = vo->geom;
    g.src = e.source(stream);   // the record's source must be the destination stream's
    StreamRecord rec(g);
    CHK(read_record(static_cast<const uint8_t*>(buf), size, g, rec));
    rec.s.src = g.src;
    CHK(e.check_start_pose(stream, rec.s.start));
    CHK(e.adopt(stream, rec.s, &rec.map.rec, rec.has_ref ? &rec.ref.rec : nullptr));
    if (rec.s.has_depth) CHK(e.set_depth(stream, rec.depth.data()));
    return YGZB_OK;
}

void ygz_vo_destroy(ygz_vo* vo) { delete vo; }

}  // extern "C"
