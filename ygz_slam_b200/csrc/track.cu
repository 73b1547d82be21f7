// track.cu -- device-resident local map and the fused tracking entry points (ygzb_tracker_*).
//
// Replaces the CALLER-SIDE data flow of the reference's per-frame path, so that nothing but one small record per frame
// crosses PCIe:
//   VisualOdometry::TrackRefFrame / LocalMapping::TrackLocalMap     src/Module/VisualOdometry.cpp:281-302,
//                                                                   src/Module/LocalMapping.cpp:24-140
//   VisualOdometry::SetKeyframe (Detect, map points, LocalBA)       src/Module/VisualOdometry.cpp:182-218,
//                                                                   src/Module/LocalMapping.cpp:149-172
// The numeric stages are the kernels of align.cu (sparse alignment, direct projection), ba.cu (pose-only), fast.cu /
// describe.cu (Detect) and ba2.cu (LocalBAG2O); this file owns the key-frame ring, the key-frame insertion kernel, the
// assembly of the local-BA problems (landmark-major, straight from the ring) and the write-back of the BA result.
// Compiled with -fmad=false: the map-point creation and candidate bookkeeping follow the host loops
// (host/vo_driver.cpp, ygz_slam_b200/vo.py) operation by operation.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <new>

#include "ba2.cuh"
#include "common.cuh"
#include "se3.cuh"
#include "track.cuh"

using namespace ygzb;

struct ygzb_tracker {
    ygzb_frames* f;
    ygzb_ctx* ctx;
    TrackStore st;
    TrackBatch b;          // arrays sized for max_jobs
    int max_jobs;
    void* d_store;         // one allocation behind st.*
    void* d_batch;         // one allocation behind b.*
    double* d_depth;       // [S][W*H]
    // staging (page-locked) + device copies of the job arrays; a key-frame batch of n jobs is followed by n start poses
    // (kf_stage_bytes per stream), so a job's pose travels with it in the same copy
    ygzb_track_job* h_jobs;
    ygzb_keyframe_job* h_kfjobs;
    ygzb_keyframe_job* d_kfjobs;
    std::vector<double> start_T;   // [S][12] pose of each stream's next first key-frame (ygzb_tracker_set_start_pose)
    ygzb_keyframe_result* d_kfres;
    cudaEvent_t staged;    // the last H2D copy out of the staging buffers
    int last_J;
    // local BA problems of a key-frame batch (device-built, capacity based)
    void* d_ba;            // problem arrays + scratch of ba2
    size_t ba_bytes;
    int pcap, ocap;        // points / observations capacity per problem
    cudaStream_t front;    // second stream: uploads + pyramid + sparse alignment of the next batch run here, concurrently with a
                           // local BA on the context's stream (they need the new key-frame's features, not its refined pose)
    cudaEvent_t e_fill;    // recorded on the main stream after the key-frame insertion kernel (features + ring entry written)
    cudaEvent_t e_front;   // recorded on the front stream after the sparse alignment
    cudaEvent_t e_up;      // recorded on the front stream after every upload: a key-frame insertion (Detect) waits for it
    cudaEvent_t e_main;    // recorded on the main stream after a tracking chain: the front stream must not overwrite its arrays earlier
    int cluster;           // CTAs per tracking problem (sparse alignment, pose-only): fixed, so that a frame's result does not
                           // depend on how many other frames share its batch (the summation order follows the cluster size)
    void* d_xfer;          // staging of a map record (ygzb_tracker_export / _import), allocated on first use
    // previous-frame reference (ygzb_tracker_set_reference_mode)
    int ref_mode;
    bool kf_inserted;              // a key-frame insertion has been enqueued: the mode is fixed from then on
    std::vector<int32_t> ref_slots; // the caller's reference slot of every stream (pyramid of the last tracked frame)
    std::vector<int32_t> cur_ref;   // slot the stream's reference pyramid is in now (ref_slots[s] or a key-frame's slot), -1: none
    std::vector<int32_t> pos_of;    // caller's job index -> position in the wave-ordered batch
    void* d_ref;                   // reference store + the wave scratch of the sparse alignment (ref_cap features per problem)
    int32_t* h_aux;                // pinned [2][max_jobs]: job_ref_slot, orig
    int32_t* d_aux;
    ygzb_observation* d_obs;       // device view of the caller's page-locked observation rows (ygzb_tracker_set_observations), or NULL
    ygzb_pose_information* d_info; // device view of the caller's page-locked information records (ygzb_tracker_set_information), or NULL
    ygzb_map_point* d_map;         // device view of the caller's page-locked map rows (ygzb_tracker_set_map_updates), or NULL
    // the camera table (ygzb_tracker_set_camera): st.cam_K / st.cam_F on the device, and the host's copy of both
    void* d_cam;
    std::vector<double> cam_K;     // [S][4]
    std::vector<float> cam_F;      // [S][4]
    // per stream: what ygzb_tracker_upload_stream reads its frames through
    struct Source {
        RawFormat raw;                  // the raw frames (ygzb_tracker_set_source)
        // undistortion maps (ygzb_tracker_set_undistort), allocated on the stream's first maps and kept until destroy:
        // map_xy then map_a on the device, read only by the stream's uploads on the front stream, and their page-locked
        // staging with an event behind its last copy
        uint8_t* d_maps = nullptr;
        uint8_t* h_maps = nullptr;
        cudaEvent_t e_maps = nullptr;
        bool has_maps = false;          // maps set: uploads remap level 0 through them
    };
    std::vector<Source> sources;
};

namespace {

static_assert(sizeof(ygzb_observation) == 48, "an observation row is 48 bytes");
static_assert(sizeof(ygzb_pose_information) == 336, "an information record is 336 bytes");
static_assert(sizeof(ygzb_map_point) == 32 && offsetof(ygzb_map_point, pw) == 8, "a map point row is 32 bytes: id, pw[3]");
// a stream's maps: map_xy (short2 per pixel), then map_a (uint16 per pixel) from a 256-byte boundary
size_t lens_a_offset(size_t pixels) { return (pixels * sizeof(short2) + 255) & ~(size_t)255; }
size_t lens_bytes(size_t pixels) { return lens_a_offset(pixels) + pixels * sizeof(uint16_t); }
constexpr size_t kf_stage_bytes = sizeof(ygzb_keyframe_job) + 12 * sizeof(double);   // a key-frame job and its start pose
static_assert(sizeof(ygzb_keyframe_job) % sizeof(double) == 0, "the start poses behind the key-frame jobs are 8-byte aligned");

template <typename T>
int dalloc(ygzb_ctx* ctx, T** p, size_t count) {
    return check_cuda(ctx, cudaMalloc((void**)p, std::max(count, (size_t)1) * sizeof(T)), "cudaMalloc");
}

__device__ __forceinline__ void mat34_inv(const double* A, double* C) {
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) C[4 * r + c] = A[4 * c + r];
        C[4 * r + 3] = -(A[r] * A[3] + A[4 + r] * A[7] + A[8 + r] * A[11]);
    }
}

__global__ void track_finish_kernel(TrackBatch b) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= b.J) return;
    ygzb_track_result r;
    for (int c = 0; c < 12; ++c) r.T_cw[c] = b.T_cur[12 * (size_t)j + c];
    r.n_meas = b.n_meas[j];
    r.aligned = b.aligned[j];
    r.n_candidates = b.n_cand[j];
    r.n_projected = b.c_cnt[j];
    r.n_inliers = b.aligned[j] ? b.n_inl[j] : 0;
    r.pad[0] = r.pad[1] = r.pad[2] = 0;
    b.results[b.orig ? b.orig[j] : j] = r;
}

// inclusive scan of one int per thread over a 1024-thread CTA: shuffles inside the warps, the 32 warp totals scanned by warp 0
// (two barriers instead of the twenty of a shared-memory Hillis-Steele scan); s_w = 33 ints; returns the CTA total in *total
__device__ __forceinline__ int block_scan_1024(int v, int* s_w, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xFFFFFFFFu, v, o);
        if (lane >= o) v += u;
    }
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    if (warp == 0) {
        int w = s_w[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xFFFFFFFFu, w, o);
            if (lane >= o) w += u;
        }
        s_w[lane] = w;
        if (lane == 31) s_w[32] = w;
    }
    __syncthreads();
    const int out = v + (warp ? s_w[warp - 1] : 0);
    *total = s_w[32];
    __syncthreads();   // s_w may be rewritten by the next call
    return out;
}

// the pose-only inliers of tracking job tj (batch position) in candidate order -- none when it did not align -- as rows
// 0, 1, ...: emit(row, r, at, id) with the row's index r within its chunk of 1024 candidates, the candidate's index `at`
// in the batch arrays and its map point's id; then, in every thread, chunk(first row of the chunk, rows of the chunk).
// Called by a whole 1024-thread CTA (s_w as in block_scan_1024); returns the row count.  Both the key-frame observations
// (kf_fill_kernel) and the frame observations (track_obs_kernel) are made here, so they follow one rule.
template <typename Emit, typename Chunk>
__device__ __forceinline__ int for_each_inlier(const TrackStore& st, const TrackBatch& b, int tj, int* s_w, Emit emit, Chunk chunk) {
    const ygzb_track_job* job = b.jobs + tj;   // (read in place: a local copy would be indexed by k in local memory)
    const int cnt = b.aligned[tj] ? b.c_cnt[tj] : 0;
    int carry = 0;
    for (int base = 0; base < cnt; base += 1024) {
        const int q = base + (int)threadIdx.x;
        const size_t at = (size_t)tj * b.cap + q;
        const int flag = (q < cnt && b.inlier[at]) ? 1 : 0;
        int chunk_total;
        const int incl = block_scan_1024(flag, s_w, &chunk_total);
        if (flag) {
            const int c = b.c_src[at], k = c / st.cells, f = c - k * st.cells;
            emit(carry + incl - 1, incl - 1, at, st.kf_mp0[job->stream * st.R + job->entry[k]] + f);
        }
        chunk(carry, chunk_total);
        carry += chunk_total;   // (the same total in every thread; block_scan_1024 ends on a barrier)
    }
    return carry;
}

// SetKeyframe for job blockIdx.x: the features Detect left in the frame slot's store become the key-frame's features and
// map points (depth image -> camera point -> world, VisualOdometry.cpp:182-218 with the depth initialisation of
// test/test_feature_alignment.cpp:72-85), the inlier observations of its tracking job become its observations of older points.
// A first key-frame (track_job < 0) takes the start pose staged with its job (start_T[blockIdx.x], identity by default).
__global__ void __launch_bounds__(1024) kf_fill_kernel(TrackStore st, TrackBatch b, const ygzb_keyframe_job* __restrict__ jobs,
                                                      const double* __restrict__ start_T, const int32_t* __restrict__ f_count,
                                                      const int16_t* __restrict__ f_x, const int16_t* __restrict__ f_y,
                                                      const uint8_t* __restrict__ f_level, int n_cells, ygzb_keyframe_result* __restrict__ res) {
    __shared__ int s_scan[33];
    __shared__ double s_T[12], s_Tin[12], s_K[4];
    const ygzb_keyframe_job kj = jobs[blockIdx.x];
    const int tid = threadIdx.x, e = kj.stream * st.R + kj.entry;
    const int n = min(f_count[kj.frame_slot], st.cells);
    if (tid < 12) s_T[tid] = kj.track_job >= 0 ? b.T_cur[12 * (size_t)kj.track_job + tid] : start_T[12 * (size_t)blockIdx.x + tid];
    if (tid >= 32 && tid < 36) s_K[tid - 32] = st.cam_K[4 * kj.stream + tid - 32];   // the camera of the key-frame's stream
    __syncthreads();
    if (tid == 0) mat34_inv(s_T, s_Tin);
    __syncthreads();
    if (tid < 12) st.kf_T[12 * (size_t)e + tid] = s_T[tid];
    if (tid == 0) {
        st.kf_n[e] = n;
        st.kf_slot[e] = kj.kf_slot;
        st.kf_mp0[e] = kj.mp0;
        res[blockIdx.x].n_features = n;
    }
    const double* depth = st.depth_map + (size_t)kj.stream * st.W * st.H;
    for (int g = tid; g < n; g += 1024) {
        const size_t s = (size_t)kj.frame_slot * n_cells + g, fe = (size_t)e * st.cells + g;
        const int L = f_level[s];
        const double x = (double)((int)f_x[s] << L), y = (double)((int)f_y[s] << L);   // Feature::_pixel = level coordinate * 2^level
        const double d = depth[(size_t)(int)y * st.W + (int)x];
        st.kf_px[2 * fe] = x;
        st.kf_px[2 * fe + 1] = y;
        st.kf_level[fe] = (uint8_t)L;
        st.kf_depth[fe] = d;
        const volatile double* K = s_K;   // (read where it is used: held in registers across the loop, it spills more)
        const double pc0 = (x - K[2]) * d / K[0], pc1 = (y - K[3]) * d / K[1], pc2 = d;
        for (int r = 0; r < 3; ++r)
            st.kf_pw[3 * fe + r] = s_Tin[4 * r] * pc0 + s_Tin[4 * r + 1] * pc1 + s_Tin[4 * r + 2] * pc2 + s_Tin[4 * r + 3];
    }
    // observations of older map points: the inliers of the tracking job, in candidate order
    int total = 0;
    if (kj.track_job >= 0) {
        long long* obs_id = st.kf_obs_id + (size_t)e * b.cap;
        double* obs_px = st.kf_obs_px + 2 * (size_t)e * b.cap;
        total = for_each_inlier(
            st, b, kj.track_job, s_scan,
            [&](int row, int, size_t at, long long id) {
                obs_id[row] = id;
                obs_px[2 * row] = b.c_px[2 * at];
                obs_px[2 * row + 1] = b.c_px[2 * at + 1];
            },
            [](int, int) {});
    }
    if (tid == 0) st.kf_nobs[e] = total;
}

// the observations of job blockIdx.x (batch position) behind its pose-only: its inliers as rows (map point id, measured
// pixel, world point), written straight into the caller's page-locked buffer `out` (a mapped device pointer) at the rows
// of the caller's job index -- only the live rows cross PCIe.  The rows of a chunk of candidates are assembled in shared
// memory and leave as one contiguous run of 16-byte stores (full lines over PCIe, not 8-byte pieces 48 bytes apart).
constexpr size_t kObsSmem = 1024 * sizeof(ygzb_observation);   // dynamic shared memory of track_obs_kernel: one chunk of rows
__global__ void __launch_bounds__(1024) track_obs_kernel(TrackStore st, TrackBatch b, ygzb_observation* __restrict__ out) {
    extern __shared__ int4 s_rows[];   // [1024 * 3]: the chunk's rows
    __shared__ int s_scan[33];
    const int j = blockIdx.x;
    ygzb_observation* rows = out + (size_t)(b.orig ? b.orig[j] : j) * b.cap;
    ygzb_observation* s_obs = reinterpret_cast<ygzb_observation*>(s_rows);
    for_each_inlier(
        st, b, j, s_scan,
        [&](int, int r, size_t at, long long id) {
            ygzb_observation& o = s_obs[r];
            o.id = id;
            o.px[0] = b.c_px[2 * at];
            o.px[1] = b.c_px[2 * at + 1];
            o.pw[0] = b.c_pw[3 * at];
            o.pw[1] = b.c_pw[3 * at + 1];
            o.pw[2] = b.c_pw[3 * at + 2];
        },
        [&](int first, int n) {   // (the next chunk's scan begins with a barrier: s_rows is read before it is rewritten)
            __syncthreads();
            int4* dst = reinterpret_cast<int4*>(rows + first);   // 48-byte rows: every row starts 16-byte aligned
            for (int i = threadIdx.x; i < 3 * n; i += 1024) dst[i] = s_rows[i];
        });
}

// the pose information of job blockIdx.x (batch position) behind its pose-only, written straight into the caller's
// page-locked record `out` (a mapped device pointer) of the caller's job index: the alignment's H scaled to
// getFisherInformation, and sum J^T J over the job's inliers -- the set its observation rows hold (for_each_inlier) -- with
// J = d pi(exp(delta) T_cw P_w) / d delta at delta = 0 (left perturbation [upsilon; omega]) at the job's pose-only result.
// Each thread sums the candidates it visits in candidate order, the warps and then the 32 warp sums are added in a fixed
// order: a record depends on its job alone, not on the batch, the wave or the pacing.
__global__ void __launch_bounds__(1024) track_info_kernel(TrackStore st, TrackBatch b, ygzb_pose_information* __restrict__ out) {
    __shared__ int s_scan[33];
    __shared__ double s_T[12], s_f[2];
    __shared__ double s_red[32][21];
    const int j = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 12) s_T[tid] = b.T_cur[12 * (size_t)j + tid];
    if (tid >= 32 && tid < 34) s_f[tid - 32] = b.cam[4 * (size_t)j + tid - 32];   // the float focal lengths of the job's stream
    __syncthreads();
    const double fx = s_f[0], fy = s_f[1];
    double acc[21];
#pragma unroll
    for (int k = 0; k < 21; ++k) acc[k] = 0.0;
    for_each_inlier(
        st, b, j, s_scan,
        [&](int, int, size_t at, long long) {
            const double* P = b.c_pw + 3 * at;
            const double x = s_T[0] * P[0] + s_T[1] * P[1] + s_T[2] * P[2] + s_T[3];
            const double y = s_T[4] * P[0] + s_T[5] * P[1] + s_T[6] * P[2] + s_T[7];
            const double z = s_T[8] * P[0] + s_T[9] * P[1] + s_T[10] * P[2] + s_T[11];
            const double zi = 1.0 / z, u = x * zi, v = y * zi;
            // d pi / d P_c times d P_c / d delta = [I | -P_c^]
            const double Ju[6] = {fx * zi, 0.0, -fx * u * zi, -fx * u * v, fx * (1.0 + u * u), -fx * v};
            const double Jv[6] = {0.0, fy * zi, -fy * v * zi, -fy * (1.0 + v * v), fy * u * v, fy * u};
            int t = 0;
#pragma unroll
            for (int r = 0; r < 6; ++r)
#pragma unroll
                for (int c = r; c < 6; ++c, ++t) acc[t] += Ju[r] * Ju[c] + Jv[r] * Jv[c];
        },
        [](int, int) {});
#pragma unroll
    for (int k = 0; k < 21; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
        if (lane == 0) s_red[warp][k] = v;
    }
    __syncthreads();
    ygzb_pose_information* rec = out + (b.orig ? b.orig[j] : j);
    if (tid < 21) {
        double v = 0.0;
        for (int w = 0; w < 32; ++w) v += s_red[w][tid];
        rec->pose_info[tid] = v;
    } else if (tid < 42) {
        rec->align_fisher[tid - 21] = b.align_H[21 * (size_t)j + tid - 21] / kFisherNoise;
    }
}

// previous-frame reference of job blockIdx.x after its pose-only refinement, into the stream's other buffer: its pose and its
// projected candidates in candidate order; an inlier at the depth of its map point under that pose (OptimizeCurrent,
// LocalMapping.cpp:130-134), an outlier at the depth pose-only left it (its last inlier round's, or -1).  Outliers stay:
// SparseImgAlign tests only _mappoint and the border, not _bad.
__global__ void __launch_bounds__(256) track_ref_write_kernel(TrackStore st, TrackBatch b) {
    __shared__ double s_T[12];
    const int j = blockIdx.x, tid = threadIdx.x;
    const int s = b.jobs[j].stream, nb = 1 - st.ref_cur[s], r = 2 * s + nb;
    const int n = b.aligned[j] ? b.c_cnt[j] : 0;
    if (tid < 12) s_T[tid] = b.T_cur[12 * (size_t)j + tid];
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
        const size_t at = (size_t)j * b.cap + i, o = (size_t)r * st.ref_cap + i;
        const double* X = b.c_pw + 3 * at;
        st.ref_px[2 * o] = b.c_px[2 * at];
        st.ref_px[2 * o + 1] = b.c_px[2 * at + 1];
        st.ref_depth[o] = b.inlier[at] ? s_T[8] * X[0] + s_T[9] * X[1] + s_T[10] * X[2] + s_T[11] : b.c_depth[at];
    }
    if (tid < 12) st.ref_T[12 * (size_t)r + tid] = s_T[tid];
    __syncthreads();
    if (tid == 0) {
        st.ref_n[r] = n;
        st.ref_cur[s] = nb;
    }
}

// previous-frame reference after key-frame job blockIdx.x (SetKeyframe + LocalBA, VisualOdometry.cpp:182-218,
// LocalMapping.cpp:192-206), over the stream's current buffer: the key-frame's pose after the BA write-back; its tracked
// features, inliers at the depth of their map point after the BA, outliers unchanged; then its new features with their
// depth-image depth
__global__ void __launch_bounds__(256) kf_ref_kernel(TrackStore st, TrackBatch b, const ygzb_keyframe_job* __restrict__ jobs) {
    __shared__ double s_T[12];
    const ygzb_keyframe_job kj = jobs[blockIdx.x];
    const int tid = threadIdx.x, e = kj.stream * st.R + kj.entry, r = 2 * kj.stream + st.ref_cur[kj.stream];
    if (tid < 12) s_T[tid] = st.kf_T[12 * (size_t)e + tid];
    __syncthreads();
    int n_tr = 0;
    if (kj.track_job >= 0) {
        const int tj = kj.track_job;
        const ygzb_track_job job = b.jobs[tj];
        n_tr = b.aligned[tj] ? b.c_cnt[tj] : 0;
        for (int i = tid; i < n_tr; i += blockDim.x) {
            const size_t at = (size_t)tj * b.cap + i, o = (size_t)r * st.ref_cap + i;
            st.ref_px[2 * o] = b.c_px[2 * at];
            st.ref_px[2 * o + 1] = b.c_px[2 * at + 1];
            double d = b.c_depth[at];
            if (b.inlier[at]) {
                const int c = b.c_src[at], k = c / st.cells, f = c - k * st.cells;
                const double* X = st.kf_pw + 3 * ((size_t)(job.stream * st.R + job.entry[k]) * st.cells + f);
                d = s_T[8] * X[0] + s_T[9] * X[1] + s_T[10] * X[2] + s_T[11];
            }
            st.ref_depth[o] = d;
        }
    }
    const int n_new = st.kf_n[e];
    for (int g = tid; g < n_new; g += blockDim.x) {
        const size_t fe = (size_t)e * st.cells + g, o = (size_t)r * st.ref_cap + n_tr + g;
        st.ref_px[2 * o] = st.kf_px[2 * fe];
        st.ref_px[2 * o + 1] = st.kf_px[2 * fe + 1];
        st.ref_depth[o] = st.kf_depth[fe];
    }
    if (tid < 12) st.ref_T[12 * (size_t)r + tid] = s_T[tid];
    if (tid == 0) st.ref_n[r] = n_tr + n_new;
}

// the batch arrays of wave jobs [j0, j0 + J): every per-job array shifted to job j0; the workspaces of the solvers and the
// sparse alignment's per-feature scratch (wave-local, sized for the stream count) are not
TrackBatch wave_batch(const TrackBatch& b, int j0, int J) {
    TrackBatch w = b;
    const size_t c = (size_t)j0 * b.cap;
    w.J = J;
    w.jobs += j0; w.ref_slot += j0; w.cur_slot += j0; w.offsets += j0; w.in_off += j0; w.n_feat += j0; w.n_meas += j0;
    w.T_ref += 12 * (size_t)j0; w.T_cur += 12 * (size_t)j0; w.T_aligned += 12 * (size_t)j0;
    w.aligned += j0; w.rel += 12 * (size_t)kTrackMaxLocal * j0; w.cam += 4 * (size_t)j0;
    w.cand_ok += c; w.cand_px += 2 * c; w.n_cand += j0; w.c_cnt += j0; w.c_off += j0; w.c_src += c;
    w.c_pw += 3 * c; w.c_px += 2 * c; w.c_depth += c; w.inlier += c; w.enable += c; w.n_inl += j0;
    w.results += j0; w.job_ref_slot += j0; w.orig += j0;
    if (w.align_H) w.align_H += 21 * (size_t)j0;
    return w;
}

struct BABuild {   // device arrays of the batch of local-BA problems (capacity based: problem p owns fixed ranges)
    int32_t *kf_off, *pt_off, *obs_off;   // [P + 1]
    int32_t *n_kf, *n_pt;                 // [P]
    double* poses;                        // [P][kTrackMaxLocal][6]
    uint8_t* fixed;                       // [P][kTrackMaxLocal]
    double* pts;                          // [P][pcap][3]
    int32_t* lm_start;                    // [P][pcap]
    int32_t* so_kf;                       // [P][ocap]
    double* so_uv;                        // [P][ocap][2]
    int32_t* owner;                       // [P][pcap]  dense index (local key-frame * cells + feature) of every BA point
    int32_t* tab;                         // [P][kTrackMaxLocal][kTrackMaxLocal * cells]  observation of point i in key-frame k' (+1)
    int32_t* prob_of;                     // [n key-frame jobs] -> problem or -1
    int pcap, ocap;
};

// LocalMapping::LocalBA problem of key-frame job kf_job[blockIdx.x] (if it runs a BA): the local key-frames and the points
// at least two of them observe (a key-frame observes its own points and the older points tracked into it), landmark-major
__global__ void __launch_bounds__(1024) ba_build_kernel(TrackStore st, const ygzb_keyframe_job* __restrict__ jobs, BABuild B, int cap_obs) {
    __shared__ int s_scan[1024];
    __shared__ int s_cpt, s_cobs;
    const int p = B.prob_of[blockIdx.x];
    if (p < 0) return;
    const ygzb_keyframe_job kj = jobs[blockIdx.x];
    const int tid = threadIdx.x, nk = kj.n_local, dense = nk * st.cells;
    int e[kTrackMaxLocal], nf[kTrackMaxLocal];
    long long m0[kTrackMaxLocal];
    for (int k = 0; k < kTrackMaxLocal; ++k) {
        e[k] = kj.stream * st.R + kj.local_entry[k < nk ? k : 0];
        nf[k] = k < nk ? st.kf_n[e[k]] : 0;
        m0[k] = st.kf_mp0[e[k]];
    }
    int32_t* tab = B.tab + (size_t)p * kTrackMaxLocal * kTrackMaxLocal * st.cells;
    for (int i = tid; i < nk * dense; i += 1024) tab[(size_t)(i / dense) * kTrackMaxLocal * st.cells + (i % dense)] = 0;
    if (tid == 0) s_cpt = s_cobs = 0;
    __syncthreads();
    for (int k2 = 0; k2 < nk; ++k2) {
        const int nobs = st.kf_nobs[e[k2]];
        for (int q = tid; q < nobs; q += 1024) {
            const long long id = st.kf_obs_id[(size_t)e[k2] * cap_obs + q];
            for (int k = 0; k < nk; ++k)
                if (id >= m0[k] && id < m0[k] + nf[k]) {
                    tab[(size_t)k2 * kTrackMaxLocal * st.cells + k * st.cells + (int)(id - m0[k])] = q + 1;
                    break;
                }
        }
    }
    __syncthreads();
    const int p0 = p * B.pcap, o0 = p * B.ocap;
    // every thread takes `per` CONSECUTIVE dense indices (so the output order is the dense order), finds their degrees with all
    // the table loads in flight at once, and ONE block scan of the per-thread (points, observations) totals places them
    constexpr int kMaxPer = (kTrackMaxLocal * 4096 + 1023) / 1024;   // cells <= 4096
    const int per = (dense + 1023) / 1024;
    int degs[kMaxPer];
    int my_pts = 0, my_obs = 0;
#pragma unroll
    for (int r = 0; r < kMaxPer; ++r) {
        degs[r] = 0;
        const int i = tid * per + r;
        if (r < per && i < dense) {
            const int k = i / st.cells, g = i - k * st.cells;
            if (g < nf[k]) {
                int deg = 1;
                for (int k2 = 0; k2 < nk; ++k2) deg += tab[(size_t)k2 * kTrackMaxLocal * st.cells + i] != 0;
                if (deg >= 2) {
                    degs[r] = deg;
                    my_pts += 1;
                    my_obs += deg;
                }
            }
        }
    }
    int total_packed;
    const int incl = block_scan_1024(my_pts | (my_obs << 15), s_scan, &total_packed);   // 15 bits of points, 17 of observations
    int pt = (incl & 0x7FFF) - my_pts, ob = (int)((unsigned)incl >> 15) - my_obs;   // exclusive prefix of this thread
#pragma unroll
    for (int r = 0; r < kMaxPer; ++r) {
        const int deg = degs[r];
        if (!deg) continue;
        const int i = tid * per + r, k = i / st.cells, g = i - k * st.cells;
        const size_t P = (size_t)p0 + pt, fe = (size_t)e[k] * st.cells + g;
        B.pts[3 * P] = st.kf_pw[3 * fe];
        B.pts[3 * P + 1] = st.kf_pw[3 * fe + 1];
        B.pts[3 * P + 2] = st.kf_pw[3 * fe + 2];
        B.lm_start[P] = o0 + ob;
        B.owner[P] = i;
        size_t o = (size_t)o0 + ob;
        B.so_kf[o] = k;
        B.so_uv[2 * o] = st.kf_px[2 * fe];
        B.so_uv[2 * o + 1] = st.kf_px[2 * fe + 1];
        ++o;
        for (int k2 = 0; k2 < nk; ++k2) {
            const int q = tab[(size_t)k2 * kTrackMaxLocal * st.cells + i];
            if (!q) continue;
            B.so_kf[o] = k2;
            B.so_uv[2 * o] = st.kf_obs_px[2 * ((size_t)e[k2] * cap_obs + q - 1)];
            B.so_uv[2 * o + 1] = st.kf_obs_px[2 * ((size_t)e[k2] * cap_obs + q - 1) + 1];
            ++o;
        }
        pt += 1;
        ob += deg;
    }
    if (tid == 0) {
        s_cpt = total_packed & 0x7FFF;
        s_cobs = (int)((unsigned)total_packed >> 15);
    }
    __syncthreads();
    if (tid == 0) {
        B.lm_start[(size_t)p0 + s_cpt] = o0 + s_cobs;
        B.n_kf[p] = nk;
        B.n_pt[p] = s_cpt;
        B.kf_off[p] = p * kTrackMaxLocal;
        B.pt_off[p] = p0;
        B.obs_off[p] = o0;
    }
    if (tid < nk) {
        double lg[6];
        se3_log(se3_from_mat(st.kf_T + 12 * (size_t)e[tid]), lg);
        double* g2o = B.poses + 6 * ((size_t)p * kTrackMaxLocal + tid);
        g2o[0] = lg[3]; g2o[1] = lg[4]; g2o[2] = lg[5]; g2o[3] = lg[0]; g2o[4] = lg[1]; g2o[5] = lg[2];   // VertexSE3Sophus: [omega; upsilon]
        B.fixed[p * kTrackMaxLocal + tid] = tid == 0 ? 1 : 0;   // the oldest local key-frame fixes the gauge (key-frame 0 in the reference)
    }
}

// BA result back into the ring (poses of every local key-frame, refined map points) and into the result records
__global__ void __launch_bounds__(256) ba_writeback_kernel(TrackStore st, const ygzb_keyframe_job* __restrict__ jobs, BABuild B,
                                                           const double* __restrict__ ba_stats, ygzb_keyframe_result* __restrict__ res) {
    const ygzb_keyframe_job kj = jobs[blockIdx.x];
    const int p = B.prob_of[blockIdx.x], tid = threadIdx.x, nk = kj.n_local;
    ygzb_keyframe_result* r = res + blockIdx.x;
    if (p >= 0) {
        if (tid < nk) {
            const double* g = B.poses + 6 * ((size_t)p * kTrackMaxLocal + tid);
            const double v[6] = {g[3], g[4], g[5], g[0], g[1], g[2]};
            se3_to_mat(se3_exp(v), st.kf_T + 12 * (size_t)(kj.stream * st.R + kj.local_entry[tid]));
        }
        const int npt = B.n_pt[p];
        for (int q = tid; q < npt; q += 256) {
            const int i = B.owner[(size_t)p * B.pcap + q], k = i / st.cells, g = i - k * st.cells;
            const size_t fe = (size_t)(kj.stream * st.R + kj.local_entry[k]) * st.cells + g;
            for (int c = 0; c < 3; ++c) st.kf_pw[3 * fe + c] = B.pts[3 * ((size_t)p * B.pcap + q) + c];
        }
        if (tid == 0) {
            const double* s = ba_stats + 8 * (size_t)p;
            r->ba_points = npt;
            r->ba_observations = B.lm_start[(size_t)p * B.pcap + npt] - p * B.ocap;
            r->ba_iters = (int)s[0];
            r->ba_trials = (int)s[1];
            r->chi2_initial = s[2];
            r->chi2_final = s[3];
            r->pad = 0;
        }
    } else if (tid == 0) {
        r->ba_points = r->ba_observations = r->ba_iters = r->ba_trials = r->pad = 0;
        r->chi2_initial = r->chi2_final = 0;
    }
    __syncthreads();
    if (tid < 12 * nk) r->T_cw[tid / 12][tid % 12] = st.kf_T[12 * (size_t)(kj.stream * st.R + kj.local_entry[tid / 12]) + tid % 12];
}

size_t babuild_carve(Carver& c, BABuild& B, size_t P, int cells, int n_jobs) {
    B.kf_off = c.take<int32_t>(P + 1); B.pt_off = c.take<int32_t>(P + 1); B.obs_off = c.take<int32_t>(P + 1);
    B.n_kf = c.take<int32_t>(P); B.n_pt = c.take<int32_t>(P);
    B.poses = c.take<double>(P * kTrackMaxLocal * 6);
    B.fixed = c.take<uint8_t>(P * kTrackMaxLocal);
    B.pts = c.take<double>(P * B.pcap * 3);
    B.lm_start = c.take<int32_t>(P * B.pcap);
    B.so_kf = c.take<int32_t>(P * B.ocap);
    B.so_uv = c.take<double>(P * B.ocap * 2);
    B.owner = c.take<int32_t>(P * B.pcap);
    B.tab = c.take<int32_t>(P * kTrackMaxLocal * kTrackMaxLocal * cells);
    B.prob_of = c.take<int32_t>((size_t)n_jobs);
    return c.bytes();
}

// the map rows of key-frame job blockIdx.x behind its BA write-back (ygzb_tracker_set_map_updates): the BA's points in its
// landmark order (B.owner), then the new key-frame's points in feature order, each with its id and the ring's kf_pw as the
// write-back left it, written straight into the caller's page-locked buffer `out` (a mapped device pointer) at
// out[blockIdx.x * YGZB_TRACK_RING * cells].  The rows of a chunk are assembled in shared memory and leave as one
// contiguous run of 16-byte stores, as track_obs_kernel's do.
__global__ void __launch_bounds__(1024) kf_points_kernel(TrackStore st, const ygzb_keyframe_job* __restrict__ jobs, BABuild B,
                                                        ygzb_map_point* __restrict__ out) {
    __shared__ int4 s_rows[1024 * sizeof(ygzb_map_point) / sizeof(int4)];   // one chunk of 1024 rows
    const ygzb_keyframe_job* kj = jobs + blockIdx.x;   // (read in place: local_entry is indexed by k)
    const int p = B.prob_of[blockIdx.x];
    const int n_moved = p >= 0 ? B.n_pt[p] : 0, e_new = kj->stream * st.R + kj->entry;
    const int total = n_moved + st.kf_n[e_new];
    ygzb_map_point* rows = out + (size_t)blockIdx.x * YGZB_TRACK_RING * st.cells;
    ygzb_map_point* s_pts = reinterpret_cast<ygzb_map_point*>(s_rows);
    for (int base = 0; base < total; base += 1024) {
        const int q = base + (int)threadIdx.x;
        if (q < total) {
            int e = e_new, g = q - n_moved;
            if (q < n_moved) {
                const int i = B.owner[(size_t)p * B.pcap + q], k = i / st.cells;
                e = kj->stream * st.R + kj->local_entry[k];
                g = i - k * st.cells;
            }
            const size_t fe = (size_t)e * st.cells + g;
            ygzb_map_point& m = s_pts[threadIdx.x];
            m.id = st.kf_mp0[e] + g;
            m.pw[0] = st.kf_pw[3 * fe];
            m.pw[1] = st.kf_pw[3 * fe + 1];
            m.pw[2] = st.kf_pw[3 * fe + 2];
        }
        __syncthreads();
        const int n = min(1024, total - base);
        int4* dst = reinterpret_cast<int4*>(rows + base);   // 32-byte rows: every row starts 16-byte aligned
        for (int i = threadIdx.x; i < 2 * n; i += 1024) dst[i] = s_rows[i];
        __syncthreads();   // s_rows is read before the next chunk rewrites it
    }
}

// ---- map records (ygzb_tracker_export / _import) -----------------------------------------------------------------------
static_assert(YGZB_MAP_OBS_PER_CELL == kTrackMaxLocal, "a key-frame's observation capacity is kTrackMaxLocal * cells");
static_assert(YGZB_TRACK_REF_FEATURES_PER_CELL == kTrackMaxLocal + 1, "the reference store holds (kTrackMaxLocal + 1) * cells features");
constexpr int kXferChunks = 16;   // CTAs per key-frame of the pack / unpack kernels (per reference record of theirs)

struct MapXfer {   // device staging of one record: at most YGZB_TRACK_RING key-frames, packed like ygzb_map_record
    double* T;
    long long* mp0;
    int32_t *n_feat, *n_obs;
    double *px, *depth, *pw, *obs_px;
    uint8_t *level, *image;
    long long* obs_id;
    // and of one reference record (ygzb_tracker_export_reference / _import_reference): ref_cap rows and one image
    double *ref_T, *ref_px, *ref_depth;
    int32_t* ref_n;
    uint8_t* ref_image;
};

struct MapXferJob {   // kernel argument: the ring entries of a record and, for an import, its packed offsets and slots
    int n, stream, with_image;
    int entry[YGZB_TRACK_RING], slot[YGZB_TRACK_RING];
    int foff[YGZB_TRACK_RING + 1], ooff[YGZB_TRACK_RING + 1];
};

size_t xfer_carve(Carver& c, MapXfer& X, size_t cells, size_t cap_obs, size_t WH) {
    const size_t R = YGZB_TRACK_RING;
    X.T = c.take<double>(R * 12); X.mp0 = c.take<long long>(R); X.n_feat = c.take<int32_t>(R); X.n_obs = c.take<int32_t>(R);
    X.px = c.take<double>(R * cells * 2); X.level = c.take<uint8_t>(R * cells); X.depth = c.take<double>(R * cells);
    X.pw = c.take<double>(R * cells * 3); X.obs_id = c.take<long long>(R * cap_obs); X.obs_px = c.take<double>(R * cap_obs * 2);
    X.image = c.take<uint8_t>(R * WH);
    const size_t ref_cap = YGZB_TRACK_REF_FEATURES_PER_CELL * cells;
    X.ref_T = c.take<double>(12); X.ref_n = c.take<int32_t>(1); X.ref_px = c.take<double>(ref_cap * 2); X.ref_depth = c.take<double>(ref_cap);
    X.ref_image = c.take<uint8_t>(WH);
    return c.bytes();
}

// export: CTA (k, y) fills rows [k * cells, (k + 1) * cells) of the packed feature arrays and [k * cap_obs, (k + 1) * cap_obs)
// of the observation arrays -- the live rows of all requested entries, back to back, then zeros up to the record's capacity
// -- and the level-0 image of key-frame k
__global__ void __launch_bounds__(256) map_pack_kernel(TrackStore st, MapXfer X, MapXferJob job, int cap_obs, const uint8_t* __restrict__ pyr,
                                                       size_t slot_stride, unsigned lv0_off, int lv0_pitch) {
    const int k = blockIdx.x, tid = threadIdx.x, n = job.n;
    int foff[YGZB_TRACK_RING + 1], ooff[YGZB_TRACK_RING + 1];
    foff[0] = ooff[0] = 0;
    for (int q = 0; q < YGZB_TRACK_RING; ++q) {
        const int e = job.stream * st.R + job.entry[q < n ? q : 0];
        foff[q + 1] = foff[q] + (q < n ? st.kf_n[e] : 0);
        ooff[q + 1] = ooff[q] + (q < n ? st.kf_nobs[e] : 0);
    }
    const int e = job.stream * st.R + job.entry[k];
    if (blockIdx.y == 0) {
        if (tid < 12) X.T[12 * k + tid] = st.kf_T[12 * (size_t)e + tid];
        if (tid == 0) {
            X.mp0[k] = st.kf_mp0[e];
            X.n_feat[k] = foff[k + 1] - foff[k];
            X.n_obs[k] = ooff[k + 1] - ooff[k];
        }
    }
    const int step = gridDim.y * blockDim.x, first = blockIdx.y * blockDim.x + tid;
    for (int i = k * st.cells + first; i < (k + 1) * st.cells; i += step) {
        double p0 = 0, p1 = 0, d = 0, w0 = 0, w1 = 0, w2 = 0;
        uint8_t L = 0;
        if (i < foff[n]) {
            int kk = 0;
            while (i >= foff[kk + 1]) ++kk;
            const size_t fe = (size_t)(job.stream * st.R + job.entry[kk]) * st.cells + (i - foff[kk]);
            p0 = st.kf_px[2 * fe]; p1 = st.kf_px[2 * fe + 1];
            L = st.kf_level[fe];
            d = st.kf_depth[fe];
            w0 = st.kf_pw[3 * fe]; w1 = st.kf_pw[3 * fe + 1]; w2 = st.kf_pw[3 * fe + 2];
        }
        X.px[2 * (size_t)i] = p0; X.px[2 * (size_t)i + 1] = p1;
        X.level[i] = L;
        X.depth[i] = d;
        X.pw[3 * (size_t)i] = w0; X.pw[3 * (size_t)i + 1] = w1; X.pw[3 * (size_t)i + 2] = w2;
    }
    for (int i = k * cap_obs + first; i < (k + 1) * cap_obs; i += step) {
        long long id = 0;
        double u = 0, v = 0;
        if (i < ooff[n]) {
            int kk = 0;
            while (i >= ooff[kk + 1]) ++kk;
            const size_t q = (size_t)(job.stream * st.R + job.entry[kk]) * cap_obs + (i - ooff[kk]);
            id = st.kf_obs_id[q];
            u = st.kf_obs_px[2 * q]; v = st.kf_obs_px[2 * q + 1];
        }
        X.obs_id[i] = id;
        X.obs_px[2 * (size_t)i] = u; X.obs_px[2 * (size_t)i + 1] = v;
    }
    if (job.with_image) {
        const uint8_t* src = pyr + (size_t)st.kf_slot[e] * slot_stride + lv0_off;
        uint8_t* dst = X.image + (size_t)k * st.W * st.H;
        for (int i = first; i < st.W * st.H; i += step) {
            const int y = i / st.W, x = i - y * st.W;
            dst[i] = src[(size_t)y * lv0_pitch + x];
        }
    }
}

// import: CTA (k, y) scatters key-frame k of the packed record into its ring entry (live rows only)
__global__ void __launch_bounds__(256) map_unpack_kernel(TrackStore st, MapXfer X, MapXferJob job, int cap_obs) {
    const int k = blockIdx.x, tid = threadIdx.x;
    const int e = job.stream * st.R + job.entry[k];
    const int nf = job.foff[k + 1] - job.foff[k], no = job.ooff[k + 1] - job.ooff[k];
    if (blockIdx.y == 0) {
        if (tid < 12) st.kf_T[12 * (size_t)e + tid] = X.T[12 * k + tid];
        if (tid == 0) {
            st.kf_n[e] = nf;
            st.kf_nobs[e] = no;
            st.kf_slot[e] = job.slot[k];
            st.kf_mp0[e] = X.mp0[k];
        }
    }
    const int step = gridDim.y * blockDim.x, first = blockIdx.y * blockDim.x + tid;
    for (int g = first; g < nf; g += step) {
        const size_t s = (size_t)job.foff[k] + g, fe = (size_t)e * st.cells + g;
        st.kf_px[2 * fe] = X.px[2 * s]; st.kf_px[2 * fe + 1] = X.px[2 * s + 1];
        st.kf_level[fe] = X.level[s];
        st.kf_depth[fe] = X.depth[s];
        st.kf_pw[3 * fe] = X.pw[3 * s]; st.kf_pw[3 * fe + 1] = X.pw[3 * s + 1]; st.kf_pw[3 * fe + 2] = X.pw[3 * s + 2];
    }
    for (int q = first; q < no; q += step) {
        const size_t s = (size_t)job.ooff[k] + q, d = (size_t)e * cap_obs + q;
        st.kf_obs_id[d] = X.obs_id[s];
        st.kf_obs_px[2 * d] = X.obs_px[2 * s]; st.kf_obs_px[2 * d + 1] = X.obs_px[2 * s + 1];
    }
}

// reference export: the live rows of stream s's current reference buffer, zeros up to ref_cap, and level 0 of the slot its
// pyramid is in (`lv0`, the host knows the slot when it enqueues); kXferChunks CTAs stride over rows and pixels
__global__ void __launch_bounds__(256) ref_pack_kernel(TrackStore st, MapXfer X, int s, const uint8_t* __restrict__ lv0, int lv0_pitch) {
    const int r = 2 * s + st.ref_cur[s], n = st.ref_n[r], tid = threadIdx.x;
    if (blockIdx.x == 0) {
        if (tid < 12) X.ref_T[tid] = st.ref_T[12 * (size_t)r + tid];
        if (tid == 0) X.ref_n[0] = n;
    }
    const int step = gridDim.x * blockDim.x, first = blockIdx.x * blockDim.x + tid;
    for (int i = first; i < st.ref_cap; i += step) {
        double u = 0, v = 0, d = 0;
        if (i < n) {
            const size_t o = (size_t)r * st.ref_cap + i;
            u = st.ref_px[2 * o]; v = st.ref_px[2 * o + 1];
            d = st.ref_depth[o];
        }
        X.ref_px[2 * (size_t)i] = u; X.ref_px[2 * (size_t)i + 1] = v;
        X.ref_depth[i] = d;
    }
    for (int i = first; i < st.W * st.H; i += step) {
        const int y = i / st.W, x = i - y * st.W;
        X.ref_image[i] = lv0[(size_t)y * lv0_pitch + x];
    }
}

// reference import: the first n rows of an uploaded record, its pose and count into stream s's current reference buffer
__global__ void __launch_bounds__(256) ref_unpack_kernel(TrackStore st, MapXfer X, int s, int n) {
    const int r = 2 * s + st.ref_cur[s], tid = threadIdx.x;
    if (blockIdx.x == 0) {
        if (tid < 12) st.ref_T[12 * (size_t)r + tid] = X.ref_T[tid];
        if (tid == 0) st.ref_n[r] = n;
    }
    for (int i = blockIdx.x * blockDim.x + tid; i < n; i += gridDim.x * blockDim.x) {
        const size_t o = (size_t)r * st.ref_cap + i;
        st.ref_px[2 * o] = X.ref_px[2 * (size_t)i]; st.ref_px[2 * o + 1] = X.ref_px[2 * (size_t)i + 1];
        st.ref_depth[o] = X.ref_depth[i];
    }
}

int tracker_xfer(ygzb_tracker* t, MapXfer& X) {
    const TrackStore& st = t->st;
    Carver c(nullptr);
    const size_t bytes = xfer_carve(c, X, (size_t)st.cells, (size_t)t->b.cap, (size_t)st.W * st.H);
    if (!t->d_xfer) YGZB_CUDA(t->ctx, cudaMalloc(&t->d_xfer, bytes));
    Carver d(t->d_xfer);
    xfer_carve(d, X, (size_t)st.cells, (size_t)t->b.cap, (size_t)st.W * st.H);
    return YGZB_OK;
}

// the batch arrays of a tracking batch of n_jobs jobs (the sparse alignment keeps its Hessians for the information records only)
TrackBatch job_batch(ygzb_tracker* t, int n_jobs) {
    TrackBatch b = t->b;
    b.J = n_jobs;
    if (!t->d_info) b.align_H = nullptr;
    t->last_J = n_jobs;
    return b;
}

// the tail of a tracking batch whose jobs have all been through pose-only: the observation rows and information records
// (when the caller asked for them), the results and their copy back, then e_main; before_copy() enqueues what has to come
// between the results and their copy
template <typename BeforeCopy>
int finish_batch(ygzb_tracker* t, const TrackBatch& b, ygzb_track_result* results, BeforeCopy before_copy) {
    ygzb_ctx* ctx = t->ctx;
    if (t->d_obs) {
        ProfScope ps(ctx, kStageOther);
        track_obs_kernel<<<(unsigned)b.J, 1024, kObsSmem, ctx->stream>>>(t->st, b, t->d_obs);
        YGZB_LAUNCHED(ctx);
    }
    if (t->d_info) {
        ProfScope ps(ctx, kStageOther);
        track_info_kernel<<<(unsigned)b.J, 1024, 0, ctx->stream>>>(t->st, b, t->d_info);
        YGZB_LAUNCHED(ctx);
    }
    {
        ProfScope ps(ctx, kStageOther);
        track_finish_kernel<<<(b.J + 63) / 64, 64, 0, ctx->stream>>>(b);
        YGZB_LAUNCHED(ctx);
    }
    TRY(before_copy());
    YGZB_CUDA(ctx, cudaMemcpyAsync(results, b.results, sizeof(ygzb_track_result) * (size_t)b.J, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaEventRecord(t->e_main, ctx->stream));
    return YGZB_OK;
}

// the device view of `bytes` bytes of page-locked host memory at `host` (ygzb_host_alloc), which a kernel writes through:
// both ends must be page-locked host memory with a device mapping, in one allocation; pageable memory has neither
int mapped_view(ygzb_ctx* ctx, const void* host, size_t bytes, size_t align, const char* what, void** out) {
    void* dev[2] = {nullptr, nullptr};
    const char* ends[2] = {static_cast<const char*>(host), static_cast<const char*>(host) + bytes - 1};
    for (int k = 0; k < 2; ++k) {
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, ends[k]) != cudaSuccess) {
            cudaGetLastError();
            return set_error(ctx, YGZB_ERR_INVALID, "%s: not a page-locked host buffer", what);
        }
        if (a.type != cudaMemoryTypeHost || !a.devicePointer)
            return set_error(ctx, YGZB_ERR_INVALID, "%s: not a page-locked host buffer (ygzb_host_alloc)", what);
        dev[k] = a.devicePointer;
    }
    if (static_cast<char*>(dev[1]) - static_cast<char*>(dev[0]) != ends[1] - ends[0])
        return set_error(ctx, YGZB_ERR_INVALID, "%s: the buffer spans more than one page-locked allocation", what);
    if (reinterpret_cast<uintptr_t>(dev[0]) % align) return set_error(ctx, YGZB_ERR_INVALID, "%s: buffer not %zu-byte aligned", what, align);
    *out = dev[0];
    return YGZB_OK;
}

#define STRINGIFY_(x) #x
#define STRINGIFY(x) STRINGIFY_(x)

// one of the tracker's optional outputs: *dev becomes the device view of the caller's page-locked buffer `host` of `capacity`
// elements, `need` of which the tracker writes (`rule` spells `need` out in the message), or NULL for a NULL host, which
// switches the writes off.  A call that fails leaves *dev as it was
template <typename T>
int attach_output(ygzb_tracker* t, T* host, size_t capacity, size_t need, size_t align, const char* what, const char* rule, T** dev) {
    if (!host) {
        *dev = nullptr;
        return YGZB_OK;
    }
    ygzb_ctx* ctx = t->ctx;
    if (capacity < need) return set_error(ctx, YGZB_ERR_INVALID, "%s: capacity %zu %s = %zu", what, capacity, rule, need);
    cudaSetDevice(ctx->device);
    void* view = nullptr;
    TRY(mapped_view(ctx, host, need * sizeof(T), align, what, &view));
    *dev = static_cast<T*>(view);
    return YGZB_OK;
}

// distinct ring entries in range (and distinct frame slots in range when `slots` is given)
int check_entries(ygzb_tracker* t, int n, const int32_t* entries, const int32_t* slots, const char* what) {
    ygzb_ctx* ctx = t->ctx;
    for (int k = 0; k < n; ++k) {
        if (entries[k] < 0 || entries[k] >= YGZB_TRACK_RING) return set_error(ctx, YGZB_ERR_INVALID, "%s: ring entry %d out of range", what, entries[k]);
        if (slots && (slots[k] < 0 || slots[k] >= t->f->capacity)) return set_error(ctx, YGZB_ERR_INVALID, "%s: frame slot %d out of range", what, slots[k]);
        for (int k2 = 0; k2 < k; ++k2) {
            if (entries[k2] == entries[k]) return set_error(ctx, YGZB_ERR_INVALID, "%s: ring entry %d given twice", what, entries[k]);
            if (slots && slots[k2] == slots[k]) return set_error(ctx, YGZB_ERR_INVALID, "%s: frame slot %d given twice", what, slots[k]);
        }
    }
    return YGZB_OK;
}

// the checks an export and an import of a reference record share: the mode, the stream, the capacity and the arrays
int check_reference_call(ygzb_tracker* t, int stream, const ygzb_reference_record* rec, const char* what) {
    ygzb_ctx* ctx = t->ctx;
    if (t->ref_mode != YGZB_TRACK_REF_PREVIOUS) return set_error(ctx, YGZB_ERR_INVALID, "%s: not in previous-frame reference mode", what);
    if (stream < 0 || stream >= t->st.S) return set_error(ctx, YGZB_ERR_INVALID, "%s: stream %d out of range", what, stream);
    if (rec->capacity < t->st.ref_cap)
        return set_error(ctx, YGZB_ERR_INVALID, "%s: capacity %d below the reference store's %d", what, rec->capacity, t->st.ref_cap);
    if (!rec->px || !rec->depth || !rec->image) return set_error(ctx, YGZB_ERR_INVALID, "%s: null array in the record", what);
    return YGZB_OK;
}

}  // namespace

// the previous-frame reference store of st.S streams (two records each, st.ref_cap features per record)
void ref_store_carve(Carver& c, TrackStore& st) {
    const size_t R2 = 2 * (size_t)st.S, cap = st.ref_cap;
    st.ref_px = c.take<double>(R2 * cap * 2); st.ref_depth = c.take<double>(R2 * cap); st.ref_n = c.take<int32_t>(R2);
    st.ref_T = c.take<double>(R2 * 12); st.ref_cur = c.take<int32_t>(st.S);
}

size_t ref_store_bytes(TrackStore st) {
    Carver c(nullptr);
    ref_store_carve(c, st);
    return (c.bytes() + 255) & ~(size_t)255;
}

// ygzb_tracker_track in YGZB_TRACK_REF_PREVIOUS mode.  A stream's jobs are tracked in batch order, each against the one
// before it (its first against the stream's reference).  The batch runs in waves (wave w = the w-th job of every stream),
// each wave the whole chain -- sparse alignment, candidates, direct projection, pose-only -- followed by the kernel that
// makes every job the next reference of its stream; all on the context's stream, without a host synchronisation.  Behind
// the last wave the last job's pyramid is copied into the stream's reference slot.  The alignment needs the refined pose
// and depths of a key-frame, so nothing overlaps a local BA here.
int track_previous(ygzb_tracker* t, int n_jobs, const ygzb_track_job* jobs, ygzb_track_result* results) {
    ygzb_ctx* ctx = t->ctx;
    const int S = t->st.S;
    std::vector<int> wave_of(n_jobs), count(S, 0), last(S, -1);
    int n_waves = 0;
    for (int j = 0; j < n_jobs; ++j) {
        const int s = jobs[j].stream;
        if (t->cur_ref[s] < 0) return set_error(ctx, YGZB_ERR_INVALID, "track job %d: stream %d has no reference frame yet", j, s);
        wave_of[j] = count[s]++;
        n_waves = std::max(n_waves, wave_of[j] + 1);
    }
    YGZB_CUDA(ctx, cudaEventSynchronize(t->staged));
    std::vector<int> wave_start(n_waves + 1, 0);
    for (int j = 0; j < n_jobs; ++j) wave_start[wave_of[j] + 1] += 1;
    for (int w = 0; w < n_waves; ++w) wave_start[w + 1] += wave_start[w];
    std::vector<int> fill(wave_start.begin(), wave_start.end() - 1);
    t->pos_of.assign(n_jobs, 0);
    int32_t* h_ref_slot = t->h_aux;
    int32_t* h_orig = t->h_aux + t->max_jobs;
    for (int j = 0; j < n_jobs; ++j) {   // wave-major order, batch order inside a wave
        const int p = fill[wave_of[j]]++, s = jobs[j].stream;
        t->pos_of[j] = p;
        t->h_jobs[p] = jobs[j];
        h_orig[p] = j;
        h_ref_slot[p] = last[s] < 0 ? t->cur_ref[s] : jobs[last[s]].cur_slot;
        last[s] = j;
    }
    TrackBatch b = job_batch(t, n_jobs);
    b.prev = 1;
    b.job_ref_slot = t->d_aux;
    b.orig = t->d_aux + t->max_jobs;
    // the sparse alignment's per-feature scratch, for ref_cap features per problem (a wave has at most one job per stream)
    b.sa2_scratch = static_cast<uint8_t*>(t->d_ref) + ref_store_bytes(t->st);
    const int cl = t->cluster;
    // uploads ran on the front stream; a key-frame insertion (and its BA) is on this stream already
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_up, 0));
    YGZB_CUDA(ctx, cudaMemcpyAsync(const_cast<ygzb_track_job*>(t->b.jobs), t->h_jobs, sizeof(ygzb_track_job) * (size_t)n_jobs,
                                   cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(t->d_aux, t->h_aux, sizeof(int32_t) * 2 * (size_t)t->max_jobs, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaEventRecord(t->staged, ctx->stream));
    for (int w = 0; w < n_waves; ++w) {
        TrackBatch wb = wave_batch(b, wave_start[w], wave_start[w + 1] - wave_start[w]);
        int rc = launch_track_chain_front(t->f, t->st, wb, cl);
        if (rc == YGZB_OK) rc = launch_track_chain_mid(t->f, t->st, wb);
        if (rc == YGZB_OK)
            rc = launch_pose_only_dev(ctx, wb.J, wb.c_off, wb.c_cnt, wb.c_pw, wb.c_px, wb.T_cur, wb.inlier, wb.c_depth, wb.n_inl, wb.enable,
                                      wb.pose_ws, cl, wb.cap, wb.cam);
        if (rc != YGZB_OK) return rc;
        ProfScope ps(ctx, kStageOther);
        track_ref_write_kernel<<<(unsigned)wb.J, 256, 0, ctx->stream>>>(t->st, wb);
        YGZB_LAUNCHED(ctx);
    }
    // (every wave's jobs keep their rows of the batch arrays)
    return finish_batch(t, b, results, [&] {
        for (int s = 0; s < S; ++s)
            if (last[s] >= 0) {
                TRY(ygzb_frames_copy(t->f, jobs[last[s]].cur_slot, t->ref_slots[s]));
                t->cur_ref[s] = t->ref_slots[s];
            }
        return YGZB_OK;
    });
}

extern "C" {

int ygzb_tracker_create(ygzb_frames* f, int n_streams, int max_jobs, const double K[4], ygzb_tracker** out) {
    if (!f || !out || n_streams < 1 || max_jobs < 1 || !K) return YGZB_ERR_INVALID;
    *out = nullptr;
    ygzb_ctx* ctx = f->ctx;
    cudaSetDevice(ctx->device);
    if (ctx->geo.n_cells > 4096) return set_error(ctx, YGZB_ERR_CAPACITY, "tracker: %d grid cells (the BA assembly handles up to 4096)", ctx->geo.n_cells);
    ygzb_tracker* t = new (std::nothrow) ygzb_tracker();
    if (!t) return YGZB_ERR_INVALID;
    t->f = f;
    t->ctx = ctx;
    t->max_jobs = max_jobs;
    t->cluster = cluster_knob("YGZB_TRACK_CLUSTER", kTrackCluster, false);
    const Geometry& g = ctx->geo;
    const size_t S = (size_t)n_streams, R = YGZB_TRACK_RING, cells = (size_t)g.n_cells, E = S * R, cap = kTrackMaxLocal * cells;
    TrackStore& st = t->st;
    st.S = n_streams; st.R = (int)R; st.cells = (int)cells; st.W = g.W; st.H = g.H;
    // every stream starts with K, and with the context's float camera in the solvers
    t->cam_K.resize(4 * S);
    t->cam_F.resize(4 * S);
    for (size_t s = 0; s < S; ++s) {
        std::copy(K, K + 4, &t->cam_K[4 * s]);
        t->cam_F[4 * s] = ctx->prm.fx; t->cam_F[4 * s + 1] = ctx->prm.fy; t->cam_F[4 * s + 2] = ctx->prm.cx; t->cam_F[4 * s + 3] = ctx->prm.cy;
    }
    int rc = check_cuda(ctx, cudaMalloc(&t->d_cam, 4 * S * (sizeof(double) + sizeof(float))), "cudaMalloc(tracker cameras)");
    if (rc == YGZB_OK) {
        st.cam_K = static_cast<double*>(t->d_cam);
        st.cam_F = reinterpret_cast<float*>(static_cast<double*>(t->d_cam) + 4 * S);
        rc = check_cuda(ctx, cudaMemcpyAsync(t->d_cam, t->cam_K.data(), 4 * S * sizeof(double), cudaMemcpyHostToDevice, ctx->stream), "H2D");
    }
    if (rc == YGZB_OK)
        rc = check_cuda(ctx, cudaMemcpyAsync(const_cast<float*>(st.cam_F), t->cam_F.data(), 4 * S * sizeof(float), cudaMemcpyHostToDevice, ctx->stream),
                        "H2D");
    {
        auto carve = [&](Carver& c) {
            st.kf_T = c.take<double>(E * 12); st.kf_n = c.take<int32_t>(E); st.kf_slot = c.take<int32_t>(E); st.kf_mp0 = c.take<long long>(E);
            st.kf_px = c.take<double>(E * cells * 2); st.kf_level = c.take<uint8_t>(E * cells); st.kf_depth = c.take<double>(E * cells);
            st.kf_pw = c.take<double>(E * cells * 3); st.kf_nobs = c.take<int32_t>(E); st.kf_obs_id = c.take<long long>(E * cap);
            st.kf_obs_px = c.take<double>(E * cap * 2);
        };
        Carver sz(nullptr);
        carve(sz);
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMalloc(&t->d_store, sz.bytes()), "cudaMalloc(tracker store)");
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMemsetAsync(t->d_store, 0, sz.bytes(), ctx->stream), "memset");
        if (rc == YGZB_OK) {
            Carver c(t->d_store);
            carve(c);
        }
    }
    if (rc == YGZB_OK) rc = dalloc(ctx, &t->d_depth, S * g.W * g.H);
    st.depth_map = t->d_depth;
    if (rc == YGZB_OK) {
        const size_t J = (size_t)max_jobs, Cn = J * cap;
        TrackBatch& b = t->b;
        b.J = 0;
        b.cap = (int)cap;
        auto carve = [&](Carver& c) {
            b.jobs = c.take<ygzb_track_job>(J);
            b.ref_slot = c.take<int32_t>(J); b.cur_slot = c.take<int32_t>(J); b.offsets = c.take<int32_t>(J + 1); b.in_off = c.take<int32_t>(J);
            b.n_feat = c.take<int32_t>(J); b.n_meas = c.take<int32_t>(J);
            b.T_ref = c.take<double>(J * 12); b.T_cur = c.take<double>(J * 12); b.T_aligned = c.take<double>(J * 12);
            b.sa2_scratch = c.take<double>(sparse_align2_scratch_bytes((int)J, (int)cells) / 8 + 1);
            b.aligned = c.take<int32_t>(J); b.rel = c.take<double>(J * kTrackMaxLocal * 12);
            b.cand_ok = c.take<uint8_t>(Cn); b.cand_px = c.take<double>(Cn * 2); b.n_cand = c.take<int32_t>(J);
            b.c_cnt = c.take<int32_t>(J); b.c_off = c.take<int32_t>(J + 1); b.c_src = c.take<int32_t>(Cn);
            b.c_pw = c.take<double>(Cn * 3); b.c_px = c.take<double>(Cn * 2); b.c_depth = c.take<double>(Cn);
            b.inlier = c.take<uint8_t>(Cn); b.enable = c.take<uint8_t>(Cn); b.n_inl = c.take<int32_t>(J);
            b.pose_ws = c.take<double>(pose_only_ws_doubles((int)J));
            b.results = c.take<ygzb_track_result>(J);
            b.align_H = c.take<double>(J * 21);
            b.cam = c.take<float>(J * 4);
        };
        Carver sz(nullptr);
        carve(sz);
        rc = check_cuda(ctx, cudaMalloc(&t->d_batch, sz.bytes()), "cudaMalloc(tracker batch)");
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMemsetAsync(t->d_batch, 0, sz.bytes(), ctx->stream), "memset");
        if (rc == YGZB_OK) {
            Carver c(t->d_batch);
            carve(c);
        }
    }
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMallocHost((void**)&t->h_jobs, sizeof(ygzb_track_job) * (size_t)max_jobs), "cudaMallocHost");
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMallocHost((void**)&t->h_kfjobs, kf_stage_bytes * S), "cudaMallocHost");
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMalloc((void**)&t->d_kfjobs, kf_stage_bytes * S), "cudaMalloc");
    if (rc == YGZB_OK) {
        t->start_T.assign(12 * S, 0.0);
        for (size_t s = 0; s < S; ++s) t->start_T[12 * s] = t->start_T[12 * s + 5] = t->start_T[12 * s + 10] = 1.0;
        t->sources.assign(S, {RawFormat{st.W, st.H, 1}});
    }
    if (rc == YGZB_OK) rc = dalloc(ctx, &t->d_kfres, S);
    // (a result record carries YGZB_TRACK_RING pose slots and only the first n_local are written by a job: the whole record is
    //  copied back, so start from zeros rather than from whatever cudaMalloc returned)
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMemsetAsync(t->d_kfres, 0, sizeof(ygzb_keyframe_result) * S, ctx->stream), "memset");
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaEventCreateWithFlags(&t->staged, cudaEventDisableTiming), "cudaEventCreate");
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaStreamCreateWithFlags(&t->front, cudaStreamNonBlocking), "cudaStreamCreate");
    for (cudaEvent_t* e : {&t->e_fill, &t->e_front, &t->e_main, &t->e_up})
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaEventCreateWithFlags(e, cudaEventDisableTiming), "cudaEventCreate");
    if (rc == YGZB_OK) {   // (events start out "completed": recorded once on an idle stream)
        rc = check_cuda(ctx, cudaEventRecord(t->e_fill, ctx->stream), "cudaEventRecord");
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaEventRecord(t->e_main, ctx->stream), "cudaEventRecord");
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaEventRecord(t->e_up, ctx->stream), "cudaEventRecord");
    }
    if (rc == YGZB_OK) {
        t->pcap = (int)(kTrackMaxLocal * cells + 1);
        t->ocap = (int)(kTrackMaxLocal * kTrackMaxLocal * cells);
        BABuild B{};
        B.pcap = t->pcap;
        B.ocap = t->ocap;
        Carver sz(nullptr);
        const size_t head = babuild_carve(sz, B, S, (int)cells, (int)S);
        t->ba_bytes = head + ba2_scratch_bytes(S * t->pcap, S * t->ocap, S) + 512;
        rc = check_cuda(ctx, cudaMalloc(&t->d_ba, t->ba_bytes), "cudaMalloc(tracker BA)");
    }
    if (rc != YGZB_OK) {
        ygzb_tracker_destroy(t);
        return rc;
    }
    *out = t;
    return YGZB_OK;
}

void ygzb_tracker_destroy(ygzb_tracker* t) {
    if (!t) return;
    cudaSetDevice(t->ctx->device);
    cudaStreamSynchronize(t->ctx->stream);
    if (t->d_store) cudaFree(t->d_store);
    if (t->d_batch) cudaFree(t->d_batch);
    if (t->d_depth) cudaFree(t->d_depth);
    if (t->h_jobs) cudaFreeHost(t->h_jobs);
    if (t->h_kfjobs) cudaFreeHost(t->h_kfjobs);
    if (t->d_kfjobs) cudaFree(t->d_kfjobs);
    if (t->d_kfres) cudaFree(t->d_kfres);
    if (t->d_ba) cudaFree(t->d_ba);
    if (t->d_xfer) cudaFree(t->d_xfer);
    if (t->d_ref) cudaFree(t->d_ref);
    if (t->h_aux) cudaFreeHost(t->h_aux);
    if (t->d_aux) cudaFree(t->d_aux);
    if (t->d_cam) cudaFree(t->d_cam);
    if (t->staged) cudaEventDestroy(t->staged);
    if (t->front) {
        cudaStreamSynchronize(t->front);
        cudaStreamDestroy(t->front);
    }
    for (cudaEvent_t e : {t->e_fill, t->e_front, t->e_main, t->e_up})
        if (e) cudaEventDestroy(e);
    for (const ygzb_tracker::Source& s : t->sources) {
        if (s.e_maps) cudaEventDestroy(s.e_maps);
        if (s.d_maps) cudaFree(s.d_maps);
        if (s.h_maps) cudaFreeHost(s.h_maps);
    }
    delete t;
}

int ygzb_tracker_set_reference_mode(ygzb_tracker* t, int mode, const int32_t* ref_slots) {
    if (!t) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (mode != YGZB_TRACK_REF_KEYFRAME && mode != YGZB_TRACK_REF_PREVIOUS) return set_error(ctx, YGZB_ERR_INVALID, "reference mode %d", mode);
    if (t->kf_inserted) return set_error(ctx, YGZB_ERR_INVALID, "the reference mode is fixed once a key-frame has been inserted");
    const int S = t->st.S;
    if (mode == YGZB_TRACK_REF_PREVIOUS) {
        if (!ref_slots) return set_error(ctx, YGZB_ERR_INVALID, "previous-frame reference: no reference slots");
        for (int s = 0; s < S; ++s) {
            if (ref_slots[s] < 0 || ref_slots[s] >= t->f->capacity) return set_error(ctx, YGZB_ERR_INVALID, "reference slot of stream %d out of range", s);
            for (int q = 0; q < s; ++q)
                if (ref_slots[q] == ref_slots[s]) return set_error(ctx, YGZB_ERR_INVALID, "streams %d and %d share reference slot %d", q, s, ref_slots[s]);
        }
    }
    cudaSetDevice(ctx->device);
    if (mode == YGZB_TRACK_REF_PREVIOUS && !t->d_ref) {
        TrackStore st = t->st;
        st.ref_cap = (kTrackMaxLocal + 1) * st.cells;
        const size_t head = ref_store_bytes(st);   // (256-byte multiple) the store, then the sparse alignment's wave scratch
        int rc = check_cuda(ctx, cudaMalloc(&t->d_ref, head + sparse_align2_scratch_bytes(S, st.ref_cap)), "cudaMalloc(reference store)");
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMemsetAsync(t->d_ref, 0, head, ctx->stream), "memset");
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMallocHost((void**)&t->h_aux, sizeof(int32_t) * 2 * (size_t)t->max_jobs), "cudaMallocHost");
        if (rc == YGZB_OK) rc = dalloc(ctx, &t->d_aux, 2 * (size_t)t->max_jobs);
        if (rc != YGZB_OK) {
            if (t->d_ref) cudaFree(t->d_ref);
            if (t->h_aux) cudaFreeHost(t->h_aux);
            t->d_ref = nullptr;
            t->h_aux = nullptr;
            return rc;
        }
        Carver c(t->d_ref);
        ref_store_carve(c, st);
        t->st = st;
    }
    t->ref_mode = mode;
    t->ref_slots.assign(ref_slots && mode == YGZB_TRACK_REF_PREVIOUS ? ref_slots : nullptr, ref_slots && mode == YGZB_TRACK_REF_PREVIOUS ? ref_slots + S : nullptr);
    t->cur_ref.assign(S, -1);
    return YGZB_OK;
}

int ygzb_tracker_debug_reference(ygzb_tracker* t, int stream, ygzb_track_reference* out) {
    if (!t || !out) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (t->ref_mode != YGZB_TRACK_REF_PREVIOUS) return set_error(ctx, YGZB_ERR_INVALID, "debug_reference: not in previous-frame reference mode");
    if (stream < 0 || stream >= t->st.S) return set_error(ctx, YGZB_ERR_INVALID, "debug_reference: stream %d out of range", stream);
    if (!out->px || !out->depth) return set_error(ctx, YGZB_ERR_INVALID, "debug_reference: null array");
    cudaSetDevice(ctx->device);
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    int32_t cur = 0, n = 0;
    YGZB_CUDA(ctx, cudaMemcpy(&cur, t->st.ref_cur + stream, sizeof(int32_t), cudaMemcpyDeviceToHost));
    const size_t r = 2 * (size_t)stream + cur;
    YGZB_CUDA(ctx, cudaMemcpy(&n, t->st.ref_n + r, sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (n > out->capacity) return set_error(ctx, YGZB_ERR_CAPACITY, "debug_reference: %d features exceed the capacity %d", n, out->capacity);
    out->slot = t->cur_ref[stream];
    out->n = n;
    YGZB_CUDA(ctx, cudaMemcpy(out->T_cw, t->st.ref_T + 12 * r, 12 * sizeof(double), cudaMemcpyDeviceToHost));
    YGZB_CUDA(ctx, cudaMemcpy(out->px, t->st.ref_px + 2 * r * t->st.ref_cap, 2 * (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
    YGZB_CUDA(ctx, cudaMemcpy(out->depth, t->st.ref_depth + r * t->st.ref_cap, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
    return YGZB_OK;
}

int ygzb_tracker_set_depth(ygzb_tracker* t, int stream, const double* depth) {
    if (!t || !depth || stream < 0 || stream >= t->st.S) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    cudaSetDevice(ctx->device);
    const size_t n = (size_t)t->st.W * t->st.H;
    YGZB_CUDA(ctx, cudaMemcpyAsync(t->d_depth + (size_t)stream * n, depth, n * sizeof(double), cudaMemcpyDefault, ctx->stream));
    return YGZB_OK;
}

int ygzb_tracker_get_depth(ygzb_tracker* t, int stream, double* out) {
    if (!t || !out) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (stream < 0 || stream >= t->st.S) return set_error(ctx, YGZB_ERR_INVALID, "get_depth: stream %d out of range", stream);
    cudaSetDevice(ctx->device);
    const size_t n = (size_t)t->st.W * t->st.H;
    YGZB_CUDA(ctx, cudaMemcpyAsync(out, t->d_depth + (size_t)stream * n, n * sizeof(double), cudaMemcpyDefault, ctx->stream));
    return YGZB_OK;
}

int ygzb_tracker_set_start_pose(ygzb_tracker* t, int stream, const double T_cw[12]) {
    if (!t || !T_cw) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (stream < 0 || stream >= t->st.S) return set_error(ctx, YGZB_ERR_INVALID, "start pose: stream %d out of range", stream);
    for (int c = 0; c < 12; ++c)
        if (!std::isfinite(T_cw[c])) return set_error(ctx, YGZB_ERR_INVALID, "start pose: entry %d is not finite", c);
    // a rotation: R R^T = I and det R = +1, entry by entry within 1e-6
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            const double d = T_cw[4 * r] * T_cw[4 * c] + T_cw[4 * r + 1] * T_cw[4 * c + 1] + T_cw[4 * r + 2] * T_cw[4 * c + 2];
            if (!(std::fabs(d - (r == c ? 1.0 : 0.0)) <= 1e-6)) return set_error(ctx, YGZB_ERR_INVALID, "start pose: rotation is not orthonormal");
        }
    const double det = T_cw[0] * (T_cw[5] * T_cw[10] - T_cw[6] * T_cw[9]) - T_cw[1] * (T_cw[4] * T_cw[10] - T_cw[6] * T_cw[8]) +
                       T_cw[2] * (T_cw[4] * T_cw[9] - T_cw[5] * T_cw[8]);
    if (!(std::fabs(det - 1.0) <= 1e-6)) return set_error(ctx, YGZB_ERR_INVALID, "start pose: rotation has determinant %g", det);
    memcpy(&t->start_T[12 * (size_t)stream], T_cw, 12 * sizeof(double));
    return YGZB_OK;
}

int ygzb_tracker_set_camera(ygzb_tracker* t, int stream, const double K[4]) {
    if (!t || !K) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (stream < 0 || stream >= t->st.S) return set_error(ctx, YGZB_ERR_INVALID, "set_camera: stream %d out of range", stream);
    for (int c = 0; c < 4; ++c)
        if (!std::isfinite(K[c])) return set_error(ctx, YGZB_ERR_INVALID, "set_camera: entry %d is not finite", c);
    if (!(K[0] > 0 && K[1] > 0)) return set_error(ctx, YGZB_ERR_INVALID, "set_camera: focal lengths %g, %g must be positive", K[0], K[1]);
    cudaSetDevice(ctx->device);
    double* hk = &t->cam_K[4 * (size_t)stream];
    float* hf = &t->cam_F[4 * (size_t)stream];
    for (int c = 0; c < 4; ++c) {
        hk[c] = K[c];
        hf[c] = (float)K[c];
    }
    // ordered as an upload (ygzb_tracker_upload): on the front stream, behind the last key-frame insertion's kf_fill_kernel
    // and the last tracking chain, the table's readers on the context's stream, but NOT behind a local BA in flight (its
    // cameras are kernel parameters); the next tracking chain is on the front stream, and a key-frame insertion, an import
    // and previous-frame tracking wait for e_up
    YGZB_CUDA(ctx, cudaStreamWaitEvent(t->front, t->e_fill, 0));
    YGZB_CUDA(ctx, cudaStreamWaitEvent(t->front, t->e_main, 0));
    YGZB_CUDA(ctx, cudaMemcpyAsync(const_cast<double*>(t->st.cam_K) + 4 * stream, hk, 4 * sizeof(double), cudaMemcpyHostToDevice, t->front));
    YGZB_CUDA(ctx, cudaMemcpyAsync(const_cast<float*>(t->st.cam_F) + 4 * stream, hf, 4 * sizeof(float), cudaMemcpyHostToDevice, t->front));
    YGZB_CUDA(ctx, cudaEventRecord(t->e_up, t->front));
    return YGZB_OK;
}

int ygzb_tracker_set_undistort(ygzb_tracker* t, int stream, const int16_t* map_xy, const uint16_t* map_a) {
    if (!t) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (stream < 0 || stream >= t->st.S) return set_error(ctx, YGZB_ERR_INVALID, "set_undistort: stream %d out of range", stream);
    if (!map_xy != !map_a) return set_error(ctx, YGZB_ERR_INVALID, "set_undistort: map_xy and map_a must both be given, or both be NULL");
    ygzb_tracker::Source& s = t->sources[stream];
    if (!map_xy) {   // uploads enqueued before keep reading the maps, which stay allocated until the tracker is destroyed
        s.has_maps = false;
        return YGZB_OK;
    }
    ygzb_frames* f = t->f;
    if (f->undistort) return set_error(ctx, YGZB_ERR_INVALID, "set_undistort: the frame pool has undistortion maps of its own");
    cudaSetDevice(ctx->device);
    const size_t n = (size_t)t->st.W * t->st.H, a_off = lens_a_offset(n);
    if (!s.h_maps) {
        YGZB_CUDA(ctx, cudaMallocHost((void**)&s.h_maps, lens_bytes(n)));
        YGZB_CUDA(ctx, cudaMalloc((void**)&s.d_maps, lens_bytes(n)));
        YGZB_CUDA(ctx, cudaEventCreateWithFlags(&s.e_maps, cudaEventDisableTiming));
    } else {   // the staging's last copy to the device has run (it waited for nothing but earlier front-stream work)
        YGZB_CUDA(ctx, cudaEventSynchronize(s.e_maps));
    }
    if (!f->e_stage) YGZB_CUDA(ctx, cudaEventCreateWithFlags(&f->e_stage, cudaEventDisableTiming));
    // the maps (host or device memory) are read into the staging and checked before anything an upload reads changes
    uint8_t* h = s.h_maps;
    const uint16_t* a = reinterpret_cast<const uint16_t*>(h + a_off);
    YGZB_CUDA(ctx, cudaMemcpy(h, map_xy, n * sizeof(short2), cudaMemcpyDefault));
    YGZB_CUDA(ctx, cudaMemcpy(h + a_off, map_a, n * sizeof(uint16_t), cudaMemcpyDefault));
    for (size_t i = 0; i < n; ++i)
        if (a[i] >= 1024)
            return set_error(ctx, YGZB_ERR_INVALID, "set_undistort: map_a[%zu] = %d is not a 5 + 5-bit fraction (< 1024)", i, (int)a[i]);
    // in order on the front stream, which runs every upload: the ones enqueued before read the old maps, the ones enqueued
    // after the new; nothing waits for the key-frame insertion or a local BA in flight
    YGZB_CUDA(ctx, cudaMemcpyAsync(s.d_maps, h, lens_bytes(n), cudaMemcpyHostToDevice, t->front));
    YGZB_CUDA(ctx, cudaEventRecord(s.e_maps, t->front));
    s.has_maps = true;
    return YGZB_OK;
}

int ygzb_tracker_set_source(ygzb_tracker* t, int stream, int width, int height, int channels) {
    if (!t) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (stream < 0 || stream >= t->st.S) return set_error(ctx, YGZB_ERR_INVALID, "set_source: stream %d out of range", stream);
    // (the maps' int16 source coordinates reach 32767)
    if (width < 1 || height < 1 || width > 32767 || height > 32767)
        return set_error(ctx, YGZB_ERR_INVALID, "set_source: a raw frame of %d x %d is not within 1 .. 32767 each way", width, height);
    if (channels != 1 && channels != 3) return set_error(ctx, YGZB_ERR_INVALID, "set_source: channels must be 1 or 3, not %d", channels);
    // read when an upload is enqueued, so the uploads enqueued before the call read the old format and those after it the new
    // one, in order on the front stream like the maps (ygzb_tracker_set_undistort)
    t->sources[stream].raw = RawFormat{width, height, channels};
    return YGZB_OK;
}

// on the front stream, behind the last key-frame insertion (which still reads the frame slots of the previous window) and
// behind the last tracking chain (ditto); NOT behind a local BA in flight.  Frames of format `src`; map_xy / map_a: the
// undistortion maps of level 0, or NULL
static int upload_front(ygzb_tracker* t, int first, int count, const uint8_t* host, RawFormat src, size_t frame_stride, const short2* map_xy,
                        const uint16_t* map_a) {
    ygzb_ctx* ctx = t->ctx;
    cudaSetDevice(ctx->device);
    YGZB_CUDA(ctx, cudaStreamWaitEvent(t->front, t->e_fill, 0));
    YGZB_CUDA(ctx, cudaStreamWaitEvent(t->front, t->e_main, 0));
    cudaStream_t main = ctx->stream;
    ctx->stream = t->front;
    int rc = frames_upload(t->f, first, count, host, src, frame_stride, map_xy, map_a);
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaEventRecord(t->e_up, ctx->stream), "cudaEventRecord");
    ctx->stream = main;
    return rc;
}

int ygzb_tracker_upload(ygzb_tracker* t, int first, int count, const uint8_t* host, size_t frame_stride) {
    if (!t) return YGZB_ERR_INVALID;
    ygzb_frames* f = t->f;
    return upload_front(t, first, count, host, RawFormat{t->st.W, t->st.H, 1}, frame_stride, f->undistort ? f->d_map_xy : nullptr, f->d_map_a);
}

int ygzb_tracker_upload_stream(ygzb_tracker* t, int stream, int first, int count, const uint8_t* host, size_t frame_stride) {
    if (!t) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (stream < 0 || stream >= t->st.S) return set_error(ctx, YGZB_ERR_INVALID, "upload_stream: stream %d out of range", stream);
    const ygzb_tracker::Source& s = t->sources[stream];
    ygzb_frames* f = t->f;
    if (s.has_maps && f->undistort)
        return set_error(ctx, YGZB_ERR_INVALID, "upload_stream: stream %d and the frame pool both have undistortion maps", stream);
    // level 0 is remapped through the stream's maps, else through the pool's, else converted or copied at level 0's size
    const short2* map_xy = s.has_maps ? reinterpret_cast<const short2*>(s.d_maps) : f->undistort ? f->d_map_xy : nullptr;
    const uint16_t* map_a = s.has_maps ? reinterpret_cast<const uint16_t*>(s.d_maps + lens_a_offset((size_t)t->st.W * t->st.H)) : f->d_map_a;
    return upload_front(t, first, count, host, s.raw, frame_stride, map_xy, map_a);
}

int ygzb_tracker_track(ygzb_tracker* t, int n_jobs, const ygzb_track_job* jobs, ygzb_track_result* results) {
    if (!t || n_jobs < 0 || (n_jobs && (!jobs || !results))) return YGZB_ERR_INVALID;
    if (n_jobs == 0) return YGZB_OK;
    ygzb_ctx* ctx = t->ctx;
    cudaSetDevice(ctx->device);
    if (n_jobs > t->max_jobs) return set_error(ctx, YGZB_ERR_CAPACITY, "%d jobs exceed the tracker's max_jobs %d", n_jobs, t->max_jobs);
    for (int j = 0; j < n_jobs; ++j) {
        const ygzb_track_job& q = jobs[j];
        if (q.stream < 0 || q.stream >= t->st.S || q.cur_slot < 0 || q.cur_slot >= t->f->capacity || q.n_local < 1 || q.n_local > kTrackMaxLocal - 1)
            return set_error(ctx, YGZB_ERR_INVALID, "track job %d: stream / slot / n_local out of range", j);
        for (int k = 0; k < q.n_local; ++k)
            if (q.entry[k] < 0 || q.entry[k] >= YGZB_TRACK_RING) return set_error(ctx, YGZB_ERR_INVALID, "track job %d: ring entry out of range", j);
    }
    if (t->ref_mode == YGZB_TRACK_REF_PREVIOUS) return track_previous(t, n_jobs, jobs, results);
    YGZB_CUDA(ctx, cudaEventSynchronize(t->staged));   // the previous copy out of the staging buffer has finished
    memcpy(t->h_jobs, jobs, sizeof(ygzb_track_job) * (size_t)n_jobs);
    const TrackBatch b = job_batch(t, n_jobs);
    t->pos_of.clear();
    const int cl = t->cluster;
    int rc;
    {   // part 1 on the front stream: behind the key-frame insertion (new reference features, and the batch arrays it still
        // reads) and the previous chain, concurrent with a local BA on the main stream
        cudaStream_t main = ctx->stream;
        YGZB_CUDA(ctx, cudaStreamWaitEvent(t->front, t->e_fill, 0));
        YGZB_CUDA(ctx, cudaStreamWaitEvent(t->front, t->e_main, 0));
        ctx->stream = t->front;
        cudaError_t ce = cudaMemcpyAsync(const_cast<ygzb_track_job*>(t->b.jobs), t->h_jobs, sizeof(ygzb_track_job) * (size_t)n_jobs,
                                         cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess) ce = cudaEventRecord(t->staged, ctx->stream);
        rc = ce == cudaSuccess ? launch_track_chain_front(t->f, t->st, b, cl) : check_cuda(ctx, ce, "H2D(track jobs)");
        if (rc == YGZB_OK) rc = check_cuda(ctx, cudaEventRecord(t->e_front, ctx->stream), "cudaEventRecord");
        ctx->stream = main;
        if (rc != YGZB_OK) return rc;
        YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_front, 0));
    }
    rc = launch_track_chain_mid(t->f, t->st, b);
    if (rc != YGZB_OK) return rc;
    rc = launch_pose_only_dev(ctx, n_jobs, b.c_off, b.c_cnt, b.c_pw, b.c_px, b.T_cur, b.inlier, b.c_depth, b.n_inl, b.enable, b.pose_ws, cl, b.cap,
                              b.cam);
    if (rc != YGZB_OK) return rc;
    return finish_batch(t, b, results, [] { return YGZB_OK; });
}

int ygzb_tracker_make_keyframes(ygzb_tracker* t, int n, const ygzb_keyframe_job* jobs, const ygzb_ba_params* ba,
                                ygzb_keyframe_result* results) {
    if (!t || n < 0 || (n && (!jobs || !results || !ba))) return YGZB_ERR_INVALID;
    if (n == 0) return YGZB_OK;
    ygzb_ctx* ctx = t->ctx;
    ygzb_frames* f = t->f;
    cudaSetDevice(ctx->device);
    if (n > t->st.S) return set_error(ctx, YGZB_ERR_CAPACITY, "%d key-frame jobs for %d streams", n, t->st.S);
    std::vector<int32_t> slots(n), prob_of(n);
    int P = 0;
    for (int i = 0; i < n; ++i) {
        const ygzb_keyframe_job& q = jobs[i];
        if (q.stream < 0 || q.stream >= t->st.S || q.frame_slot < 0 || q.frame_slot >= f->capacity || q.kf_slot < 0 || q.kf_slot >= f->capacity ||
            q.entry < 0 || q.entry >= YGZB_TRACK_RING || q.track_job >= t->last_J || q.n_local < 1 || q.n_local > kTrackMaxLocal - 1)
            return set_error(ctx, YGZB_ERR_INVALID, "key-frame job %d: field out of range", i);
        for (int k = 0; k < q.n_local; ++k)
            if (q.local_entry[k] < 0 || q.local_entry[k] >= YGZB_TRACK_RING) return set_error(ctx, YGZB_ERR_INVALID, "key-frame job %d: ring entry out of range", i);
        if (q.local_entry[q.n_local - 1] != q.entry) return set_error(ctx, YGZB_ERR_INVALID, "key-frame job %d: the newest local key-frame must be the inserted one", i);
        for (int i2 = 0; i2 < i; ++i2)
            if (jobs[i2].stream == q.stream) return set_error(ctx, YGZB_ERR_INVALID, "two key-frame jobs for stream %d", q.stream);
        slots[i] = q.frame_slot;
        prob_of[i] = (q.run_ba && q.n_local >= 2) ? P++ : -1;
    }
    // FeatureDetector::Detect on the frames (results stay in the slots' feature store); the frames may have been uploaded on
    // the front stream without a tracking chain behind them (first frame of a stream)
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_up, 0));
    int rc = ygzb_detect(f, slots.data(), n, nullptr, nullptr);
    if (rc != YGZB_OK) return rc;
    for (int i = 0; i < n; ++i)
        if (jobs[i].frame_slot != jobs[i].kf_slot) {
            rc = ygzb_frames_copy(f, jobs[i].frame_slot, jobs[i].kf_slot);   // the key-frame keeps its pyramid (Frame.h:138)
            if (rc != YGZB_OK) return rc;
        }
    YGZB_CUDA(ctx, cudaEventSynchronize(t->staged));
    memcpy(t->h_kfjobs, jobs, sizeof(ygzb_keyframe_job) * (size_t)n);
    // the start pose of every job's stream as it is now, right behind the n jobs: a later ygzb_tracker_set_start_pose does
    // not reach an insertion already enqueued
    double* h_start = reinterpret_cast<double*>(t->h_kfjobs + n);
    for (int i = 0; i < n; ++i) memcpy(h_start + 12 * (size_t)i, &t->start_T[12 * (size_t)jobs[i].stream], 12 * sizeof(double));
    const bool prev = t->ref_mode == YGZB_TRACK_REF_PREVIOUS;
    for (int i = 0; i < n; ++i)   // (previous-frame mode keeps the batch in wave order)
        if (jobs[i].track_job >= 0 && !t->pos_of.empty()) t->h_kfjobs[i].track_job = t->pos_of[jobs[i].track_job];
    t->kf_inserted = true;
    YGZB_CUDA(ctx, cudaMemcpyAsync(t->d_kfjobs, t->h_kfjobs, kf_stage_bytes * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    const double* d_start = reinterpret_cast<const double*>(t->d_kfjobs + n);
    BABuild B{};
    B.pcap = t->pcap;
    B.ocap = t->ocap;
    Carver c(t->d_ba);
    const size_t head = babuild_carve(c, B, (size_t)t->st.S, t->st.cells, t->st.S);
    // the problem indices travel behind the jobs in the same staging buffer's lifetime: small synchronous-safe copy from a
    // host vector is fine because the stream is synchronised on `staged` before the vector dies (cudaMemcpyAsync from pageable
    // memory returns after the data has been staged)
    YGZB_CUDA(ctx, cudaMemcpyAsync(B.prob_of, prob_of.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaEventRecord(t->staged, ctx->stream));
    TrackBatch b = t->b;
    b.J = t->last_J;
    {
        ProfScope ps(ctx, kStageOther);
        kf_fill_kernel<<<(unsigned)n, 1024, 0, ctx->stream>>>(t->st, b, t->d_kfjobs, d_start, f->d_count, f->d_fx, f->d_fy, f->d_flevel,
                                                             ctx->geo.n_cells, t->d_kfres);
        YGZB_LAUNCHED(ctx);
    }
    // from here on only the BA runs: the next batch's front part may start (key-frame mode: the alignment is relative to the
    // key-frame and needs its features only; previous-frame mode records this behind the reference, below)
    if (!prev) YGZB_CUDA(ctx, cudaEventRecord(t->e_fill, ctx->stream));
    double* d_ba_stats = nullptr;
    if (P > 0) {
        {
            ProfScope ps(ctx, kStageOther);
            ba_build_kernel<<<(unsigned)n, 1024, 0, ctx->stream>>>(t->st, t->d_kfjobs, B, b.cap);
            YGZB_LAUNCHED(ctx);
        }
        BA2Problem in{};
        in.n_problems = P;
        in.kf_off = B.kf_off; in.pt_off = B.pt_off; in.obs_off = B.obs_off;
        in.n_kf = B.n_kf; in.n_pt = B.n_pt;
        in.poses = B.poses; in.fixed = B.fixed; in.pts = B.pts;
        in.kf_idx = B.so_kf; in.pt_idx = nullptr; in.obs = B.so_uv; in.lm_start = B.lm_start;
        in.total_pts = (size_t)P * t->pcap;
        in.total_obs = (size_t)P * t->ocap;
        int max_local = 1;
        for (int i = 0; i < n; ++i) max_local = std::max(max_local, jobs[i].n_local);
        in.max_pts = (size_t)(max_local - 1) * t->st.cells;   // the newest key-frame's own points have one observation: never in the BA
        in.max_obs = (size_t)max_local * in.max_pts;
        in.max_free = max_local - 1;
        in.max_kf = max_local;
        std::vector<float> cams(4 * (size_t)P);   // the float camera of every problem's stream
        for (int i = 0; i < n; ++i)
            if (prob_of[i] >= 0) std::copy_n(&t->cam_F[4 * (size_t)jobs[i].stream], 4, &cams[4 * (size_t)prob_of[i]]);
        in.cam = reinterpret_cast<const float(*)[4]>(cams.data());
        void* scratch = static_cast<uint8_t*>(t->d_ba) + ((head + 255) & ~(size_t)255);
        rc = launch_local_ba2(ctx, in, scratch, ba, nullptr, &d_ba_stats);
        if (rc != YGZB_OK) return rc;
    }
    {
        ProfScope ps(ctx, kStageOther);
        ba_writeback_kernel<<<(unsigned)n, 256, 0, ctx->stream>>>(t->st, t->d_kfjobs, B, d_ba_stats, t->d_kfres);
        YGZB_LAUNCHED(ctx);
    }
    if (prev) {   // the key-frame becomes its stream's reference, with the BA's pose and points
        {
            ProfScope ps(ctx, kStageOther);
            kf_ref_kernel<<<(unsigned)n, 256, 0, ctx->stream>>>(t->st, b, t->d_kfjobs);
            YGZB_LAUNCHED(ctx);
        }
        for (int i = 0; i < n; ++i) t->cur_ref[jobs[i].stream] = jobs[i].kf_slot;
        YGZB_CUDA(ctx, cudaEventRecord(t->e_fill, ctx->stream));
    }
    if (t->d_map) {   // (behind the reference, so that previous-frame mode's next alignment does not wait for the rows)
        ProfScope ps(ctx, kStageOther);
        kf_points_kernel<<<(unsigned)n, 1024, 0, ctx->stream>>>(t->st, t->d_kfjobs, B, t->d_map);
        YGZB_LAUNCHED(ctx);
    }
    YGZB_CUDA(ctx, cudaMemcpyAsync(results, t->d_kfres, sizeof(ygzb_keyframe_result) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    return YGZB_OK;
}

// (the row buffers are 16-byte aligned: their kernels write the rows as 16-byte stores)
int ygzb_tracker_set_observations(ygzb_tracker* t, ygzb_observation* host, size_t capacity) {
    if (!t) return YGZB_ERR_INVALID;
    TRY(attach_output(t, host, capacity, (size_t)t->max_jobs * t->b.cap, 16, "set_observations",
                      "rows below max_jobs * " STRINGIFY(YGZB_TRACK_RING) " * cells", &t->d_obs));
    if (host) YGZB_CUDA(t->ctx, cudaFuncSetAttribute(track_obs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kObsSmem));
    return YGZB_OK;
}

int ygzb_tracker_set_information(ygzb_tracker* t, ygzb_pose_information* host, size_t capacity) {
    if (!t) return YGZB_ERR_INVALID;
    return attach_output(t, host, capacity, (size_t)t->max_jobs, alignof(double), "set_information", "records below max_jobs", &t->d_info);
}

int ygzb_tracker_set_map_updates(ygzb_tracker* t, ygzb_map_point* host, size_t capacity) {
    if (!t) return YGZB_ERR_INVALID;
    // a key-frame batch has at most one job per stream
    return attach_output(t, host, capacity, (size_t)t->st.S * YGZB_TRACK_RING * t->st.cells, 16, "set_map_updates",
                         "rows below n_streams * " STRINGIFY(YGZB_TRACK_RING) " * cells", &t->d_map);
}

int ygzb_tracker_export(ygzb_tracker* t, int stream, int n_entries, const int32_t* entries, ygzb_map_record* out) {
    if (!t || !out) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    const TrackStore& st = t->st;
    if (stream < 0 || stream >= st.S) return set_error(ctx, YGZB_ERR_INVALID, "export: stream %d out of range", stream);
    if (n_entries < 0 || n_entries > YGZB_TRACK_RING || (n_entries && !entries))
        return set_error(ctx, YGZB_ERR_INVALID, "export: %d entries (at most %d)", n_entries, YGZB_TRACK_RING);
    if (n_entries && (!out->entry || !out->T_cw || !out->mp0 || !out->n_features || !out->n_obs || !out->px || !out->level || !out->depth ||
                      !out->pw || !out->obs_id || !out->obs_px))
        return set_error(ctx, YGZB_ERR_INVALID, "export: null array in the record");
    int rc = check_entries(t, n_entries, entries, nullptr, "export");
    if (rc != YGZB_OK) return rc;
    cudaSetDevice(ctx->device);
    out->width = st.W; out->height = st.H; out->cells = st.cells; out->n_levels = ctx->geo.n_levels;
    std::copy_n(&t->cam_K[4 * (size_t)stream], 4, out->K);
    out->n_keyframes = n_entries;
    out->pad = 0;
    for (int k = 0; k < n_entries; ++k) out->entry[k] = entries[k];
    if (n_entries == 0) return YGZB_OK;
    MapXfer X;
    rc = tracker_xfer(t, X);
    if (rc != YGZB_OK) return rc;
    MapXferJob job{};
    job.n = n_entries;
    job.stream = stream;
    job.with_image = out->image != nullptr;
    for (int k = 0; k < n_entries; ++k) job.entry[k] = entries[k];
    // on the context's stream: behind every key-frame insertion and local BA enqueued so far; behind the front stream's
    // uploads as well, in case a caller uploads into a key-frame's slot
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_up, 0));
    {
        ProfScope ps(ctx, kStageOther);
        const LevelGeom& lv = ctx->geo.lv[0];
        map_pack_kernel<<<dim3((unsigned)n_entries, kXferChunks), 256, 0, ctx->stream>>>(st, X, job, t->b.cap, t->f->d_pyr, ctx->slot_stride,
                                                                                          lv.off, lv.pitch);
        YGZB_LAUNCHED(ctx);
    }
    const size_t n = (size_t)n_entries, F = n * st.cells, O = n * t->b.cap;
    auto d2h = [&](void* dst, const void* src, size_t bytes) {
        return check_cuda(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream), "D2H(map record)");
    };
    if (rc == YGZB_OK) rc = d2h(out->T_cw, X.T, n * 12 * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->mp0, X.mp0, n * sizeof(int64_t));
    if (rc == YGZB_OK) rc = d2h(out->n_features, X.n_feat, n * sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(out->n_obs, X.n_obs, n * sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(out->px, X.px, F * 2 * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->level, X.level, F);
    if (rc == YGZB_OK) rc = d2h(out->depth, X.depth, F * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->pw, X.pw, F * 3 * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->obs_id, X.obs_id, O * sizeof(int64_t));
    if (rc == YGZB_OK) rc = d2h(out->obs_px, X.obs_px, O * 2 * sizeof(double));
    if (rc == YGZB_OK && out->image) rc = d2h(out->image, X.image, n * st.W * st.H);
    return rc;
}

int ygzb_tracker_import(ygzb_tracker* t, int stream, const int32_t* entries, const int32_t* kf_slots, const ygzb_map_record* in) {
    if (!t || !in) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    const TrackStore& st = t->st;
    // ---- the whole record is checked before anything is enqueued
    if (stream < 0 || stream >= st.S) return set_error(ctx, YGZB_ERR_INVALID, "import: stream %d out of range", stream);
    if (in->width != st.W || in->height != st.H || in->cells != st.cells || in->n_levels != ctx->geo.n_levels)
        return set_error(ctx, YGZB_ERR_INVALID, "import: record geometry %dx%d, %d cells, %d levels; tracker %dx%d, %d cells, %d levels", in->width,
                         in->height, in->cells, in->n_levels, st.W, st.H, st.cells, ctx->geo.n_levels);
    const double* K = &t->cam_K[4 * (size_t)stream];
    if (!(in->K[0] == K[0] && in->K[1] == K[1] && in->K[2] == K[2] && in->K[3] == K[3]))
        return set_error(ctx, YGZB_ERR_INVALID, "import: record intrinsics differ from the stream's camera");
    const int n = in->n_keyframes;
    if (n < 0 || n > YGZB_TRACK_RING) return set_error(ctx, YGZB_ERR_INVALID, "import: %d key-frames (at most %d)", n, YGZB_TRACK_RING);
    if (n == 0) return YGZB_OK;
    if (!entries || !kf_slots || !in->T_cw || !in->mp0 || !in->n_features || !in->n_obs)
        return set_error(ctx, YGZB_ERR_INVALID, "import: null array in the record");
    if (!in->image) return set_error(ctx, YGZB_ERR_INVALID, "import: the record has no images");
    int rc = check_entries(t, n, entries, kf_slots, "import");
    if (rc != YGZB_OK) return rc;
    MapXferJob job{};
    job.n = n;
    job.stream = stream;
    for (int k = 0; k < n; ++k) {
        if (in->n_features[k] < 0 || in->n_features[k] > st.cells)
            return set_error(ctx, YGZB_ERR_INVALID, "import: key-frame %d has %d features (capacity %d)", k, in->n_features[k], st.cells);
        if (in->n_obs[k] < 0 || in->n_obs[k] > t->b.cap)
            return set_error(ctx, YGZB_ERR_INVALID, "import: key-frame %d has %d observations (capacity %d)", k, in->n_obs[k], t->b.cap);
        job.entry[k] = entries[k];
        job.slot[k] = kf_slots[k];
        job.foff[k + 1] = job.foff[k] + in->n_features[k];
        job.ooff[k + 1] = job.ooff[k] + in->n_obs[k];
    }
    const size_t F = (size_t)job.foff[n], O = (size_t)job.ooff[n];
    if ((F && (!in->px || !in->level || !in->depth || !in->pw)) || (O && (!in->obs_id || !in->obs_px)))
        return set_error(ctx, YGZB_ERR_INVALID, "import: null array in the record");
    for (size_t i = 0; i < F; ++i)
        if (in->level[i] >= ctx->geo.n_levels)
            return set_error(ctx, YGZB_ERR_INVALID, "import: feature %zu on level %d of a %d-level pyramid", i, (int)in->level[i], ctx->geo.n_levels);
    // ---- enqueue on the context's stream, behind the front stream's uploads and sparse alignment (they read the ring and
    //      the key-frame slots); the next upload or tracking chain waits for e_fill
    cudaSetDevice(ctx->device);
    MapXfer X;
    rc = tracker_xfer(t, X);
    if (rc != YGZB_OK) return rc;
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_up, 0));
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_front, 0));
    auto h2d = [&](void* dst, const void* src, size_t bytes) {
        return bytes ? check_cuda(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream), "H2D(map record)") : YGZB_OK;
    };
    const size_t nk = (size_t)n;
    if (rc == YGZB_OK) rc = h2d(X.T, in->T_cw, nk * 12 * sizeof(double));
    if (rc == YGZB_OK) rc = h2d(X.mp0, in->mp0, nk * sizeof(int64_t));
    if (rc == YGZB_OK) rc = h2d(X.px, in->px, F * 2 * sizeof(double));
    if (rc == YGZB_OK) rc = h2d(X.level, in->level, F);
    if (rc == YGZB_OK) rc = h2d(X.depth, in->depth, F * sizeof(double));
    if (rc == YGZB_OK) rc = h2d(X.pw, in->pw, F * 3 * sizeof(double));
    if (rc == YGZB_OK) rc = h2d(X.obs_id, in->obs_id, O * sizeof(int64_t));
    if (rc == YGZB_OK) rc = h2d(X.obs_px, in->obs_px, O * 2 * sizeof(double));
    if (rc != YGZB_OK) return rc;
    {
        ProfScope ps(ctx, kStageOther);
        map_unpack_kernel<<<dim3((unsigned)n, kXferChunks), 256, 0, ctx->stream>>>(st, X, job, t->b.cap);
        YGZB_LAUNCHED(ctx);
    }
    const size_t WH = (size_t)st.W * st.H;
    // the record's images are level 0 of key-frames, undistorted already: the pool's undistortion maps must not warp them again
    for (int k = 0; k < n && rc == YGZB_OK; ++k) rc = frames_upload(t->f, kf_slots[k], 1, in->image + k * WH, RawFormat{st.W, st.H, 1}, WH, nullptr, nullptr);
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaEventRecord(t->e_fill, ctx->stream), "cudaEventRecord");
    return rc;
}

int ygzb_tracker_export_reference(ygzb_tracker* t, int stream, ygzb_reference_record* out) {
    if (!t || !out) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    const TrackStore& st = t->st;
    int rc = check_reference_call(t, stream, out, "export_reference");
    if (rc != YGZB_OK) return rc;
    const int slot = t->cur_ref[stream];
    if (slot < 0) return set_error(ctx, YGZB_ERR_INVALID, "export_reference: stream %d has no reference yet", stream);
    cudaSetDevice(ctx->device);
    out->width = st.W; out->height = st.H; out->cells = st.cells; out->n_levels = ctx->geo.n_levels;
    std::copy_n(&t->cam_K[4 * (size_t)stream], 4, out->K);
    MapXfer X;
    rc = tracker_xfer(t, X);
    if (rc != YGZB_OK) return rc;
    // on the context's stream, where previous-frame tracking (its copy into the reference slot included) and key-frame
    // insertion (kf_ref_kernel included) run; behind the front stream's uploads, in case a caller uploads into the slot
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_up, 0));
    {
        ProfScope ps(ctx, kStageOther);
        const LevelGeom& lv = ctx->geo.lv[0];
        ref_pack_kernel<<<kXferChunks, 256, 0, ctx->stream>>>(st, X, stream, t->f->d_pyr + (size_t)slot * ctx->slot_stride + lv.off, lv.pitch);
        YGZB_LAUNCHED(ctx);
    }
    const size_t cap = st.ref_cap;
    auto d2h = [&](void* dst, const void* src, size_t bytes) {
        return check_cuda(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream), "D2H(reference record)");
    };
    if (rc == YGZB_OK) rc = d2h(&out->n, X.ref_n, sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(out->T_cw, X.ref_T, 12 * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->px, X.ref_px, cap * 2 * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->depth, X.ref_depth, cap * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->image, X.ref_image, (size_t)st.W * st.H);
    if (rc == YGZB_OK && (size_t)out->capacity > cap) {   // rows the store cannot hold: zero, like the store's rows past n
        memset(out->px + 2 * cap, 0, ((size_t)out->capacity - cap) * 2 * sizeof(double));
        memset(out->depth + cap, 0, ((size_t)out->capacity - cap) * sizeof(double));
    }
    return rc;
}

int ygzb_tracker_import_reference(ygzb_tracker* t, int stream, const ygzb_reference_record* in) {
    if (!t || !in) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    const TrackStore& st = t->st;
    // ---- the whole record is checked before anything is enqueued
    int rc = check_reference_call(t, stream, in, "import_reference");
    if (rc != YGZB_OK) return rc;
    if (in->width != st.W || in->height != st.H || in->cells != st.cells || in->n_levels != ctx->geo.n_levels)
        return set_error(ctx, YGZB_ERR_INVALID, "import_reference: record geometry %dx%d, %d cells, %d levels; tracker %dx%d, %d cells, %d levels",
                         in->width, in->height, in->cells, in->n_levels, st.W, st.H, st.cells, ctx->geo.n_levels);
    const double* K = &t->cam_K[4 * (size_t)stream];
    if (!(in->K[0] == K[0] && in->K[1] == K[1] && in->K[2] == K[2] && in->K[3] == K[3]))
        return set_error(ctx, YGZB_ERR_INVALID, "import_reference: record intrinsics differ from the stream's camera");
    const int n = in->n;
    if (n < 0 || n > st.ref_cap) return set_error(ctx, YGZB_ERR_INVALID, "import_reference: %d features (capacity %d)", n, st.ref_cap);
    // ---- enqueue on the context's stream, behind the front stream's uploads and sparse alignment, like an import of a map;
    //      the next upload waits for e_fill
    cudaSetDevice(ctx->device);
    MapXfer X;
    rc = tracker_xfer(t, X);
    if (rc != YGZB_OK) return rc;
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_up, 0));
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, t->e_front, 0));
    auto h2d = [&](void* dst, const void* src, size_t bytes) {
        return bytes ? check_cuda(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream), "H2D(reference record)") : YGZB_OK;
    };
    if (rc == YGZB_OK) rc = h2d(X.ref_T, in->T_cw, 12 * sizeof(double));
    if (rc == YGZB_OK) rc = h2d(X.ref_px, in->px, (size_t)n * 2 * sizeof(double));
    if (rc == YGZB_OK) rc = h2d(X.ref_depth, in->depth, (size_t)n * sizeof(double));
    if (rc != YGZB_OK) return rc;
    {
        ProfScope ps(ctx, kStageOther);
        ref_unpack_kernel<<<kXferChunks, 256, 0, ctx->stream>>>(st, X, stream, n);
        YGZB_LAUNCHED(ctx);
    }
    const size_t WH = (size_t)st.W * st.H;
    rc = frames_upload(t->f, t->ref_slots[stream], 1, in->image, RawFormat{st.W, st.H, 1}, WH, nullptr, nullptr);   // undistorted already, like a map record's images
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaEventRecord(t->e_fill, ctx->stream), "cudaEventRecord");
    if (rc != YGZB_OK) return rc;
    t->cur_ref[stream] = t->ref_slots[stream];
    t->kf_inserted = true;   // the stream has a reference of the previous-frame mode: the mode is fixed from here on
    return YGZB_OK;
}

int ygzb_tracker_debug_job(ygzb_tracker* t, int job, ygzb_track_debug* out) {
    if (!t || !out) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = t->ctx;
    if (job < 0 || job >= t->last_J) return set_error(ctx, YGZB_ERR_INVALID, "debug: job %d is not in the last batch (%d jobs)", job, t->last_J);
    if (!out->cand_ok || !out->cand_px || !out->c_src || !out->c_px || !out->c_pw || !out->inlier)
        return set_error(ctx, YGZB_ERR_INVALID, "debug: null array");
    cudaSetDevice(ctx->device);
    const TrackBatch& b = t->b;
    if (!t->pos_of.empty()) job = t->pos_of[job];   // previous-frame mode keeps the batch in wave order
    const size_t j = (size_t)job, cap = (size_t)b.cap;
    auto d2h = [&](void* dst, const void* src, size_t bytes) {
        return check_cuda(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream), "D2H(track debug)");
    };
    int rc = d2h(out->T_aligned, b.T_aligned + 12 * j, 12 * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->rel, b.rel + 12 * kTrackMaxLocal * j, 12 * kTrackMaxLocal * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(&out->n_meas, b.n_meas + j, sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(&out->aligned, b.aligned + j, sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(&out->n_candidates, b.n_cand + j, sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(&out->n_projected, b.c_cnt + j, sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(&out->n_inliers, b.n_inl + j, sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(out->cand_ok, b.cand_ok + cap * j, cap);
    if (rc == YGZB_OK) rc = d2h(out->cand_px, b.cand_px + 2 * cap * j, 2 * cap * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->c_src, b.c_src + cap * j, cap * sizeof(int32_t));
    if (rc == YGZB_OK) rc = d2h(out->c_px, b.c_px + 2 * cap * j, 2 * cap * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->c_pw, b.c_pw + 3 * cap * j, 3 * cap * sizeof(double));
    if (rc == YGZB_OK) rc = d2h(out->inlier, b.inlier + cap * j, cap);
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize");
    out->n_local = t->h_jobs[job].n_local;
    return rc;
}

}  // extern "C"
