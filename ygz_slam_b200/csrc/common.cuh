// common.cuh -- shared declarations of libygz_b200.so (context, slot storage, launch helpers).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <utility>
#include <vector>

#include "../../include/ygz_b200.h"

namespace ygzb {

constexpr int kMaxLevels = YGZB_MAX_LEVELS;

// FAST / cell-selection tile (level pixels).  80 x 40 is a whole number of 10-px grid cells on the
// three levels that can yield features (8x4, 16x8, 32x16 cells).
constexpr int kTileW = 80;
constexpr int kTileH = 40;

struct LevelGeom {
    int w, h, pitch;   // pitch in bytes, multiple of 16
    unsigned off;      // byte offset of the level inside a slot
};

struct Geometry {
    LevelGeom lv[kMaxLevels];
    int n_levels;
    int n_sel_levels;  // levels [0, n_sel_levels) can pass Frame::InFrame(px, 20, L); the others never yield features
    int W, H;          // full resolution (image.width / image.height)
    int cell_size, grid_cols, grid_rows, n_cells;
    int threshold;
    int tile_begin[kMaxLevels + 1];  // prefix sums of tiles per level
    int tiles_x[kMaxLevels];
    // exact division by small runtime constants without the ~20-instruction integer divide: n / d == (n * magic) >> 24
    // with magic = ceil(2^24 / d), valid while n * d < 2^24 (checked by build_geometry)
    unsigned tiles_x_magic[kMaxLevels];
    unsigned cell_magic;
    int cpt_x[kMaxLevels], cpt_y[kMaxLevels];  // grid cells per FAST tile row / column on the selectable levels
};

__host__ __device__ __forceinline__ unsigned div_magic(unsigned n, unsigned magic) {
    return (unsigned)(((unsigned long long)n * magic) >> 24);
}

}  // namespace ygzb

struct ygzb_ctx {
    int device;
    cudaStream_t stream;
    ygzb_params prm;
    ygzb::Geometry geo;
    size_t slot_stride;  // bytes per frame slot (pyramid), multiple of 256
    int sm_count;
    long long launches;
    char err[512];
    // growable device / pinned scratch owned by the context
    void* d_scratch[8];
    size_t d_scratch_bytes[8];
    void* h_scratch[4];
    size_t h_scratch_bytes[4];
    // optional per-stage CUDA-event timing (ygzb_profile_*): events bracket each kernel on ctx->stream
    int prof_on;
    void* prof;  // std::vector<ygzb::ProfRec>*
    cudaEvent_t timer[2];   // ygzb_timer_start / ygzb_timer_stop
    cudaEvent_t block_ev;   // ygzb_synchronize_blocking (created on first use)
};

struct ygzb_frames {
    ygzb_ctx* ctx;
    int capacity;
    uint8_t* d_pyr;       // capacity * slot_stride
    // device feature store, per slot, capacity n_cells features each (cell-index order)
    int32_t* d_count;     // [capacity]
    int16_t* d_fx;        // level coordinates
    int16_t* d_fy;
    uint8_t* d_flevel;
    float* d_fscore;
    float* d_fangle;
    int32_t* d_fcell;
    uint8_t* d_fdesc;     // [capacity][n_cells][32]
    // detect scratch (sized for `capacity` items)
    unsigned long long* d_best_key;   // [capacity][n_sel][n_cells]
    unsigned long long* d_first_key;  // [capacity][n_sel][n_cells]
    int32_t* d_stats;                 // [capacity][n_levels][2]
    int32_t* d_slots;                 // [capacity] slot list of the current call
    uint8_t* d_occupied;              // [capacity][n_cells]
    // TMA descriptors (CUtensorMap, 128 B each) of the first pyramid levels: 3-D tensors (x, y, slot) of u8 with a
    // 112 x 50 x 1 box = one FAST tile + halo; tma_levels == 0 disables the TMA path
    alignas(64) unsigned char tile_maps[3][128];
    void* d_tile_maps;                // device copy of tile_maps
    int tma_levels;
    int32_t* d_offsets;               // [capacity+1]
    int last_n;
    // lens undistortion (ygzb_frames_set_undistort): OpenCV fixed-point maps, [H][W] each, and the pool's own staging of the
    // raw frames a remap reads (uploads run on the context's stream and on a tracker's front stream: no shared scratch)
    bool undistort;                   // maps set: uploads remap level 0
    short2* d_map_xy;
    uint16_t* d_map_a;
    uint8_t* d_stage;
    size_t stage_bytes;
    cudaEvent_t e_stage;              // recorded behind the last remap, on whichever stream ran it: reuse of d_stage waits for it
};

namespace ygzb {

int set_error(ygzb_ctx* ctx, int code, const char* fmt, ...);
int check_cuda(ygzb_ctx* ctx, cudaError_t e, const char* what);
// offsets arrays of the batched entry points: off[0] == 0, non-decreasing, int-range total (returns YGZB_ERR_INVALID before
// anything is allocated or indexed)
inline int check_offsets(ygzb_ctx* ctx, const int32_t* off, int n, const char* what) {
    if (!off || n < 0) return set_error(ctx, YGZB_ERR_INVALID, "%s: null offsets", what);
    if (off[0] != 0) return set_error(ctx, YGZB_ERR_INVALID, "%s[0] must be 0", what);
    for (int i = 0; i < n; ++i)
        if (off[i + 1] < off[i]) return set_error(ctx, YGZB_ERR_INVALID, "%s must be non-decreasing (entry %d)", what, i + 1);
    return YGZB_OK;
}
// grow-only scratch buffers
void* dev_scratch(ygzb_ctx* ctx, int which, size_t bytes);
void* host_scratch(ygzb_ctx* ctx, int which, size_t bytes);

#define YGZB_CUDA(ctx, call)                                               \
    do {                                                                   \
        int _rc = ygzb::check_cuda((ctx), (call), #call);                  \
        if (_rc != YGZB_OK) return _rc;                                    \
    } while (0)

#define YGZB_LAUNCHED(ctx)                                                 \
    do {                                                                   \
        (ctx)->launches++;                                                 \
        int _rc = ygzb::check_cuda((ctx), cudaGetLastError(), "kernel launch"); \
        if (_rc != YGZB_OK) return _rc;                                    \
    } while (0)

#define TRY(x)                          \
    do {                                \
        int _rc = (x);                  \
        if (_rc != YGZB_OK) return _rc; \
    } while (0)

// typed copies on the context's stream (nothing is enqueued for a count of zero)
template <typename T>
int h2d(ygzb_ctx* ctx, T* dst, const T* src, size_t count) {
    if (!count) return YGZB_OK;
    return check_cuda(ctx, cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream), "H2D");
}
template <typename T>
int d2h(ygzb_ctx* ctx, T* dst, const T* src, size_t count) {
    if (!count) return YGZB_OK;
    return check_cuda(ctx, cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream), "D2H");
}

// ---- per-stage device timing -------------------------------------------------------------------
enum Stage {
    kStageBgr2Gray = 0, kStagePyrDown, kStageFastCells, kStageMergeCells, kStageDescribe, kStageMatch,
    kStageMatchFinalize, kStagePack, kStageOther, kStageAlign2D, kStageProjectAlign, kStageSparseAlign, kStagePoseOnly,
    kStageLocalBA, kStageKLT, kNumStages
};
struct ProfRec {
    cudaEvent_t a, b;
    int stage;
};
void prof_begin(ygzb_ctx* ctx, int stage);
void prof_end(ygzb_ctx* ctx);
struct ProfScope {
    ygzb_ctx* c;
    ProfScope(ygzb_ctx* ctx, int stage) : c(ctx) { if (c->prof_on) prof_begin(c, stage); }
    ~ProfScope() { if (c->prof_on) prof_end(c); }
};

// ---- stage launchers (one .cu each) -----------------------------------------------------------
// d_src = raw frames staged on the device (`channels` 1 or 3) or null (level 0 already in the slots); remap: level 0 =
// remap_gray_kernel of d_src through the pool's undistortion maps, otherwise d_src must be BGR (bgr2gray_kernel)
int launch_pyramid(ygzb_frames* f, int first, int count, const uint8_t* d_src, int channels, bool remap);
// ygzb_frames_upload; undistort = false skips the pool's undistortion maps (images that are undistorted already, e.g. the
// key-frame and reference images of the tracker's records)
int frames_upload(ygzb_frames* f, int first, int count, const uint8_t* host, int channels, size_t frame_stride, bool undistort);
int launch_pyrdown_ptrs(ygzb_ctx* ctx, const uint8_t* const* d_src_ptr, uint8_t* const* d_dst_ptr, int sw, int sh, int spitch,
                        int dw, int dh, int dpitch, int count);
int launch_detect(ygzb_frames* f, int n, bool have_occupied);
int build_tile_maps(ygzb_frames* f);
int launch_describe_store(ygzb_frames* f, int n);
int launch_describe_list(ygzb_frames* f, int n, const int32_t* d_slot_of, int total, const double* d_x, const double* d_y,
                         const uint8_t* d_level, float* d_angle, uint8_t* d_desc);
int launch_fast_debug(ygzb_frames* f, int slot, int level, uint8_t* d_score_map, uint8_t* d_nonmax_map);
int launch_offsets(ygzb_ctx* ctx, const int32_t* d_counts, const int32_t* d_sets, int n, int32_t* d_offsets);
int launch_match(ygzb_ctx* ctx, const uint8_t* d_base, size_t set_stride, const int32_t* d_counts, const int32_t* d_a_sets,
                 const int32_t* d_b_sets, int n_pairs, int cap, int cross_check, unsigned* d_fwd_key, unsigned* d_col_key,
                 const int32_t* d_q_offsets, int32_t* d_train_idx, int32_t* d_dist);
int launch_hamming_pairs(ygzb_ctx* ctx, const uint8_t* d_A, const uint8_t* d_B, const int32_t* d_ia, const int32_t* d_ib,
                         int n, int32_t* d_dist);
int launch_align2d(ygzb_frames* f, int n, const int32_t* d_slot, const uint8_t* d_level, const uint8_t* d_ref_border,
                   const uint8_t* d_ref, int n_iter, double* d_uv, uint8_t* d_ok);
int launch_align1d(ygzb_frames* f, int n, const int32_t* d_slot, const uint8_t* d_level, const float* d_dir, const uint8_t* d_ref_border,
                   const uint8_t* d_ref, int n_iter, double* d_uv, uint8_t* d_ok, double* d_hinv);
int launch_project_align(ygzb_frames* f, int n, const int32_t* d_ref_slot, const int32_t* d_cur_slot, const double* d_poses,
                         const int32_t* d_ref_pose, const int32_t* d_cur_pose, const double* d_ref_px, const double* d_ref_depth,
                         const uint8_t* d_ref_level, double* d_cur_px, uint8_t* d_search_level, uint8_t* d_ok);
int launch_sparse_align(ygzb_frames* f, int n_problems, const int32_t* d_ref_slot, const int32_t* d_cur_slot,
                        const int32_t* d_offsets, const double* d_px, const double* d_depth, const uint8_t* d_has_mp,
                        const double* d_T_ref, double* d_T_cur, int max_level, int min_level, int n_iter, double eps,
                        int32_t* d_n_meas, int32_t* d_iters, void* d_feat_scratch, size_t feat_stride);
// sparse_align2_kernel on kTrackCluster CTAs per problem (YGZB_TRACK_CLUSTER, as in the tracker).  d_feat_scratch holds feat_stride bytes per problem, at least
// sparse_align2_scratch_bytes(1, features of the largest problem): the global fall-back for CTAs whose share of the features
// does not fit shared memory.
size_t sparse_align2_scratch_bytes(int n_problems, int max_features);
constexpr int kTrackCluster = 4;   // CTAs per problem of the tracker's sparse alignment and pose-only (YGZB_TRACK_CLUSTER: 1, 2, 4 or 8)

// bump allocator over one scratch buffer (all sub-buffers 256-byte aligned)
struct Carver {
    uint8_t* base;
    size_t off = 0;
    explicit Carver(void* p) : base(static_cast<uint8_t*>(p)) {}
    template <typename T>
    T* take(size_t count) {
        off = (off + 255) & ~(size_t)255;
        T* r = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += count * sizeof(T);
        return r;
    }
    size_t bytes() const { return off + 256; }
};

// One scratch buffer, described once.  `layout(Carver&)` takes the sub-buffers in order and assigns the caller's pointers; it
// runs on a null Carver to size the buffer and again on the buffer dev_scratch returned for that size (a slot may move when it
// grows, so only the pointers of that second run are used).  `extra` bytes follow the layout; `sized` receives the layout's
// Carver::bytes().  Null if the allocation fails.
template <typename Layout>
void* carve_scratch(ygzb_ctx* ctx, int which, Layout&& layout, size_t extra = 0, size_t* sized = nullptr) {
    Carver sz(nullptr);
    layout(sz);
    if (sized) *sized = sz.bytes();
    void* buf = dev_scratch(ctx, which, sz.bytes() + extra);
    if (buf) {
        Carver c(buf);
        layout(c);
    }
    return buf;
}

// The inputs of an entry point are the first sub-buffers of its device buffer `buf`, contiguous up to in_bytes: they are
// assembled in pinned memory (host slot 1) with the same layout and travel as ONE host-to-device copy instead of one pageable
// copy each.  begin, put every input at its device address, commit.
struct StagedUpload {
    ygzb_ctx* ctx;
    void* buf;
    size_t in_bytes;
    uint8_t* stage;
    int begin(ygzb_ctx* ctx_, void* buf_, size_t in_bytes_) {
        ctx = ctx_; buf = buf_; in_bytes = in_bytes_;
        stage = static_cast<uint8_t*>(host_scratch(ctx, 1, in_bytes));
        if (!stage) return YGZB_ERR_CUDA;
        YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // an earlier copy may still read the staging buffer
        return YGZB_OK;
    }
    void put(const void* dev_ptr, const void* src, size_t bytes) const {
        if (bytes) memcpy(stage + (static_cast<const uint8_t*>(dev_ptr) - static_cast<uint8_t*>(buf)), src, bytes);
    }
    int commit() const {
        YGZB_CUDA(ctx, cudaMemcpyAsync(buf, stage, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
        return YGZB_OK;
    }
};

// `kernel` on n_ctas CTAs of `threads` threads, grouped into clusters of `cluster` CTAs (n_ctas is a multiple of it)
template <typename... Params, typename... Args>
cudaError_t launch_cluster(void (*kernel)(Params...), unsigned n_ctas, unsigned threads, int cluster, size_t smem_bytes, cudaStream_t stream,
                           Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_ctas);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// cluster-size tuning knobs (YGZB_BA_CLUSTER, YGZB_TRACK_CLUSTER): the variable's value if it is 1, 2, 4 or 8 -- or 16 where
// the kernel can run on the non-portable size --, `dflt` if it is unset or anything else
inline int cluster_knob(const char* name, int dflt, bool allow_16) {
    if (const char* e = getenv(name)) {
        const int v = atoi(e);
        if (v == 1 || v == 2 || v == 4 || v == 8 || (allow_16 && v == 16)) return v;
    }
    return dflt;
}

// device helpers shared by kernels ---------------------------------------------------------------
__device__ __forceinline__ unsigned float_orderable(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float orderable_float(unsigned o) {
    unsigned u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
    return __uint_as_float(u);
}

// c ? a : b on values, opaque to the compiler.  Written as `c ? v[i] : v[j]` on an array, the choice may be folded into a load
// from a selected ADDRESS; as a select of two registers pose_only_kernel spills 16 bytes less (sm_90a).
__device__ __forceinline__ double select_f64(bool c, double a, double b) {
    double r;
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\tselp.f64 %0, %2, %3, p;\n\t}" : "=d"(r) : "r"((unsigned)c), "d"(a), "d"(b));
    return r;
}

// Sums of N per-lane values over the warp, all at once (a "reduce-scatter" butterfly): at every step a lane keeps one half of
// its values and hands the other half to its partner, so N values cost N - 1 (+ log2(32 / N)) shuffles instead of 5 N.
// N = 32: lane l returns the total of v[l]; N = 16: lanes 2 i and 2 i + 1 return the total of v[i].  Only v[0, M) is read:
// v[M, N) count as zeros (padding that need not be kept in registers).  v is overwritten.
// Every loop has a trip count that is a compile-time constant before any loop is unrolled (the inner loop runs to N / 2 and
// skips i >= n): the compiler unrolls inner loops first and leaves `for (i < n)` inside `for (n = N / 2; n >= 1; n >>= 1)`
// rolled.  A rolled loop indexes v at run time, and v -- the caller's accumulators -- then lives in local memory, not registers.
template <int N, int M = N>
__device__ __forceinline__ double warp_reduce_scatter(double* v, int lane) {
    static_assert((N == 16 || N == 32) && 2 * M > N && M <= N, "warp_reduce_scatter: N = 16 or 32 values, at most N / 2 of them padding");
#pragma unroll
    for (int s = 0; s < 5; ++s) {
        const int n = (N >> 1) >> s, off = 16 >> s;
        if (n == 0) {
            v[0] += __shfl_xor_sync(0xFFFFFFFFu, v[0], off);
            continue;
        }
        const bool up = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
            if (i >= n) continue;
            const double hi = i + n < M ? v[i + n] : 0.0;
            const double keep = select_f64(up, hi, v[i]);
            const double send = select_f64(up, v[i], hi);
            v[i] = keep + __shfl_xor_sync(0xFFFFFFFFu, send, off);
        }
    }
    return v[0];
}

}  // namespace ygzb
