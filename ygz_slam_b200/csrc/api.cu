// api.cu -- extern "C" entry points of libygz_b200.so (include/ygz_b200.h): context, frame slots,
// host<->device marshalling around the stage launchers.  No computation happens on the host.
#include <stdarg.h>

#include <algorithm>
#include <cmath>
#include <new>

#include "common.cuh"

namespace ygzb {

int set_error(ygzb_ctx* ctx, int code, const char* fmt, ...) {
    if (ctx) {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
        va_end(ap);
    }
    return code;
}

int check_cuda(ygzb_ctx* ctx, cudaError_t e, const char* what) {
    if (e == cudaSuccess) return YGZB_OK;
    return set_error(ctx, YGZB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

void* dev_scratch(ygzb_ctx* ctx, int which, size_t bytes) {
    if (ctx->d_scratch_bytes[which] >= bytes && ctx->d_scratch[which]) return ctx->d_scratch[which];
    if (ctx->d_scratch[which]) {
        cudaStreamSynchronize(ctx->stream);
        cudaFree(ctx->d_scratch[which]);
        ctx->d_scratch[which] = nullptr;
        ctx->d_scratch_bytes[which] = 0;
    }
    const size_t want = std::max(bytes + bytes / 4, (size_t)4096);
    void* p = nullptr;
    if (check_cuda(ctx, cudaMalloc(&p, want), "cudaMalloc(scratch)") != YGZB_OK) return nullptr;
    ctx->d_scratch[which] = p;
    ctx->d_scratch_bytes[which] = want;
    return p;
}

void* host_scratch(ygzb_ctx* ctx, int which, size_t bytes) {
    if (ctx->h_scratch_bytes[which] >= bytes && ctx->h_scratch[which]) return ctx->h_scratch[which];
    if (ctx->h_scratch[which]) {
        cudaStreamSynchronize(ctx->stream);
        cudaFreeHost(ctx->h_scratch[which]);
        ctx->h_scratch[which] = nullptr;
        ctx->h_scratch_bytes[which] = 0;
    }
    const size_t want = std::max(bytes + bytes / 4, (size_t)4096);
    void* p = nullptr;
    if (check_cuda(ctx, cudaMallocHost(&p, want), "cudaMallocHost(scratch)") != YGZB_OK) return nullptr;
    ctx->h_scratch[which] = p;
    ctx->h_scratch_bytes[which] = want;
    return p;
}

void prof_begin(ygzb_ctx* ctx, int stage) {
    auto* v = static_cast<std::vector<ProfRec>*>(ctx->prof);
    if (!v) ctx->prof = v = new std::vector<ProfRec>();
    ProfRec r;
    r.stage = stage;
    cudaEventCreate(&r.a);
    cudaEventCreate(&r.b);
    cudaEventRecord(r.a, ctx->stream);
    v->push_back(r);
}

void prof_end(ygzb_ctx* ctx) {
    auto* v = static_cast<std::vector<ProfRec>*>(ctx->prof);
    if (v && !v->empty()) cudaEventRecord(v->back().b, ctx->stream);
}

namespace {

// gather the per-slot feature store of the n items of a call into packed SoA arrays
__global__ void pack_features_kernel(const int32_t* __restrict__ slots, const int32_t* __restrict__ offsets, int n_cells,
                                     const int32_t* __restrict__ count, const int16_t* __restrict__ fx,
                                     const int16_t* __restrict__ fy, const uint8_t* __restrict__ flevel,
                                     const float* __restrict__ fscore, const float* __restrict__ fangle,
                                     const int32_t* __restrict__ fcell, const uint8_t* __restrict__ fdesc, float* ox,
                                     float* oy, uint8_t* olevel, float* oscore, float* oangle, int32_t* ocell,
                                     uint8_t* odesc) {
    const int item = blockIdx.y, slot = slots[item];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count[slot]) return;
    const size_t s = (size_t)slot * n_cells + i, d = (size_t)offsets[item] + i;
    const int L = flevel[s];
    ox[d] = (float)((int)fx[s] << L);  // Feature::_pixel = level coordinate * 2^level (FeatureDetector.cpp:415-424)
    oy[d] = (float)((int)fy[s] << L);
    olevel[d] = (uint8_t)L;
    oscore[d] = fscore[s];
    oangle[d] = fangle[s];
    ocell[d] = fcell[s];
    const uint4* src = reinterpret_cast<const uint4*>(fdesc) + s * 2;
    uint4* dst = reinterpret_cast<uint4*>(odesc) + d * 2;
    dst[0] = src[0];
    dst[1] = src[1];
}

__global__ void expand_slots_kernel(const int32_t* __restrict__ slots, const int32_t* __restrict__ offsets, int n,
                                    int32_t* __restrict__ slot_of) {
    const int item = blockIdx.y;
    const int i = offsets[item] + blockIdx.x * blockDim.x + threadIdx.x;
    if (i < offsets[item + 1]) slot_of[i] = slots[item];
}

int build_geometry(ygzb_ctx* ctx) {
    const ygzb_params& p = ctx->prm;
    Geometry& g = ctx->geo;
    memset(&g, 0, sizeof(g));
    if (p.n_levels < 1 || p.n_levels > kMaxLevels) return set_error(ctx, YGZB_ERR_INVALID, "n_levels out of range");
    if (p.image_width < 16 || p.image_height < 16 || p.image_width > 8192 || p.image_height > 8192)
        return set_error(ctx, YGZB_ERR_INVALID, "unsupported image size");
    if (p.cell_size < 1) return set_error(ctx, YGZB_ERR_INVALID, "cell_size must be positive");
    // the FAST kernel keeps scores in u8 with 0 = "not a corner" and builds SWAR constants from 127 - threshold
    if (p.fast_threshold < 1 || p.fast_threshold > 254) return set_error(ctx, YGZB_ERR_INVALID, "fast_threshold must be in [1, 254]");
    g.n_levels = p.n_levels;
    g.W = p.image_width;
    g.H = p.image_height;
    g.cell_size = p.cell_size;
    g.grid_cols = (p.image_width + p.cell_size - 1) / p.cell_size;   // ceil(double(w)/cell) FeatureDetector.cpp:336-337
    g.grid_rows = (p.image_height + p.cell_size - 1) / p.cell_size;
    g.n_cells = g.grid_cols * g.grid_rows;
    g.threshold = p.fast_threshold;
    int w = p.image_width, h = p.image_height;
    size_t off = 0;
    g.tile_begin[0] = 0;
    for (int L = 0; L < p.n_levels; ++L) {
        g.lv[L].w = w;
        g.lv[L].h = h;
        g.lv[L].pitch = (w + 15) & ~15;
        g.lv[L].off = (unsigned)off;
        off += (size_t)g.lv[L].pitch * h;
        off = (off + 255) & ~(size_t)255;
        g.tiles_x[L] = (w + kTileW - 1) / kTileW;
        g.tile_begin[L + 1] = g.tile_begin[L] + g.tiles_x[L] * ((h + kTileH - 1) / kTileH);
        w = (w + 1) / 2;
        h = (h + 1) / 2;
    }
    ctx->slot_stride = off;
    // levels whose corners can pass Frame::InFrame(px, 20, L): need a FAST pixel x in [3, w_L-3) with
    // x >= 20 * 2^L (and the same vertically)
    g.n_sel_levels = 0;
    for (int L = 0; L < p.n_levels; ++L) {
        const bool can = (20 << L) < g.lv[L].w - 3 && (20 << L) < g.lv[L].h - 3;
        if (!can) break;
        g.n_sel_levels = L + 1;
    }
    for (int L = 0; L < g.n_sel_levels; ++L) {
        const int sx = kTileW << L, sy = kTileH << L;
        if (sx % p.cell_size || sy % p.cell_size || (sx / p.cell_size) * (sy / p.cell_size) > 512)
            return set_error(ctx, YGZB_ERR_INVALID,
                             "cell_size %d does not tile the %dx%d FAST tile at level %d (supported: divisors of 40 such as 5, 8, 10, 20)",
                             p.cell_size, kTileW, kTileH, L);
    }
    if (g.n_cells > 8 * 1024) return set_error(ctx, YGZB_ERR_INVALID, "grid has too many cells");
    // magic multipliers for the divisions of the FAST kernel (see common.cuh)
    g.cell_magic = (unsigned)(((1ull << 24) + p.cell_size - 1) / p.cell_size);
    for (int L = 0; L < p.n_levels; ++L) {
        g.tiles_x_magic[L] = (unsigned)(((1ull << 24) + g.tiles_x[L] - 1) / g.tiles_x[L]);
        const long long n_tiles = g.tile_begin[L + 1] - g.tile_begin[L];
        if (n_tiles * g.tiles_x[L] >= (1ll << 24)) return set_error(ctx, YGZB_ERR_INVALID, "image too large for the tile index arithmetic");
        if (L < g.n_sel_levels) {
            g.cpt_x[L] = (kTileW << L) / p.cell_size;
            g.cpt_y[L] = (kTileH << L) / p.cell_size;
            if ((long long)(kTileW << L) * p.cell_size >= (1ll << 24)) return set_error(ctx, YGZB_ERR_INVALID, "cell arithmetic out of range");
        }
    }
    return YGZB_OK;
}

template <typename T>
int dalloc(ygzb_ctx* ctx, T** p, size_t count) {
    return check_cuda(ctx, cudaMalloc((void**)p, std::max(count, (size_t)1) * sizeof(T)), "cudaMalloc");
}

}  // namespace
}  // namespace ygzb

using namespace ygzb;

extern "C" {

void ygzb_default_params(ygzb_params* p) {
    p->image_width = 640;
    p->image_height = 480;
    p->n_levels = 3;
    p->cell_size = 10;
    p->fast_threshold = 15;
    p->fx = 520.9f;
    p->fy = 521.0f;
    p->cx = 325.1f;
    p->cy = 249.7f;
}

int ygzb_create(int device, const ygzb_params* p, ygzb_ctx** out) {
    if (!p || !out) return YGZB_ERR_INVALID;
    *out = nullptr;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0 || device < 0 || device >= n_dev) return YGZB_ERR_NO_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return YGZB_ERR_NO_DEVICE;
    if (prop.major != 9 || prop.minor != 0) return YGZB_ERR_NO_DEVICE;  // the kernels are built for sm_90a only
    ygzb_ctx* ctx = new (std::nothrow) ygzb_ctx();
    if (!ctx) return YGZB_ERR_INVALID;
    memset(ctx, 0, sizeof(*ctx));
    ctx->device = device;
    ctx->prm = *p;
    ctx->sm_count = prop.multiProcessorCount;
    if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete ctx;
        return YGZB_ERR_CUDA;
    }
    const int rc = build_geometry(ctx);
    if (rc != YGZB_OK) {
        // keep the message reachable: hand the context back so ygzb_last_error works, caller destroys it
        *out = ctx;
        return rc;
    }
    *out = ctx;
    return YGZB_OK;
}

void ygzb_destroy(ygzb_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (int i = 0; i < 8; ++i)
        if (ctx->d_scratch[i]) cudaFree(ctx->d_scratch[i]);
    for (int i = 0; i < 4; ++i)
        if (ctx->h_scratch[i]) cudaFreeHost(ctx->h_scratch[i]);
    if (ctx->prof) {
        auto* v = static_cast<std::vector<ProfRec>*>(ctx->prof);
        for (ProfRec& r : *v) {
            cudaEventDestroy(r.a);
            cudaEventDestroy(r.b);
        }
        delete v;
    }
    for (cudaEvent_t e : ctx->timer)
        if (e) cudaEventDestroy(e);
    if (ctx->block_ev) cudaEventDestroy(ctx->block_ev);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* ygzb_last_error(const ygzb_ctx* ctx) { return ctx ? ctx->err : "null context"; }

int ygzb_synchronize(ygzb_ctx* ctx) {
    if (!ctx) return YGZB_ERR_INVALID;
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

// waits on a cudaEventBlockingSync event recorded behind everything enqueued so far: the calling thread sleeps instead of
// spinning (cudaStreamSynchronize spins under the default scheduling flags) -- for hosts with fewer CPUs than waiting threads
int ygzb_synchronize_blocking(ygzb_ctx* ctx) {
    if (!ctx) return YGZB_ERR_INVALID;
    cudaSetDevice(ctx->device);
    if (!ctx->block_ev) YGZB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->block_ev, cudaEventBlockingSync | cudaEventDisableTiming));
    YGZB_CUDA(ctx, cudaEventRecord(ctx->block_ev, ctx->stream));
    YGZB_CUDA(ctx, cudaEventSynchronize(ctx->block_ev));
    return YGZB_OK;
}

int ygzb_profile_enable(ygzb_ctx* ctx, int on) {
    if (!ctx) return YGZB_ERR_INVALID;
    ctx->prof_on = on ? 1 : 0;
    return YGZB_OK;
}

int ygzb_profile_read(ygzb_ctx* ctx, double* ms, int32_t* launches) {
    if (!ctx || !ms || !launches) return YGZB_ERR_INVALID;
    cudaSetDevice(ctx->device);
    for (int i = 0; i < kNumStages; ++i) {
        ms[i] = 0.0;
        launches[i] = 0;
    }
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    auto* v = static_cast<std::vector<ProfRec>*>(ctx->prof);
    if (!v) return YGZB_OK;
    for (ProfRec& r : *v) {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) {
            ms[r.stage] += t;
            launches[r.stage] += 1;
        }
        cudaEventDestroy(r.a);
        cudaEventDestroy(r.b);
    }
    v->clear();
    return YGZB_OK;
}

int ygzb_profile_stage_count(void) { return kNumStages; }
const char* ygzb_profile_stage_name(int i) {
    static const char* names[kNumStages] = {"bgr2gray", "pyrdown", "fast_cells", "merge_cells", "describe", "match",
                                            "match_finalize", "pack", "other", "align2d", "project_align", "sparse_align",
                                            "pose_only", "local_ba", "klt"};
    return (i >= 0 && i < kNumStages) ? names[i] : "";
}

void* ygzb_stream(ygzb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

int ygzb_timer_start(ygzb_ctx* ctx) {
    if (!ctx) return YGZB_ERR_INVALID;
    cudaSetDevice(ctx->device);
    if (!ctx->timer[0]) {
        YGZB_CUDA(ctx, cudaEventCreate(&ctx->timer[0]));
        YGZB_CUDA(ctx, cudaEventCreate(&ctx->timer[1]));
    }
    YGZB_CUDA(ctx, cudaEventRecord(ctx->timer[0], ctx->stream));
    return YGZB_OK;
}

int ygzb_timer_stop(ygzb_ctx* ctx, double* ms) {
    if (!ctx || !ms || !ctx->timer[0]) return YGZB_ERR_INVALID;
    cudaSetDevice(ctx->device);
    YGZB_CUDA(ctx, cudaEventRecord(ctx->timer[1], ctx->stream));
    YGZB_CUDA(ctx, cudaEventSynchronize(ctx->timer[1]));
    float t = 0.f;
    YGZB_CUDA(ctx, cudaEventElapsedTime(&t, ctx->timer[0], ctx->timer[1]));
    *ms = t;
    return YGZB_OK;
}
long long ygzb_launch_count(const ygzb_ctx* ctx) { return ctx ? ctx->launches : 0; }

int ygzb_host_alloc(void** ptr, size_t bytes) {
    return cudaMallocHost(ptr, bytes) == cudaSuccess ? YGZB_OK : YGZB_ERR_CUDA;
}
int ygzb_host_free(void* ptr) { return cudaFreeHost(ptr) == cudaSuccess ? YGZB_OK : YGZB_ERR_CUDA; }

int ygzb_get_params(const ygzb_ctx* ctx, ygzb_params* out) {
    if (!ctx || !out) return YGZB_ERR_INVALID;
    *out = ctx->prm;
    return YGZB_OK;
}

int ygzb_grid_dims(const ygzb_ctx* ctx, int* rows, int* cols) {
    if (!ctx) return YGZB_ERR_INVALID;
    if (rows) *rows = ctx->geo.grid_rows;
    if (cols) *cols = ctx->geo.grid_cols;
    return YGZB_OK;
}

// ---- frames -------------------------------------------------------------------------------------
int ygzb_frames_create(ygzb_ctx* ctx, int capacity, ygzb_frames** out) {
    if (!ctx || !out || capacity < 1) return YGZB_ERR_INVALID;
    *out = nullptr;
    cudaSetDevice(ctx->device);
    ygzb_frames* f = new (std::nothrow) ygzb_frames();
    if (!f) return YGZB_ERR_INVALID;
    memset(f, 0, sizeof(*f));
    f->ctx = ctx;
    f->capacity = capacity;
    const Geometry& g = ctx->geo;
    const size_t cap = (size_t)capacity, nc = (size_t)g.n_cells;
    int rc = YGZB_OK;
    auto A = [&](int r) { if (rc == YGZB_OK) rc = r; };
    A(dalloc(ctx, &f->d_pyr, cap * ctx->slot_stride));
    A(dalloc(ctx, &f->d_count, cap));
    A(dalloc(ctx, &f->d_fx, cap * nc));
    A(dalloc(ctx, &f->d_fy, cap * nc));
    A(dalloc(ctx, &f->d_flevel, cap * nc));
    A(dalloc(ctx, &f->d_fscore, cap * nc));
    A(dalloc(ctx, &f->d_fangle, cap * nc));
    A(dalloc(ctx, &f->d_fcell, cap * nc));
    A(dalloc(ctx, &f->d_fdesc, cap * nc * 32));
    A(dalloc(ctx, &f->d_best_key, cap * std::max(g.n_sel_levels, 1) * nc));
    A(dalloc(ctx, &f->d_first_key, cap * std::max(g.n_sel_levels, 1) * nc));
    A(dalloc(ctx, &f->d_stats, cap * g.n_levels * 2));
    A(dalloc(ctx, &f->d_slots, cap));
    A(dalloc(ctx, &f->d_occupied, cap * nc));
    A(dalloc(ctx, &f->d_offsets, cap + 1));
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMemsetAsync(f->d_count, 0, cap * sizeof(int32_t), ctx->stream), "memset");
    if (rc == YGZB_OK) rc = check_cuda(ctx, cudaMemsetAsync(f->d_pyr, 0, cap * ctx->slot_stride, ctx->stream), "memset");
    if (rc == YGZB_OK) rc = build_tile_maps(f);
    if (rc != YGZB_OK) {
        ygzb_frames_destroy(f);
        return rc;
    }
    *out = f;
    return YGZB_OK;
}

void ygzb_frames_destroy(ygzb_frames* f) {
    if (!f) return;
    cudaSetDevice(f->ctx->device);
    cudaStreamSynchronize(f->ctx->stream);
    void* ptrs[] = {f->d_pyr,   f->d_count,    f->d_fx,        f->d_fy,    f->d_flevel, f->d_fscore,   f->d_fangle, f->d_fcell,
                    f->d_fdesc, f->d_best_key, f->d_first_key, f->d_stats, f->d_slots,  f->d_occupied, f->d_offsets};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    if (f->d_tile_maps) cudaFree(f->d_tile_maps);
    if (f->e_stage) {
        cudaEventSynchronize(f->e_stage);
        cudaEventDestroy(f->e_stage);
    }
    for (void* p : {(void*)f->d_map_xy, (void*)f->d_map_a, (void*)f->d_stage})
        if (p) cudaFree(p);
    delete f;
}

int ygzb_frames_layout(const ygzb_frames* f, int* lw, int* lh, int* lpitch, size_t* loff, size_t* slot_stride) {
    if (!f) return YGZB_ERR_INVALID;
    const Geometry& g = f->ctx->geo;
    for (int L = 0; L < g.n_levels; ++L) {
        if (lw) lw[L] = g.lv[L].w;
        if (lh) lh[L] = g.lv[L].h;
        if (lpitch) lpitch[L] = g.lv[L].pitch;
        if (loff) loff[L] = g.lv[L].off;
    }
    if (slot_stride) *slot_stride = f->ctx->slot_stride;
    return YGZB_OK;
}

void* ygzb_frames_device_ptr(ygzb_frames* f) { return f ? f->d_pyr : nullptr; }

int ygzb_frames_build_pyramid(ygzb_frames* f, int first, int count) {
    if (!f || first < 0 || count < 0 || first + count > f->capacity) return YGZB_ERR_INVALID;
    cudaSetDevice(f->ctx->device);
    const RawFormat l0{f->ctx->geo.lv[0].w, f->ctx->geo.lv[0].h, 1};
    return launch_pyramid(f, first, count, nullptr, l0, nullptr, nullptr);
}

int ygzb_frames_copy(ygzb_frames* f, int src_slot, int dst_slot) {
    if (!f || src_slot < 0 || dst_slot < 0 || src_slot >= f->capacity || dst_slot >= f->capacity) return YGZB_ERR_INVALID;
    if (src_slot == dst_slot) return YGZB_OK;
    ygzb_ctx* ctx = f->ctx;
    cudaSetDevice(ctx->device);
    YGZB_CUDA(ctx, cudaMemcpyAsync(f->d_pyr + (size_t)dst_slot * ctx->slot_stride, f->d_pyr + (size_t)src_slot * ctx->slot_stride,
                                   ctx->slot_stride, cudaMemcpyDeviceToDevice, ctx->stream));
    return YGZB_OK;
}

}  // extern "C"

namespace {

// host or device memory -> device staging of `count` raw frames, packed (one frame after the other)
int stage_frames(ygzb_ctx* ctx, uint8_t* dst, const uint8_t* src, int count, size_t frame_bytes, size_t frame_stride) {
    // cudaMemcpyDefault: `src` may also be a device pointer (frames already resident in HBM, unified addressing).
    // A strided batch copy treats one image as a "row", so its pitch is limited (cudaDeviceProp::memPitch, 2^31 - 1):
    // longer strides (a stacked [stream][frame] array of thousands of frames) fall back to one copy per image.
    if (frame_stride <= (size_t)0x7FFFFFFF) {
        YGZB_CUDA(ctx, cudaMemcpy2DAsync(dst, frame_bytes, src, frame_stride, frame_bytes, count, cudaMemcpyDefault, ctx->stream));
    } else {
        for (int i = 0; i < count; ++i)
            YGZB_CUDA(ctx, cudaMemcpyAsync(dst + (size_t)i * frame_bytes, src + (size_t)i * frame_stride, frame_bytes, cudaMemcpyDefault,
                                           ctx->stream));
    }
    return YGZB_OK;
}

// staged upload: the raw frames go to the pool's staging buffer, and remap_gray_kernel (through the maps: the pool's, or a
// tracker stream's, ygzb_tracker_set_undistort) or bgr2gray_kernel writes level 0.  The buffer is the pool's own, not a
// context scratch buffer, because a tracker uploads on its front stream while the context's stream runs a local BA; e_stage,
// recorded behind every kernel that reads the buffer on whichever stream ran it, orders each reuse of the buffer (a copy
// into it, or its reallocation) behind the last read of it, so a frame in flight is never overwritten.
int upload_staged(ygzb_frames* f, int first, int count, const uint8_t* src, RawFormat fmt, size_t frame_stride, const short2* map_xy,
                  const uint16_t* map_a) {
    ygzb_ctx* ctx = f->ctx;
    const size_t frame = fmt.bytes(), bytes = frame * count;
    if (!f->e_stage) YGZB_CUDA(ctx, cudaEventCreateWithFlags(&f->e_stage, cudaEventDisableTiming));
    if (f->stage_bytes < bytes) {
        YGZB_CUDA(ctx, cudaEventSynchronize(f->e_stage));
        if (f->d_stage) cudaFree(f->d_stage);
        f->d_stage = nullptr;
        f->stage_bytes = 0;
        YGZB_CUDA(ctx, cudaMalloc((void**)&f->d_stage, bytes));
        f->stage_bytes = bytes;
    }
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, f->e_stage, 0));
    int rc = stage_frames(ctx, f->d_stage, src, count, frame, frame_stride);
    if (rc == YGZB_OK) rc = launch_pyramid(f, first, count, f->d_stage, fmt, map_xy, map_a);
    // recorded even after a failed launch: a copy into the buffer may be in flight
    const int rc_ev = check_cuda(ctx, cudaEventRecord(f->e_stage, ctx->stream), "cudaEventRecord");
    return rc != YGZB_OK ? rc : rc_ev;
}

}  // namespace

int ygzb::frames_upload(ygzb_frames* f, int first, int count, const uint8_t* host, RawFormat src, size_t frame_stride, const short2* map_xy,
                        const uint16_t* map_a) {
    if (!f || !host || first < 0 || count < 0 || first + count > f->capacity) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    const Geometry& g = ctx->geo;
    cudaSetDevice(ctx->device);
    if (src.channels != 1 && src.channels != 3) return set_error(ctx, YGZB_ERR_INVALID, "channels must be 1 or 3");
    if (src.w < 1 || src.h < 1) return set_error(ctx, YGZB_ERR_INVALID, "raw frame size %d x %d", src.w, src.h);
    if ((src.w != g.lv[0].w || src.h != g.lv[0].h) && !map_xy)
        return set_error(ctx, YGZB_ERR_INVALID, "a raw frame of %d x %d needs undistortion maps to become level 0 (%d x %d)", src.w, src.h,
                         g.lv[0].w, g.lv[0].h);
    if (frame_stride < src.bytes()) return set_error(ctx, YGZB_ERR_INVALID, "frame_stride smaller than one image");
    if (count == 0) return YGZB_OK;
    if (map_xy || src.channels == 3) return upload_staged(f, first, count, host, src, frame_stride, map_xy, map_a);
    // a grey frame of level 0's size, straight into the slots.
    // cudaMemcpyDefault: `host` may also be a device pointer (frames already resident in HBM, unified addressing).
    // A strided batch copy treats one image as a "row", so its pitch is limited (cudaDeviceProp::memPitch, 2^31 - 1):
    // longer strides (a stacked [stream][frame] array of thousands of frames) fall back to one copy per image.
    const size_t row = (size_t)g.lv[0].w;
    uint8_t* dst = f->d_pyr + (size_t)first * ctx->slot_stride + g.lv[0].off;
    if (g.lv[0].pitch == g.lv[0].w && frame_stride <= (size_t)0x7FFFFFFF) {
        // level 0 of a slot is one contiguous run: a single strided copy moves the whole batch
        YGZB_CUDA(ctx, cudaMemcpy2DAsync(dst, ctx->slot_stride, host, frame_stride, row * g.lv[0].h, count, cudaMemcpyDefault,
                                         ctx->stream));
    } else {
        for (int i = 0; i < count; ++i)
            YGZB_CUDA(ctx, cudaMemcpy2DAsync(dst + (size_t)i * ctx->slot_stride, g.lv[0].pitch, host + (size_t)i * frame_stride,
                                             row, row, g.lv[0].h, cudaMemcpyDefault, ctx->stream));
    }
    return launch_pyramid(f, first, count, nullptr, src, nullptr, nullptr);
}

extern "C" {

int ygzb_frames_upload(ygzb_frames* f, int first, int count, const uint8_t* host, int channels, size_t frame_stride) {
    if (!f) return YGZB_ERR_INVALID;
    const RawFormat src{f->ctx->geo.lv[0].w, f->ctx->geo.lv[0].h, channels};
    return frames_upload(f, first, count, host, src, frame_stride, f->undistort ? f->d_map_xy : nullptr, f->d_map_a);
}

int ygzb_frames_set_undistort(ygzb_frames* f, const int16_t* map_xy, const uint16_t* map_a) {
    if (!f) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    if (!map_xy != !map_a) return set_error(ctx, YGZB_ERR_INVALID, "set_undistort: map_xy and map_a must both be given, or both be NULL");
    cudaSetDevice(ctx->device);
    if (!map_xy) {   // uploads in flight keep reading the maps, which stay allocated until the pool is destroyed
        f->undistort = false;
        return YGZB_OK;
    }
    // the maps are read into host memory and checked before anything of the pool changes
    const size_t n = (size_t)ctx->geo.W * ctx->geo.H;
    std::vector<int16_t> xy(2 * n);
    std::vector<uint16_t> a(n);
    YGZB_CUDA(ctx, cudaMemcpy(xy.data(), map_xy, 2 * n * sizeof(int16_t), cudaMemcpyDefault));
    YGZB_CUDA(ctx, cudaMemcpy(a.data(), map_a, n * sizeof(uint16_t), cudaMemcpyDefault));
    for (size_t i = 0; i < n; ++i)
        if (a[i] >= 1024)
            return set_error(ctx, YGZB_ERR_INVALID, "set_undistort: map_a[%zu] = %d is not a 5 + 5-bit fraction (< 1024)", i, (int)a[i]);
    if (!f->e_stage) YGZB_CUDA(ctx, cudaEventCreateWithFlags(&f->e_stage, cudaEventDisableTiming));
    if (!f->d_map_xy) YGZB_CUDA(ctx, cudaMalloc((void**)&f->d_map_xy, n * sizeof(short2)));
    if (!f->d_map_a) YGZB_CUDA(ctx, cudaMalloc((void**)&f->d_map_a, n * sizeof(uint16_t)));
    // behind the last remap (which may still read the old maps, on a tracker's front stream), and complete on return
    YGZB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, f->e_stage, 0));
    YGZB_CUDA(ctx, cudaMemcpyAsync(f->d_map_xy, xy.data(), 2 * n * sizeof(int16_t), cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(f->d_map_a, a.data(), n * sizeof(uint16_t), cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    f->undistort = true;
    return YGZB_OK;
}

// cv::initUndistortRectifyMap(K, D, R = I, newK, size, CV_16SC2) (OpenCV modules/calib3d, undistort), restated as OpenCV's
// x86-64 build computes it (its AVX2 + FMA code path, 8 columns per step): the inverse of newK by the cofactor formula of
// cv::invert for 3x3; per row the ray start _y = fma(i, iR11, iR12); per column _x = start of its group of 8 (advanced by
// 8 iR00 per group) + k iR00, the columns after the last full group advanced by iR00 one by one; then the radial-tangential
// model with its multiply-adds fused as OpenCV's vector code fuses them, projection with K, rounding to 1/32 pixel (cvRound:
// half to even) and the split into the integer pixel and the 5 + 5-bit fraction.  Every other step is one IEEE double
// operation (the host build does not contract them).  The fusing matters at exact ties only: on the TUM and EuRoC cameras the
// plain sums give the same maps.
int ygzb_undistort_map(int width, int height, const double K[4], const double dist[5], const double newK[4], int16_t* map_xy,
                       uint16_t* map_a) {
    if (width < 1 || height < 1 || width > 32767 || height > 32767 || !K || !dist || !map_xy || !map_a) return YGZB_ERR_INVALID;
    const double* A = newK ? newK : K;
    const double afx = A[0], afy = A[1], acx = A[2], acy = A[3];
    if (!(afx * afy != 0.0)) return YGZB_ERR_INVALID;
    // iR = newK^-1 (cv::invert, DECOMP_LU, 3x3: d = 1 / det3, cofactors times d), the zero entries dropped
    const double d = 1.0 / (afx * afy);
    const double ir0 = afy * d, ir2 = -(acx * afy) * d, ir4 = afx * d, ir5 = -(afx * acy) * d, ir8 = (afx * afy) * d;
    const double fx = K[0], fy = K[1], u0 = K[2], v0 = K[3];
    const double k1 = dist[0], k2 = dist[1], p1 = dist[2], p2 = dist[3], k3 = dist[4];
    const double w = 1.0 / ir8;
    std::vector<double> xs(width);
    {
        double base = ir2;
        const int full = width / 8 * 8;
        for (int j = 0; j < full; j += 8, base += 8 * ir0)
            for (int k = 0; k < 8; ++k) xs[j + k] = base + k * ir0;
        for (int j = full; j < width; ++j, base += ir0) xs[j] = base;
    }
    for (int i = 0; i < height; ++i) {
        const double y = std::fma((double)i, ir4, ir5) * w;
        for (int j = 0; j < width; ++j) {
            const double x = xs[j] * w;
            const double x2 = x * x, y2 = y * y;
            const double r2 = x2 + y2, _2xy = 2 * x * y;
            const double kr = std::fma(std::fma(std::fma(k3, r2, k2), r2, k1), r2, 1.0);
            const double xd = std::fma(p2, r2 + 2 * x2, std::fma(p1, _2xy, x * kr));
            const double yd = std::fma(p2, _2xy, std::fma(p1, r2 + 2 * y2, y * kr));
            const double u = std::fma(fx, xd, u0), v = std::fma(fy, yd, v0);
            const double su = u * 32.0, sv = v * 32.0;
            // saturate_cast<int>: round half to even, clamped to the int range (NaN: INT_MIN, as x86's cvtsd2si gives it)
            const int iu = su >= 2147483647.0 ? INT32_MAX : (su <= -2147483648.0 || su != su) ? INT32_MIN : (int)std::nearbyint(su);
            const int iv = sv >= 2147483647.0 ? INT32_MAX : (sv <= -2147483648.0 || sv != sv) ? INT32_MIN : (int)std::nearbyint(sv);
            const size_t o = (size_t)i * width + j;
            // saturate_cast<short> of the integer pixel: a ray that leaves the image far away must not wrap back into it
            map_xy[2 * o] = (int16_t)std::min(std::max(iu >> 5, -32768), 32767);
            map_xy[2 * o + 1] = (int16_t)std::min(std::max(iv >> 5, -32768), 32767);
            map_a[o] = (uint16_t)((iv & 31) * 32 + (iu & 31));
        }
    }
    return YGZB_OK;
}

int ygzb_frames_download_level(ygzb_frames* f, int slot, int level, uint8_t* host) {
    if (!f || !host || slot < 0 || slot >= f->capacity || level < 0 || level >= f->ctx->geo.n_levels) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    const LevelGeom& lv = ctx->geo.lv[level];
    cudaSetDevice(ctx->device);
    YGZB_CUDA(ctx, cudaMemcpy2DAsync(host, lv.w, f->d_pyr + (size_t)slot * ctx->slot_stride + lv.off, lv.pitch, lv.w, lv.h,
                                     cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

// ---- FeatureDetector ------------------------------------------------------------------------------
static int upload_slots(ygzb_frames* f, const int32_t* slots, int n) {
    ygzb_ctx* ctx = f->ctx;
    if (!slots || n < 1 || n > f->capacity) return set_error(ctx, YGZB_ERR_INVALID, "bad slot list (n=%d, capacity=%d)", n, f->capacity);
    for (int i = 0; i < n; ++i)
        if (slots[i] < 0 || slots[i] >= f->capacity) return set_error(ctx, YGZB_ERR_INVALID, "slot %d out of range", slots[i]);
    // staged through pinned memory so the async copy does not read a caller buffer that may go away
    int32_t* h = (int32_t*)host_scratch(ctx, 0, (size_t)f->capacity * sizeof(int32_t));
    if (!h) return YGZB_ERR_CUDA;
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(h, slots, (size_t)n * sizeof(int32_t));
    YGZB_CUDA(ctx, cudaMemcpyAsync(f->d_slots, h, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    return YGZB_OK;
}

int ygzb_detect(ygzb_frames* f, const int32_t* slots, int n, const uint8_t* occupied, ygzb_keypoints* out) {
    if (!f) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    const Geometry& g = ctx->geo;
    cudaSetDevice(ctx->device);
    int rc = upload_slots(f, slots, n);
    if (rc != YGZB_OK) return rc;
    if (occupied)
        YGZB_CUDA(ctx, cudaMemcpyAsync(f->d_occupied, occupied, (size_t)n * g.n_cells, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = launch_detect(f, n, occupied != nullptr)) != YGZB_OK) return rc;
    if ((rc = launch_describe_store(f, n)) != YGZB_OK) return rc;
    f->last_n = n;
    if (!out) return YGZB_OK;

    // packed copy-back: offsets first (one sync), then exactly `total` features per array
    if ((rc = launch_offsets(ctx, f->d_count, f->d_slots, n, f->d_offsets)) != YGZB_OK) return rc;
    // array stride rounded up to 4 elements: the descriptor rows behind the five 4-byte arrays are moved as uint4
    const size_t cap = ((size_t)n * g.n_cells + 3) & ~(size_t)3;
    uint8_t* pk = (uint8_t*)dev_scratch(ctx, 1, cap * 56);
    if (!pk) return YGZB_ERR_CUDA;
    float* ox = (float*)pk;
    float* oy = ox + cap;
    float* oscore = oy + cap;
    float* oangle = oscore + cap;
    int32_t* ocell = (int32_t*)(oangle + cap);
    uint8_t* odesc = (uint8_t*)(ocell + cap);
    uint8_t* olevel = odesc + cap * 32;
    dim3 grid((g.n_cells + 255) / 256, n);
    ProfScope ps(ctx, kStagePack);
    pack_features_kernel<<<grid, 256, 0, ctx->stream>>>(f->d_slots, f->d_offsets, g.n_cells, f->d_count, f->d_fx, f->d_fy,
                                                        f->d_flevel, f->d_fscore, f->d_fangle, f->d_fcell, f->d_fdesc, ox, oy,
                                                        olevel, oscore, oangle, ocell, odesc);
    YGZB_LAUNCHED(ctx);
    YGZB_CUDA(ctx, cudaMemcpyAsync(out->offsets, f->d_offsets, (size_t)(n + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const size_t total = (size_t)out->offsets[n];
    if ((size_t)out->capacity < total)
        return set_error(ctx, YGZB_ERR_CAPACITY, "ygzb_keypoints.capacity %d < %zu features", out->capacity, total);
    if (total) {
        YGZB_CUDA(ctx, cudaMemcpyAsync(out->x, ox, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(out->y, oy, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(out->level, olevel, total, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(out->score, oscore, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(out->angle, oangle, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(out->desc, odesc, total * 32, cudaMemcpyDeviceToHost, ctx->stream));
        if (out->cell) YGZB_CUDA(ctx, cudaMemcpyAsync(out->cell, ocell, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return YGZB_OK;
}

int ygzb_detect_stats(ygzb_frames* f, int n, int32_t* stats) {
    if (!f || !stats || n < 1 || n > f->capacity) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    cudaSetDevice(ctx->device);
    YGZB_CUDA(ctx, cudaMemcpyAsync(stats, f->d_stats, (size_t)n * ctx->geo.n_levels * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                   ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

int ygzb_describe(ygzb_frames* f, const int32_t* slots, int n, const int32_t* offsets, const double* x, const double* y,
                  const uint8_t* level, float* angle, uint8_t* desc) {
    if (!f || !offsets || !x || !y || !level || !angle || !desc) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    cudaSetDevice(ctx->device);
    int rc = upload_slots(f, slots, n);
    if (rc != YGZB_OK) return rc;
    if (n < 0) return YGZB_ERR_INVALID;
    rc = check_offsets(ctx, offsets, n, "offsets");
    if (rc != YGZB_OK) return rc;
    const int total = offsets[n];
    if (total <= 0) return YGZB_OK;
    for (int i = 0; i < total; ++i)
        if (level[i] >= ctx->geo.n_levels) return set_error(ctx, YGZB_ERR_INVALID, "feature %d: level %d out of range", i, level[i]);
    int max_per = 0;
    for (int i = 0; i < n; ++i) max_per = std::max(max_per, offsets[i + 1] - offsets[i]);
    const size_t T = (size_t)total;
    uint8_t* buf = (uint8_t*)dev_scratch(ctx, 2, T * (8 + 8 + 4 + 4 + 32 + 1) + (size_t)(n + 1) * 4 + 64);
    if (!buf) return YGZB_ERR_CUDA;
    double* dx = (double*)buf;
    double* dy = dx + T;
    float* dangle = (float*)(dy + T);
    int32_t* dslot_of = (int32_t*)(dangle + T);
    int32_t* doff = dslot_of + T;
    uint8_t* ddesc = (uint8_t*)(doff + n + 1);
    ddesc = (uint8_t*)(((uintptr_t)ddesc + 15) & ~(uintptr_t)15);
    uint8_t* dlevel = ddesc + T * 32;
    YGZB_CUDA(ctx, cudaMemcpyAsync(dx, x, T * 8, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(dy, y, T * 8, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(dlevel, level, T, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(doff, offsets, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    dim3 grid((max_per + 255) / 256, n);
    expand_slots_kernel<<<grid, 256, 0, ctx->stream>>>(f->d_slots, doff, n, dslot_of);
    YGZB_LAUNCHED(ctx);
    if ((rc = launch_describe_list(f, n, dslot_of, total, dx, dy, dlevel, dangle, ddesc)) != YGZB_OK) return rc;
    YGZB_CUDA(ctx, cudaMemcpyAsync(angle, dangle, T * 4, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(desc, ddesc, T * 32, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

int ygzb_fast_debug(ygzb_frames* f, int slot, int level, int capacity, int16_t* xy, int32_t* scores, int32_t* n_corners,
                    int32_t* nonmax_idx, int32_t* n_nonmax) {
    if (!f || !xy || !scores || !n_corners || !nonmax_idx || !n_nonmax) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    const Geometry& g = ctx->geo;
    if (slot < 0 || slot >= f->capacity || level < 0 || level >= g.n_levels) return YGZB_ERR_INVALID;
    cudaSetDevice(ctx->device);
    const LevelGeom& lv = g.lv[level];
    const size_t px = (size_t)lv.w * lv.h;
    uint8_t* d = (uint8_t*)dev_scratch(ctx, 3, 2 * px);
    uint8_t* h = (uint8_t*)host_scratch(ctx, 1, 2 * px);
    if (!d || !h) return YGZB_ERR_CUDA;
    int rc = launch_fast_debug(f, slot, level, d, d + px);
    if (rc != YGZB_OK) return rc;
    YGZB_CUDA(ctx, cudaMemcpyAsync(h, d, 2 * px, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    // enumeration only (no decisions): raster-order corner list and the positions of the survivors in it
    int nc = 0, nn = 0;
    for (int y = 0; y < lv.h; ++y)
        for (int x = 0; x < lv.w; ++x) {
            const size_t i = (size_t)y * lv.w + x;
            if (!h[i]) continue;
            if (nc < capacity) {
                xy[2 * nc] = (int16_t)x;
                xy[2 * nc + 1] = (int16_t)y;
                scores[nc] = h[i];
                if (h[px + i]) {
                    if (nn < capacity) nonmax_idx[nn] = nc;
                    ++nn;
                }
            }
            ++nc;
        }
    *n_corners = nc;
    *n_nonmax = nn;
    return nc > capacity ? set_error(ctx, YGZB_ERR_CAPACITY, "%d corners > capacity %d", nc, capacity) : YGZB_OK;
}

// ---- Matcher: descriptors ---------------------------------------------------------------------------
int ygzb_match_bf(ygzb_ctx* ctx, const uint8_t* A, int nA, const uint8_t* B, int nB, int cross_check, int32_t* train_idx,
                  int32_t* dist) {
    if (!ctx || nA < 0 || nB < 0 || (nA && !A) || (nB && !B) || !train_idx || !dist) return YGZB_ERR_INVALID;
    if (nA > 65535 || nB > 65535) return set_error(ctx, YGZB_ERR_INVALID, "at most 65535 descriptors per set");
    if (nA == 0) return YGZB_OK;
    cudaSetDevice(ctx->device);
    const int cap = std::max(nA, nB);
    const size_t stride = (size_t)cap * 32;
    // [descs A | descs B | counts(2) a_set b_set q_off(2) | fwd | col | idx | dist]
    uint8_t* buf = (uint8_t*)dev_scratch(ctx, 4, 2 * stride + 64 + (size_t)cap * 16);
    int32_t* h = (int32_t*)host_scratch(ctx, 2, 64);
    if (!buf || !h) return YGZB_ERR_CUDA;
    int32_t* meta = (int32_t*)(buf + 2 * stride);
    unsigned* fwd = (unsigned*)(meta + 16);
    unsigned* col = fwd + cap;
    int32_t* didx = (int32_t*)(col + cap);
    int32_t* ddist = didx + cap;
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    h[0] = nA; h[1] = nB; h[2] = 0; h[3] = 1; h[4] = 0; h[5] = nA;
    YGZB_CUDA(ctx, cudaMemcpyAsync(meta, h, 6 * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(buf, A, (size_t)nA * 32, cudaMemcpyHostToDevice, ctx->stream));
    if (nB) YGZB_CUDA(ctx, cudaMemcpyAsync(buf + stride, B, (size_t)nB * 32, cudaMemcpyHostToDevice, ctx->stream));
    int rc = launch_match(ctx, buf, stride, meta, meta + 2, meta + 3, 1, cap, cross_check, fwd, col, meta + 4, didx, ddist);
    if (rc != YGZB_OK) return rc;
    YGZB_CUDA(ctx, cudaMemcpyAsync(train_idx, didx, (size_t)nA * 4, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(dist, ddist, (size_t)nA * 4, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

int ygzb_match_frames(ygzb_frames* f, const int32_t* a_slots, const int32_t* b_slots, int n_pairs, int cross_check,
                      int32_t* q_offsets, int32_t* train_idx, int32_t* dist, int capacity) {
    if (!f || !a_slots || !b_slots || n_pairs < 1) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    const Geometry& g = ctx->geo;
    cudaSetDevice(ctx->device);
    for (int i = 0; i < n_pairs; ++i)
        if (a_slots[i] < 0 || a_slots[i] >= f->capacity || b_slots[i] < 0 || b_slots[i] >= f->capacity)
            return set_error(ctx, YGZB_ERR_INVALID, "pair %d: slot out of range", i);
    const size_t P = (size_t)n_pairs, cap = (size_t)g.n_cells;
    // [a_sets | b_sets | q_off (P+1) | fwd | col | idx | dist]
    uint8_t* buf = (uint8_t*)dev_scratch(ctx, 5, (3 * P + 1) * 4 + 64 + P * cap * 16);
    int32_t* h = (int32_t*)host_scratch(ctx, 3, 2 * P * 4);
    if (!buf || !h) return YGZB_ERR_CUDA;
    int32_t* d_a = (int32_t*)buf;
    int32_t* d_b = d_a + P;
    int32_t* d_qoff = d_b + P;
    unsigned* fwd = (unsigned*)(((uintptr_t)(d_qoff + P + 1) + 15) & ~(uintptr_t)15);
    unsigned* col = fwd + P * cap;
    int32_t* didx = (int32_t*)(col + P * cap);
    int32_t* ddist = didx + P * cap;
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(h, a_slots, P * 4);
    memcpy(h + P, b_slots, P * 4);
    YGZB_CUDA(ctx, cudaMemcpyAsync(d_a, h, 2 * P * 4, cudaMemcpyHostToDevice, ctx->stream));
    int rc = launch_offsets(ctx, f->d_count, d_a, n_pairs, d_qoff);
    if (rc != YGZB_OK) return rc;
    rc = launch_match(ctx, f->d_fdesc, cap * 32, f->d_count, d_a, d_b, n_pairs, (int)cap, cross_check, fwd, col, d_qoff, didx,
                      ddist);
    if (rc != YGZB_OK) return rc;
    if (!q_offsets) return YGZB_OK;  // results stay on the device (bench "value" leg)
    YGZB_CUDA(ctx, cudaMemcpyAsync(q_offsets, d_qoff, (P + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const size_t total = (size_t)q_offsets[n_pairs];
    if ((size_t)capacity < total) return set_error(ctx, YGZB_ERR_CAPACITY, "match capacity %d < %zu queries", capacity, total);
    if (total && train_idx && dist) {
        YGZB_CUDA(ctx, cudaMemcpyAsync(train_idx, didx, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(dist, ddist, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return YGZB_OK;
}

int ygzb_hamming_pairs(ygzb_ctx* ctx, const uint8_t* A, int nA, const uint8_t* B, int nB, const int32_t* ia, const int32_t* ib,
                       int n, int32_t* dist) {
    if (!ctx || !A || !B || !ia || !ib || !dist || n < 0 || nA < 1 || nB < 1) return YGZB_ERR_INVALID;
    if (n == 0) return YGZB_OK;
    for (int k = 0; k < n; ++k)
        if (ia[k] < 0 || ia[k] >= nA || ib[k] < 0 || ib[k] >= nB) return set_error(ctx, YGZB_ERR_INVALID, "pair %d: index out of range", k);
    cudaSetDevice(ctx->device);
    const size_t sa = ((size_t)nA * 32 + 15) & ~(size_t)15, sb = ((size_t)nB * 32 + 15) & ~(size_t)15;
    uint8_t* buf = (uint8_t*)dev_scratch(ctx, 4, sa + sb + (size_t)n * 12);
    if (!buf) return YGZB_ERR_CUDA;
    int32_t* dia = (int32_t*)(buf + sa + sb);
    int32_t* dib = dia + n;
    int32_t* dd = dib + n;
    YGZB_CUDA(ctx, cudaMemcpyAsync(buf, A, (size_t)nA * 32, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(buf + sa, B, (size_t)nB * 32, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(dia, ia, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(dib, ib, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    int rc = launch_hamming_pairs(ctx, buf, buf + sa, dia, dib, n, dd);
    if (rc != YGZB_OK) return rc;
    YGZB_CUDA(ctx, cudaMemcpyAsync(dist, dd, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

}  // extern "C"
