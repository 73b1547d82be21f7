// api_align.cu -- extern "C" entry points for the photometric alignment stages (marshalling only).
#include <algorithm>

#include <cstring>

#include "common.cuh"

using namespace ygzb;

namespace {

int check_slots(ygzb_frames* f, const int32_t* s, int n, const char* what) {
    for (int i = 0; i < n; ++i)
        if (s[i] < 0 || s[i] >= f->capacity) return set_error(f->ctx, YGZB_ERR_INVALID, "%s[%d] = %d out of range", what, i, s[i]);
    return YGZB_OK;
}

}  // namespace

extern "C" {

int ygzb_align2d(ygzb_frames* f, int n, const int32_t* slot, const uint8_t* level, const uint8_t* ref_border, const uint8_t* ref,
                 int n_iter, double* uv, uint8_t* ok) {
    if (!f || n < 0 || (n && (!slot || !level || !ref_border || !uv || !ok))) return YGZB_ERR_INVALID;
    if (n == 0) return YGZB_OK;
    ygzb_ctx* ctx = f->ctx;
    cudaSetDevice(ctx->device);
    TRY(check_slots(f, slot, n, "slot"));
    for (int i = 0; i < n; ++i)
        if (level[i] >= ctx->geo.n_levels) return set_error(ctx, YGZB_ERR_INVALID, "level[%d] out of range", i);
    const size_t N = (size_t)n;
    int32_t* d_slot;
    uint8_t *d_level, *d_rb, *d_ref, *d_ok;
    double* d_uv;
    void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
        d_slot = c.take<int32_t>(N);
        d_level = c.take<uint8_t>(N);
        d_rb = c.take<uint8_t>(N * 100);
        d_ref = c.take<uint8_t>(N * 64);
        d_uv = c.take<double>(2 * N);
        d_ok = c.take<uint8_t>(N);
    });
    if (!buf) return YGZB_ERR_CUDA;
    TRY(h2d(ctx, d_slot, slot, N));
    TRY(h2d(ctx, d_level, level, N));
    TRY(h2d(ctx, d_rb, ref_border, N * 100));
    if (ref) TRY(h2d(ctx, d_ref, ref, N * 64));
    TRY(h2d(ctx, d_uv, uv, 2 * N));
    TRY(launch_align2d(f, n, d_slot, d_level, d_rb, ref ? d_ref : nullptr, n_iter, d_uv, d_ok));
    TRY(d2h(ctx, uv, d_uv, 2 * N));
    TRY(d2h(ctx, ok, d_ok, N));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

int ygzb_align1d(ygzb_frames* f, int n, const int32_t* slot, const uint8_t* level, const float* dir, const uint8_t* ref_border,
                 const uint8_t* ref, int n_iter, double* uv, uint8_t* ok, double* h_inv) {
    if (!f || n < 0 || (n && (!slot || !level || !dir || !ref_border || !uv || !ok || !h_inv))) return YGZB_ERR_INVALID;
    if (n == 0) return YGZB_OK;
    ygzb_ctx* ctx = f->ctx;
    cudaSetDevice(ctx->device);
    TRY(check_slots(f, slot, n, "slot"));
    for (int i = 0; i < n; ++i)
        if (level[i] >= ctx->geo.n_levels) return set_error(ctx, YGZB_ERR_INVALID, "level[%d] out of range", i);
    const size_t N = (size_t)n;
    int32_t* d_slot;
    uint8_t *d_level, *d_rb, *d_ref, *d_ok;
    float* d_dir;
    double *d_uv, *d_h;
    void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
        d_slot = c.take<int32_t>(N);
        d_level = c.take<uint8_t>(N);
        d_dir = c.take<float>(2 * N);
        d_rb = c.take<uint8_t>(N * 100);
        d_ref = c.take<uint8_t>(N * 64);
        d_uv = c.take<double>(2 * N);
        d_ok = c.take<uint8_t>(N);
        d_h = c.take<double>(N);
    });
    if (!buf) return YGZB_ERR_CUDA;
    TRY(h2d(ctx, d_slot, slot, N));
    TRY(h2d(ctx, d_level, level, N));
    TRY(h2d(ctx, d_dir, dir, 2 * N));
    TRY(h2d(ctx, d_rb, ref_border, N * 100));
    if (ref) TRY(h2d(ctx, d_ref, ref, N * 64));
    TRY(h2d(ctx, d_uv, uv, 2 * N));
    TRY(launch_align1d(f, n, d_slot, d_level, d_dir, d_rb, ref ? d_ref : nullptr, n_iter, d_uv, d_ok, d_h));
    TRY(d2h(ctx, uv, d_uv, 2 * N));
    TRY(d2h(ctx, ok, d_ok, N));
    TRY(d2h(ctx, h_inv, d_h, N));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

int ygzb_project_align(ygzb_frames* f, int n, const int32_t* ref_slot, const int32_t* cur_slot, int n_poses, const double* poses,
                       const int32_t* ref_pose, const int32_t* cur_pose, const double* ref_px, const double* ref_depth,
                       const uint8_t* ref_level, double* cur_px, uint8_t* search_level, uint8_t* ok) {
    if (!f || n < 0 || n_poses < 1 || !poses) return YGZB_ERR_INVALID;
    if (n == 0) return YGZB_OK;
    if (!ref_slot || !cur_slot || !ref_pose || !cur_pose || !ref_px || !ref_depth || !ref_level || !cur_px || !search_level || !ok)
        return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    cudaSetDevice(ctx->device);
    TRY(check_slots(f, ref_slot, n, "ref_slot"));
    TRY(check_slots(f, cur_slot, n, "cur_slot"));
    for (int i = 0; i < n; ++i) {
        if (ref_pose[i] < 0 || ref_pose[i] >= n_poses || cur_pose[i] < 0 || cur_pose[i] >= n_poses)
            return set_error(ctx, YGZB_ERR_INVALID, "candidate %d: pose index out of range", i);
        if (ref_level[i] >= ctx->geo.n_levels) return set_error(ctx, YGZB_ERR_INVALID, "ref_level[%d] out of range", i);
    }
    const size_t N = (size_t)n, P = (size_t)n_poses;
    int32_t* d_idx;
    double *d_poses, *d_rpx, *d_depth, *d_cpx;
    uint8_t *d_rlevel, *d_slevel, *d_ok;
    void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
        d_idx = c.take<int32_t>(4 * N);
        d_poses = c.take<double>(12 * P);
        d_rpx = c.take<double>(2 * N);
        d_depth = c.take<double>(N);
        d_cpx = c.take<double>(2 * N);
        d_rlevel = c.take<uint8_t>(N);
        d_slevel = c.take<uint8_t>(N);
        d_ok = c.take<uint8_t>(N);
    });
    if (!buf) return YGZB_ERR_CUDA;
    // the inputs are the first six sub-buffers: one staged copy (nine pageable copies cost more than the kernel itself)
    StagedUpload up;
    TRY(up.begin(ctx, buf, (size_t)((uint8_t*)(d_rlevel + N) - (uint8_t*)buf)));
    up.put(d_idx, ref_slot, N * 4);
    up.put(d_idx + N, cur_slot, N * 4);
    up.put(d_idx + 2 * N, ref_pose, N * 4);
    up.put(d_idx + 3 * N, cur_pose, N * 4);
    up.put(d_poses, poses, 12 * P * 8);
    up.put(d_rpx, ref_px, 2 * N * 8);
    up.put(d_depth, ref_depth, N * 8);
    up.put(d_cpx, cur_px, 2 * N * 8);
    up.put(d_rlevel, ref_level, N);
    TRY(up.commit());
    TRY(launch_project_align(f, n, d_idx, d_idx + N, d_poses, d_idx + 2 * N, d_idx + 3 * N, d_rpx, d_depth, d_rlevel, d_cpx, d_slevel,
                             d_ok));
    TRY(d2h(ctx, cur_px, d_cpx, 2 * N));
    TRY(d2h(ctx, search_level, d_slevel, N));
    TRY(d2h(ctx, ok, d_ok, N));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

int ygzb_sparse_align(ygzb_frames* f, int n_problems, const int32_t* ref_slot, const int32_t* cur_slot, const int32_t* offsets,
                      const double* px, const double* depth, const uint8_t* has_mappoint, const double* T_cw_ref, double* T_cw_cur,
                      int max_level, int min_level, int n_iter, double eps, int32_t* n_meas, int32_t* iters_per_level) {
    return ygzb_sparse_align_fisher(f, n_problems, ref_slot, cur_slot, offsets, px, depth, has_mappoint, T_cw_ref, T_cw_cur, max_level,
                                    min_level, n_iter, eps, n_meas, iters_per_level, nullptr);
}

int ygzb_sparse_align_fisher(ygzb_frames* f, int n_problems, const int32_t* ref_slot, const int32_t* cur_slot, const int32_t* offsets,
                             const double* px, const double* depth, const uint8_t* has_mappoint, const double* T_cw_ref, double* T_cw_cur,
                             int max_level, int min_level, int n_iter, double eps, int32_t* n_meas, int32_t* iters_per_level,
                             double* fisher) {
    if (!f || n_problems < 1 || !ref_slot || !cur_slot || !offsets || !T_cw_ref || !T_cw_cur || !n_meas) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    cudaSetDevice(ctx->device);
    TRY(check_slots(f, ref_slot, n_problems, "ref_slot"));
    TRY(check_slots(f, cur_slot, n_problems, "cur_slot"));
    if (max_level >= ctx->geo.n_levels || min_level < 0 || min_level > max_level)
        return set_error(ctx, YGZB_ERR_INVALID, "levels [%d, %d] outside the %d-level pyramid", min_level, max_level, ctx->geo.n_levels);
    TRY(check_offsets(ctx, offsets, n_problems, "offsets"));
    const size_t P = (size_t)n_problems, T = (size_t)offsets[n_problems];
    if (T && (!px || !depth || !has_mappoint)) return YGZB_ERR_INVALID;
    // one per-problem region of feature records, sized by the largest problem, for CTAs whose share exceeds shared memory
    int max_nf = 0;
    for (int p = 0; p < n_problems; ++p) max_nf = std::max(max_nf, offsets[p + 1] - offsets[p]);
    const size_t feat_stride = sparse_align2_scratch_bytes(1, max_nf);
    int32_t *d_slots, *d_off, *d_nmeas, *d_iters;
    double *d_px, *d_depth, *d_Tref, *d_Tcur, *d_H;
    uint8_t *d_mp, *d_feat;
    void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
        d_slots = c.take<int32_t>(2 * P);
        d_off = c.take<int32_t>(P + 1);
        d_px = c.take<double>(2 * T);
        d_depth = c.take<double>(T);
        d_mp = c.take<uint8_t>(T);
        d_Tref = c.take<double>(12 * P);
        d_Tcur = c.take<double>(12 * P);
        d_nmeas = c.take<int32_t>(P);
        d_iters = c.take<int32_t>(P * kMaxLevels);
        d_feat = c.take<uint8_t>(P * feat_stride);
        d_H = c.take<double>(21 * P);
    });
    if (!buf) return YGZB_ERR_CUDA;
    {   // the inputs are the first seven sub-buffers of `buf`: one staged copy instead of eight pageable ones
        StagedUpload up;
        TRY(up.begin(ctx, buf, (size_t)((uint8_t*)(d_Tcur + 12 * P) - (uint8_t*)buf)));
        up.put(d_slots, ref_slot, P * 4);
        up.put(d_slots + P, cur_slot, P * 4);
        up.put(d_off, offsets, (P + 1) * 4);
        up.put(d_px, px, 2 * T * 8);
        up.put(d_depth, depth, T * 8);
        up.put(d_mp, has_mappoint, T);
        up.put(d_Tref, T_cw_ref, 12 * P * 8);
        up.put(d_Tcur, T_cw_cur, 12 * P * 8);
        TRY(up.commit());
    }
    YGZB_CUDA(ctx, cudaMemsetAsync(d_iters, 0, P * kMaxLevels * sizeof(int32_t), ctx->stream));
    TRY(launch_sparse_align(f, n_problems, d_slots, d_slots + P, d_off, d_px, d_depth, d_mp, d_Tref, d_Tcur, max_level, min_level,
                            n_iter, eps, d_nmeas, d_iters, d_feat, feat_stride, fisher ? d_H : nullptr));
    TRY(d2h(ctx, T_cw_cur, d_Tcur, 12 * P));
    TRY(d2h(ctx, n_meas, d_nmeas, P));
    if (iters_per_level) TRY(d2h(ctx, iters_per_level, d_iters, P * kMaxLevels));
    if (fisher) TRY(d2h(ctx, fisher, d_H, 21 * P));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (fisher)   // SparseImgAlign::getFisherInformation: H_ / (5e-4 * 255 * 255), the image noise
        for (size_t k = 0; k < 21 * P; ++k) fisher[k] /= kFisherNoise;
    return YGZB_OK;
}

}  // extern "C"
