// klt.cu -- pyramidal Lucas-Kanade tracking of feature points, one warp per point.
//
// Replaces Tracker::TrackKLT (reference src/Algorithm/Tracker.cpp:65-113), i.e.
//     cv::calcOpticalFlowPyrLK(ref.pyr[0], cur.pyr[0], pt_ref, pt_cur, status, err, Size(21,21), 4,
//                              TermCriteria(COUNT+EPS, 30, 0.001), OPTFLOW_USE_INITIAL_FLOW)
// OpenCV's algorithm (video/lkpyramid.cpp; not in the reference tree) as pinned by oracle/klt.cpp:
// pyrDown pyramid (levels stop while larger than the window), Scharr (3,10,3) derivatives with reflect-101
// inside the image and 0 outside, 2^14 fixed-point bilinear weights, int16 template (x32), 2x2 normal equations
// scaled by 2^-20, min-eigenvalue test, <= 30 iterations with the eps^2 and |delta + prev| < 0.01 stops.
//
// A warp walks one point from the coarsest level down.  Per level it stages a 24x24 reflect-101 window of I in
// shared memory, derives the 22x22 Scharr gradients from it, builds the 21x21 template (I, Ix, Iy as int16) and
// iterates on J with 14 window pixels per lane.  The window sums are EXACT 64-bit integer sums (OpenCV accumulates
// the same integer products in f32; its SIMD and scalar builds already differ in the last bits), reduced with warp
// shuffles.  Roofline class: L1/L2-resident gather, latency bound (2.6 kB first touch per point and level).
#include <algorithm>
#include <exception>
#include <vector>

#include "common.cuh"

namespace ygzb {

namespace {

constexpr int kWin = 21;
constexpr int kKltWarps = 4;
constexpr int kMaxKltLevels = 8;

struct KltLevel {
    int w, h, pitch;
};

struct KltArgs {
    const uint8_t* const* level_ptr;  // [n_images][kMaxKltLevels]
    KltLevel lv[kMaxKltLevels];
    int max_level;
    const int32_t* ref_img;           // per point: image index of the reference / current frame
    const int32_t* cur_img;
    const float* ref_xy;
    float* cur_xy;
    uint8_t* status;
    float* err;
    int n;
    int max_count;
    double eps2;
    float min_eig;
};

__device__ __forceinline__ int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * (n - 1) - i;
    return i;
}
__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }
__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
    return __shfl_sync(0xFFFFFFFFu, v, 0);
}

struct Weights {
    int w00, w01, w10, w11;
};
__device__ __forceinline__ Weights make_weights(float a, float b) {
    Weights w;
    const float s = (float)(1 << 14);
    w.w00 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), __fsub_rn(1.f, b)), s));
    w.w01 = __float2int_rn(__fmul_rn(__fmul_rn(a, __fsub_rn(1.f, b)), s));
    w.w10 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), b), s));
    w.w11 = (1 << 14) - w.w00 - w.w01 - w.w10;
    return w;
}

// stage a (rows x cols) reflect-101 window of `img` whose top-left pixel is (x0, y0)
__device__ __forceinline__ void stage(uint8_t* s, int pitch_s, const uint8_t* __restrict__ img, const KltLevel& lv, int x0, int y0,
                                      int cols, int rows, int lane) {
    for (int i = lane; i < rows * cols; i += 32) {
        const int r = i / cols, c = i - r * cols;
        s[r * pitch_s + c] = img[(size_t)reflect101(y0 + r, lv.h) * lv.pitch + reflect101(x0 + c, lv.w)];
    }
}

__global__ void __launch_bounds__(kKltWarps * 32) klt_kernel(const KltArgs a) {
    __shared__ uint8_t s_patch[kKltWarps][24 * 24];
    __shared__ short s_grad[kKltWarps][22 * 22 * 2];
    __shared__ short s_I[kKltWarps][kWin * kWin];
    __shared__ short s_dI[kKltWarps][kWin * kWin * 2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kKltWarps + warp;
    if (i >= a.n) return;
    uint8_t* patch = s_patch[warp];
    short* grad = s_grad[warp];
    short* Iw = s_I[warp];
    short* dIw = s_dI[warp];
    const float half = (kWin - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (1 << 20);
    float cx = a.cur_xy[2 * i], cy = a.cur_xy[2 * i + 1];
    const float rx = a.ref_xy[2 * i], ry = a.ref_xy[2 * i + 1];
    bool status = true;
    float errv = 0.f;

    for (int level = a.max_level; level >= 0; --level) {
        const KltLevel lv = a.lv[level];
        const uint8_t* __restrict__ I = a.level_ptr[(size_t)a.ref_img[i] * kMaxKltLevels + level];
        const uint8_t* __restrict__ J = a.level_ptr[(size_t)a.cur_img[i] * kMaxKltLevels + level];
        const float sc = (float)(1. / (1 << level));
        float prevx = __fmul_rn(rx, sc), prevy = __fmul_rn(ry, sc);
        float nx, ny;
        if (level == a.max_level) {
            nx = __fmul_rn(cx, sc);
            ny = __fmul_rn(cy, sc);
        } else {
            nx = __fmul_rn(cx, 2.f);
            ny = __fmul_rn(cy, 2.f);
        }
        cx = nx;
        cy = ny;
        prevx = __fsub_rn(prevx, half);
        prevy = __fsub_rn(prevy, half);
        const int ipx = (int)floorf(prevx), ipy = (int)floorf(prevy);
        if (ipx < -kWin || ipx >= lv.w || ipy < -kWin || ipy >= lv.h) {
            if (level == 0) {
                status = false;
                errv = 0.f;
            }
            continue;
        }
        // template: 24x24 window of I starting at (ipx-1, ipy-1); gradients on the inner 22x22
        __syncwarp();
        stage(patch, 24, I, lv, ipx - 1, ipy - 1, 24, 24, lane);
        __syncwarp();
        for (int k = lane; k < 22 * 22; k += 32) {
            const int r = k / 22, c = k - r * 22;
            const int X = ipx + c, Y = ipy + r;
            int dx = 0, dy = 0;
            if (X >= 0 && X < lv.w && Y >= 0 && Y < lv.h) {
                // calcSharrDeriv reflects at the IMAGE border: the staged window is the reflect-101 padded image, and
                // reflect101(reflect101(x) +- 1) differs from reflect101(x +- 1) only outside the image, which is excluded here
                const uint8_t* q = patch + (r + 1) * 24 + (c + 1);
                const int t0m = (q[-24 - 1] + q[24 - 1]) * 3 + q[-1] * 10, t0p = (q[-24 + 1] + q[24 + 1]) * 3 + q[1] * 10;
                const int t1m = q[24 - 1] - q[-24 - 1], t1c = q[24] - q[-24], t1p = q[24 + 1] - q[-24 + 1];
                dx = t0p - t0m;
                dy = (t1p + t1m) * 3 + t1c * 10;
            }
            grad[2 * k] = (short)dx;
            grad[2 * k + 1] = (short)dy;
        }
        __syncwarp();
        Weights w = make_weights(__fsub_rn(prevx, (float)ipx), __fsub_rn(prevy, (float)ipy));
        long long sA11 = 0, sA12 = 0, sA22 = 0;
        for (int k = lane; k < kWin * kWin; k += 32) {
            const int y = k / kWin, x = k - y * kWin;
            const uint8_t* q = patch + (y + 1) * 24 + (x + 1);
            const short* g = grad + 2 * (y * 22 + x);
            const int ival = descale(q[0] * w.w00 + q[1] * w.w01 + q[24] * w.w10 + q[25] * w.w11, 14 - 5);
            const int ixval = descale(g[0] * w.w00 + g[2] * w.w01 + g[44] * w.w10 + g[46] * w.w11, 14);
            const int iyval = descale(g[1] * w.w00 + g[3] * w.w01 + g[45] * w.w10 + g[47] * w.w11, 14);
            Iw[k] = (short)ival;
            dIw[2 * k] = (short)ixval;
            dIw[2 * k + 1] = (short)iyval;
            sA11 += (long long)ixval * ixval;
            sA12 += (long long)ixval * iyval;
            sA22 += (long long)iyval * iyval;
        }
        sA11 = warp_sum_ll(sA11);
        sA12 = warp_sum_ll(sA12);
        sA22 = warp_sum_ll(sA22);
        const float A11 = __fmul_rn((float)sA11, FLT_SCALE), A12 = __fmul_rn((float)sA12, FLT_SCALE), A22 = __fmul_rn((float)sA22, FLT_SCALE);
        float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
        const float dd = __fsub_rn(A11, A22);
        const float minEig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(__fadd_rn(__fmul_rn(dd, dd), __fmul_rn(__fmul_rn(4.f, A12), A12)))),
                                       (float)(2 * kWin * kWin));
        if (minEig < a.min_eig || D < 1.1920929e-07f) {
            if (level == 0) status = false;
            continue;
        }
        D = __fdiv_rn(1.f, D);
        nx = __fsub_rn(nx, half);
        ny = __fsub_rn(ny, half);
        float pdx = 0.f, pdy = 0.f;
        for (int j = 0; j < a.max_count; ++j) {
            const int inx = (int)floorf(nx), iny = (int)floorf(ny);
            if (inx < -kWin || inx >= lv.w || iny < -kWin || iny >= lv.h) {
                if (level == 0) status = false;
                break;
            }
            __syncwarp();
            stage(patch, 24, J, lv, inx, iny, 22, 22, lane);
            __syncwarp();
            w = make_weights(__fsub_rn(nx, (float)inx), __fsub_rn(ny, (float)iny));
            long long sb1 = 0, sb2 = 0;
            for (int k = lane; k < kWin * kWin; k += 32) {
                const int y = k / kWin, x = k - y * kWin;
                const uint8_t* q = patch + y * 24 + x;
                const int diff = descale(q[0] * w.w00 + q[1] * w.w01 + q[24] * w.w10 + q[25] * w.w11, 14 - 5) - Iw[k];
                sb1 += (long long)(diff * dIw[2 * k]);
                sb2 += (long long)(diff * dIw[2 * k + 1]);
            }
            sb1 = warp_sum_ll(sb1);
            sb2 = warp_sum_ll(sb2);
            const float b1 = __fmul_rn((float)sb1, FLT_SCALE), b2 = __fmul_rn((float)sb2, FLT_SCALE);
            const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, b2), __fmul_rn(A22, b1)), D);
            const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, b1), __fmul_rn(A11, b2)), D);
            nx = __fadd_rn(nx, dx);
            ny = __fadd_rn(ny, dy);
            cx = __fadd_rn(nx, half);
            cy = __fadd_rn(ny, half);
            if ((double)dx * dx + (double)dy * dy <= a.eps2) break;
            if (j > 0 && fabs((double)__fadd_rn(dx, pdx)) < 0.01 && fabs((double)__fadd_rn(dy, pdy)) < 0.01) {
                cx = __fsub_rn(cx, __fmul_rn(dx, 0.5f));
                cy = __fsub_rn(cy, __fmul_rn(dy, 0.5f));
                break;
            }
            pdx = dx;
            pdy = dy;
        }
        if (status && level == 0) {
            const float fx = __fsub_rn(cx, half), fy = __fsub_rn(cy, half);
            const int inx = (int)floorf(fx), iny = (int)floorf(fy);
            if (inx < -kWin || inx >= lv.w || iny < -kWin || iny >= lv.h) {
                status = false;
                continue;
            }
            __syncwarp();
            stage(patch, 24, J, lv, inx, iny, 22, 22, lane);
            __syncwarp();
            w = make_weights(__fsub_rn(fx, (float)inx), __fsub_rn(fy, (float)iny));
            long long se = 0;
            for (int k = lane; k < kWin * kWin; k += 32) {
                const int y = k / kWin, x = k - y * kWin;
                const uint8_t* q = patch + y * 24 + x;
                const int diff = descale(q[0] * w.w00 + q[1] * w.w01 + q[24] * w.w10 + q[25] * w.w11, 14 - 5) - Iw[k];
                se += diff < 0 ? -diff : diff;
            }
            se = warp_sum_ll(se);
            errv = __fdiv_rn(__fmul_rn((float)se, 1.f), (float)(32 * kWin * kWin));
        }
    }
    if (lane == 0) {
        a.cur_xy[2 * i] = cx;
        a.cur_xy[2 * i + 1] = cy;
        a.status[i] = status ? 1 : 0;
        a.err[i] = errv;
    }
}

}  // namespace
}  // namespace ygzb

using namespace ygzb;

extern "C" {

void ygzb_default_klt_params(ygzb_klt_params* p) {
    p->win = 21;         // Tracker::Option::klt_win_size (include/ygz/Algorithm/Tracker.h:25)
    p->max_level = 4;    // Tracker.cpp:97
    p->max_iter = 30;    // klt_max_iter
    p->eps = 0.001;      // klt_eps
    p->min_eig = 1e-4;   // cv::calcOpticalFlowPyrLK default minEigThreshold
}

static int klt_impl(ygzb_frames* f, int n_pairs, const int32_t* ref_slot, const int32_t* cur_slot, const int32_t* offsets,
                    const float* ref_xy, float* cur_xy, uint8_t* status, float* err, const ygzb_klt_params* prm);

int ygzb_klt(ygzb_frames* f, int n_pairs, const int32_t* ref_slot, const int32_t* cur_slot, const int32_t* offsets,
             const float* ref_xy, float* cur_xy, uint8_t* status, float* err, const ygzb_klt_params* prm) {
    try {   // never throws (header): host-side bookkeeping failures become an error code
        return klt_impl(f, n_pairs, ref_slot, cur_slot, offsets, ref_xy, cur_xy, status, err, prm);
    } catch (const std::exception& e) {
        return f ? set_error(f->ctx, YGZB_ERR_INVALID, "ygzb_klt: %s", e.what()) : YGZB_ERR_INVALID;
    }
}

static int klt_impl(ygzb_frames* f, int n_pairs, const int32_t* ref_slot, const int32_t* cur_slot, const int32_t* offsets,
                    const float* ref_xy, float* cur_xy, uint8_t* status, float* err, const ygzb_klt_params* prm) {
    if (!f || n_pairs < 1 || !ref_slot || !cur_slot || !offsets || !prm) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = f->ctx;
    const Geometry& g = ctx->geo;
    cudaSetDevice(ctx->device);
    if (prm->win != kWin) return set_error(ctx, YGZB_ERR_INVALID, "only the reference's 21x21 window is supported (got %d)", prm->win);
    {
        const int rc = check_offsets(ctx, offsets, n_pairs, "offsets");
        if (rc != YGZB_OK) return rc;
    }
    const int total = offsets[n_pairs];
    if (total <= 0) return YGZB_OK;
    if (!ref_xy || !cur_xy || !status || !err) return YGZB_ERR_INVALID;
    for (int p = 0; p < n_pairs; ++p)
        if (ref_slot[p] < 0 || ref_slot[p] >= f->capacity || cur_slot[p] < 0 || cur_slot[p] >= f->capacity)
            return set_error(ctx, YGZB_ERR_INVALID, "pair %d: slot out of range", p);
    // pyramid depth like buildOpticalFlowPyramid: stop when a level is not larger than the window
    KltArgs a;
    int w = g.lv[0].w, h = g.lv[0].h, max_level = 0;
    a.lv[0] = KltLevel{w, h, g.lv[0].pitch};
    for (int L = 1; L <= std::min(prm->max_level, kMaxKltLevels - 1); ++L) {
        const int nw = (w + 1) / 2, nh = (h + 1) / 2;
        if (nw <= kWin || nh <= kWin) break;
        w = nw;
        h = nh;
        a.lv[L] = KltLevel{w, h, (w + 15) & ~15};
        max_level = L;
    }
    const int n_img = 2 * n_pairs;
    // levels the slot pyramid does not hold are built into scratch with the same pyrDown kernel
    size_t extra_bytes = 0;
    std::vector<size_t> extra_off(kMaxKltLevels, 0);
    for (int L = g.n_levels; L <= max_level; ++L) {
        extra_off[L] = extra_bytes;
        extra_bytes += ((size_t)a.lv[L].pitch * a.lv[L].h + 255) & ~(size_t)255;
    }
    const size_t T = (size_t)total;
    uint8_t *d_extra, *d_status;
    const uint8_t **d_ptrs, **d_src;
    uint8_t** d_dst;
    int32_t* d_img;
    float *d_ref, *d_cur, *d_err;
    void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
        d_extra = c.take<uint8_t>(extra_bytes * n_img);
        d_ptrs = c.take<const uint8_t*>((size_t)n_img * kMaxKltLevels);
        d_img = c.take<int32_t>(2 * T);
        d_ref = c.take<float>(2 * T);
        d_cur = c.take<float>(2 * T);
        d_status = c.take<uint8_t>(T);
        d_err = c.take<float>(T);
        d_src = c.take<const uint8_t*>((size_t)n_img);
        d_dst = c.take<uint8_t*>((size_t)n_img);
    });
    if (!buf) return YGZB_ERR_CUDA;
    std::vector<const uint8_t*> ptrs((size_t)n_img * kMaxKltLevels, nullptr);
    for (int im = 0; im < n_img; ++im) {
        const int slot = (im & 1) ? cur_slot[im / 2] : ref_slot[im / 2];
        for (int L = 0; L <= max_level; ++L) {
            if (L < g.n_levels) {
                ptrs[(size_t)im * kMaxKltLevels + L] = f->d_pyr + (size_t)slot * ctx->slot_stride + g.lv[L].off;
                a.lv[L].pitch = g.lv[L].pitch;
            } else {
                ptrs[(size_t)im * kMaxKltLevels + L] = d_extra + (size_t)im * extra_bytes + extra_off[L];
            }
        }
    }
    std::vector<int32_t> img_of(2 * T);
    for (int p = 0; p < n_pairs; ++p)
        for (int i = offsets[p]; i < offsets[p + 1]; ++i) {
            img_of[i] = 2 * p;
            img_of[T + i] = 2 * p + 1;
        }
    YGZB_CUDA(ctx, cudaMemcpyAsync(d_ptrs, ptrs.data(), ptrs.size() * sizeof(void*), cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(d_img, img_of.data(), 2 * T * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(d_ref, ref_xy, 2 * T * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(d_cur, cur_xy, 2 * T * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    for (int L = std::max(g.n_levels, 1); L <= max_level; ++L) {
        std::vector<const uint8_t*> src(n_img);
        std::vector<uint8_t*> dst(n_img);
        for (int im = 0; im < n_img; ++im) {
            src[im] = ptrs[(size_t)im * kMaxKltLevels + L - 1];
            dst[im] = const_cast<uint8_t*>(ptrs[(size_t)im * kMaxKltLevels + L]);
        }
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_src, src.data(), n_img * sizeof(void*), cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_dst, dst.data(), n_img * sizeof(void*), cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // src/dst host vectors are reused per level
        int rc = launch_pyrdown_ptrs(ctx, d_src, d_dst, a.lv[L - 1].w, a.lv[L - 1].h, a.lv[L - 1].pitch, a.lv[L].w, a.lv[L].h, a.lv[L].pitch, n_img);
        if (rc != YGZB_OK) return rc;
    }
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    a.level_ptr = d_ptrs;
    a.max_level = max_level;
    a.ref_img = d_img;
    a.cur_img = d_img + T;
    a.ref_xy = d_ref;
    a.cur_xy = d_cur;
    a.status = d_status;
    a.err = d_err;
    a.n = total;
    a.max_count = std::min(std::max(prm->max_iter, 0), 100);
    const double e = std::min(std::max(prm->eps, 0.), 10.);
    a.eps2 = e * e;
    a.min_eig = (float)prm->min_eig;
    {
        ProfScope ps(ctx, kStageKLT);
        klt_kernel<<<(total + kKltWarps - 1) / kKltWarps, kKltWarps * 32, 0, ctx->stream>>>(a);
    }
    YGZB_LAUNCHED(ctx);
    YGZB_CUDA(ctx, cudaMemcpyAsync(cur_xy, d_cur, 2 * T * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(status, d_status, T, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(err, d_err, T * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

}  // extern "C"
