// pyramid.cu -- Frame::InitFrame / CreateImagePyramid on the device.
//
// Replaces (reference src/Basic/Frame.cpp:22-40):
//     cv::cvtColor(_color, gray, CV_BGR2GRAY);  _pyramid[0] = gray;
//     for i in 1..levels: cv::pyrDown(_pyramid[i-1], _pyramid[i]);
// Arithmetic (OpenCV-owned, pinned against cv2 4.13 by the oracle tests):
//     gray = (B*3735 + G*19235 + R*9798 + 16384) >> 15
//     pyrDown: separable [1 4 6 4 1], (sum + 128) >> 8, BORDER_REFLECT_101, dst = ((w+1)/2, (h+1)/2)
//
// Layout: every frame slot holds all levels back to back, each level pitch-linear with a 16-byte
// multiple pitch (so level rows can be moved with 16-byte vectors / TMA boxes).
// Roofline class: HBM.  Algorithmic bytes per frame (8 levels, grey in): 307,200 read + 102,400
// written = 409,600 B.  One launch handles one level of `count` frames.
#include <algorithm>

#include "common.cuh"

namespace ygzb {

namespace {

constexpr int kDW = 64;               // dst tile width
constexpr int kDH = 16;               // dst tile height
constexpr int kSrcRows = 2 * kDH + 3; // 35
constexpr int kSrcWords = 34;         // 136 bytes: src x in [2*x0-4, 2*x0+132)

__device__ __forceinline__ int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = (i < 0) ? -i : 2 * (n - 1) - i;
    return i;
}

__device__ __forceinline__ void pyrdown_tile(const uint8_t* __restrict__ sp, uint8_t* __restrict__ dp, const LevelGeom& src,
                                             const LevelGeom& dst) {
    __shared__ __align__(16) uint8_t s_src[kSrcRows][kSrcWords * 4];
    __shared__ uint16_t s_h[kSrcRows][kDW];

    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * kDW, y0 = blockIdx.y * kDH;

    // stage the source window (reflect-101 at the image border)
    const int xs = 2 * x0 - 4, ys = 2 * y0 - 2;
    for (int i = tid; i < kSrcRows * kSrcWords; i += 256) {
        const int r = i / kSrcWords, k = i - r * kSrcWords;
        const int y = reflect101(ys + r, src.h);
        const int x = xs + 4 * k;
        const uint8_t* row = sp + (size_t)y * src.pitch;
        uint32_t v;
        if (x >= 0 && x + 3 < src.w) {
            v = *reinterpret_cast<const uint32_t*>(row + x);
        } else {
            v = (uint32_t)row[reflect101(x, src.w)] | ((uint32_t)row[reflect101(x + 1, src.w)] << 8) |
                ((uint32_t)row[reflect101(x + 2, src.w)] << 16) | ((uint32_t)row[reflect101(x + 3, src.w)] << 24);
        }
        *reinterpret_cast<uint32_t*>(&s_src[r][4 * k]) = v;
    }
    __syncthreads();

    // horizontal [1 4 6 4 1]: dst column dx is centred on smem column 2*dx + 4
    for (int i = tid; i < kSrcRows * kDW; i += 256) {
        const int r = i / kDW, dx = i - r * kDW;
        const uint8_t* s = &s_src[r][2 * dx + 2];
        s_h[r][dx] = (uint16_t)(s[0] + 4 * s[1] + 6 * s[2] + 4 * s[3] + s[4]);
    }
    __syncthreads();

    // vertical pass, 4 consecutive dst pixels per thread
    const int dy = tid >> 4, dx4 = (tid & 15) * 4;
    const int oy = y0 + dy, ox = x0 + dx4;
    if (oy >= dst.h || ox >= dst.w) return;
    uint32_t packed = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int dx = dx4 + j;
        const int v = s_h[2 * dy][dx] + 4 * s_h[2 * dy + 1][dx] + 6 * s_h[2 * dy + 2][dx] + 4 * s_h[2 * dy + 3][dx] +
                      s_h[2 * dy + 4][dx];
        packed |= (uint32_t)((v + 128) >> 8) << (8 * j);
    }
    uint8_t* out = dp + (size_t)oy * dst.pitch + ox;
    if (ox + 3 < dst.w) {
        *reinterpret_cast<uint32_t*>(out) = packed;  // pitch % 16 == 0 and ox % 4 == 0
    } else {
        for (int j = 0; j < 4 && ox + j < dst.w; ++j) out[j] = (uint8_t)(packed >> (8 * j));
    }
}

// ---- streaming variant for the large levels (source width a multiple of 8) ------------------------------------
// No shared memory: a thread owns 4 adjacent destination pixels (one 32-bit store) of a strip of kStripRows
// destination rows and walks down the source rows with a rolling window of five horizontally filtered rows in
// registers.  All arithmetic is packed u16x2: the horizontal sums are <= 16*255 and the vertical ones <= 256*255,
// so two pixels share one 32-bit register without carries between the halves.  Source bytes come in as one
// aligned 8-byte load (the thread's own 8 source columns) plus the 4-byte words left and right of it (L1 hits:
// they are the neighbours' columns); reflect-101 at the left / right image border is a byte permute of the
// thread's own columns instead of a load, at the top / bottom it is a row index.
// HBM traffic = source read once + destination written once; neighbouring strips share 3 source rows through L1/L2.
constexpr int kStripRows = 8;

struct HRow {
    uint32_t lo, hi;  // (h0, h1) and (h2, h3): horizontal [1 4 6 4 1] sums of the thread's 4 destination columns
};

struct RawRow {
    uint2 m;       // columns 8k .. 8k+7
    uint32_t a;    // bytes 2,3 = columns 8k-2, 8k-1
    uint32_t r;    // byte 0 = column 8k+8
};

// the three loads of one source row (issued early, consumed by hfilter one iteration later)
__device__ __forceinline__ RawRow load_row(const uint8_t* __restrict__ row, int k, bool first, bool last) {
    RawRow w;
    w.m = *reinterpret_cast<const uint2*>(row + 8 * k);
    // reflect-101 at the image border is a byte permute of the thread's own columns instead of a load
    w.a = first ? __byte_perm(w.m.x, 0, 0x1200) : *reinterpret_cast<const uint32_t*>(row + 8 * k - 4);   // columns 2, 1
    w.r = last ? (w.m.y >> 16) : *reinterpret_cast<const uint32_t*>(row + 8 * k + 8);                   // column 8k+6
    return w;
}

__device__ __forceinline__ HRow hfilter(const RawRow& w) {
    const uint2 m = w.m;
    const uint32_t a = w.a, r = w.r;
    const uint32_t e_lo = __byte_perm(m.x, 0, 0x4240), e_hi = __byte_perm(m.y, 0, 0x4240);  // even columns (e0,e1) (e2,e3)
    const uint32_t o_lo = __byte_perm(m.x, 0, 0x4341), o_hi = __byte_perm(m.y, 0, 0x4341);  // odd columns  (o0,o1) (o2,o3)
    const uint32_t em_lo = __byte_perm(e_lo, a, 0x1016);          // (e-1, e0)
    const uint32_t e12 = __funnelshift_r(e_lo, e_hi, 16);         // (e1, e2) = left neighbours of hi = right neighbours of lo
    const uint32_t ep_hi = __byte_perm(e_hi, r, 0x3432);          // (e3, e4)
    const uint32_t om_lo = __byte_perm(o_lo, a, 0x1017);          // (o-1, o0)
    const uint32_t om_hi = __funnelshift_r(o_lo, o_hi, 16);       // (o1, o2)
    HRow h;
    h.lo = em_lo + e12 + 6u * e_lo + 4u * (om_lo + o_lo);
    h.hi = e12 + ep_hi + 6u * e_hi + 4u * (om_hi + o_hi);
    return h;
}

__device__ __forceinline__ uint32_t vfilter_pack(const HRow& h0, const HRow& h1, const HRow& h2, const HRow& h3, const HRow& h4) {
    const uint32_t lo = h0.lo + h4.lo + 4u * (h1.lo + h3.lo) + 6u * h2.lo + 0x00800080u;
    const uint32_t hi = h0.hi + h4.hi + 4u * (h1.hi + h3.hi) + 6u * h2.hi + 0x00800080u;
    return __byte_perm(lo, hi, 0x7531);  // byte 1 of every 16-bit half = (v + 128) >> 8
}

__global__ void __launch_bounds__(256) pyrdown_stream_kernel(uint8_t* __restrict__ pyr, size_t slot_stride, int first_slot,
                                                             LevelGeom src, LevelGeom dst, int strips) {
    const int tpr = src.w >> 3;  // threads per row
    const int id = blockIdx.x * 256 + threadIdx.x;
    const int strip = id / tpr, k = id - strip * tpr;
    if (strip >= strips) return;
    uint8_t* slot = pyr + (size_t)(first_slot + blockIdx.y) * slot_stride;
    const uint8_t* __restrict__ sp = slot + src.off;
    uint8_t* __restrict__ dp = slot + dst.off + 4 * k;
    const bool first = k == 0, last = k == tpr - 1;
    const int dy0 = strip * kStripRows;
    const int sh = src.h;
    // rows -2 .. sh+1 only (sh >= 4 on this path): one reflection, branch-free
    auto raw = [&](int sy) {
        const int r = sy < 0 ? -sy : (sy >= sh ? 2 * (sh - 1) - sy : sy);
        return load_row(sp + (size_t)r * src.pitch, k, first, last);
    };
    HRow h0 = hfilter(raw(2 * dy0 - 2)), h1 = hfilter(raw(2 * dy0 - 1)), h2 = hfilter(raw(2 * dy0));
    // software pipeline: the two source rows of destination row j + 1 are in flight while row j is filtered and stored
    RawRow n3 = raw(2 * dy0 + 1), n4 = raw(2 * dy0 + 2);
#pragma unroll
    for (int j = 0; j < kStripRows; ++j) {
        const int dy = dy0 + j;
        if (dy >= dst.h) break;
        const RawRow c3 = n3, c4 = n4;
        if (j + 1 < kStripRows && dy + 1 < dst.h) {
            n3 = raw(2 * dy + 3);
            n4 = raw(2 * dy + 4);
        }
        const HRow h3 = hfilter(c3), h4 = hfilter(c4);
        *reinterpret_cast<uint32_t*>(dp + (size_t)dy * dst.pitch) = vfilter_pack(h0, h1, h2, h3, h4);
        h0 = h2;
        h1 = h3;
        h2 = h4;
    }
}

// one level of `count` consecutive slots
__global__ void __launch_bounds__(256) pyrdown_kernel(uint8_t* __restrict__ pyr, size_t slot_stride, int first_slot,
                                                      LevelGeom src, LevelGeom dst) {
    uint8_t* slot = pyr + (size_t)(first_slot + blockIdx.z) * slot_stride;
    pyrdown_tile(slot + src.off, slot + dst.off, src, dst);
}

// same, with explicit per-image source / destination pointers (levels beyond the slot pyramid, e.g. for KLT)
__global__ void __launch_bounds__(256) pyrdown_ptr_kernel(const uint8_t* const* __restrict__ src_ptr,
                                                          uint8_t* const* __restrict__ dst_ptr, LevelGeom src, LevelGeom dst) {
    pyrdown_tile(src_ptr[blockIdx.z], dst_ptr[blockIdx.z], src, dst);
}

// all remaining small levels of one frame in ONE CTA: level `first-1` (<= kTailBytes) is staged in shared memory and
// every further level is produced from the previous one there (no launch or HBM round trip per level)
constexpr int kTailBytes = 5120;   // 80 x 60 at 640 x 480: larger sources go through the streaming kernel (measured faster)

__global__ void __launch_bounds__(256) pyrdown_tail_kernel(uint8_t* __restrict__ pyr, size_t slot_stride, int first_slot, Geometry g,
                                                           int first) {
    __shared__ uint8_t s_a[kTailBytes];
    // next level of a w x h source (w * h <= kTailBytes): ((w+1)/2) * ((h+1)/2) <= (w*h + w + h + 1) / 4 <= kTailBytes / 2 + 1
    // (elongated levels such as 341 x 15 -> 171 x 8 = 1368 pixels exceed a quarter of the source)
    __shared__ uint8_t s_b[kTailBytes / 2 + 64];
    uint8_t* slot = pyr + (size_t)(first_slot + blockIdx.x) * slot_stride;
    const int tid = threadIdx.x;
    uint8_t* cur = s_a;
    uint8_t* nxt = s_b;
    {
        const LevelGeom s0 = g.lv[first - 1];
        for (int i = tid; i < s0.w * s0.h; i += 256) {
            const int y = i / s0.w, x = i - y * s0.w;
            cur[i] = slot[s0.off + (size_t)y * s0.pitch + x];
        }
    }
    __syncthreads();
    for (int L = first; L < g.n_levels; ++L) {
        const LevelGeom src = g.lv[L - 1], dst = g.lv[L];
        for (int i = tid; i < dst.w * dst.h; i += 256) {
            const int dy = i / dst.w, dx = i - dy * dst.w;
            int acc = 0;
#pragma unroll
            for (int ky = 0; ky < 5; ++ky) {
                const uint8_t* row = cur + reflect101(2 * dy + ky - 2, src.h) * src.w;
                const int wy = (ky == 0 || ky == 4) ? 1 : (ky == 2 ? 6 : 4);
                const int hsum = row[reflect101(2 * dx - 2, src.w)] + 4 * row[reflect101(2 * dx - 1, src.w)] + 6 * row[2 * dx] +
                                 4 * row[reflect101(2 * dx + 1, src.w)] + row[reflect101(2 * dx + 2, src.w)];
                acc += wy * hsum;
            }
            const uint8_t v = (uint8_t)((acc + 128) >> 8);
            nxt[i] = v;
            slot[dst.off + (size_t)dy * dst.pitch + dx] = v;
        }
        __syncthreads();
        uint8_t* t = cur;
        cur = nxt;
        nxt = t;
    }
}

// cv::cvtColor(BGR2GRAY), 4 pixels per thread
__global__ void __launch_bounds__(256) bgr2gray_kernel(const uint8_t* __restrict__ bgr, size_t bgr_frame_stride,
                                                       uint8_t* __restrict__ pyr, size_t slot_stride, int first_slot,
                                                       LevelGeom l0) {
    const int quads_per_row = (l0.w + 3) / 4;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= quads_per_row * l0.h) return;
    const int y = q / quads_per_row, x = (q - y * quads_per_row) * 4;
    const uint8_t* in = bgr + (size_t)blockIdx.y * bgr_frame_stride + ((size_t)y * l0.w + x) * 3;
    uint8_t* out = pyr + (size_t)(first_slot + blockIdx.y) * slot_stride + l0.off + (size_t)y * l0.pitch + x;
    for (int j = 0; j < 4 && x + j < l0.w; ++j) {
        const int b = in[3 * j], g = in[3 * j + 1], r = in[3 * j + 2];
        out[j] = (uint8_t)((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15);
    }
}

}  // namespace

int launch_pyramid(ygzb_frames* f, int first, int count, const uint8_t* d_bgr) {
    ygzb_ctx* ctx = f->ctx;
    const Geometry& g = ctx->geo;
    if (count <= 0) return YGZB_OK;
    if (d_bgr) {
        const int quads = ((g.lv[0].w + 3) / 4) * g.lv[0].h;
        dim3 grid((quads + 255) / 256, count);
        ProfScope ps(ctx, kStageBgr2Gray);
        bgr2gray_kernel<<<grid, 256, 0, ctx->stream>>>(d_bgr, (size_t)g.lv[0].w * g.lv[0].h * 3, f->d_pyr,
                                                       ctx->slot_stride, first, g.lv[0]);
        YGZB_LAUNCHED(ctx);
    }
    // big levels: one tiled launch each; the small tail (source level <= kTailBytes): one CTA per frame for all of them
    int tail = g.n_levels;
    for (int L = 1; L < g.n_levels; ++L)
        if (g.lv[L - 1].w * g.lv[L - 1].h <= kTailBytes) {
            tail = L;
            break;
        }
    for (int L = 1; L < tail; ++L) {
        ProfScope ps(ctx, kStagePyrDown);
        if (g.lv[L - 1].w % 8 == 0 && g.lv[L - 1].w >= 16 && g.lv[L - 1].h >= 4) {
            const int strips = (g.lv[L].h + kStripRows - 1) / kStripRows;
            dim3 grid((strips * (g.lv[L - 1].w / 8) + 255) / 256, count);
            pyrdown_stream_kernel<<<grid, 256, 0, ctx->stream>>>(f->d_pyr, ctx->slot_stride, first, g.lv[L - 1], g.lv[L], strips);
        } else {
            dim3 grid((g.lv[L].w + kDW - 1) / kDW, (g.lv[L].h + kDH - 1) / kDH, count);
            pyrdown_kernel<<<grid, 256, 0, ctx->stream>>>(f->d_pyr, ctx->slot_stride, first, g.lv[L - 1], g.lv[L]);
        }
        YGZB_LAUNCHED(ctx);
    }
    if (tail < g.n_levels) {
        ProfScope ps(ctx, kStagePyrDown);
        pyrdown_tail_kernel<<<count, 256, 0, ctx->stream>>>(f->d_pyr, ctx->slot_stride, first, g, tail);
        YGZB_LAUNCHED(ctx);
    }
    return YGZB_OK;
}

int launch_pyrdown_ptrs(ygzb_ctx* ctx, const uint8_t* const* d_src_ptr, uint8_t* const* d_dst_ptr, int sw, int sh, int spitch,
                        int dw, int dh, int dpitch, int count) {
    if (count <= 0) return YGZB_OK;
    const LevelGeom src{sw, sh, spitch, 0}, dst{dw, dh, dpitch, 0};
    // one image per gridDim.z index, which is limited to 65,535: larger batches (KLT with > 32,767 pairs) go in chunks
    constexpr int kMaxGridZ = 65535;
    for (int first = 0; first < count; first += kMaxGridZ) {
        dim3 grid((dw + kDW - 1) / kDW, (dh + kDH - 1) / kDH, std::min(count - first, kMaxGridZ));
        ProfScope ps(ctx, kStagePyrDown);
        pyrdown_ptr_kernel<<<grid, 256, 0, ctx->stream>>>(d_src_ptr + first, d_dst_ptr + first, src, dst);
        YGZB_LAUNCHED(ctx);
    }
    return YGZB_OK;
}

}  // namespace ygzb
