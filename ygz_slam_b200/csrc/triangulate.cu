// triangulate.cu -- the matching / geometry kernels behind LocalMapping::CreateNewMapPoints (SURVEY.md 8f row 1):
//   Matcher::SearchForTriangulation        reference src/Algorithm/Matcher.cpp:86-193
//   Matcher::CheckDistEpipolarLine         reference src/Algorithm/Matcher.cpp:338-354
//   cvutils::DepthFromTriangulation        reference include/ygz/Algorithm/CVUtils.h:18-38
// SearchForTriangulation walks the DBoW3 feature vectors of two key-frames (vocabulary node -> feature indices) and
// matches, inside every common node, each feature of key-frame 1 against the features of key-frame 2 by Hamming distance
// under the epipolar constraint.  Here the feature vectors arrive as ONE NODE ID PER FEATURE (-1 = the feature is in no
// node); a thread owns a feature of key-frame 1 and scans the features of key-frame 2 in index order -- the order of a
// DBoW3 feature vector's index lists -- so the reference's tie rule (a later candidate of EQUAL distance replaces the
// earlier one, `dist > bestDist` skips) is kept and the result is index-exact.  The descriptors of key-frame 2 are staged
// through shared memory in chunks like the brute-force matcher (match.cu); the distance is 8 x POPC per candidate of the
// same node only.  Compiled with -fmad=false: the double sums behind the epipolar line and its distance, and the normal
// matrix, determinant and right-hand side of DepthFromTriangulation, are rounded after every operation as in the oracle.
// A fused multiply-add changes them in their last bits, which moves the `dsqr < th` and `det < det_th` decisions on
// boundary cases and the depths themselves.  The f32 steps also use explicit round-to-nearest intrinsics.
#include <exception>
#include <vector>

#include "common.cuh"
#include "se3.cuh"

namespace ygzb {
namespace {

constexpr int kChunk = 128;   // key-frame-2 features staged per pass

// Matcher::CheckDistEpipolarLine with pt = Pixel2Camera(px) (Camera.h:56-62: double maths on float intrinsics)
__device__ __forceinline__ bool epipolar_ok(double x1, double y1, double x2, double y2, const double* E, float th) {
    const float a = (float)(x1 * E[0] + y1 * E[3] + E[6]);
    const float b = (float)(x1 * E[1] + y1 * E[4] + E[7]);
    const float c = (float)(x1 * E[2] + y1 * E[5] + E[8]);
    // const float num = a * pt2[0] + b * pt2[1] + c: float * double promotes, the sum is rounded to float once
    const float num = (float)((double)a * x2 + (double)b * y2 + (double)c);
    const float den = __fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b));
    if (den < 1e-6) return false;   // (float compared with a double literal)
    const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
    return (double)fabsf(dsqr) < (double)th;
}

__global__ void __launch_bounds__(128) search_triangulation_kernel(const int32_t* __restrict__ off1, const int32_t* __restrict__ off2,
                                                                   const uint8_t* __restrict__ desc1, const double* __restrict__ px1,
                                                                   const int32_t* __restrict__ node1, const uint8_t* __restrict__ desc2,
                                                                   const double* __restrict__ px2, const int32_t* __restrict__ node2,
                                                                   const double* __restrict__ E12, float fx, float fy, float cx, float cy, int th_low,
                                                                   float epipolar_dsqr, int32_t* __restrict__ match12) {
    __shared__ uint4 s_desc[kChunk][2];
    __shared__ int s_node[kChunk];
    __shared__ double s_pt[kChunk][2];
    const int p = blockIdx.y, tid = threadIdx.x;
    const int a0 = off1[p], n1 = off1[p + 1] - a0, b0 = off2[p], n2 = off2[p + 1] - b0;
    const int i = blockIdx.x * blockDim.x + tid;
    const bool live = i < n1;
    uint4 d0 = make_uint4(0, 0, 0, 0), d1 = d0;
    int my_node = -1;
    double x1 = 0, y1 = 0;
    if (live) {
        const uint4* q = reinterpret_cast<const uint4*>(desc1) + 2 * (size_t)(a0 + i);
        d0 = q[0];
        d1 = q[1];
        my_node = node1[a0 + i];
        x1 = (px1[2 * (size_t)(a0 + i)] - cx) * 1.0 / fx;       // Pixel2Camera(p, depth = 1)
        y1 = (px1[2 * (size_t)(a0 + i) + 1] - cy) * 1.0 / fy;
    }
    const double* E = E12 + 9 * (size_t)p;
    int bestDist = 256, bestIdx = -1;
    for (int base = 0; base < n2; base += kChunk) {
        __syncthreads();
        for (int k = tid; k < kChunk && base + k < n2; k += blockDim.x) {
            const uint4* q = reinterpret_cast<const uint4*>(desc2) + 2 * (size_t)(b0 + base + k);
            s_desc[k][0] = q[0];
            s_desc[k][1] = q[1];
            s_node[k] = node2[b0 + base + k];
            s_pt[k][0] = (px2[2 * (size_t)(b0 + base + k)] - cx) * 1.0 / fx;
            s_pt[k][1] = (px2[2 * (size_t)(b0 + base + k) + 1] - cy) * 1.0 / fy;
        }
        __syncthreads();
        if (!live || my_node < 0) continue;
        const int m = min(kChunk, n2 - base);
        for (int k = 0; k < m; ++k) {
            if (s_node[k] != my_node) continue;
            const uint4 e0 = s_desc[k][0], e1 = s_desc[k][1];
            const int dist = __popc(d0.x ^ e0.x) + __popc(d0.y ^ e0.y) + __popc(d0.z ^ e0.z) + __popc(d0.w ^ e0.w) + __popc(d1.x ^ e1.x) +
                             __popc(d1.y ^ e1.y) + __popc(d1.z ^ e1.z) + __popc(d1.w ^ e1.w);
            if (dist > th_low || dist > bestDist) continue;
            if (epipolar_ok(x1, y1, s_pt[k][0], s_pt[k][1], E, epipolar_dsqr)) {
                bestIdx = base + k;
                bestDist = dist;
            }
        }
    }
    if (live) match12[a0 + i] = bestIdx;
}

__global__ void depth_from_triangulation_kernel(int n, const double* __restrict__ T, const int32_t* __restrict__ pose_of,
                                                const double* __restrict__ f_ref, const double* __restrict__ f_cur, double det_th,
                                                double* __restrict__ depth1, double* __restrict__ depth2, uint8_t* __restrict__ ok) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* M = T + 12 * (size_t)(pose_of ? pose_of[i] : 0);
    const double fr[3] = {f_ref[3 * (size_t)i], f_ref[3 * (size_t)i + 1], f_ref[3 * (size_t)i + 2]};
    // A = [R f_ref, -f_cur] (3 x 2)
    double a0[3], a1[3];
    for (int r = 0; r < 3; ++r) {
        a0[r] = M[4 * r] * fr[0] + M[4 * r + 1] * fr[1] + M[4 * r + 2] * fr[2];
        a1[r] = -f_cur[3 * (size_t)i + r];
    }
    const double m00 = a0[0] * a0[0] + a0[1] * a0[1] + a0[2] * a0[2], m01 = a0[0] * a1[0] + a0[1] * a1[1] + a0[2] * a1[2],
                 m11 = a1[0] * a1[0] + a1[1] * a1[1] + a1[2] * a1[2];
    const double det = m00 * m11 - m01 * m01;
    depth1[i] = depth2[i] = 0;
    if (det < det_th) {
        ok[i] = 0;
        return;
    }
    // depth = -(A^T A)^-1 A^T t   (Eigen's 2x2 inverse: adjugate / determinant)
    const double t0 = M[3], t1 = M[7], t2 = M[11];
    const double b0 = a0[0] * t0 + a0[1] * t1 + a0[2] * t2, b1 = a1[0] * t0 + a1[1] * t1 + a1[2] * t2;
    const double id = 1.0 / det;
    const double i00 = m11 * id, i01 = -m01 * id, i11 = m00 * id;
    depth1[i] = fabs(-(i00 * b0 + i01 * b1));
    depth2[i] = fabs(-(i01 * b0 + i11 * b1));
    ok[i] = 1;
}

}  // namespace
}  // namespace ygzb

using namespace ygzb;

extern "C" {

int ygzb_search_for_triangulation(ygzb_ctx* ctx, int n_pairs, const int32_t* off1, const int32_t* off2, const uint8_t* desc1,
                                  const double* px1, const int32_t* node1, const uint8_t* desc2, const double* px2, const int32_t* node2,
                                  const double* E12, int th_low, double epipolar_dsqr, int32_t* match12) {
    if (!ctx || n_pairs < 1 || !off1 || !off2 || !E12) return YGZB_ERR_INVALID;
    cudaSetDevice(ctx->device);
    int rc = check_offsets(ctx, off1, n_pairs, "off1");
    if (rc == YGZB_OK) rc = check_offsets(ctx, off2, n_pairs, "off2");
    if (rc != YGZB_OK) return rc;
    const size_t P = (size_t)n_pairs, N1 = (size_t)off1[n_pairs], N2 = (size_t)off2[n_pairs];
    if (N1 == 0) return YGZB_OK;
    if (!desc1 || !px1 || !node1 || !match12 || (N2 && (!desc2 || !px2 || !node2))) return YGZB_ERR_INVALID;
    int max1 = 0;
    for (size_t p = 0; p < P; ++p) max1 = std::max(max1, off1[p + 1] - off1[p]);
    int32_t *d_off, *d_n1, *d_n2, *d_m;
    double *d_E, *d_p1, *d_p2;
    uint8_t *d_d1, *d_d2;
    void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
        d_off = c.take<int32_t>(2 * (P + 1));
        d_E = c.take<double>(9 * P);
        d_d1 = c.take<uint8_t>(32 * N1);
        d_d2 = c.take<uint8_t>(32 * N2 + 32);
        d_p1 = c.take<double>(2 * N1);
        d_p2 = c.take<double>(2 * N2 + 2);
        d_n1 = c.take<int32_t>(N1);
        d_n2 = c.take<int32_t>(N2 + 1);
        d_m = c.take<int32_t>(N1);
    });
    if (!buf) return YGZB_ERR_CUDA;
    auto H2D = [&](void* dst, const void* src, size_t bytes) {
        return bytes ? check_cuda(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream), "H2D") : YGZB_OK;
    };
    if ((rc = H2D(d_off, off1, (P + 1) * 4)) || (rc = H2D(d_off + P + 1, off2, (P + 1) * 4)) || (rc = H2D(d_E, E12, 9 * P * 8)) ||
        (rc = H2D(d_d1, desc1, 32 * N1)) || (rc = H2D(d_d2, desc2, 32 * N2)) || (rc = H2D(d_p1, px1, 16 * N1)) || (rc = H2D(d_p2, px2, 16 * N2)) ||
        (rc = H2D(d_n1, node1, 4 * N1)) || (rc = H2D(d_n2, node2, 4 * N2)))
        return rc;
    {
        ProfScope ps(ctx, kStageMatch);
        const dim3 grid((unsigned)((max1 + 127) / 128), (unsigned)P);
        search_triangulation_kernel<<<grid, 128, 0, ctx->stream>>>(d_off, d_off + P + 1, d_d1, d_p1, d_n1, d_d2, d_p2, d_n2, d_E, ctx->prm.fx,
                                                                  ctx->prm.fy, ctx->prm.cx, ctx->prm.cy, th_low, (float)epipolar_dsqr, d_m);
        YGZB_LAUNCHED(ctx);
    }
    YGZB_CUDA(ctx, cudaMemcpyAsync(match12, d_m, 4 * N1, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

int ygzb_depth_from_triangulation(ygzb_ctx* ctx, int n, int n_poses, const double* T_search_ref, const int32_t* pose_of, const double* f_ref,
                                  const double* f_cur, double determinant_th, double* depth1, double* depth2, uint8_t* ok) {
    if (!ctx || n < 0 || n_poses < 1 || !T_search_ref) return YGZB_ERR_INVALID;
    if (n == 0) return YGZB_OK;
    if (!f_ref || !f_cur || !depth1 || !depth2 || !ok || (n_poses > 1 && !pose_of)) return YGZB_ERR_INVALID;
    cudaSetDevice(ctx->device);
    if (pose_of)
        for (int i = 0; i < n; ++i)
            if (pose_of[i] < 0 || pose_of[i] >= n_poses) return set_error(ctx, YGZB_ERR_INVALID, "pose_of[%d] out of range", i);
    const size_t N = (size_t)n, P = (size_t)n_poses;
    double *d_T, *d_fr, *d_fc, *d_d1, *d_d2;
    int32_t* d_po;
    uint8_t* d_ok;
    void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
        d_T = c.take<double>(12 * P);
        d_po = c.take<int32_t>(N);
        d_fr = c.take<double>(3 * N);
        d_fc = c.take<double>(3 * N);
        d_d1 = c.take<double>(N);
        d_d2 = c.take<double>(N);
        d_ok = c.take<uint8_t>(N);
    });
    if (!buf) return YGZB_ERR_CUDA;
    YGZB_CUDA(ctx, cudaMemcpyAsync(d_T, T_search_ref, 12 * P * 8, cudaMemcpyHostToDevice, ctx->stream));
    if (pose_of) YGZB_CUDA(ctx, cudaMemcpyAsync(d_po, pose_of, 4 * N, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(d_fr, f_ref, 24 * N, cudaMemcpyHostToDevice, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(d_fc, f_cur, 24 * N, cudaMemcpyHostToDevice, ctx->stream));
    {
        ProfScope ps(ctx, kStageOther);
        depth_from_triangulation_kernel<<<(unsigned)((N + 127) / 128), 128, 0, ctx->stream>>>(n, d_T, pose_of ? d_po : nullptr, d_fr, d_fc, determinant_th,
                                                                                          d_d1, d_d2, d_ok);
        YGZB_LAUNCHED(ctx);
    }
    YGZB_CUDA(ctx, cudaMemcpyAsync(depth1, d_d1, 8 * N, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(depth2, d_d2, 8 * N, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaMemcpyAsync(ok, d_ok, N, cudaMemcpyDeviceToHost, ctx->stream));
    YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return YGZB_OK;
}

}  // extern "C"
