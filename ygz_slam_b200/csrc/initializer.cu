// initializer.cu -- the RANSAC half of the monocular initialiser (SURVEY.md 8f row 4):
//   Initializer::FindHomography / Normalize / ComputeH21 / CheckHomography   reference src/Algorithm/Initializer.cpp:89-318
//   Initializer::FindFundamental / ComputeF21 / CheckFundamental             reference src/Algorithm/Initializer.cpp:670-853
// "200 hypotheses x N-point scoring is embarrassingly parallel": three kernels for a batch of point-pair lists --
//   init_normalize_kernel   per list: Normalize() of both images, T1, T2^-1, T2^T
//   init_models_kernel      ONE THREAD PER HYPOTHESIS (list, iteration, H or F): the 16 x 9 / 8 x 9 design matrix of the
//                           iteration's 8-point set, its null vector by a one-sided Jacobi SVD (working set in shared memory,
//                           element-major so the 64 threads of a CTA never conflict), the rank-2 projection for F, de-normalisation
//   init_score_kernel       ONE WARP PER HYPOTHESIS: the lanes evaluate CheckHomography / CheckFundamental for 32 points at a
//                           time; the float score is then accumulated IN POINT ORDER (shuffles, every lane keeps the same
//                           running sum), so it is the reference's sequential float sum bit for bit
//   init_select_kernel      per (list, model): the reference's `if (currentScore > score)` scan, the inlier flags of the winner
// Compiled without FMA contraction (build.py) and written operation by operation like oracle/initializer.cpp, whose header
// lists what is restated from third parties (cv::RNG sets are drawn by the caller; Eigen::JacobiSVD -> Hestenes Jacobi).
#include <algorithm>
#include <exception>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace ygzb {
namespace {

constexpr int kModelThreads = 64;
constexpr int kWork = 16 * 9 + 81;   // doubles of a hypothesis' Jacobi working set: A (up to 16 x 9) and V (9 x 9)

struct Norm {   // per list: the similarity transforms of Normalize()
    double T1[9], T2inv[9], T2t[9];
};

// element e of this thread's working set
#define WS(e) ws[(e) * kModelThreads + threadIdx.x]

// one-sided Jacobi SVD of the M x N matrix at WS(a0 + r * N + c); right vectors at WS(v0 + r * N + c)
template <int M, int N>
__device__ void jacobi_svd(double* ws, int a0, int v0) {
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < N; ++j) WS(v0 + i * N + j) = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 40; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < N - 1; ++p)
            for (int q = p + 1; q < N; ++q) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int r = 0; r < M; ++r) {
                    const double x = WS(a0 + r * N + p), y = WS(a0 + r * N + q);
                    alpha += x * x;
                    beta += y * y;
                    gamma += x * y;
                }
                if (gamma == 0.0 || fabs(gamma) <= 1e-15 * sqrt(alpha * beta)) continue;
                rotated = true;
                const double zeta = (beta - alpha) / (2.0 * gamma);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
                for (int r = 0; r < M; ++r) {
                    const double x = WS(a0 + r * N + p), y = WS(a0 + r * N + q);
                    WS(a0 + r * N + p) = c * x - s * y;
                    WS(a0 + r * N + q) = s * x + c * y;
                }
                for (int r = 0; r < N; ++r) {
                    const double x = WS(v0 + r * N + p), y = WS(v0 + r * N + q);
                    WS(v0 + r * N + p) = c * x - s * y;
                    WS(v0 + r * N + q) = s * x + c * y;
                }
            }
        if (!rotated) break;
    }
}

template <int M, int N>
__device__ int smallest_column(const double* ws, int a0) {
    int best = 0;
    double best2 = 0;
    for (int c = 0; c < N; ++c) {
        double n2 = 0;
        for (int r = 0; r < M; ++r) n2 += WS(a0 + r * N + c) * WS(a0 + r * N + c);
        if (c == 0 || n2 < best2) {
            best = c;
            best2 = n2;
        }
    }
    return best;
}

template <int M>
__device__ void null_vector(double* ws, double* out9) {
    jacobi_svd<M, 9>(ws, 0, 16 * 9);
    const int c = smallest_column<M, 9>(ws, 0);
    int big = 0;
    for (int r = 1; r < 9; ++r)
        if (fabs(WS(16 * 9 + r * 9 + c)) > fabs(WS(16 * 9 + big * 9 + c))) big = r;
    const double sg = WS(16 * 9 + big * 9 + c) < 0 ? -1.0 : 1.0;
    for (int r = 0; r < 9; ++r) out9[r] = sg * WS(16 * 9 + r * 9 + c);
}

__device__ __forceinline__ void mul3(const double* A, const double* B, double* C) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

__device__ __forceinline__ void inverse3(const double* m, double* inv) {
    const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
    const double id = 1.0 / det;
    inv[0] = c00 * id;
    inv[1] = (m[2] * m[7] - m[1] * m[8]) * id;
    inv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    inv[3] = c01 * id;
    inv[4] = (m[0] * m[8] - m[2] * m[6]) * id;
    inv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    inv[6] = c02 * id;
    inv[7] = (m[1] * m[6] - m[0] * m[7]) * id;
    inv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}

// Initializer::Normalize for both point lists of every pair: the sums run in point order on one thread (they are the
// reference's sequential double sums), the scaling of the points is parallel
__global__ void __launch_bounds__(256) init_normalize_kernel(const int32_t* __restrict__ off, const double* __restrict__ px1,
                                                             const double* __restrict__ px2, double* __restrict__ pn1, double* __restrict__ pn2,
                                                             Norm* __restrict__ norm) {
    __shared__ double s_mean[2][2];
    __shared__ float s_scale[2][2];
    const int p = blockIdx.x, a0 = off[p], n = off[p + 1] - a0;
    if (threadIdx.x < 2) {
        const double* px = (threadIdx.x == 0 ? px1 : px2) + 2 * (size_t)a0;
        double m0 = 0, m1 = 0;
        for (int i = 0; i < n; ++i) {
            m0 += px[2 * i];
            m1 += px[2 * i + 1];
        }
        m0 = m0 / n;
        m1 = m1 / n;
        double d0 = 0, d1 = 0;
        for (int i = 0; i < n; ++i) {
            d0 += fabs(px[2 * i] - m0);
            d1 += fabs(px[2 * i + 1] - m1);
        }
        d0 /= n;
        d1 /= n;
        s_mean[threadIdx.x][0] = m0;
        s_mean[threadIdx.x][1] = m1;
        s_scale[threadIdx.x][0] = (float)(1.0 / d0);
        s_scale[threadIdx.x][1] = (float)(1.0 / d1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        pn1[2 * (size_t)(a0 + i)] = (px1[2 * (size_t)(a0 + i)] - s_mean[0][0]) * s_scale[0][0];
        pn1[2 * (size_t)(a0 + i) + 1] = (px1[2 * (size_t)(a0 + i) + 1] - s_mean[0][1]) * s_scale[0][1];
        pn2[2 * (size_t)(a0 + i)] = (px2[2 * (size_t)(a0 + i)] - s_mean[1][0]) * s_scale[1][0];
        pn2[2 * (size_t)(a0 + i) + 1] = (px2[2 * (size_t)(a0 + i) + 1] - s_mean[1][1]) * s_scale[1][1];
    }
    if (threadIdx.x == 0) {
        const float sX1 = s_scale[0][0], sY1 = s_scale[0][1], sX2 = s_scale[1][0], sY2 = s_scale[1][1];
        const double T1[9] = {sX1, 0, -s_mean[0][0] * sX1, 0, sY1, -s_mean[0][1] * sY1, 0, 0, 1};
        const double T2[9] = {sX2, 0, -s_mean[1][0] * sX2, 0, sY2, -s_mean[1][1] * sY2, 0, 0, 1};
        Norm o;
        for (int k = 0; k < 9; ++k) o.T1[k] = T1[k];
        inverse3(T2, o.T2inv);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) o.T2t[r * 3 + c] = T2[c * 3 + r];
        norm[p] = o;
    }
}

// hypothesis h = (list * max_iter + iteration) * 2 + model (0 = H, 1 = F); models[h] = H21i or F21i, aux[h] = H12i (H only)
__global__ void __launch_bounds__(kModelThreads) init_models_kernel(int n_hyp, int max_iter, const int32_t* __restrict__ off,
                                                                    const int32_t* __restrict__ sets, const double* __restrict__ pn1,
                                                                    const double* __restrict__ pn2, const Norm* __restrict__ norm,
                                                                    double* __restrict__ models, double* __restrict__ aux) {
    extern __shared__ double ws[];
    const int h = blockIdx.x * kModelThreads + threadIdx.x;
    if (h >= n_hyp) return;
    const int model = h & 1, pi = h >> 1, p = pi / max_iter, it = pi - p * max_iter;
    const int a0 = off[p];
    const int32_t* set = sets + ((size_t)p * max_iter + it) * 8;
    const Norm& nm = norm[p];
    double tmp[9], out[9];
    if (model == 0) {   // ComputeH21 (:196-239)
        for (int j = 0; j < 8; ++j) {
            const int idx = a0 + set[j];
            const double u1 = pn1[2 * (size_t)idx], v1 = pn1[2 * (size_t)idx + 1], u2 = pn2[2 * (size_t)idx], v2 = pn2[2 * (size_t)idx + 1];
            const int r0 = (2 * j) * 9, r1 = r0 + 9;
            WS(r0 + 0) = 0.0; WS(r0 + 1) = 0.0; WS(r0 + 2) = 0.0; WS(r0 + 3) = -u1; WS(r0 + 4) = -v1; WS(r0 + 5) = -1;
            WS(r0 + 6) = v2 * u1; WS(r0 + 7) = v2 * v1; WS(r0 + 8) = v2;
            WS(r1 + 0) = u1; WS(r1 + 1) = v1; WS(r1 + 2) = 1; WS(r1 + 3) = 0.0; WS(r1 + 4) = 0.0; WS(r1 + 5) = 0.0;
            WS(r1 + 6) = -u2 * u1; WS(r1 + 7) = -u2 * v1; WS(r1 + 8) = -u2;
        }
        double Hn[9];
        null_vector<16>(ws, Hn);
        mul3(nm.T2inv, Hn, tmp);
        mul3(tmp, nm.T1, out);
        double H12[9];
        inverse3(out, H12);
        for (int k = 0; k < 9; ++k) aux[9 * (size_t)h + k] = H12[k];
    } else {            // ComputeF21 (:730-762)
        for (int j = 0; j < 8; ++j) {
            const int idx = a0 + set[j];
            const double u1 = pn1[2 * (size_t)idx], v1 = pn1[2 * (size_t)idx + 1], u2 = pn2[2 * (size_t)idx], v2 = pn2[2 * (size_t)idx + 1];
            const int r = j * 9;
            WS(r + 0) = u2 * u1; WS(r + 1) = u2 * v1; WS(r + 2) = u2; WS(r + 3) = v2 * u1; WS(r + 4) = v2 * v1; WS(r + 5) = v2;
            WS(r + 6) = u1; WS(r + 7) = v1; WS(r + 8) = 1;
        }
        double Fpre[9], Fn[9];
        null_vector<8>(ws, Fpre);
        // rank 2: the 3 x 3 SVD in the same working set (A at 0, V at 9)
        for (int k = 0; k < 9; ++k) WS(k) = Fpre[k];
        jacobi_svd<3, 3>(ws, 0, 9);
        const int cz = smallest_column<3, 3>(ws, 0);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) Fn[r * 3 + c] = Fpre[r * 3 + c] - WS(r * 3 + cz) * WS(9 + c * 3 + cz);
        mul3(nm.T2t, Fn, tmp);
        mul3(tmp, nm.T1, out);
    }
    for (int k = 0; k < 9; ++k) models[9 * (size_t)h + k] = out[k];
}

// per-point terms of CheckHomography (:284-313): chi <= th ? th - chi : (not an inlier)
__device__ __forceinline__ bool homography_term(const double* H12, double u1, double v1, double u2, double v2, float invSigmaSquare, float* add) {
    const float th = 5.991f;
    const float w2in1inv = (float)(1.0 / (H12[6] * u2 + H12[7] * v2 + H12[8]));
    const float u2in1 = (float)((H12[0] * u2 + H12[1] * v2 + H12[2]) * w2in1inv);
    const float v2in1 = (float)((H12[3] * u2 + H12[4] * v2 + H12[5]) * w2in1inv);
    const float squareDist1 = (float)((u1 - u2in1) * (u1 - u2in1) + (v1 - v2in1) * (v1 - v2in1));
    const float chiSquare1 = squareDist1 * invSigmaSquare;
    *add = th - chiSquare1;
    return !(chiSquare1 > th);
}

// per-point terms of CheckFundamental (:798-850): two conditional additions, in this order
__device__ __forceinline__ void fundamental_terms(const float* f, float u1, float v1, float u2, float v2, float invSigmaSquare, bool* ok1,
                                                  float* add1, bool* ok2, float* add2) {
    const float th = 3.841f, thScore = 5.991f;
    const float a2 = f[0] * u1 + f[1] * v1 + f[2], b2 = f[3] * u1 + f[4] * v1 + f[5], c2 = f[6] * u1 + f[7] * v1 + f[8];
    const float num2 = a2 * u2 + b2 * v2 + c2;
    const float squareDist1 = num2 * num2 / (a2 * a2 + b2 * b2);
    const float chiSquare1 = squareDist1 * invSigmaSquare;
    *ok1 = !(chiSquare1 > th);
    *add1 = thScore - chiSquare1;
    const float a1 = f[0] * u2 + f[3] * v2 + f[6], b1 = f[1] * u2 + f[4] * v2 + f[7], c1 = f[2] * u2 + f[5] * v2 + f[8];
    const float num1 = a1 * u1 + b1 * v1 + c1;
    const float squareDist2 = num1 * num1 / (a1 * a1 + b1 * b1);
    const float chiSquare2 = squareDist2 * invSigmaSquare;
    *ok2 = !(chiSquare2 > th);
    *add2 = thScore - chiSquare2;
}

__global__ void __launch_bounds__(128) init_score_kernel(int n_hyp, int max_iter, const int32_t* __restrict__ off, const double* __restrict__ px1,
                                                         const double* __restrict__ px2, const double* __restrict__ models,
                                                         const double* __restrict__ aux, float sigma, float* __restrict__ scores) {
    const int h = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (h >= n_hyp) return;
    const int model = h & 1, p = (h >> 1) / max_iter;
    const int a0 = off[p], n = off[p + 1] - a0;
    const float invSigmaSquare = (float)(1.0 / (sigma * sigma));
    float score = 0;
    double M[9];
    float f[9];
    for (int k = 0; k < 9; ++k) {
        M[k] = model == 0 ? aux[9 * (size_t)h + k] : models[9 * (size_t)h + k];
        f[k] = (float)M[k];
    }
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        bool ok1 = false, ok2 = false;
        float add1 = 0, add2 = 0;
        if (i < n) {
            const double u1 = px1[2 * (size_t)(a0 + i)], v1 = px1[2 * (size_t)(a0 + i) + 1], u2 = px2[2 * (size_t)(a0 + i)],
                         v2 = px2[2 * (size_t)(a0 + i) + 1];
            if (model == 0) ok1 = homography_term(M, u1, v1, u2, v2, invSigmaSquare, &add1);
            else fundamental_terms(f, (float)u1, (float)v1, (float)u2, (float)v2, invSigmaSquare, &ok1, &add1, &ok2, &add2);
        }
        const unsigned m1 = __ballot_sync(0xFFFFFFFFu, ok1), m2 = __ballot_sync(0xFFFFFFFFu, ok2);
        const int cnt = min(32, n - base);
        for (int l = 0; l < cnt; ++l) {   // the reference's order: point by point, first term then second
            const float t1 = __shfl_sync(0xFFFFFFFFu, add1, l), t2 = __shfl_sync(0xFFFFFFFFu, add2, l);
            if (m1 >> l & 1) score += t1;
            if (m2 >> l & 1) score += t2;
        }
    }
    if (lane == 0) scores[h] = score;
}

// per (list, model): the winner of `if (currentScore > score)` over the iterations in order, its model and inlier flags
__global__ void __launch_bounds__(128) init_select_kernel(int max_iter, const int32_t* __restrict__ off, const double* __restrict__ px1,
                                                          const double* __restrict__ px2, const double* __restrict__ models,
                                                          const double* __restrict__ aux, const float* __restrict__ scores, float sigma,
                                                          double* __restrict__ out_model, float* __restrict__ out_score,
                                                          int32_t* __restrict__ out_best, uint8_t* __restrict__ inl_H, uint8_t* __restrict__ inl_F) {
    __shared__ int s_best;
    const int p = blockIdx.x, model = blockIdx.y;
    const int a0 = off[p], n = off[p + 1] - a0;
    if (threadIdx.x == 0) {
        float score = 0;
        int best = -1;
        for (int it = 0; it < max_iter; ++it) {
            const float s = scores[((size_t)p * max_iter + it) * 2 + model];
            if (s > score) {
                score = s;
                best = it;
            }
        }
        s_best = best;
        out_score[2 * p + model] = score;
        out_best[2 * p + model] = best;
    }
    __syncthreads();
    const int best = s_best;
    uint8_t* inl = (model == 0 ? inl_H : inl_F) + a0;
    if (best < 0) {
        if (threadIdx.x < 9) out_model[(2 * (size_t)p + model) * 9 + threadIdx.x] = 0.0;
        for (int i = threadIdx.x; i < n; i += blockDim.x) inl[i] = 0;
        return;
    }
    const size_t h = ((size_t)p * max_iter + best) * 2 + model;
    if (threadIdx.x < 9) out_model[(2 * (size_t)p + model) * 9 + threadIdx.x] = models[9 * h + threadIdx.x];
    const float invSigmaSquare = (float)(1.0 / (sigma * sigma));
    double M[9];
    float f[9];
    for (int k = 0; k < 9; ++k) {
        M[k] = model == 0 ? aux[9 * h + k] : models[9 * h + k];
        f[k] = (float)M[k];
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double u1 = px1[2 * (size_t)(a0 + i)], v1 = px1[2 * (size_t)(a0 + i) + 1], u2 = px2[2 * (size_t)(a0 + i)], v2 = px2[2 * (size_t)(a0 + i) + 1];
        bool ok1, ok2 = true;
        float a1, a2;
        if (model == 0) ok1 = homography_term(M, u1, v1, u2, v2, invSigmaSquare, &a1);
        else fundamental_terms(f, (float)u1, (float)v1, (float)u2, (float)v2, invSigmaSquare, &ok1, &a1, &ok2, &a2);
        inl[i] = (ok1 && ok2) ? 1 : 0;
    }
}

// =====================================================================================================================
// Second half: Initializer::ReconstructH / ReconstructF with CheckRT, Triangulate, DecomposeE (Initializer.cpp:330-675, 855-963).
// One CTA per list: thread 0 decomposes the model into its pose candidates (eight for H, four for F; 3 x 3 SVDs -- a few
// hundred operations), then ALL threads run CheckRT for every candidate over the point pairs (a 4 x 4 SVD per pair and
// candidate: the parallel part), the block selects the 51st smallest parallax cosine by repeated minimum extraction (a k-th
// element is order-free, unlike the reference's sort it needs no staging), and thread 0 takes the reference's decisions.
// Same operation order as oracle/initializer.cpp, no FMA contraction: poses, points, flags and counts are bit-exact; only
// acosf() may differ from glibc's in the last bit (parallax in degrees, compared with a tolerance).

template <int M, int N>
__device__ void jacobi_svd_local(double* a, double* v) {
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < N; ++j) v[i * N + j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 40; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < N - 1; ++p)
            for (int q = p + 1; q < N; ++q) {
                double alpha = 0, beta = 0, gamma = 0;
                for (int r = 0; r < M; ++r) {
                    const double x = a[r * N + p], y = a[r * N + q];
                    alpha += x * x;
                    beta += y * y;
                    gamma += x * y;
                }
                if (gamma == 0.0 || fabs(gamma) <= 1e-15 * sqrt(alpha * beta)) continue;
                rotated = true;
                const double zeta = (beta - alpha) / (2.0 * gamma);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
                for (int r = 0; r < M; ++r) {
                    const double x = a[r * N + p], y = a[r * N + q];
                    a[r * N + p] = c * x - s * y;
                    a[r * N + q] = s * x + c * y;
                }
                for (int r = 0; r < N; ++r) {
                    const double x = v[r * N + p], y = v[r * N + q];
                    v[r * N + p] = c * x - s * y;
                    v[r * N + q] = s * x + c * y;
                }
            }
        if (!rotated) break;
    }
}

struct Svd3 {
    double U[9], V[9], s[3];
};

__device__ void svd3_sorted(const double* A, Svd3* r) {
    double a[9], v[9], n2[3];
    for (int k = 0; k < 9; ++k) a[k] = A[k];
    jacobi_svd_local<3, 3>(a, v);
    for (int c = 0; c < 3; ++c) n2[c] = a[c] * a[c] + a[3 + c] * a[3 + c] + a[6 + c] * a[6 + c];
    int ord[3] = {0, 1, 2};
    for (int i = 0; i < 2; ++i)
        for (int j = i + 1; j < 3; ++j)
            if (n2[ord[j]] > n2[ord[i]]) {
                const int t = ord[i];
                ord[i] = ord[j];
                ord[j] = t;
            }
    for (int c = 0; c < 3; ++c) {
        const int o = ord[c];
        r->s[c] = sqrt(n2[o]);
        for (int k = 0; k < 3; ++k) r->V[k * 3 + c] = v[k * 3 + o];
    }
    for (int c = 0; c < 3; ++c) {
        const int o = ord[c];
        if (c < 2 || r->s[2] > 1e-12 * r->s[0]) {
            for (int k = 0; k < 3; ++k) r->U[k * 3 + c] = a[k * 3 + o] / r->s[c];
        } else {
            r->U[2] = r->U[3] * r->U[7] - r->U[6] * r->U[4];
            r->U[5] = r->U[6] * r->U[1] - r->U[0] * r->U[7];
            r->U[8] = r->U[0] * r->U[4] - r->U[3] * r->U[1];
        }
    }
}

__device__ __forceinline__ double det3(const double* m) {
    return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

__device__ __forceinline__ void transpose3(const double* A, double* T) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) T[r * 3 + c] = A[c * 3 + r];
}

__device__ void mat_R(const double* U, double s, const double* Rp, const double* V, double* R) {   // (s U) Rp V^T
    double sU[9], t1[9], Vt[9];
    for (int k = 0; k < 9; ++k) sU[k] = s * U[k];
    mul3(sU, Rp, t1);
    transpose3(V, Vt);
    mul3(t1, Vt, R);
}

struct ReconArgs {
    const int32_t* off;
    const double *px1, *px2;
    const int32_t* use_h;
    const double* model;       // [lists][9]
    const uint8_t* inliers;    // [N]
    double K[4];               // fx fy cx cy (the camera's float intrinsics)
    float sigma2, min_parallax;
    int min_triangulated;
    double ratio_h;
    // scratch: per candidate
    double* p3d_all;           // [8][3 N]
    uint8_t* good_all;         // [8][N]
    float* cos_all;            // [8][N]; NaN = the point was not counted
    size_t n_total;
    // out
    int32_t* ok;               // [lists]
    double *R21, *t21;         // [lists][9], [lists][3]
    double* p3d;               // [3 N]
    uint8_t* triangulated;     // [N]
    int32_t* n_good;           // [lists][8]
    double* parallax;          // [lists]
    double* candidates;        // [lists][8][12] or null
};

__device__ __forceinline__ unsigned long long cos_key(float v, int i) {   // total order of (value, index)
    unsigned u = __float_as_uint(v);
    u ^= (u >> 31) ? 0xFFFFFFFFu : 0x80000000u;
    return ((unsigned long long)u << 32) | (unsigned)i;
}

__global__ void __launch_bounds__(256) init_reconstruct_kernel(const ReconArgs a) {
    __shared__ double s_R[8][9], s_t[8][3];
    __shared__ int s_ncand, s_N, s_cnt[8];
    __shared__ float s_cosk[8];
    __shared__ unsigned long long s_min[8];
    __shared__ int s_best, s_ok;
    const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int a0 = a.off[p], n = a.off[p + 1] - a0;
    const double fx = a.K[0], fy = a.K[1], cx = a.K[2], cy = a.K[3];
    const bool use_h = a.use_h[p] != 0;
    if (tid < 8) s_cnt[tid] = 0;
    if (tid == 0) {
        int N = 0;
        for (int i = 0; i < n; ++i) N += a.inliers[a0 + i] ? 1 : 0;
        s_N = N;
        const double Km[9] = {fx, 0, cx, 0, fy, cy, 0, 0, 1};
        const double* model = a.model + 9 * (size_t)p;
        int ncand = 0;
        if (use_h) {
            double invK[9], t1[9], A[9];
            inverse3(Km, invK);
            mul3(invK, model, t1);
            mul3(t1, Km, A);
            Svd3 sv;
            svd3_sorted(A, &sv);
            const double d1 = sv.s[0], d2 = sv.s[1], d3 = sv.s[2];
            const double s = det3(sv.U) * det3(sv.V);
            if (!(d1 / d2 < 1.00001 || d2 / d3 < 1.00001)) {
                const float aux1 = (float)sqrt((d1 * d1 - d2 * d2) / (d1 * d1 - d3 * d3));
                const float aux3 = (float)sqrt((d2 * d2 - d3 * d3) / (d1 * d1 - d3 * d3));
                const float x1[4] = {aux1, aux1, -aux1, -aux1}, x3[4] = {aux3, -aux3, aux3, -aux3};
                const float aux_stheta = (float)(sqrt((d1 * d1 - d2 * d2) * (d2 * d2 - d3 * d3)) / ((d1 + d3) * d2));
                const float ctheta = (float)((d2 * d2 + d1 * d3) / ((d1 + d3) * d2));
                const float stheta[4] = {aux_stheta, -aux_stheta, -aux_stheta, aux_stheta};
                for (int i = 0; i < 4; ++i) {
                    const double Rp[9] = {ctheta, 0, -stheta[i], 0, 1, 0, stheta[i], 0, ctheta};
                    mat_R(sv.U, s, Rp, sv.V, s_R[i]);
                    const double tp[3] = {x1[i] * (d1 - d3), 0.0 * (d1 - d3), -x3[i] * (d1 - d3)};
                    double tt[3];
                    for (int r = 0; r < 3; ++r) tt[r] = sv.U[r * 3] * tp[0] + sv.U[r * 3 + 1] * tp[1] + sv.U[r * 3 + 2] * tp[2];
                    const double nn = sqrt(tt[0] * tt[0] + tt[1] * tt[1] + tt[2] * tt[2]);
                    for (int r = 0; r < 3; ++r) s_t[i][r] = tt[r] / nn;
                }
                const float aux_sphi = (float)(sqrt((d1 * d1 - d2 * d2) * (d2 * d2 - d3 * d3)) / ((d1 - d3) * d2));
                const float cphi = (float)((d1 * d3 - d2 * d2) / ((d1 - d3) * d2));
                const float sphi[4] = {aux_sphi, -aux_sphi, -aux_sphi, aux_sphi};
                for (int i = 0; i < 4; ++i) {
                    const double Rp[9] = {cphi, 0, sphi[i], 0, -1, 0, sphi[i], 0, -cphi};
                    mat_R(sv.U, s, Rp, sv.V, s_R[4 + i]);
                    const double tp[3] = {x1[i] * (d1 + d3), 0.0 * (d1 + d3), x3[i] * (d1 + d3)};
                    double tt[3];
                    for (int r = 0; r < 3; ++r) tt[r] = sv.U[r * 3] * tp[0] + sv.U[r * 3 + 1] * tp[1] + sv.U[r * 3 + 2] * tp[2];
                    const double nn = sqrt(tt[0] * tt[0] + tt[1] * tt[1] + tt[2] * tt[2]);
                    for (int r = 0; r < 3; ++r) s_t[4 + i][r] = tt[r] / nn;
                }
                ncand = 8;
            }
        } else {
            double Kt[9], t1[9], E[9];
            transpose3(Km, Kt);
            mul3(Kt, model, t1);
            mul3(t1, Km, E);
            Svd3 sv;
            svd3_sorted(E, &sv);
            double tv[3] = {sv.U[2], sv.U[5], sv.U[8]};
            {
                const double nn = sqrt(tv[0] * tv[0] + tv[1] * tv[1] + tv[2] * tv[2]);
                for (int r = 0; r < 3; ++r) tv[r] = tv[r] / nn;
            }
            const double W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1}, Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
            double Vt[9], R1[9], R2[9];
            transpose3(sv.V, Vt);
            mul3(sv.U, W, t1);
            mul3(t1, Vt, R1);
            if (det3(R1) < 0)
                for (int k = 0; k < 9; ++k) R1[k] = -R1[k];
            mul3(sv.U, Wt, t1);
            mul3(t1, Vt, R2);
            if (det3(R2) < 0)
                for (int k = 0; k < 9; ++k) R2[k] = -R2[k];
            for (int i = 0; i < 4; ++i) {
                const double* Rc = (i & 1) ? R2 : R1;
                for (int k = 0; k < 9; ++k) s_R[i][k] = Rc[k];
                for (int r = 0; r < 3; ++r) s_t[i][r] = i < 2 ? tv[r] : -tv[r];
            }
            ncand = 4;
        }
        s_ncand = ncand;
        if (a.candidates)
            for (int i = 0; i < 8; ++i)
                for (int k = 0; k < 12; ++k)
                    a.candidates[(8 * (size_t)p + i) * 12 + k] = i < ncand ? (k < 9 ? s_R[i][k] : s_t[i][k - 9]) : 0.0;
    }
    __syncthreads();
    const int ncand = s_ncand;
    const float th2 = use_h ? 4.0f * a.sigma2 : 24.0f * a.sigma2;
    // ---- CheckRT of every candidate
    for (int h = 0; h < ncand; ++h) {
        const double* R = s_R[h];
        const double* t = s_t[h];
        const double P1[12] = {fx, 0, cx, 0, 0, fy, cy, 0, 0, 0, 1, 0};
        const double Rt[12] = {R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2]};
        double P2[12];
        for (int c = 0; c < 4; ++c) {
            P2[c] = fx * Rt[c] + 0.0 * Rt[4 + c] + cx * Rt[8 + c];
            P2[4 + c] = 0.0 * Rt[c] + fy * Rt[4 + c] + cy * Rt[8 + c];
            P2[8 + c] = 0.0 * Rt[c] + 0.0 * Rt[4 + c] + 1.0 * Rt[8 + c];
        }
        const double O2[3] = {-(R[0] * t[0] + R[3] * t[1] + R[6] * t[2]), -(R[1] * t[0] + R[4] * t[1] + R[7] * t[2]),
                              -(R[2] * t[0] + R[5] * t[1] + R[8] * t[2])};
        double* p3d = a.p3d_all + 3 * ((size_t)h * a.n_total + a0);
        uint8_t* good = a.good_all + (size_t)h * a.n_total + a0;
        float* cosv = a.cos_all + (size_t)h * a.n_total + a0;
        int cnt = 0;
        for (int i = tid; i < n; i += blockDim.x) {
            good[i] = 0;
            p3d[3 * i] = p3d[3 * i + 1] = p3d[3 * i + 2] = 0;
            cosv[i] = __int_as_float(0x7FC00000);
            const double* kp1 = a.px1 + 2 * (size_t)(a0 + i);
            const double* kp2 = a.px2 + 2 * (size_t)(a0 + i);
            double A[16], v[16], X[3];
            for (int c = 0; c < 4; ++c) {
                A[c] = kp1[0] * P1[8 + c] - P1[c];
                A[4 + c] = kp1[1] * P1[8 + c] - P1[4 + c];
                A[8 + c] = kp2[0] * P2[8 + c] - P2[c];
                A[12 + c] = kp2[1] * P2[8 + c] - P2[4 + c];
            }
            jacobi_svd_local<4, 4>(A, v);
            int cs = 0;
            double best2 = 0;
            for (int c = 0; c < 4; ++c) {
                double n2 = 0;
                for (int r = 0; r < 4; ++r) n2 += A[r * 4 + c] * A[r * 4 + c];
                if (c == 0 || n2 < best2) {
                    cs = c;
                    best2 = n2;
                }
            }
            for (int k = 0; k < 3; ++k) X[k] = v[k * 4 + cs] / v[12 + cs];
            if (!isfinite(X[0])) continue;
            const double dist1 = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
            const double n2v[3] = {X[0] - O2[0], X[1] - O2[1], X[2] - O2[2]};
            const double dist2 = sqrt(n2v[0] * n2v[0] + n2v[1] * n2v[1] + n2v[2] * n2v[2]);
            const double cosParallax = (X[0] * n2v[0] + X[1] * n2v[1] + X[2] * n2v[2]) / (dist1 * dist2);
            if (X[2] < 0 && cosParallax < 0.99998) continue;
            const double Y[3] = {R[0] * X[0] + R[1] * X[1] + R[2] * X[2] + t[0], R[3] * X[0] + R[4] * X[1] + R[5] * X[2] + t[1],
                                 R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2]};
            if (Y[2] < 0 && cosParallax < 0.99998) continue;
            if (use_h) {   // ReconstructH checks the reprojection error, ReconstructF does not (:877-880)
                const double invZ1 = 1.0 / X[2];
                const double im1x = fx * X[0] * invZ1 + cx, im1y = fy * X[1] * invZ1 + cy;
                const double e1 = (im1x - kp1[0]) * (im1x - kp1[0]) + (im1y - kp1[1]) * (im1y - kp1[1]);
                if (e1 > th2) continue;
                const double invZ2 = 1.0 / Y[2];
                const double im2x = fx * Y[0] * invZ2 + cx, im2y = fy * Y[1] * invZ2 + cy;
                const double e2 = (im2x - kp2[0]) * (im2x - kp2[0]) + (im2y - kp2[1]) * (im2y - kp2[1]);
                if (e2 > th2) continue;
            }
            cosv[i] = (float)cosParallax;
            p3d[3 * i] = X[0];
            p3d[3 * i + 1] = X[1];
            p3d[3 * i + 2] = X[2];
            ++cnt;
            if (cosParallax < 0.99998) good[i] = 1;
        }
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_down_sync(0xFFFFFFFFu, cnt, o);
        if (lane == 0 && cnt) atomicAdd(&s_cnt[h], cnt);
        __syncthreads();
        // the (min(50, count - 1) + 1)-th smallest counted cosine: repeated extraction of the minimum above the last one
        const int total = s_cnt[h];
        if (total > 0) {
            const int idx = min(50, total - 1);
            unsigned long long last = 0;
            bool have_last = false;
            for (int round = 0; round <= idx; ++round) {
                unsigned long long mine = ~0ULL;
                for (int i = tid; i < n; i += blockDim.x) {
                    const float c = cosv[i];
                    if (c != c) continue;
                    const unsigned long long k = cos_key(c, i);
                    if ((!have_last || k > last) && k < mine) mine = k;
                }
                for (int o = 16; o > 0; o >>= 1) {
                    const unsigned long long other = __shfl_down_sync(0xFFFFFFFFu, mine, o);
                    mine = other < mine ? other : mine;
                }
                if (lane == 0) s_min[warp] = mine;
                __syncthreads();
                unsigned long long m = s_min[0];
                for (int w = 1; w < 8; ++w) m = s_min[w] < m ? s_min[w] : m;
                __syncthreads();
                if (m == ~0ULL) break;   // (fewer comparable values than counted: a NaN cosine; uniform)
                last = m;
                have_last = true;
            }
            if (tid == 0) s_cosk[h] = have_last ? cosv[(int)(last & 0xFFFFFFFFu)] : __int_as_float(0x7FC00000);
        }
        __syncthreads();
    }
    // ---- the reference's decisions
    if (tid == 0) {
        int best = -1, ok = 0;
        double par_out = 0;
        int g[8];
        double par[8];
        for (int h = 0; h < 8; ++h) {
            g[h] = h < ncand ? s_cnt[h] : 0;
            par[h] = (h < ncand && g[h] > 0) ? (double)(acosf(s_cosk[h]) * 180) / M_PI : 0.0;
            a.n_good[8 * (size_t)p + h] = g[h];
        }
        if (use_h && ncand == 8) {
            int bestGood = 0, secondBestGood = 0;
            float bestParallax = -1;
            for (int i = 0; i < 8; ++i) {
                if (g[i] > bestGood) {
                    secondBestGood = bestGood;
                    bestGood = g[i];
                    best = i;
                    bestParallax = (float)par[i];
                } else if (g[i] > secondBestGood) {
                    secondBestGood = g[i];
                }
            }
            par_out = bestParallax;
            ok = (secondBestGood < 0.75 * bestGood && bestParallax >= a.min_parallax && bestGood > a.min_triangulated && bestGood > a.ratio_h * n) ? 1 : 0;
        } else if (!use_h) {
            const int maxGood = max(g[0], max(g[1], max(g[2], g[3])));
            const int minGood = max((int)(0.9 * s_N), a.min_triangulated);
            int similar = 0;
            for (int i = 0; i < 4; ++i)
                if (g[i] > 0.7 * maxGood) ++similar;
            if (!(maxGood < minGood || similar > 1)) {
                for (int i = 0; i < 4; ++i)
                    if (maxGood == g[i]) {
                        best = i;
                        par_out = par[i];
                        ok = par[i] > a.min_parallax ? 1 : 0;
                        break;
                    }
            }
        }
        s_best = best;
        s_ok = ok;
        a.ok[p] = ok;
        a.parallax[p] = par_out;
        for (int k = 0; k < 9; ++k) a.R21[9 * (size_t)p + k] = ok ? s_R[best][k] : 0.0;
        for (int k = 0; k < 3; ++k) a.t21[3 * (size_t)p + k] = ok ? s_t[best][k] : 0.0;
    }
    __syncthreads();
    const int best = s_best, ok = s_ok;
    for (int i = tid; i < n; i += blockDim.x) {
        const double* src = a.p3d_all + 3 * ((size_t)max(best, 0) * a.n_total + a0 + i);
        for (int k = 0; k < 3; ++k) a.p3d[3 * (size_t)(a0 + i) + k] = ok ? src[k] : 0.0;
        a.triangulated[a0 + i] = ok ? a.good_all[(size_t)best * a.n_total + a0 + i] : 0;
    }
}

}  // namespace
}  // namespace ygzb

using namespace ygzb;

extern "C" {

int ygzb_initializer_ransac(ygzb_ctx* ctx, int n_lists, const int32_t* offsets, const double* px1, const double* px2, int max_iter,
                            const int32_t* sets, float sigma, double* H21, float* score_H, int32_t* best_H, uint8_t* inlier_H, double* F21,
                            float* score_F, int32_t* best_F, uint8_t* inlier_F, double* all_models) {
    if (!ctx || n_lists < 1 || !offsets || !px1 || !px2 || max_iter < 1 || !sets || !(sigma > 0) || !H21 || !score_H || !best_H || !inlier_H ||
        !F21 || !score_F || !best_F || !inlier_F)
        return YGZB_ERR_INVALID;
    try {
        cudaSetDevice(ctx->device);
        int rc = check_offsets(ctx, offsets, n_lists, "offsets");
        if (rc != YGZB_OK) return rc;
        const size_t P = (size_t)n_lists, N = (size_t)offsets[n_lists], I = (size_t)max_iter;
        for (size_t p = 0; p < P; ++p) {
            const int n = offsets[p + 1] - offsets[p];
            if (n < 8) return set_error(ctx, YGZB_ERR_INVALID, "initializer: list %zu has %d point pairs, 8 are needed", p, n);
            for (size_t k = 0; k < I * 8; ++k)
                if (sets[p * I * 8 + k] < 0 || sets[p * I * 8 + k] >= n) return set_error(ctx, YGZB_ERR_INVALID, "initializer: set index out of range (list %zu)", p);
        }
        const size_t Hn = P * I * 2;
        int32_t *d_off, *d_sets, *d_obest;
        double *d_px1, *d_px2, *d_pn1, *d_pn2, *d_models, *d_aux, *d_out;
        Norm* d_norm;
        float *d_scores, *d_oscore;
        uint8_t *d_inlH, *d_inlF;
        void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
            d_off = c.take<int32_t>(P + 1);
            d_px1 = c.take<double>(2 * N);
            d_px2 = c.take<double>(2 * N);
            d_pn1 = c.take<double>(2 * N);
            d_pn2 = c.take<double>(2 * N);
            d_sets = c.take<int32_t>(P * I * 8);
            d_norm = c.take<Norm>(P);
            d_models = c.take<double>(9 * Hn);
            d_aux = c.take<double>(9 * Hn);
            d_scores = c.take<float>(Hn);
            d_out = c.take<double>(18 * P);
            d_oscore = c.take<float>(2 * P);
            d_obest = c.take<int32_t>(2 * P);
            d_inlH = c.take<uint8_t>(N);
            d_inlF = c.take<uint8_t>(N);
        });
        if (!buf) return YGZB_ERR_CUDA;
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_off, offsets, (P + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_px1, px1, 16 * N, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_px2, px2, 16 * N, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_sets, sets, P * I * 8 * 4, cudaMemcpyHostToDevice, ctx->stream));
        {
            ProfScope ps(ctx, kStageOther);
            init_normalize_kernel<<<(unsigned)P, 256, 0, ctx->stream>>>(d_off, d_px1, d_px2, d_pn1, d_pn2, d_norm);
            YGZB_LAUNCHED(ctx);
            static std::once_flag once;
            std::call_once(once, [] {
                cudaFuncSetAttribute(init_models_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kWork * kModelThreads * sizeof(double)));
            });
            init_models_kernel<<<(unsigned)((Hn + kModelThreads - 1) / kModelThreads), kModelThreads, kWork * kModelThreads * sizeof(double),
                                 ctx->stream>>>((int)Hn, max_iter, d_off, d_sets, d_pn1, d_pn2, d_norm, d_models, d_aux);
            YGZB_LAUNCHED(ctx);
            init_score_kernel<<<(unsigned)((Hn * 32 + 127) / 128), 128, 0, ctx->stream>>>((int)Hn, max_iter, d_off, d_px1, d_px2, d_models, d_aux,
                                                                                        sigma, d_scores);
            YGZB_LAUNCHED(ctx);
            init_select_kernel<<<dim3((unsigned)P, 2), 128, 0, ctx->stream>>>(max_iter, d_off, d_px1, d_px2, d_models, d_aux, d_scores, sigma, d_out,
                                                                            d_oscore, d_obest, d_inlH, d_inlF);
            YGZB_LAUNCHED(ctx);
        }
        std::vector<double> h_out(18 * P);
        std::vector<float> h_score(2 * P);
        std::vector<int32_t> h_best(2 * P);
        YGZB_CUDA(ctx, cudaMemcpyAsync(h_out.data(), d_out, 18 * P * 8, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(h_score.data(), d_oscore, 2 * P * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(h_best.data(), d_obest, 2 * P * 4, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(inlier_H, d_inlH, N, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(inlier_F, d_inlF, N, cudaMemcpyDeviceToHost, ctx->stream));
        if (all_models) YGZB_CUDA(ctx, cudaMemcpyAsync(all_models, d_models, 9 * Hn * 8, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (size_t p = 0; p < P; ++p) {
            std::copy(h_out.begin() + 18 * p, h_out.begin() + 18 * p + 9, H21 + 9 * p);
            std::copy(h_out.begin() + 18 * p + 9, h_out.begin() + 18 * p + 18, F21 + 9 * p);
            score_H[p] = h_score[2 * p];
            score_F[p] = h_score[2 * p + 1];
            best_H[p] = h_best[2 * p];
            best_F[p] = h_best[2 * p + 1];
        }
        return YGZB_OK;
    } catch (const std::exception& e) {
        return set_error(ctx, YGZB_ERR_INVALID, "initializer_ransac: %s", e.what());
    }
}

int ygzb_initializer_reconstruct(ygzb_ctx* ctx, int n_lists, const int32_t* offsets, const double* px1, const double* px2, const int32_t* use_h,
                                 const double* model, const uint8_t* inliers, float sigma2, float min_parallax, int min_triangulated,
                                 double good_point_ratio_h, int32_t* ok, double* R21, double* t21, double* p3d, uint8_t* triangulated,
                                 int32_t* n_good, double* parallax, double* candidates) {
    if (!ctx || n_lists < 1 || !offsets || !px1 || !px2 || !use_h || !model || !inliers || !ok || !R21 || !t21 || !p3d || !triangulated ||
        !n_good || !parallax)
        return YGZB_ERR_INVALID;
    try {
        cudaSetDevice(ctx->device);
        int rc = check_offsets(ctx, offsets, n_lists, "offsets");
        if (rc != YGZB_OK) return rc;
        const size_t P = (size_t)n_lists, N = (size_t)offsets[n_lists];
        if (N == 0) return set_error(ctx, YGZB_ERR_INVALID, "initializer_reconstruct: no point pairs");
        ReconArgs a;
        int32_t *d_off, *d_use;
        double *d_px1, *d_px2, *d_model;
        uint8_t* d_inl;
        void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
            d_off = c.take<int32_t>(P + 1);
            d_px1 = c.take<double>(2 * N);
            d_px2 = c.take<double>(2 * N);
            d_use = c.take<int32_t>(P);
            d_model = c.take<double>(9 * P);
            d_inl = c.take<uint8_t>(N);
            a.p3d_all = c.take<double>(8 * 3 * N);
            a.good_all = c.take<uint8_t>(8 * N);
            a.cos_all = c.take<float>(8 * N);
            a.ok = c.take<int32_t>(P);
            a.R21 = c.take<double>(9 * P);
            a.t21 = c.take<double>(3 * P);
            a.p3d = c.take<double>(3 * N);
            a.triangulated = c.take<uint8_t>(N);
            a.n_good = c.take<int32_t>(8 * P);
            a.parallax = c.take<double>(P);
            a.candidates = c.take<double>(96 * P);   // (laid out whether or not the caller asks for them)
        });
        if (!buf) return YGZB_ERR_CUDA;
        if (!candidates) a.candidates = nullptr;
        a.off = d_off; a.px1 = d_px1; a.px2 = d_px2; a.use_h = d_use; a.model = d_model; a.inliers = d_inl;
        a.K[0] = ctx->prm.fx; a.K[1] = ctx->prm.fy; a.K[2] = ctx->prm.cx; a.K[3] = ctx->prm.cy;
        a.sigma2 = sigma2; a.min_parallax = min_parallax; a.min_triangulated = min_triangulated; a.ratio_h = good_point_ratio_h;
        a.n_total = N;
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_off, offsets, (P + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_px1, px1, 16 * N, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_px2, px2, 16 * N, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_use, use_h, 4 * P, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_model, model, 72 * P, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_inl, inliers, N, cudaMemcpyHostToDevice, ctx->stream));
        {
            ProfScope ps(ctx, kStageOther);
            init_reconstruct_kernel<<<(unsigned)P, 256, 0, ctx->stream>>>(a);
            YGZB_LAUNCHED(ctx);
        }
        YGZB_CUDA(ctx, cudaMemcpyAsync(ok, a.ok, 4 * P, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(R21, a.R21, 72 * P, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(t21, a.t21, 24 * P, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(p3d, a.p3d, 24 * N, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(triangulated, a.triangulated, N, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(n_good, a.n_good, 32 * P, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(parallax, a.parallax, 8 * P, cudaMemcpyDeviceToHost, ctx->stream));
        if (candidates) YGZB_CUDA(ctx, cudaMemcpyAsync(candidates, a.candidates, 96 * 8 * P, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return YGZB_OK;
    } catch (const std::exception& e) {
        return set_error(ctx, YGZB_ERR_INVALID, "initializer_reconstruct: %s", e.what());
    }
}

}  // extern "C"
