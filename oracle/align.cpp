// oracle/align.cpp -- patch alignment and sparse image alignment.
// TEST INFRASTRUCTURE ONLY (see oracle.h).
//   cvutils::Align2D / Align1D          reference src/Algorithm/CVUtils.cpp:186-318, :64-184
//   cvutils::GetBilateralInterpUchar    reference include/ygz/Algorithm/CVUtils.h:59-71
//   cvutils::JacobXYZ2Cam               reference include/ygz/Algorithm/CVUtils.h:77-99
//   Matcher::FindDirectProjection       reference src/Algorithm/Matcher.cpp:385-417 (Feature* overload)
//   Matcher::GetWarpAffineMatrix        reference src/Algorithm/Matcher.cpp:420-436
//   Matcher::WarpAffine                 reference src/Algorithm/Matcher.cpp:438-466
//   Matcher::GetBestSearchLevel         reference include/ygz/Algorithm/Matcher.h:123-134
//   SparseImgAlign::*                   reference src/Algorithm/SparseImageAlign.cpp:21-238
//   NLLSSolver::optimizeGaussNewton     reference include/ygz/Algorithm/NLSSolver_impl.hpp:16-88
//   Matcher::SparseImageAlignment       reference src/Algorithm/Matcher.cpp:468-492
// f32 / f64 operations are written in the reference's order; Eigen's fixed-size 3x3 / 2x2 inverse is
// restated as cofactors * (1/det); H.ldlt().solve() (6x6) as an unpivoted LDL^T (tolerances: SURVEY 8d).
#include <cmath>
#include <cstring>
#include <vector>

#include "oracle.h"
#include "se3.h"

using namespace ora;

namespace {

struct Img {
    const uint8_t* d;
    int w, h;
};

// Eigen compute_inverse for 3x3: cofactors, det from the first column, multiply by 1/det
void inverse3f(const float H[3][3], float inv[3][3]) {
    auto cof = [&](int i, int j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        return H[i1][j1] * H[i2][j2] - H[i1][j2] * H[i2][j1];
    };
    const float c00 = cof(0, 0), c10 = cof(1, 0), c20 = cof(2, 0);
    const float det = (c00 * H[0][0] + c10 * H[1][0]) + c20 * H[2][0];
    const float invdet = 1.0f / det;
    inv[0][0] = c00 * invdet;
    inv[0][1] = c10 * invdet;
    inv[0][2] = c20 * invdet;
    inv[1][0] = cof(0, 1) * invdet;
    inv[1][1] = cof(1, 1) * invdet;
    inv[1][2] = cof(2, 1) * invdet;
    inv[2][0] = cof(0, 2) * invdet;
    inv[2][1] = cof(1, 2) * invdet;
    inv[2][2] = cof(2, 2) * invdet;
}

}  // namespace

// cvutils::Align2D (CVUtils.cpp:186-318), the portable (non-NEON) body
extern "C" int ora_align2d(const uint8_t* img, int w, int h, const uint8_t* ref_with_border, const uint8_t* ref, int n_iter,
                           double* pu, double* pv) {
    const int halfpatch = 4, patch = 8;
    bool converged = false;
    float dxs[64], dys[64];
    float H[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    const int ref_step = patch + 2;
    for (int y = 0, k = 0; y < patch; ++y) {
        const uint8_t* it = ref_with_border + (y + 1) * ref_step + 1;
        for (int x = 0; x < patch; ++x, ++it, ++k) {
            float J[3];
            J[0] = (float)(0.5 * (it[1] - it[-1]));
            J[1] = (float)(0.5 * (it[ref_step] - it[-ref_step]));
            J[2] = 1;
            dxs[k] = J[0];
            dys[k] = J[1];
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) H[a][b] += J[a] * J[b];
        }
    }
    float Hinv[3][3];
    inverse3f(H, Hinv);
    float mean_diff = 0;
    float u = (float)*pu, v = (float)*pv;
    const float min_update_squared = (float)(0.03 * 0.03);
    float chi2 = 0;
    for (int iter = 0; iter < n_iter; ++iter) {
        chi2 = 0;
        const int u_r = (int)std::floor(u), v_r = (int)std::floor(v);
        if (u_r < halfpatch || v_r < halfpatch || u_r >= w - halfpatch || v_r >= h - halfpatch) break;
        if (std::isnan(u) || std::isnan(v)) return 0;  // (unreachable after the floor test; kept for fidelity)
        const float sx = u - u_r, sy = v - v_r;
        const float wTL = (float)((1.0 - sx) * (1.0 - sy));
        const float wTR = (float)(sx * (1.0 - sy));
        const float wBL = (float)((1.0 - sx) * sy);
        const float wBR = sx * sy;
        float Jres[3] = {0, 0, 0};
        for (int y = 0, k = 0; y < patch; ++y) {
            const uint8_t* it = img + (size_t)(v_r + y - halfpatch) * w + u_r - halfpatch;
            for (int x = 0; x < patch; ++x, ++it, ++k) {
                const float search_pixel = wTL * it[0] + wTR * it[1] + wBL * it[w] + wBR * it[w + 1];
                const float res = search_pixel - ref[k] + mean_diff;
                Jres[0] -= res * dxs[k];
                Jres[1] -= res * dys[k];
                Jres[2] -= res;
                chi2 += res * res;
            }
        }
        float upd[3];
        for (int a = 0; a < 3; ++a) upd[a] = (Hinv[a][0] * Jres[0] + Hinv[a][1] * Jres[1]) + Hinv[a][2] * Jres[2];
        u += upd[0];
        v += upd[1];
        mean_diff += upd[2];
        if (upd[0] * upd[0] + upd[1] * upd[1] < min_update_squared) {
            converged = true;
            break;
        }
    }
    *pu = u;
    *pv = v;
    return (converged && chi2 < 20000) ? 1 : 0;
}

// cvutils::Align1D (CVUtils.cpp:64-184)
extern "C" int ora_align1d(const uint8_t* img, int w, int h, float dirx, float diry, const uint8_t* ref_with_border,
                           const uint8_t* ref, int n_iter, double* pu, double* pv, double* h_inv) {
    const int halfpatch = 4, patch = 8;
    bool converged = false;
    float dvs[64];
    float H[2][2] = {{0, 0}, {0, 0}};
    const int ref_step = patch + 2;
    for (int y = 0, k = 0; y < patch; ++y) {
        const uint8_t* it = ref_with_border + (y + 1) * ref_step + 1;
        for (int x = 0; x < patch; ++x, ++it, ++k) {
            float J[2];
            J[0] = (float)(0.5 * (dirx * (it[1] - it[-1]) + diry * (it[ref_step] - it[-ref_step])));
            J[1] = 1;
            dvs[k] = J[0];
            for (int a = 0; a < 2; ++a)
                for (int b = 0; b < 2; ++b) H[a][b] += J[a] * J[b];
        }
    }
    *h_inv = 1.0 / H[0][0] * patch * patch;
    // Eigen 2x2 inverse: adjugate * (1/det)
    const float invdet = 1.0f / (H[0][0] * H[1][1] - H[1][0] * H[0][1]);
    const float Hinv[2][2] = {{H[1][1] * invdet, -H[0][1] * invdet}, {-H[1][0] * invdet, H[0][0] * invdet}};
    float mean_diff = 0;
    float u = (float)*pu, v = (float)*pv;
    const float min_update_squared = (float)(0.03 * 0.03);
    float chi2 = 0;
    float upd[2] = {0, 0};
    for (int iter = 0; iter < n_iter; ++iter) {
        const int u_r = (int)std::floor(u), v_r = (int)std::floor(v);
        if (u_r < halfpatch || v_r < halfpatch || u_r >= w - halfpatch || v_r >= h - halfpatch) break;
        if (std::isnan(u) || std::isnan(v)) return 0;
        const float sx = u - u_r, sy = v - v_r;
        const float wTL = (float)((1.0 - sx) * (1.0 - sy));
        const float wTR = (float)(sx * (1.0 - sy));
        const float wBL = (float)((1.0 - sx) * sy);
        const float wBR = sx * sy;
        float new_chi2 = 0;
        float Jres[2] = {0, 0};
        for (int y = 0, k = 0; y < patch; ++y) {
            const uint8_t* it = img + (size_t)(v_r + y - halfpatch) * w + u_r - halfpatch;
            for (int x = 0; x < patch; ++x, ++it, ++k) {
                const float search_pixel = wTL * it[0] + wTR * it[1] + wBL * it[w] + wBR * it[w + 1];
                const float res = search_pixel - ref[k] + mean_diff;
                Jres[0] -= res * dvs[k];
                Jres[1] -= res;
                new_chi2 += res * res;
            }
        }
        if (iter > 0 && new_chi2 > chi2) {
            u -= upd[0];
            v -= upd[1];
            break;
        }
        chi2 = new_chi2;
        upd[0] = Hinv[0][0] * Jres[0] + Hinv[0][1] * Jres[1];
        upd[1] = Hinv[1][0] * Jres[0] + Hinv[1][1] * Jres[1];
        u += upd[0] * dirx;
        v += upd[0] * diry;
        mean_diff += upd[1];
        if (upd[0] * upd[0] + upd[1] * upd[1] < min_update_squared) {
            converged = true;
            break;
        }
    }
    *pu = u;
    *pv = v;
    return converged ? 1 : 0;
}

namespace {

struct Cam {
    float fx, fy, cx, cy;  // Camera.h:105-107: stored as float, maths in double
    V3 pixel2camera(double px, double py, double depth) const {
        return {(px - cx) * depth / fx, (py - cy) * depth / fy, depth};
    }
    void camera2pixel(V3 p, double* u, double* v) const {
        *u = fx * p.x / p.z + cx;
        *v = fy * p.y / p.z + cy;
    }
    double focal() const { return (float)((fx + fy) / 2); }  // _f = (_fx+_fy)/2, a float member
};

Img level(const uint8_t* pyr, int w, int h, int n_levels, int L) {
    int lw[ORA_MAX_LEVELS], lh[ORA_MAX_LEVELS];
    size_t off[ORA_MAX_LEVELS];
    ora_pyramid_layout(w, h, n_levels, lw, lh, off);
    return Img{pyr + off[L], lw[L], lh[L]};
}

// cvutils::GetBilateralInterpUchar
uint8_t interp_uchar(double x, double y, const Img& im) {
    const double xx = x - std::floor(x), yy = y - std::floor(y);
    const uint8_t* d = im.d + (size_t)(int)y * im.w + (int)x;
    return (uint8_t)((1 - xx) * (1 - yy) * d[0] + xx * (1 - yy) * d[1] + (1 - xx) * yy * d[im.w] + xx * yy * d[im.w + 1]);
}

}  // namespace

extern "C" void ora_find_direct_projection(const uint8_t* ref_pyr, const uint8_t* cur_pyr, int w, int h, int n_levels,
                                           const ora_camera* camp, const double* T_cw_ref, const double* T_cw_cur, int n,
                                           const double* ref_px, const double* ref_depth, const int32_t* ref_level,
                                           double* cur_px, int32_t* search_level, uint8_t* ok) {
    const Cam cam{camp->fx, camp->fy, camp->cx, camp->cy};
    const SE3 Tr = SE3::from_mat(T_cw_ref), Tc = SE3::from_mat(T_cw_cur);
    const SE3 TCR = Tc * Tr.inverse();
    const SE3 Tr_inv = Tr.inverse();
    const int half = 4;  // WarpHalfPatchSize
    for (int i = 0; i < n; ++i) {
        ok[i] = 0;
        search_level[i] = 0;
        if (ref_depth[i] < 0) continue;
        const double pxr = ref_px[2 * i], pyr_ = ref_px[2 * i + 1];
        const int lvl = ref_level[i];
        const V3 pt_ref = cam.pixel2camera(pxr, pyr_, ref_depth[i]);
        // GetWarpAffineMatrix (sic: the WORLD point is transformed with T_CR, Matcher.cpp:425-430)
        const V3 pt_ref_world = Tr_inv * pt_ref;
        const V3 pt_du = cam.pixel2camera(pxr + (double)half * (1 << lvl), pyr_, pt_ref.z);
        const V3 pt_dv = cam.pixel2camera(pxr, pyr_ + (double)half * (1 << lvl), pt_ref.z);
        double cu, cv, du_u, du_v, dv_u, dv_v;
        cam.camera2pixel(TCR * pt_ref_world, &cu, &cv);
        cam.camera2pixel(TCR * pt_du, &du_u, &du_v);
        cam.camera2pixel(TCR * pt_dv, &dv_u, &dv_v);
        const double A00 = (du_u - cu) / half, A10 = (du_v - cv) / half, A01 = (dv_u - cu) / half, A11 = (dv_v - cv) / half;
        // GetBestSearchLevel(ACR, pyramid_level - 1)
        int sl = 0;
        double D = A00 * A11 - A01 * A10;
        while (D > 3.0 && sl < n_levels - 1) {
            sl += 1;
            D *= 0.25;
        }
        search_level[i] = sl;
        // WarpAffine(ACR, ref pyramid[lvl], px_ref, lvl, sl, 5, patch_with_border)
        const double det = A00 * A11 - A10 * A01;
        const double invdet = 1.0 / det;
        const double R00 = A11 * invdet, R01 = -A01 * invdet, R10 = -A10 * invdet, R11 = A00 * invdet;  // ARC = ACR^-1
        const Img im = level(ref_pyr, w, h, n_levels, lvl);
        uint8_t pwb[100], patch[64];
        const double rx = pxr / (1 << lvl), ry = pyr_ / (1 << lvl);
        for (int y = 0, k = 0; y < 10; ++y)
            for (int x = 0; x < 10; ++x, ++k) {
                const double ppx = (double)(x - 5) * (1 << sl), ppy = (double)(y - 5) * (1 << sl);
                const double qx = (R00 * ppx + R01 * ppy) + rx, qy = (R10 * ppx + R11 * ppy) + ry;
                // (a NaN warp fails every comparison in the reference and would index out of range there: -> 0)
                if (!(qx >= 0 && qy >= 0 && qx < im.w - 1 && qy < im.h - 1)) pwb[k] = 0;
                else pwb[k] = interp_uchar(qx, qy, im);
            }
        for (int y = 1; y < 9; ++y)
            for (int x = 0; x < 8; ++x) patch[(y - 1) * 8 + x] = pwb[y * 10 + 1 + x];
        double su = cur_px[2 * i] / (1 << sl), sv = cur_px[2 * i + 1] / (1 << sl);
        const Img ci = level(cur_pyr, w, h, n_levels, sl);
        const int success = ora_align2d(ci.d, ci.w, ci.h, pwb, patch, 10, &su, &sv);
        cur_px[2 * i] = su * (1 << sl);
        cur_px[2 * i + 1] = sv * (1 << sl);
        // curr->InFrame(px_curr) with the default border 10 against the full-res size
        const bool in = cur_px[2 * i] >= 10 && cur_px[2 * i] < w - 10 && cur_px[2 * i + 1] >= 10 && cur_px[2 * i + 1] < h - 10;
        ok[i] = (in && success) ? 1 : 0;
    }
}

// ---- SparseImgAlign ---------------------------------------------------------------------------------
namespace {

// unpivoted LDL^T solve of the 6x6 normal equations (Eigen's ldlt() pivots; the system is SPD here)
bool ldlt_solve6(const double H[6][6], const double b[6], double x[6]) {
    double L[6][6] = {}, D[6];
    for (int j = 0; j < 6; ++j) {
        double d = H[j][j];
        for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k] * D[k];
        D[j] = d;
        if (!(std::fabs(d) > 0)) return false;
        L[j][j] = 1;
        for (int i = j + 1; i < 6; ++i) {
            double s = H[i][j];
            for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k] * D[k];
            L[i][j] = s / d;
        }
    }
    double y[6];
    for (int i = 0; i < 6; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= L[i][k] * y[k];
        y[i] = s;
    }
    for (int i = 0; i < 6; ++i) y[i] /= D[i];
    for (int i = 5; i >= 0; --i) {
        double s = y[i];
        for (int k = i + 1; k < 6; ++k) s -= L[k][i] * x[k];
        x[i] = s;
    }
    return true;
}

struct SparseAlign {
    const uint8_t *ref_pyr, *cur_pyr;
    int w, h, n_levels;
    Cam cam;
    int n;
    const double *px, *depth;
    const uint8_t* has_mp;
    int level_ = 0;
    std::vector<float> ref_patch_cache;   // n x 16
    std::vector<double> jac;              // 6 x (16 n), column major like Eigen
    std::vector<uint8_t> visible;
    bool have_ref_patch_cache = false;
    double H[6][6], Jres[6], x[6];
    size_t n_meas = 0;
    double chi2_ = 1e10;
    bool exact_chi2 = false;   // sum the squared residuals in double and round to float once (the kernel's order-free sum)

    // SparseImgAlign::precomputeReferencePatches (:59-122)
    void precompute() {
        const int border = 3;  // patch_halfsize_ + 1
        const Img im = level(ref_pyr, w, h, n_levels, level_);
        const int stride = im.w;
        const float scale = 1.0f / (1 << level_);
        const double focal = cam.focal();
        for (int i = 0; i < n; ++i) {
            const float u_ref = (float)(px[2 * i] * scale), v_ref = (float)(px[2 * i + 1] * scale);
            const int ui = (int)floorf(u_ref), vi = (int)floorf(v_ref);
            if (!has_mp[i] || ui - border < 0 || vi - border < 0 || ui + border >= im.w || vi + border >= im.h) continue;
            visible[i] = 1;
            const V3 xyz = cam.pixel2camera(px[2 * i], px[2 * i + 1], depth[i]);
            // cvutils::JacobXYZ2Cam
            double J[2][6];
            const double X = xyz.x, Y = xyz.y, zi = 1. / xyz.z, zi2 = zi * zi;
            J[0][0] = -zi; J[0][1] = 0; J[0][2] = X * zi2; J[0][3] = Y * J[0][2]; J[0][4] = -(1.0 + X * J[0][2]); J[0][5] = Y * zi;
            J[1][0] = 0; J[1][1] = -zi; J[1][2] = Y * zi2; J[1][3] = 1.0 + Y * J[1][2]; J[1][4] = -J[0][3]; J[1][5] = -X * zi;
            const float su = u_ref - ui, sv = v_ref - vi;
            const float wtl = (float)((1.0 - su) * (1.0 - sv)), wtr = (float)(su * (1.0 - sv)), wbl = (float)((1.0 - su) * sv),
                        wbr = su * sv;
            float* cache = &ref_patch_cache[16 * (size_t)i];
            int pc = 0;
            for (int y = 0; y < 4; ++y) {
                const uint8_t* p = im.d + (size_t)(vi + y - 2) * stride + (ui - 2);
                for (int xx = 0; xx < 4; ++xx, ++p, ++pc) {
                    cache[pc] = wtl * p[0] + wtr * p[1] + wbl * p[stride] + wbr * p[stride + 1];
                    const float dx = 0.5f * ((wtl * p[1] + wtr * p[2] + wbl * p[stride + 1] + wbr * p[stride + 2]) -
                                             (wtl * p[-1] + wtr * p[0] + wbl * p[stride - 1] + wbr * p[stride]));
                    const float dy = 0.5f * ((wtl * p[stride] + wtr * p[1 + stride] + wbl * p[stride * 2] + wbr * p[stride * 2 + 1]) -
                                             (wtl * p[-stride] + wtr * p[1 - stride] + wbl * p[0] + wbr * p[1]));
                    double* col = &jac[6 * (16 * (size_t)i + pc)];
                    for (int k = 0; k < 6; ++k) col[k] = (dx * J[0][k] + dy * J[1][k]) * (focal / (1 << level_));
                }
            }
        }
        have_ref_patch_cache = true;
    }

    // SparseImgAlign::computeResiduals (:124-223), use_weights_ == false
    double residuals(const SE3& T, bool linearize) {
        const Img im = level(cur_pyr, w, h, n_levels, level_);
        if (!have_ref_patch_cache) precompute();
        const int stride = im.w, border = 3;
        const float scale = 1.0f / (1 << level_);
        float chi2 = 0.0f;
        double chi2_d = 0.0;
        for (int i = 0; i < n; ++i) {
            if (!visible[i]) continue;
            const V3 xyz_ref = cam.pixel2camera(px[2 * i], px[2 * i + 1], depth[i]);
            const V3 xyz_cur = T * xyz_ref;
            double pu, pv;
            cam.camera2pixel(xyz_cur, &pu, &pv);
            const float u_cur = (float)pu * scale, v_cur = (float)pv * scale;
            const int ui = (int)floorf(u_cur), vi = (int)floorf(v_cur);
            if (ui < 0 || vi < 0 || ui - border < 0 || vi - border < 0 || ui + border >= im.w || vi + border >= im.h) continue;
            const float su = u_cur - ui, sv = v_cur - vi;
            const float wtl = (float)((1.0 - su) * (1.0 - sv)), wtr = (float)(su * (1.0 - sv)), wbl = (float)((1.0 - su) * sv),
                        wbr = su * sv;
            const float* cache = &ref_patch_cache[16 * (size_t)i];
            int pc = 0;
            for (int y = 0; y < 4; ++y) {
                const uint8_t* p = im.d + (size_t)(vi + y - 2) * stride + (ui - 2);
                for (int xx = 0; xx < 4; ++xx, ++pc, ++p) {
                    const float inten = wtl * p[0] + wtr * p[1] + wbl * p[stride] + wbr * p[stride + 1];
                    const float res = inten - cache[pc];
                    const float weight = 1.0;
                    chi2 += res * res * weight;
                    chi2_d += (double)(res * res * weight);
                    n_meas++;
                    if (linearize) {
                        const double* J = &jac[6 * (16 * (size_t)i + pc)];
                        for (int a = 0; a < 6; ++a) {
                            for (int b = 0; b < 6; ++b) H[a][b] += J[a] * J[b] * weight;
                            Jres[a] -= J[a] * res * weight;
                        }
                    }
                }
            }
        }
        if (exact_chi2) return (float)chi2_d / (float)n_meas;
        return chi2 / n_meas;
    }
};

}  // namespace

extern "C" size_t ora_sparse_align(const uint8_t* ref_pyr, const uint8_t* cur_pyr, int w, int h, int n_levels,
                                   const ora_camera* camp, int n, const double* px, const double* depth,
                                   const uint8_t* has_mappoint, const double* T_cw_ref, double* T_cw_cur, int max_level,
                                   int min_level, int n_iter, double eps, int32_t* iters_per_level, int exact_chi2) {
    if (n == 0) return 0;  // run(): ref_frame->_features.empty()
    SparseAlign s;
    s.exact_chi2 = exact_chi2 != 0;
    s.ref_pyr = ref_pyr; s.cur_pyr = cur_pyr; s.w = w; s.h = h; s.n_levels = n_levels;
    s.cam = Cam{camp->fx, camp->fy, camp->cx, camp->cy};
    s.n = n; s.px = px; s.depth = depth; s.has_mp = has_mappoint;
    s.ref_patch_cache.assign(16 * (size_t)n, 0.f);
    s.jac.assign(6 * 16 * (size_t)n, 0.0);
    s.visible.assign(n, 0);   // TODO in the reference: never reset per level -- kept
    const SE3 Tref = SE3::from_mat(T_cw_ref);
    SE3 T = SE3::from_mat(T_cw_cur) * Tref.inverse();  // T_cur_from_ref
    for (int lvl = max_level; lvl >= min_level; --lvl) {
        s.level_ = lvl;
        std::fill(s.jac.begin(), s.jac.end(), 0.0);  // jacobian_cache_.setZero()
        s.have_ref_patch_cache = false;
        // NLLSSolver::optimizeGaussNewton
        SE3 old_model = T;
        int it = 0;
        bool stop = false;
        for (it = 0; it < n_iter; ++it) {
            std::memset(s.H, 0, sizeof(s.H));
            std::memset(s.Jres, 0, sizeof(s.Jres));
            s.n_meas = 0;
            const double new_chi2 = s.residuals(T, true);
            if (!ldlt_solve6(s.H, s.Jres, s.x) || std::isnan(s.x[0])) stop = true;
            if ((it > 0 && new_chi2 > s.chi2_) || stop) {
                T = old_model;  // rollback
                break;
            }
            double mx[6];
            for (int k = 0; k < 6; ++k) mx[k] = -s.x[k];
            const SE3 Tnew = T * SE3::exp(mx);  // update(): T_new = T_old * exp(-x)
            old_model = T;
            T = Tnew;
            s.chi2_ = new_chi2;
            double nm = -1;
            for (int k = 0; k < 6; ++k) nm = std::fabs(s.x[k]) > nm ? std::fabs(s.x[k]) : nm;
            if (nm <= eps) break;
        }
        if (iters_per_level) iters_per_level[lvl] = it;
    }
    (T * Tref).to_mat(T_cw_cur);
    return s.n_meas / 16;
}

extern "C" int ora_matcher_sparse_alignment(const uint8_t* ref_pyr, const uint8_t* cur_pyr, int w, int h, int n_levels,
                                            const ora_camera* cam, int n, const double* px, const double* depth,
                                            const uint8_t* has_mappoint, const double* T_cw_ref, double* T_cw_cur) {
    // current->_TCW = ref->_TCW; _align->run(ref, current) with SparseImgAlign(2, 0, 30, GaussNewton) (Matcher.cpp:18)
    double T[12];
    std::memcpy(T, T_cw_ref, sizeof(T));
    ora_sparse_align(ref_pyr, cur_pyr, w, h, n_levels, cam, n, px, depth, has_mappoint, T_cw_ref, T, 2, 0, 30, 0.000001, nullptr, 0);
    const SE3 TCR = SE3::from_mat(T) * SE3::from_mat(T_cw_ref).inverse();
    double lg[6];
    TCR.log(lg);
    double nrm = 0;
    for (int k = 0; k < 6; ++k) nrm += lg[k] * lg[k];
    if (std::sqrt(nrm) > 0.2) {  // _max_alignment_motion
        std::memcpy(T_cw_cur, T_cw_ref, sizeof(T));
        return 0;
    }
    std::memcpy(T_cw_cur, T, sizeof(T));
    return 1;
}

extern "C" void ora_se3_exp(const double* v, double* T) { SE3::exp(v).to_mat(T); }
extern "C" void ora_se3_log(const double* T, double* v) { SE3::from_mat(T).log(v); }
