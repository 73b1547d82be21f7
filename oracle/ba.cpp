// oracle/ba.cpp -- local bundle adjustment and pose-only refinement.
// TEST INFRASTRUCTURE ONLY (see oracle.h).
//
//   ba::LocalBAG2O                    reference src/Algorithm/BA.cpp:386-543
//   VertexSE3Sophus::oplusImpl        reference include/ygz/G2oTypes.h:38-45   (estimate = [omega; upsilon],
//                                     update est <- log(exp(delta) * exp(est)))
//   EdgeSophusSE3ProjectXYZ           reference include/ygz/G2oTypes.h:50-146  (error = obs - (f X/Z + c), analytic J)
//   ba::OptimizeCurrentPoseOnly       reference src/Algorithm/BA.cpp:188-264
//   CeresReprojectionErrorPoseOnly    reference include/ygz/Ceres/CeresReprojectionErrorPoseOnly.h:27-58
//
// The optimisers themselves (g2o, Ceres) are NOT in the reference tree and are unpinned (SURVEY.md 8c):
// PARITY UNPINNED.  They are restated from the published algorithms (SURVEY.md appendix A.3 / A.4):
//   g2o   OptimizationAlgorithmLevenberg + BlockSolver_6_3 with marginalised landmarks (Schur complement onto
//         the free poses, dense Cholesky in place of CSparse), RobustKernelHuber, tau = 1e-5, <= 10 trials.
//   Ceres trust-region Levenberg-Marquardt with Jacobi scaling, default Solver::Options, AutoDiff (forward jets).
// Known-answer pin: the ground-truth scene of test/test_local_ba.cpp (tests/test_oracle_ba.py).
#include <cmath>
#include <cstring>
#include <vector>

#include "oracle.h"
#include "se3.h"

using namespace ora;

namespace {

struct CamD {
    double fx, fy, cx, cy;  // EdgeSophusSE3ProjectXYZ::setCamera copies the float intrinsics into doubles
};

// g2o order [omega; upsilon] -> SE3
SE3 pose_from_g2o(const double* est) {
    const double v[6] = {est[3], est[4], est[5], est[0], est[1], est[2]};
    return SE3::exp(v);
}

// dense Cholesky solve A x = b (A symmetric positive definite, n x n, row major); false if not SPD
bool cholesky_solve(std::vector<double>& A, std::vector<double>& b, int n) {
    for (int j = 0; j < n; ++j) {
        double d = A[j * n + j];
        for (int k = 0; k < j; ++k) d -= A[j * n + k] * A[j * n + k];
        if (!(d > 0)) return false;
        d = std::sqrt(d);
        A[j * n + j] = d;
        for (int i = j + 1; i < n; ++i) {
            double s = A[i * n + j];
            for (int k = 0; k < j; ++k) s -= A[i * n + k] * A[j * n + k];
            A[i * n + j] = s / d;
        }
    }
    for (int i = 0; i < n; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= A[i * n + k] * b[k];
        b[i] = s / A[i * n + i];
    }
    for (int i = n - 1; i >= 0; --i) {
        double s = b[i];
        for (int k = i + 1; k < n; ++k) s -= A[k * n + i] * b[k];
        b[i] = s / A[i * n + i];
    }
    return true;
}

void inverse3d(const double H[3][3], double inv[3][3]) {
    auto cof = [&](int i, int j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        return H[i1][j1] * H[i2][j2] - H[i1][j2] * H[i2][j1];
    };
    const double c00 = cof(0, 0), c10 = cof(1, 0), c20 = cof(2, 0);
    const double det = (c00 * H[0][0] + c10 * H[1][0]) + c20 * H[2][0];
    const double invdet = 1.0 / det;
    inv[0][0] = c00 * invdet; inv[0][1] = c10 * invdet; inv[0][2] = c20 * invdet;
    inv[1][0] = cof(0, 1) * invdet; inv[1][1] = cof(1, 1) * invdet; inv[1][2] = cof(2, 1) * invdet;
    inv[2][0] = cof(0, 2) * invdet; inv[2][1] = cof(1, 2) * invdet; inv[2][2] = cof(2, 2) * invdet;
}

struct BAProblem {
    CamD cam;
    int n_kf, n_pt, n_obs;
    std::vector<double> poses;   // g2o order
    std::vector<double> pts;
    const uint8_t* fixed;
    const int32_t *kf_idx, *pt_idx;
    const double* obs;
    double delta;                // Huber delta, <= 0: none
    std::vector<int> free_index; // pose -> index among free poses or -1
    int n_free = 0;

    // EdgeSophusSE3ProjectXYZ::computeError
    void error(const SE3& T, const double* X, const double* z, double e[2], V3* pc = nullptr) const {
        const V3 p = T * V3{X[0], X[1], X[2]};
        if (pc) *pc = p;
        e[0] = z[0] - (p.x / p.z * cam.fx + cam.cx);
        e[1] = z[1] - (p.y / p.z * cam.fy + cam.cy);
    }

    // activeRobustChi2 (RobustKernelHuber::robustify rho[0])
    double robust_chi2(const std::vector<double>& P, const std::vector<double>& X) const {
        std::vector<SE3> T(n_kf);
        for (int k = 0; k < n_kf; ++k) T[k] = pose_from_g2o(&P[6 * k]);
        double chi = 0;
        for (int o = 0; o < n_obs; ++o) {
            double e[2];
            error(T[kf_idx[o]], &X[3 * pt_idx[o]], obs + 2 * o, e);
            const double e2 = e[0] * e[0] + e[1] * e[1];
            if (delta > 0 && e2 > delta * delta) chi += 2 * std::sqrt(e2) * delta - delta * delta;
            else chi += e2;
        }
        return chi;
    }
};

}  // namespace

extern "C" int ora_local_ba_g2o(const ora_camera* camp, int n_kf, double* poses, const uint8_t* fixed, int n_pt, double* pts,
                                int n_obs, const int32_t* kf_idx, const int32_t* pt_idx, const double* obs_px,
                                const ora_ba_params* prm, uint8_t* outlier, ora_ba_stats* stats) {
    BAProblem pb;
    pb.cam = CamD{camp->fx, camp->fy, camp->cx, camp->cy};
    pb.n_kf = n_kf; pb.n_pt = n_pt; pb.n_obs = n_obs;
    pb.poses.assign(poses, poses + 6 * (size_t)n_kf);
    pb.pts.assign(pts, pts + 3 * (size_t)n_pt);
    pb.fixed = fixed; pb.kf_idx = kf_idx; pb.pt_idx = pt_idx; pb.obs = obs_px;
    pb.delta = prm->huber_delta;
    pb.free_index.assign(n_kf, -1);
    for (int k = 0; k < n_kf; ++k)
        if (!fixed[k]) pb.free_index[k] = pb.n_free++;
    const int np = pb.n_free, dimp = 6 * np;

    // observations grouped by landmark (g2o walks each landmark's edge set when it builds the Schur complement)
    std::vector<std::vector<int>> obs_of_pt(n_pt);
    for (int o = 0; o < n_obs; ++o) obs_of_pt[pt_idx[o]].push_back(o);

    std::vector<double> Hpp((size_t)np * 36), bp(dimp), Hll((size_t)n_pt * 9), bl((size_t)3 * n_pt), Hpl((size_t)n_obs * 18);
    std::vector<double> xp(dimp), xl((size_t)3 * n_pt);
    double lambda = 0, ni = 2;
    int iters = 0, trials_total = 0;
    double chi_first = 0, chi_last = 0;

    // computeActiveErrors + buildSystem at the current estimate; returns its robust chi2
    auto build_system = [&]() {
        const double chi = pb.robust_chi2(pb.poses, pb.pts);
        std::fill(Hpp.begin(), Hpp.end(), 0.0); std::fill(bp.begin(), bp.end(), 0.0);
        std::fill(Hll.begin(), Hll.end(), 0.0); std::fill(bl.begin(), bl.end(), 0.0);
        std::fill(Hpl.begin(), Hpl.end(), 0.0);
        std::vector<SE3> T(n_kf);
        std::vector<M3> R(n_kf);
        for (int k = 0; k < n_kf; ++k) {
            T[k] = pose_from_g2o(&pb.poses[6 * k]);
            R[k] = T[k].so3.matrix();
        }
        for (int o = 0; o < n_obs; ++o) {
            const int k = kf_idx[o], j = pt_idx[o];
            double e[2];
            V3 pc;
            pb.error(T[k], &pb.pts[3 * j], obs_px + 2 * o, e, &pc);
            const double e2 = e[0] * e[0] + e[1] * e[1];
            double w = 1.0;  // rho[1]
            if (pb.delta > 0 && e2 > pb.delta * pb.delta) w = pb.delta / std::sqrt(e2);
            const double x = pc.x, y = pc.y, z = pc.z, z_2 = z * z;
            const double fx = pb.cam.fx, fy = pb.cam.fy;
            // linearizeOplus (G2oTypes.h:93-132)
            double tmp[2][3] = {{fx, 0, -x / z * fx}, {0, fy, -y / z * fy}};
            double Jl[2][3], Jp[2][6];
            for (int r = 0; r < 2; ++r)
                for (int c = 0; c < 3; ++c)
                    Jl[r][c] = -1. / z * (tmp[r][0] * R[k].m[0][c] + tmp[r][1] * R[k].m[1][c] + tmp[r][2] * R[k].m[2][c]);
            Jp[0][0] = x * y / z_2 * fx; Jp[0][1] = -(1 + (x * x / z_2)) * fx; Jp[0][2] = y / z * fx;
            Jp[0][3] = -1. / z * fx; Jp[0][4] = 0; Jp[0][5] = x / z_2 * fx;
            Jp[1][0] = (1 + y * y / z_2) * fy; Jp[1][1] = -x * y / z_2 * fy; Jp[1][2] = -x / z * fy;
            Jp[1][3] = 0; Jp[1][4] = -1. / z * fy; Jp[1][5] = y / z_2 * fy;
            // constructQuadraticForm with the robust weight: H += w J^T J, b += -w J^T e
            for (int a = 0; a < 3; ++a) {
                for (int b = 0; b < 3; ++b) Hll[9 * (size_t)j + 3 * a + b] += w * (Jl[0][a] * Jl[0][b] + Jl[1][a] * Jl[1][b]);
                bl[3 * (size_t)j + a] += -w * (Jl[0][a] * e[0] + Jl[1][a] * e[1]);
            }
            const int fi = pb.free_index[k];
            if (fi >= 0) {
                for (int a = 0; a < 6; ++a) {
                    for (int b = 0; b < 6; ++b) Hpp[36 * (size_t)fi + 6 * a + b] += w * (Jp[0][a] * Jp[0][b] + Jp[1][a] * Jp[1][b]);
                    bp[6 * fi + a] += -w * (Jp[0][a] * e[0] + Jp[1][a] * e[1]);
                    for (int b = 0; b < 3; ++b) Hpl[18 * (size_t)o + 3 * a + b] = w * (Jp[0][a] * Jl[0][b] + Jp[1][a] * Jl[1][b]);
                }
            }
        }
        return chi;
    };
    // g2o linearises before the first iteration: chi2_initial and computeLambdaInit (tau * max |diag H| over all free
    // vertices) exist even when max_iters = 0, which then reports them and returns the input
    chi_first = chi_last = build_system();
    {
        double mx = 0;
        for (int i = 0; i < np; ++i)
            for (int a = 0; a < 6; ++a) mx = std::max(mx, std::fabs(Hpp[36 * (size_t)i + 7 * a]));
        for (int j = 0; j < n_pt; ++j)
            for (int a = 0; a < 3; ++a) mx = std::max(mx, std::fabs(Hll[9 * (size_t)j + 4 * a]));
        lambda = prm->tau * mx;
    }
    for (int iteration = 0; iteration < prm->max_iters; ++iteration) {
        double currentChi = iteration == 0 ? chi_first : build_system();
        double rho = 0;
        int qmax = 0;
        do {
            const std::vector<double> poses_backup = pb.poses, pts_backup = pb.pts;  // _optimizer->push()
            // Schur complement with lambda on every diagonal entry
            std::vector<double> S((size_t)dimp * dimp, 0.0), bs(bp);
            for (int i = 0; i < np; ++i)
                for (int a = 0; a < 6; ++a)
                    for (int b = 0; b < 6; ++b) S[(size_t)(6 * i + a) * dimp + 6 * i + b] = Hpp[36 * (size_t)i + 6 * a + b] + (a == b ? lambda : 0.0);
            std::vector<double> Dinv_all((size_t)9 * n_pt);
            for (int j = 0; j < n_pt; ++j) {
                double D[3][3], Di[3][3];
                for (int a = 0; a < 3; ++a)
                    for (int b = 0; b < 3; ++b) D[a][b] = Hll[9 * (size_t)j + 3 * a + b] + (a == b ? lambda : 0.0);
                inverse3d(D, Di);
                std::memcpy(&Dinv_all[9 * (size_t)j], Di, sizeof(Di));
                for (int o1 : obs_of_pt[j]) {
                    const int f1 = pb.free_index[kf_idx[o1]];
                    if (f1 < 0) continue;
                    double BD[6][3];
                    for (int a = 0; a < 6; ++a)
                        for (int b = 0; b < 3; ++b)
                            BD[a][b] = Hpl[18 * (size_t)o1 + 3 * a] * Di[0][b] + Hpl[18 * (size_t)o1 + 3 * a + 1] * Di[1][b] +
                                       Hpl[18 * (size_t)o1 + 3 * a + 2] * Di[2][b];
                    for (int a = 0; a < 6; ++a)
                        bs[6 * f1 + a] -= BD[a][0] * bl[3 * (size_t)j] + BD[a][1] * bl[3 * (size_t)j + 1] + BD[a][2] * bl[3 * (size_t)j + 2];
                    for (int o2 : obs_of_pt[j]) {
                        const int f2 = pb.free_index[kf_idx[o2]];
                        if (f2 < 0) continue;
                        for (int a = 0; a < 6; ++a)
                            for (int b = 0; b < 6; ++b)
                                S[(size_t)(6 * f1 + a) * dimp + 6 * f2 + b] -= BD[a][0] * Hpl[18 * (size_t)o2 + 3 * b] +
                                                                              BD[a][1] * Hpl[18 * (size_t)o2 + 3 * b + 1] +
                                                                              BD[a][2] * Hpl[18 * (size_t)o2 + 3 * b + 2];
                    }
                }
            }
            std::vector<double> sol(bs);
            bool ok2 = dimp == 0 || cholesky_solve(S, sol, dimp);
            // a failed factorisation leaves sol unsolved: the trial's pose step is zero (the landmarks follow from it)
            if (ok2) xp = sol;
            else std::fill(xp.begin(), xp.end(), 0.0);
            for (int j = 0; j < n_pt; ++j) {
                double r[3] = {bl[3 * (size_t)j], bl[3 * (size_t)j + 1], bl[3 * (size_t)j + 2]};
                for (int o1 : obs_of_pt[j]) {
                    const int f1 = pb.free_index[kf_idx[o1]];
                    if (f1 < 0) continue;
                    for (int b = 0; b < 3; ++b)
                        for (int a = 0; a < 6; ++a) r[b] -= Hpl[18 * (size_t)o1 + 3 * a + b] * xp[6 * f1 + a];
                }
                const double* Di = &Dinv_all[9 * (size_t)j];
                for (int a = 0; a < 3; ++a) xl[3 * (size_t)j + a] = Di[3 * a] * r[0] + Di[3 * a + 1] * r[1] + Di[3 * a + 2] * r[2];
            }
            // _optimizer->update(x): oplusImpl
            for (int k = 0; k < n_kf; ++k) {
                const int fi = pb.free_index[k];
                if (fi < 0) continue;
                const double* u = &xp[6 * fi];
                const double v[6] = {u[3], u[4], u[5], u[0], u[1], u[2]};
                const SE3 Tn = SE3::exp(v) * pose_from_g2o(&pb.poses[6 * k]);
                double lg[6];
                Tn.log(lg);
                double* est = &pb.poses[6 * k];
                est[0] = lg[3]; est[1] = lg[4]; est[2] = lg[5]; est[3] = lg[0]; est[4] = lg[1]; est[5] = lg[2];
            }
            for (size_t i = 0; i < 3 * (size_t)n_pt; ++i) pb.pts[i] += xl[i];
            double tempChi = pb.robust_chi2(pb.poses, pb.pts);
            if (!ok2) tempChi = 1.7976931348623157e308;
            rho = currentChi - tempChi;
            double scale = 0;  // computeScale: sum_j x_j (lambda x_j + b_j)
            for (int i = 0; i < dimp; ++i) scale += xp[i] * (lambda * xp[i] + bp[i]);
            for (size_t i = 0; i < 3 * (size_t)n_pt; ++i) scale += xl[i] * (lambda * xl[i] + bl[i]);
            scale += 1e-3;
            rho /= scale;
            if (rho > 0 && std::isfinite(tempChi)) {
                double alpha = 1. - std::pow((2 * rho - 1), 3);
                alpha = std::min(alpha, 2. / 3.);
                const double scaleFactor = std::max(1. / 3., alpha);
                lambda *= scaleFactor;
                ni = 2;
                currentChi = tempChi;
            } else {
                lambda *= ni;
                ni *= 2;
                pb.poses = poses_backup;  // _optimizer->pop()
                pb.pts = pts_backup;
            }
            ++qmax;
            ++trials_total;
        } while (rho < 0 && qmax < prm->max_trials);
        ++iters;
        chi_last = currentChi;
        if (qmax == prm->max_trials || rho == 0) break;  // OptimizationAlgorithm::Terminate
    }

    // BA.cpp:505-515: edges with chi2 > 5.991 are outliers (plain |e|^2, not the Huber cost)
    int n_out = 0;
    {
        std::vector<SE3> T(n_kf);
        for (int k = 0; k < n_kf; ++k) T[k] = pose_from_g2o(&pb.poses[6 * k]);
        for (int o = 0; o < n_obs; ++o) {
            double e[2];
            pb.error(T[kf_idx[o]], &pb.pts[3 * pt_idx[o]], obs_px + 2 * o, e);
            outlier[o] = (e[0] * e[0] + e[1] * e[1] > prm->chi2_outlier) ? 1 : 0;
            n_out += outlier[o];
        }
    }
    std::memcpy(poses, pb.poses.data(), sizeof(double) * 6 * n_kf);
    std::memcpy(pts, pb.pts.data(), sizeof(double) * 3 * n_pt);
    if (stats) {
        stats->iters = iters;
        stats->lm_trials = trials_total;
        stats->chi2_initial = chi_first;
        stats->chi2_final = chi_last;
        stats->lambda_final = lambda;
        stats->n_outliers = n_out;
    }
    return iters;
}

// ---- pose-only refinement (Ceres restatement) -------------------------------------------------------------
namespace {

// forward-mode dual number with 6 partials: what ceres::AutoDiffCostFunction<.., 2, 6> evaluates
struct Jet6 {
    double a;
    double v[6];
};
inline Jet6 jc(double c) {
    Jet6 r{c, {0, 0, 0, 0, 0, 0}};
    return r;
}
inline Jet6 operator+(const Jet6& x, const Jet6& y) {
    Jet6 r{x.a + y.a, {}};
    for (int i = 0; i < 6; ++i) r.v[i] = x.v[i] + y.v[i];
    return r;
}
inline Jet6 operator-(const Jet6& x, const Jet6& y) {
    Jet6 r{x.a - y.a, {}};
    for (int i = 0; i < 6; ++i) r.v[i] = x.v[i] - y.v[i];
    return r;
}
inline Jet6 operator*(const Jet6& x, const Jet6& y) {
    Jet6 r{x.a * y.a, {}};
    for (int i = 0; i < 6; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a;
    return r;
}
inline Jet6 operator/(const Jet6& x, const Jet6& y) {
    const double inv = 1.0 / y.a, q = x.a * inv;
    Jet6 r{q, {}};
    for (int i = 0; i < 6; ++i) r.v[i] = (x.v[i] - q * y.v[i]) * inv;
    return r;
}
inline Jet6 jsqrt(const Jet6& x) {
    const double s = std::sqrt(x.a), d = 1.0 / (2.0 * s);
    Jet6 r{s, {}};
    for (int i = 0; i < 6; ++i) r.v[i] = x.v[i] * d;
    return r;
}
inline Jet6 jcos(const Jet6& x) {
    const double c = std::cos(x.a), s = -std::sin(x.a);
    Jet6 r{c, {}};
    for (int i = 0; i < 6; ++i) r.v[i] = s * x.v[i];
    return r;
}
inline Jet6 jsin(const Jet6& x) {
    const double s = std::sin(x.a), c = std::cos(x.a);
    Jet6 r{s, {}};
    for (int i = 0; i < 6; ++i) r.v[i] = c * x.v[i];
    return r;
}

// ceres::AngleAxisRotatePoint on jets (ceres/rotation.h)
void angle_axis_rotate(const Jet6 aa[3], const Jet6 pt[3], Jet6 out[3]) {
    const Jet6 theta2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
    if (theta2.a > 2.2204460492503131e-16) {
        const Jet6 theta = jsqrt(theta2);
        const Jet6 costheta = jcos(theta), sintheta = jsin(theta);
        const Jet6 inv = jc(1.0) / theta;
        const Jet6 w[3] = {aa[0] * inv, aa[1] * inv, aa[2] * inv};
        const Jet6 wxp[3] = {w[1] * pt[2] - w[2] * pt[1], w[2] * pt[0] - w[0] * pt[2], w[0] * pt[1] - w[1] * pt[0]};
        const Jet6 tmp = (w[0] * pt[0] + w[1] * pt[1] + w[2] * pt[2]) * (jc(1.0) - costheta);
        for (int i = 0; i < 3; ++i) out[i] = pt[i] * costheta + wxp[i] * sintheta + w[i] * tmp;
    } else {
        const Jet6 wxp[3] = {aa[1] * pt[2] - aa[2] * pt[1], aa[2] * pt[0] - aa[0] * pt[2], aa[0] * pt[1] - aa[1] * pt[0]};
        for (int i = 0; i < 3; ++i) out[i] = pt[i] + wxp[i];
    }
}

struct PoseOnly {
    int n;
    const double* pw;            // world points
    std::vector<double> ptcam;   // normalised observations (Pixel2Camera2D)
    std::vector<uint8_t> enable;

    // evaluates residuals (2n) and, optionally, the Jacobian (2n x 6); false = a residual block returned false
    bool evaluate(const double pose[6], std::vector<double>& r, std::vector<double>* J) const {
        Jet6 P[6];
        for (int i = 0; i < 6; ++i) {
            P[i] = jc(pose[i]);
            P[i].v[i] = 1.0;
        }
        const Jet6 rot[3] = {P[3], P[4], P[5]};
        for (int i = 0; i < n; ++i) {
            double* ri = &r[2 * i];
            double* Ji = J ? &(*J)[12 * (size_t)i] : nullptr;
            if (!enable[i]) {
                ri[0] = ri[1] = 0;
                if (Ji) std::memset(Ji, 0, sizeof(double) * 12);
                continue;
            }
            const Jet6 X[3] = {jc(pw[3 * i]), jc(pw[3 * i + 1]), jc(pw[3 * i + 2])};
            Jet6 p[3];
            angle_axis_rotate(rot, X, p);
            p[0] = p[0] + P[0];
            p[1] = p[1] + P[1];
            p[2] = p[2] + P[2];
            if (p[2].a < 0) return false;  // the functor returns false: Ceres treats the evaluation as failed
            const Jet6 r0 = jc(ptcam[2 * i]) - p[0] / p[2], r1 = jc(ptcam[2 * i + 1]) - p[1] / p[2];
            ri[0] = r0.a;
            ri[1] = r1.a;
            if (Ji)
                for (int k = 0; k < 6; ++k) {
                    Ji[k] = r0.v[k];
                    Ji[6 + k] = r1.v[k];
                }
        }
        return true;
    }
};

// Ceres TrustRegionMinimizer + LevenbergMarquardtStrategy with default Solver::Options, dense 6x6 normal equations
void ceres_lm(const PoseOnly& pb, double pose[6]) {
    const int m = 2 * pb.n;
    std::vector<double> r(m), rn(m), J((size_t)m * 6);
    if (!pb.evaluate(pose, r, &J)) return;  // initial evaluation failed: Solve() returns FAILURE, parameters untouched
    double cost = 0;
    for (double v : r) cost += v * v;
    cost *= 0.5;
    // Jacobi scaling computed once at the start
    double scale[6];
    for (int k = 0; k < 6; ++k) {
        double s = 0;
        for (int i = 0; i < m; ++i) s += J[(size_t)i * 6 + k] * J[(size_t)i * 6 + k];
        scale[k] = 1.0 / (1.0 + std::sqrt(s));
    }
    auto gradient_max = [&](const std::vector<double>& Jm, const std::vector<double>& rm) {
        double g = 0;
        for (int k = 0; k < 6; ++k) {
            double s = 0;
            for (int i = 0; i < m; ++i) s += Jm[(size_t)i * 6 + k] * rm[i];
            g = std::max(g, std::fabs(s));
        }
        return g;
    };
    if (gradient_max(J, r) <= 1e-10) return;
    double radius = 1e4, decrease_factor = 2.0;
    for (int iter = 0; iter < 50; ++iter) {
        // scaled Jacobian Js = J diag(scale); normal equations (Js^T Js + D^T D) y = -Js^T r
        std::vector<double> A(36, 0.0), g(6, 0.0);
        for (int i = 0; i < m; ++i) {
            double row[6];
            for (int k = 0; k < 6; ++k) row[k] = J[(size_t)i * 6 + k] * scale[k];
            for (int a = 0; a < 6; ++a) {
                g[a] += row[a] * r[i];
                for (int b = 0; b < 6; ++b) A[a * 6 + b] += row[a] * row[b];
            }
        }
        double diag[6];
        for (int k = 0; k < 6; ++k) diag[k] = std::min(std::max(A[k * 6 + k], 1e-6), 1e32);
        std::vector<double> An(A), y(6);
        for (int k = 0; k < 6; ++k) {
            An[k * 6 + k] += diag[k] / radius;  // lm_diagonal^2 = diagonal / radius
            y[k] = -g[k];
        }
        bool step_ok = cholesky_solve(An, y, 6);
        double model_cost_change = 0;
        if (step_ok) {
            // model_cost_change = -(Js y)^T (r + Js y / 2)
            for (int i = 0; i < m; ++i) {
                double jy = 0;
                for (int k = 0; k < 6; ++k) jy += J[(size_t)i * 6 + k] * scale[k] * y[k];
                model_cost_change -= jy * (r[i] + jy / 2);
            }
            step_ok = model_cost_change > 0;
        }
        bool accepted = false;
        double delta[6], new_cost = 0, step_norm = 0, x_norm = 0;
        if (step_ok) {
            double cand[6];
            for (int k = 0; k < 6; ++k) {
                delta[k] = y[k] * scale[k];
                cand[k] = pose[k] + delta[k];
                step_norm += delta[k] * delta[k];
                x_norm += pose[k] * pose[k];
            }
            step_norm = std::sqrt(step_norm);
            x_norm = std::sqrt(x_norm);
            if (pb.evaluate(cand, rn, nullptr)) {
                for (double v : rn) new_cost += v * v;
                new_cost *= 0.5;
                const double relative_decrease = (cost - new_cost) / model_cost_change;
                if (relative_decrease > 1e-3) {
                    accepted = true;
                    // parameter tolerance (checked before the step is taken)
                    if (step_norm <= 1e-8 * (x_norm + 1e-8)) return;
                    const double cost_change = cost - new_cost;
                    for (int k = 0; k < 6; ++k) pose[k] = cand[k];
                    pb.evaluate(pose, r, &J);
                    const double old_cost = cost;
                    cost = new_cost;
                    if (std::fabs(cost_change) <= 1e-6 * old_cost) return;   // function tolerance
                    if (gradient_max(J, r) <= 1e-10) return;                 // gradient tolerance
                    radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * relative_decrease - 1.0, 3));
                    radius = std::min(1e16, radius);
                    decrease_factor = 2.0;
                }
            }
        }
        if (!accepted) {
            radius = radius / decrease_factor;
            decrease_factor *= 2.0;
            if (radius < 1e-32) return;
        }
    }
}

}  // namespace

extern "C" int ora_pose_only(const ora_camera* camp, int n, const double* pt_world, const double* px, double* T_cw,
                             uint8_t* inlier, double* depth) {
    const float fx = camp->fx, fy = camp->fy, cx = camp->cx, cy = camp->cy;
    SE3 T = SE3::from_mat(T_cw);
    // pose = [t; so3.log()] (BA.cpp:190-193)
    double pose[6], backup[6];
    const V3 rlog = T.so3.log();
    pose[0] = T.t.x; pose[1] = T.t.y; pose[2] = T.t.z; pose[3] = rlog.x; pose[4] = rlog.y; pose[5] = rlog.z;
    std::memcpy(backup, pose, sizeof(pose));
    PoseOnly pb;
    pb.n = n;
    pb.pw = pt_world;
    pb.ptcam.resize(2 * (size_t)n);
    pb.enable.assign(n, 1);
    for (int i = 0; i < n; ++i) {  // Pixel2Camera2D
        pb.ptcam[2 * i] = (px[2 * i] - cx) / fx;
        pb.ptcam[2 * i + 1] = (px[2 * i + 1] - cy) / fy;
        inlier[i] = 1;    // Feature::_bad defaults to false
        depth[i] = -1;
    }
    const float chi2Mono = 5.991f;
    int cntInlier = 0;
    for (int it = 0; it < 4; ++it) {
        std::memcpy(pose, backup, sizeof(pose));
        ceres_lm(pb, pose);
        cntInlier = 0;
        for (int i = 0; i < n; ++i) {
            // classification uses current->_TCW, which is only refreshed at the END of a round (BA.cpp:251)
            const V3 pc = T * V3{pt_world[3 * i], pt_world[3 * i + 1], pt_world[3 * i + 2]};
            const double u = fx * pc.x / pc.z + cx, v = fy * pc.y / pc.z + cy;
            const double dx = u - px[2 * i], dy = v - px[2 * i + 1];
            const double error2 = dx * dx + dy * dy;
            if (error2 > chi2Mono) {
                inlier[i] = 0;
                pb.enable[i] = 0;
            } else {
                depth[i] = pc.z;
                inlier[i] = 1;
                ++cntInlier;
                pb.enable[i] = 1;
            }
        }
        if (cntInlier < 10) break;
        T.so3 = SO3::exp(V3{pose[3], pose[4], pose[5]});
        T.t = V3{pose[0], pose[1], pose[2]};
    }
    T.to_mat(T_cw);
    return cntInlier;
}

// ---- ba::LocalBA, the Ceres twin of the local BA (reference src/Algorithm/BA.cpp:324-384) ---------------------
//   CeresReprojectionError           reference include/ygz/Ceres/CeresReprojectionError.h:33-69
//       pose = [t; angle-axis], residual = pt_cam - p / p.z in NORMALISED image coordinates, AutoDiff<2, 6, 3>
//   CeresReprojectionErrorPointOnly  reference include/ygz/Ceres/CeresReprojectionErrorPointOnly.h:14-67
//       the same residual with the pose held constant: used for the key-frame with _keyframe_id == 0 (BA.cpp:340-349)
//       = `fixed[k] != 0` here; observations in frames outside the local set are not added at all (BA.cpp:338).
// Solver: default ceres::Solver::Options -- trust-region Levenberg-Marquardt, Jacobi scaling, no loss function, <= 50
// iterations, function / gradient / parameter tolerances 1e-6 / 1e-10 / 1e-8, initial radius 1e4.  The sparse normal
// Cholesky of the full system is restated as its exact equivalent, the Schur complement onto the free poses.
namespace {

struct Jet9 {
    double a;
    double v[9];
};
inline Jet9 j9c(double c) {
    Jet9 r{c, {}};
    return r;
}
inline Jet9 operator+(const Jet9& x, const Jet9& y) {
    Jet9 r{x.a + y.a, {}};
    for (int i = 0; i < 9; ++i) r.v[i] = x.v[i] + y.v[i];
    return r;
}
inline Jet9 operator-(const Jet9& x, const Jet9& y) {
    Jet9 r{x.a - y.a, {}};
    for (int i = 0; i < 9; ++i) r.v[i] = x.v[i] - y.v[i];
    return r;
}
inline Jet9 operator*(const Jet9& x, const Jet9& y) {
    Jet9 r{x.a * y.a, {}};
    for (int i = 0; i < 9; ++i) r.v[i] = x.a * y.v[i] + x.v[i] * y.a;
    return r;
}
inline Jet9 operator/(const Jet9& x, const Jet9& y) {
    const double inv = 1.0 / y.a, q = x.a * inv;
    Jet9 r{q, {}};
    for (int i = 0; i < 9; ++i) r.v[i] = (x.v[i] - q * y.v[i]) * inv;
    return r;
}

// ceres::AngleAxisRotatePoint on 9-partial jets
void angle_axis_rotate9(const Jet9 aa[3], const Jet9 pt[3], Jet9 out[3]) {
    const Jet9 theta2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
    if (theta2.a > 2.2204460492503131e-16) {
        const double th = std::sqrt(theta2.a), dth = 1.0 / (2.0 * th);
        Jet9 theta{th, {}}, costheta{std::cos(th), {}}, sintheta{std::sin(th), {}};
        for (int i = 0; i < 9; ++i) {
            theta.v[i] = theta2.v[i] * dth;
            costheta.v[i] = -sintheta.a * theta.v[i];
            sintheta.v[i] = costheta.a * theta.v[i];
        }
        const Jet9 inv = j9c(1.0) / theta;
        const Jet9 w[3] = {aa[0] * inv, aa[1] * inv, aa[2] * inv};
        const Jet9 wxp[3] = {w[1] * pt[2] - w[2] * pt[1], w[2] * pt[0] - w[0] * pt[2], w[0] * pt[1] - w[1] * pt[0]};
        const Jet9 tmp = (w[0] * pt[0] + w[1] * pt[1] + w[2] * pt[2]) * (j9c(1.0) - costheta);
        for (int i = 0; i < 3; ++i) out[i] = pt[i] * costheta + wxp[i] * sintheta + w[i] * tmp;
    } else {
        const Jet9 wxp[3] = {aa[1] * pt[2] - aa[2] * pt[1], aa[2] * pt[0] - aa[0] * pt[2], aa[0] * pt[1] - aa[1] * pt[0]};
        for (int i = 0; i < 3; ++i) out[i] = pt[i] + wxp[i];
    }
}

struct CeresBA {
    int n_kf, n_pt, n_obs, np;
    const int32_t *kf_idx, *pt_idx;
    std::vector<int> free_index;
    std::vector<double> ptcam;
    std::vector<std::vector<int>> obs_of_pt;

    // residuals (2 per observation) and, optionally, the Jacobian blocks Jp (2x6) / Jl (2x3) per observation
    void evaluate(const std::vector<double>& P, const std::vector<double>& X, std::vector<double>& r, std::vector<double>* Jp,
                  std::vector<double>* Jl) const {
        for (int o = 0; o < n_obs; ++o) {
            const double* pose = &P[6 * (size_t)kf_idx[o]];
            const double* x = &X[3 * (size_t)pt_idx[o]];
            Jet9 T[6], Xj[3];
            for (int i = 0; i < 6; ++i) {
                T[i] = j9c(pose[i]);
                T[i].v[i] = 1.0;
            }
            for (int i = 0; i < 3; ++i) {
                Xj[i] = j9c(x[i]);
                Xj[i].v[6 + i] = 1.0;
            }
            const Jet9 rot[3] = {T[3], T[4], T[5]};
            Jet9 p[3];
            angle_axis_rotate9(rot, Xj, p);
            p[0] = p[0] + T[0];
            p[1] = p[1] + T[1];
            p[2] = p[2] + T[2];
            const Jet9 r0 = j9c(ptcam[2 * (size_t)o]) - p[0] / p[2], r1 = j9c(ptcam[2 * (size_t)o + 1]) - p[1] / p[2];
            r[2 * (size_t)o] = r0.a;
            r[2 * (size_t)o + 1] = r1.a;
            if (Jp)
                for (int k = 0; k < 6; ++k) {
                    (*Jp)[12 * (size_t)o + k] = r0.v[k];
                    (*Jp)[12 * (size_t)o + 6 + k] = r1.v[k];
                }
            if (Jl)
                for (int k = 0; k < 3; ++k) {
                    (*Jl)[6 * (size_t)o + k] = r0.v[6 + k];
                    (*Jl)[6 * (size_t)o + 3 + k] = r1.v[6 + k];
                }
        }
    }
};

}  // namespace

static int ceres_ba_impl(const ora_camera* camp, int n_kf, double* poses, const uint8_t* fixed, int n_pt, double* pts,
                         int n_obs, const int32_t* kf_idx, const int32_t* pt_idx, const double* obs_px, int max_iters,
                         double huber_a, const uint8_t* loss_mask, ora_ceres_stats* stats);

extern "C" int ora_local_ba_ceres(const ora_camera* camp, int n_kf, double* poses, const uint8_t* fixed, int n_pt, double* pts,
                                  int n_obs, const int32_t* kf_idx, const int32_t* pt_idx, const double* obs_px, int max_iters,
                                  double huber_a, ora_ceres_stats* stats) {
    return ceres_ba_impl(camp, n_kf, poses, fixed, n_pt, pts, n_obs, kf_idx, pt_idx, obs_px, max_iters, huber_a, nullptr, stats);
}

// loss_mask (may be NULL = every block): the residual blocks that carry ceres::HuberLoss(huber_a); the others have no loss
// (AddResidualBlock(cost, inlier ? nullptr : new HuberLoss(0.1), ...), BA.cpp:38-56)
static int ceres_ba_impl(const ora_camera* camp, int n_kf, double* poses, const uint8_t* fixed, int n_pt, double* pts,
                         int n_obs, const int32_t* kf_idx, const int32_t* pt_idx, const double* obs_px, int max_iters,
                         double huber_a, const uint8_t* loss_mask, ora_ceres_stats* stats) {
    const float fx = camp->fx, fy = camp->fy, cx = camp->cx, cy = camp->cy;
    CeresBA pb;
    pb.n_kf = n_kf; pb.n_pt = n_pt; pb.n_obs = n_obs;
    pb.kf_idx = kf_idx; pb.pt_idx = pt_idx;
    pb.free_index.assign(n_kf, -1);
    pb.np = 0;
    for (int k = 0; k < n_kf; ++k)
        if (!fixed[k]) pb.free_index[k] = pb.np++;
    const int np = pb.np, dimp = 6 * np;
    pb.ptcam.resize(2 * (size_t)n_obs);
    for (int o = 0; o < n_obs; ++o) {  // PinholeCamera::Pixel2Camera2D (float intrinsics, double maths)
        pb.ptcam[2 * (size_t)o] = (obs_px[2 * (size_t)o] - cx) / fx;
        pb.ptcam[2 * (size_t)o + 1] = (obs_px[2 * (size_t)o + 1] - cy) / fy;
    }
    pb.obs_of_pt.assign(n_pt, {});
    for (int o = 0; o < n_obs; ++o) pb.obs_of_pt[pt_idx[o]].push_back(o);

    std::vector<double> P(poses, poses + 6 * (size_t)n_kf), X(pts, pts + 3 * (size_t)n_pt);
    std::vector<double> r(2 * (size_t)n_obs), rn(2 * (size_t)n_obs), Jp(12 * (size_t)n_obs), Jl(6 * (size_t)n_obs);
    std::vector<double> Hpp((size_t)np * 36), gp(dimp), Hll((size_t)n_pt * 9), gl(3 * (size_t)n_pt), Hpl(18 * (size_t)n_obs);
    double cost = 0;

    // ceres::HuberLoss(a) through the Corrector (ceres/corrector.cc): rho'' <= 0 for Huber, so residuals and Jacobians of
    // a block are both scaled by sqrt(rho') -- i.e. the block enters the normal equations with the weight w = rho' --
    // and the cost is 1/2 sum rho(s), s = |r|^2: rho = s, w = 1 for s <= a^2, else rho = 2 a sqrt(s) - a^2, w = a / sqrt(s)
    std::vector<double> wgt(n_obs, 1.0);
    auto robust_cost = [&](const std::vector<double>& res, std::vector<double>* w) {
        double c = 0;
        for (int o = 0; o < n_obs; ++o) {
            const double s2 = res[2 * (size_t)o] * res[2 * (size_t)o] + res[2 * (size_t)o + 1] * res[2 * (size_t)o + 1];
            if (huber_a > 0 && (!loss_mask || loss_mask[o]) && s2 > huber_a * huber_a) {
                const double rt = std::sqrt(s2);
                c += 2 * huber_a * rt - huber_a * huber_a;
                if (w) (*w)[o] = huber_a / rt;
            } else {
                c += s2;
                if (w) (*w)[o] = 1.0;
            }
        }
        return 0.5 * c;
    };
    auto build = [&]() {  // normal-equation blocks of the UNSCALED (loss-corrected) Jacobian and the gradient g = J^T r
        pb.evaluate(P, X, r, &Jp, &Jl);
        cost = robust_cost(r, &wgt);
        std::fill(Hpp.begin(), Hpp.end(), 0.0); std::fill(gp.begin(), gp.end(), 0.0);
        std::fill(Hll.begin(), Hll.end(), 0.0); std::fill(gl.begin(), gl.end(), 0.0);
        for (int o = 0; o < n_obs; ++o) {
            const int j = pt_idx[o], fi = pb.free_index[kf_idx[o]];
            const double* J0 = &Jl[6 * (size_t)o];
            const double* J1 = J0 + 3;
            const double e0 = r[2 * (size_t)o], e1 = r[2 * (size_t)o + 1], w = wgt[o];
            for (int a = 0; a < 3; ++a) {
                for (int b = 0; b < 3; ++b) Hll[9 * (size_t)j + 3 * a + b] += w * (J0[a] * J0[b] + J1[a] * J1[b]);
                gl[3 * (size_t)j + a] += w * (J0[a] * e0 + J1[a] * e1);
            }
            if (fi >= 0) {
                const double* Q0 = &Jp[12 * (size_t)o];
                const double* Q1 = Q0 + 6;
                for (int a = 0; a < 6; ++a) {
                    for (int b = 0; b < 6; ++b) Hpp[36 * (size_t)fi + 6 * a + b] += w * (Q0[a] * Q0[b] + Q1[a] * Q1[b]);
                    gp[6 * fi + a] += w * (Q0[a] * e0 + Q1[a] * e1);
                    for (int b = 0; b < 3; ++b) Hpl[18 * (size_t)o + 3 * a + b] = w * (Q0[a] * J0[b] + Q1[a] * J1[b]);
                }
            }
        }
    };
    auto gradient_max = [&]() {
        double g = 0;
        for (double v : gp) g = std::max(g, std::fabs(v));
        for (double v : gl) g = std::max(g, std::fabs(v));
        return g;
    };

    build();
    const double cost_initial = cost;
    // Jacobi scaling, computed once from the initial Jacobian: 1 / (1 + ||column||)
    std::vector<double> sp(dimp), sl(3 * (size_t)n_pt);
    for (int i = 0; i < np; ++i)
        for (int a = 0; a < 6; ++a) sp[6 * i + a] = 1.0 / (1.0 + std::sqrt(Hpp[36 * (size_t)i + 7 * a]));
    for (int j = 0; j < n_pt; ++j)
        for (int a = 0; a < 3; ++a) sl[3 * (size_t)j + a] = 1.0 / (1.0 + std::sqrt(Hll[9 * (size_t)j + 4 * a]));

    int iters = 0, n_success = 0, termination = 0;  // 0 = max iterations, 1 = gradient, 2 = parameter, 3 = function, 4 = radius
    double radius = 1e4, decrease_factor = 2.0;
    if (gradient_max() <= 1e-10) termination = 1;
    std::vector<double> xp(dimp), xl(3 * (size_t)n_pt), Pc, Xc;
    for (int iter = 0; termination == 0 && iter < max_iters; ++iter) {
        ++iters;
        // (Js^T Js + D / radius) y = -Js^T r with D = clamp(diag(Js^T Js), 1e-6, 1e32), delta = S y
        //   <=>  (H + diag(d)) delta = -g,  d_k = clamp(s_k^2 H_kk) / (radius s_k^2)
        auto damp = [&](double hkk, double s) { return std::min(std::max(s * s * hkk, 1e-6), 1e32) / radius / (s * s); };
        std::vector<double> S((size_t)dimp * dimp, 0.0), bs(dimp);
        for (int i = 0; i < np; ++i)
            for (int a = 0; a < 6; ++a) {
                for (int b = 0; b < 6; ++b) S[(size_t)(6 * i + a) * dimp + 6 * i + b] = Hpp[36 * (size_t)i + 6 * a + b];
                S[(size_t)(6 * i + a) * dimp + 6 * i + a] += damp(Hpp[36 * (size_t)i + 7 * a], sp[6 * i + a]);
                bs[6 * i + a] = -gp[6 * i + a];
            }
        std::vector<double> Dinv_all(9 * (size_t)n_pt);
        for (int j = 0; j < n_pt; ++j) {
            double D[3][3], Di[3][3];
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) D[a][b] = Hll[9 * (size_t)j + 3 * a + b];
            for (int a = 0; a < 3; ++a) D[a][a] += damp(Hll[9 * (size_t)j + 4 * a], sl[3 * (size_t)j + a]);
            inverse3d(D, Di);
            std::memcpy(&Dinv_all[9 * (size_t)j], Di, sizeof(Di));
            for (int o1 : pb.obs_of_pt[j]) {
                const int f1 = pb.free_index[kf_idx[o1]];
                if (f1 < 0) continue;
                double BD[6][3];
                for (int a = 0; a < 6; ++a)
                    for (int b = 0; b < 3; ++b)
                        BD[a][b] = Hpl[18 * (size_t)o1 + 3 * a] * Di[0][b] + Hpl[18 * (size_t)o1 + 3 * a + 1] * Di[1][b] +
                                   Hpl[18 * (size_t)o1 + 3 * a + 2] * Di[2][b];
                for (int a = 0; a < 6; ++a)
                    bs[6 * f1 + a] -= BD[a][0] * -gl[3 * (size_t)j] + BD[a][1] * -gl[3 * (size_t)j + 1] + BD[a][2] * -gl[3 * (size_t)j + 2];
                for (int o2 : pb.obs_of_pt[j]) {
                    const int f2 = pb.free_index[kf_idx[o2]];
                    if (f2 < 0) continue;
                    for (int a = 0; a < 6; ++a)
                        for (int b = 0; b < 6; ++b)
                            S[(size_t)(6 * f1 + a) * dimp + 6 * f2 + b] -= BD[a][0] * Hpl[18 * (size_t)o2 + 3 * b] +
                                                                          BD[a][1] * Hpl[18 * (size_t)o2 + 3 * b + 1] +
                                                                          BD[a][2] * Hpl[18 * (size_t)o2 + 3 * b + 2];
                }
            }
        }
        std::vector<double> sol(bs);
        bool step_ok = dimp == 0 || cholesky_solve(S, sol, dimp);
        xp = sol;
        for (int j = 0; j < n_pt; ++j) {
            double rr[3] = {-gl[3 * (size_t)j], -gl[3 * (size_t)j + 1], -gl[3 * (size_t)j + 2]};
            for (int o1 : pb.obs_of_pt[j]) {
                const int f1 = pb.free_index[kf_idx[o1]];
                if (f1 < 0) continue;
                for (int b = 0; b < 3; ++b)
                    for (int a = 0; a < 6; ++a) rr[b] -= Hpl[18 * (size_t)o1 + 3 * a + b] * xp[6 * f1 + a];
            }
            const double* Di = &Dinv_all[9 * (size_t)j];
            for (int a = 0; a < 3; ++a) xl[3 * (size_t)j + a] = Di[3 * a] * rr[0] + Di[3 * a + 1] * rr[1] + Di[3 * a + 2] * rr[2];
        }
        double model_cost_change = 0;
        if (step_ok) {  // -(J delta)^T (r + J delta / 2)
            for (int o = 0; o < n_obs; ++o) {
                const int fi = pb.free_index[kf_idx[o]];
                for (int row = 0; row < 2; ++row) {
                    double jy = 0;
                    if (fi >= 0)
                        for (int k = 0; k < 6; ++k) jy += Jp[12 * (size_t)o + 6 * row + k] * xp[6 * fi + k];
                    for (int k = 0; k < 3; ++k) jy += Jl[6 * (size_t)o + 3 * row + k] * xl[3 * (size_t)pt_idx[o] + k];
                    model_cost_change -= wgt[o] * jy * (r[2 * (size_t)o + row] + jy / 2);
                }
            }
            step_ok = model_cost_change > 0;
        }
        bool accepted = false;
        if (step_ok) {
            Pc = P;
            Xc = X;
            double step_norm = 0, x_norm = 0;
            for (int k = 0; k < n_kf; ++k) {
                const int fi = pb.free_index[k];
                if (fi < 0) continue;
                for (int a = 0; a < 6; ++a) {
                    Pc[6 * (size_t)k + a] += xp[6 * fi + a];
                    step_norm += xp[6 * fi + a] * xp[6 * fi + a];
                    x_norm += P[6 * (size_t)k + a] * P[6 * (size_t)k + a];
                }
            }
            for (size_t i = 0; i < 3 * (size_t)n_pt; ++i) {
                Xc[i] += xl[i];
                step_norm += xl[i] * xl[i];
                x_norm += X[i] * X[i];
            }
            step_norm = std::sqrt(step_norm);
            x_norm = std::sqrt(x_norm);
            pb.evaluate(Pc, Xc, rn, nullptr, nullptr);
            const double new_cost = robust_cost(rn, nullptr);
            const double relative_decrease = (cost - new_cost) / model_cost_change;
            if (relative_decrease > 1e-3) {
                accepted = true;
                if (step_norm <= 1e-8 * (x_norm + 1e-8)) {  // parameter tolerance (checked before the step is taken)
                    termination = 2;
                    break;
                }
                const double old_cost = cost;
                P = Pc;
                X = Xc;
                build();
                ++n_success;
                if (std::fabs(old_cost - cost) <= 1e-6 * old_cost) {  // function tolerance
                    termination = 3;
                    break;
                }
                if (gradient_max() <= 1e-10) {
                    termination = 1;
                    break;
                }
                radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * relative_decrease - 1.0, 3));
                radius = std::min(1e16, radius);
                decrease_factor = 2.0;
            }
        }
        if (!accepted) {
            radius = radius / decrease_factor;
            decrease_factor *= 2.0;
            if (radius < 1e-32) {
                termination = 4;
                break;
            }
        }
    }
    std::memcpy(poses, P.data(), sizeof(double) * 6 * n_kf);
    std::memcpy(pts, X.data(), sizeof(double) * 3 * n_pt);
    if (stats) {
        stats->iters = iters;
        stats->successful_steps = n_success;
        stats->cost_initial = cost_initial;
        stats->cost_final = cost;
        stats->radius_final = radius;
        stats->termination = termination;
    }
    return iters;
}

// ba::TwoViewBACeres (src/Algorithm/BA.cpp:11-89): two-view bundle adjustment after the monocular initialisation.  The
// reference frame is fixed (CeresReprojectionErrorPointOnly blocks), the current pose [t; angle-axis] and every point are
// free; points that are not inliers are reset to (0, 0, 1) and their two blocks carry HuberLoss(0.1) (:31-56); afterwards a
// point is an inlier iff both pixel errors are <= 5.991 (squared) and both depths are positive (:70-84).
// The reference solves with DENSE_SCHUR + DOGLEG; Ceres is not in the reference tree, and this restatement (like the CUDA
// path) runs the same trust-region LEVENBERG-MARQUARDT as ba::LocalBA on the identical cost -- both strategies stop at the
// same local minimum up to the solver's function tolerance (1e-6), which the tests bound.
extern "C" int ora_two_view_ba(const ora_camera* cam, int n, const double* T_cw_ref, double* T_cw_cur, const double* px_ref,
                               const double* px_cur, uint8_t* inlier, double* pts, ora_ceres_stats* stats) {
    const SE3 Tr = SE3::from_mat(T_cw_ref), Tc = SE3::from_mat(T_cw_cur);
    double poses[12];
    const V3 lr = Tr.so3.log(), lc = Tc.so3.log();
    poses[0] = Tr.t.x; poses[1] = Tr.t.y; poses[2] = Tr.t.z; poses[3] = lr.x; poses[4] = lr.y; poses[5] = lr.z;
    poses[6] = Tc.t.x; poses[7] = Tc.t.y; poses[8] = Tc.t.z; poses[9] = lc.x; poses[10] = lc.y; poses[11] = lc.z;
    const uint8_t fixed[2] = {1, 0};
    std::vector<int32_t> kf(2 * (size_t)n), pt(2 * (size_t)n);
    std::vector<double> obs(4 * (size_t)n);
    std::vector<uint8_t> mask(2 * (size_t)n);
    for (int i = 0; i < n; ++i) {
        if (!inlier[i]) {
            pts[3 * i] = 0; pts[3 * i + 1] = 0; pts[3 * i + 2] = 1;
        }
        kf[2 * i] = 0; kf[2 * i + 1] = 1;
        pt[2 * i] = pt[2 * i + 1] = i;
        obs[4 * i] = px_ref[2 * i]; obs[4 * i + 1] = px_ref[2 * i + 1]; obs[4 * i + 2] = px_cur[2 * i]; obs[4 * i + 3] = px_cur[2 * i + 1];
        mask[2 * i] = mask[2 * i + 1] = inlier[i] ? 0 : 1;
    }
    ceres_ba_impl(cam, 2, poses, fixed, n, pts, 2 * n, kf.data(), pt.data(), obs.data(), 50, 0.1, mask.data(), stats);
    SE3 Tn;
    Tn.so3 = SO3::exp(V3{poses[9], poses[10], poses[11]});
    Tn.t = V3{poses[6], poses[7], poses[8]};
    Tn.to_mat(T_cw_cur);
    const float fx = cam->fx, fy = cam->fy, cx = cam->cx, cy = cam->cy;
    int n_in = 0;
    for (int i = 0; i < n; ++i) {
        const V3 X{pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        const V3 p1 = Tr * X, p2 = Tn * X;
        const double e1x = px_ref[2 * i] - (fx * p1.x / p1.z + cx), e1y = px_ref[2 * i + 1] - (fy * p1.y / p1.z + cy);
        const double e2x = px_cur[2 * i] - (fx * p2.x / p2.z + cx), e2y = px_cur[2 * i + 1] - (fy * p2.y / p2.z + cy);
        if (e1x * e1x + e1y * e1y > 5.991 || e2x * e2x + e2y * e2y > 5.991) inlier[i] = 0;
        else if (p1.z < 0 || p2.z < 0) inlier[i] = 0;
        else inlier[i] = 1;
        n_in += inlier[i];
    }
    return n_in;
}
