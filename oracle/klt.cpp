// oracle/klt.cpp -- Tracker::TrackKLT's optical flow (reference src/Algorithm/Tracker.cpp:65-113):
//     cv::calcOpticalFlowPyrLK(ref.pyr[0], cur.pyr[0], pt_ref, pt_cur, status, err, Size(21,21), 4,
//                              TermCriteria(COUNT+EPS, 30, 0.001), OPTFLOW_USE_INITIAL_FLOW)
// TEST INFRASTRUCTURE ONLY (see oracle.h).
// The arithmetic lives in OpenCV (video/lkpyramid.cpp), not in the reference tree: restated from the published
// algorithm (SURVEY.md appendix A.2) -- pyrDown pyramid, Scharr derivatives (3,10,3) with reflect-101 inside
// the image and zero outside, W_BITS = 14 fixed-point bilinear weights, int16 template scaled by 2^5,
// f32 normal equations scaled by 2^-20, min-eigenvalue test, <= 30 iterations, eps^2 stop, the |delta + prev| <
// 0.01 oscillation stop -- and pinned against cv2.calcOpticalFlowPyrLK in tests/test_oracle_klt.py (OpenCV's SIMD
// build sums the f32 terms in a different order, so the pin is a tolerance, not bit-exactness).
// The min-eigenvalue threshold is compared in float, as OpenCV stores it.  exact_sums = 1 adds the window sums in int64
// and converts each once to float, which is klt.cu's arithmetic: in that mode the GPU must match bit for bit.
#include <cmath>
#include <cstring>
#include <vector>

#include "oracle.h"

namespace {

inline int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * (n - 1) - i;
    return i;
}
inline int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }
inline int cv_round(float v) { return (int)lrintf(v); }

struct Lvl {
    std::vector<uint8_t> img;
    int w, h;
    int I(int x, int y) const { return img[(size_t)reflect101(y, h) * w + reflect101(x, w)]; }  // padded pyramid (REFLECT_101)
    // Scharr derivative image: reflect-101 inside calcSharrDeriv, constant 0 outside the image (derivBorder)
    void deriv(int x, int y, int* dx, int* dy) const {
        if (x < 0 || x >= w || y < 0 || y >= h) {
            *dx = *dy = 0;
            return;
        }
        auto P = [&](int xx, int yy) { return (int)img[(size_t)reflect101(yy, h) * w + reflect101(xx, w)]; };
        auto t0 = [&](int xx) { return (P(xx, y - 1) + P(xx, y + 1)) * 3 + P(xx, y) * 10; };
        auto t1 = [&](int xx) { return P(xx, y + 1) - P(xx, y - 1); };
        *dx = t0(x + 1) - t0(x - 1);
        *dy = (t1(x + 1) + t1(x - 1)) * 3 + t1(x) * 10;
    }
};

}  // namespace

extern "C" void ora_klt(const uint8_t* ref, const uint8_t* cur, int w, int h, int n, const float* ref_xy, float* cur_xy,
                        uint8_t* status, float* err, const ora_klt_params* p) {
    const int win = p->win;
    // buildOpticalFlowPyramid: stop when a level is not larger than the window
    std::vector<Lvl> A, B;
    {
        Lvl a{std::vector<uint8_t>(ref, ref + (size_t)w * h), w, h}, b{std::vector<uint8_t>(cur, cur + (size_t)w * h), w, h};
        A.push_back(a);
        B.push_back(b);
        for (int L = 1; L <= p->max_level; ++L) {
            const int pw = A.back().w, ph = A.back().h, nw = (pw + 1) / 2, nh = (ph + 1) / 2;
            if (nw <= win || nh <= win) break;
            Lvl a2{std::vector<uint8_t>((size_t)nw * nh), nw, nh}, b2{std::vector<uint8_t>((size_t)nw * nh), nw, nh};
            ora_pyrdown(A.back().img.data(), pw, ph, a2.img.data());
            ora_pyrdown(B.back().img.data(), pw, ph, b2.img.data());
            A.push_back(a2);
            B.push_back(b2);
        }
    }
    const int max_level = (int)A.size() - 1;
    const float half = (win - 1) * 0.5f;
    const int W_BITS = 14;
    const float FLT_SCALE = 1.f / (1 << 20);
    const int max_count = std::min(std::max(p->max_iter, 0), 100);
    const float min_eig = (float)p->min_eig;
    const bool exact = p->exact_sums != 0;
    double eps = std::min(std::max(p->eps, 0.), 10.);
    eps *= eps;
    std::vector<short> Iw((size_t)win * win), dIw((size_t)2 * win * win);
    for (int i = 0; i < n; ++i) {
        status[i] = 1;
        err[i] = 0;
    }
    for (int level = max_level; level >= 0; --level) {
        const Lvl& I = A[level];
        const Lvl& J = B[level];
        for (int i = 0; i < n; ++i) {
            const float sc = (float)(1. / (1 << level));
            float prevx = ref_xy[2 * i] * sc, prevy = ref_xy[2 * i + 1] * sc;
            float nx, ny;
            if (level == max_level) {  // OPTFLOW_USE_INITIAL_FLOW
                nx = cur_xy[2 * i] * sc;
                ny = cur_xy[2 * i + 1] * sc;
            } else {
                nx = cur_xy[2 * i] * 2.f;
                ny = cur_xy[2 * i + 1] * 2.f;
            }
            cur_xy[2 * i] = nx;
            cur_xy[2 * i + 1] = ny;
            prevx -= half;
            prevy -= half;
            const int ipx = (int)std::floor(prevx), ipy = (int)std::floor(prevy);
            if (ipx < -win || ipx >= I.w || ipy < -win || ipy >= I.h) {
                if (level == 0) {
                    status[i] = 0;
                    err[i] = 0;
                }
                continue;
            }
            float a = prevx - ipx, b = prevy - ipy;
            int iw00 = cv_round((1.f - a) * (1.f - b) * (1 << W_BITS)), iw01 = cv_round(a * (1.f - b) * (1 << W_BITS)),
                iw10 = cv_round((1.f - a) * b * (1 << W_BITS)), iw11 = (1 << W_BITS) - iw00 - iw01 - iw10;
            float iA11 = 0, iA12 = 0, iA22 = 0;
            int64_t xA11 = 0, xA12 = 0, xA22 = 0;
            for (int y = 0; y < win; ++y)
                for (int x = 0; x < win; ++x) {
                    const int X = ipx + x, Y = ipy + y;
                    int dx00, dy00, dx01, dy01, dx10, dy10, dx11, dy11;
                    I.deriv(X, Y, &dx00, &dy00);
                    I.deriv(X + 1, Y, &dx01, &dy01);
                    I.deriv(X, Y + 1, &dx10, &dy10);
                    I.deriv(X + 1, Y + 1, &dx11, &dy11);
                    const int ival = descale(I.I(X, Y) * iw00 + I.I(X + 1, Y) * iw01 + I.I(X, Y + 1) * iw10 + I.I(X + 1, Y + 1) * iw11, W_BITS - 5);
                    const int ixval = descale(dx00 * iw00 + dx01 * iw01 + dx10 * iw10 + dx11 * iw11, W_BITS);
                    const int iyval = descale(dy00 * iw00 + dy01 * iw01 + dy10 * iw10 + dy11 * iw11, W_BITS);
                    Iw[(size_t)y * win + x] = (short)ival;
                    dIw[2 * ((size_t)y * win + x)] = (short)ixval;
                    dIw[2 * ((size_t)y * win + x) + 1] = (short)iyval;
                    if (exact) {
                        xA11 += (int64_t)ixval * ixval;
                        xA12 += (int64_t)ixval * iyval;
                        xA22 += (int64_t)iyval * iyval;
                    } else {
                        iA11 += (float)(ixval * ixval);
                        iA12 += (float)(ixval * iyval);
                        iA22 += (float)(iyval * iyval);
                    }
                }
            if (exact) {
                iA11 = (float)xA11;
                iA12 = (float)xA12;
                iA22 = (float)xA22;
            }
            const float A11 = iA11 * FLT_SCALE, A12 = iA12 * FLT_SCALE, A22 = iA22 * FLT_SCALE;
            float D = A11 * A22 - A12 * A12;
            const float minEig = (A22 + A11 - std::sqrt((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (2 * win * win);
            if (p->get_min_eig) err[i] = minEig;  // the last write is level 0's
            if (minEig < min_eig || D < 1.1920929e-07f) {
                if (level == 0) status[i] = 0;
                continue;
            }
            D = 1.f / D;
            nx -= half;
            ny -= half;
            float pdx = 0, pdy = 0;
            for (int j = 0; j < max_count; ++j) {
                const int inx = (int)std::floor(nx), iny = (int)std::floor(ny);
                if (inx < -win || inx >= J.w || iny < -win || iny >= J.h) {
                    if (level == 0) status[i] = 0;
                    break;
                }
                a = nx - inx;
                b = ny - iny;
                iw00 = cv_round((1.f - a) * (1.f - b) * (1 << W_BITS));
                iw01 = cv_round(a * (1.f - b) * (1 << W_BITS));
                iw10 = cv_round((1.f - a) * b * (1 << W_BITS));
                iw11 = (1 << W_BITS) - iw00 - iw01 - iw10;
                float ib1 = 0, ib2 = 0;
                int64_t xb1 = 0, xb2 = 0;
                for (int y = 0; y < win; ++y)
                    for (int x = 0; x < win; ++x) {
                        const int X = inx + x, Y = iny + y;
                        const int diff = descale(J.I(X, Y) * iw00 + J.I(X + 1, Y) * iw01 + J.I(X, Y + 1) * iw10 + J.I(X + 1, Y + 1) * iw11, W_BITS - 5) -
                                         Iw[(size_t)y * win + x];
                        if (exact) {
                            xb1 += diff * dIw[2 * ((size_t)y * win + x)];
                            xb2 += diff * dIw[2 * ((size_t)y * win + x) + 1];
                        } else {
                            ib1 += (float)(diff * dIw[2 * ((size_t)y * win + x)]);
                            ib2 += (float)(diff * dIw[2 * ((size_t)y * win + x) + 1]);
                        }
                    }
                if (exact) {
                    ib1 = (float)xb1;
                    ib2 = (float)xb2;
                }
                const float b1 = ib1 * FLT_SCALE, b2 = ib2 * FLT_SCALE;
                const float dx = (float)((A12 * b2 - A22 * b1) * D), dy = (float)((A12 * b1 - A11 * b2) * D);
                nx += dx;
                ny += dy;
                cur_xy[2 * i] = nx + half;
                cur_xy[2 * i + 1] = ny + half;
                if ((double)dx * dx + (double)dy * dy <= eps) break;
                if (j > 0 && std::abs(dx + pdx) < 0.01 && std::abs(dy + pdy) < 0.01) {
                    cur_xy[2 * i] -= dx * 0.5f;
                    cur_xy[2 * i + 1] -= dy * 0.5f;
                    break;
                }
                pdx = dx;
                pdy = dy;
            }
            if (status[i] && level == 0 && !p->get_min_eig) {  // err = mean |diff| / 32 at the final position
                const float fx = cur_xy[2 * i] - half, fy = cur_xy[2 * i + 1] - half;
                const int inx = (int)std::floor(fx), iny = (int)std::floor(fy);
                if (inx < -win || inx >= J.w || iny < -win || iny >= J.h) {
                    status[i] = 0;
                    continue;
                }
                const float aa = fx - inx, bb = fy - iny;
                iw00 = cv_round((1.f - aa) * (1.f - bb) * (1 << W_BITS));
                iw01 = cv_round(aa * (1.f - bb) * (1 << W_BITS));
                iw10 = cv_round((1.f - aa) * bb * (1 << W_BITS));
                iw11 = (1 << W_BITS) - iw00 - iw01 - iw10;
                float errval = 0.f;
                int64_t xerr = 0;
                for (int y = 0; y < win; ++y)
                    for (int x = 0; x < win; ++x) {
                        const int X = inx + x, Y = iny + y;
                        const int diff = descale(J.I(X, Y) * iw00 + J.I(X + 1, Y) * iw01 + J.I(X, Y + 1) * iw10 + J.I(X + 1, Y + 1) * iw11, W_BITS - 5) -
                                         Iw[(size_t)y * win + x];
                        if (exact)
                            xerr += std::abs(diff);
                        else
                            errval += std::abs((float)diff);
                    }
                if (exact) errval = (float)xerr;
                err[i] = errval * 1.f / (32 * win * win);
            }
        }
    }
}
