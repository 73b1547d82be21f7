/*
 * oracle.h -- CPU restatement of the ygz-slam tracking + local-BA hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library, and only as the checker / the timed CPU baseline.
 * The product (ygz_slam_b200/csrc) never links or calls it.
 *
 * Every function cites the reference file:line it restates (paths relative to
 * /root/reference).  Arithmetic owned by third-party code that is NOT in the
 * reference tree (uzh-rpg `fast`, OpenCV, g2o, Ceres -- SURVEY.md 8c) is restated
 * from the published algorithm; the OpenCV-owned pieces are pinned against
 * cv2 4.13 in tests/test_oracle_cv2.py, FAST / g2o / Ceres are "parity unpinned"
 * (no reference test asserts a value for them) and are pinned only structurally
 * (brute-force cross-implementations, known-answer scenes).
 *
 * Build: oracle/Makefile.  Two flavours of the same sources:
 *   liboracle.so       -O2 -ffp-contract=off      (the parity checker: no FMA contraction)
 *   liboracle_native.so -O3 -march=native         (the reference's own flags, CMakeLists.txt:14-16;
 *                                                  the timed CPU baseline)
 */
#ifndef YGZ_ORACLE_H_
#define YGZ_ORACLE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORA_MAX_LEVELS 10

/* ---- image pyramid (src/Basic/Frame.cpp:22-40; OpenCV cvtColor / pyrDown) ------------- */
void ora_bgr2gray(const uint8_t* bgr, int w, int h, uint8_t* gray);
void ora_pyrdown(const uint8_t* src, int w, int h, uint8_t* dst);
/* packed pyramid: levels stored back to back, each level continuous (pitch == width), like the
 * cv::Mat outputs of pyrDown.  Fills lw/lh/off for n_levels and returns the total byte count. */
size_t ora_pyramid_layout(int w, int h, int n_levels, int* lw, int* lh, size_t* off);
void ora_build_pyramid(const uint8_t* gray, int w, int h, int n_levels, uint8_t* pyr);

/* ---- FAST-10 (uzh-rpg/fast; call sites src/Algorithm/FeatureDetector.cpp:365-381) ------- */
/* raster-order corner list; returns the number found (corners beyond `cap` are counted but not stored) */
int ora_fast10_detect(const uint8_t* img, int w, int h, int stride, int barrier, int16_t* xy, int cap);
void ora_fast10_score(const uint8_t* img, int stride, const int16_t* xy, int n, int barrier, int32_t* scores);
int ora_fast_nonmax_3x3(const int16_t* xy, const int32_t* scores, int n, int32_t* keep_idx);
/* neighbour rule of fast_nonmax_3x3: 0 = ">=" (default, restated from memory of uzh-rpg/fast), 1 = ">" */
void ora_set_fast_nonmax_strict(int strict);

/* ---- FeatureDetector (src/Algorithm/FeatureDetector.cpp:299-596) ------------------------ */
typedef struct {
    int image_width, image_height; /* image.width / image.height            */
    int cell_size;                 /* feature.cell (10)                     */
    int threshold;                 /* short(feature.detection_threshold)=15 */
    int n_levels;                  /* Frame::Option::_pyramid_level (3)     */
} ora_detect_params;

typedef struct {
    int n;
    double* px;      /* full-resolution pixel = level coord * 2^level */
    double* py;
    int32_t* level;
    float* score;    /* Shi-Tomasi */
    float* angle;    /* degrees */
    uint8_t* desc;   /* n x 32 */
    int32_t* cell;   /* grid cell index of each feature */
} ora_features;

/* FeatureDetector::Detect.  `occupied` = grid_rows*grid_cols bytes (non-zero = cell already holds an
 * old feature, SetExistingFeatures) or NULL.  Output arrays must hold grid_rows*grid_cols entries. */
int ora_detect(const uint8_t* pyr, const ora_detect_params* p, const uint8_t* occupied, ora_features* out);
float ora_shi_tomasi(const uint8_t* img, int w, int h, int u, int v);
/* IC_Angle + ComputeOrbDescriptor for given full-res pixels (ComputeAngleAndDescriptor, :580-588) */
void ora_describe(const uint8_t* pyr, int w, int h, int n_levels, int n, const double* px, const double* py,
                  const int32_t* level, float* angle, uint8_t* desc);
float ora_fast_atan2(float y, float x);
int ora_cv_round_f(float v);
int ora_cv_round_d(double v);

/* ---- matching (src/Algorithm/Matcher.cpp:30-84; test/test_orb_match.cpp:86-105) --------- */
int ora_descriptor_distance(const uint8_t* a, const uint8_t* b);
/* cv::BFMatcher(NORM_HAMMING, crossCheck).match: train_idx[i] = -1 when query i has no match */
void ora_match_bf(const uint8_t* A, int nA, const uint8_t* B, int nB, int cross_check, int32_t* train_idx,
                  int32_t* dist);
/* test_orb_match.cpp:97-105: keep[i]=1 iff matched and dist < 3*clamp(min dist,20,50); returns count */
int ora_good_matches(const int32_t* train_idx, const int32_t* dist, int nA, uint8_t* keep);
/* Matcher::CheckFrameDescriptors core: keep[k]=1 iff d_k < 3.0*clamp(min d, init_low, init_high) */
int ora_check_descriptors(const uint8_t* A, const uint8_t* B, const int32_t* ia, const int32_t* ib, int n,
                          int init_low, int init_high, int32_t* dist, uint8_t* keep);

typedef struct { float fx, fy, cx, cy; } ora_camera; /* Camera.h:14-22: stored as float */

/* Matcher::SearchForTriangulation + CheckDistEpipolarLine (Matcher.cpp:86-193, 338-354): node1 / node2 = vocabulary node of
 * every feature in the key-frame's DBoW3 feature vector (-1 = none); match12[i] = index in key-frame 2 or -1 */
void ora_search_for_triangulation(const ora_camera* cam, int n1, const uint8_t* desc1, const double* px1, const int32_t* node1,
                                  int n2, const uint8_t* desc2, const double* px2, const int32_t* node2, const double* E12,
                                  int th_low, double epipolar_dsqr, int32_t* match12);
/* cvutils::DepthFromTriangulation (CVUtils.h:18-38); returns the function's bool */
int ora_depth_from_triangulation(const double* T_search_ref, const double* f_ref, const double* f_cur, double determinant_th,
                                 double* depth1, double* depth2);

/* ---- DBoW3 (thirdparty/DBoW3/src/Vocabulary.cpp; bow.cpp) --------------------------------------------------------------- */
typedef struct ora_vocab ora_vocab;
/* Vocabulary::loadFromBinaryFile (Vocabulary.cpp:1180-1225) from the file's bytes; NULL if malformed */
ora_vocab* ora_vocab_load(const uint8_t* bytes, size_t n_bytes);
void ora_vocab_free(ora_vocab* v);
void ora_vocab_info(const ora_vocab* v, int32_t* info /* k, L, scoring, weighting, nodes, words */);
/* Vocabulary::transform(features, bow, feature vector, levelsup) (Vocabulary.cpp:706-832), Frame::ComputeBoW (Frame.cpp:190-201) */
int ora_bow_transform(const ora_vocab* v, int n, const uint8_t* desc, int levelsup, int32_t* word, int32_t* node, double* weight,
                      int32_t* bow_word, double* bow_value);
/* Matcher::SearchByBoW (Matcher.cpp:196-292) */
int ora_search_by_bow(int n1, const uint8_t* desc1, const int32_t* node1, const float* angle1, int n2, const uint8_t* desc2,
                      const int32_t* node2, const float* angle2, int th_low, float knn_ratio, int check_orientation, int32_t* match12);

/* ---- monocular initialiser, RANSAC half (src/Algorithm/Initializer.cpp:9-318, 670-853; initializer.cpp) ----------------- */
/* the 8-point minimal sets TryInitialize draws from a default-constructed cv::RNG (:25-49): sets[it * 8 + j] */
void ora_initializer_sets(int n_points, int max_iter, int32_t* sets);
/* FindHomography + FindFundamental: best model, float score, winning iteration (-1: no model scored above 0) and inlier
 * flags of each; models (may be NULL) = max_iter x 18 doubles, every iteration's H21i then F21i */
void ora_initializer_ransac(int n, const double* px1, const double* px2, int max_iter, const int32_t* sets, float sigma, double* H21,
                            float* score_H, int32_t* best_H, uint8_t* inl_H, double* F21, float* score_F, int32_t* best_F, uint8_t* inl_F,
                            double* models);

/* Initializer::ReconstructH (use_h != 0) / ReconstructF with CheckRT, Triangulate, DecomposeE (Initializer.cpp:330-675, 855-963) on
 * the model TryInitialize chose; K = {fx, fy, cx, cy}; returns the function's bool; n_good[8] = CheckRT's count per candidate */
int ora_initializer_reconstruct(int n, const double* px1, const double* px2, int use_h, const double* model, const uint8_t* inliers,
                                const double* K, float sigma2, float min_parallax, int min_triangulated, double ratio_h, double* R21,
                                double* t21, double* p3d, uint8_t* triangulated, int32_t* n_good, double* parallax,
                                double* candidates /* may be NULL: 8 x 12 */);

/* ---- patch alignment (src/Algorithm/CVUtils.cpp:186-318; Matcher.cpp:356-466) ----------- */
int ora_align2d(const uint8_t* img, int w, int h, const uint8_t* ref_with_border /*100*/,
                const uint8_t* ref /*64*/, int n_iter, double* u, double* v);
int ora_align1d(const uint8_t* img, int w, int h, float dirx, float diry, const uint8_t* ref_with_border,
                const uint8_t* ref, int n_iter, double* u, double* v, double* h_inv);


/* pose = T_cw as 3x4 row-major [R|t] (12 doubles) at this boundary; quaternion inside like Sophus */
/* Matcher::FindDirectProjection(ref,curr,Feature*,px,level) (Matcher.cpp:385-417) for a batch */
void ora_find_direct_projection(const uint8_t* ref_pyr, const uint8_t* cur_pyr, int w, int h, int n_levels,
                                const ora_camera* cam, const double* T_cw_ref, const double* T_cw_cur, int n,
                                const double* ref_px /*2n*/, const double* ref_depth, const int32_t* ref_level,
                                double* cur_px_inout /*2n*/, int32_t* search_level, uint8_t* ok);

/* ---- sparse image alignment (src/Algorithm/SparseImageAlign.cpp; NLSSolver_impl.hpp) ---- */
/* returns n_meas/16 (SparseImgAlign::run); T_cw_cur updated in place.  exact_chi2 = 0: the reference's float running
 * sum of the squared residuals; 1: their sum in double, rounded to float once, so that the rollback test chi2_new > chi2
 * decides as in the CUDA kernel, whose sum has no fixed order */
size_t ora_sparse_align(const uint8_t* ref_pyr, const uint8_t* cur_pyr, int w, int h, int n_levels,
                        const ora_camera* cam, int n, const double* px /*2n*/, const double* depth,
                        const uint8_t* has_mappoint, const double* T_cw_ref, double* T_cw_cur, int max_level,
                        int min_level, int n_iter, double eps, int32_t* iters_per_level /*may be NULL*/, int exact_chi2);
/* Matcher::SparseImageAlignment (Matcher.cpp:468-492): returns 1/0, T_cw_cur in/out */
int ora_matcher_sparse_alignment(const uint8_t* ref_pyr, const uint8_t* cur_pyr, int w, int h, int n_levels,
                                 const ora_camera* cam, int n, const double* px, const double* depth,
                                 const uint8_t* has_mappoint, const double* T_cw_ref, double* T_cw_cur);

/* ---- Sophus (thirdparty/Sophus/sophus/so3.cpp:127-202, se3.cpp:59-95,170-220) ----------- */
void ora_se3_exp(const double* upsilon_omega /*6*/, double* T /*12*/);
void ora_se3_log(const double* T /*12*/, double* upsilon_omega /*6*/);

/* ---- bundle adjustment (src/Algorithm/BA.cpp; include/ygz/G2oTypes.h) ------------------- */
typedef struct {
    int max_iters;        /* optimizer.optimize(20)            */
    double huber_delta;   /* 5.991 (BA.cpp:451); <=0 : no loss */
    double chi2_outlier;  /* 5.991 (BA.cpp:508)                */
    double tau;           /* g2o LM tau 1e-5                   */
    int max_trials;       /* g2o LM maxTrialsAfterFailure 10   */
} ora_ba_params;

typedef struct {
    int iters;
    int lm_trials;
    double chi2_initial, chi2_final, lambda_final;
    int n_outliers;
} ora_ba_stats;

/* ba::LocalBAG2O.  poses: n_kf x 6 in g2o order [omega; upsilon] (G2oTypes.h:38-45), in/out.
 * fixed[k] != 0 : vertex fixed.  pts: n_pt x 3 in/out.  obs: (kf_idx, pt_idx, px) x n_obs. */
int ora_local_ba_g2o(const ora_camera* cam, int n_kf, double* poses, const uint8_t* fixed, int n_pt, double* pts,
                     int n_obs, const int32_t* kf_idx, const int32_t* pt_idx, const double* obs_px,
                     const ora_ba_params* prm, uint8_t* outlier, ora_ba_stats* stats);

/* ba::LocalBA, the Ceres twin (BA.cpp:324-384).  poses: n_kf x 6 as [t; angle-axis] (CeresReprojectionError.h:33-69),
 * in/out; fixed[k] != 0 : the key-frame with _keyframe_id == 0 (point-only residual blocks, BA.cpp:340-349).
 * Default ceres::Solver::Options (trust-region LM, Jacobi scaling); max_iters = 50 in the reference.  huber_a > 0 adds the
 * ceres::HuberLoss(a) of ba::OptimizeCurrent (BA.cpp:91-186, a = 0.1 in normalised image coordinates).
 * termination: 0 max iterations, 1 gradient, 2 parameter, 3 function tolerance, 4 trust region collapsed. */
typedef struct {
    int iters, successful_steps;
    double cost_initial, cost_final, radius_final;
    int termination;
} ora_ceres_stats;
int ora_local_ba_ceres(const ora_camera* cam, int n_kf, double* poses, const uint8_t* fixed, int n_pt, double* pts,
                       int n_obs, const int32_t* kf_idx, const int32_t* pt_idx, const double* obs_px, int max_iters,
                       double huber_a /* ceres::HuberLoss(a) on every block, 0 = no loss */, ora_ceres_stats* stats);

/* ba::TwoViewBACeres (BA.cpp:11-89): ref pose fixed, current pose and points free, HuberLoss(0.1) on the blocks of the
 * non-inlier points (which restart from (0,0,1)); inlier[] in/out, returns the inlier count.  Trust-region LM instead of the
 * reference's DOGLEG strategy (same cost, same minimum up to the function tolerance). */
int ora_two_view_ba(const ora_camera* cam, int n, const double* T_cw_ref, double* T_cw_cur, const double* px_ref,
                    const double* px_cur, uint8_t* inlier, double* pts, ora_ceres_stats* stats);

/* ba::OptimizeCurrentPoseOnly (BA.cpp:188-264).  T_cw in/out, inlier[] out (1 = !_bad), depth[] out */
int ora_pose_only(const ora_camera* cam, int n, const double* pt_world /*3n*/, const double* px /*2n*/,
                  double* T_cw, uint8_t* inlier, double* depth);

/* ---- KLT (src/Algorithm/Tracker.cpp:65-113 -> cv::calcOpticalFlowPyrLK) ------------------ */
/* min_eig is compared in float, as OpenCV stores minEigThreshold: the threshold is (float)min_eig.
 * exact_sums = 0 adds the window sums (A11, A12, A22, b1, b2 and the err sum) in f32 like OpenCV's scalar code;
 * exact_sums = 1 adds the same integer products in int64 and converts each sum to float once, which is klt.cu's
 * arithmetic (every other step is the same round-to-nearest f32 on both sides, so this mode matches it bit for bit).
 * get_min_eig = 1 writes the level-0 minimum eigenvalue into err instead of the mean |diff| (OPTFLOW_LK_GET_MIN_EIGENVALS). */
typedef struct {
    int win;         /* 21 */
    int max_level;   /* 4  */
    int max_iter;    /* 30 */
    double eps;      /* 0.001 */
    double min_eig;  /* 1e-4  */
    int exact_sums;  /* 0 */
    int get_min_eig; /* 0 */
} ora_klt_params;
void ora_klt(const uint8_t* ref, const uint8_t* cur, int w, int h, int n, const float* ref_xy,
             float* cur_xy_inout, uint8_t* status, float* err, const ora_klt_params* p);

#ifdef __cplusplus
}
#endif
#endif
