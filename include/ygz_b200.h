/*
 * ygz_b200.h -- C ABI of libygz_b200.so: the H100 (sm_90a) implementation of the ygz-slam
 * per-frame tracking + local-BA hot path.
 *
 * The reference (PaoPaoRobot/ygz-slam) has no plugin / FFI layer: its boundary for this path is the
 * public C++ API of libygz-algorithm.so (SURVEY.md 8b).  Every entry point below names the reference
 * interface it replaces (paths relative to the reference root).  The C++ shim classes in
 * ygz_slam_b200/host/ keep the reference's class/method names on top of this ABI so that
 * the reference callers under src/Module compile against them unchanged (INTEGRATION.md).
 *
 * Conventions
 *   - plain pointers and sizes only; the caller owns every host buffer, the context owns device memory;
 *   - every call returns YGZB_OK (0) or a negative error code and never throws; ygzb_last_error()
 *     returns the message of the last failure on that context;
 *   - one context = one device + one stream; thread-compatible (one context per host thread), like
 *     the reference's per-instance scratch (Matcher.h:143-150, FeatureDetector.h:93-98);
 *   - all batched calls take `n` independent items (frames, pairs, patches) -- n = 1 is the
 *     reference's one-frame-at-a-time call;
 *   - there is NO CPU fallback: without a usable sm_90 device ygzb_create fails.
 *   - poses T_cw are 3x4 row-major [R|t] doubles (12 per pose) unless stated otherwise.
 */
#ifndef YGZ_B200_H_
#define YGZ_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YGZB_OK 0
#define YGZB_ERR_INVALID (-1)   /* bad argument */
#define YGZB_ERR_CUDA (-2)      /* CUDA runtime error (message in ygzb_last_error) */
#define YGZB_ERR_NO_DEVICE (-3) /* no sm_90 device: there is no CPU fallback */
#define YGZB_ERR_CAPACITY (-4)  /* an output or scratch capacity was exceeded */

#define YGZB_MAX_LEVELS 10

typedef struct ygzb_ctx ygzb_ctx;
typedef struct ygzb_frames ygzb_frames;

/* Filled from the reference's YAML keys (config/default.yaml) and Option structs.            */
typedef struct {
    int image_width;     /* image.width  (640)                                                */
    int image_height;    /* image.height (480)                                                */
    int n_levels;        /* Frame::Option::_pyramid_level (include/ygz/Basic/Frame.h:22-24)   */
    int cell_size;       /* feature.cell (10)           FeatureDetector.cpp:335               */
    int fast_threshold;  /* short(feature.detection_threshold) = 15   FeatureDetector.cpp:338 */
    float fx, fy, cx, cy;/* camera.* -- stored as float like PinholeCamera (Camera.h:14-22)   */
} ygzb_params;

void ygzb_default_params(ygzb_params* p);
int ygzb_create(int device, const ygzb_params* p, ygzb_ctx** out);
/* the parameters the context was created with (image size and camera for callers that size their buffers from it) */
int ygzb_get_params(const ygzb_ctx* ctx, ygzb_params* out);
void ygzb_destroy(ygzb_ctx* ctx);
const char* ygzb_last_error(const ygzb_ctx* ctx);
int ygzb_synchronize(ygzb_ctx* ctx);
/* the same, but the calling thread sleeps on a blocking event instead of spinning: for hosts where more threads wait on
 * the GPU than there are CPUs to spin on (a few tens of microseconds of extra wake-up latency per call) */
int ygzb_synchronize_blocking(ygzb_ctx* ctx);
/* the context's cudaStream_t, for callers that time or order work themselves */
void* ygzb_stream(ygzb_ctx* ctx);
/* device time between two points of the context's stream (CUDA events): start records an event, stop records a second
 * one, waits for it and returns the elapsed milliseconds -- what bench.py reports as the device-timed step */
int ygzb_timer_start(ygzb_ctx* ctx);
int ygzb_timer_stop(ygzb_ctx* ctx, double* ms);
/* number of kernels this library launched on the context since creation (bench.py: gpu_launches) */
long long ygzb_launch_count(const ygzb_ctx* ctx);

/* optional per-stage device timing: when enabled every kernel launch is bracketed by CUDA events on
 * the context stream; ygzb_profile_read synchronises, sums the elapsed ms and launch counts per stage
 * (arrays of ygzb_profile_stage_count() entries) and resets the record.                          */
int ygzb_profile_enable(ygzb_ctx* ctx, int on);
int ygzb_profile_read(ygzb_ctx* ctx, double* ms, int32_t* launches);
int ygzb_profile_stage_count(void);
const char* ygzb_profile_stage_name(int stage);

/* page-locked host memory for the batched entry points (plain malloc'ed buffers also work) */
int ygzb_host_alloc(void** ptr, size_t bytes);
int ygzb_host_free(void* ptr);

/* ---- frames: device-resident image pyramids -------------------------------------------------
 * replaces Frame::InitFrame / CreateImagePyramid (src/Basic/Frame.cpp:22-40: cvtColor + pyrDown). */
int ygzb_frames_create(ygzb_ctx* ctx, int capacity, ygzb_frames** out);
void ygzb_frames_destroy(ygzb_frames* f);
/* host -> device copy of `count` images into slots [first, first+count) and pyramid build.
 * channels 1 (grey) or 3 (BGR); frame_stride = bytes between consecutive host images.  `host` may also be a
 * device pointer (frames that are already resident in HBM): the copy uses unified addressing.  */
int ygzb_frames_upload(ygzb_frames* f, int first, int count, const uint8_t* host, int channels,
                       size_t frame_stride);
/* device-to-device copy of the whole pyramid of one slot into another (asynchronous on the context stream): lets a
 * caller keep a frame beyond its staging slot, e.g. when Frame becomes a key-frame (the reference keeps the cv::Mat
 * pyramid alive through the Frame object, include/ygz/Basic/Frame.h:138).  The slot's feature store is not copied. */
int ygzb_frames_copy(ygzb_frames* f, int src_slot, int dst_slot);
/* pyramid build only, for level-0 images already resident in slot storage (bench "value" leg) */
int ygzb_frames_build_pyramid(ygzb_frames* f, int first, int count);
/* device pointer / geometry of slot storage, level 0 first, every level pitch-linear */
int ygzb_frames_layout(const ygzb_frames* f, int* lw, int* lh, int* lpitch, size_t* loff, size_t* slot_stride);
void* ygzb_frames_device_ptr(ygzb_frames* f);
/* copy one level of one slot back to the host (tests) */
int ygzb_frames_download_level(ygzb_frames* f, int slot, int level, uint8_t* host /* lw*lh, packed */);

/* ---- lens undistortion on upload ----------------------------------------------------------------------------------
 * The reference's camera reads the radial-tangential coefficients camera.k1 k2 p1 p2 (include/ygz/Basic/Camera.h:19-22)
 * and declares UndistortPoint (:96-104), but nothing on its path applies them.  Here a frame pool can undistort every
 * frame on the device as it enters the pyramid: level 0 becomes cv::remap(cv::cvtColor(image), map, INTER_LINEAR,
 * BORDER_CONSTANT, 0), bit for bit, with the maps in OpenCV's fixed-point format (cv::initUndistortRectifyMap with
 * CV_16SC2), so a caller with OpenCV can pass the maps it already has:
 *   map_xy [H][W][2] int16   (CV_16SC2: integer source pixel x, y)
 *   map_a  [H][W]    uint16  (CV_16UC1: (fy << 5) | fx, the 1/32-pixel fractions, < 1024)
 * Source pixels outside the image read as 0.
 *
 * Host code, no device needed: cv::initUndistortRectifyMap(K, D, R = I, newK, (width, height), CV_16SC2) restated in
 * double precision, D = {k1, k2, p1, p2, k3} (k3 = 0 is the model of the reference's UndistortPoint).  K and newK are
 * {fx, fy, cx, cy}; newK == NULL means newK = K (unlike OpenCV, whose empty newK centres the principal point).       */
int ygzb_undistort_map(int width, int height, const double K[4], const double dist[5], const double newK[4], int16_t* map_xy,
                       uint16_t* map_a);
/* copies the maps (image_width x image_height entries, host or device memory) to the device, one set per frame pool;
 * map_xy == map_a == NULL clears them.  While they are set, every ygzb_frames_upload (grey or BGR, host or device source)
 * and every ygzb_tracker_upload writes level 0 undistorted before the pyramid is built; ygzb_frames_build_pyramid, which
 * starts from the level 0 already in the slot, is unchanged.  Then the camera of everything downstream is the
 * undistorted one: the tracker's K (ygzb_tracker_create), the context's fx..cy and every depth map passed to
 * ygzb_tracker_set_depth belong to newK.  Images the tracker re-uploads from a map or reference record
 * (ygzb_tracker_import, ygzb_tracker_import_reference) are undistorted already and are not remapped again.
 * Synchronous: the call waits for the uploads in flight that read the old maps.  An entry map_a >= 1024, or only one
 * of the two pointers, returns YGZB_ERR_INVALID with the pool's maps unchanged.                                         */
int ygzb_frames_set_undistort(ygzb_frames* f, const int16_t* map_xy, const uint16_t* map_a);

/* ---- FeatureDetector ------------------------------------------------------------------------
 * replaces FeatureDetector::Detect (src/Algorithm/FeatureDetector.cpp:345-444; header
 * include/ygz/Algorithm/FeatureDetector.h:63): grid FAST-10 over the pyramid, 3x3 non-max, best
 * Shi-Tomasi per cell, IC angle, rotated-BRIEF descriptor.  Results stay on the device (slot feature
 * store) for ygzb_match_frames and are returned packed, frame after frame, in cell-index order. */
typedef struct {
    int32_t* offsets; /* n+1 : features of item i are [offsets[i], offsets[i+1])                 */
    float* x;         /* full-resolution pixel = level coordinate * 2^level  (Feature::_pixel)   */
    float* y;
    uint8_t* level;   /* Feature::_level */
    float* score;     /* Feature::_score (Shi-Tomasi) */
    float* angle;     /* Feature::_angle, degrees */
    uint8_t* desc;    /* 32 bytes per feature (Feature::_desc) */
    int32_t* cell;    /* grid cell of the feature (may be NULL) */
    int capacity;     /* capacity of the packed arrays, in features */
} ygzb_keypoints;

/* slots[i] selects the frame of item i.  occupied: n * grid_rows*grid_cols bytes (non-zero = cell
 * holds an old feature: SetExistingFeatures, :446-464) or NULL (= overwrite_existing_features).
 * out may be NULL (results only kept on the device).                                          */
int ygzb_detect(ygzb_frames* f, const int32_t* slots, int n, const uint8_t* occupied, ygzb_keypoints* out);
int ygzb_grid_dims(const ygzb_ctx* ctx, int* rows, int* cols);

/* replaces FeatureDetector::ComputeAngleAndDescriptor (:580-588) for caller-supplied pixels:
 * item i owns features [offsets[i], offsets[i+1]) of x/y/level (full-res pixels, double like
 * Feature::_pixel); angle/desc are outputs.                                                  */
int ygzb_describe(ygzb_frames* f, const int32_t* slots, int n, const int32_t* offsets, const double* x,
                  const double* y, const uint8_t* level, float* angle, uint8_t* desc);

/* parity/debug view of the FAST stage of one slot and level (the call sites at
 * FeatureDetector.cpp:365-381): raster-order corner list, bisection scores and the indices kept by
 * fast_nonmax_3x3 -- the "FAST keypoint indices" the north star asks to match bit-exactly.     */
int ygzb_fast_debug(ygzb_frames* f, int slot, int level, int capacity, int16_t* xy, int32_t* scores,
                    int32_t* n_corners, int32_t* nonmax_idx, int32_t* n_nonmax);
/* per-level counters of the last ygzb_detect: stats[(i*n_levels + L)*2 + {0,1}] = corners, nonmax */
int ygzb_detect_stats(ygzb_frames* f, int n, int32_t* stats);

/* ---- Matcher: descriptors -------------------------------------------------------------------
 * replaces cv::BFMatcher(cv::NORM_HAMMING, crossCheck).match (test/test_orb_match.cpp:87-92) with
 * Matcher::DescriptorDistance (src/Algorithm/Matcher.cpp:30-43) as the metric.
 * train_idx[i] = -1 / dist[i] = -1 when query i has no (cross-checked) match.                  */
int ygzb_match_bf(ygzb_ctx* ctx, const uint8_t* A, int nA, const uint8_t* B, int nB, int cross_check,
                  int32_t* train_idx, int32_t* dist);
/* same, on the device-resident features of n_pairs slot pairs (a_slots[i] = query frame,
 * b_slots[i] = train frame); results packed per pair: query q of pair i is at q_offsets[i]+q.  */
int ygzb_match_frames(ygzb_frames* f, const int32_t* a_slots, const int32_t* b_slots, int n_pairs,
                      int cross_check, int32_t* q_offsets /* n_pairs+1 */, int32_t* train_idx, int32_t* dist,
                      int capacity);
/* replaces the distance loop of Matcher::CheckFrameDescriptors (Matcher.cpp:45-84) */
int ygzb_hamming_pairs(ygzb_ctx* ctx, const uint8_t* A, int nA, const uint8_t* B, int nB, const int32_t* ia,
                       const int32_t* ib, int n, int32_t* dist);

/* replaces Matcher::SearchForTriangulation (src/Algorithm/Matcher.cpp:86-193; Matcher.h:61-67) with
 * Matcher::CheckDistEpipolarLine (:338-354) for n_pairs key-frame pairs: pair p matches features [off1[p], off1[p+1]) of
 * key-frame 1 against [off2[p], off2[p+1]) of key-frame 2.  node1 / node2 = the vocabulary node of every feature in the
 * key-frame's DBoW3 feature vector (Frame::_feature_vec, levelsup = 4, Frame.cpp:199), -1 if the feature is in no node;
 * only features of the same node are compared, candidates in ascending index like the vector's index lists.  E12 = 9
 * doubles per pair (row major); th_low = matcher.th_low (65 in default.yaml, 50 in Matcher::Options), epipolar_dsqr =
 * Options::_epipolar_dsqr (1e-4).  match12[i] = index of the match inside key-frame 2 of the pair, or -1.          */
int ygzb_search_for_triangulation(ygzb_ctx* ctx, int n_pairs, const int32_t* off1, const int32_t* off2, const uint8_t* desc1,
                                  const double* px1, const int32_t* node1, const uint8_t* desc2, const double* px2,
                                  const int32_t* node2, const double* E12, int th_low, double epipolar_dsqr, int32_t* match12);
/* replaces cvutils::DepthFromTriangulation (include/ygz/Algorithm/CVUtils.h:18-38) for n bearing pairs: T_search_ref =
 * n_poses x 12 (3x4), pose_of[i] selects the pose of item i (NULL when n_poses == 1); f_ref / f_cur = unit-depth camera
 * rays; ok[i] = the function's bool (determinant >= determinant_th, 1e-5 in the reference), depth1 / depth2 = |depth|.  */
int ygzb_depth_from_triangulation(ygzb_ctx* ctx, int n, int n_poses, const double* T_search_ref, const int32_t* pose_of,
                                  const double* f_ref, const double* f_cur, double determinant_th, double* depth1, double* depth2,
                                  uint8_t* ok);

/* ---- DBoW3 vocabulary: Frame::ComputeBoW and BoW-guided matching ---------------------------------
 * replaces DBoW3::Vocabulary::loadFromBinaryFile (thirdparty/DBoW3/src/Vocabulary.cpp:1180-1225; the call
 * test/test_orb_match.cpp:74 `vocab.loadFromBinaryFile("./vocab/ORBvoc.bin")`): file_bytes = the whole file (u32 nb_nodes,
 * u32 size_node, i32 k, i32 L, i32 scoring, i32 weighting, then {i32 parent, u8 descriptor[32], f32 weight, u8 is_leaf}
 * records).  The tree is uploaded once and stays resident (39 MB for ORBvoc.bin).  Malformed data -> YGZB_ERR_INVALID.    */
typedef struct ygzb_vocab ygzb_vocab;
int ygzb_vocab_create(ygzb_ctx* ctx, const void* file_bytes, size_t n_bytes, ygzb_vocab** out);
void ygzb_vocab_destroy(ygzb_vocab* v);
/* info[6] = k, L, scoring (DBoW3::ScoringType), weighting (DBoW3::WeightingType), nodes, words -- like the reference, the
 * counts include the copy of the last record its `while (!f.eof())` loop appends */
int ygzb_vocab_info(const ygzb_vocab* v, int32_t* info);
/* replaces DBoW3::Vocabulary::transform(features, BowVector&, FeatureVector&, levelsup) (Vocabulary.cpp:706-832) as called by
 * Frame::ComputeBoW (src/Basic/Frame.cpp:190-201, levelsup = 4) for n_frames frames: frame f owns descriptors
 * [offsets[f], offsets[f+1]) (32 bytes each, at most 16384 per frame).  Per descriptor: word[i], weight[i] (the word's
 * weight) and node[i] = the id of its ancestor at level L - levelsup = the key of the FeatureVector entry the feature
 * index is appended to (-1 when the word is stopped, weight <= 0: such a feature enters neither vector).  The BowVector
 * of frame f = bow_count[f] pairs (bow_word ascending, bow_value) stored from index offsets[f] of bow_word / bow_value.
 * Word, node and count outputs are exact; bow_value differs from the reference's map-order sum in the last bits only.    */
int ygzb_bow_transform(ygzb_vocab* v, int n_frames, const int32_t* offsets, const uint8_t* desc, int levelsup, int32_t* word,
                       int32_t* node, double* weight, int32_t* bow_count, int32_t* bow_word, double* bow_value);
/* replaces Matcher::SearchByBoW (src/Algorithm/Matcher.cpp:196-292; Matcher.h:52-58) for n_pairs key-frame pairs, the
 * feature vectors given as one node id per feature (ygzb_bow_transform's `node`).  th_low / knn_ratio / check_orientation =
 * Matcher::Options (Matcher.h:21-24: 50, 0.9, false).  match12[i] = index inside key-frame 2 of the pair or -1; count[p] =
 * the function's return value (with check_orientation the matches outside the three dominant rotation bins are counted
 * out but -- as in the reference, Matcher.cpp:280-285 -- stay in match12); angle1 / angle2 may be NULL without it.       */
int ygzb_search_by_bow(ygzb_ctx* ctx, int n_pairs, const int32_t* off1, const int32_t* off2, const uint8_t* desc1,
                       const int32_t* node1, const float* angle1, const uint8_t* desc2, const int32_t* node2, const float* angle2,
                       int th_low, float knn_ratio, int check_orientation, int32_t* match12, int32_t* count);

/* ---- Initializer: the RANSAC half of the monocular initialisation -----------------------------
 * replaces Initializer::FindHomography + FindFundamental (src/Algorithm/Initializer.cpp:89-138, 670-717; with Normalize
 * :140-175, ComputeH21 :196-239, CheckHomography :251-318, ComputeF21 :730-762, CheckFundamental :772-853) as called from
 * Initializer::TryInitialize (:52-60) for n_lists pairs of matched pixel lists: list l owns point pairs
 * [offsets[l], offsets[l+1]) of px1 / px2 (x, y doubles; at least 8).  sets = n_lists x max_iter x 8 indices into the list:
 * the minimal sets TryInitialize draws with cv::RNG (:25-49; ygz::Initializer in the shim restates the generator).
 * sigma = Options::_sigma (2.0), max_iter = Options::_max_iter (200).  Per list: H21 / F21 (9 doubles, row major) = the
 * model of the best-scoring iteration, score_* = the float scores sh / sf of TryInitialize (:66), best_* = that iteration
 * or -1 when no model scored above 0 (the reference then leaves the matrix untouched; here it is zero), inlier_* = the
 * flags of the best model.  all_models (may be NULL) = n_lists x max_iter x 18 doubles, every iteration's H21i then F21i.
 * Every hypothesis is evaluated in parallel; scores are the reference's sequential float sums (same order of additions). */
int ygzb_initializer_ransac(ygzb_ctx* ctx, int n_lists, const int32_t* offsets, const double* px1, const double* px2, int max_iter,
                            const int32_t* sets, float sigma, double* H21, float* score_H, int32_t* best_H, uint8_t* inlier_H,
                            double* F21, float* score_F, int32_t* best_F, uint8_t* inlier_F, double* all_models);

/* replaces Initializer::ReconstructH / ReconstructF with CheckRT, Triangulate and DecomposeE (src/Algorithm/Initializer.cpp:
 * 330-675, 855-963) as called from TryInitialize (:74-78): per list the model TryInitialize chose (use_h[l] != 0: model[l] =
 * H21 and ReconstructH, else F21 and ReconstructF), inliers = that model's flags (only their count enters, :861-864, 882).
 * The camera is the context's (ygzb_params fx fy cx cy, float like Camera.h:14-22); sigma2 = Options::_sigma2 (4.0),
 * min_parallax = _min_parallex (1.0), min_triangulated = _min_triangulated_pts (8), good_point_ratio_h (0.9).
 * Out per list: ok = the function's bool; R21 (9, row major), t21 (3), zero unless ok; n_good[8] = CheckRT's count of every
 * pose candidate (8 for H, 4 for F); parallax = the selected candidate's (degrees); per point pair: p3d (3 doubles, camera-1
 * frame; zero where not reconstructed) and triangulated flags of the selected candidate; candidates (may be NULL) = n_lists x
 * 8 x 12, every candidate's R then t.  All point pairs of all candidates are triangulated in parallel.                     */
int ygzb_initializer_reconstruct(ygzb_ctx* ctx, int n_lists, const int32_t* offsets, const double* px1, const double* px2,
                                 const int32_t* use_h, const double* model, const uint8_t* inliers, float sigma2, float min_parallax,
                                 int min_triangulated, double good_point_ratio_h, int32_t* ok, double* R21, double* t21, double* p3d,
                                 uint8_t* triangulated, int32_t* n_good, double* parallax, double* candidates);

/* ---- cvutils / Matcher: direct (photometric) alignment ---------------------------------------
 * replaces cvutils::Align2D (src/Algorithm/CVUtils.cpp:186-318; include/ygz/Algorithm/CVUtils.h:163-169):
 * inverse-compositional alignment of an 8x8 template.  Patch i is searched on pyramid level level[i] of
 * frame slot[i]; ref_border = n x 100 bytes (10x10 template with border), ref = n x 64 bytes or NULL
 * (then the inner 8x8 of ref_border); uv = level coordinates in/out; ok = the function's bool.
 * One thread per patch with the reference's summation order: bit-exact (u, v, ok).               */
int ygzb_align2d(ygzb_frames* f, int n, const int32_t* slot, const uint8_t* level, const uint8_t* ref_border,
                 const uint8_t* ref, int n_iter, double* uv, uint8_t* ok);

/* replaces cvutils::Align1D (src/Algorithm/CVUtils.cpp:64-184; CVUtils.h:146-153): the same alignment restricted to
 * the direction dir = (dx, dy) per patch (epipolar search); h_inv = the function's double& output.     */
int ygzb_align1d(ygzb_frames* f, int n, const int32_t* slot, const uint8_t* level, const float* dir,
                 const uint8_t* ref_border, const uint8_t* ref, int n_iter, double* uv, uint8_t* ok, double* h_inv);

/* replaces Matcher::FindDirectProjection (src/Algorithm/Matcher.cpp:356-417, both overloads: the caller
 * supplies the reference depth) incl. GetWarpAffineMatrix / GetBestSearchLevel / WarpAffine
 * (:420-466, Matcher.h:123-134).  poses = n_poses x 12 (T_cw); candidate i uses frames ref_slot[i] /
 * cur_slot[i] and poses ref_pose[i] / cur_pose[i]; ref_px = full-res pixel of the reference feature,
 * cur_px = predicted full-res pixel in/out, search_level / ok = outputs.                          */
int ygzb_project_align(ygzb_frames* f, int n, const int32_t* ref_slot, const int32_t* cur_slot, int n_poses,
                       const double* poses, const int32_t* ref_pose, const int32_t* cur_pose, const double* ref_px,
                       const double* ref_depth, const uint8_t* ref_level, double* cur_px, uint8_t* search_level,
                       uint8_t* ok);

/* replaces SparseImgAlign::run (src/Algorithm/SparseImageAlign.cpp:21-50; ctor args SparseImageAlign.h:21-27)
 * for n_problems independent (ref, cur) pairs; problem p owns features [offsets[p], offsets[p+1]) of
 * px (full-res, 2 per feature) / depth / has_mappoint.  T_cw_cur is the initial pose in, the aligned
 * pose out; n_meas[p] = the function's return value (n_meas_/16).  Matcher::SparseImageAlignment
 * (Matcher.cpp:468-492) = this with (2, 0, 30, eps 1e-6) plus the host-side motion-norm check.       */
int ygzb_sparse_align(ygzb_frames* f, int n_problems, const int32_t* ref_slot, const int32_t* cur_slot,
                      const int32_t* offsets, const double* px, const double* depth, const uint8_t* has_mappoint,
                      const double* T_cw_ref, double* T_cw_cur, int max_level, int min_level, int n_iter, double eps,
                      int32_t* n_meas, int32_t* iters_per_level /* n_problems x YGZB_MAX_LEVELS or NULL */);

/* ---- ba:: ---------------------------------------------------------------------------------------
 * replaces ba::LocalBAG2O (src/Algorithm/BA.cpp:386-543; include/ygz/Algorithm/BA.h:60-66) with
 * VertexSE3Sophus / EdgeSophusSE3ProjectXYZ (include/ygz/G2oTypes.h:13-146): Levenberg + Schur
 * complement over marginalised landmarks, Huber kernel.  Batched: problem p owns keyframes
 * [kf_off[p], kf_off[p+1]), points [pt_off[p], ..), observations [obs_off[p], ..); kf_idx / pt_idx are
 * indices LOCAL to the problem.  poses = 6 doubles per keyframe in the vertex' order [omega; upsilon]
 * (in/out), fixed[k] != 0 = setFixed(true) (keyframe id 0 and non-local observers, BA.cpp:404-405,458-492),
 * pts in/out, outlier[o] = 1 iff chi2 > chi2_outlier after the optimisation (Feature::_bad, :505-515).
 * The system is linearised once before the first iteration: chi2_initial is the robust cost of the input
 * and lambda starts at tau * max |diag H| (free poses and landmarks), so max_iters = 0 evaluates once and
 * reports chi2_initial = chi2_final = that cost and lambda_final = that lambda.  A pose keeps its input
 * bits unless an LM step was accepted.  When the dense factorisation of the reduced system fails (a
 * non-positive pivot), the trial's pose step is zero, the landmarks are back-substituted from it, its
 * cost counts as DBL_MAX and the trial is rejected or accepted by the usual gain ratio.  With the landmark
 * blocks (Hll + lambda I) positive definite the gain ratio's denominator is then bl^T (Hll + lambda I)^-1 bl +
 * lambda |x_l|^2 + 1e-3 > 0, so the trial is always rejected; any pose step of that kind -- the unsolved
 * right-hand side b_s included, which gives |b_s|^2 + the same terms -- decides alike, so which one is taken
 * changes no result and no test can tell them apart.  A point observed
 * twice by one key-frame makes the call fail with YGZB_ERR_INVALID.                                     */
typedef struct {
    int max_iters;        /* optimizer.optimize(20)        */
    double huber_delta;   /* 5.991 (<= 0: no robust kernel) */
    double chi2_outlier;  /* 5.991                          */
    double tau;           /* g2o Levenberg tau (1e-5)       */
    int max_trials;       /* g2o maxTrialsAfterFailure (10) */
} ygzb_ba_params;
typedef struct {
    int iters, lm_trials;
    double chi2_initial, chi2_final, lambda_final;
    int n_outliers;
} ygzb_ba_stats;
void ygzb_default_ba_params(ygzb_ba_params* p);
int ygzb_local_ba(ygzb_ctx* ctx, int n_problems, const int32_t* kf_off, const int32_t* pt_off, const int32_t* obs_off,
                  double* poses, const uint8_t* fixed, double* pts, const int32_t* kf_idx, const int32_t* pt_idx,
                  const double* obs_px, const ygzb_ba_params* prm, uint8_t* outlier, ygzb_ba_stats* stats);

/* replaces ba::LocalBA, the Ceres twin of the local BA (src/Algorithm/BA.cpp:324-384; BA.h:52-58) with
 * CeresReprojectionError / CeresReprojectionErrorPointOnly (include/ygz/Ceres/CeresReprojectionError.h:33-69,
 * CeresReprojectionErrorPointOnly.h:14-67): residual pt_cam - p / p.z in normalised image coordinates, no loss,
 * default ceres::Solver::Options (trust-region LM with Jacobi scaling; max_iters = 50 there).  Same batching and index
 * conventions as ygzb_local_ba, except that a pose is 6 doubles [t(3); angle-axis(3)] (the Vector6d of BA.cpp:353-357)
 * and fixed[k] != 0 marks the key-frame with _keyframe_id == 0, whose observations become point-only residual blocks
 * (BA.cpp:340-349).  Observations in frames outside the local set are not part of the problem (BA.cpp:338): the
 * caller leaves them out.  obs_px are pixels; Pixel2Camera2D (float intrinsics of the context) is applied inside.
 * huber_a > 0 puts ceres::HuberLoss(huber_a) on every residual block (normalised image units): with it and the right
 * choice of free / fixed poses the same entry point is ba::OptimizeCurrent (BA.cpp:91-186: the current frame free, its
 * map points free, their other observers fixed, HuberLoss(0.1)) and ba::OptimizeCurrentPointOnly (:266-322: every pose
 * fixed, no loss); a problem without free poses is a pure point refinement.
 * termination: 0 max_iters reached, 1 gradient, 2 parameter, 3 function tolerance, 4 trust region collapsed.
 * The statistics follow the solver restated in oracle/ba.cpp, which may differ from ceres::Solver::Summary: the gradient
 * test runs before the iteration limit (max_iters = 0 evaluates once and reports 1 if the gradient is already below
 * 1e-10; a step accepted on the last allowed trial is still followed by the gradient test), and after a gradient exit
 * radius_final is the radius before the last step's update.  A landmark observed twice by one free pose returns
 * YGZB_ERR_INVALID, as in ygzb_local_ba.                                                                        */
typedef struct {
    int iters, successful_steps;
    double cost_initial, cost_final, radius_final;
    int termination;
} ygzb_ceres_stats;
int ygzb_local_ba_ceres(ygzb_ctx* ctx, int n_problems, const int32_t* kf_off, const int32_t* pt_off, const int32_t* obs_off,
                        double* poses, const uint8_t* fixed, double* pts, const int32_t* kf_idx, const int32_t* pt_idx,
                        const double* obs_px, int max_iters, double huber_a, ygzb_ceres_stats* stats);

/* replaces ba::TwoViewBACeres (src/Algorithm/BA.cpp:11-89; BA.h:23-30), the two-view bundle adjustment after the monocular
 * initialisation, for n_problems independent frame pairs: pair p owns points [offsets[p], offsets[p+1]) of px_ref / px_cur
 * (pixels), inlier (in/out) and pts (world points, in/out); T_cw_ref stays fixed (point-only residual blocks), T_cw_cur and
 * the points are refined; points that come in as non-inliers restart from (0,0,1) with ceres::HuberLoss(0.1) on their two
 * blocks (:31-56); afterwards inlier[i] = both squared pixel errors <= 5.991 and both depths positive (:70-84).
 * Solver: the trust-region Levenberg-Marquardt of ygzb_local_ba_ceres on the identical cost (the reference selects
 * ceres::DOGLEG; both strategies converge to the same minimum within the function tolerance).                   */
int ygzb_two_view_ba(ygzb_ctx* ctx, int n_problems, const int32_t* offsets, const double* T_cw_ref, double* T_cw_cur,
                     const double* px_ref, const double* px_cur, uint8_t* inlier, double* pts, ygzb_ceres_stats* stats);

/* replaces ba::OptimizeCurrentPoseOnly (src/Algorithm/BA.cpp:188-264; BA.h:44-46) with
 * CeresReprojectionErrorPoseOnly (include/ygz/Ceres/CeresReprojectionErrorPoseOnly.h): four rounds of
 * trust-region LM on [t; angle-axis] with re-classification of the observations between rounds.
 * Problem p owns points [offsets[p], offsets[p+1]); T_cw (3x4) in/out; inlier[i] = !Feature::_bad;
 * depth[i] = Feature::_depth written for inliers (-1 otherwise); n_inlier[p] = cntInlier.            */
int ygzb_pose_only(ygzb_ctx* ctx, int n_problems, const int32_t* offsets, const double* pt_world, const double* px,
                   double* T_cw, uint8_t* inlier, double* depth, int32_t* n_inlier);

/* ---- Tracker ------------------------------------------------------------------------------------
 * replaces Tracker::TrackKLT (src/Algorithm/Tracker.cpp:65-113; include/ygz/Algorithm/Tracker.h:31-58), i.e.
 * cv::calcOpticalFlowPyrLK(ref.pyr[0], cur.pyr[0], ..., Size(21,21), 4, (COUNT+EPS, 30, 0.001),
 * OPTFLOW_USE_INITIAL_FLOW).  Pair p tracks points [offsets[p], offsets[p+1]) from frame ref_slot[p] to
 * cur_slot[p]; ref_xy / cur_xy are full-resolution pixels (cur_xy = initial flow in, tracked position out),
 * status / err as OpenCV returns them.  The status filtering and Frame::InFrame(pt, 20) test of
 * Tracker.cpp:104-112 and MeanDisparity (:115-127) stay host bookkeeping in the shim.            */
typedef struct {
    int win;        /* Tracker::Option::klt_win_size = 21 (only 21 is supported) */
    int max_level;  /* 4 (Tracker.cpp:97)                                       */
    int max_iter;   /* klt_max_iter = 30                                        */
    double eps;     /* klt_eps = 0.001                                          */
    double min_eig; /* OpenCV default minEigThreshold 1e-4                      */
} ygzb_klt_params;
void ygzb_default_klt_params(ygzb_klt_params* p);
int ygzb_klt(ygzb_frames* f, int n_pairs, const int32_t* ref_slot, const int32_t* cur_slot, const int32_t* offsets,
             const float* ref_xy, float* cur_xy, uint8_t* status, float* err, const ygzb_klt_params* prm);


/* ---- device-resident tracking (VisualOdometry::TrackRefFrame + LocalMapping::TrackLocalMap + SetKeyframe) -----------
 * The per-stage calls above move every intermediate through host memory.  A tracker keeps the LOCAL MAP of `n_streams`
 * independent sequences on the device -- per stream a ring of YGZB_TRACK_RING key-frame entries (pose, features, depth,
 * map points, tracked observations; the reference keeps them in Memory / Frame / MapPoint objects, src/Basic) -- and runs
 * the whole per-frame chain as ONE asynchronous enqueue:
 *   Matcher::SparseImageAlignment against the reference key-frame (Matcher.cpp:468-492, VisualOdometry.cpp:281-302)
 *   -> LocalMapping::FindCandidates (LocalMapping.cpp:47-80: project the map points of the local key-frames, border 20)
 *   -> Matcher::FindDirectProjection per candidate (LocalMapping.cpp:82-111)
 *   -> ba::OptimizeCurrentPoseOnly on the projected points (LocalMapping.cpp:126, BA.cpp:188-264)
 * for a batch of (stream, frame) jobs; one small record per job comes back.  Frames of ONE stream may be batched as
 * long as none of them can become a key-frame before the last one (the tracker aligns every frame against the newest
 * key-frame, which is how a caller keeps several frames per stream in flight without changing any result).  This is
 * the engine's batching choice: the reference aligns a frame against the previous tracked frame, or the key-frame it
 * became (VisualOdometry.cpp:66, :88-90); ygz_slam_b200/vo.py implements that rule as ref_mode="previous".
 * ygzb_tracker_make_keyframes is VisualOdometry::SetKeyframe (:182-218) for a batch of streams: FeatureDetector::Detect
 * on the frame, map points from the depth image, insertion into the ring, and ba::LocalBAG2O over the local key-frames
 * and the points at least two of them observe (LocalMapping::LocalBA, LocalMapping.cpp:149-172) -- problem assembly,
 * optimisation and write-back all on the device.                                                                    */
#define YGZB_TRACK_RING 4
typedef struct ygzb_tracker ygzb_tracker;
typedef struct {
    int32_t stream;        /* sequence index                                                              */
    int32_t cur_slot;      /* frame slot with the current frame's pyramid (ygzb_frames_upload)             */
    int32_t n_local;       /* local key-frames, oldest first; the last one is the reference key-frame      */
    int32_t entry[YGZB_TRACK_RING]; /* their ring entries                                                  */
    int32_t pad;
} ygzb_track_job;
typedef struct {
    double T_cw[12];       /* pose after OptimizeCurrentPoseOnly (after the alignment if that failed)      */
    int32_t n_meas;        /* SparseImgAlign::run return value                                             */
    int32_t aligned;       /* Matcher::SparseImageAlignment's bool (motion norm <= 0.2)                    */
    int32_t n_candidates, n_projected, n_inliers;
    int32_t pad[3];
} ygzb_track_result;
typedef struct {
    int32_t stream;
    int32_t frame_slot;    /* slot of the frame that becomes a key-frame                                    */
    int32_t kf_slot;       /* slot that keeps its pyramid from now on (copied device-to-device)             */
    int32_t entry;         /* ring entry to (over)write                                                     */
    int32_t track_job;     /* job index in the LAST ygzb_tracker_track batch whose pose and inlier observations
                              the key-frame takes over, or -1: first key-frame (at the stream's start pose,
                              ygzb_tracker_set_start_pose; nothing tracked)                                  */
    int32_t n_local;       /* local key-frames AFTER the insertion, oldest first (the last one is `entry`)  */
    int32_t local_entry[YGZB_TRACK_RING];
    int32_t run_ba;        /* non-zero: LocalBAG2O over the local key-frames                                */
    int32_t pad;
    int64_t mp0;           /* id of the first map point the key-frame creates                               */
} ygzb_keyframe_job;
typedef struct {
    int32_t n_features;
    int32_t ba_points, ba_observations, ba_iters, ba_trials, pad;
    double chi2_initial, chi2_final;
    double T_cw[YGZB_TRACK_RING][12];   /* poses of the local key-frames after the BA, order of local_entry  */
} ygzb_keyframe_result;

/* K = {fx, fy, cx, cy} of the caller (doubles: the reference's callers project with PinholeCamera in double); with
 * undistortion maps on the pool (ygzb_frames_set_undistort), the undistorted camera newK. */
int ygzb_tracker_create(ygzb_frames* f, int n_streams, int max_jobs, const double K[4], ygzb_tracker** out);
void ygzb_tracker_destroy(ygzb_tracker* t);
/* depth image (image_width * image_height doubles, host or device) that initialises the map points of the next key-frame
 * of `stream` (the reference's drivers read it from the TUM depth frame, test/test_feature_alignment.cpp:72-85)   */
int ygzb_tracker_set_depth(ygzb_tracker* t, int stream, const double* depth);
/* T_cw (3x4 row-major) that the next first key-frame of `stream` (a key-frame job with track_job = -1) takes: it places a
 * sequence in the caller's world frame, as the reference's drivers do for their first frame
 * (test/test_feature_alignment.cpp:63); the key-frame's map points go to that world frame.  Identity from
 * ygzb_tracker_create.  Like ygzb_tracker_set_depth it applies to the insertions enqueued after it: the pose is read
 * before the call returns and travels with the key-frame jobs, so a later call never changes an insertion already
 * enqueued.  YGZB_ERR_INVALID, with the tracker untouched, for a NULL tracker or pose, a stream out of range, an entry
 * that is not finite, or a rotation that is not orthonormal with determinant +1 (within 1e-6 per entry).           */
int ygzb_tracker_set_start_pose(ygzb_tracker* t, int stream, const double T_cw[12]);
/* host -> device copy of `count` grey frames into slots [first, first+count) and their pyramids, like ygzb_frames_upload,
 * but on the tracker's second CUDA stream: behind the last key-frame insertion and tracking chain (which still read the
 * slots), concurrent with a local BA in flight.  ygzb_tracker_track orders itself behind these uploads.              */
int ygzb_tracker_upload(ygzb_tracker* t, int first, int count, const uint8_t* host, size_t frame_stride);
/* asynchronous: enqueues the chain on the context's stream and a copy of the n_jobs result records into `results`
 * (host memory, page-locked for a truly asynchronous copy); valid after ygzb_synchronize(ctx).                    */
int ygzb_tracker_track(ygzb_tracker* t, int n_jobs, const ygzb_track_job* jobs, ygzb_track_result* results);
/* asynchronous like ygzb_tracker_track; local BA problems of a batch run as one cluster launch.                   */
int ygzb_tracker_make_keyframes(ygzb_tracker* t, int n, const ygzb_keyframe_job* jobs, const ygzb_ba_params* ba,
                                ygzb_keyframe_result* results);

/* ---- map record: the local map of one stream, out of a tracker and back into one ----------------------------------
 * The reference keeps its map in Memory / MapPoint objects any caller can read, and its System declares SaveMap /
 * LoadMap (include/ygz/system.h:63-67, never defined).  A map record is the tracker's side of that: `n_keyframes` ring
 * entries of one stream as structure-of-arrays, sized by the caller from capacities (C = grid cells):
 *   per key-frame [n_keyframes]      entry, T_cw[12], mp0, n_features, n_obs, image (W*H bytes of level 0; may be NULL)
 *   per feature   [n_keyframes * C]  px[2], level, depth, pw[3]    packed key-frame after key-frame (n_features each)
 *   per observation [n_keyframes * 4 * C]  obs_id, obs_px[2]      packed the same way (n_obs each): the older map
 *                                                                   points tracked into the key-frame
 * The header carries the geometry the record was made under; an import checks it.  Serialising a record is the
 * caller's business.                                                                                               */
#define YGZB_MAP_OBS_PER_CELL 4   /* observation capacity of a key-frame per grid cell */
typedef struct {
    int32_t width, height, cells, n_levels;   /* image size, grid cells, pyramid levels                             */
    double K[4];                              /* fx, fy, cx, cy of the tracker (ygzb_tracker_create)                */
    int32_t n_keyframes, pad;
    int32_t* entry;        /* [n_keyframes] ring entry the key-frame was exported from                                */
    double* T_cw;          /* [n_keyframes][12]                                                                      */
    int64_t* mp0;          /* [n_keyframes] id of its first map point; ids are [mp0, mp0 + n_features)               */
    int32_t* n_features;   /* [n_keyframes]                                                                          */
    int32_t* n_obs;        /* [n_keyframes]                                                                          */
    uint8_t* image;        /* [n_keyframes][height][width] or NULL                                                   */
    double* px;            /* [n_keyframes * C][2] full-resolution pixel (Feature::_pixel)                            */
    uint8_t* level;        /* [n_keyframes * C]                                                                      */
    double* depth;         /* [n_keyframes * C]                                                                      */
    double* pw;            /* [n_keyframes * C][3] MapPoint::_pos_world                                              */
    int64_t* obs_id;       /* [n_keyframes * 4 * C] map point id                                                     */
    double* obs_px;        /* [n_keyframes * 4 * C][2] measured pixel                                                */
} ygzb_map_record;

/* asynchronous like ygzb_tracker_track, and ordered behind every key-frame insertion and local BA already enqueued (it
 * sees the BA's write-back): one kernel packs the live rows of ring entries entries[0 .. n_entries) of `stream` (and
 * their level-0 images when out->image != NULL) into a staging buffer, one copy per array moves them to `out`.  The
 * header, out->entry and out->n_keyframes are written before the call returns; everything else is valid after
 * ygzb_synchronize(ctx).  The per-feature and per-observation arrays are copied at their full capacity: the rows past
 * the live ones are zero.  Entries must be distinct and in [0, YGZB_TRACK_RING).                                     */
int ygzb_tracker_export(ygzb_tracker* t, int stream, int n_entries, const int32_t* entries, ygzb_map_record* out);
/* writes record `in` into ring entries entries[0 .. in->n_keyframes) of `stream` (any stream of any tracker with the same
 * geometry and K), uploads image k into frame slot kf_slots[k] and builds its pyramid (ygzb_frames_upload); the
 * entries' key-frame slots become kf_slots.  Asynchronous on the context's stream; the record is read before the call
 * returns unless its arrays are page-locked, then it must stay valid until ygzb_synchronize(ctx).  The whole record is
 * checked on the host first: a different geometry or K, a count over capacity, an entry or slot out of range or twice,
 * a level >= the pyramid depth or a missing image returns YGZB_ERR_INVALID with the tracker untouched.             */
int ygzb_tracker_import(ygzb_tracker* t, int stream, const int32_t* entries, const int32_t* kf_slots, const ygzb_map_record* in);

/* ---- reference record: what a stream in YGZB_TRACK_REF_PREVIOUS mode aligns its next frame against ------------------
 * In previous-frame mode (ygzb_tracker_set_reference_mode, below) a stream's state is its ring plus its current
 * reference: the pose, projected pixels and depths of the previous tracked frame or key-frame, and the pyramid of that
 * frame.  A reference record carries both out of a tracker and into another; together with the map record of the
 * stream's ring it is everything a stream tracked the reference's way needs to continue bit for bit.  The pyramid
 * travels as its level-0 image, from which the destination rebuilds it.  Capacity: at most
 * YGZB_TRACK_REF_FEATURES_PER_CELL * C features (C = grid cells), every tracked candidate of the local key-frames plus
 * the new features of a key-frame.                                                                                     */
#define YGZB_TRACK_REF_FEATURES_PER_CELL (YGZB_TRACK_RING + 1)
typedef struct {
    int32_t width, height, cells, n_levels;   /* as in ygzb_map_record                                              */
    double K[4];
    int32_t capacity;      /* in: rows px / depth hold; at least YGZB_TRACK_REF_FEATURES_PER_CELL * cells              */
    int32_t n;             /* features of the reference                                                              */
    double T_cw[12];       /* its pose                                                                               */
    double* px;            /* [capacity][2] full-resolution pixels, in the order the alignment reads them             */
    double* depth;         /* [capacity]                                                                             */
    uint8_t* image;        /* [height][width] level 0 of the pyramid the stream aligns its next frame against         */
} ygzb_reference_record;

/* asynchronous like ygzb_tracker_export, on the context's stream: ordered behind every tracking batch already enqueued
 * (including the copy of its last frame into the stream's reference slot) and every key-frame insertion (including the
 * key-frame's reference, written after its local BA).  One kernel packs the reference's rows, zeros up to the store's
 * capacity and level 0 of its pyramid into a staging buffer; one copy per field moves them to `out`.  The header is
 * written before the call returns; n, T_cw, px, depth and image are valid after ygzb_synchronize(ctx).  Rows past n are
 * zero.  YGZB_ERR_INVALID for a tracker in key-frame mode, a stream out of range or without a reference yet, a capacity
 * below YGZB_TRACK_REF_FEATURES_PER_CELL * cells, or a missing px, depth or image.                                    */
int ygzb_tracker_export_reference(ygzb_tracker* t, int stream, ygzb_reference_record* out);
/* writes record `in` as the current reference of `stream` (any stream of a previous-mode tracker with the same geometry
 * and K): pose, pixels and depths into the stream's reference store, the image into its reference slot with the pyramid
 * rebuilt (ygzb_frames_upload).  A reference that was a key-frame in the source lives in the reference slot here; the
 * pixels are the same, and so are the results.  Like a key-frame insertion, it fixes the reference mode.  Asynchronous
 * on the context's stream like ygzb_tracker_import.  The whole record is checked first: a tracker in key-frame mode, a
 * stream out of range, a capacity below the store's, n < 0 or above it, a different geometry or K, or a missing px,
 * depth or image returns YGZB_ERR_INVALID with the tracker untouched.
 * A stream moves to another tracker in this order: ygzb_tracker_set_reference_mode(YGZB_TRACK_REF_PREVIOUS, ref_slots),
 * ygzb_tracker_import (its map), ygzb_tracker_import_reference.                                                     */
int ygzb_tracker_import_reference(ygzb_tracker* t, int stream, const ygzb_reference_record* in);

/* ---- parity / debug view of the last tracking batch (tests; not part of the tracking path, like ygzb_fast_debug) ------
 * Synchronous: waits for the context's stream, then copies out the intermediate state of job `job` of the most recent
 * ygzb_tracker_track batch (valid until the next ygzb_tracker_track).  The caller sizes every array for
 * YGZB_MAP_OBS_PER_CELL * C entries (C = grid cells): the dense arrays are indexed by local key-frame k * C + feature, the
 * compacted ones by the candidate order; entries of cand_px are only written for candidates, entries past n_projected
 * of the compacted arrays are left over from earlier batches.                                                      */
typedef struct {
    double T_aligned[12];               /* T_cw after the sparse alignment and the key-frame pose (pose-only's start) */
    double rel[YGZB_TRACK_RING][12];    /* T_aligned * T_cw(local key-frame k)^-1, first n_local rows               */
    int32_t n_local, n_meas, aligned;
    int32_t n_candidates;               /* FindCandidates: z > 0 and inside the border of 20 px                      */
    int32_t n_projected;                /* FindDirectProjection succeeded: the compacted count                       */
    int32_t n_inliers;                  /* pose-only's count (also when aligned == 0)                                */
    uint8_t* cand_ok;                   /* [4 C] direct projection succeeded                                         */
    double* cand_px;                    /* [4 C][2] its result                                                       */
    int32_t* c_src;                     /* [4 C] dense index of compacted candidate i                                */
    double* c_px;                       /* [4 C][2]                                                                  */
    double* c_pw;                       /* [4 C][3] the map point                                                    */
    uint8_t* inlier;                    /* [4 C] pose-only's inlier flag                                             */
} ygzb_track_debug;
int ygzb_tracker_debug_job(ygzb_tracker* t, int job, ygzb_track_debug* out);

/* ---- what a frame is aligned against --------------------------------------------------------------------------------
 * YGZB_TRACK_REF_KEYFRAME (the default): the newest local key-frame (job.entry[n_local - 1]); the frames of a batch are
 * independent, and the alignment of a batch overlaps the local BA in flight.
 * YGZB_TRACK_REF_PREVIOUS: the reference's rule (VisualOdometry.cpp:66, :88-90) -- the stream's previous tracked frame,
 * with its pose-only pose and its projected candidates in candidate order (inliers at the depth of their map point
 * under that pose, outliers at the depth pose-only left them: that of their last inlier round, or -1), or, after
 * ygzb_tracker_make_keyframes, the key-frame with its pose after the local BA, its tracked features (inlier depths
 * from the BA's points) and then its new features.  The jobs of one stream in a batch are tracked in batch order, each
 * against the one before it, the first against the stream's reference; a batch runs as waves (the w-th job of every
 * stream) without a host synchronisation.  Behind the batch, the pyramid of the stream's last job is copied into
 * ref_slots[stream], which must be distinct slots that no frame or key-frame uses; a key-frame reference uses its kf_slot.
 * The next batch's alignment waits for the local BA.  The mode can only be set before the first key-frame insertion;
 * otherwise, and for an unknown mode or missing, out-of-range or shared reference slots, YGZB_ERR_INVALID with the
 * tracker untouched.                                                                                                  */
#define YGZB_TRACK_REF_KEYFRAME 0
#define YGZB_TRACK_REF_PREVIOUS 1
int ygzb_tracker_set_reference_mode(ygzb_tracker* t, int mode, const int32_t* ref_slots /* [n_streams] */);

/* synchronous, for tests (like ygzb_tracker_debug_job): the current reference of a stream in YGZB_TRACK_REF_PREVIOUS
 * mode.  The caller sets capacity and sizes px [capacity][2] and depth [capacity]; a larger reference returns
 * YGZB_ERR_CAPACITY.  At most YGZB_TRACK_REF_FEATURES_PER_CELL * grid cells features.  ygzb_tracker_export_reference
 * reads the same reference asynchronously, with its image.                                                           */
typedef struct {
    int32_t slot;          /* slot of its pyramid */
    int32_t n;             /* features */
    int32_t capacity;      /* in: entries px / depth can hold */
    int32_t pad;
    double T_cw[12];
    double* px;
    double* depth;
} ygzb_track_reference;
int ygzb_tracker_debug_reference(ygzb_tracker* t, int stream, ygzb_track_reference* out);

#ifdef __cplusplus
}
#endif
#endif /* YGZ_B200_H_ */
