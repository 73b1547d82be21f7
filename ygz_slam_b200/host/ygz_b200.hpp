// ygz_b200.hpp -- host-side C++ mirror of the reference's call surface for the tracking + local-BA hot path,
// implemented on top of the C ABI (include/ygz_b200.h).  Same class / method names, argument meaning and
// bool/enum error behaviour as the reference headers, so the callers in src/Module compile against it:
//
//   ygz::FeatureDetector   include/ygz/Algorithm/FeatureDetector.h:43-101
//   ygz::Matcher           include/ygz/Algorithm/Matcher.h:15-155
//   ygz::Tracker           include/ygz/Algorithm/Tracker.h:11-76
//   ygz::cvutils::Align2D  include/ygz/Algorithm/CVUtils.h:163-169
//   ygz::SparseImgAlign    include/ygz/Algorithm/SparseImageAlign.h:12-58
//   ygz::ba::*             include/ygz/Algorithm/BA.h:23-66
//   ygz::Frame / Feature / MapPoint / PinholeCamera   include/ygz/Basic/*.h (data carriers only)
//   ygz::Optimizer         facade over ygz::ba for the north star's vocabulary (the reference has no such class)
//
// The reference's data types depend on Eigen / OpenCV / Sophus, which are not part of this repo: minimal
// stand-ins with the same member names are provided (Vector2d, Vector3d, SE3, Mat).  A port that keeps the
// real Eigen/Sophus types only has to replace the conversions in b200::detail.
// No computation happens here: every method marshals AoS <-> SoA and calls ygzb_*.
#pragma once

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <list>
#include <cmath>
#include <map>
#include <memory>
#include <set>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/ygz_b200.h"
#include "../csrc/se3.cuh"

namespace ygz {

struct Vector2d {
    double v[2]{0, 0};
    Vector2d() = default;
    Vector2d(double x, double y) : v{x, y} {}
    double& operator[](int i) { return v[i]; }
    double operator[](int i) const { return v[i]; }
};
struct Vector3d {
    double v[3]{0, 0, 0};
    Vector3d() = default;
    Vector3d(double x, double y, double z) : v{x, y, z} {}
    double& operator[](int i) { return v[i]; }
    double operator[](int i) const { return v[i]; }
};

// stand-in for Sophus::SE3 (quaternion + translation, same arithmetic as thirdparty/Sophus)
struct SE3 {
    ygzb::SE3d T{{1, 0, 0, 0}, {0, 0, 0}};
    SE3() = default;
    explicit SE3(const ygzb::SE3d& t) : T(t) {}
    SE3 operator*(const SE3& o) const { return SE3(ygzb::se3_mul(T, o.T)); }
    Vector3d operator*(const Vector3d& p) const {
        const ygzb::V3d r = ygzb::transform(T, ygzb::V3d{p[0], p[1], p[2]});
        return Vector3d(r.x, r.y, r.z);
    }
    SE3 inverse() const { return SE3(ygzb::se3_inverse(T)); }
    Vector3d translation() const { return Vector3d(T.t.x, T.t.y, T.t.z); }
    void matrix3x4(double* out) const { ygzb::se3_to_mat(T, out); }
    static SE3 from3x4(const double* m) { return SE3(ygzb::se3_from_mat(m)); }
    static SE3 exp(const double* upsilon_omega) { return SE3(ygzb::se3_exp(upsilon_omega)); }
    void log(double* upsilon_omega) const { ygzb::se3_log(T, upsilon_omega); }
};

// 8-bit image view (stand-in for the CV_8U cv::Mat members)
struct Mat {
    std::vector<uint8_t> buf;
    int rows = 0, cols = 0, channels = 1;
    uint8_t* data = nullptr;
    void create(int r, int c, int ch = 1) {
        rows = r; cols = c; channels = ch;
        buf.assign((size_t)r * c * ch, 0);
        data = buf.data();
    }
};

struct Frame;
struct MapPoint;

struct Feature {  // include/ygz/Basic/Feature.h:15-36
    Feature(const Vector2d& pixel, const int& level = 0, const double& score = 0) : _pixel(pixel), _level(level), _score(score) {}
    Vector2d _pixel;
    double _depth = -1;
    int _level = -1;
    double _angle = 0;
    uint8_t _desc[32]{};
    Frame* _frame = nullptr;
    MapPoint* _mappoint = nullptr;
    bool _bad = false;
    double _score = 0;
};

struct MapPoint {  // include/ygz/Basic/MapPoint.h:17-46 (fields used on the hot path)
    unsigned long _id = 0;
    Vector3d _pos_world;
    bool _bad = false;
    int _cnt_found = 0, _cnt_visible = 0;
    unsigned long _first_seen = 0, _last_seen = 0;
    std::map<unsigned long, Feature*> _obs;  // keyframe id -> feature
};

class PinholeCamera {  // include/ygz/Basic/Camera.h:10-112
  public:
    PinholeCamera(float fx = 520.9f, float fy = 521.0f, float cx = 325.1f, float cy = 249.7f, float k1 = 0.f, float k2 = 0.f, float p1 = 0.f,
                  float p2 = 0.f)
        : _fx(fx), _fy(fy), _cx(cx), _cy(cy), _k1(k1), _k2(k2), _p1(p1), _p2(p2) {}
    // camera.k1 k2 p1 p2 (Camera.h:19-22): the radial-tangential model of UndistortPoint (:96-104).  The reference stores
    // them and never applies them; b200::Runtime::SetUndistortion(camera) undistorts every later InitFrame with them.
    float k1() const { return _k1; }
    float k2() const { return _k2; }
    float p1() const { return _p1; }
    float p2() const { return _p2; }
    Vector3d World2Camera(const Vector3d& p_w, const SE3& T_c_w) const { return T_c_w * p_w; }
    Vector2d Camera2Pixel(const Vector3d& p) const { return Vector2d(_fx * p[0] / p[2] + _cx, _fy * p[1] / p[2] + _cy); }
    Vector2d World2Pixel(const Vector3d& p_w, const SE3& T) const { return Camera2Pixel(World2Camera(p_w, T)); }
    Vector3d Camera2World(const Vector3d& p_c, const SE3& T_c_w) const { return T_c_w.inverse() * p_c; }             // Camera.h:45-47
    Vector3d Pixel2Camera(const Vector2d& p, double depth = 1) const {                                                // Camera.h:56-62
        return Vector3d((p[0] - _cx) * depth / _fx, (p[1] - _cy) * depth / _fy, depth);
    }
    float fx() const { return _fx; }
    float fy() const { return _fy; }
    float cx() const { return _cx; }
    float cy() const { return _cy; }
  protected:
    float _fx, _fy, _cx, _cy;
    float _k1, _k2, _p1, _p2;
};

class ORBVocabulary;

struct Frame {  // include/ygz/Basic/Frame.h:20-166 (fields used on the hot path)
    struct Option { int _pyramid_level = 3; } _option;
    ~Frame();          // releases the device pyramid slot: a frame pins its slot for as long as it lives (key-frames in Memory: for good)
    void InitFrame();  // cvtColor + pyrDown chain (src/Basic/Frame.cpp:22-40) -> device pyramid
    bool InFrame(const Vector2d& px, const int& boarder = 10) const {
        return px[0] >= boarder && px[0] < _color.cols - boarder && px[1] >= boarder && px[1] < _color.rows - boarder;
    }
    void CleanAllFeatures() {
        for (Feature* f : _features) delete f;
        _features.clear();
    }
    static void SetCamera(PinholeCamera* c) { _camera = c; }
    static void SetORBVocabulary(ORBVocabulary* v) { _vocab = v; }   // Frame.h:101
    Vector3d GetCamCenter() const { return _TCW.inverse().translation(); }                  // Frame.h:77-80
    bool GetMeanAndMinDepth(double& mean_depth, double& min_depth) const {                   // Frame.cpp:42-71
        mean_depth = 0;
        min_depth = 9999;
        int cnt = 0;
        for (const Feature* f : _features) {
            if (f->_mappoint == nullptr || f->_mappoint->_bad) continue;
            const double depth = (_TCW * f->_mappoint->_pos_world)[2];
            if (depth < 0) continue;
            ++cnt;
            mean_depth += depth;
            if (depth < min_depth) min_depth = depth;
        }
        if (cnt == 0) {
            mean_depth = min_depth = 0;
            return false;
        }
        mean_depth /= cnt;
        return true;
    }
    void ComputeBoW();   // Frame.cpp:190-201: _vocab->transform(all descriptors, _bow_vec, _feature_vec, 4)
    unsigned long _id = 0, _keyframe_id = 0;
    SE3 _TCW;
    bool _is_keyframe = false;
    std::vector<Feature*> _features;
    Mat _color;                 // BGR (3 channels) or grey (1 channel) input image
    std::map<unsigned, std::vector<unsigned>> _feature_vec;   // DBoW3::FeatureVector of Frame::ComputeBoW (Frame.cpp:190-201): node -> feature indices
    std::map<unsigned, double> _bow_vec;                      // DBoW3::BowVector: word -> normalised tf-idf
    int _slot = -1;             // device pyramid slot (set by InitFrame)
    static inline PinholeCamera* _camera = nullptr;
    static inline ORBVocabulary* _vocab = nullptr;
};

// ---------------------------------------------------------------------------------------------------
namespace b200 {

struct Error : std::runtime_error { using std::runtime_error::runtime_error; };

// process-wide device runtime: one ygzb context + a pool of frame slots (one context per host thread:
// like the reference, the algorithm classes are single-threaded)
class Runtime {
  public:
    static Runtime& Get() {
        static Runtime r;
        return r;
    }
    void Configure(const ygzb_params& p, int device = 0, int slots = 64) {
        Release();
        if (ygzb_create(device, &p, &ctx_) != YGZB_OK) {
            std::string m = ctx_ ? ygzb_last_error(ctx_) : "no sm_90 device (there is no CPU fallback)";
            if (ctx_) ygzb_destroy(ctx_);
            ctx_ = nullptr;
            throw Error("ygzb_create: " + m);
        }
        Check(ygzb_frames_create(ctx_, slots, &frames_), "ygzb_frames_create");
        params_ = p;
        owner_.assign(slots, nullptr);
        free_.clear();
        for (int i = slots - 1; i >= 0; --i) free_.push_back(i);   // slot 0 is handed out first
    }
    ygzb_ctx* ctx() { Ensure(); return ctx_; }
    ygzb_frames* frames() { Ensure(); return frames_; }
    const ygzb_params& params() { Ensure(); return params_; }
    // explicit slot ownership: a Frame pins its slot from InitFrame until it is destroyed (the reference keeps the cv::Mat
    // pyramid alive through the Frame object, Frame.h:138; Memory keeps key-frames forever, Memory.cpp:7-19), so a live
    // key-frame can never lose its pyramid.  Running out of slots is an error the caller sees: Configure(.., slots) sizes the pool.
    int AcquireSlot(Frame* f) {
        Ensure();
        if (free_.empty()) throw Error("out of device frame slots: " + std::to_string(owner_.size()) +
                                       " frames are alive; raise the `slots` argument of b200::Runtime::Configure");
        const int s = free_.back();
        free_.pop_back();
        owner_[s] = f;
        return s;
    }
    void ReleaseSlot(Frame* f, int s) {
        if (s >= 0 && s < (int)owner_.size() && owner_[s] == f) {
            owner_[s] = nullptr;
            free_.push_back(s);
        }
    }
    int FreeSlots() const { return (int)free_.size(); }
    // undistort every later Frame::InitFrame with the camera's k1 k2 p1 p2 (k3 = 0, the model of Camera.h:96-104): the maps of
    // cv::initUndistortRectifyMap(K, D, I, K) are built on the host (ygzb_undistort_map) and set on the pool
    // (ygzb_frames_set_undistort).  The undistorted camera keeps K, so the same PinholeCamera projects the undistorted
    // frames.  A camera without distortion clears the maps.
    void SetUndistortion(const PinholeCamera& cam) {
        Ensure();
        if (cam.k1() == 0.f && cam.k2() == 0.f && cam.p1() == 0.f && cam.p2() == 0.f) {
            Check(ygzb_frames_set_undistort(frames_, nullptr, nullptr), "ygzb_frames_set_undistort");
            return;
        }
        const int w = params_.image_width, h = params_.image_height;
        const double K[4] = {cam.fx(), cam.fy(), cam.cx(), cam.cy()};
        const double D[5] = {cam.k1(), cam.k2(), cam.p1(), cam.p2(), 0.0};
        std::vector<int16_t> xy((size_t)w * h * 2);
        std::vector<uint16_t> a((size_t)w * h);
        Check(ygzb_undistort_map(w, h, K, D, nullptr, xy.data(), a.data()), "ygzb_undistort_map");
        Check(ygzb_frames_set_undistort(frames_, xy.data(), a.data()), "ygzb_frames_set_undistort");
    }
    void Check(int rc, const char* what) {
        if (rc != YGZB_OK) throw Error(std::string(what) + ": " + (ctx_ ? ygzb_last_error(ctx_) : "?"));
    }
    void Release() {
        if (frames_) ygzb_frames_destroy(frames_);
        if (ctx_) ygzb_destroy(ctx_);
        frames_ = nullptr;
        ctx_ = nullptr;
    }
    ~Runtime() { Release(); }
  private:
    void Ensure() {
        if (!ctx_) {
            ygzb_params p;
            ygzb_default_params(&p);
            Configure(p);
        }
    }
    ygzb_ctx* ctx_ = nullptr;
    ygzb_frames* frames_ = nullptr;
    ygzb_params params_{};
    std::vector<Frame*> owner_;
    std::vector<int> free_;
};

inline int SlotOf(Frame* f) {
    if (f->_slot < 0) throw Error("Frame::InitFrame() has not been called");
    return f->_slot;
}
inline void PoseTo3x4(const SE3& T, double* out) { T.matrix3x4(out); }

}  // namespace b200

inline Frame::~Frame() {
    CleanAllFeatures();
    if (_slot >= 0) b200::Runtime::Get().ReleaseSlot(this, _slot);
}

inline void Frame::InitFrame() {
    auto& rt = b200::Runtime::Get();
    if (_slot < 0) _slot = rt.AcquireSlot(this);   // (a second InitFrame of the same frame re-uses its slot)
    rt.Check(ygzb_frames_upload(rt.frames(), _slot, 1, _color.data, _color.channels, (size_t)_color.rows * _color.cols * _color.channels),
             "ygzb_frames_upload");
}

// DBoW3::Vocabulary as the reference uses it (typedef DBoW3::Vocabulary ORBVocabulary, Common.h): the tree lives on the device
class ORBVocabulary {
  public:
    typedef std::map<unsigned, double> BowVector;                        // DBoW3/BowVector.h:52
    typedef std::map<unsigned, std::vector<unsigned>> FeatureVector;     // DBoW3/FeatureVector.h
    ORBVocabulary() = default;
    ORBVocabulary(const ORBVocabulary&) = delete;
    ORBVocabulary& operator=(const ORBVocabulary&) = delete;
    ~ORBVocabulary() { clear(); }
    // Vocabulary.cpp:1180-1225; false if the file cannot be read or is malformed (the reference does not check)
    bool loadFromBinaryFile(const std::string& filename) {
        std::FILE* f = std::fopen(filename.c_str(), "rb");
        if (!f) return false;
        std::vector<uint8_t> bytes;
        uint8_t buf[1 << 16];
        size_t got;
        while ((got = std::fread(buf, 1, sizeof buf, f)) > 0) bytes.insert(bytes.end(), buf, buf + got);
        std::fclose(f);
        return loadFromMemory(bytes.data(), bytes.size());
    }
    bool loadFromMemory(const void* bytes, size_t n) {
        clear();
        auto& rt = b200::Runtime::Get();
        if (ygzb_vocab_create(rt.ctx(), bytes, n, &v_) != YGZB_OK) {
            v_ = nullptr;
            return false;
        }
        return true;
    }
    bool empty() const { return v_ == nullptr; }
    unsigned size() const { return (unsigned)info(5); }                   // number of words
    int getBranchingFactor() const { return info(0); }
    int getDepthLevels() const { return info(1); }
    // Vocabulary.cpp:706-776; features = 32-byte descriptors
    void transform(const std::vector<const uint8_t*>& features, BowVector& v, FeatureVector& fv, int levelsup) const {
        v.clear();
        fv.clear();
        if (empty() || features.empty()) return;
        auto& rt = b200::Runtime::Get();
        const int n = (int)features.size();
        std::vector<uint8_t> desc((size_t)n * 32);
        for (int i = 0; i < n; ++i) std::memcpy(&desc[(size_t)i * 32], features[i], 32);
        const int32_t off[2] = {0, n};
        std::vector<int32_t> word(n), node(n), bw(n);
        std::vector<double> weight(n), bv(n);
        int32_t cnt = 0;
        rt.Check(ygzb_bow_transform(v_, 1, off, desc.data(), levelsup, word.data(), node.data(), weight.data(), &cnt, bw.data(), bv.data()),
                 "ygzb_bow_transform");
        for (int q = 0; q < cnt; ++q) v.emplace_hint(v.end(), (unsigned)bw[q], bv[q]);
        for (int i = 0; i < n; ++i)
            if (node[i] >= 0) fv[(unsigned)node[i]].push_back((unsigned)i);
    }
    void clear() {
        if (v_) ygzb_vocab_destroy(v_);
        v_ = nullptr;
    }
  private:
    int info(int i) const {
        int32_t a[6] = {0, 0, 0, 0, 0, 0};
        if (v_) ygzb_vocab_info(v_, a);
        return a[i];
    }
    ygzb_vocab* v_ = nullptr;
};

inline void Frame::ComputeBoW() {
    if (_vocab != nullptr && _bow_vec.empty()) {
        std::vector<const uint8_t*> alldesp;
        for (Feature* fea : _features) alldesp.push_back(fea->_desc);
        _vocab->transform(alldesp, _bow_vec, _feature_vec, 4);
    }
}

// ---------------------------------------------------------------------------------------------------
class FeatureDetector {  // include/ygz/Algorithm/FeatureDetector.h
  public:
    struct Option {
        int _image_width = 640, _image_height = 480;
        int _cell_size = 10;
        int _grid_rows = 0, _grid_cols = 0;
        double _detection_threshold = 15.0;
    } _option;
    FeatureDetector() { LoadParams(); }
    void LoadParams() {
        const ygzb_params& p = b200::Runtime::Get().params();
        _option._image_width = p.image_width;
        _option._image_height = p.image_height;
        _option._cell_size = p.cell_size;
        _option._detection_threshold = p.fast_threshold;
        ygzb_grid_dims(b200::Runtime::Get().ctx(), &_option._grid_rows, &_option._grid_cols);
    }
    // FeatureDetector.cpp:345-444
    void Detect(Frame* frame, bool overwrite_existing_features = true) {
        auto& rt = b200::Runtime::Get();
        const int n_cells = _option._grid_rows * _option._grid_cols;
        std::vector<uint8_t> occ;
        if (overwrite_existing_features) {
            frame->CleanAllFeatures();
        } else {  // SetExistingFeatures (:446-464)
            occ.assign(n_cells, 0);
            for (Feature* fea : frame->_features) {
                const int gx = (int)(fea->_pixel[0] / _option._cell_size), gy = (int)(fea->_pixel[1] / _option._cell_size);
                const size_t k = (size_t)gy * _option._grid_cols + gx;
                if (k < occ.size()) occ[k] = 1;
            }
        }
        std::vector<int32_t> off(2), cell(n_cells);
        std::vector<float> x(n_cells), y(n_cells), score(n_cells), angle(n_cells);
        std::vector<uint8_t> level(n_cells), desc((size_t)n_cells * 32);
        ygzb_keypoints kp{off.data(), x.data(), y.data(), level.data(), score.data(), angle.data(), desc.data(), cell.data(), n_cells};
        const int32_t slot = b200::SlotOf(frame);
        rt.Check(ygzb_detect(rt.frames(), &slot, 1, occ.empty() ? nullptr : occ.data(), &kp), "ygzb_detect");
        for (int i = 0; i < off[1]; ++i) {
            Feature* fea = new Feature(Vector2d(x[i], y[i]), level[i], score[i]);
            fea->_frame = frame;
            fea->_angle = angle[i];
            std::memcpy(fea->_desc, &desc[(size_t)i * 32], 32);
            frame->_features.push_back(fea);
        }
    }
    // FeatureDetector.cpp:580-588
    void ComputeAngleAndDescriptor(Frame* frame) {
        auto& rt = b200::Runtime::Get();
        const int n = (int)frame->_features.size();
        if (!n) return;
        std::vector<double> x(n), y(n);
        std::vector<uint8_t> level(n), desc((size_t)n * 32);
        std::vector<float> angle(n);
        for (int i = 0; i < n; ++i) {
            x[i] = frame->_features[i]->_pixel[0];
            y[i] = frame->_features[i]->_pixel[1];
            level[i] = (uint8_t)frame->_features[i]->_level;
        }
        const int32_t slot = b200::SlotOf(frame), off[2] = {0, n};
        rt.Check(ygzb_describe(rt.frames(), &slot, 1, off, x.data(), y.data(), level.data(), angle.data(), desc.data()), "ygzb_describe");
        for (int i = 0; i < n; ++i) {
            frame->_features[i]->_angle = angle[i];
            std::memcpy(frame->_features[i]->_desc, &desc[(size_t)i * 32], 32);
        }
    }
    // FeatureDetector.cpp:591-594 (no caller in the reference).  The reference rebuilds the descriptor with the angle the
    // feature carries; a feature that came out of Detect / ComputeAngleAndDescriptor carries the IC angle of its pixel, which is
    // what the device computes, so the descriptor is the same and the angle is left untouched.
    void ComputeDescriptor(Feature* fea) {
        auto& rt = b200::Runtime::Get();
        const double x = fea->_pixel[0], y = fea->_pixel[1];
        const uint8_t level = (uint8_t)fea->_level;
        float angle = 0;
        const int32_t slot = b200::SlotOf(fea->_frame), off[2] = {0, 1};
        rt.Check(ygzb_describe(rt.frames(), &slot, 1, off, &x, &y, &level, &angle, fea->_desc), "ygzb_describe");
    }
};

namespace cvutils {
// Host-side helpers of include/ygz/Algorithm/CVUtils.h that the reference's callers use directly (pure arithmetic: the device
// kernels carry their own copies).  Matrix<double,2,6> is a plain row-major array here.
struct Matrix26d {
    double m[2][6];
    double operator()(int r, int c) const { return m[r][c]; }
    double& operator()(int r, int c) { return m[r][c]; }
};
// CVUtils.h:77-99 (translation first, already negated)
inline Matrix26d JacobXYZ2Cam(const Vector3d& xyz) {
    Matrix26d J;
    const double x = xyz[0], y = xyz[1], z_inv = 1. / xyz[2], z_inv_2 = z_inv * z_inv;
    J(0, 0) = -z_inv; J(0, 1) = 0.0; J(0, 2) = x * z_inv_2; J(0, 3) = y * J(0, 2); J(0, 4) = -(1.0 + x * J(0, 2)); J(0, 5) = y * z_inv;
    J(1, 0) = 0.0; J(1, 1) = -z_inv; J(1, 2) = y * z_inv_2; J(1, 3) = 1.0 + y * J(1, 2); J(1, 4) = -J(0, 3); J(1, 5) = -x * z_inv;
    return J;
}
// CVUtils.h:101-126
inline Matrix26d JacobXYZ2Pixel(const Vector3d& xyz, PinholeCamera* cam) {
    Matrix26d J;
    const double x = xyz[0], y = xyz[1], z_inv = 1. / xyz[2], z_inv_2 = z_inv * z_inv;
    J(0, 0) = -z_inv * cam->fx(); J(0, 1) = 0.0; J(0, 2) = x * z_inv_2 * cam->fx(); J(0, 3) = cam->fx() * y * J(0, 2);
    J(0, 4) = -cam->fx() * (1.0 + x * J(0, 2)); J(0, 5) = cam->fx() * y * z_inv;
    J(1, 0) = 0.0; J(1, 1) = -cam->fy() * z_inv; J(1, 2) = cam->fy() * y * z_inv_2; J(1, 3) = cam->fy() * (1.0 + y * J(1, 2));
    J(1, 4) = -cam->fy() * x * J(1, 2); J(1, 5) = -cam->fy() * x * z_inv;
    return J;
}
// CVUtils.h:59-71 / :41-57 on a host-resident single-channel image (row pitch = cols)
inline uint8_t GetBilateralInterpUchar(const double& x, const double& y, const Mat& gray) {
    const double xx = x - std::floor(x), yy = y - std::floor(y);
    const uint8_t* d = &gray.data[(size_t)int(y) * gray.cols + int(x)];
    return uint8_t((1 - xx) * (1 - yy) * d[0] + xx * (1 - yy) * d[1] + (1 - xx) * yy * d[gray.cols] + xx * yy * d[gray.cols + 1]);
}
inline float GetBilateralInterp(const double& x, const double& y, const Mat& gray) {
    const double xx = x - std::floor(x), yy = y - std::floor(y);
    const uint8_t* d = &gray.data[(size_t)int(y) * gray.cols + int(x)];
    return float((1 - xx) * (1 - yy) * d[0] + xx * (1 - yy) * d[1] + (1 - xx) * yy * d[gray.cols] + xx * yy * d[gray.cols + 1]);
}
// CVUtils.h:18-38
inline bool DepthFromTriangulation(const SE3& T_search_ref, const Vector3d& f_ref, const Vector3d& f_cur, double& depth1, double& depth2,
                                   const double& determinant_th = 1e-5) {
    auto& rt = b200::Runtime::Get();
    double T[12];
    T_search_ref.matrix3x4(T);
    const double fr[3] = {f_ref[0], f_ref[1], f_ref[2]}, fc[3] = {f_cur[0], f_cur[1], f_cur[2]};
    uint8_t ok = 0;
    rt.Check(ygzb_depth_from_triangulation(rt.ctx(), 1, 1, T, nullptr, fr, fc, determinant_th, &depth1, &depth2, &ok), "ygzb_depth_from_triangulation");
    return ok != 0;
}
// include/ygz/Algorithm/CVUtils.h:163-169 -- cur_img is identified by (frame, level) instead of a cv::Mat
inline bool Align2D(Frame* cur, int level, uint8_t* ref_patch_with_border, uint8_t* ref_patch, const int n_iter, Vector2d& cur_px_estimate) {
    auto& rt = b200::Runtime::Get();
    const int32_t slot = b200::SlotOf(cur);
    const uint8_t lv = (uint8_t)level;
    double uv[2] = {cur_px_estimate[0], cur_px_estimate[1]};
    uint8_t ok = 0;
    rt.Check(ygzb_align2d(rt.frames(), 1, &slot, &lv, ref_patch_with_border, ref_patch, n_iter, uv, &ok), "ygzb_align2d");
    cur_px_estimate = Vector2d(uv[0], uv[1]);
    return ok != 0;
}
}  // namespace cvutils

// Matrix<double,6,6> is a plain row-major array here (SparseImgAlign::getFisherInformation's return type)
struct Matrix66d {
    double m[6][6] = {};
    double operator()(int r, int c) const { return m[r][c]; }
    double& operator()(int r, int c) { return m[r][c]; }
};

class SparseImgAlign {  // include/ygz/Algorithm/SparseImageAlign.h:12-58
  public:
    enum Method { GaussNewton, LevenbergMarquardt };
    SparseImgAlign(int max_level, int min_level, int n_iter, Method = GaussNewton, bool = false, bool = false)
        : max_level_(max_level), min_level_(min_level), n_iter_(n_iter) {}
    size_t run(Frame* ref_frame, Frame* cur_frame) {
        auto& rt = b200::Runtime::Get();
        const int n = (int)ref_frame->_features.size();
        fisher_ = Matrix66d{};
        if (!n) return 0;
        std::vector<double> px(2 * (size_t)n), depth(n);
        std::vector<uint8_t> has(n);
        for (int i = 0; i < n; ++i) {
            const Feature* f = ref_frame->_features[i];
            px[2 * i] = f->_pixel[0];
            px[2 * i + 1] = f->_pixel[1];
            depth[i] = f->_depth;
            has[i] = f->_mappoint != nullptr;
        }
        double Tr[12], Tc[12];
        b200::PoseTo3x4(ref_frame->_TCW, Tr);
        b200::PoseTo3x4(cur_frame->_TCW, Tc);
        const int32_t rs = b200::SlotOf(ref_frame), cs = b200::SlotOf(cur_frame), off[2] = {0, n};
        int32_t n_meas = 0;
        double packed[21];
        rt.Check(ygzb_sparse_align_fisher(rt.frames(), 1, &rs, &cs, off, px.data(), depth.data(), has.data(), Tr, Tc, max_level_, min_level_,
                                          n_iter_, 0.000001, &n_meas, nullptr, packed),
                 "ygzb_sparse_align_fisher");
        for (int r = 0, t = 0; r < 6; ++r)
            for (int c = r; c < 6; ++c, ++t) fisher_(r, c) = fisher_(c, r) = packed[t];
        cur_frame->_TCW = SE3::from3x4(Tc);
        return (size_t)n_meas;
    }
    // SparseImageAlign.cpp:52-57: H_ / (5e-4 * 255^2) of the last run (zeros before any run, or after one that had no feature
    // or n_iter = 0, where the reference keeps a stale H_)
    Matrix66d getFisherInformation() const { return fisher_; }
  private:
    int max_level_, min_level_, n_iter_;
    Matrix66d fisher_;
};

class Matcher {  // include/ygz/Algorithm/Matcher.h
  public:
    struct Options {
        float initMatchRatio = 3.0;
        int init_low = 30, init_high = 100;  // matcher.init_low / init_high (config/default.yaml:59-60)
        double _max_alignment_motion = 0.2;
        int th_low = 65;                      // matcher.th_low (config/default.yaml:54)
        double _epipolar_dsqr = 1e-4;         // Matcher.h:31
        float knnRatio = 0.9f;                // Matcher.h:22
        bool checkOrientation = false;        // Matcher.h:24
    } _options;
    Matcher() : _align(new SparseImgAlign(2, 0, 30, SparseImgAlign::GaussNewton, false, false)) {}
    // Matcher.cpp:30-43
    static int DescriptorDistance(const uint8_t* a, const uint8_t* b) {
        auto& rt = b200::Runtime::Get();
        const int32_t z = 0;
        int32_t d = 0;
        rt.Check(ygzb_hamming_pairs(rt.ctx(), a, 1, b, 1, &z, &z, 1, &d), "ygzb_hamming_pairs");
        return d;
    }
    // Matcher.cpp:45-84
    int CheckFrameDescriptors(Frame* frame1, Frame* frame2, std::list<std::pair<int, int>>& matches) {
        auto& rt = b200::Runtime::Get();
        const int n = (int)matches.size(), n1 = (int)frame1->_features.size(), n2 = (int)frame2->_features.size();
        if (!n) return 0;
        std::vector<uint8_t> A((size_t)n1 * 32), B((size_t)n2 * 32);
        for (int i = 0; i < n1; ++i) std::memcpy(&A[(size_t)i * 32], frame1->_features[i]->_desc, 32);
        for (int i = 0; i < n2; ++i) std::memcpy(&B[(size_t)i * 32], frame2->_features[i]->_desc, 32);
        std::vector<int32_t> ia, ib, dist(n);
        for (auto& m : matches) { ia.push_back(m.first); ib.push_back(m.second); }
        rt.Check(ygzb_hamming_pairs(rt.ctx(), A.data(), n1, B.data(), n2, ia.data(), ib.data(), n, dist.data()), "ygzb_hamming_pairs");
        int best = dist[0];
        for (int d : dist) best = d < best ? d : best;
        best = best > _options.init_low ? best : _options.init_low;
        best = best < _options.init_high ? best : _options.init_high;
        int cnt_good = 0, i = 0;
        for (auto it = matches.begin(); it != matches.end(); ++i) {
            if (dist[i] < _options.initMatchRatio * best) { ++cnt_good; ++it; }
            else it = matches.erase(it);
        }
        return cnt_good;
    }
    // brute-force cross-checked matching of two frames (cv::BFMatcher in test/test_orb_match.cpp:87-92)
    // Matcher.cpp:86-193 (+ CheckDistEpipolarLine :338-354): matches inside the common nodes of the two feature vectors
    int SearchForTriangulation(Frame* kf1, Frame* kf2, const double E12[9] /* row major */, std::vector<std::pair<int, int>>& matched_points,
                               const bool& onlyStereo = false) {
        (void)onlyStereo;
        auto& rt = b200::Runtime::Get();
        auto flatten = [](Frame* f, std::vector<uint8_t>& desc, std::vector<double>& px, std::vector<int32_t>& node) {
            const size_t n = f->_features.size();
            desc.resize(32 * n); px.resize(2 * n); node.assign(n, -1);
            for (size_t i = 0; i < n; ++i) {
                std::memcpy(&desc[32 * i], f->_features[i]->_desc, 32);
                px[2 * i] = f->_features[i]->_pixel[0];
                px[2 * i + 1] = f->_features[i]->_pixel[1];
            }
            for (const auto& kv : f->_feature_vec)
                for (unsigned idx : kv.second)
                    if (idx < n) node[idx] = (int32_t)kv.first;
        };
        std::vector<uint8_t> d1, d2;
        std::vector<double> p1, p2;
        std::vector<int32_t> n1, n2;
        flatten(kf1, d1, p1, n1);
        flatten(kf2, d2, p2, n2);
        const int32_t off1[2] = {0, (int32_t)n1.size()}, off2[2] = {0, (int32_t)n2.size()};
        std::vector<int32_t> m12(n1.size(), -1);
        rt.Check(ygzb_search_for_triangulation(rt.ctx(), 1, off1, off2, d1.data(), p1.data(), n1.data(), d2.data(), p2.data(), n2.data(), E12,
                                               _options.th_low, _options._epipolar_dsqr, m12.data()), "ygzb_search_for_triangulation");
        matched_points.clear();
        for (size_t i = 0; i < m12.size(); ++i)
            if (m12[i] >= 0) matched_points.push_back(std::make_pair((int)i, (int)m12[i]));
        return (int)matched_points.size();
    }
    // Matcher.cpp:196-292: best / second-best Hamming match inside the common vocabulary nodes of the two feature vectors
    int SearchByBoW(Frame* kf1, Frame* kf2, std::map<int, int>& matches) {
        auto& rt = b200::Runtime::Get();
        auto flatten = [](Frame* f, std::vector<uint8_t>& desc, std::vector<float>& angle, std::vector<int32_t>& node) {
            const size_t n = f->_features.size();
            desc.resize(32 * n); angle.resize(n); node.assign(n, -1);
            for (size_t i = 0; i < n; ++i) {
                std::memcpy(&desc[32 * i], f->_features[i]->_desc, 32);
                angle[i] = (float)f->_features[i]->_angle;
            }
            for (const auto& kv : f->_feature_vec)
                for (unsigned idx : kv.second)
                    if (idx < n) node[idx] = (int32_t)kv.first;
        };
        std::vector<uint8_t> d1, d2;
        std::vector<float> a1, a2;
        std::vector<int32_t> n1, n2;
        flatten(kf1, d1, a1, n1);
        flatten(kf2, d2, a2, n2);
        const int32_t off1[2] = {0, (int32_t)n1.size()}, off2[2] = {0, (int32_t)n2.size()};
        std::vector<int32_t> m12(n1.size(), -1);
        int32_t cnt = 0;
        rt.Check(ygzb_search_by_bow(rt.ctx(), 1, off1, off2, d1.data(), n1.data(), a1.data(), d2.data(), n2.data(), a2.data(), _options.th_low,
                                    _options.knnRatio, _options.checkOrientation ? 1 : 0, m12.data(), &cnt), "ygzb_search_by_bow");
        for (size_t i = 0; i < m12.size(); ++i)
            if (m12[i] >= 0) matches[(int)i] = (int)m12[i];
        return cnt;
    }
    static void BruteForceMatch(Frame* f1, Frame* f2, std::vector<int>& train_idx, std::vector<int>& dist, bool cross_check = true) {
        auto& rt = b200::Runtime::Get();
        const int n1 = (int)f1->_features.size(), n2 = (int)f2->_features.size();
        std::vector<uint8_t> A((size_t)n1 * 32), B((size_t)n2 * 32);
        for (int i = 0; i < n1; ++i) std::memcpy(&A[(size_t)i * 32], f1->_features[i]->_desc, 32);
        for (int i = 0; i < n2; ++i) std::memcpy(&B[(size_t)i * 32], f2->_features[i]->_desc, 32);
        train_idx.assign(n1, -1);
        dist.assign(n1, -1);
        rt.Check(ygzb_match_bf(rt.ctx(), A.data(), n1, B.data(), n2, cross_check, train_idx.data(), dist.data()), "ygzb_match_bf");
    }
    // Matcher.cpp:385-417 (Feature* overload) and :356-383 (MapPoint* overload)
    bool FindDirectProjection(Frame* ref, Frame* curr, Feature* fea_ref, Vector2d& px_curr, int& search_level) {
        if (fea_ref->_depth < 0) return false;
        return Project(ref, curr, fea_ref->_pixel, fea_ref->_depth, fea_ref->_level, px_curr, search_level);
    }
    bool FindDirectProjection(Frame* ref, Frame* curr, MapPoint* mp, Vector2d& px_curr, int& search_level) {
        Feature* fea = mp->_obs[ref->_keyframe_id];
        const double depth = Frame::_camera->World2Camera(mp->_pos_world, ref->_TCW)[2];
        return Project(ref, curr, fea->_pixel, depth, fea->_level, px_curr, search_level);
    }
    // Matcher.cpp:468-492
    bool SparseImageAlignment(Frame* ref, Frame* current) {
        current->_TCW = ref->_TCW;
        _align->run(ref, current);
        _TCR_esti = current->_TCW * ref->_TCW.inverse();
        double lg[6], n2 = 0;
        _TCR_esti.log(lg);
        for (double v : lg) n2 += v * v;
        if (std::sqrt(n2) > _options._max_alignment_motion) {
            _TCR_esti = SE3();
            current->_TCW = ref->_TCW;
            return false;
        }
        return true;
    }
    void SetTCR(const SE3& TCR) { _TCR_esti = TCR; }
    SE3 GetTCR() const { return _TCR_esti; }
  private:
    bool Project(Frame* ref, Frame* curr, const Vector2d& px_ref, double depth, int level, Vector2d& px_curr, int& search_level) {
        auto& rt = b200::Runtime::Get();
        double poses[24];
        b200::PoseTo3x4(ref->_TCW, poses);
        b200::PoseTo3x4(curr->_TCW, poses + 12);
        const int32_t rs = b200::SlotOf(ref), cs = b200::SlotOf(curr), rp = 0, cp = 1;
        const double rpx[2] = {px_ref[0], px_ref[1]};
        double cpx[2] = {px_curr[0], px_curr[1]};
        const uint8_t lv = (uint8_t)level;
        uint8_t sl = 0, ok = 0;
        rt.Check(ygzb_project_align(rt.frames(), 1, &rs, &cs, 2, poses, &rp, &cp, rpx, &depth, &lv, cpx, &sl, &ok), "ygzb_project_align");
        px_curr = Vector2d(cpx[0], cpx[1]);
        search_level = sl;
        return ok != 0;
    }
    std::unique_ptr<SparseImgAlign> _align;
    SE3 _TCR_esti;
};

class Tracker {  // include/ygz/Algorithm/Tracker.h:11-76
  public:
    enum TrackerStatusType { TRACK_NOT_READY, TRACK_GOOD, TRACK_LOST };
    struct Option {
        int _min_feature_tracking = 50;  // tracker.min_features (config/default.yaml:42)
        double klt_win_size = 21.0;
        int klt_max_iter = 30;
        double klt_eps = 0.001;
    } _option;
    // Tracker.cpp:13-32
    void SetReference(Frame* ref) {
        if ((int)ref->_features.size() < _option._min_feature_tracking) {
            _status = TRACK_NOT_READY;
            return;
        }
        _ref = ref;
        _curr = ref;
        _status = TRACK_GOOD;
        for (Feature* fea : ref->_features) {
            _tracked_features.push_back(fea);
            _px_curr.push_back({(float)fea->_pixel[0], (float)fea->_pixel[1]});
        }
    }
    // Tracker.cpp:34-53
    void Track(Frame* curr) {
        if (_status != TRACK_GOOD) return;
        _curr = curr;
        TrackKLT();
        if ((int)_px_curr.size() < _option._min_feature_tracking) _status = TRACK_LOST;
    }
    // Tracker.cpp:115-127
    float MeanDisparity() const {
        float mean = 0;
        size_t i = 0;
        for (auto it = _tracked_features.begin(); it != _tracked_features.end(); ++it, ++i) {
            const double dx = (*it)->_pixel[0] - _px_curr[i].x, dy = (*it)->_pixel[1] - _px_curr[i].y;
            mean += (float)std::sqrt(dx * dx + dy * dy);
        }
        return mean / _tracked_features.size();
    }
    // Tracker.cpp:55-63
    void GetTrackedPixel(std::vector<Feature*>& feature1, std::vector<Vector2d>& pixels2) const {
        for (Feature* f : _tracked_features) feature1.push_back(f);
        for (auto& p : _px_curr) pixels2.push_back(Vector2d(p.x, p.y));
    }
    TrackerStatusType Status() const { return _status; }
  private:
    struct P2f { float x, y; };
    // Tracker.cpp:65-113: cv::calcOpticalFlowPyrLK(ref.pyr[0], cur.pyr[0], ..., 21x21, 4, (COUNT+EPS, 30, 0.001), USE_INITIAL_FLOW)
    void TrackKLT() {
        auto& rt = b200::Runtime::Get();
        const int n = (int)_tracked_features.size();
        if (!n) return;
        std::vector<float> ref(2 * (size_t)n), cur(2 * (size_t)n), err(n);
        std::vector<uint8_t> status(n);
        int i = 0;
        for (Feature* f : _tracked_features) {
            ref[2 * i] = (float)f->_pixel[0];
            ref[2 * i + 1] = (float)f->_pixel[1];
            cur[2 * i] = _px_curr[i].x;
            cur[2 * i + 1] = _px_curr[i].y;
            ++i;
        }
        ygzb_klt_params prm;
        ygzb_default_klt_params(&prm);
        prm.win = (int)_option.klt_win_size;
        prm.max_iter = _option.klt_max_iter;
        prm.eps = _option.klt_eps;
        const int32_t rs = b200::SlotOf(_ref), cs = b200::SlotOf(_curr), off[2] = {0, n};
        rt.Check(ygzb_klt(rt.frames(), 1, &rs, &cs, off, ref.data(), cur.data(), status.data(), err.data(), &prm), "ygzb_klt");
        _px_curr.clear();
        i = 0;
        for (auto it = _tracked_features.begin(); it != _tracked_features.end(); ++i) {
            const Vector2d p(cur[2 * i], cur[2 * i + 1]);
            if (!status[i] || !_curr->InFrame(p, 20)) {
                it = _tracked_features.erase(it);
            } else {
                ++it;
                _px_curr.push_back({cur[2 * i], cur[2 * i + 1]});
            }
        }
    }
    Frame* _ref = nullptr;
    Frame* _curr = nullptr;
    std::list<Feature*> _tracked_features;
    std::vector<P2f> _px_curr;
    TrackerStatusType _status = TRACK_NOT_READY;
};

// LocalMapping::CreateNewMapPoints (src/Module/LocalMapping.cpp:375-571) as a caller of the device entry points:
// SearchForTriangulation per neighbour key-frame, then per match DepthFromTriangulation -> FindDirectProjection ->
// DepthFromTriangulation -> reprojection test, or the association with an already triangulated point.  The neighbours
// (Frame::GetBestCovisibilityKeyframes in the reference) and the owner of new map points (Memory::CreateMapPoint) are the
// caller's; E12 = hat(t12) R12.
struct LocalMapping {
    std::vector<std::unique_ptr<MapPoint>> _new_points;   // the map points this call created (stand-in for Memory)
    int _cnt_new_mappoints = 0, _cnt_associate_mps = 0;
    void CreateNewMapPoints(Frame* current_kf, const std::vector<Frame*>& neighbour_kf) {
        PinholeCamera* cam = Frame::_camera;
        const Vector3d cam_current = current_kf->GetCamCenter();
        _cnt_new_mappoints = _cnt_associate_mps = 0;
        for (Frame* f2 : neighbour_kf) {
            const Vector3d c2 = f2->GetCamCenter();
            const double bl = std::sqrt((cam_current[0] - c2[0]) * (cam_current[0] - c2[0]) + (cam_current[1] - c2[1]) * (cam_current[1] - c2[1]) +
                                        (cam_current[2] - c2[2]) * (cam_current[2] - c2[2]));
            double mean_depth, min_depth;
            f2->GetMeanAndMinDepth(mean_depth, min_depth);
            if (bl / mean_depth < 0.01) continue;
            const SE3 T12 = current_kf->_TCW * f2->_TCW.inverse();
            double M[12];
            T12.matrix3x4(M);
            const double t[3] = {M[3], M[7], M[11]};
            const double hat[9] = {0, -t[2], t[1], t[2], 0, -t[0], -t[1], t[0], 0};
            double E12[9];
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) E12[3 * r + c] = hat[3 * r] * M[c] + hat[3 * r + 1] * M[4 + c] + hat[3 * r + 2] * M[8 + c];
            std::vector<std::pair<int, int>> matched_pairs;
            Matcher matcher;
            const int matches = matcher.SearchForTriangulation(current_kf, f2, E12, matched_pairs);
            const SE3 T21 = T12.inverse();
            for (int im = 0; im < matches; ++im) {
                Feature* fea1 = current_kf->_features[matched_pairs[im].first];
                Feature* fea2 = f2->_features[matched_pairs[im].second];
                if (fea2->_mappoint == nullptr && fea1->_mappoint == nullptr) {
                    const Vector3d pt1 = cam->Pixel2Camera(fea1->_pixel);
                    Vector3d pt2 = cam->Pixel2Camera(fea2->_pixel);
                    const double n1 = std::sqrt(pt1[0] * pt1[0] + pt1[1] * pt1[1] + pt1[2] * pt1[2]),
                                 n2 = std::sqrt(pt2[0] * pt2[0] + pt2[1] * pt2[1] + pt2[2] * pt2[2]);
                    const double cos_para_rays = (pt1[0] * pt2[0] + pt1[1] * pt2[1] + pt1[2] * pt2[2]) / (n1 * n2);
                    if (cos_para_rays >= 0.9998) continue;
                    double depth1 = 0, depth2 = 0;
                    bool ret = cvutils::DepthFromTriangulation(T21, pt1, pt2, depth1, depth2);
                    if (ret == false || depth1 < 0 || depth2 < 0) continue;
                    fea1->_depth = depth1;
                    Vector2d px_curr = fea2->_pixel;
                    int level = 0;
                    ret = matcher.FindDirectProjection(current_kf, f2, fea1, px_curr, level);
                    if (ret == false) continue;
                    fea2->_pixel = px_curr;
                    pt2 = cam->Pixel2Camera(fea2->_pixel);
                    ret = cvutils::DepthFromTriangulation(T21, pt1, pt2, depth1, depth2);
                    if (ret == false || depth1 < 0 || depth2 < 0) continue;
                    const Vector3d pt1_tri(pt1[0] * depth1, pt1[1] * depth1, pt1[2] * depth1);
                    const Vector2d px2_reproj = cam->Camera2Pixel(T21 * pt1_tri);
                    const double reproj_error = std::sqrt((px2_reproj[0] - fea2->_pixel[0]) * (px2_reproj[0] - fea2->_pixel[0]) +
                                                          (px2_reproj[1] - fea2->_pixel[1]) * (px2_reproj[1] - fea2->_pixel[1]));
                    if (reproj_error > 5.991) continue;
                    _new_points.emplace_back(new MapPoint());
                    MapPoint* mp = _new_points.back().get();
                    mp->_id = _next_id++;
                    mp->_first_seen = mp->_last_seen = current_kf->_keyframe_id;
                    mp->_obs[current_kf->_keyframe_id] = fea1;
                    mp->_obs[f2->_keyframe_id] = fea2;
                    mp->_cnt_visible = 2;
                    mp->_cnt_found = 2;
                    mp->_pos_world = cam->Camera2World(pt1_tri, current_kf->_TCW);
                    fea1->_mappoint = mp;
                    fea2->_mappoint = mp;
                    fea1->_depth = depth1;
                    fea2->_depth = depth2;
                    fea1->_bad = fea2->_bad = false;
                    ++_cnt_new_mappoints;
                } else if (fea2->_mappoint && fea1->_mappoint == nullptr) {
                    const Vector2d px_reproj = cam->World2Pixel(fea2->_mappoint->_pos_world, current_kf->_TCW);
                    const double e = std::sqrt((px_reproj[0] - fea1->_pixel[0]) * (px_reproj[0] - fea1->_pixel[0]) +
                                               (px_reproj[1] - fea1->_pixel[1]) * (px_reproj[1] - fea1->_pixel[1]));
                    if (e > 5.991) continue;
                    fea1->_mappoint = fea2->_mappoint;
                    fea1->_depth = cam->World2Camera(fea2->_mappoint->_pos_world, current_kf->_TCW)[2];
                    fea1->_mappoint->_obs[current_kf->_keyframe_id] = fea1;
                    ++_cnt_associate_mps;
                } else if (fea1->_mappoint && fea2->_mappoint == nullptr) {
                    const Vector2d px_reproj = cam->World2Pixel(fea1->_mappoint->_pos_world, f2->_TCW);
                    const double e = std::sqrt((px_reproj[0] - fea2->_pixel[0]) * (px_reproj[0] - fea2->_pixel[0]) +
                                               (px_reproj[1] - fea2->_pixel[1]) * (px_reproj[1] - fea2->_pixel[1]));
                    if (e > 5.991) continue;
                    fea2->_mappoint = fea1->_mappoint;
                    fea2->_depth = cam->World2Camera(fea2->_mappoint->_pos_world, f2->_TCW)[2];
                    fea2->_mappoint->_obs[f2->_keyframe_id] = fea2;
                    ++_cnt_associate_mps;
                }
            }
        }
    }
    unsigned long _next_id = 0;
};

// include/ygz/Algorithm/Initializer.h:27-145: TryInitialize (src/Algorithm/Initializer.cpp:9-87) = the RANSAC over 200 minimal
// sets for H and F, the model choice, and ReconstructH / ReconstructF (pose + structure), all on the device
class Initializer {
  public:
    struct Option {
        float _sigma = 2.0f;    // Initializer.h:45
        float _sigma2 = 4.0f;
        int _max_iter = 200;    // Initializer.h:47
        double _min_parallex = 1.0;
        int _min_triangulated_pts = 8;
        double good_point_ratio_H = 0.9;
    } _options;
    struct Matrix3 { double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}; double operator()(int r, int c) const { return m[3 * r + c]; } };
    // the minimal sets of TryInitialize (:25-49): a default-constructed cv::RNG (multiply-with-carry, state 0xffffffff,
    // uniform(0, b) = next() % b), 8 draws without replacement per iteration by swap-with-last
    static std::vector<int32_t> DrawSets(int num_points, int max_iter) {
        std::vector<int32_t> sets((size_t)max_iter * 8), avail;
        uint64_t state = 0xffffffffULL;
        for (int it = 0; it < max_iter; ++it) {
            avail.resize(num_points);
            for (int i = 0; i < num_points; ++i) avail[i] = i;
            for (int j = 0; j < 8; ++j) {
                state = (uint64_t)(uint32_t)state * 4164903690ULL + (uint32_t)(state >> 32);
                const int r = avail.empty() ? 0 : (int)((uint32_t)state % (uint32_t)avail.size());
                sets[(size_t)it * 8 + j] = avail[r];
                avail[r] = avail.back();
                avail.pop_back();
            }
        }
        return sets;
    }
    // TryInitialize up to the choice of the model (:9-78): returns true if the homography is preferred (rh > 0.4)
    bool FindModels(const std::vector<Vector2d>& px1, const std::vector<Vector2d>& px2) {
        if (px1.size() != px2.size() || px1.size() < 8) throw b200::Error("Initializer: at least 8 matched pixels are needed");
        auto& rt = b200::Runtime::Get();
        const int n = (int)px1.size();
        std::vector<double> a(2 * (size_t)n), b(2 * (size_t)n);
        for (int i = 0; i < n; ++i) {
            a[2 * i] = px1[i][0]; a[2 * i + 1] = px1[i][1];
            b[2 * i] = px2[i][0]; b[2 * i + 1] = px2[i][1];
        }
        const std::vector<int32_t> sets = DrawSets(n, _options._max_iter);
        const int32_t off[2] = {0, n};
        std::vector<uint8_t> ih(n), jf(n);
        int32_t bh = -1, bf = -1;
        rt.Check(ygzb_initializer_ransac(rt.ctx(), 1, off, a.data(), b.data(), _options._max_iter, sets.data(), _options._sigma, _H21.m, &_score_H,
                                         &bh, ih.data(), _F21.m, &_score_F, &bf, jf.data(), nullptr), "ygzb_initializer_ransac");
        _inliers_H.assign(ih.begin(), ih.end());
        _inliers_F.assign(jf.begin(), jf.end());
        const float rh = _score_H / (_score_H + _score_F);   // :66
        return rh > 0.4f;
    }
    // Initializer.cpp:9-87.  The camera is the runtime's (ygzb_params); `ref` / `curr` are kept like the reference does.
    bool TryInitialize(std::vector<Vector2d>& px1, std::vector<Vector2d>& px2, Frame* ref, Frame* curr) {
        _ref = ref;
        _curr = curr;
        const bool use_h = FindModels(px1, px2);
        auto& rt = b200::Runtime::Get();
        const int n = (int)px1.size();
        std::vector<double> a(2 * (size_t)n), b(2 * (size_t)n), p3d(3 * (size_t)n);
        std::vector<uint8_t> inl(n), tri(n);
        for (int i = 0; i < n; ++i) {
            a[2 * i] = px1[i][0]; a[2 * i + 1] = px1[i][1];
            b[2 * i] = px2[i][0]; b[2 * i + 1] = px2[i][1];
            inl[i] = (use_h ? _inliers_H[i] : _inliers_F[i]) ? 1 : 0;
        }
        const int32_t off[2] = {0, n}, uh = use_h ? 1 : 0;
        int32_t ok = 0, n_good[8];
        double R[9], t[3], parallax = 0;
        rt.Check(ygzb_initializer_reconstruct(rt.ctx(), 1, off, a.data(), b.data(), &uh, use_h ? _H21.m : _F21.m, inl.data(), _options._sigma2,
                                              (float)_options._min_parallex, _options._min_triangulated_pts, _options.good_point_ratio_H, &ok, R, t,
                                              p3d.data(), tri.data(), n_good, &parallax, nullptr), "ygzb_initializer_reconstruct");
        const double Rt[12] = {R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2]};
        _T21 = ok ? SE3::from3x4(Rt) : SE3();
        _inliers.assign(n, true);
        if (!ok) return false;
        _pts_triangulated.resize(n);
        for (int i = 0; i < n; ++i) {
            _inliers[i] = tri[i] != 0;
            _pts_triangulated[i] = Vector3d(p3d[3 * i], p3d[3 * i + 1], p3d[3 * i + 2]);
        }
        return true;
    }
    Matrix3 _H21, _F21;
    float _score_H = 0, _score_F = 0;
    std::vector<bool> _inliers_H, _inliers_F;
    std::vector<bool> _inliers;                  // Initializer.h:118
    std::vector<Vector3d> _pts_triangulated;     // Initializer.h:119
    SE3 _T21;                                    // Initializer.h:120
    Frame* _ref = nullptr;
    Frame* _curr = nullptr;
};

namespace ba {  // include/ygz/Algorithm/BA.h:23-66

// BA.h:23-30 / BA.cpp:11-89: two-view bundle adjustment after the monocular initialisation (VisualOdometry.cpp:148)
inline void TwoViewBACeres(const SE3& ref, SE3& curr, const std::vector<Vector2d> px_ref, const std::vector<Vector2d> px_curr,
                           std::vector<bool>& inlier, std::vector<Vector3d>& pts_ref) {
    auto& rt = b200::Runtime::Get();
    const int n = (int)px_ref.size();
    const int32_t off[2] = {0, n};
    double Tr[12], Tc[12];
    ref.matrix3x4(Tr);
    curr.matrix3x4(Tc);
    std::vector<double> pr(2 * (size_t)n), pc(2 * (size_t)n), X(3 * (size_t)n);
    std::vector<uint8_t> in(n);
    for (int i = 0; i < n; ++i) {
        pr[2 * i] = px_ref[i][0]; pr[2 * i + 1] = px_ref[i][1];
        pc[2 * i] = px_curr[i][0]; pc[2 * i + 1] = px_curr[i][1];
        X[3 * i] = pts_ref[i][0]; X[3 * i + 1] = pts_ref[i][1]; X[3 * i + 2] = pts_ref[i][2];
        in[i] = inlier[i] ? 1 : 0;
    }
    rt.Check(ygzb_two_view_ba(rt.ctx(), 1, off, Tr, Tc, pr.data(), pc.data(), in.data(), X.data(), nullptr), "ygzb_two_view_ba");
    curr = SE3::from3x4(Tc);
    for (int i = 0; i < n; ++i) {
        pts_ref[i] = Vector3d(X[3 * i], X[3 * i + 1], X[3 * i + 2]);
        inlier[i] = in[i] != 0;
    }
}
// BA.cpp:188-264
inline void OptimizeCurrentPoseOnly(Frame* current) {
    auto& rt = b200::Runtime::Get();
    const int n = (int)current->_features.size();
    if (!n) return;
    std::vector<double> pw(3 * (size_t)n), px(2 * (size_t)n), depth(n);
    std::vector<uint8_t> inl(n);
    for (int i = 0; i < n; ++i) {
        const Feature* f = current->_features[i];
        for (int k = 0; k < 3; ++k) pw[3 * i + k] = f->_mappoint->_pos_world[k];
        px[2 * i] = f->_pixel[0];
        px[2 * i + 1] = f->_pixel[1];
    }
    double T[12];
    b200::PoseTo3x4(current->_TCW, T);
    const int32_t off[2] = {0, n};
    int32_t cnt = 0;
    rt.Check(ygzb_pose_only(rt.ctx(), 1, off, pw.data(), px.data(), T, inl.data(), depth.data(), &cnt), "ygzb_pose_only");
    current->_TCW = SE3::from3x4(T);
    for (int i = 0; i < n; ++i) {
        Feature* f = current->_features[i];
        f->_bad = !inl[i];
        if (inl[i]) f->_depth = depth[i];
        if (!f->_bad && f->_mappoint && !f->_mappoint->_bad) f->_mappoint->_cnt_found++;  // BA.cpp:255-261
    }
}

// BA.cpp:386-543.  `keyframe_of` resolves keyframe ids (Memory::GetKeyFrame in the reference).
inline void LocalBAG2O(std::set<Frame*>& local_keyframes, std::set<MapPoint*>& local_map_points,
                       const std::map<unsigned long, Frame*>& keyframe_of) {
    auto& rt = b200::Runtime::Get();
    std::vector<Frame*> kfs;
    std::map<Frame*, int> index;
    std::vector<uint8_t> fixed;
    auto add_kf = [&](Frame* f, bool fix) {
        auto it = index.find(f);
        if (it == index.end()) {
            index[f] = (int)kfs.size();
            kfs.push_back(f);
            fixed.push_back(fix || f->_keyframe_id == 0);
        } else if (fix) {
            fixed[it->second] = 1;
        }
        return index[f];
    };
    for (Frame* f : local_keyframes) add_kf(f, false);
    std::vector<MapPoint*> pts;
    std::vector<int32_t> kf_idx, pt_idx;
    std::vector<double> obs;
    std::vector<Feature*> feats;
    for (MapPoint* mp : local_map_points) {
        if (mp->_bad) continue;
        const int j = (int)pts.size();
        pts.push_back(mp);
        for (auto& o : mp->_obs) {
            if (o.second->_bad) continue;
            Frame* f = keyframe_of.at(o.first);
            const bool local = local_keyframes.count(f) != 0;
            kf_idx.push_back(add_kf(f, !local));  // observers outside the local set are added / set fixed (:458-492)
            pt_idx.push_back(j);
            obs.push_back(o.second->_pixel[0]);
            obs.push_back(o.second->_pixel[1]);
            feats.push_back(o.second);
        }
    }
    const int nk = (int)kfs.size(), np = (int)pts.size(), no = (int)kf_idx.size();
    std::vector<double> poses(6 * (size_t)nk), X(3 * (size_t)np);
    for (int k = 0; k < nk; ++k) {  // esti = [log.tail<3>; log.head<3>]
        double lg[6];
        kfs[k]->_TCW.log(lg);
        for (int c = 0; c < 3; ++c) { poses[6 * k + c] = lg[3 + c]; poses[6 * k + 3 + c] = lg[c]; }
    }
    for (int j = 0; j < np; ++j)
        for (int c = 0; c < 3; ++c) X[3 * j + c] = pts[j]->_pos_world[c];
    ygzb_ba_params prm;
    ygzb_default_ba_params(&prm);
    std::vector<uint8_t> outl(no ? no : 1);
    const int32_t ko[2] = {0, nk}, po[2] = {0, np}, oo[2] = {0, no};
    rt.Check(ygzb_local_ba(rt.ctx(), 1, ko, po, oo, poses.data(), fixed.data(), X.data(), kf_idx.data(), pt_idx.data(), obs.data(), &prm,
                           outl.data(), nullptr), "ygzb_local_ba");
    for (int o = 0; o < no; ++o)
        if (outl[o]) feats[o]->_bad = true;
    for (Frame* f : local_keyframes) {
        const int k = index[f];
        const double v[6] = {poses[6 * k + 3], poses[6 * k + 4], poses[6 * k + 5], poses[6 * k], poses[6 * k + 1], poses[6 * k + 2]};
        f->_TCW = SE3::exp(v);
    }
    for (int j = 0; j < np; ++j) pts[j]->_pos_world = Vector3d(X[3 * j], X[3 * j + 1], X[3 * j + 2]);
}

// BA.cpp:324-384: the Ceres flavour.  Only observations in local key-frames enter (:338); the key-frame with
// _keyframe_id == 0 keeps its pose (point-only residual blocks, :340-349); poses travel as [t; so3.log()] (:353-357)
// and come back through SE3(SO3::exp(r), t) (:378-382).
inline void LocalBA(std::set<Frame*>& local_keyframes, std::set<MapPoint*>& local_map_points,
                    const std::map<unsigned long, Frame*>& keyframe_of) {
    auto& rt = b200::Runtime::Get();
    std::vector<Frame*> kfs(local_keyframes.begin(), local_keyframes.end());
    std::map<Frame*, int> index;
    std::vector<uint8_t> fixed;
    for (size_t k = 0; k < kfs.size(); ++k) {
        index[kfs[k]] = (int)k;
        fixed.push_back(kfs[k]->_keyframe_id == 0);
    }
    std::vector<MapPoint*> pts;
    std::vector<int32_t> kf_idx, pt_idx;
    std::vector<double> obs;
    for (MapPoint* mp : local_map_points) {
        const int j = (int)pts.size();
        pts.push_back(mp);
        for (auto& o : mp->_obs) {
            auto it = index.find(keyframe_of.at(o.first));
            if (it == index.end()) continue;
            kf_idx.push_back(it->second);
            pt_idx.push_back(j);
            obs.push_back(o.second->_pixel[0]);
            obs.push_back(o.second->_pixel[1]);
        }
    }
    const int nk = (int)kfs.size(), np = (int)pts.size(), no = (int)kf_idx.size();
    if (!nk || !np || !no) return;
    std::vector<double> poses(6 * (size_t)nk), X(3 * (size_t)np);
    for (int k = 0; k < nk; ++k) {
        double th;
        const ygzb::V3d r = ygzb::so3_log(kfs[k]->_TCW.T.q, &th);
        const ygzb::V3d t = kfs[k]->_TCW.T.t;
        poses[6 * k] = t.x; poses[6 * k + 1] = t.y; poses[6 * k + 2] = t.z;
        poses[6 * k + 3] = r.x; poses[6 * k + 4] = r.y; poses[6 * k + 5] = r.z;
    }
    for (int j = 0; j < np; ++j)
        for (int c = 0; c < 3; ++c) X[3 * j + c] = pts[j]->_pos_world[c];
    const int32_t ko[2] = {0, nk}, po[2] = {0, np}, oo[2] = {0, no};
    rt.Check(ygzb_local_ba_ceres(rt.ctx(), 1, ko, po, oo, poses.data(), fixed.data(), X.data(), kf_idx.data(), pt_idx.data(), obs.data(),
                                 50, 0.0, nullptr), "ygzb_local_ba_ceres");
    for (int k = 0; k < nk; ++k) {
        if (fixed[k]) continue;   // the map `poses` of the reference only holds the key-frames with pose blocks
        ygzb::SE3d T;
        double th;
        T.q = ygzb::so3_exp(ygzb::V3d{poses[6 * k + 3], poses[6 * k + 4], poses[6 * k + 5]}, &th);
        T.t = ygzb::V3d{poses[6 * k], poses[6 * k + 1], poses[6 * k + 2]};
        kfs[k]->_TCW = SE3(T);
    }
    for (int j = 0; j < np; ++j) pts[j]->_pos_world = Vector3d(X[3 * j], X[3 * j + 1], X[3 * j + 2]);
}

namespace detail {
// shared body of OptimizeCurrent / OptimizeCurrentPointOnly: the current frame (free or fixed) observes the map points of
// its usable features; every other observer of those points enters as a constant pose (CeresReprojectionErrorPointOnly)
inline void OptimizeCurrentImpl(Frame* current, const std::map<unsigned long, Frame*>& keyframe_of, bool pose_free, double huber_a,
                                bool skip_bad) {
    auto& rt = b200::Runtime::Get();
    std::vector<const Frame*> frames{current};
    std::vector<uint8_t> fixed{(uint8_t)!pose_free};
    std::map<const Frame*, int> fixed_index;
    std::vector<MapPoint*> pts;
    std::map<MapPoint*, int> pt_index;
    std::vector<int32_t> kf_idx, pt_idx;
    std::vector<double> obs;
    for (Feature* fea : current->_features) {
        if (!fea->_mappoint || (skip_bad && fea->_bad)) continue;
        auto it = pt_index.find(fea->_mappoint);
        if (it == pt_index.end()) {
            it = pt_index.emplace(fea->_mappoint, (int)pts.size()).first;
            pts.push_back(fea->_mappoint);
        }
        const int j = it->second;
        kf_idx.push_back(0); pt_idx.push_back(j);
        obs.push_back(fea->_pixel[0]); obs.push_back(fea->_pixel[1]);
        for (auto& o : fea->_mappoint->_obs) {   // the covisible key-frames, poses held constant
            const Frame* f = keyframe_of.at(o.first);
            auto fi = fixed_index.find(f);
            if (fi == fixed_index.end()) {
                fi = fixed_index.emplace(f, (int)frames.size()).first;
                frames.push_back(f);
                fixed.push_back(1);
            }
            kf_idx.push_back(fi->second); pt_idx.push_back(j);
            obs.push_back(o.second->_pixel[0]); obs.push_back(o.second->_pixel[1]);
        }
    }
    const int nk = (int)frames.size(), np = (int)pts.size(), no = (int)kf_idx.size();
    if (!np || !no) return;
    std::vector<double> poses(6 * (size_t)nk), X(3 * (size_t)np);
    for (int k = 0; k < nk; ++k) {
        double th;
        const ygzb::V3d r = ygzb::so3_log(frames[k]->_TCW.T.q, &th);
        const ygzb::V3d t = frames[k]->_TCW.T.t;
        poses[6 * k] = t.x; poses[6 * k + 1] = t.y; poses[6 * k + 2] = t.z;
        poses[6 * k + 3] = r.x; poses[6 * k + 4] = r.y; poses[6 * k + 5] = r.z;
    }
    for (int j = 0; j < np; ++j)
        for (int c = 0; c < 3; ++c) X[3 * j + c] = pts[j]->_pos_world[c];
    const int32_t ko[2] = {0, nk}, po[2] = {0, np}, oo[2] = {0, no};
    rt.Check(ygzb_local_ba_ceres(rt.ctx(), 1, ko, po, oo, poses.data(), fixed.data(), X.data(), kf_idx.data(), pt_idx.data(), obs.data(),
                                 50, huber_a, nullptr), "ygzb_local_ba_ceres");
    if (pose_free) {
        ygzb::SE3d T;
        double th;
        T.q = ygzb::so3_exp(ygzb::V3d{poses[3], poses[4], poses[5]}, &th);
        T.t = ygzb::V3d{poses[0], poses[1], poses[2]};
        current->_TCW = SE3(T);
    }
    for (int j = 0; j < np; ++j) pts[j]->_pos_world = Vector3d(X[3 * j], X[3 * j + 1], X[3 * j + 2]);
}
}  // namespace detail

// BA.cpp:91-186: pose of the current frame + its map points, HuberLoss(0.1) on every block, then the 4 * 5.991 px^2 test
inline void OptimizeCurrent(Frame* current, const std::map<unsigned long, Frame*>& keyframe_of) {
    detail::OptimizeCurrentImpl(current, keyframe_of, true, 0.1, false);
    const float chi2Mono = 5.991 * 4;
    for (Feature* fea : current->_features) {
        if (!fea->_mappoint) continue;
        const Vector2d px = current->_camera->World2Pixel(fea->_mappoint->_pos_world, current->_TCW);
        const double dx = px[0] - fea->_pixel[0], dy = px[1] - fea->_pixel[1];
        if (dx * dx + dy * dy > chi2Mono) fea->_bad = true;
        else fea->_depth = current->_camera->World2Camera(fea->_mappoint->_pos_world, current->_TCW)[2];
    }
}

// BA.cpp:266-322: only the map points move; every pose (the current frame's too) is a constant of its residual block
inline void OptimizeCurrentPointOnly(Frame* current, const std::map<unsigned long, Frame*>& keyframe_of) {
    detail::OptimizeCurrentImpl(current, keyframe_of, false, 0.0, true);
}
}  // namespace ba

// facade for the vocabulary of the north star ("ygz::Optimizer"); the reference's live API is namespace ygz::ba
class Optimizer {
  public:
    static void PoseOnly(Frame* current) { ba::OptimizeCurrentPoseOnly(current); }
    static void LocalBA(std::set<Frame*>& kfs, std::set<MapPoint*>& mps, const std::map<unsigned long, Frame*>& keyframe_of) {
        ba::LocalBAG2O(kfs, mps, keyframe_of);
    }
};

}  // namespace ygz
