// pslam_adapter.hpp — header-only C++ adapter that re-creates the reference's class interfaces on top of the C ABI
// (include/pslam_abi.h), so Frame / Tracking can switch to the GPU path without changing their call sites.
//
// This header carries the reference's method names and argument order over plain pointers / std::vector (no OpenCV, Eigen or PCL needed;
// tests/test_adapter_compiles.py builds it).  The calls WITH the reference's own argument types (Frame*, KeyFrame*, cv::InputArray,
// std::vector<MapPoint*> ...) are in include/pslam_reference_adapter.hpp, which is compiled inside the PlanarSLAM tree.
//
//   Planar_SLAM::ORBextractor::operator()      include/ORBextractor.h:59-61   -> pslam_orb_extract
//   ORBextractor getters                       include/ORBextractor.h:63-83   -> pslam_orb_get_scale_tables
//   PlaneDetection::readDepthImage / run...    include/PlaneExtractor.h:36-56 -> pslam_peac_run_batch
//   Optimizer::PoseOptimization                include/Optimizer.h:38         -> pslam_pose_optimization
//   Optimizer::LocalBundleAdjustment           include/Optimizer.h:34         -> pslam_local_bundle_adjustment
//   LineSegment::ExtractLineSegment            include/LSDextractor.h:349     -> pslam_lines_extract_batch
//   Frame::isLineGood                          include/Frame.h (src/Frame.cc:189)  -> pslam_lines3d_batch
//   Frame::ComputeStereoFromRGBD               src/Frame.cc:603               -> pslam_compute_stereo_from_rgbd_batch
//   Frame::isInFrustum(MapLine*, float)        src/Frame.cc:369               -> pslam_lines_in_frustum
//   Tracking::TrackManhattanFrame              src/Tracking.cc:963            -> pslam_track_manhattan_batch
#pragma once
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "pslam_abi.h"

namespace pslam_adapter {

struct Image8 { const uint8_t* data; int width, height, stride; };       // CV_8UC1 view
struct Image16 { const uint16_t* data; int width, height; };             // CV_16UC1 view, dense

class Context {
public:
    Context(int width, int height, const pslam_config* overrides = nullptr) {
        pslam_config cfg;
        if (overrides) cfg = *overrides; else pslam_default_config(&cfg, width, height, 1);
        cfg.width = width; cfg.height = height;
        if (pslam_create(&cfg, &ctx_) != PSLAM_OK) throw std::runtime_error("pslam_create failed: no sm_90 GPU or bad configuration");
        cfg_ = cfg;
    }
    ~Context() { pslam_destroy(ctx_); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    pslam_ctx* get() const { return ctx_; }
    const pslam_config& config() const { return cfg_; }
private:
    pslam_ctx* ctx_ = nullptr;
    pslam_config cfg_;
};

// Same constructor arguments, getters and call operator as Planar_SLAM::ORBextractor.
class ORBextractor {
public:
    ORBextractor(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST)
        : nfeatures_(nfeatures), scaleFactor_(scaleFactor), nlevels_(nlevels), iniThFAST_(iniThFAST), minThFAST_(minThFAST) {}
    ~ORBextractor() { delete ctx_; }

    // void operator()(InputArray image, InputArray mask, vector<KeyPoint>& keypoints, OutputArray descriptors)
    void operator()(const Image8& image, const void* /*mask, ignored like the reference*/, std::vector<pslam_keypoint>& keypoints,
                    std::vector<uint8_t>& descriptors) {
        keypoints.clear(); descriptors.clear();
        if (!image.data || image.width <= 0 || image.height <= 0) return;           // reference: silent return on empty input
        ensure(image.width, image.height);
        const int cap = pslam_orb_max_keypoints(ctx_->get());
        keypoints.resize(cap); descriptors.resize((size_t)cap * 32);
        int32_t n = 0;
        const int rc = pslam_orb_extract(ctx_->get(), image.data, image.stride, keypoints.data(), descriptors.data(), cap, &n);
        if (rc != PSLAM_OK) throw std::runtime_error(pslam_last_error(ctx_->get()));
        keypoints.resize(n); descriptors.resize((size_t)n * 32);
    }
    int GetLevels() const { return nlevels_; }
    float GetScaleFactor() const { return scaleFactor_; }
    std::vector<float> GetScaleFactors() { return table(0); }
    std::vector<float> GetInverseScaleFactors() { return table(1); }
    std::vector<float> GetScaleSigmaSquares() { return table(2); }
    std::vector<float> GetInverseScaleSigmaSquares() { return table(3); }

private:
    void ensure(int w, int h) {
        if (ctx_ && ctx_->config().width == w && ctx_->config().height == h) return;
        delete ctx_; ctx_ = nullptr;
        pslam_config cfg;
        pslam_default_config(&cfg, w, h, 1);
        cfg.nfeatures = nfeatures_; cfg.scale_factor = scaleFactor_; cfg.nlevels = nlevels_; cfg.ini_th_fast = iniThFAST_; cfg.min_th_fast = minThFAST_;
        ctx_ = new Context(w, h, &cfg);
    }
    std::vector<float> table(int which) {
        if (!ctx_) ensure(640, 480);
        std::vector<float> t[4];
        for (auto& v : t) v.resize(nlevels_);
        pslam_orb_get_scale_tables(ctx_->get(), t[0].data(), t[1].data(), t[2].data(), t[3].data(), nullptr);
        return t[which];
    }
    int nfeatures_; float scaleFactor_; int nlevels_, iniThFAST_, minThFAST_;
    Context* ctx_ = nullptr;
};

// Same public surface as the reference's PlaneDetection (global namespace there).
class PlaneDetection {
public:
    std::vector<std::vector<int>> plane_vertices_;     // vertex (pixel) indices each plane contains
    std::vector<pslam_plane> extractedPlanes;          // plane_filter.extractedPlanes[i]->{normal, center, N, mse}
    std::vector<int32_t> membershipImg;                // plane_filter.membershipImg (int32 per pixel)
    int plane_num_ = 0;
    ~PlaneDetection() { delete ctx_; }

    // bool readDepthImage(cv::Mat depthImg, cv::Mat& K, float kScaleFactor); K = {fx, fy, cx, cy} of the float 3x3
    bool readDepthImage(const Image16& depthImg, const float K[4], float kScaleFactor) {
        if (!depthImg.data || depthImg.width <= 0) return false;
        if (!ctx_ || ctx_->config().width != depthImg.width || ctx_->config().height != depthImg.height || std::memcmp(K, K_, sizeof K_) || kScaleFactor != scale_) {
            delete ctx_; ctx_ = nullptr;
            pslam_config cfg;
            pslam_default_config(&cfg, depthImg.width, depthImg.height, 1);
            cfg.fx = K[0]; cfg.fy = K[1]; cfg.cx = K[2]; cfg.cy = K[3]; cfg.depth_scale = kScaleFactor;
            ctx_ = new Context(depthImg.width, depthImg.height, &cfg);
            std::memcpy(K_, K, sizeof K_); scale_ = kScaleFactor;
        }
        depth_ = depthImg;
        return true;
    }
    // void runPlaneDetection(int kDepthHeight, int kDepthWidth)
    void runPlaneDetection(int /*kDepthHeight*/, int /*kDepthWidth*/) {
        const size_t px = (size_t)depth_.width * depth_.height;
        const int maxp = pslam_peac_max_planes(ctx_->get());
        membershipImg.assign(px, -1);
        std::vector<pslam_plane> planes(maxp);
        std::vector<int32_t> midx(px), moff(maxp + 1);
        int32_t n = 0;
        const int rc = pslam_peac_run_batch(ctx_->get(), depth_.data, 1, membershipImg.data(), planes.data(), &n, midx.data(), moff.data());
        if (rc != PSLAM_OK) throw std::runtime_error(pslam_last_error(ctx_->get()));
        plane_num_ = n;
        extractedPlanes.assign(planes.begin(), planes.begin() + n);
        plane_vertices_.assign(n, {});
        for (int k = 0; k < n; ++k) plane_vertices_[k].assign(midx.begin() + moff[k], midx.begin() + moff[k + 1]);
    }
private:
    Context* ctx_ = nullptr;
    Image16 depth_{nullptr, 0, 0};
    float K_[4] = {0, 0, 0, 0}, scale_ = 0;
};

// Same method name and argument order as Planar_SLAM::LineSegment (include/LSDextractor.h:349); the descriptor matrix is not
// produced (LBD stays with OpenCV's BinaryDescriptor on the returned key lines).
class LineSegment {
public:
    ~LineSegment() { delete ctx_; }
    // void ExtractLineSegment(const Mat& img, vector<KeyLine>& keylines, Mat& ldesc, vector<Vector3d>& keylineFunctions, float scale, int numOctaves)
    void ExtractLineSegment(const Image8& img, std::vector<pslam_keyline>& keylines, std::vector<double>& keylineFunctions /* 3 per line, appended */,
                            float /*scale*/ = 1.2f, int /*numOctaves*/ = 1) {
        keylines.clear();
        if (!img.data || img.width <= 0 || img.height <= 0) return;
        if (!ctx_ || ctx_->config().width != img.width || ctx_->config().height != img.height) { delete ctx_; ctx_ = new Context(img.width, img.height); }
        std::vector<uint8_t> dense;
        const uint8_t* src = img.data;
        if (img.stride != img.width) {
            dense.resize((size_t)img.width * img.height);
            for (int y = 0; y < img.height; ++y) std::memcpy(&dense[(size_t)y * img.width], img.data + (size_t)y * img.stride, img.width);
            src = dense.data();
        }
        const int max_lines = 40;                                             // lsdNFeatures, src/LSDextractor.cpp:18
        keylines.resize(max_lines);
        std::vector<double> lf((size_t)max_lines * 3);
        int32_t n = 0;
        if (pslam_lines_extract_batch(ctx_->get(), src, 1, max_lines, keylines.data(), lf.data(), &n) != PSLAM_OK)
            throw std::runtime_error(pslam_last_error(ctx_->get()));
        keylines.resize(n);
        keylineFunctions.insert(keylineFunctions.end(), lf.begin(), lf.begin() + 3 * n);
    }
private:
    Context* ctx_ = nullptr;
};


// static int Optimizer::PoseOptimization(Frame* pFrame): the Frame fields it reads are gathered into a pslam_pose_problem
// by the caller under the same mutexes the reference takes (MapPoint/MapLine/MapPlane::mGlobalMutex, src/Optimizer.cc:590,691,786).
class Optimizer {
public:
    explicit Optimizer(Context& ctx) : ctx_(ctx) {}
    int PoseOptimization(const pslam_pose_problem& prob, float Tcw_io[16], std::vector<uint8_t>& mvbOutlier, std::vector<uint8_t>& mvbLineOutlier,
                         std::vector<uint8_t>& mvbPlaneOutlier, std::vector<uint8_t>& mvbParPlaneOutlier, std::vector<uint8_t>& mvbVerPlaneOutlier) {
        mvbOutlier.assign(prob.n_points > 0 ? prob.n_points : 1, 0); mvbLineOutlier.assign(prob.n_lines > 0 ? prob.n_lines : 1, 0);
        mvbPlaneOutlier.assign(prob.n_planes > 0 ? prob.n_planes : 1, 0); mvbParPlaneOutlier.assign(prob.n_par > 0 ? prob.n_par : 1, 0);
        mvbVerPlaneOutlier.assign(prob.n_ver > 0 ? prob.n_ver : 1, 0);
        const int rc = pslam_pose_optimization(ctx_.get(), &prob, Tcw_io, mvbOutlier.data(), mvbLineOutlier.data(), mvbPlaneOutlier.data(),
                                               mvbParPlaneOutlier.data(), mvbVerPlaneOutlier.data());
        if (rc < 0) throw std::runtime_error(pslam_last_error(ctx_.get()));
        mvbOutlier.resize(prob.n_points); mvbLineOutlier.resize(prob.n_lines); mvbPlaneOutlier.resize(prob.n_planes);
        mvbParPlaneOutlier.resize(prob.n_par); mvbVerPlaneOutlier.resize(prob.n_ver);
        return rc;      // nInitialCorrespondences - nBad
    }
private:
    Context& ctx_;
};


// static void Optimizer::LocalBundleAdjustment(KeyFrame*, bool*, Map*): the caller gathers the local map into a
// pslam_lba_problem (INTEGRATION.md section 3c) and owns the output arrays of pslam_lba_result.
inline void LocalBundleAdjustment(Context& ctx, const pslam_lba_problem& prob, pslam_lba_result& res) {
    if (pslam_local_bundle_adjustment(ctx.get(), &prob, &res) != PSLAM_OK) throw std::runtime_error(pslam_last_error(ctx.get()));
}

// void Frame::isLineGood(const cv::Mat& imGray, const cv::Mat& imDepth, cv::Mat K): fills what the reference stores per key line.
// rand_draws: the number of libc rand() calls the process has made so far (the reference never seeds: srand(1)); it is advanced by
// the draws this frame makes, so consecutive frames see the stream the reference's single libc stream would give them.
inline void isLineGood(Context& ctx, const std::vector<pslam_keyline>& mvKeylinesUn, const Image16& rawDepth, float depthMapFactor, const float K[4] /* fx fy cx cy */,
                       int32_t& rand_draws, std::vector<pslam_line3d>& lines3d) {
    const int32_t n = (int32_t)mvKeylinesUn.size();
    lines3d.assign(n > 0 ? n : 1, pslam_line3d());
    if (n == 0) { lines3d.clear(); return; }
    if (rawDepth.width != ctx.config().width || rawDepth.height != ctx.config().height) throw std::runtime_error("depth size differs from the context");
    const uint32_t seed = 1;
    int32_t drawn = 0;
    if (pslam_lines3d_batch(ctx.get(), mvKeylinesUn.data(), &n, n, rawDepth.data, 1, depthMapFactor, K, &seed, &rand_draws, lines3d.data(), &drawn) != PSLAM_OK)
        throw std::runtime_error(pslam_last_error(ctx.get()));
    rand_draws += drawn;
}

// void Frame::ComputeStereoFromRGBD(const cv::Mat& imDepth): mvuRight / mvDepth for N key points (mvKeysUn may alias mvKeys).
inline void ComputeStereoFromRGBD(Context& ctx, const std::vector<pslam_keypoint>& mvKeys, const std::vector<pslam_keypoint>& mvKeysUn, const Image16& rawDepth,
                                  float depthMapFactor, float mbf, std::vector<float>& mvuRight, std::vector<float>& mvDepth) {
    const int32_t n = (int32_t)mvKeys.size();
    mvuRight.assign(n, -1.f); mvDepth.assign(n, -1.f);
    if (n == 0) return;
    if (mvKeysUn.size() != mvKeys.size()) throw std::runtime_error("mvKeysUn and mvKeys differ in size");
    if (pslam_compute_stereo_from_rgbd_batch(ctx.get(), mvKeys.data(), mvKeysUn.data(), &n, n, rawDepth.data, 1, depthMapFactor, mbf, mvuRight.data(), mvDepth.data()) !=
        PSLAM_OK)
        throw std::runtime_error(pslam_last_error(ctx.get()));
}

// cv::Mat Tracking::TrackManhattanFrame(cv::Mat& mLastRcm, vector<SurfaceNormal>&, vector<FrameLine>&): normals = SurfaceNormal::normal
// (3 floats each), directions = FrameLine::direction (3 doubles each); returns the result record (R = the returned matrix) and the
// per-element membership masks (bit a-1: appended to vSurfaceNormal{x,y,z} / vVanishingLine{x,y,z}).
inline pslam_manhattan_result TrackManhattanFrame(Context& ctx, const float mLastRcm[9], const std::vector<float>& normals, const std::vector<double>& directions,
                                                  std::vector<uint8_t>& normal_mask, std::vector<uint8_t>& direction_mask) {
    const int32_t nn = (int32_t)(normals.size() / 3), nd = (int32_t)(directions.size() / 3);
    const int mn = nn > 0 ? nn : 1, md = nd > 0 ? nd : 1;
    normal_mask.assign(mn, 0); direction_mask.assign(md, 0);
    const float zero3f[3] = {0, 0, 0};
    const double zero3d[3] = {0, 0, 0};
    pslam_manhattan_result r;
    if (pslam_track_manhattan_batch(ctx.get(), mLastRcm, nn ? normals.data() : zero3f, &nn, mn, nd ? directions.data() : zero3d, &nd, md, 1, &r, normal_mask.data(),
                                    direction_mask.data()) != PSLAM_OK)
        throw std::runtime_error(pslam_last_error(ctx.get()));
    normal_mask.resize(nn); direction_mask.resize(nd);
    return r;
}

// bool Frame::isInFrustum(MapLine* pML, float viewingCosLimit) for the local map lines gathered into plain arrays (GetWorldPos: 6 doubles,
// GetNormal: 3 doubles, mfMaxDistance, mfMinDistance); returns nToMatch and fills the MapLine tracking fields.
inline int LinesInFrustum(Context& ctx, const pslam_line_frustum_frame& frame, const std::vector<double>& worldPos, const std::vector<double>& normal,
                          const std::vector<float>& mfMaxDistance, const std::vector<float>& mfMinDistance, float viewingCosLimit, std::vector<uint8_t>& mbTrackInView,
                          std::vector<float>& mTrackProj /* X1 Y1 X2 Y2 */, std::vector<int32_t>& mnTrackScaleLevel, std::vector<float>& mTrackViewCos) {
    const int n = (int)mfMaxDistance.size();
    mbTrackInView.assign(n, 0); mTrackProj.assign((size_t)4 * n, 0.f); mnTrackScaleLevel.assign(n, 0); mTrackViewCos.assign(n, 0.f);
    if (n == 0) return 0;
    if (worldPos.size() != (size_t)6 * n || normal.size() != (size_t)3 * n || mfMinDistance.size() != (size_t)n) throw std::runtime_error("map line arrays differ in size");
    const int rc = pslam_lines_in_frustum(ctx.get(), &frame, n, worldPos.data(), normal.data(), mfMaxDistance.data(), mfMinDistance.data(), viewingCosLimit,
                                          mbTrackInView.data(), mTrackProj.data(), mnTrackScaleLevel.data(), mTrackViewCos.data());
    if (rc < 0) throw std::runtime_error(pslam_last_error(ctx.get()));
    return rc;
}

}  // namespace pslam_adapter
