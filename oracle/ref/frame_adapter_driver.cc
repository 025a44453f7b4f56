// TEST INFRASTRUCTURE ONLY.  The product's pslam_adapter::ref::FrameConstructor (include/pslam_reference_adapter.hpp) on the reference's own Frame class
// (src/Frame.cc, linked from libmatch_ref.so), with plain-array entry points for tests/test_frame_adapter_gpu.py: arrays in -> cv::Mat inputs -> adapter ->
// the filled Frame's members back out as arrays.  The reference functions the test compares against (ComputeImageBounds, AssignFeaturesToGrid,
// GetFeaturesInArea, isLineGood, ComputeStereoFromRGBD) are called here as they are, on reference Frames that hold the adapter's key points / key lines, and
// ORBmatcher::SearchByProjection + Optimizer::PoseOptimization on the adapted Frame itself.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <sstream>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#define private public
#define protected public
#include "Frame.h"
#include "KeyFrame.h"
#include "Map.h"
#include "MapPoint.h"
#include "MapLine.h"
#include "MapPlane.h"
#include "ORBextractor.h"
#include "ORBmatcher.h"
#include "Optimizer.h"
#include "Config.h"
#include "KeyFrameDatabase.h"
#undef private
#undef protected
#include "pslam_reference_adapter.hpp"

using Planar_SLAM::Frame;

namespace {

std::string g_error;

struct Handle {
    std::unique_ptr<Planar_SLAM::ORBextractor> extractor;
    std::unique_ptr<pslam_adapter::ref::FrameConstructor> fc;
    int w, h;
};

cv::Mat image_mat(const uint8_t* image, int channels, int w, int h) { return cv::Mat(h, w, CV_MAKETYPE(CV_8U, channels), (void*)image); }
cv::Mat depth_mat(const void* depth, int type, int w, int h) { return cv::Mat(h, w, type, (void*)depth); }

// the members the early return of :106-107 does not reach get recognisable values first
void mark(Frame& F) {
    F.mnPlaneNum = -12345; F.mb = -1.5f; F.N = -1;
}

}  // namespace

extern "C" {

const char* fad_error() { return g_error.c_str(); }

// K = fx, fy, cx, cy (CV_32F 3x3 like Tracking's mK); dist = 4 distortion coefficients (CV_32F 4x1)
void* fad_create(int nfeatures, float scale, int nlevels, int ini_th, int min_th, const float* K4, const float* dist4, float bf, float th_depth, float depth_factor,
                 float plane_th, int w, int h, int rgb, int max_batch, int cap_plane_pts) {
    try {
        auto H = std::make_unique<Handle>();
        H->extractor = std::make_unique<Planar_SLAM::ORBextractor>(nfeatures, scale, nlevels, ini_th, min_th);
        cv::Mat K = cv::Mat::eye(3, 3, CV_32F);
        K.at<float>(0, 0) = K4[0]; K.at<float>(1, 1) = K4[1]; K.at<float>(0, 2) = K4[2]; K.at<float>(1, 2) = K4[3];
        cv::Mat D(4, 1, CV_32F);
        for (int i = 0; i < 4; ++i) D.at<float>(i) = dist4[i];
        H->fc = std::make_unique<pslam_adapter::ref::FrameConstructor>(H->extractor.get(), nfeatures, scale, nlevels, ini_th, min_th, K, D, bf, th_depth, depth_factor,
                                                                      plane_th, w, h, rgb != 0, max_batch, cap_plane_pts);
        H->w = w; H->h = h;
        return H.release();
    } catch (const std::exception& e) {
        g_error = e.what();
        return nullptr;
    }
}
void fad_destroy(void* h) { delete static_cast<Handle*>(h); }

// operator(): depth_type CV_16UC1 (the supported input) or anything else the test wants refused.  Returns the new Frame, NULL on an exception (fad_error).
void* fad_frame(void* h, const uint8_t* image, int channels, const void* depth, int depth_type, double stamp, void* voc) {
    Handle* H = static_cast<Handle*>(h);
    Frame* F = new Frame();
    mark(*F);
    try {
        (*H->fc)(*F, cv::Mat(), image_mat(image, channels, H->w, H->h), depth_mat(depth, depth_type, H->w, H->h), stamp, (Planar_SLAM::ORBVocabulary*)voc);
        return F;
    } catch (const std::exception& e) {
        g_error = e.what();
        delete F;
        return nullptr;
    }
}

// batch(): n frames of the same channel count, images [n][h][w][channels], depth [n][h][w] uint16; frames_out[n]
int fad_batch(void* h, int n, const uint8_t* images, int channels, const uint16_t* depths, const double* stamps, void* voc, void** frames_out) {
    Handle* H = static_cast<Handle*>(h);
    const size_t npx = (size_t)H->w * H->h;
    std::vector<Frame*> frames(n);
    std::vector<cv::Mat> ims(n), deps(n);
    for (int i = 0; i < n; ++i) {
        frames[i] = new Frame(); mark(*frames[i]);
        ims[i] = image_mat(images + i * npx * channels, channels, H->w, H->h);
        deps[i] = depth_mat(depths + i * npx, CV_16UC1, H->w, H->h);
    }
    try {
        H->fc->batch(frames, ims, deps, std::vector<double>(stamps, stamps + n), (Planar_SLAM::ORBVocabulary*)voc);
    } catch (const std::exception& e) {
        g_error = e.what();
        for (Frame* F : frames) delete F;
        return -1;
    }
    for (int i = 0; i < n; ++i) frames_out[i] = frames[i];
    return 0;
}

int64_t fad_draws(void* h) { return static_cast<Handle*>(h)->fc->draws(); }
void fad_advance(void* h, int64_t n) { static_cast<Handle*>(h)->fc->advance(n); }
void fad_timing(void* h, double* out) {
    const auto& fc = *static_cast<Handle*>(h)->fc;
    out[0] = fc.call_seconds(); out[1] = fc.unpack_seconds(); out[2] = fc.support_seconds();
}
void* fad_extractor(void* h) { return static_cast<Handle*>(h)->extractor.get(); }
void fad_free_frame(void* F) { delete static_cast<Frame*>(F); }

// the extractor's scale tables (what Frame.cc:65-71 reads): [4][nlevels] scale, inverse scale, sigma2, inverse sigma2
void fad_extractor_tables(void* h, float* out) {
    Planar_SLAM::ORBextractor* e = static_cast<Handle*>(h)->extractor.get();
    const int n = e->GetLevels();
    const std::vector<float> t[4] = {e->GetScaleFactors(), e->GetInverseScaleFactors(), e->GetScaleSigmaSquares(), e->GetInverseScaleSigmaSquares()};
    for (int k = 0; k < 4; ++k) std::copy(t[k].begin(), t[k].end(), out + k * n);
}

// ---- statics ----------------------------------------------------------------------------------------------------------------------------------------------
// fx fy cx cy invfx invfy mnMinX mnMaxX mnMinY mnMaxY mfGridElementWidthInv mfGridElementHeightInv mbInitialComputations nNextId
void fad_statics(double* s) {
    const double v[14] = {Frame::fx, Frame::fy, Frame::cx, Frame::cy, Frame::invfx, Frame::invfy, Frame::mnMinX, Frame::mnMaxX, Frame::mnMinY, Frame::mnMaxY,
                          Frame::mfGridElementWidthInv, Frame::mfGridElementHeightInv, (double)Frame::mbInitialComputations, (double)Frame::nNextId};
    std::copy(v, v + 14, s);
}
void fad_set_statics(int initial_computations, float fill) {       // fill: a value no frame computes, so the test sees what the adapter writes
    Frame::mbInitialComputations = initial_computations != 0;
    Frame::fx = Frame::fy = Frame::cx = Frame::cy = Frame::invfx = Frame::invfy = fill;
    Frame::mnMinX = Frame::mnMaxX = Frame::mnMinY = Frame::mnMaxY = Frame::mfGridElementWidthInv = Frame::mfGridElementHeightInv = fill;
}

// ---- read-back of a Frame ---------------------------------------------------------------------------------------------------------------------------------
// scalars: mnId mTimeStamp N NL mbf mb mThDepth mnScaleLevels mfScaleFactor mfLogScaleFactor mnPlaneNum dealWithLine, then mK (9), mDistCoef (4),
// mpORBvocabulary, mpORBextractorLeft, mpORBextractorRight (as integers)
void fad_scalars(void* f, double* s) {
    Frame& F = *static_cast<Frame*>(f);
    const double v[12] = {(double)F.mnId, F.mTimeStamp, (double)F.N, (double)F.NL, F.mbf, F.mb, F.mThDepth, (double)F.mnScaleLevels, F.mfScaleFactor,
                          F.mfLogScaleFactor, (double)F.mnPlaneNum, (double)F.dealWithLine};
    std::copy(v, v + 12, s);
    for (int i = 0; i < 9; ++i) s[12 + i] = F.mK.empty() ? NAN : F.mK.at<float>(i / 3, i % 3);
    for (int i = 0; i < 4; ++i) s[21 + i] = F.mDistCoef.empty() ? NAN : F.mDistCoef.at<float>(i);
    s[25] = (double)(uintptr_t)F.mpORBvocabulary; s[26] = (double)(uintptr_t)F.mpORBextractorLeft; s[27] = (double)(uintptr_t)F.mpORBextractorRight;
}

// per-feature vector sizes and contents: [0] mvKeys [1] mvKeysUn [2] mvuRight [3] mvDepth [4] mDescriptors rows [5] mvpMapPoints [6] mvbOutlier
// [7] mvpMapLines [8] mvbLineOutlier [9] mvpMapPlanes [10] mvpParallelPlanes [11] mvpVerticalPlanes [12] mvPlanePointMatches [13] mvPlaneLineMatches
// [14] mvbPlaneOutlier [15] mvbVerPlaneOutlier [16] mvbParPlaneOutlier [17] mvPlanePoints [18] mvPlaneCoefficients [19] vSurfaceNormal [20] mVF3DLines
// [21] mvScaleFactors; [22] 1 if every pointer of [5] [7] [9]-[11] is NULL, every flag of [6] [8] [14]-[16] false and every list of [12] [13] empty
// [23] mDescriptors type (-1: empty)
void fad_sizes(void* f, int64_t* s) {
    Frame& F = *static_cast<Frame*>(f);
    const int64_t v[22] = {(int64_t)F.mvKeys.size(), (int64_t)F.mvKeysUn.size(), (int64_t)F.mvuRight.size(), (int64_t)F.mvDepth.size(), F.mDescriptors.rows,
                           (int64_t)F.mvpMapPoints.size(), (int64_t)F.mvbOutlier.size(), (int64_t)F.mvpMapLines.size(), (int64_t)F.mvbLineOutlier.size(),
                           (int64_t)F.mvpMapPlanes.size(), (int64_t)F.mvpParallelPlanes.size(), (int64_t)F.mvpVerticalPlanes.size(),
                           (int64_t)F.mvPlanePointMatches.size(), (int64_t)F.mvPlaneLineMatches.size(), (int64_t)F.mvbPlaneOutlier.size(),
                           (int64_t)F.mvbVerPlaneOutlier.size(), (int64_t)F.mvbParPlaneOutlier.size(), (int64_t)F.mvPlanePoints.size(),
                           (int64_t)F.mvPlaneCoefficients.size(), (int64_t)F.vSurfaceNormal.size(), (int64_t)F.mVF3DLines.size(), (int64_t)F.mvScaleFactors.size()};
    std::copy(v, v + 22, s);
    bool clean = true;
    for (auto* p : F.mvpMapPoints) clean &= p == nullptr;
    for (auto* p : F.mvpMapLines) clean &= p == nullptr;
    for (auto* v2 : {&F.mvpMapPlanes, &F.mvpParallelPlanes, &F.mvpVerticalPlanes}) for (auto* p : *v2) clean &= p == nullptr;
    for (auto* v2 : {&F.mvbOutlier, &F.mvbLineOutlier, &F.mvbPlaneOutlier, &F.mvbVerPlaneOutlier, &F.mvbParPlaneOutlier}) for (bool b : *v2) clean &= !b;
    for (const auto& l : F.mvPlanePointMatches) clean &= l.empty();
    for (const auto& l : F.mvPlaneLineMatches) clean &= l.empty();
    s[22] = clean ? 1 : 0;
    s[23] = F.mDescriptors.empty() ? -1 : F.mDescriptors.type();
}

// scale tables [4][mvScaleFactors.size()]: mvScaleFactors, mvInvScaleFactors, mvLevelSigma2, mvInvLevelSigma2
void fad_scale_tables(void* f, float* out) {
    Frame& F = *static_cast<Frame*>(f);
    const size_t n = F.mvScaleFactors.size();
    const std::vector<float>* t[4] = {&F.mvScaleFactors, &F.mvInvScaleFactors, &F.mvLevelSigma2, &F.mvInvLevelSigma2};
    for (int k = 0; k < 4; ++k) for (size_t i = 0; i < n && i < t[k]->size(); ++i) out[k * n + i] = (*t[k])[i];
}

// mvKeys / mvKeysUn as pslam_keypoint records, mDescriptors [N][32], mvuRight, mvDepth
void fad_keys(void* f, pslam_keypoint* keys, pslam_keypoint* keys_un, uint8_t* desc, float* u_right, float* depth) {
    Frame& F = *static_cast<Frame*>(f);
    auto put = [](const cv::KeyPoint& k, pslam_keypoint& o) { o.x = k.pt.x; o.y = k.pt.y; o.size = k.size; o.angle = k.angle; o.response = k.response; o.octave = k.octave; o.class_id = k.class_id; };
    for (size_t i = 0; i < F.mvKeys.size(); ++i) put(F.mvKeys[i], keys[i]);
    for (size_t i = 0; i < F.mvKeysUn.size(); ++i) put(F.mvKeysUn[i], keys_un[i]);
    for (int i = 0; i < F.mDescriptors.rows; ++i) std::memcpy(desc + 32 * (size_t)i, F.mDescriptors.ptr(i), 32);
    std::copy(F.mvuRight.begin(), F.mvuRight.end(), u_right);
    std::copy(F.mvDepth.begin(), F.mvDepth.end(), depth);
}

// mGrid as CSR over the cells in [col][row] order: off [64 * 48 + 1], idx [N]
void fad_grid(void* f, int32_t* off, int32_t* idx) {
    Frame& F = *static_cast<Frame*>(f);
    int n = 0;
    off[0] = 0;
    for (int i = 0; i < FRAME_GRID_COLS; ++i)
        for (int j = 0; j < FRAME_GRID_ROWS; ++j) {
            for (size_t v : F.mGrid[i][j]) idx[n++] = (int32_t)v;
            off[i * FRAME_GRID_ROWS + j + 1] = n;
        }
}

int fad_features_in_area(void* f, float x, float y, float r, int min_level, int max_level, int32_t* out) {
    const std::vector<size_t> v = static_cast<Frame*>(f)->GetFeaturesInArea(x, y, r, min_level, max_level);
    for (size_t i = 0; i < v.size(); ++i) out[i] = (int32_t)v[i];
    return (int)v.size();
}

// mvKeylinesUn as pslam_keyline records (field by field), mvKeyLineFunctions [NL][3], mLdesc [NL][32], mvDepthLine, mvLines3D [NL][6]
void fad_lines(void* f, pslam_keyline* kl, double* lf, uint8_t* ldesc, float* depth_line, double* lines3d) {
    Frame& F = *static_cast<Frame*>(f);
    for (size_t i = 0; i < F.mvKeylinesUn.size(); ++i) {
        const auto& L = F.mvKeylinesUn[i];
        pslam_keyline& o = kl[i];
        o.angle = L.angle; o.class_id = L.class_id; o.octave = L.octave; o.pt_x = L.pt.x; o.pt_y = L.pt.y; o.response = L.response; o.size = L.size;
        o.startPointX = L.startPointX; o.startPointY = L.startPointY; o.endPointX = L.endPointX; o.endPointY = L.endPointY;
        o.sPointInOctaveX = L.sPointInOctaveX; o.sPointInOctaveY = L.sPointInOctaveY; o.ePointInOctaveX = L.ePointInOctaveX; o.ePointInOctaveY = L.ePointInOctaveY;
        o.lineLength = L.lineLength; o.numOfPixels = L.numOfPixels;
    }
    for (size_t i = 0; i < F.mvKeyLineFunctions.size(); ++i) for (int c = 0; c < 3; ++c) lf[3 * i + c] = F.mvKeyLineFunctions[i](c);
    for (int i = 0; i < F.mLdesc.rows; ++i) std::memcpy(ldesc + 32 * (size_t)i, F.mLdesc.ptr(i), 32);
    std::copy(F.mvDepthLine.begin(), F.mvDepthLine.end(), depth_line);
    for (size_t i = 0; i < F.mvLines3D.size(); ++i) for (int c = 0; c < 6; ++c) lines3d[6 * i + c] = F.mvLines3D[i](c);
}

// mVF3DLines: head [n][15] = p (2), q (2), direction (3), direct1 (3), direct2 (3), haveDepth, rndpts3d.size(); pts [sum][27] = pos (3), xyz (3), W_sqrt (3),
// DU (9), dux (3), cov diagonal + upper triangle (6).  Returns the total number of points (call with NULL pointers to size the buffers).
int fad_vf3d(void* f, double* head, double* pts) {
    Frame& F = *static_cast<Frame*>(f);
    int n = 0;
    for (size_t i = 0; i < F.mVF3DLines.size(); ++i) {
        const FrameLine& L = F.mVF3DLines[i];
        if (head) {
            double* h = head + 15 * i;
            const double v[15] = {L.p.x, L.p.y, L.q.x, L.q.y, L.direction.x, L.direction.y, L.direction.z, L.direct1.x, L.direct1.y, L.direct1.z,
                                  L.direct2.x, L.direct2.y, L.direct2.z, (double)L.haveDepth, (double)L.rndpts3d.size()};
            std::copy(v, v + 15, h);
        }
        for (const RandomPoint3d& p : L.rndpts3d) {
            if (pts) {
                double* o = pts + 27 * (size_t)n;
                o[0] = p.pos.x; o[1] = p.pos.y; o[2] = p.pos.z;
                for (int c = 0; c < 3; ++c) { o[3 + c] = p.xyz[c]; o[6 + c] = p.W_sqrt[c]; o[18 + c] = p.dux[c]; }
                for (int c = 0; c < 9; ++c) o[9 + c] = p.DU[c];
                const int rc[6][2] = {{0, 0}, {1, 1}, {2, 2}, {0, 1}, {0, 2}, {1, 2}};
                for (int c = 0; c < 6; ++c) o[21 + c] = p.cov.at<double>(rc[c][0], rc[c][1]);
            }
            ++n;
        }
    }
    return n;
}

// mvPlanePoints as off [n + 1] / pts [total][3] (+ width, height per cloud in wh [n][2]), mvPlaneCoefficients [n][4] (+ their type and shape in meta [n][3]).
// Returns the total number of points (call with NULL pointers to size the buffers).
int fad_planes(void* f, int32_t* off, float* pts, int32_t* wh, float* coef, int32_t* meta) {
    Frame& F = *static_cast<Frame*>(f);
    int n = 0;
    if (off) off[0] = 0;
    for (size_t q = 0; q < F.mvPlanePoints.size(); ++q) {
        for (const auto& p : F.mvPlanePoints[q].points) {
            if (pts) { pts[3 * n] = p.x; pts[3 * n + 1] = p.y; pts[3 * n + 2] = p.z; }
            ++n;
        }
        if (off) off[q + 1] = n;
        if (wh) { wh[2 * q] = (int32_t)F.mvPlanePoints[q].width; wh[2 * q + 1] = (int32_t)F.mvPlanePoints[q].height; }
    }
    for (size_t q = 0; coef && q < F.mvPlaneCoefficients.size(); ++q) {
        const cv::Mat& c = F.mvPlaneCoefficients[q];
        meta[3 * q] = c.type(); meta[3 * q + 1] = c.rows; meta[3 * q + 2] = c.cols;
        for (int k = 0; k < 4; ++k) coef[4 * q + k] = c.at<float>(k);
    }
    return n;
}

// vSurfaceNormal [n][8] = normal, cameraPosition, FramePosition
void fad_normals(void* f, float* out) {
    Frame& F = *static_cast<Frame*>(f);
    for (size_t i = 0; i < F.vSurfaceNormal.size(); ++i) {
        const SurfaceNormal& s = F.vSurfaceNormal[i];
        const float v[8] = {s.normal.x, s.normal.y, s.normal.z, s.cameraPosition.x, s.cameraPosition.y, s.cameraPosition.z, (float)s.FramePosition.x, (float)s.FramePosition.y};
        std::copy(v, v + 8, out + 8 * i);
    }
}

// ---- the reference's functions on reference Frames holding the adapter's features --------------------------------------------------------------------
// Frame::ComputeImageBounds(imGray) + Frame::AssignFeaturesToGrid() on a Frame with the adapter Frame's mvKeysUn and mDistCoef; returns that Frame
void* fad_ref_grid_frame(void* f, int w, int h) {
    const Frame& A = *static_cast<Frame*>(f);
    Frame* R = new Frame();
    R->N = A.N; R->mvKeysUn = A.mvKeysUn; R->mDistCoef = A.mDistCoef.clone(); R->mK = A.mK.clone();
    cv::Mat imGray(h, w, CV_8UC1);
    R->ComputeImageBounds(imGray);
    R->AssignFeaturesToGrid();
    return R;
}

// Frame::ComputeStereoFromRGBD(depth) on a Frame with the adapter Frame's mvKeys / mvKeysUn / mbf; depth: metres [h][w] float
void fad_ref_stereo(void* f, const float* depth_m, int w, int h, float* u_right, float* depth) {
    const Frame& A = *static_cast<Frame*>(f);
    Frame R;
    R.N = A.N; R.mbf = A.mbf; R.mvKeys = A.mvKeys; R.mvKeysUn = A.mvKeysUn;
    R.ComputeStereoFromRGBD(cv::Mat(h, w, CV_32F, (void*)depth_m));
    std::copy(R.mvuRight.begin(), R.mvuRight.end(), u_right);
    std::copy(R.mvDepth.begin(), R.mvDepth.end(), depth);
}

// Frame::isLineGood(imGray, depth, tmpK) on n Frames in a row holding the adapter Frames' mvKeylinesUn, with srand(seed) and `skip` draws before the first only
// (no srand in between, like consecutive reference constructors); tmpK from the Frame statics (:84-86).  Returns the Frames; next4 receives the next four
// rand() values after the last frame (where the stream stands).
void fad_ref_is_line_good(void** adapter_frames, int n, const float* depth_m, int w, int h, uint32_t seed, int64_t skip, void** out, int32_t* next4) {
    const cv::Mat K = (cv::Mat_<double>(3, 3) << Frame::fx, 0, Frame::cx, 0, Frame::fy, Frame::cy, 0, 0, 1);
    srand(seed);
    for (int64_t i = 0; i < skip; ++i) (void)rand();
    for (int k = 0; k < n; ++k) {
        Frame* R = new Frame();
        R->mvKeylinesUn = static_cast<Frame*>(adapter_frames[k])->mvKeylinesUn;
        R->NL = (int)R->mvKeylinesUn.size();
        R->isLineGood(cv::Mat(), cv::Mat(h, w, CV_32F, (void*)(depth_m + (size_t)k * w * h)), K);
        out[k] = R;
    }
    for (int i = 0; i < 4; ++i) next4[i] = rand();
}

// the next four rand() values after srand(seed) and `skip` draws
void fad_rand_after(uint32_t seed, int64_t skip, int32_t* next4) {
    srand(seed);
    for (int64_t i = 0; i < skip; ++i) (void)rand();
    for (int i = 0; i < 4; ++i) next4[i] = rand();
}

// Tracking::SearchLocalPoints' frustum loop (isInFrustum(pMP, 0.5) on every point that is not skipped), ORBmatcher::SearchByProjection(F, points, th), then
// Optimizer::PoseOptimization(&F) from the pose Tcw0 - the reference's own code on the ADAPTED Frame, against map points built from the pslam_map_points arrays
// (as oracle/ref/match_driver.cc builds them).  settings = Plane.AngleInfo, DistanceInfo, ParallelInfo, VerticalInfo, Chi, VPChi.  Writes the match of every
// key point (-1: none), the optimised pose and mvbOutlier; returns the number of matches, *n_inliers = PoseOptimization's return.
int fad_ref_track_local(void* f, const float* Tcw, const float* Tcw0, const pslam_map_points* m, float th, float nnratio, const double* settings, int32_t* matches,
                        float* Tcw_out, uint8_t* outlier, int32_t* n_inliers) {
    Frame& F = *static_cast<Frame*>(f);
    auto& t = cv::FileStorage::table();
    t["Plane.AngleInfo"] = settings[0]; t["Plane.DistanceInfo"] = settings[1]; t["Plane.ParallelInfo"] = settings[2]; t["Plane.VerticalInfo"] = settings[3];
    t["Plane.Chi"] = settings[4]; t["Plane.VPChi"] = settings[5];
    Planar_SLAM::Config::SetParameterFile("pslam-settings-table");
    auto mat44 = [](const float* T) { cv::Mat M(4, 4, CV_32F); for (int i = 0; i < 16; ++i) M.at<float>(i / 4, i % 4) = T[i]; return M; };
    Planar_SLAM::Map map;
    Frame anchor_frame;
    anchor_frame.N = 0;
    anchor_frame.SetPose(cv::Mat::eye(4, 4, CV_32F));
    Planar_SLAM::KeyFrame* anchor = new Planar_SLAM::KeyFrame(anchor_frame, &map, static_cast<Planar_SLAM::KeyFrameDatabase*>(NULL));
    std::vector<Planar_SLAM::MapPoint*> pts(m->n);
    std::map<Planar_SLAM::MapPoint*, int> index;
    for (int i = 0; i < m->n; ++i) {
        cv::Mat X(3, 1, CV_32F);
        for (int c = 0; c < 3; ++c) X.at<float>(c) = m->pos[3 * i + c];
        Planar_SLAM::MapPoint* p = new Planar_SLAM::MapPoint(X, anchor, &map);
        p->mNormalVector = cv::Mat(3, 1, CV_32F);
        for (int c = 0; c < 3; ++c) p->mNormalVector.at<float>(c) = m->normal[3 * i + c];
        p->mfMaxDistance = m->max_distance[i]; p->mfMinDistance = m->min_distance[i];
        p->mDescriptor = cv::Mat(1, 32, CV_8U);
        std::memcpy(p->mDescriptor.ptr(0), m->desc + 32 * (size_t)i, 32);
        p->nObs = m->has_obs[i] ? 1 : 0;
        p->mbTrackInView = false;
        pts[i] = p; index[p] = i;
    }
    F.SetPose(mat44(Tcw));
    for (int i = 0; i < m->n; ++i) if (!m->skip[i]) F.isInFrustum(pts[i], 0.5);
    Planar_SLAM::ORBmatcher matcher(nnratio);
    const int n = matcher.SearchByProjection(F, pts, th);
    for (int i = 0; i < F.N; ++i) matches[i] = F.mvpMapPoints[i] ? index.at(F.mvpMapPoints[i]) : -1;
    F.SetPose(mat44(Tcw0));
    *n_inliers = Planar_SLAM::Optimizer::PoseOptimization(&F);
    for (int i = 0; i < 16; ++i) Tcw_out[i] = F.mTcw.at<float>(i / 4, i % 4);
    for (int i = 0; i < F.N; ++i) { outlier[i] = F.mvbOutlier[i] ? 1 : 0; F.mvpMapPoints[i] = static_cast<Planar_SLAM::MapPoint*>(NULL); }
    for (Planar_SLAM::MapPoint* p : pts) delete p;
    delete anchor;
    return n;
}

}  // extern "C"
