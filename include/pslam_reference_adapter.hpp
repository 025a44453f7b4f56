// pslam_reference_adapter.hpp - drop-in replacements WITH THE REFERENCE'S OWN SIGNATURES (Frame*, Frame&, std::vector<MapPoint*>, MapPlane* ...)
// on top of the C ABI (include/pslam_abi.h).  Header-only; compile it inside the PlanarSLAM tree after the reference's own headers:
//
//     #include "Frame.h"  "MapPoint.h"  "MapPlane.h"  "MapLine.h"  "Config.h"          (the reference's)
//     #include "pslam_reference_adapter.hpp"
//     ...
//     int nInliers = pslam_adapter::ref::Optimizer::PoseOptimization(&mCurrentFrame);                       // was Optimizer::PoseOptimization   (include/Optimizer.h:38)
//     pslam_adapter::ref::ORBmatcher matcher(0.8);  matcher.SearchByProjection(mCurrentFrame, mvpLocalMapPoints, th);    // include/ORBmatcher.h:43
//
// Each entry point gathers what the reference function reads from the object graph - under the same mutexes the reference takes -, calls the C ABI
// (one context per calling thread, created on first use), and writes back exactly what the reference function writes (mvpMapPoints, mvbOutlier...,
// mTcw through Frame::SetPose).  Return values are the reference's.
//
//   static int  Optimizer::PoseOptimization(Frame*)                                   include/Optimizer.h:38   src/Optimizer.cc:550-1275
//   static int  Optimizer::TranslationOptimization(Frame*)                            include/Optimizer.h:40   src/Optimizer.cc:2995-3737
//   static void Optimizer::LocalBundleAdjustment(KeyFrame*, bool*, Map*)              include/Optimizer.h:34   src/Optimizer.cc:1853-2678
//   int ORBmatcher::SearchByProjection(Frame&, const vector<MapPoint*>&, float th)    include/ORBmatcher.h:43  src/ORBmatcher.cc:46-130
//   int ORBmatcher::SearchByProjection(Frame&, const Frame&, float th, bool bMono)    include/ORBmatcher.h:47  src/ORBmatcher.cc:1396-1535
//   int ORBmatcher::SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&)                include/ORBmatcher.h:53  src/ORBmatcher.cc:160-292
//   int ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, vector<MapPoint*>&)             include/ORBmatcher.h:56  src/ORBmatcher.cc:526-659
//   int LSDmatcher::SearchByProjection(Frame&, const vector<MapLine*>&, float th)     include/LSDmatcher.h:24  src/LSDmatcher.cpp:141-211
//   int LSDmatcher::SearchByDescriptor(KeyFrame*, Frame&, vector<MapLine*>&)          include/LSDmatcher.h:21  src/LSDmatcher.cpp:242-279
//   int PlaneMatcher::SearchMapByCoefficients(Frame&, const vector<MapPlane*>&)       include/PlaneMatcher.h:18 src/PlaneMatcher.cpp:10-67
//   KeyFrameDatabase::add / erase / clear / DetectLoopCandidates(KeyFrame*, float) / DetectRelocalizationCandidates(Frame*)
//                                                                                     include/KeyFrameDatabase.h:43-75  src/KeyFrameDatabase.cc:38-305
//   void ORBextractor::operator()(cv::InputArray, cv::InputArray, vector<cv::KeyPoint>&, cv::OutputArray)   include/ORBextractor.h:59-61
//   Frame::Frame(imRGB, imGray, imDepth, timeStamp, extractor, voc, K, distCoef, bf, thDepth, depthMapFactor) include/Frame.h:57  src/Frame.cc:55-152
//                                                                                     (FrameConstructor: fills a default-constructed Frame; batch() for replays)
//
// Two reference members read here are protected in the reference (MapPoint::mfMaxDistance / mfMinDistance: the getters return them scaled by 1.2 / 0.8
// and a float division does not undo a float multiplication): add `friend struct pslam_adapter::ref::Access;` to MapPoint, or two raw getters - see
// INTEGRATION.md.  tests/ builds this header against the reference's headers with the stand-in OpenCV / Eigen of oracle/ref/shims
// (oracle/ref/adapter_driver.cc) and compares every entry point with the reference function on the same objects (tests/test_reference_adapter_gpu.py).
#pragma once
#include <cmath>
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <string>
#include <list>
#include <map>
#include <mutex>
#include <set>
#include <stdexcept>
#include <unordered_map>
#include <vector>

#include "pslam_abi.h"

namespace pslam_adapter {
namespace ref {

using Planar_SLAM::Frame;
using Planar_SLAM::KeyFrame;
using Planar_SLAM::MapLine;
using Planar_SLAM::MapPlane;
using Planar_SLAM::MapPoint;

struct Access {          // the two protected MapPoint members (see the header comment)
    static float max_distance(MapPoint* p) { return p->mfMaxDistance; }
    static float min_distance(MapPoint* p) { return p->mfMinDistance; }
};

// one context per calling thread (the reference calls its matchers / optimiser from the tracking thread and from three SearchLocal* threads)
inline pslam_ctx* context(int width = 640, int height = 480) {
    struct Holder {
        pslam_ctx* c = nullptr; int w = 0, h = 0;
        ~Holder() { if (c) pslam_destroy(c); }
    };
    thread_local Holder H;
    if (!H.c || H.w != width || H.h != height) {
        if (H.c) pslam_destroy(H.c);
        pslam_config cfg;
        pslam_default_config(&cfg, width, height, 1);
        if (pslam_create(&cfg, &H.c) != PSLAM_OK) { H.c = nullptr; throw std::runtime_error("pslam_create failed: no sm_90 GPU"); }
        H.w = width; H.h = height;
    }
    return H.c;
}

struct Optimizer {
    static int PoseOptimization(Frame* pFrame) { return run(pFrame, false); }
    static int TranslationOptimization(Frame* pFrame) { return run(pFrame, true); }

    // Local bundle adjustment around pKF (include/Optimizer.h:34, src/Optimizer.cc:1853-2678).  The walk that selects the local / fixed key frames and the local
    // points, lines and planes is the reference's (same marker fields mnBALocalForKF / mnBAFixedForKF, same list orders); the graph it would hand to g2o goes to
    // pslam_local_bundle_adjustment as plain arrays; erasures, poses and landmark positions are written back under pMap->mMutexMapUpdate like the reference does.
    // pbStopFlag is only honoured before the optimisation starts (a result that depends on when another thread raises the flag cannot be reproduced).
    static void LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Planar_SLAM::Map* pMap) {
        std::list<KeyFrame*> lLocalKeyFrames;
        lLocalKeyFrames.push_back(pKF);
        pKF->mnBALocalForKF = pKF->mnId;
        for (KeyFrame* pKFi : pKF->GetVectorCovisibleKeyFrames()) {
            pKFi->mnBALocalForKF = pKF->mnId;
            if (!pKFi->isBad()) lLocalKeyFrames.push_back(pKFi);
        }
        std::list<MapPoint*> lLocalMapPoints;
        std::list<MapLine*> lLocalMapLines;
        std::list<MapPlane*> lLocalMapPlanes;
        for (KeyFrame* k : lLocalKeyFrames)
            for (MapPoint* pMP : k->GetMapPointMatches())
                if (pMP && !pMP->isBad() && pMP->mnBALocalForKF != pKF->mnId) { lLocalMapPoints.push_back(pMP); pMP->mnBALocalForKF = pKF->mnId; }
        for (KeyFrame* k : lLocalKeyFrames)
            for (MapLine* pML : k->GetMapLineMatches())
                if (pML && !pML->isBad() && pML->mnBALocalForKF != pKF->mnId) { lLocalMapLines.push_back(pML); pML->mnBALocalForKF = pKF->mnId; }
        for (KeyFrame* k : lLocalKeyFrames)
            for (MapPlane* pMP : k->GetMapPlaneMatches())
                if (pMP && !pMP->isBad() && pMP->mnBALocalForKF != pKF->mnId) { lLocalMapPlanes.push_back(pMP); pMP->mnBALocalForKF = pKF->mnId; }
        std::list<KeyFrame*> lFixedCameras;
        auto fix = [&](const std::map<KeyFrame*, size_t>& observations) {
            for (const auto& o : observations) {
                KeyFrame* pKFi = o.first;
                if (pKFi->mnBALocalForKF != pKF->mnId && pKFi->mnBAFixedForKF != pKF->mnId) {
                    pKFi->mnBAFixedForKF = pKF->mnId;
                    if (!pKFi->isBad()) lFixedCameras.push_back(pKFi);
                }
            }
        };
        for (MapPoint* p : lLocalMapPoints) fix(p->GetObservations());
        for (MapLine* l : lLocalMapLines) fix(l->GetObservations());
        for (MapPlane* q : lLocalMapPlanes) fix(q->GetObservations());
        if (pbStopFlag && *pbStopFlag) return;

        // vertices in g2o's order (ascending id): key frames by mnId, then points, line end points and planes by mnId
        std::vector<KeyFrame*> kfs(lLocalKeyFrames.begin(), lLocalKeyFrames.end());
        const size_t n_local = kfs.size();
        kfs.insert(kfs.end(), lFixedCameras.begin(), lFixedCameras.end());
        std::vector<uint8_t> is_fixed_cam(kfs.size(), 0);
        for (size_t i = n_local; i < kfs.size(); ++i) is_fixed_cam[i] = 1;
        std::vector<int> kf_order(kfs.size());
        for (size_t i = 0; i < kfs.size(); ++i) kf_order[i] = (int)i;
        std::sort(kf_order.begin(), kf_order.end(), [&](int a, int b) { return kfs[a]->mnId < kfs[b]->mnId; });
        std::unordered_map<KeyFrame*, int> kf_index;
        std::vector<KeyFrame*> kf_sorted(kfs.size());
        std::vector<float> kf_Tcw(kfs.size() * 16), kf_K(kfs.size() * 5);
        std::vector<uint8_t> kf_fixed(kfs.size());
        unsigned long maxKFid = 0;
        for (size_t r = 0; r < kfs.size(); ++r) {
            KeyFrame* k = kfs[kf_order[r]];
            kf_sorted[r] = k; kf_index[k] = (int)r;
            kf_fixed[r] = (is_fixed_cam[kf_order[r]] || k->mnId == 0) ? 1 : 0;
            const cv::Mat T = k->GetPose();
            for (int i = 0; i < 16; ++i) kf_Tcw[r * 16 + i] = T.at<float>(i / 4, i % 4);
            kf_K[r * 5] = k->fx; kf_K[r * 5 + 1] = k->fy; kf_K[r * 5 + 2] = k->cx; kf_K[r * 5 + 3] = k->cy; kf_K[r * 5 + 4] = k->mbf;
            if (k->mnId > maxKFid) maxKFid = k->mnId;
        }
        auto by_id = [](auto& v) { std::stable_sort(v.begin(), v.end(), [](auto* a, auto* b) { return a->mnId < b->mnId; }); };
        std::vector<MapPoint*> pts(lLocalMapPoints.begin(), lLocalMapPoints.end());
        std::vector<MapLine*> lines(lLocalMapLines.begin(), lLocalMapLines.end());
        std::vector<MapPlane*> planes(lLocalMapPlanes.begin(), lLocalMapPlanes.end());
        by_id(pts); by_id(lines); by_id(planes);
        std::unordered_map<MapPoint*, int> pt_index; std::unordered_map<MapLine*, int> line_index; std::unordered_map<MapPlane*, int> plane_index;
        std::vector<float> pt_Xw(pts.size() * 3 + 3), plane_Xw(planes.size() * 4 + 4);
        std::vector<double> line_Xw(lines.size() * 6 + 6);
        for (size_t i = 0; i < pts.size(); ++i) { pt_index[pts[i]] = (int)i; const cv::Mat X = pts[i]->GetWorldPos(); for (int c = 0; c < 3; ++c) pt_Xw[i * 3 + c] = X.at<float>(c); }
        for (size_t i = 0; i < lines.size(); ++i) { line_index[lines[i]] = (int)i; const auto X = lines[i]->GetWorldPos(); for (int c = 0; c < 6; ++c) line_Xw[i * 6 + c] = X(c); }
        for (size_t i = 0; i < planes.size(); ++i) { plane_index[planes[i]] = (int)i; const cv::Mat X = planes[i]->GetWorldPos(); for (int c = 0; c < 4; ++c) plane_Xw[i * 4 + c] = X.at<float>(c); }

        // edges in creation order: the local lists as the reference walks them, every landmark's observations in its std::map order
        struct PtObs { KeyFrame* kf; MapPoint* p; };
        struct LineObs { KeyFrame* kf; MapLine* l; };
        struct PlaneObs { KeyFrame* kf; MapPlane* q; };
        std::vector<PtObs> pt_obs; std::vector<LineObs> line_obs; std::vector<PlaneObs> plane_obs[3];
        std::vector<int32_t> po_kf, po_pt, lo_kf, lo_line, plo_kf[3], plo_plane[3];
        std::vector<float> po_uvr, po_is2, plo_meas[3];
        std::vector<double> lo_l;
        for (MapPoint* pMP : lLocalMapPoints)
            for (const auto& o : pMP->GetObservations()) {
                KeyFrame* pKFi = o.first;
                if (pKFi->isBad()) continue;
                const auto it = kf_index.find(pKFi);
                if (it == kf_index.end()) continue;                         // (cannot happen: every observer is local or was made a fixed camera above)
                const cv::KeyPoint& kpUn = pKFi->mvKeysUn[o.second];
                po_kf.push_back(it->second); po_pt.push_back(pt_index[pMP]);
                po_uvr.push_back(kpUn.pt.x); po_uvr.push_back(kpUn.pt.y); po_uvr.push_back(pKFi->mvuRight[o.second] < 0 ? -1.0f : pKFi->mvuRight[o.second]);
                po_is2.push_back(pKFi->mvInvLevelSigma2[kpUn.octave]);
                pt_obs.push_back(PtObs{pKFi, pMP});
            }
        const int cur = kf_index[pKF];
        for (MapLine* pML : lLocalMapLines)
            for (const auto& o : pML->GetObservations()) {
                KeyFrame* pKFi = o.first;
                if (pKFi->isBad()) continue;
                const Eigen::Vector3d lineObs = pKF->mvKeyLineFunctions[o.second];   // the reference reads the CURRENT key frame's line function and hangs both
                lo_kf.push_back(cur); lo_line.push_back(line_index[pML]);            // end-point edges on the current key frame (src/Optimizer.cc:2169-2201)
                for (int c = 0; c < 3; ++c) lo_l.push_back(lineObs(c));
                line_obs.push_back(LineObs{pKFi, pML});
            }
        for (MapPlane* pMP : lLocalMapPlanes)
            for (int fam = 0; fam < 3; ++fam) {                             // [0] EdgePlane, [1] EdgeVerticalPlane, [2] EdgeParallelPlane
                const std::map<KeyFrame*, size_t> observations = fam == 0 ? pMP->GetObservations() : fam == 1 ? pMP->GetVerObservations() : pMP->GetParObservations();
                for (const auto& o : observations) {
                    KeyFrame* k = o.first;
                    if (k->isBad() || k->mnId > maxKFid) continue;
                    const auto it = kf_index.find(k);
                    if (it == kf_index.end()) continue;                     // no vertex with that id in the reference's graph either (it would dereference NULL)
                    plo_kf[fam].push_back(it->second); plo_plane[fam].push_back(plane_index[pMP]);
                    for (int c = 0; c < 4; ++c) plo_meas[fam].push_back(k->mvPlaneCoefficients[o.second].at<float>(c));
                    plane_obs[fam].push_back(PlaneObs{k, pMP});
                }
            }

        pslam_lba_problem P;
        std::memset(&P, 0, sizeof P);
        P.n_kf = (int)kfs.size(); P.kf_Tcw = kf_Tcw.data(); P.kf_fixed = kf_fixed.data(); P.kf_K = kf_K.data();
        P.n_points = (int)pts.size(); P.pt_Xw = pt_Xw.data();
        P.n_pt_obs = (int)pt_obs.size(); P.pt_obs_kf = po_kf.data(); P.pt_obs_pt = po_pt.data(); P.pt_obs_uvr = po_uvr.data(); P.pt_obs_inv_sigma2 = po_is2.data();
        P.n_lines = (int)lines.size(); P.line_Xw = line_Xw.data();
        P.n_line_obs = (int)line_obs.size(); P.line_obs_kf = lo_kf.data(); P.line_obs_line = lo_line.data(); P.line_obs_l = lo_l.data();
        P.n_planes = (int)planes.size(); P.plane_Xw = plane_Xw.data();
        for (int fam = 0; fam < 3; ++fam) {
            P.n_plane_obs[fam] = (int)plane_obs[fam].size(); P.plane_obs_kf[fam] = plo_kf[fam].data(); P.plane_obs_plane[fam] = plo_plane[fam].data();
            P.plane_obs_meas[fam] = plo_meas[fam].data();
        }
        P.angle_info = Planar_SLAM::Config::Get<double>("Plane.AngleInfo"); P.dist_info = Planar_SLAM::Config::Get<double>("Plane.DistanceInfo");
        P.plane_chi = Planar_SLAM::Config::Get<double>("Plane.Chi"); P.vp_chi = Planar_SLAM::Config::Get<double>("Plane.VPChi");
        std::vector<float> r_T(kfs.size() * 16), r_pt(pts.size() * 3 + 3), r_pl(planes.size() * 4 + 4);
        std::vector<double> r_line(lines.size() * 6 + 6);
        std::vector<uint8_t> e_pt(pt_obs.size() + 1), e_line(line_obs.size() + 1), e_pl[3];
        pslam_lba_result R;
        std::memset(&R, 0, sizeof R);
        R.kf_Tcw = r_T.data(); R.pt_Xw = r_pt.data(); R.line_Xw = r_line.data(); R.plane_Xw = r_pl.data(); R.erase_pt = e_pt.data(); R.erase_line = e_line.data();
        for (int fam = 0; fam < 3; ++fam) { e_pl[fam].assign(plane_obs[fam].size() + 1, 0); R.erase_plane[fam] = e_pl[fam].data(); }
        pslam_ctx* c = context();
        if (pslam_local_bundle_adjustment(c, &P, &R) != PSLAM_OK) throw std::runtime_error(pslam_last_error(c));

        std::unique_lock<std::mutex> lock(pMap->mMutexMapUpdate);
        // vToErase lists monocular edges before stereo ones (:2462-2490); a (key frame, point) pair occurs once, so only the order of the cascades differs
        for (int pass = 0; pass < 2; ++pass)
            for (size_t j = 0; j < pt_obs.size(); ++j) {
                if (!e_pt[j] || (po_uvr[3 * j + 2] < 0) != (pass == 0)) continue;
                pt_obs[j].kf->EraseMapPointMatch(pt_obs[j].p); pt_obs[j].p->EraseObservation(pt_obs[j].kf);
            }
        for (size_t j = 0; j < line_obs.size(); ++j) if (e_line[j]) { line_obs[j].kf->EraseMapLineMatch(line_obs[j].l); line_obs[j].l->EraseObservation(line_obs[j].kf); }
        for (size_t j = 0; j < plane_obs[0].size(); ++j) if (e_pl[0][j]) { plane_obs[0][j].kf->EraseMapPlaneMatch(plane_obs[0][j].q); plane_obs[0][j].q->EraseObservation(plane_obs[0][j].kf); }
        for (size_t j = 0; j < plane_obs[1].size(); ++j) if (e_pl[1][j]) { plane_obs[1][j].kf->EraseMapVerticalPlaneMatch(plane_obs[1][j].q); plane_obs[1][j].q->EraseVerObservation(plane_obs[1][j].kf); }
        for (size_t j = 0; j < plane_obs[2].size(); ++j) if (e_pl[2][j]) { plane_obs[2][j].kf->EraseMapParallelPlaneMatch(plane_obs[2][j].q); plane_obs[2][j].q->EraseParObservation(plane_obs[2][j].kf); }
        for (KeyFrame* k : lLocalKeyFrames) {
            cv::Mat T(4, 4, CV_32F);
            const float* t = &r_T[(size_t)kf_index[k] * 16];
            for (int i = 0; i < 16; ++i) T.at<float>(i / 4, i % 4) = t[i];
            k->SetPose(T);
        }
        for (MapPoint* pMP : lLocalMapPoints) {
            cv::Mat X(3, 1, CV_32F);
            for (int c2 = 0; c2 < 3; ++c2) X.at<float>(c2) = r_pt[(size_t)pt_index[pMP] * 3 + c2];
            pMP->SetWorldPos(X);
            pMP->UpdateNormalAndDepth();
        }
        for (MapLine* pML : lLocalMapLines) {
            Planar_SLAM::Vector6d LinePos;
            for (int c2 = 0; c2 < 6; ++c2) LinePos(c2) = r_line[(size_t)line_index[pML] * 6 + c2];
            pML->SetWorldPos(LinePos);
            pML->UpdateAverageDir();
        }
        for (MapPlane* pMP : lLocalMapPlanes) {
            cv::Mat X(4, 1, CV_32F);
            for (int c2 = 0; c2 < 4; ++c2) X.at<float>(c2) = r_pl[(size_t)plane_index[pMP] * 4 + c2];
            pMP->SetWorldPos(X);
            pMP->UpdateCoefficientsAndPoints();
        }
    }

private:
    static int run(Frame* pFrame, bool translation_only) {
        pslam_pose_problem P;
        std::memset(&P, 0, sizeof P);
        P.fx = pFrame->fx; P.fy = pFrame->fy; P.cx = pFrame->cx; P.cy = pFrame->cy; P.bf = pFrame->mbf;
        const int N = pFrame->N;
        std::vector<float> Xw, obs, inv_sigma2;
        std::vector<int> pt_index;
        {
            std::unique_lock<std::mutex> lock(MapPoint::mGlobalMutex);
            for (int i = 0; i < N; ++i) {
                MapPoint* pMP = pFrame->mvpMapPoints[i];
                if (!pMP) continue;
                pFrame->mvbOutlier[i] = false;
                const cv::KeyPoint& kpUn = pFrame->mvKeysUn[i];
                const cv::Mat X = pMP->GetWorldPos();
                for (int k = 0; k < 3; ++k) Xw.push_back(X.at<float>(k));
                obs.push_back(kpUn.pt.x); obs.push_back(kpUn.pt.y); obs.push_back(pFrame->mvuRight[i] < 0 ? -1.0f : pFrame->mvuRight[i]);
                inv_sigma2.push_back(pFrame->mvInvLevelSigma2[kpUn.octave]);
                pt_index.push_back(i);
            }
        }
        const int NL = pFrame->NL;
        std::vector<double> line_Xw, line_obs;
        std::vector<int> line_index;
        {
            std::unique_lock<std::mutex> lock(MapLine::mGlobalMutex);
            for (int i = 0; i < NL; ++i) {
                MapLine* pML = pFrame->mvpMapLines[i];
                if (!pML) continue;
                pFrame->mvbLineOutlier[i] = false;
                for (int k = 0; k < 6; ++k) line_Xw.push_back(pML->mWorldPos(k));
                for (int k = 0; k < 3; ++k) line_obs.push_back(pFrame->mvKeyLineFunctions[i](k));
                line_index.push_back(i);
            }
        }
        const int M = pFrame->mnPlaneNum;
        std::vector<float> meas[3], mapc[3];
        std::vector<int> plane_index[3];
        {
            std::unique_lock<std::mutex> lock(MapPlane::mGlobalMutex);
            for (int fam = 0; fam < (translation_only ? 1 : 3); ++fam) {          // TranslationOptimization adds plane edges only (src/Optimizer.cc:3215-3220)
                std::vector<MapPlane*>& held = fam == 0 ? pFrame->mvpMapPlanes : fam == 1 ? pFrame->mvpParallelPlanes : pFrame->mvpVerticalPlanes;
                std::vector<bool>& flags = fam == 0 ? pFrame->mvbPlaneOutlier : fam == 1 ? pFrame->mvbParPlaneOutlier : pFrame->mvbVerPlaneOutlier;
                for (int i = 0; i < M; ++i) {
                    MapPlane* pMP = held[i];
                    if (!pMP) continue;
                    flags[i] = false;
                    const cv::Mat w = pMP->GetWorldPos();
                    for (int k = 0; k < 4; ++k) { meas[fam].push_back(pFrame->mvPlaneCoefficients[i].at<float>(k)); mapc[fam].push_back(w.at<float>(k)); }
                    plane_index[fam].push_back(i);
                }
            }
        }
        P.n_points = (int)pt_index.size(); P.Xw = Xw.data(); P.obs = obs.data(); P.inv_sigma2 = inv_sigma2.data();
        P.n_lines = (int)line_index.size(); P.line_Xw = line_Xw.data(); P.line_obs = line_obs.data();
        P.n_planes = (int)plane_index[0].size(); P.n_par = (int)plane_index[1].size(); P.n_ver = (int)plane_index[2].size();
        P.plane_meas = meas[0].data(); P.plane_map = mapc[0].data(); P.par_meas = meas[1].data(); P.par_map = mapc[1].data();
        P.ver_meas = meas[2].data(); P.ver_map = mapc[2].data();
        P.angle_info = Planar_SLAM::Config::Get<double>("Plane.AngleInfo"); P.dist_info = Planar_SLAM::Config::Get<double>("Plane.DistanceInfo");
        P.par_info = Planar_SLAM::Config::Get<double>("Plane.ParallelInfo"); P.ver_info = Planar_SLAM::Config::Get<double>("Plane.VerticalInfo");
        P.plane_chi = Planar_SLAM::Config::Get<double>("Plane.Chi"); P.vp_chi = Planar_SLAM::Config::Get<double>("Plane.VPChi");
        float T[16];
        for (int i = 0; i < 16; ++i) T[i] = pFrame->mTcw.at<float>(i / 4, i % 4);
        std::vector<uint8_t> o_pt(P.n_points + 1), o_line(P.n_lines + 1), o_pl(P.n_planes + 1), o_par(P.n_par + 1), o_ver(P.n_ver + 1);
        pslam_ctx* c = context();
        const int rc = translation_only ? pslam_translation_optimization(c, &P, T, o_pt.data(), o_line.data(), o_pl.data())
                                        : pslam_pose_optimization(c, &P, T, o_pt.data(), o_line.data(), o_pl.data(), o_par.data(), o_ver.data());
        if (rc < 0) throw std::runtime_error(pslam_last_error(c));
        const int n_initial = translation_only ? P.n_points : P.n_points + P.n_lines + P.n_planes + P.n_par + P.n_ver;
        if (n_initial < 3) return 0;                                              // the reference returns before touching the flags or the pose
        for (int k = 0; k < P.n_points; ++k) pFrame->mvbOutlier[pt_index[k]] = o_pt[k] != 0;
        for (int k = 0; k < P.n_lines; ++k) pFrame->mvbLineOutlier[line_index[k]] = o_line[k] != 0;
        for (int k = 0; k < P.n_planes; ++k) pFrame->mvbPlaneOutlier[plane_index[0][k]] = o_pl[k] != 0;
        for (int k = 0; k < P.n_par; ++k) pFrame->mvbParPlaneOutlier[plane_index[1][k]] = o_par[k] != 0;
        for (int k = 0; k < P.n_ver; ++k) pFrame->mvbVerPlaneOutlier[plane_index[2][k]] = o_ver[k] != 0;
        cv::Mat pose(4, 4, CV_32F);
        for (int i = 0; i < 16; ++i) pose.at<float>(i / 4, i % 4) = T[i];
        pFrame->SetPose(pose);
        return rc;
    }
};

// gathers the arrays of pslam_frame_view from a Frame (mvKeysUn, mvuRight, mDescriptors, mTcw, statics, scale tables)
struct FrameArrays {
    std::vector<pslam_keypoint> keys; std::vector<uint8_t> desc; pslam_frame_view v;
    explicit FrameArrays(const Frame& F) {
        const int n = F.N;
        keys.resize(n); desc.resize((size_t)n * 32);
        for (int i = 0; i < n; ++i) {
            const cv::KeyPoint& k = F.mvKeysUn[i];
            keys[i].x = k.pt.x; keys[i].y = k.pt.y; keys[i].size = k.size; keys[i].angle = k.angle; keys[i].response = k.response; keys[i].octave = k.octave;
            keys[i].class_id = k.class_id;
            std::memcpy(&desc[(size_t)i * 32], F.mDescriptors.ptr(i), 32);
        }
        std::memset(&v, 0, sizeof v);
        v.n = n; v.keys_un = keys.data(); v.u_right = F.mvuRight.data(); v.desc = desc.data();
        for (int i = 0; i < 16; ++i) v.Tcw[i] = F.mTcw.at<float>(i / 4, i % 4);
        v.fx = Frame::fx; v.fy = Frame::fy; v.cx = Frame::cx; v.cy = Frame::cy; v.bf = F.mbf;
        v.min_x = Frame::mnMinX; v.max_x = Frame::mnMaxX; v.min_y = Frame::mnMinY; v.max_y = Frame::mnMaxY;
        v.n_levels = F.mnScaleLevels; v.scale_factors = F.mvScaleFactors.data(); v.log_scale_factor = F.mfLogScaleFactor;
    }
};

struct MapArrays {       // pslam_map_points over a list of distinct MapPoint*
    std::vector<float> pos, normal, maxd, mind; std::vector<uint8_t> desc, skip, has_obs; pslam_map_points v;
    std::unordered_map<MapPoint*, int> index; std::vector<MapPoint*> pts;
    int add(MapPoint* p, bool skipped) {
        auto it = index.find(p);
        if (it != index.end()) return it->second;
        const int id = (int)pts.size();
        index[p] = id; pts.push_back(p);
        const cv::Mat X = p->GetWorldPos(), Nv = p->GetNormal(), D = p->GetDescriptor();
        for (int k = 0; k < 3; ++k) { pos.push_back(X.at<float>(k)); normal.push_back(Nv.empty() ? 0.f : Nv.at<float>(k)); }
        maxd.push_back(Access::max_distance(p)); mind.push_back(Access::min_distance(p));
        desc.resize(desc.size() + 32);
        if (!D.empty()) std::memcpy(&desc[desc.size() - 32], D.ptr(0), 32);
        skip.push_back(skipped ? 1 : 0); has_obs.push_back(p->Observations() > 0 ? 1 : 0);
        return id;
    }
    const pslam_map_points* view() {
        v.n = (int)pts.size(); v.pos = pos.data(); v.normal = normal.data(); v.max_distance = maxd.data(); v.min_distance = mind.data();
        v.desc = desc.data(); v.skip = skip.data(); v.has_obs = has_obs.data();
        return &v;
    }
};

class ORBmatcher {
public:
    ORBmatcher(float nnratio = 0.6, bool checkOri = true) : mfNNratio(nnratio), mbCheckOrientation(checkOri) {}

    // Search matches between Frame keypoints and projected MapPoints (the caller ran Frame::isInFrustum on them: mbTrackInView)
    int SearchByProjection(Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th = 3) {
        // the kernel walks the map arrays in index order = the order of vpMapPoints; points the frame already holds are appended (skipped: they only
        // take part as "this key point is taken", src/ORBmatcher.cc:83-85)
        MapArrays L;
        std::vector<int32_t> matches(F.N, -1);
        for (MapPoint* p : vpMapPoints) L.add(p, !p->mbTrackInView || p->isBad());
        for (int i = 0; i < F.N; ++i) matches[i] = F.mvpMapPoints[i] ? L.add(F.mvpMapPoints[i], true) : -1;
        FrameArrays A(F);
        pslam_ctx* c = context();
        const int n = pslam_search_by_projection_map(c, &A.v, L.view(), th, mfNNratio, matches.data(), nullptr);
        if (n < 0) throw std::runtime_error(pslam_last_error(c));
        for (int i = 0; i < F.N; ++i) F.mvpMapPoints[i] = matches[i] >= 0 ? L.pts[matches[i]] : static_cast<MapPoint*>(NULL);
        return n;
    }

    // Project MapPoints tracked in the last frame into the current frame and search matches (motion-model tracking)
    int SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono) {
        MapArrays M;
        std::vector<int32_t> last_mp(LastFrame.N, -1), matches(CurrentFrame.N, -1);
        std::vector<uint8_t> last_out(LastFrame.N, 0);
        std::vector<pslam_keypoint> last_keys(LastFrame.N);
        for (int i = 0; i < LastFrame.N; ++i) {
            if (LastFrame.mvpMapPoints[i]) last_mp[i] = M.add(LastFrame.mvpMapPoints[i], false);
            last_out[i] = LastFrame.mvbOutlier[i] ? 1 : 0;
            const cv::KeyPoint& k = LastFrame.mvKeys[i];
            last_keys[i].x = k.pt.x; last_keys[i].y = k.pt.y; last_keys[i].size = k.size; last_keys[i].angle = k.angle; last_keys[i].response = k.response;
            last_keys[i].octave = k.octave; last_keys[i].class_id = k.class_id;
        }
        for (int i = 0; i < CurrentFrame.N; ++i) if (CurrentFrame.mvpMapPoints[i]) matches[i] = M.add(CurrentFrame.mvpMapPoints[i], false);
        pslam_last_frame Lf;
        std::memset(&Lf, 0, sizeof Lf);
        Lf.n = LastFrame.N; Lf.keys = last_keys.data(); Lf.map_point = last_mp.data(); Lf.outlier = last_out.data();
        for (int i = 0; i < 16; ++i) Lf.Tcw[i] = LastFrame.mTcw.at<float>(i / 4, i % 4);
        FrameArrays A(CurrentFrame);
        pslam_ctx* c = context();
        const int n = pslam_search_by_projection_last(c, &A.v, &Lf, M.view(), th, bMono ? 1 : 0, mbCheckOrientation ? 1 : 0, matches.data());
        if (n < 0) throw std::runtime_error(pslam_last_error(c));
        for (int i = 0; i < CurrentFrame.N; ++i) CurrentFrame.mvpMapPoints[i] = matches[i] >= 0 ? M.pts[matches[i]] : static_cast<MapPoint*>(NULL);
        return n;
    }

    // Search matches between MapPoints in a KeyFrame and ORB in a Frame, brute force constrained to the same vocabulary node (relocalisation, tracking
    // with the reference key frame)
    int SearchByBoW(KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches) {
        const std::vector<MapPoint*> vpMapPointsKF = pKF->GetMapPointMatches();
        vpMapPointMatches = std::vector<MapPoint*>(F.N, static_cast<MapPoint*>(NULL));
        BowSide A(pKF->mDescriptors, pKF->mvKeysUn, pKF->mFeatVec, &vpMapPointsKF), B(F.mDescriptors, F.mvKeys, F.mFeatVec, nullptr);
        std::vector<int32_t> match((size_t)std::max(F.N, 1), -1);
        pslam_ctx* c = context();
        const int n = pslam_search_by_bow(c, A.n, A.desc.data(), A.angle.data(), A.has_mp.data(), (int)A.node_id.size(), A.node_id.data(), A.node_off.data(),
                                          A.node_feat.data(), B.n, B.desc.data(), B.angle.data(), (int)B.node_id.size(), B.node_id.data(), B.node_off.data(),
                                          B.node_feat.data(), mfNNratio, mbCheckOrientation ? 1 : 0, match.data());
        if (n < 0) throw std::runtime_error(pslam_last_error(c));
        for (int j = 0; j < F.N; ++j) if (match[j] >= 0) vpMapPointMatches[j] = vpMapPointsKF[match[j]];
        return n;
    }

    // Matching between two key frames for loop detection (LoopClosing::ComputeSim3): the consumer of the key-frame exchange
    int SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12) {
        const std::vector<MapPoint*> vpMapPoints1 = pKF1->GetMapPointMatches(), vpMapPoints2 = pKF2->GetMapPointMatches();
        vpMatches12 = std::vector<MapPoint*>(vpMapPoints1.size(), static_cast<MapPoint*>(NULL));
        BowSide A(pKF1->mDescriptors, pKF1->mvKeysUn, pKF1->mFeatVec, &vpMapPoints1), B(pKF2->mDescriptors, pKF2->mvKeysUn, pKF2->mFeatVec, &vpMapPoints2);
        std::vector<int32_t> match12((size_t)std::max(A.n, 1), -1);
        pslam_ctx* c = context();
        const int n = pslam_search_by_bow_kf(c, A.n, A.desc.data(), A.angle.data(), A.has_mp.data(), (int)A.node_id.size(), A.node_id.data(), A.node_off.data(),
                                             A.node_feat.data(), B.n, B.desc.data(), B.angle.data(), B.has_mp.data(), (int)B.node_id.size(), B.node_id.data(),
                                             B.node_off.data(), B.node_feat.data(), mfNNratio, mbCheckOrientation ? 1 : 0, match12.data());
        if (n < 0) throw std::runtime_error(pslam_last_error(c));
        for (int i = 0; i < A.n; ++i) if (match12[i] >= 0) vpMatches12[i] = vpMapPoints2[match12[i]];
        return n;
    }

private:
    struct BowSide {          // descriptors, key-point angles, map-point flags and the DBoW2 FeatureVector (std::map<NodeId, vector<unsigned>>) as CSR
        int n; std::vector<uint8_t> desc, has_mp; std::vector<float> angle; std::vector<int32_t> node_id, node_off, node_feat;
        BowSide(const cv::Mat& D, const std::vector<cv::KeyPoint>& keys, const DBoW2::FeatureVector& fv, const std::vector<MapPoint*>* mps) : n((int)keys.size()) {
            desc.resize((size_t)std::max(n, 1) * 32); has_mp.assign((size_t)std::max(n, 1), 1); angle.resize((size_t)std::max(n, 1));
            for (int i = 0; i < n; ++i) {
                std::memcpy(&desc[32 * (size_t)i], D.ptr(i), 32);
                angle[i] = keys[i].angle;
                if (mps) { MapPoint* p = (*mps)[i]; has_mp[i] = (p && !p->isBad()) ? 1 : 0; }
            }
            node_off.push_back(0);
            for (const auto& kv : fv) {
                node_id.push_back((int32_t)kv.first);
                for (unsigned f : kv.second) node_feat.push_back((int32_t)f);
                node_off.push_back((int32_t)node_feat.size());
            }
        }
    };
    float mfNNratio; bool mbCheckOrientation;
};

class LSDmatcher {
public:
    LSDmatcher(float nnratio = 0.6, bool checkOri = true) : mfNNratio(nnratio), mbCheckOrientation(checkOri) {}

    // Search matches between Frame key lines and projected MapLines (the caller ran Frame::isInFrustum(MapLine*) on them: mbTrackInView, mTrackProj*)
    int SearchByProjection(Frame& F, const std::vector<MapLine*>& vpMapLines, const float th = 3) {
        const int nf = F.NL, nm = (int)vpMapLines.size();
        std::vector<float> pt((size_t)std::max(nf, 1) * 2), angle((size_t)std::max(nf, 1)), view_cos((size_t)std::max(nm, 1)), proj((size_t)std::max(nm, 1) * 4);
        std::vector<int32_t> octave((size_t)std::max(nf, 1)), level((size_t)std::max(nm, 1)), assigned((size_t)std::max(nf, 1), -1);
        std::vector<uint8_t> desc((size_t)std::max(nf, 1) * 32), has_obs((size_t)std::max(nf, 1)), skip((size_t)std::max(nm, 1), 1), mdesc((size_t)std::max(nm, 1) * 32),
            m_has_obs((size_t)std::max(nm, 1));
        for (int i = 0; i < nf; ++i) {
            const auto& k = F.mvKeylinesUn[i];
            pt[2 * i] = k.pt.x; pt[2 * i + 1] = k.pt.y; angle[i] = k.angle; octave[i] = k.octave;
            std::memcpy(&desc[32 * (size_t)i], F.mLdesc.ptr(i), 32);
            has_obs[i] = (F.mvpMapLines[i] && F.mvpMapLines[i]->Observations() > 0) ? 1 : 0;
        }
        for (int j = 0; j < nm; ++j) {
            MapLine* p = vpMapLines[j];
            if (!p || p->isBad() || !p->mbTrackInView) continue;
            skip[j] = 0;
            level[j] = p->mnTrackScaleLevel; view_cos[j] = p->mTrackViewCos;
            proj[4 * j] = p->mTrackProjX1; proj[4 * j + 1] = p->mTrackProjY1; proj[4 * j + 2] = p->mTrackProjX2; proj[4 * j + 3] = p->mTrackProjY2;
            const cv::Mat d = p->GetDescriptor();
            std::memcpy(&mdesc[32 * (size_t)j], d.ptr(0), 32);
            m_has_obs[j] = p->Observations() > 0 ? 1 : 0;
        }
        pslam_ctx* c = context();
        const int n = pslam_line_search_by_projection(c, nf, pt.data(), angle.data(), octave.data(), desc.data(), has_obs.data(), F.mvScaleFactors.data(),
                                                      (int)F.mvScaleFactors.size(), nm, skip.data(), level.data(), view_cos.data(), proj.data(), mdesc.data(),
                                                      m_has_obs.data(), th, mfNNratio, assigned.data());
        if (n < 0) throw std::runtime_error(pslam_last_error(c));
        for (int i = 0; i < nf; ++i) if (assigned[i] >= 0) F.mvpMapLines[i] = vpMapLines[assigned[i]];
        return n;
    }

    // Matching of the key frame's map lines to the frame's key lines by LBD descriptor: cv::BFMatcher(NORM_HAMMING).knnMatch(k = 2) + the 1 / 1.5 ratio test
    // (include/LSDmatcher.h:21, src/LSDmatcher.cpp:242-279; the thresholds lineDescriptorMAD computes there are never read)
    int SearchByDescriptor(KeyFrame* pKF, Frame& currentF, std::vector<MapLine*>& vpMapLineMatches) {
        const std::vector<MapLine*> vpMapLinesKF = pKF->GetMapLineMatches();
        vpMapLineMatches = std::vector<MapLine*>(currentF.NL, static_cast<MapLine*>(NULL));
        const cv::Mat& ldesc1 = pKF->mLineDescriptors;
        const cv::Mat& ldesc2 = currentF.mLdesc;
        const int nq = ldesc1.rows, nt = ldesc2.rows;
        if (nq == 0 || nt < 2) return 0;                                  // (the reference indexes lmatches[i][1]: it needs two frame lines)
        std::vector<uint8_t> q((size_t)nq * 32), t((size_t)nt * 32);
        for (int i = 0; i < nq; ++i) std::memcpy(&q[32 * (size_t)i], ldesc1.ptr(i), 32);
        for (int i = 0; i < nt; ++i) std::memcpy(&t[32 * (size_t)i], ldesc2.ptr(i), 32);
        std::vector<int32_t> idx2((size_t)nq * 2), dist2((size_t)nq * 2);
        pslam_ctx* c = context();
        if (pslam_hamming_knn2(c, q.data(), nq, t.data(), nt, idx2.data(), dist2.data(), nullptr, nullptr) != PSLAM_OK) throw std::runtime_error(pslam_last_error(c));
        const float minRatio = 1.0f / 1.5f;
        int nmatches = 0;
        for (int i = 0; i < nq; ++i) {
            const double dist_12 = (float)dist2[2 * i] / (float)dist2[2 * i + 1];
            if (dist_12 < minRatio) {
                MapLine* mapLine = i < (int)vpMapLinesKF.size() ? vpMapLinesKF[i] : static_cast<MapLine*>(NULL);
                if (mapLine) { vpMapLineMatches[idx2[2 * i]] = mapLine; nmatches++; }
            }
        }
        return nmatches;
    }

private:
    float mfNNratio; bool mbCheckOrientation;
};

// The candidate searches of Planar_SLAM::KeyFrameDatabase.  The reference keeps only the inverted file; this class keeps the key frames in insertion order
// (the order every inverted-file list has) and mirrors their BowVectors into HBM when the set changed since the last query.  mnLoopQuery / mnLoopWords /
// mLoopScore (mnReloc*) of the key frames are written like the reference writes them, so code that reads them afterwards (LoopClosing) sees the same values.
class KeyFrameDatabase {
public:
    void add(KeyFrame* pKF) { std::unique_lock<std::mutex> lock(mMutex); mvKeyFrames.push_back(pKF); mbDirty = true; }
    void erase(KeyFrame* pKF) {
        std::unique_lock<std::mutex> lock(mMutex);
        auto it = std::find(mvKeyFrames.begin(), mvKeyFrames.end(), pKF);
        if (it != mvKeyFrames.end()) { mvKeyFrames.erase(it); mbDirty = true; }
    }
    void clear() { std::unique_lock<std::mutex> lock(mMutex); mvKeyFrames.clear(); mbDirty = true; }

    std::vector<KeyFrame*> DetectLoopCandidates(KeyFrame* pKF, float minScore) {
        std::unique_lock<std::mutex> lock(mMutex);
        const int n_kf = (int)mvKeyFrames.size();
        if (!n_kf) return std::vector<KeyFrame*>();
        pslam_ctx* c = context();
        upload(c);
        const std::set<KeyFrame*> spConnected = pKF->GetConnectedKeyFrames();
        std::vector<uint8_t> connected(n_kf);
        for (int k = 0; k < n_kf; ++k) connected[k] = spConnected.count(mvKeyFrames[k]) ? 1 : 0;
        Query q(pKF->mBowVec);
        std::vector<int32_t> covis = covisibility(), cand(n_kf), words(n_kf);
        const float unset = -2.f;
        std::vector<float> score(n_kf, unset);
        const int n = pslam_detect_loop_candidates(c, (int)q.word.size(), q.word.data(), q.val.data(), covis.data(), 10, connected.data(), minScore, cand.data(),
                                                   words.data(), score.data());
        if (n < 0) throw std::runtime_error(pslam_last_error(c));
        for (int k = 0; k < n_kf; ++k) {
            KeyFrame* kf = mvKeyFrames[k];
            if (words[k] > 0) { kf->mnLoopWords = words[k]; if (!connected[k]) kf->mnLoopQuery = pKF->mnId; }
            if (score[k] != unset) kf->mLoopScore = score[k];
        }
        std::vector<KeyFrame*> r(n);
        for (int i = 0; i < n; ++i) r[i] = mvKeyFrames[cand[i]];
        return r;
    }

    std::vector<KeyFrame*> DetectRelocalizationCandidates(Frame* F) {
        std::unique_lock<std::mutex> lock(mMutex);
        const int n_kf = (int)mvKeyFrames.size();
        if (!n_kf) return std::vector<KeyFrame*>();
        pslam_ctx* c = context();
        upload(c);
        Query q(F->mBowVec);
        std::vector<int32_t> covis = covisibility(), cand(n_kf), words(n_kf);
        std::vector<float> score(n_kf);
        for (int k = 0; k < n_kf; ++k) score[k] = mvKeyFrames[k]->mRelocScore;
        const int n = pslam_detect_relocalization_candidates(c, (int)q.word.size(), q.word.data(), q.val.data(), covis.data(), 10, score.data(), cand.data(), words.data());
        if (n < 0) throw std::runtime_error(pslam_last_error(c));
        for (int k = 0; k < n_kf; ++k) {
            KeyFrame* kf = mvKeyFrames[k];
            if (words[k] > 0) { kf->mnRelocWords = words[k]; kf->mnRelocQuery = F->mnId; }
            kf->mRelocScore = score[k];
        }
        std::vector<KeyFrame*> r(n);
        for (int i = 0; i < n; ++i) r[i] = mvKeyFrames[cand[i]];
        return r;
    }

private:
    struct Query {
        std::vector<int32_t> word; std::vector<double> val;
        explicit Query(const DBoW2::BowVector& v) { for (const auto& kv : v) { word.push_back((int32_t)kv.first); val.push_back(kv.second); } }
    };
    void upload(pslam_ctx* c) {
        if (!mbDirty && c == mpUploadedTo) return;
        std::vector<int32_t> off(1, 0), word; std::vector<double> val;
        for (KeyFrame* kf : mvKeyFrames) {
            for (const auto& kv : kf->mBowVec) { word.push_back((int32_t)kv.first); val.push_back(kv.second); }
            off.push_back((int32_t)word.size());
        }
        if (pslam_bow_database_set(c, (int)mvKeyFrames.size(), off.data(), word.data(), val.data()) != PSLAM_OK) throw std::runtime_error(pslam_last_error(c));
        mbDirty = false; mpUploadedTo = c;
    }
    std::vector<int32_t> covisibility() {          // KeyFrame::GetBestCovisibilityKeyFrames(10) as database indices; neighbours outside the database cannot
        std::unordered_map<KeyFrame*, int> index;  // carry this query's id and are left out, like the reference's mnLoopQuery / mnRelocQuery test skips them
        for (size_t k = 0; k < mvKeyFrames.size(); ++k) index[mvKeyFrames[k]] = (int)k;
        std::vector<int32_t> t(mvKeyFrames.size() * 10, -1);
        for (size_t k = 0; k < mvKeyFrames.size(); ++k) {
            int j = 0;
            for (KeyFrame* nb : mvKeyFrames[k]->GetBestCovisibilityKeyFrames(10)) {
                auto it = index.find(nb);
                if (it != index.end()) t[k * 10 + j++] = it->second;
            }
        }
        return t;
    }
    std::vector<KeyFrame*> mvKeyFrames; bool mbDirty = true; pslam_ctx* mpUploadedTo = nullptr; std::mutex mMutex;
};

class PlaneMatcher {
public:
    PlaneMatcher(float dTh = 0.1, float aTh = 0.86, float verTh = 0.08716, float parTh = 0.9962) : dTh(dTh), aTh(aTh), verTh(verTh), parTh(parTh) {}
    int SearchMapByCoefficients(Frame& pF, const std::vector<MapPlane*>& vpMapPlanes) {
        pF.mbNewPlane = false;
        const int nf = pF.mnPlaneNum, nm = (int)vpMapPlanes.size();
        std::vector<float> fc((size_t)nf * 4), mc((size_t)nm * 4), pts;
        std::vector<uint8_t> bad(nm);
        std::vector<int32_t> off(nm + 1, 0);
        for (int i = 0; i < nf; ++i) for (int k = 0; k < 4; ++k) fc[4 * i + k] = pF.mvPlaneCoefficients[i].at<float>(k);
        for (int j = 0; j < nm; ++j) {
            MapPlane* p = vpMapPlanes[j];
            bad[j] = p->isBad() ? 1 : 0;
            const cv::Mat w = p->GetWorldPos();
            for (int k = 0; k < 4; ++k) mc[4 * j + k] = w.at<float>(k);
            for (const auto& q : p->mvPlanePoints->points) { pts.push_back(q.x); pts.push_back(q.y); pts.push_back(q.z); }
            off[j + 1] = (int32_t)(pts.size() / 3);
        }
        float T[16];
        for (int i = 0; i < 16; ++i) T[i] = pF.mTcw.at<float>(i / 4, i % 4);
        std::vector<int32_t> m(nf + 1, -1), v(nf + 1, -1), pr(nf + 1, -1);
        pslam_ctx* c = context();
        const int n = pslam_plane_match(c, T, nf, fc.data(), nm, mc.data(), bad.data(), off.data(), pts.empty() ? fc.data() : pts.data(), dTh, aTh, verTh, parTh,
                                        m.data(), v.data(), pr.data());
        if (n < 0) throw std::runtime_error(pslam_last_error(c));
        for (int i = 0; i < nf; ++i) {                 // the reference only overwrites a slot when it finds a candidate
            if (m[i] >= 0) pF.mvpMapPlanes[i] = vpMapPlanes[m[i]];
            if (v[i] >= 0) pF.mvpVerticalPlanes[i] = vpMapPlanes[v[i]];
            if (pr[i] >= 0) pF.mvpParallelPlanes[i] = vpMapPlanes[pr[i]];
        }
        return n;
    }

private:
    float dTh, aTh, verTh, parTh;
};

// Planar_SLAM::ORBextractor with cv types: same constructor, getters and call operator (mask ignored like the reference, empty image -> silent return)
class ORBextractor {
public:
    ORBextractor(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST)
        : nfeatures(nfeatures), scaleFactor(scaleFactor), nlevels(nlevels), iniThFAST(iniThFAST), minThFAST(minThFAST) {}
    ~ORBextractor() { if (ctx) pslam_destroy(ctx); }
    ORBextractor(const ORBextractor&) = delete;
    ORBextractor& operator=(const ORBextractor&) = delete;

    void operator()(cv::InputArray _image, cv::InputArray /*mask*/, std::vector<cv::KeyPoint>& _keypoints, cv::OutputArray _descriptors) {
        if (_image.empty()) return;
        cv::Mat image = _image.getMat();
        if (image.type() != CV_8UC1) throw std::invalid_argument("ORBextractor: CV_8UC1 expected");            // the reference asserts (src/ORBextractor.cc:1050)
        if (!ctx || w != image.cols || h != image.rows) {
            if (ctx) pslam_destroy(ctx);
            pslam_config cfg;
            pslam_default_config(&cfg, image.cols, image.rows, 1);
            cfg.nfeatures = nfeatures; cfg.scale_factor = scaleFactor; cfg.nlevels = nlevels; cfg.ini_th_fast = iniThFAST; cfg.min_th_fast = minThFAST;
            if (pslam_create(&cfg, &ctx) != PSLAM_OK) { ctx = nullptr; throw std::runtime_error("pslam_create failed: no sm_90 GPU"); }
            w = image.cols; h = image.rows;
        }
        const int cap = pslam_orb_max_keypoints(ctx);
        std::vector<pslam_keypoint> kps(cap);
        std::vector<uint8_t> desc((size_t)cap * 32);
        int32_t n = 0;
        if (pslam_orb_extract(ctx, image.ptr(0), (int)image.step, kps.data(), desc.data(), cap, &n) != PSLAM_OK) throw std::runtime_error(pslam_last_error(ctx));
        _keypoints.resize(n);
        for (int i = 0; i < n; ++i) {
            cv::KeyPoint& k = _keypoints[i];
            k.pt.x = kps[i].x; k.pt.y = kps[i].y; k.size = kps[i].size; k.angle = kps[i].angle; k.response = kps[i].response; k.octave = kps[i].octave;
            k.class_id = kps[i].class_id;
        }
        if (n == 0) { _descriptors.release(); return; }
        _descriptors.create(n, 32, CV_8U);
        cv::Mat d = _descriptors.getMat();
        for (int i = 0; i < n; ++i) std::memcpy(d.ptr(i), &desc[(size_t)i * 32], 32);
    }
    int inline GetLevels() { return nlevels; }
    float inline GetScaleFactor() { return scaleFactor; }

private:
    int nfeatures; float scaleFactor; int nlevels, iniThFAST, minThFAST;
    pslam_ctx* ctx = nullptr; int w = 0, h = 0;
};

// Planar_SLAM::Frame's RGB-D constructor  Frame(imRGB, imGray, imDepth, timeStamp, extractor, voc, K, distCoef, bf, thDepth, depthMapFactor)  (include/Frame.h:57,
// src/Frame.cc:55-152) as a call that fills a default-constructed Frame (Frame::Frame(), src/Frame.cc:19): ExtractORB, ExtractLSD with isLineGood, ComputePlanes,
// ComputeStereoFromRGBD run in one pslam_frame_construct_batch_ex call; this class writes every member the constructor writes, the Frame statics included
// (fx ... invfy every frame, mnMinX ... mfGridElement*Inv on the first frame only, as mbInitialComputations says).
// Refused with std::invalid_argument: a non-zero distCoef[0] (there is no distortion model on this path: the reference would undistort mvKeysUn and the image
// bounds), a grey image other than CV_8UC1 / CV_8UC3 / CV_8UC4 (colour is converted as Tracking::GrabImageRGBD does, Camera.RGB = rgb), a depth image other than
// CV_16UC1, or a size other than the constructor's.  A capacity error throws std::runtime_error and leaves the Frame untouched.
// rand(): the reference's isLineGood draws from the process-wide libc stream, never seeded (srand(1)).  operator() continues one stream from frame to frame
// (seed, draws()); MapPlane's constructor and Tracking.cc:513 draw from the same stream in the reference, so a caller that runs them reports their draws with
// advance(n).  batch() starts every frame of the call at the stream position of the call's start and leaves draws() where it was (the replay convention:
// frame k's start would depend on the draws of frames 0 .. k-1, which are only known after they ran).
class FrameConstructor {
public:
    FrameConstructor(Planar_SLAM::ORBextractor* extractor, int nFeatures, float scaleFactor, int nLevels, int iniThFAST, int minThFAST, const cv::Mat& K,
                     const cv::Mat& distCoef, float bf, float thDepth, float depthMapFactor, float planeDistanceThreshold, int width, int height, bool rgb = true,
                     int max_batch = 1, int cap_plane_pts = 16384)
        : extractor(extractor), K(K.clone()), distCoef(distCoef.clone()), bf(bf), thDepth(thDepth), depthMapFactor(depthMapFactor),
          planeDistanceThreshold(planeDistanceThreshold), width(width), height(height), rgb(rgb), max_batch(max_batch), cap_plane_pts(cap_plane_pts),
          nLevels(nLevels), scaleFactor(scaleFactor) {
        if (K.type() != CV_32F || K.rows != 3 || K.cols != 3) throw std::invalid_argument("FrameConstructor: K must be a 3x3 CV_32F matrix");
        if (distCoef.empty() || distCoef.type() != CV_32F) throw std::invalid_argument("FrameConstructor: distCoef must be a CV_32F vector");
        if (distCoef.at<float>(0) != 0.0f) throw std::invalid_argument("FrameConstructor: distorted cameras (distCoef[0] != 0) are not supported");
        if (max_batch < 1 || cap_plane_pts < 1) throw std::invalid_argument("FrameConstructor: max_batch and cap_plane_pts must be positive");
        pslam_config cfg;
        pslam_default_config(&cfg, width, height, max_batch);
        cfg.nfeatures = nFeatures; cfg.scale_factor = scaleFactor; cfg.nlevels = nLevels; cfg.ini_th_fast = iniThFAST; cfg.min_th_fast = minThFAST;
        cfg.fx = K.at<float>(0, 0); cfg.fy = K.at<float>(1, 1); cfg.cx = K.at<float>(0, 2); cfg.cy = K.at<float>(1, 2); cfg.depth_scale = depthMapFactor;
        const int rc = pslam_create(&cfg, &ctx);
        if (rc != PSLAM_OK) { ctx = nullptr; throw std::runtime_error(rc == PSLAM_E_NO_DEVICE ? "pslam_create failed: no sm_90 GPU" : "pslam_create failed: bad settings"); }
        capk = pslam_orb_max_keypoints(ctx); maxp = pslam_peac_max_planes(ctx); nsn = pslam_surface_normals_count(ctx);
        scale.resize(nLevels); inv_scale.resize(nLevels); sigma2.resize(nLevels); inv_sigma2.resize(nLevels);
        pslam_orb_get_scale_tables(ctx, scale.data(), inv_scale.data(), sigma2.data(), inv_sigma2.data(), nullptr);
        const size_t nb = (size_t)max_batch, npx = (size_t)width * height;
        image = stage<uint8_t>(nb * npx * 4); depth = stage<uint16_t>(nb * npx); skip = stage<int32_t>(nb);
        o.keys = stage<pslam_keypoint>(nb * capk); o.desc = stage<uint8_t>(nb * capk * 32); o.n_keys = stage<int32_t>(nb);
        o.u_right = stage<float>(nb * capk); o.depth_kp = stage<float>(nb * capk);
        o.keylines = stage<pslam_keyline>(nb * kMaxLines); o.line_functions = stage<double>(nb * kMaxLines * 3); o.line_desc = stage<uint8_t>(nb * kMaxLines * 32);
        o.lines3d = stage<pslam_line3d>(nb * kMaxLines); o.n_lines = stage<int32_t>(nb); o.n_rand_drawn = stage<int32_t>(nb);
        o.n_planes = stage<int32_t>(nb); o.plane_src = stage<int32_t>(nb * maxp); o.plane_coef = stage<float>(nb * maxp * 4);
        o.plane_pt_off = stage<int32_t>(nb * (maxp + 1)); o.plane_pts = stage<float>(nb * cap_plane_pts * 3); o.cap_plane_pts = cap_plane_pts;
        o.surface_normals8 = stage<float>(nb * nsn * 8);
    }
    ~FrameConstructor() {
        for (void* p : pinned) pslam_host_free(p);
        if (ctx) pslam_destroy(ctx);
    }
    FrameConstructor(const FrameConstructor&) = delete;
    FrameConstructor& operator=(const FrameConstructor&) = delete;

    // Frame(imRGB, imGray, imDepth, timeStamp, extractor, voc, K, distCoef, bf, thDepth, depthMapFactor) on F, a default-constructed Frame
    void operator()(Frame& F, const cv::Mat& imRGB, const cv::Mat& imGray, const cv::Mat& imDepth, const double& timeStamp, Planar_SLAM::ORBVocabulary* voc) {
        (void)imRGB;                                   // ComputePlanes hands it to PlaneDetection::readColorImage, which nothing reads
        const int channels = check_image(imGray, imDepth, -1);
        put(0, imGray, imDepth);
        skip[0] = (int32_t)mDraws;
        run(1, channels, timeStamp);
        const int32_t drawn = o.n_rand_drawn[0];
        unpack(F, 0, timeStamp, voc);
        mDraws += drawn;
    }

    // The constructor for a sequence of frames, max_batch frames per call; frames[i] receives what operator() would put there with the rand() stream at
    // draws() for every frame (see the class comment).  mnId follows the order of `frames`.
    void batch(std::vector<Frame*>& frames, const std::vector<cv::Mat>& gray_or_colour, const std::vector<cv::Mat>& depth_images, const std::vector<double>& stamps,
               Planar_SLAM::ORBVocabulary* voc) {
        const size_t n = frames.size();
        if (gray_or_colour.size() != n || depth_images.size() != n || stamps.size() != n) throw std::invalid_argument("FrameConstructor::batch: list lengths differ");
        const int channels = n ? check_image(gray_or_colour[0], depth_images[0], -1) : 1;
        for (size_t i = 0; i < n; ++i) {
            if (!frames[i]) throw std::invalid_argument("FrameConstructor::batch: null Frame");
            check_image(gray_or_colour[i], depth_images[i], channels);
        }
        for (size_t b = 0; b < n; b += (size_t)max_batch) {
            const int nf = (int)std::min(n - b, (size_t)max_batch);
            for (int k = 0; k < nf; ++k) { put(k, gray_or_colour[b + k], depth_images[b + k]); skip[k] = (int32_t)mDraws; }
            run(nf, channels, stamps[b]);
            for (int k = 0; k < nf; ++k) unpack(*frames[b + k], k, stamps[b + k], voc);
        }
    }

    // libc rand() calls made by isLineGood since the stream started (srand(seed)); advance(n) accounts for n draws made elsewhere (a negative n rewinds)
    int64_t draws() const { return mDraws; }
    void advance(int64_t n) {
        if (mDraws + n < 0 || mDraws + n > INT32_MAX) throw std::invalid_argument("FrameConstructor::advance: stream position out of range");
        mDraws += n;
    }
    // host seconds spent in pslam_frame_construct_batch_ex and in filling Frames since construction
    double call_seconds() const { return mCallSeconds; }
    double unpack_seconds() const { return mUnpackSeconds; }
    double support_seconds() const { return mSupportSeconds; }      // the part of unpack_seconds() that rebuilds FrameLine::rndpts3d (compPt3dCov)

    static constexpr int kMaxLines = 40;         // ExtractLineSegment keeps the 40 strongest segments (src/LSDextractor.cpp:18-26)
    static constexpr uint32_t kSeed = 1;         // libc's stream before any srand

private:
    template <typename T>
    T* stage(size_t n) {
        void* p = nullptr;
        if (pslam_host_alloc(ctx, std::max(n, (size_t)1) * sizeof(T), &p) != PSLAM_OK) throw std::runtime_error(pslam_last_error(ctx));
        pinned.push_back(p);
        return static_cast<T*>(p);
    }
    int check_image(const cv::Mat& im, const cv::Mat& dep, int channels) const {
        const int t = im.type();
        if (t != CV_8UC1 && t != CV_MAKETYPE(CV_8U, 3) && t != CV_MAKETYPE(CV_8U, 4)) throw std::invalid_argument("FrameConstructor: imGray must be CV_8UC1, CV_8UC3 or CV_8UC4");
        if (dep.type() != CV_16UC1) throw std::invalid_argument("FrameConstructor: imDepth must be CV_16UC1");
        if (im.cols != width || im.rows != height || dep.cols != width || dep.rows != height) throw std::invalid_argument("FrameConstructor: image size differs from the constructor's");
        if (channels > 0 && im.channels() != channels) throw std::invalid_argument("FrameConstructor::batch: grey and colour images mixed in one call");
        return im.channels();
    }
    void put(int k, const cv::Mat& im, const cv::Mat& dep) {
        const size_t npx = (size_t)width * height, row = (size_t)width * im.channels();
        for (int y = 0; y < height; ++y) {
            std::memcpy(image + k * npx * im.channels() + y * row, im.ptr(y), row);
            std::memcpy(depth + k * npx + (size_t)y * width, dep.ptr(y), (size_t)width * 2);
        }
    }
    void run(int nf, int channels, double first_stamp) {
        const auto t0 = std::chrono::steady_clock::now();
        const int rc = pslam_frame_construct_batch_ex(ctx, image, channels, rgb ? 1 : 0, depth, nf, depthMapFactor, bf, planeDistanceThreshold, kMaxLines, kSeed, skip, &o);
        mCallSeconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        if (rc == PSLAM_OK) return;
        char what[96];
        std::snprintf(what, sizeof what, "FrameConstructor: frame at %.6f%s: ", first_stamp, nf > 1 ? " (or a later one of its batch)" : "");
        throw std::runtime_error(std::string(what) + pslam_last_error(ctx));
    }

    // the one unpacking routine of operator() and batch(): slot k of the staged outputs into F, member by member as src/Frame.cc:58-152 writes them
    void unpack(Frame& F, int k, double timeStamp, Planar_SLAM::ORBVocabulary* voc) {
        const auto t0 = std::chrono::steady_clock::now();
        F.mpORBvocabulary = voc; F.mpORBextractorLeft = extractor; F.mpORBextractorRight = static_cast<Planar_SLAM::ORBextractor*>(NULL);
        F.mTimeStamp = timeStamp; F.mK = K.clone(); F.mDistCoef = distCoef.clone(); F.mbf = bf; F.mThDepth = thDepth;
        F.mnId = Frame::nNextId++;
        F.mnScaleLevels = nLevels; F.mfScaleFactor = scaleFactor; F.mfLogScaleFactor = std::log(F.mfScaleFactor);
        F.mvScaleFactors = scale; F.mvInvScaleFactors = inv_scale; F.mvLevelSigma2 = sigma2; F.mvInvLevelSigma2 = inv_sigma2;
        set_intrinsics();
        F.dealWithLine = true;

        // ExtractLSD: ExtractLineSegment, then isLineGood (:189-267)
        const int NL = o.n_lines[k];
        const pslam_keyline* kl = o.keylines + (size_t)k * kMaxLines;
        const pslam_line3d* l3 = o.lines3d + (size_t)k * kMaxLines;
        F.mvKeylinesUn.resize(NL);
        F.mvKeyLineFunctions.resize(NL);
        F.mLdesc = NL ? cv::Mat(NL, 32, CV_8U) : cv::Mat();
        for (int i = 0; i < NL; ++i) {
            cv::line_descriptor::KeyLine& L = F.mvKeylinesUn[i];
            const pslam_keyline& s = kl[i];
            L.angle = s.angle; L.class_id = s.class_id; L.octave = s.octave; L.pt = cv::Point2f(s.pt_x, s.pt_y); L.response = s.response; L.size = s.size;
            L.startPointX = s.startPointX; L.startPointY = s.startPointY; L.endPointX = s.endPointX; L.endPointY = s.endPointY;
            L.sPointInOctaveX = s.sPointInOctaveX; L.sPointInOctaveY = s.sPointInOctaveY; L.ePointInOctaveX = s.ePointInOctaveX; L.ePointInOctaveY = s.ePointInOctaveY;
            L.lineLength = s.lineLength; L.numOfPixels = s.numOfPixels;
            const double* lf = o.line_functions + ((size_t)k * kMaxLines + i) * 3;
            F.mvKeyLineFunctions[i] = Eigen::Vector3d(lf[0], lf[1], lf[2]);
            std::memcpy(F.mLdesc.ptr(i), o.line_desc + ((size_t)k * kMaxLines + i) * 32, 32);
        }
        F.mvDepthLine = std::vector<float>(NL, -1.0f);
        F.mvLines3D = std::vector<Planar_SLAM::Vector6d>(NL, Eigen::Matrix<double, 6, 1>::Zero());
        const cv::Mat tmpK = (cv::Mat_<double>(3, 3) << Frame::fx, 0, Frame::cx, 0, Frame::fy, Frame::cy, 0, 0, 1);     // :84-86
        const uint16_t* raw = depth + (size_t)k * width * height;
        for (int i = 0; i < NL; ++i) {
            if (!l3[i].valid) continue;
            F.mvDepthLine[i] = l3[i].depth;
            F.mvLines3D[i] << l3[i].A[0], l3[i].A[1], l3[i].A[2], l3[i].B[0], l3[i].B[1], l3[i].B[2];
            FrameLine tempLine;
            tempLine.haveDepth = true;
            const auto ts = std::chrono::steady_clock::now();
            tempLine.rndpts3d = line_support(F.mvKeylinesUn[i], l3[i], raw, tmpK);
            mSupportSeconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - ts).count();
            tempLine.direction = cv::Point3d(l3[i].director[0], l3[i].director[1], l3[i].director[2]);
            tempLine.direct1 = cv::Point3d(); tempLine.direct2 = cv::Point3d();       // RandomLine3d leaves both unset (src/LineExtractor.cpp:1353-1354)
            tempLine.p = cv::Point2d(F.mvKeylinesUn[i].endPointX, F.mvKeylinesUn[i].endPointY);
            tempLine.q = cv::Point2d(F.mvKeylinesUn[i].startPointX, F.mvKeylinesUn[i].startPointY);
            F.mVF3DLines.push_back(tempLine);
        }

        // ComputePlanes (:647-753): the kept planes' voxel clouds and refitted coefficients, the surface normals of every other cell of the 3x3 grid
        const int np = o.n_planes[k];
        const int32_t* off = o.plane_pt_off + (size_t)k * (maxp + 1);
        const float* pts = o.plane_pts + (size_t)k * cap_plane_pts * 3;
        for (int q = 0; q < np; ++q) {
            Frame::PointCloud cloud;
            for (int j = off[q]; j < off[q + 1]; ++j) {
                Frame::PointT p;
                p.x = pts[3 * j]; p.y = pts[3 * j + 1]; p.z = pts[3 * j + 2];
                cloud.points.push_back(p);
            }
            cloud.width = (unsigned)cloud.points.size(); cloud.height = 1;     // VoxelGrid's output: one row
            F.mvPlanePoints.push_back(cloud);
            const float* c = o.plane_coef + ((size_t)k * maxp + q) * 4;
            F.mvPlaneCoefficients.push_back((cv::Mat_<float>(4, 1) << c[0], c[1], c[2], c[3]));
        }
        const float* sn = o.surface_normals8 + (size_t)k * nsn * 8;
        F.vSurfaceNormal.resize(nsn);
        for (int i = 0; i < nsn; ++i) {
            SurfaceNormal& s = F.vSurfaceNormal[i];
            const float* r = sn + 8 * (size_t)i;
            s.normal = cv::Point3f(r[0], r[1], r[2]); s.cameraPosition = cv::Point3f(r[3], r[4], r[5]); s.FramePosition = cv::Point2i((int)r[6], (int)r[7]);
        }

        // ExtractORB, then :99-152
        const int N = o.n_keys[k];
        F.N = N;
        F.NL = NL;
        F.mvKeys.resize(N);
        const pslam_keypoint* kp = o.keys + (size_t)k * capk;
        for (int i = 0; i < N; ++i) {
            cv::KeyPoint& q = F.mvKeys[i];
            q.pt.x = kp[i].x; q.pt.y = kp[i].y; q.size = kp[i].size; q.angle = kp[i].angle; q.response = kp[i].response; q.octave = kp[i].octave;
            q.class_id = kp[i].class_id;
        }
        if (N == 0) {                                 // :106-107 (ORBextractor releases the descriptors when it finds nothing)
            F.mDescriptors.release();
            mUnpackSeconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            return;
        }
        F.mDescriptors = cv::Mat(N, 32, CV_8U);
        std::memcpy(F.mDescriptors.ptr(0), o.desc + (size_t)k * capk * 32, (size_t)N * 32);
        F.mvKeysUn = F.mvKeys;                        // UndistortKeyPoints with distCoef[0] == 0 (:546-548)
        F.mvuRight.assign(o.u_right + (size_t)k * capk, o.u_right + (size_t)k * capk + N);
        F.mvDepth.assign(o.depth_kp + (size_t)k * capk, o.depth_kp + (size_t)k * capk + N);
        F.mvpMapPoints = std::vector<MapPoint*>(N, static_cast<MapPoint*>(NULL));
        F.mvpMapLines = std::vector<MapLine*>(NL, static_cast<MapLine*>(NULL));
        F.mvbOutlier = std::vector<bool>(N, false);
        F.mvbLineOutlier = std::vector<bool>(NL, false);
        if (Frame::mbInitialComputations) {           // ComputeImageBounds without distortion (:595-600), then :122-132
            Frame::mnMinX = 0.0f; Frame::mnMaxX = width; Frame::mnMinY = 0.0f; Frame::mnMaxY = height;
            Frame::mfGridElementWidthInv = static_cast<float>(FRAME_GRID_COLS) / static_cast<float>(Frame::mnMaxX - Frame::mnMinX);
            Frame::mfGridElementHeightInv = static_cast<float>(FRAME_GRID_ROWS) / static_cast<float>(Frame::mnMaxY - Frame::mnMinY);
            set_intrinsics();
            Frame::mbInitialComputations = false;
        }
        F.mb = F.mbf / Frame::fx;
        for (int i = 0; i < N; ++i) {                 // AssignFeaturesToGrid (:155-168)
            int gx, gy;
            if (F.PosInGrid(F.mvKeysUn[i], gx, gy)) F.mGrid[gx][gy].push_back(i);
        }
        F.mnPlaneNum = (int)F.mvPlanePoints.size();
        F.mvpMapPlanes = std::vector<MapPlane*>(F.mnPlaneNum, static_cast<MapPlane*>(nullptr));
        F.mvpParallelPlanes = std::vector<MapPlane*>(F.mnPlaneNum, static_cast<MapPlane*>(nullptr));
        F.mvpVerticalPlanes = std::vector<MapPlane*>(F.mnPlaneNum, static_cast<MapPlane*>(nullptr));
        F.mvPlanePointMatches = std::vector<std::vector<MapPoint*>>(F.mnPlaneNum);
        F.mvPlaneLineMatches = std::vector<std::vector<MapLine*>>(F.mnPlaneNum);
        F.mvbPlaneOutlier = std::vector<bool>(F.mnPlaneNum, false);
        F.mvbVerPlaneOutlier = std::vector<bool>(F.mnPlaneNum, false);
        F.mvbParPlaneOutlier = std::vector<bool>(F.mnPlaneNum, false);
        mUnpackSeconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    }

    void set_intrinsics() const {                     // :73-78 (and :125-130)
        Frame::fx = K.at<float>(0, 0); Frame::fy = K.at<float>(1, 1); Frame::cx = K.at<float>(0, 2); Frame::cy = K.at<float>(1, 2);
        Frame::invfx = 1.0f / Frame::fx; Frame::invfy = 1.0f / Frame::fy;
    }

    // FrameLine::rndpts3d of an accepted line: the samples of isLineGood (:193-232, the same expressions on the same types) that the fit kept (l.inliers, in
    // sampling order like RandomLine3d::pts), each with the reference's own compPt3dCov
    std::vector<RandomPoint3d> line_support(const cv::line_descriptor::KeyLine& kl, const pslam_line3d& l, const uint16_t* raw, const cv::Mat& tmpK) const {
        const double len = cv::norm(kl.getStartPoint() - kl.getEndPoint());
        const double numSmp = (double)std::min((int)len, 50);
        std::vector<cv::Point3d> pts3d;
        for (int j = 0; j <= numSmp; ++j) {
            const cv::Point2d pt = kl.getStartPoint() * (1 - j / numSmp) + kl.getEndPoint() * (j / numSmp);
            if (pt.x < 0 || pt.y < 0 || pt.x >= width || pt.y >= height) continue;
            int row, col;
            if ((std::floor(pt.x) == pt.x) && (std::floor(pt.y) == pt.y)) { col = std::max(int(pt.x - 1), 0); row = std::max(int(pt.y - 1), 0); }
            else { col = int(pt.x); row = int(pt.y); }
            const float d = (float)raw[(size_t)row * width + col] * depthMapFactor;     // imDepth.convertTo(depth, CV_32F, depthMapFactor) (:81-82)
            if (d <= 0.01) continue;
            cv::Point3d p;
            p.z = d;
            p.x = (col - Frame::cx) * p.z * Frame::invfx;
            p.y = (row - Frame::cy) * p.z * Frame::invfy;
            pts3d.push_back(p);
        }
        if ((int)pts3d.size() != l.n_points) throw std::logic_error("FrameConstructor: isLineGood samples differ from the device's");
        std::vector<RandomPoint3d> r;
        for (int j = 0; j < (int)pts3d.size() && j < 64; ++j)
            if (l.inliers >> j & 1) r.push_back(compPt3dCov(pts3d[j], tmpK, 1));
        if ((int)r.size() != l.n_inliers) throw std::logic_error("FrameConstructor: isLineGood support differs from the device's");
        return r;
    }

    Planar_SLAM::ORBextractor* extractor;
    cv::Mat K, distCoef;
    float bf, thDepth, depthMapFactor, planeDistanceThreshold;
    int width, height; bool rgb; int max_batch, cap_plane_pts, nLevels; float scaleFactor;
    pslam_ctx* ctx = nullptr;
    int capk = 0, maxp = 0, nsn = 0;
    std::vector<float> scale, inv_scale, sigma2, inv_sigma2;
    std::vector<void*> pinned;
    uint8_t* image = nullptr; uint16_t* depth = nullptr; int32_t* skip = nullptr;
    pslam_frame_outputs o{};
    int64_t mDraws = 0;
    double mCallSeconds = 0, mUnpackSeconds = 0, mSupportSeconds = 0;
};

}  // namespace ref
}  // namespace pslam_adapter
