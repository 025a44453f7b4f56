// Device-resident tracking chain (BASELINE.json config 3): a recorded RGB-D sequence is tracked against a POD map snapshot that lives in HBM,
// with no host round trip between the stages of a frame or between frames.
//
//   stage A, batched over the whole sequence (frames are independent):
//     ORBextractor::operator()            src/ORBextractor.cc:1043-1105      orb_run_dev (orb_pipeline.cu)
//     Frame::ComputeStereoFromRGBD        src/Frame.cc:603-621               pslam_compute_stereo_from_rgbd_batch_dev (mvKeysUn = mvKeys: no distortion)
//   stage B, frame after frame on the context's stream (frame t needs the pose of frame t - 1):
//     Tracking::TrackWithMotionModel      src/Tracking.cc:1739-1859          pose prediction mVelocity * mLastFrame.mTcw (:1754), SearchByProjection(cur, last,
//                                                                            th = 15, mono = false; :1764), PoseOptimization (:1782), outliers dropped (:1788-1800)
//     Tracking::TrackLocalMap             src/Tracking.cc:1954-2046          SearchLocalPoints: points already matched are skipped (:2290-2306), isInFrustum +
//                                                                            SearchByProjection(F, map, th = 3; :2321-2328), PoseOptimization (:1969), outliers dropped
//     velocity update                     src/Tracking.cc:270-278            mVelocity = mCurrentFrame.mTcw * LastTwc
//   Kernels reused as they are: k_search_grid / k_candidates_* / k_resolve_* (search_kernels.cuh) and k_pose_optimization (pose_kernels.cuh); new here: the
//   device-side problem packer (matches -> edge records in key-point order, the order Optimizer::PoseOptimization walks mvpMapPoints), the outlier sweep and the
//   4x4 float pose algebra (cv::Mat float products accumulate in double, like the oracle's search conventions).
// Not modelled (documented in DESIGN.md): UpdateLastFrame's temporary RGB-D points, key-frame insertion, lines / planes in this chain.
// The planar chain below (pslam_track_planar_sequence*) is PlanarSLAM's Track(): Manhattan rotation, TranslationWithMotionModel with the MatchORBPoints fallback,
// line and plane matching, TrackLocalMap with point / line / plane / parallel / vertical edges; see include/pslam_abi.h for its conventions.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "mapplane_body.cuh"
#include "pose_kernels.cuh"
#include "search_kernels.cuh"

namespace pslam {

int orb_run_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, pslam_keypoint* d_kps, uint8_t* d_desc, int cap, int32_t* d_n);

struct TrackBuffers {
    // map snapshot
    DevArray<uint8_t> map_blob; SearchMapDev M{}; DevArray<uint8_t> d_skip, d_skip0; int n_map = 0;
    // sequence products (stage A)
    DevArray<pslam_keypoint> d_kps; DevArray<uint8_t> d_desc; DevArray<int32_t> d_n; DevArray<float> d_ur, d_dz; int cap = 0;
    // chain state
    DevArray<float> d_T;                 // [3][16]: current pose, last pose, velocity
    DevArray<int32_t> d_matches;         // [2][cap]: current / last frame's map point per key point
    DevArray<uint8_t> d_zero;            // [cap] zeros (mvbOutlier of the last frame after the sweep)
    // search scratch
    DevArray<int32_t> d_cell_start, d_items, d_cand_n, d_scalar, d_hist_idx; DevArray<uint32_t> d_cand;
    DevArray<int8_t> d_hist_bin; DevArray<uint8_t> d_in_view;
    // pose problem
    DevArray<PoseHeaderDev> d_hdr; DevArray<float4> d_pa, d_pb; DevArray<uint8_t> d_level, d_flags;
    DevArray<PoseOutDev> d_out; DevArray<int32_t> d_kp_of_edge; DevArray<float> d_inv_sigma2;
    // per-frame outputs
    DevArray<float> d_T_all; DevArray<int32_t> d_stats;      // [n][16], [n][4] = matches / inliers after the motion-model stage and after the local-map stage
};

struct TrackCam { float fx, fy, cx, cy, bf; };

// ---- 4x4 float pose algebra in cv::Mat conventions (float storage, double accumulation) ----
__device__ __forceinline__ void mat4_mul(const float* A, const float* B, float* C) {
    float out[16];
    for (int r = 0; r < 4; ++r)
        for (int q = 0; q < 4; ++q) {
            double s = 0;
            for (int k = 0; k < 4; ++k) s += (double)A[4 * r + k] * (double)B[4 * k + q];
            out[4 * r + q] = (float)s;
        }
    for (int i = 0; i < 16; ++i) C[i] = out[i];
}
// T[0] = cur, T[1] = last, T[2] = velocity.  mode 0: start of a frame (t > 0): last <- cur; cur <- velocity * last (SetPose(mVelocity * mLastFrame.mTcw)).
// mode 1: end of a frame: velocity <- cur * LastTwc with LastTwc = [Rlw^T | -Rlw^T tlw] (Tracking.cc:270-278) unless ok is given and 0; record the pose.
__global__ void k_track_pose_algebra(float* __restrict__ T, int mode, int use_velocity, float* __restrict__ T_out, const int32_t* __restrict__ ok = nullptr) {
    if (threadIdx.x != 0) return;
    float* cur = T; float* last = T + 16; float* vel = T + 32;
    if (mode == 0) {
        for (int i = 0; i < 16; ++i) last[i] = cur[i];
        if (use_velocity) mat4_mul(vel, last, cur);
    } else {
        float Twc[16] = {0};
        for (int r = 0; r < 3; ++r) {
            for (int q = 0; q < 3; ++q) Twc[4 * r + q] = last[4 * q + r];                               // Rwc = Rcw^T
            double s = 0;
            for (int k = 0; k < 3; ++k) s += (double)(-last[4 * k + r]) * (double)last[4 * k + 3];      // Ow = -Rcw^T tcw
            Twc[4 * r + 3] = (float)s;
        }
        Twc[15] = 1.0f;
        if (!ok || *ok) mat4_mul(cur, Twc, vel);
        for (int i = 0; i < 16; ++i) T_out[i] = cur[i];
    }
}

// skip[m] = skip0[m] || (m is matched in the current frame)   (SearchLocalPoints: mnLastFrameSeen == current id, mbTrackInView = false, :2290-2306)
__global__ void k_track_skip(const uint8_t* __restrict__ skip0, uint8_t* __restrict__ skip, int n_map) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_map) skip[i] = skip0[i];
}
__global__ void k_track_skip_mark(uint8_t* __restrict__ skip, const int32_t* __restrict__ matches, const int32_t* __restrict__ n_kp, int cap) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < min(*n_kp, cap)) { const int m = matches[i]; if (m >= 0) skip[m] = 1; }
}
__global__ void k_track_fill(int32_t* __restrict__ a, int n, int32_t v) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = v;
}

// Optimizer::PoseOptimization's graph construction for the point edges (src/Optimizer.cc:593-690): key points in index order, matched ones become an edge -
// monocular when mvuRight[i] < 0, stereo otherwise; the record of pose_records.h (information = mvInvLevelSigma2[octave], float Huber deltas).
__global__ void __launch_bounds__(256) k_track_pack(const pslam_keypoint* __restrict__ keys, const float* __restrict__ u_right, const int32_t* __restrict__ n_kp, int cap,
                                                    const int32_t* __restrict__ matches, const float* __restrict__ map_pos, const float* __restrict__ inv_sigma2,
                                                    TrackCam K, const float* __restrict__ Tcw, PoseHeaderDev* __restrict__ hdr, float4* __restrict__ pt_a,
                                                    float4* __restrict__ pt_b, int32_t* __restrict__ kp_of_edge) {
    __shared__ int s_part[256];
    const int tid = threadIdx.x;
    const int n = min(*n_kp, cap);
    const int per = (n + 255) / 256, b0 = tid * per, b1 = min(n, b0 + per);
    int mine = 0;
    for (int i = b0; i < b1; ++i) mine += matches[i] >= 0;
    s_part[tid] = mine;
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int t = 0; t < 256; ++t) { const int v = s_part[t]; s_part[t] = run; run += v; }
        PoseHeaderDev H;
        memset(&H, 0, sizeof H);
        H.edge_off = 0; H.n_edges = run; H.n_pt = run; H.n_initial = run; H.mode = 0;
        H.fx = K.fx; H.fy = K.fy; H.cx = K.cx; H.cy = K.cy; H.bf = K.bf; H.plane_chi = 0; H.vp_chi = 0;
        for (int i = 0; i < 16; ++i) H.Tcw0[i] = Tcw[i];
        *hdr = H;
    }
    __syncthreads();
    int pos = s_part[tid];
    for (int i = b0; i < b1; ++i) {
        const int m = matches[i];
        if (m < 0) continue;
        const pslam_keypoint kp = keys[i];
        pose_point_record(map_pos + 3 * m, kp.x, kp.y, u_right[i], inv_sigma2[kp.octave], 0, Tcw, pt_a[pos], pt_b[pos]);
        kp_of_edge[pos] = i;
        ++pos;
    }
}

// After PoseOptimization: outliers lose their map point (mvpMapPoints[i] = NULL, :1791-1799 / :1978-1990), the optimised pose becomes the frame's pose;
// stats = {matches fed to the optimiser, inliers}.
__global__ void __launch_bounds__(256) k_track_sweep(const PoseHeaderDev* __restrict__ hdr, const PoseOutDev* __restrict__ out, const uint8_t* __restrict__ flags,
                                                     const int32_t* __restrict__ kp_of_edge, int32_t* __restrict__ matches, float* __restrict__ Tcw,
                                                     int32_t* __restrict__ stats) {
    const int n = hdr->n_pt;
    for (int j = threadIdx.x; j < n; j += 256) if (flags[j]) matches[kp_of_edge[j]] = -1;
    if (threadIdx.x == 0) {
        if (n >= 3) for (int i = 0; i < 16; ++i) Tcw[i] = out->Tcw[i];          // < 3 correspondences: PoseOptimization returns 0 and leaves mTcw alone (:985-986)
        stats[0] = n; stats[1] = out->n_inliers;
    }
}


// ============================================================================================================================================================
// Planar chain (pslam_track_planar_sequence*): PlanarSLAM's Tracking::Track() per frame.  Reuses the kernels above (pose algebra, skip kernels, grid and
// search kernels, k_pose_optimization) and the per-function kernels through their device launchers; new here: the compaction of the 3-D line directions for
// the Manhattan kernel, the rotation products, the MatchORBPoints / SearchByDescriptor assignments, the device packers (edge records of pose_records.h)
// and the two outlier sweeps.  st[0] = the local-map stage runs (the motion-model stage passed), st[1] = the frame tracked; kernels of a stage that is off
// do nothing.
#include "linefrustum_body.h"

struct PlanarTrackBuffers {
    // snapshot
    DevArray<uint8_t> map_blob; SearchMapDev M{}; DevArray<uint8_t> d_skip, d_skip0; int n_map = 0;
    const double *l_pos = nullptr, *l_normal = nullptr; const float *l_maxd = nullptr, *l_mind = nullptr; const uint8_t *l_desc = nullptr, *l_bad = nullptr,
        *l_has_obs = nullptr;
    DevArray<uint8_t> d_lskip; int n_lines = 0;
    const float* p_coef = nullptr; const uint8_t* p_bad = nullptr; const int32_t* p_off = nullptr; const float* p_pts = nullptr; int n_planes = 0;
    const uint8_t* ref_desc = nullptr; const int32_t* ref_map = nullptr; const int32_t* n_ref_dev = nullptr; int n_ref = 0;
    const float* R_cm = nullptr; bool ready = false;
    // sequence products and chain state
    DevArray<uint8_t> seq, state;
    // MapPlane::UpdateCoefficientsAndPoints after every frame (pslam_track_planar_set_map_plane_updates): map plane j's current cloud is
    // seg_pts[seg_begin[j] .. seg_end[j]) with seg_begin[j] = j * MP_SLOTS.  seg_live: the segments hold the current clouds; otherwise the next call in update
    // mode seeds them from the upload.  rows [rows_frames][3][maxp]: the associations of every frame of the last call in update mode.
    bool update_planes = false, seg_live = false; int max_plane_pts = 0; std::vector<int32_t> h_off;
    DevArray<float> seg_pts; DevArray<int32_t> seg_begin, seg_end, rows; int rows_frames = 0;
};

struct PlanarCam { float fx, fy, cx, cy, bf, min_x, max_x, min_y, max_y, log_scale_factor; };

// cv::Mat 3x3 float product (double accumulation); ta / tb: use the transpose of A / B
__device__ __forceinline__ void mat3_mul(const float* A, bool ta, const float* B, bool tb, float* C) {
    float out[9];
    for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 3; ++q) {
            double s = 0;
            for (int k = 0; k < 3; ++k) s += (double)(ta ? A[3 * k + r] : A[3 * r + k]) * (double)(tb ? B[3 * q + k] : B[3 * k + q]);
            out[3 * r + q] = (float)s;
        }
    for (int i = 0; i < 9; ++i) C[i] = out[i];
}

// start of a frame: the directions of the lines isLineGood accepted (mVF3DLines, in key-line order) for the Manhattan kernel; pred <- cur; the stage
// word, the counters, the frame's line matches and its plane associations (a new Frame's NULL entries) are reset.
__global__ void k_planar_begin(const pslam_line3d* __restrict__ l3d, const int32_t* __restrict__ n_lines, int max_lines, double* __restrict__ dirs,
                               int32_t* __restrict__ n_dirs, float* __restrict__ T, int32_t* __restrict__ st, int32_t* __restrict__ cnt,
                               int32_t* __restrict__ lmatch, int32_t* __restrict__ match3, int maxp) {
    const int tid = threadIdx.x;
    for (int i = tid; i < 3 * maxp; i += blockDim.x) match3[i] = -1;
    if (tid < 16) T[48 + tid] = T[tid];
    if (tid < max_lines) lmatch[tid] = -1;
    if (tid < 8) cnt[tid] = 0;
    if (tid == 0) {
        st[0] = 1; st[1] = 0; st[2] = 0; st[3] = 0;
        const int n = min(*n_lines, max_lines);
        int m = 0;
        for (int i = 0; i < n; ++i)
            if (l3d[i].valid) { for (int q = 0; q < 3; ++q) dirs[3 * m + q] = l3d[i].director[q]; ++m; }
        *n_dirs = m;
    }
}

// mode 0, after TrackManhattanFrame: mLastRcm = MF_can, R_cw = (Rotation_cm * MF_can^T)^T (:247-254).  mode 1, end of frame t >= 1: mLastRcm =
// (Rotation_cm^T * R_cw^T)^T from the final pose (:281-284).  Both record mLastRcm in R_out when given.
__global__ void k_planar_rotation(int mode, const pslam_manhattan_result* __restrict__ res, const float* __restrict__ R_cm, float* __restrict__ Rcm,
                                  float* __restrict__ Rcw, const float* __restrict__ T, float* __restrict__ R_out) {
    if (threadIdx.x != 0) return;
    if (mode == 0) {
        float M[9];
        for (int i = 0; i < 9; ++i) { M[i] = res->R[i]; Rcm[i] = M[i]; }
        float Rwc[9];
        mat3_mul(R_cm, false, M, true, Rwc);
        for (int r = 0; r < 3; ++r) for (int q = 0; q < 3; ++q) Rcw[3 * r + q] = Rwc[3 * q + r];
    } else if (mode == 1) {
        float Rcw_new[9], MT[9];
        for (int r = 0; r < 3; ++r) for (int q = 0; q < 3; ++q) Rcw_new[3 * r + q] = T[4 * r + q];
        mat3_mul(R_cm, true, Rcw_new, true, MT);
        for (int r = 0; r < 3; ++r) for (int q = 0; q < 3; ++q) Rcm[3 * r + q] = MT[3 * q + r];
    }
    if (R_out) for (int i = 0; i < 9; ++i) R_out[i] = Rcm[i];
}

// MatchORBPoints (src/ORBmatcher.cc:1332-1394) when SearchByProjection found fewer than 50 matches: fb_n = the descriptor counts of the current and the
// last frame, zero otherwise (the matcher launches then have nothing to do)
__global__ void k_planar_fallback_prep(const int32_t* __restrict__ nmatches, const int32_t* __restrict__ n_cur, const int32_t* __restrict__ n_last, int cap,
                                       int32_t* __restrict__ fb_n) {
    if (threadIdx.x != 0) return;
    const bool fb = *nmatches < 50;
    fb_n[0] = fb ? min(*n_cur, cap) : 0; fb_n[1] = fb ? min(*n_last, cap) : 0;
}
// ... and its assignment: the current frame's matches are cleared, good match i (query order) takes the last frame's map point of its train key point
// unless mvbOutlier[i] of the last frame is set (the reference indexes mvbOutlier with the match counter); nmatches = the number of good matches.
__global__ void __launch_bounds__(256) k_planar_fallback_apply(const int32_t* __restrict__ fb_n, const int32_t* __restrict__ idx2, const int32_t* __restrict__ good,
                                                               const int32_t* __restrict__ n_good, const int32_t* __restrict__ m_last,
                                                               const uint8_t* __restrict__ outl_last, int cap, int32_t* __restrict__ m_cur,
                                                               int32_t* __restrict__ nmatches, int32_t* __restrict__ stats) {
    if (fb_n[0] == 0 && *nmatches >= 50) return;
    const int tid = threadIdx.x;
    for (int i = tid; i < cap; i += 256) m_cur[i] = -1;
    __syncthreads();
    const int ng = *n_good, nl = fb_n[1];
    for (int k = tid; k < ng; k += 256) {
        const int q = good[k], mp = m_last[idx2[2 * q]];
        if (mp >= 0 && !(k < nl && outl_last[k])) m_cur[q] = mp;
    }
    if (tid == 0) { *nmatches = ng; stats[3] = 1; }
}

// LSDmatcher::SearchByDescriptor(mpReferenceKF, cur) (src/LSDmatcher.cpp:242-279) on k_hamming_knn2's output (query = the key frame's lines): rows in query
// order, ratio dist0 / dist1 < 1 / 1.5 (float quotient), the key line's map line goes to the matched frame line (later rows overwrite), every accepted row
// counts.  A row without a second neighbour (a frame with fewer than two lines) is skipped.
__global__ void k_planar_line_desc(int n_ref, const int32_t* __restrict__ idx2, const int32_t* __restrict__ dist2, const int32_t* __restrict__ ref_map,
                                   int32_t* __restrict__ lmatch, int32_t* __restrict__ cnt) {
    if (threadIdx.x != 0) return;
    int n = 0;
    for (int i = 0; i < n_ref; ++i) {
        if (idx2[2 * i] < 0 || idx2[2 * i + 1] < 0) continue;
        const float ratio = (float)dist2[2 * i] / (float)dist2[2 * i + 1];
        if (!((double)ratio < (double)(1.0f / 1.5f))) continue;
        const int m = ref_map[i];
        if (m >= 0) { lmatch[idx2[2 * i]] = m; ++n; }
    }
    *cnt = n;
}

// Frame::ComputePlaneWorldCoeff for PlaneMatcher::SearchMapByCoefficients: pi_w = Tcw^T pi_c (float storage, double accumulation); rows past the frame's
// planes, and all rows when the stage is off, are NaN (they fail every test of k_plane_assign).  This call's associations (found3, same layout as match3)
// start at -1, the count at 0.
__global__ void k_planar_plane_world(const int32_t* __restrict__ on, const float* __restrict__ T, const float* __restrict__ coef, const int32_t* __restrict__ n_kept,
                                     int maxp, float* __restrict__ pM, int32_t* __restrict__ found3, int32_t* __restrict__ cnt) {
    const int i = threadIdx.x + blockIdx.x * blockDim.x;
    if (i == 0) *cnt = 0;
    if (i >= maxp) return;
    found3[i] = -1; found3[maxp + i] = -1; found3[2 * maxp + i] = -1;
    const bool live = *on && i < *n_kept;
    for (int r = 0; r < 4; ++r) {
        double s = 0;
        for (int k = 0; k < 4; ++k) s += (double)T[4 * k + r] * (double)coef[4 * i + k];
        pM[4 * i + r] = live ? (float)s : __int_as_float(0x7fc00000);
    }
}

// SearchMapByCoefficients writes mvpMapPlanes / mvpParallelPlanes / mvpVerticalPlanes[i] only where it finds a candidate (src/PlaneMatcher.cpp:36-58): the
// local-map call keeps the motion-model stage's entries it does not replace
__global__ void k_planar_plane_merge(const int32_t* __restrict__ found3, int32_t* __restrict__ match3, int n) {
    const int i = threadIdx.x + blockIdx.x * blockDim.x;
    if (i < n && found3[i] >= 0) match3[i] = found3[i];
}

// Frame::isInFrustum(MapLine*, 0.6) at the pose in HBM (the shared body of k_lines_in_frustum); out_skip = the line search's skip flag (!mbTrackInView)
__global__ void k_planar_lines_in_frustum(PlanarCam K, const float* __restrict__ T, int n, const double* __restrict__ pos, const double* __restrict__ normal,
                                          const float* __restrict__ max_distance, const float* __restrict__ min_distance, const uint8_t* __restrict__ skip,
                                          float cos_limit, uint8_t* __restrict__ out_skip, float* __restrict__ proj, int32_t* __restrict__ level,
                                          float* __restrict__ view_cos) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    LfFrame F;
    for (int i = 0; i < 16; ++i) F.Tcw[i] = T[i];
    F.fx = K.fx; F.fy = K.fy; F.cx = K.cx; F.cy = K.cy; F.min_x = K.min_x; F.max_x = K.max_x; F.min_y = K.min_y; F.max_y = K.max_y;
    F.log_scale_factor = K.log_scale_factor;
    lf_camera_center(F);
    float p[4] = {0, 0, 0, 0}, vc = 0;
    int32_t lvl = 0;
    const bool ok = !skip[k] && lf_line_in_frustum(F, pos + 6 * (size_t)k, normal + 3 * (size_t)k, max_distance[k], min_distance[k], cos_limit, p, lvl, vc);
    out_skip[k] = ok ? 0 : 1; level[k] = lvl; view_cos[k] = vc;
    for (int q = 0; q < 4; ++q) proj[4 * (size_t)k + q] = p[q];
}

// before the local-map searches: a stage that is off skips every map point and map line; map lines held by the frame are skipped (SearchLocalLines step 1:
// mnLastFrameSeen); the frame-side arrays of the line search (pt, angle, octave; occupied = holds a map line with observations, padding rows occupied)
__global__ void k_planar_local_prep(const int32_t* __restrict__ st, uint8_t* __restrict__ skip, int n_map, uint8_t* __restrict__ lskip, int n_lines,
                                    const int32_t* __restrict__ lmatch, const uint8_t* __restrict__ l_has_obs, const pslam_keyline* __restrict__ kl,
                                    const int32_t* __restrict__ n_kl, int max_lines, float* __restrict__ f_pt, float* __restrict__ f_angle,
                                    int32_t* __restrict__ f_octave, uint8_t* __restrict__ f_occ) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool on = st[0] != 0;
    if (!on) { if (i < n_map) skip[i] = 1; if (i < n_lines) lskip[i] = 1; }
    if (i < max_lines) {
        const int nl = min(*n_kl, max_lines);
        const int m = i < nl ? lmatch[i] : -1;
        if (m >= 0) lskip[m] = 1;
        f_pt[2 * i] = i < nl ? kl[i].pt_x : 0.f; f_pt[2 * i + 1] = i < nl ? kl[i].pt_y : 0.f;
        f_angle[i] = i < nl ? kl[i].angle : 0.f; f_octave[i] = i < nl ? kl[i].octave : 0;
        f_occ[i] = i >= nl || (m >= 0 && l_has_obs[m]);
    }
}

struct PlanarEdges {          // what a packed problem came from, for the sweeps
    int32_t* kp_of_edge; int32_t* line_of_edge; int32_t* plane_of_edge;   // [cap], [max_lines], [3][maxp]
};

// Optimizer::TranslationOptimization (mode 1, after TranslationWithMotionModel's "< 10 matches" gate and the copy of R_cw into mTcw) or PoseOptimization
// (mode 0) problem of the frame: points in key-point order, lines in key-line order (two records each), matched / parallel / vertical planes in plane
// order; records of pose_records.h.  In mode 0 the line matches of SearchLocalLines (assigned) are merged into the frame's first.  A stage that is off (or
// fails the gate) packs an empty problem.
__global__ void __launch_bounds__(256) k_planar_pack(int mode, int32_t* __restrict__ st, const int32_t* __restrict__ cnt3, const float* __restrict__ Rcw,
                                                     float* __restrict__ T, const pslam_keypoint* __restrict__ keys, const float* __restrict__ u_right,
                                                     const int32_t* __restrict__ n_kp, int cap, const int32_t* __restrict__ matches,
                                                     const float* __restrict__ map_pos, const float* __restrict__ inv_sigma2, const double* __restrict__ lf,
                                                     const int32_t* __restrict__ n_kl, int max_lines, int32_t* __restrict__ lmatch,
                                                     const int32_t* __restrict__ assigned, const double* __restrict__ l_pos, const float* __restrict__ coef,
                                                     const int32_t* __restrict__ n_kept, int maxp, const int32_t* __restrict__ match3,
                                                     const float* __restrict__ p_coef, TrackCam K, PoseEdgeConsts EK, double plane_chi, double vp_chi,
                                                     PoseHeaderDev* __restrict__ hdr, float4* __restrict__ pt_a, float4* __restrict__ pt_b,
                                                     PoseEdgeDev* __restrict__ wide, PlanarEdges E, int32_t* __restrict__ stats) {
    __shared__ int s_part[256];
    __shared__ int s_on;
    const int tid = threadIdx.x;
    if (tid == 0) {
        int on = st[0];
        if (on && mode == 1) {                                    // :1776-1782
            const int initial = cnt3[0] + cnt3[1] + cnt3[2];
            stats[0] = cnt3[0]; stats[1] = cnt3[1]; stats[2] = cnt3[2];
            if (initial < 10) { on = 0; st[0] = 0; }
            else for (int r = 0; r < 3; ++r) for (int q = 0; q < 3; ++q) T[4 * r + q] = Rcw[3 * r + q];
        }
        s_on = on;
    }
    __syncthreads();
    const int n = s_on ? min(*n_kp, cap) : 0;
    const int per = (n + 255) / 256, b0 = tid * per, b1 = min(n, b0 + per);
    int mine = 0;
    for (int i = b0; i < b1; ++i) mine += matches[i] >= 0;
    s_part[tid] = mine;
    __syncthreads();
    if (tid == 0) { int run = 0; for (int t = 0; t < 256; ++t) { const int v = s_part[t]; s_part[t] = run; run += v; } }
    __syncthreads();
    int pos = s_part[tid];
    for (int i = b0; i < b1; ++i) {
        const int m = matches[i];
        if (m < 0) continue;
        const pslam_keypoint kp = keys[i];
        pose_point_record(map_pos + 3 * m, kp.x, kp.y, u_right[i], inv_sigma2[kp.octave], mode, T, pt_a[pos], pt_b[pos]);
        E.kp_of_edge[pos] = i;
        ++pos;
    }
    __syncthreads();
    if (tid != 0) return;
    int np = 0;
    for (int i = 255 * per; i < n; ++i) np += matches[i] >= 0;   // the last thread's share
    const int n_points = s_part[255] + np;
    int w = 0, nl = 0, npl[3] = {0, 0, 0};
    if (s_on) {
        const int nkl = min(*n_kl, max_lines);
        for (int i = 0; i < nkl; ++i) {
            if (mode == 0 && assigned[i] >= 0) lmatch[i] = assigned[i];
            const int m = lmatch[i];
            if (m < 0) continue;
            for (int s = 0; s < 2; ++s) pose_line_record(l_pos + 6 * (size_t)m, lf + 3 * i, nl, s, mode, T, wide[w++]);
            E.line_of_edge[nl++] = i;
        }
        const int nk = min(*n_kept, maxp);
        const int kinds[3] = {mode == 0 ? PK_PLANE : PK_PLANE_T, PK_PAR, PK_VER};
        for (int f = 0; f < (mode == 0 ? 3 : (n_points >= 3 ? 1 : 0)); ++f)     // TranslationOptimization: matched planes only, none below 3 points
            for (int i = 0; i < nk; ++i) {
                const int j = match3[f * maxp + i];                   // match3 = [mvpMapPlanes | mvpParallelPlanes | mvpVerticalPlanes], the families' order
                if (j < 0) continue;
                pose_plane_record(kinds[f], npl[f], p_coef + 4 * j, coef + 4 * i, T, EK, wide[w++]);
                E.plane_of_edge[f * maxp + npl[f]++] = i;
            }
    }
    PoseHeaderDev H;
    memset(&H, 0, sizeof H);
    H.n_pt = n_points; H.n_line = nl; H.n_plane = npl[0]; H.n_par = npl[1]; H.n_ver = npl[2];
    H.n_edges = n_points + w;
    H.n_initial = mode == 0 ? n_points + nl + npl[0] + npl[1] + npl[2] : n_points;
    H.mode = mode;
    H.fx = K.fx; H.fy = K.fy; H.cx = K.cx; H.cy = K.cy; H.bf = K.bf; H.plane_chi = plane_chi; H.vp_chi = vp_chi;
    for (int i = 0; i < 16; ++i) H.Tcw0[i] = T[i];
    *hdr = H;
}

// the outlier sweeps.  mode 1 (TranslationWithMotionModel :1795-1855): outlier points / lines lose their match and are skipped by the local-map searches
// (mnLastFrameSeen); nmatchesMap / line / plane inliers; fail below 3 (pose back to the prediction).  mode 0 (TrackLocalMap :1971-2044): outlier points
// keep their match with mvbOutlier set (the next frame's last-frame flags); mnMatchesInliers; fail below 7; a tracked frame drops the matches of points
// without observations ("Clean VO matches", :320-327).  Mode 0 also drops the parallel / vertical associations PoseOptimization flagged
// (mvpParallelPlanes / mvpVerticalPlanes[i] = NULL, :2018-2030); matched planes keep theirs (the reference's nulling is commented out).  Mode 1 has no
// parallel / vertical edges, so its identical loop (:1828-1840) has nothing to drop.
__global__ void __launch_bounds__(256) k_planar_sweep(int mode, int32_t* __restrict__ st, const PoseHeaderDev* __restrict__ hdr, const PoseOutDev* __restrict__ out,
                                                      const uint8_t* __restrict__ f_pt, const uint8_t* __restrict__ f_line, const uint8_t* __restrict__ f_plane,
                                                      PlanarEdges E, int32_t* __restrict__ matches, uint8_t* __restrict__ outl, uint8_t* __restrict__ skip,
                                                      const uint8_t* __restrict__ has_obs, int32_t* __restrict__ lmatch, uint8_t* __restrict__ lskip,
                                                      const uint8_t* __restrict__ l_has_obs, const int32_t* __restrict__ n_kept, int maxp,
                                                      int32_t* __restrict__ match3, float* __restrict__ T, int32_t* __restrict__ stats) {
    __shared__ int s_cnt[3];
    const int tid = threadIdx.x;
    if (!st[0]) {
        if (tid == 0) { if (mode == 1) { stats[4] = 0; stats[5] = 0; } else { st[1] = 0; } }
        return;
    }
    const PoseHeaderDev H = *hdr;
    if (tid < 3) s_cnt[tid] = 0;
    __syncthreads();
    int c_pt = 0;
    for (int j = tid; j < H.n_pt; j += 256) {
        const int i = E.kp_of_edge[j], m = matches[i];
        if (f_pt[j]) {
            if (mode == 1) { matches[i] = -1; skip[m] = 1; } else outl[i] = 1;
        } else if (has_obs[m]) ++c_pt;
    }
    atomicAdd(&s_cnt[0], c_pt);
    if (tid == 0) {
        int c_l = 0, c_p = 0;
        for (int j = 0; j < H.n_line; ++j) {
            const int i = E.line_of_edge[j], m = lmatch[i];
            if (f_line[j]) { if (mode == 1) { lmatch[i] = -1; lskip[m] = 1; } }
            else if (l_has_obs[m]) ++c_l;
        }
        // matched planes count unless flagged; a plane without an edge (TranslationOptimization with < 3 points) keeps mvbPlaneOutlier = false
        const int nk = min(*n_kept, maxp);
        int e = 0;
        for (int i = 0; i < nk; ++i) {
            if (match3[i] < 0) continue;
            const bool has_edge = e < H.n_plane && E.plane_of_edge[e] == i;
            if (!(has_edge && f_plane[e])) ++c_p;
            if (has_edge) ++e;
        }
        s_cnt[1] = c_l; s_cnt[2] = c_p;
    }
    if (mode == 0)             // after the plane count above read match3; edge e of family f came from frame plane plane_of_edge[f * maxp + e]
        for (int f = 1; f < 3; ++f) {
            const int n_f = f == 1 ? H.n_par : H.n_ver;
            for (int e = tid; e < n_f; e += 256)
                if (f_plane[f * maxp + e]) match3[f * maxp + E.plane_of_edge[f * maxp + e]] = -1;
        }
    __syncthreads();
    if (tid != 0) return;
    const int n_map_in = s_cnt[0], total = s_cnt[0] + s_cnt[1] + s_cnt[2];
    if (H.n_initial >= 3) for (int i = 0; i < 16; ++i) T[i] = out->Tcw[i];
    if (mode == 1) {
        const bool ok = !(n_map_in < 3 || total < 3);
        if (!ok) { for (int i = 0; i < 16; ++i) T[i] = T[48 + i]; st[0] = 0; }
        stats[4] = n_map_in; stats[5] = ok;
    } else {
        const bool ok = total >= 7;
        st[1] = ok;
        stats[6] = H.n_pt; stats[7] = H.n_line; stats[8] = H.n_plane; stats[9] = H.n_par; stats[10] = H.n_ver; stats[11] = total; stats[12] = ok;
    }
}
// the three match counts of TranslationWithMotionModel's gate in one place: cnt = {nmatches, line matches, plane matches}
__global__ void k_planar_counts(const int32_t* __restrict__ nmatches, int32_t* __restrict__ cnt) {
    if (threadIdx.x == 0) cnt[0] = *nmatches;
}
// "Clean VO matches" of a tracked frame (after the local-map sweep)
__global__ void k_planar_clean(const int32_t* __restrict__ st, int32_t* __restrict__ matches, uint8_t* __restrict__ outl, const uint8_t* __restrict__ has_obs,
                               const int32_t* __restrict__ n_kp, int cap) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!st[1] || i >= min(*n_kp, cap)) return;
    const int m = matches[i];
    if (m >= 0 && !has_obs[m]) { matches[i] = -1; outl[i] = 0; }
}

// update mode, before the first frame: map plane j's uploaded cloud into its segment
__global__ void __launch_bounds__(256) k_planar_seed_planes(const int32_t* __restrict__ p_off, const float* __restrict__ p_pts, float* __restrict__ seg_pts,
                                                            int32_t* __restrict__ seg_begin, int32_t* __restrict__ seg_end) {
    const int j = blockIdx.x, b = p_off[j], n = p_off[j + 1] - b;
    for (int k = threadIdx.x; k < 3 * n; k += 256) seg_pts[(size_t)j * MP_SLOTS * 3 + k] = p_pts[(size_t)b * 3 + k];
    if (threadIdx.x == 0) { seg_begin[j] = j * MP_SLOTS; seg_end[j] = j * MP_SLOTS + n; }
}

// MapPlane::UpdateCoefficientsAndPoints(mCurrentFrame, i) for every frame plane i with mvpMapPlanes[i] (src/Tracking.cc:296-304), after every frame, tracked
// or not, at the frame's final pose.  CTA j = map plane j walks the frame planes in ascending i; each i with match3[i] == j rebuilds the cloud from the frame
// cloud i at T = toSE3Quat(mTcw).inverse() and the current cloud at the identity, one merge after the other as the reference's loop does.  A merge that
// does not fit (more than MP_SLOTS voxels, or a point beyond the key range) leaves the cloud as it was and sets bit 0 of the frame's status.  CTA 0 also
// records the frame's associations (row [3][maxp], the match3 layout).  Segments are read and written in place: no restrict on seg_pts.
__global__ void __launch_bounds__(MP_THREADS, 1) k_planar_map_plane_update(const float* __restrict__ T, const int32_t* __restrict__ match3,
                                                                          const int32_t* __restrict__ n_kept, int maxp, const int32_t* __restrict__ f_off,
                                                                          const float* __restrict__ f_pts, int n_planes, float* seg_pts,
                                                                          const int32_t* __restrict__ seg_begin, int32_t* seg_end, int32_t* __restrict__ row,
                                                                          int32_t* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char mp_smem[];
    __shared__ int s_flag, s_n;
    __shared__ double s_T[12], s_I[12];
    const int j = blockIdx.x, tid = threadIdx.x;
    if (j == 0) for (int k = tid; k < 3 * maxp; k += MP_THREADS) row[k] = match3[k];
    if (j >= n_planes) return;
    const int nk = min(*n_kept, maxp);
    bool any = false;
    for (int i = 0; i < nk; ++i) any |= match3[i] == j;
    if (!any) return;
    if (tid == 0) mp_pose_inverse(T, s_T);
    if (tid < 12) s_I[tid] = tid % 5 == 0 ? 1.0 : 0.0;          // the identity's rows
    const MpTable S = mp_table(mp_smem, &s_flag, &s_n);
    const int b = seg_begin[j];
    for (int i = 0; i < nk; ++i) {
        if (match3[i] != j) continue;
        mp_clear(S, tid);
        __syncthreads();                                         // also publishes s_T, s_I and the previous merge's cloud and seg_end
        mp_add(S, tid, f_pts, f_off[i], f_off[i + 1], s_T);
        mp_add(S, tid, seg_pts, b, seg_end[j], s_I);
        mp_sort(S, tid);
        const int N = s_n;
        if (s_flag || N > MP_SLOTS) {
            if (tid == 0) atomicOr(status, 1);
        } else {
            mp_emit(S, tid, MP_SLOTS, seg_pts + (size_t)b * 3);
            if (tid == 0) seg_end[j] = b + N;
        }
        __syncthreads();
    }
}

void track_free(pslam_ctx* c) {
    delete c->track;
    c->track = nullptr;
    delete c->ptrack;
    c->ptrack = nullptr;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_track_set_map(pslam_ctx* c, const pslam_map_points* m) {
    if (!c) return PSLAM_E_INVALID;
    if (!m || m->n < 1 || !m->pos || !m->normal || !m->max_distance || !m->min_distance || !m->desc || !m->skip || !m->has_obs)
        return set_error(c, PSLAM_E_INVALID, "null or empty map snapshot");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->track) c->track = new TrackBuffers();
    TrackBuffers& B = *c->track;
    const size_t nm = (size_t)m->n;
    Slab s;
    const auto pos = s.add<float>(nm * 3), normal = s.add<float>(nm * 3), max_d = s.add<float>(nm), min_d = s.add<float>(nm);
    const auto desc = s.add<uint8_t>(nm * 32), has_obs = s.add<uint8_t>(nm);
    int rc;
    B.n_map = 0;                // no snapshot until this one is uploaded
    if ((rc = s.alloc(c, B.map_blob)) || (rc = B.d_skip.reserve(c, nm)) || (rc = B.d_skip0.reserve(c, nm))) return rc;
    cudaStream_t st = c->stream;
    s.up(pos, m->pos, st); s.up(normal, m->normal, st); s.up(max_d, m->max_distance, st); s.up(min_d, m->min_distance, st);
    s.up(desc, m->desc, st); s.up(has_obs, m->has_obs, st);
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_skip0, m->skip, nm, cudaMemcpyHostToDevice, st));
    B.M.n = m->n; B.n_map = m->n;
    B.M.pos = s[pos]; B.M.normal = s[normal]; B.M.max_distance = s[max_d]; B.M.min_distance = s[min_d]; B.M.desc = s[desc]; B.M.has_obs = s[has_obs];
    B.M.skip = B.d_skip;
    return s.sync(c, st);       // the caller's arrays may be pageable
}

int pslam_track_sequence_dev(pslam_ctx* c, const uint8_t* d_gray, const uint16_t* d_depth, int nframes, const pslam_track_params* prm, const float* Tcw0,
                             float* Tcw_out, int32_t* stats_out) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_gray || !d_depth || !prm || !Tcw0 || !Tcw_out || nframes < 1 || nframes > c->cfg.max_batch) return set_error(c, PSLAM_E_INVALID, "bad tracking arguments");
    if (!c->track || c->track->n_map < 1) return set_error(c, PSLAM_E_INVALID, "no map snapshot (pslam_track_set_map)");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    TrackBuffers& B = *c->track;
    const OrbGeom& g = c->geom;
    const int cap = std::min(pslam_orb_max_keypoints(c), SEARCH_MAX_KP);
    cudaStream_t st = c->stream;
    const size_t nf = (size_t)nframes;
    int rc;
    if ((rc = B.d_kps.reserve(c, nf * cap)) || (rc = B.d_desc.reserve(c, nf * cap * 32)) || (rc = B.d_n.reserve(c, nf)) || (rc = B.d_ur.reserve(c, nf * cap)) ||
        (rc = B.d_dz.reserve(c, nf * cap)) || (rc = B.d_T_all.reserve(c, nf * 16)) || (rc = B.d_stats.reserve(c, nf * 4)))
        return rc;
    if (cap != B.cap) {
        if ((rc = B.d_T.reserve(c, 3 * 16)) || (rc = B.d_matches.reserve(c, (size_t)2 * cap)) || (rc = B.d_zero.reserve(c, cap)) ||
            (rc = B.d_cell_start.reserve(c, SG_CELLS + 1)) || (rc = B.d_items.reserve(c, SEARCH_MAX_KP)) || (rc = B.d_scalar.reserve(c, 4)) ||
            (rc = B.d_hdr.reserve(c, 1)) || (rc = B.d_pa.reserve(c, cap)) || (rc = B.d_pb.reserve(c, cap)) || (rc = B.d_level.reserve(c, cap)) ||
            (rc = B.d_flags.reserve(c, cap)) || (rc = B.d_out.reserve(c, 1)) || (rc = B.d_kp_of_edge.reserve(c, cap)) || (rc = B.d_inv_sigma2.reserve(c, PSLAM_MAX_LEVELS)))
            return rc;
        PSLAM_CUDA(c, cudaMemsetAsync(B.d_zero, 0, cap, st));
        PSLAM_CUDA(c, cudaMemcpyAsync(B.d_inv_sigma2, c->inv_sigma2.data(), g.nlevels * 4, cudaMemcpyHostToDevice, st));
        B.cap = cap;
    }
    const size_t npts = (size_t)std::max(B.n_map, cap);
    if ((rc = B.d_cand.reserve(c, npts * SEARCH_CAND_CAP)) || (rc = B.d_cand_n.reserve(c, npts)) || (rc = B.d_hist_idx.reserve(c, npts)) ||
        (rc = B.d_hist_bin.reserve(c, npts)) || (rc = B.d_in_view.reserve(c, npts)))
        return rc;
    // ---- stage A: ORB + stereo association for every frame of the sequence ----
    if ((rc = orb_run_dev(c, d_gray, nframes, B.d_kps, B.d_desc, cap, B.d_n)) != PSLAM_OK) return rc;
    if ((rc = pslam_compute_stereo_from_rgbd_batch_dev(c, B.d_kps, B.d_kps, B.d_n, cap, d_depth, nframes, prm->depth_factor, prm->bf, B.d_ur, B.d_dz)) != PSLAM_OK) return rc;
    // ---- stage B ----
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_T, Tcw0, 64, cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemsetAsync(B.d_T + 16, 0, 128, st));
    PSLAM_CUDA(c, cudaMemsetAsync(B.d_scalar, 0, 16, st));
    SearchFrameDev F;
    memset(&F, 0, sizeof F);
    F.n = cap; F.fx = prm->fx; F.fy = prm->fy; F.cx = prm->cx; F.cy = prm->cy; F.bf = prm->bf;
    F.min_x = prm->min_x; F.max_x = prm->max_x; F.min_y = prm->min_y; F.max_y = prm->max_y;
    F.n_levels = g.nlevels; F.log_scale_factor = std::log(c->cfg.scale_factor);
    for (int i = 0; i < g.nlevels; ++i) F.scale[i] = c->scale[i];
    F.inv_w = (float)SG_COLS / (F.max_x - F.min_x); F.inv_h = (float)SG_ROWS / (F.max_y - F.min_y);
    F.Tcw_dev = B.d_T;
    const TrackCam K{prm->fx, prm->fy, prm->cx, prm->cy, prm->bf};
    int32_t* m_cur = B.d_matches; int32_t* m_last = B.d_matches + cap;
    auto optimise = [&](int t, int stage) -> int {
        PSLAM_LAUNCH(c, "track_pack", k_track_pack<<<1, 256, 0, st>>>(F.keys_un, F.u_right, F.n_dev, cap, m_cur, B.M.pos, B.d_inv_sigma2, K, B.d_T, B.d_hdr, B.d_pa,
                     B.d_pb, B.d_kp_of_edge));
        PSLAM_LAUNCH(c, "pose_optimization", k_pose_optimization<<<1, POSE_THREADS, 0, st>>>(B.d_hdr, B.d_pa, B.d_pb, nullptr, nullptr, B.d_level, B.d_flags,
                     B.d_flags, B.d_flags, B.d_flags, B.d_flags, B.d_out));
        PSLAM_LAUNCH(c, "track_sweep", k_track_sweep<<<1, 256, 0, st>>>(B.d_hdr, B.d_out, B.d_flags, B.d_kp_of_edge, m_cur, B.d_T, B.d_stats + 4 * t + 2 * stage));
        return PSLAM_OK;
    };
    for (int t = 0; t < nframes; ++t) {
        F.keys_un = B.d_kps + (size_t)t * cap; F.u_right = B.d_ur + (size_t)t * cap; F.desc = B.d_desc + (size_t)t * cap * 32; F.n_dev = B.d_n + t;
        std::swap(m_cur, m_last);
        PSLAM_LAUNCH(c, "track_fill", k_track_fill<<<(cap + 255) / 256, 256, 0, st>>>(m_cur, cap, -1));
        PSLAM_LAUNCH(c, "search_grid", k_search_grid<<<1, 1024, 0, st>>>(F, B.d_cell_start, B.d_items));
        if (t > 0) {
            PSLAM_LAUNCH(c, "track_pose_algebra", k_track_pose_algebra<<<1, 32, 0, st>>>(B.d_T, 0, t > 1 && prm->use_motion_model, nullptr));
            SearchLastDev L;
            memset(&L, 0, sizeof L);
            L.n = cap; L.keys = B.d_kps + (size_t)(t - 1) * cap; L.map_point = m_last; L.outlier = B.d_zero; L.Tcw_dev = B.d_T + 16; L.n_dev = B.d_n + t - 1;
            PSLAM_LAUNCH(c, "search_candidates_last", k_candidates_last<<<(cap + 7) / 8, 256, 0, st>>>(F, L, B.M, prm->th_last, 0, B.d_cell_start, B.d_items, B.d_cand,
                         B.d_cand_n, B.d_scalar + 1));
            PSLAM_LAUNCH(c, "search_resolve_last", k_resolve_last<<<1, 32, 0, st>>>(F, L, B.M, 1, B.d_cand, B.d_cand_n, m_cur, B.d_scalar, B.d_hist_idx, B.d_hist_bin));
            if ((rc = optimise(t, 0)) != PSLAM_OK) return rc;
        } else {
            PSLAM_CUDA(c, cudaMemsetAsync(B.d_stats + 4 * t, 0, 8, st));
        }
        // TrackLocalMap
        PSLAM_LAUNCH(c, "track_skip", k_track_skip<<<(B.n_map + 255) / 256, 256, 0, st>>>(B.d_skip0, B.d_skip, B.n_map));
        PSLAM_LAUNCH(c, "track_skip_mark", k_track_skip_mark<<<(cap + 255) / 256, 256, 0, st>>>(B.d_skip, m_cur, F.n_dev, cap));
        PSLAM_LAUNCH(c, "search_candidates_map", k_candidates_map<<<(B.n_map + 7) / 8, 256, 0, st>>>(F, B.M, prm->th_map, B.d_cell_start, B.d_items, B.d_cand, B.d_cand_n,
                     B.d_in_view, B.d_scalar + 1));
        PSLAM_LAUNCH(c, "search_resolve_map", k_resolve_map<<<1, 32, 0, st>>>(B.M, prm->nnratio_map, B.d_cand, B.d_cand_n, m_cur, B.d_scalar));
        if ((rc = optimise(t, 1)) != PSLAM_OK) return rc;
        PSLAM_LAUNCH(c, "track_pose_algebra", k_track_pose_algebra<<<1, 32, 0, st>>>(B.d_T, 1, 0, B.d_T_all + 16 * t));
    }
    PSLAM_CUDA(c, cudaGetLastError());
    int32_t sc[2] = {0, 0};
    PSLAM_CUDA(c, cudaMemcpyAsync(Tcw_out, B.d_T_all, (size_t)nframes * 64, cudaMemcpyDeviceToHost, st));
    if (stats_out) PSLAM_CUDA(c, cudaMemcpyAsync(stats_out, B.d_stats, (size_t)nframes * 16, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(sc, B.d_scalar, sizeof sc, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    if (sc[1]) return set_error(c, PSLAM_E_CAPACITY, "more than 128 candidates in one search window");
    return PSLAM_OK;
}

// host-pointer convenience: uploads the frames, tracks, returns poses (the frames are the only per-sequence transfer)
int pslam_track_sequence(pslam_ctx* c, const uint8_t* gray, const uint16_t* depth, int nframes, const pslam_track_params* prm, const float* Tcw0, float* Tcw_out,
                         int32_t* stats_out) {
    if (!c) return PSLAM_E_INVALID;
    if (!gray || !depth || nframes < 1) return set_error(c, PSLAM_E_INVALID, "bad tracking arguments");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const size_t npx = (size_t)c->cfg.width * c->cfg.height;
    Slab s;
    const auto dg = s.add<uint8_t>((size_t)nframes * npx);
    const auto dd = s.add<uint16_t>((size_t)nframes * npx);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.up(dg, gray, c->stream); s.up(dd, depth, c->stream);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    rc = pslam_track_sequence_dev(c, s[dg], s[dd], nframes, prm, Tcw0, Tcw_out, stats_out);
    const int src = s.sync(c, c->stream);
    return rc != PSLAM_OK ? rc : src;
}


int pslam_track_set_planar_map(pslam_ctx* c, const pslam_planar_map* pm) {
    if (!c) return PSLAM_E_INVALID;
    if (!pm) return set_error(c, PSLAM_E_INVALID, "null planar map");
    const pslam_map_points* m = &pm->points;
    const pslam_map_lines* l = &pm->lines;
    const pslam_map_planes* p = &pm->planes;
    if (m->n < 1 || !m->pos || !m->normal || !m->max_distance || !m->min_distance || !m->desc || !m->skip || !m->has_obs)
        return set_error(c, PSLAM_E_INVALID, "planar map: null or empty point arrays");
    if (l->n < 0 || (l->n && (!l->pos || !l->normal || !l->max_distance || !l->min_distance || !l->desc || !l->skip || !l->has_obs)))
        return set_error(c, PSLAM_E_INVALID, "planar map: bad line arrays");
    if (p->n < 0 || (p->n && (!p->coef || !p->bad || !p->pts_off || (p->pts_off[p->n] > 0 && !p->pts))))
        return set_error(c, PSLAM_E_INVALID, "planar map: bad plane arrays");
    if (pm->n_ref_lines < 0 || (pm->n_ref_lines && (!pm->ref_line_desc || !pm->ref_line_map)))
        return set_error(c, PSLAM_E_INVALID, "planar map: bad reference key-frame lines");
    for (int i = 0; i < pm->n_ref_lines; ++i)
        if (pm->ref_line_map[i] < -1 || pm->ref_line_map[i] >= l->n) return set_error(c, PSLAM_E_INVALID, "planar map: ref_line_map outside the map lines");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->ptrack) c->ptrack = new PlanarTrackBuffers();
    PlanarTrackBuffers& B = *c->ptrack;
    B.ready = false;
    B.seg_live = false;                                           // the map planes' clouds restart from this upload
    B.h_off.assign(p->pts_off, p->pts_off + (p->n ? p->n + 1 : 0));
    B.max_plane_pts = 0;
    for (int j = 0; j < p->n; ++j) B.max_plane_pts = std::max(B.max_plane_pts, p->pts_off[j + 1] - p->pts_off[j]);
    const size_t nm = (size_t)m->n, nl = (size_t)l->n, np = (size_t)p->n, npts = np ? (size_t)p->pts_off[p->n] : 0, nr = (size_t)pm->n_ref_lines;
    Slab s;
    const auto pos = s.add<float>(nm * 3), normal = s.add<float>(nm * 3), max_d = s.add<float>(nm), min_d = s.add<float>(nm);
    const auto desc = s.add<uint8_t>(nm * 32), has_obs = s.add<uint8_t>(nm);
    const auto lpos = s.add<double>(nl * 6), lnormal = s.add<double>(nl * 3);
    const auto lmax = s.add<float>(nl), lmin = s.add<float>(nl);
    const auto ldesc = s.add<uint8_t>(nl * 32), lbad = s.add<uint8_t>(nl), lobs = s.add<uint8_t>(nl);
    const auto pcoef = s.add<float>(np * 4);
    const auto pbad = s.add<uint8_t>(np);
    const auto poff = s.add<int32_t>(np + 1);
    const auto ppts = s.add<float>(npts * 3 + 3);
    const auto rdesc = s.add<uint8_t>(nr * 32 + 32);
    const auto rmap = s.add<int32_t>(nr + 1), rn = s.add<int32_t>(1);
    const auto rcm = s.add<float>(9);
    int rc;
    if ((rc = s.alloc(c, B.map_blob)) || (rc = B.d_skip.reserve(c, nm)) || (rc = B.d_skip0.reserve(c, nm)) || (rc = B.d_lskip.reserve(c, nl + 1))) return rc;
    cudaStream_t st = c->stream;
    s.up(pos, m->pos, st); s.up(normal, m->normal, st); s.up(max_d, m->max_distance, st); s.up(min_d, m->min_distance, st); s.up(desc, m->desc, st);
    s.up(has_obs, m->has_obs, st);
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_skip0, m->skip, nm, cudaMemcpyHostToDevice, st));
    if (nl) { s.up(lpos, l->pos, st); s.up(lnormal, l->normal, st); s.up(lmax, l->max_distance, st); s.up(lmin, l->min_distance, st); s.up(ldesc, l->desc, st);
              s.up(lbad, l->skip, st); s.up(lobs, l->has_obs, st); }
    if (np) { s.up(pcoef, p->coef, st); s.up(pbad, p->bad, st); s.up(poff, p->pts_off, st); if (npts) s.up(ppts, p->pts, st, npts * 3); }
    if (nr) { s.up(rdesc, pm->ref_line_desc, st, nr * 32); s.up(rmap, pm->ref_line_map, st, nr); }
    const int32_t n_ref = pm->n_ref_lines;
    s.up(rn, &n_ref, st); s.up(rcm, pm->R_cm, st);
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;          // the caller's arrays may be pageable
    B.M.n = m->n; B.n_map = m->n;
    B.M.pos = s[pos]; B.M.normal = s[normal]; B.M.max_distance = s[max_d]; B.M.min_distance = s[min_d]; B.M.desc = s[desc]; B.M.has_obs = s[has_obs];
    B.M.skip = B.d_skip;
    B.l_pos = s[lpos]; B.l_normal = s[lnormal]; B.l_maxd = s[lmax]; B.l_mind = s[lmin]; B.l_desc = s[ldesc]; B.l_bad = s[lbad]; B.l_has_obs = s[lobs];
    B.n_lines = l->n;
    B.p_coef = s[pcoef]; B.p_bad = s[pbad]; B.p_off = s[poff]; B.p_pts = s[ppts]; B.n_planes = p->n;
    B.ref_desc = s[rdesc]; B.ref_map = s[rmap]; B.n_ref_dev = s[rn]; B.n_ref = n_ref; B.R_cm = s[rcm];
    B.ready = true;
    return PSLAM_OK;
}

int pslam_track_planar_sequence_dev(pslam_ctx* c, const uint8_t* d_gray, const uint16_t* d_depth, int nframes, const pslam_planar_track_params* prm,
                                    const float* Tcw0, const float* vel0, const float* Rcm0, float* Tcw_out, float* Rcm_out, int32_t* stats_out) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_gray || !d_depth || !prm || !Tcw0 || !Rcm0 || !Tcw_out || nframes < 1 || nframes > c->cfg.max_batch || prm->max_lines < 1 || prm->max_lines > 64)
        return set_error(c, PSLAM_E_INVALID, "bad planar tracking arguments");
    if (!c->ptrack || !c->ptrack->ready) return set_error(c, PSLAM_E_INVALID, "no planar map snapshot (pslam_track_set_planar_map)");
    PlanarTrackBuffers& B = *c->ptrack;
    const bool upd = B.update_planes;
    if (upd && B.max_plane_pts > MP_SLOTS) return set_error(c, PSLAM_E_CAPACITY, "map plane updates: a snapshot plane has more points than pslam_map_plane_max_points()");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const pslam_track_params& bp = prm->base;
    const OrbGeom& g = c->geom;
    const int cap = std::min(pslam_orb_max_keypoints(c), SEARCH_MAX_KP), maxp = pslam_peac_max_planes(c), n_sn = pslam_surface_normals_count(c);
    const int ml = prm->max_lines, cap_pts = 4096;
    const size_t nf = (size_t)nframes, npx = (size_t)c->cfg.width * c->cfg.height;
    cudaStream_t st = c->stream;
    // ---- HBM: the sequence's frame products, then the chain state (both owned by the context, they only grow) ----
    Slab q;
    const auto kps = q.add<pslam_keypoint>(nf * cap);
    const auto desc = q.add<uint8_t>(nf * cap * 32);
    const auto nk = q.add<int32_t>(nf);
    const auto ur = q.add<float>(nf * cap), dz = q.add<float>(nf * cap);
    const auto kl = q.add<pslam_keyline>(nf * ml);
    const auto lf = q.add<double>(nf * ml * 3);
    const auto ldesc = q.add<uint8_t>(nf * ml * 32);
    const auto l3d = q.add<pslam_line3d>(nf * ml);
    const auto nkl = q.add<int32_t>(nf), seed = q.add<int32_t>(nf), drawn = q.add<int32_t>(nf);
    const auto labels = q.add<int32_t>(nf * npx), members = q.add<int32_t>(nf * npx);
    const auto planes = q.add<pslam_plane>(nf * maxp);
    const auto npl = q.add<int32_t>(nf), moff = q.add<int32_t>(nf * (maxp + 1)), ppn = q.add<int32_t>(nf), ppsrc = q.add<int32_t>(nf * maxp);
    const auto ppcoef = q.add<float>(nf * maxp * 4);
    const auto ppoff = q.add<int32_t>(nf * (maxp + 1));
    const auto pppts = q.add<float>(nf * cap_pts * 3);
    const auto ppst = q.add<int32_t>(nf);
    const auto sn8 = q.add<float>(nf * n_sn * 8), sn3 = q.add<float>(nf * n_sn * 3);
    Slab w;
    const auto T = w.add<float>(64);                  // cur, last, velocity, prediction
    const auto Rcm = w.add<float>(9), Rcw = w.add<float>(9);
    const auto mh = w.add<pslam_manhattan_result>(1);
    const auto nmask = w.add<uint8_t>(n_sn), dmask = w.add<uint8_t>(ml);
    const auto dirs = w.add<double>(ml * 3);
    const auto ndirs = w.add<int32_t>(1), nsn = w.add<int32_t>(1), stw = w.add<int32_t>(4), cnt = w.add<int32_t>(8), scalar = w.add<int32_t>(8);
    const auto mt = w.add<int32_t>(2 * (size_t)cap);
    const auto outl = w.add<uint8_t>(2 * (size_t)cap);
    const auto cell_start = w.add<int32_t>(SG_CELLS + 1), items = w.add<int32_t>(SEARCH_MAX_KP);
    const size_t npts = (size_t)std::max(B.n_map, cap);
    const auto cand = w.add<uint32_t>(npts * SEARCH_CAND_CAP);
    const auto cand_n = w.add<int32_t>(npts), hist_idx = w.add<int32_t>(npts);
    const auto hist_bin = w.add<int8_t>(npts);
    const auto in_view = w.add<uint8_t>(npts);
    const auto fb_n = w.add<int32_t>(2), kidx = w.add<int32_t>(2 * (size_t)cap), kdist = w.add<int32_t>(2 * (size_t)cap), good = w.add<int32_t>(cap),
               ngood = w.add<int32_t>(1);
    const size_t nr = (size_t)std::max(B.n_ref, 1), nlm = (size_t)std::max(B.n_lines, 1);
    const auto lidx = w.add<int32_t>(2 * nr), ldist = w.add<int32_t>(2 * nr);
    const auto lmatch = w.add<int32_t>(ml), lassigned = w.add<int32_t>(ml);
    const auto lskip_s = w.add<uint8_t>(nlm);
    const auto lproj = w.add<float>(nlm * 4);
    const auto llevel = w.add<int32_t>(nlm);
    const auto lvcos = w.add<float>(nlm), f_pt = w.add<float>(2 * (size_t)ml);
    const auto f_ang = w.add<float>(ml);
    const auto f_oct = w.add<int32_t>(ml);
    const auto f_occ = w.add<uint8_t>(ml);
    const auto scale = w.add<float>(PSLAM_MAX_LEVELS), isig = w.add<float>(PSLAM_MAX_LEVELS);
    const auto pM = w.add<float>((size_t)maxp * 4), pang = w.add<float>((size_t)maxp * std::max(B.n_planes, 1)), pmind = w.add<float>((size_t)maxp * std::max(B.n_planes, 1));
    const auto match3 = w.add<int32_t>((size_t)maxp * 3), found3 = w.add<int32_t>((size_t)maxp * 3);
    const size_t n_wide = 2 * (size_t)ml + 3 * (size_t)maxp, n_edges = cap + n_wide;
    const auto hdr = w.add<PoseHeaderDev>(1);
    const auto pa = w.add<float4>(n_edges), pb = w.add<float4>(n_edges);
    const auto wide = w.add<PoseEdgeDev>(n_wide);
    const auto pjac = w.add<double>(3 * (size_t)maxp * 36);
    const auto level = w.add<uint8_t>(n_edges);
    const auto fpt = w.add<uint8_t>(cap), fline = w.add<uint8_t>(ml);
    const auto fplane = w.add<uint8_t>(3 * (size_t)maxp);
    const auto pout = w.add<PoseOutDev>(1);
    const auto kp_of_edge = w.add<int32_t>(cap), line_of_edge = w.add<int32_t>(ml), plane_of_edge = w.add<int32_t>(3 * (size_t)maxp);
    const auto T_all = w.add<float>(nf * 16), R_all = w.add<float>(nf * 9);
    const auto stats = w.add<int32_t>(nf * PSLAM_PLANAR_STATS);
    const auto mpst = w.add<int32_t>(upd ? nf : 0);              // map plane update status per frame
    int rc;
    if ((q.bytes() > B.seq.cap || w.bytes() > B.state.cap)) PSLAM_CUDA(c, cudaStreamSynchronize(st));     // an earlier call may still read the old buffers
    if ((rc = q.alloc(c, B.seq)) || (rc = w.alloc(c, B.state))) return rc;
    const size_t np = (size_t)B.n_planes;
    if (upd) {
        if ((rc = B.rows.reserve(c, nf * 3 * maxp))) return rc;
        if (!B.seg_live) {
            if ((rc = B.seg_pts.reserve(c, np * MP_SLOTS * 3)) || (rc = B.seg_begin.reserve(c, np)) || (rc = B.seg_end.reserve(c, np))) return rc;
            if (np) PSLAM_LAUNCH(c, "planar_seed_planes", k_planar_seed_planes<<<B.n_planes, 256, 0, st>>>(B.p_off, B.p_pts, B.seg_pts, B.seg_begin, B.seg_end));
            B.seg_live = true;
        }
        PSLAM_CUDA(c, cudaFuncSetAttribute(k_planar_map_plane_update, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MP_SMEM));
        B.rows_frames = 0;
    }
    // ---- stage A: the Frame constructor's products for every frame of the sequence ----
    PSLAM_LAUNCH(c, "track_fill", k_track_fill<<<(nframes + 255) / 256, 256, 0, st>>>(q[seed], nframes, (int32_t)prm->line_seed));
    if ((rc = pslam_peac_run_batch_dev(c, d_depth, nframes, q[labels], q[planes], q[npl], q[members], q[moff])) != PSLAM_OK) return rc;
    if ((rc = pslam_planes_post_batch_dev(c, d_depth, nframes, q[planes], q[npl], q[members], q[moff], prm->plane_dist_th, q[ppn], q[ppsrc], q[ppcoef], q[ppoff],
                                          q[pppts], cap_pts, q[ppst])) != PSLAM_OK) return rc;
    if ((rc = pslam_surface_normals_batch_dev(c, d_depth, nframes, q[sn8], q[sn3])) != PSLAM_OK) return rc;
    if ((rc = orb_run_dev(c, d_gray, nframes, q[kps], q[desc], cap, q[nk])) != PSLAM_OK) return rc;
    if ((rc = pslam_compute_stereo_from_rgbd_batch_dev(c, q[kps], q[kps], q[nk], cap, d_depth, nframes, bp.depth_factor, bp.bf, q[ur], q[dz])) != PSLAM_OK) return rc;
    if ((rc = pslam_lines_extract_describe_batch_dev(c, d_gray, nframes, ml, q[kl], q[lf], q[ldesc], q[nkl])) != PSLAM_OK) return rc;
    const float cam[4] = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    if ((rc = pslam_lines3d_batch_dev(c, q[kl], q[nkl], ml, d_depth, nframes, bp.depth_factor, cam, reinterpret_cast<const uint32_t*>(q[seed]), nullptr, q[l3d],
                                      q[drawn])) != PSLAM_OK) return rc;
    // ---- stage B ----
    static const float I4[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    w.up(T, Tcw0, st, 16);
    PSLAM_CUDA(c, cudaMemcpyAsync(w[T] + 32, vel0 ? vel0 : I4, 64, cudaMemcpyHostToDevice, st));
    w.up(Rcm, Rcm0, st, 9);
    const int32_t n_sn_i = n_sn;
    w.up(nsn, &n_sn_i, st); w.up(scale, c->scale.data(), st, g.nlevels); w.up(isig, c->inv_sigma2.data(), st, g.nlevels);
    w.zero(scalar, st); w.zero(stats, st); w.zero(outl, st);
    if (upd) w.zero(mpst, st);
    if ((rc = w.check(c)) != PSLAM_OK) return rc;
    PSLAM_CUDA(c, cudaStreamSynchronize(st));        // the host arguments above may be pageable; nothing is synchronised from here to the end of the sequence
    SearchFrameDev F;
    memset(&F, 0, sizeof F);
    F.n = cap; F.fx = bp.fx; F.fy = bp.fy; F.cx = bp.cx; F.cy = bp.cy; F.bf = bp.bf;
    F.min_x = bp.min_x; F.max_x = bp.max_x; F.min_y = bp.min_y; F.max_y = bp.max_y;
    F.n_levels = g.nlevels; F.log_scale_factor = std::log(c->cfg.scale_factor);
    for (int i = 0; i < g.nlevels; ++i) F.scale[i] = c->scale[i];
    F.inv_w = (float)SG_COLS / (F.max_x - F.min_x); F.inv_h = (float)SG_ROWS / (F.max_y - F.min_y);
    F.Tcw_dev = w[T];
    const TrackCam K{bp.fx, bp.fy, bp.cx, bp.cy, bp.bf};
    const PlanarCam PK{bp.fx, bp.fy, bp.cx, bp.cy, bp.bf, bp.min_x, bp.max_x, bp.min_y, bp.max_y, F.log_scale_factor};
    const PoseEdgeConsts EK = pose_edge_consts(prm->angle_info, prm->dist_info, prm->par_info, prm->ver_info, prm->plane_chi, prm->vp_chi);
    const PlanarEdges E{w[kp_of_edge], w[line_of_edge], w[plane_of_edge]};
    int32_t *m_cur = w[mt], *m_last = w[mt] + cap;
    uint8_t *o_cur = w[outl], *o_last = w[outl] + cap;
    float* Tp = w[T];
    int32_t* S = w[stw];
    const int gmax = (std::max(std::max(B.n_map, B.n_lines), ml) + 255) / 256;
    auto planes_match = [&](int t) -> int {
        PSLAM_LAUNCH(c, "planar_plane_world", k_planar_plane_world<<<(maxp + 127) / 128, 128, 0, st>>>(S, Tp, q[ppcoef] + (size_t)t * maxp * 4, q[ppn] + t, maxp, w[pM],
                     w[found3], w[cnt] + 2));
        if (B.n_planes > 0)
            plane_match_run_dev(c, maxp, B.n_planes, w[pM], B.p_coef, B.p_bad, upd ? B.seg_begin : B.p_off, upd ? B.seg_end : B.p_off + 1,
                                upd ? B.seg_pts : B.p_pts, w[pang], w[pmind], prm->plane_dist_ref, prm->plane_ang_ref,
                                prm->plane_ver_th, prm->plane_par_th, w[found3], w[found3] + 2 * maxp, w[found3] + maxp, w[cnt] + 2);
        PSLAM_LAUNCH(c, "planar_plane_merge", k_planar_plane_merge<<<(3 * maxp + 127) / 128, 128, 0, st>>>(w[found3], w[match3], 3 * maxp));
        return PSLAM_OK;
    };
    auto optimise = [&](int t, int mode) -> int {
        int32_t* srow = w[stats] + (size_t)t * PSLAM_PLANAR_STATS;
        PSLAM_LAUNCH(c, "planar_pack", k_planar_pack<<<1, 256, 0, st>>>(mode, S, mode == 1 ? w[cnt] : nullptr, w[Rcw], Tp, F.keys_un, F.u_right, F.n_dev, cap, m_cur,
                     B.M.pos, w[isig], q[lf] + (size_t)t * ml * 3, q[nkl] + t, ml, w[lmatch], w[lassigned], B.l_pos, q[ppcoef] + (size_t)t * maxp * 4, q[ppn] + t,
                     maxp, w[match3], B.p_coef, K, EK, prm->plane_chi, prm->vp_chi, w[hdr], w[pa], w[pb], w[wide], E, srow));
        PSLAM_LAUNCH(c, "pose_optimization", k_pose_optimization<<<1, POSE_THREADS, 0, st>>>(w[hdr], w[pa], w[pb], w[wide], w[pjac], w[level], w[fpt], w[fline],
                     w[fplane], w[fplane] + maxp, w[fplane] + 2 * maxp, w[pout]));
        PSLAM_LAUNCH(c, "planar_sweep", k_planar_sweep<<<1, 256, 0, st>>>(mode, S, w[hdr], w[pout], w[fpt], w[fline], w[fplane], E, m_cur, o_cur, B.d_skip,
                     B.M.has_obs, w[lmatch], B.d_lskip, B.l_has_obs, q[ppn] + t, maxp, w[match3], Tp, srow));
        return PSLAM_OK;
    };
    for (int t = 0; t < nframes; ++t) {
        F.keys_un = q[kps] + (size_t)t * cap; F.u_right = q[ur] + (size_t)t * cap; F.desc = q[desc] + (size_t)t * cap * 32; F.n_dev = q[nk] + t;
        std::swap(m_cur, m_last); std::swap(o_cur, o_last);
        int32_t* srow = w[stats] + (size_t)t * PSLAM_PLANAR_STATS;
        PSLAM_LAUNCH(c, "track_fill", k_track_fill<<<(cap + 255) / 256, 256, 0, st>>>(m_cur, cap, -1));
        PSLAM_CUDA(c, cudaMemsetAsync(o_cur, 0, cap, st));
        PSLAM_LAUNCH(c, "search_grid", k_search_grid<<<1, 1024, 0, st>>>(F, w[cell_start], w[items]));
        PSLAM_LAUNCH(c, "track_skip", k_track_skip<<<(B.n_map + 255) / 256, 256, 0, st>>>(B.d_skip0, B.d_skip, B.n_map));
        if (B.n_lines) PSLAM_LAUNCH(c, "track_skip", k_track_skip<<<(B.n_lines + 255) / 256, 256, 0, st>>>(B.l_bad, B.d_lskip, B.n_lines));
        if (t > 0) PSLAM_LAUNCH(c, "track_pose_algebra", k_track_pose_algebra<<<1, 32, 0, st>>>(Tp, 0, 1, nullptr));
        PSLAM_LAUNCH(c, "planar_begin", k_planar_begin<<<1, 64, 0, st>>>(q[l3d] + (size_t)t * ml, q[nkl] + t, ml, w[dirs], w[ndirs], Tp, S, w[cnt], w[lmatch],
                     w[match3], maxp));
        // TrackManhattanFrame(mLastRcm, vSurfaceNormal, mVF3DLines)
        if ((rc = pslam_track_manhattan_batch_dev(c, w[Rcm], q[sn3] + (size_t)t * n_sn * 3, w[nsn], n_sn, w[dirs], w[ndirs], ml, 1, w[mh], w[nmask], w[dmask])) != PSLAM_OK)
            return rc;
        PSLAM_LAUNCH(c, "planar_rotation", k_planar_rotation<<<1, 32, 0, st>>>(0, w[mh], B.R_cm, w[Rcm], w[Rcw], Tp, nullptr));
        if (t > 0) {
            // TranslationWithMotionModel
            SearchLastDev L;
            memset(&L, 0, sizeof L);
            L.n = cap; L.keys = q[kps] + (size_t)(t - 1) * cap; L.map_point = m_last; L.outlier = o_last; L.Tcw_dev = Tp + 16; L.n_dev = q[nk] + t - 1;
            PSLAM_LAUNCH(c, "search_candidates_last", k_candidates_last<<<(cap + 7) / 8, 256, 0, st>>>(F, L, B.M, bp.th_last, 0, w[cell_start], w[items], w[cand],
                         w[cand_n], w[scalar] + 1));
            PSLAM_LAUNCH(c, "search_resolve_last", k_resolve_last<<<1, 32, 0, st>>>(F, L, B.M, 1, w[cand], w[cand_n], m_cur, w[scalar], w[hist_idx], w[hist_bin]));
            PSLAM_LAUNCH(c, "planar_fallback_prep", k_planar_fallback_prep<<<1, 32, 0, st>>>(w[scalar], q[nk] + t, q[nk] + t - 1, cap, w[fb_n]));
            if ((rc = pslam_hamming_knn2_batch_dev(c, F.desc, w[fb_n], cap, q[desc] + (size_t)(t - 1) * cap * 32, w[fb_n] + 1, cap, 1, w[kidx], w[kdist], w[good],
                                                   w[ngood])) != PSLAM_OK) return rc;
            PSLAM_LAUNCH(c, "planar_fallback_apply", k_planar_fallback_apply<<<1, 256, 0, st>>>(w[fb_n], w[kidx], w[good], w[ngood], m_last, o_last, cap, m_cur,
                         w[scalar], srow));
            if (B.n_ref > 0) {
                if ((rc = pslam_hamming_knn2_batch_dev(c, B.ref_desc, B.n_ref_dev, B.n_ref, q[ldesc] + (size_t)t * ml * 32, q[nkl] + t, ml, 1, w[lidx], w[ldist],
                                                       nullptr, nullptr)) != PSLAM_OK) return rc;
                PSLAM_LAUNCH(c, "planar_line_desc", k_planar_line_desc<<<1, 32, 0, st>>>(B.n_ref, w[lidx], w[ldist], B.ref_map, w[lmatch], w[cnt] + 1));
            }
            if ((rc = planes_match(t)) != PSLAM_OK) return rc;
            // the pack kernel reads the three counts: nmatches (scalar[0]), line matches (cnt[1]), plane matches (cnt[2])
            PSLAM_LAUNCH(c, "planar_counts", k_planar_counts<<<1, 32, 0, st>>>(w[scalar], w[cnt]));
            if ((rc = optimise(t, 1)) != PSLAM_OK) return rc;
        }
        // TrackLocalMap (a no-op when the motion-model stage failed)
        PSLAM_LAUNCH(c, "track_skip_mark", k_track_skip_mark<<<(cap + 255) / 256, 256, 0, st>>>(B.d_skip, m_cur, F.n_dev, cap));
        PSLAM_LAUNCH(c, "planar_local_prep", k_planar_local_prep<<<gmax, 256, 0, st>>>(S, B.d_skip, B.n_map, B.d_lskip, B.n_lines, w[lmatch], B.l_has_obs,
                     q[kl] + (size_t)t * ml, q[nkl] + t, ml, w[f_pt], w[f_ang], w[f_oct], w[f_occ]));
        PSLAM_LAUNCH(c, "search_candidates_map", k_candidates_map<<<(B.n_map + 7) / 8, 256, 0, st>>>(F, B.M, bp.th_map, w[cell_start], w[items], w[cand], w[cand_n],
                     w[in_view], w[scalar] + 1));
        PSLAM_LAUNCH(c, "search_resolve_map", k_resolve_map<<<1, 32, 0, st>>>(B.M, bp.nnratio_map, w[cand], w[cand_n], m_cur, w[scalar] + 2));
        PSLAM_LAUNCH(c, "track_fill", k_track_fill<<<1, 64, 0, st>>>(w[lassigned], ml, -1));
        if (B.n_lines > 0) {
            PSLAM_LAUNCH(c, "planar_lines_in_frustum", k_planar_lines_in_frustum<<<(B.n_lines + 127) / 128, 128, 0, st>>>(PK, Tp, B.n_lines, B.l_pos, B.l_normal,
                         B.l_maxd, B.l_mind, B.d_lskip, 0.6f, w[lskip_s], w[lproj], w[llevel], w[lvcos]));
            line_search_run_dev(c, ml, w[f_pt], w[f_ang], w[f_oct], q[ldesc] + (size_t)t * ml * 32, w[f_occ], w[scale], g.nlevels, B.n_lines, w[lskip_s], w[llevel],
                                w[lvcos], w[lproj], B.l_desc, B.l_has_obs, prm->line_th, prm->line_nnratio, w[lassigned], w[scalar] + 3);
        }
        if ((rc = planes_match(t)) != PSLAM_OK) return rc;
        if ((rc = optimise(t, 0)) != PSLAM_OK) return rc;
        PSLAM_LAUNCH(c, "planar_clean", k_planar_clean<<<(cap + 255) / 256, 256, 0, st>>>(S, m_cur, o_cur, B.M.has_obs, F.n_dev, cap));
        // the velocity of a tracked frame (not after frame 0: frame 1 uses vel0), mLastRcm from the final pose
        PSLAM_LAUNCH(c, "track_pose_algebra", k_track_pose_algebra<<<1, 32, 0, st>>>(Tp, 1, 0, w[T_all] + 16 * (size_t)t, t > 0 ? S + 1 : S + 3));
        PSLAM_LAUNCH(c, "planar_rotation", k_planar_rotation<<<1, 32, 0, st>>>(t > 0 ? 1 : 2, w[mh], B.R_cm, w[Rcm], w[Rcw], Tp, w[R_all] + 9 * (size_t)t));
        if (upd)       // (:294-304) with the frame's final pose and final mvpMapPlanes
            PSLAM_LAUNCH(c, "planar_map_plane_update", k_planar_map_plane_update<<<std::max(B.n_planes, 1), MP_THREADS, MP_SMEM, st>>>(Tp, w[match3], q[ppn] + t, maxp,
                         q[ppoff] + (size_t)t * (maxp + 1), q[pppts] + (size_t)t * cap_pts * 3, B.n_planes, B.seg_pts, B.seg_begin, B.seg_end,
                         B.rows + (size_t)t * 3 * maxp, w[mpst] + t));
    }
    PSLAM_CUDA(c, cudaGetLastError());
    int32_t sc[2] = {0, 0};
    std::vector<int32_t> pst(nf), mps(upd ? nf : 0);
    PSLAM_CUDA(c, cudaMemcpyAsync(Tcw_out, w[T_all], nf * 64, cudaMemcpyDeviceToHost, st));
    if (Rcm_out) PSLAM_CUDA(c, cudaMemcpyAsync(Rcm_out, w[R_all], nf * 36, cudaMemcpyDeviceToHost, st));
    if (stats_out) PSLAM_CUDA(c, cudaMemcpyAsync(stats_out, w[stats], nf * PSLAM_PLANAR_STATS * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(sc, w[scalar], sizeof sc, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(pst.data(), q[ppst], nf * 4, cudaMemcpyDeviceToHost, st));
    if (upd) PSLAM_CUDA(c, cudaMemcpyAsync(mps.data(), w[mpst], nf * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    if (upd) B.rows_frames = nframes;
    if (sc[1]) return set_error(c, PSLAM_E_CAPACITY, "more than 128 candidates in one search window");
    for (int f = 0; f < nframes; ++f)
        if (pst[f] & (32 | 64)) return set_error(c, PSLAM_E_CAPACITY, "planar tracking: more plane voxels than the per-frame capacity");
    for (int f = 0; f < (int)mps.size(); ++f)
        if (mps[f]) return set_error(c, PSLAM_E_CAPACITY, "map plane updates: a merged cloud exceeds pslam_map_plane_max_points() voxels (the plane kept its cloud)");
    return PSLAM_OK;
}

int pslam_track_planar_sequence(pslam_ctx* c, const uint8_t* gray, const uint16_t* depth, int nframes, const pslam_planar_track_params* prm, const float* Tcw0,
                                const float* vel0, const float* Rcm0, float* Tcw_out, float* Rcm_out, int32_t* stats_out) {
    if (!c) return PSLAM_E_INVALID;
    if (!gray || !depth || nframes < 1 || nframes > c->cfg.max_batch) return set_error(c, PSLAM_E_INVALID, "bad planar tracking arguments");
    if (!c->ptrack || !c->ptrack->ready) return set_error(c, PSLAM_E_INVALID, "no planar map snapshot (pslam_track_set_planar_map)");
    if (c->ptrack->update_planes && c->ptrack->max_plane_pts > MP_SLOTS)       // refused before the frames are staged
        return set_error(c, PSLAM_E_CAPACITY, "map plane updates: a snapshot plane has more points than pslam_map_plane_max_points()");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const size_t npx = (size_t)c->cfg.width * c->cfg.height;
    Slab s;
    const auto dg = s.add<uint8_t>((size_t)nframes * npx);
    const auto dd = s.add<uint16_t>((size_t)nframes * npx);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.up(dg, gray, c->stream); s.up(dd, depth, c->stream);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    rc = pslam_track_planar_sequence_dev(c, s[dg], s[dd], nframes, prm, Tcw0, vel0, Rcm0, Tcw_out, Rcm_out, stats_out);
    const int src = s.sync(c, c->stream);
    return rc != PSLAM_OK ? rc : src;
}

int pslam_track_planar_set_map_plane_updates(pslam_ctx* c, int on) {
    if (!c) return PSLAM_E_INVALID;
    if (!c->ptrack) c->ptrack = new PlanarTrackBuffers();
    PlanarTrackBuffers& B = *c->ptrack;
    if (!on) B.seg_live = false;                                  // mode off: the uploaded clouds; a later update-mode call starts from them again
    B.update_planes = on != 0;
    return PSLAM_OK;
}

int pslam_track_planar_get_map_plane_updates(const pslam_ctx* c) {
    if (!c) return PSLAM_E_INVALID;
    return c->ptrack && c->ptrack->update_planes ? 1 : 0;
}

int pslam_track_planar_map_planes(pslam_ctx* c, int32_t* pts_off, float* pts, int cap) {
    if (!c) return PSLAM_E_INVALID;
    if (!c->ptrack || !c->ptrack->ready || !pts_off || cap < 0 || (cap && !pts)) return set_error(c, PSLAM_E_INVALID, "bad map plane readback (or no planar map snapshot)");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    PlanarTrackBuffers& B = *c->ptrack;
    const int n = B.n_planes;
    cudaStream_t st = c->stream;
    const bool seg = B.update_planes && B.seg_live;
    std::vector<int32_t> end(n);
    if (seg && n) {
        PSLAM_CUDA(c, cudaMemcpyAsync(end.data(), B.seg_end, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
        PSLAM_CUDA(c, cudaStreamSynchronize(st));
    }
    pts_off[0] = 0;
    for (int j = 0; j < n; ++j) pts_off[j + 1] = pts_off[j] + (seg ? end[j] - j * MP_SLOTS : B.h_off[j + 1] - B.h_off[j]);
    if (pts_off[n] > cap) return set_error(c, PSLAM_E_CAPACITY, "map plane readback: more points than cap (pts_off holds the sizes)");
    for (int j = 0; j < n; ++j) {
        const size_t k = (size_t)(pts_off[j + 1] - pts_off[j]);
        const float* src = seg ? B.seg_pts + (size_t)j * MP_SLOTS * 3 : B.p_pts + (size_t)B.h_off[j] * 3;
        if (k) PSLAM_CUDA(c, cudaMemcpyAsync(pts + (size_t)pts_off[j] * 3, src, k * 12, cudaMemcpyDeviceToHost, st));
    }
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    return PSLAM_OK;
}

int pslam_track_planar_plane_matches(pslam_ctx* c, int32_t* out, int nframes) {
    if (!c) return PSLAM_E_INVALID;
    if (!c->ptrack || c->ptrack->rows_frames < 1 || !out || nframes < 1 || nframes > c->ptrack->rows_frames)
        return set_error(c, PSLAM_E_INVALID, "plane association readback: no call in map plane update mode, or nframes beyond its length");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const size_t maxp = (size_t)pslam_peac_max_planes(c);
    PSLAM_CUDA(c, cudaMemcpyAsync(out, c->ptrack->rows, (size_t)nframes * 3 * maxp * 4, cudaMemcpyDeviceToHost, c->stream));
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSLAM_OK;
}

}  // extern "C"
