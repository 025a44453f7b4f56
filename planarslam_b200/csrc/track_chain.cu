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
// Not modelled (documented in DESIGN.md): UpdateLastFrame's temporary RGB-D points, key-frame insertion, lines / planes in the chain (their stages run batched).
#include <algorithm>
#include <cmath>
#include <cstring>

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
// mode 1: end of a frame: velocity <- cur * LastTwc with LastTwc = [Rlw^T | -Rlw^T tlw] (Tracking.cc:270-278); record the pose.
__global__ void k_track_pose_algebra(float* __restrict__ T, int mode, int use_velocity, float* __restrict__ T_out) {
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
        mat4_mul(cur, Twc, vel);
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
// monocular when mvuRight[i] < 0, stereo otherwise; information = mvInvLevelSigma2[octave]; Huber deltas sqrt(5.991) / sqrt(7.815) as float.
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
    const float deltaMono = sqrtf(5.991f), deltaStereo = sqrtf(7.815f);
    for (int i = b0; i < b1; ++i) {
        const int m = matches[i];
        if (m < 0) continue;
        const float ur = u_right[i];
        const bool mono = ur < 0;
        const pslam_keypoint kp = keys[i];
        pt_a[pos] = make_float4(map_pos[3 * m], map_pos[3 * m + 1], map_pos[3 * m + 2], kp.x);     // the point record of pose_kernels.cuh
        pt_b[pos] = make_float4(kp.y, ur, inv_sigma2[kp.octave], mono ? deltaMono : deltaStereo);
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

void track_free(pslam_ctx* c) {
    delete c->track;
    c->track = nullptr;
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

}  // extern "C"
