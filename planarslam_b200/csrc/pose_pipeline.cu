// Host side of the pose optimisation: packs the caller's problems (the arrays Optimizer::PoseOptimization reads from a
// Frame, src/Optimizer.cc:593-981) into flat device records, launches one CTA per problem, unpacks the results.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "pose_kernels.cuh"

namespace pslam {

struct PoseBuffers {
    // host staging
    std::vector<PoseHeaderDev> h_hdr;
    std::vector<float4> h_pa, h_pb;          // point records (one slot per edge; line / plane slots stay zero)
    std::vector<PoseEdgeDev> h_wide;         // line and plane records
    // device
    PoseHeaderDev* d_hdr = nullptr; float4* d_pa = nullptr; float4* d_pb = nullptr; PoseEdgeDev* d_wide = nullptr; double* d_pjac = nullptr;
    uint8_t* d_level = nullptr;
    uint8_t* d_flags[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    PoseOutDev* d_out = nullptr;
    size_t cap_prob = 0, cap_out = 0, cap_pa = 0, cap_pb = 0, cap_wide = 0, cap_pjac = 0, cap_level = 0, cap_flags[5] = {0, 0, 0, 0, 0};   // one capacity per buffer (elements)
    int n_prob = 0;
    int tot_flags[5] = {0, 0, 0, 0, 0};
    std::vector<PoseOutDev> h_out;
    std::vector<uint8_t> h_flags[5];
};

static void plane_from_float4(const float* v, double out[4]) {     // Converter::toPlane3D + Plane3D::normalize
    double p[4] = {v[0], v[1], v[2], v[3]};
    if (v[3] < 0.0f) for (int i = 0; i < 4; ++i) p[i] = -p[i];
    const double n = std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    const double s = 1. / n;
    for (int i = 0; i < 4; ++i) p[i] = p[i] * s;
    if (p[3] < 0.0) for (int i = 0; i < 4; ++i) p[i] = -p[i];
    for (int i = 0; i < 4; ++i) out[i] = p[i];
}

template <typename T>
static int grow(pslam_ctx* c, T** p, size_t* cap, size_t need) {
    if (need <= *cap) return PSLAM_OK;
    if (*p) cudaFree(*p);
    *p = nullptr;
    const size_t n = std::max<size_t>(need * 3 / 2, 64);
    int rc = check_cuda(c, cudaMalloc((void**)p, n * sizeof(T)), "cudaMalloc(pose)");
    *cap = rc == PSLAM_OK ? n : 0;
    return rc;
}

int pose_pack_upload(pslam_ctx* c, const pslam_pose_problem* probs, int n, const float* Tcw0, int mode) {
    if (!c->pose) c->pose = new PoseBuffers();
    PoseBuffers& B = *c->pose;
    B.h_hdr.assign(n, PoseHeaderDev());
    B.h_pa.clear(); B.h_pb.clear(); B.h_wide.clear();
    int off[5] = {0, 0, 0, 0, 0}, n_plane_edges = 0;
    for (int p = 0; p < n; ++p) {
        const pslam_pose_problem& P = probs[p];
        PoseHeaderDev& H = B.h_hdr[p];
        if (P.n_points < 0 || P.n_lines < 0 || P.n_planes < 0 || P.n_par < 0 || P.n_ver < 0) return set_error(c, PSLAM_E_INVALID, "negative count in pose problem");
        if ((P.n_points && (!P.Xw || !P.obs || !P.inv_sigma2)) || (P.n_lines && (!P.line_Xw || !P.line_obs)) ||
            (P.n_planes && (!P.plane_meas || !P.plane_map)) || (P.n_par && (!P.par_meas || !P.par_map)) || (P.n_ver && (!P.ver_meas || !P.ver_map)))
            return set_error(c, PSLAM_E_INVALID, "null array in pose problem");
        H.edge_off = (int)B.h_pa.size(); H.wide_off = (int)B.h_wide.size(); H.plane_off = n_plane_edges;
        H.n_pt = P.n_points; H.n_line = P.n_lines; H.n_plane = P.n_planes; H.n_par = P.n_par; H.n_ver = P.n_ver;
        for (int k = 0; k < 5; ++k) H.flag_off[k] = off[k];
        off[0] += P.n_points; off[1] += P.n_lines; off[2] += P.n_planes; off[3] += P.n_par; off[4] += P.n_ver;
        H.n_initial = mode == 0 ? P.n_points + P.n_lines + P.n_planes + P.n_par + P.n_ver : P.n_points;   // :3137-3139, :3245-3246
        H.mode = mode;
        const float* T0 = Tcw0 + 16 * p;
        // R_cw * X as cv::Mat(CV_32F) products do it: double accumulation, float result (TranslationOptimization :3019,:3066,:3161)
        auto rot_f = [&](double x, double y, double z, int row) -> double {
            return (double)(float)((double)T0[row * 4 + 0] * (double)(float)x + (double)T0[row * 4 + 1] * (double)(float)y + (double)T0[row * 4 + 2] * (double)(float)z);
        };
        H.fx = P.fx; H.fy = P.fy; H.cx = P.cx; H.cy = P.cy; H.bf = P.bf; H.plane_chi = P.plane_chi; H.vp_chi = P.vp_chi;
        std::memcpy(H.Tcw0, Tcw0 + 16 * p, sizeof H.Tcw0);
        const float deltaMono = std::sqrt(5.991), deltaStereo = std::sqrt(7.815);       // const float in the reference (:583-584)
        const float deltaPlane = std::sqrt(P.plane_chi), deltaVP = std::sqrt(P.vp_chi);
        const double angleInfo = 3282.8 / (P.angle_info * P.angle_info), disInfo = P.dist_info * P.dist_info;
        const double parInfo = 3282.8 / (P.par_info * P.par_info), verInfo = 3282.8 / (P.ver_info * P.ver_info);
        for (int i = 0; i < P.n_points; ++i) {     // monocular when uR < 0; every field is a float, so the float record loses nothing
            const bool mono = P.obs[3 * i + 2] < 0;
            float X[3];
            for (int k = 0; k < 3; ++k) X[k] = mode == 0 ? P.Xw[3 * i + k] : (float)rot_f(P.Xw[3 * i], P.Xw[3 * i + 1], P.Xw[3 * i + 2], k);
            B.h_pa.push_back(make_float4(X[0], X[1], X[2], P.obs[3 * i]));
            B.h_pb.push_back(make_float4(P.obs[3 * i + 1], P.obs[3 * i + 2], P.inv_sigma2[i], mono ? deltaMono : deltaStereo));
        }
        auto add_wide = [&](const PoseEdgeDev& e) {
            B.h_wide.push_back(e);
            B.h_pa.push_back(make_float4(0, 0, 0, 0)); B.h_pb.push_back(make_float4(0, 0, 0, 0));
        };
        for (int i = 0; i < P.n_lines; ++i)
            for (int s = 0; s < 2; ++s) {
                PoseEdgeDev e;
                std::memset(&e, 0, sizeof e);
                e.kind = mode == 0 ? PK_LINE : PK_LINE_T; e.idx = i;
                const double* X = P.line_Xw + 6 * i + 3 * s;
                for (int k = 0; k < 3; ++k) { e.a[k] = mode == 0 ? X[k] : rot_f(X[0], X[1], X[2], k); e.a[3 + k] = P.line_obs[3 * i + k]; e.info[k] = 1.0; }
                e.delta = deltaStereo;
                add_wide(e);
            }
        auto add_planes = [&](int kind, int cnt, const float* meas, const float* map, double i0, double i1, double i2, double delta) {
            for (int i = 0; i < cnt; ++i) {
                PoseEdgeDev e;
                std::memset(&e, 0, sizeof e);
                e.kind = kind; e.idx = i;
                plane_from_float4(map + 4 * i, e.a); plane_from_float4(meas + 4 * i, e.a + 4);
                e.info[0] = i0; e.info[1] = i1; e.info[2] = i2; e.delta = delta;
                add_wide(e);
            }
        };
        if (mode == 0) {
            add_planes(PK_PLANE, P.n_planes, P.plane_meas, P.plane_map, angleInfo, angleInfo, disInfo, deltaPlane);
            add_planes(PK_PAR, P.n_par, P.par_meas, P.par_map, parInfo, parInfo, 0, deltaVP);
            add_planes(PK_VER, P.n_ver, P.ver_meas, P.ver_map, verInfo, verInfo, 0, deltaVP);
        } else if (P.n_points >= 3) {          // the reference returns before adding planes when < 3 points are matched (:3198-3200)
            const size_t first = B.h_wide.size();
            add_planes(PK_PLANE_T, P.n_planes, P.plane_meas, P.plane_map, angleInfo, angleInfo, disInfo, deltaPlane);
            for (size_t k = first; k < B.h_wide.size(); ++k) {     // Xw.rotateNormal(toMatrix3d(R_cw)): widened float rotation, not renormalised
                double* a = B.h_wide[k].a;
                const double nrm[3] = {a[0], a[1], a[2]};
                for (int r = 0; r < 3; ++r) a[r] = (double)T0[r * 4 + 0] * nrm[0] + (double)T0[r * 4 + 1] * nrm[1] + (double)T0[r * 4 + 2] * nrm[2];
            }
        }
        H.n_edges = (int)B.h_pa.size() - H.edge_off;
        n_plane_edges += H.n_edges - H.n_pt - 2 * H.n_line;
    }
    B.n_prob = n;
    for (int k = 0; k < 5; ++k) B.tot_flags[k] = off[k];
    const size_t n_edges = B.h_pa.size();
    int rc;
    if ((rc = grow(c, &B.d_hdr, &B.cap_prob, (size_t)n)) != PSLAM_OK) return rc;
    if ((rc = grow(c, &B.d_out, &B.cap_out, (size_t)n)) != PSLAM_OK) return rc;
    if ((rc = grow(c, &B.d_pa, &B.cap_pa, n_edges)) != PSLAM_OK) return rc;
    if ((rc = grow(c, &B.d_pb, &B.cap_pb, n_edges)) != PSLAM_OK) return rc;
    if ((rc = grow(c, &B.d_wide, &B.cap_wide, B.h_wide.size())) != PSLAM_OK) return rc;
    if ((rc = grow(c, &B.d_pjac, &B.cap_pjac, (size_t)n_plane_edges * 36)) != PSLAM_OK) return rc;
    if ((rc = grow(c, &B.d_level, &B.cap_level, n_edges)) != PSLAM_OK) return rc;
    for (int k = 0; k < 5; ++k) if ((rc = grow(c, &B.d_flags[k], &B.cap_flags[k], (size_t)std::max(off[k], 1))) != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_hdr, B.h_hdr.data(), n * sizeof(PoseHeaderDev), cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_pa, B.h_pa.data(), n_edges * sizeof(float4), cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_pb, B.h_pb.data(), n_edges * sizeof(float4), cudaMemcpyHostToDevice, st));
    if (!B.h_wide.empty()) PSLAM_CUDA(c, cudaMemcpyAsync(B.d_wide, B.h_wide.data(), B.h_wide.size() * sizeof(PoseEdgeDev), cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));       // the staging vectors are pageable
    return PSLAM_OK;
}

int pose_run_packed(pslam_ctx* c) {
    if (!c->pose || c->pose->n_prob < 1) return set_error(c, PSLAM_E_INVALID, "no packed pose problems");
    PoseBuffers& B = *c->pose;
    // a batch runs 64-thread CTAs.  Measured on the benchmark's 1584 problems (H100 SXM, 400 W; tools/pose_profile.py): 7.9 ms per call at 64 threads,
    // 8.0 at 32 and 8.6 at 128.  64 also keeps the parent's per-thread edge sets and reduction tree, so results are bit-identical to it.
    PSLAM_LAUNCH(c, "pose_optimization", k_pose_optimization<<<B.n_prob, POSE_BATCH_THREADS, 0, c->stream>>>(B.d_hdr, B.d_pa, B.d_pb, B.d_wide, B.d_pjac, B.d_level,
                 B.d_flags[0], B.d_flags[1], B.d_flags[2], B.d_flags[3], B.d_flags[4], B.d_out));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

int pose_fetch(pslam_ctx* c, float* Tcw, double* Tcw_d, uint8_t* o_pt, uint8_t* o_line, uint8_t* o_plane, uint8_t* o_par, uint8_t* o_ver,
               int32_t* n_inliers, int32_t* trace_i, double* trace_d) {
    if (!c->pose || c->pose->n_prob < 1) return set_error(c, PSLAM_E_INVALID, "no packed pose problems");
    PoseBuffers& B = *c->pose;
    B.h_out.resize(B.n_prob);
    cudaStream_t st = c->stream;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_out.data(), B.d_out, B.n_prob * sizeof(PoseOutDev), cudaMemcpyDeviceToHost, st));
    uint8_t* dst[5] = {o_pt, o_line, o_plane, o_par, o_ver};
    for (int k = 0; k < 5; ++k)
        if (dst[k] && B.tot_flags[k]) PSLAM_CUDA(c, cudaMemcpyAsync(dst[k], B.d_flags[k], B.tot_flags[k], cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    for (int p = 0; p < B.n_prob; ++p) {
        const PoseOutDev& o = B.h_out[p];
        if (Tcw) std::memcpy(Tcw + 16 * p, o.Tcw, sizeof o.Tcw);
        if (Tcw_d) std::memcpy(Tcw_d + 16 * p, o.Tcw_d, sizeof o.Tcw_d);
        if (n_inliers) n_inliers[p] = o.n_inliers;
        if (trace_i) std::memcpy(trace_i + 12 * p, o.trace_i, sizeof o.trace_i);
        if (trace_d) std::memcpy(trace_d + 8 * p, o.trace_d, sizeof o.trace_d);
    }
    return PSLAM_OK;
}

void pose_free(pslam_ctx* c) {
    if (!c->pose) return;
    PoseBuffers& B = *c->pose;
    cudaFree(B.d_hdr); cudaFree(B.d_pa); cudaFree(B.d_pb); cudaFree(B.d_wide); cudaFree(B.d_pjac); cudaFree(B.d_level); cudaFree(B.d_out);
    for (int k = 0; k < 5; ++k) cudaFree(B.d_flags[k]);
    delete c->pose;
    c->pose = nullptr;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

static int pack_mode(pslam_ctx* c, const pslam_pose_problem* probs, int n, const float* Tcw0, int mode) {
    if (!c) return PSLAM_E_INVALID;
    if (!probs || !Tcw0 || n < 1) return set_error(c, PSLAM_E_INVALID, "null problems or n < 1");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return pose_pack_upload(c, probs, n, Tcw0, mode);
}
int pslam_pose_pack(pslam_ctx* c, const pslam_pose_problem* probs, int n, const float* Tcw0) { return pack_mode(c, probs, n, Tcw0, 0); }
int pslam_translation_pack(pslam_ctx* c, const pslam_pose_problem* probs, int n, const float* Tcw0) { return pack_mode(c, probs, n, Tcw0, 1); }

int pslam_pose_run_packed(pslam_ctx* c) {
    if (!c) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return pose_run_packed(c);
}

int pslam_pose_fetch(pslam_ctx* c, float* Tcw, double* Tcw_d, uint8_t* o_pt, uint8_t* o_line, uint8_t* o_plane, uint8_t* o_par, uint8_t* o_ver,
                     int32_t* n_inliers, int32_t* trace_i, double* trace_d) {
    if (!c) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return pose_fetch(c, Tcw, Tcw_d, o_pt, o_line, o_plane, o_par, o_ver, n_inliers, trace_i, trace_d);
}

int pslam_pose_optimization_batch(pslam_ctx* c, const pslam_pose_problem* probs, int n, float* Tcw_io, uint8_t* o_pt, uint8_t* o_line,
                                  uint8_t* o_plane, uint8_t* o_par, uint8_t* o_ver, int32_t* n_inliers) {
    int rc = pslam_pose_pack(c, probs, n, Tcw_io);
    if (rc != PSLAM_OK) return rc;
    if ((rc = pose_run_packed(c)) != PSLAM_OK) return rc;
    return pose_fetch(c, Tcw_io, nullptr, o_pt, o_line, o_plane, o_par, o_ver, n_inliers, nullptr, nullptr);
}

int pslam_pose_optimization(pslam_ctx* c, const pslam_pose_problem* prob, float* Tcw_io, uint8_t* o_pt, uint8_t* o_line, uint8_t* o_plane,
                            uint8_t* o_par, uint8_t* o_ver) {
    int32_t n_inl = 0;
    const int rc = pslam_pose_optimization_batch(c, prob, 1, Tcw_io, o_pt, o_line, o_plane, o_par, o_ver, &n_inl);
    return rc != PSLAM_OK ? rc : n_inl;
}

int pslam_translation_optimization_batch(pslam_ctx* c, const pslam_pose_problem* probs, int n, float* Tcw_io, uint8_t* o_pt, uint8_t* o_line,
                                         uint8_t* o_plane, int32_t* n_inliers) {
    int rc = pslam_translation_pack(c, probs, n, Tcw_io);
    if (rc != PSLAM_OK) return rc;
    if ((rc = pose_run_packed(c)) != PSLAM_OK) return rc;
    return pose_fetch(c, Tcw_io, nullptr, o_pt, o_line, o_plane, nullptr, nullptr, n_inliers, nullptr, nullptr);
}

int pslam_translation_optimization(pslam_ctx* c, const pslam_pose_problem* prob, float* Tcw_io, uint8_t* o_pt, uint8_t* o_line, uint8_t* o_plane) {
    int32_t n_inl = 0;
    const int rc = pslam_translation_optimization_batch(c, prob, 1, Tcw_io, o_pt, o_line, o_plane, &n_inl);
    return rc != PSLAM_OK ? rc : n_inl;
}

}  // extern "C"
