// The edge-record format of k_pose_optimization (pose_kernels.cuh) and the conversions Optimizer::PoseOptimization / TranslationOptimization apply to a
// Frame's fields before they become edges (src/Optimizer.cc:583-981, :3019-3220).  Shared by the host packer (pose_pipeline.cu) and the device packers of the
// planar tracking chain (track_chain.cu), so both produce the same bytes for the same inputs.  Host/device: plain float / double arithmetic, no fused
// multiply-add (the library is built with --fmad=false).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <cuda_runtime.h>

#if defined(__CUDACC__)
#define PR_HD __host__ __device__
#else
#define PR_HD
#endif

namespace pslam {

enum { PK_MONO = 0, PK_STEREO = 1, PK_LINE = 2, PK_PLANE = 3, PK_PAR = 4, PK_VER = 5,
       PK_MONO_T = 6, PK_STEREO_T = 7, PK_LINE_T = 8, PK_PLANE_T = 9 };   // translation-only variants (TranslationOptimization)

// A problem's edges are numbered points first, then the start / end edge of every line, then the plane, parallel-plane
// and vertical-plane edges.  Point edge i is two float4 records (every field is a float in the reference's Frame, so
// widening on load gives the same doubles): pt_a[edge_off + i] = (Xw, u), pt_b[edge_off + i] = (v, uR, inv_sigma2, Huber
// delta); uR < 0 makes it monocular.  Line and plane edges are PoseEdgeDev records, wide[wide_off + i - n_pt].
struct PoseEdgeDev {            // 104 bytes
    int32_t kind, idx;          // idx: index inside its family (line i / plane i)
    double a[8];                // lines: Xw[3], obs[3]; planes: world plane[4], measured plane[4] (normalised)
    double info[3];
    double delta;               // Huber delta
};

// Huber deltas of the point and line edges: const float deltaMono = sqrt(5.991), deltaStereo = sqrt(7.815) (:583-584)
PR_HD inline float pose_delta_mono() { return (float)sqrt(5.991); }
PR_HD inline float pose_delta_stereo() { return (float)sqrt(7.815); }

// Huber deltas and information of the plane families: sqrt(Plane.Chi) / sqrt(Plane.VPChi), 3282.8 / info^2 for the angle terms and DistanceInfo^2 for the
// distance term (:771-783)
struct PoseEdgeConsts {
    float delta_plane, delta_vp;
    double angle_info, dist_info, par_info, ver_info;
};
PR_HD inline PoseEdgeConsts pose_edge_consts(double angle_info, double dist_info, double par_info, double ver_info, double plane_chi, double vp_chi) {
    PoseEdgeConsts k;
    k.delta_plane = (float)sqrt(plane_chi); k.delta_vp = (float)sqrt(vp_chi);
    k.angle_info = 3282.8 / (angle_info * angle_info); k.dist_info = dist_info * dist_info;
    k.par_info = 3282.8 / (par_info * par_info); k.ver_info = 3282.8 / (ver_info * ver_info);
    return k;
}

// Converter::toPlane3D + Plane3D::normalize of a float plane
PR_HD inline void plane_from_float4(const float* v, double out[4]) {
    double p[4] = {v[0], v[1], v[2], v[3]};
    if (v[3] < 0.0f) for (int i = 0; i < 4; ++i) p[i] = -p[i];
    const double n = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    const double s = 1. / n;
    for (int i = 0; i < 4; ++i) p[i] = p[i] * s;
    if (p[3] < 0.0) for (int i = 0; i < 4; ++i) p[i] = -p[i];
    for (int i = 0; i < 4; ++i) out[i] = p[i];
}

// row `row` of R_cw * X as cv::Mat(CV_32F) products compute it: double accumulation, float result (TranslationOptimization :3019, :3066, :3161)
PR_HD inline double rot_f(const float* T, double x, double y, double z, int row) {
    return (double)(float)((double)T[row * 4 + 0] * (double)(float)x + (double)T[row * 4 + 1] * (double)(float)y + (double)T[row * 4 + 2] * (double)(float)z);
}

// point edge: Xw (pre-rotated by the float R_cw of T in mode 1), observation u, v, uR, mvInvLevelSigma2[octave]
PR_HD inline void pose_point_record(const float* Xw, float u, float v, float ur, float inv_sigma2, int mode, const float* T, float4& a, float4& b) {
    float X[3];
    for (int q = 0; q < 3; ++q) X[q] = mode == 0 ? Xw[q] : (float)rot_f(T, Xw[0], Xw[1], Xw[2], q);
    a = make_float4(X[0], X[1], X[2], u);
    b = make_float4(v, ur, inv_sigma2, ur < 0 ? pose_delta_mono() : pose_delta_stereo());
}

// start (s = 0) or end (s = 1) edge of line i: endpoint line_Xw[3 s ..] (double), line function obs[3]
PR_HD inline void pose_line_record(const double* line_Xw6, const double* obs, int i, int s, int mode, const float* T, PoseEdgeDev& e) {
    memset(&e, 0, sizeof e);
    e.kind = mode == 0 ? PK_LINE : PK_LINE_T; e.idx = i;
    const double* X = line_Xw6 + 3 * s;
    for (int q = 0; q < 3; ++q) { e.a[q] = mode == 0 ? X[q] : rot_f(T, X[0], X[1], X[2], q); e.a[3 + q] = obs[q]; e.info[q] = 1.0; }
    e.delta = pose_delta_stereo();
}

// plane edge of family kind (PK_PLANE, PK_PAR, PK_VER, PK_PLANE_T): map plane GetWorldPos() and the frame's mvPlaneCoefficients, both float.  PK_PLANE_T
// rotates the world normal by the widened float R_cw of T (Xw.rotateNormal(toMatrix3d(R_cw)), not renormalised).
PR_HD inline void pose_plane_record(int kind, int i, const float* map, const float* meas, const float* T, const PoseEdgeConsts& k, PoseEdgeDev& e) {
    memset(&e, 0, sizeof e);
    e.kind = kind; e.idx = i;
    plane_from_float4(map, e.a); plane_from_float4(meas, e.a + 4);
    if (kind == PK_PLANE || kind == PK_PLANE_T) { e.info[0] = k.angle_info; e.info[1] = k.angle_info; e.info[2] = k.dist_info; e.delta = k.delta_plane; }
    else if (kind == PK_PAR) { e.info[0] = k.par_info; e.info[1] = k.par_info; e.delta = k.delta_vp; }
    else { e.info[0] = k.ver_info; e.info[1] = k.ver_info; e.delta = k.delta_vp; }
    if (kind == PK_PLANE_T) {
        const double nrm[3] = {e.a[0], e.a[1], e.a[2]};
        for (int r = 0; r < 3; ++r) e.a[r] = (double)T[r * 4 + 0] * nrm[0] + (double)T[r * 4 + 1] * nrm[1] + (double)T[r * 4 + 2] * nrm[2];
    }
}

}  // namespace pslam
