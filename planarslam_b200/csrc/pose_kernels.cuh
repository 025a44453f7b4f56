// Pose optimisation on sm_90a: one CTA per frame runs the reference's whole PoseOptimization — four rounds of
// Levenberg-Marquardt (<= 10 iterations each, g2o's control flow) over point / line / plane unary edges with chi-square
// re-classification between rounds.  Edges are evaluated edge-parallel (one thread per edge, strided), the 6x6 normal
// equations (21 unique entries of J^T W J plus 6 of J^T W r) and the robust chi2 are reduced with warp shuffles and a
// fixed-order cross-warp sum (deterministic), the 6x6 LDL^T solve and the SE(3) update are done redundantly per thread.
// FP64 throughout (inputs are widened from float like the reference does); no tensor cores: the "GEMM" is K x 6 by 6 x K
// with K ~ 1e3 in double, a reduction, not a dense MMA tile (SURVEY.md §8d).
//
// Reference semantics: src/Optimizer.cc:550-1275; vendored g2o LM optimization_algorithm_levenberg.cpp:61-189,
// sparse_optimizer.cpp:61-114,354-419, base_unary_edge.hpp:43-122, robust_kernel_impl.cpp:78-91, linear_solver_dense.h:65-113,
// se3quat.h, types_six_dof_expmap.{h,cpp}, include/EdgeLine.h:155-245, g2oAddition/{EdgePlane,EdgeParallelPlane,
// EdgeVerticalPlane,Plane3D}.h, src/Converter.cc:37-45,171-180.
#pragma once
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

#include "pslam_internal.h"
#include "geom_device.cuh"

namespace pslam {

enum { PK_MONO = 0, PK_STEREO = 1, PK_LINE = 2, PK_PLANE = 3, PK_PAR = 4, PK_VER = 5,
       PK_MONO_T = 6, PK_STEREO_T = 7, PK_LINE_T = 8, PK_PLANE_T = 9 };   // translation-only variants (TranslationOptimization)
__host__ __device__ inline bool pk_is_plane(int k) { return k == PK_PLANE || k == PK_PAR || k == PK_VER || k == PK_PLANE_T; }
__host__ __device__ inline bool pk_is_point(int k) { return k == PK_MONO || k == PK_STEREO || k == PK_MONO_T || k == PK_STEREO_T; }
__host__ __device__ inline bool pk_is_line(int k) { return k == PK_LINE || k == PK_LINE_T; }

struct PoseEdgeDev {            // 104 bytes
    int32_t kind, idx;          // idx: index inside its family (point i / line i / plane i)
    double a[8];                // points & lines: Xw[3], obs[3]; planes: world plane[4], measured plane[4] (normalised)
    double info[3];
    double delta;               // Huber delta
};

struct PoseHeaderDev {
    int32_t edge_off, n_edges;
    int32_t n_pt, n_line, n_plane, n_par, n_ver;
    int32_t flag_off[5];        // offsets of this problem's outlier flags inside the five concatenated flag arrays
    int32_t n_initial;          // nInitialCorrespondences
    int32_t mode;               // 0 = PoseOptimization, 1 = TranslationOptimization
    double fx, fy, cx, cy, bf, plane_chi, vp_chi;
    float Tcw0[16];
};

struct PoseOutDev {
    float Tcw[16];
    double Tcw_d[16];
    int32_t n_inliers;
    int32_t trace_i[12];        // per round: LM iterations, trials, nBad (-1 when the round did not run)
    double trace_d[8];          // per round: final robust chi2, final lambda
};

struct PoseCam { double fx, fy, cx, cy, bf; };

// residual of one edge at pose T (computeError of the six edge classes)
static __device__ __noinline__ void pose_edge_error(const PoseEdgeDev& e, const dSE3& T, const PoseCam& K, double err[3]) {
    if (e.kind <= PK_LINE || (e.kind >= PK_MONO_T && e.kind <= PK_LINE_T)) {
        const bool tonly = e.kind >= PK_MONO_T;                                   // mapTrans: Xc + t (se3quat.h:221)
        const dV3 p = tonly ? dv(e.a[0], e.a[1], e.a[2]) + T.t : qrot(T.q, dv(e.a[0], e.a[1], e.a[2])) + T.t;
        if (e.kind == PK_MONO || e.kind == PK_MONO_T) {
            err[0] = e.a[3] - (p.x / p.z * K.fx + K.cx);
            err[1] = e.a[4] - (p.y / p.z * K.fy + K.cy);
            err[2] = 0;
        } else if (e.kind == PK_STEREO || e.kind == PK_STEREO_T) {
            const float invz = 1.0f / (float)p.z;                             // sic: float reciprocal (types_six_dof_expmap.cpp:300,369)
            const double r0 = p.x * invz * K.fx + K.cx, r1 = p.y * invz * K.fy + K.cy, r2 = r0 - K.bf * invz;
            err[0] = e.a[3] - r0; err[1] = e.a[4] - r1; err[2] = e.a[5] - r2;
        } else {
            const double u = p.x / p.z * K.fx + K.cx, v = p.y / p.z * K.fy + K.cy;
            err[0] = e.a[3] * u + e.a[4] * v + e.a[5]; err[1] = 0; err[2] = 0;
        }
        return;
    }
    // localPlane = T * Xw  (Plane3D operator*, Plane3D.h:186-199), or T + Xc for the translation-only edge (:201-209)
    dV3 n = dv(e.a[0], e.a[1], e.a[2]);
    if (e.kind != PK_PLANE_T) n = mmul(quat_to_matrix(T.q), n);
    double lp[4] = {n.x, n.y, n.z, e.a[3] - ddot(T.t, n)};
    if (lp[3] < 0.0) { lp[0] = -lp[0]; lp[1] = -lp[1]; lp[2] = -lp[2]; lp[3] = -lp[3]; }
    plane_normalize(lp);
    const dV3 ln = dv(lp[0], lp[1], lp[2]), mn = dv(e.a[4], e.a[5], e.a[6]);
    dV3 base = ln;
    if (e.kind == PK_PAR) {
        if (ddot(mn, ln) < 0) base = -1.0 * ln;
    } else if (e.kind == PK_VER) {
        const dV3 v = dcross(ln, mn);
        const dV3 ax = (1.0 / sqrt(ddot(v, v))) * v;
        const double ang = 3.14159265358979323846 / 2, c = cos(ang), s = sin(ang);
        base = c * ln + s * dcross(ax, ln) + ((1 - c) * ddot(ax, ln)) * ax;
    }
    const dV3 nn = mmul(plane_rotation_T(base), mn);
    err[0] = azimuth(nn); err[1] = elevation(nn);
    err[2] = (e.kind == PK_PLANE || e.kind == PK_PLANE_T) ? ((-lp[3]) - (-e.a[7])) : 0.0;
}

__device__ __forceinline__ int pose_edge_dim(int kind) { return kind == PK_MONO || kind == PK_MONO_T || kind == PK_PAR || kind == PK_VER ? 2 : 3; }

static __device__ __noinline__ void pose_edge_jacobian(const PoseEdgeDev& e, const dSE3& T, const PoseCam& K, double J[3][6]) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) J[i][j] = 0;
    if (e.kind <= PK_LINE) {
        const dV3 p = qrot(T.q, dv(e.a[0], e.a[1], e.a[2])) + T.t;
        const double x = p.x, y = p.y, invz = 1.0 / p.z, invz_2 = invz * invz;
        if (e.kind == PK_LINE) {
            const double lx = e.a[3], ly = e.a[4], fx = K.fx, fy = K.fy;
            J[0][0] = -fy * ly - fx * lx * x * y * invz_2 - fy * ly * y * y * invz_2;
            J[0][1] = fx * lx + fx * lx * x * x * invz_2 + fy * ly * x * y * invz_2;
            J[0][2] = -fx * lx * y * invz + fy * ly * x * invz;
            J[0][3] = fx * lx * invz;
            J[0][4] = fy * ly * invz;
            J[0][5] = -(fx * lx * x + fy * ly * y) * invz_2;
            return;
        }
        J[0][0] = x * y * invz_2 * K.fx; J[0][1] = -(1 + (x * x * invz_2)) * K.fx; J[0][2] = y * invz * K.fx;
        J[0][3] = -invz * K.fx; J[0][4] = 0; J[0][5] = x * invz_2 * K.fx;
        J[1][0] = (1 + y * y * invz_2) * K.fy; J[1][1] = -x * y * invz_2 * K.fy; J[1][2] = -x * invz * K.fy;
        J[1][3] = 0; J[1][4] = -invz * K.fy; J[1][5] = y * invz_2 * K.fy;
        if (e.kind == PK_STEREO) {
            J[2][0] = J[0][0] - K.bf * y * invz_2; J[2][1] = J[0][1] + K.bf * x * invz_2; J[2][2] = J[0][2];
            J[2][3] = J[0][3]; J[2][4] = 0; J[2][5] = J[0][5] - K.bf * invz_2;
        }
        return;
    }
    if (e.kind >= PK_MONO_T && e.kind <= PK_LINE_T) {          // rotation columns are zero (types_six_dof_expmap.cpp:404-485, EdgeLine.h:283-310)
        const dV3 p = dv(e.a[0], e.a[1], e.a[2]) + T.t;
        const double x = p.x, y = p.y, invz = 1.0 / p.z, invz_2 = invz * invz;
        if (e.kind == PK_LINE_T) {
            const double lx = e.a[3], ly = e.a[4];
            J[0][3] = K.fx * lx * invz; J[0][4] = K.fy * ly * invz; J[0][5] = -(K.fx * lx * x + K.fy * ly * y) * invz_2;
            return;
        }
        J[0][3] = -invz * K.fx; J[0][5] = x * invz_2 * K.fx;
        J[1][4] = -invz * K.fy; J[1][5] = y * invz_2 * K.fy;
        if (e.kind == PK_STEREO_T) { J[2][3] = J[0][3]; J[2][5] = J[0][5] - K.bf * invz_2; }
        return;
    }
    // numeric central differences with delta = 1e-9 like BaseUnaryEdge::linearizeOplus (the reference does this for
    // every plane edge; an analytic Jacobian would change the iterates)
    const double delta = 1e-9, scalar = 1.0 / (2 * delta);
    const int dim = pose_edge_dim(e.kind);
    for (int d = 0; d < 6; ++d) {
        double add[6] = {0, 0, 0, 0, 0, 0}, e1[3], e2[3];
        add[d] = delta;
        pose_edge_error(e, se3_mul(se3_exp(add), T), K, e1);
        add[d] = -delta;
        pose_edge_error(e, se3_mul(se3_exp(add), T), K, e2);
        for (int i = 0; i < dim; ++i) J[i][d] = scalar * (e1[i] - e2[i]);
    }
    if (e.kind == PK_PLANE_T)                                  // EdgePlaneOnlyTranslation zeroes the rotation columns (EdgePlane.h:292-308)
        for (int i = 0; i < 3; ++i) { J[i][0] = 0; J[i][1] = 0; J[i][2] = 0; }
}

__device__ __forceinline__ void huber(double e2, double delta, double& rho0, double& rho1) {
    const double dsqr = delta * delta;
    if (e2 <= dsqr) { rho0 = e2; rho1 = 1.; }
    else { const double s = sqrt(e2); rho0 = 2 * s * delta - dsqr; rho1 = delta / s; }
}

static __device__ __noinline__ bool solve6(const double H[6][6], const double b[6], double x[6]) {
    double L[6][6], D[6], y[6];
    for (int j = 0; j < 6; ++j) {
        double d = H[j][j];
        for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k] * D[k];
        if (!(d > 0)) return false;
        D[j] = d;
        for (int i = j + 1; i < 6; ++i) {
            double v = H[i][j];
            for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k] * D[k];
            L[i][j] = v / d;
        }
    }
    for (int i = 0; i < 6; ++i) { double v = b[i]; for (int k = 0; k < i; ++k) v -= L[i][k] * y[k]; y[i] = v; }
    for (int i = 0; i < 6; ++i) y[i] /= D[i];
    for (int i = 5; i >= 0; --i) { double v = y[i]; for (int k = i + 1; k < 6; ++k) v -= L[k][i] * x[k]; x[i] = v; }
    return true;
}

#define POSE_THREADS 256                 // upper bound of the block size (single problems, track_chain.cu); batches launch PSLAM_POSE_THREADS (pose_pipeline.cu)
#define POSE_WARPS (POSE_THREADS / 32)
#define POSE_NT ((int)blockDim.x)

// deterministic block reduction of NV doubles held per thread: result broadcast in out[] (shared)
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV], double* s_part /*[POSE_WARPS][NV]*/, double* s_out /*[NV]*/) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        double t = v[k];
#pragma unroll
        for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) s_part[wid * NV + k] = t;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        double t = 0;
        for (int w = 0; w < (POSE_NT >> 5); ++w) t += s_part[w * NV + threadIdx.x];
        s_out[threadIdx.x] = t;
    }
    __syncthreads();
}

// errors of the active edges at pose Tq, and the robust chi2 (computeActiveErrors + activeRobustChi2)
static __device__ __noinline__ double pose_active_chi(const PoseEdgeDev* E, int ne, const uint8_t* level, double* err, const dSE3& Tq, const PoseCam& K,
                                               bool robust, double* s_part, double* s_red) {
    double acc[1] = {0};
    for (int i = threadIdx.x; i < ne; i += POSE_NT) {
        if (level[i]) continue;
        const PoseEdgeDev& e = E[i];
        double e3[3];
        pose_edge_error(e, Tq, K, e3);
        err[3 * i] = e3[0]; err[3 * i + 1] = e3[1]; err[3 * i + 2] = e3[2];
        const int dim = pose_edge_dim(e.kind);
        double c = 0;
        for (int r = 0; r < dim; ++r) c += e3[r] * e.info[r] * e3[r];
        if (robust) { double r0, r1; huber(c, e.delta, r0, r1); c = r0; }
        acc[0] += c;
    }
    block_sum<1>(acc, s_part, s_red);
    return s_red[0];
}

static __global__ void __launch_bounds__(POSE_THREADS) k_pose_optimization(const PoseHeaderDev* __restrict__ headers, const PoseEdgeDev* __restrict__ edges,
                                                                    double* __restrict__ err_all, uint8_t* __restrict__ level_all,
                                                                    uint8_t* __restrict__ f_pt, uint8_t* __restrict__ f_line, uint8_t* __restrict__ f_plane,
                                                                    uint8_t* __restrict__ f_par, uint8_t* __restrict__ f_ver, PoseOutDev* __restrict__ outs) {
    const int prob = blockIdx.x, tid = threadIdx.x;
    const PoseHeaderDev& hd = headers[prob];
    const PoseEdgeDev* E = edges + hd.edge_off;
    double* err = err_all + (size_t)hd.edge_off * 3;
    uint8_t* level = level_all + hd.edge_off;
    const int ne = hd.n_edges;
    PoseCam K;
    K.fx = hd.fx; K.fy = hd.fy; K.cx = hd.cx; K.cy = hd.cy; K.bf = hd.bf;
    uint8_t* fl[5] = {f_pt + hd.flag_off[0], f_line + hd.flag_off[1], f_plane + hd.flag_off[2], f_par + hd.flag_off[3], f_ver + hd.flag_off[4]};

    __shared__ double s_part[POSE_WARPS * 28];
    __shared__ double s_red[28];
    __shared__ double s_T[7], s_x[6];
    __shared__ int s_i[4];

    // initial pose: Converter::toSE3Quat(mTcw) — float entries widened, quaternion from the (not exactly orthonormal) matrix
    dSE3 T0;
    {
        dM3 R;
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R.m[i][j] = hd.Tcw0[i * 4 + j];
        T0.q = qnorm_pos(quat_from_matrix(R));
        T0.t = dv(hd.Tcw0[3], hd.Tcw0[7], hd.Tcw0[11]);
    }
    PoseOutDev& out = outs[prob];
    for (int i = tid; i < 12; i += POSE_NT) out.trace_i[i] = -1;
    for (int i = tid; i < 8; i += POSE_NT) out.trace_d[i] = 0;
    for (int i = tid; i < hd.n_pt; i += POSE_NT) fl[0][i] = 0;
    for (int i = tid; i < hd.n_line; i += POSE_NT) fl[1][i] = 0;
    for (int i = tid; i < hd.n_plane; i += POSE_NT) fl[2][i] = 0;
    for (int i = tid; i < hd.n_par; i += POSE_NT) fl[3][i] = 0;
    for (int i = tid; i < hd.n_ver; i += POSE_NT) fl[4][i] = 0;
    for (int i = tid; i < ne; i += POSE_NT) {
        level[i] = 0;
        double e3[3] = {0, 0, 0};
        if (pk_is_plane(E[i].kind)) pose_edge_error(E[i], T0, K, e3);      // computeError() while the graph is built (:896,:935,:975,:3300)
        err[3 * i] = e3[0]; err[3 * i + 1] = e3[1]; err[3 * i + 2] = e3[2];
    }
    __syncthreads();

    auto write_pose = [&](const dSE3& T, int n_inl) {
        if (tid == 0) {
            const dM3 R = quat_to_matrix(T.q);
            const double tt[3] = {T.t.x, T.t.y, T.t.z};
            for (int i = 0; i < 16; ++i) out.Tcw_d[i] = (i == 15) ? 1.0 : 0.0;
            for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) out.Tcw_d[i * 4 + j] = R.m[i][j]; out.Tcw_d[i * 4 + 3] = tt[i]; }
            for (int i = 0; i < 16; ++i) out.Tcw[i] = (float)out.Tcw_d[i];
            out.n_inliers = n_inl;
        }
    };
    if (hd.n_initial < 3) {                       // :985-986: return 0, pose untouched
        if (tid == 0) { for (int i = 0; i < 16; ++i) { out.Tcw[i] = hd.Tcw0[i]; out.Tcw_d[i] = hd.Tcw0[i]; } out.n_inliers = 0; }
        return;
    }

    bool robust = true;                           // Huber is dropped for every edge after round index 2
    dSE3 T = T0;
    int nBad_total = 0;
    double lambda = 0, ni = 2;
    double x[6] = {0, 0, 0, 0, 0, 0};

    auto active_chi = [&](const dSE3& Tq) -> double { return pose_active_chi(E, ne, level, err, Tq, K, robust, s_part, s_red); };

    for (int it = 0; it < 4; ++it) {
        T = T0;
        int iters = 0, trials_total = 0, nBadLm = 0;
        double chi_final = 0;
        bool ok = true;
        for (int iter = 0; iter < 10 && ok; ++iter) {
            // ---- OptimizationAlgorithmLevenberg::solve ----
            double currentChi = active_chi(T);
            const double iniChi = currentChi;
            double tempChi = currentChi;
            // buildSystem: H = sum rho1 J^T Omega J, b = -sum rho1 J^T Omega e
            double acc[27];
#pragma unroll
            for (int k = 0; k < 27; ++k) acc[k] = 0;
            for (int i = tid; i < ne; i += POSE_NT) {
                if (level[i]) continue;
                const PoseEdgeDev& e = E[i];
                double J[3][6];
                pose_edge_jacobian(e, T, K, J);
                const int dim = pose_edge_dim(e.kind);
                double w = 1.0;
                if (robust) {
                    double c = 0;
                    for (int r = 0; r < dim; ++r) c += err[3 * i + r] * e.info[r] * err[3 * i + r];
                    double r0;
                    huber(c, e.delta, r0, w);
                }
                for (int r = 0; r < dim; ++r) {
                    const double oe = e.info[r] * err[3 * i + r];
                    int k = 0;
#pragma unroll
                    for (int a = 0; a < 6; ++a) {
                        acc[21 + a] -= w * J[r][a] * oe;
                        const double wa = w * e.info[r] * J[r][a];
#pragma unroll
                        for (int b2 = a; b2 < 6; ++b2) acc[k++] += wa * J[r][b2];
                    }
                }
            }
            block_sum<27>(acc, s_part, s_red);
            double H[6][6], b[6];
            {
                int k = 0;
                for (int a = 0; a < 6; ++a) for (int b2 = a; b2 < 6; ++b2) { H[a][b2] = s_red[k]; H[b2][a] = s_red[k]; ++k; }
                for (int a = 0; a < 6; ++a) b[a] = s_red[21 + a];
            }
            __syncthreads();
            if (iter == 0) {
                double mx = 0;
                for (int j = 0; j < 6; ++j) mx = fmax(fabs(H[j][j]), mx);
                lambda = 1e-5 * mx; ni = 2; nBadLm = 0;
            }
            double rho = 0;
            int qmax = 0;
            do {
                const dSE3 backup = T;
                double Hl[6][6];
                for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) Hl[i][j] = H[i][j] + (i == j ? lambda : 0.0);
                const bool ok2 = solve6(Hl, b, x);                 // on failure x keeps the previous solution (g2o applies it anyway)
                T = se3_mul(se3_exp(x), T);
                tempChi = active_chi(T);
                if (!ok2) tempChi = DBL_MAX;
                rho = currentChi - tempChi;
                double scale = 0;
                for (int j = 0; j < 6; ++j) scale += x[j] * (lambda * x[j] + b[j]);
                scale += 1e-3;
                rho /= scale;
                if (rho > 0 && isfinite(tempChi)) {
                    double alpha = 1. - pow((2 * rho - 1), 3.0);
                    alpha = fmin(alpha, 2. / 3.);
                    const double sf = fmax(1. / 3., alpha);
                    lambda *= sf; ni = 2; currentChi = tempChi;
                } else {
                    lambda *= ni; ni *= 2; T = backup;
                }
                ++qmax;
            } while (rho < 0 && qmax < 10);
            trials_total += qmax;
            chi_final = currentChi;
            ++iters;
            if (qmax == 10 || rho == 0) { ok = false; }
            else {
                if ((iniChi - currentChi) * 1e3 < iniChi) ++nBadLm; else nBadLm = 0;
                if (nBadLm >= 3) ok = false;
            }
        }
        // ---- classify every edge against its chi-square threshold (:1006-1259) ----
        double nb[1] = {0};
        for (int i = tid; i < ne; i += POSE_NT) {
            const PoseEdgeDev& e = E[i];
            if (pk_is_point(e.kind)) {
                uint8_t& f = fl[0][e.idx];
                if (f) { double e3[3]; pose_edge_error(e, T, K, e3); err[3 * i] = e3[0]; err[3 * i + 1] = e3[1]; err[3 * i + 2] = e3[2]; }
                const int dim = pose_edge_dim(e.kind);
                double c = 0;
                for (int r = 0; r < dim; ++r) c += err[3 * i + r] * e.info[r] * err[3 * i + r];
                const float cf = (float)c;
                if (cf > ((e.kind == PK_MONO || e.kind == PK_MONO_T) ? 5.991f : 7.815f)) { f = 1; level[i] = 1; nb[0] += 1; } else { f = 0; level[i] = 0; }
            } else if (pk_is_line(e.kind)) {
                // start (even) and end (odd) edges of a line are adjacent; the thread owning the start edge classifies both
                const int first = hd.n_pt;               // first line edge
                if (((i - first) & 1) == 0) {
                    uint8_t& f = fl[1][e.idx];
                    // PoseOptimization recomputes both endpoint errors unconditionally (:1087-1088); TranslationOptimization only
                    // for lines currently flagged as outliers (:3598-3601) and keeps a separate nLineBad
                    if (hd.mode == 0 || f) {
                        double ea[3], eb[3];
                        pose_edge_error(E[i], T, K, ea); pose_edge_error(E[i + 1], T, K, eb);
                        err[3 * i] = ea[0]; err[3 * i + 1] = 0; err[3 * i + 2] = 0;
                        err[3 * (i + 1)] = eb[0]; err[3 * (i + 1) + 1] = 0; err[3 * (i + 1) + 2] = 0;
                    }
                    const float cs = (float)(err[3 * i] * err[3 * i]), ce = (float)(err[3 * (i + 1)] * err[3 * (i + 1)]);
                    if (cs > 2 * 5.991f || ce > 2 * 5.991f) { f = 1; level[i] = 1; level[i + 1] = 1; if (hd.mode == 0) nb[0] += 1; }
                    else { f = 0; level[i] = 0; level[i + 1] = 0; }
                }
            } else {
                uint8_t& f = fl[e.kind == PK_PLANE_T ? 2 : e.kind - PK_PLANE + 2][e.idx];
                if (f) { double e3[3]; pose_edge_error(e, T, K, e3); err[3 * i] = e3[0]; err[3 * i + 1] = e3[1]; err[3 * i + 2] = e3[2]; }
                const int dim = pose_edge_dim(e.kind);
                double c = 0;
                for (int r = 0; r < dim; ++r) c += err[3 * i + r] * e.info[r] * err[3 * i + r];
                const float cf = (float)c;
                const double th = (e.kind == PK_PLANE || e.kind == PK_PLANE_T) ? hd.plane_chi : hd.vp_chi;
                if ((double)cf > th) { f = 1; level[i] = 1; nb[0] += 1; } else { f = 0; level[i] = 0; }
            }
        }
        block_sum<1>(nb, s_part, s_red);
        nBad_total = (int)(s_red[0] + 0.5);
        __syncthreads();
        if (it == 2) robust = false;
        if (tid == 0) {
            out.trace_i[3 * it] = iters; out.trace_i[3 * it + 1] = trials_total; out.trace_i[3 * it + 2] = nBad_total;
            out.trace_d[2 * it] = chi_final; out.trace_d[2 * it + 1] = lambda;
        }
        if (ne < 10) break;
    }
    write_pose(T, hd.n_initial - nBad_total);
}

}  // namespace pslam
