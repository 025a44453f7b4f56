// Pose optimisation on sm_90a: one CTA per frame runs the reference's whole PoseOptimization — four rounds of
// Levenberg-Marquardt (<= 10 iterations each, g2o's control flow) over point / line / plane unary edges with chi-square
// re-classification between rounds.  Edges are evaluated edge-parallel (one thread per edge, strided); each pass keeps the
// residual, the Jacobian and the accumulators in registers.  One pass per LM iteration evaluates the residuals, the robust
// chi2 and the 6x6 normal equations (21 unique entries of J^T W J plus 6 of J^T W r) at the same pose (g2o's
// computeActiveErrors + buildSystem); one chi2 pass per trial.  The sums are reduced with warp shuffles and a fixed-order
// cross-warp sum (deterministic).  The 6x6 LDL^T solve and the SE(3) update run once per trial on thread 0 and reach the
// other threads through shared memory.  FP64 throughout (inputs are widened from float like the reference does); no tensor
// cores: the "GEMM" is K x 6 by 6 x K with K ~ 1e3 in double, a reduction, not a dense MMA tile (SURVEY.md §8d).
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
#include "pose_records.h"

namespace pslam {

struct PoseHeaderDev {
    int32_t edge_off, n_edges;  // first edge in the point records and the level bytes, edge count
    int32_t wide_off;           // first line / plane record
    int32_t plane_off;          // first plane edge in the numeric-Jacobian scratch (36 doubles per plane edge)
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

struct PoseErr3 { double e[3]; };

// residual of a plane, parallel-plane or vertical-plane edge at pose T (computeError of EdgePlane & co.).  Out of line: a
// problem has a handful of plane edges, and inlining this trigonometry at every call site would only lengthen the passes'
// code and raise their register count.
static __device__ __noinline__ PoseErr3 pose_plane_error(const PoseEdgeDev& e, const dSE3 T) {
    PoseErr3 r;
    double (&err)[3] = r.e;
    // localPlane = T * Xw  (Plane3D operator*, Plane3D.h:186-199), or T + Xc for the translation-only edge (:201-209)
    const int kind = e.kind;
    dV3 n = dv(e.a[0], e.a[1], e.a[2]);
    if (kind != PK_PLANE_T) n = mmul(quat_to_matrix(T.q), n);
    double lp[4] = {n.x, n.y, n.z, e.a[3] - ddot(T.t, n)};
    if (lp[3] < 0.0) { lp[0] = -lp[0]; lp[1] = -lp[1]; lp[2] = -lp[2]; lp[3] = -lp[3]; }
    plane_normalize(lp);
    const dV3 ln = dv(lp[0], lp[1], lp[2]), mn = dv(e.a[4], e.a[5], e.a[6]);
    dV3 base = ln;
    if (kind == PK_PAR) {
        if (ddot(mn, ln) < 0) base = -1.0 * ln;
    } else if (kind == PK_VER) {
        const dV3 v = dcross(ln, mn);
        const dV3 ax = (1.0 / sqrt(ddot(v, v))) * v;
        const double ang = 3.14159265358979323846 / 2, c = cos(ang), s = sin(ang);
        base = c * ln + s * dcross(ax, ln) + ((1 - c) * ddot(ax, ln)) * ax;
    }
    const dV3 nn = mmul(plane_rotation_T(base), mn);
    err[0] = azimuth(nn); err[1] = elevation(nn);
    err[2] = (kind == PK_PLANE || kind == PK_PLANE_T) ? ((-lp[3]) - (-e.a[7])) : 0.0;
    return r;
}

// one problem's edge arrays, as the kernel sees them
struct PoseView {
    const float4* A; const float4* B;   // point records of edge 0
    const PoseEdgeDev* W;               // line / plane record of edge n_pt
    const double* PJ;                   // numeric-Jacobian scratch of the first plane edge
    int n_pt, p0, mode;                 // p0: first plane edge
};

// residual of edge i at pose T (computeError of the edge classes), its information diagonal and Huber delta, and with JAC its
// Jacobian (linearizeOplus; plane edges combine the 12 perturbed residuals left in PJ by the pass prologue).  Returns the
// residual dimension.  Everything stays in registers: the caller indexes e / info / J with constants only.
template <bool JAC>
__device__ __forceinline__ int pose_edge_eval(const PoseView& P, int i, const dSE3& T, const PoseCam& K, double (&e)[3], double (&info)[3], double& delta,
                                              double (&J)[3][6]) {
    if (JAC) {
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 6; ++c) J[r][c] = 0;
    }
    if (i < P.n_pt) {
        const float4 a = __ldg(P.A + i), b = __ldg(P.B + i);
        const bool mono = b.y < 0.f;
        const dV3 X = dv(a.x, a.y, a.z);
        const dV3 p = P.mode ? X + T.t : qrot(T.q, X) + T.t;       // mapTrans: Xc + t (se3quat.h:221)
        info[0] = info[1] = info[2] = b.z;
        delta = b.w;
        if (mono) {
            e[0] = (double)a.w - (p.x / p.z * K.fx + K.cx);
            e[1] = (double)b.x - (p.y / p.z * K.fy + K.cy);
            e[2] = 0;
        } else {
            const float invzf = 1.0f / (float)p.z;                  // sic: float reciprocal (types_six_dof_expmap.cpp:300,369)
            const double r0 = p.x * invzf * K.fx + K.cx, r1 = p.y * invzf * K.fy + K.cy, r2 = r0 - K.bf * invzf;
            e[0] = (double)a.w - r0; e[1] = (double)b.x - r1; e[2] = (double)b.y - r2;
        }
        if (JAC) {
            const double x = p.x, y = p.y, invz = 1.0 / p.z, invz_2 = invz * invz;
            if (P.mode == 0) {
                J[0][0] = x * y * invz_2 * K.fx; J[0][1] = -(1 + (x * x * invz_2)) * K.fx; J[0][2] = y * invz * K.fx;
                J[0][3] = -invz * K.fx; J[0][4] = 0; J[0][5] = x * invz_2 * K.fx;
                J[1][0] = (1 + y * y * invz_2) * K.fy; J[1][1] = -x * y * invz_2 * K.fy; J[1][2] = -x * invz * K.fy;
                J[1][3] = 0; J[1][4] = -invz * K.fy; J[1][5] = y * invz_2 * K.fy;
                if (!mono) {
                    J[2][0] = J[0][0] - K.bf * y * invz_2; J[2][1] = J[0][1] + K.bf * x * invz_2; J[2][2] = J[0][2];
                    J[2][3] = J[0][3]; J[2][4] = 0; J[2][5] = J[0][5] - K.bf * invz_2;
                }
            } else {                                                // rotation columns are zero (types_six_dof_expmap.cpp:404-485)
                J[0][3] = -invz * K.fx; J[0][5] = x * invz_2 * K.fx;
                J[1][4] = -invz * K.fy; J[1][5] = y * invz_2 * K.fy;
                if (!mono) { J[2][3] = J[0][3]; J[2][5] = J[0][5] - K.bf * invz_2; }
            }
        }
        return mono ? 2 : 3;
    }
    const PoseEdgeDev& E = P.W[i - P.n_pt];
    info[0] = E.info[0]; info[1] = E.info[1]; info[2] = E.info[2];
    delta = E.delta;
    if (i < P.p0) {                                                 // line start / end edge (EdgeLine.h:155-245)
        const dV3 X = dv(E.a[0], E.a[1], E.a[2]);
        const dV3 p = P.mode ? X + T.t : qrot(T.q, X) + T.t;
        const double lx = E.a[3], ly = E.a[4];
        const double u = p.x / p.z * K.fx + K.cx, v = p.y / p.z * K.fy + K.cy;
        e[0] = lx * u + ly * v + E.a[5]; e[1] = 0; e[2] = 0;
        if (JAC) {
            const double x = p.x, y = p.y, invz = 1.0 / p.z, invz_2 = invz * invz, fx = K.fx, fy = K.fy;
            if (P.mode == 0) {
                J[0][0] = -fy * ly - fx * lx * x * y * invz_2 - fy * ly * y * y * invz_2;
                J[0][1] = fx * lx + fx * lx * x * x * invz_2 + fy * ly * x * y * invz_2;
                J[0][2] = -fx * lx * y * invz + fy * ly * x * invz;
                J[0][3] = fx * lx * invz;
                J[0][4] = fy * ly * invz;
                J[0][5] = -(fx * lx * x + fy * ly * y) * invz_2;
            } else {                                                // EdgeLine.h:283-310
                J[0][3] = fx * lx * invz; J[0][4] = fy * ly * invz; J[0][5] = -(fx * lx * x + fy * ly * y) * invz_2;
            }
        }
        return 3;
    }
    {
        const PoseErr3 r = pose_plane_error(E, T);
        e[0] = r.e[0]; e[1] = r.e[1]; e[2] = r.e[2];
    }
    const int kind = E.kind, dim = kind == PK_PAR || kind == PK_VER ? 2 : 3;
    if (JAC) {
        // numeric central differences with delta = 1e-9 like BaseUnaryEdge::linearizeOplus (the reference does this for
        // every plane edge; an analytic Jacobian would change the iterates)
        const double scalar = 1.0 / (2 * 1e-9);
        const double* q = P.PJ + 36 * (i - P.p0);
#pragma unroll
        for (int d = 0; d < 6; ++d)
#pragma unroll
            for (int r = 0; r < 3; ++r)
                if (r < dim) J[r][d] = scalar * (q[6 * d + r] - q[6 * d + 3 + r]);
        if (kind == PK_PLANE_T) {                                   // EdgePlaneOnlyTranslation zeroes the rotation columns (EdgePlane.h:292-308)
#pragma unroll
            for (int r = 0; r < 3; ++r) { J[r][0] = 0; J[r][1] = 0; J[r][2] = 0; }
        }
    }
    return dim;
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

#define POSE_THREADS 256                 // upper bound of the block size; the single-problem launch of the tracking chain uses it
#define POSE_BATCH_THREADS 64            // block size of batched launches (pose_pipeline.cu)
#define POSE_WARPS (POSE_THREADS / 32)

// deterministic block reduction of NV doubles held per thread; every thread gets the sums in v.  Multi-warp blocks stage
// the warp sums in one of two shared buffers, alternating per call, so one barrier per reduction suffices.
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV], double* s_part /*[2][POSE_WARPS * 28]*/, int& parity) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
        for (int o = 16; o; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (nw == 1) return;
    double* sp = s_part + parity * (POSE_WARPS * 28);
    parity ^= 1;
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < NV; ++k) sp[wid * NV + k] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        double t = 0;
        for (int w = 0; w < nw; ++w) t += sp[w * NV + k];
        v[k] = t;
    }
}

static __device__ __forceinline__ void pose_load(const double* s, dSE3& T) {
    T.q.x = s[0]; T.q.y = s[1]; T.q.z = s[2]; T.q.w = s[3]; T.t = dv(s[4], s[5], s[6]);
}
static __device__ __forceinline__ void pose_store(double* s, const dSE3& T) {
    s[0] = T.q.x; s[1] = T.q.y; s[2] = T.q.z; s[3] = T.q.w; s[4] = T.t.x; s[5] = T.t.y; s[6] = T.t.z;
}

static __global__ void __launch_bounds__(POSE_THREADS) k_pose_optimization(const PoseHeaderDev* __restrict__ headers, const float4* __restrict__ pt_a,
                                                                    const float4* __restrict__ pt_b, const PoseEdgeDev* __restrict__ wide,
                                                                    double* __restrict__ plane_jac, uint8_t* __restrict__ level_all,
                                                                    uint8_t* f_pt, uint8_t* f_line, uint8_t* f_plane, uint8_t* f_par, uint8_t* f_ver,   // may alias (tracking chain)
                                                                    PoseOutDev* __restrict__ outs) {
    const int prob = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const PoseHeaderDev& hd = headers[prob];
    const int ne = hd.n_edges, n_pt = hd.n_pt, mode = hd.mode;
    PoseView P;
    P.A = pt_a + hd.edge_off; P.B = pt_b + hd.edge_off; P.W = wide + hd.wide_off;
    P.n_pt = n_pt; P.p0 = n_pt + 2 * hd.n_line; P.mode = mode;
    double* PJ = plane_jac + (size_t)hd.plane_off * 36;
    P.PJ = PJ;
    const int n_planes = ne - P.p0;
    uint8_t* level = level_all + hd.edge_off;
    PoseCam K;
    K.fx = hd.fx; K.fy = hd.fy; K.cx = hd.cx; K.cy = hd.cy; K.bf = hd.bf;
    uint8_t* fl[5] = {f_pt + hd.flag_off[0], f_line + hd.flag_off[1], f_plane + hd.flag_off[2], f_par + hd.flag_off[3], f_ver + hd.flag_off[4]};

    __shared__ double s_part[2 * POSE_WARPS * 28];
    __shared__ double s_TP[12][7];            // the 12 perturbed poses of the numeric plane Jacobians
    __shared__ double s_H[21];                // upper triangle of H, for thread 0's solves
    __shared__ double s_T[7], s_x[6];         // trial pose, LM step (thread 0 -> all)
    __shared__ int s_ok;
    int parity = 0;

    // initial pose: Converter::toSE3Quat(mTcw) — float entries widened, quaternion from the (not exactly orthonormal) matrix
    dSE3 T0;
    {
        dM3 R;
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R.m[i][j] = hd.Tcw0[i * 4 + j];
        T0.q = qnorm_pos(quat_from_matrix(R));
        T0.t = dv(hd.Tcw0[3], hd.Tcw0[7], hd.Tcw0[11]);
    }
    PoseOutDev& out = outs[prob];
    for (int i = tid; i < 12; i += nt) out.trace_i[i] = -1;
    for (int i = tid; i < 8; i += nt) out.trace_d[i] = 0;
    for (int i = tid; i < hd.n_pt; i += nt) fl[0][i] = 0;
    for (int i = tid; i < hd.n_line; i += nt) fl[1][i] = 0;
    for (int i = tid; i < hd.n_plane; i += nt) fl[2][i] = 0;
    for (int i = tid; i < hd.n_par; i += nt) fl[3][i] = 0;
    for (int i = tid; i < hd.n_ver; i += nt) fl[4][i] = 0;
    for (int i = tid; i < ne; i += nt) level[i] = 0;
    if (tid < 6) s_x[tid] = 0;                // on a failed solve g2o applies the previous step again, even from an earlier round
    __syncthreads();

    if (hd.n_initial < 3) {                       // :985-986: return 0, pose untouched
        if (tid == 0) { for (int i = 0; i < 16; ++i) { out.Tcw[i] = hd.Tcw0[i]; out.Tcw_d[i] = hd.Tcw0[i]; } out.n_inliers = 0; }
        return;
    }

    bool robust = true;                           // Huber is dropped for every edge after round index 2
    dSE3 T = T0, Tt = T0;                         // Tt: pose of the last trial, where the active edges' residuals were last computed
    int nBad_total = 0;
    double lambda = 0, ni = 2;

    for (int it = 0; it < 4; ++it) {
        T = T0;
        int iters = 0, trials_total = 0, nBadLm = 0;
        double chi_final = 0;
        bool ok = true;
        for (int iter = 0; iter < 10 && ok; ++iter) {
            // ---- OptimizationAlgorithmLevenberg::solve: computeActiveErrors and buildSystem at T, in one pass ----
            // H = sum rho1 J^T Omega J (acc[0..20]), b = -sum rho1 J^T Omega e (acc[21..26]), robust chi2 (acc[27])
            if (n_planes > 0) {
                if (tid < 12) {                   // T perturbed by +-1e-9 along each of the 6 coordinates
                    double add[6] = {0, 0, 0, 0, 0, 0};
                    add[tid >> 1] = (tid & 1) ? -1e-9 : 1e-9;
                    pose_store(s_TP[tid], se3_mul(se3_exp(add), T));
                }
                __syncthreads();
                for (int k = tid; k < 12 * n_planes; k += nt) {
                    const int j = k / 12, m = k - 12 * j;
                    dSE3 Tp;
                    pose_load(s_TP[m], Tp);
                    const PoseErr3 r = pose_plane_error(P.W[P.p0 - n_pt + j], Tp);
                    double* q = PJ + 36 * j + 3 * m;
                    q[0] = r.e[0]; q[1] = r.e[1]; q[2] = r.e[2];
                }
                __syncthreads();
            }
            double acc[28];
#pragma unroll
            for (int k = 0; k < 28; ++k) acc[k] = 0;
            for (int i = tid; i < ne; i += nt) {
                if (level[i]) continue;
                double e[3], info[3], delta, J[3][6];
                const int dim = pose_edge_eval<true>(P, i, T, K, e, info, delta, J);
                double c = 0;
#pragma unroll
                for (int r = 0; r < 3; ++r)
                    if (r < dim) c += e[r] * info[r] * e[r];
                double w = 1.0;
                if (robust) { double r0; huber(c, delta, r0, w); c = r0; }
                acc[27] += c;
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    if (r >= dim) break;
                    const double oe = info[r] * e[r];
                    int k = 0;
#pragma unroll
                    for (int a = 0; a < 6; ++a) {
                        acc[21 + a] -= w * J[r][a] * oe;
                        const double wa = w * info[r] * J[r][a];
#pragma unroll
                        for (int b2 = a; b2 < 6; ++b2) acc[k++] += wa * J[r][b2];
                    }
                }
            }
            block_sum<28>(acc, s_part, parity);
            if (tid == 0) {
#pragma unroll
                for (int k = 0; k < 21; ++k) s_H[k] = acc[k];
            }
            double b[6];
#pragma unroll
            for (int j = 0; j < 6; ++j) b[j] = acc[21 + j];
            double currentChi = acc[27];
            const double iniChi = currentChi;
            double tempChi = currentChi;
            if (iter == 0) {
                double mx = 0;
                for (int j = 0; j < 6; ++j) mx = fmax(fabs(acc[j * (13 - j) / 2]), mx);
                lambda = 1e-5 * mx; ni = 2; nBadLm = 0;
            }
            double rho = 0;
            int qmax = 0;
            do {
                const dSE3 backup = T;
                __syncthreads();                  // every thread has read the previous trial's s_T / s_x
                if (tid == 0) {
                    double Hl[6][6], bl[6];
                    int k = 0;
                    for (int a = 0; a < 6; ++a) for (int b2 = a; b2 < 6; ++b2) { Hl[a][b2] = s_H[k]; Hl[b2][a] = s_H[k]; ++k; }
                    for (int a = 0; a < 6; ++a) { Hl[a][a] += lambda; bl[a] = b[a]; }
                    s_ok = solve6(Hl, bl, s_x);   // on failure s_x keeps the previous solution (g2o applies it anyway)
                    pose_store(s_T, se3_mul(se3_exp(s_x), T));
                }
                __syncthreads();
                double x[6];
#pragma unroll
                for (int j = 0; j < 6; ++j) x[j] = s_x[j];
                pose_load(s_T, Tt);
                const bool ok2 = s_ok != 0;
                T = Tt;
                double chi[1] = {0};
                for (int i = tid; i < ne; i += nt) {
                    if (level[i]) continue;
                    double e[3], info[3], delta, J[3][6];
                    const int dim = pose_edge_eval<false>(P, i, T, K, e, info, delta, J);
                    double c = 0;
#pragma unroll
                    for (int r = 0; r < 3; ++r)
                        if (r < dim) c += e[r] * info[r] * e[r];
                    if (robust) { double r0, r1; huber(c, delta, r0, r1); c = r0; }
                    chi[0] += c;
                }
                block_sum<1>(chi, s_part, parity);
                tempChi = chi[0];
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
        // an active edge is judged by its residual at the last trial pose Tt (g2o's stored _error), an outlier by its
        // residual recomputed at the optimised pose T
        double nb[1] = {0};
        for (int i = tid; i < ne; i += nt) {
            double e[3], info[3], delta, J[3][6];
            if (i < n_pt) {
                uint8_t& f = fl[0][i];
                const int dim = pose_edge_eval<false>(P, i, f ? T : Tt, K, e, info, delta, J);
                double c = 0;
#pragma unroll
                for (int r = 0; r < 3; ++r)
                    if (r < dim) c += e[r] * info[r] * e[r];
                const float cf = (float)c;
                if (cf > (dim == 2 ? 5.991f : 7.815f)) { f = 1; level[i] = 1; nb[0] += 1; } else { f = 0; level[i] = 0; }
            } else if (i < P.p0) {
                // start (even) and end (odd) edges of a line are adjacent; the thread owning the start edge classifies both
                if (((i - n_pt) & 1) == 0) {
                    uint8_t& f = fl[1][(i - n_pt) >> 1];
                    // PoseOptimization recomputes both endpoint errors unconditionally (:1087-1088); TranslationOptimization only
                    // for lines currently flagged as outliers (:3598-3601) and keeps a separate nLineBad
                    const dSE3 Tc = (mode == 0 || f) ? T : Tt;
                    double eb[3];
                    pose_edge_eval<false>(P, i, Tc, K, e, info, delta, J);
                    pose_edge_eval<false>(P, i + 1, Tc, K, eb, info, delta, J);
                    const float cs = (float)(e[0] * e[0]), ce = (float)(eb[0] * eb[0]);
                    if (cs > 2 * 5.991f || ce > 2 * 5.991f) { f = 1; level[i] = 1; level[i + 1] = 1; if (mode == 0) nb[0] += 1; }
                    else { f = 0; level[i] = 0; level[i + 1] = 0; }
                }
            } else {
                const PoseEdgeDev& E = P.W[i - n_pt];
                const int kind = E.kind;
                uint8_t& f = (kind == PK_PLANE || kind == PK_PLANE_T ? f_plane + hd.flag_off[2] : kind == PK_PAR ? f_par + hd.flag_off[3] : f_ver + hd.flag_off[4])[E.idx];
                const int dim = pose_edge_eval<false>(P, i, f ? T : Tt, K, e, info, delta, J);
                double c = 0;
#pragma unroll
                for (int r = 0; r < 3; ++r)
                    if (r < dim) c += e[r] * info[r] * e[r];
                const float cf = (float)c;
                const double th = (kind == PK_PLANE || kind == PK_PLANE_T) ? hd.plane_chi : hd.vp_chi;
                if ((double)cf > th) { f = 1; level[i] = 1; nb[0] += 1; } else { f = 0; level[i] = 0; }
            }
        }
        block_sum<1>(nb, s_part, parity);
        nBad_total = (int)(nb[0] + 0.5);
        __syncthreads();                          // the new levels are visible to the next round
        if (it == 2) robust = false;
        if (tid == 0) {
            out.trace_i[3 * it] = iters; out.trace_i[3 * it + 1] = trials_total; out.trace_i[3 * it + 2] = nBad_total;
            out.trace_d[2 * it] = chi_final; out.trace_d[2 * it + 1] = lambda;
        }
        if (ne < 10) break;
    }
    if (tid == 0) {
        const dM3 R = quat_to_matrix(T.q);
        const double tt[3] = {T.t.x, T.t.y, T.t.z};
        for (int i = 0; i < 16; ++i) out.Tcw_d[i] = (i == 15) ? 1.0 : 0.0;
        for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) out.Tcw_d[i * 4 + j] = R.m[i][j]; out.Tcw_d[i * 4 + 3] = tt[i]; }
        for (int i = 0; i < 16; ++i) out.Tcw[i] = (float)out.Tcw_d[i];
        out.n_inliers = hd.n_initial - nBad_total;
    }
}

}  // namespace pslam
