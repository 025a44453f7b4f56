// Local bundle adjustment on sm_90a: one CTA per problem runs the reference's whole LocalBundleAdjustment numeric core
// (src/Optimizer.cc:2361-2460 around g2o's BlockSolver_6_3 + Levenberg): optimize(5) with Huber kernels, chi-square gating,
// optimize(10) without kernels.  Every stage is a block-wide loop over a static work list built at pack time, so all sums
// have a fixed order (deterministic, and - up to libm ulps in sin/cos/atan2 - the order the CPU restatement uses):
//   edges        thread per edge: residual, analytic Jacobians A (d e / d landmark) and B (d e / d pose), Huber weight,
//                W_e = B^T (w Omega) A;  plane-type edges get g2o's numeric Jacobians, one thread per (edge, column)
//   landmarks    thread per landmark over its CSR edge list: H_ll (3x3), b_l;  per trial D^-1 = (H_ll + lambda I)^-1
//   poses        thread per (key frame, entry) over the key frame's CSR edge list: H_pp (6x6), b_p
//   Schur        thread per (pose-pair block, entry) over the block's precomputed list of (edge, edge) terms:
//                S = H_pp + lambda I - sum W_e1 D^-1 W_e2^T  into shared memory (global memory for windows > 26 free poses)
//   solve        in-place right-looking LDL^T of S in shared memory + column-oriented substitutions, all 512 threads
//   back-subst.  thread per landmark: x_l = D^-1 (b_l - sum W_e^T x_p)
// FP64 throughout, no tensor cores: S is at most a few hundred rows and every product is a 6x3 / 3x3 / 3x6 chain.
//
// Reference semantics: src/Optimizer.cc:1971-2678; Thirdparty/g2o/g2o/core/{block_solver.hpp:140-600,
// base_binary_edge.hpp:55-203, optimization_algorithm_levenberg.cpp:61-189, sparse_optimizer.cpp:166-267,354-435};
// types_six_dof_expmap.cpp:103-232; include/EdgeLine.h:53-153; g2oAddition/{EdgePlane.h:24-126, EdgeVerticalPlane.h:21-108,
// EdgeParallelPlane.h:21-108, VertexPlane.h:24-27, Plane3D.h:84-97}; types_sba.h:52-56.
#pragma once
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

#include "geom_device.cuh"
#include "pslam_internal.h"

namespace pslam {

enum { LK_MONO = 0, LK_STEREO = 1, LK_LINE = 2, LK_PLANE = 3, LK_VER = 4, LK_PAR = 5 };
__host__ __device__ inline int lk_dim(int k) { return (k == LK_MONO || k == LK_VER || k == LK_PAR) ? 2 : 3; }
__host__ __device__ inline bool lk_is_plane(int k) { return k >= LK_PLANE; }

struct LbaEdgeDev {             // 80 bytes, static part of an edge (sorted landmark-major, creation order inside a landmark)
    int32_t kind, kf, lm, orig; // kf / lm: indices local to the problem; orig: creation index (family-major)
    double obs[4];              // points & lines: obs[3]; planes: measured plane (normalised)
    double info[3];
    double delta;               // Huber delta
};

struct LbaHeaderDev {
    int32_t n_kf, n_free, n_lm, n_edges, n_blk, n_plane_edges;
    int32_t kf_off, lm_off, edge_off;        // this problem's slice of the per-key-frame / per-landmark / per-edge arrays
    int32_t kfcsr_off, lmcsr_off, blk_off, blkcsr_off;   // slices of kf_edge_off (n_kf + 1), lm_edge_off (n_lm + 1), blk_ij (n_blk), blk_term_off (n_blk + 1)
    int32_t plane_list_off;                  // slice of plane_edges (sorted edge indices of plane-type edges)
    int32_t col_off;                         // slice of per-free-pose arrays (bp, xp, ...), n_free entries of 6
    int64_t term_off;                        // slice of terms
    int64_t hs_off;                          // slice of the global S buffer (used when S does not fit in shared memory)
    int32_t use_smem, ld;                    // leading dimension of S (odd)
    int32_t n_pt_obs, n_line_obs, n_plane_obs[3];
    int32_t fam_off[5];                      // creation index of the first edge of each family (pt, line, plane, ver, par)
    int32_t flag_off;                        // slice of the erase flags (pt | line | plane | ver | par)
    double plane_chi, vp_chi;
};

struct LbaOutDev {
    int32_t iterations[2], trials[2];
    double chi2[2], lambda[2];
};

struct LbaArrays {
    const LbaHeaderDev* hdr;
    // per key frame
    const float* kf_Tcw0; const uint8_t* kf_fixed; const double* kf_K; const int32_t* kf_col;
    double* kf_T; double* kf_Tb;             // [8] each: quaternion xyzw, translation, pad
    uint8_t* kf_active;
    double* out_Tcw;                         // [16]
    // per free pose column
    double* Hpp; double* bp; double* coeff; double* xp;   // 36, 6, 6, 6
    // per landmark
    const int32_t* lm_type; const double* lm_val0;
    double* lm_val; double* lm_valb;         // [4]
    double* Hll; double* bl; double* Dinv; double* db; double* xl;   // 9, 3, 9, 3, 3
    uint8_t* lm_active;
    // per edge
    const LbaEdgeDev* edges;
    double* err; double* JA; double* JB; double* we; double* re; double* W; double* Y;    // 3, 9, 18, 3, 3, 18, 18
    uint8_t* level;
    const int32_t* orig2sorted;
    // work lists
    const int32_t* kf_edge_off; const int32_t* kf_edge_idx;     // per key frame, creation order
    const int32_t* lm_edge_off;                                 // per landmark (edges are sorted landmark-major: a range)
    const int32_t* plane_edges;
    const int32_t* blk_ij; const int32_t* blk_term_off; const int2* terms;
    double* hs_global;
    uint8_t* flags;
    LbaOutDev* out;
};

#define LBA_THREADS 512
#define LBA_WARPS (LBA_THREADS / 32)

__device__ __forceinline__ double lba_block_sum(double v, double* s_part, double* s_out) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();                         // s_out of the previous call may still be read
    if (lane == 0) s_part[wid] = v;
    __syncthreads();
    if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < LBA_WARPS; ++w) t += s_part[w]; s_out[0] = t; }
    __syncthreads();
    return s_out[0];
}
__device__ __forceinline__ double lba_block_max(double v, double* s_part, double* s_out) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) s_part[wid] = v;
    __syncthreads();
    if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < LBA_WARPS; ++w) t = fmax(t, s_part[w]); s_out[0] = t; }
    __syncthreads();
    return s_out[0];
}
__device__ __forceinline__ int lba_block_or(int v, int* s_flag) {
    __syncthreads();
    if (threadIdx.x == 0) *s_flag = 0;
    __syncthreads();
    if (v) atomicOr(s_flag, 1);
    __syncthreads();
    return *s_flag;
}

__device__ __forceinline__ dSE3 lba_load_pose(const double* p) {
    dSE3 T;
    T.q.x = p[0]; T.q.y = p[1]; T.q.z = p[2]; T.q.w = p[3]; T.t = dv(p[4], p[5], p[6]);
    return T;
}
__device__ __forceinline__ void lba_store_pose(double* p, const dSE3& T) {
    p[0] = T.q.x; p[1] = T.q.y; p[2] = T.q.z; p[3] = T.q.w; p[4] = T.t.x; p[5] = T.t.y; p[6] = T.t.z;
}

// Plane3D::oplus (g2oAddition/Plane3D.h:84-97)
__device__ __noinline__ void lba_plane_oplus(double p[4], const double v[3]) {
    const double az = v[0], el = v[1];
    const double s = sin(el), c = cos(el);
    const dV3 n = dv(c * cos(az), c * sin(az), s);
    const dM3 Rt = plane_rotation_T(dv(p[0], p[1], p[2]));
    const double d = (-p[3]) + v[2];
    p[0] = Rt.m[0][0] * n.x + Rt.m[1][0] * n.y + Rt.m[2][0] * n.z;
    p[1] = Rt.m[0][1] * n.x + Rt.m[1][1] * n.y + Rt.m[2][1] * n.z;
    p[2] = Rt.m[0][2] * n.x + Rt.m[1][2] * n.y + Rt.m[2][2] * n.z;
    p[3] = -d;
    plane_normalize(p);
}

// computeError of EdgePlane / EdgeVerticalPlane / EdgeParallelPlane: (T * plane).ominus*(measurement)
__device__ __noinline__ void lba_plane_error(int kind, const dSE3& T, const double pw[4], const double pm[4], double err[3]) {
    const dV3 n = mmul(quat_to_matrix(T.q), dv(pw[0], pw[1], pw[2]));
    double lp[4] = {n.x, n.y, n.z, pw[3] - ddot(T.t, n)};
    if (lp[3] < 0.0) { lp[0] = -lp[0]; lp[1] = -lp[1]; lp[2] = -lp[2]; lp[3] = -lp[3]; }
    plane_normalize(lp);
    const dV3 ln = dv(lp[0], lp[1], lp[2]), mn = dv(pm[0], pm[1], pm[2]);
    dV3 base = ln;
    if (kind == LK_PAR) {
        if (ddot(mn, ln) < 0) base = -1.0 * ln;
    } else if (kind == LK_VER) {
        const dV3 v = dcross(ln, mn);
        const dV3 ax = (1.0 / sqrt(ddot(v, v))) * v;
        const double ang = 3.14159265358979323846 / 2, c = cos(ang), s = sin(ang);
        base = c * ln + s * dcross(ax, ln) + ((1 - c) * ddot(ax, ln)) * ax;
    }
    const dV3 nn = mmul(plane_rotation_T(base), mn);
    err[0] = azimuth(nn); err[1] = elevation(nn);
    err[2] = kind == LK_PLANE ? ((-lp[3]) - (-pm[3])) : 0.0;
}

__device__ __forceinline__ void lba_point_error(const LbaEdgeDev& e, const dSE3& T, const double* K, const double* X, double err[3]) {
    const dV3 p = qrot(T.q, dv(X[0], X[1], X[2])) + T.t;
    if (e.kind == LK_MONO) {
        err[0] = e.obs[0] - (p.x / p.z * K[0] + K[2]);
        err[1] = e.obs[1] - (p.y / p.z * K[1] + K[3]);
        err[2] = 0;
    } else if (e.kind == LK_STEREO) {
        const float invz = 1.0f / (float)p.z;                       // sic: float reciprocal (types_six_dof_expmap.cpp:150-157)
        const double r0 = p.x * invz * K[0] + K[2], r1 = p.y * invz * K[1] + K[3], r2 = r0 - K[4] * invz;
        err[0] = e.obs[0] - r0; err[1] = e.obs[1] - r1; err[2] = e.obs[2] - r2;
    } else {
        const double u = p.x / p.z * K[0] + K[2], v = p.y / p.z * K[1] + K[3];
        err[0] = e.obs[0] * u + e.obs[1] * v + e.obs[2]; err[1] = 0; err[2] = 0;
    }
}

// in-place LDL^T of the symmetric S (lower triangle, row-major, leading dimension ld) and solution of S x = b.
// Right-looking, so every entry receives its updates in ascending pivot order like the sequential algorithm.
// Returns false (uniformly) when a pivot is not positive.
__device__ __noinline__ bool lba_ldlt_solve(double* S, int n, int ld, double* b /* in: rhs, out: x */, double* s_col, int* s_flag) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int j = 0; j < n; ++j) {
        const double d = S[(size_t)j * ld + j];
        if (!(d > 0)) return false;                                 // same value for every thread
        for (int i = j + 1 + tid; i < n; i += LBA_THREADS) {
            const double v = S[(size_t)i * ld + j] / d;
            S[(size_t)i * ld + j] = v;
            s_col[i] = v;
        }
        __syncthreads();
        for (int i = j + 1 + wid; i < n; i += LBA_WARPS) {
            const double li = s_col[i];
            double* row = S + (size_t)i * ld;
            for (int k = j + 1 + lane; k <= i; k += 32) row[k] -= li * s_col[k] * d;
        }
        __syncthreads();
    }
    // forward: L y = b (column-oriented: ascending k for every row, like the row-oriented sequential loop)
    for (int k = 0; k < n; ++k) {
        const double yk = b[k];
        for (int i = k + 1 + tid; i < n; i += LBA_THREADS) b[i] -= S[(size_t)i * ld + k] * yk;
        __syncthreads();
    }
    for (int i = tid; i < n; i += LBA_THREADS) b[i] /= S[(size_t)i * ld + i];
    __syncthreads();
    // backward: L^T x = y (descending k for every row)
    for (int k = n - 1; k >= 0; --k) {
        const double xk = b[k];
        for (int i = tid; i < k; i += LBA_THREADS) b[i] -= S[(size_t)k * ld + i] * xk;
        __syncthreads();
    }
    (void)s_flag;
    return true;
}

__global__ void __launch_bounds__(LBA_THREADS) k_local_bundle_adjustment(LbaArrays A) {
    extern __shared__ double s_dyn[];
    __shared__ double s_part[LBA_WARPS];
    __shared__ double s_out[1];
    __shared__ int s_flag;

    const int tid = threadIdx.x;
    const LbaHeaderDev& hd = A.hdr[blockIdx.x];
    const int nkf = hd.n_kf, nfree = hd.n_free, nlm = hd.n_lm, ne = hd.n_edges, n = 6 * nfree, ld = hd.ld;
    // slices
    const float* kf_Tcw0 = A.kf_Tcw0 + (size_t)hd.kf_off * 16;
    const uint8_t* kf_fixed = A.kf_fixed + hd.kf_off;
    const double* kf_K = A.kf_K + (size_t)hd.kf_off * 5;
    const int32_t* kf_col = A.kf_col + hd.kf_off;
    double* kf_T = A.kf_T + (size_t)hd.kf_off * 8;
    double* kf_Tb = A.kf_Tb + (size_t)hd.kf_off * 8;
    uint8_t* kf_active = A.kf_active + hd.kf_off;
    double* Hpp = A.Hpp + (size_t)hd.col_off * 36;
    double* bp = A.bp + (size_t)hd.col_off * 6;
    double* coeff = A.coeff + (size_t)hd.col_off * 6;
    double* xp = A.xp + (size_t)hd.col_off * 6;
    const int32_t* lm_type = A.lm_type + hd.lm_off;
    double* lm_val = A.lm_val + (size_t)hd.lm_off * 4;
    double* lm_valb = A.lm_valb + (size_t)hd.lm_off * 4;
    double* Hll = A.Hll + (size_t)hd.lm_off * 9;
    double* bl = A.bl + (size_t)hd.lm_off * 3;
    double* Dinv = A.Dinv + (size_t)hd.lm_off * 9;
    double* db = A.db + (size_t)hd.lm_off * 3;
    double* xl = A.xl + (size_t)hd.lm_off * 3;
    uint8_t* lm_active = A.lm_active + hd.lm_off;
    const LbaEdgeDev* E = A.edges + hd.edge_off;
    double* err = A.err + (size_t)hd.edge_off * 3;
    double* JA = A.JA + (size_t)hd.edge_off * 9;
    double* JB = A.JB + (size_t)hd.edge_off * 18;
    double* we = A.we + (size_t)hd.edge_off * 3;
    double* re = A.re + (size_t)hd.edge_off * 3;
    double* W = A.W + (size_t)hd.edge_off * 18;
    double* Y = A.Y + (size_t)hd.edge_off * 18;
    uint8_t* level = A.level + hd.edge_off;
    const int32_t* o2s = A.orig2sorted + hd.edge_off;
    const int32_t* kf_eoff = A.kf_edge_off + hd.kfcsr_off;
    const int32_t* kf_eidx = A.kf_edge_idx + hd.edge_off;
    const int32_t* lm_eoff = A.lm_edge_off + hd.lmcsr_off;
    const int32_t* plane_edges = A.plane_edges + hd.plane_list_off;
    const int32_t* blk_ij = A.blk_ij + (size_t)hd.blk_off * 2;
    const int32_t* blk_toff = A.blk_term_off + hd.blkcsr_off;
    const int2* terms = A.terms + hd.term_off;
    uint8_t* flags = A.flags + hd.flag_off;
    LbaOutDev& out = A.out[blockIdx.x];

    double* S = hd.use_smem ? s_dyn : A.hs_global + hd.hs_off;
    double* s_bs = hd.use_smem ? s_dyn + (size_t)n * ld : A.hs_global + hd.hs_off + (size_t)n * ld;    // rhs / solution, n
    double* s_col = s_bs + n;                                                                              // n

    // ---- initial estimates: Converter::toSE3Quat(GetPose()), toVector3d(GetWorldPos()), toPlane3D ----
    for (int k = tid; k < nkf; k += LBA_THREADS) {
        const float* T0 = kf_Tcw0 + 16 * k;
        dM3 R;
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R.m[i][j] = T0[i * 4 + j];
        dSE3 T;
        T.q = qnorm_pos(quat_from_matrix(R));
        T.t = dv(T0[3], T0[7], T0[11]);
        lba_store_pose(kf_T + 8 * k, T);
    }
    for (int l = tid; l < nlm; l += LBA_THREADS) for (int i = 0; i < 4; ++i) lm_val[4 * l + i] = A.lm_val0[(size_t)(hd.lm_off + l) * 4 + i];
    for (int i = tid; i < ne; i += LBA_THREADS) { level[i] = 0; err[3 * i] = 0; err[3 * i + 1] = 0; err[3 * i + 2] = 0; }
    for (int i = tid; i < n; i += LBA_THREADS) xp[i] = 0;
    for (int i = tid; i < 3 * nlm; i += LBA_THREADS) xl[i] = 0;
    __syncthreads();

    bool robust = true;
    double lambda = 0, ni = 2;

    // computeActiveErrors + activeRobustChi2
    auto active_chi = [&]() -> double {
        double acc = 0;
        for (int i = tid; i < ne; i += LBA_THREADS) {
            if (level[i]) continue;
            const LbaEdgeDev& e = E[i];
            double e3[3];
            const dSE3 T = lba_load_pose(kf_T + 8 * e.kf);
            if (lk_is_plane(e.kind)) lba_plane_error(e.kind, T, lm_val + 4 * e.lm, e.obs, e3);
            else lba_point_error(e, T, kf_K + 5 * e.kf, lm_val + 4 * e.lm, e3);
            err[3 * i] = e3[0]; err[3 * i + 1] = e3[1]; err[3 * i + 2] = e3[2];
            const int dim = lk_dim(e.kind);
            double c = 0;
            for (int r = 0; r < dim; ++r) c += e3[r] * e.info[r] * e3[r];
            if (robust) { double r0, r1; const double dsqr = e.delta * e.delta;
                if (c <= dsqr) { r0 = c; } else { const double s = sqrt(c); r0 = 2 * s * e.delta - dsqr; } (void)r1; c = r0; }
            acc += c;
        }
        return lba_block_sum(acc, s_part, s_out);
    };

    for (int pass = 0; pass < 2; ++pass) {
        // ---- initializeOptimization(0): active vertices = those with at least one level-0 edge ----
        for (int k = tid; k < nkf; k += LBA_THREADS) {
            int a = 0;
            if (!kf_fixed[k]) for (int q = kf_eoff[k]; q < kf_eoff[k + 1]; ++q) a |= level[kf_eidx[q]] == 0;
            kf_active[k] = (uint8_t)a;
        }
        int any = 0;
        for (int l = tid; l < nlm; l += LBA_THREADS) {
            int a = 0;
            for (int q = lm_eoff[l]; q < lm_eoff[l + 1]; ++q) a |= level[q] == 0;
            lm_active[l] = (uint8_t)a;
            any |= a;
        }
        any = lba_block_or(any, &s_flag);
        for (int i = tid; i < n; i += LBA_THREADS) xp[i] = 0;        // buildStructure -> resizeVector
        for (int i = tid; i < 3 * nlm; i += LBA_THREADS) xl[i] = 0;
        __syncthreads();

        int iters = 0, trials_total = 0, nBad = 0;
        double chi_final = 0;
        bool ok = any != 0;
        const int max_it = pass == 0 ? 5 : 10;
        for (int iter = 0; iter < max_it && ok; ++iter) {
            // ================= OptimizationAlgorithmLevenberg::solve =================
            double currentChi = active_chi();
            const double iniChi = currentChi;
            double tempChi = currentChi;
            // ---- buildSystem: Jacobians ----
            for (int i = tid; i < ne; i += LBA_THREADS) {
                const LbaEdgeDev& e = E[i];
                if (level[i] || lk_is_plane(e.kind)) continue;
                const dSE3 T = lba_load_pose(kf_T + 8 * e.kf);
                const double* K = kf_K + 5 * e.kf;
                const double* X = lm_val + 4 * e.lm;
                const dV3 p = qrot(T.q, dv(X[0], X[1], X[2])) + T.t;
                const dM3 R = quat_to_matrix(T.q);
                const double x = p.x, y = p.y, z = p.z, fx = K[0], fy = K[1], bf = K[4];
                double a[3][3], b[3][6];
#pragma unroll
                for (int r = 0; r < 3; ++r) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) a[r][c] = 0;
#pragma unroll
                    for (int c = 0; c < 6; ++c) b[r][c] = 0;
                }
                if (e.kind == LK_LINE) {                                  // include/EdgeLine.h:73-114
                    const double invz = 1.0 / z, invz_2 = invz * invz, lx = e.obs[0], ly = e.obs[1];
                    b[0][0] = -fy * ly - fx * lx * x * y * invz_2 - fy * ly * y * y * invz_2;
                    b[0][1] = fx * lx + fx * lx * x * x * invz_2 + fy * ly * x * y * invz_2;
                    b[0][2] = -fx * lx * y * invz + fy * ly * x * invz;
                    b[0][3] = fx * lx * invz;
                    b[0][4] = fy * ly * invz;
                    b[0][5] = -(fx * lx * x + fy * ly * y) * invz_2;
                    const double t0 = fx * lx, t1 = fy * ly, t2 = -(fx * lx * x + fy * ly * y) * invz;
#pragma unroll
                    for (int c = 0; c < 3; ++c) a[0][c] = 1. * invz * (t0 * R.m[0][c] + t1 * R.m[1][c] + t2 * R.m[2][c]);
                } else {
                    const double z_2 = z * z;
                    if (e.kind == LK_MONO) {                              // types_six_dof_expmap.cpp:103-139
                        const double t02 = -x / z * fx, t12 = -y / z * fy;
#pragma unroll
                        for (int c = 0; c < 3; ++c) {
                            a[0][c] = -1. / z * (fx * R.m[0][c] + t02 * R.m[2][c]);
                            a[1][c] = -1. / z * (fy * R.m[1][c] + t12 * R.m[2][c]);
                        }
                    } else {                                              // :188-232
#pragma unroll
                        for (int c = 0; c < 3; ++c) {
                            a[0][c] = -fx * R.m[0][c] / z + fx * x * R.m[2][c] / z_2;
                            a[1][c] = -fy * R.m[1][c] / z + fy * y * R.m[2][c] / z_2;
                            a[2][c] = a[0][c] - bf * R.m[2][c] / z_2;
                        }
                    }
                    b[0][0] = x * y / z_2 * fx; b[0][1] = -(1 + (x * x / z_2)) * fx; b[0][2] = y / z * fx;
                    b[0][3] = -1. / z * fx; b[0][4] = 0; b[0][5] = x / z_2 * fx;
                    b[1][0] = (1 + y * y / z_2) * fy; b[1][1] = -x * y / z_2 * fy; b[1][2] = -x / z * fy;
                    b[1][3] = 0; b[1][4] = -1. / z * fy; b[1][5] = y / z_2 * fy;
                    if (e.kind == LK_STEREO) {
                        b[2][0] = b[0][0] - bf * y / z_2; b[2][1] = b[0][1] + bf * x / z_2; b[2][2] = b[0][2];
                        b[2][3] = b[0][3]; b[2][4] = 0; b[2][5] = b[0][5] - bf / z_2;
                    }
                }
#pragma unroll
                for (int r = 0; r < 3; ++r) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) JA[9 * i + 3 * r + c] = a[r][c];
#pragma unroll
                    for (int c = 0; c < 6; ++c) JB[18 * i + 6 * r + c] = b[r][c];
                }
            }
            // numeric Jacobians of the plane-type edges (BaseBinaryEdge::linearizeOplus, delta = 1e-9): one thread per column
            for (int w = tid; w < hd.n_plane_edges * 9; w += LBA_THREADS) {
                const int i = plane_edges[w / 9], d = w % 9;
                if (level[i]) continue;
                const LbaEdgeDev& e = E[i];
                const double delta = 1e-9, scalar = 1.0 / (2 * delta);
                const dSE3 T = lba_load_pose(kf_T + 8 * e.kf);
                double e1[3], e2[3];
                if (d < 3) {
                    double add[3] = {0, 0, 0}, pl[4];
                    add[d] = delta;
                    for (int q = 0; q < 4; ++q) pl[q] = lm_val[4 * e.lm + q];
                    lba_plane_oplus(pl, add);
                    lba_plane_error(e.kind, T, pl, e.obs, e1);
                    add[d] = -delta;
                    for (int q = 0; q < 4; ++q) pl[q] = lm_val[4 * e.lm + q];
                    lba_plane_oplus(pl, add);
                    lba_plane_error(e.kind, T, pl, e.obs, e2);
                    for (int r = 0; r < 3; ++r) JA[9 * i + 3 * r + d] = scalar * (e1[r] - e2[r]);
                } else {
                    double add[6] = {0, 0, 0, 0, 0, 0};
                    add[d - 3] = delta;
                    lba_plane_error(e.kind, se3_mul(se3_exp(add), T), lm_val + 4 * e.lm, e.obs, e1);
                    add[d - 3] = -delta;
                    lba_plane_error(e.kind, se3_mul(se3_exp(add), T), lm_val + 4 * e.lm, e.obs, e2);
                    for (int r = 0; r < 3; ++r) JB[18 * i + 6 * r + d - 3] = scalar * (e1[r] - e2[r]);
                }
            }
            __syncthreads();
            // ---- constructQuadraticForm, per edge: weights and W = B^T (w Omega) A ----
            for (int i = tid; i < ne; i += LBA_THREADS) {
                const LbaEdgeDev& e = E[i];
                const int dim = lk_dim(e.kind);
                double wgt[3] = {0, 0, 0}, rr[3] = {0, 0, 0};
                if (!level[i]) {
                    double w = 1.0;
                    if (robust) {
                        double c = 0;
                        for (int r = 0; r < dim; ++r) c += err[3 * i + r] * e.info[r] * err[3 * i + r];
                        const double dsqr = e.delta * e.delta;
                        if (c > dsqr) w = e.delta / sqrt(c);            // RobustKernelHuber::robustify rho[1] (robust_kernel_impl.cpp:78-91)
                    }
                    for (int r = 0; r < dim; ++r) { wgt[r] = w * e.info[r]; rr[r] = -(e.info[r] * err[3 * i + r]) * w; }
                }
                for (int r = 0; r < 3; ++r) { we[3 * i + r] = wgt[r]; re[3 * i + r] = rr[r]; }
                const bool has_col = !level[i] && kf_col[e.kf] >= 0;
#pragma unroll
                for (int a = 0; a < 6; ++a)
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        double s = 0;
                        if (has_col) for (int r = 0; r < dim; ++r) s += (JB[18 * i + 6 * r + a] * wgt[r]) * JA[9 * i + 3 * r + c];
                        W[18 * i + 3 * a + c] = s;
                    }
            }
            __syncthreads();
            // ---- H_ll, b_l per landmark; H_pp, b_p per (key frame, entry) ----
            double mx = 0;
            for (int l = tid; l < nlm; l += LBA_THREADS) {
                double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, bb[3] = {0, 0, 0};
                for (int i = lm_eoff[l]; i < lm_eoff[l + 1]; ++i) {
                    if (level[i]) continue;
                    const int dim = lk_dim(E[i].kind);
                    for (int r = 0; r < dim; ++r)
#pragma unroll
                        for (int a = 0; a < 3; ++a) {
                            const double ja = JA[9 * i + 3 * r + a];
                            bb[a] += ja * re[3 * i + r];
                            const double wa = ja * we[3 * i + r];
#pragma unroll
                            for (int c = 0; c < 3; ++c) h[3 * a + c] += wa * JA[9 * i + 3 * r + c];
                        }
                }
                for (int q = 0; q < 9; ++q) Hll[9 * l + q] = h[q];
                for (int q = 0; q < 3; ++q) bl[3 * l + q] = bb[q];
                if (lm_active[l]) mx = fmax(mx, fmax(fabs(h[0]), fmax(fabs(h[4]), fabs(h[8]))));
            }
            for (int w = tid; w < nkf * 42; w += LBA_THREADS) {
                const int k = w / 42, q = w % 42, col = kf_col[k];
                if (col < 0) continue;
                double s = 0;
                if (q < 36) {
                    const int a = q / 6, c = q % 6;
                    for (int t = kf_eoff[k]; t < kf_eoff[k + 1]; ++t) {
                        const int i = kf_eidx[t];
                        if (level[i]) continue;
                        const int dim = lk_dim(E[i].kind);
                        for (int r = 0; r < dim; ++r) s += (JB[18 * i + 6 * r + a] * we[3 * i + r]) * JB[18 * i + 6 * r + c];
                    }
                    Hpp[36 * col + q] = s;
                    if (a == c && kf_active[k]) mx = fmax(mx, fabs(s));
                } else {
                    const int a = q - 36;
                    for (int t = kf_eoff[k]; t < kf_eoff[k + 1]; ++t) {
                        const int i = kf_eidx[t];
                        if (level[i]) continue;
                        const int dim = lk_dim(E[i].kind);
                        for (int r = 0; r < dim; ++r) s += JB[18 * i + 6 * r + a] * re[3 * i + r];
                    }
                    bp[6 * col + a] = s;
                }
            }
            mx = lba_block_max(mx, s_part, s_out);
            if (iter == 0) { lambda = 1e-5 * mx; ni = 2; nBad = 0; }      // computeLambdaInit

            double rho = 0;
            int qmax = 0;
            do {
                // push
                for (int i = tid; i < nkf * 8; i += LBA_THREADS) kf_Tb[i] = kf_T[i];
                for (int i = tid; i < nlm * 4; i += LBA_THREADS) lm_valb[i] = lm_val[i];
                // ---- Schur complement (BlockSolver::solve) ----
                for (int l = tid; l < nlm; l += LBA_THREADS) {
                    const double* D = Hll + 9 * l;
                    const double d00 = D[0] + lambda, d11 = D[4] + lambda, d22 = D[8] + lambda;
                    const double c00 = d11 * d22 - D[5] * D[7];
                    const double c10 = D[5] * D[6] - D[3] * d22;
                    const double c20 = D[3] * D[7] - d11 * D[6];
                    const double det = c00 * d00 + c10 * D[1] + c20 * D[2];
                    const double id = 1.0 / det;
                    double I[9];
                    I[0] = c00 * id; I[3] = c10 * id; I[6] = c20 * id;
                    I[1] = (D[2] * D[7] - D[1] * d22) * id;
                    I[4] = (d00 * d22 - D[2] * D[6]) * id;
                    I[7] = (D[1] * D[6] - d00 * D[7]) * id;
                    I[2] = (D[1] * D[5] - D[2] * d11) * id;
                    I[5] = (D[2] * D[3] - d00 * D[5]) * id;
                    I[8] = (d00 * d11 - D[1] * D[3]) * id;
                    for (int q = 0; q < 9; ++q) Dinv[9 * l + q] = I[q];
                    for (int a = 0; a < 3; ++a) db[3 * l + a] = I[3 * a] * bl[3 * l] + I[3 * a + 1] * bl[3 * l + 1] + I[3 * a + 2] * bl[3 * l + 2];
                }
                __syncthreads();
                for (int i = tid; i < ne; i += LBA_THREADS) {
                    const double* I = Dinv + 9 * E[i].lm;
#pragma unroll
                    for (int a = 0; a < 6; ++a)
#pragma unroll
                        for (int c = 0; c < 3; ++c)
                            Y[18 * i + 3 * a + c] = W[18 * i + 3 * a] * I[c] + W[18 * i + 3 * a + 1] * I[3 + c] + W[18 * i + 3 * a + 2] * I[6 + c];
                }
                for (int w = tid; w < nkf * 6; w += LBA_THREADS) {
                    const int k = w / 6, a = w % 6, col = kf_col[k];
                    if (col < 0) continue;
                    double s = 0;
                    for (int t = kf_eoff[k]; t < kf_eoff[k + 1]; ++t) {
                        const int i = kf_eidx[t];
                        const double* dbl = db + 3 * E[i].lm;
                        s += W[18 * i + 3 * a] * dbl[0] + W[18 * i + 3 * a + 1] * dbl[1] + W[18 * i + 3 * a + 2] * dbl[2];
                    }
                    coeff[6 * col + a] = s;
                }
                __syncthreads();
                for (int w = tid; w < hd.n_blk * 36; w += LBA_THREADS) {
                    const int bk = w / 36, a = (w % 36) / 6, c = w % 6;
                    const int ci = blk_ij[2 * bk], cj = blk_ij[2 * bk + 1];
                    double s = 0;
                    if (ci == cj) { s = Hpp[36 * ci + 6 * a + c]; if (a == c) s += lambda; }
                    for (int t = blk_toff[bk]; t < blk_toff[bk + 1]; ++t) {
                        const int2 tm = terms[t];
                        const double* y = Y + 18 * tm.x + 3 * a;
                        const double* ww = W + 18 * tm.y + 3 * c;
                        s -= y[0] * ww[0] + y[1] * ww[1] + y[2] * ww[2];
                    }
                    // lower triangle, row-major: element (row 6 cj + c, column 6 ci + a) of the symmetric S
                    const int row = 6 * cj + c, colm = 6 * ci + a;
                    if (row >= colm) S[(size_t)row * ld + colm] = s;
                }
                for (int i = tid; i < n; i += LBA_THREADS) s_bs[i] = bp[i] - coeff[i];
                __syncthreads();
                const bool ok2 = n == 0 ? true : lba_ldlt_solve(S, n, ld, s_bs, s_col, &s_flag);
                __syncthreads();
                if (ok2) {
                    for (int i = tid; i < n; i += LBA_THREADS) xp[i] = s_bs[i];
                    __syncthreads();
                    for (int l = tid; l < nlm; l += LBA_THREADS) {
                        double cl[3] = {bl[3 * l], bl[3 * l + 1], bl[3 * l + 2]};
                        for (int i = lm_eoff[l]; i < lm_eoff[l + 1]; ++i) {
                            const int col = kf_col[E[i].kf];
                            if (col < 0 || level[i]) continue;
                            const double* x6 = xp + 6 * col;
#pragma unroll
                            for (int c = 0; c < 3; ++c) {
                                double s = 0;
#pragma unroll
                                for (int a = 0; a < 6; ++a) s += W[18 * i + 3 * a + c] * x6[a];
                                cl[c] -= s;
                            }
                        }
                        const double* I = Dinv + 9 * l;
                        for (int a = 0; a < 3; ++a) xl[3 * l + a] = I[3 * a] * cl[0] + I[3 * a + 1] * cl[1] + I[3 * a + 2] * cl[2];
                    }
                }
                __syncthreads();
                // ---- update (oplus); on a failed solve g2o applies the previous x as well ----
                for (int k = tid; k < nkf; k += LBA_THREADS) {
                    if (!kf_active[k]) continue;
                    const dSE3 T = lba_load_pose(kf_T + 8 * k);
                    lba_store_pose(kf_T + 8 * k, se3_mul(se3_exp(xp + 6 * kf_col[k]), T));
                }
                for (int l = tid; l < nlm; l += LBA_THREADS) {
                    if (!lm_active[l]) continue;
                    if (lm_type[l]) lba_plane_oplus(lm_val + 4 * l, xl + 3 * l);
                    else { lm_val[4 * l] += xl[3 * l]; lm_val[4 * l + 1] += xl[3 * l + 1]; lm_val[4 * l + 2] += xl[3 * l + 2]; }
                }
                __syncthreads();
                tempChi = active_chi();
                if (!ok2) tempChi = DBL_MAX;
                rho = currentChi - tempChi;
                double sc = 0;
                for (int k = tid; k < nkf; k += LBA_THREADS) {
                    if (!kf_active[k]) continue;
                    const int col = kf_col[k];
                    for (int a = 0; a < 6; ++a) sc += xp[6 * col + a] * (lambda * xp[6 * col + a] + bp[6 * col + a]);
                }
                for (int l = tid; l < nlm; l += LBA_THREADS) {
                    if (!lm_active[l]) continue;
                    for (int a = 0; a < 3; ++a) sc += xl[3 * l + a] * (lambda * xl[3 * l + a] + bl[3 * l + a]);
                }
                double scale = lba_block_sum(sc, s_part, s_out);
                scale += 1e-3;
                rho /= scale;
                if (rho > 0 && isfinite(tempChi)) {
                    double alpha = 1. - pow((2 * rho - 1), 3.0);
                    alpha = fmin(alpha, 2. / 3.);
                    const double sf = fmax(1. / 3., alpha);
                    lambda *= sf; ni = 2; currentChi = tempChi;
                } else {
                    lambda *= ni; ni *= 2;
                    for (int i = tid; i < nkf * 8; i += LBA_THREADS) kf_T[i] = kf_Tb[i];     // pop
                    for (int i = tid; i < nlm * 4; i += LBA_THREADS) lm_val[i] = lm_valb[i];
                    __syncthreads();
                }
                ++qmax;
            } while (rho < 0 && qmax < 10);
            trials_total += qmax;
            chi_final = currentChi;
            ++iters;
            if (qmax == 10 || rho == 0) ok = false;
            else {
                if ((iniChi - currentChi) * 1e3 < iniChi) ++nBad; else nBad = 0;
                if (nBad >= 3) ok = false;
            }
        }
        if (tid == 0) { out.iterations[pass] = iters; out.trials[pass] = trials_total; out.chi2[pass] = chi_final; out.lambda[pass] = lambda; }

        if (pass == 0) {
            // ---- chi-square gating with the errors left by the last LM trial (:2373-2455), kernels removed ----
            for (int o = tid; o < hd.n_pt_obs; o += LBA_THREADS) {
                const int i = o2s[hd.fam_off[0] + o];
                const LbaEdgeDev& e = E[i];
                double c = 0;
                for (int r = 0; r < lk_dim(e.kind); ++r) c += err[3 * i + r] * e.info[r] * err[3 * i + r];
                const dSE3 T = lba_load_pose(kf_T + 8 * e.kf);
                const double* X = lm_val + 4 * e.lm;
                const double z = (qrot(T.q, dv(X[0], X[1], X[2])) + T.t).z;
                if (c > (e.kind == LK_MONO ? 5.991 : 7.815) || !(z > 0.0)) level[i] = 1;
            }
            for (int o = tid; o < hd.n_line_obs; o += LBA_THREADS) {
                const int i0 = o2s[hd.fam_off[1] + 2 * o], i1 = o2s[hd.fam_off[1] + 2 * o + 1];
                if (err[3 * i0] * err[3 * i0] > 7.815 || err[3 * i1] * err[3 * i1] > 7.815) { level[i0] = 1; level[i1] = 1; }
            }
            for (int t = 0; t < 3; ++t)
                for (int o = tid; o < hd.n_plane_obs[t]; o += LBA_THREADS) {
                    const int i = o2s[hd.fam_off[2 + t] + o];
                    const LbaEdgeDev& e = E[i];
                    double c = 0;
                    for (int r = 0; r < lk_dim(e.kind); ++r) c += err[3 * i + r] * e.info[r] * err[3 * i + r];
                    if (c > (t == 0 ? hd.plane_chi : hd.vp_chi)) level[i] = 1;
                }
            robust = false;
            __syncthreads();
        }
    }

    // ---- erase lists (:2462-2560) and optimised estimates (:2620-2677) ----
    {
        uint8_t* f = flags;
        for (int o = tid; o < hd.n_pt_obs; o += LBA_THREADS) {
            const int i = o2s[hd.fam_off[0] + o];
            const LbaEdgeDev& e = E[i];
            double c = 0;
            for (int r = 0; r < lk_dim(e.kind); ++r) c += err[3 * i + r] * e.info[r] * err[3 * i + r];
            const dSE3 T = lba_load_pose(kf_T + 8 * e.kf);
            const double* X = lm_val + 4 * e.lm;
            const double z = (qrot(T.q, dv(X[0], X[1], X[2])) + T.t).z;
            f[o] = (c > (e.kind == LK_MONO ? 5.991 : 7.815) || !(z > 0.0)) ? 1 : 0;
        }
        f += hd.n_pt_obs;
        for (int o = tid; o < hd.n_line_obs; o += LBA_THREADS) {
            const int i0 = o2s[hd.fam_off[1] + 2 * o], i1 = o2s[hd.fam_off[1] + 2 * o + 1];
            f[o] = (err[3 * i0] * err[3 * i0] > 7.815 || err[3 * i1] * err[3 * i1] > 7.815) ? 1 : 0;
        }
        f += hd.n_line_obs;
        for (int t = 0; t < 3; ++t) {
            for (int o = tid; o < hd.n_plane_obs[t]; o += LBA_THREADS) {
                const int i = o2s[hd.fam_off[2 + t] + o];
                const LbaEdgeDev& e = E[i];
                double c = 0;
                for (int r = 0; r < lk_dim(e.kind); ++r) c += err[3 * i + r] * e.info[r] * err[3 * i + r];
                f[o] = c > (t == 0 ? hd.plane_chi : hd.vp_chi) ? 1 : 0;
            }
            f += hd.n_plane_obs[t];
        }
    }
    for (int k = tid; k < nkf; k += LBA_THREADS) {
        const dSE3 T = lba_load_pose(kf_T + 8 * k);
        const dM3 R = quat_to_matrix(T.q);
        double* M = A.out_Tcw + (size_t)(hd.kf_off + k) * 16;
        const double tt[3] = {T.t.x, T.t.y, T.t.z};
        for (int i = 0; i < 16; ++i) M[i] = (i == 15) ? 1.0 : 0.0;
        for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) M[i * 4 + j] = R.m[i][j]; M[i * 4 + 3] = tt[i]; }
    }
}

}  // namespace pslam
