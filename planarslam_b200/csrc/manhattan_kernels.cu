// Manhattan-frame tracking step on sm_90a - Tracking::TrackManhattanFrame (src/Tracking.cc:763-1157).
// One thread per frame, 8 frames per block (manhattan_body.h: six ordered passes over the frame's surface normals; the sums keep the
// reference's order).  ~0.1 MB of normals per frame are streamed six times from L2; latency-bound, hidden behind the detector kernels
// when thousands of frames are in flight.  Round 2: a warp per frame with an ordered tree reduction once it can be timed.
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "manhattan_body.h"
#include "pslam_internal.h"

namespace pslam {

#define MH_BLOCK 8
static_assert(sizeof(MhResult) == sizeof(pslam_manhattan_result) && sizeof(MhResult) == 92, "pslam_manhattan_result layout");

__global__ void __launch_bounds__(MH_BLOCK) k_track_manhattan(const float* __restrict__ R_last, const float* __restrict__ normals, const int32_t* __restrict__ n_normals,
                                                              int max_normals, const double* __restrict__ dirs, const int32_t* __restrict__ n_dirs, int max_dirs,
                                                              int nframes, pslam_manhattan_result* __restrict__ res, uint8_t* __restrict__ nmask,
                                                              uint8_t* __restrict__ dmask) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    int n = n_normals[f], m = n_dirs[f];
    n = n < 0 ? 0 : (n > max_normals ? max_normals : n);
    m = m < 0 ? 0 : (m > max_dirs ? max_dirs : m);
    MhResult r;
    mh_track(R_last + 9 * (size_t)f, normals + 3 * (size_t)f * max_normals, n, dirs + 3 * (size_t)f * max_dirs, m, r, nmask + (size_t)f * max_normals,
             dmask + (size_t)f * max_dirs);
    for (int i = n; i < max_normals; ++i) nmask[(size_t)f * max_normals + i] = 0;
    for (int i = m; i < max_dirs; ++i) dmask[(size_t)f * max_dirs + i] = 0;
    *reinterpret_cast<MhResult*>(res + f) = r;
}

// ---- warp per frame ------------------------------------------------------------------------------------------------------------------------------------
// Lanes stride over the surface normals / line directions.  Cone membership and all counts are exact; the three mean-shift sums of an axis (double) are
// reduced with a butterfly instead of the reference's index order: they differ from the ordered sums by rounding of doubles (1e-16 relative) before they are
// narrowed to float - the counts, flags and masks are identical, the rotation agrees to float rounding (tests use 2e-6).  Axes stay sequential: the cones of
// axes 2 and 3 are rebuilt from the partly updated matrix (the reference's R_cm aliasing).
__device__ __forceinline__ double mh_warp_sum(double v) { for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o); return v; }
__device__ __forceinline__ int mh_warp_sum(int v) { for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o); return v; }

__global__ void __launch_bounds__(128) k_track_manhattan_warp(const float* __restrict__ R_last, const float* __restrict__ normals_all, const int32_t* __restrict__ n_normals,
                                                              int max_normals, const double* __restrict__ dirs_all, const int32_t* __restrict__ n_dirs, int max_dirs,
                                                              int nframes, pslam_manhattan_result* __restrict__ res_all, uint8_t* __restrict__ nmask_all,
                                                              uint8_t* __restrict__ dmask_all) {
    const int lane = threadIdx.x & 31, f = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (f >= nframes) return;
    int n = n_normals[f], m = n_dirs[f];
    n = n < 0 ? 0 : (n > max_normals ? max_normals : n);
    m = m < 0 ? 0 : (m > max_dirs ? max_dirs : m);
    const float* normals = normals_all + 3 * (size_t)f * max_normals;
    const double* dirs = dirs_all + 3 * (size_t)f * max_dirs;
    uint8_t* nmask = nmask_all + (size_t)f * max_normals;
    uint8_t* dmask = dmask_all + (size_t)f * max_dirs;
    MhResult res;
    float R[9];
    for (int i = 0; i < 9; ++i) { R[i] = R_last[9 * (size_t)f + i]; res.R[i] = 0; }
    for (int a = 0; a < 3; ++a) { res.density[a] = 0; res.found[a] = 0; res.n_cone[a] = 0; res.n_selected[a] = 0; }
    res.svd_applied = 0;
    {   // ProjectSN2Conic, the three axes in one pass over the data
        float T[3][9];
        for (int a = 1; a < 4; ++a) mh_axis_rotation(R, a, T[a - 1]);
        int cnt[3] = {0, 0, 0};
        for (int i = lane; i < max_normals; i += 32) {
            uint8_t mk = 0;
            if (i < n) {
                float q[3];
                for (int a = 1; a < 4; ++a) { mh_rotate_normal(T[a - 1], normals + 3 * i, q); if (mh_lambda(q) < MH_SIN_2018) { mk |= (uint8_t)(8 << a); ++cnt[a - 1]; } }
            }
            nmask[i] = mk;
        }
        for (int i = lane; i < max_dirs; i += 32) {
            uint8_t mk = 0;
            if (i < m) {
                float q[3];
                for (int a = 1; a < 4; ++a) { mh_rotate_dir(T[a - 1], dirs + 3 * i, q); if (mh_lambda(q) < MH_SIN_1018) mk |= (uint8_t)(8 << a); }
            }
            dmask[i] = mk;
        }
        for (int a = 0; a < 3; ++a) res.n_cone[a] = mh_warp_sum(cnt[a]);
    }
    __syncwarp();
    int minNum = n / 20;
    {
        int a = res.n_cone[0], b = res.n_cone[1], c = res.n_cone[2], t;
        if (a > b) { t = a; a = b; b = t; }
        if (b > c) { t = b; b = c; c = t; }
        if (a > b) { t = a; a = b; b = t; }
        if (b < minNum) minNum = (b + a) / 2;
    }
    res.min_num = minNum;
    int nfound = 0;
    for (int a = 1; a < 4; ++a) {
        float T[9], q[3];
        mh_axis_rotation(R, a, T);
        MhShift S;
        S.nx = 0; S.ny = 0; S.den = 0; S.count = 0;
        for (int i = lane; i < n; i += 32) {
            const uint8_t mk = nmask[i];
            if (!(mk & (8 << a))) continue;
            mh_rotate_normal(T, normals + 3 * i, q);
            if (mh_consider(q, S)) nmask[i] = mk | (uint8_t)(1 << (a - 1));
        }
        for (int i = lane; i < m; i += 32) {
            const uint8_t mk = dmask[i];
            if (!(mk & (8 << a))) continue;
            mh_rotate_dir(T, dirs + 3 * i, q);
            if (mh_consider(q, S)) dmask[i] = mk | (uint8_t)(1 << (a - 1));
        }
        S.nx = mh_warp_sum(S.nx); S.ny = mh_warp_sum(S.ny); S.den = mh_warp_sum(S.den); S.count = mh_warp_sum(S.count);
        res.n_selected[a - 1] = S.count;
        if (S.count > minNum) {
            const double sx = S.nx / S.den, sy = S.ny / S.den;
            const float density = (float)(S.den / S.count);
            const float alfa = (float)sqrt(sx * sx + sy * sy);
            const float tr = tanf(alfa) / alfa;
            const float t1[3] = {(float)(tr * sx), (float)(tr * sy), 1.0f};
            float rec[3];
            double nn = 0;
            for (int r = 0; r < 3; ++r) {
                double s = 0;
                for (int k = 0; k < 3; ++k) s += (double)T[3 * k + r] * t1[k];
                rec[r] = (float)s;
            }
            for (int r = 0; r < 3; ++r) nn += (double)rec[r] * rec[r];
            const float inv = (float)(1.0 / sqrt(nn));
            for (int r = 0; r < 3; ++r) rec[r] = rec[r] * inv;
            const double sum = (double)rec[0] + (double)rec[1] + (double)rec[2];
            if (sum != 0) {
                ++nfound;
                res.found[a - 1] = 1;
                res.density[a - 1] = density;
                for (int r = 0; r < 3; ++r) R[3 * r + a - 1] = rec[r];
            }
        }
        __syncwarp();
    }
    if (nfound < 2) {
        for (int i = 0; i < 9; ++i) res.R[i] = R[i];
    } else {
        if (nfound == 2) {
            int ca, cb, target;
            bool swap;
            if (res.found[0] && res.found[1]) { ca = 0; cb = 1; target = 2; swap = false; }
            else if (res.found[1] && res.found[2]) { ca = 1; cb = 2; target = 0; swap = true; }
            else { ca = 0; cb = 2; target = 1; swap = false; }
            float u[3], w[3], x[3];
            for (int r = 0; r < 3; ++r) { u[r] = R[3 * r + (swap ? cb : ca)]; w[r] = R[3 * r + (swap ? ca : cb)]; }
            x[0] = u[1] * w[2] - u[2] * w[1]; x[1] = u[2] * w[0] - u[0] * w[2]; x[2] = u[0] * w[1] - u[1] * w[0];
            for (int r = 0; r < 3; ++r) R[3 * r + target] = x[r];
            const double det = (double)R[0] * ((double)R[4] * R[8] - (double)R[5] * R[7]) - (double)R[1] * ((double)R[3] * R[8] - (double)R[5] * R[6]) +
                               (double)R[2] * ((double)R[3] * R[7] - (double)R[4] * R[6]);
            if (fabs(det + 1) < 0.5)
                for (int r = 0; r < 3; ++r) R[3 * r + target] = -x[r];
        }
        float U[9], Vt[9];
        mh_svd3f(R, U, Vt);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) {
                double s = 0;
                for (int k = 0; k < 3; ++k) s += (double)U[3 * r + k] * Vt[3 * k + c];
                res.R[3 * r + c] = (float)s;
            }
        res.svd_applied = 1;
    }
    if (lane == 0) *reinterpret_cast<MhResult*>(res_all + f) = res;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_track_manhattan_batch_dev(pslam_ctx* c, const float* R_last, const float* normals, const int32_t* n_normals, int max_normals, const double* dirs,
                                    const int32_t* n_dirs, int max_dirs, int nframes, pslam_manhattan_result* res, uint8_t* normal_mask, uint8_t* dir_mask) {
    if (!c) return PSLAM_E_INVALID;
    if (!R_last || !normals || !n_normals || !dirs || !n_dirs || !res || !normal_mask || !dir_mask || nframes < 1 || max_normals < 1 || max_dirs < 1)
        return set_error(c, PSLAM_E_INVALID, "bad manhattan arguments");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    static const bool per_thread = [] { const char* e = std::getenv("PSLAM_MANHATTAN"); return e && !std::strcmp(e, "thread"); }();      // the host-checkable first version
    if (per_thread)
        PSLAM_LAUNCH(c, "track_manhattan", k_track_manhattan<<<(nframes + MH_BLOCK - 1) / MH_BLOCK, MH_BLOCK, 0, c->stream>>>(R_last, normals, n_normals, max_normals, dirs,
                     n_dirs, max_dirs, nframes, res, normal_mask, dir_mask));
    else
        PSLAM_LAUNCH(c, "track_manhattan", k_track_manhattan_warp<<<(nframes + 3) / 4, 128, 0, c->stream>>>(R_last, normals, n_normals, max_normals, dirs, n_dirs, max_dirs,
                     nframes, res, normal_mask, dir_mask));
    return PSLAM_OK;
}

int pslam_track_manhattan_batch(pslam_ctx* c, const float* R_last, const float* normals, const int32_t* n_normals, int max_normals, const double* dirs,
                                const int32_t* n_dirs, int max_dirs, int nframes, pslam_manhattan_result* res, uint8_t* normal_mask, uint8_t* dir_mask) {
    if (!c) return PSLAM_E_INVALID;
    if (!R_last || !normals || !n_normals || !dirs || !n_dirs || !res || !normal_mask || !dir_mask || nframes < 1 || max_normals < 1 || max_dirs < 1)
        return set_error(c, PSLAM_E_INVALID, "bad manhattan arguments");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    const size_t nf = (size_t)nframes;
    Slab s;
    const auto d_R = s.add<float>(nf * 9), d_normals = s.add<float>(nf * max_normals * 3);
    const auto d_n_normals = s.add<int32_t>(nf);
    const auto d_dirs = s.add<double>(nf * max_dirs * 3);
    const auto d_n_dirs = s.add<int32_t>(nf);
    const auto d_res = s.add<pslam_manhattan_result>(nf);
    const auto d_normal_mask = s.add<uint8_t>(nf * max_normals), d_dir_mask = s.add<uint8_t>(nf * max_dirs);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.up(d_R, R_last, st); s.up(d_normals, normals, st); s.up(d_n_normals, n_normals, st); s.up(d_dirs, dirs, st); s.up(d_n_dirs, n_dirs, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    rc = pslam_track_manhattan_batch_dev(c, s[d_R], s[d_normals], s[d_n_normals], max_normals, s[d_dirs], s[d_n_dirs], max_dirs, nframes, s[d_res], s[d_normal_mask],
                                         s[d_dir_mask]);
    if (rc != PSLAM_OK) return rc;
    s.down(res, d_res, st); s.down(normal_mask, d_normal_mask, st); s.down(dir_mask, d_dir_mask, st);
    return s.sync(c, st);
}

}
