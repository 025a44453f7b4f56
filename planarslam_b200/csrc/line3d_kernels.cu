// Per-frame 3-D line fit on sm_90a - Frame::isLineGood (src/Frame.cc:189-267) and the LineExtractor.cpp routines it calls.
// One thread per frame (line3d_body.h explains why the lines of a frame are a sequential chain); a batch of frames is one launch.
// The per-thread scratch (51 points x 96 B + a 3 x 51 SVD panel) lives in local memory.  Latency-bound, about 3-4 MFLOP per frame
// (2 040 3x3 Jacobi SVDs dominate); with thousands of frames in flight it is hidden behind the detector kernels.
#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "line3d_body.h"
#include "pslam_internal.h"

namespace pslam {

// frames per block: the threads of a warp run different frames and diverge (RANSAC early exits, Jacobi sweep counts), so a warp
// carries only 8 frames; 2 368 frames -> 296 blocks, two per SM
#define L3D_BLOCK 8

static_assert(sizeof(L3dKeyLine) == sizeof(pslam_keyline), "KeyLine layout");
static_assert(sizeof(pslam_line3d) == 96, "pslam_line3d layout");

__global__ void __launch_bounds__(L3D_BLOCK) k_lines3d(const pslam_keyline* __restrict__ kl, const int32_t* __restrict__ n_lines, int max_lines,
                                                const uint16_t* __restrict__ depth, int nframes, L3dCam cam, const uint32_t* __restrict__ seed,
                                                const int32_t* __restrict__ skip, pslam_line3d* __restrict__ out, int32_t* __restrict__ n_drawn) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    L3dPoint pts[L3D_MAX_PTS];
    double At[3 * L3D_MAX_PTS];
    int n = n_lines[f];
    if (n < 0) n = 0;
    if (n > max_lines) n = max_lines;
    L3dRand rng;
    l3d_srand(rng, seed[f], skip ? skip[f] : 0);
    const uint16_t* dframe = depth + (size_t)f * cam.w * cam.h;
    for (int i = 0; i < max_lines; ++i) {
        pslam_line3d o;
        if (i < n) {
            L3dLineOut R;
            l3d_line(reinterpret_cast<const L3dKeyLine*>(kl)[(size_t)f * max_lines + i], dframe, cam, rng, pts, At, R);
            for (int c = 0; c < 3; ++c) { o.A[c] = R.A[c]; o.B[c] = R.B[c]; o.director[c] = R.director[c]; }
            o.inliers = R.inliers; o.depth = R.depth; o.n_points = R.n_points; o.n_inliers = R.n_inliers; o.valid = R.valid;
        } else {
            for (int c = 0; c < 3; ++c) { o.A[c] = 0; o.B[c] = 0; o.director[c] = 0; }
            o.inliers = 0; o.depth = -1.0f; o.n_points = 0; o.n_inliers = 0; o.valid = 0;
        }
        out[(size_t)f * max_lines + i] = o;
    }
    n_drawn[f] = rng.drawn;
}

// ---- warp per frame ------------------------------------------------------------------------------------------------------------------------------------
// The lines of a frame stay a sequential chain (one rand() stream), but inside a line the <= 51 samples are independent: lanes own samples j = lane and
// lane + 32 - depth look-up, back-projection, the 3x3 covariance SVD (compPt3dCov), every Mahalanobis distance of a RANSAC hypothesis - and the inlier sets
// are two ballots.  What the reference computes as ordered double sums (the inlier mean, the M x 3 Jacobi SVD of computeLine3d_svd) is evaluated by lane 0 with
// the code of line3d_body.h; arg-min / arg-max scans with "first index wins" become warp reductions on (value, index).  Same bits as l3d_line (tested).
struct L3dWarp {                       // shared memory of one warp
    L3dPoint pts[L3D_MAX_PTS];
    double At[3 * L3D_MAX_PTS];
    int indexes[L3D_MAX_PTS];
    L3dRand rng;
};

__device__ __forceinline__ uint64_t l3d_ballot64(bool lo, bool hi) { return (uint64_t)__ballot_sync(0xffffffffu, lo) | ((uint64_t)__ballot_sync(0xffffffffu, hi) << 32); }

// first index with the smallest value (strict <, scan order) over the points of `set`; lanes hold points lane and lane + 32.  init: the scan's start value
__device__ __forceinline__ int l3d_warp_argmin(double v0, bool ok0, double v1, bool ok1, int lane, double init) {
    double v = init; int idx = -1;
    if (ok0 && v0 < v) { v = v0; idx = lane; }
    if (ok1 && v1 < v) { v = v1; idx = lane + 32; }
    for (int o = 16; o; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (oi >= 0 && (idx < 0 || ov < v || (ov == v && oi < idx))) { v = ov; idx = oi; }
    }
    return idx;
}

// verify3dLine on the warp: same decisions as l3d_verify
__device__ bool l3d_verify_warp(const L3dPoint* pts, int n, uint64_t set, const double* A, const double* B, int lane) {
    const double BA[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]};
    const int j0 = lane, j1 = lane + 32;
    const bool ok0 = j0 < n && ((set >> j0) & 1), ok1 = j1 < n && ((set >> j1) & 1);
    double v0 = 0, v1 = 0;
    if (ok0) { const double d[3] = {pts[j0].pos[0] - A[0], pts[j0].pos[1] - A[1], pts[j0].pos[2] - A[2]}; v0 = l3d_dot3(d, BA); }
    if (ok1) { const double d[3] = {pts[j1].pos[0] - A[0], pts[j1].pos[1] - A[1], pts[j1].pos[2] - A[2]}; v1 = l3d_dot3(d, BA); }
    int idx1 = l3d_warp_argmin(v0, ok0, v1, ok1, lane, 100.0);
    int idx2 = l3d_warp_argmin(-v0, ok0, -v1, ok1, lane, 100.0);                 // v > maxv from -100  <=>  -v < 100
    const int first = set ? (int)(__ffsll((long long)set) - 1) : -1;
    if (idx1 < 0) idx1 = first;
    if (idx2 < 0) idx2 = first;
    const double mid[3] = {(A[0] + B[0]) * 0.5, (A[1] + B[1]) * 0.5, (A[2] + B[2]) * 0.5};
    double C[3], D[3];
    l3d_project(pts[idx1].pos, mid, BA, C);
    l3d_project(pts[idx2].pos, mid, BA, D);
    const double DC[3] = {D[0] - C[0], D[1] - C[1], D[2] - C[2]};
    const double cd = sqrt(DC[0] * DC[0] + DC[1] * DC[1] + DC[2] * DC[2]);
    if (cd < 1e-10) return false;
    unsigned cells = 0;
    if (ok0) { const double d[3] = {pts[j0].pos[0] - C[0], pts[j0].pos[1] - C[1], pts[j0].pos[2] - C[2]}; const double l = fabs(l3d_dot3(d, DC) / cd / cd); cells |= l >= 1 ? 1u << 9 : 1u << (unsigned)floor(l * 10); }
    if (ok1) { const double d[3] = {pts[j1].pos[0] - C[0], pts[j1].pos[1] - C[1], pts[j1].pos[2] - C[2]}; const double l = fabs(l3d_dot3(d, DC) / cd / cd); cells |= l >= 1 ? 1u << 9 : 1u << (unsigned)floor(l * 10); }
    for (int o = 16; o; o >>= 1) cells |= __shfl_xor_sync(0xffffffffu, cells, o);
    return (double)__popc(cells & 1023u) / 10 > 0.7;
}

__device__ void l3d_extract_warp(L3dWarp& S, int n, L3dLineOut& R, int lane) {
    const L3dPoint* pts = S.pts;
    const int pairs = (int)(n * (n - 1) * 0.5);
    const int maxIterNo = pairs < 10 ? pairs : 10;
    const double distThresh = 1.5;
    for (int i = lane; i < n; i += 32) S.indexes[i] = i;
    __syncwarp();
    uint64_t maxSet = 0;
    int maxCount = 0, bestA = 0, bestB = 0;
    const int j0 = lane, j1 = lane + 32;
    for (int iter = 0; iter < maxIterNo; ++iter) {
        if (lane == 0) {
            const int r0 = (int)((uint64_t)l3d_rand(S.rng) % (uint64_t)n);
            int t = S.indexes[0]; S.indexes[0] = S.indexes[r0]; S.indexes[r0] = t;
            const int r1 = 1 + (int)((uint64_t)l3d_rand(S.rng) % (uint64_t)(n - 1));
            t = S.indexes[1]; S.indexes[1] = S.indexes[r1]; S.indexes[r1] = t;
        }
        __syncwarp();
        const int ia = S.indexes[0], ib = S.indexes[1];
        const double* A = pts[ia].pos;
        const double* B = pts[ib].pos;
        const double dAB[3] = {B[0] - A[0], B[1] - A[1], B[2] - A[2]};
        if (sqrt(dAB[0] * dAB[0] + dAB[1] * dAB[1] + dAB[2] * dAB[2]) < 1e-10) continue;
        const uint64_t set = l3d_ballot64(j0 < n && l3d_mah_dist(pts[j0 < n ? j0 : 0], A, B) < distThresh, j1 < n && l3d_mah_dist(pts[j1 < n ? j1 : 0], A, B) < distThresh);
        const int count = __popcll(set);
        if (count > maxCount && l3d_verify_warp(pts, n, set, A, B, lane)) { maxSet = set; maxCount = count; bestA = ia; bestB = ib; }
        if ((double)maxCount > n * 0.6) break;
    }
    double rA[3] = {0, 0, 0}, rB[3] = {0, 0, 0};
    if (maxCount >= 2) {
        double m[3], d[3];
        for (int c = 0; c < 3; ++c) { m[c] = (pts[bestA].pos[c] + pts[bestB].pos[c]) * 0.5; d[c] = pts[bestB].pos[c] - pts[bestA].pos[c]; }
        while (true) {
            double mean[3], vt0[3];
            if (lane == 0) {           // computeLine3d_svd: ordered sums, lane 0 with the code of line3d_body.h
                double mm[3] = {0, 0, 0}, w[3], vt[9];
                for (int i = 0; i < n; ++i)
                    if ((maxSet >> i) & 1) for (int c = 0; c < 3; ++c) mm[c] = mm[c] + pts[i].pos[c];
                const double inv = 1.0 / maxCount;
                for (int c = 0; c < 3; ++c) mm[c] = mm[c] * inv;
                int q = 0;
                for (int i = 0; i < n; ++i)
                    if ((maxSet >> i) & 1) { for (int c = 0; c < 3; ++c) S.At[c * L3D_MAX_PTS + q] = pts[i].pos[c] - mm[c]; ++q; }
                l3d_jacobi3(S.At, maxCount, L3D_MAX_PTS, w, vt);
                for (int c = 0; c < 3; ++c) { mean[c] = mm[c]; vt0[c] = vt[c]; }
            }
            for (int c = 0; c < 3; ++c) { mean[c] = __shfl_sync(0xffffffffu, mean[c], 0); vt0[c] = __shfl_sync(0xffffffffu, vt0[c], 0); }
            const double e2[3] = {mean[0] + vt0[0], mean[1] + vt0[1], mean[2] + vt0[2]};
            const uint64_t set = l3d_ballot64(j0 < n && l3d_mah_dist(pts[j0 < n ? j0 : 0], mean, e2) < distThresh, j1 < n && l3d_mah_dist(pts[j1 < n ? j1 : 0], mean, e2) < distThresh);
            const int count = __popcll(set);
            if (count > maxCount) { maxSet = set; maxCount = count; for (int c = 0; c < 3; ++c) { m[c] = mean[c]; d[c] = vt0[c]; } }
            else break;
        }
        const bool ok0 = j0 < n && ((maxSet >> j0) & 1), ok1 = j1 < n && ((maxSet >> j1) & 1);
        double v0 = 0, v1 = 0;
        if (ok0) { const double dd[3] = {pts[j0].pos[0] - m[0], pts[j0].pos[1] - m[1], pts[j0].pos[2] - m[2]}; v0 = l3d_dot3(dd, d); }
        if (ok1) { const double dd[3] = {pts[j1].pos[0] - m[0], pts[j1].pos[1] - m[1], pts[j1].pos[2] - m[2]}; v1 = l3d_dot3(dd, d); }
        int e1 = l3d_warp_argmin(v0, ok0, v1, ok1, lane, 100.0), e2i = l3d_warp_argmin(-v0, ok0, -v1, ok1, lane, 100.0);
        const int first = maxSet ? (int)(__ffsll((long long)maxSet) - 1) : -1;
        if (e1 < 0) e1 = first;
        if (e2i < 0) e2i = first;
        for (int c = 0; c < 3; ++c) { rA[c] = pts[e1].pos[c]; rB[c] = pts[e2i].pos[c]; }
    }
    const double ab[3] = {rA[0] - rB[0], rA[1] - rB[1], rA[2] - rB[2]};
    const double nn = sqrt(l3d_dot3(ab, ab));
    for (int c = 0; c < 3; ++c) { R.director[c] = ab[c] / nn; R.A[c] = rA[c]; R.B[c] = rB[c]; }
    R.inliers = maxSet;
    R.n_inliers = maxCount;
}

#define L3D_WARPS 4
__global__ void __launch_bounds__(L3D_WARPS * 32) k_lines3d_warp(const pslam_keyline* __restrict__ kl, const int32_t* __restrict__ n_lines, int max_lines,
                                                                 const uint16_t* __restrict__ depth, int nframes, L3dCam cam, const uint32_t* __restrict__ seed,
                                                                 const int32_t* __restrict__ skip, pslam_line3d* __restrict__ out, int32_t* __restrict__ n_drawn) {
    extern __shared__ __align__(16) unsigned char l3d_smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int f = blockIdx.x * L3D_WARPS + wid;
    if (f >= nframes) return;
    L3dWarp& S = reinterpret_cast<L3dWarp*>(l3d_smem)[wid];
    int n = n_lines[f];
    if (n < 0) n = 0;
    if (n > max_lines) n = max_lines;
    if (lane == 0) l3d_srand(S.rng, seed[f], skip ? skip[f] : 0);
    __syncwarp();
    const uint16_t* dframe = depth + (size_t)f * cam.w * cam.h;
    for (int i = 0; i < max_lines; ++i) {
        L3dLineOut R;
        R.valid = 0; R.depth = -1.0f; R.n_points = 0; R.n_inliers = 0; R.inliers = 0;
        for (int c = 0; c < 3; ++c) { R.A[c] = 0; R.B[c] = 0; R.director[c] = 0; }
        if (i < n) {
            const L3dKeyLine k = reinterpret_cast<const L3dKeyLine*>(kl)[(size_t)f * max_lines + i];
            const float ddx = k.startPointX - k.endPointX, ddy = k.startPointY - k.endPointY;
            const double len = sqrt((double)ddx * ddx + (double)ddy * ddy);
            const int ilen = (int)len;
            const double numSmp = (double)(ilen < 50 ? ilen : 50);
            int np = 0;
            if (numSmp >= 1) {
                // lanes own samples j = lane, lane + 32 (j <= numSmp <= 50); the kept ones are compacted in order
                double px3[2][3]; bool keep[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int j = lane + 32 * h;
                    keep[h] = false;
                    if ((double)j <= numSmp) {
                        const double t1 = 1 - j / numSmp, t2 = j / numSmp;
                        const float px = (float)(k.startPointX * t1) + (float)(k.endPointX * t2);
                        const float py = (float)(k.startPointY * t1) + (float)(k.endPointY * t2);
                        const double ptx = px, pty = py;
                        if (!(ptx < 0 || pty < 0 || ptx >= cam.w || pty >= cam.h)) {
                            int row, col;
                            if (floor(ptx) == ptx && floor(pty) == pty) { col = (int)(ptx - 1); if (col < 0) col = 0; row = (int)(pty - 1); if (row < 0) row = 0; }
                            else { col = (int)ptx; row = (int)pty; }
                            const float dv = (float)dframe[(size_t)row * cam.w + col] * cam.depth_factor;
                            if (!((double)dv <= 0.01)) {
                                keep[h] = true;
                                px3[h][2] = dv;
                                px3[h][0] = (double)((float)col - cam.cx) * px3[h][2] * (double)cam.invfx;
                                px3[h][1] = (double)((float)row - cam.cy) * px3[h][2] * (double)cam.invfy;
                            }
                        }
                    }
                }
                const unsigned m0 = __ballot_sync(0xffffffffu, keep[0]), m1 = __ballot_sync(0xffffffffu, keep[1]);
                const unsigned lt = (1u << lane) - 1u;
                if (keep[0]) { L3dPoint& p = S.pts[__popc(m0 & lt)]; p.pos[0] = px3[0][0]; p.pos[1] = px3[0][1]; p.pos[2] = px3[0][2]; }
                if (keep[1]) { L3dPoint& p = S.pts[__popc(m0) + __popc(m1 & lt)]; p.pos[0] = px3[1][0]; p.pos[1] = px3[1][1]; p.pos[2] = px3[1][2]; }
                np = __popc(m0) + __popc(m1);
                __syncwarp();
            }
            R.n_points = np;
            if (np >= 10) {
                for (int j = lane; j < np; j += 32) l3d_point_cov(S.pts[j], (double)cam.fx);
                __syncwarp();
                l3d_extract_warp(S, np, R, lane);
                const double ab[3] = {R.A[0] - R.B[0], R.A[1] - R.B[1], R.A[2] - R.B[2]};
                if ((double)R.n_inliers / len > 0.4 && sqrt(l3d_dot3(ab, ab)) > 0.02) {
                    R.valid = 1;
                    const float de = (float)dframe[(size_t)(int)k.endPointY * cam.w + (int)k.endPointX] * cam.depth_factor;
                    const float ds = (float)dframe[(size_t)(int)k.startPointY * cam.w + (int)k.startPointX] * cam.depth_factor;
                    R.depth = ds < de ? ds : de;
                } else {
                    for (int c = 0; c < 3; ++c) { R.A[c] = 0; R.B[c] = 0; }
                }
                __syncwarp();
            }
        }
        if (lane == 0) {
            pslam_line3d o;
            for (int c = 0; c < 3; ++c) { o.A[c] = R.A[c]; o.B[c] = R.B[c]; o.director[c] = R.director[c]; }
            o.inliers = R.inliers; o.depth = R.depth; o.n_points = R.n_points; o.n_inliers = R.n_inliers; o.valid = R.valid;
            out[(size_t)f * max_lines + i] = o;
        }
    }
    __syncwarp();
    if (lane == 0) n_drawn[f] = S.rng.drawn;
}

static int lines3d_launch(pslam_ctx* c, const pslam_keyline* d_kl, const int32_t* d_nl, int max_lines, const uint16_t* d_depth, int nframes, float depth_factor,
                          const float* cam4, const uint32_t* d_seed, const int32_t* d_skip, pslam_line3d* d_out, int32_t* d_drawn) {
    L3dCam cam;
    cam.w = c->cfg.width; cam.h = c->cfg.height;
    cam.fx = cam4[0]; cam.fy = cam4[1]; cam.cx = cam4[2]; cam.cy = cam4[3];
    cam.invfx = 1.0f / cam.fx; cam.invfy = 1.0f / cam.fy;                      // src/Frame.cc:77-78
    cam.depth_factor = depth_factor;
    static const bool per_thread = [] { const char* e = std::getenv("PSLAM_LINES3D"); return e && !std::strcmp(e, "thread"); }();      // the host-checkable first version
    if (per_thread) {
        PSLAM_LAUNCH(c, "lines3d", k_lines3d<<<(nframes + L3D_BLOCK - 1) / L3D_BLOCK, L3D_BLOCK, 0, c->stream>>>(d_kl, d_nl, max_lines, d_depth, nframes, cam, d_seed, d_skip, d_out, d_drawn));
    } else {
        const size_t smem = L3D_WARPS * sizeof(L3dWarp);
        PSLAM_CUDA(c, cudaFuncSetAttribute(k_lines3d_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        PSLAM_LAUNCH(c, "lines3d", k_lines3d_warp<<<(nframes + L3D_WARPS - 1) / L3D_WARPS, L3D_WARPS * 32, smem, c->stream>>>(d_kl, d_nl, max_lines, d_depth, nframes, cam, d_seed,
                     d_skip, d_out, d_drawn));
    }
    return PSLAM_OK;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_lines3d_batch_dev(pslam_ctx* c, const pslam_keyline* keylines, const int32_t* n_lines, int max_lines, const uint16_t* depth, int nframes,
                            float depth_factor, const float* cam, const uint32_t* seed, const int32_t* skip, pslam_line3d* out, int32_t* n_drawn) {
    if (!c) return PSLAM_E_INVALID;
    if (!keylines || !n_lines || !depth || !cam || !seed || !out || !n_drawn || nframes < 1 || max_lines < 1 || cam[0] == 0 || cam[1] == 0)        // fy < 0 is legal (Examples/RGB-D/ICL.yaml:9)
        return set_error(c, PSLAM_E_INVALID, "bad lines3d arguments");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return lines3d_launch(c, keylines, n_lines, max_lines, depth, nframes, depth_factor, cam, seed, skip, out, n_drawn);
}

int pslam_lines3d_batch(pslam_ctx* c, const pslam_keyline* keylines, const int32_t* n_lines, int max_lines, const uint16_t* depth, int nframes, float depth_factor,
                        const float* cam, const uint32_t* seed, const int32_t* skip, pslam_line3d* out, int32_t* n_drawn) {
    if (!c) return PSLAM_E_INVALID;
    if (!keylines || !n_lines || !depth || !cam || !seed || !out || !n_drawn || nframes < 1 || max_lines < 1 || cam[0] == 0 || cam[1] == 0)        // fy < 0 is legal (Examples/RGB-D/ICL.yaml:9)
        return set_error(c, PSLAM_E_INVALID, "bad lines3d arguments");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    const size_t npx = (size_t)c->cfg.width * c->cfg.height, nf = (size_t)nframes;
    Slab s;
    const auto d_kl = s.add<pslam_keyline>(nf * max_lines);
    const auto d_n_lines = s.add<int32_t>(nf);
    const auto d_depth = s.add<uint16_t>(nf * npx);
    const auto d_seed = s.add<uint32_t>(nf);
    const auto d_skip = s.add<int32_t>(nf);
    const auto d_out = s.add<pslam_line3d>(nf * max_lines);
    const auto d_n_drawn = s.add<int32_t>(nf);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.up(d_kl, keylines, st); s.up(d_n_lines, n_lines, st); s.up(d_depth, depth, st); s.up(d_seed, seed, st);
    if (skip) s.up(d_skip, skip, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    rc = lines3d_launch(c, s[d_kl], s[d_n_lines], max_lines, s[d_depth], nframes, depth_factor, cam, s[d_seed], skip ? s[d_skip] : nullptr, s[d_out], s[d_n_drawn]);
    if (rc != PSLAM_OK) return rc;
    s.down(out, d_out, st); s.down(n_drawn, d_n_drawn, st);
    return s.sync(c, st);
}

}
