// PlaneMatcher::SearchMapByCoefficients on sm_90a (src/PlaneMatcher.cpp:10-80, Frame::ComputePlaneWorldCoeff src/Frame.cc:815-820).
// Stage 1 (one warp per (frame plane, map plane) pair): normal dot product and the minimum point-to-plane distance over the
// map plane's voxel points (warp-shuffle min).  Stage 2 (one thread per frame plane): the reference's sequential scan over
// the map planes with its shrinking thresholds (closest association, most perpendicular, most parallel).
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "pslam_internal.h"

namespace pslam {

__global__ void __launch_bounds__(256) k_plane_pairs(int n_frame, int n_map, const float* __restrict__ pM /*[n_frame][4]*/, const float* __restrict__ map_coef,
                                                     const int32_t* __restrict__ pts_begin, const int32_t* __restrict__ pts_end, const float* __restrict__ pts,
                                                     float* __restrict__ angle, float* __restrict__ mind) {
    const int pair = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (pair >= n_frame * n_map) return;
    const int i = pair / n_map, j = pair - i * n_map;
    const float a = pM[4 * i], b = pM[4 * i + 1], c = pM[4 * i + 2], d = pM[4 * i + 3];
    float res = 100.f;       // the reference keeps the minimum in a double initialised to 100; every candidate is a float value
    for (int p = pts_begin[j] + lane; p < pts_end[j]; p += 32) res = fminf(res, fabsf(a * pts[3 * p] + b * pts[3 * p + 1] + c * pts[3 * p + 2] + d));
#pragma unroll
    for (int o = 16; o; o >>= 1) res = fminf(res, __shfl_xor_sync(0xffffffffu, res, o));
    if (lane == 0) { angle[pair] = a * map_coef[4 * j] + b * map_coef[4 * j + 1] + c * map_coef[4 * j + 2]; mind[pair] = res; }
}

__global__ void k_plane_assign(int n_frame, int n_map, const uint8_t* __restrict__ map_bad, const float* __restrict__ angle, const float* __restrict__ mind,
                               float dTh, float aTh, float verTh, float parTh, int32_t* __restrict__ match, int32_t* __restrict__ ver,
                               int32_t* __restrict__ par, int32_t* __restrict__ nmatches) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frame) return;
    float ldTh = dTh, lverTh = verTh, lparTh = parTh;
    int m = -1, v = -1, p = -1;
    for (int j = 0; j < n_map; ++j) {
        if (map_bad[j]) continue;
        const float ang = angle[i * n_map + j];
        if (ang > aTh || ang < -aTh) {
            const double res = (double)mind[i * n_map + j];
            if (res < (double)ldTh) { ldTh = (float)res; m = j; continue; }
        }
        if (ang < lverTh && ang > -lverTh) { lverTh = fabsf(ang); v = j; continue; }
        if (ang > lparTh || ang < -lparTh) { lparTh = fabsf(ang); p = j; }
    }
    match[i] = m; ver[i] = v; par[i] = p;
    if (m >= 0) atomicAdd(nmatches, 1);
}

// pM: the frame planes in world coordinates ([n_frame][4]); map plane j's points are pts[pts_begin[j] .. pts_end[j]) (a CSR offset array passes itself and
// itself + 1; the minimum does not depend on the order); ang / mind: [n_frame][n_map] scratch; *nmatches is incremented per matched frame plane
int plane_match_run_dev(pslam_ctx* c, int n_frame, int n_map, const float* pM, const float* map_coef, const uint8_t* map_bad, const int32_t* pts_begin,
                        const int32_t* pts_end, const float* pts, float* ang, float* mind, float dTh, float aTh, float verTh, float parTh, int32_t* match, int32_t* ver, int32_t* par, int32_t* nmatches) {
    PSLAM_LAUNCH(c, "plane_pairs", k_plane_pairs<<<(n_frame * n_map + 7) / 8, 256, 0, c->stream>>>(n_frame, n_map, pM, map_coef, pts_begin, pts_end, pts, ang, mind));
    PSLAM_LAUNCH(c, "plane_assign", k_plane_assign<<<(n_frame + 63) / 64, 64, 0, c->stream>>>(n_frame, n_map, map_bad, ang, mind, dTh, aTh, verTh, parTh, match, ver, par,
                 nmatches));
    return PSLAM_OK;
}

}  // namespace pslam

using namespace pslam;

extern "C" int pslam_plane_match(pslam_ctx* c, const float* Tcw, int n_frame, const float* frame_coef, int n_map, const float* map_coef,
                                 const uint8_t* map_bad, const int32_t* pts_off, const float* pts, float dTh, float aTh, float verTh, float parTh,
                                 int32_t* match, int32_t* ver, int32_t* par) {
    if (!c) return PSLAM_E_INVALID;
    if (n_frame < 0 || n_map < 0 || !Tcw || (n_frame && (!frame_coef || !match || !ver || !par)) || (n_map && (!map_coef || !map_bad || !pts_off)))
        return set_error(c, PSLAM_E_INVALID, "bad plane arrays");
    for (int i = 0; i < n_frame; ++i) match[i] = ver[i] = par[i] = -1;
    if (n_frame == 0 || n_map == 0) return 0;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    // pi_w = Tcw^T pi_c: a 4x4 float product per frame plane, done while packing (double accumulation like cv::gemm)
    std::vector<float> pM((size_t)n_frame * 4);
    for (int i = 0; i < n_frame; ++i)
        for (int r = 0; r < 4; ++r) {
            double s = 0;
            for (int k = 0; k < 4; ++k) s += (double)Tcw[k * 4 + r] * (double)frame_coef[4 * i + k];
            pM[4 * i + r] = (float)s;
        }
    const int npts = pts_off[n_map];
    Slab s;
    const auto d_pM = s.add<float>(pM.size()), d_mc = s.add<float>((size_t)n_map * 4);
    const auto d_bad = s.add<uint8_t>(n_map);
    const auto d_off = s.add<int32_t>(n_map + 1);
    const auto d_pts = s.add<float>((size_t)npts * 3 + 1), d_ang = s.add<float>((size_t)n_frame * n_map), d_min = s.add<float>((size_t)n_frame * n_map);
    const auto d_out = s.add<int32_t>((size_t)n_frame * 3), d_cnt = s.add<int32_t>(1);      // match, ver, par; number of matches
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    s.up(d_pM, pM.data(), st); s.up(d_mc, map_coef, st); s.up(d_bad, map_bad, st); s.up(d_off, pts_off, st); s.up(d_pts, pts, st, (size_t)npts * 3);
    s.zero(d_cnt, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    int32_t* out_d = s[d_out];
    plane_match_run_dev(c, n_frame, n_map, s[d_pM], s[d_mc], s[d_bad], s[d_off], s[d_off] + 1, s[d_pts], s[d_ang], s[d_min], dTh, aTh, verTh, parTh, out_d, out_d + n_frame,
                        out_d + 2 * n_frame, s[d_cnt]);
    std::vector<int32_t> out((size_t)3 * n_frame + 1);
    s.down(out.data(), d_out, st); s.down(out.data() + 3 * n_frame, d_cnt, st);
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    for (int i = 0; i < n_frame; ++i) { match[i] = out[i]; ver[i] = out[n_frame + i]; par[i] = out[2 * n_frame + i]; }
    return out[3 * n_frame];
}
