// LSDmatcher::SearchByProjection(Frame&, const vector<MapLine*>&, th) on sm_90a (src/LSDmatcher.cpp:141-211, Frame::GetLinesInArea
// src/Frame.cc:491-523).  One warp per frame: the map lines are visited in order (an assignment changes which frame lines
// later map lines may take), the <= 64 frame lines of a frame are evaluated by the lanes (gates + 256-bit Hamming distance),
// and the best / second-best bookkeeping of the reference's scan is replayed in index order over the lane results.
#include <cuda_runtime.h>

#include <cstdint>

#include "pslam_internal.h"

namespace pslam {

#define LS_MAX_LINES 64

__global__ void __launch_bounds__(32) k_line_search(int nf, const float* __restrict__ pt, const float* __restrict__ angle, const int32_t* __restrict__ octave,
                                                    const uint8_t* __restrict__ desc, const uint8_t* __restrict__ has_obs, const float* __restrict__ scale,
                                                    int n_levels, int nm, const uint8_t* __restrict__ skip, const int32_t* __restrict__ level,
                                                    const float* __restrict__ view_cos, const float* __restrict__ proj, const uint8_t* __restrict__ mdesc,
                                                    const uint8_t* __restrict__ m_has_obs, float th, float nnratio, int32_t* __restrict__ assigned,
                                                    int32_t* __restrict__ nmatches) {
    const int lane = threadIdx.x;
    __shared__ uint32_t s_desc[LS_MAX_LINES][8];
    __shared__ uint8_t s_occ[LS_MAX_LINES];
    for (int i = lane; i < nf * 8; i += 32) s_desc[i / 8][i % 8] = reinterpret_cast<const uint32_t*>(desc)[i];
    for (int i = lane; i < nf; i += 32) { s_occ[i] = has_obs[i]; assigned[i] = -1; }
    __syncwarp();
    const bool bFactor = th != 1.0f;
    int count = 0;
    for (int m = 0; m < nm; ++m) {
        if (skip[m]) continue;
        const int lv = level[m];
        float r = view_cos[m] > 0.998 ? 5.0f : 8.0f;
        if (bFactor) r = __fmul_rn(r, th);
        const float x1 = proj[4 * m], y1 = proj[4 * m + 1], x2 = proj[4 * m + 2], y2 = proj[4 * m + 3];
        const float rr = __fmul_rn(r, scale[min(max(lv, 0), n_levels - 1)]);   // MapLine::PredictScale does not clamp and the reference reads past mvScaleFactors;
                                                                               // the scale index is clamped here, the level gate below keeps the raw level
        const int minLevel = lv - 1, maxLevel = lv;
        const bool bCheckLevels = (minLevel > 0) || (maxLevel > 0);
        uint32_t md[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) md[q] = reinterpret_cast<const uint32_t*>(mdesc)[8 * m + q];
        int dist_l[2] = {-1, -1};            // -1: not in area, -2: in area but occupied, >= 0: Hamming distance
        bool any = false;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = lane + 32 * h;
            if (i >= nf) continue;
            const double mx = 0.5 * (double)__fadd_rn(x1, x2) - (double)pt[2 * i], my = 0.5 * (double)__fadd_rn(y1, y2) - (double)pt[2 * i + 1];
            const float distance = (float)(mx * mx + my * my);
            if (distance > __fmul_rn(rr, rr)) continue;
            const float slope = __fsub_rn(__fdiv_rn(__fsub_rn(y1, y2), __fsub_rn(x1, x2)), angle[i]);
            if ((double)slope > (double)rr * 0.01) continue;
            if (bCheckLevels) {
                if (octave[i] < minLevel) continue;
                if (maxLevel >= 0 && octave[i] > maxLevel) continue;
            }
            any = true;
            if (s_occ[i]) { dist_l[h] = -2; continue; }
            int d = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) d += __popc(md[q] ^ s_desc[i][q]);
            dist_l[h] = d;
        }
        if (!__any_sync(0xffffffffu, any)) continue;
        int bestDist = 256, bestLevel = -1, bestDist2 = 256, bestLevel2 = -1, bestIdx = -1;
        for (int i = 0; i < nf; ++i) {                       // the reference's scan, in index order
            const int d = __shfl_sync(0xffffffffu, dist_l[i >> 5], i & 31);
            if (d < 0) continue;
            if (d < bestDist) { bestDist2 = bestDist; bestDist = d; bestLevel2 = bestLevel; bestLevel = octave[i]; bestIdx = i; }
            else if (d < bestDist2) { bestLevel2 = octave[i]; bestDist2 = d; }
        }
        if (bestDist <= 100) {
            if (bestLevel == bestLevel2 && (float)bestDist > __fmul_rn(nnratio, (float)bestDist2)) continue;
            if (lane == 0) { assigned[bestIdx] = m; s_occ[bestIdx] = m_has_obs[m]; }
            __syncwarp();
            ++count;
        }
    }
    if (lane == 0) *nmatches = count;
}

int line_search_run_dev(pslam_ctx* c, int nf, const float* pt, const float* angle, const int32_t* octave, const uint8_t* desc, const uint8_t* has_obs, const float* scale,
                        int n_levels, int nm, const uint8_t* skip, const int32_t* level, const float* view_cos, const float* proj, const uint8_t* mdesc,
                        const uint8_t* m_has_obs, float th, float nnratio, int32_t* assigned, int32_t* nmatches) {
    PSLAM_LAUNCH(c, "line_search", k_line_search<<<1, 32, 0, c->stream>>>(nf, pt, angle, octave, desc, has_obs, scale, n_levels, nm, skip, level, view_cos, proj, mdesc,
                 m_has_obs, th, nnratio, assigned, nmatches));
    return PSLAM_OK;
}

}  // namespace pslam

using namespace pslam;

extern "C" int pslam_line_search_by_projection(pslam_ctx* c, int nf, const float* pt, const float* angle, const int32_t* octave, const uint8_t* desc,
                                               const uint8_t* has_obs, const float* scale_factors, int n_levels, int nm, const uint8_t* skip,
                                               const int32_t* level, const float* view_cos, const float* proj, const uint8_t* mdesc,
                                               const uint8_t* m_has_obs, float th, float nnratio, int32_t* assigned) {
    if (!c) return PSLAM_E_INVALID;
    if (nf < 0 || nf > LS_MAX_LINES || nm < 0 || n_levels < 1 || (nf && (!pt || !angle || !octave || !desc || !has_obs || !assigned)) || !scale_factors ||
        (nm && (!skip || !level || !view_cos || !proj || !mdesc || !m_has_obs)))
        return set_error(c, PSLAM_E_INVALID, "bad line-search arrays (at most 64 frame lines)");
    for (int i = 0; i < nf; ++i) assigned[i] = -1;
    if (nf == 0 || nm == 0) return 0;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    // small POD arrays: one staging allocation per call (a live tracker calls this once per frame)
    Slab s;
    const auto d_pt = s.add<float>((size_t)nf * 2), d_angle = s.add<float>(nf);
    const auto d_octave = s.add<int32_t>(nf);
    const auto d_desc = s.add<uint8_t>((size_t)nf * 32), d_has_obs = s.add<uint8_t>(nf);
    const auto d_scale = s.add<float>(n_levels);
    const auto d_skip = s.add<uint8_t>(nm);
    const auto d_level = s.add<int32_t>(nm);
    const auto d_view_cos = s.add<float>(nm), d_proj = s.add<float>((size_t)nm * 4);
    const auto d_mdesc = s.add<uint8_t>((size_t)nm * 32), d_m_has_obs = s.add<uint8_t>(nm);
    const auto d_assigned = s.add<int32_t>(nf), d_n = s.add<int32_t>(1);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.up(d_pt, pt, st); s.up(d_angle, angle, st); s.up(d_octave, octave, st); s.up(d_desc, desc, st); s.up(d_has_obs, has_obs, st); s.up(d_scale, scale_factors, st);
    s.up(d_skip, skip, st); s.up(d_level, level, st); s.up(d_view_cos, view_cos, st); s.up(d_proj, proj, st); s.up(d_mdesc, mdesc, st); s.up(d_m_has_obs, m_has_obs, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    line_search_run_dev(c, nf, s[d_pt], s[d_angle], s[d_octave], s[d_desc], s[d_has_obs], s[d_scale], n_levels, nm, s[d_skip], s[d_level], s[d_view_cos], s[d_proj],
                        s[d_mdesc], s[d_m_has_obs], th, nnratio, s[d_assigned], s[d_n]);
    int32_t n = 0;
    s.down(assigned, d_assigned, st); s.down(&n, d_n, st);
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    return n;
}
