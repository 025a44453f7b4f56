// Projection-guided descriptor search for sm_90a (one frame + one map snapshot per call; frames of a replayed
// sequence are issued back to back on the context's stream).
//
// Reference semantics: Frame::AssignFeaturesToGrid / PosInGrid src/Frame.cc:155-168,526-535; Frame::GetFeaturesInArea :440-489;
// Frame::isInFrustum :312-367; MapPoint::PredictScale src/MapPoint.cc:419-434; ORBmatcher::SearchByProjection(Frame&,
// vector<MapPoint*>&, th) src/ORBmatcher.cc:46-130; ORBmatcher::SearchByProjection(Frame&, const Frame&, th, bMono)
// :1396-1535; ComputeThreeMaxima :1666-1707.  Arithmetic conventions as in oracle/search.h (float cv::Mat products and
// cv::norm accumulate in double; log() of PredictScale in double; no FMA: the file is built with --fmad=false).
//
// Work decomposition:
//   k_search_grid        one CTA: sort keypoints by (cell, index) -> the reference's per-cell lists in push order
//   k_candidates_*       one warp per map point / last-frame keypoint: projection, window cells in (ix, iy) order, level and
//                        stereo gates, 256-bit Hamming distance by popcount; ordered candidate list per point (ballot compaction)
//   k_resolve_*          one warp: the reference's sequential greedy assignment (a keypoint that already holds a map point
//                        with observations is skipped by later points), top-2 / top-1 by warp-shuffle merge per point
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <vector>

#include "pslam_internal.h"

namespace pslam {

#define SG_COLS 64
#define SG_ROWS 48
#define SG_CELLS (SG_COLS * SG_ROWS)
#define SEARCH_CAND_CAP 128
#define SEARCH_MAX_KP 4096

struct SearchFrameDev {
    int n;
    const pslam_keypoint* keys_un; const float* u_right; const uint8_t* desc;
    float Tcw[16];
    const float* Tcw_dev;      // device-resident chain (track_chain.cu): pose and key-point count live in HBM; nullptr -> the by-value fields
    const int32_t* n_dev;
    float fx, fy, cx, cy, bf, min_x, max_x, min_y, max_y;
    int n_levels; float scale[PSLAM_MAX_LEVELS]; float log_scale_factor;
    float inv_w, inv_h;
};
struct SearchMapDev {
    int n;
    const float *pos, *normal, *max_distance, *min_distance; const uint8_t *desc, *skip, *has_obs;
};

__device__ __forceinline__ const float* frame_T(const SearchFrameDev& F) { return F.Tcw_dev ? F.Tcw_dev : F.Tcw; }
__device__ __forceinline__ int frame_n(const SearchFrameDev& F) { return F.n_dev ? min(*F.n_dev, F.n) : F.n; }

// ---- grid: sorted (cell << 16 | index) keys; keypoints outside the grid get cell = SG_CELLS (sorted to the end) ----
static __global__ void __launch_bounds__(1024) k_search_grid(SearchFrameDev F, int32_t* __restrict__ cell_start /*[SG_CELLS+1]*/, int32_t* __restrict__ items /*[n]*/) {
    __shared__ uint32_t keys[SEARCH_MAX_KP];
    const int tid = threadIdx.x;
    const int Fn = frame_n(F);
    for (int i = tid; i < SEARCH_MAX_KP; i += 1024) {
        uint32_t k = 0xffffffffu;
        if (i < Fn) {
            const int px = (int)roundf((F.keys_un[i].x - F.min_x) * F.inv_w), py = (int)roundf((F.keys_un[i].y - F.min_y) * F.inv_h);
            const int cell = (px < 0 || px >= SG_COLS || py < 0 || py >= SG_ROWS) ? SG_CELLS : px * SG_ROWS + py;     // mGrid[x][y]
            k = ((uint32_t)cell << 16) | (uint32_t)i;
        }
        keys[i] = k;
    }
    __syncthreads();
    for (int size = 2; size <= SEARCH_MAX_KP; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < SEARCH_MAX_KP / 2; i += 1024) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool up = ((lo & size) == 0);
                const uint32_t a = keys[lo], b = keys[hi];
                if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
            }
            __syncthreads();
        }
    for (int i = tid; i < Fn; i += 1024) items[i] = (int)(keys[i] & 0xffff);
    for (int c = tid; c <= SG_CELLS; c += 1024) {      // cell_start[c] = first position whose cell >= c (binary search)
        int lo = 0, hi = Fn;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if ((int)(keys[mid] >> 16) < c) lo = mid + 1; else hi = mid; }
        cell_start[c] = lo;
    }
}

__device__ __forceinline__ void mat_rt(const float* T, const float* P, float out[3]) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float m = (float)((double)T[4 * r] * P[0] + (double)T[4 * r + 1] * P[1] + (double)T[4 * r + 2] * P[2]);
        out[r] = m + T[4 * r + 3];
    }
}
__device__ __forceinline__ void camera_center(const float* T, float Ow[3]) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float a = -T[0 + r], b = -T[4 + r], c = -T[8 + r];
        Ow[r] = (float)((double)a * T[3] + (double)b * T[7] + (double)c * T[11]);
    }
}
__device__ __forceinline__ int hamming32(const uint8_t* a, const uint8_t* b) {
    const uint4* pa = reinterpret_cast<const uint4*>(a);
    const uint4* pb = reinterpret_cast<const uint4*>(b);
    const uint4 a0 = pa[0], a1 = pa[1], b0 = pb[0], b1 = pb[1];
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) +
           __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// Ordered candidate gathering shared by both searches: all keypoints in the window cells (ix outer, iy inner, push order inside
// a cell) that pass the level gate, the |dx|,|dy| < r gate and the stereo gate; entry = idx | dist << 16 | octave << 26.
__device__ __forceinline__ int gather_candidates(const SearchFrameDev& F, const int32_t* cell_start, const int32_t* items, float x, float y, float r,
                                                 int minLevel, int maxLevel, bool stereo_gate, float ur_proj, float er_max, const uint8_t* qdesc,
                                                 uint32_t* out, bool& overflow) {
    const int lane = threadIdx.x & 31;
    const int cx0 = max(0, (int)floorf((x - F.min_x - r) * F.inv_w));
    if (cx0 >= SG_COLS) return 0;
    const int cx1 = min(SG_COLS - 1, (int)ceilf((x - F.min_x + r) * F.inv_w));
    if (cx1 < 0) return 0;
    const int cy0 = max(0, (int)floorf((y - F.min_y - r) * F.inv_h));
    if (cy0 >= SG_ROWS) return 0;
    const int cy1 = min(SG_ROWS - 1, (int)ceilf((y - F.min_y + r) * F.inv_h));
    if (cy1 < 0) return 0;
    const bool check = (minLevel > 0) || (maxLevel >= 0);
    int cnt = 0;
    for (int ix = cx0; ix <= cx1; ++ix) {
        // cells (ix, cy0..cy1) are contiguous in the sorted order: one run per column
        const int beg = cell_start[ix * SG_ROWS + cy0], end = cell_start[ix * SG_ROWS + cy1 + 1];
        for (int p0 = beg; p0 < end; p0 += 32) {
            const int p = p0 + lane;
            bool ok = p < end;
            int j = 0, d = 0, oct = 0;
            if (ok) {
                j = items[p];
                const pslam_keypoint kp = F.keys_un[j];
                oct = kp.octave;
                if (check) { if (oct < minLevel) ok = false; if (maxLevel >= 0 && oct > maxLevel) ok = false; }
                const float dx = kp.x - x, dy = kp.y - y;
                if (!(fabsf(dx) < r && fabsf(dy) < r)) ok = false;
                if (ok && stereo_gate) { const float urj = F.u_right[j]; if (urj > 0 && fabsf(ur_proj - urj) > er_max) ok = false; }
                if (ok) d = hamming32(qdesc, F.desc + (size_t)j * 32);
            }
            const uint32_t m = __ballot_sync(0xffffffffu, ok);
            if (ok) {
                const int pos = cnt + __popc(m & ((1u << lane) - 1));
                if (pos < SEARCH_CAND_CAP) out[pos] = (uint32_t)j | ((uint32_t)d << 16) | ((uint32_t)oct << 26); else overflow = true;
            }
            cnt += __popc(m);
        }
    }
    return min(cnt, SEARCH_CAND_CAP);
}

// ---- SearchByProjection(Frame, local map points): candidates ----
static __global__ void __launch_bounds__(256) k_candidates_map(SearchFrameDev F, SearchMapDev M, float th, const int32_t* __restrict__ cell_start,
                                                        const int32_t* __restrict__ items, uint32_t* __restrict__ cand, int32_t* __restrict__ cand_n,
                                                        uint8_t* __restrict__ in_view, int32_t* __restrict__ status) {
    const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (k >= M.n) return;
    int n_c = 0;
    bool view = false;
    if (!M.skip[k]) {
        float Ow[3], Pc[3];
        camera_center(frame_T(F), Ow);
        const float* P = M.pos + 3 * k;
        mat_rt(frame_T(F), P, Pc);
        if (!(Pc[2] < 0.0f)) {
            const float invz = 1.0f / Pc[2];
            const float u = F.fx * Pc[0] * invz + F.cx, v = F.fy * Pc[1] * invz + F.cy;
            if (!(u < F.min_x || u > F.max_x) && !(v < F.min_y || v > F.max_y)) {
                const float maxD = 1.2f * M.max_distance[k], minD = 0.8f * M.min_distance[k];
                const float PO[3] = {P[0] - Ow[0], P[1] - Ow[1], P[2] - Ow[2]};
                const float dist = (float)sqrt((double)PO[0] * PO[0] + (double)PO[1] * PO[1] + (double)PO[2] * PO[2]);
                if (!(dist < minD || dist > maxD)) {
                    const float* Pn = M.normal + 3 * k;
                    const float view_cos = (float)(((double)PO[0] * Pn[0] + (double)PO[1] * Pn[1] + (double)PO[2] * Pn[2]) / dist);
                    if (!(view_cos < 0.5f)) {
                        const float ratio = M.max_distance[k] / dist;
                        int lvl = (int)ceilf((float)log((double)ratio) / F.log_scale_factor);
                        if (lvl < 0) lvl = 0; else if (lvl >= F.n_levels) lvl = F.n_levels - 1;
                        view = true;
                        float r = ((double)view_cos > 0.998) ? 2.5f : 4.0f;
                        if (th != 1.0f) r *= th;
                        const float rs = r * F.scale[lvl];
                        bool overflow = false;
                        n_c = gather_candidates(F, cell_start, items, u, v, rs, lvl - 1, lvl, true, u - F.bf * invz, rs, M.desc + (size_t)k * 32,
                                                cand + (size_t)k * SEARCH_CAND_CAP, overflow);
                        if (__any_sync(0xffffffffu, overflow) && lane == 0) atomicOr(status, 64);
                    }
                }
            }
        }
    }
    if (lane == 0) { cand_n[k] = n_c; in_view[k] = view ? 1 : 0; }
}

// warp top-2 over keys (dist << 8 | position): returns the two smallest
__device__ __forceinline__ void warp_top2(uint32_t& k0, uint32_t& k1) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const uint32_t o0 = __shfl_xor_sync(0xffffffffu, k0, o), o1 = __shfl_xor_sync(0xffffffffu, k1, o);
        const uint32_t lo = min(k0, o0), hi = max(k0, o0);
        k1 = min(hi, min(k1, o1));
        k0 = lo;
    }
}

static __global__ void __launch_bounds__(32) k_resolve_map(SearchMapDev M, float nnratio, const uint32_t* __restrict__ cand, const int32_t* __restrict__ cand_n,
                                                    int32_t* __restrict__ matches, int32_t* __restrict__ n_matches) {
    const int lane = threadIdx.x;
    const uint32_t NONE = 0xffffffffu;
    int nm = 0;
    for (int k = 0; k < M.n; ++k) {
        const int nc = cand_n[k];
        if (nc == 0) continue;
        uint32_t k0 = NONE, k1 = NONE;
        for (int p = lane; p < nc; p += 32) {
            const uint32_t e = cand[(size_t)k * SEARCH_CAND_CAP + p];
            const int idx = e & 0xffff;
            const int cur = matches[idx];
            if (cur >= 0 && M.has_obs[cur]) continue;                 // already holds a map point with observations (:83-85)
            const uint32_t key = (((e >> 16) & 0x3ff) << 8) | (uint32_t)p;
            if (key < k0) { k1 = k0; k0 = key; } else if (key < k1) k1 = key;
        }
        warp_top2(k0, k1);
        if (k0 == NONE) continue;
        const int bestDist = k0 >> 8;
        if (bestDist <= 100) {
            const uint32_t e0 = cand[(size_t)k * SEARCH_CAND_CAP + (k0 & 0xff)];
            const int bestLevel = e0 >> 26;
            int bestDist2 = 256, bestLevel2 = -1;
            if (k1 != NONE) { const uint32_t e1 = cand[(size_t)k * SEARCH_CAND_CAP + (k1 & 0xff)]; bestDist2 = k1 >> 8; bestLevel2 = e1 >> 26; }
            if (bestLevel == bestLevel2 && (float)bestDist > nnratio * (float)bestDist2) continue;
            if (lane == 0) matches[e0 & 0xffff] = k;
            ++nm;
            __syncwarp();
        }
    }
    if (lane == 0) *n_matches = nm;
}

// ---- SearchByProjection(current, last): candidates per last-frame keypoint ----
struct SearchLastDev { int n; const pslam_keypoint* keys; const int32_t* map_point; const uint8_t* outlier; float Tcw[16];
                       const float* Tcw_dev; const int32_t* n_dev; };      // device-resident chain: see SearchFrameDev
__device__ __forceinline__ const float* last_T(const SearchLastDev& L) { return L.Tcw_dev ? L.Tcw_dev : L.Tcw; }
__device__ __forceinline__ int last_n(const SearchLastDev& L) { return L.n_dev ? min(*L.n_dev, L.n) : L.n; }

static __global__ void __launch_bounds__(256) k_candidates_last(SearchFrameDev C, SearchLastDev L, SearchMapDev M, float th, int mono,
                                                         const int32_t* __restrict__ cell_start, const int32_t* __restrict__ items,
                                                         uint32_t* __restrict__ cand, int32_t* __restrict__ cand_n, int32_t* __restrict__ status) {
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= last_n(L)) return;
    int n_c = 0;
    const int mp = L.map_point[i];
    if (mp >= 0 && !L.outlier[i]) {
        float twc[3], tlc[3], xc[3];
        camera_center(frame_T(C), twc);
        mat_rt(last_T(L), twc, tlc);
        const float mb = C.bf / C.fx;
        const bool fwd = tlc[2] > mb && !mono, bwd = -tlc[2] > mb && !mono;
        mat_rt(frame_T(C), M.pos + 3 * mp, xc);
        const float invzc = (float)(1.0 / (double)xc[2]);
        if (!(invzc < 0)) {
            const float u = C.fx * xc[0] * invzc + C.cx, v = C.fy * xc[1] * invzc + C.cy;
            if (!(u < C.min_x || u > C.max_x) && !(v < C.min_y || v > C.max_y)) {
                const int oct = L.keys[i].octave;
                const float radius = th * C.scale[oct];
                int lo, hi;
                if (fwd) { lo = oct; hi = -1; } else if (bwd) { lo = 0; hi = oct; } else { lo = oct - 1; hi = oct + 1; }
                bool overflow = false;
                n_c = gather_candidates(C, cell_start, items, u, v, radius, lo, hi, true, u - C.bf * invzc, radius, M.desc + (size_t)mp * 32,
                                        cand + (size_t)i * SEARCH_CAND_CAP, overflow);
                if (__any_sync(0xffffffffu, overflow) && lane == 0) atomicOr(status, 64);
            }
        }
    }
    if (lane == 0) cand_n[i] = n_c;
}

static __global__ void __launch_bounds__(32) k_resolve_last(SearchFrameDev C, SearchLastDev L, SearchMapDev M, int check_ori, const uint32_t* __restrict__ cand,
                                                     const int32_t* __restrict__ cand_n, int32_t* __restrict__ matches, int32_t* __restrict__ n_matches,
                                                     int32_t* __restrict__ hist_idx /*[L.n]*/, int8_t* __restrict__ hist_bin /*[L.n]*/) {
    const int lane = threadIdx.x;
    const uint32_t NONE = 0xffffffffu;
    __shared__ int s_cnt[32];
    if (lane < 30) s_cnt[lane] = 0;
    __syncwarp();
    int nm = 0, n_push = 0;
    const int Ln = last_n(L);
    for (int i = 0; i < Ln; ++i) {
        const int nc = cand_n[i];
        if (nc == 0) continue;
        const int mp = L.map_point[i];
        uint32_t k0 = NONE, k1 = NONE;
        for (int p = lane; p < nc; p += 32) {
            const uint32_t e = cand[(size_t)i * SEARCH_CAND_CAP + p];
            const int cur = matches[e & 0xffff];
            if (cur >= 0 && M.has_obs[cur]) continue;
            const uint32_t key = (((e >> 16) & 0x3ff) << 8) | (uint32_t)p;
            if (key < k0) { k1 = k0; k0 = key; } else if (key < k1) k1 = key;
        }
        warp_top2(k0, k1);
        if (k0 == NONE || (int)(k0 >> 8) > 100) continue;
        const int idx2 = cand[(size_t)i * SEARCH_CAND_CAP + (k0 & 0xff)] & 0xffff;
        if (lane == 0) matches[idx2] = mp;
        ++nm;
        if (check_ori) {
            float rot = L.keys[i].angle - C.keys_un[idx2].angle;
            if (rot < 0.0f) rot += 360.0f;
            int bin = (int)roundf(rot * (1.0f / 30));
            if (bin == 30) bin = 0;
            if (lane == 0) { hist_idx[n_push] = idx2; hist_bin[n_push] = (int8_t)bin; ++s_cnt[bin]; }
            ++n_push;
        }
        __syncwarp();
    }
    if (check_ori) {
        __syncwarp();
        int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
        for (int b = 0; b < 30; ++b) {
            const int s = s_cnt[b];
            if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = b; }
            else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = b; }
            else if (s > max3) { max3 = s; ind3 = b; }
        }
        if ((float)max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; } else if ((float)max3 < 0.1f * (float)max1) ind3 = -1;
        int removed = 0;
        for (int j = lane; j < n_push; j += 32) {
            const int b = hist_bin[j];
            if (b != ind1 && b != ind2 && b != ind3) { matches[hist_idx[j]] = -1; ++removed; }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) removed += __shfl_xor_sync(0xffffffffu, removed, o);
        nm -= removed;
    }
    if (lane == 0) *n_matches = nm;
}


}  // namespace pslam
