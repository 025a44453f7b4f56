// ORB extraction kernels for sm_90a (batched over frames: blockIdx.y or .z selects the frame).
//
// Reference semantics (file:line under /root/reference): ComputePyramid src/ORBextractor.cc:1107-1132,
// ComputeKeyPointsOctTree :765-853, DistributeOctTree :539-763, IC_Angle :77-104, GaussianBlur call :1086,
// computeOrbDescriptor :108-147.  OpenCV primitive arithmetic (resize / FAST / GaussianBlur / fastAtan2) is
// restated from OpenCV's published algorithms; the whole file is compiled with --fmad=false so float/double
// expressions round exactly like the unfused CPU oracle.
#pragma once
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

#include "orb_common.h"
#include "pslam_internal.h"
#include "tma_util.cuh"

namespace pslam {

__device__ __forceinline__ const uint8_t* level_ptr(const OrbGeom& g, const uint8_t* gray, const uint8_t* pyr,
                                                    int frame, int level, int& pitch) {
    if (level == 0) { pitch = g.width; return gray + (size_t)frame * g.width * g.height; }
    pitch = g.lv[level].pitch;
    return pyr + (size_t)frame * g.pyr_bytes + g.lv[level].pyr_off;
}

// ------------------------------------------------------------------------------------------------------
// K1: one pyramid level = cv::resize(INTER_LINEAR) of the previous one. 11-bit fixed-point coefficients from
// precomputed tables; 4 output pixels per thread, one aligned uchar4 store.
// grid (ceil(dw/128), ceil(dh/8), frames), block (32, 8).
__global__ void __launch_bounds__(256) k_resize_level(const uint8_t* __restrict__ src, size_t src_frame_stride, int src_pitch, int sw,
                                                      int sh, uint8_t* __restrict__ dst, size_t dst_frame_stride, int dst_pitch, int dw,
                                                      int dh, const int16_t* __restrict__ xofs, const int16_t* __restrict__ xa,
                                                      const int16_t* __restrict__ yofs, const int16_t* __restrict__ ya) {
    const int dx0 = (blockIdx.x * 32 + threadIdx.x) * 4;
    const int dy = blockIdx.y * 8 + threadIdx.y;
    if (dx0 >= dw || dy >= dh) return;
    const uint8_t* S = src + (size_t)blockIdx.z * src_frame_stride;
    uint8_t* D = dst + (size_t)blockIdx.z * dst_frame_stride;
    int sy0 = yofs[dy], sy1 = sy0 + 1;
    sy0 = min(max(sy0, 0), sh - 1); sy1 = min(max(sy1, 0), sh - 1);
    const int b0 = ya[2 * dy], b1 = ya[2 * dy + 1];
    const uint8_t* R0 = S + (size_t)sy0 * src_pitch;
    const uint8_t* R1 = S + (size_t)sy1 * src_pitch;
    uint32_t out = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int dx = min(dx0 + k, dw - 1);
        const int sx = xofs[dx], sx1 = min(sx + 1, sw - 1);
        const int a0 = xa[2 * dx], a1 = xa[2 * dx + 1];
        const int r0 = R0[sx] * a0 + R0[sx1] * a1;
        const int r1 = R1[sx] * a0 + R1[sx1] * a1;
        int v = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;
        v = min(255, max(0, v));
        out |= (uint32_t)v << (8 * k);
    }
    *reinterpret_cast<uint32_t*>(D + (size_t)dy * dst_pitch + dx0) = out;
}

// ------------------------------------------------------------------------------------------------------
// K2: per-cell FAST-9/16 with the reference's per-cell threshold fallback (src/ORBextractor.cc:789-829).
// One CTA per (cell, frame): the cell window (cell + 6 px) is staged in shared memory, every interior pixel
// gets its FAST score (largest threshold at which it is still a corner; 0 below min_th), non-maximum
// suppression sees zeros outside the window interior exactly like cv::FAST on the sub-image, and the
// survivors are emitted in row-major order: those with score >= ini_th if any exist, otherwise all.
#define FAST_WIN_MAX 68
__device__ __forceinline__ int fast_score(const uint8_t (*win)[FAST_WIN_MAX + 4], int x, int y, int min_th) {
    const int v = win[y][x];
    const int p0 = win[y + 3][x], p4 = win[y][x + 3], p8 = win[y - 3][x], p12 = win[y][x - 3];
    {   // any 9-arc of the 16-circle contains at least two of the four compass points
        const int hi = v + min_th, lo = v - min_th;
        const int nb = (p0 > hi) + (p4 > hi) + (p8 > hi) + (p12 > hi);
        const int nd = (p0 < lo) + (p4 < lo) + (p8 < lo) + (p12 < lo);
        if (nb < 2 && nd < 2) return 0;
    }
    // d = centre - circle (dark arcs), e = circle - centre (bright arcs).  Both polarities use min-chains only:
    // nvcc 12.9 has been seen to miscompile max(x, -y) when it is folded into a 3-input VIMNMX (observed on sm_100a:
    // max(0, max(-4, -203)) evaluated to 203), so no negation may appear inside a min/max operand here.
    int d[16], e[16];
    const int c1 = win[y + 3][x + 1], c2 = win[y + 2][x + 2], c3 = win[y + 1][x + 3], c5 = win[y - 1][x + 3];
    const int c6 = win[y - 2][x + 2], c7 = win[y - 3][x + 1], c9 = win[y - 3][x - 1], c10 = win[y - 2][x - 2];
    const int c11 = win[y - 1][x - 3], c13 = win[y + 1][x - 3], c14 = win[y + 2][x - 2], c15 = win[y + 3][x - 1];
    d[0] = v - p0;   d[1] = v - c1;   d[2] = v - c2;   d[3] = v - c3;   d[4] = v - p4;   d[5] = v - c5;   d[6] = v - c6;   d[7] = v - c7;
    d[8] = v - p8;   d[9] = v - c9;   d[10] = v - c10; d[11] = v - c11; d[12] = v - p12; d[13] = v - c13; d[14] = v - c14; d[15] = v - c15;
    e[0] = p0 - v;   e[1] = c1 - v;   e[2] = c2 - v;   e[3] = c3 - v;   e[4] = p4 - v;   e[5] = c5 - v;   e[6] = c6 - v;   e[7] = c7 - v;
    e[8] = p8 - v;   e[9] = c9 - v;   e[10] = c10 - v; e[11] = c11 - v; e[12] = p12 - v; e[13] = c13 - v; e[14] = c14 - v; e[15] = c15 - v;
    int d2[16], e2[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) { d2[i] = min(d[i], d[(i + 1) & 15]); e2[i] = min(e[i], e[(i + 1) & 15]); }           // arcs of 2
    int d4[16], e4[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) { d4[i] = min(d2[i], d2[(i + 2) & 15]); e4[i] = min(e2[i], e2[(i + 2) & 15]); }       // arcs of 4
    int best = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int d9 = min(min(d4[i], d4[(i + 4) & 15]), d[(i + 8) & 15]);                                            // arcs of 9
        const int e9 = min(min(e4[i], e4[(i + 4) & 15]), e[(i + 8) & 15]);
        best = max(best, d9);
        best = max(best, e9);
    }
    const int s = best - 1;
    return s >= min_th ? s : 0;
}

// Two horizontally adjacent pixels at once in packed 16-bit lanes (DPX three-input min / max on u16x2, native on sm_90+): every difference is kept biased,
// d' = centre - circle + 256 in [1, 511] and e' = 512 - d', so plain 32-bit subtraction never borrows across the lanes.  The score is the one fast_score()
// returns (the largest threshold at which a 9-arc exists, or 0 below min_th); the compass-point test is evaluated for the pair and the whole warp skips the
// arc search when no lane passes it.  win row r holds image bytes from column xa0; X = column of the left pixel inside the window row.
__device__ __forceinline__ uint32_t fast_pair(uint32_t w, int k) {            // bytes k, k+1 of a word as u16x2 (k = 0..2)
    return __byte_perm(w, 0u, k == 0 ? 0x4140u : k == 1 ? 0x4241u : 0x4342u);
}
__device__ __forceinline__ void fast_score_pair(const uint8_t (*win)[FAST_WIN_MAX + 4], int X, int y, int min_th, int& s0, int& s1) {
    const int base = (X - 3) & ~3, sh = 8 * ((X - 3) & 3);
    uint32_t lo[7], hi[7];                                                     // row y - 3 + r: bytes of columns X-3 .. X+4
#pragma unroll
    for (int r = 0; r < 7; ++r) {
        const uint32_t* rp = reinterpret_cast<const uint32_t*>(&win[y - 3 + r][base]);
        const uint32_t w0 = rp[0], w1 = rp[1], w2 = rp[2];
        lo[r] = __funnelshift_r(w0, w1, sh); hi[r] = __funnelshift_r(w1, w2, sh);
    }
    // byte offset of dx inside the 8-byte row: dx + 3
    const uint32_t VB = (fast_pair(__funnelshift_r(lo[3], hi[3], 24), 0)) + 0x01000100u;      // (centre + 256) per lane; centre = bytes 3, 4
    uint32_t D[16];
    D[0]  = VB - fast_pair(__funnelshift_r(lo[6], hi[6], 24), 0);      // ( 0, +3)
    D[1]  = VB - fast_pair(hi[6], 0);                                  // (+1, +3)
    D[2]  = VB - fast_pair(hi[5], 1);                                  // (+2, +2)
    D[3]  = VB - fast_pair(hi[4], 2);                                  // (+3, +1)
    D[4]  = VB - fast_pair(hi[3], 2);                                  // (+3,  0)
    D[5]  = VB - fast_pair(hi[2], 2);                                  // (+3, -1)
    D[6]  = VB - fast_pair(hi[1], 1);                                  // (+2, -2)
    D[7]  = VB - fast_pair(hi[0], 0);                                  // (+1, -3)
    D[8]  = VB - fast_pair(__funnelshift_r(lo[0], hi[0], 24), 0);      // ( 0, -3)
    D[9]  = VB - fast_pair(lo[0], 2);                                  // (-1, -3)
    D[10] = VB - fast_pair(lo[1], 1);                                  // (-2, -2)
    D[11] = VB - fast_pair(lo[2], 0);                                  // (-3, -1)
    D[12] = VB - fast_pair(lo[3], 0);                                  // (-3,  0)
    D[13] = VB - fast_pair(lo[4], 0);                                  // (-3, +1)
    D[14] = VB - fast_pair(lo[5], 1);                                  // (-2, +2)
    D[15] = VB - fast_pair(lo[6], 2);                                  // (-1, +3)
    {   // any 9-arc of the 16-circle contains at least two of the four compass points: second smallest / second largest of d'[0, 4, 8, 12]
        const uint32_t a = __vimin3_u16x2(D[0], D[4], D[4]), b = __vimax3_u16x2(D[0], D[4], D[4]);
        const uint32_t c = __vimin3_u16x2(D[8], D[12], D[12]), d = __vimax3_u16x2(D[8], D[12], D[12]);
        const uint32_t t1 = __vimax3_u16x2(a, c, c), t2 = __vimin3_u16x2(b, d, d);
        const uint32_t s2 = __vimin3_u16x2(t1, t2, t2), l2 = __vimax3_u16x2(t1, t2, t2);
        const int brt = 256 - min_th, drk = 256 + min_th;                      // circle > centre + th  <=>  d' < 256 - th
        const bool pass = (int)(s2 & 0xffffu) < brt || (int)(s2 >> 16) < brt || (int)(l2 & 0xffffu) > drk || (int)(l2 >> 16) > drk;
        if (!__any_sync(__activemask(), pass)) { s0 = 0; s1 = 0; return; }
    }
    uint32_t best = 0;
    uint32_t m3[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) m3[i] = __vimin3_u16x2(D[i], D[(i + 1) & 15], D[(i + 2) & 15]);
#pragma unroll
    for (int i = 0; i < 16; i += 2) {
        const uint32_t q0 = __vimin3_u16x2(m3[i], m3[(i + 3) & 15], m3[(i + 6) & 15]), q1 = __vimin3_u16x2(m3[i + 1], m3[(i + 4) & 15], m3[(i + 7) & 15]);
        best = __vimax3_u16x2(best, q0, q1);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) D[i] = 0x02000200u - D[i];                    // e' = circle - centre + 256
#pragma unroll
    for (int i = 0; i < 16; ++i) m3[i] = __vimin3_u16x2(D[i], D[(i + 1) & 15], D[(i + 2) & 15]);
#pragma unroll
    for (int i = 0; i < 16; i += 2) {
        const uint32_t q0 = __vimin3_u16x2(m3[i], m3[(i + 3) & 15], m3[(i + 6) & 15]), q1 = __vimin3_u16x2(m3[i + 1], m3[(i + 4) & 15], m3[(i + 7) & 15]);
        best = __vimax3_u16x2(best, q0, q1);
    }
    const int b0 = (int)(best & 0xffffu) - 257, b1 = (int)(best >> 16) - 257;
    s0 = b0 >= min_th ? b0 : 0;
    s1 = b1 >= min_th ? b1 : 0;
}

__global__ void __launch_bounds__(128) k_fast_cells(const uint8_t* __restrict__ gray, const uint8_t* __restrict__ pyr,
                                                    OrbGeom g, uint32_t* __restrict__ slots, int32_t* __restrict__ cell_cnt,
                                                    int32_t* __restrict__ status) {
    __shared__ __align__(16) uint8_t win[FAST_WIN_MAX + 1][FAST_WIN_MAX + 4];      // one spare row: the pair scorer reads whole words past a row's last pixel
    __shared__ uint8_t sc[FAST_WIN_MAX][FAST_WIN_MAX + 4];
    __shared__ int s_tot20, s_warp[4];

    const int frame = blockIdx.y;
    int cell = blockIdx.x, level = 0;
    while (level + 1 < g.nlevels && cell >= g.lv[level + 1].cell_base) ++level;
    const LevelGeom& L = g.lv[level];
    const int lc = cell - L.cell_base;
    const int ci = lc / L.n_cols, cj = lc - ci * L.n_cols;
    int32_t* my_cnt = cell_cnt + (size_t)frame * g.total_cells + cell;

    const int x0 = 16 + cj * L.w_cell, y0 = 16 + ci * L.h_cell;
    const int x1 = min(x0 + L.w_cell + 6, L.max_bx), y1 = min(y0 + L.h_cell + 6, L.max_by);
    const int ww = x1 - x0, wh = y1 - y0;
    if (y0 >= L.max_by - 3 || x0 >= L.max_bx - 6 || ww < 7 || wh < 7) {   // reference :794-795, :803-804
        if (threadIdx.x == 0) *my_cnt = 0;
        return;
    }
    int pitch;
    const uint8_t* img = level_ptr(g, gray, pyr, frame, level, pitch);

    // stage the window: aligned 32-bit loads; smem column 0 corresponds to image column (x0 & ~3).  One warp per row, one lane per word (no index division)
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int xa0 = x0 & ~3, ox = x0 - xa0;
    const int words = ((x1 + 3) >> 2) - (xa0 >> 2);                  // <= 19
    for (int r = wid; r < wh; r += 4) {
        if (lane < words) *reinterpret_cast<uint32_t*>(&win[r][4 * lane]) = *reinterpret_cast<const uint32_t*>(img + (size_t)(y0 + r) * pitch + xa0 + 4 * lane);
        if (lane < (FAST_WIN_MAX + 4) / 4) *reinterpret_cast<uint32_t*>(&sc[r][4 * lane]) = 0u;
    }
    if (threadIdx.x == 0) s_tot20 = 0;
    __syncthreads();

    const int wi = ww - 6, hi = wh - 6, P = wi * hi;
    {
        // pixel pairs: a warp iteration covers 32 >> lg rows of (1 << lg) pairs each (lg chosen so that a row of pairs fits), warps interleave
        const int wi2 = (wi + 1) >> 1;
        const int lg = wi2 <= 8 ? 3 : wi2 <= 16 ? 4 : 5;
        const int rows_per_it = 32 >> lg, x2 = lane & ((1 << lg) - 1), yl = lane >> lg;
        for (int yb = wid * rows_per_it; yb < hi; yb += 4 * rows_per_it) {          // warp-uniform trip count: fast_score_pair votes across the warp
            const int y = yb + yl, x = 2 * x2;
            if (x2 < wi2 && y < hi) {
                int sa, sb;
                fast_score_pair(win, x + 3 + ox, y + 3, g.min_th, sa, sb);
                sc[y + 3][x + 3] = (uint8_t)sa;
                if (x + 1 < wi) sc[y + 3][x + 4] = (uint8_t)sb;
            }
        }
    }
    __syncthreads();

    // contiguous row-major chunk per thread so that a block-wide exclusive scan gives the output order
    const int chunk = (P + 127) / 128;      // <= 32 for windows up to 68x68
    const int pbeg = threadIdx.x * chunk, pend = min(P, pbeg + chunk);
    uint32_t m_max = 0, m_ini = 0;
    {
        int y = pbeg / wi, x = pbeg - y * wi;                        // one division per thread, then the walk wraps by comparison
        for (int p = pbeg; p < pend; ++p) {
            const int s = sc[y + 3][x + 3];
            if (s != 0) {
                const uint8_t* r0 = &sc[y + 2][x + 2]; const uint8_t* r1 = &sc[y + 3][x + 2]; const uint8_t* r2 = &sc[y + 4][x + 2];
                const bool is_max = s > r0[0] && s > r0[1] && s > r0[2] && s > r1[0] && s > r1[2] && s > r2[0] && s > r2[1] && s > r2[2];
                if (is_max) {
                    m_max |= 1u << (p - pbeg);
                    if (s >= g.ini_th) m_ini |= 1u << (p - pbeg);
                }
            }
            if (++x == wi) { x = 0; ++y; }
        }
    }
    if (m_ini) atomicAdd(&s_tot20, __popc(m_ini));
    __syncthreads();
    const uint32_t sel = s_tot20 > 0 ? m_ini : m_max;
    const int cnt = __popc(sel);
    // block exclusive scan of cnt
    int inc = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < wid; ++w) base += s_warp[w];
    const int total = s_warp[0] + s_warp[1] + s_warp[2] + s_warp[3];
    int off = base + inc - cnt;
    uint32_t* my_slots = slots + ((size_t)frame * g.total_slots + L.slot_base + (size_t)lc * L.slot_cap);
    for (uint32_t m = sel; m; m &= m - 1) {
        const int p = pbeg + __ffs(m) - 1;
        const int y = p / wi, x = p - y * wi;
        if (off < L.slot_cap) my_slots[off] = pack_kp(x + 3 + cj * L.w_cell, y + 3 + ci * L.h_cell, sc[y + 3][x + 3]);
        ++off;
    }
    if (threadIdx.x == 0) {
        *my_cnt = min(total, L.slot_cap);
        if (total > L.slot_cap) atomicOr(status + frame, ST_SLOT_OVERFLOW);
    }
}

// ------------------------------------------------------------------------------------------------------
// K3: quadtree distribution (DistributeOctTree), one warp per (level, frame).  Control flow is warp-uniform
// and follows the reference's list semantics exactly (children pushed to the list front in the order
// 1,2,3,4, parent erased, "largest first" expansion near the quota with ties broken by creation order);
// the per-node key partition is done cooperatively by the 32 lanes (stable 4-way partition by ballot).
struct QtScratch {
    uint32_t* keys[2];   // ping-pong candidate buffers
    int4* nodes;         // {ulx | uly<<16, urx | bry<<16, kbeg, kcnt | buf<<29 | nomore<<30}
    int2* links;         // {prev, next}
    int32_t* exp_a;      // expandable node ids (current generation)
    int32_t* exp_b;
    int32_t* order;      // node ids in final list order
};

__device__ __forceinline__ int qt_group(uint32_t key, int midx, int midy) {
    const int x = kp_x(key), y = kp_y(key);
    return (x < midx) ? ((y < midy) ? 0 : 2) : ((y < midy) ? 1 : 3);
}

// Stable 4-way partition of src[beg, beg+n) into dst[beg, beg+n); returns the four group sizes in cnt[].
template <typename GroupFn>
__device__ __forceinline__ void qt_partition(const uint32_t* src, uint32_t* dst, int beg, int n, GroupFn grp, int cnt[4]) {
    const int lane = threadIdx.x & 31;
    int c0 = 0, c1 = 0, c2 = 0, c3 = 0;
    for (int i = lane; i < n; i += 32) {
        const int gq = grp(src[beg + i]);
        c0 += gq == 0; c1 += gq == 1; c2 += gq == 2; c3 += gq == 3;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        c0 += __shfl_xor_sync(0xffffffffu, c0, o); c1 += __shfl_xor_sync(0xffffffffu, c1, o);
        c2 += __shfl_xor_sync(0xffffffffu, c2, o); c3 += __shfl_xor_sync(0xffffffffu, c3, o);
    }
    cnt[0] = c0; cnt[1] = c1; cnt[2] = c2; cnt[3] = c3;
    int run[4] = {beg, beg + c0, beg + c0 + c1, beg + c0 + c1 + c2};
    const uint32_t lt = (1u << lane) - 1;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const bool ok = i < n;
        const uint32_t key = ok ? src[beg + i] : 0u;
        const int gq = ok ? grp(key) : -1;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint32_t m = __ballot_sync(0xffffffffu, gq == q);
            if (gq == q) dst[run[q] + __popc(m & lt)] = key;
            run[q] += __popc(m);
        }
    }
    __syncwarp();
}

__global__ void __launch_bounds__(32) k_quadtree(OrbGeom g, const uint32_t* __restrict__ slots, const int32_t* __restrict__ cell_cnt,
                                                 uint32_t* __restrict__ cand, int32_t* __restrict__ cand_cnt, int4* __restrict__ nodes_all,
                                                 int2* __restrict__ links_all, int32_t* __restrict__ work_all,
                                                 uint32_t* __restrict__ lvl_kp, int32_t* __restrict__ lvl_cnt, int32_t* __restrict__ status) {
    const int level = blockIdx.x, frame = blockIdx.y, lane = threadIdx.x;
    const LevelGeom& L = g.lv[level];
    QtScratch S;
    S.keys[0] = cand + ((size_t)frame * g.total_cand + L.cand_base) * 2;
    S.keys[1] = S.keys[0] + L.cand_cap;
    S.nodes = nodes_all + (size_t)frame * g.total_nodes + L.node_base;
    S.links = links_all + (size_t)frame * g.total_nodes + L.node_base;
    int32_t* work = work_all + (size_t)frame * g.total_work + L.work_base;
    S.exp_a = work; S.exp_b = work + 4 * L.kp_cap; S.order = work + 8 * L.kp_cap;
    uint32_t* out = lvl_kp + (size_t)frame * g.total_kp + L.kp_base;
    int32_t* out_cnt = lvl_cnt + frame * g.nlevels + level;
    const int N = L.quota;

    // ---- gather this level's candidates in the reference order: cells row-major, row-major inside a cell ----
    const int ncell = L.n_cols * L.n_rows;
    const int32_t* cc = cell_cnt + (size_t)frame * g.total_cells + L.cell_base;
    const uint32_t* sl = slots + (size_t)frame * g.total_slots + L.slot_base;
    int ncand = 0;
    bool overflow = false;
    for (int c0 = 0; c0 < ncell; c0 += 32) {
        const int c = c0 + lane;
        const int n = c < ncell ? cc[c] : 0;
        int inc = n;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        const int tot = __shfl_sync(0xffffffffu, inc, 31);
        // every lane copies its own cell (cells hold a handful of candidates)
        int dstp = ncand + inc - n;
        for (int k = 0; k < n; ++k, ++dstp) {
            if (dstp < L.cand_cap) S.keys[0][dstp] = sl[(size_t)c * L.slot_cap + k]; else overflow = true;
        }
        ncand += tot;
    }
    if (__any_sync(0xffffffffu, overflow)) { if (lane == 0) atomicOr(status + frame, ST_CAND_OVERFLOW); ncand = min(ncand, L.cand_cap); }
    if (lane == 0) cand_cnt[frame * g.nlevels + level] = ncand;
    __syncwarp();
    if (ncand == 0 || L.n_ini <= 0 || L.n_ini > 4) { if (lane == 0) *out_cnt = 0; return; }

    int nn = 0;            // nodes created
    int head = -1;         // list head
    int size = 0;          // list length
    bool node_overflow = false;

    auto push_front = [&](int id) {   // lane 0 writes; all lanes track head
        if (lane == 0) { S.links[id] = make_int2(-1, head); if (head >= 0) S.links[head].x = id; }
        head = id; ++size;
    };
    auto unlink = [&](int id) {
        const int2 l = S.links[id];
        if (lane == 0) { if (l.x >= 0) S.links[l.x].y = l.y; if (l.y >= 0) S.links[l.y].x = l.x; }
        if (head == id) head = l.y;
        --size;
        __syncwarp();
    };

    // ---- roots (reference :543-585) ----
    {
        int cnt[4];
        const float hX = L.h_x;
        qt_partition(S.keys[0], S.keys[1], 0, ncand, [&](uint32_t k) { return min((int)__fdiv_rn((float)kp_x(k), hX), 3); }, cnt);
        int kb = 0;
        int tail = -1;
        for (int i = 0; i < L.n_ini; ++i) {
            if (cnt[i] > 0) {        // empty roots are erased right away; roots keep their left-to-right order
                const int id = nn++;
                const int ulx = (int)(hX * (float)i), urx = (int)(hX * (float)(i + 1));
                if (lane == 0) {
                    S.nodes[id] = make_int4(ulx, urx | ((L.max_by - 16) << 16), kb, cnt[i] | (1 << 29) | ((cnt[i] == 1) << 30));
                    S.links[id] = make_int2(tail, -1);
                    if (tail >= 0) S.links[tail].y = id;
                }
                if (head < 0) head = id;
                tail = id; ++size;
            }
            kb += cnt[i];
        }
        __syncwarp();
    }

    // split node `id`: children pushed to the list front in order 1..4; those with >1 keys appended to exp_out
    auto split = [&](int id, int32_t* exp_out, int& n_exp) {
        const int4 nd = S.nodes[id];
        const int ulx = nd.x & 0xffff, uly = nd.x >> 16, urx = nd.y & 0xffff, bry = nd.y >> 16;
        const int kbeg = nd.z, kcnt = nd.w & 0x1fffffff, buf = (nd.w >> 29) & 1;
        const int midx = ulx + ((urx - ulx + 1) >> 1), midy = uly + ((bry - uly + 1) >> 1);   // ceil(d / 2)
        int cnt[4];
        qt_partition(S.keys[buf], S.keys[buf ^ 1], kbeg, kcnt, [&](uint32_t k) { return qt_group(k, midx, midy); }, cnt);
        int kb = kbeg;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (cnt[q] > 0) {
                if (nn >= L.node_cap) { node_overflow = true; }
                else {
                    const int cid = nn++;
                    const int cx0 = (q & 1) ? midx : ulx, cx1 = (q & 1) ? urx : midx;
                    const int cy0 = (q & 2) ? midy : uly, cy1 = (q & 2) ? bry : midy;
                    if (lane == 0) S.nodes[cid] = make_int4(cx0 | (cy0 << 16), cx1 | (cy1 << 16), kb, cnt[q] | ((buf ^ 1) << 29) | ((cnt[q] == 1) << 30));
                    push_front(cid);
                    if (cnt[q] > 1) { if (lane == 0) exp_out[n_exp] = cid; ++n_exp; }
                }
            }
            kb += cnt[q];
        }
        __syncwarp();
    };

    int32_t* exp_cur = S.exp_a;
    int32_t* exp_nxt = S.exp_b;
    bool finish = false;
    while (!finish && !node_overflow) {
        const int prev_size = size;
        int n_exp = 0;
        int cur = head;
        while (cur >= 0 && !node_overflow) {
            const int nxt = S.links[cur].y;
            const int meta = S.nodes[cur].w;
            if (!((meta >> 30) & 1)) { split(cur, exp_cur, n_exp); unlink(cur); }
            cur = nxt;
        }
        if (size >= N || size == prev_size) {
            finish = true;
        } else if (size + 3 * n_exp > N) {
            while (!finish && !node_overflow) {
                const int prev2 = size;
                int n_exp2 = 0;
                // expand in descending (key count, creation id) order; stop as soon as the quota is reached
                for (int it = 0; it < n_exp; ++it) {
                    unsigned long long best = 0ull;
                    for (int i = lane; i < n_exp; i += 32) {
                        const int id = exp_cur[i];
                        if (id >= 0) {
                            const unsigned long long key = ((unsigned long long)(S.nodes[id].w & 0x1fffffff) << 32) | (unsigned)(id + 1);
                            best = key > best ? key : best;
                        }
                    }
#pragma unroll
                    for (int o = 16; o; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o); best = t > best ? t : best; }
                    const int id = (int)(unsigned)(best & 0xffffffffu) - 1;
                    // entries were appended in creation order, so the slot of `id` is found by scanning
                    for (int i = lane; i < n_exp; i += 32) if (exp_cur[i] == id) exp_cur[i] = -1;
                    __syncwarp();
                    split(id, exp_nxt, n_exp2);
                    unlink(id);
                    if (size >= N || node_overflow) break;
                }
                if (size >= N || size == prev2) finish = true;
                int32_t* t = exp_cur; exp_cur = exp_nxt; exp_nxt = t;
                n_exp = n_exp2;
            }
        }
    }
    if (node_overflow && lane == 0) atomicOr(status + frame, ST_NODE_OVERFLOW);

    // ---- keep the best response of every node, in list order (reference :741-760) ----
    int nout = 0;
    for (int cur = head; cur >= 0; cur = S.links[cur].y) { if (lane == 0 && nout < L.kp_cap) S.order[nout] = cur; ++nout; }
    nout = min(nout, L.kp_cap);
    __syncwarp();
    for (int i = lane; i < nout; i += 32) {
        const int4 nd = S.nodes[S.order[i]];
        const uint32_t* ks = S.keys[(nd.w >> 29) & 1] + nd.z;
        const int kcnt = nd.w & 0x1fffffff;
        uint32_t best = ks[0];
        for (int k = 1; k < kcnt; ++k) if (kp_s(ks[k]) > kp_s(best)) best = ks[k];
        out[i] = best;
    }
    if (lane == 0) *out_cnt = nout;
}

// ------------------------------------------------------------------------------------------------------
// K4a: cv::GaussianBlur(7x7, sigma 2, BORDER_REFLECT_101) in OpenCV's 8.8 fixed point (taps 18 34 48 56 48 34 18,
// horizontal pass exact 16-bit, vertical pass 32-bit, round half up at >> 16).  Tile 64x16, block 256.
__device__ __forceinline__ int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = (i < 0) ? -i : 2 * (n - 1) - i;
    return i;
}

__global__ void __launch_bounds__(256) k_blur_level(const uint8_t* __restrict__ src, size_t src_frame_stride, int src_pitch,
                                                    uint8_t* __restrict__ dst, size_t dst_frame_stride, int dst_pitch, int w, int h) {
    constexpr int TW = 64, TH = 16;
    __shared__ uint8_t in[TH + 6][TW + 8];
    __shared__ uint16_t hz[TH + 6][TW];
    const uint8_t* S = src + (size_t)blockIdx.z * src_frame_stride;
    uint8_t* D = dst + (size_t)blockIdx.z * dst_frame_stride;
    const int tx0 = blockIdx.x * TW, ty0 = blockIdx.y * TH;
    for (int i = threadIdx.x; i < (TH + 6) * (TW + 6); i += 256) {
        const int r = i / (TW + 6), c = i - r * (TW + 6);
        in[r][c] = S[(size_t)reflect101(ty0 + r - 3, h) * src_pitch + reflect101(tx0 + c - 3, w)];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (TH + 6) * TW; i += 256) {
        const int r = i / TW, c = i - r * TW;
        const uint8_t* p = &in[r][c];
        hz[r][c] = (uint16_t)(18 * (p[0] + p[6]) + 34 * (p[1] + p[5]) + 48 * (p[2] + p[4]) + 56 * p[3]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TH * TW; i += 256) {
        const int r = i / TW, c = i - r * TW;
        const int x = tx0 + c, y = ty0 + r;
        if (x < w && y < h) {
            const uint32_t acc = 18u * (hz[r][c] + hz[r + 6][c]) + 34u * (hz[r + 1][c] + hz[r + 5][c]) +
                                 48u * (hz[r + 2][c] + hz[r + 4][c]) + 56u * hz[r + 3][c];
            D[(size_t)y * dst_pitch + x] = (uint8_t)min(255u, (acc + 32768u) >> 16);
        }
    }
}

// K4a (TMA): the same blur, every level of every frame in ONE launch.  A CTA owns a 128 x 64 output tile; its 160 x 70 source box
// (3-pixel halo; starting 16 columns left of the tile so that the box start is 16-byte aligned) is fetched by one cp.async.bulk.tensor copy into shared memory (zero fill outside the image),
// the REFLECT_101 halo of border tiles is rebuilt in shared memory from the interior, and each thread slides a 7-row window down a
// 4-pixel-wide, 16-row strip: horizontal taps by two __dp4a per pixel on byte windows cut from three aligned words, vertical taps on
// the 8.8 sums held in registers, one 32-bit store per row.  Arithmetic identical to k_blur_level (8.8 -> 16.16, round half up).
__device__ __forceinline__ void blur_hrow(const uint8_t* __restrict__ row, int lane, uint32_t hv[4]) {
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(row) + lane + (BT_X_PAD - 4) / 4;        // bytes x - 4 .. x + 7 of the row, x = x0 + 4 lane
    const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2];
    const uint32_t c0 = 18u | (34u << 8) | (48u << 16) | (56u << 24), c1 = 48u | (34u << 8) | (18u << 16);
    hv[0] = __dp4a(__funnelshift_r(w0, w1, 8), c0, __dp4a(__funnelshift_r(w1, w2, 8), c1, 0u));
    hv[1] = __dp4a(__funnelshift_r(w0, w1, 16), c0, __dp4a(__funnelshift_r(w1, w2, 16), c1, 0u));
    hv[2] = __dp4a(__funnelshift_r(w0, w1, 24), c0, __dp4a(__funnelshift_r(w1, w2, 24), c1, 0u));
    hv[3] = __dp4a(w1, c0, __dp4a(w2, c1, 0u));
}

// The tensor maps are read by the copy engine from `maps`: device global memory (the context's copy, default) or - MAPS_IN_PARAM - the kernel's own
// __grid_constant__ parameter block.
template <bool MAPS_IN_PARAM>
__global__ void __launch_bounds__(128) k_blur_tma(const __grid_constant__ BlurTmaParams P, const CUtensorMap* __restrict__ maps, uint8_t* __restrict__ blur,
                                                  size_t blur_frame_bytes) {
    __shared__ __align__(128) uint8_t tile[BT_BOX_H][BT_BOX_W];
    __shared__ __align__(8) uint64_t bar;
    const int tid = threadIdx.x, lane = tid & 31, strip = tid >> 5, frame = blockIdx.y;
    int level = 0;
    while (level + 1 < P.nlevels && (int)blockIdx.x >= P.tile_base[level + 1]) ++level;
    const int t = blockIdx.x - P.tile_base[level];
    const int ty = t / P.tiles_x[level], tx = t - ty * P.tiles_x[level];
    const int x0 = tx * BT_W, y0 = ty * BT_H, w = P.w[level], h = P.h[level];
    if (tid == 0) mbar_init(&bar, 1);
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(&bar, BT_BOX_W * BT_BOX_H);
        tma_load_3d(&tile[0][0], MAPS_IN_PARAM ? &P.map[level] : maps + level, x0 - BT_X_PAD, y0 - 3, frame, &bar);     // smem (r, c) <-> image (y0 - 3 + r, x0 - 16 + c)
    }
    mbar_wait(&bar, 0);
    // REFLECT_101 halo of border tiles: rows first (whole rows, halo columns included), then columns (all rows): the reflection is separable
    if (y0 == 0 || y0 + BT_H + 3 > h) {
        for (int i = tid; i < 6 * (BT_BOX_W / 4); i += 128) {
            const int k = i / (BT_BOX_W / 4), cw = i - k * (BT_BOX_W / 4);
            const int Y = k < 3 ? k - 3 : h + (k - 3);                             // rows -3..-1 and h..h+2
            const int r = Y - (y0 - 3);
            if (r < 0 || r >= BT_BOX_H) continue;
            const int rs = (Y < 0 ? -Y : 2 * (h - 1) - Y) - (y0 - 3);
            if (rs < 0 || rs >= BT_BOX_H) continue;
            reinterpret_cast<uint32_t*>(&tile[r][0])[cw] = reinterpret_cast<const uint32_t*>(&tile[rs][0])[cw];
        }
        __syncthreads();
    }
    if (x0 == 0 || x0 + BT_W + 3 > w) {
        for (int i = tid; i < 6 * BT_BOX_H; i += 128) {
            const int r = i / 6, k = i - r * 6;
            const int X = k < 3 ? k - 3 : w + (k - 3);
            const int c = X - (x0 - BT_X_PAD);
            if (c < 0 || c >= BT_BOX_W) continue;
            const int cs = (X < 0 ? -X : 2 * (w - 1) - X) - (x0 - BT_X_PAD);
            if (cs < 0 || cs >= BT_BOX_W) continue;
            tile[r][c] = tile[r][cs];
        }
        __syncthreads();
    }
    const int x = x0 + 4 * lane, ys = y0 + 16 * strip;
    if (x >= w || ys >= h) return;
    uint8_t* D = blur + (size_t)frame * blur_frame_bytes + P.dst_off[level];
    const int pitch = P.dst_pitch[level];
    uint32_t hw[7][4];
#pragma unroll
    for (int k = 0; k < 6; ++k) blur_hrow(&tile[16 * strip + k][0], lane, hw[k]);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        blur_hrow(&tile[16 * strip + j + 6][0], lane, hw[(j + 6) % 7]);
        if (ys + j < h) {
            // acc + 32768 <= 255 * 65536 + 32768 (the taps sum to 256 in both passes), so bits 16..23 are the rounded pixel and no clamp is needed:
            // the four result bytes are gathered with three byte permutes instead of shift / or chains
            uint32_t r[4];
#pragma unroll
            for (int q = 0; q < 4; ++q)
                r[q] = 18u * (hw[j % 7][q] + hw[(j + 6) % 7][q]) + 34u * (hw[(j + 1) % 7][q] + hw[(j + 5) % 7][q]) +
                       48u * (hw[(j + 2) % 7][q] + hw[(j + 4) % 7][q]) + 56u * hw[(j + 3) % 7][q] + 32768u;
            const uint32_t out = __byte_perm(__byte_perm(r[0], r[1], 0x0062), __byte_perm(r[2], r[3], 0x0062), 0x5410);
            *reinterpret_cast<uint32_t*>(D + (size_t)(ys + j) * pitch + x) = out;
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// K4b: intensity-centroid angle (IC_Angle) + steered BRIEF (computeOrbDescriptor) + final keypoint record.
// One warp per keypoint slot; 8 warps per CTA. grid (ceil(total_kp / 8), frames).
__device__ __align__(16) const int8_t g_pattern[1024] = {
#include "orb_pattern.inc"
};

__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float p1 = 0.9997878412794807f * (float)(180 / 3.14159265358979323846);
    const float p3 = -0.3258083974640975f * (float)(180 / 3.14159265358979323846);
    const float p5 = 0.1555786518463281f * (float)(180 / 3.14159265358979323846);
    const float p7 = -0.04432655554792128f * (float)(180 / 3.14159265358979323846);
    const float ax = fabsf(x), ay = fabsf(y);
    float a, c, c2;
    if (ax >= ay) {
        c = __fdiv_rn(ay, __fadd_rn(ax, (float)DBL_EPSILON));
        c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = __fdiv_rn(ax, __fadd_rn(ay, (float)DBL_EPSILON));
        c2 = __fmul_rn(c, c);
        a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

#define OD_R 18                       // the pattern's largest radius is 18.38: a rotated, rounded coordinate stays within +-18.  Key points are >= 19 pixels from
                                      // the level border, so the staged rows (and the word-aligned overshoot of <= 3 bytes either side) stay inside the level
#define OD_ROWS (2 * OD_R + 1)
#define OD_WORDS 10                   // 37 bytes + up to 3 bytes of misalignment = 40
__global__ void __launch_bounds__(256) k_orient_describe(OrbGeom g, const uint8_t* __restrict__ gray, const uint8_t* __restrict__ pyr,
                                                         const uint8_t* __restrict__ blur, int blur_frame_bytes,
                                                         const uint32_t* __restrict__ lvl_kp, const int32_t* __restrict__ lvl_cnt,
                                                         pslam_keypoint* __restrict__ kps, uint8_t* __restrict__ desc, int32_t* __restrict__ n_out,
                                                         int cap, int32_t* __restrict__ status) {
    const int frame = blockIdx.y, lane = threadIdx.x & 31;
    const int slot = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (slot >= g.total_kp) return;
    int level = 0;
    while (level + 1 < g.nlevels && slot >= g.lv[level + 1].kp_base) ++level;
    const LevelGeom& L = g.lv[level];
    const int idx = slot - L.kp_base;
    const int32_t* cnts = lvl_cnt + frame * g.nlevels;
    int row = idx, total = 0;
    for (int l = 0; l < g.nlevels; ++l) { const int c = cnts[l]; if (l < level) row += c; total += c; }
    if (slot == 0 && lane == 0) {
        n_out[frame] = total;
        if (total > cap) atomicOr(status + frame, ST_OUT_OVERFLOW);
    }
    if (idx >= cnts[level] || row >= cap) return;

    const uint32_t pk = lvl_kp[(size_t)frame * g.total_kp + slot];
    const int x = kp_x(pk) + 16, y = kp_y(pk) + 16;
    int pitch;
    const uint8_t* img = level_ptr(g, gray, pyr, frame, level, pitch);
    const uint8_t* c = img + (size_t)y * pitch + x;

    // IC_Angle over the radius-15 disc: lane = column u = lane - 15, rows walked in order, so that every load instruction of the warp reads 31 consecutive
    // bytes (one or two sectors) instead of one byte from each of 31 rows; integer moments, so the summation order is free
    int m10 = 0, m01 = 0;
    {
        const int u = lane - 15, au = u < 0 ? -u : u;
        int col = 0;
        if (lane < 31) {
#pragma unroll
            for (int v = -15; v <= 15; ++v) {
                const int val = (au <= g.umax[v < 0 ? -v : v]) ? (int)c[v * pitch + u] : 0;
                col += val; m01 += v * val;
            }
        }
        m10 = u * col;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { m10 += __shfl_xor_sync(0xffffffffu, m10, o); m01 += __shfl_xor_sync(0xffffffffu, m01, o); }
    const float angle = fast_atan2_deg((float)m01, (float)m10);

    // steered BRIEF on the blurred level: the 37 x 37 patch around the key point (the rotated pattern stays within +-18) is staged in shared memory with
    // coalesced word loads, then lane i gathers its 16 samples from there and produces descriptor byte i
    const float ar = __fmul_rn(angle, (float)(3.14159265358979323846 / 180.f));
    const float a = (float)cos((double)ar), b = (float)sin((double)ar);
    const int bp = L.blur_pitch;
    const uint8_t* bc = blur + (size_t)frame * blur_frame_bytes + L.blur_off + (size_t)y * bp + x;
    __shared__ uint32_t s_patch[8][OD_ROWS * OD_WORDS];
    uint32_t* sp = s_patch[threadIdx.x >> 5];
    const uintptr_t left = reinterpret_cast<uintptr_t>(bc - OD_R);
    const int sh = (int)(left & 3);                                    // the patch row starts sh bytes into its first word; bp is a multiple of 4
    const uint8_t* base = bc - OD_R - sh - (size_t)OD_R * bp;           // word-aligned start of the top row
    for (int i = lane; i < OD_ROWS * OD_WORDS; i += 32) {
        const int r = i / OD_WORDS, wd = i - r * OD_WORDS;
        sp[i] = *reinterpret_cast<const uint32_t*>(base + (size_t)r * bp + 4 * wd);
    }
    __syncwarp();
    const uint8_t* sb = reinterpret_cast<const uint8_t*>(sp) + OD_R * (OD_WORDS * 4) + OD_R + sh;      // the key point inside the staged patch
    // lane i owns pattern bytes [32 i, 32 i + 32): eight words read once from global memory (a per-lane index into __constant__ memory would be serialised
    // 32 ways by the constant cache - that was this kernel's limiter)
    uint32_t pw[8];
    {
        const uint4* pp = reinterpret_cast<const uint4*>(g_pattern) + lane * 2;
        const uint4 p0 = __ldg(pp), p1 = __ldg(pp + 1);
        pw[0] = p0.x; pw[1] = p0.y; pw[2] = p0.z; pw[3] = p0.w; pw[4] = p1.x; pw[5] = p1.y; pw[6] = p1.z; pw[7] = p1.w;
    }
    int val = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        int t[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float px = (float)(int)(int8_t)(pw[k] >> (16 * e)), py = (float)(int)(int8_t)(pw[k] >> (16 * e + 8));
            const int yy = __float2int_rn(__fadd_rn(__fmul_rn(px, b), __fmul_rn(py, a)));
            const int xx = __float2int_rn(__fsub_rn(__fmul_rn(px, a), __fmul_rn(py, b)));
            t[e] = sb[yy * (OD_WORDS * 4) + xx];
        }
        val |= (t[0] < t[1]) << k;
    }
    desc[((size_t)frame * cap + row) * 32 + lane] = (uint8_t)val;
    if (lane == 0) {
        pslam_keypoint k;
        k.x = (float)x; k.y = (float)y;
        if (level != 0) { k.x = __fmul_rn(k.x, L.scale); k.y = __fmul_rn(k.y, L.scale); }
        k.size = (float)L.patch_size; k.angle = angle; k.response = (float)kp_s(pk);
        k.octave = level; k.class_id = -1;
        kps[(size_t)frame * cap + row] = k;
    }
}

}  // namespace pslam
