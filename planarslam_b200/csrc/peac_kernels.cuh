// PEAC plane extraction kernels for sm_90a (batched over frames).
//
// Reference semantics (file:line under /root/reference): PlaneDetection::readDepthImage src/PlaneExtractor.cpp:26-57,
// ImagePointCloud::get include/PlaneExtractor.h:25-33, ahc::PlaneSeg ctor include/peac/AHCPlaneSeg.hpp:211-285,
// Stats::compute :125-156, PlaneFitter::initGraph include/peac/AHCPlaneFitter.hpp:786-972, ahCluster :983-1189,
// mergeNbsFrom AHCPlaneSeg.hpp:379-410, findBlockMembership AHCPlaneFitter.hpp:485-587, floodFill :428-476,
// refineDetails :299-379, DisjointSet include/peac/DisjointSet.hpp:64-92.
// Compiled with --fmad=false: every double operation rounds like the unfused CPU oracle.
//
// Work decomposition:
//   k_peac_blocks   one thread per 10x10 block: validity, the nine running sums in row-major order, PCA
//   k_peac_cluster  one warp per frame: graph edges, agglomerative clustering (serial pops, the neighbours of the
//                   popped node are evaluated in parallel by the 32 lanes), plane list, eroded block map
//   k_peac_seed     one CTA per frame: label image / distance map initialisation, region-growing seed queue
//   k_peac_flood    one warp per frame: the FIFO region growing, 8 queue items x 4 neighbours per step with an
//                   exact-order fallback whenever two lanes touch the same pixel
//   k_peac_final    one CTA per frame: last merge over the coarse planes, relabel, per-plane pixel index lists
#pragma once
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

#include "pslam_internal.h"

namespace pslam {

#define PEAC_MAX_PLANES 128          // capacity (640x480 / minSupport = 102 at most); overflow raises a status flag
#define PEAC_PL_WORDS (PEAC_MAX_PLANES / 32)

// ---------------------------------------------------------------------------------------------------------
// cyclic Jacobi eigen-decomposition of a symmetric 3x3 (only + - * / sqrt: bit-identical to oracle/peac.cc)
__device__ __forceinline__ void eig33sym_jacobi(const double K[3][3], double s[3], double V[3][3]) {
    double a[3][3], d[3], b[3], z[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) { a[i][j] = K[i][j]; V[i][j] = (i == j) ? 1.0 : 0.0; }
        d[i] = b[i] = a[i][i];
        z[i] = 0.0;
    }
    for (int sweep = 0; sweep < 50; ++sweep) {
        const double sm = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
        if (sm == 0.0) break;
        const double tresh = (sweep < 3) ? 0.2 * sm / 9.0 : 0.0;
#pragma unroll
        for (int p = 0; p < 2; ++p)
#pragma unroll
            for (int q = p + 1; q < 3; ++q) {
                const double g = 100.0 * fabs(a[p][q]);
                if (sweep > 3 && fabs(d[p]) + g == fabs(d[p]) && fabs(d[q]) + g == fabs(d[q])) {
                    a[p][q] = 0.0;
                } else if (fabs(a[p][q]) > tresh) {
                    double h = d[q] - d[p], t;
                    if (fabs(h) + g == fabs(h)) {
                        t = a[p][q] / h;
                    } else {
                        const double theta = 0.5 * h / a[p][q];
                        t = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));
                        if (theta < 0.0) t = -t;
                    }
                    const double c = 1.0 / sqrt(1.0 + t * t), sn = t * c, tau = sn / (1.0 + c);
                    h = t * a[p][q];
                    z[p] -= h; z[q] += h; d[p] -= h; d[q] += h;
                    a[p][q] = 0.0;
#define PEAC_ROT(i, j, k, l) { const double gg = a[i][j], hh = a[k][l]; a[i][j] = gg - sn * (hh + gg * tau); a[k][l] = hh + sn * (gg - hh * tau); }
                    // for a 3x3 the rotation touches exactly one off-diagonal pair besides (p,q)
                    if (p == 0 && q == 1) { PEAC_ROT(0, 2, 1, 2) }
                    else if (p == 0 && q == 2) { PEAC_ROT(0, 1, 1, 2) }
                    else { PEAC_ROT(0, 1, 0, 2) }
#undef PEAC_ROT
#pragma unroll
                    for (int j = 0; j < 3; ++j) {
                        const double gg = V[j][p], hh = V[j][q];
                        V[j][p] = gg - sn * (hh + gg * tau);
                        V[j][q] = hh + sn * (gg - hh * tau);
                    }
                }
            }
#pragma unroll
        for (int i = 0; i < 3; ++i) { b[i] += z[i]; d[i] = b[i]; z[i] = 0.0; }
    }
    // ascending eigenvalues; the three compare-swaps of the oracle's index sort applied in place (static indices keep
    // everything in registers)
#define PEAC_CSWAP(i, j) if (d[j] < d[i]) { double t_ = d[i]; d[i] = d[j]; d[j] = t_; \
        t_ = V[0][i]; V[0][i] = V[0][j]; V[0][j] = t_; t_ = V[1][i]; V[1][i] = V[1][j]; V[1][j] = t_; t_ = V[2][i]; V[2][i] = V[2][j]; V[2][j] = t_; }
    PEAC_CSWAP(0, 1)
    PEAC_CSWAP(0, 2)
    PEAC_CSWAP(1, 2)
#undef PEAC_CSWAP
    s[0] = d[0]; s[1] = d[1]; s[2] = d[2];
}

// Stats::compute (AHCPlaneSeg.hpp:125-156): geo = {center[3], normal[3], mse, curvature}
__device__ __forceinline__ void peac_stats_compute(const double st[9], int N, double geo[8]) {
    const double sc = 1.0 / N;
    const double sx = st[0], sy = st[1], sz = st[2];
    geo[0] = sx * sc; geo[1] = sy * sc; geo[2] = sz * sc;
    double K[3][3];
    K[0][0] = st[3] - sx * sx * sc; K[0][1] = st[6] - sx * sy * sc; K[0][2] = st[8] - sx * sz * sc;
    K[1][1] = st[4] - sy * sy * sc; K[1][2] = st[7] - sy * sz * sc; K[2][2] = st[5] - sz * sz * sc;
    K[1][0] = K[0][1]; K[2][0] = K[0][2]; K[2][1] = K[1][2];
    double sv[3], V[3][3];
    eig33sym_jacobi(K, sv, V);
    if (V[0][0] * geo[0] + V[1][0] * geo[1] + V[2][0] * geo[2] <= 0) { geo[3] = V[0][0]; geo[4] = V[1][0]; geo[5] = V[2][0]; }
    else { geo[3] = -V[0][0]; geo[4] = -V[1][0]; geo[5] = -V[2][0]; }
    geo[6] = sv[0] * sc;
    geo[7] = sv[0] / (sv[0] + sv[1] + sv[2]);
}

__device__ __forceinline__ double peac_t_mse(const PeacGeom& g, double tol, double z) { const double v = g.depth_sigma * z * z + tol; return v * v; }
__device__ __forceinline__ double peac_t_ang_init(const PeacGeom& g, double z) {
    if (z <= g.z_near) return g.t_ang_init_near;               // the only branch reachable with metre-valued clouds
    const double cz = fmin(z, g.z_far);
    const double factor = (g.angle_far - g.angle_near) / (g.z_far - g.z_near);
    return cos(factor * cz + g.angle_near - factor * g.z_near);
}
__device__ __forceinline__ double peac_sim(const double* ga, const double* gb) {
    return fabs(ga[3] * gb[3] + ga[4] * gb[4] + ga[5] * gb[5]);
}

// ---------------------------------------------------------------------------------------------------------
// K-P1: per-block statistics. grid (ceil(nblk/128), frames), block 128.
__global__ void __launch_bounds__(128) k_peac_blocks(PeacGeom g, const uint16_t* __restrict__ depth, double* __restrict__ blk_st,
                                                     double* __restrict__ blk_geo, int32_t* __restrict__ blk_n, uint8_t* __restrict__ blk_valid) {
    const int b = blockIdx.x * 128 + threadIdx.x, frame = blockIdx.y;
    if (b >= g.nblk) return;
    const int bi = b / g.nbw, bj = b - bi * g.nbw;
    const uint16_t* D = depth + (size_t)frame * g.w * g.h;
    const double scale = (double)g.scale, fx = (double)g.fx, fy = (double)g.fy, cx = (double)g.cx, cy = (double)g.cy;
    double st[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    int n = 0;
    bool valid = true;
    for (int i = bi * g.win, ic = 0; ic < g.win && i < g.h && valid; ++i, ++ic)
        for (int j = bj * g.win, jc = 0; jc < g.win && j < g.w; ++j, ++jc) {
            const int dv = D[(size_t)i * g.w + j];
            if (dv == 0) { valid = false; break; }
            const double z = (double)dv * scale;
            const double tdz = g.depth_alpha * fabs(z) + g.depth_change_tol;
            if (j + 1 < g.w) { const int dn = D[(size_t)i * g.w + j + 1]; if (dn != 0 && fabs(z - (double)dn * scale) > tdz) { valid = false; break; } }
            if (i + 1 < g.h) { const int dn = D[(size_t)(i + 1) * g.w + j]; if (dn != 0 && fabs(z - (double)dn * scale) > tdz) { valid = false; break; } }
            const double x = ((double)j - cx) * z / fx, y = ((double)i - cy) * z / fy;
            st[0] += x; st[1] += y; st[2] += z;
            st[3] += x * x; st[4] += y * y; st[5] += z * z;
            st[6] += x * y; st[7] += y * z; st[8] += x * z;
            ++n;
        }
    double geo[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    bool keep = false;
    if (!valid) { n = 0; for (int k = 0; k < 9; ++k) st[k] = 0; }
    if (n >= 4) {
        peac_stats_compute(st, n, geo);
        keep = valid && geo[6] < peac_t_mse(g, g.std_tol_init, geo[2]);
    } else {
        geo[6] = geo[7] = __longlong_as_double(0x7ff8000000000000LL);
    }
    const size_t o = (size_t)frame * g.nblk + b;
    for (int k = 0; k < 9; ++k) blk_st[o * 9 + k] = st[k];
    for (int k = 0; k < 8; ++k) blk_geo[o * 8 + k] = geo[k];
    blk_n[o] = n;
    blk_valid[o] = keep ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------
// Agglomerative clustering shared by the coarse pass (nodes = blocks) and the last merge (nodes = coarse planes).
struct AhcState {
    int nslots;              // node slots (a merged node reuses the slot of the popped parent)
    int words;               // adjacency bitset words per row
    double* st;              // [nslots][9]
    double* geo;             // [nslots][8]
    int32_t* N;              // [nslots]
    int32_t* rid;            // [nslots]
    int32_t* cid;            // [nslots] creation order (canonical neighbour order)
    uint8_t* alive;          // [nslots] still in the graph
    uint32_t* adj;           // [nslots][words]
    int16_t* wlo;            // [nslots] first / last adjacency word that can hold a set bit (scans are limited to it)
    int16_t* whi;
    uint16_t* heap;          // [nslots]  slot ids (shared memory; nslots <= 65535 is checked at context creation)
    float* keyf;             // [nslots]  float(mse) of every slot (shared memory): the heap orders by it and falls back to the
                             //           double mse in geo[slot*8+6] only when two float keys are equal (rounding is monotone, so
                             //           the order is exactly the double order)
    int32_t* nb_list;        // [nslots] scratch
    int32_t* ds_parent;      // disjoint set over initial blocks
    int32_t* ds_size;
};

__device__ __forceinline__ int ds_find(int32_t* parent, int x) {
    int r = x;
    while (parent[r] != r) r = parent[r];
    while (parent[x] != r) { const int nx = parent[x]; parent[x] = r; x = nx; }
    return r;
}
__device__ __forceinline__ void ds_union(int32_t* parent, int32_t* size, int x, int y) {
    const int xr = ds_find(parent, x), yr = ds_find(parent, y);
    if (xr == yr) return;
    if (size[xr] < size[yr]) { parent[xr] = yr; size[yr] += size[xr]; }
    else { parent[yr] = xr; size[xr] += size[yr]; }
}

// libstdc++ binary-heap algorithms (std::priority_queue<.., PlaneSegMinMSECmp>): comp(a,b) = mse[b] < mse[a]
struct HeapKey {
    const float* kf; const double* geo;
    __device__ __forceinline__ bool comp(int a, int b) const {
        const float fa = kf[a], fb = kf[b];
        if (fb < fa) return true;
        if (fb > fa) return false;
        return geo[(size_t)b * 8 + 6] < geo[(size_t)a * 8 + 6];
    }
};
__device__ __forceinline__ void heap_sift_up(uint16_t* h, const HeapKey& key, int hole, int top, int value) {
    int parent = (hole - 1) / 2;
    while (hole > top && key.comp(h[parent], value)) { h[hole] = h[parent]; hole = parent; parent = (hole - 1) / 2; }
    h[hole] = (uint16_t)value;
}
__device__ __forceinline__ void heap_push(uint16_t* h, int& len, const HeapKey& key, int id) { h[len] = (uint16_t)id; ++len; heap_sift_up(h, key, len - 1, 0, id); }
__device__ __forceinline__ int heap_pop(uint16_t* h, int& len, const HeapKey& key) {
    const int top = h[0], value = h[len - 1];
    --len;
    if (len > 0) {
        int hole = 0, child = 0;
        while (child < (len - 1) / 2) {
            child = 2 * (child + 1);
            if (key.comp(h[child], h[child - 1])) --child;
            h[hole] = h[child]; hole = child;
        }
        if ((len & 1) == 0 && child == (len - 2) / 2) { child = 2 * (child + 1); h[hole] = h[child - 1]; hole = child - 1; }
        heap_sift_up(h, key, hole, 0, value);
    }
    return top;
}

// One warp. heap_len: current heap size (entries already pushed in the reference's order). next_cid: next creation id.
// Extracted slots are appended to ex[i * exs] (at most PEAC_MAX_PLANES; exs = +1 or -1) and finally stable-sorted by N
// descending.  The coarse pass stores them downwards from the last heap entry: every extraction follows a pop that is
// not pushed back, so heap_len + n_ex < nslots whenever an entry is written.
__device__ void ahc_run(const PeacGeom& g, AhcState S, int heap_len, int& next_cid, uint16_t* ex, const int exs, int& n_ex, bool& overflow) {
    const int lane = threadIdx.x & 31;
    const uint32_t full = 0xffffffffu;
    const HeapKey hkey{S.keyf, S.geo};
    int step = 0;
    while (heap_len > 0 && step <= g.max_step) {
        int p = 0;
        if (lane == 0) p = heap_pop(S.heap, heap_len, hkey);
        p = __shfl_sync(full, p, 0);
        heap_len = __shfl_sync(full, heap_len, 0);
        if (!S.alive[p]) continue;
        const int plo = S.wlo[p], phi = S.whi[p];
        // ---- neighbours of p (set bits of its adjacency row), compacted in slot order ----
        int cnt = 0;
        for (int w0 = plo; w0 <= phi; w0 += 32) {
            const int w = w0 + lane;
            uint32_t bits = (w <= phi) ? S.adj[(size_t)p * S.words + w] : 0u;
            const int c = __popc(bits);
            int inc = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(full, inc, o); if (lane >= o) inc += t; }
            int pos = cnt + inc - c;
            while (bits) { const int bpos = __ffs(bits) - 1; bits &= bits - 1; S.nb_list[pos++] = w * 32 + bpos; }
            cnt += __shfl_sync(full, inc, 31);
        }
        __syncwarp();
        // ---- every lane tries the merges lane, lane+32, ... and keeps its best (mse, then creation id) ----
        const double* gp = S.geo + (size_t)p * 8;
        const double* sp = S.st + (size_t)p * 9;
        const int Np = S.N[p];
        double bst[9], bgeo[8];
        int best_nb = -1, best_cid = 0x7fffffff, best_N = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) bgeo[k] = 0;
        for (int i = lane; i < cnt; i += 32) {
            const int q = S.nb_list[i];
            const double* gq = S.geo + (size_t)q * 8;
            if (peac_sim(gp, gq) < g.sim_merge) continue;
            double st[9], geo[8];
            const double* sq = S.st + (size_t)q * 9;
#pragma unroll
            for (int k = 0; k < 9; ++k) st[k] = sp[k] + sq[k];
            const int Nq = S.N[q];
            peac_stats_compute(st, Np + Nq, geo);
            const int cq = S.cid[q];
            if (best_nb < 0 || geo[6] < bgeo[6] || (geo[6] == bgeo[6] && cq < best_cid)) {
                best_nb = q; best_cid = cq; best_N = Np + Nq;
#pragma unroll
                for (int k = 0; k < 9; ++k) bst[k] = st[k];
#pragma unroll
                for (int k = 0; k < 8; ++k) bgeo[k] = geo[k];
            }
        }
        // warp argmin over (mse, cid); lanes without a candidate carry best_nb = -1
        double w_mse = bgeo[6];
        int w_nb = best_nb, w_cid = best_cid;
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const double om = __shfl_xor_sync(full, w_mse, o);
            const int onb = __shfl_xor_sync(full, w_nb, o), oc = __shfl_xor_sync(full, w_cid, o);
            if (onb >= 0 && (w_nb < 0 || om < w_mse || (om == w_mse && oc < w_cid))) { w_mse = om; w_nb = onb; w_cid = oc; }
        }
        // (The reference's tie rule `cand.N < merge.mse` (AHCPlaneFitter.hpp:1045) can only fire when two merges have
        //  bit-identical mse AND mse exceeds the point count; with metre-valued clouds mse << 1, so the first
        //  candidate in canonical order wins a tie, which is what the (mse, cid) order above implements.)
        bool merged = false;
        if (w_nb >= 0) {
            const int nb = w_nb;
            // the lane that evaluated the winning merge broadcasts its sums and PCA
            const int src = __ffs(__ballot_sync(full, best_nb == nb)) - 1;
            double st[9], geo[8];
#pragma unroll
            for (int k = 0; k < 9; ++k) st[k] = __shfl_sync(full, bst[k], src);
#pragma unroll
            for (int k = 0; k < 8; ++k) geo[k] = __shfl_sync(full, bgeo[k], src);
            const int Nc = __shfl_sync(full, best_N, src);
            if (geo[6] < peac_t_mse(g, g.std_tol_merge, geo[2])) {
                merged = true;
                // mergeNbsFrom: union in the disjoint set, new neighbour set = nbs(p) | nbs(nb) - {p, nb}
                const int rid_c = Np >= S.N[nb] ? S.rid[p] : S.rid[nb];
                if (lane == 0) ds_union(S.ds_parent, S.ds_size, S.rid[p], S.rid[nb]);
                const int nlo = S.wlo[nb], nhi = S.whi[nb];
                // every neighbour q of nb: forget nb, learn p (the merged node lives in p's slot)
                for (int w = nlo + lane; w <= nhi; w += 32) {
                    uint32_t bits = S.adj[(size_t)nb * S.words + w];
                    while (bits) {
                        const int q = w * 32 + __ffs(bits) - 1;
                        bits &= bits - 1;
                        if (q == p) continue;
                        atomicAnd(&S.adj[(size_t)q * S.words + (nb >> 5)], ~(1u << (nb & 31)));
                        atomicOr(&S.adj[(size_t)q * S.words + (p >> 5)], 1u << (p & 31));
                        if ((p >> 5) < S.wlo[q]) S.wlo[q] = (int16_t)(p >> 5);      // q is touched by exactly one lane here
                        if ((p >> 5) > S.whi[q]) S.whi[q] = (int16_t)(p >> 5);
                    }
                }
                __syncwarp();
                const int clo = min(plo, nlo), chi = max(phi, nhi);
                for (int w = clo + lane; w <= chi; w += 32) {
                    uint32_t u = S.adj[(size_t)p * S.words + w] | S.adj[(size_t)nb * S.words + w];
                    if (w == (p >> 5)) u &= ~(1u << (p & 31));
                    if (w == (nb >> 5)) u &= ~(1u << (nb & 31));
                    S.adj[(size_t)p * S.words + w] = u;
                    S.adj[(size_t)nb * S.words + w] = 0u;
                }
                if (lane == 0) {      // static indices: st / geo stay in registers
#pragma unroll
                    for (int k = 0; k < 9; ++k) S.st[(size_t)p * 9 + k] = st[k];
#pragma unroll
                    for (int k = 0; k < 8; ++k) S.geo[(size_t)p * 8 + k] = geo[k];
                    S.N[p] = Nc; S.rid[p] = rid_c; S.cid[p] = next_cid; S.alive[nb] = 0; S.keyf[p] = (float)geo[6];
                    S.wlo[p] = (int16_t)clo; S.whi[p] = (int16_t)chi;
                }
                ++next_cid;
                __syncwarp();
                if (lane == 0) heap_push(S.heap, heap_len, hkey, p);
                heap_len = __shfl_sync(full, heap_len, 0);
            }
        }
        if (!merged) {
            if (Np >= g.min_support) { if (n_ex < PEAC_MAX_PLANES) { if (lane == 0) ex[n_ex * exs] = (uint16_t)p; ++n_ex; } else overflow = true; }
            // disconnectAllNbs(p)
            for (int w = plo + lane; w <= phi; w += 32) {
                uint32_t bits = S.adj[(size_t)p * S.words + w];
                while (bits) { const int q = w * 32 + __ffs(bits) - 1; bits &= bits - 1; atomicAnd(&S.adj[(size_t)q * S.words + (p >> 5)], ~(1u << (p & 31))); }
                S.adj[(size_t)p * S.words + w] = 0u;
            }
            if (lane == 0) S.alive[p] = 0;
        }
        __syncwarp();
        ++step;
    }
    // (maxStep is never reached in practice; the reference then just drains the queue, :1168-1175)
    while (heap_len > 0) {
        int p = 0;
        if (lane == 0) p = heap_pop(S.heap, heap_len, hkey);
        p = __shfl_sync(full, p, 0);
        heap_len = __shfl_sync(full, heap_len, 0);
        if (S.alive[p] && S.N[p] >= g.min_support) { if (n_ex < PEAC_MAX_PLANES) { if (lane == 0) ex[n_ex * exs] = (uint16_t)p; ++n_ex; } else overflow = true; }
    }
    __syncwarp();
    if (lane == 0)      // stable insertion sort by N descending (std::sort on <= 16 elements is exactly this)
        for (int i = 1; i < n_ex; ++i) {
            const int v = ex[i * exs];
            int j = i - 1;
            while (j >= 0 && S.N[ex[j * exs]] < S.N[v]) { ex[(j + 1) * exs] = ex[j * exs]; --j; }
            ex[(j + 1) * exs] = (uint16_t)v;
        }
    __syncwarp();
}

// Per-frame plane record written by the cluster / final kernels (also what the ABI returns)
struct PeacPlaneRec {
    double normal[3], center[3], mse, curvature;
    double st[9];
    int32_t N, rid, cid, valid;
};

// K-P2: graph edges + coarse clustering + eroded block map. grid (frames), block 32.
// OCC = resident CTAs per SM the build targets.  12 is what 168 registers and 18 KB of shared memory (float heap keys + u16 heap) allow; the variants above it
// cap the registers at 65536 / (32 OCC) and keep only the 6 KB heap in shared memory (keys in global memory, L1-resident): the kernel is bound by the latency of
// its dependent FP64 chains at ~3 warps per scheduler, so more resident frames trade a little per-frame speed for throughput (PSLAM_PEAC_OCC, measured in DESIGN.md).
template <int OCC>
__global__ void __launch_bounds__(32, OCC) k_peac_cluster(PeacGeom g, const double* __restrict__ blk_st, const double* __restrict__ blk_geo,
                                                     const int32_t* __restrict__ blk_n, const uint8_t* __restrict__ blk_valid,
                                                     double* node_st, double* node_geo, int32_t* node_n, int32_t* node_rid, int32_t* node_cid,
                                                     uint8_t* node_alive, uint32_t* adj, int16_t* wlo_all, int16_t* whi_all, int32_t* nb_list, int32_t* ds_parent,
                                                     int32_t* ds_size, PeacPlaneRec* planes, int32_t* n_planes, int32_t* blk_map,
                                                     int32_t* next_cid_out, int32_t* status, float* keyf_all) {
    const int frame = blockIdx.x, lane = threadIdx.x;
    const size_t fo = (size_t)frame * g.nblk;
    AhcState S;
    S.nslots = g.nblk; S.words = g.adj_words;
    S.st = node_st + fo * 9; S.geo = node_geo + fo * 8; S.N = node_n + fo; S.rid = node_rid + fo; S.cid = node_cid + fo;
    extern __shared__ __align__(16) unsigned char cluster_smem[];
    if (OCC > 12) {
        S.keyf = keyf_all + fo;                                                        // [nblk] in global memory
        S.heap = reinterpret_cast<uint16_t*>(cluster_smem);                            // [nblk]
    } else {
        S.keyf = reinterpret_cast<float*>(cluster_smem);                               // [nblk]
        S.heap = reinterpret_cast<uint16_t*>(cluster_smem + (size_t)g.nblk * sizeof(float));   // [nblk]
    }
    S.alive = node_alive + fo; S.adj = adj + fo * g.adj_words; S.nb_list = nb_list + fo;
    S.wlo = wlo_all + fo; S.whi = whi_all + fo;
    S.ds_parent = ds_parent + fo; S.ds_size = ds_size + fo;
    const uint8_t* valid = blk_valid + fo;
    // node slots = blocks
    for (int b = lane; b < g.nblk; b += 32) {
        for (int k = 0; k < 9; ++k) S.st[(size_t)b * 9 + k] = blk_st[(fo + b) * 9 + k];
        for (int k = 0; k < 8; ++k) S.geo[(size_t)b * 8 + k] = blk_geo[(fo + b) * 8 + k];
        S.N[b] = blk_n[fo + b]; S.rid[b] = b; S.cid[b] = b; S.alive[b] = valid[b];
        S.ds_parent[b] = b; S.ds_size[b] = 1;
        S.keyf[b] = (float)blk_geo[(fo + b) * 8 + 6];
        // a block can only be connected to b-1, b+1, b-Nw, b+Nw
        S.wlo[b] = (int16_t)(max(b - g.nbw, 0) >> 5); S.whi[b] = (int16_t)(min(b + g.nbw, g.nblk - 1) >> 5);
    }
    __syncwarp();
    auto connect = [&](int a, int b) {
        atomicOr(&S.adj[(size_t)a * S.words + (b >> 5)], 1u << (b & 31));
        atomicOr(&S.adj[(size_t)b * S.words + (a >> 5)], 1u << (a & 31));
    };
    const int Nh = g.nbh, Nw = g.nbw;
    // row pass (AHCPlaneFitter.hpp:896-924): rows are independent, the walk along a row is sequential
    for (int i = lane; i < Nh; i += 32)
        for (int j = 1; j < Nw; j += 2) {
            const int c = i * Nw + j;
            if (!valid[c - 1]) { --j; continue; }
            if (!valid[c]) continue;
            if (j < Nw - 1 && !valid[c + 1]) { ++j; continue; }
            const double th = peac_t_ang_init(g, S.geo[(size_t)c * 8 + 2]);
            if ((j < Nw - 1 && peac_sim(S.geo + (size_t)(c - 1) * 8, S.geo + (size_t)(c + 1) * 8) >= th) ||
                (j == Nw - 1 && peac_sim(S.geo + (size_t)c * 8, S.geo + (size_t)(c - 1) * 8) >= th)) {
                connect(c, c - 1);
                if (j < Nw - 1) connect(c, c + 1);
            } else {
                --j;
            }
        }
    // column pass (:926-954)
    for (int j = lane; j < Nw; j += 32)
        for (int i = 1; i < Nh; i += 2) {
            const int c = i * Nw + j;
            if (!valid[c - Nw]) { --i; continue; }
            if (!valid[c]) continue;
            if (i < Nh - 1 && !valid[c + Nw]) { ++i; continue; }
            const double th = peac_t_ang_init(g, S.geo[(size_t)c * 8 + 2]);
            if ((i < Nh - 1 && peac_sim(S.geo + (size_t)(c - Nw) * 8, S.geo + (size_t)(c + Nw) * 8) >= th) ||
                (i == Nh - 1 && peac_sim(S.geo + (size_t)c * 8, S.geo + (size_t)(c - Nw) * 8) >= th)) {
                connect(c, c - Nw);
                if (i < Nh - 1) connect(c, c + Nw);
            } else {
                --i;
            }
        }
    __syncwarp();
    // initial heap: valid blocks pushed in block order (:810-811)
    int heap_len = 0;
    if (lane == 0)
        { const HeapKey hkey{S.keyf, S.geo}; for (int b = 0; b < g.nblk; ++b) if (valid[b]) heap_push(S.heap, heap_len, hkey, b); }
    heap_len = __shfl_sync(0xffffffffu, heap_len, 0);
    __syncwarp();

    uint16_t* ex = S.heap + (g.nblk - 1);          // grows downwards inside the heap array (see ahc_run)
    int n_ex = 0, next_cid = g.nblk;
    bool overflow = false;
    ahc_run(g, S, heap_len, next_cid, ex, -1, n_ex, overflow);
    if (overflow && lane == 0) atomicOr(status + frame, 16);

    PeacPlaneRec* P = planes + (size_t)frame * PEAC_MAX_PLANES;
    for (int i = lane; i < n_ex; i += 32) {
        const int s = ex[-i];
        PeacPlaneRec r;
        for (int k = 0; k < 3; ++k) { r.center[k] = S.geo[(size_t)s * 8 + k]; r.normal[k] = S.geo[(size_t)s * 8 + 3 + k]; }
        r.mse = S.geo[(size_t)s * 8 + 6]; r.curvature = S.geo[(size_t)s * 8 + 7];
        for (int k = 0; k < 9; ++k) r.st[k] = S.st[(size_t)s * 9 + k];
        r.N = S.N[s]; r.rid = S.rid[s]; r.cid = S.cid[s]; r.valid = 0;
        P[i] = r;
    }
    __syncwarp();
    // findBlockMembership (:485-531): a block keeps its plane only if all its 4-neighbours are in the same set
    int32_t* bm = blk_map + fo;
    const int PP = g.win * g.win;
    for (int b = lane; b < g.nblk; b += 32) {
        const int i = b / Nw, j = b - i * Nw;
        const int setid = ds_find(S.ds_parent, b);      // lanes touch disjoint chains only through benign idempotent compression
        int plid = -1;
        if (S.ds_size[setid] * PP >= g.min_support) {
            bool same = true;
            if (j > 0 && ds_find(S.ds_parent, b - 1) != setid) same = false;
            if (same && j < Nw - 1 && ds_find(S.ds_parent, b + 1) != setid) same = false;
            if (same && i > 0 && ds_find(S.ds_parent, b - Nw) != setid) same = false;
            if (same && i < Nh - 1 && ds_find(S.ds_parent, b + Nw) != setid) same = false;
            if (same) {
                plid = 0;                                   // std::map::operator[] default when the root is unknown
                for (int k = 0; k < n_ex; ++k) if (P[k].rid == setid) { plid = k; break; }
                P[plid].valid = 1;
            }
        }
        bm[b] = plid;
    }
    if (lane == 0) { n_planes[frame] = n_ex; next_cid_out[frame] = next_cid; }
}

// ---------------------------------------------------------------------------------------------------------
// K-P3: labels = -1 / plane id of kept blocks, distance map = FLT_MAX, seed queue in block-scan order (:532-575).
// queue entry: pixel index | plane id << 24.  grid (frames), block 256.
__device__ __forceinline__ int peac_seed_count(const PeacGeom& g, const int32_t* bm, int b) {
    const int i = b / g.nbw, j = b - i * g.nbw, W = g.win;
    int n = 0;
    if (bm[b] < 0) {
        if (i > 0 && bm[b - g.nbw] >= 0) n += W - 1;
        if (j > 0 && bm[b - 1] >= 0) n += W - 1;
    } else {
        if (i > 0 && bm[b - g.nbw] != bm[b]) n += W - 1;
        if (j > 0 && bm[b - 1] != bm[b]) n += W - 1;
    }
    return n;
}

// region-growing queue entry: x | y << 12 | plane << 24
__host__ __device__ __forceinline__ uint32_t peac_q_pack(int x, int y, uint32_t plane) { return (uint32_t)x | ((uint32_t)y << 12) | (plane << 24); }

__global__ void __launch_bounds__(256) k_peac_seed(PeacGeom g, const int32_t* __restrict__ blk_map, int32_t* __restrict__ labels,
                                                   float* __restrict__ dist, uint32_t* __restrict__ queue, int32_t* __restrict__ q_len) {
    const int frame = blockIdx.x, tid = threadIdx.x;
    const int32_t* bm = blk_map + (size_t)frame * g.nblk;
    int32_t* lab = labels + (size_t)frame * g.w * g.h;
    float* dm = dist + (size_t)frame * g.w * g.h;
    uint32_t* q = queue + (size_t)frame * g.queue_cap;
    const int npx = g.w * g.h;
    for (int p = tid; p < npx; p += 256) {
        const int y = p / g.w, x = p - y * g.w;
        const int by = y / g.win, bx = x / g.win;
        lab[p] = (by < g.nbh && bx < g.nbw) ? (bm[by * g.nbw + bx] >= 0 ? bm[by * g.nbw + bx] : -1) : -1;
        dm[p] = FLT_MAX;
    }
    // exclusive scan of per-block seed counts: each thread owns a contiguous run of blocks
    __shared__ int s_part[256];
    const int per = (g.nblk + 255) / 256;
    const int b0 = tid * per, b1 = min(g.nblk, b0 + per);
    int mine = 0;
    for (int b = b0; b < b1; ++b) mine += peac_seed_count(g, bm, b);
    s_part[tid] = mine;
    __syncthreads();
    if (tid == 0) { int run = 0; for (int t = 0; t < 256; ++t) { const int v = s_part[t]; s_part[t] = run; run += v; } q_len[frame] = run; }
    __syncthreads();
    int pos = s_part[tid];
    const int W = g.win;
    for (int b = b0; b < b1; ++b) {
        const int i = b / g.nbw, j = b - i * g.nbw;
        if (bm[b] < 0) {
            if (i > 0 && bm[b - g.nbw] >= 0) { const uint32_t pl = (uint32_t)bm[b - g.nbw]; for (int k = 1; k < W; ++k) q[pos++] = peac_q_pack(j * W + k, i * W - 1, pl); }
            if (j > 0 && bm[b - 1] >= 0) { const uint32_t pl = (uint32_t)bm[b - 1]; for (int k = 0; k < W - 1; ++k) q[pos++] = peac_q_pack(j * W - 1, i * W + k, pl); }
        } else {
            const uint32_t pl = (uint32_t)bm[b];
            if (i > 0 && bm[b - g.nbw] != bm[b]) { for (int k = 0; k < W - 1; ++k) q[pos++] = peac_q_pack(j * W + k, i * W, pl); }
            if (j > 0 && bm[b - 1] != bm[b]) { for (int k = 1; k < W; ++k) q[pos++] = peac_q_pack(j * W, i * W + k, pl); }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// K-P4: region growing (floodFill :428-476). One warp per frame; lane = (queue item % 8) * 4 + neighbour.
// The 32 (item, neighbour) touches of a step are independent unless two lanes address the same pixel; lanes that share
// a pixel are applied in lane (= queue) order — exact FIFO semantics, at most 4 rounds.  A touch is split in two:
//   stage A  everything that depends only on immutable data (queue entry, depth, plane records, kept-block map): the
//            neighbour pixel, its distance to the plane and the inlier test.  It is computed ONE STEP AHEAD for the entries
//            already in the queue, so its depth load and FP64 arithmetic overlap the current step instead of extending it.
//   stage B  the order-dependent decision on (label, best distance): the pixel state is loaded once per step, passed
//            between the lanes that share the pixel by shuffles (no memory round trip per round) and stored once.
// Queue entries: x | y << 12 | plane << 24.  Plane records and the block map live in shared memory.
struct FloodPlane { double n[3], c[3], th; };     // th = 9 * mse + 1e-5

__global__ void __launch_bounds__(32) k_peac_flood(PeacGeom g, const uint16_t* __restrict__ depth, const int32_t* __restrict__ blk_map,
                                                   const PeacPlaneRec* __restrict__ planes, const int32_t* __restrict__ n_planes,
                                                   int32_t* __restrict__ labels, float* __restrict__ dist,
                                                   uint32_t* __restrict__ queue, int32_t* __restrict__ q_len, uint32_t* __restrict__ pl_adj,
                                                   int32_t* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char flood_smem[];
    FloodPlane* sP = reinterpret_cast<FloodPlane*>(flood_smem);                       // [PEAC_MAX_PLANES]
    int8_t* sbm = reinterpret_cast<int8_t*>(flood_smem + PEAC_MAX_PLANES * sizeof(FloodPlane));   // [nblk] plane id or -1
    const int frame = blockIdx.x, lane = threadIdx.x;
    const uint32_t full = 0xffffffffu;
    const uint16_t* D = depth + (size_t)frame * g.w * g.h;
    const int32_t* bm = blk_map + (size_t)frame * g.nblk;
    const PeacPlaneRec* P = planes + (size_t)frame * PEAC_MAX_PLANES;
    int32_t* lab = labels + (size_t)frame * g.w * g.h;
    float* dm = dist + (size_t)frame * g.w * g.h;
    uint32_t* q = queue + (size_t)frame * g.queue_cap;
    uint32_t* padj = pl_adj + (size_t)frame * PEAC_MAX_PLANES * PEAC_PL_WORDS;
    const int np = n_planes[frame];
    for (int i = lane; i < np; i += 32) {
        FloodPlane f;
        for (int k = 0; k < 3; ++k) { f.n[k] = P[i].normal[k]; f.c[k] = P[i].center[k]; }
        f.th = 9 * P[i].mse + 1e-5;
        sP[i] = f;
    }
    for (int b = lane; b < g.nblk; b += 32) sbm[b] = (int8_t)bm[b];
    __syncwarp();
    int tail = q_len[frame];
    const double scale = (double)g.scale, fx = (double)g.fx, fy = (double)g.fy, cx = (double)g.cx, cy = (double)g.cy;
    const int item_in_group = lane >> 2, nbr = lane & 3;
    const uint32_t lt_mask = (1u << lane) - 1;
    bool overflow = false;

    struct Touch { int c, x, y, plid; float cdist; bool have, ok; };
    // stage A in three parts, so that the two dependent global loads of a touch - its queue entry, then the depth sample of the neighbour that entry names -
    // are issued a whole step before their values are needed (ncu: 40 % of the kernel's stall samples sat on those two loads when stage A was one function):
    //   a_geom   neighbour pixel of queue entry e for this lane's slot (order of getValid4Neighbor :393-405: left, right, up, down, skipping the ones outside the
    //            image); pixels inside a kept block are skipped by every touch and never change: dropped here, before the conflict test
    //   (load)   the neighbour's depth sample
    //   a_math   distance to the plane and the inlier test
    auto a_geom = [&](uint32_t e) -> Touch {
        Touch t;
        const int sx = e & 0xfff, sy = (e >> 12) & 0xfff;
        t.plid = e >> 24; t.c = -1; t.x = 0; t.y = 0; t.cdist = -1.f; t.ok = false; t.have = false;
        int n = nbr;
        if (sx > 0) { if (n == 0) { t.x = sx - 1; t.y = sy; t.have = true; } --n; }
        if (sx < g.w - 1) { if (n == 0 && !t.have) { t.x = sx + 1; t.y = sy; t.have = true; } --n; }
        if (sy > 0) { if (n == 0 && !t.have) { t.x = sx; t.y = sy - 1; t.have = true; } --n; }
        if (sy < g.h - 1) { if (n == 0 && !t.have) { t.x = sx; t.y = sy + 1; t.have = true; } --n; }
        if (t.have) {
            const int by = (t.y * g.win_magic) >> 16, bx = (t.x * g.win_magic) >> 16;
            if (by < g.nbh && bx < g.nbw && sbm[by * g.nbw + bx] >= 0) t.have = false;
        }
        if (t.have) t.c = t.y * g.w + t.x;
        return t;
    };
    auto a_math = [&](Touch& t, int dv) {
        if (t.have && dv != 0) {
            const FloodPlane& pr = sP[t.plid];
            const double z = (double)dv * scale;
            const double x = ((double)t.x - cx) * z / fx, y = ((double)t.y - cy) * z / fy;
            const double sd = pr.n[0] * (x - pr.c[0]) + pr.n[1] * (y - pr.c[1]) + pr.n[2] * (z - pr.c[2]);
            t.cdist = (float)fabs(sd);
            t.ok = (double)t.cdist * (double)t.cdist < pr.th;
        }
    };

    Touch nxt;
    nxt.c = -1; nxt.x = nxt.y = nxt.plid = 0; nxt.cdist = -1.f; nxt.have = nxt.ok = false;
    int nxt_dv = 0;                                     // depth sample of nxt's pixel, requested during the previous step
    uint32_t e_far = 0;                                 // queue entry head + 16 + item_in_group, requested during the previous step
    bool next_ready = false, far_ready = false;         // nxt / e_far belong to the coming step (warp-uniform)
    for (int head = 0; head < tail;) {
        const int group = min(8, tail - head);          // items consumed by this step (a partial group must not skip later pushes)
        const int k = head + item_in_group;
        Touch t = nxt;
        if (next_ready) a_math(t, nxt_dv);
        else {
            t.have = false; t.c = -1;
            if (item_in_group < group) { t = a_geom(q[k]); a_math(t, t.have ? (int)D[t.c] : 0); }
        }
        // pixel state for this step (mutable: always loaded after the previous step's stores)
        int tr = 0;
        float old = 0.f;
        if (t.have) { tr = lab[t.c]; old = dm[t.c]; }
        // the next step's neighbour and its depth request, for entries that already exist (entries never change once written), plus an L1 prefetch of the two
        // mutable lines it will read; and the queue entries of the step after it
        const bool whole_next = group == 8 && head + 16 <= tail;            // the whole next group is already queued (warp-uniform)
        if (whole_next) {
            nxt = a_geom(far_ready ? e_far : q[k + 8]);
            nxt_dv = nxt.have ? (int)D[nxt.c] : 0;
            if (nxt.have) {
                asm volatile("prefetch.global.L1 [%0];" ::"l"(lab + nxt.c));
                asm volatile("prefetch.global.L1 [%0];" ::"l"(dm + nxt.c));
            }
        }
        next_ready = whole_next;
        far_ready = group == 8 && head + 24 <= tail;                         // then the next step is a whole group with a whole successor: it takes e_far
        if (far_ready) e_far = q[k + 16];
        // ---- stage B: lanes that address the same pixel apply their touches in lane order (:444-473) ----
        const uint32_t peers = __match_any_sync(full, t.have ? t.c : -1 - lane);
        const int rank = __popc(peers & lt_mask);
        int rounds = t.have ? __popc(peers) : 0;
#pragma unroll
        for (int o = 16; o; o >>= 1) rounds = max(rounds, __shfl_xor_sync(full, rounds, o));
        const int tr0 = tr;
        const float old0 = old;
        bool pushed = false;
        uint32_t rem = peers;
        for (int r = 0; r < rounds; ++r) {
            int ntr = tr;
            float nold = old;
            if (t.have && rank == r && tr > -6 && !(tr >= 0 && tr == t.plid)) {
                if (t.ok) {
                    if (tr >= 0) {
                        const FloodPlane& pr = sP[t.plid];
                        const FloodPlane& other = sP[tr];
                        const double sim = fabs(pr.n[0] * other.n[0] + pr.n[1] * other.n[1] + pr.n[2] * other.n[2]);
                        if (sim >= g.sim_refine) {
                            atomicOr(&padj[tr * PEAC_PL_WORDS + (t.plid >> 5)], 1u << (t.plid & 31));
                            atomicOr(&padj[t.plid * PEAC_PL_WORDS + (tr >> 5)], 1u << (tr & 31));
                        }
                    }
                    if (t.cdist < old) { ntr = t.plid; nold = t.cdist; pushed = true; }
                    else if (tr < 0) ntr = tr - 1;
                } else if (tr < 0) ntr = tr - 1;
            }
            // the r-th lane of every pixel group hands the new state to its peers
            const int src = rem ? (__ffs(rem) - 1) : lane;
            rem &= rem - 1;
            tr = __shfl_sync(full, ntr, src);
            old = __shfl_sync(full, nold, src);
        }
        if (t.have && rank == 0) {                       // one store per pixel
            if (tr != tr0) lab[t.c] = tr;
            if (old != old0) dm[t.c] = old;
        }
        const uint32_t pm = __ballot_sync(full, pushed);
        if (pushed) {
            const int pos = tail + __popc(pm & lt_mask);
            if (pos < g.queue_cap) q[pos] = peac_q_pack(t.x, t.y, (uint32_t)t.plid); else overflow = true;
        }
        tail = min(tail + __popc(pm), g.queue_cap);
        head += group;
        __syncwarp();
    }
    if (__any_sync(full, overflow) && lane == 0) atomicOr(status + frame, 32);
    if (lane == 0) q_len[frame] = tail;
}

// ---------------------------------------------------------------------------------------------------------
// K-P5a: last merge over the coarse planes (plane_merge, PlaneExtractor / AHCPlaneFitter.hpp:303-360). grid (frames), block 32.
// Writes the final plane records, the coarse plane -> final plane map (-1: dropped) and the final plane count.
__global__ void __launch_bounds__(32) k_peac_final_merge(PeacGeom g, PeacPlaneRec* __restrict__ planes, const int32_t* __restrict__ n_planes,
                                                         const int32_t* __restrict__ next_cid_in, uint32_t* __restrict__ pl_adj,
                                                         int32_t* ds_parent, int32_t* ds_size, PeacPlaneRec* __restrict__ out_planes,
                                                         pslam_plane* __restrict__ abi_planes, int32_t* __restrict__ out_n,
                                                         int32_t* __restrict__ final_map, int32_t* __restrict__ status) {
    const int frame = blockIdx.x, tid = threadIdx.x;
    __shared__ double s_st[PEAC_MAX_PLANES * 9];
    __shared__ double s_geo[PEAC_MAX_PLANES * 8];
    __shared__ int32_t s_n[PEAC_MAX_PLANES], s_rid[PEAC_MAX_PLANES], s_cid[PEAC_MAX_PLANES], s_nb[PEAC_MAX_PLANES];
    __shared__ uint16_t s_heap[PEAC_MAX_PLANES];
    __shared__ uint8_t s_alive[PEAC_MAX_PLANES];
    __shared__ float s_key[PEAC_MAX_PLANES];
    __shared__ int16_t s_wlo[PEAC_MAX_PLANES], s_whi[PEAC_MAX_PLANES];
    __shared__ uint16_t s_ex[PEAC_MAX_PLANES];
    PeacPlaneRec* P = planes + (size_t)frame * PEAC_MAX_PLANES;
    PeacPlaneRec* O = out_planes + (size_t)frame * PEAC_MAX_PLANES;
    int32_t* fmap = final_map + (size_t)frame * PEAC_MAX_PLANES;
    const int np = n_planes[frame];
    const size_t fo = (size_t)frame * g.nblk;
    for (int i = tid; i < np; i += 32) {
        for (int k = 0; k < 9; ++k) s_st[i * 9 + k] = P[i].st[k];
        for (int k = 0; k < 3; ++k) { s_geo[i * 8 + k] = P[i].center[k]; s_geo[i * 8 + 3 + k] = P[i].normal[k]; }
        s_geo[i * 8 + 6] = P[i].mse; s_geo[i * 8 + 7] = P[i].curvature;
        s_n[i] = P[i].N; s_rid[i] = P[i].rid; s_cid[i] = P[i].cid; s_alive[i] = (uint8_t)P[i].valid;
        s_key[i] = (float)P[i].mse; s_wlo[i] = 0; s_whi[i] = PEAC_PL_WORDS - 1;
    }
    for (int i = tid; i < PEAC_MAX_PLANES; i += 32) fmap[i] = -1;
    __syncwarp();
    AhcState S;
    S.nslots = np; S.words = PEAC_PL_WORDS;
    S.st = s_st; S.geo = s_geo; S.N = s_n; S.rid = s_rid; S.cid = s_cid; S.alive = s_alive;
    S.adj = pl_adj + (size_t)frame * PEAC_MAX_PLANES * PEAC_PL_WORDS;
    S.heap = s_heap; S.keyf = s_key; S.wlo = s_wlo; S.whi = s_whi; S.nb_list = s_nb; S.ds_parent = ds_parent + fo; S.ds_size = ds_size + fo;
    // planes that were eroded completely take no part: drop their adjacency (they never got any) and skip the push
    int heap_len = 0;
    if (tid == 0) { const HeapKey hkey{S.keyf, S.geo}; for (int i = 0; i < np; ++i) if (s_alive[i]) heap_push(S.heap, heap_len, hkey, i); }
    heap_len = __shfl_sync(0xffffffffu, heap_len, 0);
    __syncwarp();
    int n_ex = 0, next_cid = next_cid_in[frame];
    bool overflow = false;
    ahc_run(g, S, heap_len, next_cid, s_ex, 1, n_ex, overflow);
    if (overflow && tid == 0) atomicOr(status + frame, 16);
    // final plane records, and old plane -> final plane map through the disjoint set (:329-344)
    for (int j = tid; j < n_ex; j += 32) {
        const int s = s_ex[j];
        PeacPlaneRec r;
        for (int k = 0; k < 3; ++k) { r.center[k] = s_geo[s * 8 + k]; r.normal[k] = s_geo[s * 8 + 3 + k]; }
        r.mse = s_geo[s * 8 + 6]; r.curvature = s_geo[s * 8 + 7];
        for (int k = 0; k < 9; ++k) r.st[k] = s_st[s * 9 + k];
        r.N = s_n[s]; r.rid = s_rid[s]; r.cid = s_cid[s]; r.valid = 1;
        O[j] = r;
        pslam_plane a;
        for (int k = 0; k < 3; ++k) { a.normal[k] = r.normal[k]; a.center[k] = r.center[k]; }
        a.mse = r.mse; a.curvature = r.curvature; a.N = r.N; a.rid = r.rid;
        abi_planes[(size_t)frame * PEAC_MAX_PLANES + j] = a;
    }
    __syncwarp();
    if (tid == 0) {
        for (int i = 0; i < np; ++i) {
            if (!P[i].valid) continue;
            const int root = ds_find(S.ds_parent, P[i].rid);
            for (int j = 0; j < n_ex; ++j) if (O[j].rid == root) { fmap[i] = j; break; }
        }
        out_n[frame] = n_ex;
    }
}

// K-P5b/c/d: relabel (:362-372) + per-plane pixel lists in ascending pixel order.  The image is cut into sub-chunks of
// PEAC_SUB pixels, one warp each (32 coalesced pixels per row); per-(sub-chunk, plane) counts -> exclusive scan over the
// sub-chunks of a frame -> ordered scatter.  Within a row the rank among pixels of the same plane comes from match_any.
#define PEAC_SUB 1024
#define PEAC_SUB_WARPS 4
__host__ __device__ inline int peac_num_sub(const PeacGeom& g) { return (g.w * g.h + PEAC_SUB - 1) / PEAC_SUB; }
__device__ __forceinline__ int peac_final_id(const int32_t* __restrict__ s_map, int v) { return (v >= 0 && v < PEAC_MAX_PLANES) ? s_map[v] : -1; }

// grid (ceil(nsub / 4), frames), block 128.  counts[frame][sub][plane]
__global__ void __launch_bounds__(32 * PEAC_SUB_WARPS) k_peac_member_count(PeacGeom g, const int32_t* __restrict__ labels, const int32_t* __restrict__ final_map,
                                                                           const int32_t* __restrict__ out_n, int32_t* __restrict__ counts, int nsub) {
    __shared__ int32_t s_map[PEAC_MAX_PLANES];
    __shared__ int32_t s_cnt[PEAC_SUB_WARPS][PEAC_MAX_PLANES];
    const int frame = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sub = blockIdx.x * PEAC_SUB_WARPS + warp;
    const int npx = g.w * g.h;
    for (int i = threadIdx.x; i < PEAC_MAX_PLANES; i += blockDim.x) s_map[i] = final_map[(size_t)frame * PEAC_MAX_PLANES + i];
    for (int i = lane; i < PEAC_MAX_PLANES; i += 32) s_cnt[warp][i] = 0;
    __syncthreads();
    if (sub >= nsub) return;
    const int nf = out_n[frame];
    const int32_t* lab = labels + (size_t)frame * npx;
    const int p0 = sub * PEAC_SUB, p1 = min(npx, p0 + PEAC_SUB);
    for (int base = p0; base < p1; base += 32) {
        const int p = base + lane;
        const int nv = (p < p1) ? peac_final_id(s_map, lab[p]) : -1;
        const uint32_t peers = __match_any_sync(0xffffffffu, nv);
        if (nv >= 0 && (peers & ((1u << lane) - 1)) == 0) s_cnt[warp][nv] += __popc(peers);     // one leader per plane per row
        __syncwarp();
    }
    int32_t* out = counts + ((size_t)frame * nsub + sub) * PEAC_MAX_PLANES;
    for (int k = lane; k < nf; k += 32) out[k] = s_cnt[warp][k];
}

// grid (frames), block 128: thread = plane.  counts -> exclusive prefix over sub-chunks (in place); member_off
__global__ void __launch_bounds__(PEAC_MAX_PLANES) k_peac_member_scan(const int32_t* __restrict__ out_n, int32_t* __restrict__ counts,
                                                                      int32_t* __restrict__ member_off, int nsub) {
    __shared__ int32_t s_tot[PEAC_MAX_PLANES];
    const int frame = blockIdx.x, k = threadIdx.x;
    const int nf = out_n[frame];
    int32_t* cf = counts + (size_t)frame * nsub * PEAC_MAX_PLANES;
    int run = 0;
    if (k < nf)
        for (int sb = 0; sb < nsub; ++sb) { const int v = cf[(size_t)sb * PEAC_MAX_PLANES + k]; cf[(size_t)sb * PEAC_MAX_PLANES + k] = run; run += v; }
    s_tot[k] = (k < nf) ? run : 0;
    __syncthreads();
    if (k == 0) {
        int32_t* moff = member_off + (size_t)frame * (PEAC_MAX_PLANES + 1);
        int acc = 0;
        for (int j = 0; j < nf; ++j) { moff[j] = acc; acc += s_tot[j]; }
        moff[nf] = acc;
    }
}

// grid (ceil(nsub / 4), frames), block 128
__global__ void __launch_bounds__(32 * PEAC_SUB_WARPS) k_peac_member_scatter(PeacGeom g, int32_t* __restrict__ labels, const int32_t* __restrict__ final_map,
                                                                             const int32_t* __restrict__ out_n, const int32_t* __restrict__ counts,
                                                                             const int32_t* __restrict__ member_off, int32_t* __restrict__ member_idx, int nsub) {
    __shared__ int32_t s_map[PEAC_MAX_PLANES];
    __shared__ int32_t s_pos[PEAC_SUB_WARPS][PEAC_MAX_PLANES];
    const int frame = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sub = blockIdx.x * PEAC_SUB_WARPS + warp;
    const int npx = g.w * g.h;
    for (int i = threadIdx.x; i < PEAC_MAX_PLANES; i += blockDim.x) s_map[i] = final_map[(size_t)frame * PEAC_MAX_PLANES + i];
    __syncthreads();
    if (sub >= nsub) return;
    const int nf = out_n[frame];
    const int32_t* base_cnt = counts + ((size_t)frame * nsub + sub) * PEAC_MAX_PLANES;
    const int32_t* moff = member_off + (size_t)frame * (PEAC_MAX_PLANES + 1);
    for (int k = lane; k < nf; k += 32) s_pos[warp][k] = moff[k] + base_cnt[k];
    __syncwarp();
    int32_t* lab = labels + (size_t)frame * npx;
    int32_t* midx = member_idx + (size_t)frame * npx;
    const int p0 = sub * PEAC_SUB, p1 = min(npx, p0 + PEAC_SUB);
    for (int base = p0; base < p1; base += 32) {
        const int p = base + lane;
        const int nv = (p < p1) ? peac_final_id(s_map, lab[p]) : -1;
        const uint32_t peers = __match_any_sync(0xffffffffu, nv);
        if (nv >= 0) {                                  // pixels of other values keep their raw trail counter (:369-371)
            const int rank = __popc(peers & ((1u << lane) - 1));
            const int at = s_pos[warp][nv] + rank;
            lab[p] = nv;
            midx[at] = p;
        }
        __syncwarp();
        if (nv >= 0 && (peers & ((1u << lane) - 1)) == 0) s_pos[warp][nv] += __popc(peers);
        __syncwarp();
    }
}

}  // namespace pslam
