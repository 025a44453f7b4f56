// Plane post-processing of Frame::ComputePlanes (src/Frame.cc:647-753) and Frame::MaxPointDistanceFromPlane (:755-813) on sm_90a: what turns the PEAC result into
// mvPlanePoints / mvPlaneCoefficients, and the surface normals (vSurfaceNormal) that TrackManhattanFrame consumes.  The three PCL algorithms behind those calls
// are not in /root/reference; oracle/planepost.cc restates them (parity unpinned upstream, see its header) and the kernels here are held to that restatement.
//
//   k_planes_post    one CTA per (PEAC plane, frame): bounding box of the member points, voxel accumulation (leaf 0.1 m) into a shared-memory hash table with
//                    ORDER-FREE 64-bit fixed-point sums (atomics), voxels sorted by index, the all-centroids-within-threshold test against the PEAC plane, PCL's
//                    RANSAC (mt19937(12345) sample shuffling, <= 50 iterations, inlier counts by the whole CTA) and the float least-squares refit through the
//                    closed-form eigen33, sign kept like the reference
//   k_planes_compact one thread block per frame: the planes that survive, in PEAC order, with their voxel clouds packed
//   k_sn_*           surface normals of the 3x sub-sampled organised cloud: points + depth-change map (parallel), the two chamfer passes (one warp per frame: the lanes
//                    evaluate the terms from the neighbouring row, lane 0 walks the in-row chain of rounded additions), 3-D gradients + integral images in
//                    double (one warp per frame: rows of gradients built by all lanes, the recurrence walked by one lane per image and component), normals from rectangle sums (parallel), odd rows / columns gathered into vSurfaceNormal
#include <cuda_runtime.h>

#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "pslam_internal.h"

namespace pslam {

#define PP_SLOTS 2048            // occupied voxels per plane (a 20 m^2 plane at 0.1 m); more raise a status flag
#define PP_THREADS 256
#define PP_EMPTY 0xffffffffu
#define PP_MAX_PLANES 128        // >= pslam_peac_max_planes()

struct PlanePostBuffers {
    int max_batch = 0, maxp = 0, w3 = 0, h3 = 0;
    // per (frame, plane) working records
    float* d_coef = nullptr; int32_t* d_valid = nullptr; int32_t* d_npts = nullptr; float* d_pts = nullptr; int32_t* d_stats = nullptr;     // [B][maxp][...]
    // surface normals scratch
    float* d_cloud = nullptr; float* d_dist = nullptr; double *d_ix = nullptr, *d_iy = nullptr;
    float* d_nrm = nullptr;
};

struct PPCam { float fx, fy, cx, cy, scale; };

__device__ __forceinline__ void pp_vertex(const uint16_t* __restrict__ depth, int w, const PPCam& K, int pix, float& x, float& y, float& z) {
    const int i = pix / w, j = pix - i * w;
    const double zz = (double)depth[pix] * (double)K.scale;
    x = (float)(((double)j - (double)K.cx) * zz / (double)K.fx);
    y = (float)(((double)i - (double)K.cy) * zz / (double)K.fy);
    z = (float)zz;
}
__device__ __forceinline__ void pp_vertex_d(uint16_t dval, int w, const PPCam& K, int pix, float& x, float& y, float& z) {      // pp_vertex with the depth sample already loaded
    const int i = pix / w, j = pix - i * w;
    const double zz = (double)dval * (double)K.scale;
    x = (float)(((double)j - (double)K.cx) * zz / (double)K.fx);
    y = (float)(((double)i - (double)K.cy) * zz / (double)K.fy);
    z = (float)zz;
}
__device__ __forceinline__ float pp_dot4(const float c[4], float x, float y, float z) { return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c[0], x), __fmul_rn(c[1], y)), __fmul_rn(c[2], z)), c[3]); }

__device__ uint32_t g_pp_mt[624];    // boost::mt19937(12345) after the first regeneration: identical for every plane, computed once on the host

struct PPRng {                    // boost::mt19937(12345) >> 1, as pcl::SampleConsensusModel::rnd() draws it
    uint32_t* mt; int idx;
    __device__ void seed(uint32_t s) { mt[0] = s; for (int i = 1; i < 624; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i; idx = 624; }
    __device__ uint32_t next() {
        if (idx >= 624) {
            for (int i = 0; i < 624; ++i) {
                const uint32_t y = (mt[i] & 0x80000000u) | (mt[(i + 1) % 624] & 0x7fffffffu);
                mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
            }
            idx = 0;
        }
        uint32_t y = mt[idx++];
        y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
        return y;
    }
    __device__ int rnd() { return (int)(next() >> 1); }
};

// pcl::eigen33 in float (closed-form roots + cross-product eigenvector), see oracle/planepost.cc pcl_eigen33
__device__ void pp_eigen33(const float m_in[3][3], float v[3]) {
    float scale = 0;
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) scale = fmaxf(scale, fabsf(m_in[i][j]));
    if (scale <= FLT_MIN) scale = 1.0f;
    float m[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) m[i][j] = __fdiv_rn(m_in[i][j], scale);
    float r0, r1, r2;
    auto roots2 = [&](float b, float c) {
        r0 = 0.f;
        float d = __fsub_rn(__fmul_rn(b, b), __fmul_rn(4.0f, c));
        if (d < 0.0f) d = 0.0f;
        const float sd = sqrtf(d);
        r2 = __fmul_rn(0.5f, __fadd_rn(b, sd));
        r1 = __fmul_rn(0.5f, __fsub_rn(b, sd));
    };
#define MUL3(a, b, c) __fmul_rn(__fmul_rn(a, b), c)
    float c0 = MUL3(m[0][0], m[1][1], m[2][2]);
    c0 = __fadd_rn(c0, __fmul_rn(MUL3(2.0f, m[0][1], m[0][2]), m[1][2]));
    c0 = __fsub_rn(c0, MUL3(m[0][0], m[1][2], m[1][2]));
    c0 = __fsub_rn(c0, MUL3(m[1][1], m[0][2], m[0][2]));
    c0 = __fsub_rn(c0, MUL3(m[2][2], m[0][1], m[0][1]));
#undef MUL3
    float c1 = __fsub_rn(__fmul_rn(m[0][0], m[1][1]), __fmul_rn(m[0][1], m[0][1]));
    c1 = __fadd_rn(c1, __fmul_rn(m[0][0], m[2][2])); c1 = __fsub_rn(c1, __fmul_rn(m[0][2], m[0][2]));
    c1 = __fadd_rn(c1, __fmul_rn(m[1][1], m[2][2])); c1 = __fsub_rn(c1, __fmul_rn(m[1][2], m[1][2]));
    const float c2 = __fadd_rn(__fadd_rn(m[0][0], m[1][1]), m[2][2]);
    if (fabsf(c0) < FLT_EPSILON) roots2(c2, c1);
    else {
        const float s_inv3 = (float)(1.0 / 3.0), s_sqrt3 = sqrtf(3.0f);
        const float c2_over_3 = __fmul_rn(c2, s_inv3);
        float a_over_3 = __fmul_rn(__fsub_rn(c1, __fmul_rn(c2, c2_over_3)), s_inv3);
        if (a_over_3 > 0.0f) a_over_3 = 0.0f;
        const float half_b = __fmul_rn(0.5f, __fadd_rn(c0, __fmul_rn(c2_over_3, __fsub_rn(__fmul_rn(__fmul_rn(2.0f, c2_over_3), c2_over_3), c1))));
        float q = __fadd_rn(__fmul_rn(half_b, half_b), __fmul_rn(__fmul_rn(a_over_3, a_over_3), a_over_3));
        if (q > 0.0f) q = 0.0f;
        const float rho = sqrtf(-a_over_3);
        const float theta = __fmul_rn(atan2f(sqrtf(-q), half_b), s_inv3);
        const float cos_theta = cosf(theta), sin_theta = sinf(theta);
        r0 = __fadd_rn(c2_over_3, __fmul_rn(__fmul_rn(2.0f, rho), cos_theta));
        r1 = __fsub_rn(c2_over_3, __fmul_rn(rho, __fadd_rn(cos_theta, __fmul_rn(s_sqrt3, sin_theta))));
        r2 = __fsub_rn(c2_over_3, __fmul_rn(rho, __fsub_rn(cos_theta, __fmul_rn(s_sqrt3, sin_theta))));
        if (r0 >= r1) { const float t = r0; r0 = r1; r1 = t; }
        if (r1 >= r2) { const float t = r1; r1 = r2; r2 = t; if (r0 >= r1) { const float u = r0; r0 = r1; r1 = u; } }
        if (r0 <= 0) roots2(c2, c1);
    }
    for (int i = 0; i < 3; ++i) m[i][i] = __fsub_rn(m[i][i], r0);
    auto cross = [](const float a[3], const float b[3], float o[3]) {
        o[0] = __fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1])); o[1] = __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2]));
        o[2] = __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]));
    };
    auto sq = [](const float a[3]) { return __fadd_rn(__fadd_rn(__fmul_rn(a[0], a[0]), __fmul_rn(a[1], a[1])), __fmul_rn(a[2], a[2])); };
    float v1[3], v2[3], v3[3];
    cross(m[0], m[1], v1); cross(m[0], m[2], v2); cross(m[1], m[2], v3);
    const float l1 = sq(v1), l2 = sq(v2), l3 = sq(v3);
    const float* best = (l1 >= l2 && l1 >= l3) ? v1 : (l2 >= l1 && l2 >= l3) ? v2 : v3;
    const float len = sqrtf((l1 >= l2 && l1 >= l3) ? l1 : (l2 >= l1 && l2 >= l3) ? l2 : l3);
    for (int k = 0; k < 3; ++k) v[k] = __fdiv_rn(best[k], len);
}

__global__ void __launch_bounds__(PP_THREADS) k_planes_post(const uint16_t* __restrict__ depth_all, int w, int h, PPCam K, const pslam_plane* __restrict__ planes_all,
                                                            const int32_t* __restrict__ n_planes, const int32_t* __restrict__ midx_all,
                                                            const int32_t* __restrict__ moff_all, int maxp, double dist_th, float* __restrict__ coef_out,
                                                            int32_t* __restrict__ valid_out, int32_t* __restrict__ npts_out, float* __restrict__ pts_out,
                                                            int32_t* __restrict__ stats_out, int32_t* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char pp_smem[];
    unsigned long long* s_sum = reinterpret_cast<unsigned long long*>(pp_smem);                 // [3][PP_SLOTS]
    uint32_t* s_key = reinterpret_cast<uint32_t*>(s_sum + 3 * PP_SLOTS);                          // [PP_SLOTS]
    uint32_t* s_cnt = s_key + PP_SLOTS;                                                           // [PP_SLOTS]
    float* s_px = reinterpret_cast<float*>(s_cnt + PP_SLOTS);                                     // [3][PP_SLOTS] sorted centroids
    uint32_t* s_ord = reinterpret_cast<uint32_t*>(s_px + 3 * PP_SLOTS);                           // [PP_SLOTS] sort keys (voxel index << 11 | slot) / shuffled indices
    uint32_t* s_mt = s_ord + PP_SLOTS;                                                            // [624]
    __shared__ int s_i[8];
    __shared__ float s_model[4];
    const int pl = blockIdx.x, frame = blockIdx.y, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const size_t rec = (size_t)frame * maxp + pl;
    if (pl >= min(n_planes[frame], maxp)) { if (tid == 0) { valid_out[rec] = 0; npts_out[rec] = 0; } return; }
    const uint16_t* depth = depth_all + (size_t)frame * w * h;
    const int32_t* moff = moff_all + (size_t)frame * (maxp + 1);
    const int32_t* midx = midx_all + (size_t)frame * w * h + moff[pl];
    const int nm = moff[pl + 1] - moff[pl];
    for (int i = tid; i < PP_SLOTS; i += PP_THREADS) { s_key[i] = PP_EMPTY; s_cnt[i] = 0; s_sum[i] = 0; s_sum[PP_SLOTS + i] = 0; s_sum[2 * PP_SLOTS + i] = 0; }
    for (int i = tid; i < 624; i += PP_THREADS) s_mt[i] = g_pp_mt[i];
    if (tid == 0) { s_i[0] = 0; s_i[1] = 0; }
    __syncthreads();
    // ---- voxel accumulation (leaf 0.1 m, order-free fixed-point sums) ----
    // pcl::VoxelGrid numbers a voxel i0 + i1 * div0 + i2 * div0 * div1 with i* = floor(coordinate * 10) - floor(minimum * 10): ascending index = lexicographic
    // (i2, i1, i0), which the packed absolute key (iz, iy, ix) below orders identically - so no bounding-box pass is needed.  The members of a plane are in pixel
    // order and neighbouring pixels mostly share a voxel: every thread walks a contiguous run of members and only touches the table when the voxel changes.
    const float inv = 10.0f;                                      // 1.0f / 0.1f rounds to 10.0f
    {
        const int chunk = (nm + PP_THREADS - 1) / PP_THREADS;
        const int i_end = min(nm, (tid + 1) * chunk);
        uint32_t run_key = PP_EMPTY, run_cnt = 0;
        long long rx = 0, ry = 0, rz = 0;
        auto flush = [&]() {
            if (run_key == PP_EMPTY) return;
            uint32_t slot = (run_key * 2654435761u) >> 21;         // 11 bits
            bool placed = false;
            for (int probe = 0; probe < PP_SLOTS; ++probe) {
                const uint32_t cur = atomicCAS(&s_key[slot], PP_EMPTY, run_key);
                if (cur == PP_EMPTY || cur == run_key) { placed = true; break; }
                slot = (slot + 1) & (PP_SLOTS - 1);
            }
            if (!placed) { atomicOr(&s_i[1], 1); return; }
            atomicAdd(&s_cnt[slot], run_cnt);
            atomicAdd(&s_sum[slot], (unsigned long long)rx);
            atomicAdd(&s_sum[PP_SLOTS + slot], (unsigned long long)ry);
            atomicAdd(&s_sum[2 * PP_SLOTS + slot], (unsigned long long)rz);
        };
        // four members per trip: their index and depth loads are issued together (the walk was bound by the latency of one dependent load pair per member)
        for (int ib = tid * chunk; ib < i_end; ib += 4) {
          int pixv[4]; uint16_t dv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) pixv[u] = ib + u < i_end ? midx[ib + u] : -1;
#pragma unroll
          for (int u = 0; u < 4; ++u) dv[u] = pixv[u] >= 0 ? depth[pixv[u]] : (uint16_t)0;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (pixv[u] < 0) continue;
            float x, y, z;
            pp_vertex_d(dv[u], w, K, pixv[u], x, y, z);
            const int i0 = (int)floorf(__fmul_rn(x, inv)) + 512, i1 = (int)floorf(__fmul_rn(y, inv)) + 512, i2 = (int)floorf(__fmul_rn(z, inv));
            if ((unsigned)i0 > 1023u || (unsigned)i1 > 1023u || (unsigned)i2 >= 4095u) { atomicOr(&s_i[1], 1); continue; }      // > 51 m sideways / 409 m deep: capacity flag
            const uint32_t key = ((uint32_t)i2 << 20) | ((uint32_t)i1 << 10) | (uint32_t)i0;
            if (key != run_key) { flush(); run_key = key; run_cnt = 0; rx = ry = rz = 0; }
            ++run_cnt;
            rx += llrint((double)x * 1048576.0); ry += llrint((double)y * 1048576.0); rz += llrint((double)z * 1048576.0);
          }
        }
        flush();
    }
    __syncthreads();
    // ---- order the occupied voxels by index: bitonic sort of (key, slot) pairs; empty slots sort last ----
    // keys can exceed 21 bits, so the pair is sorted as 64-bit values held in two arrays: s_ord (slot) ordered by s_key through an index sort
    for (int i = tid; i < PP_SLOTS; i += PP_THREADS) s_ord[i] = (uint32_t)i;
    __syncthreads();
    for (int size = 2; size <= PP_SLOTS; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < PP_SLOTS / 2; i += PP_THREADS) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool up = ((lo & size) == 0);
                const uint32_t a = s_ord[lo], b = s_ord[hi];
                if ((s_key[a] > s_key[b]) == up) { s_ord[lo] = b; s_ord[hi] = a; }
            }
            __syncthreads();
        }
    if (tid == 0) { int n = 0; while (n < PP_SLOTS && s_key[s_ord[n]] != PP_EMPTY) ++n; s_i[0] = n; }
    __syncthreads();
    const int N = s_i[0];
    for (int i = tid; i < N; i += PP_THREADS) {
        const uint32_t sl = s_ord[i];
        const double n = (double)s_cnt[sl] * 1048576.0;
        s_px[i] = (float)((double)(long long)s_sum[sl] / n);
        s_px[PP_SLOTS + i] = (float)((double)(long long)s_sum[PP_SLOTS + sl] / n);
        s_px[2 * PP_SLOTS + i] = (float)((double)(long long)s_sum[2 * PP_SLOTS + sl] / n);
    }
    __syncthreads();
    // ---- MaxPointDistanceFromPlane: every centroid within the threshold of the PEAC plane ----
    const pslam_plane P = planes_all[rec];
    float coef[4] = {(float)P.normal[0], (float)P.normal[1], (float)P.normal[2],
                     (float)-(P.normal[0] * P.center[0] + P.normal[1] * P.center[1] + P.normal[2] * P.center[2])};
    int bad = 0;
    for (int i = tid; i < N; i += PP_THREADS) bad |= (double)fabsf(pp_dot4(coef, s_px[i], s_px[PP_SLOTS + i], s_px[2 * PP_SLOTS + i])) > dist_th;
    bad = __syncthreads_or(bad);
    if (bad || N < 3) { if (tid == 0) { valid_out[rec] = 0; npts_out[rec] = 0; stats_out[2 * rec] = 0; stats_out[2 * rec + 1] = 0; if (s_i[1]) atomicOr(status + frame, 32); } return; }
    // ---- RANSAC (pcl::RandomSampleConsensus on SampleConsensusModelPlane) ----
    uint32_t* shuffled = s_ord;                                   // the sort order is no longer needed
    for (int i = tid; i < N; i += PP_THREADS) shuffled[i] = (uint32_t)i;
    PPRng rng; rng.mt = s_mt; rng.idx = 0;                       // s_mt: mt19937(12345) after its first twist (copied from g_pp_mt above)
    __syncthreads();
    int best_count = -INT_MAX, iterations = 0;
    double k = 1.0;
    const double log_probability = log(1.0 - 0.99), one_over = 1.0 / (double)N;
    float best[4] = {0, 0, 0, 0};
    bool have = false;
    unsigned skipped = 0;
    while (iterations < k && skipped < 500u) {
        if (tid == 0) {
            int s0 = 0, s1 = 0, s2 = 0;
            bool good = false;
            for (unsigned it = 0; it < 1000 && !good; ++it) {
                for (int i = 0; i < 3; ++i) { const int j = i + (rng.rnd() % (N - i)); const uint32_t t = shuffled[i]; shuffled[i] = shuffled[j]; shuffled[j] = t; }
                s0 = shuffled[0]; s1 = shuffled[1]; s2 = shuffled[2];
                const float d0 = __fdiv_rn(__fsub_rn(s_px[s1], s_px[s0]), __fsub_rn(s_px[s2], s_px[s0]));
                const float d1 = __fdiv_rn(__fsub_rn(s_px[PP_SLOTS + s1], s_px[PP_SLOTS + s0]), __fsub_rn(s_px[PP_SLOTS + s2], s_px[PP_SLOTS + s0]));
                const float d2 = __fdiv_rn(__fsub_rn(s_px[2 * PP_SLOTS + s1], s_px[2 * PP_SLOTS + s0]), __fsub_rn(s_px[2 * PP_SLOTS + s2], s_px[2 * PP_SLOTS + s0]));
                good = (d0 != d1) || (d2 != d1);
            }
            int state = good ? 1 : 0;                             // 0: no sample, 1: model, 2: degenerate (skipped)
            if (good) {
                const float a[3] = {__fsub_rn(s_px[s1], s_px[s0]), __fsub_rn(s_px[PP_SLOTS + s1], s_px[PP_SLOTS + s0]), __fsub_rn(s_px[2 * PP_SLOTS + s1], s_px[2 * PP_SLOTS + s0])};
                const float b[3] = {__fsub_rn(s_px[s2], s_px[s0]), __fsub_rn(s_px[PP_SLOTS + s2], s_px[PP_SLOTS + s0]), __fsub_rn(s_px[2 * PP_SLOTS + s2], s_px[2 * PP_SLOTS + s0])};
                const float e0 = __fdiv_rn(a[0], b[0]), e1 = __fdiv_rn(a[1], b[1]), e2 = __fdiv_rn(a[2], b[2]);
                if (e0 == e1 && e2 == e1) state = 2;
                else {
                    float c[3] = {__fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1])), __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2])),
                                  __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]))};
                    const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(c[0], c[0]), __fmul_rn(c[1], c[1])), __fmul_rn(c[2], c[2])));
                    for (int q = 0; q < 3; ++q) c[q] = __fdiv_rn(c[q], nrm);
                    s_model[0] = c[0]; s_model[1] = c[1]; s_model[2] = c[2];
                    s_model[3] = -1 * __fadd_rn(__fadd_rn(__fmul_rn(c[0], s_px[s0]), __fmul_rn(c[1], s_px[PP_SLOTS + s0])), __fmul_rn(c[2], s_px[2 * PP_SLOTS + s0]));
                }
            }
            s_i[2] = state; s_i[3] = 0;
        }
        __syncthreads();
        const int state = s_i[2];
        if (state == 0) break;
        if (state == 2) { ++skipped; __syncthreads(); continue; }
        const float c[4] = {s_model[0], s_model[1], s_model[2], s_model[3]};
        int cnt = 0;
        for (int i = tid; i < N; i += PP_THREADS) cnt += (double)fabsf(pp_dot4(c, s_px[i], s_px[PP_SLOTS + i], s_px[2 * PP_SLOTS + i])) < dist_th;
        for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if (lane == 0) atomicAdd(&s_i[3], cnt);
        __syncthreads();
        cnt = s_i[3];
        if (cnt > best_count) {
            best_count = cnt; best[0] = c[0]; best[1] = c[1]; best[2] = c[2]; best[3] = c[3]; have = true;
            const double wv = (double)best_count * one_over;
            double p_no = 1.0 - pow(wv, 3.0);
            p_no = fmax(DBL_EPSILON, p_no);
            p_no = fmin(1.0 - DBL_EPSILON, p_no);
            k = log_probability / log(p_no);
        }
        ++iterations;
        __syncthreads();
        if (iterations > 50) break;
    }
    if (!have) { if (tid == 0) { valid_out[rec] = 0; npts_out[rec] = 0; stats_out[2 * rec] = 0; stats_out[2 * rec + 1] = iterations; } return; }
    // ---- optimizeModelCoefficients (thread 0: sequential float moments in index order) + selectWithinDistance with the refined model ----
    if (tid == 0) {
        float acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        int ninl = 0;
        for (int i = 0; i < N; ++i) {
            const float x = s_px[i], y = s_px[PP_SLOTS + i], z = s_px[2 * PP_SLOTS + i];
            if (!((double)fabsf(pp_dot4(best, x, y, z)) < dist_th)) continue;
            ++ninl;
            acc[0] = __fadd_rn(acc[0], __fmul_rn(x, x)); acc[1] = __fadd_rn(acc[1], __fmul_rn(x, y)); acc[2] = __fadd_rn(acc[2], __fmul_rn(x, z));
            acc[3] = __fadd_rn(acc[3], __fmul_rn(y, y)); acc[4] = __fadd_rn(acc[4], __fmul_rn(y, z)); acc[5] = __fadd_rn(acc[5], __fmul_rn(z, z));
            acc[6] = __fadd_rn(acc[6], x); acc[7] = __fadd_rn(acc[7], y); acc[8] = __fadd_rn(acc[8], z);
        }
        float opt[4] = {best[0], best[1], best[2], best[3]};
        if (ninl > 3) {
            for (int q = 0; q < 9; ++q) acc[q] = __fdiv_rn(acc[q], (float)ninl);
            float cov[3][3];
            cov[0][0] = __fsub_rn(acc[0], __fmul_rn(acc[6], acc[6])); cov[0][1] = __fsub_rn(acc[1], __fmul_rn(acc[6], acc[7])); cov[0][2] = __fsub_rn(acc[2], __fmul_rn(acc[6], acc[8]));
            cov[1][1] = __fsub_rn(acc[3], __fmul_rn(acc[7], acc[7])); cov[1][2] = __fsub_rn(acc[4], __fmul_rn(acc[7], acc[8])); cov[2][2] = __fsub_rn(acc[5], __fmul_rn(acc[8], acc[8]));
            cov[1][0] = cov[0][1]; cov[2][0] = cov[0][2]; cov[2][1] = cov[1][2];
            float vec[3];
            pp_eigen33(cov, vec);
            opt[0] = vec[0]; opt[1] = vec[1]; opt[2] = vec[2];
            opt[3] = -1 * __fadd_rn(__fadd_rn(__fmul_rn(opt[0], acc[6]), __fmul_rn(opt[1], acc[7])), __fmul_rn(opt[2], acc[8]));
        }
        s_model[0] = opt[0]; s_model[1] = opt[1]; s_model[2] = opt[2]; s_model[3] = opt[3];
        s_i[3] = 0; s_i[4] = ninl;
    }
    __syncthreads();
    {
        const float c[4] = {s_model[0], s_model[1], s_model[2], s_model[3]};
        int cnt = 0;
        for (int i = tid; i < N; i += PP_THREADS) cnt += (double)fabsf(pp_dot4(c, s_px[i], s_px[PP_SLOTS + i], s_px[2 * PP_SLOTS + i])) < dist_th;
        for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if (lane == 0) atomicAdd(&s_i[3], cnt);
    }
    __syncthreads();
    const int final_inl = s_i[3];
    if (final_inl == 0 || s_i[4] == 0) { if (tid == 0) { valid_out[rec] = 0; npts_out[rec] = 0; } return; }
    float outc[4] = {s_model[0], s_model[1], s_model[2], s_model[3]};
    const float old_d = coef[3], new_d = outc[3];
    if ((new_d < 0 && old_d > 0) || (new_d > 0 && old_d < 0)) for (int q = 0; q < 4; ++q) outc[q] = -outc[q];
    if (tid == 0) {
        for (int q = 0; q < 4; ++q) coef_out[rec * 4 + q] = outc[q];
        valid_out[rec] = 1; npts_out[rec] = N; stats_out[2 * rec] = final_inl; stats_out[2 * rec + 1] = iterations;
        if (s_i[1]) atomicOr(status + frame, 32);
    }
    float* po = pts_out + rec * (size_t)PP_SLOTS * 3;
    for (int i = tid; i < N; i += PP_THREADS) { po[3 * i] = s_px[i]; po[3 * i + 1] = s_px[PP_SLOTS + i]; po[3 * i + 2] = s_px[2 * PP_SLOTS + i]; }
}

// the surviving planes of a frame, in PEAC order: src [maxp], coef [maxp][4], pt_off [maxp + 1], pts packed
__global__ void __launch_bounds__(256) k_planes_compact(int maxp, int cap_pts, const float* __restrict__ coef_w, const int32_t* __restrict__ valid_w, const int32_t* __restrict__ npts_w,
                                                        const float* __restrict__ pts_w, int32_t* __restrict__ n_kept, int32_t* __restrict__ src, float* __restrict__ coef,
                                                        int32_t* __restrict__ pt_off, float* __restrict__ pts, int32_t* __restrict__ status) {
    const int frame = blockIdx.x, tid = threadIdx.x;
    __shared__ int s_slot[PP_MAX_PLANES], s_off[PP_MAX_PLANES + 1], s_n;
    if (tid == 0) {
        int n = 0, off = 0;
        for (int p = 0; p < maxp; ++p) {
            const size_t rec = (size_t)frame * maxp + p;
            if (!valid_w[rec]) continue;
            s_slot[n] = p; s_off[n] = off; off += npts_w[rec]; ++n;
        }
        s_off[n] = off; s_n = n;
        n_kept[frame] = n;
        if (off > cap_pts) atomicOr(status + frame, 64);
    }
    __syncthreads();
    const int n = s_n;
    for (int k = tid; k <= maxp; k += 256) pt_off[(size_t)frame * (maxp + 1) + k] = k <= n ? min(s_off[k], cap_pts) : min(s_off[n], cap_pts);
    for (int k = tid; k < n; k += 256) {
        src[(size_t)frame * maxp + k] = s_slot[k];
        for (int q = 0; q < 4; ++q) coef[((size_t)frame * maxp + k) * 4 + q] = coef_w[((size_t)frame * maxp + s_slot[k]) * 4 + q];
    }
    for (int k = 0; k < n; ++k) {
        const size_t rec = (size_t)frame * maxp + s_slot[k];
        const int cnt = npts_w[rec];
        for (int i = tid; i < cnt * 3; i += 256) { const int o = s_off[k] * 3 + i; if (o < cap_pts * 3) pts[(size_t)frame * cap_pts * 3 + o] = pts_w[rec * (size_t)PP_SLOTS * 3 + i]; }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------------------------------
// surface normals (IntegralImageNormalEstimation, AVERAGE_3D_GRADIENT, max depth change factor 0.05, smoothing size 10, BORDER_POLICY_IGNORE)
__global__ void k_sn_points(const uint16_t* __restrict__ depth_all, int w, int h, int W3, int H3, PPCam K, float* __restrict__ cloud) {
    const int frame = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W3 * H3) return;
    const int r = i / W3, c = i - r * W3, m = 3 * r, n = 3 * c;
    const float d = __fmul_rn((float)depth_all[((size_t)frame * h + m) * w + n], K.scale);
    float* p = cloud + ((size_t)frame * W3 * H3 + i) * 3;
    p[2] = d; p[0] = __fdiv_rn(__fmul_rn(__fsub_rn((float)n, K.cx), d), K.fx); p[1] = __fdiv_rn(__fmul_rn(__fsub_rn((float)m, K.cy), d), K.fy);
}
// depth-change map -> initial distance map (0 at a depth change, W3 + H3 elsewhere): one thread per point.  The reference loop visits (ri, ci) with ri < H3 - 1,
// ci < W3 - 1 and clears the visited point and its right / lower neighbour when the depth step exceeds the tolerance: a point is cleared by its own two tests, by
// the right-test of its left neighbour or by the down-test of its upper neighbour.  dist has one guard element before and after the image.
__device__ __forceinline__ bool sn_step(float dep, float other) {
    const float tol = __fmul_rn(__fmul_rn(0.05f, __fadd_rn(fabsf(dep), 1.0f)), 2.0f);
    return fabsf(__fsub_rn(dep, other)) > tol || !isfinite(dep) || !isfinite(other);
}
__global__ void k_sn_change(int W3, int H3, const float* __restrict__ cloud_all, float* __restrict__ dist_all) {
    const int frame = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t NP = (size_t)W3 * H3;
    if (i >= W3 * H3) return;
    const float* pts = cloud_all + (size_t)frame * NP * 3;
    float* dist = dist_all + (size_t)frame * (NP + 2);
    const int r = i / W3, c = i - r * W3;
    const float dep = pts[(size_t)i * 3 + 2];
    bool cleared = false;
    if (r < H3 - 1 && c < W3 - 1) cleared = sn_step(dep, pts[((size_t)i + 1) * 3 + 2]) || sn_step(dep, pts[((size_t)i + W3) * 3 + 2]);
    if (!cleared && c >= 1 && r < H3 - 1) cleared = sn_step(pts[((size_t)i - 1) * 3 + 2], dep);
    if (!cleared && r >= 1 && c < W3 - 1) cleared = sn_step(pts[((size_t)i - W3) * 3 + 2], dep);
    const float far = (float)(W3 + H3);
    dist[1 + i] = cleared ? 0.0f : far;
    if (i == 0) { dist[0] = far; dist[NP + 1] = far; }
}
// The two chamfer passes (1.0 / 1.4 weights, float): one warp per frame.  Each row's three terms from the neighbouring row are evaluated by all lanes; what
// remains is d[c] = min(m[c], d[c -+ 1] + 1.0f) along the row, a chain of rounded float additions that lane 0 walks in order (the rounding of x + 1.0f + 1.0f ...
// is not that of x + n, so the chain is kept).  Like the reference loop, the forward pass reads prev[W3] = cur[0] and the backward pass next[-1] = cur[W3 - 1].
#define SN_WARPS 4
__global__ void __launch_bounds__(SN_WARPS * 32) k_sn_chamfer(int nframes, int W3, int H3, float* __restrict__ dist_all) {
    extern __shared__ __align__(16) unsigned char sn_smem[];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, frame = blockIdx.x * SN_WARPS + wid;
    if (frame >= nframes) return;
    const int RS = W3 + 2;                                             // row stride in shared memory: element c lives at [c + 1]
    float* rowA = reinterpret_cast<float*>(sn_smem) + (size_t)wid * 3 * RS;
    float* rowB = rowA + RS;
    float* m = rowB + RS;
    const size_t NP = (size_t)W3 * H3;
    float* dm = dist_all + (size_t)frame * (NP + 2) + 1;
    float* prev = rowA; float* cur = rowB;
    for (int c = lane; c < W3; c += 32) prev[c + 1] = dm[c];
    for (int ri = 1; ri < H3; ++ri) {
        float* g = dm + (size_t)ri * W3;
        for (int c = lane; c < W3; c += 32) cur[c + 1] = g[c];
        __syncwarp();
        if (lane == 0) prev[W3 + 1] = cur[1];
        __syncwarp();
        for (int c = 1 + lane; c < W3; c += 32)
            m[c] = fminf(fminf(cur[c + 1], __fadd_rn(prev[c], 1.4f)), fminf(__fadd_rn(prev[c + 1], 1.0f), __fadd_rn(prev[c + 2], 1.4f)));
        __syncwarp();
        if (lane == 0) {
            float d = cur[1];
#pragma unroll 8
            for (int c = 1; c < W3; ++c) { d = fminf(m[c], __fadd_rn(d, 1.0f)); cur[c + 1] = d; }
        }
        __syncwarp();
        for (int c = lane; c < W3; c += 32) g[c] = cur[c + 1];
        float* t = prev; prev = cur; cur = t;
    }
    // backward: `prev` holds the last row (its final values)
    float* next = prev;
    for (int ri = H3 - 2; ri >= 0; --ri) {
        float* g = dm + (size_t)ri * W3;
        for (int c = lane; c < W3; c += 32) cur[c + 1] = g[c];
        __syncwarp();
        if (lane == 0) next[0] = cur[W3];
        __syncwarp();
        for (int c = lane; c < W3 - 1; c += 32)
            m[c] = fminf(fminf(cur[c + 1], __fadd_rn(next[c], 1.4f)), fminf(__fadd_rn(next[c + 1], 1.0f), __fadd_rn(next[c + 2], 1.4f)));
        __syncwarp();
        if (lane == 0) {
            float d = cur[W3];
#pragma unroll 8
            for (int c = W3 - 2; c >= 0; --c) { d = fminf(m[c], __fadd_rn(d, 1.0f)); cur[c + 1] = d; }
        }
        __syncwarp();
        for (int c = lane; c < W3; c += 32) g[c] = cur[c + 1];
        float* t = next; next = cur; cur = t;
    }
}
// 3-D gradients (central differences of the organised cloud, zero on the image border) and their integral images in double, one warp per frame: all lanes
// build row r of the six gradient components in shared memory; lanes 0..5 (image x / y, component) then walk the recurrence
//     I[r+1][c+1] = (I[r][c+1] + I[r+1][c]) - I[r][c]  (+ element when the 3-vector is finite)
// along the row in place over the previous row (the rounding of every step is the reference's), and all lanes store the finished row.
__global__ void __launch_bounds__(SN_WARPS * 32) k_sn_integral(int nframes, int W3, int H3, const float* __restrict__ cloud_all, double* __restrict__ ix_all, double* __restrict__ iy_all) {
    extern __shared__ __align__(16) unsigned char sn_smem[];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, frame = blockIdx.x * SN_WARPS + wid;
    if (frame >= nframes) return;
    const int RI = (W3 + 1) * 3, RE = W3 * 3;
    const size_t per_warp = (size_t)2 * RI * sizeof(double) + (size_t)2 * RE * sizeof(float);
    double* buf = reinterpret_cast<double*>(sn_smem + (size_t)wid * ((per_warp + 15) & ~(size_t)15));     // [2][RI]
    float* e = reinterpret_cast<float*>(buf + 2 * RI);                                                    // [2][RE]
    const size_t NP = (size_t)W3 * H3, NI = (size_t)(W3 + 1) * (H3 + 1);
    const float* pts = cloud_all + (size_t)frame * NP * 3;
    double* IX = ix_all + (size_t)frame * NI * 3;
    double* IY = iy_all + (size_t)frame * NI * 3;
    for (int i = lane; i < 2 * RI; i += 32) buf[i] = 0.0;
    for (int i = lane; i < RI; i += 32) { IX[i] = 0.0; IY[i] = 0.0; }
    __syncwarp();
    for (int r = 0; r < H3; ++r) {
        const bool inner_r = r >= 1 && r < H3 - 1;
        const float* row = pts + (size_t)r * W3 * 3;
        for (int i = lane; i < RE; i += 32) {
            float gx = 0.0f, gy = 0.0f;
            if (inner_r && i >= 3 && i < RE - 3) { gx = __fsub_rn(row[i + 3], row[i - 3]); gy = __fsub_rn(row[i + RE], row[i - RE]); }
            e[i] = gx; e[RE + i] = gy;
        }
        __syncwarp();
        if (lane < 6) {
            const int which = lane / 3, k = lane - which * 3;
            double* b = buf + which * RI;
            const float* ev = e + which * RE;
            double left = 0.0, pc = b[k];                                 // I[r][0] (= 0)
            b[k] = 0.0;                                                   // I[r + 1][0]
            for (int c = 0; c < W3; ++c) {
                const double pc1 = b[(c + 1) * 3 + k];
                double v = __dsub_rn(__dadd_rn(pc1, left), pc);
                const float e0 = ev[c * 3], e1 = ev[c * 3 + 1], e2 = ev[c * 3 + 2];
                if (isfinite(e0) && isfinite(e1) && isfinite(e2)) v = __dadd_rn(v, (double)ev[c * 3 + k]);
                b[(c + 1) * 3 + k] = v;
                left = v; pc = pc1;
            }
        }
        __syncwarp();
        double* ox = IX + (size_t)(r + 1) * RI; double* oy = IY + (size_t)(r + 1) * RI;
        for (int i = lane; i < RI; i += 32) { ox[i] = buf[i]; oy[i] = buf[RI + i]; }
        __syncwarp();
    }
}
__global__ void k_sn_normals(int W3, int H3, const float* __restrict__ cloud_all, const float* __restrict__ dist_all, const double* __restrict__ ix_all,
                             const double* __restrict__ iy_all, float* __restrict__ nrm_all) {
    const int frame = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W3 * H3) return;
    const int ri = i / W3, ci = i - ri * W3;
    const size_t NP = (size_t)W3 * H3, NI = (size_t)(W3 + 1) * (H3 + 1);
    const float nanv = __int_as_float(0x7fc00000);
    float out[3] = {nanv, nanv, nanv};
    const int border = 10, bottom = H3 > border ? H3 - border : 0, right = W3 > border ? W3 - border : 0;
    const float* p = cloud_all + ((size_t)frame * NP + i) * 3;
    if (ri >= border && ri < bottom && ci >= border && ci < right && isfinite(p[2])) {
        const float smoothing = fminf(dist_all[(size_t)frame * (NP + 2) + 1 + i], 10.0f);
        if (smoothing > 2.0f) {
            const int rw = (int)smoothing, rw2 = rw / 2, sx = ci - rw2, sy = ri - rw2;
            const double* IX = ix_all + (size_t)frame * NI * 3;
            const double* IY = iy_all + (size_t)frame * NI * 3;
            const size_t ul = (size_t)sy * (W3 + 1) + sx, ur = ul + rw, ll = (size_t)(sy + rw) * (W3 + 1) + sx, lr = ll + rw;
            double gx[3], gy[3];
            for (int k = 0; k < 3; ++k) {
                gx[k] = __dsub_rn(__dsub_rn(__dadd_rn(IX[lr * 3 + k], IX[ul * 3 + k]), IX[ur * 3 + k]), IX[ll * 3 + k]);
                gy[k] = __dsub_rn(__dsub_rn(__dadd_rn(IY[lr * 3 + k], IY[ul * 3 + k]), IY[ur * 3 + k]), IY[ll * 3 + k]);
            }
            const double nv[3] = {__dsub_rn(__dmul_rn(gy[1], gx[2]), __dmul_rn(gy[2], gx[1])), __dsub_rn(__dmul_rn(gy[2], gx[0]), __dmul_rn(gy[0], gx[2])),
                                  __dsub_rn(__dmul_rn(gy[0], gx[1]), __dmul_rn(gy[1], gx[0]))};
            const double len = __dadd_rn(__dadd_rn(__dmul_rn(nv[0], nv[0]), __dmul_rn(nv[1], nv[1])), __dmul_rn(nv[2], nv[2]));
            if (len != 0.0) {
                const double s = sqrt(len);
                float nx = (float)(nv[0] / s), ny = (float)(nv[1] / s), nz = (float)(nv[2] / s);
                const float vx = __fsub_rn(0.f, p[0]), vy = __fsub_rn(0.f, p[1]), vz = __fsub_rn(0.f, p[2]);
                const float cos_theta = __fadd_rn(__fadd_rn(__fmul_rn(vx, nx), __fmul_rn(vy, ny)), __fmul_rn(vz, nz));
                if (cos_theta < 0) { nx = -nx; ny = -ny; nz = -nz; }
                out[0] = nx; out[1] = ny; out[2] = nz;
            }
        }
    }
    for (int k = 0; k < 3; ++k) nrm_all[((size_t)frame * NP + i) * 3 + k] = out[k];
}
// vSurfaceNormal: odd rows and columns of the sub-sampled grid -> [n][8] = normal, camera position, frame position
__global__ void k_sn_gather(int W3, int H3, const float* __restrict__ cloud_all, const float* __restrict__ nrm_all, float* __restrict__ out8, float* __restrict__ out3, int n_out) {
    const int frame = blockIdx.y, o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= n_out) return;
    const int cols = W3 / 2, r = o / cols, c = o - r * cols, m = 2 * r + 1, n = 2 * c + 1;
    const size_t NP = (size_t)W3 * H3, idx = (size_t)m * W3 + n;
    float* d = out8 + ((size_t)frame * n_out + o) * 8;
    for (int k = 0; k < 3; ++k) { d[k] = nrm_all[((size_t)frame * NP + idx) * 3 + k]; d[3 + k] = cloud_all[((size_t)frame * NP + idx) * 3 + k]; }
    d[6] = (float)(n * 3); d[7] = (float)(m * 3);
    if (out3) for (int k = 0; k < 3; ++k) out3[((size_t)frame * n_out + o) * 3 + k] = d[k];      // the normals alone, the layout pslam_track_manhattan_batch_dev reads
}

void planepost_free(pslam_ctx* c) {
    if (!c->planepost) return;
    PlanePostBuffers& B = *c->planepost;
    for (void* p : {(void*)B.d_coef, (void*)B.d_valid, (void*)B.d_npts, (void*)B.d_pts, (void*)B.d_stats, (void*)B.d_cloud, (void*)B.d_dist, (void*)B.d_ix, (void*)B.d_iy, (void*)B.d_nrm})
        if (p) cudaFree(p);
    delete c->planepost;
    c->planepost = nullptr;
}

static int planepost_alloc(pslam_ctx* c) {
    if (c->planepost) return PSLAM_OK;
    PlanePostBuffers* Bp = new PlanePostBuffers();
    PlanePostBuffers& B = *Bp;
    c->planepost = Bp;
    B.max_batch = c->cfg.max_batch; B.maxp = pslam_peac_max_planes(c);
    if (B.maxp > PP_MAX_PLANES) { planepost_free(c); return set_error(c, PSLAM_E_INVALID, "plane capacity above the post-processing limit"); }
    B.w3 = (c->cfg.width + 2) / 3; B.h3 = (c->cfg.height + 2) / 3;
    {   // mt19937(12345) seeded and regenerated once (what the first draw of every RANSAC run sees)
        uint32_t mt[624];
        mt[0] = 12345u;
        for (int i = 1; i < 624; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
        for (int i = 0; i < 624; ++i) {
            const uint32_t y = (mt[i] & 0x80000000u) | (mt[(i + 1) % 624] & 0x7fffffffu);
            mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        const int rc_ = check_cuda(c, cudaMemcpyToSymbol(g_pp_mt, mt, sizeof mt), "cudaMemcpyToSymbol(mt19937)");
        if (rc_ != PSLAM_OK) { planepost_free(c); return rc_; }
    }
    const size_t nb = B.max_batch, np = (size_t)B.w3 * B.h3, ni = (size_t)(B.w3 + 1) * (B.h3 + 1);
#define PA(ptr, bytes) do { const int rc_ = check_cuda(c, cudaMalloc((void**)&(ptr), (bytes)), "cudaMalloc(planepost)"); if (rc_ != PSLAM_OK) { planepost_free(c); return rc_; } } while (0)
    PA(B.d_coef, nb * B.maxp * 16); PA(B.d_valid, nb * B.maxp * 4); PA(B.d_npts, nb * B.maxp * 4); PA(B.d_stats, nb * B.maxp * 8);
    PA(B.d_pts, nb * B.maxp * (size_t)PP_SLOTS * 12);
    PA(B.d_cloud, nb * np * 12); PA(B.d_dist, nb * (np + 2) * 4);
    PA(B.d_ix, nb * ni * 24); PA(B.d_iy, nb * ni * 24); PA(B.d_nrm, nb * np * 12);
#undef PA
    return PSLAM_OK;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_surface_normals_count(const pslam_ctx* c) { return c ? (((c->cfg.width + 2) / 3) / 2) * (((c->cfg.height + 2) / 3) / 2) : 0; }
int pslam_planes_post_max_points(const pslam_ctx*) { return PP_SLOTS; }

int pslam_planes_post_batch_dev(pslam_ctx* c, const uint16_t* d_depth, int nframes, const pslam_plane* d_planes, const int32_t* d_nplanes, const int32_t* d_member_idx,
                                const int32_t* d_member_off, float dist_th, int32_t* d_n_kept, int32_t* d_src, float* d_coef, int32_t* d_pt_off, float* d_pts, int cap_pts,
                                int32_t* d_status) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_depth || !d_planes || !d_nplanes || !d_member_idx || !d_member_off || !d_n_kept || !d_src || !d_coef || !d_pt_off || !d_pts || !d_status || cap_pts < 1 || nframes < 1 ||
        nframes > c->cfg.max_batch)
        return set_error(c, PSLAM_E_INVALID, "planes post: null pointer or nframes outside [1, max_batch]");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    int rc = planepost_alloc(c);
    if (rc != PSLAM_OK) return rc;
    PlanePostBuffers& B = *c->planepost;
    cudaStream_t st = c->stream;
    const PPCam K{c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy, c->cfg.depth_scale};
    const size_t smem = (size_t)PP_SLOTS * (3 * 8 + 4 + 4 + 3 * 4 + 4) + 624 * 4;
    PSLAM_CUDA(c, cudaFuncSetAttribute(k_planes_post, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PSLAM_CUDA(c, cudaMemsetAsync(d_status, 0, (size_t)nframes * 4, st));
    PSLAM_LAUNCH(c, "planes_post", k_planes_post<<<dim3(B.maxp, nframes), PP_THREADS, smem, st>>>(d_depth, c->cfg.width, c->cfg.height, K, d_planes, d_nplanes, d_member_idx,
                 d_member_off, B.maxp, (double)dist_th, B.d_coef, B.d_valid, B.d_npts, B.d_pts, B.d_stats, d_status));
    PSLAM_LAUNCH(c, "planes_compact", k_planes_compact<<<nframes, 256, 0, st>>>(B.maxp, cap_pts, B.d_coef, B.d_valid, B.d_npts, B.d_pts, d_n_kept, d_src, d_coef, d_pt_off,
                 d_pts, d_status));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

int pslam_surface_normals_batch_dev(pslam_ctx* c, const uint16_t* d_depth, int nframes, float* d_normals8, float* d_normals3) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_depth || !d_normals8 || nframes < 1 || nframes > c->cfg.max_batch) return set_error(c, PSLAM_E_INVALID, "surface normals: null pointer or nframes outside [1, max_batch]");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    int rc = planepost_alloc(c);
    if (rc != PSLAM_OK) return rc;
    PlanePostBuffers& B = *c->planepost;
    cudaStream_t st = c->stream;
    const PPCam K{c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy, c->cfg.depth_scale};
    const int np = B.w3 * B.h3, n_out = pslam_surface_normals_count(c);
    const dim3 gp((np + 255) / 256, nframes);
    PSLAM_LAUNCH(c, "sn_points", k_sn_points<<<gp, 256, 0, st>>>(d_depth, c->cfg.width, c->cfg.height, B.w3, B.h3, K, B.d_cloud));
    const size_t smem_ch = (size_t)SN_WARPS * 3 * (B.w3 + 2) * sizeof(float);
    const size_t smem_ii = (size_t)SN_WARPS * (((size_t)2 * (B.w3 + 1) * 3 * sizeof(double) + (size_t)2 * B.w3 * 3 * sizeof(float) + 15) & ~(size_t)15);
    if (smem_ch > 227 * 1024 || smem_ii > 227 * 1024) return set_error(c, PSLAM_E_INVALID, "surface normals: image too wide for the row buffers");
    // (the attribute is per device and contexts may live on several devices of one process: set it on every call, it is a cheap driver query)
    if (smem_ch > 48 * 1024) PSLAM_CUDA(c, cudaFuncSetAttribute(k_sn_chamfer, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ch));
    if (smem_ii > 48 * 1024) PSLAM_CUDA(c, cudaFuncSetAttribute(k_sn_integral, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ii));
    PSLAM_LAUNCH(c, "sn_change", k_sn_change<<<gp, 256, 0, st>>>(B.w3, B.h3, B.d_cloud, B.d_dist));
    PSLAM_LAUNCH(c, "sn_chamfer", k_sn_chamfer<<<(nframes + SN_WARPS - 1) / SN_WARPS, SN_WARPS * 32, smem_ch, st>>>(nframes, B.w3, B.h3, B.d_dist));
    PSLAM_LAUNCH(c, "sn_integral", k_sn_integral<<<(nframes + SN_WARPS - 1) / SN_WARPS, SN_WARPS * 32, smem_ii, st>>>(nframes, B.w3, B.h3, B.d_cloud, B.d_ix, B.d_iy));
    PSLAM_LAUNCH(c, "sn_normals", k_sn_normals<<<gp, 256, 0, st>>>(B.w3, B.h3, B.d_cloud, B.d_dist, B.d_ix, B.d_iy, B.d_nrm));
    PSLAM_LAUNCH(c, "sn_gather", k_sn_gather<<<dim3((n_out + 255) / 256, nframes), 256, 0, st>>>(B.w3, B.h3, B.d_cloud, B.d_nrm, d_normals8, d_normals3, n_out));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

// Frame::ComputePlanes for nframes host depth images: PEAC + the post-processing + the surface normals.  Outputs: n_kept [nframes], src / coef [nframes][maxp] ([4]),
// pt_off [nframes][maxp + 1], pts [nframes][cap_pts][3], normals8 [nframes][pslam_surface_normals_count()][8] (may be NULL)
int pslam_compute_planes_batch(pslam_ctx* c, const uint16_t* depth, int nframes, float dist_th, int32_t* n_kept, int32_t* src, float* coef, int32_t* pt_off, float* pts,
                               int cap_pts, float* normals8) {
    if (!c) return PSLAM_E_INVALID;
    if (!depth || !n_kept || !src || !coef || !pt_off || !pts || cap_pts < 1 || nframes < 1 || nframes > c->cfg.max_batch) return set_error(c, PSLAM_E_INVALID, "compute planes: bad arguments");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const int maxp = pslam_peac_max_planes(c), n_sn = pslam_surface_normals_count(c);
    const size_t npx = (size_t)c->cfg.width * c->cfg.height, nf = (size_t)nframes;
    const size_t sz[] = {nf * npx * 2, nf * npx * 4, nf * maxp * sizeof(pslam_plane), nf * 4, nf * npx * 4, nf * (maxp + 1) * 4, nf * 4, nf * maxp * 4, nf * maxp * 16,
                         nf * (maxp + 1) * 4, nf * cap_pts * 12, nf * 4, nf * n_sn * 32};
    size_t off[14]; off[0] = 0;
    for (int i = 0; i < 13; ++i) off[i + 1] = (off[i] + sz[i] + 255) & ~(size_t)255;
    uint8_t* d = nullptr;
    PSLAM_CUDA(c, cudaMalloc((void**)&d, off[13]));
    cudaStream_t st = c->stream;
    cudaMemcpyAsync(d + off[0], depth, sz[0], cudaMemcpyHostToDevice, st);
    int rc = pslam_peac_run_batch_dev(c, (const uint16_t*)(d + off[0]), nframes, (int32_t*)(d + off[1]), (pslam_plane*)(d + off[2]), (int32_t*)(d + off[3]), (int32_t*)(d + off[4]),
                                      (int32_t*)(d + off[5]));
    if (rc == PSLAM_OK)
        rc = pslam_planes_post_batch_dev(c, (const uint16_t*)(d + off[0]), nframes, (const pslam_plane*)(d + off[2]), (const int32_t*)(d + off[3]), (const int32_t*)(d + off[4]),
                                         (const int32_t*)(d + off[5]), dist_th, (int32_t*)(d + off[6]), (int32_t*)(d + off[7]), (float*)(d + off[8]), (int32_t*)(d + off[9]),
                                         (float*)(d + off[10]), cap_pts, (int32_t*)(d + off[11]));
    if (rc == PSLAM_OK && normals8) rc = pslam_surface_normals_batch_dev(c, (const uint16_t*)(d + off[0]), nframes, (float*)(d + off[12]), nullptr);
    if (rc != PSLAM_OK) { cudaStreamSynchronize(st); cudaFree(d); return rc; }
    std::vector<int32_t> status(nframes);
    cudaMemcpyAsync(n_kept, d + off[6], sz[6], cudaMemcpyDeviceToHost, st); cudaMemcpyAsync(src, d + off[7], sz[7], cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(coef, d + off[8], sz[8], cudaMemcpyDeviceToHost, st); cudaMemcpyAsync(pt_off, d + off[9], sz[9], cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(pts, d + off[10], sz[10], cudaMemcpyDeviceToHost, st); cudaMemcpyAsync(status.data(), d + off[11], sz[11], cudaMemcpyDeviceToHost, st);
    if (normals8) cudaMemcpyAsync(normals8, d + off[12], sz[12], cudaMemcpyDeviceToHost, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    cudaFree(d);
    if (e != cudaSuccess) return check_cuda(c, e, "compute planes");
    for (int f = 0; f < nframes; ++f) if (status[f] & (32 | 64)) return set_error(c, PSLAM_E_CAPACITY, "more voxels than the plane post-processing capacity");
    return PSLAM_OK;
}

}  // extern "C"
