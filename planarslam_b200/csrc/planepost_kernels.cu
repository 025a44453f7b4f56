// Plane post-processing of Frame::ComputePlanes (src/Frame.cc:647-753) and Frame::MaxPointDistanceFromPlane (:755-813) on sm_90a: what turns the PEAC result into
// mvPlanePoints / mvPlaneCoefficients, and the surface normals (vSurfaceNormal) that TrackManhattanFrame consumes.  The three PCL algorithms behind those calls
// are not in /root/reference; oracle/planepost.cc restates them (parity unpinned upstream, see its header) and the kernels here are held to that restatement.
//
//   k_planes_worklist the (frame, plane) records of the planes PEAC found, plane-major
//   k_planes_post    persistent CTAs (four per SM) that take one record at a time: voxel accumulation (leaf 0.1 m) into a shared-memory hash table with
//                    ORDER-FREE fixed-point sums (32-bit atomics, see pp_base), the all-centroids-within-threshold test against the PEAC plane, occupied voxels
//                    sorted by index, then on one warp PCL's RANSAC (mt19937(12345) sample shuffling, <= 50 iterations) and the float least-squares refit
//                    through the closed-form eigen33, sign kept like the reference
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
#define PP_CTAS_PER_SM 4         // 48 KB of shared memory per CTA
#define PP_SMEM ((size_t)PP_SLOTS * 6 * 4)
#define PP_EMPTY 0xffffffffu
#define PP_MAX_PLANES 128        // >= pslam_peac_max_planes()
#define PP_MAX_PIXELS (1 << 25)  // members of one voxel: keeps the carry fields of the voxel sums below 2^10 (pp_base)

struct PlanePostBuffers {
    int max_batch = 0, maxp = 0, w3 = 0, h3 = 0, workers = 0;
    // per (frame, plane) working records
    DevArray<float> d_coef; DevArray<int32_t> d_valid, d_npts; DevArray<float> d_pts; DevArray<int32_t> d_stats;     // [B][maxp][...]
    DevArray<int32_t> d_work, d_ctl;                                                                                   // [B * maxp] records, [2] count / fetch counter
    // surface normals scratch
    DevArray<float> d_cloud, d_dist; DevArray<double> d_ix, d_iy;
    DevArray<float> d_nrm;
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

// Exact, order-free voxel sums.  A member's coordinate enters as v = llrint(coordinate * 2^20); the sum of a voxel is kept relative to a base B(idx) of its
// voxel index idx = floor(coordinate * 10) along that axis: every v - B lies in [0, 2^17) (v is within 26 units of [idx, idx + 1) * 104857.6 after the float
// rounding of coordinate * 10, and idx is in [-512, 4094]), so a warp's group of at most 32 members sums to below 2^22 and enters the low 32-bit word of the
// voxel with one atomicAdd.  Wraps of the low word are counted in a 10-bit field per axis of a shared carry word, which holds (sum >> 32) exactly while a voxel
// has fewer than 2^25 members (PP_MAX_PIXELS).  The sums are integers, so the centroids do not depend on the order of the atomics.
__device__ __forceinline__ int pp_base(int idx) { return idx * 104857 - 1024; }

__device__ __forceinline__ float pp_centroid(uint32_t lo, uint32_t carries, uint32_t n, int idx, double n_fixed) {
    const long long sum = (long long)(((unsigned long long)carries << 32) | lo) + (long long)n * pp_base(idx);
    return (float)((double)sum / n_fixed);
}

// the (frame, plane) records of the planes PEAC found, plane-major: every frame's plane 0 comes first, and PEAC orders a frame's planes by size, so the largest
// work is taken first and the launch ends on small planes.  ctl[0] = number of records, ctl[1] = the fetch counter of k_planes_post.  The order of the frames
// within one plane index is that of the atomics; no output depends on it.
__global__ void __launch_bounds__(1024) k_planes_worklist(int nframes, int maxp, const int32_t* __restrict__ n_planes, int32_t* __restrict__ work,
                                                          int32_t* __restrict__ ctl) {
    __shared__ int s_cnt[PP_MAX_PLANES], s_cur[PP_MAX_PLANES];
    const int tid = threadIdx.x;
    for (int p = tid; p < maxp; p += blockDim.x) s_cnt[p] = 0;
    __syncthreads();
    for (int f = tid; f < nframes; f += blockDim.x) {
        const int n = min(n_planes[f], maxp);
        for (int p = 0; p < n; ++p) atomicAdd(&s_cnt[p], 1);
    }
    __syncthreads();
    if (tid == 0) {
        int off = 0;
        for (int p = 0; p < maxp; ++p) { s_cur[p] = off; off += s_cnt[p]; }
        ctl[0] = off; ctl[1] = 0;
    }
    __syncthreads();
    for (int f = tid; f < nframes; f += blockDim.x) {
        const int n = min(n_planes[f], maxp);
        for (int p = 0; p < n; ++p) work[atomicAdd(&s_cur[p], 1)] = f * maxp + p;
    }
}

// one group of members that share a voxel: probe for its slot, then add the count and the three relative sums (leader lane only)
__device__ __forceinline__ void pp_voxel_add(uint32_t* s_key, uint32_t* s_cnt, uint32_t* s_carry, uint32_t* s_lo, uint32_t key, uint32_t n, uint32_t sx,
                                             uint32_t sy, uint32_t sz, int* flag) {
    uint32_t slot = (key * 2654435761u) >> 21;                    // 11 bits
    bool placed = false;
    for (int probe = 0; probe < PP_SLOTS; ++probe) {
        const uint32_t cur = atomicCAS(&s_key[slot], PP_EMPTY, key);
        if (cur == PP_EMPTY || cur == key) { placed = true; break; }
        slot = (slot + 1) & (PP_SLOTS - 1);
    }
    if (!placed) { atomicOr(flag, 1); return; }
    atomicAdd(&s_cnt[slot], n);
    const uint32_t d[3] = {sx, sy, sz};
    uint32_t carry = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const uint32_t old = atomicAdd(&s_lo[a * PP_SLOTS + slot], d[a]);
        if (old + d[a] < old) carry += 1u << (10 * a);
    }
    if (carry) atomicAdd(&s_carry[slot], carry);
}

__global__ void __launch_bounds__(PP_THREADS, PP_CTAS_PER_SM) k_planes_post(const uint16_t* __restrict__ depth_all, int w, int h, PPCam K,
                                                                            const pslam_plane* __restrict__ planes_all, const int32_t* __restrict__ work,
                                                                            int32_t* __restrict__ ctl, const int32_t* __restrict__ midx_all,
                                                                            const int32_t* __restrict__ moff_all, int maxp, double dist_th, float* __restrict__ coef_out,
                                                                            int32_t* __restrict__ valid_out, int32_t* __restrict__ npts_out, float* __restrict__ pts_out,
                                                                            int32_t* __restrict__ stats_out, int32_t* __restrict__ status) {
    constexpr int PER_THREAD = PP_SLOTS / PP_THREADS;
    constexpr uint32_t FULL = 0xffffffffu;
    extern __shared__ __align__(16) uint32_t pp_smem[];
    // 48 KB, reused from phase to phase: voxel table -> centroids by slot + sort order -> sorted centroids + RANSAC state
    uint32_t* s_key = pp_smem;                     // [PP_SLOTS] voxel keys; then sorted x
    uint32_t* s_cnt = s_key + PP_SLOTS;            // [PP_SLOTS] member counts; then the sort order; then the mt19937 state
    uint32_t* s_carry = s_cnt + PP_SLOTS;          // [PP_SLOTS] carry fields of the sums; then sorted y
    uint32_t* s_lo = s_carry + PP_SLOTS;           // [3][PP_SLOTS] low words of the sums; then the centroids by slot; then sorted z, shuffled indices, inlier list
    float* s_px = reinterpret_cast<float*>(s_lo);
    __shared__ int s_i[4];                         // occupied voxels, capacity flag, record
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const float inv = 10.0f;                       // 1.0f / 0.1f rounds to 10.0f
    for (;;) {
        __syncthreads();                           // the previous record's shared memory is no longer read
        if (tid == 0) { s_i[0] = 0; s_i[1] = 0; const int item = atomicAdd(ctl + 1, 1); s_i[2] = item < ctl[0] ? item : -1; }
        {
            uint4* t = reinterpret_cast<uint4*>(pp_smem);
            for (int i = tid; i < PP_SLOTS / 4; i += PP_THREADS) t[i] = make_uint4(PP_EMPTY, PP_EMPTY, PP_EMPTY, PP_EMPTY);
            for (int i = PP_SLOTS / 4 + tid; i < 6 * PP_SLOTS / 4; i += PP_THREADS) t[i] = make_uint4(0, 0, 0, 0);
        }
        __syncthreads();
        const int item = s_i[2];
        if (item < 0) return;
        const int rec = work[item], frame = rec / maxp, pl = rec - frame * maxp;
        const uint16_t* depth = depth_all + (size_t)frame * w * h;
        const int32_t* moff = moff_all + (size_t)frame * (maxp + 1);
        const int32_t* midx = midx_all + (size_t)frame * w * h + moff[pl];
        const int nm = moff[pl + 1] - moff[pl];
        // ---- voxel accumulation (leaf 0.1 m) ----
        // pcl::VoxelGrid numbers a voxel i0 + i1 * div0 + i2 * div0 * div1 with i* = floor(coordinate * 10) - floor(minimum * 10): ascending index = lexicographic
        // (i2, i1, i0), which the packed absolute key (iz, iy, ix) below orders identically - so no bounding-box pass is needed.  A warp reads 4 x 32 consecutive
        // members per trip (their index loads, then their depth loads, issued together); lanes of one trip that share a voxel are grouped by __match_any_sync and
        // their sums reduced, so the table sees one update per distinct voxel and trip.
        for (int base = wid * 128; base < nm; base += PP_THREADS * 4) {
            int pix[4]; uint16_t dv[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { const int i = base + 32 * u + lane; pix[u] = i < nm ? midx[i] : -1; }
#pragma unroll
            for (int u = 0; u < 4; ++u) dv[u] = pix[u] >= 0 ? depth[pix[u]] : (uint16_t)0;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (base + 32 * u >= nm) break;
                uint32_t key = PP_EMPTY, dx = 0, dy = 0, dz = 0;
                if (pix[u] >= 0) {
                    float x, y, z;
                    pp_vertex_d(dv[u], w, K, pix[u], x, y, z);
                    const int j0 = (int)floorf(__fmul_rn(x, inv)), j1 = (int)floorf(__fmul_rn(y, inv)), j2 = (int)floorf(__fmul_rn(z, inv));
                    const int i0 = j0 + 512, i1 = j1 + 512, i2 = j2;
                    if ((unsigned)i0 > 1023u || (unsigned)i1 > 1023u || (unsigned)i2 >= 4095u) atomicOr(&s_i[1], 1);      // > 51 m sideways / 409 m deep: capacity flag
                    else {
                        key = ((uint32_t)i2 << 20) | ((uint32_t)i1 << 10) | (uint32_t)i0;
                        // llrint((double)x * 2^20): the scaling is exact in float as well, and |v| < 2^29 inside the key range
                        dx = (uint32_t)(__float2int_rn(__fmul_rn(x, 1048576.0f)) - pp_base(j0));
                        dy = (uint32_t)(__float2int_rn(__fmul_rn(y, 1048576.0f)) - pp_base(j1));
                        dz = (uint32_t)(__float2int_rn(__fmul_rn(z, 1048576.0f)) - pp_base(j2));
                    }
                }
                const uint32_t grp = __match_any_sync(FULL, key);
                uint32_t leaders = __ballot_sync(FULL, key != PP_EMPTY && (grp & ((1u << lane) - 1u)) == 0);
                while (leaders) {
                    const int ld = __ffs(leaders) - 1;
                    leaders &= leaders - 1;
                    const uint32_t g = __shfl_sync(FULL, grp, ld);
                    const bool in = (g >> lane) & 1u;
                    const uint32_t sx = __reduce_add_sync(FULL, in ? dx : 0u), sy = __reduce_add_sync(FULL, in ? dy : 0u), sz = __reduce_add_sync(FULL, in ? dz : 0u);
                    if (lane == ld) pp_voxel_add(s_key, s_cnt, s_carry, s_lo, key, __popc(g), sx, sy, sz, &s_i[1]);
                }
            }
        }
        __syncthreads();
        // ---- centroids (each thread overwrites the sums of its own slots) and MaxPointDistanceFromPlane: every centroid within the threshold of the PEAC plane ----
        const pslam_plane P = planes_all[rec];
        const float coef[4] = {(float)P.normal[0], (float)P.normal[1], (float)P.normal[2],
                               (float)-(P.normal[0] * P.center[0] + P.normal[1] * P.center[1] + P.normal[2] * P.center[2])};
        int bad = 0;
        for (int s = tid; s < PP_SLOTS; s += PP_THREADS) {
            const uint32_t key = s_key[s];
            if (key == PP_EMPTY) continue;
            const uint32_t n = s_cnt[s], carries = s_carry[s];
            const double n_fixed = (double)n * 1048576.0;
            const float x = pp_centroid(s_lo[s], carries & 1023u, n, (int)(key & 1023u) - 512, n_fixed);
            const float y = pp_centroid(s_lo[PP_SLOTS + s], (carries >> 10) & 1023u, n, (int)((key >> 10) & 1023u) - 512, n_fixed);
            const float z = pp_centroid(s_lo[2 * PP_SLOTS + s], carries >> 20, n, (int)(key >> 20), n_fixed);
            s_px[s] = x; s_px[PP_SLOTS + s] = y; s_px[2 * PP_SLOTS + s] = z;
            bad |= (double)fabsf(pp_dot4(coef, x, y, z)) > dist_th;
        }
        bad = __syncthreads_or(bad);
        uint32_t* s_ord = s_cnt;
        int N = 0;
        if (!bad) {                                // the occupied slots, compacted
            for (int s = tid; s < PP_SLOTS; s += PP_THREADS) {
                const bool o = s_key[s] != PP_EMPTY;
                const uint32_t m = __ballot_sync(FULL, o);
                int at = 0;
                if (lane == 0 && m) at = atomicAdd(&s_i[0], __popc(m));
                at = __shfl_sync(FULL, at, 0);
                if (o) s_ord[at + __popc(m & ((1u << lane) - 1u))] = (uint32_t)s;
            }
            __syncthreads();
            N = s_i[0];
        }
        if (bad || N < 3) {
            if (tid == 0) { valid_out[rec] = 0; npts_out[rec] = 0; stats_out[2 * rec] = 0; stats_out[2 * rec + 1] = 0; if (s_i[1]) atomicOr(status + frame, 32); }
            continue;
        }
        // ---- order the occupied voxels by index: bitonic sort of their slots by key over the next power of two (keys are unique, pads sort last) ----
        int n2 = 4;
        while (n2 < N) n2 <<= 1;
        for (int i = N + tid; i < n2; i += PP_THREADS) s_ord[i] = PP_EMPTY;
        __syncthreads();
        for (int size = 2; size <= n2; size <<= 1)
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int i = tid; i < n2 / 2; i += PP_THREADS) {
                    const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                    const bool up = ((lo & size) == 0);
                    const uint32_t a = s_ord[lo], b = s_ord[hi];
                    const uint32_t ka = a == PP_EMPTY ? PP_EMPTY : s_key[a], kb = b == PP_EMPTY ? PP_EMPTY : s_key[b];
                    if ((ka > kb) == up) { s_ord[lo] = b; s_ord[hi] = a; }
                }
                __syncthreads();
            }
        // sorted centroids: x over the keys, y over the carries, z (through registers) over the slot-order x
        float* px = reinterpret_cast<float*>(s_key);
        float* py = reinterpret_cast<float*>(s_carry);
        float* pz = s_px;
        float zk[PER_THREAD];
#pragma unroll
        for (int k = 0; k < PER_THREAD; ++k) {
            const int i = tid + k * PP_THREADS;
            zk[k] = 0.f;
            if (i < N) { const uint32_t o = s_ord[i]; px[i] = s_px[o]; py[i] = s_px[PP_SLOTS + o]; zk[k] = s_px[2 * PP_SLOTS + o]; }
        }
        __syncthreads();
        uint32_t* shuffled = s_lo + PP_SLOTS;
        uint32_t* s_inl = s_lo + 2 * PP_SLOTS;
#pragma unroll
        for (int k = 0; k < PER_THREAD; ++k) {
            const int i = tid + k * PP_THREADS;
            if (i < N) { pz[i] = zk[k]; shuffled[i] = (uint32_t)i; }
        }
        for (int i = tid; i < 624; i += PP_THREADS) s_cnt[i] = g_pp_mt[i];      // mt19937(12345) after its first twist
        __syncthreads();
        if (wid != 0) continue;
        // ---- RANSAC (pcl::RandomSampleConsensus on SampleConsensusModelPlane) on warp 0: lane 0 draws the samples in the reference's order, the lanes count ----
        PPRng rng; rng.mt = s_cnt; rng.idx = 0;
        int best_count = -INT_MAX, iterations = 0;
        double k = 1.0;
        const double log_probability = log(1.0 - 0.99), one_over = 1.0 / (double)N;
        float best[4] = {0, 0, 0, 0};
        bool have = false;
        unsigned skipped = 0;
        while (iterations < k && skipped < 500u) {
            int state = 0;                                            // 0: no sample, 1: model, 2: degenerate (skipped)
            float c[4] = {0, 0, 0, 0};
            if (lane == 0) {
                int s0 = 0, s1 = 0, s2 = 0;
                bool good = false;
                for (unsigned it = 0; it < 1000 && !good; ++it) {
                    for (int i = 0; i < 3; ++i) { const int j = i + (rng.rnd() % (N - i)); const uint32_t t = shuffled[i]; shuffled[i] = shuffled[j]; shuffled[j] = t; }
                    s0 = shuffled[0]; s1 = shuffled[1]; s2 = shuffled[2];
                    const float d0 = __fdiv_rn(__fsub_rn(px[s1], px[s0]), __fsub_rn(px[s2], px[s0]));
                    const float d1 = __fdiv_rn(__fsub_rn(py[s1], py[s0]), __fsub_rn(py[s2], py[s0]));
                    const float d2 = __fdiv_rn(__fsub_rn(pz[s1], pz[s0]), __fsub_rn(pz[s2], pz[s0]));
                    good = (d0 != d1) || (d2 != d1);
                }
                state = good ? 1 : 0;
                if (good) {
                    const float a[3] = {__fsub_rn(px[s1], px[s0]), __fsub_rn(py[s1], py[s0]), __fsub_rn(pz[s1], pz[s0])};
                    const float b[3] = {__fsub_rn(px[s2], px[s0]), __fsub_rn(py[s2], py[s0]), __fsub_rn(pz[s2], pz[s0])};
                    const float e0 = __fdiv_rn(a[0], b[0]), e1 = __fdiv_rn(a[1], b[1]), e2 = __fdiv_rn(a[2], b[2]);
                    if (e0 == e1 && e2 == e1) state = 2;
                    else {
                        c[0] = __fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1]));
                        c[1] = __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2]));
                        c[2] = __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]));
                        const float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(c[0], c[0]), __fmul_rn(c[1], c[1])), __fmul_rn(c[2], c[2])));
                        for (int q = 0; q < 3; ++q) c[q] = __fdiv_rn(c[q], nrm);
                        c[3] = -1 * __fadd_rn(__fadd_rn(__fmul_rn(c[0], px[s0]), __fmul_rn(c[1], py[s0])), __fmul_rn(c[2], pz[s0]));
                    }
                }
            }
            state = __shfl_sync(FULL, state, 0);
            if (state == 0) break;
            if (state == 2) { ++skipped; continue; }
#pragma unroll
            for (int q = 0; q < 4; ++q) c[q] = __shfl_sync(FULL, c[q], 0);
            unsigned cnt = 0;
            for (int i = lane; i < N; i += 32) cnt += (double)fabsf(pp_dot4(c, px[i], py[i], pz[i])) < dist_th;
            const int total = (int)__reduce_add_sync(FULL, cnt);
            if (total > best_count) {
                best_count = total; best[0] = c[0]; best[1] = c[1]; best[2] = c[2]; best[3] = c[3]; have = true;
                if (lane == 0) {
                    const double wv = (double)best_count * one_over;
                    double p_no = 1.0 - pow(wv, 3.0);
                    p_no = fmax(DBL_EPSILON, p_no);
                    p_no = fmin(1.0 - DBL_EPSILON, p_no);
                    k = log_probability / log(p_no);
                }
                k = __shfl_sync(FULL, k, 0);
            }
            ++iterations;
            if (iterations > 50) break;
        }
        if (!have) {
            if (lane == 0) { valid_out[rec] = 0; npts_out[rec] = 0; stats_out[2 * rec] = 0; stats_out[2 * rec + 1] = iterations; }
            continue;
        }
        // ---- optimizeModelCoefficients: the inliers of the best model listed in index order, then nine lanes walk one float moment each in that order (the
        //      sequential loop's chains of rounded additions, term by term; the first-order terms are x * 1.0f = x) ----
        int ninl = 0;
        for (int b = 0; b < N; b += 32) {
            const int i = b + lane;
            const bool in = i < N && (double)fabsf(pp_dot4(best, px[i], py[i], pz[i])) < dist_th;
            const uint32_t m = __ballot_sync(FULL, in);
            if (in) s_inl[ninl + __popc(m & ((1u << lane) - 1u))] = (uint32_t)i;
            ninl += __popc(m);
        }
        __syncwarp();
        float acc = 0.f;
        if (lane < 9) {
            const int ua = lane < 3 ? 0 : lane < 5 ? 1 : lane < 6 ? 2 : -1;
            const int vb = lane < 6 ? (lane < 3 ? lane : lane < 5 ? lane - 2 : 2) : lane - 6;
            const float* pu = ua == 1 ? py : ua == 2 ? pz : px;
            const float* pv = vb == 0 ? px : vb == 1 ? py : pz;
#pragma unroll 4
            for (int t = 0; t < ninl; ++t) {
                const uint32_t i = s_inl[t];
                const float u = ua < 0 ? 1.0f : pu[i];
                acc = __fadd_rn(acc, __fmul_rn(u, pv[i]));
            }
        }
        float m9[9];
#pragma unroll
        for (int q = 0; q < 9; ++q) m9[q] = __shfl_sync(FULL, acc, q);
        float opt[4] = {best[0], best[1], best[2], best[3]};
        if (ninl > 3) {
            for (int q = 0; q < 9; ++q) m9[q] = __fdiv_rn(m9[q], (float)ninl);
            float cov[3][3];
            cov[0][0] = __fsub_rn(m9[0], __fmul_rn(m9[6], m9[6])); cov[0][1] = __fsub_rn(m9[1], __fmul_rn(m9[6], m9[7])); cov[0][2] = __fsub_rn(m9[2], __fmul_rn(m9[6], m9[8]));
            cov[1][1] = __fsub_rn(m9[3], __fmul_rn(m9[7], m9[7])); cov[1][2] = __fsub_rn(m9[4], __fmul_rn(m9[7], m9[8])); cov[2][2] = __fsub_rn(m9[5], __fmul_rn(m9[8], m9[8]));
            cov[1][0] = cov[0][1]; cov[2][0] = cov[0][2]; cov[2][1] = cov[1][2];
            float vec[3];
            pp_eigen33(cov, vec);
            opt[0] = vec[0]; opt[1] = vec[1]; opt[2] = vec[2];
            opt[3] = -1 * __fadd_rn(__fadd_rn(__fmul_rn(opt[0], m9[6]), __fmul_rn(opt[1], m9[7])), __fmul_rn(opt[2], m9[8]));
        }
        // ---- selectWithinDistance with the refined model ----
        unsigned cnt = 0;
        for (int i = lane; i < N; i += 32) cnt += (double)fabsf(pp_dot4(opt, px[i], py[i], pz[i])) < dist_th;
        const int final_inl = (int)__reduce_add_sync(FULL, cnt);
        if (final_inl == 0 || ninl == 0) {
            if (lane == 0) { valid_out[rec] = 0; npts_out[rec] = 0; }
            continue;
        }
        const float old_d = coef[3], new_d = opt[3];
        if ((new_d < 0 && old_d > 0) || (new_d > 0 && old_d < 0)) for (int q = 0; q < 4; ++q) opt[q] = -opt[q];
        if (lane == 0) {
            for (int q = 0; q < 4; ++q) coef_out[(size_t)rec * 4 + q] = opt[q];
            valid_out[rec] = 1; npts_out[rec] = N; stats_out[2 * rec] = final_inl; stats_out[2 * rec + 1] = iterations;
            if (s_i[1]) atomicOr(status + frame, 32);
        }
        float* po = pts_out + (size_t)rec * PP_SLOTS * 3;
        for (int i = lane; i < 3 * N; i += 32) { const int v = i / 3, q = i - 3 * v; po[i] = (q == 0 ? px : q == 1 ? py : pz)[v]; }
    }
}

// the surviving planes of a frame, in PEAC order: src [maxp], coef [maxp][4], pt_off [maxp + 1], pts packed
__global__ void __launch_bounds__(256) k_planes_compact(int maxp, int cap_pts, const int32_t* __restrict__ n_planes, const float* __restrict__ coef_w,
                                                        const int32_t* __restrict__ valid_w, const int32_t* __restrict__ npts_w, const float* __restrict__ pts_w,
                                                        int32_t* __restrict__ n_kept, int32_t* __restrict__ src, float* __restrict__ coef, int32_t* __restrict__ pt_off,
                                                        float* __restrict__ pts, int32_t* __restrict__ status) {
    const int frame = blockIdx.x, tid = threadIdx.x;
    __shared__ int s_slot[PP_MAX_PLANES], s_off[PP_MAX_PLANES + 1], s_n;
    if (tid == 0) {
        int n = 0, off = 0;
        const int np = min(n_planes[frame], maxp);                // records past n_planes are not written by k_planes_post
        for (int p = 0; p < np; ++p) {
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
    if ((size_t)c->cfg.width * c->cfg.height > (size_t)PP_MAX_PIXELS) { planepost_free(c); return set_error(c, PSLAM_E_INVALID, "image above the plane post-processing limit"); }
    B.w3 = (c->cfg.width + 2) / 3; B.h3 = (c->cfg.height + 2) / 3;
    {   // the persistent grid of k_planes_post: as many CTAs as are resident at once
        int sms = 0, per_sm = 0;
        int rc_ = check_cuda(c, cudaFuncSetAttribute(k_planes_post, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PP_SMEM), "cudaFuncSetAttribute(k_planes_post)");
        if (rc_ == PSLAM_OK) rc_ = check_cuda(c, cudaFuncSetAttribute(k_planes_post, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared),
                                              "cudaFuncSetAttribute(k_planes_post)");
        if (rc_ == PSLAM_OK) rc_ = check_cuda(c, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->cfg.device), "cudaDeviceGetAttribute");
        if (rc_ == PSLAM_OK) rc_ = check_cuda(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_planes_post, PP_THREADS, PP_SMEM), "cudaOccupancy");
        if (rc_ == PSLAM_OK && per_sm < 1) rc_ = set_error(c, PSLAM_E_INVALID, "planes post: kernel does not fit on an SM");
        if (rc_ != PSLAM_OK) { planepost_free(c); return rc_; }
        B.workers = sms * per_sm;
    }
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
    int rc;
    if ((rc = B.d_coef.reserve(c, nb * B.maxp * 4)) || (rc = B.d_valid.reserve(c, nb * B.maxp)) || (rc = B.d_npts.reserve(c, nb * B.maxp)) ||
        (rc = B.d_stats.reserve(c, nb * B.maxp * 2)) || (rc = B.d_pts.reserve(c, nb * B.maxp * (size_t)PP_SLOTS * 3)) ||
        (rc = B.d_work.reserve(c, nb * B.maxp)) || (rc = B.d_ctl.reserve(c, 2)) ||
        (rc = B.d_cloud.reserve(c, nb * np * 3)) || (rc = B.d_dist.reserve(c, nb * (np + 2))) ||
        (rc = B.d_ix.reserve(c, nb * ni * 3)) || (rc = B.d_iy.reserve(c, nb * ni * 3)) || (rc = B.d_nrm.reserve(c, nb * np * 3))) {
        planepost_free(c);
        return rc;
    }
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
    PSLAM_CUDA(c, cudaMemsetAsync(d_status, 0, (size_t)nframes * 4, st));
    PSLAM_LAUNCH(c, "planes_worklist", k_planes_worklist<<<1, 1024, 0, st>>>(nframes, B.maxp, d_nplanes, B.d_work, B.d_ctl));
    PSLAM_LAUNCH(c, "planes_post", k_planes_post<<<B.workers, PP_THREADS, PP_SMEM, st>>>(d_depth, c->cfg.width, c->cfg.height, K, d_planes, B.d_work, B.d_ctl,
                 d_member_idx, d_member_off, B.maxp, (double)dist_th, B.d_coef, B.d_valid, B.d_npts, B.d_pts, B.d_stats, d_status));
    PSLAM_LAUNCH(c, "planes_compact", k_planes_compact<<<nframes, 256, 0, st>>>(B.maxp, cap_pts, d_nplanes, B.d_coef, B.d_valid, B.d_npts, B.d_pts, d_n_kept, d_src,
                 d_coef, d_pt_off, d_pts, d_status));
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
    Slab s;
    const auto d_depth = s.add<uint16_t>(nf * npx);
    const auto labels = s.add<int32_t>(nf * npx);
    const auto planes = s.add<pslam_plane>(nf * maxp);
    const auto nplanes = s.add<int32_t>(nf), members = s.add<int32_t>(nf * npx), moff = s.add<int32_t>(nf * (maxp + 1));
    const auto d_kept = s.add<int32_t>(nf), d_src = s.add<int32_t>(nf * maxp);
    const auto d_coef = s.add<float>(nf * maxp * 4);
    const auto d_off = s.add<int32_t>(nf * (maxp + 1));
    const auto d_pts = s.add<float>(nf * cap_pts * 3);
    const auto d_status = s.add<int32_t>(nf);
    const auto d_normals8 = s.add<float>(nf * n_sn * 8);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    s.up(d_depth, depth, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    rc = pslam_peac_run_batch_dev(c, s[d_depth], nframes, s[labels], s[planes], s[nplanes], s[members], s[moff]);
    if (rc == PSLAM_OK)
        rc = pslam_planes_post_batch_dev(c, s[d_depth], nframes, s[planes], s[nplanes], s[members], s[moff], dist_th, s[d_kept], s[d_src], s[d_coef], s[d_off], s[d_pts],
                                         cap_pts, s[d_status]);
    if (rc == PSLAM_OK && normals8) rc = pslam_surface_normals_batch_dev(c, s[d_depth], nframes, s[d_normals8], nullptr);
    if (rc != PSLAM_OK) { cudaStreamSynchronize(st); return rc; }
    std::vector<int32_t> status(nframes);
    s.down(n_kept, d_kept, st); s.down(src, d_src, st); s.down(coef, d_coef, st); s.down(pt_off, d_off, st); s.down(pts, d_pts, st); s.down(status.data(), d_status, st);
    if (normals8) s.down(normals8, d_normals8, st);
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    for (int f = 0; f < nframes; ++f) if (status[f] & (32 | 64)) return set_error(c, PSLAM_E_CAPACITY, "more voxels than the plane post-processing capacity");
    return PSLAM_OK;
}

}  // extern "C"
