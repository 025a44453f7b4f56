// The body of MapPlane::UpdateCoefficientsAndPoints (src/MapPlane.cc:298-365), shared by k_map_plane_update (mapplane_kernels.cu, a batch of jobs) and
// k_planar_map_plane_update (track_chain.cu, the planar chain's per-frame update): clouds transformed like pcl::transformPointCloud (double 4x4 on float
// points, rounded to float), merged into an order-free fixed-point voxel table (leaf 0.1 m), then one centroid per occupied voxel in ascending voxel index.
// One CTA of MP_THREADS threads runs one merge; the table lives in MP_SMEM bytes of dynamic shared memory.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "geom_device.cuh"

namespace pslam {

#define MP_SLOTS 4096
#define MP_THREADS 256
#define MP_EMPTY 0xffffffffu
#define MP_SMEM ((size_t)MP_SLOTS * (3 * 8 + 3 * 4))

struct MpTable {
    unsigned long long* sum;      // [3][MP_SLOTS]
    uint32_t *key, *cnt, *ord;    // [MP_SLOTS] each
    int* flag;                    // a point did not fit (table full or beyond the key range)
    int* n;                       // occupied voxels (after mp_sort)
};

__device__ __forceinline__ MpTable mp_table(unsigned char* smem, int* flag, int* n) {
    MpTable S;
    S.sum = reinterpret_cast<unsigned long long*>(smem);
    S.key = reinterpret_cast<uint32_t*>(S.sum + 3 * MP_SLOTS);
    S.cnt = S.key + MP_SLOTS;
    S.ord = S.cnt + MP_SLOTS;
    S.flag = flag; S.n = n;
    return S;
}

// empties the table; the caller synchronises before the first mp_add
__device__ __forceinline__ void mp_clear(const MpTable& S, int tid) {
    for (int i = tid; i < MP_SLOTS; i += MP_THREADS) { S.key[i] = MP_EMPTY; S.cnt[i] = 0; S.sum[i] = 0; S.sum[MP_SLOTS + i] = 0; S.sum[2 * MP_SLOTS + i] = 0; }
    if (tid == 0) { *S.flag = 0; *S.n = 0; }
}

// adds the points [p0, p1) of pts, transformed by the first three rows of the row-major 4x4 t (pts is not restrict: the planar chain merges a cloud into
// itself)
__device__ __forceinline__ void mp_add(const MpTable& S, int tid, const float* pts, int p0, int p1, const double* t) {
    const float inv = 10.0f;                                     // 1.0f / 0.1f rounds to 10.0f
    const double t0 = t[0], t1 = t[1], t2 = t[2], t3 = t[3], t4 = t[4], t5 = t[5], t6 = t[6], t7 = t[7], t8 = t[8], t9 = t[9], t10 = t[10], t11 = t[11];
    for (int i = p0 + tid; i < p1; i += MP_THREADS) {
        const double px = (double)pts[3 * (size_t)i], py = (double)pts[3 * (size_t)i + 1], pz = (double)pts[3 * (size_t)i + 2];
        const float x = (float)(((t0 * px + t1 * py) + t2 * pz) + t3), y = (float)(((t4 * px + t5 * py) + t6 * pz) + t7), z = (float)(((t8 * px + t9 * py) + t10 * pz) + t11);
        // ascending pcl::VoxelGrid index = lexicographic (iz, iy, ix): the packed absolute key orders the voxels identically (world frame: all three signed)
        const int i0 = (int)floorf(__fmul_rn(x, inv)) + 1024, i1 = (int)floorf(__fmul_rn(y, inv)) + 512, i2 = (int)floorf(__fmul_rn(z, inv)) + 1024;
        if ((unsigned)i0 > 2047u || (unsigned)i1 > 1023u || (unsigned)i2 > 2047u) { *S.flag = 1; continue; }        // beyond +-102 m (x, z) / +-51 m (y): capacity flag
        const uint32_t key = ((uint32_t)i2 << 21) | ((uint32_t)i1 << 11) | (uint32_t)i0;
        uint32_t slot = (key * 2654435761u) >> 20;            // 12 bits
        bool placed = false;
        for (int probe = 0; probe < MP_SLOTS; ++probe) {
            const uint32_t cur = atomicCAS(&S.key[slot], MP_EMPTY, key);
            if (cur == MP_EMPTY || cur == key) { placed = true; break; }
            slot = (slot + 1) & (MP_SLOTS - 1);
        }
        if (!placed) { *S.flag = 1; continue; }
        atomicAdd(&S.cnt[slot], 1u);
        atomicAdd(&S.sum[slot], (unsigned long long)llrint((double)x * 1048576.0));
        atomicAdd(&S.sum[MP_SLOTS + slot], (unsigned long long)llrint((double)y * 1048576.0));
        atomicAdd(&S.sum[2 * MP_SLOTS + slot], (unsigned long long)llrint((double)z * 1048576.0));
    }
}

// orders the occupied voxels by key (bitonic index sort, empty slots last) and counts them into *S.n; synchronises on entry and on exit
__device__ __forceinline__ void mp_sort(const MpTable& S, int tid) {
    __syncthreads();
    for (int i = tid; i < MP_SLOTS; i += MP_THREADS) S.ord[i] = (uint32_t)i;
    __syncthreads();
    for (int size = 2; size <= MP_SLOTS; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < MP_SLOTS / 2; i += MP_THREADS) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool up = ((lo & size) == 0);
                const uint32_t a = S.ord[lo], b = S.ord[hi];
                if ((S.key[a] > S.key[b]) == up) { S.ord[lo] = b; S.ord[hi] = a; }
            }
            __syncthreads();
        }
    int occupied = 0;
    for (int i = tid; i < MP_SLOTS; i += MP_THREADS) occupied += S.key[i] != MP_EMPTY;
    atomicAdd(S.n, occupied);
    __syncthreads();
}

// the first min(*S.n, cap) centroids, in key order, to out [cap][3]
__device__ __forceinline__ void mp_emit(const MpTable& S, int tid, int cap, float* out) {
    const int N = *S.n;
    for (int i = tid; i < min(N, cap); i += MP_THREADS) {
        const uint32_t sl = S.ord[i];
        const double n = (double)S.cnt[sl] * 1048576.0;
        float* o = out + (size_t)i * 3;
        o[0] = (float)((double)(long long)S.sum[sl] / n);
        o[1] = (float)((double)(long long)S.sum[MP_SLOTS + sl] / n);
        o[2] = (float)((double)(long long)S.sum[2 * MP_SLOTS + sl] / n);
    }
}

// T = Converter::toSE3Quat(Tcw).inverse() as the 3x4 rows pcl::transformPointCloud reads (MapPlane::UpdateCoefficientsAndPoints(const Frame&, int)):
// R and t of the float pose widened to double; R' = quat_to_matrix(qnorm_pos(quat_from_matrix(R))) (g2o::SE3Quat's constructor, then its Isometry3d);
// inverse [R'^T | -(R'^T t)] with (R'^T t)_r = (R'[0][r] t0 + R'[1][r] t1) + R'[2][r] t2 (DESIGN.md section 5).
__device__ __forceinline__ void mp_pose_inverse(const float* Tcw, double* T) {
    dM3 R;
    for (int r = 0; r < 3; ++r) for (int q = 0; q < 3; ++q) R.m[r][q] = (double)Tcw[4 * r + q];
    const double t0 = (double)Tcw[3], t1 = (double)Tcw[7], t2 = (double)Tcw[11];
    const dM3 Rq = quat_to_matrix(qnorm_pos(quat_from_matrix(R)));
    for (int r = 0; r < 3; ++r) {
        for (int q = 0; q < 3; ++q) T[4 * r + q] = Rq.m[q][r];
        T[4 * r + 3] = -((Rq.m[0][r] * t0 + Rq.m[1][r] * t1) + Rq.m[2][r] * t2);
    }
}

}  // namespace pslam
