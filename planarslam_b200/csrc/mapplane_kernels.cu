// MapPlane::UpdateCoefficientsAndPoints() and (const Frame&, int id) on sm_90a (src/MapPlane.cc:298-365): the plane clouds of a map plane's observations
// (KeyFrame::mvPlanePoints[id], camera frame) are brought into the world frame by pcl::transformPointCloud (double 4x4 on float points, rounded to float),
// concatenated - the second overload appends the map plane's current cloud - and reduced by pcl::VoxelGrid (leaf 0.1 m): one centroid per occupied voxel in
// ascending voxel index becomes MapPlane::mvPlanePoints.  The pcl::SACSegmentation call that follows in the reference writes into locals nobody reads.
// One CTA per map plane ("job"): the same order-free fixed-point voxel table as k_planes_post (planepost_kernels.cu), 4096 slots here because a map plane
// accumulates the extent of many views.  Oracle: oracle/planepost.cc map_plane_update (PCL absent: parity unpinned).
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "pslam_internal.h"

namespace pslam {

#define MP_SLOTS 4096
#define MP_THREADS 256
#define MP_EMPTY 0xffffffffu

__global__ void __launch_bounds__(MP_THREADS) k_map_plane_update(const int32_t* __restrict__ job_off, const int32_t* __restrict__ cloud_off, const float* __restrict__ pts,
                                                                 const double* __restrict__ T, int cap, float* __restrict__ out_pts, int32_t* __restrict__ n_out,
                                                                 int32_t* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char mp_smem[];
    unsigned long long* s_sum = reinterpret_cast<unsigned long long*>(mp_smem);       // [3][MP_SLOTS]
    uint32_t* s_key = reinterpret_cast<uint32_t*>(s_sum + 3 * MP_SLOTS);               // [MP_SLOTS]
    uint32_t* s_cnt = s_key + MP_SLOTS;                                                // [MP_SLOTS]
    uint32_t* s_ord = s_cnt + MP_SLOTS;                                                // [MP_SLOTS]
    __shared__ int s_flag, s_n;
    const int job = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < MP_SLOTS; i += MP_THREADS) { s_key[i] = MP_EMPTY; s_cnt[i] = 0; s_sum[i] = 0; s_sum[MP_SLOTS + i] = 0; s_sum[2 * MP_SLOTS + i] = 0; }
    if (tid == 0) { s_flag = 0; s_n = 0; }
    __syncthreads();
    const float inv = 10.0f;                                     // 1.0f / 0.1f rounds to 10.0f
    for (int c = job_off[job]; c < job_off[job + 1]; ++c) {
        const double* t = T + 16 * (size_t)c;
        const double t0 = t[0], t1 = t[1], t2 = t[2], t3 = t[3], t4 = t[4], t5 = t[5], t6 = t[6], t7 = t[7], t8 = t[8], t9 = t[9], t10 = t[10], t11 = t[11];
        for (int i = cloud_off[c] + tid; i < cloud_off[c + 1]; i += MP_THREADS) {
            const double px = (double)pts[3 * (size_t)i], py = (double)pts[3 * (size_t)i + 1], pz = (double)pts[3 * (size_t)i + 2];
            const float x = (float)(((t0 * px + t1 * py) + t2 * pz) + t3), y = (float)(((t4 * px + t5 * py) + t6 * pz) + t7), z = (float)(((t8 * px + t9 * py) + t10 * pz) + t11);
            // ascending pcl::VoxelGrid index = lexicographic (iz, iy, ix): the packed absolute key orders the voxels identically (world frame: all three signed)
            const int i0 = (int)floorf(__fmul_rn(x, inv)) + 1024, i1 = (int)floorf(__fmul_rn(y, inv)) + 512, i2 = (int)floorf(__fmul_rn(z, inv)) + 1024;
            if ((unsigned)i0 > 2047u || (unsigned)i1 > 1023u || (unsigned)i2 > 2047u) { s_flag = 1; continue; }        // beyond +-102 m (x, z) / +-51 m (y): capacity flag
            const uint32_t key = ((uint32_t)i2 << 21) | ((uint32_t)i1 << 11) | (uint32_t)i0;
            uint32_t slot = (key * 2654435761u) >> 20;            // 12 bits
            bool placed = false;
            for (int probe = 0; probe < MP_SLOTS; ++probe) {
                const uint32_t cur = atomicCAS(&s_key[slot], MP_EMPTY, key);
                if (cur == MP_EMPTY || cur == key) { placed = true; break; }
                slot = (slot + 1) & (MP_SLOTS - 1);
            }
            if (!placed) { s_flag = 1; continue; }
            atomicAdd(&s_cnt[slot], 1u);
            atomicAdd(&s_sum[slot], (unsigned long long)llrint((double)x * 1048576.0));
            atomicAdd(&s_sum[MP_SLOTS + slot], (unsigned long long)llrint((double)y * 1048576.0));
            atomicAdd(&s_sum[2 * MP_SLOTS + slot], (unsigned long long)llrint((double)z * 1048576.0));
        }
    }
    __syncthreads();
    // order the occupied voxels by key: bitonic index sort, empty slots (key 0xffffffff) last
    for (int i = tid; i < MP_SLOTS; i += MP_THREADS) s_ord[i] = (uint32_t)i;
    __syncthreads();
    for (int size = 2; size <= MP_SLOTS; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < MP_SLOTS / 2; i += MP_THREADS) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool up = ((lo & size) == 0);
                const uint32_t a = s_ord[lo], b = s_ord[hi];
                if ((s_key[a] > s_key[b]) == up) { s_ord[lo] = b; s_ord[hi] = a; }
            }
            __syncthreads();
        }
    int occupied = 0;
    for (int i = tid; i < MP_SLOTS; i += MP_THREADS) occupied += s_key[i] != MP_EMPTY;
    atomicAdd(&s_n, occupied);
    __syncthreads();
    const int N = s_n;
    for (int i = tid; i < min(N, cap); i += MP_THREADS) {
        const uint32_t sl = s_ord[i];
        const double n = (double)s_cnt[sl] * 1048576.0;
        float* o = out_pts + ((size_t)job * cap + i) * 3;
        o[0] = (float)((double)(long long)s_sum[sl] / n);
        o[1] = (float)((double)(long long)s_sum[MP_SLOTS + sl] / n);
        o[2] = (float)((double)(long long)s_sum[2 * MP_SLOTS + sl] / n);
    }
    if (tid == 0) { n_out[job] = min(N, cap); if (s_flag || N > cap) atomicOr(status, 1); }
}

}  // namespace pslam

using namespace pslam;

extern "C" int pslam_map_plane_max_points(const pslam_ctx*) { return MP_SLOTS; }

extern "C" int pslam_map_plane_update_batch(pslam_ctx* c, int n_jobs, const int32_t* job_cloud_off, const int32_t* cloud_pt_off, const float* pts, const double* T,
                                            int cap, float* out_pts, int32_t* n_out) {
    if (!c) return PSLAM_E_INVALID;
    if (n_jobs < 0 || cap <= 0 || (n_jobs && (!job_cloud_off || !cloud_pt_off || !out_pts || !n_out || job_cloud_off[0] != 0)))
        return set_error(c, PSLAM_E_INVALID, "bad MapPlane update arguments");
    if (n_jobs == 0) return PSLAM_OK;
    for (int j = 0; j < n_jobs; ++j) if (job_cloud_off[j + 1] < job_cloud_off[j]) return set_error(c, PSLAM_E_INVALID, "job offsets must not decrease");
    const int n_clouds = job_cloud_off[n_jobs];
    if (n_clouds && cloud_pt_off[0] != 0) return set_error(c, PSLAM_E_INVALID, "cloud offsets must start at 0");
    for (int k = 0; k < n_clouds; ++k) if (cloud_pt_off[k + 1] < cloud_pt_off[k]) return set_error(c, PSLAM_E_INVALID, "cloud offsets must not decrease");
    const int n_pts = n_clouds ? cloud_pt_off[n_clouds] : 0;
    if ((n_pts && !pts) || (n_clouds && !T)) return set_error(c, PSLAM_E_INVALID, "bad MapPlane update arrays");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    Slab s;
    const auto d_job_off = s.add<int32_t>(n_jobs + 1), d_cloud_off = s.add<int32_t>(n_clouds + 1);
    const auto d_pts = s.add<float>((size_t)n_pts * 3);
    const auto d_T = s.add<double>((size_t)n_clouds * 16);
    const auto d_out = s.add<float>((size_t)n_jobs * cap * 3);
    const auto d_n_out = s.add<int32_t>(n_jobs), d_flag = s.add<int32_t>(1);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.zero(d_flag, st);
    s.up(d_job_off, job_cloud_off, st); s.up(d_cloud_off, cloud_pt_off, st); s.up(d_pts, pts, st); s.up(d_T, T, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    const size_t smem = (size_t)MP_SLOTS * (3 * 8 + 3 * 4);
    PSLAM_CUDA(c, cudaFuncSetAttribute(k_map_plane_update, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PSLAM_LAUNCH(c, "map_plane_update", k_map_plane_update<<<n_jobs, MP_THREADS, smem, st>>>(s[d_job_off], s[d_cloud_off], s[d_pts], s[d_T], cap, s[d_out], s[d_n_out],
                 s[d_flag]));
    PSLAM_CUDA(c, cudaGetLastError());
    int32_t flag = 0;
    s.down(out_pts, d_out, st); s.down(n_out, d_n_out, st); s.down(&flag, d_flag, st);
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    if (flag) return set_error(c, PSLAM_E_CAPACITY, "MapPlane update: more occupied voxels than the capacity (or a point beyond the voxel key range)");
    return PSLAM_OK;
}
