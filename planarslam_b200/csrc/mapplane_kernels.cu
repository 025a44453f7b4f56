// MapPlane::UpdateCoefficientsAndPoints() and (const Frame&, int id) on sm_90a (src/MapPlane.cc:298-365): the plane clouds of a map plane's observations
// (KeyFrame::mvPlanePoints[id], camera frame) are brought into the world frame by pcl::transformPointCloud (double 4x4 on float points, rounded to float),
// concatenated - the second overload appends the map plane's current cloud - and reduced by pcl::VoxelGrid (leaf 0.1 m): one centroid per occupied voxel in
// ascending voxel index becomes MapPlane::mvPlanePoints.  The pcl::SACSegmentation call that follows in the reference writes into locals nobody reads.
// One CTA per map plane ("job"): the same order-free fixed-point voxel table as k_planes_post (planepost_kernels.cu), 4096 slots here because a map plane
// accumulates the extent of many views; the body (mapplane_body.cuh) is shared with the planar chain's per-frame update (track_chain.cu).
// Oracle: oracle/planepost.cc map_plane_update (PCL absent: parity unpinned).
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "pslam_internal.h"
#include "mapplane_body.cuh"

namespace pslam {

__global__ void __launch_bounds__(MP_THREADS) k_map_plane_update(const int32_t* __restrict__ job_off, const int32_t* __restrict__ cloud_off, const float* __restrict__ pts,
                                                                 const double* __restrict__ T, int cap, float* __restrict__ out_pts, int32_t* __restrict__ n_out,
                                                                 int32_t* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char mp_smem[];
    __shared__ int s_flag, s_n;
    const int job = blockIdx.x, tid = threadIdx.x;
    const MpTable S = mp_table(mp_smem, &s_flag, &s_n);
    mp_clear(S, tid);
    __syncthreads();
    for (int c = job_off[job]; c < job_off[job + 1]; ++c) mp_add(S, tid, pts, cloud_off[c], cloud_off[c + 1], T + 16 * (size_t)c);
    mp_sort(S, tid);
    mp_emit(S, tid, cap, out_pts + (size_t)job * cap * 3);
    const int N = s_n;
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
    const size_t smem = MP_SMEM;
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
