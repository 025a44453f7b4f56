// Host side of the PEAC plane extractor: parameters (compiled-in defaults of the reference), buffers, launch sequence.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "peac_kernels.cuh"

namespace pslam {

int peac_build_geometry(pslam_ctx* c) {
    const pslam_config& cf = c->cfg;
    PeacGeom& g = c->pgeom;
    std::memset(&g, 0, sizeof(g));
    g.w = cf.width; g.h = cf.height; g.win = 10;                       // windowWidth/Height, AHCPlaneFitter.hpp:156
    g.nbw = g.w / g.win; g.nbh = g.h / g.win; g.nblk = g.nbw * g.nbh;
    g.min_support = 3000; g.max_step = 100000;                         // :155
    g.adj_words = (g.nblk + 31) / 32;
    g.queue_cap = 2 * g.w * g.h;
    g.scale = cf.depth_scale; g.fx = cf.fx; g.fy = cf.fy; g.cx = cf.cx; g.cy = cf.cy;
    g.depth_sigma = 1.6e-6; g.std_tol_init = 5; g.std_tol_merge = 8;   // AHCParamSet.hpp:68-76
    g.z_near = 500; g.z_far = 4000;
    g.angle_near = 15.0 * M_PI / 180.0; g.angle_far = 90.0 * M_PI / 180.0;
    {   // T_ang(P_INIT, z <= z_near), AHCParamSet.hpp:120-127, evaluated with the host libm like the CPU path does
        const double factor = (g.angle_far - g.angle_near) / (g.z_far - g.z_near);
        g.t_ang_init_near = std::cos(factor * g.z_near + g.angle_near - factor * g.z_near);
    }
    g.sim_merge = std::cos(60.0 * M_PI / 180.0);
    g.sim_refine = std::cos(30.0 * M_PI / 180.0);
    g.depth_alpha = 0.04; g.depth_change_tol = 0.02;
    // PEAC_MAX_PLANES (128) is a capacity, not a bound derived from the frame size: a frame with more planes of >= 3000
    // points each raises PSLAM_E_CAPACITY at run time (status flag 16).
    if (g.w > 4096 || g.h > 4096) return set_error(c, PSLAM_E_INVALID, "frame larger than 4096 in one dimension (12-bit queue coordinates)");
    g.win_magic = (65536 + g.win - 1) / g.win;
    for (int x = 0; x < std::max(g.w, g.h); ++x)
        if (((x * g.win_magic) >> 16) != x / g.win) return set_error(c, PSLAM_E_INVALID, "block index reciprocal is not exact for this frame size");
    if (g.nblk < 1) return set_error(c, PSLAM_E_INVALID, "frame smaller than one PEAC block");
    if (g.nblk > 65535) return set_error(c, PSLAM_E_INVALID, "more than 65535 PEAC blocks per frame (the clustering heap holds 16-bit slot ids)");
    if (!(cf.fx != 0.f) || !(cf.fy != 0.f) || !(cf.depth_scale > 0.f)) return set_error(c, PSLAM_E_INVALID, "fx, fy must be non-zero and depth_scale > 0");
    return PSLAM_OK;
}

int peac_alloc(pslam_ctx* c) {
    const PeacGeom& g = c->pgeom;
    const size_t B = c->cfg.max_batch, nb = g.nblk, px = (size_t)g.w * g.h;
    int rc;
    if ((rc = c->d_depth.reserve(c, B * px)) ||
        (rc = c->d_blk_st.reserve(c, B * nb * 9)) || (rc = c->d_blk_geo.reserve(c, B * nb * 8)) || (rc = c->d_blk_n.reserve(c, B * nb)) || (rc = c->d_blk_valid.reserve(c, B * nb)) ||
        (rc = c->d_node_st.reserve(c, B * nb * 9)) || (rc = c->d_node_geo.reserve(c, B * nb * 8)) || (rc = c->d_node_n.reserve(c, B * nb)) ||
        (rc = c->d_node_rid.reserve(c, B * nb)) || (rc = c->d_node_cid.reserve(c, B * nb)) || (rc = c->d_node_alive.reserve(c, B * nb)) ||
        (rc = c->d_adj.reserve(c, B * nb * g.adj_words)) || (rc = c->d_wlo.reserve(c, B * nb)) || (rc = c->d_whi.reserve(c, B * nb)) ||
        (rc = c->d_nb_list.reserve(c, B * nb)) || (rc = c->d_keyf.reserve(c, B * nb)) ||
        (rc = c->d_ds_parent.reserve(c, B * nb)) || (rc = c->d_ds_size.reserve(c, B * nb)) ||
        (rc = c->d_coarse.reserve(c, B * PEAC_MAX_PLANES)) || (rc = c->d_ncoarse.reserve(c, B)) || (rc = c->d_next_cid.reserve(c, B)) ||
        (rc = c->d_blk_map.reserve(c, B * nb)) ||
        (rc = c->d_dist.reserve(c, B * px)) || (rc = c->d_queue.reserve(c, B * g.queue_cap)) || (rc = c->d_qlen.reserve(c, B)) ||
        (rc = c->d_pl_adj.reserve(c, B * PEAC_MAX_PLANES * PEAC_PL_WORDS)) ||
        (rc = c->d_final.reserve(c, B * PEAC_MAX_PLANES)) || (rc = c->d_scratch.reserve(c, B * (size_t)peac_num_sub(g) * PEAC_MAX_PLANES)) ||
        (rc = c->d_final_map.reserve(c, B * PEAC_MAX_PLANES)) ||
        (rc = c->d_labels.reserve(c, B * px)) || (rc = c->d_planes.reserve(c, B * PEAC_MAX_PLANES)) || (rc = c->d_nplanes.reserve(c, B)) ||
        (rc = c->d_midx.reserve(c, B * px)) || (rc = c->d_moff.reserve(c, B * (PEAC_MAX_PLANES + 1))) ||
        (rc = c->h_depth.reserve(c, B * px)))
        return rc;
    c->peac_ready = true;
    return PSLAM_OK;
}

// resident-CTA target of the clustering kernel (see k_peac_cluster): PSLAM_PEAC_OCC = 12 (default), 16 or 20
static int peac_cluster_occ() {
    static const int occ = [] { const char* e = std::getenv("PSLAM_PEAC_OCC"); const int v = e ? std::atoi(e) : 12; return (v == 16 || v == 20) ? v : 12; }();
    return occ;
}
static size_t peac_cluster_smem(const PeacGeom& g, int occ) {
    return (size_t)g.nblk * (occ > 12 ? sizeof(uint16_t) : sizeof(float) + sizeof(uint16_t));      // u16 heap (+ float heap keys)
}

int peac_run_dev(pslam_ctx* c, const uint16_t* d_depth, int nframes, int32_t* d_labels, pslam_plane* d_planes, int32_t* d_nplanes,
                 int32_t* d_member_idx, int32_t* d_member_off) {
    const PeacGeom& g = c->pgeom;
    if (nframes < 1 || nframes > c->cfg.max_batch) return set_error(c, PSLAM_E_INVALID, "nframes outside [1, max_batch]");
    if (!d_depth || !d_labels || !d_planes || !d_nplanes || !d_member_idx || !d_member_off) return set_error(c, PSLAM_E_INVALID, "null device pointer");
    if (!c->peac_ready) { const int arc = peac_alloc(c); if (arc != PSLAM_OK) return arc; }
    cudaStream_t st = c->stream;
    c->last_nframes = nframes;
    PSLAM_CUDA(c, cudaMemsetAsync(c->d_status, 0, nframes * sizeof(int32_t), st));
    PSLAM_CUDA(c, cudaMemsetAsync(c->d_adj, 0, (size_t)nframes * g.nblk * g.adj_words * sizeof(uint32_t), st));
    PSLAM_CUDA(c, cudaMemsetAsync(c->d_pl_adj, 0, (size_t)nframes * PEAC_MAX_PLANES * PEAC_PL_WORDS * sizeof(uint32_t), st));
    PSLAM_LAUNCH(c, "peac_blocks", k_peac_blocks<<<dim3((g.nblk + 127) / 128, nframes), 128, 0, st>>>(g, d_depth, c->d_blk_st, c->d_blk_geo, c->d_blk_n, c->d_blk_valid));
    const int occ = peac_cluster_occ();
    const size_t cluster_smem = peac_cluster_smem(g, occ);
#define PEAC_CLUSTER(V) do { \
        PSLAM_CUDA(c, cudaFuncSetAttribute(k_peac_cluster<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cluster_smem)); \
        PSLAM_CUDA(c, cudaFuncSetAttribute(k_peac_cluster<V>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared)); \
        PSLAM_LAUNCH(c, "peac_cluster", k_peac_cluster<V><<<nframes, 32, cluster_smem, st>>>(g, c->d_blk_st, c->d_blk_geo, c->d_blk_n, c->d_blk_valid, c->d_node_st, \
                     c->d_node_geo, c->d_node_n, c->d_node_rid, c->d_node_cid, c->d_node_alive, c->d_adj, c->d_wlo, c->d_whi, c->d_nb_list, c->d_ds_parent, c->d_ds_size, \
                     c->d_coarse, c->d_ncoarse, c->d_blk_map, c->d_next_cid, c->d_status, c->d_keyf)); } while (0)
    if (occ == 16) PEAC_CLUSTER(16); else if (occ == 20) PEAC_CLUSTER(20); else PEAC_CLUSTER(12);
#undef PEAC_CLUSTER
    PSLAM_LAUNCH(c, "peac_seed", k_peac_seed<<<nframes, 256, 0, st>>>(g, c->d_blk_map, d_labels, c->d_dist, c->d_queue, c->d_qlen));
    const size_t flood_smem = PEAC_MAX_PLANES * sizeof(FloodPlane) + (size_t)g.nblk;
    PSLAM_CUDA(c, cudaFuncSetAttribute(k_peac_flood, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)flood_smem));
    PSLAM_LAUNCH(c, "peac_flood", k_peac_flood<<<nframes, 32, flood_smem, st>>>(g, d_depth, c->d_blk_map, c->d_coarse, c->d_ncoarse, d_labels, c->d_dist, c->d_queue,
                 c->d_qlen, c->d_pl_adj, c->d_status));
    PSLAM_LAUNCH(c, "peac_final_merge", k_peac_final_merge<<<nframes, 32, 0, st>>>(g, c->d_coarse, c->d_ncoarse, c->d_next_cid, c->d_pl_adj, c->d_ds_parent,
                 c->d_ds_size, c->d_final, d_planes, d_nplanes, c->d_final_map, c->d_status));
    const int nsub = peac_num_sub(g);
    const dim3 mgrid((nsub + PEAC_SUB_WARPS - 1) / PEAC_SUB_WARPS, nframes);
    PSLAM_LAUNCH(c, "peac_member_count", k_peac_member_count<<<mgrid, 32 * PEAC_SUB_WARPS, 0, st>>>(g, d_labels, c->d_final_map, d_nplanes, c->d_scratch, nsub));
    PSLAM_LAUNCH(c, "peac_member_scan", k_peac_member_scan<<<nframes, PEAC_MAX_PLANES, 0, st>>>(d_nplanes, c->d_scratch, d_member_off, nsub));
    PSLAM_LAUNCH(c, "peac_member_scatter", k_peac_member_scatter<<<mgrid, 32 * PEAC_SUB_WARPS, 0, st>>>(g, d_labels, c->d_final_map, d_nplanes, c->d_scratch,
                 d_member_off, d_member_idx, nsub));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_peac_max_planes(const pslam_ctx*) { return PEAC_MAX_PLANES; }
int pslam_peac_num_blocks(const pslam_ctx* c) { return c ? c->pgeom.nblk : 0; }

int pslam_peac_wave_frames(const pslam_ctx* c) {
    if (!c) return 0;
    const int occ = peac_cluster_occ();
    const size_t cluster_smem = peac_cluster_smem(c->pgeom, occ);
    int per_sm = 0, sms = 0, dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
#define PEAC_OCCUPANCY(V) do { \
        if (cudaFuncSetAttribute(k_peac_cluster<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cluster_smem) != cudaSuccess) return 0; \
        cudaFuncSetAttribute(k_peac_cluster<V>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared); \
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_peac_cluster<V>, 32, cluster_smem) != cudaSuccess) return 0; } while (0)
    if (occ == 16) PEAC_OCCUPANCY(16); else if (occ == 20) PEAC_OCCUPANCY(20); else PEAC_OCCUPANCY(12);
#undef PEAC_OCCUPANCY
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return per_sm * sms;
}

int pslam_peac_run_batch_dev(pslam_ctx* c, const uint16_t* d_depth, int nframes, int32_t* d_labels, pslam_plane* d_planes, int32_t* d_nplanes,
                             int32_t* d_member_idx, int32_t* d_member_off) {
    if (!c) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return peac_run_dev(c, d_depth, nframes, d_labels, d_planes, d_nplanes, d_member_idx, d_member_off);
}

int pslam_peac_run_batch(pslam_ctx* c, const uint16_t* depth, int nframes, int32_t* labels, pslam_plane* planes, int32_t* nplanes,
                         int32_t* member_idx, int32_t* member_off) {
    if (!c) return PSLAM_E_INVALID;
    if (!depth || !labels || !planes || !nplanes) return set_error(c, PSLAM_E_INVALID, "null pointer");
    if (nframes < 1 || nframes > c->cfg.max_batch) return set_error(c, PSLAM_E_INVALID, "nframes outside [1, max_batch]");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->peac_ready) { const int arc = peac_alloc(c); if (arc != PSLAM_OK) return arc; }
    const PeacGeom& g = c->pgeom;
    const size_t px = (size_t)g.w * g.h;
    cudaStream_t st = c->stream;
    const uint16_t* src = depth;                       // page-locked caller memory goes straight to the copy engine
    if (!host_ptr_is_pinned(depth)) { std::memcpy(c->h_depth, depth, px * nframes * sizeof(uint16_t)); src = c->h_depth; }
    PSLAM_CUDA(c, cudaMemcpyAsync(c->d_depth, src, px * nframes * sizeof(uint16_t), cudaMemcpyHostToDevice, st));
    int rc = peac_run_dev(c, c->d_depth, nframes, c->d_labels, c->d_planes, c->d_nplanes, c->d_midx, c->d_moff);
    if (rc != PSLAM_OK) return rc;
    PSLAM_CUDA(c, cudaMemcpyAsync(labels, c->d_labels, px * nframes * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(planes, c->d_planes, (size_t)nframes * PEAC_MAX_PLANES * sizeof(pslam_plane), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(nplanes, c->d_nplanes, nframes * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (member_idx) PSLAM_CUDA(c, cudaMemcpyAsync(member_idx, c->d_midx, px * nframes * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (member_off) PSLAM_CUDA(c, cudaMemcpyAsync(member_off, c->d_moff, (size_t)nframes * (PEAC_MAX_PLANES + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(c->h_status, c->d_status, nframes * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    int bits = 0;
    for (int i = 0; i < nframes; ++i) bits |= c->h_status[i];
    if (bits) return set_error(c, PSLAM_E_CAPACITY, "PEAC capacity exceeded (16: more than PEAC_MAX_PLANES planes, 32: region-growing queue)");
    return PSLAM_OK;
}

int pslam_peac_debug_blocks(pslam_ctx* c, int frame, double* st9, double* geo8, int32_t* n, uint8_t* valid) {
    if (!c || !c->peac_ready || frame < 0 || frame >= c->last_nframes) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    const size_t nb = c->pgeom.nblk, o = (size_t)frame * nb;
    if (st9) PSLAM_CUDA(c, cudaMemcpy(st9, c->d_blk_st + o * 9, nb * 9 * sizeof(double), cudaMemcpyDeviceToHost));
    if (geo8) PSLAM_CUDA(c, cudaMemcpy(geo8, c->d_blk_geo + o * 8, nb * 8 * sizeof(double), cudaMemcpyDeviceToHost));
    if (n) PSLAM_CUDA(c, cudaMemcpy(n, c->d_blk_n + o, nb * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (valid) PSLAM_CUDA(c, cudaMemcpy(valid, c->d_blk_valid + o, nb, cudaMemcpyDeviceToHost));
    return PSLAM_OK;
}

int pslam_peac_debug_coarse(pslam_ctx* c, int frame, int32_t* blk_map, int32_t* n_coarse) {
    if (!c || !c->peac_ready || frame < 0 || frame >= c->last_nframes) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    const size_t nb = c->pgeom.nblk;
    if (blk_map) PSLAM_CUDA(c, cudaMemcpy(blk_map, c->d_blk_map + (size_t)frame * nb, nb * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (n_coarse) PSLAM_CUDA(c, cudaMemcpy(n_coarse, c->d_ncoarse + frame, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return PSLAM_OK;
}

}  // extern "C"
