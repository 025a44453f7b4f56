// Internal declarations shared by the translation units of libpslam_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/pslam_abi.h"

#define PSLAM_MAX_LEVELS 8

namespace pslam {

// Geometry of one pyramid level and of its FAST cell grid (reference: src/ORBextractor.cc:771-806, :1107-1116).
struct LevelGeom {
    int w, h, pitch;          // pitch: bytes per row in the pyramid buffer (multiple of 16); level 0 lives in the input
    int pyr_off;              // byte offset of the level inside one frame's pyramid buffer (level 0: unused)
    int blur_off, blur_pitch; // the blurred copy of the level (all levels, incl. 0) inside one frame's blur buffer
    int n_cols, n_rows;       // FAST cell grid
    int w_cell, h_cell;
    int max_bx, max_by;       // maxBorderX/Y (minBorder is 16)
    int cell_base;            // index of this level's first cell among all cells of a frame
    int slot_cap;             // candidate slots per cell
    int slot_base;            // index of this level's first slot among all slots of a frame
    int quota;                // mnFeaturesPerLevel
    int kp_cap;               // quota + 3 (the quadtree can overshoot by at most 2)
    int kp_base;              // first row of this level in the per-frame level-keypoint scratch
    int cand_cap;             // capacity of the ordered candidate list fed to the quadtree
    int cand_base;            // first entry of this level in the per-frame candidate scratch
    int node_cap, node_base;  // quadtree node pool
    int tabx_off, taby_off;   // offsets of this level's resize tables (x: w entries, y: h entries) in the table buffers
    int n_ini; float h_x;     // quadtree roots (reference DistributeOctTree :543-545)
    int work_base;            // first int of this level in the per-frame quadtree scratch
    float scale;              // mvScaleFactor[level]
    int patch_size;           // (int)(31 * scale)
};

struct OrbGeom {
    int nlevels;
    int width, height;
    int total_cells, total_slots, total_kp, total_cand, total_nodes, total_work, total_tabx, total_taby;
    int pyr_bytes;            // per frame, levels 1..n-1
    LevelGeom lv[PSLAM_MAX_LEVELS];
    int ini_th, min_th;
    int umax[16];
};

// TMA-staged Gaussian blur of the ORB path (orb_kernels.cuh k_blur_tma): tile / box geometry and the kernel parameter block
#define BT_W 128
#define BT_H 64
#define BT_BOX_W 160          // 16 + 128 + 3 rounded up to 16: the box must START at a 16-byte multiple of the row (a start column that is not a
                              // multiple of 16 bytes raised "illegal instruction" in tools/dbg/tma_min.cu), so it starts 16 columns left of the tile
#define BT_X_PAD 16
#define BT_BOX_H 70
struct BlurTmaParams {
    CUtensorMap map[PSLAM_MAX_LEVELS];
    int tile_base[PSLAM_MAX_LEVELS + 1];    // first tile of each level in blockIdx.x
    int tiles_x[PSLAM_MAX_LEVELS];
    int w[PSLAM_MAX_LEVELS], h[PSLAM_MAX_LEVELS], dst_pitch[PSLAM_MAX_LEVELS], dst_off[PSLAM_MAX_LEVELS];
    int nlevels;
};

// PEAC parameters and sizes (compiled-in defaults of the reference: AHCPlaneFitter.hpp:154-158, AHCParamSet.hpp:68-76)
struct PeacGeom {
    int w, h, nbw, nbh, nblk, win;
    int win_magic;            // ceil(2^16 / win): (x * win_magic) >> 16 == x / win for every pixel coordinate (checked at creation)
    int min_support, max_step;
    int adj_words, queue_cap;
    float scale, fx, fy, cx, cy;
    double depth_sigma, std_tol_init, std_tol_merge;
    double z_near, z_far, angle_near, angle_far, t_ang_init_near;
    double sim_merge, sim_refine;
    double depth_alpha, depth_change_tol;
};

struct PeacPlaneRec;
struct PoseBuffers;
struct SearchBuffers;
struct LbaBuffers;
struct LsdBuffers;
struct TrackBuffers;
struct ExchangeBuffers;
struct PlanePostBuffers;
struct BowDbBuffers;
struct BowVocBuffers;
struct FrameBuffers;

}  // namespace pslam

struct pslam_ctx {
    pslam_config cfg;
    pslam::OrbGeom geom;
    std::vector<float> scale, inv_scale, sigma2, inv_sigma2;
    std::vector<int> quota;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    int64_t launches = 0;
    // optional per-kernel timing (pslam_profile_enable): one CUDA event pair per launch on the launching stream
    bool profile = false;
    struct ProfRec { const char* name; cudaEvent_t a, b; };
    std::vector<ProfRec> prof;
    std::string err;
    int last_nframes = 0;
    bool orb_ready = false, peac_ready = false;   // stage buffers are allocated on first use of the stage

    // device buffers (sized for cfg.max_batch frames)
    uint8_t* d_gray = nullptr;        // staging copy of host input (host-pointer entry points)
    const uint8_t* d_gray_cur = nullptr;  // input of the most recent call (staging or caller's device buffer)
    uint8_t* d_pyr = nullptr;         // levels 1.. of every frame
    uint8_t* d_blur = nullptr;        // blurred levels 0.. of every frame (same layout incl. level 0)
    int blur_frame_bytes = 0;
    pslam::BlurTmaParams blur_tma;    // tensor maps of the TMA-staged blur (orb_pipeline.cu); valid for (blur_tma_src, blur_tma_n)
    const uint8_t* blur_tma_src = nullptr; int blur_tma_n = 0;
    CUtensorMap* d_blur_maps = nullptr;      // device copy of blur_tma.map (what the copy engine reads)
    int16_t* d_xofs = nullptr; int16_t* d_xa = nullptr;   // resize tables: source column, (alpha0, alpha1) pairs
    int16_t* d_yofs = nullptr; int16_t* d_ya = nullptr;
    uint32_t* d_slots = nullptr;      // per-cell candidate slots (packed x | y<<11 | score<<22)
    int32_t* d_cell_cnt = nullptr;    // per-cell candidate counts
    uint32_t* d_cand = nullptr;       // ordered candidates per (frame, level), ping-pong x2
    int32_t* d_cand_cnt = nullptr;    // [frame][level]
    int4* d_nodes = nullptr;          // quadtree node pool
    int2* d_links = nullptr;
    int32_t* d_work = nullptr;        // quadtree scratch (expandable lists, list-order array)
    uint32_t* d_lvl_kp = nullptr;     // selected keypoints per (frame, level) in list order (packed)
    int32_t* d_lvl_cnt = nullptr;     // [frame][level]
    int32_t* d_status = nullptr;      // per-frame capacity flags
    pslam_keypoint* d_kps = nullptr;  // outputs for host-pointer entry points
    uint8_t* d_desc = nullptr;
    int32_t* d_n = nullptr;
    // ---- PEAC ----
    pslam::PeacGeom pgeom;
    uint16_t* d_depth = nullptr;                 // staging copy of host depth
    double* d_blk_st = nullptr; double* d_blk_geo = nullptr; int32_t* d_blk_n = nullptr; uint8_t* d_blk_valid = nullptr;
    double* d_node_st = nullptr; double* d_node_geo = nullptr; int32_t* d_node_n = nullptr; int32_t* d_node_rid = nullptr;
    int32_t* d_node_cid = nullptr; uint8_t* d_node_alive = nullptr; uint32_t* d_adj = nullptr; int16_t* d_wlo = nullptr; int16_t* d_whi = nullptr;
    int32_t* d_nb_list = nullptr; float* d_keyf = nullptr; int32_t* d_ds_parent = nullptr; int32_t* d_ds_size = nullptr;
    pslam::PeacPlaneRec* d_coarse = nullptr; int32_t* d_ncoarse = nullptr; int32_t* d_next_cid = nullptr; int32_t* d_blk_map = nullptr;
    float* d_dist = nullptr; uint32_t* d_queue = nullptr; int32_t* d_qlen = nullptr; uint32_t* d_pl_adj = nullptr;
    pslam::PeacPlaneRec* d_final = nullptr; int32_t* d_scratch = nullptr; int32_t* d_final_map = nullptr;
    int32_t* d_labels = nullptr; pslam_plane* d_planes = nullptr; int32_t* d_nplanes = nullptr; int32_t* d_midx = nullptr; int32_t* d_moff = nullptr;
    uint16_t* h_depth = nullptr;                 // pinned
    pslam::PoseBuffers* pose = nullptr;          // pose-optimisation staging (pose_pipeline.cu)
    pslam::SearchBuffers* search = nullptr;      // projection-search staging (search_kernels.cu)
    pslam::LbaBuffers* lba = nullptr;            // local bundle adjustment staging (lba_pipeline.cu)
    pslam::LsdBuffers* lsd = nullptr;            // line-segment detector buffers (lsd_pipeline.cu)
    pslam::TrackBuffers* track = nullptr;        // device-resident tracking chain (track_chain.cu)
    pslam::PlanePostBuffers* planepost = nullptr; // Frame::ComputePlanes post-processing + surface normals (planepost_kernels.cu)
    pslam::FrameBuffers* frame = nullptr;        // staging of pslam_frame_construct_batch (frame_pipeline.cu)
    pslam::BowDbBuffers* bowdb = nullptr;        // key-frame database BowVectors for loop / relocalisation candidates (bow_kernels.cu)
    pslam::BowVocBuffers* bowvoc = nullptr;      // resident DBoW2 vocabulary + batched-transform scratch (bow_transform_kernels.cu)
    pslam::ExchangeBuffers* exchange = nullptr;  // key-frame descriptor exchange over peer memory (exchange_kernels.cu)
    // pinned host staging
    uint8_t* h_gray = nullptr; pslam_keypoint* h_kps = nullptr; uint8_t* h_desc = nullptr; int32_t* h_n = nullptr;
    int32_t* h_status = nullptr;
};

namespace pslam {
int set_error(pslam_ctx* c, int code, const std::string& msg);
int check_cuda(pslam_ctx* c, cudaError_t e, const char* what);
// ORB pipeline (orb_pipeline.cu)
int orb_build_geometry(pslam_ctx* c);
int orb_alloc(pslam_ctx* c);
void orb_free(pslam_ctx* c);
int orb_run_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, pslam_keypoint* d_kps, uint8_t* d_desc, int cap,
                int32_t* d_n);
// pose optimisation (pose_pipeline.cu)
void pose_free(pslam_ctx* c);
void search_free(pslam_ctx* c);
void lba_free(pslam_ctx* c);
void lsd_free(pslam_ctx* c);
void track_free(pslam_ctx* c);
void exchange_free(pslam_ctx* c);
void planepost_free(pslam_ctx* c);
void bowdb_free(pslam_ctx* c);
void bowvoc_free(pslam_ctx* c);
void frame_free(pslam_ctx* c);
int lsd_status_fetch_async(pslam_ctx* c, int nframes, int32_t* h_pinned);
// PEAC pipeline (peac_pipeline.cu)
int peac_build_geometry(pslam_ctx* c);
int peac_alloc(pslam_ctx* c);
void peac_free(pslam_ctx* c);
int peac_run_dev(pslam_ctx* c, const uint16_t* d_depth, int nframes, int32_t* d_labels, pslam_plane* d_planes, int32_t* d_nplanes,
                 int32_t* d_member_idx, int32_t* d_member_off);
}  // namespace pslam

// Launch wrapper: counts the launch and, when profiling is on, brackets it with events on the same stream.
#define PSLAM_LAUNCH(c, name, ...)                                            \
    do {                                                                      \
        pslam_ctx::ProfRec _r{name, nullptr, nullptr};                        \
        if ((c)->profile) { cudaEventCreate(&_r.a); cudaEventCreate(&_r.b); cudaEventRecord(_r.a, (c)->stream); } \
        __VA_ARGS__;                                                          \
        if ((c)->profile) { cudaEventRecord(_r.b, (c)->stream); (c)->prof.push_back(_r); } \
        ++(c)->launches;                                                      \
    } while (0)

// true when p is page-locked host memory known to the CUDA runtime (cudaMallocHost / cudaHostRegister / torch pin_memory)
static inline bool host_ptr_is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

#define PSLAM_CUDA(c, call)                                                   \
    do {                                                                      \
        int _rc = pslam::check_cuda((c), (call), #call);                      \
        if (_rc != PSLAM_OK) return _rc;                                      \
    } while (0)
