// Internal declarations shared by the translation units of libpslam_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/pslam_abi.h"
#include "devmem.h"

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
struct PlanarTrackBuffers;
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
    pslam::DevArray<uint8_t> d_gray;          // staging copy of host input (host-pointer entry points)
    const uint8_t* d_gray_cur = nullptr;      // input of the most recent call (staging or caller's device buffer)
    pslam::DevArray<uint8_t> d_pyr;           // levels 1.. of every frame
    pslam::DevArray<uint8_t> d_blur;          // blurred levels 0.. of every frame (same layout incl. level 0)
    int blur_frame_bytes = 0;
    pslam::BlurTmaParams blur_tma;            // tensor maps of the TMA-staged blur (orb_pipeline.cu); valid for (blur_tma_src, blur_tma_n)
    const uint8_t* blur_tma_src = nullptr; int blur_tma_n = 0;
    pslam::DevArray<CUtensorMap> d_blur_maps; // device copy of blur_tma.map (what the copy engine reads)
    pslam::DevArray<int16_t> d_xofs, d_xa;    // resize tables: source column, (alpha0, alpha1) pairs
    pslam::DevArray<int16_t> d_yofs, d_ya;
    pslam::DevArray<uint32_t> d_slots;        // per-cell candidate slots (packed x | y<<11 | score<<22)
    pslam::DevArray<int32_t> d_cell_cnt;      // per-cell candidate counts
    pslam::DevArray<uint32_t> d_cand;         // ordered candidates per (frame, level), ping-pong x2
    pslam::DevArray<int32_t> d_cand_cnt;      // [frame][level]
    pslam::DevArray<int4> d_nodes;            // quadtree node pool
    pslam::DevArray<int2> d_links;
    pslam::DevArray<int32_t> d_work;          // quadtree scratch (expandable lists, list-order array)
    pslam::DevArray<uint32_t> d_lvl_kp;       // selected keypoints per (frame, level) in list order (packed)
    pslam::DevArray<int32_t> d_lvl_cnt;       // [frame][level]
    pslam::DevArray<int32_t> d_status;        // per-frame capacity flags
    pslam::DevArray<pslam_keypoint> d_kps;    // outputs for host-pointer entry points
    pslam::DevArray<uint8_t> d_desc;
    pslam::DevArray<int32_t> d_n;
    // ---- PEAC ----
    pslam::PeacGeom pgeom;
    pslam::DevArray<uint16_t> d_depth;        // staging copy of host depth
    pslam::DevArray<double> d_blk_st, d_blk_geo; pslam::DevArray<int32_t> d_blk_n; pslam::DevArray<uint8_t> d_blk_valid;
    pslam::DevArray<double> d_node_st, d_node_geo; pslam::DevArray<int32_t> d_node_n, d_node_rid, d_node_cid; pslam::DevArray<uint8_t> d_node_alive;
    pslam::DevArray<uint32_t> d_adj; pslam::DevArray<int16_t> d_wlo, d_whi;
    pslam::DevArray<int32_t> d_nb_list; pslam::DevArray<float> d_keyf; pslam::DevArray<int32_t> d_ds_parent, d_ds_size;
    pslam::DevArray<pslam::PeacPlaneRec> d_coarse; pslam::DevArray<int32_t> d_ncoarse, d_next_cid, d_blk_map;
    pslam::DevArray<float> d_dist; pslam::DevArray<uint32_t> d_queue; pslam::DevArray<int32_t> d_qlen; pslam::DevArray<uint32_t> d_pl_adj;
    pslam::DevArray<pslam::PeacPlaneRec> d_final; pslam::DevArray<int32_t> d_scratch, d_final_map;
    pslam::DevArray<int32_t> d_labels; pslam::DevArray<pslam_plane> d_planes; pslam::DevArray<int32_t> d_nplanes, d_midx, d_moff;
    pslam::PinnedArray<uint16_t> h_depth;
    pslam::PoseBuffers* pose = nullptr;          // pose-optimisation staging (pose_pipeline.cu)
    pslam::SearchBuffers* search = nullptr;      // projection-search staging (search_kernels.cu)
    pslam::LbaBuffers* lba = nullptr;            // local bundle adjustment staging (lba_pipeline.cu)
    pslam::LsdBuffers* lsd = nullptr;            // line-segment detector buffers (lsd_pipeline.cu)
    pslam::TrackBuffers* track = nullptr;        // device-resident tracking chain (track_chain.cu)
    pslam::PlanarTrackBuffers* ptrack = nullptr; // device-resident planar tracking chain (track_chain.cu)
    pslam::PlanePostBuffers* planepost = nullptr; // Frame::ComputePlanes post-processing + surface normals (planepost_kernels.cu)
    pslam::FrameBuffers* frame = nullptr;        // staging of pslam_frame_construct_batch (frame_pipeline.cu)
    pslam::BowDbBuffers* bowdb = nullptr;        // key-frame database BowVectors for loop / relocalisation candidates (bow_kernels.cu)
    pslam::BowVocBuffers* bowvoc = nullptr;      // resident DBoW2 vocabulary + batched-transform scratch (bow_transform_kernels.cu)
    pslam::ExchangeBuffers* exchange = nullptr;  // key-frame descriptor exchange over peer memory (exchange_kernels.cu)
    // pinned host staging
    pslam::PinnedArray<uint8_t> h_gray; pslam::PinnedArray<pslam_keypoint> h_kps; pslam::PinnedArray<uint8_t> h_desc; pslam::PinnedArray<int32_t> h_n;
    pslam::PinnedArray<int32_t> h_status;
};

namespace pslam {
int set_error(pslam_ctx* c, int code, const std::string& msg);
int check_cuda(pslam_ctx* c, cudaError_t e, const char* what);
// ORB pipeline (orb_pipeline.cu)
int orb_build_geometry(pslam_ctx* c);
int orb_alloc(pslam_ctx* c);
int orb_run_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, pslam_keypoint* d_kps, uint8_t* d_desc, int cap,
                int32_t* d_n);
// device-pointer launchers of the per-function kernels, for the tracking chains (track_chain.cu); enqueue on the context's stream
int line_search_run_dev(pslam_ctx* c, int nf, const float* pt, const float* angle, const int32_t* octave, const uint8_t* desc, const uint8_t* has_obs, const float* scale,
                        int n_levels, int nm, const uint8_t* skip, const int32_t* level, const float* view_cos, const float* proj, const uint8_t* mdesc,
                        const uint8_t* m_has_obs, float th, float nnratio, int32_t* assigned, int32_t* nmatches);   // linesearch_kernels.cu
int plane_match_run_dev(pslam_ctx* c, int n_frame, int n_map, const float* pM, const float* map_coef, const uint8_t* map_bad, const int32_t* pts_begin,
                        const int32_t* pts_end, const float* pts, float* ang, float* mind, float dTh, float aTh, float verTh, float parTh, int32_t* match, int32_t* ver, int32_t* par,
                        int32_t* nmatches);                                                                                   // planematch_kernels.cu
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
const int32_t* lsd_status_dev(const pslam_ctx* c);
// PEAC pipeline (peac_pipeline.cu)
int peac_build_geometry(pslam_ctx* c);
int peac_alloc(pslam_ctx* c);
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
