/* pslam_abi.h — C ABI of the H100-native PlanarSLAM per-frame hot path (libpslam_b200.so).
 *
 * The reference (yanyan-li/PlanarSLAM) has no plugin/FFI layer: its seam is a set of C++ methods called
 * from Frame / Tracking (SURVEY.md §8b).  Each entry point below replaces one of those methods with plain
 * pointers and sizes; include/pslam_adapter.hpp re-creates the reference's C++ signatures on top of it.
 *
 * Conventions: every function returns 0 on success or a negative pslam_status; nothing throws; the callee
 * never allocates caller-visible memory (the caller passes capacities); a context is bound to one GPU and is
 * used by one thread at a time (the reference calls ORB / LSD / PEAC from three threads: use one context
 * per thread, they are re-entrant across contexts).  There is NO CPU fallback: creation fails with
 * PSLAM_E_NO_DEVICE when no sm_90 device is present.
 *
 * "_dev" variants take device pointers and enqueue on the context's stream without synchronising
 * (inputs already resident in HBM); the plain variants take host pointers, copy in, run, copy out and
 * synchronise — that is the call a Frame-constructor replacement makes.
 */
#ifndef PSLAM_ABI_H_
#define PSLAM_ABI_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pslam_status {
    PSLAM_OK = 0,
    PSLAM_E_INVALID = -1,    /* bad argument (null pointer, size mismatch, unsupported parameter) */
    PSLAM_E_NO_DEVICE = -2,  /* no CUDA device / not sm_90 */
    PSLAM_E_CUDA = -3,       /* CUDA runtime error; see pslam_last_error() */
    PSLAM_E_CAPACITY = -4,   /* an internal or caller capacity was exceeded (results truncated) */
    PSLAM_E_NCCL = -5
} pslam_status;

/* Layout-compatible with cv::KeyPoint {Point2f pt; float size, angle, response; int octave, class_id}
 * as filled by ORBextractor::operator() (src/ORBextractor.cc:1043-1105). 28 bytes. */
typedef struct pslam_keypoint {
    float x, y, size, angle, response;
    int32_t octave, class_id;
} pslam_keypoint;

/* Parameters of the reference constructors / settings file that the hot path reads
 * (ORBextractor ctor include/ORBextractor.h:51-52; Examples/RGB-D/TUM3.yaml:8-55). */
typedef struct pslam_config {
    int32_t device;        /* CUDA ordinal */
    int32_t width, height; /* frame size, all frames of a context share it */
    int32_t max_batch;     /* frames processed per batched call (>= 1) */
    /* ORB */
    int32_t nfeatures;     /* ORBextractor.nFeatures   (1000) */
    float scale_factor;    /* ORBextractor.scaleFactor (1.2)  */
    int32_t nlevels;       /* ORBextractor.nLevels     (8, max 8) */
    int32_t ini_th_fast;   /* ORBextractor.iniThFAST   (20) */
    int32_t min_th_fast;   /* ORBextractor.minThFAST   (7), must be <= ini_th_fast */
    /* camera (Camera.fx .. DepthMapFactor); float like the reference's cv::Mat K (CV_32F) */
    float fx, fy, cx, cy;
    float depth_scale;     /* metres per depth unit = 1 / DepthMapFactor, as float (src/Tracking.cc) */
} pslam_config;

typedef struct pslam_ctx pslam_ctx;

/* Fill cfg with the reference defaults for TUM3.yaml at the given size / batch. */
void pslam_default_config(pslam_config* cfg, int width, int height, int max_batch);

int pslam_create(const pslam_config* cfg, pslam_ctx** out);
void pslam_destroy(pslam_ctx* ctx);
const char* pslam_last_error(const pslam_ctx* ctx);
/* Run on a caller-owned CUDA stream (cudaStream_t / CUstream as void*); NULL restores the context's own. */
int pslam_set_stream(pslam_ctx* ctx, void* cuda_stream);
int pslam_synchronize(pslam_ctx* ctx);
/* Number of kernel launches this context has issued since creation (bench.py's gpu_launches claim). */
int64_t pslam_launch_count(const pslam_ctx* ctx);

/* Per-kernel timing for the roofline report: when enabled every kernel launch is bracketed by a CUDA event pair
 * on the launching stream (do not enable inside a timed throughput region).  pslam_profile_report() synchronises
 * and writes one line per kernel name: "<name> <launches> <total_ms>\n". Enabling again clears the records. */
int pslam_profile_enable(pslam_ctx* ctx, int on);
int pslam_profile_report(pslam_ctx* ctx, char* buf, int cap);

/* ---- ORB extraction -------------------------------------------------------------------------------
 * Replaces  void ORBextractor::operator()(InputArray image, InputArray mask, vector<KeyPoint>&, OutputArray desc)
 *           include/ORBextractor.h:59-61, src/ORBextractor.cc:1043-1105   (mask is ignored there too).
 * Scale tables replace the getters include/ORBextractor.h:63-83 (read by Frame.cc:65-71).
 */
int pslam_orb_get_scale_tables(const pslam_ctx* ctx, float* scale, float* inv_scale, float* sigma2,
                               float* inv_sigma2, int32_t* features_per_level /* each nlevels long, may be NULL */);

/* One frame, host buffers. gray: height rows of `stride` bytes. kps/desc: room for `cap` keypoints
 * (desc is cap x 32 bytes).  *n receives the number found; if it exceeds cap the first cap are written and
 * PSLAM_E_CAPACITY is returned.  pslam_orb_max_keypoints() is always enough. */
int pslam_orb_extract(pslam_ctx* ctx, const uint8_t* gray, int stride, pslam_keypoint* kps, uint8_t* desc,
                      int cap, int32_t* n);
int pslam_orb_max_keypoints(const pslam_ctx* ctx);

/* Batched: nframes <= max_batch images, each height x width, densely packed (frame stride = width*height).
 * Outputs are [nframes][cap] keypoints, [nframes][cap][32] descriptor bytes, [nframes] counts. */
int pslam_orb_extract_batch(pslam_ctx* ctx, const uint8_t* gray, int nframes, pslam_keypoint* kps,
                            uint8_t* desc, int cap, int32_t* n);
/* Same with device pointers; asynchronous on the context's stream. */
int pslam_orb_extract_batch_dev(pslam_ctx* ctx, const uint8_t* d_gray, int nframes, pslam_keypoint* d_kps,
                                uint8_t* d_desc, int cap, int32_t* d_n);

/* Stage outputs of the most recent ORB call, for stage-by-stage parity tests (host buffers; synchronises).
 * Level pixels are the borderless level (the reference's mvImagePyramid ROI, include/ORBextractor.h:85). */
int pslam_orb_debug_level_size(const pslam_ctx* ctx, int level, int32_t* w, int32_t* h);
int pslam_orb_debug_level_pixels(pslam_ctx* ctx, int frame, int level, uint8_t* out /* w*h */);
int pslam_orb_debug_level_blurred(pslam_ctx* ctx, int frame, int level, uint8_t* out /* w*h */);
/* FAST candidates of a level in the reference's order (cell-major, row-major inside a cell), as int32
 * triples (x, y, score) relative to (16,16) like vToDistributeKeys (src/ORBextractor.cc:820-825). */
int pslam_orb_debug_level_candidates(pslam_ctx* ctx, int frame, int level, int32_t* xys, int cap, int32_t* n);

/* ---- PEAC plane extraction ------------------------------------------------------------------------
 * Replaces  bool PlaneDetection::readDepthImage(cv::Mat depth16U, cv::Mat& K, float kScaleFactor)   src/PlaneExtractor.cpp:26-57
 *           void PlaneDetection::runPlaneDetection(int H, int W)                                     src/PlaneExtractor.cpp:59-65
 * and the public results Frame::ComputePlanes reads (src/Frame.cc:652-672): plane_num_, plane_vertices_
 * (member_idx / member_off), plane_filter.extractedPlanes[i]->{normal, center, N, mse} (pslam_plane), membershipImg (labels).
 * Camera intrinsics and the depth scale come from pslam_config (fx, fy, cx, cy, depth_scale).
 * The organised cloud is never materialised: x = (j - cx) z / fx etc. are recomputed in double where needed. */
typedef struct pslam_plane {
    double normal[3];   /* unit normal pointing towards the camera (n . c <= 0) */
    double center[3];   /* centre of mass; plane coefficients are (n, -n . c) as in src/Frame.cc:664-672 */
    double mse, curvature;
    int32_t N, rid;     /* supporting points before refinement; root block id */
} pslam_plane;

int pslam_peac_max_planes(const pslam_ctx* ctx);

/* nframes depth images, each height x width uint16, densely packed.  Outputs per frame:
 *   labels     [height*width] int32: final plane index, or a negative value for unlabelled pixels (the raw
 *              region-growing trail counters -1..-6 of the reference's membershipImg)
 *   planes     [pslam_peac_max_planes()] records, the first nplanes[f] valid, sorted by N descending
 *   member_idx [height*width] pixel indices grouped by plane, ascending inside a plane (plane_vertices_)
 *   member_off [pslam_peac_max_planes()+1] start offsets into member_idx; member_off[nplanes] = total
 * member_idx / member_off may be NULL in the host variant. */
int pslam_peac_run_batch(pslam_ctx* ctx, const uint16_t* depth, int nframes, int32_t* labels, pslam_plane* planes,
                         int32_t* nplanes, int32_t* member_idx, int32_t* member_off);
/* Device pointers (all required); asynchronous on the context's stream. */
int pslam_peac_run_batch_dev(pslam_ctx* ctx, const uint16_t* d_depth, int nframes, int32_t* d_labels, pslam_plane* d_planes,
                             int32_t* d_nplanes, int32_t* d_member_idx, int32_t* d_member_off);

/* ---- Plane post-processing of Frame::ComputePlanes (src/Frame.cc:647-753) + Frame::MaxPointDistanceFromPlane (:755-813) ----------------------
 * What turns the PEAC result into  mvPlanePoints / mvPlaneCoefficients  and  vSurfaceNormal:
 *   per PEAC plane: pcl::VoxelGrid(0.1) of its member points -> reject the plane when a voxel centroid is farther than dist_th (Plane.DistanceThreshold) from
 *   (n, -n . c) -> pcl::SACSegmentation plane RANSAC + least-squares refit, sign of d kept (MaxPointDistanceFromPlane) -> coefficients + voxel cloud;
 *   pcl::IntegralImageNormalEstimation(AVERAGE_3D_GRADIENT, 0.05, 10) on the 3x sub-sampled cloud, every 2nd row / column -> surface normals.
 * PCL is not part of the reference tree: the three algorithms are restated (oracle/planepost.cc, parity unpinned upstream; voxel centroids are an order-free
 * fixed-point mean - PCL's float sum runs in the unspecified order std::sort leaves).
 * Outputs per frame: n_kept; src [maxp] = PEAC plane index of every kept plane (PEAC order); coef [maxp][4] float = mvPlaneCoefficients; pt_off [maxp + 1] +
 * pts [cap_pts][3] = mvPlanePoints concatenated; normals8 [pslam_surface_normals_count()][8] = SurfaceNormal {normal xyz (NaN where PCL leaves NaN), cameraPosition
 * xyz, FramePosition xy}.  maxp = pslam_peac_max_planes(); at most pslam_planes_post_max_points() voxels per plane (PSLAM_E_CAPACITY beyond). */
int pslam_surface_normals_count(const pslam_ctx* ctx);
int pslam_planes_post_max_points(const pslam_ctx* ctx);
int pslam_planes_post_batch_dev(pslam_ctx* ctx, const uint16_t* d_depth, int nframes, const pslam_plane* d_planes, const int32_t* d_nplanes, const int32_t* d_member_idx,
                                const int32_t* d_member_off, float dist_th, int32_t* d_n_kept, int32_t* d_src, float* d_coef, int32_t* d_pt_off, float* d_pts, int cap_pts,
                                int32_t* d_status);
/* d_normals3 (optional): the normals alone, [nframes][pslam_surface_normals_count()][3] - the layout pslam_track_manhattan_batch_dev reads (NaN normals stay NaN and fail
 * every cone test there, like in the reference) */
int pslam_surface_normals_batch_dev(pslam_ctx* ctx, const uint16_t* d_depth, int nframes, float* d_normals8, float* d_normals3);
/* Replaces  void MapPlane::UpdateCoefficientsAndPoints()  and  (const Frame& pF, int id)      include/MapPlane.h, src/MapPlane.cc:298-365
 * (called from src/Optimizer.cc:541, 2676, 2989, src/Tracking.cc:300, 1207, 2270; SURVEY.md 8 f4): per map plane ("job") the clouds of its observations - KeyFrame::mvPlanePoints[id] with T = Converter::toMatrix4d(GetPoseInverse());
 * for the second overload the frame's cloud with T = toSE3Quat(mTcw).inverse() plus the plane's current cloud with the identity - are transformed like
 * pcl::transformPointCloud (double 4x4, row-major here, on float points), concatenated and reduced by pcl::VoxelGrid (leaf 0.1 m).  out_pts [n_jobs][cap][3]
 * receives the new MapPlane::mvPlanePoints (voxel centroids in ascending voxel index), n_out [n_jobs] their counts.  Clouds as CSR: job_cloud_off [n_jobs + 1]
 * into the cloud list, cloud_pt_off [n_clouds + 1] into pts (xyz), T [n_clouds][16].  The reference's SACSegmentation call after the filter writes into
 * locals that are never read and is not reproduced.  PSLAM_E_CAPACITY when a plane occupies more than cap (<= pslam_map_plane_max_points()) voxels. */
int pslam_map_plane_max_points(const pslam_ctx* ctx);
int pslam_map_plane_update_batch(pslam_ctx* ctx, int n_jobs, const int32_t* job_cloud_off, const int32_t* cloud_pt_off, const float* pts, const double* T,
                                 int cap, float* out_pts, int32_t* n_out);

/* PEAC + post-processing + normals on host depth images (the whole Frame::ComputePlanes); normals8 may be NULL */
int pslam_compute_planes_batch(pslam_ctx* ctx, const uint16_t* depth, int nframes, float dist_th, int32_t* n_kept, int32_t* src, float* coef, int32_t* pt_off, float* pts,
                               int cap_pts, float* normals8);

/* Stage outputs of the most recent PEAC call (host buffers; synchronises): per 10x10 block the nine running sums
 * (sx sy sz sxx syy szz sxy syz sxz), {center[3], normal[3], mse, curvature}, point count and the "node kept" flag;
 * the eroded block -> coarse plane map and the number of coarse planes before the last merge. */
int pslam_peac_debug_blocks(pslam_ctx* ctx, int frame, double* st9, double* geo8, int32_t* n, uint8_t* valid);
int pslam_peac_debug_coarse(pslam_ctx* ctx, int frame, int32_t* blk_map, int32_t* n_coarse);
int pslam_peac_num_blocks(const pslam_ctx* ctx);
/* Frames the clustering kernel (one warp per frame, the longest stage) keeps resident at once on this device: SM count x
 * resident CTAs per SM.  A replay batch that is a multiple of this number runs in full waves (no reference counterpart). */
int pslam_peac_wave_frames(const pslam_ctx* ctx);

/* ---- Descriptor matching --------------------------------------------------------------------------
 * Replaces the brute-force searches on the tracking path:
 *   static int ORBmatcher::DescriptorDistance(const cv::Mat&, const cv::Mat&)            src/ORBmatcher.cc:1712-1728
 *   int ORBmatcher::MatchORBPoints(Frame& cur, const Frame& last)                        src/ORBmatcher.cc:1332-1394
 *       (cv::BFMatcher(NORM_HAMMING).match(cur.mDescriptors, last.mDescriptors) + the "dist < max(2*min_dist, 15)" gate;
 *        the MapPoint* copy that follows, incl. its mvbOutlier[i] index quirk, stays in the caller)
 *   int LSDmatcher::SearchByDescriptor(KeyFrame*, Frame&, vector<MapLine*>&)             src/LSDmatcher.cpp:242-279
 *       (BFMatcher knnMatch k=2; the ratio test dist0/dist1 < 1/1.5 is one compare per row in the caller)
 * For every query row: the two nearest train rows in (distance, train index) order -> idx2[i][0..1], dist2[i][0..1]
 * (-1 / 256 when missing).  good / n_good (optional): MatchORBPoints' kept query indices in ascending order. */
int pslam_hamming_knn2(pslam_ctx* ctx, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* idx2, int32_t* dist2,
                       int32_t* good, int32_t* n_good);
/* Batched, device pointers, asynchronous: q [nframes][capq][32], t [nframes][capt][32], per-frame counts d_nq / d_nt,
 * outputs [nframes][capq][2]; d_good [nframes][capq] and d_ngood [nframes] may be NULL. capt <= 65535. */
int pslam_hamming_knn2_batch_dev(pslam_ctx* ctx, const uint8_t* d_q, const int32_t* d_nq, int capq, const uint8_t* d_t,
                                 const int32_t* d_nt, int capt, int nframes, int32_t* d_idx2, int32_t* d_dist2, int32_t* d_good,
                                 int32_t* d_ngood);

/* ---- RGB-D "stereo" fields -------------------------------------------------------------------------
 * Replaces  void Frame::ComputeStereoFromRGBD(const cv::Mat& imDepth)   src/Frame.cc:603-621
 * keys = mvKeys, keys_un = mvKeysUn (the same pointer when the camera has no distortion, Frame::UndistortKeyPoints :545-549), both
 * [nframes][cap] with n[f] valid entries; depth: raw uint16 [nframes][height][width], metres = (float)raw * depth_factor (the Frame
 * constructor's convertTo, :80-83); bf = mbf.  Outputs [nframes][cap]: u_right = mvuRight, depth_out = mvDepth (-1 where there is
 * no depth, and for the padding entries). */
int pslam_compute_stereo_from_rgbd_batch(pslam_ctx* ctx, const pslam_keypoint* keys, const pslam_keypoint* keys_un, const int32_t* n, int cap,
                                         const uint16_t* depth, int nframes, float depth_factor, float bf, float* u_right, float* depth_out);
/* Same with device pointers; only enqueues on the context's stream (chains after pslam_orb_extract_batch_dev). */
int pslam_compute_stereo_from_rgbd_batch_dev(pslam_ctx* ctx, const pslam_keypoint* d_keys, const pslam_keypoint* d_keys_un, const int32_t* d_n, int cap,
                                             const uint16_t* d_depth, int nframes, float depth_factor, float bf, float* d_u_right, float* d_depth_out);

/* ---- Projection-guided search ---------------------------------------------------------------------
 * Replaces  int ORBmatcher::SearchByProjection(Frame& F, const vector<MapPoint*>& vpMapPoints, float th)        src/ORBmatcher.cc:46-130
 *           (together with the Frame::isInFrustum pass of Tracking::SearchLocalPoints, src/Tracking.cc:2286-2329, src/Frame.cc:312-367)
 *           int ORBmatcher::SearchByProjection(Frame& cur, const Frame& last, float th, bool bMono)              src/ORBmatcher.cc:1396-1535
 * The Frame / MapPoint objects are passed as plain-array views gathered by the caller under the map mutex:
 *   pslam_frame_view   N, mvKeysUn, mvuRight, mDescriptors, mTcw, fx..mbf, mnMinX..mnMaxY, mvScaleFactors, mfLogScaleFactor
 *   pslam_map_points   GetWorldPos, GetNormal, mfMaxDistance, mfMinDistance, GetDescriptor, skip (= mnLastFrameSeen == frame id or
 *                      isBad()), has_obs (= Observations() > 0)
 *   pslam_last_frame   mvKeys (octave, angle), index of mvpMapPoints[i] in the map arrays (-1: none), mvbOutlier, mTcw
 * matches_io[i] is the index (into the map arrays) held by F.mvpMapPoints[i], -1 for none; it is updated in place with the
 * reference's greedy order-dependent assignment.  Both calls return nmatches (>= 0) or a negative pslam_status. */
typedef struct pslam_frame_view {
    int32_t n; const pslam_keypoint* keys_un; const float* u_right; const uint8_t* desc; float Tcw[16];
    float fx, fy, cx, cy, bf, min_x, max_x, min_y, max_y; int32_t n_levels; const float* scale_factors; float log_scale_factor;
} pslam_frame_view;
typedef struct pslam_map_points {
    int32_t n; const float *pos, *normal, *max_distance, *min_distance; const uint8_t *desc, *skip, *has_obs;
} pslam_map_points;
typedef struct pslam_last_frame { int32_t n; const pslam_keypoint* keys; const int32_t* map_point; const uint8_t* outlier; float Tcw[16]; } pslam_last_frame;

int pslam_search_by_projection_map(pslam_ctx* ctx, const pslam_frame_view* frame, const pslam_map_points* map, float th, float nnratio,
                                   int32_t* matches_io, uint8_t* in_view /* [map.n] mbTrackInView, may be NULL */);
int pslam_search_by_projection_last(pslam_ctx* ctx, const pslam_frame_view* cur, const pslam_last_frame* last, const pslam_map_points* map,
                                    float th, int mono, int check_orientation, int32_t* matches_io);

/* ---- Device-resident tracking chain (BASELINE.json config 3; SURVEY.md section 8 f1) ------------------------------------
 * Replaces the per-frame part of  void Tracking::Track()  src/Tracking.cc:239-304  for a replayed sequence against a fixed map snapshot:
 *   Frame::Frame (ORB + ComputeStereoFromRGBD, src/Frame.cc:90-110, 603-621)                          batched over the sequence
 *   bool Tracking::TrackWithMotionModel()   src/Tracking.cc:1739-1859   pose prediction, SearchByProjection(cur, last), PoseOptimization, outlier sweep
 *   bool Tracking::TrackLocalMap()          src/Tracking.cc:1954-2046   SearchLocalPoints (isInFrustum + SearchByProjection(F, map)), PoseOptimization
 *   mVelocity update                        src/Tracking.cc:270-278
 * The map snapshot (pslam_track_set_map: the arrays of pslam_map_points, copied once) and every intermediate product stay in HBM; nothing is read back
 * between the stages of a frame or between frames.  Frame 0 starts from Tcw0 and runs the local-map stage only; frame 1 predicts with the last pose,
 * later frames with mVelocity when use_motion_model is set.  Tcw_out [nframes][16] float row-major; stats [nframes][4] = {matches, inliers} of the
 * motion-model stage and of the local-map stage.  Not modelled: UpdateLastFrame's temporary RGB-D points, key-frame insertion, line / plane edges. */
typedef struct pslam_track_params {
    float fx, fy, cx, cy, bf;           /* Frame::fx .. mbf */
    float depth_factor;                 /* metres per raw depth unit (1 / DepthMapFactor) */
    float min_x, max_x, min_y, max_y;   /* mnMinX .. mnMaxY */
    float th_last;                      /* window of SearchByProjection(cur, last): 15 for RGB-D (src/Tracking.cc:1757-1764) */
    float th_map;                       /* th of SearchByProjection(F, local map): 3 (src/Tracking.cc:2321-2328) */
    float nnratio_map;                  /* ORBmatcher(0.8) of SearchLocalPoints */
    int32_t use_motion_model;           /* 0: always predict with the last pose */
} pslam_track_params;
int pslam_track_set_map(pslam_ctx* ctx, const pslam_map_points* map);
int pslam_track_sequence_dev(pslam_ctx* ctx, const uint8_t* d_gray, const uint16_t* d_depth, int nframes, const pslam_track_params* params, const float* Tcw0,
                             float* Tcw_out, int32_t* stats /* may be NULL */);
int pslam_track_sequence(pslam_ctx* ctx, const uint8_t* gray, const uint16_t* depth, int nframes, const pslam_track_params* params, const float* Tcw0,
                         float* Tcw_out, int32_t* stats /* may be NULL */);

/* ---- Key-frame descriptor exchange over NVLink peer memory, fused with the Hamming matcher (SURVEY.md section 8e) -------------------
 * The one exchange step of the multi-GPU layout: every rank (one process per GPU) publishes the ORB block of a key frame - descriptors [n][32], key points
 * [n] (28 B), count - into a record in ITS OWN HBM; peers map the records through CUDA IPC (NVLink / NVSwitch P2P) and pslam_exchange_match_dev finds, for
 * every query descriptor, the two nearest rows over the concatenation rank 0 | rank 1 | ... by reading the peers' records in place: the CTA working on peer
 * p starts as soon as p's epoch flag lands, no gathered copy is built.  Same result as pslam_hamming_knn2_batch on the concatenated set (cv::BFMatcher::knnMatch
 * k = 2 - the matcher behind KeyFrameDatabase::DetectLoopCandidates / LoopClosing::ComputeSim3's candidates, src/KeyFrameDatabase.cc:76-197, src/LoopClosing.cc:231-400).
 *   create   allocates `slots` records of capacity cap_kp on the context's device and returns its CUDA IPC handle (PSLAM_IPC_HANDLE_BYTES bytes)
 *   attach   handles = the handles of all ranks in rank order (exchanged by the caller, e.g. torch.distributed.all_gather); world = 1 needs no handles
 *   publish  enqueues the copy + release of `epoch` (> 0) on the context's stream; a slot may be re-published once every rank has matched the old epoch
 *   match    enqueues the fused wait + match; idx [capq][2] = row in the concatenation (-1: none), dist [capq][2] (256: none)
 * Errors: PSLAM_E_NCCL when a peer record cannot be mapped (no P2P path). */
#define PSLAM_IPC_HANDLE_BYTES 64
int pslam_exchange_create(pslam_ctx* ctx, int cap_kp, int slots, void* ipc_handle_out);
int pslam_exchange_attach(pslam_ctx* ctx, int world, int rank, const void* handles /* [world][PSLAM_IPC_HANDLE_BYTES] */);
int pslam_exchange_publish_dev(pslam_ctx* ctx, int slot, const uint8_t* d_desc, const pslam_keypoint* d_kps /* may be NULL */, const int32_t* d_n, uint32_t epoch);
int pslam_exchange_match_dev(pslam_ctx* ctx, int slot, uint32_t epoch, const uint8_t* d_qdesc, const int32_t* d_nq, int capq, int32_t* d_idx, int32_t* d_dist);
/* A matcher CTA that waits more than 20 s for a peer's epoch flag treats that peer's record as empty and counts the wait; this returns the count since create
 * (synchronises the context's stream).  Non-zero means a peer died or the epochs / slots of the ranks are out of step. */
int pslam_exchange_timeouts(pslam_ctx* ctx, int32_t* n_out);

/* ---- Plane association -------------------------------------------------------------------------
 * Replaces  int PlaneMatcher::SearchMapByCoefficients(Frame& pF, const vector<MapPlane*>& vpMapPlanes)   src/PlaneMatcher.cpp:10-67
 * (with Frame::ComputePlaneWorldCoeff, src/Frame.cc:815-820).  frame_coef: mvPlaneCoefficients [n_frame][4]; map_coef: GetWorldPos()
 * [n_map][4]; map_bad: isBad(); pts / pts_off: the map planes' mvPlanePoints concatenated ([pts_off[n_map]][3], plane j owns
 * [pts_off[j], pts_off[j+1])).  Outputs per frame plane: index of the associated map plane (mvpMapPlanes), of the most
 * perpendicular one (mvpVerticalPlanes) and of the most parallel one (mvpParallelPlanes), -1 for none.  Returns nmatches. */
int pslam_plane_match(pslam_ctx* ctx, const float* Tcw, int n_frame, const float* frame_coef, int n_map, const float* map_coef,
                      const uint8_t* map_bad, const int32_t* pts_off, const float* pts, float dTh, float aTh, float verTh, float parTh,
                      int32_t* match, int32_t* ver, int32_t* par);

/* ---- Pose optimisation ---------------------------------------------------------------------------
 * Replaces  static int Optimizer::PoseOptimization(Frame* pFrame)     include/Optimizer.h:38, src/Optimizer.cc:550-1275.
 * A pslam_pose_problem carries exactly what that function reads from the Frame and the matched map objects:
 *   points   mvpMapPoints[i]->GetWorldPos() (float), mvKeysUn[i].pt + mvuRight[i] (uR < 0 => monocular edge),
 *            mvInvLevelSigma2[octave]                                                   (:593-669)
 *   lines    mvpMapLines[i]->mWorldPos (two endpoints, double), mvKeyLineFunctions[i]   (:693-745)
 *   planes   mvPlaneCoefficients[i] (float 4) with the matched / parallel / vertical map plane's GetWorldPos()  (:789-981)
 *   settings Plane.AngleInfo, DistanceInfo, ParallelInfo, VerticalInfo, Chi, VPChi (Config::Get, :771-783); fx, fy, cx, cy, mbf
 * Tcw_io is Frame::mTcw (float 4x4, row-major) in and out; the outlier arrays are mvbOutlier, mvbLineOutlier,
 * mvbPlaneOutlier, mvbParPlaneOutlier, mvbVerPlaneOutlier.  The single-problem call returns the reference's return value
 * (nInitialCorrespondences - nBad, 0 when there are fewer than 3 correspondences) or a negative pslam_status. */
typedef struct pslam_pose_problem {
    float fx, fy, cx, cy, bf;
    int32_t n_points; const float* Xw /* [n][3] */; const float* obs /* [n][3] = u, v, uR */; const float* inv_sigma2 /* [n] */;
    int32_t n_lines; const double* line_Xw /* [n][6] */; const double* line_obs /* [n][3] */;
    int32_t n_planes, n_par, n_ver;
    const float *plane_meas, *plane_map, *par_meas, *par_map, *ver_meas, *ver_map;   /* [n][4] each */
    double angle_info, dist_info, par_info, ver_info, plane_chi, vp_chi;
} pslam_pose_problem;

int pslam_pose_optimization(pslam_ctx* ctx, const pslam_pose_problem* prob, float* Tcw_io /* [16] */, uint8_t* outlier_pt,
                            uint8_t* outlier_line, uint8_t* outlier_plane, uint8_t* outlier_par, uint8_t* outlier_ver);
/* n independent problems (replayed frames).  Tcw_io is [n][16]; each outlier array is the concatenation over the problems
 * in order; n_inliers is [n]. */
int pslam_pose_optimization_batch(pslam_ctx* ctx, const pslam_pose_problem* probs, int n, float* Tcw_io, uint8_t* outlier_pt,
                                  uint8_t* outlier_line, uint8_t* outlier_plane, uint8_t* outlier_par, uint8_t* outlier_ver,
                                  int32_t* n_inliers);
/* Split form for callers that keep the packed problems resident in HBM (bench.py's device-resident number):
 * pack + upload once, run (asynchronous on the context's stream) any number of times, fetch results.
 * Tcw_d: [n][16] double pose before the float cast; trace_i: [n][4][3] = LM iterations, trials, nBad per round (-1: round not
 * run); trace_d: [n][4][2] = final robust chi2 and lambda per round.  Any output pointer may be NULL. */
int pslam_pose_pack(pslam_ctx* ctx, const pslam_pose_problem* probs, int n, const float* Tcw0 /* [n][16] */);
int pslam_pose_run_packed(pslam_ctx* ctx);
int pslam_pose_fetch(pslam_ctx* ctx, float* Tcw, double* Tcw_d, uint8_t* outlier_pt, uint8_t* outlier_line, uint8_t* outlier_plane,
                     uint8_t* outlier_par, uint8_t* outlier_ver, int32_t* n_inliers, int32_t* trace_i, double* trace_d);

/* ---- Translation-only optimisation ---------------------------------------------------------------
 * Replaces  static int Optimizer::TranslationOptimization(Frame* pFrame)   include/Optimizer.h, src/Optimizer.cc:2995-3737
 * (rotation fixed by the Manhattan-frame tracker; map points, line endpoints and plane normals are pre-rotated by the
 * float R_cw of Tcw_io and the edges use SE3Quat::mapTrans).  Same problem struct; par / ver planes are ignored like in the
 * reference (:3215-3220); only points count as correspondences and the call returns 0 with the pose untouched when fewer
 * than 3 points are matched (:3198-3200).  pslam_translation_pack + pslam_pose_run_packed + pslam_pose_fetch is the split form. */
int pslam_translation_optimization(pslam_ctx* ctx, const pslam_pose_problem* prob, float* Tcw_io, uint8_t* outlier_pt,
                                   uint8_t* outlier_line, uint8_t* outlier_plane);
int pslam_translation_optimization_batch(pslam_ctx* ctx, const pslam_pose_problem* probs, int n, float* Tcw_io, uint8_t* outlier_pt,
                                         uint8_t* outlier_line, uint8_t* outlier_plane, int32_t* n_inliers);
int pslam_translation_pack(pslam_ctx* ctx, const pslam_pose_problem* probs, int n, const float* Tcw0);

/* ---- Local bundle adjustment ---------------------------------------------------------------------
 * Replaces  static void Optimizer::LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap)
 *           include/Optimizer.h:34, src/Optimizer.cc:1853-2678  (graph fill :1971-2358, optimize(5) :2363, chi2 gating
 *           :2373-2455, optimize(10) :2460, erase lists :2462-2560, recovery :2620-2677).
 * The Map / KeyFrame pointer walk that selects local and fixed key frames and collects observations (:1853-1969) stays on
 * the host; it hands over plain arrays (include/pslam_adapter.hpp shows the gathering loop):
 *   key frames  GetPose() (float 4x4 row-major), fixed flag (lFixedCameras, or mnId == 0), fx fy cx cy mbf; vertex order =
 *               array order (g2o orders vertices by id: pass key frames sorted by mnId)
 *   points      GetWorldPos() (float 3); observations (key frame, point, mvKeysUn pt + mvuRight (< 0 => monocular edge
 *               EdgeSE3ProjectXYZ, else EdgeStereoSE3ProjectXYZ), mvInvLevelSigma2[octave])
 *   lines       GetWorldPos() (two endpoints, double 6) -> two VertexSBAPointXYZ; one observation = two EdgeLineProjectXYZ
 *               (start, end) sharing mvKeyLineFunctions (double 3).  The reference attaches every line edge to the CURRENT
 *               key frame pKF (:2169-2201); pass pKF's index in line_obs_kf to reproduce that.
 *   planes      GetWorldPos() (float 4) -> VertexPlane; observations [0] EdgePlane, [1] EdgeVerticalPlane, [2] EdgeParallelPlane
 *               with the key frame's mvPlaneCoefficients (float 4).  The reference adds a plane's vertical / parallel
 *               observations while walking lLocalMapPlanes (:2250-2350): pass them only for planes that are LOCAL (held in
 *               mvpMapPlanes by a local key frame) - the gathering loop of the adapter does exactly that
 *   settings    Plane.AngleInfo, DistanceInfo, Chi, VPChi (vertical / parallel edges use angleInfo like the reference, :2274)
 * Outputs: optimised key-frame poses (fixed ones returned unchanged), point / line / plane positions rounded to float like
 * Converter::toCvMat, and per-observation erase flags = membership of vToErase, vLineToErase, vPlaneToErase,
 * vVerPlaneToErase, vParPlaneToErase.  pbStopFlag is not supported (the result would depend on thread timing).
 * Any output pointer may be NULL.  trace: [0] = optimize(5), [1] = optimize(10). */
typedef struct pslam_lba_problem {
    int32_t n_kf; const float* kf_Tcw /* [n_kf][16] */; const uint8_t* kf_fixed /* [n_kf] */; const float* kf_K /* [n_kf][5] */;
    int32_t n_points; const float* pt_Xw /* [n_points][3] */;
    int32_t n_pt_obs; const int32_t* pt_obs_kf; const int32_t* pt_obs_pt; const float* pt_obs_uvr /* [n][3] */; const float* pt_obs_inv_sigma2;
    int32_t n_lines; const double* line_Xw /* [n_lines][6] */;
    int32_t n_line_obs; const int32_t* line_obs_kf; const int32_t* line_obs_line; const double* line_obs_l /* [n][3] */;
    int32_t n_planes; const float* plane_Xw /* [n_planes][4] */;
    int32_t n_plane_obs[3]; const int32_t* plane_obs_kf[3]; const int32_t* plane_obs_plane[3]; const float* plane_obs_meas[3] /* [n][4] */;
    double angle_info, dist_info, plane_chi, vp_chi;
} pslam_lba_problem;

typedef struct pslam_lba_result {
    float* kf_Tcw /* [n_kf][16] */; double* kf_Tcw_d; float* pt_Xw /* [n_points][3] */; double* pt_Xw_d;
    double* line_Xw /* [n_lines][6], float-rounded */; double* line_Xw_d; float* plane_Xw /* [n_planes][4] */; double* plane_Xw_d;
    uint8_t* erase_pt; uint8_t* erase_line; uint8_t* erase_plane[3];
    int32_t iterations[2], trials[2]; double chi2[2], lambda[2];
} pslam_lba_result;

int pslam_local_bundle_adjustment(pslam_ctx* ctx, const pslam_lba_problem* prob, pslam_lba_result* res);
/* n independent problems (one per key frame of a replayed sequence), one CTA each; res is [n]. */
int pslam_local_bundle_adjustment_batch(pslam_ctx* ctx, const pslam_lba_problem* probs, int n, pslam_lba_result* res);
/* Split form (device-resident problems): pack + upload once, run asynchronously on the context's stream, fetch. */
int pslam_lba_pack(pslam_ctx* ctx, const pslam_lba_problem* probs, int n);
int pslam_lba_run_packed(pslam_ctx* ctx);
int pslam_lba_fetch(pslam_ctx* ctx, pslam_lba_result* res /* [n] */);

/* ---- Line segments ---------------------------------------------------------------------------------
 * Replaces
 *     void LineSegment::ExtractLineSegment(const cv::Mat& img, std::vector<KeyLine>& keylines, cv::Mat& ldesc,
 *                                          std::vector<Eigen::Vector3d>& keylineFunctions, float scale, int numOctaves)
 *     include/LSDextractor.h:349, src/LSDextractor.cpp:13-39  (called from Frame::ExtractLSD, src/Frame.cc:170-179)
 * i.e. LSDDetector::detect (opencv_contrib line_descriptor, one octave) = cv::LineSegmentDetector(LSD_REFINE_ADV) on the
 * input image, the KeyLine records built from the segments, the reference's "sort by response, keep 40, renumber class_id"
 * filter (:18-26) and the line functions sp x ep / |sp x ep| (:30-38).  The LBD descriptors (BinaryDescriptor::compute, :28)
 * come from pslam_lines_extract_describe_batch below (restated from the published algorithm: no upstream implementation is
 * obtainable here to pin them against, SURVEY.md section 8c); the *_extract_* entry points without "describe" stop before them.
 * pslam_keyline has the memory layout of cv::line_descriptor::KeyLine (17 four-byte fields, 68 bytes).
 * refine: 0 = LSD_REFINE_NONE, 1 = LSD_REFINE_STD, 2 = LSD_REFINE_ADV (what the reference runs). */
typedef struct pslam_keyline {
    float angle; int32_t class_id; int32_t octave; float pt_x, pt_y; float response; float size;
    float startPointX, startPointY, endPointX, endPointY, sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
    float lineLength; int32_t numOfPixels;
} pslam_keyline;

int pslam_lsd_max_segments(const pslam_ctx* ctx);     /* segment capacity per frame of the calls below */
/* Which pixels the NFA validation of LSD_REFINE_ADV counts inside a rectangle (LineSegmentDetectorImpl::rect_nfa, OpenCV
 * imgproc lsd.cpp - reached from src/LSDextractor.cpp:16): 1 = OpenCV 4.x's enumeration (DEFAULT; pinned bit for bit against
 * cv2 4.13 in the oracle, DESIGN.md section 5.7), 0 = the published LSD rectangle iterator.  The environment variable
 * PSLAM_LSD_RECT_ENUM=published selects 0 as the default of a new context. */
int pslam_lsd_set_rect_enumeration(pslam_ctx* ctx, int mode);
/* cv::LineSegmentDetector::detect on nframes frames: segs [nframes][cap][4] float (x1 y1 x2 y2), wpn [nframes][cap][3] double
 * (width, precision, log-NFA; -1 unless refine == 2), n [nframes].  PSLAM_E_CAPACITY when a frame has more than cap segments. */
int pslam_lsd_detect_batch(pslam_ctx* ctx, const uint8_t* gray, int nframes, int refine, float* segs, double* wpn, int cap, int32_t* n);
/* The whole  void LineSegment::ExtractLineSegment(const Mat& img, vector<KeyLine>&, Mat& ldesc, vector<Vector3d>& lineFunctions, ...)
 * include/LSDextractor.h:349, src/LSDextractor.cpp:13-39: detector, keep-max_lines filter, LBD descriptors (BinaryDescriptor::compute: desc [nframes][max_lines][32] =
 * the rows of ldesc / Frame::mLdesc; lbd72 [nframes][max_lines][72] optional, the float LBD vectors), line functions.  The LBD logic follows the published
 * algorithm (upstream source absent: parity unpinned, see oracle/lbd.h); its OpenCV primitives are pinned to cv2 4.13. */
int pslam_lines_extract_describe_batch(pslam_ctx* ctx, const uint8_t* gray, int nframes, int max_lines, pslam_keyline* kl, double* line_functions, uint8_t* desc,
                                       float* lbd72 /* may be NULL */, int32_t* n);
int pslam_lines_extract_describe_batch_dev(pslam_ctx* ctx, const uint8_t* d_gray, int nframes, int max_lines, pslam_keyline* d_kl, double* d_line_functions,
                                           uint8_t* d_desc, int32_t* d_n);
/* ExtractLineSegment without descriptors: kl [nframes][max_lines], line_functions [nframes][max_lines][3], n [nframes]. */
int pslam_lines_extract_batch(pslam_ctx* ctx, const uint8_t* gray, int nframes, int max_lines, pslam_keyline* kl, double* line_functions,
                              int32_t* n);
/* Same with device pointers; only enqueues on the context's stream. */
int pslam_lines_extract_batch_dev(pslam_ctx* ctx, const uint8_t* d_gray, int nframes, int max_lines, pslam_keyline* d_kl,
                                  double* d_line_functions, int32_t* d_n);
/* Debug / stage parity (after a detect or extract call): the scaled image [H][W] u8, gradient norm and level-line angle
 * [H][W] double (-1024 = undefined), the seed order (pixel indices y * W + x) and its length.  Any pointer may be NULL. */
int pslam_lsd_debug_stage(pslam_ctx* ctx, int frame, int32_t* dims /* W, H */, uint8_t* scaled, double* modgrad, double* angles,
                          int32_t* order, int32_t* n_order);

/* ---- 3-D lines ---------------------------------------------------------------------------------------
 * Replaces  void Frame::isLineGood(const cv::Mat& imGray, const cv::Mat& imDepth, cv::Mat K)            src/Frame.cc:189-267
 * with      compPt3dCov, extract3dline_mahdist, verify3dLine, mah_dist3d_pt_line, computeLine3d_svd     src/LineExtractor.cpp:1157-1470
 * and       random_unique                                                                               include/LSDextractor.h:239-251
 * Per 2-D line: up to 51 samples along the segment, nearest-pixel depth, back-projection, per-point covariance + cv::SVD, up to 10
 * RANSAC iterations on the Mahalanobis point-line distance, SVD refit, end points, accept test (inliers / length > 0.4, length > 2 cm).
 * Outputs per line what the reference stores: mvLines3D[i] (A, B), mvDepthLine[i], FrameLine::direction and the supporting samples.
 * rand(): the reference draws from the process-wide libc stream; here each frame has its own glibc-compatible stream, started
 * with srand(seed[f]) and advanced by skip[f] draws (skip may be NULL).  n_drawn[f] returns the number of rand() calls the frame
 * made, so a caller that wants the reference's single stream passes seed = its srand seed, skip = draws made so far, and adds
 * n_drawn (large skips cost O(log skip): the generator's recurrence x^31 = x^28 + 1 is jumped, not stepped).  depth: raw uint16 [nframes][height][width]; metres = (float)raw * depth_factor (imDepth.convertTo(CV_32F, factor)).
 * cam: fx, fy, cx, cy (float, as Frame::fx ... are). */
typedef struct pslam_line3d {
    double A[3], B[3];       /* mvLines3D[i]; zero unless valid */
    double director[3];      /* (A - B) / |A - B| of the fitted line (NaN when the fit found no support) */
    uint64_t inliers;        /* bit j: sample j (in sampling order, samples without depth dropped) supports the line */
    float depth;             /* mvDepthLine[i]; -1 unless valid */
    int32_t n_points;        /* samples with depth */
    int32_t n_inliers;       /* RandomLine3d::pts.size() */
    int32_t valid;           /* the accept test of isLineGood passed */
} pslam_line3d;

int pslam_lines3d_batch(pslam_ctx* ctx, const pslam_keyline* keylines /* [nframes][max_lines] */, const int32_t* n_lines /* [nframes] */, int max_lines,
                        const uint16_t* depth, int nframes, float depth_factor, const float* cam /* [4] */, const uint32_t* seed /* [nframes] */,
                        const int32_t* skip /* [nframes] or NULL */, pslam_line3d* out /* [nframes][max_lines] */, int32_t* n_drawn /* [nframes] */);
/* Same with device pointers (cam stays a host pointer); only enqueues on the context's stream - chains after
 * pslam_lines_extract_batch_dev on the key lines it leaves in HBM. */
int pslam_lines3d_batch_dev(pslam_ctx* ctx, const pslam_keyline* d_keylines, const int32_t* d_n_lines, int max_lines, const uint16_t* d_depth, int nframes,
                            float depth_factor, const float* cam, const uint32_t* d_seed, const int32_t* d_skip, pslam_line3d* d_out, int32_t* d_n_drawn);

/* ---- Manhattan frame ---------------------------------------------------------------------------------
 * Replaces  cv::Mat Tracking::TrackManhattanFrame(cv::Mat& mLastRcm, std::vector<SurfaceNormal>&, std::vector<FrameLine>&)   src/Tracking.cc:963-1137
 * with      ProjectSN2Conic :888-961, ProjectSN2MF :763-886, MeanShift :1139-1157.
 * Per axis: surface normals / 3-D line directions inside the cone around the current axis (sin 0.2018 / sin 0.1018), tangent-plane
 * coordinates of those inside sin 0.2518, one Gaussian mean-shift step (c = 20), back-projection; a missing third axis from the cross
 * product; projection onto SO(3) by cv::SVD.  The reference's aliasing of R_cm and R_cm_update (:970) is reproduced (DESIGN.md 5.8).
 * R_last / result R: row-major 3x3 float (the CV_32F cv::Mat).  normals: SurfaceNormal::normal (float x 3, camera frame); dirs:
 * FrameLine::direction (double x 3) of the lines with depth (pslam_line3d.director of the valid lines).
 * Masks (always written): bit a-1 (a = 1..3) - the element was appended to Frame::vSurfaceNormal{x,y,z} / vVanishingLine{x,y,z};
 * bit 3+a - it is inside the first-pass cone of axis a. */
typedef struct pslam_manhattan_result {
    float R[9];                  /* the returned R_cm */
    float density[3];            /* s_j_density per axis, 0 when the axis was not found */
    int32_t found[3];            /* directionFound1..3 */
    int32_t n_cone[3];           /* numInCone */
    int32_t n_selected[3];       /* m_j_selected.size() */
    int32_t min_num;             /* minNumOfSN after the (a+b)/2 fallback */
    int32_t svd_applied;         /* 0: fewer than two directions - the partially updated matrix is returned as the reference does */
} pslam_manhattan_result;

int pslam_track_manhattan_batch(pslam_ctx* ctx, const float* R_last /* [nframes][9] */, const float* normals /* [nframes][max_normals][3] */,
                                const int32_t* n_normals /* [nframes] */, int max_normals, const double* dirs /* [nframes][max_dirs][3] */,
                                const int32_t* n_dirs /* [nframes] */, int max_dirs, int nframes, pslam_manhattan_result* res /* [nframes] */,
                                uint8_t* normal_mask /* [nframes][max_normals] */, uint8_t* dir_mask /* [nframes][max_dirs] */);
/* Same with device pointers; only enqueues on the context's stream. */
int pslam_track_manhattan_batch_dev(pslam_ctx* ctx, const float* d_R_last, const float* d_normals, const int32_t* d_n_normals, int max_normals,
                                    const double* d_dirs, const int32_t* d_n_dirs, int max_dirs, int nframes, pslam_manhattan_result* d_res,
                                    uint8_t* d_normal_mask, uint8_t* d_dir_mask);

/* Replaces the  mCurrentFrame.isInFrustum(pML, 0.6)  pass of Tracking::SearchLocalLines (src/Tracking.cc:2352-2366):
 *           bool Frame::isInFrustum(MapLine* pML, float viewingCosLimit)   src/Frame.cc:369-437
 *           int MapLine::PredictScale(const float&, const float&)          src/MapLine.cpp:381-390 (no clamping)
 * for n map lines: pos [n][6] = GetWorldPos() (start, end), normal [n][3] = GetNormal(), max_distance / min_distance = mfMaxDistance /
 * mfMinDistance (the 1.2 / 0.8 factors of Get*DistanceInvariance are applied here).  Outputs the fields the function writes into the
 * MapLine: in_view = mbTrackInView, proj [n][4] = mTrackProjX1, Y1, X2, Y2, level = mnTrackScaleLevel, view_cos = mTrackViewCos (zero when
 * not in view) - exactly the inputs of pslam_line_search_by_projection below.  Returns the number of lines in view (nToMatch). */
typedef struct pslam_line_frustum_frame {
    float Tcw[16];                                   /* mTcw, row-major */
    float fx, fy, cx, cy, min_x, max_x, min_y, max_y;  /* Frame::fx.., mnMinX..mnMaxY */
    float log_scale_factor;                          /* mfLogScaleFactor */
} pslam_line_frustum_frame;
int pslam_lines_in_frustum(pslam_ctx* ctx, const pslam_line_frustum_frame* frame, int n, const double* pos, const double* normal, const float* max_distance,
                           const float* min_distance, float cos_limit, uint8_t* in_view, float* proj, int32_t* level, float* view_cos);

/* Replaces  int LSDmatcher::SearchByProjection(Frame& F, const std::vector<MapLine*>& vpMapLines, float th)
 *           include/LSDmatcher.h:24, src/LSDmatcher.cpp:141-211 (+ Frame::GetLinesInArea src/Frame.cc:491-523).
 * Frame side: KeyLine pt / angle / octave and the LBD rows of the <= 64 frame lines, has_obs[i] = (mvpMapLines[i] &&
 * mvpMapLines[i]->Observations() > 0) on entry, mvScaleFactors.  Map side, one entry per element of vpMapLines: skip (null /
 * isBad() / !mbTrackInView), mnTrackScaleLevel, mTrackViewCos, mTrackProjX1 Y1 X2 Y2, GetDescriptor(), Observations() > 0.
 * assigned[i] = index of the map line the call stores into F.mvpMapLines[i], -1 where it leaves the entry alone.
 * A predicted level outside [0, n_levels) - MapLine::PredictScale does not clamp, so pslam_lines_in_frustum produces them for lines seen
 * from close by - is accepted: the radius uses scale_factors[clamp(level)] (the reference reads past mvScaleFactors there, undefined
 * behaviour), the octave gate uses the raw level like the reference.
 * Returns nmatches (>= 0) or a negative pslam_status. */
int pslam_line_search_by_projection(pslam_ctx* ctx, int n_frame_lines, const float* pt, const float* angle, const int32_t* octave, const uint8_t* desc,
                                    const uint8_t* has_obs, const float* scale_factors, int n_levels, int n_map_lines, const uint8_t* skip,
                                    const int32_t* level, const float* view_cos, const float* proj, const uint8_t* map_desc,
                                    const uint8_t* map_has_obs, float th, float nnratio, int32_t* assigned);

/* Replaces  int ORBmatcher::SearchByBoW(KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches)
 *           include/ORBmatcher.h:53, src/ORBmatcher.cc:160-292.
 * Both sides: ORB descriptors [n][32], key-point angles (key frame: mvKeysUn, frame: mvKeys) and the DBoW2 FeatureVector as CSR
 * (node ids ascending like the std::map, offsets, feature indices in insertion order); kf_has_mp[i] = the key frame's
 * map point i exists and is not bad.  The DBoW2 transform that builds the feature vectors stays on the host (SURVEY.md 8 f2).
 * match[j] = key-frame feature whose map point the call stores into vpMapPointMatches[j] (-1: NULL).  Returns nmatches. */
int pslam_search_by_bow(pslam_ctx* ctx, int n_kf, const uint8_t* kf_desc, const float* kf_angle, const uint8_t* kf_has_mp, int kf_nodes,
                        const int32_t* kf_node_id, const int32_t* kf_node_off, const int32_t* kf_node_feat, int n_f, const uint8_t* f_desc,
                        const float* f_angle, int f_nodes, const int32_t* f_node_id, const int32_t* f_node_off, const int32_t* f_node_feat,
                        float nnratio, int check_orientation, int32_t* match);

/* Replaces  int ORBmatcher::SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12)
 *           include/ORBmatcher.h:56, src/ORBmatcher.cc:526-659 - the loop-closure matcher (LoopClosing::ComputeSim3, src/LoopClosing.cc:265), the consumer
 *           of the key-frame descriptor exchange (SURVEY.md 8 f3).
 * Same array layout as pslam_search_by_bow, both sides with map-point flags (has_mp[i] = vpMapPoints[i] && !isBad()); the distance gate is the
 * strict bestDist1 < TH_LOW of this overload.  match12[i1] = feature of key frame 2 whose map point the call stores into vpMatches12[i1] (-1: NULL).
 * Returns nmatches (>= 0) or a negative pslam_status. */
int pslam_search_by_bow_kf(pslam_ctx* ctx, int n1, const uint8_t* desc1, const float* angle1, const uint8_t* has_mp1, int nodes1, const int32_t* node_id1,
                           const int32_t* node_off1, const int32_t* node_feat1, int n2, const uint8_t* desc2, const float* angle2, const uint8_t* has_mp2,
                           int nodes2, const int32_t* node_id2, const int32_t* node_off2, const int32_t* node_feat2, float nnratio, int check_orientation,
                           int32_t* match12);

/* The key-frame database of KeyFrameDatabase (include/KeyFrameDatabase.h:43-75) as the candidate searches read it: the BowVectors of the key frames in the
 * order KeyFrameDatabase::add saw them (src/KeyFrameDatabase.cc:38-44; an erased key frame is simply left out), CSR with strictly ascending word ids per
 * key frame (std::map order).  Uploaded once and kept in HBM by the context; a second call replaces it, n_kf = 0 releases it. */
int pslam_bow_database_set(pslam_ctx* ctx, int n_kf, const int32_t* kf_off, const int32_t* kf_word, const double* kf_val);

/* Replaces  std::vector<KeyFrame*> KeyFrameDatabase::DetectLoopCandidates(KeyFrame* pKF, float minScore)
 *           include/KeyFrameDatabase.h:58, src/KeyFrameDatabase.cc:76-197 with DBoW2's L1 score (Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68).
 * Query = pKF->mBowVec (n_q words ascending + values).  covis[k][covis_stride] = KeyFrame::GetBestCovisibilityKeyFrames(10) of database key frame k as
 * database indices, -1 ends a row; connected[k] != 0: key frame k is in pKF->GetConnectedKeyFrames() (NULL: none).  candidates (capacity n_kf) receives
 * vpLoopCandidates as database indices in the reference's order.  Optional outputs, n_kf entries each: common_words[k] = mnLoopWords after the call,
 * score[k] = mLoopScore where the reference evaluates it (entries of other key frames are left untouched).
 * Not reproduced: a query key frame with mnId 0 finds nothing in the reference (mnLoopQuery starts at 0); LoopClosing never queries that key frame.
 * Returns the number of candidates (>= 0) or a negative pslam_status. */
int pslam_detect_loop_candidates(pslam_ctx* ctx, int n_q, const int32_t* q_word, const double* q_val, const int32_t* covis, int covis_stride,
                                 const uint8_t* connected, float min_score, int32_t* candidates, int32_t* common_words, float* score);

/* Replaces  std::vector<KeyFrame*> KeyFrameDatabase::DetectRelocalizationCandidates(Frame* F)   include/KeyFrameDatabase.h:61, src/KeyFrameDatabase.cc:199-305.
 * reloc_score_io[k] = KeyFrame::mRelocScore of database key frame k: the reference adds a covisible neighbour's mRelocScore whenever that neighbour shares a
 * word with the frame, also when it did not evaluate the score for this frame - the value an earlier query left (the constructor does not initialise it;
 * pass zeros for a fresh database).  Updated in place like the reference updates the key frames. */
int pslam_detect_relocalization_candidates(pslam_ctx* ctx, int n_q, const int32_t* q_word, const double* q_val, const int32_t* covis, int covis_stride,
                                           float* reloc_score_io, int32_t* candidates, int32_t* common_words);

/* Replaces  DBoW2::TemplatedVocabulary<FORB::TDescriptor, FORB>::transform(features, BowVector&, FeatureVector&, levelsup)
 *           Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1125-1252, called by Frame::ComputeBoW / KeyFrame::ComputeBoW
 *           (src/KeyFrame.cc:66-76: mpORBvocabulary->transform(vCurrentDesc, mBowVec, mFeatVec, 4); TF_IDF weights, L1 norm).
 * Vocabulary as flat arrays in DBoW2's node-id order: 32-byte node descriptors, children as CSR, word id and weight per node
 * (leaves).  Outputs (caller-allocated, n entries each, node_off n + 1): BowVector as (word_id ascending, value) pairs and the
 * FeatureVector as CSR (node_id ascending, node_off, node_feat in insertion order); counts[0] = words, counts[1] = nodes. */
int pslam_bow_transform(pslam_ctx* ctx, int n_nodes, int L, const uint8_t* voc_desc, const int32_t* child_off, const int32_t* child_id,
                        const int32_t* voc_word_id, const double* voc_weight, const uint8_t* features, int n, int levelsup, int32_t* word_id,
                        double* word_val, int32_t* node_id, int32_t* node_off, int32_t* node_feat, int32_t* counts);

/* The vocabulary for the batched transform, uploaded once (ORBvoc.txt is loaded once at System construction, src/System.cc:44) and kept in HBM by
 * the context: the same flat arrays as pslam_bow_transform in DBoW2's node-id order, child_off[0] = 0, every child id larger than its parent's.
 * A second call replaces it, n_nodes = 0 releases it.  PSLAM_E_INVALID if a node has more than 32 children.  pslam_bow_transform does not use it. */
int pslam_bow_set_vocabulary(pslam_ctx* ctx, int n_nodes, int L, const uint8_t* voc_desc, const int32_t* child_off, const int32_t* child_id,
                             const int32_t* voc_word_id, const double* voc_weight);
/* Frame::ComputeBoW / KeyFrame::ComputeBoW (transform(desc, mBowVec, mFeatVec, levelsup)) for nframes frames against the resident vocabulary;
 * PSLAM_E_INVALID if none is set.  desc [nframes][cap][32] with n[f] valid rows (the layout pslam_orb_extract_batch writes), 1 <= cap <= 3072.
 * Outputs per frame f, each [nframes][cap] (node_off [nframes][cap + 1]): word_id / word_val (BowVector, word ascending), node_id / node_off /
 * node_feat (FeatureVector CSR, node ascending, features in insertion order); counts [nframes][2] = words, nodes.  Bytes equal pslam_bow_transform's.
 * The batch size is not bounded by max_batch; device scratch belongs to the context and only grows. */
int pslam_bow_transform_batch(pslam_ctx* ctx, const uint8_t* desc, const int32_t* n, int cap, int nframes, int levelsup, int32_t* word_id,
                              double* word_val, int32_t* node_id, int32_t* node_off, int32_t* node_feat, int32_t* counts);
/* Same with device pointers (d_desc 16-byte aligned; a row count outside [0, cap] is clamped to it); only enqueues on the context's stream
 * (chains after pslam_orb_extract_batch_dev). */
int pslam_bow_transform_batch_dev(pslam_ctx* ctx, const uint8_t* d_desc, const int32_t* d_n, int cap, int nframes, int levelsup, int32_t* d_word_id,
                                  double* d_word_val, int32_t* d_node_id, int32_t* d_node_off, int32_t* d_node_feat, int32_t* d_counts);

/* ---- The RGB-D Frame constructor's compute in one call ----------------------------------------------------
 * Replaces the work of  Frame::Frame(imRGB, imGray, imDepth, ...)   src/Frame.cc:55-140 : the three extractor threads it starts (:90-95)
 *   ExtractORB (:181-186)  then  ComputeStereoFromRGBD (:603-621)            -> mvKeys (= mvKeysUn: no distortion model on this path), mDescriptors, mvuRight, mvDepth
 *   ExtractLSD (:170-179): ExtractLineSegment + LBD, isLineGood (:189-267)   -> mvKeylinesUn, mvKeyLineFunctions, mLdesc, mvLines3D / mvDepthLine
 *   ComputePlanes (:647-753)                                                 -> mvPlaneCoefficients, mvPlanePoints, vSurfaceNormal
 * for nframes frames.  gray uint8 [nframes][h][w] and depth uint16 [nframes][h][w] are host buffers and are uploaded ONCE (the per-function host-pointer
 * entry points above upload the depth frame three times and the gray frame twice); all outputs are host buffers:
 *   keys [nframes][capk], desc [nframes][capk][32], n_keys [nframes], u_right / depth_kp [nframes][capk]      capk = pslam_orb_max_keypoints()
 *   keylines [nframes][max_lines], line_functions [nframes][max_lines][3], line_desc [nframes][max_lines][32], lines3d [nframes][max_lines], n_lines [nframes],
 *   n_rand_drawn [nframes] (may be NULL; see pslam_lines3d_batch: every frame's rand() stream starts from line_seed)
 *   n_planes [nframes], plane_src / plane_coef [nframes][maxp] ([4]), plane_pt_off [nframes][maxp + 1], plane_pts [nframes][cap_plane_pts][3]   maxp = pslam_peac_max_planes()
 *   surface_normals8 [nframes][pslam_surface_normals_count()][8] (may be NULL: the normals are then not computed)
 * Pinned (page-locked) buffers make the copies asynchronous to the host; two contexts driven from two host threads overlap one batch's copies with the
 * other's kernels.  Device staging belongs to the context and only grows.  PSLAM_E_CAPACITY like the per-function calls. */
typedef struct pslam_frame_outputs {
    pslam_keypoint* keys; uint8_t* desc; int32_t* n_keys; float* u_right; float* depth_kp;
    pslam_keyline* keylines; double* line_functions; uint8_t* line_desc; struct pslam_line3d* lines3d; int32_t* n_lines; int32_t* n_rand_drawn;
    int32_t* n_planes; int32_t* plane_src; float* plane_coef; int32_t* plane_pt_off; float* plane_pts; int32_t cap_plane_pts;
    float* surface_normals8;
} pslam_frame_outputs;
int pslam_frame_construct_batch(pslam_ctx* ctx, const uint8_t* gray, const uint16_t* depth, int nframes, float depth_factor, float bf, float plane_dist_th,
                                int max_lines, uint32_t line_seed, const pslam_frame_outputs* out);

#ifdef __cplusplus
}
#endif
#endif /* PSLAM_ABI_H_ */
