// The compute of the RGB-D Frame constructor (src/Frame.cc:55-140) as ONE host-pointer call: the gray and depth frames are uploaded once and the three
// extractor chains the constructor starts as threads - ExtractORB (:181-186) followed by ComputeStereoFromRGBD (:603-621), ExtractLSD (:170-179: line segments,
// LBD descriptors, isLineGood), ComputePlanes (:647-753: PEAC, plane post-processing, surface normals) - run back to back on the context's stream over the
// resident frames; every product the constructor leaves in the Frame is copied back.  (Calling the per-function host-pointer entry points instead uploads the
// depth frame three times and the gray frame twice.)  Device staging is owned by the context and only grows.
// Copies and kernels of one call overlap: the depth frames go up first and ComputePlanes starts on them while the gray frames are still arriving on a second
// (copy) stream; the plane products - three quarters of the bytes that go back, surface normals mostly - return on that stream while ExtractORB / ExtractLSD
// run.  Only the depth upload and the ORB / line products at the end are exposed (page-locked host buffers assumed; pageable ones work, serialised).
// pslam_frame_construct_batch_dev runs the same three chains (compute_planes, extract_orb, extract_lines below) on frames the caller already holds in HBM and
// writes the products into the caller's device buffers; the capacity flags the host call reads back are folded into one status word per frame on the device.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "pslam_internal.h"

namespace pslam {

struct FrameBuffers {
    DevArray<uint8_t> slab;        // carved up per call
    DevArray<uint8_t> dev_slab;    // scratch of pslam_frame_construct_batch_dev (no outputs, no frames: those are the caller's)
    PinnedArray<int32_t> h_status;
    cudaStream_t copy = nullptr;   // second stream: gray upload / plane-product download next to the kernels
    cudaEvent_t ev_gray = nullptr, ev_planes = nullptr, ev_idle = nullptr;
};

void frame_free(pslam_ctx* c) {
    if (!c->frame) return;
    if (c->frame->copy) cudaStreamDestroy(c->frame->copy);
    for (cudaEvent_t e : {c->frame->ev_gray, c->frame->ev_planes, c->frame->ev_idle}) if (e) cudaEventDestroy(e);
    delete c->frame;
    c->frame = nullptr;
}

// Device buffers of one call that are not outputs: PEAC's label image, planes and member lists, the plane post-processing flags, the rand() seeds
struct FrameScratch {
    int32_t* labels; pslam_plane* planes; int32_t* npl; int32_t* members; int32_t* moff; int32_t* ppst; uint32_t* seed;
    const int32_t* skip;      // rand() draws to skip per frame after srand(seed), or NULL (every frame starts at its seed)
};

constexpr int kPlanePtsOverflow = 32 | 64;      // plane post-processing flags that mean "more voxels than the capacity"

// The three extractor chains of the constructor on device-resident frames, enqueued on the context's stream; o holds device pointers.
// ComputePlanes (:647-753): PEAC, plane post-processing, surface normals (when o.surface_normals8 is set).  Leaves PEAC's capacity flags in c->d_status.
static int compute_planes(pslam_ctx* c, const uint16_t* depth, int nframes, float plane_dist_th, const pslam_frame_outputs& o, const FrameScratch& s) {
    int rc;
    if ((rc = pslam_peac_run_batch_dev(c, depth, nframes, s.labels, s.planes, s.npl, s.members, s.moff)) != PSLAM_OK) return rc;
    if ((rc = pslam_planes_post_batch_dev(c, depth, nframes, s.planes, s.npl, s.members, s.moff, plane_dist_th, o.n_planes, o.plane_src, o.plane_coef, o.plane_pt_off,
                                          o.plane_pts, o.cap_plane_pts, s.ppst)) != PSLAM_OK) return rc;
    if (o.surface_normals8 && (rc = pslam_surface_normals_batch_dev(c, depth, nframes, o.surface_normals8, nullptr)) != PSLAM_OK) return rc;
    return PSLAM_OK;
}

// ExtractORB, then ComputeStereoFromRGBD on the key points it leaves in HBM (no distortion model on this path: mvKeysUn = mvKeys, Frame::UndistortKeyPoints
// :545-549).  Leaves ORB's capacity flags in c->d_status.
static int extract_orb(pslam_ctx* c, const uint8_t* gray, const uint16_t* depth, int nframes, float depth_factor, float bf, const pslam_frame_outputs& o) {
    const int cap = pslam_orb_max_keypoints(c);
    int rc;
    if ((rc = pslam_orb_extract_batch_dev(c, gray, nframes, o.keys, o.desc, cap, o.n_keys)) != PSLAM_OK) return rc;
    return pslam_compute_stereo_from_rgbd_batch_dev(c, o.keys, o.keys, o.n_keys, cap, depth, nframes, depth_factor, bf, o.u_right, o.depth_kp);
}

// ExtractLSD: segments -> key lines + line functions + LBD descriptors, then isLineGood (o.n_rand_drawn must be set)
static int extract_lines(pslam_ctx* c, const uint8_t* gray, const uint16_t* depth, int nframes, float depth_factor, int max_lines, const pslam_frame_outputs& o,
                         const FrameScratch& s) {
    const float cam[4] = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    int rc;
    if ((rc = pslam_lines_extract_describe_batch_dev(c, gray, nframes, max_lines, o.keylines, o.line_functions, o.line_desc, o.n_lines)) != PSLAM_OK) return rc;
    return pslam_lines3d_batch_dev(c, o.keylines, o.n_lines, max_lines, depth, nframes, depth_factor, cam, s.seed, s.skip, o.lines3d, o.n_rand_drawn);
}

__global__ void k_frame_seeds(uint32_t* seed, int nframes, uint32_t v) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < nframes) seed[f] = v;
}

// status[f] holds PEAC's flags on entry; the PSLAM_FRAME_CAP_* word on exit (the conditions pslam_frame_construct_batch turns into PSLAM_E_CAPACITY)
__global__ void k_frame_status(int32_t* status, int nframes, const int32_t* orb, const int32_t* n_keys, int cap, const int32_t* lines, const int32_t* ppst) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    status[f] = (orb[f] || n_keys[f] > cap ? PSLAM_FRAME_CAP_ORB : 0) | (status[f] ? PSLAM_FRAME_CAP_PEAC : 0) | (lines[f] ? PSLAM_FRAME_CAP_LINES : 0) |
                (ppst[f] & kPlanePtsOverflow ? PSLAM_FRAME_CAP_PLANE_PTS : 0);
}

}  // namespace pslam

using namespace pslam;

namespace {

// pslam_frame_construct_batch and pslam_frame_construct_batch_ex: image is grey (channels 1) or colour (3 / 4, converted on the device after its upload),
// line_skip is NULL or the per-frame rand() draws to skip.  With channels 1 and no skip the launches and copies are those of pslam_frame_construct_batch.
int construct_host(pslam_ctx* c, const uint8_t* image, int channels, int rgb, const uint16_t* depth, int nframes, float depth_factor, float bf,
                   float plane_dist_th, int max_lines, uint32_t line_seed, const int32_t* line_skip, const pslam_frame_outputs* out) {
    if (!c) return PSLAM_E_INVALID;
    if (!image || !depth || !out || nframes < 1 || nframes > c->cfg.max_batch || max_lines < 1) return set_error(c, PSLAM_E_INVALID, "frame construct: bad arguments");
    if (channels != 1 && channels != 3 && channels != 4) return set_error(c, PSLAM_E_INVALID, "frame construct: channels must be 1, 3 or 4");
    const int cap = pslam_orb_max_keypoints(c), maxp = pslam_peac_max_planes(c), n_sn = pslam_surface_normals_count(c);
    if (!out->keys || !out->desc || !out->n_keys || !out->u_right || !out->depth_kp || !out->keylines || !out->line_functions || !out->line_desc || !out->lines3d ||
        !out->n_lines || !out->n_planes || !out->plane_src || !out->plane_coef || !out->plane_pt_off || !out->plane_pts || out->cap_plane_pts < 1)
        return set_error(c, PSLAM_E_INVALID, "frame construct: null output pointer");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->frame) c->frame = new FrameBuffers();
    FrameBuffers& B = *c->frame;
    const size_t npx = (size_t)c->cfg.width * c->cfg.height, nf = (size_t)nframes, ml = (size_t)max_lines, cp = (size_t)out->cap_plane_pts;
    Slab s;
    const auto gray_d = s.add<uint8_t>(nf * npx);
    const auto depth_d = s.add<uint16_t>(nf * npx);
    const auto kps = s.add<pslam_keypoint>(nf * cap);
    const auto desc = s.add<uint8_t>(nf * cap * 32);
    const auto nk = s.add<int32_t>(nf);
    const auto ur = s.add<float>(nf * cap), dz = s.add<float>(nf * cap);
    const auto kl = s.add<pslam_keyline>(nf * ml);
    const auto lf = s.add<double>(nf * ml * 3);
    const auto ldesc = s.add<uint8_t>(nf * ml * 32);
    const auto l3d = s.add<pslam_line3d>(nf * ml);
    const auto nkl = s.add<int32_t>(nf);
    const auto seed = s.add<uint32_t>(nf);
    const auto drawn = s.add<int32_t>(nf), labels = s.add<int32_t>(nf * npx);
    const auto planes = s.add<pslam_plane>(nf * maxp);
    const auto npl = s.add<int32_t>(nf), members = s.add<int32_t>(nf * npx), moff = s.add<int32_t>(nf * (maxp + 1)), ppn = s.add<int32_t>(nf), ppsrc = s.add<int32_t>(nf * maxp);
    const auto ppcoef = s.add<float>(nf * maxp * 4);
    const auto ppoff = s.add<int32_t>(nf * (maxp + 1));
    const auto pppts = s.add<float>(nf * cp * 3);
    const auto ppst = s.add<int32_t>(nf);
    const auto sn8 = s.add<float>(out->surface_normals8 ? nf * n_sn * 8 : 0);
    const auto color_d = s.add<uint8_t>(channels != 1 ? nf * npx * channels : 0);     // empty for grey input and no skips: the slab is unchanged
    const auto skip_d = s.add<int32_t>(line_skip ? nf : 0);
    int rc;
    if (s.bytes() > B.slab.cap) PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));      // an earlier call's kernels may still read the old slab
    if ((rc = s.alloc(c, B.slab)) || (rc = B.h_status.reserve(c, nf * 4))) return rc;
    if (!B.copy) {
        PSLAM_CUDA(c, cudaStreamCreateWithFlags(&B.copy, cudaStreamNonBlocking));
        PSLAM_CUDA(c, cudaEventCreateWithFlags(&B.ev_gray, cudaEventDisableTiming));
        PSLAM_CUDA(c, cudaEventCreateWithFlags(&B.ev_planes, cudaEventDisableTiming));
        PSLAM_CUDA(c, cudaEventCreateWithFlags(&B.ev_idle, cudaEventDisableTiming));
    }
    cudaStream_t st = c->stream, cs = B.copy;
    // the copy stream starts after whatever the context's stream still holds (an earlier call's kernels may read the slab)
    PSLAM_CUDA(c, cudaEventRecord(B.ev_idle, st));
    PSLAM_CUDA(c, cudaStreamWaitEvent(cs, B.ev_idle, 0));
    s.up(depth_d, depth, st);
    if (channels == 1) s.up(gray_d, image, cs);
    else s.up(color_d, image, cs);
    PSLAM_CUDA(c, cudaEventRecord(B.ev_gray, cs));
    if (line_skip) s.up(skip_d, line_skip, st);
    {   // one rand() stream per frame, all started from the caller's seed (pslam_lines3d_batch documents the single-stream alternative)
        for (int f = 0; f < nframes; ++f) B.h_status[f] = (int32_t)line_seed;
        s.up(seed, reinterpret_cast<const uint32_t*>(B.h_status.ptr), st);
    }
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    pslam_frame_outputs dv = {s[kps], s[desc], s[nk], s[ur], s[dz], s[kl], s[lf], s[ldesc], s[l3d], s[nkl], s[drawn],
                              s[ppn], s[ppsrc], s[ppcoef], s[ppoff], s[pppts], out->cap_plane_pts, out->surface_normals8 ? s[sn8] : nullptr};
    const FrameScratch sc{s[labels], s[planes], s[npl], s[members], s[moff], s[ppst], s[seed], line_skip ? s[skip_d] : nullptr};
    // ComputePlanes on the depth frames while the gray frames arrive
    if ((rc = compute_planes(c, s[depth_d], nframes, plane_dist_th, dv, sc)) != PSLAM_OK) return rc;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_status + 2 * (size_t)nframes, c->d_status, nf * 4, cudaMemcpyDeviceToHost, st));      // PEAC capacity flags (ORB reuses the array below)
    PSLAM_CUDA(c, cudaEventRecord(B.ev_planes, st));
    // the plane products return on the copy stream while the two image chains run
    PSLAM_CUDA(c, cudaStreamWaitEvent(cs, B.ev_planes, 0));
    s.down(out->n_planes, ppn, cs); s.down(out->plane_src, ppsrc, cs); s.down(out->plane_coef, ppcoef, cs); s.down(out->plane_pt_off, ppoff, cs); s.down(out->plane_pts, pppts, cs);
    if (out->surface_normals8) s.down(out->surface_normals8, sn8, cs);
    s.down(B.h_status + nframes, ppst, cs);        // plane post-processing capacity flags
    PSLAM_CUDA(c, cudaStreamWaitEvent(st, B.ev_gray, 0));
    if (channels != 1 && (rc = pslam_gray_from_color_batch_dev(c, s[color_d], channels, rgb, nframes, s[gray_d])) != PSLAM_OK) return rc;   // GrabImageRGBD's cvtColor
    if ((rc = extract_orb(c, s[gray_d], s[depth_d], nframes, depth_factor, bf, dv)) != PSLAM_OK) return rc;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_status, c->d_status, nf * 4, cudaMemcpyDeviceToHost, st));                            // ORB capacity flags
    s.down(out->keys, kps, st); s.down(out->desc, desc, st); s.down(out->n_keys, nk, st); s.down(out->u_right, ur, st); s.down(out->depth_kp, dz, st);
    if ((rc = extract_lines(c, s[gray_d], s[depth_d], nframes, depth_factor, max_lines, dv, sc)) != PSLAM_OK) return rc;
    if ((rc = lsd_status_fetch_async(c, nframes, B.h_status + 3 * (size_t)nframes)) != PSLAM_OK) return rc;
    s.down(out->keylines, kl, st); s.down(out->line_functions, lf, st); s.down(out->line_desc, ldesc, st); s.down(out->lines3d, l3d, st); s.down(out->n_lines, nkl, st);
    if (out->n_rand_drawn) s.down(out->n_rand_drawn, drawn, st);
    PSLAM_CUDA(c, cudaStreamSynchronize(cs));
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    for (int f = 0; f < nframes; ++f) {
        if (B.h_status[nframes + f] & kPlanePtsOverflow) return set_error(c, PSLAM_E_CAPACITY, "frame construct: more voxels than the plane post-processing capacity");
        if (out->n_keys[f] > cap || B.h_status[f]) return set_error(c, PSLAM_E_CAPACITY, "frame construct: ORB candidate / key point capacity exceeded");
        if (B.h_status[2 * (size_t)nframes + f]) return set_error(c, PSLAM_E_CAPACITY, "frame construct: PEAC capacity exceeded (planes / region-growing queue)");
        if (B.h_status[3 * (size_t)nframes + f]) return set_error(c, PSLAM_E_CAPACITY, "frame construct: more line segments than the internal capacity");
    }
    return PSLAM_OK;
}

}  // namespace

extern "C" {

int pslam_frame_construct_batch(pslam_ctx* c, const uint8_t* gray, const uint16_t* depth, int nframes, float depth_factor, float bf, float plane_dist_th,
                                int max_lines, uint32_t line_seed, const pslam_frame_outputs* out) {
    return construct_host(c, gray, 1, 0, depth, nframes, depth_factor, bf, plane_dist_th, max_lines, line_seed, nullptr, out);
}

int pslam_frame_construct_batch_ex(pslam_ctx* c, const uint8_t* image, int channels, int rgb, const uint16_t* depth, int nframes, float depth_factor, float bf,
                                   float plane_dist_th, int max_lines, uint32_t line_seed, const int32_t* line_skip, const pslam_frame_outputs* out) {
    return construct_host(c, image, channels, rgb, depth, nframes, depth_factor, bf, plane_dist_th, max_lines, line_seed, line_skip, out);
}

int pslam_frame_construct_batch_dev(pslam_ctx* c, const uint8_t* d_gray, const uint16_t* d_depth, int nframes, float depth_factor, float bf, float plane_dist_th,
                                    int max_lines, uint32_t line_seed, const pslam_frame_outputs* d_out, int32_t* d_status) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_gray || !d_depth || !d_out || !d_status || nframes < 1 || nframes > c->cfg.max_batch || max_lines < 1)
        return set_error(c, PSLAM_E_INVALID, "frame construct dev: bad arguments");
    if (!d_out->keys || !d_out->desc || !d_out->n_keys || !d_out->u_right || !d_out->depth_kp || !d_out->keylines || !d_out->line_functions || !d_out->line_desc || !d_out->lines3d ||
        !d_out->n_lines || !d_out->n_planes || !d_out->plane_src || !d_out->plane_coef || !d_out->plane_pt_off || !d_out->plane_pts || d_out->cap_plane_pts < 1)
        return set_error(c, PSLAM_E_INVALID, "frame construct dev: null output pointer");
    if (((uintptr_t)d_gray | (uintptr_t)d_depth) & 3) return set_error(c, PSLAM_E_INVALID, "frame construct dev: frame pointers must be 4-byte aligned");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->frame) c->frame = new FrameBuffers();
    FrameBuffers& B = *c->frame;
    const size_t npx = (size_t)c->cfg.width * c->cfg.height, nf = (size_t)nframes, maxp = (size_t)pslam_peac_max_planes(c);
    Slab s;
    const auto labels = s.add<int32_t>(nf * npx), members = s.add<int32_t>(nf * npx);
    const auto planes = s.add<pslam_plane>(nf * maxp);
    const auto npl = s.add<int32_t>(nf), moff = s.add<int32_t>(nf * (maxp + 1)), ppst = s.add<int32_t>(nf), drawn = s.add<int32_t>(nf);
    const auto seed = s.add<uint32_t>(nf);
    int rc;
    if (s.bytes() > B.dev_slab.cap) PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));      // an earlier call's kernels may still read the old scratch
    if ((rc = s.alloc(c, B.dev_slab)) != PSLAM_OK) return rc;
    pslam_frame_outputs o = *d_out;
    if (!o.n_rand_drawn) o.n_rand_drawn = s[drawn];
    const FrameScratch sc{s[labels], s[planes], s[npl], s[members], s[moff], s[ppst], s[seed], nullptr};
    cudaStream_t st = c->stream;
    const unsigned fb = (unsigned)((nframes + 127) / 128);
    PSLAM_LAUNCH(c, "frame_seeds", k_frame_seeds<<<fb, 128, 0, st>>>(sc.seed, nframes, line_seed));
    if ((rc = compute_planes(c, d_depth, nframes, plane_dist_th, o, sc)) != PSLAM_OK) return rc;
    PSLAM_CUDA(c, cudaMemcpyAsync(d_status, c->d_status, nf * 4, cudaMemcpyDeviceToDevice, st));      // PEAC capacity flags (ORB reuses c->d_status)
    if ((rc = extract_orb(c, d_gray, d_depth, nframes, depth_factor, bf, o)) != PSLAM_OK) return rc;
    if ((rc = extract_lines(c, d_gray, d_depth, nframes, depth_factor, max_lines, o, sc)) != PSLAM_OK) return rc;
    PSLAM_LAUNCH(c, "frame_status", k_frame_status<<<fb, 128, 0, st>>>(d_status, nframes, c->d_status, o.n_keys, pslam_orb_max_keypoints(c), lsd_status_dev(c), sc.ppst));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

}  // extern "C"
