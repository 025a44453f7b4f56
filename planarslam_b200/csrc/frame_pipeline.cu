// The compute of the RGB-D Frame constructor (src/Frame.cc:55-140) as ONE host-pointer call: the gray and depth frames are uploaded once and the three
// extractor chains the constructor starts as threads - ExtractORB (:181-186) followed by ComputeStereoFromRGBD (:603-621), ExtractLSD (:170-179: line segments,
// LBD descriptors, isLineGood), ComputePlanes (:647-753: PEAC, plane post-processing, surface normals) - run back to back on the context's stream over the
// resident frames; every product the constructor leaves in the Frame is copied back.  (Calling the per-function host-pointer entry points instead uploads the
// depth frame three times and the gray frame twice.)  Device staging is owned by the context and only grows.
// Copies and kernels of one call overlap: the depth frames go up first and ComputePlanes starts on them while the gray frames are still arriving on a second
// (copy) stream; the plane products - three quarters of the bytes that go back, surface normals mostly - return on that stream while ExtractORB / ExtractLSD
// run.  Only the depth upload and the ORB / line products at the end are exposed (page-locked host buffers assumed; pageable ones work, serialised).
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "pslam_internal.h"

namespace pslam {

struct FrameBuffers {
    DevArray<uint8_t> slab;        // carved up per call
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

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_frame_construct_batch(pslam_ctx* c, const uint8_t* gray, const uint16_t* depth, int nframes, float depth_factor, float bf, float plane_dist_th,
                                int max_lines, uint32_t line_seed, const pslam_frame_outputs* out) {
    if (!c) return PSLAM_E_INVALID;
    if (!gray || !depth || !out || nframes < 1 || nframes > c->cfg.max_batch || max_lines < 1) return set_error(c, PSLAM_E_INVALID, "frame construct: bad arguments");
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
    s.up(gray_d, gray, cs);
    PSLAM_CUDA(c, cudaEventRecord(B.ev_gray, cs));
    {   // one rand() stream per frame, all started from the caller's seed (pslam_lines3d_batch documents the single-stream alternative)
        for (int f = 0; f < nframes; ++f) B.h_status[f] = (int32_t)line_seed;
        s.up(seed, reinterpret_cast<const uint32_t*>(B.h_status.ptr), st);
    }
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    const float cam[4] = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    // ComputePlanes on the depth frames while the gray frames arrive
    if ((rc = pslam_peac_run_batch_dev(c, s[depth_d], nframes, s[labels], s[planes], s[npl], s[members], s[moff])) != PSLAM_OK)
        return rc;
    if ((rc = pslam_planes_post_batch_dev(c, s[depth_d], nframes, s[planes], s[npl], s[members], s[moff], plane_dist_th,
                                          s[ppn], s[ppsrc], s[ppcoef], s[ppoff], s[pppts], out->cap_plane_pts, s[ppst])) != PSLAM_OK)
        return rc;
    if (out->surface_normals8 && (rc = pslam_surface_normals_batch_dev(c, s[depth_d], nframes, s[sn8], nullptr)) != PSLAM_OK) return rc;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_status + 2 * (size_t)nframes, c->d_status, nf * 4, cudaMemcpyDeviceToHost, st));      // PEAC capacity flags (ORB reuses the array below)
    PSLAM_CUDA(c, cudaEventRecord(B.ev_planes, st));
    // the plane products return on the copy stream while the two image chains run
    PSLAM_CUDA(c, cudaStreamWaitEvent(cs, B.ev_planes, 0));
    s.down(out->n_planes, ppn, cs); s.down(out->plane_src, ppsrc, cs); s.down(out->plane_coef, ppcoef, cs); s.down(out->plane_pt_off, ppoff, cs); s.down(out->plane_pts, pppts, cs);
    if (out->surface_normals8) s.down(out->surface_normals8, sn8, cs);
    s.down(B.h_status + nframes, ppst, cs);        // plane post-processing capacity flags
    // ExtractORB, then ComputeStereoFromRGBD on the key points it leaves in HBM (no distortion model on this path: mvKeysUn = mvKeys, Frame::UndistortKeyPoints :545-549)
    PSLAM_CUDA(c, cudaStreamWaitEvent(st, B.ev_gray, 0));
    if ((rc = pslam_orb_extract_batch_dev(c, s[gray_d], nframes, s[kps], s[desc], cap, s[nk])) != PSLAM_OK) return rc;
    if ((rc = pslam_compute_stereo_from_rgbd_batch_dev(c, s[kps], s[kps], s[nk], cap, s[depth_d], nframes, depth_factor, bf,
                                                       s[ur], s[dz])) != PSLAM_OK) return rc;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_status, c->d_status, nf * 4, cudaMemcpyDeviceToHost, st));                            // ORB capacity flags
    s.down(out->keys, kps, st); s.down(out->desc, desc, st); s.down(out->n_keys, nk, st); s.down(out->u_right, ur, st); s.down(out->depth_kp, dz, st);
    // ExtractLSD: segments -> key lines + line functions + LBD descriptors, then isLineGood
    if ((rc = pslam_lines_extract_describe_batch_dev(c, s[gray_d], nframes, max_lines, s[kl], s[lf], s[ldesc], s[nkl])) != PSLAM_OK)
        return rc;
    if ((rc = pslam_lines3d_batch_dev(c, s[kl], s[nkl], max_lines, s[depth_d], nframes, depth_factor, cam, s[seed], nullptr,
                                      s[l3d], s[drawn])) != PSLAM_OK) return rc;
    if ((rc = lsd_status_fetch_async(c, nframes, B.h_status + 3 * (size_t)nframes)) != PSLAM_OK) return rc;
    s.down(out->keylines, kl, st); s.down(out->line_functions, lf, st); s.down(out->line_desc, ldesc, st); s.down(out->lines3d, l3d, st); s.down(out->n_lines, nkl, st);
    if (out->n_rand_drawn) s.down(out->n_rand_drawn, drawn, st);
    PSLAM_CUDA(c, cudaStreamSynchronize(cs));
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    for (int f = 0; f < nframes; ++f) {
        if (B.h_status[nframes + f] & (32 | 64)) return set_error(c, PSLAM_E_CAPACITY, "frame construct: more voxels than the plane post-processing capacity");
        if (out->n_keys[f] > cap || B.h_status[f]) return set_error(c, PSLAM_E_CAPACITY, "frame construct: ORB candidate / key point capacity exceeded");
        if (B.h_status[2 * (size_t)nframes + f]) return set_error(c, PSLAM_E_CAPACITY, "frame construct: PEAC capacity exceeded (planes / region-growing queue)");
        if (B.h_status[3 * (size_t)nframes + f]) return set_error(c, PSLAM_E_CAPACITY, "frame construct: more line segments than the internal capacity");
    }
    return PSLAM_OK;
}

}  // extern "C"
