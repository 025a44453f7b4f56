// Frame::ComputeStereoFromRGBD (src/Frame.cc:603-621) on sm_90a: per key point the depth under the (distorted) key point and the
// virtual right coordinate u_un - bf / d.  One thread per key point over a batch of frames; consumes the key points
// pslam_orb_extract_batch_dev leaves in HBM and the raw depth frames the PEAC path already holds (metres = (float)raw * depth_factor,
// the Frame constructor's imDepth.convertTo(CV_32F, depthMapFactor), :80-83).  Elementwise, HBM-trivial.
#include <cstdint>

#include "pslam_internal.h"

namespace pslam {

__global__ void k_stereo_from_rgbd(const pslam_keypoint* __restrict__ keys, const pslam_keypoint* __restrict__ keys_un, const int32_t* __restrict__ n, int cap,
                                   const uint16_t* __restrict__ depth, int w, int h, float depth_factor, float bf, float* __restrict__ u_right,
                                   float* __restrict__ out_depth) {
    const int f = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    const size_t o = (size_t)f * cap + i;
    float ur = -1.0f, dz = -1.0f;
    if (i < n[f]) {
        const float u = keys[o].x, v = keys[o].y;
        const float d = __fmul_rn((float)depth[((size_t)f * h + (int)v) * w + (int)u], depth_factor);      // Mat::at<float>(float, float): truncation
        if (d > 0) { dz = d; ur = __fsub_rn(keys_un[o].x, __fdiv_rn(bf, d)); }
    }
    u_right[o] = ur; out_depth[o] = dz;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_compute_stereo_from_rgbd_batch_dev(pslam_ctx* c, const pslam_keypoint* d_keys, const pslam_keypoint* d_keys_un, const int32_t* d_n, int cap,
                                             const uint16_t* d_depth, int nframes, float depth_factor, float bf, float* d_u_right, float* d_depth_out) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_keys || !d_keys_un || !d_n || !d_depth || !d_u_right || !d_depth_out || cap < 1 || nframes < 1) return set_error(c, PSLAM_E_INVALID, "bad stereo arguments");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const dim3 grid((cap + 127) / 128, nframes);
    PSLAM_LAUNCH(c, "stereo_from_rgbd", k_stereo_from_rgbd<<<grid, 128, 0, c->stream>>>(d_keys, d_keys_un, d_n, cap, d_depth, c->cfg.width, c->cfg.height, depth_factor,
                 bf, d_u_right, d_depth_out));
    return PSLAM_OK;
}

int pslam_compute_stereo_from_rgbd_batch(pslam_ctx* c, const pslam_keypoint* keys, const pslam_keypoint* keys_un, const int32_t* n, int cap, const uint16_t* depth,
                                         int nframes, float depth_factor, float bf, float* u_right, float* depth_out) {
    if (!c) return PSLAM_E_INVALID;
    if (!keys || !keys_un || !n || !depth || !u_right || !depth_out || cap < 1 || nframes < 1) return set_error(c, PSLAM_E_INVALID, "bad stereo arguments");
    for (int f = 0; f < nframes; ++f) if (n[f] < 0 || n[f] > cap) return set_error(c, PSLAM_E_INVALID, "key point count outside [0, cap]");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    const size_t nf = (size_t)nframes, npx = (size_t)c->cfg.width * c->cfg.height;
    const bool same = keys_un == keys;
    Slab s;
    const auto d_keys = s.add<pslam_keypoint>(nf * cap), d_keys_un = s.add<pslam_keypoint>(same ? 0 : nf * cap);
    const auto d_n = s.add<int32_t>(nf);
    const auto d_depth = s.add<uint16_t>(nf * npx);
    const auto d_ur = s.add<float>(nf * cap), d_dz = s.add<float>(nf * cap);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.up(d_keys, keys, st); s.up(d_keys_un, keys_un, st); s.up(d_n, n, st); s.up(d_depth, depth, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    rc = pslam_compute_stereo_from_rgbd_batch_dev(c, s[d_keys], s[same ? d_keys : d_keys_un], s[d_n], cap, s[d_depth], nframes, depth_factor, bf, s[d_ur], s[d_dz]);
    if (rc != PSLAM_OK) return rc;
    s.down(u_right, d_ur, st); s.down(depth_out, d_dz, st);
    return s.sync(c, st);
}

}
