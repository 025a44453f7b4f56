// Frame::isInFrustum(MapLine*, cosLimit) on sm_90a - the visibility pass of Tracking::SearchLocalLines (src/Tracking.cc:2352-2366,
// src/Frame.cc:369-437) that produces the map-line fields LSDmatcher::SearchByProjection reads (pslam_line_search_by_projection).
// One thread per map line; elementwise, 88 B in / 25 B out per line: HBM-trivial, it exists so that the line match chain needs no host pass.
#include <cstdint>

#include "linefrustum_body.h"
#include "pslam_internal.h"

namespace pslam {

__global__ void k_lines_in_frustum(LfFrame F, int n, const double* __restrict__ pos, const double* __restrict__ normal, const float* __restrict__ max_distance,
                                   const float* __restrict__ min_distance, float cos_limit, uint8_t* __restrict__ in_view, float* __restrict__ proj,
                                   int32_t* __restrict__ level, float* __restrict__ view_cos, int32_t* __restrict__ count) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    bool ok = false;
    if (k < n) {
        float p[4], vc;
        int32_t lvl;
        ok = lf_line_in_frustum(F, pos + 6 * (size_t)k, normal + 3 * (size_t)k, max_distance[k], min_distance[k], cos_limit, p, lvl, vc);
        in_view[k] = ok ? 1 : 0; level[k] = lvl; view_cos[k] = vc;
        for (int q = 0; q < 4; ++q) proj[4 * (size_t)k + q] = p[q];
    }
    const unsigned b = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, __popc(b));
}

}  // namespace pslam

using namespace pslam;

extern "C" int pslam_lines_in_frustum(pslam_ctx* c, const pslam_line_frustum_frame* frame, int n, const double* pos, const double* normal, const float* max_distance,
                                      const float* min_distance, float cos_limit, uint8_t* in_view, float* proj, int32_t* level, float* view_cos) {
    if (!c) return PSLAM_E_INVALID;
    if (!frame || n < 0 || (n && (!pos || !normal || !max_distance || !min_distance || !in_view || !proj || !level || !view_cos)))
        return set_error(c, PSLAM_E_INVALID, "bad line frustum arguments");
    if (n == 0) return 0;
    static_assert(sizeof(pslam_line_frustum_frame) == 25 * 4, "pslam_line_frustum_frame layout");
    LfFrame F;
    for (int i = 0; i < 16; ++i) F.Tcw[i] = frame->Tcw[i];
    F.fx = frame->fx; F.fy = frame->fy; F.cx = frame->cx; F.cy = frame->cy; F.min_x = frame->min_x; F.max_x = frame->max_x; F.min_y = frame->min_y; F.max_y = frame->max_y;
    F.log_scale_factor = frame->log_scale_factor;
    lf_camera_center(F);
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    const size_t N = (size_t)n;
    Slab s;
    const auto d_pos = s.add<double>(N * 6), d_normal = s.add<double>(N * 3);
    const auto d_max_d = s.add<float>(N), d_min_d = s.add<float>(N);
    const auto d_in_view = s.add<uint8_t>(N);
    const auto d_proj = s.add<float>(N * 4);
    const auto d_level = s.add<int32_t>(N);
    const auto d_view_cos = s.add<float>(N);
    const auto d_cnt = s.add<int32_t>(1);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.zero(d_cnt, st);
    s.up(d_pos, pos, st); s.up(d_normal, normal, st); s.up(d_max_d, max_distance, st); s.up(d_min_d, min_distance, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    PSLAM_LAUNCH(c, "lines_in_frustum", k_lines_in_frustum<<<(n + 127) / 128, 128, 0, st>>>(F, n, s[d_pos], s[d_normal], s[d_max_d], s[d_min_d], cos_limit, s[d_in_view],
                 s[d_proj], s[d_level], s[d_view_cos], s[d_cnt]));
    int32_t cnt = 0;
    s.down(in_view, d_in_view, st); s.down(proj, d_proj, st); s.down(level, d_level, st); s.down(view_cos, d_view_cos, st); s.down(&cnt, d_cnt, st);
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    return cnt;
}
