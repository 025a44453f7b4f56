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
    const size_t sz[] = {N * 48, N * 24, N * 4, N * 4, N, N * 16, N * 4, N * 4, 4};
    const void* src[] = {pos, normal, max_distance, min_distance};
    size_t off[10]; off[0] = 0;
    for (int i = 0; i < 9; ++i) off[i + 1] = (off[i] + sz[i] + 255) & ~(size_t)255;
    uint8_t* d = nullptr;
    PSLAM_CUDA(c, cudaMalloc((void**)&d, off[9]));
    cudaError_t e = cudaMemsetAsync(d + off[8], 0, 4, st);
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = cudaMemcpyAsync(d + off[i], src[i], sz[i], cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { cudaFree(d); return check_cuda(c, e, "line frustum upload"); }
    PSLAM_LAUNCH(c, "lines_in_frustum", k_lines_in_frustum<<<(n + 127) / 128, 128, 0, st>>>(F, n, (const double*)(d + off[0]), (const double*)(d + off[1]),
                 (const float*)(d + off[2]), (const float*)(d + off[3]), cos_limit, d + off[4], (float*)(d + off[5]), (int32_t*)(d + off[6]), (float*)(d + off[7]),
                 (int32_t*)(d + off[8])));
    int32_t cnt = 0;
    void* dst[] = {in_view, proj, level, view_cos, &cnt};
    for (int i = 0; i < 5 && e == cudaSuccess; ++i) e = cudaMemcpyAsync(dst[i], d + off[4 + i], sz[4 + i], cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    if (e != cudaSuccess) return check_cuda(c, e, "line frustum");
    return cnt;
}
