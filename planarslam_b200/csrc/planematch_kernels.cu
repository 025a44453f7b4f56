// PlaneMatcher::SearchMapByCoefficients on sm_90a (src/PlaneMatcher.cpp:10-80, Frame::ComputePlaneWorldCoeff src/Frame.cc:815-820).
// Stage 1 (one warp per (frame plane, map plane) pair): normal dot product and the minimum point-to-plane distance over the
// map plane's voxel points (warp-shuffle min).  Stage 2 (one thread per frame plane): the reference's sequential scan over
// the map planes with its shrinking thresholds (closest association, most perpendicular, most parallel).
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "pslam_internal.h"

namespace pslam {

__global__ void __launch_bounds__(256) k_plane_pairs(int n_frame, int n_map, const float* __restrict__ pM /*[n_frame][4]*/, const float* __restrict__ map_coef,
                                                     const int32_t* __restrict__ pts_off, const float* __restrict__ pts, float* __restrict__ angle,
                                                     float* __restrict__ mind) {
    const int pair = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (pair >= n_frame * n_map) return;
    const int i = pair / n_map, j = pair - i * n_map;
    const float a = pM[4 * i], b = pM[4 * i + 1], c = pM[4 * i + 2], d = pM[4 * i + 3];
    float res = 100.f;       // the reference keeps the minimum in a double initialised to 100; every candidate is a float value
    for (int p = pts_off[j] + lane; p < pts_off[j + 1]; p += 32) res = fminf(res, fabsf(a * pts[3 * p] + b * pts[3 * p + 1] + c * pts[3 * p + 2] + d));
#pragma unroll
    for (int o = 16; o; o >>= 1) res = fminf(res, __shfl_xor_sync(0xffffffffu, res, o));
    if (lane == 0) { angle[pair] = a * map_coef[4 * j] + b * map_coef[4 * j + 1] + c * map_coef[4 * j + 2]; mind[pair] = res; }
}

__global__ void k_plane_assign(int n_frame, int n_map, const uint8_t* __restrict__ map_bad, const float* __restrict__ angle, const float* __restrict__ mind,
                               float dTh, float aTh, float verTh, float parTh, int32_t* __restrict__ match, int32_t* __restrict__ ver,
                               int32_t* __restrict__ par, int32_t* __restrict__ nmatches) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frame) return;
    float ldTh = dTh, lverTh = verTh, lparTh = parTh;
    int m = -1, v = -1, p = -1;
    for (int j = 0; j < n_map; ++j) {
        if (map_bad[j]) continue;
        const float ang = angle[i * n_map + j];
        if (ang > aTh || ang < -aTh) {
            const double res = (double)mind[i * n_map + j];
            if (res < (double)ldTh) { ldTh = (float)res; m = j; continue; }
        }
        if (ang < lverTh && ang > -lverTh) { lverTh = fabsf(ang); v = j; continue; }
        if (ang > lparTh || ang < -lparTh) { lparTh = fabsf(ang); p = j; }
    }
    match[i] = m; ver[i] = v; par[i] = p;
    if (m >= 0) atomicAdd(nmatches, 1);
}

}  // namespace pslam

using namespace pslam;

extern "C" int pslam_plane_match(pslam_ctx* c, const float* Tcw, int n_frame, const float* frame_coef, int n_map, const float* map_coef,
                                 const uint8_t* map_bad, const int32_t* pts_off, const float* pts, float dTh, float aTh, float verTh, float parTh,
                                 int32_t* match, int32_t* ver, int32_t* par) {
    if (!c) return PSLAM_E_INVALID;
    if (n_frame < 0 || n_map < 0 || !Tcw || (n_frame && (!frame_coef || !match || !ver || !par)) || (n_map && (!map_coef || !map_bad || !pts_off)))
        return set_error(c, PSLAM_E_INVALID, "bad plane arrays");
    for (int i = 0; i < n_frame; ++i) match[i] = ver[i] = par[i] = -1;
    if (n_frame == 0 || n_map == 0) return 0;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    // pi_w = Tcw^T pi_c: a 4x4 float product per frame plane, done while packing (double accumulation like cv::gemm)
    std::vector<float> pM((size_t)n_frame * 4);
    for (int i = 0; i < n_frame; ++i)
        for (int r = 0; r < 4; ++r) {
            double s = 0;
            for (int k = 0; k < 4; ++k) s += (double)Tcw[k * 4 + r] * (double)frame_coef[4 * i + k];
            pM[4 * i + r] = (float)s;
        }
    const int npts = pts_off[n_map];
    const size_t bytes = 256 * 12 + pM.size() * 4 + (size_t)n_map * 4 * 4 + n_map + (size_t)(n_map + 1) * 4 + (size_t)npts * 12 +
                         (size_t)n_frame * n_map * 8 + (size_t)n_frame * 12 + 16;
    uint8_t* blob = nullptr;
    PSLAM_CUDA(c, cudaMalloc((void**)&blob, bytes));
    uint8_t* p = blob;
    auto carve = [&](size_t n) { uint8_t* r = p; p += (n + 255) / 256 * 256; return r; };
    float* d_pM = (float*)carve(pM.size() * 4); float* d_mc = (float*)carve((size_t)n_map * 16); uint8_t* d_bad = carve(n_map);
    int32_t* d_off = (int32_t*)carve((size_t)(n_map + 1) * 4); float* d_pts = (float*)carve((size_t)npts * 12 + 4);
    float* d_ang = (float*)carve((size_t)n_frame * n_map * 4); float* d_min = (float*)carve((size_t)n_frame * n_map * 4);
    int32_t* d_out = (int32_t*)carve((size_t)n_frame * 12 + 16);
    cudaStream_t st = c->stream;
    int rc = PSLAM_OK;
#define TRY(call) if (rc == PSLAM_OK) rc = check_cuda(c, (call), #call)
    TRY(cudaMemcpyAsync(d_pM, pM.data(), pM.size() * 4, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(d_mc, map_coef, (size_t)n_map * 16, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(d_bad, map_bad, n_map, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(d_off, pts_off, (size_t)(n_map + 1) * 4, cudaMemcpyHostToDevice, st));
    if (npts) TRY(cudaMemcpyAsync(d_pts, pts, (size_t)npts * 12, cudaMemcpyHostToDevice, st));
    TRY(cudaMemsetAsync(d_out + 3 * n_frame, 0, sizeof(int32_t), st));
    if (rc == PSLAM_OK) {
        PSLAM_LAUNCH(c, "plane_pairs", k_plane_pairs<<<(n_frame * n_map + 7) / 8, 256, 0, st>>>(n_frame, n_map, d_pM, d_mc, d_off, d_pts, d_ang, d_min));
        PSLAM_LAUNCH(c, "plane_assign", k_plane_assign<<<(n_frame + 63) / 64, 64, 0, st>>>(n_frame, n_map, d_bad, d_ang, d_min, dTh, aTh, verTh, parTh, d_out,
                     d_out + n_frame, d_out + 2 * n_frame, d_out + 3 * n_frame));
    }
    std::vector<int32_t> out((size_t)3 * n_frame + 1);
    TRY(cudaMemcpyAsync(out.data(), d_out, out.size() * 4, cudaMemcpyDeviceToHost, st));
    TRY(cudaStreamSynchronize(st));
#undef TRY
    cudaFree(blob);
    if (rc != PSLAM_OK) return rc;
    for (int i = 0; i < n_frame; ++i) { match[i] = out[i]; ver[i] = out[n_frame + i]; par[i] = out[2 * n_frame + i]; }
    return out[3 * n_frame];
}
