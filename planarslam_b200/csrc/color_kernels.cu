// The grey conversion of Tracking::GrabImageRGBD (src/Tracking.cc:157-172): cvtColor RGB / BGR / RGBA / BGRA -> GRAY as Camera.RGB and the channel count
// select, for colour frames already on the device.  OpenCV's 8-bit path is integer arithmetic, and so is this kernel: a float conversion rounds some pixels
// to the neighbouring grey level, and FAST and LSD then see other pixels than the reference's.
#include <cuda_runtime.h>

#include <cstdint>

#include "pslam_internal.h"

namespace pslam {
namespace {

// cv2 4.13 (all 2^24 triples, tests/test_oracle_gray_from_color.py): Y = (9798 R + 19235 G + 3735 B + 2^14) >> 15; w0 / w2 weigh the first / third byte
__device__ __forceinline__ uint32_t gray_of(uint32_t b0, uint32_t b1, uint32_t b2, uint32_t w0, uint32_t w2) {
    return (b0 * w0 + b1 * 19235u + b2 * w2 + (1u << 14)) >> 15;
}

// n pixels of CH interleaved bytes -> n grey bytes.  One thread converts four pixels: CH 32-bit loads (12 or 16 bytes) and one uchar4 store; both
// pointers are 4-byte aligned (checked by the entry point), and a frame batch is one dense array, so only the last thread of the batch has a partial group.
template <int CH>
__global__ void __launch_bounds__(256) k_gray_from_color(const uint8_t* __restrict__ src, size_t n, int rgb, uint8_t* __restrict__ dst) {
    const size_t p = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (p >= n) return;
    const uint32_t w0 = rgb ? 9798u : 3735u, w2 = rgb ? 3735u : 9798u;
    if (p + 4 <= n) {
        const uint32_t* s = reinterpret_cast<const uint32_t*>(src + p * CH);
        uint32_t w[CH];
#pragma unroll
        for (int k = 0; k < CH; ++k) w[k] = __ldg(s + k);
        uint32_t g[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint32_t b[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) b[j] = (w[(i * CH + j) >> 2] >> (8 * ((i * CH + j) & 3))) & 255u;
            g[i] = gray_of(b[0], b[1], b[2], w0, w2);
        }
        *reinterpret_cast<uchar4*>(dst + p) = make_uchar4(g[0], g[1], g[2], g[3]);
    } else {
        for (size_t q = p; q < n; ++q) dst[q] = (uint8_t)gray_of(src[q * CH], src[q * CH + 1], src[q * CH + 2], w0, w2);
    }
}

}  // namespace
}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_gray_from_color_batch_dev(pslam_ctx* c, const uint8_t* d_color, int channels, int rgb, int nframes, uint8_t* d_gray) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_color || !d_gray || (channels != 3 && channels != 4) || nframes < 1 || nframes > c->cfg.max_batch)
        return set_error(c, PSLAM_E_INVALID, "gray from color: null pointer, channels not 3 or 4, or nframes outside [1, max_batch]");
    if (((uintptr_t)d_color | (uintptr_t)d_gray) & 3) return set_error(c, PSLAM_E_INVALID, "gray from color: image pointers must be 4-byte aligned");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const size_t n = (size_t)nframes * c->cfg.width * c->cfg.height;
    const unsigned grid = (unsigned)((n + 4 * 256 - 1) / (4 * 256));
    if (channels == 3) PSLAM_LAUNCH(c, "gray_from_color", k_gray_from_color<3><<<grid, 256, 0, c->stream>>>(d_color, n, rgb != 0, d_gray));
    else PSLAM_LAUNCH(c, "gray_from_color", k_gray_from_color<4><<<grid, 256, 0, c->stream>>>(d_color, n, rgb != 0, d_gray));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

}  // extern "C"
