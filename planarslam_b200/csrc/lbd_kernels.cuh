// LBD line descriptors on sm_90a - the descriptor half of LineSegment::ExtractLineSegment (src/LSDextractor.cpp:14,28: BinaryDescriptor::compute of
// opencv_contrib's line_descriptor, not vendored in /root/reference; algorithm: Zhang & Koch 2013; restated in oracle/lbd.cc, whose header says what is and
// is not pinned).  Bit-exact to that restatement: the float sums keep the upstream accumulation order (along a row of the support region, then rows in order
// into each band), so the parallel decomposition follows the order constraints:
//   k_lbd_gradients  GaussianBlur(5x5, s = 1; 8.8 fixed point) + Sobel(CV_16S, 3) of every frame -> int16 dx / dy planes (bulk per-pixel, HBM-bound)
//   k_lbd_lines      one CTA (64 threads) per key line: thread r walks row r of the 63-row support region along the line (sequential float sums, the
//                    gradient samples are L2 gathers), threads 0..8 then fold the rows into the nine bands in row order, thread 0 normalises the 72 floats,
//                    32 threads write the 32 comparison bytes
#pragma once
#include "lsd_kernels.cuh"

namespace pslam {

#define LBD_BANDS 9
#define LBD_WIDTH 7
#define LBD_HEIGHT (LBD_BANDS * LBD_WIDTH)
#define LBD_TW 32
#define LBD_TH 16

__device__ __forceinline__ int lbd_reflect101(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

// one CTA: 32 x 16 output pixels; source tile with a 3-pixel REFLECT_101 halo (a symmetric filter commutes with the symmetric extension, so blurring the
// extended source one pixel beyond the image equals OpenCV's reflection of the blurred image in the Sobel pass)
__global__ void __launch_bounds__(256) k_lbd_gradients(const uint8_t* __restrict__ gray, int w, int h, int16_t* __restrict__ dxo, int16_t* __restrict__ dyo) {
    __shared__ uint8_t s_src[LBD_TH + 6][LBD_TW + 8];
    __shared__ uint16_t s_h[LBD_TH + 6][LBD_TW + 2];
    __shared__ uint8_t s_b[LBD_TH + 2][LBD_TW + 2];
    const int frame = blockIdx.z, x0 = blockIdx.x * LBD_TW, y0 = blockIdx.y * LBD_TH;
    const uint8_t* src = gray + (size_t)frame * w * h;
    for (int t = threadIdx.x; t < (LBD_TH + 6) * (LBD_TW + 6); t += 256) {
        const int r = t / (LBD_TW + 6), c = t - r * (LBD_TW + 6);
        s_src[r][c] = src[(size_t)lbd_reflect101(y0 - 3 + r, h) * w + lbd_reflect101(x0 - 3 + c, w)];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < (LBD_TH + 6) * (LBD_TW + 2); t += 256) {           // horizontal taps 14 62 104 62 14 at columns x0 - 1 .. x0 + TW
        const int r = t / (LBD_TW + 2), c = t - r * (LBD_TW + 2);
        const uint8_t* p = &s_src[r][c];
        s_h[r][c] = (uint16_t)(14 * (p[0] + p[4]) + 62 * (p[1] + p[3]) + 104 * p[2]);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < (LBD_TH + 2) * (LBD_TW + 2); t += 256) {           // vertical taps, rows y0 - 1 .. y0 + TH
        const int r = t / (LBD_TW + 2), c = t - r * (LBD_TW + 2);
        const uint32_t acc = 14u * (s_h[r][c] + s_h[r + 4][c]) + 62u * (s_h[r + 1][c] + s_h[r + 3][c]) + 104u * s_h[r + 2][c];
        s_b[r][c] = (uint8_t)min(255u, (acc + 32768u) >> 16);
    }
    __syncthreads();
    const int lx = threadIdx.x & 31, ly0 = threadIdx.x >> 5;
    for (int ly = ly0; ly < LBD_TH; ly += 8) {
        const int x = x0 + lx, y = y0 + ly;
        if (x >= w || y >= h) continue;
        const int a = s_b[ly][lx], b = s_b[ly][lx + 1], c = s_b[ly][lx + 2], d = s_b[ly + 1][lx], f = s_b[ly + 1][lx + 2], g = s_b[ly + 2][lx], hh = s_b[ly + 2][lx + 1],
                  i = s_b[ly + 2][lx + 2];
        const size_t o = ((size_t)frame * h + y) * w + x;
        dxo[o] = (int16_t)((c + 2 * f + i) - (a + 2 * d + g));
        dyo[o] = (int16_t)((g + 2 * hh + i) - (a + 2 * b + c));
    }
}

__constant__ int c_lbd_comb[32][2] = {{0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}, {0, 6}, {1, 2}, {1, 3}, {1, 4}, {1, 5}, {1, 6}, {2, 3}, {2, 4}, {2, 5}, {2, 6}, {2, 7},
                                     {2, 8}, {3, 4}, {3, 5}, {3, 6}, {3, 7}, {3, 8}, {4, 5}, {4, 6}, {4, 7}, {4, 8}, {5, 6}, {5, 7}, {5, 8}, {6, 7}, {6, 8}, {7, 8}};

// grid (max_lines, frames), block 64
__global__ void __launch_bounds__(64) k_lbd_lines(const int16_t* __restrict__ dxI, const int16_t* __restrict__ dyI, int w, int h, const LsdKeyLine* __restrict__ kls,
                                                  const int32_t* __restrict__ n_kl, int max_lines, const float* __restrict__ g_local /*[21]*/,
                                                  const float* __restrict__ g_global /*[63]*/, uint8_t* __restrict__ desc, float* __restrict__ lbd72) {
    __shared__ float s_row[LBD_HEIGHT][4];
    __shared__ float s_band[8][LBD_BANDS];
    __shared__ float s_des[LBD_BANDS * 8];
    const int li = blockIdx.x, frame = blockIdx.y, tid = threadIdx.x;
    if (li >= min(n_kl[frame], max_lines)) return;
    const LsdKeyLine L = kls[(size_t)frame * max_lines + li];
    const int16_t* dxp = dxI + (size_t)frame * w * h;
    const int16_t* dyp = dyI + (size_t)frame * w * h;
    const short imageWidth = (short)(w - 1), imageHeight = (short)(h - 1);
    const short lengthOfLSP = (short)L.numOfPixels;
    const short halfWidth = (short)((lengthOfLSP - 1) / 2), halfHeight = (short)((LBD_HEIGHT - 1) / 2);
    const float midX = (float)(0.5 * (double)__fadd_rn(L.sPointInOctaveX, L.ePointInOctaveX)), midY = (float)(0.5 * (double)__fadd_rn(L.sPointInOctaveY, L.ePointInOctaveY));
    double sn, cs;
    lsd_sincos<0>((double)L.angle, sn, cs);
    const float dL0 = (float)cs, dL1 = (float)sn, dO0 = -dL1, dO1 = dL0;
    if (tid < LBD_HEIGHT) {
        // row hID starts at sCorX0 - hID * dL1 accumulated step by step like upstream (float running sums)
        float sCorX0 = __fadd_rn(__fadd_rn(__fmul_rn(-dL0, (float)halfWidth), __fmul_rn(dL1, (float)halfHeight)), midX);
        float sCorY0 = __fadd_rn(__fsub_rn(__fmul_rn(-dL1, (float)halfWidth), __fmul_rn(dL0, (float)halfHeight)), midY);
        for (int r = 0; r < tid; ++r) { sCorX0 = __fsub_rn(sCorX0, dL1); sCorY0 = __fadd_rn(sCorY0, dL0); }
        float sCorX = sCorX0, sCorY = sCorY0;
        float pL = 0.f, nL = 0.f, pO = 0.f, nO = 0.f;
        for (short wID = 0; wID < lengthOfLSP; ++wID) {
            short t = (short)roundf(sCorX);
            const short xCor = t < 0 ? (short)0 : (t > imageWidth ? imageWidth : t);
            t = (short)roundf(sCorY);
            const short yCor = t < 0 ? (short)0 : (t > imageHeight ? imageHeight : t);
            const float dx = (float)__ldg(dxp + (size_t)yCor * w + xCor), dy = (float)__ldg(dyp + (size_t)yCor * w + xCor);
            const float gDL = __fadd_rn(__fmul_rn(dx, dL0), __fmul_rn(dy, dL1)), gDO = __fadd_rn(__fmul_rn(dx, dO0), __fmul_rn(dy, dO1));
            if (gDL > 0) pL = __fadd_rn(pL, gDL); else nL = __fsub_rn(nL, gDL);
            if (gDO > 0) pO = __fadd_rn(pO, gDO); else nO = __fsub_rn(nO, gDO);
            sCorX = __fadd_rn(sCorX, dL0); sCorY = __fadd_rn(sCorY, dL1);
        }
        const float coef = g_global[tid];
        s_row[tid][0] = __fmul_rn(coef, pL); s_row[tid][1] = __fmul_rn(coef, nL); s_row[tid][2] = __fmul_rn(coef, pO); s_row[tid][3] = __fmul_rn(coef, nO);
    }
    __syncthreads();
    if (tid < LBD_BANDS) {                 // band b receives one contribution per row of bands b - 1, b, b + 1, in row order
        const int b = tid;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        const int h0 = max(0, (b - 1) * LBD_WIDTH), h1 = min(LBD_HEIGHT, (b + 2) * LBD_WIDTH);
        for (int hID = h0; hID < h1; ++hID) {
            const int rb = hID / LBD_WIDTH, r = hID - rb * LBD_WIDTH;
            const float c = g_local[rb == b ? r + LBD_WIDTH : (rb == b + 1 ? r + 2 * LBD_WIDTH : r)];       // own band / the row's band is below / above
            const float cc = __fmul_rn(c, c);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float v = s_row[hID][k];
                acc[k] = __fadd_rn(acc[k], __fmul_rn(c, v));
                acc[4 + k] = __fadd_rn(acc[4 + k], __fmul_rn(cc, __fmul_rn(v, v)));
            }
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) s_band[k][b] = acc[k];
    }
    __syncthreads();
    if (tid == 0) {
        const float invN2 = (float)(1.0 / (LBD_WIDTH * 2.0)), invN3 = (float)(1.0 / (LBD_WIDTH * 3.0));
        for (int b = 0; b < LBD_BANDS; ++b) {
            const float invN = (b == 0 || b == LBD_BANDS - 1) ? invN2 : invN3;
            for (int k = 0; k < 4; ++k) {
                const float m = __fmul_rn(s_band[k][b], invN);
                s_des[b * 8 + k] = m;
                const float t = __fsub_rn(__fmul_rn(s_band[4 + k][b], invN), __fmul_rn(m, m));
                s_des[b * 8 + 4 + k] = t > 0 ? sqrtf(t) : 0.f;
            }
        }
        float tM = 0.f, tS = 0.f;
        for (int b = 0; b < LBD_BANDS; ++b) {
            for (int k = 0; k < 4; ++k) tM = __fadd_rn(tM, __fmul_rn(s_des[b * 8 + k], s_des[b * 8 + k]));
            for (int k = 4; k < 8; ++k) tS = __fadd_rn(tS, __fmul_rn(s_des[b * 8 + k], s_des[b * 8 + k]));
        }
        tM = __fdiv_rn(1.f, sqrtf(tM)); tS = __fdiv_rn(1.f, sqrtf(tS));
        for (int b = 0; b < LBD_BANDS; ++b) {
            for (int k = 0; k < 4; ++k) s_des[b * 8 + k] = __fmul_rn(s_des[b * 8 + k], tM);
            for (int k = 4; k < 8; ++k) s_des[b * 8 + k] = __fmul_rn(s_des[b * 8 + k], tS);
        }
        for (int i = 0; i < LBD_BANDS * 8; ++i) if ((double)s_des[i] > 0.4) s_des[i] = (float)0.4;
        float t2 = 0.f;
        for (int i = 0; i < LBD_BANDS * 8; ++i) t2 = __fadd_rn(t2, __fmul_rn(s_des[i], s_des[i]));
        t2 = __fdiv_rn(1.f, sqrtf(t2));
        for (int i = 0; i < LBD_BANDS * 8; ++i) s_des[i] = __fmul_rn(s_des[i], t2);
    }
    __syncthreads();
    const size_t o = (size_t)frame * max_lines + li;
    if (lbd72) for (int i = tid; i < LBD_BANDS * 8; i += 64) lbd72[o * 72 + i] = s_des[i];
    if (tid < 32) {
        const float *f1 = s_des + 8 * c_lbd_comb[tid][0], *f2 = s_des + 8 * c_lbd_comb[tid][1];
        uint32_t v = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) if (f1[i] > f2[i]) v += 1u << (7 - i);
        desc[o * 32 + tid] = (uint8_t)v;
    }
}

}  // namespace pslam
