// Line-segment detector on sm_90a - the detector half of LineSegment::ExtractLineSegment (src/LSDextractor.cpp:13-39), i.e.
// cv::LineSegmentDetector(LSD_REFINE_ADV) as opencv_contrib's LSDDetector drives it for one octave (neither is vendored in
// /root/reference; semantics pinned through cv2 4.13, see oracle/lsd.h).
//   k_lsd_blur_scale   Gaussian 7x7 s=0.75 (8.8 fixed point, REFLECT_101) fused with the INTER_LINEAR_EXACT x0.8 down-scaling:
//                      source tile staged in shared memory, horizontal pass, vertical pass, bilinear taps; HBM-bound
//                      (reads the frame once, writes 0.64 of it)
//   k_lsd_gradient     2x2 gradient -> three per-pixel planes (angle | used-bit word, cosf / sinf pair, packed gx gy) + per-frame
//                      max |grad|^2; the float cos / sin come from a host-libm table indexed by (gx, gy); HBM-bound
//   k_lsd_order        stable 1024-bin counting sort of the seeds, one CTA of 32 warps per frame (bulk-parallel; gradients recomputed
//                      from the 8-bit scaled image)
//   k_lsd_regions      one warp per frame, exact sequential semantics: region growing (the 8-neighbourhoods of up to four queued
//                      region points are evaluated by the 32 lanes, acceptances are replayed in order because every accepted pixel
//                      moves the region angle), rectangle fit with in-order double sums, density refinement; emits candidate
//                      rectangles; latency-bound
//   k_lsd_validate     one thread per candidate: first NFA evaluation (aligned pixels counted on integer word intervals, lsd_alignbounds.h; the NFA
//                      from a per-context table built on the device), failures queued;
//   k_lsd_improve      one thread per queued candidate: the remaining rect_improve stages; k_lsd_emit compacts
//   k_lsd_keylines     the 40 longest segments -> cv::line_descriptor::KeyLine records + line functions
#pragma once
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

#include "lsd_alignbounds.h"
#include "lsd_detsincos.h"
#include "lsd_rectenum.h"
#include "pslam_internal.h"

namespace pslam {

struct LsdGeom {
    int w, h;                 // input image
    int W, H;                 // scaled image (cvRound(0.8 w), cvRound(0.8 h))
    int refine;               // 0 NONE, 1 STD, 2 ADV
    int seg_cap;              // segment capacity per frame
    int cand_cap;             // candidate rectangles per frame (before the NFA validation)
    int rect_enum;            // pixel enumeration of the NFA validation: 0 published LSD rectangle iterator, 1 cv2 4.x rect_nfa (lsd_rectenum.h)
    int min_reg_size;
    double rho, prec, p, log_nt, density_th, log_eps;
    const double* lgamma_tab;  // log_gamma(i) for i = 0 .. LSD_LGAMMA_N - 1, evaluated by the host with the reference's formulas
    const double* nfa_tab;     // NFA(n, k, p / 2^j) for n <= LSD_NFA_NMAX, j < LSD_NFA_NJ (lsd_nfa), built on the device by k_lsd_nfa_table
};
#define LSD_LGAMMA_N 8192

// Per scaled pixel, three planes (k_lsd_gradient writes them, 16 bytes in all):
//   ang  uint32  bits 0..30 = float bits of the level-line angle in degrees, fastAtan2(gx, -gy) (>= 0), or LSD_ANG_UNDEF (+inf) when the gradient norm is
//                <= rho; bit 31 = the pixel belongs to a region ("used").  Region growing tests a neighbour with ONE 4-byte load; only k_lsd_regions writes it.
//   cs   float2  cosf / sinf of the float angle (host-libm table indexed by (gx, gy)); region growing reads it together with the angle word
//   gxy  uint32  gx | gy << 16 (int16 each): gradient norm for the rectangle fit and the seed ordering
// (LSD_ANG_UNDEF, the angle constants, lsd_word_angle and lsd_aligned_angle live in lsd_alignbounds.h)
#define LSD_ANG_USED 0x80000000u

#define LSD_LN10 2.30258509299404568402

__device__ __forceinline__ float lsd_fast_atan2_deg(float y, float x) {       // cv::fastAtan2 (same arithmetic as the ORB path)
    const float p1 = 0.9997878412794807f * (float)(180 / 3.14159265358979323846);
    const float p3 = -0.3258083974640975f * (float)(180 / 3.14159265358979323846);
    const float p5 = 0.1555786518463281f * (float)(180 / 3.14159265358979323846);
    const float p7 = -0.04432655554792128f * (float)(180 / 3.14159265358979323846);
    const float ax = fabsf(x), ay = fabsf(y);
    const bool wide = ax >= ay;
    const float num = wide ? ay : ax, den = __fadd_rn(wide ? ax : ay, (float)DBL_EPSILON);
    const float c = __fdiv_rn(num, den);
    const float c2 = __fmul_rn(c, c);
    float a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    if (!wide) a = __fsub_rn(90.f, a);
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}
__device__ __forceinline__ double lsd_angle(int gx, int gy) { return (double)lsd_fast_atan2_deg((float)gx, (float)(-gy)) * LSD_DEG2RAD; }
__device__ __forceinline__ double lsd_norm(int gx, int gy) { return sqrt((double)(gx * gx + gy * gy) / 4.0); }

// Deterministic double sin / cos (lsd_detsincos.h, the arithmetic of oracle/detmath.h); the per-V wrapper keeps one out-of-line copy per kernel variant
template <int V>
__device__ __noinline__ void lsd_sincos(double x, double& s, double& c) { lsd_sincos_body(x, s, c); }

// ---------------------------------------------------------------------------------------------------------------------
// Gaussian blur + down-scaling.  One CTA produces a 64 x 16 tile of the scaled image.
#define LSD_TW 64
#define LSD_TH 16
#define LSD_SW 88           // source tile width bound: 64 * 1.25 + 1 + 4 (blur) + slack
#define LSD_SH 28           // 16 * 1.25 + 1 + 4 + slack
__global__ void __launch_bounds__(256) k_lsd_blur_scale(LsdGeom g, const uint8_t* __restrict__ gray, const int16_t* __restrict__ ix,
                                                        const int16_t* __restrict__ ax, const int16_t* __restrict__ iy, const int16_t* __restrict__ ay,
                                                        uint8_t* __restrict__ scaled) {
    __shared__ uint8_t s_src[LSD_SH][LSD_SW];
    __shared__ uint16_t s_h[LSD_SH][LSD_SW];
    __shared__ uint8_t s_b[LSD_SH][LSD_SW];
    const int frame = blockIdx.z, X0 = blockIdx.x * LSD_TW, Y0 = blockIdx.y * LSD_TH;
    const int X1 = min(X0 + LSD_TW, g.W) - 1, Y1 = min(Y0 + LSD_TH, g.H) - 1;
    // blurred pixels needed: columns ix[X0] .. min(ix[X1] + 1, w - 1), rows likewise; source = that range +- 2 (taps +-3 are zero)
    const int bx0 = ix[X0], bx1 = min(ix[X1] + 1, g.w - 1), by0 = iy[Y0], by1 = min(iy[Y1] + 1, g.h - 1);
    const int sx0 = bx0 - 2, sy0 = by0 - 2, sw = bx1 - bx0 + 5, sh = by1 - by0 + 5;
    const uint8_t* src = gray + (size_t)frame * g.w * g.h;
    // one warp per tile row, lanes across the columns (no index divisions; rows of <= 88 bytes are three coalesced byte loads per lane)
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int r = wid; r < sh; r += 8) {
        int y = sy0 + r;
        y = y < 0 ? -y : (y >= g.h ? 2 * (g.h - 1) - y : y);          // REFLECT_101
        const uint8_t* srow = src + (size_t)y * g.w;
        for (int c = lane; c < sw; c += 32) {
            int x = sx0 + c;
            x = x < 0 ? -x : (x >= g.w ? 2 * (g.w - 1) - x : x);
            s_src[r][c] = srow[x];
        }
    }
    __syncthreads();
    const int bw = bx1 - bx0 + 1, bh = by1 - by0 + 1;
    for (int r = wid; r < sh; r += 8)                                  // horizontal pass, taps 4 56 136 56 4 (8.8)
        for (int c = lane; c < bw; c += 32)
            s_h[r][c] = (uint16_t)(4 * (s_src[r][c] + s_src[r][c + 4]) + 56 * (s_src[r][c + 1] + s_src[r][c + 3]) + 136 * s_src[r][c + 2]);
    __syncthreads();
    for (int r = wid; r < bh; r += 8)                                  // vertical pass, 16.16, round half up (the taps sum to 256 twice: no clamp needed)
        for (int c = lane; c < bw; c += 32) {
            const uint32_t acc = 4u * (s_h[r][c] + s_h[r + 4][c]) + 56u * (s_h[r + 1][c] + s_h[r + 3][c]) + 136u * s_h[r + 2][c];
            s_b[r][c] = (uint8_t)((acc + 32768u) >> 16);
        }
    __syncthreads();
    uint8_t* dst = scaled + (size_t)frame * g.W * g.H;
    for (int t = threadIdx.x; t < LSD_TW * LSD_TH; t += 256) {
        const int X = X0 + (t % LSD_TW), Y = Y0 + (t / LSD_TW);
        if (X >= g.W || Y >= g.H) continue;
        const int x0 = ix[X] - bx0, x1 = min(ix[X] + 1, g.w - 1) - bx0, y0 = iy[Y] - by0, y1 = min(iy[Y] + 1, g.h - 1) - by0;
        const uint32_t a = (uint32_t)ax[X], b = (uint32_t)ay[Y];
        const uint32_t h0 = (256u - a) * s_b[y0][x0] + a * s_b[y0][x1];
        const uint32_t h1 = (256u - a) * s_b[y1][x0] + a * s_b[y1][x1];
        dst[(size_t)Y * g.W + X] = (uint8_t)(((256u - b) * h0 + b * h1 + 32768u) >> 16);
    }
}

// 2x2 gradient, the three per-pixel planes, per-frame maximum of gx^2 + gy^2 over the pixels whose norm exceeds rho.
__global__ void __launch_bounds__(256) k_lsd_gradient(LsdGeom g, const uint8_t* __restrict__ scaled, const float2* __restrict__ cs_lut,
                                                      uint32_t* __restrict__ ang, float2* __restrict__ cs_out, uint32_t* __restrict__ gxy, int32_t* __restrict__ smax) {
    const int frame = blockIdx.z;
    const int x = blockIdx.x * 64 + (threadIdx.x & 63), y = blockIdx.y * 4 + (threadIdx.x >> 6);
    const bool inside = x < g.W && y < g.H;
    const uint8_t* s = scaled + (size_t)frame * g.W * g.H;
    uint32_t a_w = LSD_ANG_UNDEF, g_w = 0;
    float2 cs = make_float2(0.f, 0.f);
    int sq = 0;
    if (inside && x < g.W - 1 && y < g.H - 1) {
        const size_t a = (size_t)y * g.W + x;
        const int DA = (int)s[a + g.W + 1] - (int)s[a], BC = (int)s[a + 1] - (int)s[a + g.W];
        const int gx = DA + BC, gy = DA - BC;
        g_w = ((uint32_t)gx & 0xffffu) | ((uint32_t)gy << 16);
        // (cosf, sinf) of the level-line angle is only ever read for pixels that can join a region, i.e. defined ones: the 8-byte gather from the 8.3 MB table
        // is skipped for the rest (typically three quarters of the frame), which stay (0, 0)
        if (lsd_norm(gx, gy) > g.rho) {
            sq = gx * gx + gy * gy; a_w = __float_as_uint(lsd_fast_atan2_deg((float)gx, (float)(-gy)));
            cs = __ldg(cs_lut + (gx + 510) * 1021 + (gy + 510));
        }
    }
    if (inside) {
        const size_t o = (size_t)frame * g.W * g.H + (size_t)y * g.W + x;
        ang[o] = a_w; cs_out[o] = cs; gxy[o] = g_w;
    }
    // one atomic per warp
    for (int o = 16; o; o >>= 1) sq = max(sq, __shfl_xor_sync(0xffffffffu, sq, o));
    if ((threadIdx.x & 31) == 0 && sq > 0) atomicMax(&smax[frame], sq);
}

// The same for scaled widths that are a multiple of 4 (640x480 -> 512, 1280x960 -> 1024): four pixels per thread, the two source rows as aligned words and the
// three planes as 16 / 32 / 16-byte stores (k_lsd_gradient was bound by the latency of its four byte loads per thread: 39 % of the samples on their scoreboard).
__global__ void __launch_bounds__(256) k_lsd_gradient4(LsdGeom g, const uint8_t* __restrict__ scaled, const float2* __restrict__ cs_lut,
                                                       uint32_t* __restrict__ ang, float2* __restrict__ cs_out, uint32_t* __restrict__ gxy, int32_t* __restrict__ smax) {
    const int frame = blockIdx.z;
    const int W4 = g.W >> 2;
    const int xq = blockIdx.x * 64 + (threadIdx.x & 63), y = blockIdx.y * 4 + (threadIdx.x >> 6);
    const bool inside = xq < W4 && y < g.H;
    const uint8_t* s = scaled + (size_t)frame * g.W * g.H;
    uint32_t a_w[4] = {LSD_ANG_UNDEF, LSD_ANG_UNDEF, LSD_ANG_UNDEF, LSD_ANG_UNDEF}, g_w[4] = {0, 0, 0, 0};
    float2 cs[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) cs[i] = make_float2(0.f, 0.f);
    int sq = 0;
    if (inside && y < g.H - 1) {
        const int x = xq * 4;
        const uint32_t* r0 = reinterpret_cast<const uint32_t*>(s + (size_t)y * g.W + x);
        const uint32_t* r1 = reinterpret_cast<const uint32_t*>(s + (size_t)(y + 1) * g.W + x);
        const uint32_t w0 = r0[0], w1 = r1[0];
        const bool more = x + 4 < g.W;
        const uint32_t n0 = more ? (uint32_t)s[(size_t)y * g.W + x + 4] : 0u, n1 = more ? (uint32_t)s[(size_t)(y + 1) * g.W + x + 4] : 0u;
        const uint32_t e0 = __funnelshift_r(w0, n0, 8), e1 = __funnelshift_r(w1, n1, 8);      // the rows shifted left by one pixel
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (x + i >= g.W - 1) continue;
            const int pa = (w0 >> (8 * i)) & 255, pb = (e0 >> (8 * i)) & 255, pc = (w1 >> (8 * i)) & 255, pd = (e1 >> (8 * i)) & 255;
            const int DA = pd - pa, BC = pb - pc;
            const int gx = DA + BC, gy = DA - BC;
            g_w[i] = ((uint32_t)gx & 0xffffu) | ((uint32_t)gy << 16);
            if (lsd_norm(gx, gy) > g.rho) {
                sq = max(sq, gx * gx + gy * gy); a_w[i] = __float_as_uint(lsd_fast_atan2_deg((float)gx, (float)(-gy)));
                cs[i] = __ldg(cs_lut + (gx + 510) * 1021 + (gy + 510));
            }
        }
    }
    if (inside) {
        const size_t o = (size_t)frame * g.W * g.H + (size_t)y * g.W + (size_t)xq * 4;
        *reinterpret_cast<uint4*>(ang + o) = make_uint4(a_w[0], a_w[1], a_w[2], a_w[3]);
        *reinterpret_cast<uint4*>(gxy + o) = make_uint4(g_w[0], g_w[1], g_w[2], g_w[3]);
        float4* co = reinterpret_cast<float4*>(cs_out + o);
        co[0] = make_float4(cs[0].x, cs[0].y, cs[1].x, cs[1].y);
        co[1] = make_float4(cs[2].x, cs[2].y, cs[3].x, cs[3].y);
    }
    for (int o = 16; o; o >>= 1) sq = max(sq, __shfl_xor_sync(0xffffffffu, sq, o));
    if ((threadIdx.x & 31) == 0 && sq > 0) atomicMax(&smax[frame], sq);
}

// ---------------------------------------------------------------------------------------------------------------------
struct LsdRect { double x1, y1, x2, y2, width, x, y, theta, dx, dy, prec, p; };

#define LSD_RING 64
struct LsdFrame {                 // per-frame views
    uint32_t* ang;                // angle | used plane (see above); k_lsd_validate / k_lsd_improve only read it
    const float2* cs; const uint32_t* gxy;
    uint32_t* reg; uint32_t* order;
    int W, H;
};
__device__ __forceinline__ bool lsd_word_used(uint32_t w) { return (w & LSD_ANG_USED) != 0; }
__device__ __forceinline__ bool lsd_word_defined(uint32_t w) { return (w & 0x7fffffffu) < LSD_ANG_UNDEF; }
__device__ __forceinline__ double lsd_pix_norm(const LsdFrame& F, int x, int y) {
    const uint32_t v = __ldg(F.gxy + (size_t)y * F.W + x);
    return lsd_norm((int)(short)(v & 0xffff), (int)(short)(v >> 16));
}

__device__ __forceinline__ double lsd_angle_diff_signed(double a, double b) {
    double diff = a - b;
    while (diff <= -LSD_PI) diff += LSD_2PI;
    while (diff > LSD_PI) diff -= LSD_2PI;
    return diff;
}
__device__ __forceinline__ bool lsd_double_equal(double a, double b) {
    if (a == b) return true;
    const double abs_diff = fabs(a - b), aa = fabs(a), bb = fabs(b);
    double abs_max = (aa > bb) ? aa : bb;
    if (abs_max < DBL_MIN) abs_max = DBL_MIN;
    return (abs_diff / abs_max) <= (100.0 * DBL_EPSILON);
}
__device__ __forceinline__ double lsd_dist_sq(double x1, double y1, double x2, double y2) { return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1); }

// Region growing from pixel `seed` with tolerance prec (LineSegmentDetectorImpl::region_grow).  All lanes return the same
// size / reg_angle.  The FIFO of region points is reg[] (global) with its newest LSD_RING entries mirrored in shared memory.
//
// One step handles up to FOUR queued region points at once: lane group q = lane / 8 owns queue entry i + q, lane k = lane % 8 of the
// group owns its k-th neighbour in the reference's scan order (row-major 3x3 without the centre, which is always used).  The
// reference visits candidates in (queue index, neighbour index) order and every acceptance moves the region angle, so the
// acceptances are replayed in lane order: the first lane above the last accepted one whose pixel is unused, defined and aligned
// with the CURRENT region angle is taken, the angle is updated, and every lane that looks at the pixel just taken (another
// group's overlapping neighbourhood) drops its candidate.  Entries appended during a step belong to later steps, exactly like
// the reference's queue.  The records of the next step's neighbourhoods are requested one step ahead when the queue is long
// enough; the `used` bits are read at the start of a step (they depend on the previous step's acceptances).
//
// The serial chain of a step is the replay: ballot, shuffle of the winner's (cos, sin), float sums, atan2, alignment test.  Everything
// else is kept off it: the (cos, sin) pair is loaded with the angle word (its address is known before the word arrives), and the
// replay only records which lanes accepted - the used bit, the reg[] entry and the ring slot of every accepted pixel are written
// after it by the accepting lanes at once (nothing in the step reads them; acceptances are in increasing lane order, so an
// accepted lane's rank among the accepted lanes is its queue position).  The views are plain arguments so that they stay in registers.
struct LsdGrown { double angle; int size; };
template <int V>
__device__ __noinline__ LsdGrown lsd_region_grow(uint32_t* ang, const float2* __restrict__ cs, uint32_t* reg, int W, int H, uint32_t seed, double prec) {
    __shared__ uint32_t ring[LSD_RING];           // the last LSD_RING entries appended to reg[] (reg[i] lives in ring[i % LSD_RING])
    const int lane = threadIdx.x & 31;
    const unsigned below = (1u << lane) - 1u;
    const int q = lane >> 3, k8 = lane & 7;
    const int kk = k8 + (k8 >= 4);                 // index in the 3x3 window, centre skipped
    const int dyl = kk / 3 - 1, dxl = kk % 3 - 1;
    const int sx = seed & 0xffff, sy = seed >> 16;
    const uint32_t ws = ang[(size_t)sy * W + sx];
    double reg_angle = lsd_word_angle(ws);
    float sumdx = 0.f, sumdy = 0.f;
    if (lane == 0) { reg[0] = seed; ring[0] = seed; ang[(size_t)sy * W + sx] = ws | LSD_ANG_USED; }
    __syncwarp();
    // this lane's neighbour of queue entry idx: pixel, angle word and (cos, sin); out-of-image neighbours keep npix = ~0, LSD_ANG_UNDEF
    auto probe = [&](int idx, int size, uint32_t& npix, uint32_t& w, float2& csv) {
        const uint32_t pp = size - idx <= LSD_RING ? ring[idx & (LSD_RING - 1)] : reg[idx];
        const int nx = (int)(pp & 0xffff) + dxl, ny = (int)(pp >> 16) + dyl;
        if (nx >= 0 && ny >= 0 && nx < W && ny < H) {
            const size_t o = (size_t)ny * W + nx;
            w = ang[o]; csv = __ldg(cs + o); npix = (uint32_t)nx | ((uint32_t)ny << 16);
        }
    };
    int size = 1, i = 0;
    bool have_next = false;
    uint32_t np_next = 0xffffffffu, w_next = LSD_ANG_UNDEF;
    float2 cs_next = make_float2(0.f, 0.f);
    while (true) {
        const int navail = min(4, size - i);
        uint32_t npix = 0xffffffffu, w = LSD_ANG_UNDEF;
        float2 csv = make_float2(0.f, 0.f);
        if (have_next) { npix = np_next; w = w_next; csv = cs_next; }     // navail == 4; w_next was kept up to date while the previous step accepted pixels
        else if (q < navail) probe(i + q, size, npix, w, csv);
        // request the next step's neighbourhoods (entries i + 4 .. i + 7 exist already); acceptances of THIS step are patched into w_next below
        have_next = size - i >= 8;
        np_next = 0xffffffffu; w_next = LSD_ANG_UNDEF; cs_next = make_float2(0.f, 0.f);
        if (have_next) probe(i + 4 + q, size, np_next, w_next, cs_next);
        bool cand = lsd_word_defined(w) && !lsd_word_used(w);           // out-of-image lanes carry LSD_ANG_UNDEF
        const double a_n = lsd_word_angle(w);
        // cos / sin of the seed angle start the sums; evaluated only when the seed's first step accepts a pixel (most seeds stay alone)
        if (size == 1 && __any_sync(0xffffffffu, cand && lsd_aligned_angle(a_n, reg_angle, prec))) {
            double sn0, cs0;
            lsd_sincos<V>(reg_angle, sn0, cs0);
            sumdx = (float)cs0; sumdy = (float)sn0;
        }
        int last = -1;
        unsigned taken = 0;
        while (true) {
            const bool al = cand && lane > last && lsd_aligned_angle(a_n, reg_angle, prec);
            const unsigned m = __ballot_sync(0xffffffffu, al);
            if (!m) break;
            const int j = __ffs(m) - 1;
            const float cj = __shfl_sync(0xffffffffu, csv.x, j), sj = __shfl_sync(0xffffffffu, csv.y, j);
            const uint32_t np = __shfl_sync(0xffffffffu, npix, j);
            sumdx = __fadd_rn(sumdx, cj);
            sumdy = __fadd_rn(sumdy, sj);
            reg_angle = (double)lsd_fast_atan2_deg(sumdy, sumdx) * LSD_DEG2RAD;
            if (npix == np) cand = false;                  // the pixel is used now (lane j itself and overlapping neighbourhoods of the other groups)
            if (np_next == np) w_next |= LSD_ANG_USED;     // ... and in the neighbourhoods already requested for the next step
            taken |= 1u << j;
            last = j;
        }
        if (taken >> lane & 1u) {
            const int at = size + __popc(taken & below);
            ang[(size_t)(npix >> 16) * W + (npix & 0xffff)] = w | LSD_ANG_USED;
            reg[at] = npix; ring[at & (LSD_RING - 1)] = npix;
        }
        size += __popc(taken);
        __syncwarp();
        i += navail;
        if (i >= size) break;
    }
    return {reg_angle, size};
}

// region2rect + get_theta with the order-sensitive part reduced to its minimum.  The reference's running sums are sequential double additions; what is added - the
// products x * w, (dy * dy) * w ... - does not depend on the order.  So the lanes compute the terms of 32 region points at once and park them in shared memory, and
// lanes 0, 1, 2 each fold one of the three sums in point order (one shared-memory load + one DADD per point for all three sums together, instead of four
// shuffles and five to nine double operations per point in every lane).  The extent pass is a plain min / max: l_max >= 0 >= l_min always hold (both start at 0),
// so the reference's "else if" never skips an update and the order is irrelevant.
template <int V>
__device__ __noinline__ void lsd_region2rect(const LsdFrame& F, int size, double reg_angle, double prec, double p, LsdRect& rec) {
    __shared__ double s_stage[96];                                      // [3][32] terms of the three running sums (the CTA is one warp)
    const int lane = threadIdx.x & 31;
    const double* const mine = s_stage + 32 * (lane < 3 ? lane : 2);    // the sum this lane folds (lanes above 2 fold a copy that is never read)
    double acc = 0;
    for (int base = 0; base < size; base += 32) {
        if (base + lane < size) {
            const uint32_t pp = F.reg[base + lane];
            const int mx = pp & 0xffff, my = pp >> 16;
            const double mw = lsd_pix_norm(F, mx, my);
            s_stage[lane] = (double)mx * mw; s_stage[32 + lane] = (double)my * mw; s_stage[64 + lane] = mw;
        }
        __syncwarp();
        const int cnt = min(32, size - base);
        for (int t = 0; t < cnt; ++t) acc += mine[t];
        __syncwarp();
    }
    const double sum = __shfl_sync(0xffffffffu, acc, 2);
    const double x = __shfl_sync(0xffffffffu, acc, 0) / sum, y = __shfl_sync(0xffffffffu, acc, 1) / sum;
    acc = 0;
    for (int base = 0; base < size; base += 32) {
        if (base + lane < size) {
            const uint32_t pp = F.reg[base + lane];
            const int mx = pp & 0xffff, my = pp >> 16;
            const double mw = lsd_pix_norm(F, mx, my);
            const double ddx = (double)mx - x, ddy = (double)my - y;
            s_stage[lane] = ddy * ddy * mw; s_stage[32 + lane] = ddx * ddx * mw; s_stage[64 + lane] = -(ddx * ddy * mw);      // Ixy -= t  ==  Ixy += -t
        }
        __syncwarp();
        const int cnt = min(32, size - base);
        for (int t = 0; t < cnt; ++t) acc += mine[t];
        __syncwarp();
    }
    const double Ixx = __shfl_sync(0xffffffffu, acc, 0), Iyy = __shfl_sync(0xffffffffu, acc, 1), Ixy = __shfl_sync(0xffffffffu, acc, 2);
    const double lambda = 0.5 * (Ixx + Iyy - sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
    double theta = (fabs(Ixx) > fabs(Iyy)) ? (double)lsd_fast_atan2_deg((float)(lambda - Ixx), (float)Ixy) : (double)lsd_fast_atan2_deg((float)Ixy, (float)(lambda - Iyy));
    theta *= LSD_DEG2RAD;
    if (fabs(lsd_angle_diff_signed(theta, reg_angle)) > prec) theta += LSD_PI;
    double dx, dy;
    lsd_sincos<V>(theta, dy, dx);
    double l_min = 0, l_max = 0, w_min = 0, w_max = 0;
    for (int i = lane; i < size; i += 32) {
        const uint32_t pp = F.reg[i];
        const double regdx = (double)(pp & 0xffff) - x, regdy = (double)(pp >> 16) - y;
        const double l = regdx * dx + regdy * dy;
        const double w = -regdx * dy + regdy * dx;
        if (l > l_max) l_max = l; else if (l < l_min) l_min = l;
        if (w > w_max) w_max = w; else if (w < w_min) w_min = w;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const double a = __shfl_xor_sync(0xffffffffu, l_max, o), b = __shfl_xor_sync(0xffffffffu, l_min, o);
        const double c = __shfl_xor_sync(0xffffffffu, w_max, o), d = __shfl_xor_sync(0xffffffffu, w_min, o);
        if (a > l_max) l_max = a;
        if (b < l_min) l_min = b;
        if (c > w_max) w_max = c;
        if (d < w_min) w_min = d;
    }
    rec.x1 = x + l_min * dx; rec.y1 = y + l_min * dy;
    rec.x2 = x + l_max * dx; rec.y2 = y + l_max * dy;
    rec.width = w_max - w_min;
    rec.x = x; rec.y = y; rec.theta = theta; rec.dx = dx; rec.dy = dy; rec.prec = prec; rec.p = p;
    if (rec.width < 1.0) rec.width = 1.0;
}

__device__ __forceinline__ double lsd_density(int size, const LsdRect& rec) {
    return (double)size / (sqrt(lsd_dist_sq(rec.x1, rec.y1, rec.x2, rec.y2)) * rec.width);
}

// LineSegmentDetectorImpl::refine + reduce_region_radius; returns false when the region is dropped.  size / reg_angle / rec updated.
// The angle statistics are warp-parallel like lsd_region2rect: every lane computes the terms of its point (0 for the points outside the radius: the sums start
// at +0 and never become -0, so adding +0 leaves them unchanged) and lanes 0, 1 fold the two sums in point order over shared-memory staging.
template <int V>
__device__ __noinline__ bool lsd_refine(const LsdFrame& F, const LsdGeom& g, int& size, double& reg_angle, LsdRect& rec) {
    __shared__ double s_ang[64];                                        // [2][32] terms of sum and s_sum
    const int lane = threadIdx.x & 31;
    const unsigned below = (1u << lane) - 1u;
    double density = lsd_density(size, rec);
    if (density >= g.density_th) return true;
    uint32_t* const ang = F.ang;
    uint32_t* const reg = F.reg;
    const int W = F.W;
    const uint32_t p0 = reg[0];
    const double xc = (double)(p0 & 0xffff), yc = (double)(p0 >> 16);
    const double ang_c = lsd_word_angle(ang[(size_t)(p0 >> 16) * W + (p0 & 0xffff)]);
    const double* const mine = s_ang + 32 * (lane & 1);
    double acc = 0;
    int n = 0;
    for (int base = 0; base < size; base += 32) {
        bool near = false;
        if (base + lane < size) {
            const uint32_t pp = reg[base + lane];
            const int mx = pp & 0xffff, my = pp >> 16;
            const uint32_t wv = ang[(size_t)my * W + mx];
            ang[(size_t)my * W + mx] = wv & 0x7fffffffu;               // used = NOTUSED for the whole region (every lane owns distinct pixels)
            double ang_d = 0;
            near = sqrt(lsd_dist_sq(xc, yc, (double)mx, (double)my)) < rec.width;
            if (near) ang_d = lsd_angle_diff_signed(lsd_word_angle(wv), ang_c);
            s_ang[lane] = ang_d; s_ang[32 + lane] = ang_d * ang_d;
        }
        n += __popc(__ballot_sync(0xffffffffu, near));
        __syncwarp();
        const int cnt = min(32, size - base);
        for (int t = 0; t < cnt; ++t) acc += mine[t];
        __syncwarp();
    }
    const double sum = __shfl_sync(0xffffffffu, acc, 0), s_sum = __shfl_sync(0xffffffffu, acc, 1);
    const double mean_angle = sum / (double)n;
    const double tau = 2.0 * sqrt((s_sum - 2.0 * mean_angle * sum) / (double)n + mean_angle * mean_angle);
    const LsdGrown gr = lsd_region_grow<V>(ang, F.cs, reg, W, F.H, p0, tau);
    size = gr.size; reg_angle = gr.angle;
    if (size < 2) return false;
    lsd_region2rect<V>(F, size, reg_angle, g.prec, g.p, rec);
    density = lsd_density(size, rec);
    if (density >= g.density_th) return true;
    // reduce_region_radius.  The reference walks reg[] once per radius, replacing every point farther than the radius by the last point (re-examined in its
    // place) and shrinking the region.  That leaves the m = size - (far points) near points in reg[0 .. m): the near points below m stay where they are, and the
    // k-th far point below m (in index order) is replaced by the k-th near point at or above m (in DESCENDING index order).  Three ballot passes build the same
    // order: count the far points (and clear their used bits), pack the near points of reg[m .. size) against the end of the array in descending order, and fill
    // the holes below m from there.  (The far points the reference parks in reg[m .. size) are not kept: nothing reads past the region.)
    double radSq1 = lsd_dist_sq(xc, yc, rec.x1, rec.y1), radSq2 = lsd_dist_sq(xc, yc, rec.x2, rec.y2);
    double radSq = radSq1 > radSq2 ? radSq1 : radSq2;
    while (density < g.density_th) {
        radSq *= 0.75 * 0.75;
        auto far_point = [&](uint32_t pp) { return lsd_dist_sq(xc, yc, (double)(pp & 0xffff), (double)(pp >> 16)) > radSq; };
        int nfar = 0;
        for (int base = 0; base < size; base += 32) {
            bool f = false;
            if (base + lane < size) {
                const uint32_t pp = reg[base + lane];
                f = far_point(pp);
                if (f) ang[(size_t)(pp >> 16) * W + (pp & 0xffff)] &= 0x7fffffffu;
            }
            nfar += __popc(__ballot_sync(0xffffffffu, f));
        }
        const int m = size - nfar;
        int r = 0;
        for (int top = size - 1; top >= m; top -= 32) {          // lane t reads reg[top - t]; every write lands at or above the index its lane read
            const int idx = top - lane;
            uint32_t pp = 0;
            bool keep = false;
            if (idx >= m) { pp = reg[idx]; keep = !far_point(pp); }
            const unsigned k = __ballot_sync(0xffffffffu, keep);
            if (keep) reg[size - 1 - (r + __popc(k & below))] = pp;
            r += __popc(k);
        }
        __syncwarp();
        r = 0;
        for (int base = 0; base < m; base += 32) {
            const int idx = base + lane;
            const bool hole = idx < m && far_point(reg[idx]);
            const unsigned h = __ballot_sync(0xffffffffu, hole);
            if (hole) reg[idx] = reg[size - 1 - (r + __popc(h & below))];
            r += __popc(h);
        }
        __syncwarp();
        size = m;
        if (size < 2) return false;
        lsd_region2rect<V>(F, size, reg_angle, g.prec, g.p, rec);
        density = lsd_density(size, rec);
    }
    return true;
}

// ---- single-thread NFA (k_lsd_validate runs one thread per candidate rectangle: the arithmetic is scalar, so a warp validates 32
// rectangles instead of repeating the same doubles in 32 lanes) ----
__device__ __forceinline__ double lsd_log_gamma1(double x) {
    if (x > 15.0) return 0.918938533204673 + (x - 0.5) * log(x) - x + 0.5 * x * log(x * sinh(1 / x) + 1 / (810.0 * pow(x, 6.0)));
    const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
    double a = (x + 0.5) * log(x + 5.5) - (x + 5.5);
    double b = 0;
    for (int n = 0; n < 7; ++n) {
        a -= log(x + (double)n);
        b += q[n] * pow(x, (double)n);
    }
    return a + log(b);
}
__device__ __noinline__ double lsd_nfa_scalar(int n, int k, double p, double log_nt, const double* __restrict__ lgamma_tab) {
    if (n == 0 || k == 0) return -log_nt;
    if (n == k) return -log_nt - (double)n * log10(p);
    const double p_term = p / (1 - p);
    double lg0, lg1, lg2;
    if (n + 1 < LSD_LGAMMA_N) { lg0 = __ldg(lgamma_tab + n + 1); lg1 = __ldg(lgamma_tab + k + 1); lg2 = __ldg(lgamma_tab + n - k + 1); }
    else { lg0 = lsd_log_gamma1((double)n + 1); lg1 = lsd_log_gamma1((double)k + 1); lg2 = lsd_log_gamma1((double)(n - k) + 1); }
    const double log1term = lg0 - lg1 - lg2 + (double)k * log(p) + (double)(n - k) * log(1.0 - p);
    double term = exp(log1term);
    if (lsd_double_equal(term, 0)) {
        if (k > n * p) return -log1term / LSD_LN10 - log_nt;
        return -log_nt;
    }
    double bin_tail = term;
    const double tolerance = 0.1;
    for (int i = k + 1; i <= n; ++i) {
        const double bin_term = (double)(n - i + 1) / (double)i;
        const double mult_term = bin_term * p_term;
        term *= mult_term;
        bin_tail += term;
        if (bin_term < 1) {
            const double err = term * ((1 - pow(mult_term, (double)(n - i + 1))) / (1 - mult_term) - 1);
            if (err < tolerance * fabs(-log10(bin_tail) - log_nt) * bin_tail) break;
        }
    }
    return -log10(bin_tail) - log_nt;
}

// The validation evaluates the NFA at p = g.p / 2^j only (rect_improve halves p, exactly, at most ten times) and mostly at small n (on the benchmark's frames
// 99.998 % of the calls have n <= 512, the median is 19).  lsd_alloc therefore tabulates lsd_nfa_scalar itself, on the device, for every k <= n <= LSD_NFA_NMAX
// and j < LSD_NFA_NJ: a lookup returns the very double the scalar evaluation gives.  Other arguments fall back to lsd_nfa_scalar.
#define LSD_NFA_NMAX 512
#define LSD_NFA_NJ 11
#define LSD_NFA_TRI ((LSD_NFA_NMAX + 1) * (LSD_NFA_NMAX + 2) / 2)      // entries per j, at tri(n) + k with tri(n) = n (n + 1) / 2
__global__ void __launch_bounds__(256) k_lsd_nfa_table(LsdGeom g, double* __restrict__ tab) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= LSD_NFA_NJ * LSD_NFA_TRI) return;
    const int j = i / LSD_NFA_TRI, e = i - j * LSD_NFA_TRI;
    int n = (int)((sqrt(8.0 * e + 1.0) - 1.0) / 2.0);
    while (n * (n + 1) / 2 > e) --n;
    while ((n + 1) * (n + 2) / 2 <= e) ++n;
    double p = g.p;
    for (int t = 0; t < j; ++t) p /= 2;
    tab[i] = lsd_nfa_scalar(n, e - n * (n + 1) / 2, p, g.log_nt, g.lgamma_tab);
}
__device__ __forceinline__ double lsd_nfa(int n, int k, double p, const LsdGeom& g) {
    if (n <= LSD_NFA_NMAX) {
        const int j = ilogb(g.p) - ilogb(p);
        if (j >= 0 && j < LSD_NFA_NJ && p == ldexp(g.p, -j)) return __ldg(g.nfa_tab + j * LSD_NFA_TRI + n * (n + 1) / 2 + k);
    }
    return lsd_nfa_scalar(n, k, p, g.log_nt, g.lgamma_tab);
}

__device__ __forceinline__ double lsd_inter_low(double x, double x1, double y1, double x2, double y2) {
    if (lsd_double_equal(x1, x2) && y1 < y2) return y1;
    if (lsd_double_equal(x1, x2) && y1 > y2) return y2;
    return y1 + (x - x1) * (y2 - y1) / (x2 - x1);
}
__device__ __forceinline__ double lsd_inter_hi(double x, double x1, double y1, double x2, double y2) {
    if (lsd_double_equal(x1, x2) && y1 < y2) return y2;
    if (lsd_double_equal(x1, x2) && y1 > y2) return y1;
    return y1 + (x - x1) * (y2 - y1) / (x2 - x1);
}

// Point counts of the published LSD rectangle iterator for rectangle r: this lane visits the columns xa + sub, xa + sub + stride, ...
__device__ __forceinline__ void lsd_rect_count(const LsdFrame& F, const LsdRect& r, const LsdAlignSet& S, int sub, int stride, int& n, int& k) {
    double vx[4], vy[4], rx[4], ry[4];
    vx[0] = r.x1 - r.dy * r.width / 2.0; vy[0] = r.y1 + r.dx * r.width / 2.0;
    vx[1] = r.x2 - r.dy * r.width / 2.0; vy[1] = r.y2 + r.dx * r.width / 2.0;
    vx[2] = r.x2 + r.dy * r.width / 2.0; vy[2] = r.y2 - r.dx * r.width / 2.0;
    vx[3] = r.x1 + r.dy * r.width / 2.0; vy[3] = r.y1 - r.dx * r.width / 2.0;
    int offset;
    if (r.x1 < r.x2 && r.y1 <= r.y2) offset = 0;
    else if (r.x1 >= r.x2 && r.y1 < r.y2) offset = 1;
    else if (r.x1 > r.x2 && r.y1 >= r.y2) offset = 2;
    else offset = 3;
#pragma unroll
    for (int q = 0; q < 4; ++q) { rx[q] = vx[(offset + q) & 3]; ry[q] = vy[(offset + q) & 3]; }
    n = 0; k = 0;
    const int xa = (int)ceil(rx[0]), xb = (int)floor(rx[2]);
    for (int x = xa + sub; x <= xb; x += stride) {
        if (x < 0 || x >= F.W) continue;
        const double ys = (double)x < rx[3] ? lsd_inter_low(x, rx[0], ry[0], rx[3], ry[3]) : lsd_inter_low(x, rx[3], ry[3], rx[2], ry[2]);
        const double ye = (double)x < rx[1] ? lsd_inter_hi(x, rx[0], ry[0], rx[1], ry[1]) : lsd_inter_hi(x, rx[1], ry[1], rx[2], ry[2]);
        for (int y = (int)ceil(ys); (double)y <= ye; ++y) {
            if (y < 0 || y >= F.H) continue;
            ++n;
            const uint32_t wq = __ldg(F.ang + (size_t)y * F.W + x);           // validation runs after k_lsd_regions: the plane is read-only here
            k += lsd_word_aligned(S, wq);
        }
    }
}

// Point counts of cv2 4.x's rect_nfa enumeration (row spans from lsd_rectenum.h; points outside the image are not counted)
__device__ __forceinline__ void lsd_rect_count_cv4(const LsdFrame& F, const LsdRect& r, const LsdAlignSet& A, int& n, int& k) {
    LsdRowScan S;
    lsd_cv4_setup(r.x1, r.y1, r.x2, r.y2, r.width, r.dx, r.dy, S);
    n = 0; k = 0;
    const int ya = S.y0 < 0 ? 0 : S.y0, yb = S.c2 < F.H - 1 ? S.c2 : F.H - 1;
    for (int y = ya; y <= yb; ++y) {
        int xa, xb;
        lsd_cv4_row(S, y, xa, xb);
        if (xa < 0) xa = 0;
        if (xb > F.W - 1) xb = F.W - 1;
        for (int x = xa; x <= xb; ++x) {
            ++n;
            const uint32_t wq = __ldg(F.ang + (size_t)y * F.W + x);           // validation runs after k_lsd_regions: the plane is read-only here
            k += lsd_word_aligned(A, wq);
        }
    }
}

// rect_nfa of r; S = lsd_align_set(r.theta, r.prec)
__device__ __forceinline__ double lsd_rect_nfa(const LsdFrame& F, const LsdGeom& g, const LsdRect& r, const LsdAlignSet& S) {
    int n, k;
    if (g.rect_enum == 1) lsd_rect_count_cv4(F, r, S, n, k);
    else lsd_rect_count(F, r, S, 0, 1, n, k);
    return lsd_nfa(n, k, r.p, g);
}
// LineSegmentDetectorImpl::rect_improve after its first NFA evaluation (log_nfa = rect_nfa(rec) <= log_eps), one thread per rectangle.  (A warp per rectangle -
// lanes sharing the pixel count - was measured 3.8x slower while the NFA was evaluated in FP64 per call; with the NFA a table load and the pixel test integer
// compares, a lane group per rectangle has not been measured again.)
// Five precisions on one rectangle geometry (the first and the last stage of rect_improve halve p five times without touching the rectangle): the pixel walk does
// not depend on the precision, so one pass counts the aligned pixels for all five word sets.
__device__ __forceinline__ void lsd_rect_count_cv4_prec5(const LsdFrame& F, const LsdRect& r, const LsdAlignSet A[5], int& n, int k[5]) {
    LsdRowScan S;
    lsd_cv4_setup(r.x1, r.y1, r.x2, r.y2, r.width, r.dx, r.dy, S);
    n = 0;
#pragma unroll
    for (int j = 0; j < 5; ++j) k[j] = 0;
    const int ya = S.y0 < 0 ? 0 : S.y0, yb = S.c2 < F.H - 1 ? S.c2 : F.H - 1;
    for (int y = ya; y <= yb; ++y) {
        int xa, xb;
        lsd_cv4_row(S, y, xa, xb);
        if (xa < 0) xa = 0;
        if (xb > F.W - 1) xb = F.W - 1;
        for (int x = xa; x <= xb; ++x) {
            ++n;
            const uint32_t wq = __ldg(F.ang + (size_t)y * F.W + x);
#pragma unroll
            for (int j = 0; j < 5; ++j) k[j] += lsd_word_aligned(A[j], wq);
        }
    }
}
__device__ __noinline__ double lsd_rect_improve_rest(const LsdFrame& F, const LsdGeom& g, LsdRect& rec, double log_nfa) {
    const double delta = 0.5, delta_2 = delta / 2.0;
    LsdAlignSet S;
    for (int stage = 0; stage < 5; ++stage) {
        LsdRect r = rec;
        if ((stage == 0 || stage == 4) && g.rect_enum == 1) {
            if (stage == 0 || (r.width - delta) >= 0.5) {        // (the last stage carries the width test of the stages before it, like OpenCV's)
                double pv[5], precv[5];
                LsdAlignSet S5[5];
                int nn, kk[5];
                double pp = r.p;
#pragma unroll
                for (int n = 0; n < 5; ++n) { pp /= 2; pv[n] = pp; precv[n] = pp * LSD_PI; lsd_align_set(r.theta, precv[n], S5[n]); }
                lsd_rect_count_cv4_prec5(F, r, S5, nn, kk);
#pragma unroll
                for (int n = 0; n < 5; ++n) {
                    r.p = pv[n]; r.prec = precv[n];
                    const double v = lsd_nfa(nn, kk[n], r.p, g);
                    if (v > log_nfa) { log_nfa = v; rec = r; }
                }
            }
            if (stage < 4 && log_nfa > g.log_eps) return log_nfa;
            continue;
        }
        if (stage == 1) lsd_align_set(rec.theta, rec.prec, S);       // stages 1-3 move and narrow the rectangle but keep its angle and precision
        for (int n = 0; n < 5; ++n) {
            if (stage == 0) { r.p /= 2; r.prec = r.p * LSD_PI; }
            else {
                if (!((r.width - delta) >= 0.5)) continue;
                if (stage == 1) r.width -= delta;
                else if (stage == 2) { r.x1 += -r.dy * delta_2; r.y1 += r.dx * delta_2; r.x2 += -r.dy * delta_2; r.y2 += r.dx * delta_2; r.width -= delta; }
                else if (stage == 3) { r.x1 -= -r.dy * delta_2; r.y1 -= r.dx * delta_2; r.x2 -= -r.dy * delta_2; r.y2 -= r.dx * delta_2; r.width -= delta; }
                else { r.p /= 2; r.prec = r.p * LSD_PI; }
            }
            if (stage == 0 || stage == 4) lsd_align_set(r.theta, r.prec, S);
            const double v = lsd_rect_nfa(F, g, r, S);
            if (v > log_nfa) { log_nfa = v; rec = r; }
        }
        if (stage < 4 && log_nfa > g.log_eps) return log_nfa;
    }
    return log_nfa;
}

// Pseudo-ordering of the seeds (LineSegmentDetectorImpl::ll_angle's bucket sort): bin = int(norm * 1023 / max_norm) over the pixels with
// norm > rho, bins descending, row-major order inside a bin.  One CTA of 1024 threads per frame: warp w owns the w-th contiguous
// slice of the row-major pixel sequence; pass 1 counts per (warp, bin), a block scan turns the counts into start offsets
// (bins descending, warps ascending inside a bin), pass 2 scatters each slice in order (match_any ranks inside a warp), so the
// result is the stable sort.  Both passes recompute the gradient from the 8-bit scaled image (196 KB per frame) instead of
// reading the 16-byte records.
#define LSD_ORDER_THREADS 1024
#define LSD_ORDER_SMEM (32 * 1024 * 4)
__device__ __forceinline__ int lsd_order_bin(const uint8_t* __restrict__ s, int W, int x, int y, double rho, double bin_coef) {
    const size_t a = (size_t)y * W + x;
    const int DA = (int)s[a + W + 1] - (int)s[a], BC = (int)s[a + 1] - (int)s[a + W];
    const int gx = DA + BC, gy = DA - BC;
    const double nrm = lsd_norm(gx, gy);
    return nrm > rho ? (int)(nrm * bin_coef) : -1;
}
__global__ void __launch_bounds__(LSD_ORDER_THREADS) k_lsd_order(LsdGeom g, const uint8_t* __restrict__ scaled, const int32_t* __restrict__ smax,
                                                                uint32_t* __restrict__ order_all, int32_t* __restrict__ n_order) {
    extern __shared__ uint32_t s_cnt[];            // [32 warps][1024 bins]
    __shared__ uint32_t s_tot[1024];
    __shared__ uint32_t s_wsum[32];
    const int frame = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int sm = smax[frame];
    if (sm <= 0) { if (tid == 0) n_order[frame] = 0; return; }
    const size_t npx = (size_t)g.W * g.H;
    const uint8_t* s = scaled + (size_t)frame * npx;
    uint32_t* order = order_all + (size_t)frame * npx;
    const double max_grad = sqrt((double)sm / 4.0);
    const double bin_coef = (double)(1024 - 1) / max_grad;
    for (int t = tid; t < 32 * 1024; t += LSD_ORDER_THREADS) s_cnt[t] = 0;
    __syncthreads();
    const int Wm = g.W - 1, n_scan = Wm * (g.H - 1);
    const int per = ((n_scan + 31) / 32 + 31) & ~31;               // slice length, a multiple of 32 so that a warp load never straddles slices
    const int t0 = wid * per, t1 = min(n_scan, t0 + per);
    uint32_t* cnt = s_cnt + wid * 1024;
    for (int base = t0; base < t1; base += 32) {
        const int t = base + lane;
        int bin = -1;
        if (t < t1) { const int y = t / Wm, x = t - y * Wm; bin = lsd_order_bin(s, g.W, x, y, g.rho, bin_coef); }
        const unsigned peers = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0 && lane == __ffs(peers) - 1) cnt[bin] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    {   // thread b owns bin rb = 1023 - b (descending bins come first): total over the warps, block-exclusive scan, per-warp starts
        const int rb = 1023 - tid;
        uint32_t tot = 0;
        for (int w = 0; w < 32; ++w) tot += s_cnt[w * 1024 + rb];
        uint32_t incl = tot;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        if (lane == 31) s_wsum[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            uint32_t v = s_wsum[lane], iv = v;
            for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, iv, o); if (lane >= o) iv += u; }
            s_wsum[lane] = iv - v;
            if (lane == 31) n_order[frame] = (int32_t)iv;
        }
        __syncthreads();
        uint32_t run = s_wsum[wid] + incl - tot;
        for (int w = 0; w < 32; ++w) { const uint32_t c = s_cnt[w * 1024 + rb]; s_cnt[w * 1024 + rb] = run; run += c; }
        (void)s_tot;
    }
    __syncthreads();
    for (int base = t0; base < t1; base += 32) {
        const int t = base + lane;
        int bin = -1; uint32_t pix = 0;
        if (t < t1) { const int y = t / Wm, x = t - y * Wm; bin = lsd_order_bin(s, g.W, x, y, g.rho, bin_coef); pix = (uint32_t)x | ((uint32_t)y << 16); }
        const unsigned peers = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0) {
            const int rank = __popc(peers & ((1u << lane) - 1u));
            const int leader = __ffs(peers) - 1;
            uint32_t basep = 0;
            if (lane == leader) { basep = cnt[bin]; cnt[bin] = basep + __popc(peers); }
            basep = __shfl_sync(peers, basep, leader);
            order[basep + rank] = pix;
        }
        __syncwarp();
    }
}

// One warp (= one CTA) per frame: the sequential detection loop (LineSegmentDetectorImpl::flsd) over the seeds k_lsd_order prepared.
// V = resident CTAs per SM the build targets (register budget 65536 / (32 V)); the helpers above are instantiated per V so that each variant gets
// its own register allocation.  lsd_pipeline.cu picks the variant (default LSD_REGIONS_OCC, PSLAM_LSD_OCC overrides).
template <int V>
__global__ void __launch_bounds__(32, V) k_lsd_regions(LsdGeom g, int nframes, uint32_t* __restrict__ ang_all, const float2* __restrict__ cs_all, const uint32_t* __restrict__ gxy_all,
                                                    const int32_t* __restrict__ smax, uint32_t* __restrict__ reg_all, const uint32_t* __restrict__ order_all,
                                                    const int32_t* __restrict__ n_order, double* __restrict__ cands, int32_t* __restrict__ n_cand,
                                                    int32_t* __restrict__ status) {
    const int lane = threadIdx.x & 31;
    const int frame = blockIdx.x;
    if (frame >= nframes) return;
    const size_t npx = (size_t)g.W * g.H;
    LsdFrame F;
    F.ang = ang_all + (size_t)frame * npx; F.cs = cs_all + (size_t)frame * npx; F.gxy = gxy_all + (size_t)frame * npx; F.reg = reg_all + (size_t)frame * npx;
    F.order = const_cast<uint32_t*>(order_all) + (size_t)frame * npx; F.W = g.W; F.H = g.H;
    int count_out = 0;
    const int n_def = smax[frame] > 0 ? n_order[frame] : 0;
    {
        // ---- detection loop (k_lsd_gradient leaves every pixel unused) ----
        for (int base = 0; base < n_def; base += 32) {
            const uint32_t mypix = base + lane < n_def ? F.order[base + lane] : 0u;
            int last = -1;
            while (true) {
                bool fresh = false;
                if (base + lane < n_def && lane > last) fresh = !lsd_word_used(F.ang[(size_t)(mypix >> 16) * F.W + (mypix & 0xffff)]);
                const unsigned m = __ballot_sync(0xffffffffu, fresh);
                if (!m) break;
                const int j = __ffs(m) - 1;
                last = j;
                const uint32_t seed = __shfl_sync(0xffffffffu, mypix, j);
                const LsdGrown gr = lsd_region_grow<V>(F.ang, F.cs, F.reg, F.W, F.H, seed, g.prec);
                int size = gr.size;
                double reg_angle = gr.angle;
                if (size < g.min_reg_size) continue;
                LsdRect rc;
                lsd_region2rect<V>(F, size, reg_angle, g.prec, g.p, rc);
                if (g.refine > 0 && !lsd_refine<V>(F, g, size, reg_angle, rc)) continue;
                // candidate rectangle, in detection order; the NFA validation / improvement of LSD_REFINE_ADV does not touch
                // the 'used' map, so it runs afterwards with one thread per candidate (k_lsd_validate)
                if (count_out < g.cand_cap && lane < 12) {
                    const double v = lane == 0 ? rc.x1 : lane == 1 ? rc.y1 : lane == 2 ? rc.x2 : lane == 3 ? rc.y2 : lane == 4 ? rc.width : lane == 5 ? rc.x :
                                     lane == 6 ? rc.y : lane == 7 ? rc.theta : lane == 8 ? rc.dx : lane == 9 ? rc.dy : lane == 10 ? rc.prec : rc.p;
                    cands[((size_t)frame * g.cand_cap + count_out) * 12 + lane] = v;
                }
                ++count_out;
            }
        }
    }
    if (lane == 0) {
        n_cand[frame] = count_out;
        status[frame] = count_out > g.cand_cap ? 1 : 0;
    }
}

// LSD_REFINE_ADV: rect_improve + NFA threshold.  The validation never touches the 'used' map, so it is taken off the sequential per-frame chain and run
// for all candidates at once, one thread per candidate rectangle (the NFA arithmetic is scalar: a warp validates 32 rectangles).  Two kernels: most
// rectangles are meaningful at the first NFA evaluation, the others go through up to 25 more variants - run together, every warp would wait for its
// slowest lane, so k_lsd_validate does the first evaluation and queues the failures, and k_lsd_improve runs the remaining stages on the queue
// (dense warps of long-running candidates).  Queue order is irrelevant: every candidate writes its own slot.
__device__ __forceinline__ void lsd_load_cand(const double* __restrict__ c, LsdRect& rc) {
    rc.x1 = c[0]; rc.y1 = c[1]; rc.x2 = c[2]; rc.y2 = c[3]; rc.width = c[4]; rc.x = c[5]; rc.y = c[6]; rc.theta = c[7]; rc.dx = c[8]; rc.dy = c[9];
    rc.prec = c[10]; rc.p = c[11];
}
__global__ void __launch_bounds__(64) k_lsd_validate(LsdGeom g, const uint32_t* __restrict__ ang_all, const double* __restrict__ cands, const int32_t* __restrict__ n_cand,
                                                     double* __restrict__ cand_nfa, uint32_t* __restrict__ fail_list, int32_t* __restrict__ n_fail) {
    const int frame = blockIdx.y;
    const int ci = blockIdx.x * 64 + threadIdx.x;
    const int n = min(n_cand[frame], g.cand_cap);
    if (ci >= n) return;
    LsdFrame F;
    F.ang = const_cast<uint32_t*>(ang_all) + (size_t)frame * g.W * g.H; F.cs = nullptr; F.gxy = nullptr; F.reg = nullptr; F.order = nullptr; F.W = g.W; F.H = g.H;
    LsdRect rc;
    lsd_load_cand(cands + ((size_t)frame * g.cand_cap + ci) * 12, rc);
    LsdAlignSet S;
    lsd_align_set(rc.theta, rc.prec, S);
    const double log_nfa = lsd_rect_nfa(F, g, rc, S);
    cand_nfa[(size_t)frame * g.cand_cap + ci] = log_nfa;
    if (!(log_nfa > g.log_eps)) fail_list[(size_t)frame * g.cand_cap + atomicAdd(&n_fail[frame], 1)] = (uint32_t)ci;
}
__global__ void __launch_bounds__(64) k_lsd_improve(LsdGeom g, const uint32_t* __restrict__ ang_all, double* __restrict__ cands, double* __restrict__ cand_nfa,
                                                    const uint32_t* __restrict__ fail_list, const int32_t* __restrict__ n_fail) {
    const int frame = blockIdx.y;
    const int k = blockIdx.x * 64 + threadIdx.x;
    if (k >= n_fail[frame]) return;
    const int ci = (int)fail_list[(size_t)frame * g.cand_cap + k];
    LsdFrame F;
    F.ang = const_cast<uint32_t*>(ang_all) + (size_t)frame * g.W * g.H; F.cs = nullptr; F.gxy = nullptr; F.reg = nullptr; F.order = nullptr; F.W = g.W; F.H = g.H;
    double* c = cands + ((size_t)frame * g.cand_cap + ci) * 12;
    LsdRect rc;
    lsd_load_cand(c, rc);
    const double log_nfa = lsd_rect_improve_rest(F, g, rc, cand_nfa[(size_t)frame * g.cand_cap + ci]);
    c[0] = rc.x1; c[1] = rc.y1; c[2] = rc.x2; c[3] = rc.y2; c[4] = rc.width; c[11] = rc.p;
    cand_nfa[(size_t)frame * g.cand_cap + ci] = log_nfa;
}

// Accepted candidates -> output segments, detection order kept (one CTA of 256 threads per frame).
__global__ void __launch_bounds__(256) k_lsd_emit(LsdGeom g, const double* __restrict__ cands, const int32_t* __restrict__ n_cand, const double* __restrict__ cand_nfa,
                                                  float4* __restrict__ segs, double* __restrict__ wpn, int32_t* __restrict__ n_segs, int32_t* __restrict__ status) {
    __shared__ int s_warp[8];
    __shared__ int s_base;
    const int frame = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int n = min(n_cand[frame], g.cand_cap);
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int c0 = 0; c0 < n; c0 += 256) {
        const int ci = c0 + tid;
        bool keep = false;
        double nfa = -1;
        if (ci < n) {
            if (g.refine >= 2) { nfa = cand_nfa[(size_t)frame * g.cand_cap + ci]; keep = nfa > g.log_eps; }
            else keep = true;
        }
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[wid] = __popc(m);
        __syncthreads();
        int off = s_base;
        for (int w = 0; w < wid; ++w) off += s_warp[w];
        const int slot = off + __popc(m & ((1u << lane) - 1u));
        if (keep && slot < g.seg_cap) {
            const double* c = cands + ((size_t)frame * g.cand_cap + ci) * 12;
            double x1 = c[0], y1 = c[1], x2 = c[2], y2 = c[3], width = c[4];
            x1 += 0.5; y1 += 0.5; x2 += 0.5; y2 += 0.5;
            x1 /= 0.8; y1 /= 0.8; x2 /= 0.8; y2 /= 0.8; width /= 0.8;
            segs[(size_t)frame * g.seg_cap + slot] = make_float4((float)x1, (float)y1, (float)x2, (float)y2);
            double* o = wpn + ((size_t)frame * g.seg_cap + slot) * 3;
            o[0] = width; o[1] = c[11]; o[2] = nfa;
        }
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < 8; ++w) t += s_warp[w]; s_base += t; }
        __syncthreads();
    }
    if (tid == 0) {
        n_segs[frame] = s_base;
        if (s_base > g.seg_cap) status[frame] |= 2;
    }
}

// cv::line_descriptor::KeyLine, 68 bytes (opencv_contrib line_descriptor/descriptor.hpp)
struct LsdKeyLine {
    float angle; int32_t class_id; int32_t octave; float pt_x, pt_y; float response; float size;
    float startPointX, startPointY, endPointX, endPointY, sPointInOctaveX, sPointInOctaveY, ePointInOctaveX, ePointInOctaveY;
    float lineLength; int32_t numOfPixels;
};

// LSDDetector::detectImpl's KeyLine fields for octave 0 + ExtractLineSegment's "keep the max_lines longest" + line functions.
// One CTA (128 threads) per frame; rank by (response descending, detection index ascending).
__global__ void __launch_bounds__(128) k_lsd_keylines(LsdGeom g, int max_lines, const float4* __restrict__ segs, const int32_t* __restrict__ n_segs,
                                                      LsdKeyLine* __restrict__ kls, double* __restrict__ lfs, int32_t* __restrict__ n_kl) {
    extern __shared__ float s_resp[];
    const int frame = blockIdx.x;
    const int n = min(n_segs[frame], g.seg_cap);
    const float4* S = segs + (size_t)frame * g.seg_cap;
    const float fw = (float)g.w, fh = (float)g.h;
    auto clampx = [&](float v) { if (v < 0) v = 0; if (v >= fw) v = fw - 1.0f; return v; };
    auto clampy = [&](float v) { if (v < 0) v = 0; if (v >= fh) v = fh - 1.0f; return v; };
    for (int i = threadIdx.x; i < n; i += 128) {
        const float4 e = S[i];
        const float x0 = clampx(e.x), y0 = clampy(e.y), x1 = clampx(e.z), y1 = clampy(e.w);
        const double ddx = (double)__fsub_rn(x0, x1), ddy = (double)__fsub_rn(y0, y1);      // pow(float, 2) promotes to double; x * x is exact there
        const float len = (float)sqrt(ddx * ddx + ddy * ddy);
        s_resp[i] = __fdiv_rn(len, (float)max(g.w, g.h));
    }
    __syncthreads();
    const int keep = min(n, max_lines);
    for (int i = threadIdx.x; i < n; i += 128) {
        const float r = s_resp[i];
        int rank = 0;
        for (int j = 0; j < n; ++j) { const float q = s_resp[j]; rank += (q > r) || (q == r && j < i); }
        if (n > max_lines && rank >= max_lines) continue;
        const int slot = n > max_lines ? rank : i;            // no sort when nothing is dropped (src/LSDextractor.cpp:21)
        const float4 e = S[i];
        LsdKeyLine k;
        k.startPointX = clampx(e.x); k.startPointY = clampy(e.y); k.endPointX = clampx(e.z); k.endPointY = clampy(e.w);
        k.sPointInOctaveX = k.startPointX; k.sPointInOctaveY = k.startPointY; k.ePointInOctaveX = k.endPointX; k.ePointInOctaveY = k.endPointY;
        const double ddx = (double)__fsub_rn(k.startPointX, k.endPointX), ddy = (double)__fsub_rn(k.startPointY, k.endPointY);
        k.lineLength = (float)sqrt(ddx * ddx + ddy * ddy);
        const int ax = __float2int_rn(k.startPointX), ay = __float2int_rn(k.startPointY), bx = __float2int_rn(k.endPointX), by = __float2int_rn(k.endPointY);
        k.numOfPixels = max(abs(bx - ax), abs(by - ay)) + 1;
        k.angle = (float)atan2((double)__fsub_rn(k.endPointY, k.startPointY), (double)__fsub_rn(k.endPointX, k.startPointX));
        k.class_id = slot;
        k.octave = 0;
        k.size = __fmul_rn(__fsub_rn(k.endPointX, k.startPointX), __fsub_rn(k.endPointY, k.startPointY));
        k.response = r;
        k.pt_x = __fdiv_rn(__fadd_rn(k.endPointX, k.startPointX), 2.f); k.pt_y = __fdiv_rn(__fadd_rn(k.endPointY, k.startPointY), 2.f);
        kls[(size_t)frame * max_lines + slot] = k;
        const double sp[3] = {(double)k.startPointX, (double)k.startPointY, 1.0}, ep[3] = {(double)k.endPointX, (double)k.endPointY, 1.0};
        const double l0 = sp[1] * ep[2] - sp[2] * ep[1], l1 = sp[2] * ep[0] - sp[0] * ep[2], l2 = sp[0] * ep[1] - sp[1] * ep[0];
        const double nn = sqrt(l0 * l0 + l1 * l1 + l2 * l2);
        double* lf = lfs + ((size_t)frame * max_lines + slot) * 3;
        lf[0] = l0 / nn; lf[1] = l1 / nn; lf[2] = l2 / nn;
    }
    if (threadIdx.x == 0) n_kl[frame] = keep;
}

}  // namespace pslam
