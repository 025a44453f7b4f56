// Host side of the line-segment detector: geometry / tables (down-scaling taps, the (gx, gy) -> cosf / sinf table built with
// the host libm the OpenCV binary itself would call), buffer management, launches, C ABI.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <string>

#include "lsd_kernels.cuh"
#include "lbd_kernels.cuh"

namespace pslam {

struct LsdBuffers {
    LsdGeom g;
    int max_batch = 0, last_n = 0, max_lines_cap = 0;
    int16_t *d_ix = nullptr, *d_ax = nullptr, *d_iy = nullptr, *d_ay = nullptr;
    float2* d_lut = nullptr; double* d_lgamma = nullptr; double* d_nfa = nullptr;
    uint8_t* d_gray = nullptr;        // staging for the host-pointer entry points
    uint8_t* d_scaled = nullptr; uint32_t* d_ang = nullptr; float2* d_cs = nullptr; uint32_t* d_gxy = nullptr; int32_t* d_smax = nullptr;
    uint32_t* d_reg = nullptr; uint32_t* d_order = nullptr; int32_t* d_norder = nullptr;
    double* d_cands = nullptr; double* d_cand_nfa = nullptr; int32_t* d_ncand = nullptr;
    uint32_t* d_fail = nullptr; int32_t* d_nfail = nullptr;      // candidates whose first NFA evaluation fails (queue of k_lsd_improve)
    float4* d_segs = nullptr; double* d_wpn = nullptr; int32_t* d_nsegs = nullptr; int32_t* d_status = nullptr;
    LsdKeyLine* d_kl = nullptr; double* d_lf = nullptr; int32_t* d_nkl = nullptr;
    int16_t *d_dx = nullptr, *d_dy = nullptr; float *d_glocal = nullptr, *d_gglobal = nullptr; uint8_t* d_ldesc = nullptr; float* d_lbd72 = nullptr;   // LBD (lbd_kernels.cuh)
    std::vector<int32_t> h_n, h_status;
};

static int lsd_cv_round(double v) { return (int)std::nearbyint(v); }            // round half to even (default rounding mode)

static float host_fast_atan2_deg(float y, float x) {                               // cv::fastAtan2
    const float p1 = 0.9997878412794807f * (float)(180 / 3.14159265358979323846);
    const float p3 = -0.3258083974640975f * (float)(180 / 3.14159265358979323846);
    const float p5 = 0.1555786518463281f * (float)(180 / 3.14159265358979323846);
    const float p7 = -0.04432655554792128f * (float)(180 / 3.14159265358979323846);
    const float ax = std::fabs(x), ay = std::fabs(y);
    float a, c, c2;
    if (ax >= ay) { c = ay / (ax + (float)DBL_EPSILON); c2 = c * c; a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c; }
    else { c = ax / (ay + (float)DBL_EPSILON); c2 = c * c; a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c; }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

static const int LSD_SEG_CAP = 4096;
#define LSD_REGIONS_OCC 24          // resident region-growing warps per SM the default build of k_lsd_regions targets

int lsd_alloc(pslam_ctx* c) {
    if (c->lsd) return PSLAM_OK;
    LsdBuffers* Bp = new LsdBuffers();
    LsdBuffers& B = *Bp;
    LsdGeom& g = B.g;
    g.w = c->cfg.width; g.h = c->cfg.height;
    const double SCALE = 0.8, ANG_TH = 22.5, QUANT = 2.0;
    g.W = lsd_cv_round(g.w * SCALE); g.H = lsd_cv_round(g.h * SCALE);
    if (g.W < 8 || g.H < 8 || g.W > 32767 || g.H > 32767) { delete Bp; return set_error(c, PSLAM_E_INVALID, "image size unsupported by the line-segment detector"); }
    g.refine = 2;
    // candidate / segment capacity per frame: 4096 at 640x480 (a textured frame yields a few hundred), scaled with the image area above that
    g.seg_cap = g.cand_cap = std::max(LSD_SEG_CAP, (int)(((long long)LSD_SEG_CAP * g.w * g.h / (640 * 480) + 1023) / 1024 * 1024));
    {   // default enumeration of the NFA validation = OpenCV 4.x rect_nfa (the variant the oracle pins to cv2 4.13); PSLAM_LSD_RECT_ENUM=published
        // or pslam_lsd_set_rect_enumeration(ctx, 0) select the published LSD iterator
        const char* e = std::getenv("PSLAM_LSD_RECT_ENUM");
        g.rect_enum = (e && (!std::strcmp(e, "published") || !std::strcmp(e, "0"))) ? 0 : 1;
    }
    g.prec = LSD_PI * ANG_TH / 180; g.p = ANG_TH / 180; g.rho = QUANT / std::sin(g.prec);
    g.log_nt = 5 * (std::log10(double(g.W)) + std::log10(double(g.H))) / 2 + std::log10(11.0);
    g.min_reg_size = (int)(size_t)(-g.log_nt / std::log10(g.p));
    g.density_th = 0.7; g.log_eps = 0;
    B.max_batch = c->cfg.max_batch;
    // INTER_LINEAR_EXACT taps (8.8 fixed point)
    // cv::resize(src, dst, Size(), 0.8, 0.8, INTER_LINEAR_EXACT): destination size cvRound(0.8 * size), sampling step exactly 1 / 0.8 (not src / dst;
    // the two coincide when 0.8 * size is an integer, e.g. 640 x 480 and 1280 x 960)
    auto coef = [SCALE](int dn, int sn, std::vector<int16_t>& idx, std::vector<int16_t>& a) {
        idx.resize(dn); a.resize(dn);
        const double scale = 1.0 / SCALE;
        for (int d = 0; d < dn; ++d) {
            const double f = (d + 0.5) * scale - 0.5;
            int i = (int)std::floor(f);
            double fr = f - i;
            if (i < 0) { i = 0; fr = 0; }
            if (i >= sn - 1) { i = sn - 1; fr = 0; }
            idx[d] = (int16_t)i; a[d] = (int16_t)std::floor(fr * 256 + 0.5);
        }
    };
    std::vector<int16_t> ix, ax, iy, ay;
    coef(g.W, g.w, ix, ax); coef(g.H, g.h, iy, ay);
    // the blur / scale kernel stages (tile * 1.25 + 6) source pixels: check the compiled bounds
    for (int X0 = 0; X0 < g.W; X0 += LSD_TW) {
        const int X1 = std::min(X0 + LSD_TW, g.W) - 1;
        if (std::min(ix[X1] + 1, g.w - 1) - ix[X0] + 5 > LSD_SW) { delete Bp; return set_error(c, PSLAM_E_INVALID, "LSD tile bound (width)"); }
    }
    for (int Y0 = 0; Y0 < g.H; Y0 += LSD_TH) {
        const int Y1 = std::min(Y0 + LSD_TH, g.H) - 1;
        if (std::min(iy[Y1] + 1, g.h - 1) - iy[Y0] + 5 > LSD_SH) { delete Bp; return set_error(c, PSLAM_E_INVALID, "LSD tile bound (height)"); }
    }
    // cosf / sinf of the level-line angle for every possible gradient: the float sums of region_grow use libm's float routines
    std::vector<float2> lut((size_t)1021 * 1021);
    for (int gx = -510; gx <= 510; ++gx)
        for (int gy = -510; gy <= 510; ++gy) {
            const double ang = (double)host_fast_atan2_deg((float)gx, (float)(-gy)) * LSD_DEG2RAD;
            const float af = (float)ang;
            lut[(size_t)(gx + 510) * 1021 + (gy + 510)] = make_float2(std::cos(af), std::sin(af));
        }
    // log_gamma(i), i = 0 .. LSD_LGAMMA_N - 1, with the reference's two approximations (lsd.cpp log_gamma_lanczos / _windschitl)
    std::vector<double> lgam(LSD_LGAMMA_N, 0.0);
    for (int i = 1; i < LSD_LGAMMA_N; ++i) {
        const double x = (double)i;
        if (x > 15.0) lgam[i] = 0.918938533204673 + (x - 0.5) * std::log(x) - x + 0.5 * x * std::log(x * std::sinh(1 / x) + 1 / (810.0 * std::pow(x, 6.0)));
        else {
            static const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
            double a = (x + 0.5) * std::log(x + 5.5) - (x + 5.5), b = 0;
            for (int n = 0; n < 7; ++n) { a -= std::log(x + double(n)); b += q[n] * std::pow(x, double(n)); }
            lgam[i] = a + std::log(b);
        }
    }
    const size_t npx = (size_t)g.W * g.H, nb = (size_t)B.max_batch;
#define LA(ptr, bytes) do { const int rc_ = check_cuda(c, cudaMalloc((void**)&(ptr), (bytes)), "cudaMalloc(lsd)"); if (rc_ != PSLAM_OK) { c->lsd = Bp; lsd_free(c); return rc_; } } while (0)
    LA(B.d_ix, g.W * 2); LA(B.d_ax, g.W * 2); LA(B.d_iy, g.H * 2); LA(B.d_ay, g.H * 2); LA(B.d_lut, lut.size() * sizeof(float2)); LA(B.d_lgamma, LSD_LGAMMA_N * 8);
    LA(B.d_nfa, (size_t)LSD_NFA_NJ * LSD_NFA_TRI * 8);
    LA(B.d_gray, nb * g.w * g.h); LA(B.d_scaled, nb * npx); LA(B.d_ang, nb * npx * 4); LA(B.d_cs, nb * npx * 8); LA(B.d_gxy, nb * npx * 4); LA(B.d_smax, nb * 4);
    LA(B.d_reg, nb * npx * 4); LA(B.d_order, nb * npx * 4); LA(B.d_norder, nb * 4);
    LA(B.d_fail, nb * g.cand_cap * 4); LA(B.d_nfail, nb * 4);
    LA(B.d_cands, nb * g.cand_cap * 12 * 8); LA(B.d_cand_nfa, nb * g.cand_cap * 8); LA(B.d_ncand, nb * 4);
    LA(B.d_segs, nb * g.seg_cap * sizeof(float4)); LA(B.d_wpn, nb * g.seg_cap * 3 * 8); LA(B.d_nsegs, nb * 4); LA(B.d_status, nb * 4);
#undef LA
    cudaStream_t st = c->stream;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_ix, ix.data(), g.W * 2, cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_ax, ax.data(), g.W * 2, cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_iy, iy.data(), g.H * 2, cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_ay, ay.data(), g.H * 2, cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_lut, lut.data(), lut.size() * sizeof(float2), cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_lgamma, lgam.data(), LSD_LGAMMA_N * 8, cudaMemcpyHostToDevice, st));
    g.lgamma_tab = B.d_lgamma;
    g.nfa_tab = B.d_nfa;
    // the NFA table (lsd_nfa): 11 x 131841 entries, evaluated by the device's own lsd_nfa_scalar so that every entry is the double the kernels computed without it
    k_lsd_nfa_table<<<(LSD_NFA_NJ * LSD_NFA_TRI + 255) / 256, 256, 0, st>>>(g, B.d_nfa);
    PSLAM_CUDA(c, cudaGetLastError());
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    c->lsd = Bp;
    return PSLAM_OK;
}

void lsd_free(pslam_ctx* c) {
    if (!c->lsd) return;
    LsdBuffers& B = *c->lsd;
    for (void* p : {(void*)B.d_ix, (void*)B.d_ax, (void*)B.d_iy, (void*)B.d_ay, (void*)B.d_lut, (void*)B.d_lgamma, (void*)B.d_nfa, (void*)B.d_gray, (void*)B.d_scaled, (void*)B.d_ang, (void*)B.d_cs, (void*)B.d_gxy,
                    (void*)B.d_smax, (void*)B.d_reg, (void*)B.d_order, (void*)B.d_norder, (void*)B.d_segs, (void*)B.d_wpn,
                    (void*)B.d_nsegs, (void*)B.d_status, (void*)B.d_cands, (void*)B.d_cand_nfa, (void*)B.d_ncand, (void*)B.d_fail, (void*)B.d_nfail, (void*)B.d_kl, (void*)B.d_lf, (void*)B.d_nkl, (void*)B.d_dx, (void*)B.d_dy, (void*)B.d_glocal, (void*)B.d_gglobal,
                    (void*)B.d_ldesc, (void*)B.d_lbd72})
        if (p) cudaFree(p);
    delete c->lsd;
    c->lsd = nullptr;
}

// detection on device-resident frames; results stay in the context's buffers
int lsd_detect_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, int refine) {
    int rc = lsd_alloc(c);
    if (rc != PSLAM_OK) return rc;
    LsdBuffers& B = *c->lsd;
    if (nframes < 1 || nframes > B.max_batch) return set_error(c, PSLAM_E_INVALID, "nframes outside [1, max_batch]");
    if (refine < 0 || refine > 2) return set_error(c, PSLAM_E_INVALID, "refine must be 0, 1 or 2");
    LsdGeom g = B.g;
    g.refine = refine;
    cudaStream_t st = c->stream;
    const size_t npx = (size_t)g.W * g.H;
    PSLAM_CUDA(c, cudaMemsetAsync(B.d_smax, 0, (size_t)nframes * 4, st));
    const dim3 gb((g.W + LSD_TW - 1) / LSD_TW, (g.H + LSD_TH - 1) / LSD_TH, nframes);
    PSLAM_LAUNCH(c, "lsd_blur_scale", k_lsd_blur_scale<<<gb, 256, 0, st>>>(g, d_gray, B.d_ix, B.d_ax, B.d_iy, B.d_ay, B.d_scaled));
    if ((g.W & 3) == 0 && !std::getenv("PSLAM_LSD_GRADIENT1")) {        // four pixels per thread when a row is a whole number of words (buffers are 256-byte aligned)
        const dim3 gg4(((g.W >> 2) + 63) / 64, (g.H + 3) / 4, nframes);
        PSLAM_LAUNCH(c, "lsd_gradient", k_lsd_gradient4<<<gg4, 256, 0, st>>>(g, B.d_scaled, B.d_lut, B.d_ang, B.d_cs, B.d_gxy, B.d_smax));
    } else {
        const dim3 gg((g.W + 63) / 64, (g.H + 3) / 4, nframes);
        PSLAM_LAUNCH(c, "lsd_gradient", k_lsd_gradient<<<gg, 256, 0, st>>>(g, B.d_scaled, B.d_lut, B.d_ang, B.d_cs, B.d_gxy, B.d_smax));
    }
    PSLAM_CUDA(c, cudaFuncSetAttribute(k_lsd_order, cudaFuncAttributeMaxDynamicSharedMemorySize, LSD_ORDER_SMEM));
    if ((size_t)B.g.seg_cap * sizeof(float) > 48 * 1024) {
        if ((size_t)B.g.seg_cap * sizeof(float) > 227 * 1024) return set_error(c, PSLAM_E_INVALID, "image too large for the key-line ranking buffer");
        PSLAM_CUDA(c, cudaFuncSetAttribute(k_lsd_keylines, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(B.g.seg_cap * sizeof(float))));
    }
    PSLAM_LAUNCH(c, "lsd_order", k_lsd_order<<<nframes, LSD_ORDER_THREADS, LSD_ORDER_SMEM, st>>>(g, B.d_scaled, B.d_smax, B.d_order, B.d_norder));
    {
        static const int occ = [] { const char* e = std::getenv("PSLAM_LSD_OCC"); const int v = e ? std::atoi(e) : LSD_REGIONS_OCC; return v == 16 || v == 20 || v == 24 || v == 32 ? v : LSD_REGIONS_OCC; }();
#define LSD_REGIONS_LAUNCH(V) PSLAM_LAUNCH(c, "lsd_regions", k_lsd_regions<V><<<nframes, 32, 0, st>>>(g, nframes, B.d_ang, B.d_cs, B.d_gxy, B.d_smax, B.d_reg, B.d_order, B.d_norder, \
                                                                                                B.d_cands, B.d_ncand, B.d_status))
        if (occ == 16) LSD_REGIONS_LAUNCH(16); else if (occ == 20) LSD_REGIONS_LAUNCH(20); else if (occ == 24) LSD_REGIONS_LAUNCH(24); else LSD_REGIONS_LAUNCH(32);
#undef LSD_REGIONS_LAUNCH
    }
    if (refine >= 2) {
        // grid.x covers the candidate capacity; warps beyond a frame's candidate count exit at once
        const dim3 gv((g.cand_cap + 63) / 64, nframes);
        PSLAM_CUDA(c, cudaMemsetAsync(B.d_nfail, 0, (size_t)nframes * 4, st));
        PSLAM_LAUNCH(c, "lsd_validate", k_lsd_validate<<<gv, 64, 0, st>>>(g, B.d_ang, B.d_cands, B.d_ncand, B.d_cand_nfa, B.d_fail, B.d_nfail));
        PSLAM_LAUNCH(c, "lsd_improve", k_lsd_improve<<<gv, 64, 0, st>>>(g, B.d_ang, B.d_cands, B.d_cand_nfa, B.d_fail, B.d_nfail));
    }
    PSLAM_LAUNCH(c, "lsd_emit", k_lsd_emit<<<nframes, 256, 0, st>>>(g, B.d_cands, B.d_ncand, B.d_cand_nfa, B.d_segs, B.d_wpn, B.d_nsegs, B.d_status));
    PSLAM_CUDA(c, cudaGetLastError());
    B.last_n = nframes;
    return PSLAM_OK;
}

int lsd_status_fetch_async(pslam_ctx* c, int nframes, int32_t* h_pinned) {      // capacity flags of the most recent detection (frame_pipeline.cu)
    if (!c->lsd) return set_error(c, PSLAM_E_INVALID, "no line detection has run");
    PSLAM_CUDA(c, cudaMemcpyAsync(h_pinned, c->lsd->d_status, (size_t)nframes * 4, cudaMemcpyDeviceToHost, c->stream));
    return PSLAM_OK;
}

int lsd_keylines_dev(pslam_ctx* c, int nframes, int max_lines, LsdKeyLine* d_kl, double* d_lf, int32_t* d_n) {
    LsdBuffers& B = *c->lsd;
    PSLAM_LAUNCH(c, "lsd_keylines", k_lsd_keylines<<<nframes, 128, B.g.seg_cap * sizeof(float), c->stream>>>(B.g, max_lines, B.d_segs, B.d_nsegs, d_kl, d_lf, d_n));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_lsd_max_segments(const pslam_ctx* c) {
    if (!c) return 0;
    return std::max(LSD_SEG_CAP, (int)(((long long)LSD_SEG_CAP * c->cfg.width * c->cfg.height / (640 * 480) + 1023) / 1024 * 1024));
}

int pslam_lsd_set_rect_enumeration(pslam_ctx* c, int mode) {
    if (!c) return PSLAM_E_INVALID;
    if (mode != 0 && mode != 1) return set_error(c, PSLAM_E_INVALID, "rect enumeration: 0 (published LSD iterator) or 1 (OpenCV 4.x rect_nfa)");
    const int rc = lsd_alloc(c);
    if (rc != PSLAM_OK) return rc;
    c->lsd->g.rect_enum = mode;
    return PSLAM_OK;
}

static int lsd_upload(pslam_ctx* c, const uint8_t* gray, int nframes) {
    int rc = lsd_alloc(c);
    if (rc != PSLAM_OK) return rc;
    LsdBuffers& B = *c->lsd;
    if (nframes < 1 || nframes > B.max_batch) return set_error(c, PSLAM_E_INVALID, "nframes outside [1, max_batch]");
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_gray, gray, (size_t)nframes * B.g.w * B.g.h, cudaMemcpyHostToDevice, c->stream));
    return PSLAM_OK;
}

int pslam_lsd_detect_batch(pslam_ctx* c, const uint8_t* gray, int nframes, int refine, float* segs, double* wpn, int cap, int32_t* n) {
    if (!c) return PSLAM_E_INVALID;
    if (!gray || !segs || !n || cap < 1) return set_error(c, PSLAM_E_INVALID, "null pointer or cap < 1");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    int rc = lsd_upload(c, gray, nframes);
    if (rc != PSLAM_OK) return rc;
    LsdBuffers& B = *c->lsd;
    if ((rc = lsd_detect_dev(c, B.d_gray, nframes, refine)) != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    B.h_n.resize(nframes); B.h_status.resize(nframes);
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_n.data(), B.d_nsegs, nframes * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_status.data(), B.d_status, nframes * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    rc = PSLAM_OK;
    for (int f = 0; f < nframes; ++f) {
        n[f] = B.h_n[f];
        const int m = std::min(std::min(B.h_n[f], cap), B.g.seg_cap);
        if (B.h_n[f] > cap || B.h_status[f]) rc = set_error(c, PSLAM_E_CAPACITY, "more line segments than the capacity");
        if (m) {
            PSLAM_CUDA(c, cudaMemcpyAsync(segs + (size_t)f * cap * 4, B.d_segs + (size_t)f * B.g.seg_cap, (size_t)m * 16, cudaMemcpyDeviceToHost, st));
            if (wpn) PSLAM_CUDA(c, cudaMemcpyAsync(wpn + (size_t)f * cap * 3, B.d_wpn + (size_t)f * B.g.seg_cap * 3, (size_t)m * 24, cudaMemcpyDeviceToHost, st));
        }
    }
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    return rc;
}

static int lsd_ensure_kl(pslam_ctx* c, int max_lines) {
    LsdBuffers& B = *c->lsd;
    if (max_lines <= B.max_lines_cap) return PSLAM_OK;
    if (B.d_kl) cudaFree(B.d_kl);
    if (B.d_lf) cudaFree(B.d_lf);
    if (B.d_nkl) cudaFree(B.d_nkl);
    if (B.d_ldesc) cudaFree(B.d_ldesc);
    if (B.d_lbd72) cudaFree(B.d_lbd72);
    B.d_kl = nullptr; B.d_lf = nullptr; B.d_nkl = nullptr; B.d_ldesc = nullptr; B.d_lbd72 = nullptr; B.max_lines_cap = 0;
    PSLAM_CUDA(c, cudaMalloc((void**)&B.d_kl, (size_t)B.max_batch * max_lines * sizeof(LsdKeyLine)));
    PSLAM_CUDA(c, cudaMalloc((void**)&B.d_lf, (size_t)B.max_batch * max_lines * 24));
    PSLAM_CUDA(c, cudaMalloc((void**)&B.d_nkl, (size_t)B.max_batch * 4));
    PSLAM_CUDA(c, cudaMalloc((void**)&B.d_ldesc, (size_t)B.max_batch * max_lines * 32));
    PSLAM_CUDA(c, cudaMalloc((void**)&B.d_lbd72, (size_t)B.max_batch * max_lines * 72 * 4));
    B.max_lines_cap = max_lines;
    return PSLAM_OK;
}

// BinaryDescriptor::compute on the key lines the detector left on the device (src/LSDextractor.cpp:28)
static int lbd_describe_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, int max_lines, const LsdKeyLine* d_kl, const int32_t* d_n, uint8_t* d_desc, float* d_lbd72) {
    LsdBuffers& B = *c->lsd;
    const LsdGeom& g = B.g;
    cudaStream_t st = c->stream;
    if (!B.d_dx) {
        const size_t bytes = (size_t)B.max_batch * g.w * g.h * sizeof(int16_t);
        PSLAM_CUDA(c, cudaMalloc((void**)&B.d_dx, bytes)); PSLAM_CUDA(c, cudaMalloc((void**)&B.d_dy, bytes));
        PSLAM_CUDA(c, cudaMalloc((void**)&B.d_glocal, LBD_WIDTH * 3 * 4)); PSLAM_CUDA(c, cudaMalloc((void**)&B.d_gglobal, LBD_HEIGHT * 4));
        float gl[LBD_WIDTH * 3], gg[LBD_HEIGHT];               // the two Gaussian windows, evaluated with the host libm like upstream (integer-division sigmas)
        { const double u = (double)((LBD_WIDTH * 3 - 1) / 2), sigma = (double)((LBD_WIDTH * 2 + 1) / 2), inv = -1 / (2 * sigma * sigma);
          for (int i = 0; i < LBD_WIDTH * 3; ++i) { const double d = i - u; gl[i] = (float)std::exp(d * d * inv); } }
        { const double u = (double)((LBD_HEIGHT - 1) / 2), sigma = u, inv = -1 / (2 * sigma * sigma);
          for (int i = 0; i < LBD_HEIGHT; ++i) { const double d = i - u; gg[i] = (float)std::exp(d * d * inv); } }
        PSLAM_CUDA(c, cudaMemcpy(B.d_glocal, gl, sizeof gl, cudaMemcpyHostToDevice));
        PSLAM_CUDA(c, cudaMemcpy(B.d_gglobal, gg, sizeof gg, cudaMemcpyHostToDevice));
    }
    const dim3 gb((g.w + LBD_TW - 1) / LBD_TW, (g.h + LBD_TH - 1) / LBD_TH, nframes);
    PSLAM_LAUNCH(c, "lbd_gradients", k_lbd_gradients<<<gb, 256, 0, st>>>(d_gray, g.w, g.h, B.d_dx, B.d_dy));
    PSLAM_LAUNCH(c, "lbd_lines", k_lbd_lines<<<dim3(max_lines, nframes), 64, 0, st>>>(B.d_dx, B.d_dy, g.w, g.h, d_kl, d_n, max_lines, B.d_glocal, B.d_gglobal, d_desc, d_lbd72));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

int pslam_lines_extract_describe_batch_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, int max_lines, pslam_keyline* d_kl, double* d_lf, uint8_t* d_desc, int32_t* d_n) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_desc) return set_error(c, PSLAM_E_INVALID, "null descriptor buffer");
    int rc = pslam_lines_extract_batch_dev(c, d_gray, nframes, max_lines, d_kl, d_lf, d_n);
    if (rc != PSLAM_OK) return rc;
    return lbd_describe_dev(c, d_gray, nframes, max_lines, (const LsdKeyLine*)d_kl, d_n, d_desc, nullptr);
}

int pslam_lines_extract_describe_batch(pslam_ctx* c, const uint8_t* gray, int nframes, int max_lines, pslam_keyline* kl, double* lf, uint8_t* desc, float* lbd72, int32_t* n) {
    if (!c) return PSLAM_E_INVALID;
    if (!desc) return set_error(c, PSLAM_E_INVALID, "null descriptor buffer");
    int rc = pslam_lines_extract_batch(c, gray, nframes, max_lines, kl, lf, n);       // uploads the frames into the context's staging buffer and leaves the key lines there
    if (rc != PSLAM_OK) return rc;
    LsdBuffers& B = *c->lsd;
    if ((rc = lbd_describe_dev(c, B.d_gray, nframes, max_lines, B.d_kl, B.d_nkl, B.d_ldesc, B.d_lbd72)) != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    PSLAM_CUDA(c, cudaMemcpyAsync(desc, B.d_ldesc, (size_t)nframes * max_lines * 32, cudaMemcpyDeviceToHost, st));
    if (lbd72) PSLAM_CUDA(c, cudaMemcpyAsync(lbd72, B.d_lbd72, (size_t)nframes * max_lines * 72 * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    return PSLAM_OK;
}

int pslam_lines_extract_batch_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, int max_lines, pslam_keyline* d_kl, double* d_lf, int32_t* d_n) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_gray || !d_kl || !d_lf || !d_n || max_lines < 1) return set_error(c, PSLAM_E_INVALID, "null pointer or max_lines < 1");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    int rc = lsd_detect_dev(c, d_gray, nframes, 2);
    if (rc != PSLAM_OK) return rc;
    static_assert(sizeof(LsdKeyLine) == sizeof(pslam_keyline) && sizeof(pslam_keyline) == 68, "KeyLine layout");
    return lsd_keylines_dev(c, nframes, max_lines, (LsdKeyLine*)d_kl, d_lf, d_n);
}

int pslam_lines_extract_batch(pslam_ctx* c, const uint8_t* gray, int nframes, int max_lines, pslam_keyline* kl, double* lf, int32_t* n) {
    if (!c) return PSLAM_E_INVALID;
    if (!gray || !kl || !lf || !n || max_lines < 1) return set_error(c, PSLAM_E_INVALID, "null pointer or max_lines < 1");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    int rc = lsd_upload(c, gray, nframes);
    if (rc != PSLAM_OK) return rc;
    LsdBuffers& B = *c->lsd;
    if ((rc = lsd_ensure_kl(c, max_lines)) != PSLAM_OK) return rc;
    if ((rc = lsd_detect_dev(c, B.d_gray, nframes, 2)) != PSLAM_OK) return rc;
    if ((rc = lsd_keylines_dev(c, nframes, max_lines, B.d_kl, B.d_lf, B.d_nkl)) != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    B.h_status.resize(nframes);
    PSLAM_CUDA(c, cudaMemcpyAsync(kl, B.d_kl, (size_t)nframes * max_lines * sizeof(LsdKeyLine), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(lf, B.d_lf, (size_t)nframes * max_lines * 24, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(n, B.d_nkl, (size_t)nframes * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_status.data(), B.d_status, nframes * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    for (int f = 0; f < nframes; ++f) if (B.h_status[f]) return set_error(c, PSLAM_E_CAPACITY, "more line segments than the internal capacity");
    return PSLAM_OK;
}

int pslam_lsd_debug_stage(pslam_ctx* c, int frame, int32_t* dims, uint8_t* scaled, double* modgrad, double* angles, int32_t* order, int32_t* n_order) {
    if (!c || !c->lsd || frame < 0 || frame >= c->lsd->last_n) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    LsdBuffers& B = *c->lsd;
    const LsdGeom& g = B.g;
    const size_t npx = (size_t)g.W * g.H;
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    if (dims) { dims[0] = g.W; dims[1] = g.H; }
    if (scaled) PSLAM_CUDA(c, cudaMemcpy(scaled, B.d_scaled + (size_t)frame * npx, npx, cudaMemcpyDeviceToHost));
    if (modgrad || angles) {
        std::vector<uint32_t> gxy(npx);
        PSLAM_CUDA(c, cudaMemcpy(gxy.data(), B.d_gxy + (size_t)frame * npx, npx * 4, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < npx; ++i) {
            // same formulas as the device helpers (sqrt and the float polynomial are exactly rounded operations)
            const int gx = (int16_t)(gxy[i] & 0xffff), gy = (int16_t)(gxy[i] >> 16);
            const double nrm = std::sqrt((double)(gx * gx + gy * gy) / 4.0);
            if (modgrad) modgrad[i] = nrm;
            if (angles) angles[i] = nrm > g.rho ? (double)host_fast_atan2_deg((float)gx, (float)(-gy)) * LSD_DEG2RAD : -1024.0;
        }
    }
    int no = 0;
    PSLAM_CUDA(c, cudaMemcpy(&no, B.d_norder + frame, 4, cudaMemcpyDeviceToHost));
    if (n_order) *n_order = no;
    if (order && no > 0) {
        std::vector<uint32_t> o(no);
        PSLAM_CUDA(c, cudaMemcpy(o.data(), B.d_order + (size_t)frame * npx, (size_t)no * 4, cudaMemcpyDeviceToHost));
        for (int i = 0; i < no; ++i) order[i] = (int32_t)((o[i] >> 16) * g.W + (o[i] & 0xffff));
    }
    return PSLAM_OK;
}

}  // extern "C"
