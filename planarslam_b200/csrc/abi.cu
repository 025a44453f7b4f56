// extern "C" entry points of libpslam_b200.so (declared in include/pslam_abi.h).
#include <cstdio>
#include <cstring>
#include <new>

#include "orb_common.h"
#include "pslam_internal.h"

namespace pslam {

int set_error(pslam_ctx* c, int code, const std::string& msg) {
    if (c) c->err = msg;
    return code;
}

int check_cuda(pslam_ctx* c, cudaError_t e, const char* what) {
    if (e == cudaSuccess) return PSLAM_OK;
    return set_error(c, PSLAM_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

static int status_to_rc(pslam_ctx* c, int nframes) {
    int bits = 0;
    for (int i = 0; i < nframes; ++i) bits |= c->h_status[i];
    if (!bits) return PSLAM_OK;
    char buf[160];
    std::snprintf(buf, sizeof buf, "capacity exceeded (flags 0x%x: 1 cell slots, 2 candidate list, 4 quadtree nodes, 8 output rows)", bits);
    return set_error(c, PSLAM_E_CAPACITY, buf);
}

}  // namespace pslam

using namespace pslam;

extern "C" {

void pslam_default_config(pslam_config* cfg, int width, int height, int max_batch) {
    if (!cfg) return;
    std::memset(cfg, 0, sizeof(*cfg));
    cfg->device = 0; cfg->width = width; cfg->height = height; cfg->max_batch = max_batch;
    cfg->nfeatures = 1000; cfg->scale_factor = 1.2f; cfg->nlevels = 8; cfg->ini_th_fast = 20; cfg->min_th_fast = 7;
    const float s = (float)width / 640.f;                       // Examples/RGB-D/TUM3.yaml:8-11,35 scaled to the frame width
    cfg->fx = 535.4f * s; cfg->fy = 539.2f * s; cfg->cx = 320.1f * s; cfg->cy = 247.6f * s;
    cfg->depth_scale = 1.0f / 5000.0f;
}

int pslam_create(const pslam_config* cfg, pslam_ctx** out) {
    if (!cfg || !out) return PSLAM_E_INVALID;
    *out = nullptr;
    if (cfg->max_batch < 1) return PSLAM_E_INVALID;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cfg->device < 0 || cfg->device >= ndev) return PSLAM_E_NO_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess || prop.major != 9) return PSLAM_E_NO_DEVICE;   // sm_90a only
    pslam_ctx* c = new (std::nothrow) pslam_ctx();
    if (!c) return PSLAM_E_INVALID;
    c->cfg = *cfg;
    int rc = check_cuda(c, cudaSetDevice(cfg->device), "cudaSetDevice");
    if (rc == PSLAM_OK) rc = orb_build_geometry(c);
    if (rc == PSLAM_OK) rc = peac_build_geometry(c);
    if (rc == PSLAM_OK) rc = check_cuda(c, cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking), "cudaStreamCreate");
    c->stream = c->own_stream;
    if (rc == PSLAM_OK) rc = check_cuda(c, cudaMalloc((void**)&c->d_status, (size_t)cfg->max_batch * sizeof(int32_t)), "cudaMalloc");
    if (rc == PSLAM_OK) rc = check_cuda(c, cudaMallocHost((void**)&c->h_status, (size_t)cfg->max_batch * sizeof(int32_t)), "cudaMallocHost");
    if (rc != PSLAM_OK) {
        std::fprintf(stderr, "pslam_create failed: %s\n", c->err.c_str());
        pslam_destroy(c);
        return rc;
    }
    *out = c;
    return PSLAM_OK;
}

void pslam_destroy(pslam_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->cfg.device);
    cudaDeviceSynchronize();
    if (c->orb_ready) orb_free(c);
    if (c->peac_ready) peac_free(c);
    cudaFree(c->d_status); cudaFreeHost(c->h_status);
    pose_free(c);
    lba_free(c);
    lsd_free(c);
    search_free(c);
    track_free(c);
    exchange_free(c);
    planepost_free(c);
    bowdb_free(c);
    bowvoc_free(c);
    frame_free(c);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;
}

const char* pslam_last_error(const pslam_ctx* c) { return c ? c->err.c_str() : "null context"; }

int pslam_set_stream(pslam_ctx* c, void* s) {
    if (!c) return PSLAM_E_INVALID;
    c->stream = s ? (cudaStream_t)s : c->own_stream;
    return PSLAM_OK;
}

int pslam_synchronize(pslam_ctx* c) {
    if (!c) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSLAM_OK;
}

int64_t pslam_launch_count(const pslam_ctx* c) { return c ? c->launches : 0; }

int pslam_profile_enable(pslam_ctx* c, int on) {
    if (!c) return PSLAM_E_INVALID;
    for (auto& r : c->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    c->prof.clear();
    c->profile = on != 0;
    return PSLAM_OK;
}

int pslam_profile_report(pslam_ctx* c, char* buf, int cap) {
    if (!c || !buf || cap < 2) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    struct Acc { const char* name; int n; double ms; };
    std::vector<Acc> acc;
    for (auto& r : c->prof) {
        float ms = 0.f;
        PSLAM_CUDA(c, cudaEventElapsedTime(&ms, r.a, r.b));
        bool found = false;
        for (auto& a : acc) if (!std::strcmp(a.name, r.name)) { a.n++; a.ms += ms; found = true; break; }
        if (!found) acc.push_back({r.name, 1, ms});
    }
    std::string out;
    for (auto& a : acc) { char line[160]; std::snprintf(line, sizeof line, "%s %d %.6f\n", a.name, a.n, a.ms); out += line; }
    if ((int)out.size() + 1 > cap) return set_error(c, PSLAM_E_CAPACITY, "profile report buffer too small");
    std::memcpy(buf, out.c_str(), out.size() + 1);
    return PSLAM_OK;
}

int pslam_orb_get_scale_tables(const pslam_ctx* c, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2, int32_t* fpl) {
    if (!c) return PSLAM_E_INVALID;
    for (int i = 0; i < c->geom.nlevels; ++i) {
        if (scale) scale[i] = c->scale[i];
        if (inv_scale) inv_scale[i] = c->inv_scale[i];
        if (sigma2) sigma2[i] = c->sigma2[i];
        if (inv_sigma2) inv_sigma2[i] = c->inv_sigma2[i];
        if (fpl) fpl[i] = c->quota[i];
    }
    return PSLAM_OK;
}

int pslam_orb_max_keypoints(const pslam_ctx* c) { return c ? c->geom.total_kp : 0; }

int pslam_orb_extract_batch_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, pslam_keypoint* d_kps, uint8_t* d_desc, int cap,
                                int32_t* d_n) {
    if (!c) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return orb_run_dev(c, d_gray, nframes, d_kps, d_desc, cap, d_n);
}

int pslam_orb_extract_batch(pslam_ctx* c, const uint8_t* gray, int nframes, pslam_keypoint* kps, uint8_t* desc, int cap, int32_t* n) {
    if (!c) return PSLAM_E_INVALID;
    if (!gray || !kps || !desc || !n || cap < 1) return set_error(c, PSLAM_E_INVALID, "null pointer or cap < 1");
    if (nframes < 1 || nframes > c->cfg.max_batch) return set_error(c, PSLAM_E_INVALID, "nframes outside [1, max_batch]");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->orb_ready) { const int arc = orb_alloc(c); if (arc != PSLAM_OK) return arc; }
    const OrbGeom& g = c->geom;
    const size_t frame_px = (size_t)g.width * g.height;
    const int icap = g.total_kp;                       // internal capacity is always sufficient
    cudaStream_t st = c->stream;
    const uint8_t* src = gray;                         // page-locked caller memory goes straight to the copy engine
    if (!host_ptr_is_pinned(gray)) { std::memcpy(c->h_gray, gray, frame_px * nframes); src = c->h_gray; }   // pageable -> pinned staging
    PSLAM_CUDA(c, cudaMemcpyAsync(c->d_gray, src, frame_px * nframes, cudaMemcpyHostToDevice, st));
    int rc = orb_run_dev(c, c->d_gray, nframes, c->d_kps, c->d_desc, icap, c->d_n);
    if (rc != PSLAM_OK) return rc;
    PSLAM_CUDA(c, cudaMemcpyAsync(c->h_n, c->d_n, nframes * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(c->h_status, c->d_status, nframes * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    // caller buffers with the internal row capacity that are page-locked receive the records directly
    const bool direct = cap == icap && host_ptr_is_pinned(kps) && host_ptr_is_pinned(desc);
    PSLAM_CUDA(c, cudaMemcpyAsync(direct ? kps : c->h_kps, c->d_kps, (size_t)nframes * icap * sizeof(pslam_keypoint), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(direct ? desc : c->h_desc, c->d_desc, (size_t)nframes * icap * 32, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    rc = status_to_rc(c, nframes);
    for (int f = 0; f < nframes; ++f) {
        n[f] = c->h_n[f];
        if (direct) continue;
        const int m = std::min(c->h_n[f], cap);
        if (c->h_n[f] > cap) rc = set_error(c, PSLAM_E_CAPACITY, "caller keypoint capacity too small");
        std::memcpy(kps + (size_t)f * cap, c->h_kps + (size_t)f * icap, (size_t)m * sizeof(pslam_keypoint));
        std::memcpy(desc + (size_t)f * cap * 32, c->h_desc + (size_t)f * icap * 32, (size_t)m * 32);
    }
    return rc;
}

int pslam_orb_extract(pslam_ctx* c, const uint8_t* gray, int stride, pslam_keypoint* kps, uint8_t* desc, int cap, int32_t* n) {
    if (!c) return PSLAM_E_INVALID;
    if (!gray || stride < c->geom.width) return set_error(c, PSLAM_E_INVALID, "null image or stride < width");
    if (stride == c->geom.width) return pslam_orb_extract_batch(c, gray, 1, kps, desc, cap, n);
    // repack a strided image into the pinned staging buffer, then run as a batch of one
    std::vector<uint8_t> tmp((size_t)c->geom.width * c->geom.height);
    for (int y = 0; y < c->geom.height; ++y) std::memcpy(&tmp[(size_t)y * c->geom.width], gray + (size_t)y * stride, c->geom.width);
    return pslam_orb_extract_batch(c, tmp.data(), 1, kps, desc, cap, n);
}

int pslam_orb_debug_level_size(const pslam_ctx* c, int level, int32_t* w, int32_t* h) {
    if (!c || level < 0 || level >= c->geom.nlevels || !w || !h) return PSLAM_E_INVALID;
    *w = c->geom.lv[level].w; *h = c->geom.lv[level].h;
    return PSLAM_OK;
}

int pslam_orb_debug_level_pixels(pslam_ctx* c, int frame, int level, uint8_t* out) {
    if (!c || !c->orb_ready || !out || level < 0 || level >= c->geom.nlevels || frame < 0 || frame >= c->last_nframes) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    const OrbGeom& g = c->geom;
    const LevelGeom& v = g.lv[level];
    const uint8_t* src = level == 0 ? c->d_gray_cur + (size_t)frame * g.width * g.height : c->d_pyr + (size_t)frame * g.pyr_bytes + v.pyr_off;
    PSLAM_CUDA(c, cudaMemcpy2D(out, v.w, src, v.pitch, v.w, v.h, cudaMemcpyDeviceToHost));
    return PSLAM_OK;
}

int pslam_orb_debug_level_blurred(pslam_ctx* c, int frame, int level, uint8_t* out) {
    if (!c || !c->orb_ready || !out || level < 0 || level >= c->geom.nlevels || frame < 0 || frame >= c->last_nframes) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    const LevelGeom& v = c->geom.lv[level];
    PSLAM_CUDA(c, cudaMemcpy2D(out, v.w, c->d_blur + (size_t)frame * c->blur_frame_bytes + v.blur_off, v.blur_pitch, v.w, v.h,
                               cudaMemcpyDeviceToHost));
    return PSLAM_OK;
}

int pslam_orb_debug_level_candidates(pslam_ctx* c, int frame, int level, int32_t* xys, int cap, int32_t* n) {
    if (!c || !c->orb_ready || !xys || !n || level < 0 || level >= c->geom.nlevels || frame < 0 || frame >= c->last_nframes) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    const OrbGeom& g = c->geom;
    const LevelGeom& v = g.lv[level];
    const int ncell = v.n_cols * v.n_rows;
    std::vector<int32_t> cnt(ncell);
    std::vector<uint32_t> sl((size_t)ncell * v.slot_cap);
    PSLAM_CUDA(c, cudaMemcpy(cnt.data(), c->d_cell_cnt + (size_t)frame * g.total_cells + v.cell_base, ncell * 4, cudaMemcpyDeviceToHost));
    PSLAM_CUDA(c, cudaMemcpy(sl.data(), c->d_slots + (size_t)frame * g.total_slots + v.slot_base, sl.size() * 4, cudaMemcpyDeviceToHost));
    int k = 0;
    for (int ce = 0; ce < ncell; ++ce)
        for (int i = 0; i < cnt[ce]; ++i, ++k)
            if (k < cap) { const uint32_t p = sl[(size_t)ce * v.slot_cap + i]; xys[3 * k] = kp_x(p); xys[3 * k + 1] = kp_y(p); xys[3 * k + 2] = kp_s(p); }
    *n = k;
    return k > cap ? PSLAM_E_CAPACITY : PSLAM_OK;
}

}  // extern "C"
