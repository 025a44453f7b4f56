// Host side of the ORB extractor: level / cell geometry and resize tables (float arithmetic of the reference
// constructor and ComputePyramid, src/ORBextractor.cc:410-470, :1107-1116, :771-787), buffers, launch sequence.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "orb_kernels.cuh"

namespace pslam {

static inline int cv_round(double v) { return (int)std::nearbyint(v); }   // half-to-even under FE_TONEAREST
static inline int align_up(int v, int a) { return (v + a - 1) / a * a; }
static inline short sat_short(float v) { return (short)std::min(32767, std::max(-32768, cv_round(v))); }

int orb_build_geometry(pslam_ctx* c) {
    const pslam_config& cf = c->cfg;
    OrbGeom& g = c->geom;
    std::memset(&g, 0, sizeof(g));
    const int L = cf.nlevels;
    if (L < 1 || L > PSLAM_MAX_LEVELS) return set_error(c, PSLAM_E_INVALID, "nlevels must be in [1, 8]");
    if (cf.width % 4 || cf.width < 64 || cf.height < 64 || cf.width > 2047 + 32 || cf.height > 2047 + 32)
        return set_error(c, PSLAM_E_INVALID, "width must be a multiple of 4; frame size in [64, 2079]");
    if (cf.min_th_fast < 1 || cf.ini_th_fast < cf.min_th_fast || cf.ini_th_fast > 254)
        return set_error(c, PSLAM_E_INVALID, "need 1 <= min_th_fast <= ini_th_fast <= 254");
    if (cf.nfeatures < 1 || !(cf.scale_factor > 1.0f)) return set_error(c, PSLAM_E_INVALID, "nfeatures >= 1, scale_factor > 1");
    g.nlevels = L; g.width = cf.width; g.height = cf.height; g.ini_th = cf.ini_th_fast; g.min_th = cf.min_th_fast;

    // scale tables and per-level quotas (reference ctor :415-446)
    c->scale.assign(L, 1.f); c->sigma2.assign(L, 1.f); c->inv_scale.resize(L); c->inv_sigma2.resize(L); c->quota.resize(L);
    for (int i = 1; i < L; ++i) { c->scale[i] = c->scale[i - 1] * cf.scale_factor; c->sigma2[i] = c->scale[i] * c->scale[i]; }
    for (int i = 0; i < L; ++i) { c->inv_scale[i] = 1.0f / c->scale[i]; c->inv_sigma2[i] = 1.0f / c->sigma2[i]; }
    const float factor = 1.0f / cf.scale_factor;
    float want = cf.nfeatures * (1 - factor) / (1 - (float)std::pow((double)factor, (double)L));
    int sum = 0;
    for (int l = 0; l < L - 1; ++l) { c->quota[l] = cv_round(want); sum += c->quota[l]; want *= factor; }
    c->quota[L - 1] = std::max(cf.nfeatures - sum, 0);

    // disc half-widths for the orientation patch (reference ctor :454-469)
    {
        const int HP = 15;
        int umax[17] = {0};
        const int vmax = (int)std::floor(HP * std::sqrt(2.f) / 2 + 1), vmin = (int)std::ceil(HP * std::sqrt(2.f) / 2);
        for (int v = 0; v <= vmax; ++v) umax[v] = cv_round(std::sqrt((double)HP * HP - v * v));
        for (int v = HP, v0 = 0; v >= vmin; --v) { while (umax[v0] == umax[v0 + 1]) ++v0; umax[v] = v0; ++v0; }
        for (int v = 0; v < 16; ++v) g.umax[v] = umax[v];
    }

    int pyr = 0, blur = 0, cells = 0, slots = 0, kp = 0, cand = 0, nodes = 0, work = 0, tabx = 0, taby = 0;
    for (int l = 0; l < L; ++l) {
        LevelGeom& v = g.lv[l];
        v.w = cv_round((float)cf.width * c->inv_scale[l]);
        v.h = cv_round((float)cf.height * c->inv_scale[l]);
        if (v.w < 38 + 30 || v.h < 38 + 30) return set_error(c, PSLAM_E_INVALID, "pyramid level smaller than one FAST cell; reduce nlevels");
        v.pitch = (l == 0) ? cf.width : align_up(v.w, 16);
        v.pyr_off = pyr;
        if (l > 0) pyr += align_up(v.pitch * v.h, 16);
        v.blur_pitch = align_up(v.w, 16);
        v.blur_off = blur;
        blur += align_up(v.blur_pitch * v.h, 16);
        v.max_bx = v.w - 19 + 3; v.max_by = v.h - 19 + 3;
        const float width = (float)(v.max_bx - 16), height = (float)(v.max_by - 16);
        v.n_cols = (int)(width / 30.f); v.n_rows = (int)(height / 30.f);
        v.w_cell = (int)std::ceil(width / v.n_cols); v.h_cell = (int)std::ceil(height / v.n_rows);
        if (v.w_cell > 59 || v.h_cell > 59) return set_error(c, PSLAM_E_INVALID, "FAST cell larger than 59 px");
        v.cell_base = cells; cells += v.n_cols * v.n_rows;
        v.slot_cap = ((v.w_cell + 1) / 2) * ((v.h_cell + 1) / 2);      // 8-neighbour strict maxima cannot be denser
        v.slot_base = slots; slots += v.n_cols * v.n_rows * v.slot_cap;
        v.quota = c->quota[l];
        v.kp_cap = v.quota + 3;
        v.kp_base = kp; kp += v.kp_cap;
        v.cand_cap = v.n_cols * v.n_rows * v.slot_cap;                    // every slot can be filled (noise images)
        v.cand_base = cand; cand += v.cand_cap;
        v.node_cap = 24 * v.kp_cap + 64;
        v.node_base = nodes; nodes += v.node_cap;
        v.work_base = work; work += 9 * v.kp_cap;
        v.tabx_off = tabx; v.taby_off = taby;
        if (l > 0) { tabx += v.w; taby += v.h; }
        v.n_ini = (int)std::round((float)(v.max_bx - 16) / (float)(v.max_by - 16));
        if (v.n_ini < 1 || v.n_ini > 4) return set_error(c, PSLAM_E_INVALID, "aspect ratio outside [0.5, 4.5) is not supported");
        v.h_x = (float)(v.max_bx - 16) / v.n_ini;
        v.scale = c->scale[l];
        v.patch_size = (int)(31 * c->scale[l]);
    }
    g.pyr_bytes = std::max(pyr, 16); c->blur_frame_bytes = blur;
    g.total_cells = cells; g.total_slots = slots; g.total_kp = kp; g.total_cand = cand; g.total_nodes = nodes;
    g.total_work = work; g.total_tabx = std::max(tabx, 1); g.total_taby = std::max(taby, 1);
    return PSLAM_OK;
}

int orb_alloc(pslam_ctx* c) {
    const OrbGeom& g = c->geom;
    const size_t B = c->cfg.max_batch;
    const int cap = g.total_kp;
    int rc;
    if ((rc = c->d_gray.reserve(c, B * g.width * g.height)) || (rc = c->d_pyr.reserve(c, B * g.pyr_bytes)) || (rc = c->d_blur.reserve(c, B * c->blur_frame_bytes)) ||
        (rc = c->d_xofs.reserve(c, g.total_tabx)) || (rc = c->d_xa.reserve(c, (size_t)2 * g.total_tabx)) ||
        (rc = c->d_yofs.reserve(c, g.total_taby)) || (rc = c->d_ya.reserve(c, (size_t)2 * g.total_taby)) ||
        (rc = c->d_slots.reserve(c, B * g.total_slots)) || (rc = c->d_cell_cnt.reserve(c, B * g.total_cells)) ||
        (rc = c->d_cand.reserve(c, B * g.total_cand * 2)) || (rc = c->d_cand_cnt.reserve(c, B * g.nlevels)) ||
        (rc = c->d_nodes.reserve(c, B * g.total_nodes)) || (rc = c->d_links.reserve(c, B * g.total_nodes)) || (rc = c->d_work.reserve(c, B * g.total_work)) ||
        (rc = c->d_lvl_kp.reserve(c, B * g.total_kp)) || (rc = c->d_lvl_cnt.reserve(c, B * g.nlevels)) ||
        (rc = c->d_kps.reserve(c, B * cap)) || (rc = c->d_desc.reserve(c, B * cap * 32)) || (rc = c->d_n.reserve(c, B)) ||
        (rc = c->h_gray.reserve(c, B * g.width * g.height)) || (rc = c->h_kps.reserve(c, B * cap)) || (rc = c->h_desc.reserve(c, B * cap * 32)) ||
        (rc = c->h_n.reserve(c, B)))
        return rc;
    // resize tables (cv::resize INTER_LINEAR 8-bit: 11-bit coefficients, see oracle/cvprims.cc for the pinned restatement)
    std::vector<int16_t> xofs(g.total_tabx), xa(2 * g.total_tabx), yofs(g.total_taby), ya(2 * g.total_taby);
    for (int l = 1; l < g.nlevels; ++l) {
        const LevelGeom &d = g.lv[l], &s = g.lv[l - 1];
        const double sx_ = (double)s.w / d.w, sy_ = (double)s.h / d.h;
        for (int dx = 0; dx < d.w; ++dx) {
            float fx = (float)((dx + 0.5) * sx_ - 0.5);
            int sx = (int)std::floor(fx);
            fx -= sx;
            if (sx < 0) { fx = 0; sx = 0; }
            if (sx >= s.w - 1) { fx = 0; sx = s.w - 1; }
            xofs[d.tabx_off + dx] = (int16_t)sx;
            xa[2 * (d.tabx_off + dx)] = sat_short((1.f - fx) * 2048.f);
            xa[2 * (d.tabx_off + dx) + 1] = sat_short(fx * 2048.f);
        }
        for (int dy = 0; dy < d.h; ++dy) {
            float fy = (float)((dy + 0.5) * sy_ - 0.5);
            int sy = (int)std::floor(fy);
            fy -= sy;
            yofs[d.taby_off + dy] = (int16_t)sy;
            ya[2 * (d.taby_off + dy)] = sat_short((1.f - fy) * 2048.f);
            ya[2 * (d.taby_off + dy) + 1] = sat_short(fy * 2048.f);
        }
    }
    PSLAM_CUDA(c, cudaMemcpy(c->d_xofs, xofs.data(), xofs.size() * 2, cudaMemcpyHostToDevice));
    PSLAM_CUDA(c, cudaMemcpy(c->d_xa, xa.data(), xa.size() * 2, cudaMemcpyHostToDevice));
    PSLAM_CUDA(c, cudaMemcpy(c->d_yofs, yofs.data(), yofs.size() * 2, cudaMemcpyHostToDevice));
    PSLAM_CUDA(c, cudaMemcpy(c->d_ya, ya.data(), ya.size() * 2, cudaMemcpyHostToDevice));
    c->orb_ready = true;
    return PSLAM_OK;
}

int orb_run_dev(pslam_ctx* c, const uint8_t* d_gray, int nframes, pslam_keypoint* d_kps, uint8_t* d_desc, int cap, int32_t* d_n) {
    const OrbGeom& g = c->geom;
    if (nframes < 1 || nframes > c->cfg.max_batch) return set_error(c, PSLAM_E_INVALID, "nframes outside [1, max_batch]");
    if (!d_gray || !d_kps || !d_desc || !d_n || cap < 1) return set_error(c, PSLAM_E_INVALID, "null output or cap < 1");
    if (!c->orb_ready) { const int arc = orb_alloc(c); if (arc != PSLAM_OK) return arc; }
    cudaStream_t st = c->stream;
    c->d_gray_cur = d_gray;
    c->last_nframes = nframes;
    const size_t frame_px = (size_t)g.width * g.height;
    PSLAM_CUDA(c, cudaMemsetAsync(c->d_status, 0, nframes * sizeof(int32_t), st));

    // K1: pyramid, one launch per level (each level depends on the previous one)
    for (int l = 1; l < g.nlevels; ++l) {
        const LevelGeom &d = g.lv[l], &s = g.lv[l - 1];
        const uint8_t* src = (l == 1) ? d_gray : c->d_pyr + s.pyr_off;
        const size_t sfs = (l == 1) ? frame_px : (size_t)g.pyr_bytes;
        dim3 grid((d.w + 127) / 128, (d.h + 7) / 8, nframes), block(32, 8);
        PSLAM_LAUNCH(c, "orb_resize_level", k_resize_level<<<grid, block, 0, st>>>(src, sfs, s.pitch, s.w, s.h, c->d_pyr + d.pyr_off,
                     (size_t)g.pyr_bytes, d.pitch, d.w, d.h, c->d_xofs + d.tabx_off, c->d_xa + 2 * d.tabx_off, c->d_yofs + d.taby_off,
                     c->d_ya + 2 * d.taby_off));
    }
    // K2: FAST per cell, all levels and frames in one launch
    PSLAM_LAUNCH(c, "orb_fast_cells", k_fast_cells<<<dim3(g.total_cells, nframes), 128, 0, st>>>(d_gray, c->d_pyr, g, c->d_slots, c->d_cell_cnt, c->d_status));
    // K3: quadtree, one warp per (level, frame)
    PSLAM_LAUNCH(c, "orb_quadtree", k_quadtree<<<dim3(g.nlevels, nframes), 32, 0, st>>>(g, c->d_slots, c->d_cell_cnt, c->d_cand, c->d_cand_cnt,
                 c->d_nodes, c->d_links, c->d_work, c->d_lvl_kp, c->d_lvl_cnt, c->d_status));
    // K4a: blur every level.  TMA path: one launch for all levels; the tensor maps of levels 1.. point into the context's pyramid buffer, level 0's
    // into the caller's frames (re-encoded when the pointer or the frame count changes).  Images whose rows are not 16-byte multiples cannot be
    // described by a tensor map and take the per-level kernel.
    bool tma_ok = (g.width % 16) == 0 && ((uintptr_t)d_gray % 16) == 0 && std::getenv("PSLAM_NO_TMA") == nullptr;
    if (tma_ok) {
        BlurTmaParams& P = c->blur_tma;
        if (c->blur_tma_src != d_gray || c->blur_tma_n != nframes) {
            int base = 0;
            for (int l = 0; l < g.nlevels && tma_ok; ++l) {
                const LevelGeom& v = g.lv[l];
                P.tiles_x[l] = (v.w + BT_W - 1) / BT_W;
                P.tile_base[l] = base;
                base += P.tiles_x[l] * ((v.h + BT_H - 1) / BT_H);
                P.w[l] = v.w; P.h[l] = v.h; P.dst_pitch[l] = v.blur_pitch; P.dst_off[l] = v.blur_off;
                tma_ok = l == 0 ? tma_encode_3d(&P.map[0], CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, d_gray, v.w, v.h, nframes, (size_t)g.width, frame_px, BT_BOX_W, BT_BOX_H)
                                : tma_encode_3d(&P.map[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, c->d_pyr + v.pyr_off, v.w, v.h, c->cfg.max_batch, (size_t)v.pitch,
                                                (size_t)g.pyr_bytes, BT_BOX_W, BT_BOX_H);
            }
            P.tile_base[g.nlevels] = base; P.nlevels = g.nlevels;
            c->blur_tma_src = tma_ok ? d_gray : nullptr; c->blur_tma_n = nframes;
            if (tma_ok) {
                if (const int rc = c->d_blur_maps.reserve(c, PSLAM_MAX_LEVELS)) return rc;
                PSLAM_CUDA(c, cudaMemcpyAsync(c->d_blur_maps, P.map, sizeof P.map, cudaMemcpyHostToDevice, st));      // P.map lives in the context: stable until the next re-encode
            }
        }
    }
    if (tma_ok) {
        static const bool in_param = [] { const char* e = std::getenv("PSLAM_TMA_MAPS"); return e && !std::strcmp(e, "param"); }();
        const dim3 grid(c->blur_tma.tile_base[g.nlevels], nframes);
        if (in_param) PSLAM_LAUNCH(c, "orb_blur_tma", k_blur_tma<true><<<grid, 128, 0, st>>>(c->blur_tma, c->d_blur_maps, c->d_blur, (size_t)c->blur_frame_bytes));
        else PSLAM_LAUNCH(c, "orb_blur_tma", k_blur_tma<false><<<grid, 128, 0, st>>>(c->blur_tma, c->d_blur_maps, c->d_blur, (size_t)c->blur_frame_bytes));
    } else
    for (int l = 0; l < g.nlevels; ++l) {
        const LevelGeom& v = g.lv[l];
        const uint8_t* src = (l == 0) ? d_gray : c->d_pyr + v.pyr_off;
        const size_t sfs = (l == 0) ? frame_px : (size_t)g.pyr_bytes;
        dim3 grid((v.w + 63) / 64, (v.h + 15) / 16, nframes);
        PSLAM_LAUNCH(c, "orb_blur_level", k_blur_level<<<grid, 256, 0, st>>>(src, sfs, v.pitch, c->d_blur + v.blur_off,
                     (size_t)c->blur_frame_bytes, v.blur_pitch, v.w, v.h));
    }
    // K4b: orientation + descriptors + output records
    PSLAM_LAUNCH(c, "orb_orient_describe", k_orient_describe<<<dim3((g.total_kp + 7) / 8, nframes), 256, 0, st>>>(g, d_gray, c->d_pyr, c->d_blur,
                 c->blur_frame_bytes, c->d_lvl_kp, c->d_lvl_cnt, d_kps, d_desc, d_n, cap, c->d_status));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

}  // namespace pslam
