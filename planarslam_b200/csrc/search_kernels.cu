// Host side of the projection-guided searches (kernels: search_kernels.cuh).
#include "search_kernels.cuh"

namespace pslam {

// ---------------------------------------------------------------------------------------------------------
struct SearchBuffers {
    DevArray<uint8_t> blob;                                     // the frame / map arrays of the current call
    DevArray<uint32_t> d_cand; DevArray<int32_t> d_cand_n, d_hist_idx; DevArray<int8_t> d_hist_bin; DevArray<uint8_t> d_in_view;   // per point
    DevArray<int32_t> d_cell_start, d_items, d_matches, d_scalar;
};

static int ensure(pslam_ctx* c, SearchBuffers& B, size_t npts) {
    int rc;
    if ((rc = B.d_cell_start.reserve(c, SG_CELLS + 1)) || (rc = B.d_items.reserve(c, SEARCH_MAX_KP)) || (rc = B.d_matches.reserve(c, SEARCH_MAX_KP)) ||
        (rc = B.d_scalar.reserve(c, 4)) || (rc = B.d_cand.grow(c, npts * SEARCH_CAND_CAP)) || (rc = B.d_cand_n.grow(c, npts)) ||
        (rc = B.d_hist_idx.grow(c, npts)) || (rc = B.d_hist_bin.grow(c, npts)) || (rc = B.d_in_view.grow(c, npts)))
        return rc;
    return PSLAM_OK;
}

// uploads the frame / map arrays into the staging blob; fills the device views.  Every array gets at least one element, so no view is null.
static int upload(pslam_ctx* c, SearchBuffers& B, const pslam_frame_view* f, const pslam_map_points* m, const pslam_last_frame* l, SearchFrameDev& F,
                  SearchMapDev& M, SearchLastDev& Ld) {
    const size_t nf = f->n, nm = m->n, nl = l ? l->n : 0;
    auto one = [](size_t n) { return std::max<size_t>(n, 1); };
    Slab s;
    const auto f_keys = s.add<pslam_keypoint>(one(nf)); const auto f_ur = s.add<float>(one(nf)); const auto f_desc = s.add<uint8_t>(one(nf * 32));
    const auto m_pos = s.add<float>(one(nm * 3)); const auto m_normal = s.add<float>(one(nm * 3)); const auto m_maxd = s.add<float>(one(nm));
    const auto m_mind = s.add<float>(one(nm)); const auto m_desc = s.add<uint8_t>(one(nm * 32)); const auto m_skip = s.add<uint8_t>(one(nm));
    const auto m_has_obs = s.add<uint8_t>(one(nm));
    const auto l_keys = s.add<pslam_keypoint>(one(nl)); const auto l_mp = s.add<int32_t>(one(nl)); const auto l_outlier = s.add<uint8_t>(one(nl));
    if (const int rc = s.alloc(c, B.blob, true)) return rc;
    cudaStream_t st = c->stream;
    s.up(f_keys, f->keys_un, st, nf); s.up(f_ur, f->u_right, st, nf); s.up(f_desc, f->desc, st, nf * 32);
    s.up(m_pos, m->pos, st, nm * 3); s.up(m_normal, m->normal, st, nm * 3); s.up(m_maxd, m->max_distance, st, nm); s.up(m_mind, m->min_distance, st, nm);
    s.up(m_desc, m->desc, st, nm * 32); s.up(m_skip, m->skip, st, nm); s.up(m_has_obs, m->has_obs, st, nm);
    if (l) { s.up(l_keys, l->keys, st, nl); s.up(l_mp, l->map_point, st, nl); s.up(l_outlier, l->outlier, st, nl); }
    if (const int rc = s.check(c)) return rc;
    F.n = (int)nf;
    F.keys_un = s[f_keys]; F.u_right = s[f_ur]; F.desc = s[f_desc];
    std::memcpy(F.Tcw, f->Tcw, sizeof F.Tcw); F.Tcw_dev = nullptr; F.n_dev = nullptr;
    F.fx = f->fx; F.fy = f->fy; F.cx = f->cx; F.cy = f->cy; F.bf = f->bf; F.min_x = f->min_x; F.max_x = f->max_x; F.min_y = f->min_y; F.max_y = f->max_y;
    F.n_levels = f->n_levels; F.log_scale_factor = f->log_scale_factor;
    for (int i = 0; i < f->n_levels && i < PSLAM_MAX_LEVELS; ++i) F.scale[i] = f->scale_factors[i];
    F.inv_w = (float)SG_COLS / (f->max_x - f->min_x); F.inv_h = (float)SG_ROWS / (f->max_y - f->min_y);
    M.n = (int)nm;
    M.pos = s[m_pos]; M.normal = s[m_normal]; M.max_distance = s[m_maxd]; M.min_distance = s[m_mind]; M.desc = s[m_desc]; M.skip = s[m_skip]; M.has_obs = s[m_has_obs];
    if (l) {
        Ld.n = (int)nl;
        Ld.keys = s[l_keys]; Ld.map_point = s[l_mp]; Ld.outlier = s[l_outlier];
        std::memcpy(Ld.Tcw, l->Tcw, sizeof Ld.Tcw); Ld.Tcw_dev = nullptr; Ld.n_dev = nullptr;
    }
    return PSLAM_OK;
}

static int validate(pslam_ctx* c, const pslam_frame_view* f, const pslam_map_points* m) {
    if (!f || !m || f->n < 0 || m->n < 0) return set_error(c, PSLAM_E_INVALID, "null view");
    if (f->n > SEARCH_MAX_KP || f->n > 65535) return set_error(c, PSLAM_E_INVALID, "more than 4096 keypoints in the frame view");
    if (f->n_levels < 1 || f->n_levels > PSLAM_MAX_LEVELS || !(f->max_x > f->min_x) || !(f->max_y > f->min_y)) return set_error(c, PSLAM_E_INVALID, "bad frame view");
    return PSLAM_OK;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_search_by_projection_map(pslam_ctx* c, const pslam_frame_view* f, const pslam_map_points* m, float th, float nnratio, int32_t* matches_io,
                                   uint8_t* in_view) {
    if (!c) return PSLAM_E_INVALID;
    int rc = validate(c, f, m);
    if (rc != PSLAM_OK) return rc;
    if (!matches_io) return set_error(c, PSLAM_E_INVALID, "null matches");
    if (f->n == 0 || m->n == 0) { if (in_view && m->n) std::memset(in_view, 0, m->n); return 0; }
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->search) c->search = new SearchBuffers();
    SearchBuffers& B = *c->search;
    if ((rc = ensure(c, B, (size_t)m->n)) != PSLAM_OK) return rc;
    SearchFrameDev F; SearchMapDev M; SearchLastDev Ld;
    if ((rc = upload(c, B, f, m, nullptr, F, M, Ld)) != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_matches, matches_io, f->n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemsetAsync(B.d_scalar, 0, 4 * sizeof(int32_t), st));
    PSLAM_LAUNCH(c, "search_grid", k_search_grid<<<1, 1024, 0, st>>>(F, B.d_cell_start, B.d_items));
    PSLAM_LAUNCH(c, "search_candidates_map", k_candidates_map<<<(M.n + 7) / 8, 256, 0, st>>>(F, M, th, B.d_cell_start, B.d_items, B.d_cand, B.d_cand_n,
                 B.d_in_view, B.d_scalar + 1));
    PSLAM_LAUNCH(c, "search_resolve_map", k_resolve_map<<<1, 32, 0, st>>>(M, nnratio, B.d_cand, B.d_cand_n, B.d_matches, B.d_scalar));
    int32_t sc[2] = {0, 0};
    PSLAM_CUDA(c, cudaMemcpyAsync(matches_io, B.d_matches, f->n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (in_view) PSLAM_CUDA(c, cudaMemcpyAsync(in_view, B.d_in_view, m->n, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(sc, B.d_scalar, sizeof sc, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    if (sc[1]) return set_error(c, PSLAM_E_CAPACITY, "more than 128 candidates in one search window");
    return sc[0];
}

int pslam_search_by_projection_last(pslam_ctx* c, const pslam_frame_view* cur, const pslam_last_frame* last, const pslam_map_points* m, float th,
                                    int mono, int check_orientation, int32_t* matches_io) {
    if (!c) return PSLAM_E_INVALID;
    int rc = validate(c, cur, m);
    if (rc != PSLAM_OK) return rc;
    if (!last || last->n < 0 || !matches_io) return set_error(c, PSLAM_E_INVALID, "null last-frame view or matches");
    if (cur->n == 0 || last->n == 0) return 0;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->search) c->search = new SearchBuffers();
    SearchBuffers& B = *c->search;
    if ((rc = ensure(c, B, (size_t)last->n)) != PSLAM_OK) return rc;
    SearchFrameDev F; SearchMapDev M; SearchLastDev Ld;
    if ((rc = upload(c, B, cur, m, last, F, M, Ld)) != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.d_matches, matches_io, cur->n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    PSLAM_CUDA(c, cudaMemsetAsync(B.d_scalar, 0, 4 * sizeof(int32_t), st));
    PSLAM_LAUNCH(c, "search_grid", k_search_grid<<<1, 1024, 0, st>>>(F, B.d_cell_start, B.d_items));
    PSLAM_LAUNCH(c, "search_candidates_last", k_candidates_last<<<(Ld.n + 7) / 8, 256, 0, st>>>(F, Ld, M, th, mono, B.d_cell_start, B.d_items, B.d_cand,
                 B.d_cand_n, B.d_scalar + 1));
    PSLAM_LAUNCH(c, "search_resolve_last", k_resolve_last<<<1, 32, 0, st>>>(F, Ld, M, check_orientation, B.d_cand, B.d_cand_n, B.d_matches, B.d_scalar,
                 B.d_hist_idx, B.d_hist_bin));
    int32_t sc[2] = {0, 0};
    PSLAM_CUDA(c, cudaMemcpyAsync(matches_io, B.d_matches, cur->n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(sc, B.d_scalar, sizeof sc, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    if (sc[1]) return set_error(c, PSLAM_E_CAPACITY, "more than 128 candidates in one search window");
    return sc[0];
}

}  // extern "C"

namespace pslam {
void search_free(pslam_ctx* c) {
    delete c->search;
    c->search = nullptr;
}
}  // namespace pslam
