// Host side of the local bundle adjustment: packs the caller's problems (the local map Optimizer::LocalBundleAdjustment
// gathers, src/Optimizer.cc:1853-2358) into flat device records plus the static work lists the kernel walks (landmark-major
// edge order, per-key-frame edge lists in creation order, the (edge, edge) term list of every pose-pair block of the Schur
// complement), launches one CTA per problem, unpacks the results.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>

#include "lba_kernels.cuh"

namespace pslam {

struct DevVec {                       // grow-only device array
    void* p = nullptr; size_t cap = 0;
    int ensure(pslam_ctx* c, size_t bytes) {
        if (bytes <= cap) return PSLAM_OK;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        const size_t nb = std::max<size_t>(bytes * 3 / 2, 256);
        const int rc = check_cuda(c, cudaMalloc(&p, nb), "cudaMalloc(lba)");
        if (rc == PSLAM_OK) cap = nb;
        return rc;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct LbaBuffers {
    int n_prob = 0;
    std::vector<LbaHeaderDev> hdr;
    // host staging (concatenated over the problems)
    std::vector<float> kf_Tcw0; std::vector<uint8_t> kf_fixed; std::vector<double> kf_K; std::vector<int32_t> kf_col;
    std::vector<int32_t> lm_type; std::vector<double> lm_val0;
    std::vector<LbaEdgeDev> edges; std::vector<int32_t> orig2sorted, kf_edge_off, kf_edge_idx, lm_edge_off, plane_edges, blk_ij, blk_term_off;
    std::vector<int2> terms;
    size_t tot_kf = 0, tot_lm = 0, tot_edges = 0, tot_col = 0, tot_flags = 0, tot_hs = 0;
    int max_smem = 0;
    // device
    DevVec d_hdr, d_kf_Tcw0, d_kf_fixed, d_kf_K, d_kf_col, d_kf_T, d_kf_Tb, d_kf_active, d_out_Tcw, d_Hpp, d_bp, d_coeff, d_xp, d_lm_type, d_lm_val0,
        d_lm_val, d_lm_valb, d_Hll, d_bl, d_Dinv, d_db, d_xl, d_lm_active, d_edges, d_err, d_JA, d_JB, d_we, d_re, d_W, d_Y, d_level, d_o2s,
        d_kf_eoff, d_kf_eidx, d_lm_eoff, d_plane_edges, d_blk_ij, d_blk_toff, d_terms, d_hs, d_flags, d_out;
    // fetch staging
    std::vector<double> h_Tcw, h_lm; std::vector<uint8_t> h_flags; std::vector<LbaOutDev> h_out;
    // per problem bookkeeping for fetch
    struct Shape { int n_kf, n_points, n_lines, n_planes, n_pt_obs, n_line_obs, n_plane_obs[3]; };
    std::vector<Shape> shape;
    void release() {
        for (DevVec* v : {&d_hdr, &d_kf_Tcw0, &d_kf_fixed, &d_kf_K, &d_kf_col, &d_kf_T, &d_kf_Tb, &d_kf_active, &d_out_Tcw, &d_Hpp, &d_bp, &d_coeff, &d_xp,
                          &d_lm_type, &d_lm_val0, &d_lm_val, &d_lm_valb, &d_Hll, &d_bl, &d_Dinv, &d_db, &d_xl, &d_lm_active, &d_edges, &d_err, &d_JA,
                          &d_JB, &d_we, &d_re, &d_W, &d_Y, &d_level, &d_o2s, &d_kf_eoff, &d_kf_eidx, &d_lm_eoff, &d_plane_edges, &d_blk_ij,
                          &d_blk_toff, &d_terms, &d_hs, &d_flags, &d_out})
            v->release();
    }
};

static void lba_plane_from_float4(const float* v, double out[4]) {     // Converter::toPlane3D + Plane3D::normalize
    double p[4] = {v[0], v[1], v[2], v[3]};
    if (v[3] < 0.0f) for (int i = 0; i < 4; ++i) p[i] = -p[i];
    const double n = std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    const double s = 1. / n;
    for (int i = 0; i < 4; ++i) p[i] = p[i] * s;
    if (p[3] < 0.0) for (int i = 0; i < 4; ++i) p[i] = -p[i];
    for (int i = 0; i < 4; ++i) out[i] = p[i];
}

static const int LBA_SMEM_BUDGET = 200 * 1024;      // dynamic shared memory we are willing to ask for (227 KB per CTA on sm_90)

int lba_pack_upload(pslam_ctx* c, const pslam_lba_problem* probs, int nprob) {
    if (!c->lba) c->lba = new LbaBuffers();
    LbaBuffers& B = *c->lba;
    B.n_prob = 0;
    B.hdr.assign(nprob, LbaHeaderDev());
    B.shape.assign(nprob, LbaBuffers::Shape());
    B.kf_Tcw0.clear(); B.kf_fixed.clear(); B.kf_K.clear(); B.kf_col.clear(); B.lm_type.clear(); B.lm_val0.clear(); B.edges.clear();
    B.orig2sorted.clear(); B.kf_edge_off.clear(); B.kf_edge_idx.clear(); B.lm_edge_off.clear(); B.plane_edges.clear(); B.blk_ij.clear();
    B.blk_term_off.clear(); B.terms.clear();
    B.tot_col = 0; B.tot_flags = 0; B.tot_hs = 0; B.max_smem = 0;

    for (int pi = 0; pi < nprob; ++pi) {
        const pslam_lba_problem& P = probs[pi];
        LbaHeaderDev& H = B.hdr[pi];
        std::memset(&H, 0, sizeof H);
        if (P.n_kf < 1 || P.n_points < 0 || P.n_pt_obs < 0 || P.n_lines < 0 || P.n_line_obs < 0 || P.n_planes < 0 || P.n_plane_obs[0] < 0 ||
            P.n_plane_obs[1] < 0 || P.n_plane_obs[2] < 0)
            return set_error(c, PSLAM_E_INVALID, "bad count in LBA problem");
        if (!P.kf_Tcw || !P.kf_fixed || !P.kf_K || (P.n_points && !P.pt_Xw) || (P.n_pt_obs && (!P.pt_obs_kf || !P.pt_obs_pt || !P.pt_obs_uvr || !P.pt_obs_inv_sigma2)) ||
            (P.n_lines && !P.line_Xw) || (P.n_line_obs && (!P.line_obs_kf || !P.line_obs_line || !P.line_obs_l)) || (P.n_planes && !P.plane_Xw))
            return set_error(c, PSLAM_E_INVALID, "null array in LBA problem");
        for (int t = 0; t < 3; ++t)
            if (P.n_plane_obs[t] && (!P.plane_obs_kf[t] || !P.plane_obs_plane[t] || !P.plane_obs_meas[t])) return set_error(c, PSLAM_E_INVALID, "null plane observation array");
        const int nkf = P.n_kf, nlm = P.n_points + 2 * P.n_lines + P.n_planes;
        const int lm_line0 = P.n_points, lm_plane0 = P.n_points + 2 * P.n_lines;
        H.n_kf = nkf; H.n_lm = nlm;
        H.kf_off = (int)B.kf_fixed.size(); H.lm_off = (int)B.lm_type.size(); H.edge_off = (int)B.edges.size();
        H.kfcsr_off = (int)B.kf_edge_off.size(); H.lmcsr_off = (int)B.lm_edge_off.size();
        H.plane_list_off = (int)B.plane_edges.size(); H.col_off = (int)B.tot_col; H.term_off = (int64_t)B.terms.size();
        H.blk_off = (int)(B.blk_ij.size() / 2); H.blkcsr_off = (int)B.blk_term_off.size();
        H.n_pt_obs = P.n_pt_obs; H.n_line_obs = P.n_line_obs;
        for (int t = 0; t < 3; ++t) H.n_plane_obs[t] = P.n_plane_obs[t];
        H.plane_chi = P.plane_chi; H.vp_chi = P.vp_chi;
        H.flag_off = (int)B.tot_flags;
        B.tot_flags += (size_t)P.n_pt_obs + P.n_line_obs + P.n_plane_obs[0] + P.n_plane_obs[1] + P.n_plane_obs[2];
        LbaBuffers::Shape& S = B.shape[pi];
        S.n_kf = nkf; S.n_points = P.n_points; S.n_lines = P.n_lines; S.n_planes = P.n_planes; S.n_pt_obs = P.n_pt_obs; S.n_line_obs = P.n_line_obs;
        for (int t = 0; t < 3; ++t) S.n_plane_obs[t] = P.n_plane_obs[t];

        // ---- key frames ----
        std::vector<int> col(nkf, -1);
        int nfree = 0;
        for (int k = 0; k < nkf; ++k) {
            for (int i = 0; i < 16; ++i) B.kf_Tcw0.push_back(P.kf_Tcw[16 * k + i]);
            B.kf_fixed.push_back(P.kf_fixed[k] ? 1 : 0);
            for (int i = 0; i < 5; ++i) B.kf_K.push_back((double)P.kf_K[5 * k + i]);
            if (!P.kf_fixed[k]) col[k] = nfree++;
            B.kf_col.push_back(col[k]);
        }
        H.n_free = nfree;
        B.tot_col += nfree;
        // ---- landmarks ----
        for (int i = 0; i < P.n_points; ++i) { B.lm_type.push_back(0); for (int k = 0; k < 3; ++k) B.lm_val0.push_back((double)P.pt_Xw[3 * i + k]); B.lm_val0.push_back(0.0); }
        for (int i = 0; i < P.n_lines; ++i)
            for (int s = 0; s < 2; ++s) { B.lm_type.push_back(0); for (int k = 0; k < 3; ++k) B.lm_val0.push_back(P.line_Xw[6 * i + 3 * s + k]); B.lm_val0.push_back(0.0); }
        for (int i = 0; i < P.n_planes; ++i) { B.lm_type.push_back(1); double pl[4]; lba_plane_from_float4(P.plane_Xw + 4 * i, pl); for (int k = 0; k < 4; ++k) B.lm_val0.push_back(pl[k]); }

        // ---- edges in creation order (points, line start/end pairs, plane, vertical, parallel) ----
        std::vector<LbaEdgeDev> ce;
        const float thHuberMono = std::sqrt(5.991), thHuberStereo = std::sqrt(7.815);          // const float in the reference (:2032-2033)
        const double angleInfo = 3282.8 / (P.angle_info * P.angle_info), disInfo = P.dist_info * P.dist_info;
        const float deltaPlane = std::sqrt(P.plane_chi), VPdeltaPlane = std::sqrt(P.vp_chi);
        auto bad_idx = [&](int kf, int lm, int nl) { return kf < 0 || kf >= nkf || lm < 0 || lm >= nl; };
        H.fam_off[0] = 0;
        for (int i = 0; i < P.n_pt_obs; ++i) {
            if (bad_idx(P.pt_obs_kf[i], P.pt_obs_pt[i], P.n_points)) return set_error(c, PSLAM_E_INVALID, "point observation index out of range");
            LbaEdgeDev e;
            std::memset(&e, 0, sizeof e);
            const float* o = P.pt_obs_uvr + 3 * i;
            const bool mono = o[2] < 0;
            e.kind = mono ? LK_MONO : LK_STEREO; e.kf = P.pt_obs_kf[i]; e.lm = P.pt_obs_pt[i];
            for (int k = 0; k < 3; ++k) { e.obs[k] = o[k]; e.info[k] = (double)P.pt_obs_inv_sigma2[i]; }
            e.delta = mono ? thHuberMono : thHuberStereo;
            ce.push_back(e);
        }
        H.fam_off[1] = (int)ce.size();
        for (int i = 0; i < P.n_line_obs; ++i) {
            if (bad_idx(P.line_obs_kf[i], P.line_obs_line[i], P.n_lines)) return set_error(c, PSLAM_E_INVALID, "line observation index out of range");
            for (int s = 0; s < 2; ++s) {
                LbaEdgeDev e;
                std::memset(&e, 0, sizeof e);
                e.kind = LK_LINE; e.kf = P.line_obs_kf[i]; e.lm = lm_line0 + 2 * P.line_obs_line[i] + s;
                for (int k = 0; k < 3; ++k) { e.obs[k] = P.line_obs_l[3 * i + k]; e.info[k] = 1.0; }
                e.delta = thHuberStereo;
                ce.push_back(e);
            }
        }
        for (int t = 0; t < 3; ++t) {
            H.fam_off[2 + t] = (int)ce.size();
            for (int i = 0; i < P.n_plane_obs[t]; ++i) {
                if (bad_idx(P.plane_obs_kf[t][i], P.plane_obs_plane[t][i], P.n_planes)) return set_error(c, PSLAM_E_INVALID, "plane observation index out of range");
                LbaEdgeDev e;
                std::memset(&e, 0, sizeof e);
                e.kind = t == 0 ? LK_PLANE : (t == 1 ? LK_VER : LK_PAR); e.kf = P.plane_obs_kf[t][i]; e.lm = lm_plane0 + P.plane_obs_plane[t][i];
                lba_plane_from_float4(P.plane_obs_meas[t] + 4 * i, e.obs);
                e.info[0] = e.info[1] = angleInfo; e.info[2] = t == 0 ? disInfo : 0.0;       // VPInfo uses angleInfo (:2274-2276)
                e.delta = t == 0 ? deltaPlane : VPdeltaPlane;
                ce.push_back(e);
            }
        }
        const int ne = (int)ce.size();
        H.n_edges = ne;
        for (int i = 0; i < ne; ++i) ce[i].orig = i;
        // landmark-major stable order
        std::vector<int> order(ne);
        std::iota(order.begin(), order.end(), 0);
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return ce[a].lm < ce[b].lm; });
        std::vector<int> o2s(ne);
        for (int s = 0; s < ne; ++s) o2s[order[s]] = s;
        std::vector<int> lm_off(nlm + 1, 0);
        for (int i = 0; i < ne; ++i) ++lm_off[ce[i].lm + 1];
        for (int l = 0; l < nlm; ++l) lm_off[l + 1] += lm_off[l];
        for (int s = 0; s < ne; ++s) B.edges.push_back(ce[order[s]]);
        for (int i = 0; i < ne; ++i) B.orig2sorted.push_back(o2s[i]);
        for (int l = 0; l <= nlm; ++l) B.lm_edge_off.push_back(lm_off[l]);
        // per key frame, creation order
        std::vector<int> kf_off(nkf + 1, 0);
        for (int i = 0; i < ne; ++i) ++kf_off[ce[i].kf + 1];
        for (int k = 0; k < nkf; ++k) kf_off[k + 1] += kf_off[k];
        {
            std::vector<int> cur(kf_off.begin(), kf_off.end() - 1), idx(ne);
            for (int i = 0; i < ne; ++i) idx[cur[ce[i].kf]++] = o2s[i];
            for (int k = 0; k <= nkf; ++k) B.kf_edge_off.push_back(kf_off[k]);
            for (int i = 0; i < ne; ++i) B.kf_edge_idx.push_back(idx[i]);
        }
        // plane-type edges
        int npe = 0;
        for (int s = 0; s < ne; ++s) if (lk_is_plane(ce[order[s]].kind)) { B.plane_edges.push_back(s); ++npe; }
        H.n_plane_edges = npe;
        // ---- Schur terms: for every landmark, every ordered pair (o, q) of its free-pose edges with col(o) <= col(q) ----
        const int nblk = nfree * (nfree + 1) / 2;
        H.n_blk = nblk;
        auto blk_index = [&](int ci, int cj) { return ci * nfree - ci * (ci - 1) / 2 + (cj - ci); };
        for (int ci = 0; ci < nfree; ++ci) for (int cj = ci; cj < nfree; ++cj) { B.blk_ij.push_back(ci); B.blk_ij.push_back(cj); }
        std::vector<int> cnt(nblk + 1, 0);
        std::vector<std::pair<int, int2>> tl;       // (block, (sorted e1, sorted e2)) in (landmark, o, q) order
        for (int l = 0; l < nlm; ++l) {
            std::vector<int> lst;
            for (int s = lm_off[l]; s < lm_off[l + 1]; ++s) if (col[B.edges[H.edge_off + s].kf] >= 0) lst.push_back(s);
            std::stable_sort(lst.begin(), lst.end(), [&](int a, int b) { return col[B.edges[H.edge_off + a].kf] < col[B.edges[H.edge_off + b].kf]; });
            for (size_t o = 0; o < lst.size(); ++o)
                for (size_t q = 0; q < lst.size(); ++q) {
                    const int ci = col[B.edges[H.edge_off + lst[o]].kf], cj = col[B.edges[H.edge_off + lst[q]].kf];
                    if (cj < ci) continue;
                    const int bk = blk_index(ci, cj);
                    tl.push_back({bk, make_int2(lst[o], lst[q])});
                    ++cnt[bk + 1];
                }
        }
        for (int b = 0; b < nblk; ++b) cnt[b + 1] += cnt[b];
        {
            std::vector<int> cur(cnt.begin(), cnt.end() - 1);
            const size_t base = B.terms.size();
            B.terms.resize(base + tl.size());
            for (const auto& t : tl) B.terms[base + cur[t.first]++] = t.second;       // counting sort: stable
            for (int b = 0; b <= nblk; ++b) B.blk_term_off.push_back(cnt[b]);
        }
        // ---- Schur matrix placement ----
        const int n = 6 * nfree;
        H.ld = n | 1;
        const size_t hs_doubles = (size_t)n * H.ld + 2 * (size_t)n + 8;
        H.use_smem = hs_doubles * 8 <= (size_t)LBA_SMEM_BUDGET ? 1 : 0;
        H.hs_off = (int64_t)B.tot_hs;
        if (H.use_smem) B.max_smem = std::max(B.max_smem, (int)(hs_doubles * 8)); else B.tot_hs += hs_doubles;
    }
    B.tot_kf = B.kf_fixed.size(); B.tot_lm = B.lm_type.size(); B.tot_edges = B.edges.size();

    // ---- device allocation + upload ----
    int rc;
#define ENS(v, bytes) if ((rc = B.v.ensure(c, std::max<size_t>((bytes), 8))) != PSLAM_OK) return rc
    ENS(d_hdr, nprob * sizeof(LbaHeaderDev)); ENS(d_out, nprob * sizeof(LbaOutDev));
    ENS(d_kf_Tcw0, B.tot_kf * 16 * 4); ENS(d_kf_fixed, B.tot_kf); ENS(d_kf_K, B.tot_kf * 5 * 8); ENS(d_kf_col, B.tot_kf * 4);
    ENS(d_kf_T, B.tot_kf * 8 * 8); ENS(d_kf_Tb, B.tot_kf * 8 * 8); ENS(d_kf_active, B.tot_kf); ENS(d_out_Tcw, B.tot_kf * 16 * 8);
    ENS(d_Hpp, B.tot_col * 36 * 8); ENS(d_bp, B.tot_col * 6 * 8); ENS(d_coeff, B.tot_col * 6 * 8); ENS(d_xp, B.tot_col * 6 * 8);
    ENS(d_lm_type, B.tot_lm * 4); ENS(d_lm_val0, B.tot_lm * 4 * 8); ENS(d_lm_val, B.tot_lm * 4 * 8); ENS(d_lm_valb, B.tot_lm * 4 * 8);
    ENS(d_Hll, B.tot_lm * 9 * 8); ENS(d_bl, B.tot_lm * 3 * 8); ENS(d_Dinv, B.tot_lm * 9 * 8); ENS(d_db, B.tot_lm * 3 * 8); ENS(d_xl, B.tot_lm * 3 * 8);
    ENS(d_lm_active, B.tot_lm);
    ENS(d_edges, B.tot_edges * sizeof(LbaEdgeDev)); ENS(d_err, B.tot_edges * 3 * 8); ENS(d_JA, B.tot_edges * 9 * 8); ENS(d_JB, B.tot_edges * 18 * 8);
    ENS(d_we, B.tot_edges * 3 * 8); ENS(d_re, B.tot_edges * 3 * 8); ENS(d_W, B.tot_edges * 18 * 8); ENS(d_Y, B.tot_edges * 18 * 8);
    ENS(d_level, B.tot_edges); ENS(d_o2s, B.tot_edges * 4);
    ENS(d_kf_eoff, B.kf_edge_off.size() * 4); ENS(d_kf_eidx, B.tot_edges * 4); ENS(d_lm_eoff, B.lm_edge_off.size() * 4);
    ENS(d_plane_edges, B.plane_edges.size() * 4); ENS(d_blk_ij, B.blk_ij.size() * 4); ENS(d_blk_toff, B.blk_term_off.size() * 4);
    ENS(d_terms, B.terms.size() * sizeof(int2)); ENS(d_hs, B.tot_hs * 8); ENS(d_flags, B.tot_flags);
#undef ENS
    cudaStream_t st = c->stream;
#define UP(v, vec) if (!(vec).empty()) PSLAM_CUDA(c, cudaMemcpyAsync(B.v.p, (vec).data(), (vec).size() * sizeof((vec)[0]), cudaMemcpyHostToDevice, st))
    UP(d_hdr, B.hdr); UP(d_kf_Tcw0, B.kf_Tcw0); UP(d_kf_fixed, B.kf_fixed); UP(d_kf_K, B.kf_K); UP(d_kf_col, B.kf_col);
    UP(d_lm_type, B.lm_type); UP(d_lm_val0, B.lm_val0); UP(d_edges, B.edges); UP(d_o2s, B.orig2sorted); UP(d_kf_eoff, B.kf_edge_off);
    UP(d_kf_eidx, B.kf_edge_idx); UP(d_lm_eoff, B.lm_edge_off); UP(d_plane_edges, B.plane_edges); UP(d_blk_ij, B.blk_ij);
    UP(d_blk_toff, B.blk_term_off); UP(d_terms, B.terms);
#undef UP
    PSLAM_CUDA(c, cudaStreamSynchronize(st));       // the staging vectors are pageable
    B.n_prob = nprob;
    return PSLAM_OK;
}

int lba_run_packed(pslam_ctx* c) {
    if (!c->lba || c->lba->n_prob < 1) return set_error(c, PSLAM_E_INVALID, "no packed LBA problems");
    LbaBuffers& B = *c->lba;
    LbaArrays A;
    A.hdr = (const LbaHeaderDev*)B.d_hdr.p;
    A.kf_Tcw0 = (const float*)B.d_kf_Tcw0.p; A.kf_fixed = (const uint8_t*)B.d_kf_fixed.p; A.kf_K = (const double*)B.d_kf_K.p; A.kf_col = (const int32_t*)B.d_kf_col.p;
    A.kf_T = (double*)B.d_kf_T.p; A.kf_Tb = (double*)B.d_kf_Tb.p; A.kf_active = (uint8_t*)B.d_kf_active.p; A.out_Tcw = (double*)B.d_out_Tcw.p;
    A.Hpp = (double*)B.d_Hpp.p; A.bp = (double*)B.d_bp.p; A.coeff = (double*)B.d_coeff.p; A.xp = (double*)B.d_xp.p;
    A.lm_type = (const int32_t*)B.d_lm_type.p; A.lm_val0 = (const double*)B.d_lm_val0.p; A.lm_val = (double*)B.d_lm_val.p; A.lm_valb = (double*)B.d_lm_valb.p;
    A.Hll = (double*)B.d_Hll.p; A.bl = (double*)B.d_bl.p; A.Dinv = (double*)B.d_Dinv.p; A.db = (double*)B.d_db.p; A.xl = (double*)B.d_xl.p;
    A.lm_active = (uint8_t*)B.d_lm_active.p;
    A.edges = (const LbaEdgeDev*)B.d_edges.p; A.err = (double*)B.d_err.p; A.JA = (double*)B.d_JA.p; A.JB = (double*)B.d_JB.p; A.we = (double*)B.d_we.p;
    A.re = (double*)B.d_re.p; A.W = (double*)B.d_W.p; A.Y = (double*)B.d_Y.p; A.level = (uint8_t*)B.d_level.p; A.orig2sorted = (const int32_t*)B.d_o2s.p;
    A.kf_edge_off = (const int32_t*)B.d_kf_eoff.p; A.kf_edge_idx = (const int32_t*)B.d_kf_eidx.p; A.lm_edge_off = (const int32_t*)B.d_lm_eoff.p;
    A.plane_edges = (const int32_t*)B.d_plane_edges.p; A.blk_ij = (const int32_t*)B.d_blk_ij.p; A.blk_term_off = (const int32_t*)B.d_blk_toff.p;
    A.terms = (const int2*)B.d_terms.p; A.hs_global = (double*)B.d_hs.p; A.flags = (uint8_t*)B.d_flags.p; A.out = (LbaOutDev*)B.d_out.p;
    // per device and cheap: set on every launch (contexts of one process may live on different GPUs)
    PSLAM_CUDA(c, cudaFuncSetAttribute(k_local_bundle_adjustment, cudaFuncAttributeMaxDynamicSharedMemorySize, LBA_SMEM_BUDGET));
    PSLAM_LAUNCH(c, "local_bundle_adjustment", k_local_bundle_adjustment<<<B.n_prob, LBA_THREADS, B.max_smem, c->stream>>>(A));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

int lba_fetch(pslam_ctx* c, pslam_lba_result* res) {
    if (!c->lba || c->lba->n_prob < 1) return set_error(c, PSLAM_E_INVALID, "no packed LBA problems");
    LbaBuffers& B = *c->lba;
    B.h_Tcw.resize(B.tot_kf * 16); B.h_lm.resize(B.tot_lm * 4); B.h_flags.resize(std::max<size_t>(B.tot_flags, 1)); B.h_out.resize(B.n_prob);
    cudaStream_t st = c->stream;
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_Tcw.data(), B.d_out_Tcw.p, B.tot_kf * 16 * 8, cudaMemcpyDeviceToHost, st));
    if (B.tot_lm) PSLAM_CUDA(c, cudaMemcpyAsync(B.h_lm.data(), B.d_lm_val.p, B.tot_lm * 4 * 8, cudaMemcpyDeviceToHost, st));
    if (B.tot_flags) PSLAM_CUDA(c, cudaMemcpyAsync(B.h_flags.data(), B.d_flags.p, B.tot_flags, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_out.data(), B.d_out.p, B.n_prob * sizeof(LbaOutDev), cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    for (int p = 0; p < B.n_prob; ++p) {
        const LbaHeaderDev& H = B.hdr[p];
        const LbaBuffers::Shape& S = B.shape[p];
        pslam_lba_result& R = res[p];
        const double* T = B.h_Tcw.data() + (size_t)H.kf_off * 16;
        for (int i = 0; i < S.n_kf * 16; ++i) {                       // Converter::toCvMat(SE3Quat): float
            if (R.kf_Tcw) R.kf_Tcw[i] = (float)T[i];
            if (R.kf_Tcw_d) R.kf_Tcw_d[i] = T[i];
        }
        const double* L = B.h_lm.data() + (size_t)H.lm_off * 4;
        for (int i = 0; i < S.n_points; ++i)
            for (int k = 0; k < 3; ++k) {
                if (R.pt_Xw) R.pt_Xw[3 * i + k] = (float)L[4 * i + k];
                if (R.pt_Xw_d) R.pt_Xw_d[3 * i + k] = L[4 * i + k];
            }
        const double* LL = L + (size_t)S.n_points * 4;
        for (int i = 0; i < S.n_lines; ++i)
            for (int s = 0; s < 2; ++s)
                for (int k = 0; k < 3; ++k) {
                    const double v = LL[4 * (2 * i + s) + k];
                    if (R.line_Xw) R.line_Xw[6 * i + 3 * s + k] = (double)(float)v;     // toVector3d(toCvMat(.)) round trip (:2655-2658)
                    if (R.line_Xw_d) R.line_Xw_d[6 * i + 3 * s + k] = v;
                }
        const double* LP = LL + (size_t)S.n_lines * 8;
        for (int i = 0; i < S.n_planes * 4; ++i) {
            if (R.plane_Xw) R.plane_Xw[i] = (float)LP[i];
            if (R.plane_Xw_d) R.plane_Xw_d[i] = LP[i];
        }
        const uint8_t* f = B.h_flags.data() + H.flag_off;
        if (R.erase_pt && S.n_pt_obs) std::memcpy(R.erase_pt, f, S.n_pt_obs);
        f += S.n_pt_obs;
        if (R.erase_line && S.n_line_obs) std::memcpy(R.erase_line, f, S.n_line_obs);
        f += S.n_line_obs;
        for (int t = 0; t < 3; ++t) { if (R.erase_plane[t] && S.n_plane_obs[t]) std::memcpy(R.erase_plane[t], f, S.n_plane_obs[t]); f += S.n_plane_obs[t]; }
        for (int k = 0; k < 2; ++k) {
            R.iterations[k] = B.h_out[p].iterations[k]; R.trials[k] = B.h_out[p].trials[k]; R.chi2[k] = B.h_out[p].chi2[k]; R.lambda[k] = B.h_out[p].lambda[k];
        }
    }
    return PSLAM_OK;
}

void lba_free(pslam_ctx* c) {
    if (!c->lba) return;
    c->lba->release();
    delete c->lba;
    c->lba = nullptr;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_lba_pack(pslam_ctx* c, const pslam_lba_problem* probs, int n) {
    if (!c) return PSLAM_E_INVALID;
    if (!probs || n < 1) return set_error(c, PSLAM_E_INVALID, "null problems or n < 1");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return lba_pack_upload(c, probs, n);
}
int pslam_lba_run_packed(pslam_ctx* c) {
    if (!c) return PSLAM_E_INVALID;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return lba_run_packed(c);
}
int pslam_lba_fetch(pslam_ctx* c, pslam_lba_result* res) {
    if (!c) return PSLAM_E_INVALID;
    if (!res) return set_error(c, PSLAM_E_INVALID, "null result array");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return lba_fetch(c, res);
}
int pslam_local_bundle_adjustment_batch(pslam_ctx* c, const pslam_lba_problem* probs, int n, pslam_lba_result* res) {
    int rc = pslam_lba_pack(c, probs, n);
    if (rc != PSLAM_OK) return rc;
    if ((rc = lba_run_packed(c)) != PSLAM_OK) return rc;
    return pslam_lba_fetch(c, res);
}
int pslam_local_bundle_adjustment(pslam_ctx* c, const pslam_lba_problem* prob, pslam_lba_result* res) {
    return pslam_local_bundle_adjustment_batch(c, prob, 1, res);
}

}  // extern "C"
