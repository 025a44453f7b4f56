// TEST INFRASTRUCTURE ONLY — C entry points (ctypes) onto the oracle PEAC plane extractor.
#include "peac.h"
#include <cstring>
#include <queue>
using namespace oracle;
extern "C" {
void* orc_peac_run(const uint16_t* depth, int w, int h, float fx, float fy, float cx, float cy, float scale) {
    PeacResult* r = new PeacResult();
    peac_run(depth, w, h, fx, fy, cx, cy, scale, PeacParams(), *r);
    return r;
}
void orc_peac_free(void* p) { delete (PeacResult*)p; }
int orc_peac_num_planes(void* p) { return (int)((PeacResult*)p)->planes.size(); }
int orc_peac_num_coarse(void* p) { return ((PeacResult*)p)->n_coarse_planes; }
int orc_peac_queue_len(void* p, int which) { return which ? ((PeacResult*)p)->n_queue : ((PeacResult*)p)->n_seeds; }
void orc_peac_labels(void* p, int32_t* out) { auto* r = (PeacResult*)p; std::memcpy(out, r->labels.data(), r->labels.size() * 4); }
// per plane: normal[3], center[3], mse, curvature (8 doubles); N, rid (2 ints)
void orc_peac_plane(void* p, int i, double* d8, int* i2) {
    const PeacPlane& q = ((PeacResult*)p)->planes[i];
    for (int k = 0; k < 3; ++k) { d8[k] = q.normal[k]; d8[3 + k] = q.center[k]; }
    d8[6] = q.mse; d8[7] = q.curvature; i2[0] = q.N; i2[1] = q.rid;
}
int orc_peac_membership(void* p, int i, int32_t* out, int cap) {
    const auto& m = ((PeacResult*)p)->membership[i];
    for (int k = 0; k < (int)m.size() && k < cap; ++k) out[k] = m[k];
    return (int)m.size();
}
// per block: 9 sums + center[3] + normal[3] + mse + curvature = 17 doubles; N, valid = 2 ints
int orc_peac_blocks(void* p, double* d17, int* i2) {
    auto* r = (PeacResult*)p;
    for (size_t b = 0; b < r->blocks.size(); ++b) {
        const PeacBlock& k = r->blocks[b];
        double* d = d17 + b * 17;
        d[0] = k.stats.sx; d[1] = k.stats.sy; d[2] = k.stats.sz; d[3] = k.stats.sxx; d[4] = k.stats.syy; d[5] = k.stats.szz;
        d[6] = k.stats.sxy; d[7] = k.stats.syz; d[8] = k.stats.sxz;
        for (int q = 0; q < 3; ++q) { d[9 + q] = k.center[q]; d[12 + q] = k.normal[q]; }
        d[15] = k.mse; d[16] = k.curvature;
        i2[2 * b] = k.stats.N; i2[2 * b + 1] = k.valid;
    }
    return (int)r->blocks.size();
}
void orc_peac_coarse_blocks(void* p, int32_t* out) { auto* r = (PeacResult*)p; std::memcpy(out, r->coarse_block_plane.data(), r->coarse_block_plane.size() * 4); }
void orc_eig33(const double* K9, double* s3, double* V9) {
    double K[3][3], V[3][3];
    for (int i = 0; i < 9; ++i) K[i / 3][i % 3] = K9[i];
    eig33sym_jacobi(K, s3, V);
    for (int i = 0; i < 9; ++i) V9[i] = V[i / 3][i % 3];
}
// heap order self-check: pops of a sequence of (push id with key) / (pop) ops through the oracle's explicit heap vs
// std::priority_queue with the reference comparator must agree even with tied keys.
int orc_heap_selftest(const double* keys, int n, const int* ops, int nops) {
    struct Cmp { const double* k; bool operator()(int a, int b) const { return k[b] < k[a]; } };
    std::priority_queue<int, std::vector<int>, Cmp> ref(Cmp{keys});
    // explicit heap (same code shape as peac.cc MinMseHeap)
    std::vector<int> h;
    auto comp = [&](int a, int b) { return keys[b] < keys[a]; };
    auto sift_up = [&](int hole, int top, int value) { int parent = (hole - 1) / 2; while (hole > top && comp(h[parent], value)) { h[hole] = h[parent]; hole = parent; parent = (hole - 1) / 2; } h[hole] = value; };
    int next = 0, bad = 0;
    for (int i = 0; i < nops; ++i) {
        if (ops[i] == 1 && next < n) { ref.push(next); h.push_back(next); sift_up((int)h.size() - 1, 0, next); ++next; }
        else if (!ref.empty()) {
            int a = ref.top(); ref.pop();
            int top = h[0], value = h.back(); h.pop_back();
            int len = (int)h.size();
            if (len > 0) {
                int hole = 0, child = 0;
                while (child < (len - 1) / 2) { child = 2 * (child + 1); if (comp(h[child], h[child - 1])) --child; h[hole] = h[child]; hole = child; }
                if ((len & 1) == 0 && child == (len - 2) / 2) { child = 2 * (child + 1); h[hole] = h[child - 1]; hole = child - 1; }
                sift_up(hole, 0, value);
            }
            if (a != top) ++bad;
        }
    }
    return bad;
}
}

#include "planepost.h"
extern "C" {
// Frame::ComputePlanes post-processing on the PEAC result `p`: returns the number of kept planes; src [n], coef [n][4], npts [n], pts (concatenated xyz, capacity
// cap_pts points), stats [n][2] = RANSAC inliers / iterations
int orc_planes_post(void* p, const uint16_t* depth, int w, int h, float fx, float fy, float cx, float cy, float scale, double dist_th, int32_t* src, float* coef,
                    int32_t* npts, float* pts, int cap_pts, int32_t* stats) {
    std::vector<oracle::PostPlane> out;
    oracle::compute_planes_post(depth, w, h, oracle::PlanePostParams{fx, fy, cx, cy, scale, dist_th}, *(PeacResult*)p, out);
    int tot = 0;
    for (size_t i = 0; i < out.size(); ++i) {
        src[i] = out[i].src; std::memcpy(coef + 4 * i, out[i].coef, 16); npts[i] = (int)out[i].points.size() / 3; stats[2 * i] = out[i].n_inliers; stats[2 * i + 1] = out[i].n_iterations;
        for (size_t k = 0; k < out[i].points.size() / 3 && tot < cap_pts; ++k, ++tot) std::memcpy(pts + 3 * (size_t)tot, &out[i].points[3 * k], 12);
    }
    return (int)out.size();
}
// The same post-processing on plane records given by the caller instead of a PEAC run: n_planes planes, normal_center [n][6] (PeacPlane::normal, ::center),
// member_off [n + 1] into members (pixel indices).  Outputs as orc_planes_post.
int orc_planes_post_records(const uint16_t* depth, int w, int h, float fx, float fy, float cx, float cy, float scale, double dist_th, int n_planes,
                            const double* normal_center, const int32_t* member_off, const int32_t* members, int32_t* src, float* coef, int32_t* npts, float* pts,
                            int cap_pts, int32_t* stats) {
    PeacResult r;
    r.w = w; r.h = h;
    r.planes.resize(n_planes);
    r.membership.resize(n_planes);
    for (int i = 0; i < n_planes; ++i) {
        for (int k = 0; k < 3; ++k) { r.planes[i].normal[k] = normal_center[6 * i + k]; r.planes[i].center[k] = normal_center[6 * i + 3 + k]; }
        r.membership[i].assign(members + member_off[i], members + member_off[i + 1]);
    }
    return orc_planes_post(&r, depth, w, h, fx, fy, cx, cy, scale, dist_th, src, coef, npts, pts, cap_pts, stats);
}
// vSurfaceNormal: out [n][8] = normal xyz, camera position xyz, frame position xy; returns n
int orc_surface_normals(const uint16_t* depth, int w, int h, float fx, float fy, float cx, float cy, float scale, float* out8, int cap) {
    std::vector<oracle::SurfaceNormal> v;
    oracle::surface_normals(depth, w, h, oracle::PlanePostParams{fx, fy, cx, cy, scale, 0.0}, v);
    for (size_t i = 0; i < v.size() && (int)i < cap; ++i) std::memcpy(out8 + 8 * i, &v[i], 32);
    return (int)v.size();
}
// MapPlane::UpdateCoefficientsAndPoints: clouds as CSR (cloud_off [n_clouds + 1] in points, pts xyz), T [n_clouds][16]; returns the number of voxel centroids
int orc_map_plane_update(int n_clouds, const int32_t* cloud_off, const float* pts, const double* T, float* out, int cap) {
    std::vector<std::vector<float>> clouds(n_clouds);
    std::vector<const double*> Ts(n_clouds);
    for (int c = 0; c < n_clouds; ++c) { clouds[c].assign(pts + 3 * (size_t)cloud_off[c], pts + 3 * (size_t)cloud_off[c + 1]); Ts[c] = T + 16 * (size_t)c; }
    std::vector<float> o;
    oracle::map_plane_update(clouds, Ts, o);
    for (size_t i = 0; i < o.size() && (int)(i / 3) < cap; ++i) out[i] = o[i];
    return (int)o.size() / 3;
}
uint32_t orc_pcl_rng(int n) { oracle::PclRng r; uint32_t v = 0; for (int i = 0; i < n; ++i) v = r.next_u32(); return v; }
}
