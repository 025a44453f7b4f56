// ORBmatcher::SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&) on sm_90a (src/ORBmatcher.cc:160-292).  A frame feature belongs
// to exactly one vocabulary node, so the common nodes of the two feature vectors are independent sub-problems: one warp per
// common node walks the key-frame features of the node in order (an earlier match takes its frame feature away from later
// ones), the lanes evaluate the 256-bit Hamming distances to the node's frame features, a warp top-2 gives the reference's
// best / second-best, and a second kernel applies the rotation-histogram filter (ComputeThreeMaxima, :1666-1707).
// The same kernels serve ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, vector<MapPoint*>&) (:526-659, the loop-closure matcher): both sides carry map-point
// flags there and the distance gate is strict (bestDist1 < TH_LOW instead of <=).
//
// Loop-closure / relocalisation candidates (KeyFrameDatabase::DetectLoopCandidates / DetectRelocalizationCandidates, src/KeyFrameDatabase.cc:76-305): the
// database's BowVectors live in HBM as CSR (pslam_bow_database_set); k_bow_db_scores runs one warp per key frame - lanes look the key frame's words up in the
// query (binary search), count the shared words, and fold the DBoW2 L1 terms (Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68) in ascending word order, the
// order the reference's merge loop adds them in, so the double sum (and the float it is stored as) is bit-identical.  The list logic that follows (common-word
// gate, covisibility accumulation, 0.75 x best) touches a few dozen key frames and runs on the host over the downloaded per-key-frame triples.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

#include "bowdb_select.h"
#include "pslam_internal.h"

namespace pslam {

__device__ __forceinline__ void bow_top2(uint32_t& k0, uint32_t& k1) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const uint32_t o0 = __shfl_xor_sync(0xffffffffu, k0, o), o1 = __shfl_xor_sync(0xffffffffu, k1, o);
        const uint32_t lo = min(k0, o0), hi = max(k0, o0);
        k1 = min(hi, min(k1, o1));
        k0 = lo;
    }
}

__global__ void __launch_bounds__(128) k_bow_nodes(int n_pairs, const int2* __restrict__ pairs, const uint8_t* __restrict__ kf_desc, const float* __restrict__ kf_angle,
                                                   const uint8_t* __restrict__ kf_has_mp, const int32_t* __restrict__ kf_off, const int32_t* __restrict__ kf_feat,
                                                   const uint8_t* __restrict__ f_desc, const float* __restrict__ f_angle, const int32_t* __restrict__ f_off,
                                                   const int32_t* __restrict__ f_feat, const uint8_t* __restrict__ f_has_mp, int th_low, float nnratio, int check_ori,
                                                   int32_t* __restrict__ match,
                                                   int8_t* __restrict__ bin_of, int32_t* __restrict__ hist, int32_t* __restrict__ nmatches) {
    const int lane = threadIdx.x & 31, w = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (w >= n_pairs) return;
    const int a = pairs[w].x, b = pairs[w].y;
    const int f0 = f_off[b], nfn = f_off[b + 1] - f0;
    const uint32_t NONE = 0xffffffffu;
    int nm = 0;
    for (int q = kf_off[a]; q < kf_off[a + 1]; ++q) {
        const int ik = kf_feat[q];
        if (!kf_has_mp[ik]) continue;
        uint32_t dk[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) dk[t] = reinterpret_cast<const uint32_t*>(kf_desc)[8 * ik + t];
        uint32_t k0 = NONE, k1 = NONE;
        for (int p = lane; p < nfn; p += 32) {
            const int jf = f_feat[f0 + p];
            if (match[jf] >= 0 || (f_has_mp && !f_has_mp[jf])) continue;
            int d = 0;
#pragma unroll
            for (int t = 0; t < 8; ++t) d += __popc(dk[t] ^ reinterpret_cast<const uint32_t*>(f_desc)[8 * jf + t]);
            const uint32_t key = ((uint32_t)d << 16) | (uint32_t)p;      // ties: the first frame feature of the node wins (strict <)
            if (key < k0) { k1 = k0; k0 = key; } else if (key < k1) k1 = key;
        }
        bow_top2(k0, k1);
        if (k0 == NONE) continue;
        const int bestDist1 = (int)(k0 >> 16), bestDist2 = k1 == NONE ? 256 : (int)(k1 >> 16);
        if (bestDist1 <= th_low && (float)bestDist1 < __fmul_rn(nnratio, (float)bestDist2)) {
            const int jf = f_feat[f0 + (k0 & 0xffff)];
            if (lane == 0) {
                match[jf] = ik;
                if (check_ori) {
                    float rot = __fsub_rn(kf_angle[ik], f_angle[jf]);
                    if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
                    int bin = (int)roundf(__fmul_rn(rot, 1.0f / 30));
                    if (bin == 30) bin = 0;
                    bin_of[jf] = (int8_t)bin;
                    atomicAdd(&hist[bin], 1);
                }
            }
            ++nm;
            __syncwarp();
        }
    }
    if (lane == 0 && nm) atomicAdd(nmatches, nm);
}

__global__ void __launch_bounds__(256) k_bow_orientation(int nf, int32_t* __restrict__ match, const int8_t* __restrict__ bin_of, const int32_t* __restrict__ hist,
                                                         int32_t* __restrict__ nmatches) {
    __shared__ int s_ind[3];
    if (threadIdx.x == 0) {
        int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
        for (int i = 0; i < 30; ++i) {
            const int s = hist[i];
            if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
            else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
            else if (s > max3) { max3 = s; ind3 = i; }
        }
        if ((float)max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; } else if ((float)max3 < 0.1f * (float)max1) ind3 = -1;
        s_ind[0] = ind1; s_ind[1] = ind2; s_ind[2] = ind3;
    }
    __syncthreads();
    int removed = 0;
    for (int j = blockIdx.x * 256 + threadIdx.x; j < nf; j += gridDim.x * 256) {
        if (match[j] < 0) continue;
        const int b = bin_of[j];
        if (b != s_ind[0] && b != s_ind[1] && b != s_ind[2]) { match[j] = -1; ++removed; }
    }
    if (removed) atomicSub(nmatches, removed);
}

struct BowDbBuffers {
    int n_kf = 0, total = 0;
    int32_t* d_off = nullptr; int32_t* d_word = nullptr; double* d_val = nullptr;
    int32_t* d_common = nullptr; int32_t* d_first = nullptr; float* d_score = nullptr;
    int32_t* d_qword = nullptr; double* d_qval = nullptr; int q_cap = 0;
    std::vector<int32_t> h_common, h_first; std::vector<float> h_score;
};

void bowdb_free(pslam_ctx* c) {
    if (!c->bowdb) return;
    BowDbBuffers& B = *c->bowdb;
    cudaFree(B.d_off); cudaFree(B.d_word); cudaFree(B.d_val); cudaFree(B.d_common); cudaFree(B.d_first); cudaFree(B.d_score); cudaFree(B.d_qword); cudaFree(B.d_qval);
    delete c->bowdb;
    c->bowdb = nullptr;
}

// One warp per key frame of the database.  Query and key-frame words are ascending, so the shared words come out in the order of the reference's merge loop.
__global__ void __launch_bounds__(128) k_bow_db_scores(int n_kf, const int32_t* __restrict__ off, const int32_t* __restrict__ word, const double* __restrict__ val, int n_q,
                                                       const int32_t* __restrict__ q_word, const double* __restrict__ q_val, int32_t* __restrict__ common,
                                                       int32_t* __restrict__ first, float* __restrict__ score) {
    const int lane = threadIdx.x & 31, k = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (k >= n_kf) return;
    const int b = off[k], e = off[k + 1];
    int n_common = 0, first_q = -1;
    double sum = 0.0;
    for (int base = b; base < e; base += 32) {
        const int i = base + lane;
        int qi = -1;
        double term = 0.0;
        if (i < e) {
            const int32_t w = word[i];
            int lo = 0, hi = n_q;                      // lower_bound of w in the query's words
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (q_word[mid] < w) lo = mid + 1; else hi = mid; }
            if (lo < n_q && q_word[lo] == w) {
                qi = lo;
                const double vi = q_val[lo], wi = val[i];
                term = (fabs(vi - wi) - fabs(vi)) - fabs(wi);
            }
        }
        unsigned hits = __ballot_sync(0xffffffffu, qi >= 0);
        if (hits && first_q < 0) first_q = __shfl_sync(0xffffffffu, qi, __ffs(hits) - 1);
        n_common += __popc(hits);
        while (hits) {                                 // ordered fold: every lane adds the same terms in ascending word order
            const int src = __ffs(hits) - 1;
            sum += __shfl_sync(0xffffffffu, term, src);
            hits &= hits - 1;
        }
    }
    if (lane == 0) { common[k] = n_common; first[k] = first_q; score[k] = (float)(-sum / 2.0); }
}

namespace {

struct BowSideArgs { int n; const uint8_t* desc; const float* angle; const uint8_t* has_mp; int nodes; const int32_t* node_id; const int32_t* node_off; const int32_t* node_feat; };

// match2[j2] = feature of side 1 matched to feature j2 of side 2 (-1 none); side 1 is walked in feature-vector order like the reference's outer loop
int bow_search_impl(pslam_ctx* c, const BowSideArgs& A, const BowSideArgs& Bs, int th_low, float nnratio, int check_orientation, int32_t* match2) {
    const int nkf = A.n, nf = Bs.n, kf_nodes = A.nodes, f_nodes = Bs.nodes;
    if (nkf < 0 || nf < 0 || kf_nodes < 0 || f_nodes < 0 || (nf && !match2) || (nkf && (!A.desc || !A.angle || !A.has_mp)) || (nf && (!Bs.desc || !Bs.angle)) ||
        (kf_nodes && (!A.node_id || !A.node_off || !A.node_feat)) || (f_nodes && (!Bs.node_id || !Bs.node_off || !Bs.node_feat)))
        return set_error(c, PSLAM_E_INVALID, "bad SearchByBoW arrays");
    for (int i = 0; i < nf; ++i) match2[i] = -1;
    // merge-join of the two (ascending) node-id lists, like the reference's two map iterators
    std::vector<int2> pairs;
    for (int a = 0, b = 0; a < kf_nodes && b < f_nodes;) {
        if (A.node_id[a] == Bs.node_id[b]) { pairs.push_back(make_int2(a, b)); ++a; ++b; }
        else if (A.node_id[a] < Bs.node_id[b]) a = (int)(std::lower_bound(A.node_id, A.node_id + kf_nodes, Bs.node_id[b]) - A.node_id);
        else b = (int)(std::lower_bound(Bs.node_id, Bs.node_id + f_nodes, A.node_id[a]) - Bs.node_id);
    }
    if (pairs.empty() || nf == 0 || nkf == 0) return 0;
    const int nkfeat = A.node_off[kf_nodes], nffeat = Bs.node_off[f_nodes];
    for (int i = 0; i < nkfeat; ++i) if (A.node_feat[i] < 0 || A.node_feat[i] >= nkf) return set_error(c, PSLAM_E_INVALID, "key-frame feature index out of range");
    for (int i = 0; i < nffeat; ++i) if (Bs.node_feat[i] < 0 || Bs.node_feat[i] >= nf) return set_error(c, PSLAM_E_INVALID, "frame feature index out of range");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    const size_t sz[] = {pairs.size() * 8, (size_t)nkf * 32, (size_t)nkf * 4, (size_t)nkf, (size_t)(kf_nodes + 1) * 4, (size_t)nkfeat * 4, (size_t)nf * 32,
                         (size_t)nf * 4, (size_t)(f_nodes + 1) * 4, (size_t)nffeat * 4, (size_t)nf * 4, Bs.has_mp ? (size_t)nf : 0, (size_t)nf, 31 * 4};
    const void* src[] = {pairs.data(), A.desc, A.angle, A.has_mp, A.node_off, A.node_feat, Bs.desc, Bs.angle, Bs.node_off, Bs.node_feat, match2, Bs.has_mp, nullptr, nullptr};
    size_t off[15]; off[0] = 0;
    for (int i = 0; i < 14; ++i) off[i + 1] = (off[i] + sz[i] + 15) & ~(size_t)15;
    uint8_t* d = nullptr;
    PSLAM_CUDA(c, cudaMalloc((void**)&d, off[14]));
    cudaError_t e = cudaMemsetAsync(d + off[13], 0, 31 * 4, st);
    for (int i = 0; i < 12 && e == cudaSuccess; ++i) if (sz[i]) e = cudaMemcpyAsync(d + off[i], src[i], sz[i], cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { cudaFree(d); return check_cuda(c, e, "SearchByBoW upload"); }
    int32_t* d_hist = (int32_t*)(d + off[13]);
    PSLAM_LAUNCH(c, "bow_nodes", k_bow_nodes<<<((int)pairs.size() + 3) / 4, 128, 0, st>>>((int)pairs.size(), (const int2*)(d + off[0]), d + off[1], (const float*)(d + off[2]),
                 d + off[3], (const int32_t*)(d + off[4]), (const int32_t*)(d + off[5]), d + off[6], (const float*)(d + off[7]), (const int32_t*)(d + off[8]),
                 (const int32_t*)(d + off[9]), Bs.has_mp ? d + off[11] : nullptr, th_low, nnratio, check_orientation, (int32_t*)(d + off[10]), (int8_t*)(d + off[12]),
                 d_hist, d_hist + 30));
    if (check_orientation)
        PSLAM_LAUNCH(c, "bow_orientation", k_bow_orientation<<<1, 256, 0, st>>>(nf, (int32_t*)(d + off[10]), (const int8_t*)(d + off[12]), d_hist, d_hist + 30));
    int32_t n = 0;
    e = cudaMemcpyAsync(match2, d + off[10], (size_t)nf * 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&n, d_hist + 30, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d);
    if (e != cudaSuccess) return check_cuda(c, e, "SearchByBoW");
    return n;
}

// shared words + L1 scores of every database key frame against one query BowVector, downloaded into the buffers' host vectors
int bowdb_score(pslam_ctx* c, int n_q, const int32_t* q_word, const double* q_val) {
    if (!c->bowdb || !c->bowdb->n_kf) return set_error(c, PSLAM_E_INVALID, "no key-frame database (pslam_bow_database_set)");
    if (n_q < 0 || (n_q && (!q_word || !q_val))) return set_error(c, PSLAM_E_INVALID, "bad query BowVector");
    for (int i = 1; i < n_q; ++i) if (q_word[i] <= q_word[i - 1]) return set_error(c, PSLAM_E_INVALID, "query words must be strictly ascending (std::map order)");
    BowDbBuffers& B = *c->bowdb;
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    if (n_q > B.q_cap) {
        cudaFree(B.d_qword); cudaFree(B.d_qval); B.d_qword = nullptr; B.d_qval = nullptr; B.q_cap = 0;
        const int cap = std::max(n_q * 3 / 2, 1024);
        PSLAM_CUDA(c, cudaMalloc((void**)&B.d_qword, (size_t)cap * 4));
        PSLAM_CUDA(c, cudaMalloc((void**)&B.d_qval, (size_t)cap * 8));
        B.q_cap = cap;
    }
    if (n_q) {
        PSLAM_CUDA(c, cudaMemcpyAsync(B.d_qword, q_word, (size_t)n_q * 4, cudaMemcpyHostToDevice, st));
        PSLAM_CUDA(c, cudaMemcpyAsync(B.d_qval, q_val, (size_t)n_q * 8, cudaMemcpyHostToDevice, st));
    }
    PSLAM_LAUNCH(c, "bow_db_scores", k_bow_db_scores<<<(B.n_kf + 3) / 4, 128, 0, st>>>(B.n_kf, B.d_off, B.d_word, B.d_val, n_q, B.d_qword, B.d_qval, B.d_common, B.d_first,
                                                                                      B.d_score));
    PSLAM_CUDA(c, cudaGetLastError());
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_common.data(), B.d_common, (size_t)B.n_kf * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_first.data(), B.d_first, (size_t)B.n_kf * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaMemcpyAsync(B.h_score.data(), B.d_score, (size_t)B.n_kf * 4, cudaMemcpyDeviceToHost, st));
    PSLAM_CUDA(c, cudaStreamSynchronize(st));
    return PSLAM_OK;
}

}  // namespace
}  // namespace pslam

using namespace pslam;

extern "C" int pslam_search_by_bow(pslam_ctx* c, int nkf, const uint8_t* kf_desc, const float* kf_angle, const uint8_t* kf_has_mp, int kf_nodes,
                                   const int32_t* kf_node_id, const int32_t* kf_node_off, const int32_t* kf_node_feat, int nf, const uint8_t* f_desc,
                                   const float* f_angle, int f_nodes, const int32_t* f_node_id, const int32_t* f_node_off, const int32_t* f_node_feat,
                                   float nnratio, int check_orientation, int32_t* match) {
    if (!c) return PSLAM_E_INVALID;
    const BowSideArgs A{nkf, kf_desc, kf_angle, kf_has_mp, kf_nodes, kf_node_id, kf_node_off, kf_node_feat};
    const BowSideArgs B{nf, f_desc, f_angle, nullptr, f_nodes, f_node_id, f_node_off, f_node_feat};
    return bow_search_impl(c, A, B, 50, nnratio, check_orientation, match);          // bestDist1 <= TH_LOW (src/ORBmatcher.cc:236)
}

extern "C" int pslam_search_by_bow_kf(pslam_ctx* c, int n1, const uint8_t* desc1, const float* angle1, const uint8_t* has_mp1, int nodes1, const int32_t* node_id1,
                                      const int32_t* node_off1, const int32_t* node_feat1, int n2, const uint8_t* desc2, const float* angle2, const uint8_t* has_mp2,
                                      int nodes2, const int32_t* node_id2, const int32_t* node_off2, const int32_t* node_feat2, float nnratio, int check_orientation,
                                      int32_t* match12) {
    if (!c) return PSLAM_E_INVALID;
    if (n1 < 0 || n2 < 0 || (n1 && !match12) || (n2 && !has_mp2)) return set_error(c, PSLAM_E_INVALID, "bad SearchByBoW(KeyFrame, KeyFrame) arrays");
    const BowSideArgs A{n1, desc1, angle1, has_mp1, nodes1, node_id1, node_off1, node_feat1};
    const BowSideArgs B{n2, desc2, angle2, has_mp2, nodes2, node_id2, node_off2, node_feat2};
    std::vector<int32_t> match2((size_t)std::max(n2, 1), -1);
    const int n = bow_search_impl(c, A, B, 49, nnratio, check_orientation, match2.data());     // bestDist1 < TH_LOW (src/ORBmatcher.cc:598)
    for (int i = 0; i < n1; ++i) match12[i] = -1;
    if (n < 0) return n;
    for (int j = 0; j < n2; ++j) if (match2[j] >= 0) match12[match2[j]] = j;                   // vpMatches12[idx1] = vpMapPoints2[bestIdx2]
    return n;
}

extern "C" int pslam_bow_database_set(pslam_ctx* c, int n_kf, const int32_t* kf_off, const int32_t* kf_word, const double* kf_val) {
    if (!c) return PSLAM_E_INVALID;
    if (n_kf < 0 || (n_kf && (!kf_off || kf_off[0] != 0))) return set_error(c, PSLAM_E_INVALID, "bad key-frame database offsets");
    for (int k = 0; k < n_kf; ++k) {
        if (kf_off[k + 1] < kf_off[k]) return set_error(c, PSLAM_E_INVALID, "key-frame database offsets must not decrease");
        for (int i = kf_off[k] + 1; i < kf_off[k + 1]; ++i)
            if (kf_word[i] <= kf_word[i - 1]) return set_error(c, PSLAM_E_INVALID, "BowVector words must be strictly ascending (std::map order)");
    }
    bowdb_free(c);
    if (n_kf == 0) return PSLAM_OK;
    const int total = kf_off[n_kf];
    if (total && (!kf_word || !kf_val)) return set_error(c, PSLAM_E_INVALID, "bad key-frame database arrays");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    c->bowdb = new BowDbBuffers();
    BowDbBuffers& B = *c->bowdb;
    B.n_kf = n_kf; B.total = total;
    cudaError_t e = cudaMalloc((void**)&B.d_off, (size_t)(n_kf + 1) * 4);
    if (e == cudaSuccess) e = cudaMalloc((void**)&B.d_word, (size_t)std::max(total, 1) * 4);
    if (e == cudaSuccess) e = cudaMalloc((void**)&B.d_val, (size_t)std::max(total, 1) * 8);
    if (e == cudaSuccess) e = cudaMalloc((void**)&B.d_common, (size_t)n_kf * 4);
    if (e == cudaSuccess) e = cudaMalloc((void**)&B.d_first, (size_t)n_kf * 4);
    if (e == cudaSuccess) e = cudaMalloc((void**)&B.d_score, (size_t)n_kf * 4);
    if (e == cudaSuccess) e = cudaMemcpyAsync(B.d_off, kf_off, (size_t)(n_kf + 1) * 4, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess && total) e = cudaMemcpyAsync(B.d_word, kf_word, (size_t)total * 4, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess && total) e = cudaMemcpyAsync(B.d_val, kf_val, (size_t)total * 8, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { bowdb_free(c); return check_cuda(c, e, "key-frame database upload"); }
    B.h_common.resize(n_kf); B.h_first.resize(n_kf); B.h_score.resize(n_kf);
    return PSLAM_OK;
}

extern "C" int pslam_detect_loop_candidates(pslam_ctx* c, int n_q, const int32_t* q_word, const double* q_val, const int32_t* covis, int covis_stride,
                                            const uint8_t* connected, float min_score, int32_t* candidates, int32_t* common_words, float* score) {
    if (!c) return PSLAM_E_INVALID;
    if (!candidates) return set_error(c, PSLAM_E_INVALID, "candidates is NULL");
    int rc = bowdb_score(c, n_q, q_word, q_val);
    if (rc != PSLAM_OK) return rc;
    const BowDbBuffers& B = *c->bowdb;
    if (!bowdb_covis_ok(B.n_kf, covis, covis_stride)) return set_error(c, PSLAM_E_INVALID, "bad covisibility table");
    return bowdb_select_loop(B.n_kf, B.h_common.data(), B.h_first.data(), B.h_score.data(), covis, covis_stride, connected, min_score, candidates, common_words, score);
}

extern "C" int pslam_detect_relocalization_candidates(pslam_ctx* c, int n_q, const int32_t* q_word, const double* q_val, const int32_t* covis, int covis_stride,
                                                      float* reloc_score_io, int32_t* candidates, int32_t* common_words) {
    if (!c) return PSLAM_E_INVALID;
    if (!candidates || !reloc_score_io) return set_error(c, PSLAM_E_INVALID, "candidates / reloc_score_io is NULL");
    int rc = bowdb_score(c, n_q, q_word, q_val);
    if (rc != PSLAM_OK) return rc;
    const BowDbBuffers& B = *c->bowdb;
    if (!bowdb_covis_ok(B.n_kf, covis, covis_stride)) return set_error(c, PSLAM_E_INVALID, "bad covisibility table");
    return bowdb_select_reloc(B.n_kf, B.h_common.data(), B.h_first.data(), B.h_score.data(), covis, covis_stride, reloc_score_io, candidates, common_words);
}
