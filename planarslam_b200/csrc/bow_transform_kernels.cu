// DBoW2 vocabulary transform on sm_90a: TemplatedVocabulary<FORB::TDescriptor, FORB>::transform(features, BowVector&, FeatureVector&,
// levelsup) (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1125-1193, per-feature descent :1213-1252) as Frame::ComputeBoW /
// KeyFrame::ComputeBoW use it (TF_IDF weights, L1 normalisation, levelsup = 4).
//   k_bow_descend   one warp per feature: at every level the lanes take one child each (k <= 32), 256-bit Hamming distance, warp
//                   arg-min with "first minimum wins"; L2-resident gather of k x 32 bytes per level
//   k_bow_assemble  one CTA per feature set: stable rank of the features by word id and by node id (std::map order, insertion
//                   order inside a node), word weights accumulated by repeated addition in feature order (BowVector::addWeight),
//                   L1 norm summed in word order by one thread (BowVector::normalize)
// Batched transform against the vocabulary kept resident by pslam_bow_set_vocabulary:
//   k_bow_descend_batch   the features of all frames in one launch; G = 16 or 32 lanes per feature (the vocabulary's largest branching
//                         factor rounded up), lane j scores child j.  The children of a node are stored contiguously (child-CSR order), so a
//                         level costs one coalesced k x 32-byte load plus one 16-byte record of the chosen child
//   k_bow_assemble_batch  one CTA per frame: bitonic sort of the (word, feature) and (node, feature) keys in shared memory (unique keys, so the
//                         order is the stable one), one thread per word run adds the weights in feature order, the L1 norm stays one
//                         in-order sum, the FeatureVector comes from the run heads and an exclusive scan
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "pslam_internal.h"

namespace pslam {

__global__ void __launch_bounds__(128) k_bow_descend(int n, int L, int levelsup, const uint8_t* __restrict__ vdesc, const int32_t* __restrict__ child_off,
                                                     const int32_t* __restrict__ child_id, const int32_t* __restrict__ vword, const double* __restrict__ vweight,
                                                     const uint8_t* __restrict__ feats, int32_t* __restrict__ f_word, int32_t* __restrict__ f_node,
                                                     double* __restrict__ f_weight) {
    const int lane = threadIdx.x & 31, i = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (i >= n) return;
    uint32_t f[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) f[q] = reinterpret_cast<const uint32_t*>(feats)[8 * i + q];
    const int nid_level = L - levelsup;
    int nid = 0, cur = 0, level = 0;
    while (true) {
        ++level;
        const int c0 = child_off[cur], nc = child_off[cur + 1] - c0;
        uint32_t best = 0xffffffffu;                            // (distance << 8 | child position): the first minimum wins
        for (int c = lane; c < nc; c += 32) {
            const int id = child_id[c0 + c];
            int d = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) d += __popc(f[q] ^ reinterpret_cast<const uint32_t*>(vdesc)[8 * id + q]);
            best = min(best, ((uint32_t)d << 8) | (uint32_t)c);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
        cur = child_id[c0 + (best & 0xff)];
        if (level == nid_level) nid = cur;
        if (child_off[cur + 1] == child_off[cur]) break;        // leaf
    }
    if (lane == 0) { f_word[i] = vword[cur]; f_node[i] = nid; f_weight[i] = vweight[cur]; }
}

// n <= BOW_MAX_FEATURES features of one frame
#define BOW_MAX_FEATURES 3072
__global__ void __launch_bounds__(256) k_bow_assemble(int n, const int32_t* __restrict__ f_word, const int32_t* __restrict__ f_node, const double* __restrict__ f_weight,
                                                      int32_t* __restrict__ word_id, double* __restrict__ word_val, int32_t* __restrict__ node_id,
                                                      int32_t* __restrict__ node_off, int32_t* __restrict__ node_feat, int32_t* __restrict__ counts) {
    __shared__ int32_t s_word[BOW_MAX_FEATURES], s_node[BOW_MAX_FEATURES];
    __shared__ int16_t s_byword[BOW_MAX_FEATURES], s_bynode[BOW_MAX_FEATURES];       // feature index at each sorted position
    __shared__ int s_nw, s_nn;
    const int tid = threadIdx.x;
    for (int i = tid; i < n; i += 256) { const bool keep = f_weight[i] > 0; s_word[i] = keep ? f_word[i] : 0x7fffffff; s_node[i] = keep ? f_node[i] : 0x7fffffff; }
    __syncthreads();
    // stable ranks (features with weight 0 - "stopped" words - sort to the end and are dropped)
    for (int i = tid; i < n; i += 256) {
        const int wi = s_word[i], ni = s_node[i];
        int rw = 0, rn = 0;
        for (int j = 0; j < n; ++j) {
            const int wj = s_word[j], nj = s_node[j];
            rw += (wj < wi) || (wj == wi && j < i);
            rn += (nj < ni) || (nj == ni && j < i);
        }
        s_byword[rw] = (int16_t)i; s_bynode[rn] = (int16_t)i;
    }
    __syncthreads();
    if (tid == 0) {
        // BowVector: one entry per distinct word; value = w added once per feature of the word, in feature order
        int nw = 0;
        double norm = 0.0;
        for (int p = 0; p < n;) {
            const int i0 = s_byword[p], w = s_word[i0];
            if (w == 0x7fffffff) break;
            const double wt = f_weight[i0];
            double acc = wt;
            int q = p + 1;
            while (q < n && s_word[s_byword[q]] == w) { acc += wt; ++q; }
            word_id[nw] = w; word_val[nw] = acc;
            norm += fabs(acc);
            ++nw; p = q;
        }
        if (norm > 0.0) for (int k = 0; k < nw; ++k) word_val[k] /= norm;
        s_nw = nw;
    } else if (tid == 32) {
        // FeatureVector: nodes ascending, features of a node in insertion (= feature) order
        int nn = 0, nf = 0;
        for (int p = 0; p < n; ++p) {
            const int i = s_bynode[p], nd = s_node[i];
            if (nd == 0x7fffffff) break;
            if (nn == 0 || node_id[nn - 1] != nd) { node_id[nn] = nd; node_off[nn] = nf; ++nn; }
            node_feat[nf++] = i;
        }
        node_off[nn] = nf;
        s_nn = nn;
    }
    __syncthreads();
    if (tid == 0) { counts[0] = s_nw; counts[1] = s_nn; }
}

// The vocabulary kept in HBM, in child-slot order (slot c = position c of the flat child_id array): the children of a node are adjacent
struct BowVocBuffers {
    int n_nodes = 0, L = 0, max_k = 0, root_c0 = 0, root_nc = 0;
    DevArray<uint8_t> d_cdesc;      // [n_child][32] descriptor of the node in slot c
    DevArray<int4> d_cinfo;         // {first child slot, number of children, node id, word id} of the node in slot c
    DevArray<double> d_cweight;     // weight of the node in slot c
    // scratch of the batch calls (only grows)
    DevArray<uint8_t> d_feat;       // per feature: word, node, weight
    DevArray<uint8_t> d_stage;      // host-pointer entry point: inputs and outputs
};

static void bowvoc_release_vocabulary(BowVocBuffers& V) {
    V.d_cdesc.release(); V.d_cinfo.release(); V.d_cweight.release();
    V.n_nodes = V.L = V.max_k = V.root_c0 = V.root_nc = 0;
}

void bowvoc_free(pslam_ctx* c) {
    delete c->bowvoc;
    c->bowvoc = nullptr;
}

// G lanes per feature (G >= the largest branching factor); rows >= n[f] take part in the warp's shuffles but load nothing.  The loop runs while any
// feature of the warp is still descending, so the full-warp shuffles stay convergent when leaves sit at different depths.
template <int G>
__global__ void __launch_bounds__(256) k_bow_descend_batch(long long total, int cap, const int32_t* __restrict__ nrows, int nid_level, int root_c0, int root_nc,
                                                           const uint8_t* __restrict__ cdesc, const int4* __restrict__ cinfo, const double* __restrict__ cweight,
                                                           const uint8_t* __restrict__ feats, int32_t* __restrict__ f_word, int32_t* __restrict__ f_node,
                                                           double* __restrict__ f_weight) {
    const int gl = threadIdx.x & (G - 1);
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / G;        // frame * cap + row
    bool active = false;
    if (i < total) { const int f = (int)(i / cap), r = (int)(i - (long long)f * cap); active = r < min(__ldg(nrows + f), cap); }
    uint4 fa = make_uint4(0, 0, 0, 0), fb = fa;
    if (active) { const uint4* p = reinterpret_cast<const uint4*>(feats + (size_t)i * 32); fa = __ldg(p); fb = __ldg(p + 1); }
    int c0 = root_c0, nc = active ? root_nc : 0, level = 0, nid = 0, slot = 0;
    int4 rec = make_int4(0, 0, 0, -1);
    while (__any_sync(0xffffffffu, nc > 0)) {
        ++level;
        uint32_t key = 0xffffffffu;                             // (distance << 8 | child position): the first minimum wins
        if (gl < nc) {
            const uint4* q = reinterpret_cast<const uint4*>(cdesc + (size_t)(c0 + gl) * 32);
            const uint4 a = __ldg(q), b = __ldg(q + 1);
            const int d = __popc(fa.x ^ a.x) + __popc(fa.y ^ a.y) + __popc(fa.z ^ a.z) + __popc(fa.w ^ a.w) + __popc(fb.x ^ b.x) + __popc(fb.y ^ b.y) +
                          __popc(fb.z ^ b.z) + __popc(fb.w ^ b.w);
            key = ((uint32_t)d << 8) | (uint32_t)gl;
        }
#pragma unroll
        for (int o = G / 2; o; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
        if (nc > 0) {
            slot = c0 + (int)(key & 0xff);
            rec = __ldg(cinfo + slot);
            if (level == nid_level) nid = rec.z;
            c0 = rec.x; nc = rec.y;
        }
    }
    if (active && gl == 0) { f_word[i] = rec.w; f_node[i] = nid; f_weight[i] = __ldg(cweight + slot); }
}

#define BOW_SORT_CAP 4096                                       // power of two >= BOW_MAX_FEATURES
#define BOW_ASM_THREADS 512

// ascending bitonic sort of s[0, P), P a power of two
__device__ void bow_bitonic_sort(unsigned long long* s, int P) {
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < P / 2; t += BOW_ASM_THREADS) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), l = i + j;
                const unsigned long long a = s[i], b = s[l];
                if ((a > b) == ((i & k) == 0)) { s[i] = b; s[l] = a; }
            }
            __syncthreads();
        }
}

// positions of the run heads of the sorted keys s[0, m) (a head starts a run of equal upper halves) in s_run[0, runs), s_run[runs] = m; returns runs
__device__ int bow_run_heads(const unsigned long long* s, int m, int32_t* s_run, int32_t* s_warp) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int E = (m + BOW_ASM_THREADS - 1) / BOW_ASM_THREADS, b = min(tid * E, m), e = min(b + E, m);
    auto head = [&](int p) { return p == 0 || (s[p] >> 32) != (s[p - 1] >> 32); };
    int cnt = 0;
    for (int p = b; p < e; ++p) cnt += head(p);
    int x = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < BOW_ASM_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
        if (lane < BOW_ASM_THREADS / 32) s_warp[lane] = w;
    }
    __syncthreads();
    int run = x - cnt + (warp ? s_warp[warp - 1] : 0);
    for (int p = b; p < e; ++p) if (head(p)) s_run[run++] = p;
    const int runs = s_warp[BOW_ASM_THREADS / 32 - 1];
    if (tid == 0) s_run[runs] = m;
    __syncthreads();
    return runs;
}

// order-preserving unsigned key of a signed id in the upper half, feature index in the lower half; dropped features sort last
__device__ __forceinline__ unsigned long long bow_key(int32_t id, int p) { return ((unsigned long long)((uint32_t)id ^ 0x80000000u) << 32) | (uint32_t)p; }

__global__ void __launch_bounds__(BOW_ASM_THREADS) k_bow_assemble_batch(int cap, const int32_t* __restrict__ nrows, const int32_t* __restrict__ f_word,
                                                                        const int32_t* __restrict__ f_node, const double* __restrict__ f_weight,
                                                                        int32_t* __restrict__ word_id, double* __restrict__ word_val, int32_t* __restrict__ node_id,
                                                                        int32_t* __restrict__ node_off, int32_t* __restrict__ node_feat, int32_t* __restrict__ counts) {
    __shared__ unsigned long long s_key[BOW_SORT_CAP];
    __shared__ int32_t s_run[BOW_MAX_FEATURES + 1];
    __shared__ int32_t s_warp[BOW_ASM_THREADS / 32];
    __shared__ int s_kept;
    __shared__ double s_norm;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int n = max(0, min(nrows[f], cap));
    const size_t fb = (size_t)f * cap;
    f_word += fb; f_node += fb; f_weight += fb; word_id += fb; word_val += fb; node_id += fb; node_feat += fb;
    node_off += (size_t)f * (cap + 1);
    int P = 1;
    while (P < n) P <<= 1;
    if (tid == 0) s_kept = 0;
    __syncthreads();
    int kept = 0;
    for (int p = tid; p < P; p += BOW_ASM_THREADS) {
        const bool keep = p < n && f_weight[p] > 0;                   // weight 0: a stopped word, dropped from both vectors
        s_key[p] = keep ? bow_key(f_word[p], p) : ~0ull;
        kept += keep;
    }
    if (kept) atomicAdd(&s_kept, kept);
    __syncthreads();
    const int nk = s_kept;
    bow_bitonic_sort(s_key, P);
    // BowVector: one thread per word run, value = the weights of the run's features added in feature order (BowVector::addWeight)
    const int nw = bow_run_heads(s_key, nk, s_run, s_warp);
    for (int r = tid; r < nw; r += BOW_ASM_THREADS) {
        const int p0 = s_run[r], p1 = s_run[r + 1];
        double acc = f_weight[(uint32_t)s_key[p0]];
        for (int q = p0 + 1; q < p1; ++q) acc += f_weight[(uint32_t)s_key[q]];
        word_id[r] = (int32_t)((uint32_t)(s_key[p0] >> 32) ^ 0x80000000u);
        word_val[r] = acc;
    }
    __syncthreads();
    if (tid == 0) {                                                    // BowVector::normalize(L1): one sum in ascending word order
        double norm = 0.0;
        for (int r = 0; r < nw; ++r) norm += fabs(word_val[r]);
        s_norm = norm;
    }
    for (int p = tid; p < P; p += BOW_ASM_THREADS) {
        const bool keep = p < n && f_weight[p] > 0;
        s_key[p] = keep ? bow_key(f_node[p], p) : ~0ull;
    }
    __syncthreads();
    const double norm = s_norm;
    if (norm > 0.0) for (int r = tid; r < nw; r += BOW_ASM_THREADS) word_val[r] /= norm;
    // FeatureVector: nodes ascending, the features of a node in insertion (= feature) order
    bow_bitonic_sort(s_key, P);
    const int nn = bow_run_heads(s_key, nk, s_run, s_warp);
    for (int p = tid; p < nk; p += BOW_ASM_THREADS) node_feat[p] = (int32_t)(uint32_t)s_key[p];
    for (int r = tid; r <= nn; r += BOW_ASM_THREADS) {
        node_off[r] = s_run[r];
        if (r < nn) node_id[r] = (int32_t)((uint32_t)(s_key[s_run[r]] >> 32) ^ 0x80000000u);
    }
    if (tid == 0) { counts[2 * f] = nw; counts[2 * f + 1] = nn; }
}

namespace {

int bow_batch_check(pslam_ctx* c, int cap, int nframes) {
    if (!c->bowvoc || !c->bowvoc->n_nodes) return set_error(c, PSLAM_E_INVALID, "no resident vocabulary (pslam_bow_set_vocabulary)");
    if (nframes < 0 || cap < 1 || cap > BOW_MAX_FEATURES) return set_error(c, PSLAM_E_INVALID, "bad batch shape (1 <= cap <= 3072 features per frame)");
    if ((long long)nframes * cap * 32 / 256 > 0x7fffffffLL) return set_error(c, PSLAM_E_INVALID, "batch too large for one launch");
    return PSLAM_OK;
}

// enqueues the two kernels on the context's stream
int bow_batch_run(pslam_ctx* c, const uint8_t* d_desc, const int32_t* d_n, int cap, int nframes, int levelsup, int32_t* d_word_id, double* d_word_val,
                  int32_t* d_node_id, int32_t* d_node_off, int32_t* d_node_feat, int32_t* d_counts) {
    BowVocBuffers& V = *c->bowvoc;
    const long long total = (long long)nframes * cap;
    const int rc = V.d_feat.reserve(c, (size_t)total * 16);
    if (rc != PSLAM_OK) return rc;
    int32_t* f_word = reinterpret_cast<int32_t*>(V.d_feat.ptr);
    int32_t* f_node = f_word + total;
    double* f_weight = (double*)(f_node + total);
    cudaStream_t st = c->stream;
    const int nid_level = V.L - levelsup;
    if (V.max_k <= 16)
        PSLAM_LAUNCH(c, "bow_descend_batch", k_bow_descend_batch<16><<<(unsigned)((total * 16 + 255) / 256), 256, 0, st>>>(total, cap, d_n, nid_level, V.root_c0,
                     V.root_nc, V.d_cdesc, V.d_cinfo, V.d_cweight, d_desc, f_word, f_node, f_weight));
    else
        PSLAM_LAUNCH(c, "bow_descend_batch", k_bow_descend_batch<32><<<(unsigned)((total * 32 + 255) / 256), 256, 0, st>>>(total, cap, d_n, nid_level, V.root_c0,
                     V.root_nc, V.d_cdesc, V.d_cinfo, V.d_cweight, d_desc, f_word, f_node, f_weight));
    PSLAM_LAUNCH(c, "bow_assemble_batch", k_bow_assemble_batch<<<nframes, BOW_ASM_THREADS, 0, st>>>(cap, d_n, f_word, f_node, f_weight, d_word_id, d_word_val,
                 d_node_id, d_node_off, d_node_feat, d_counts));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

}  // namespace

}  // namespace pslam

using namespace pslam;

extern "C" int pslam_bow_transform(pslam_ctx* c, int n_nodes, int L, const uint8_t* voc_desc, const int32_t* child_off, const int32_t* child_id,
                                   const int32_t* voc_word_id, const double* voc_weight, const uint8_t* features, int n, int levelsup, int32_t* word_id,
                                   double* word_val, int32_t* node_id, int32_t* node_off, int32_t* node_feat, int32_t* counts) {
    if (!c) return PSLAM_E_INVALID;
    if (n_nodes < 1 || L < 1 || n < 0 || n > BOW_MAX_FEATURES || !voc_desc || !child_off || !child_id || !voc_word_id || !voc_weight || !counts ||
        (n && (!features || !word_id || !word_val || !node_id || !node_off || !node_feat)))
        return set_error(c, PSLAM_E_INVALID, "bad vocabulary / feature arrays (at most 3072 features per call)");
    counts[0] = counts[1] = 0;
    if (n == 0) return PSLAM_OK;
    if (child_off[1] - child_off[0] < 1) return set_error(c, PSLAM_E_INVALID, "the root has no children");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->stream;
    const int n_child = child_off[n_nodes];
    // a caller that transforms many frames keeps the vocabulary resident; this entry point uploads it per call for simplicity
    Slab s;
    const auto v_desc = s.add<uint8_t>((size_t)n_nodes * 32);
    const auto v_child_off = s.add<int32_t>(n_nodes + 1), v_child_id = s.add<int32_t>(n_child), v_word_id = s.add<int32_t>(n_nodes);
    const auto v_weight = s.add<double>(n_nodes);
    const auto feat = s.add<uint8_t>((size_t)n * 32);
    const auto f_word = s.add<int32_t>(n), f_node = s.add<int32_t>(n);
    const auto f_weight = s.add<double>(n);
    const auto d_word_id = s.add<int32_t>(n);
    const auto d_word_val = s.add<double>(n);
    const auto d_node_id = s.add<int32_t>(n), d_node_off = s.add<int32_t>(n + 1), d_node_feat = s.add<int32_t>(n), d_counts = s.add<int32_t>(2);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    s.up(v_desc, voc_desc, st); s.up(v_child_off, child_off, st); s.up(v_child_id, child_id, st); s.up(v_word_id, voc_word_id, st); s.up(v_weight, voc_weight, st);
    s.up(feat, features, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    PSLAM_LAUNCH(c, "bow_descend", k_bow_descend<<<(n + 3) / 4, 128, 0, st>>>(n, L, levelsup, s[v_desc], s[v_child_off], s[v_child_id], s[v_word_id], s[v_weight], s[feat],
                 s[f_word], s[f_node], s[f_weight]));
    PSLAM_LAUNCH(c, "bow_assemble", k_bow_assemble<<<1, 256, 0, st>>>(n, s[f_word], s[f_node], s[f_weight], s[d_word_id], s[d_word_val], s[d_node_id], s[d_node_off],
                 s[d_node_feat], s[d_counts]));
    int32_t cnt[2] = {0, 0};
    s.down(cnt, d_counts, st);
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    if (cnt[0] > 0) {
        s.down(word_id, d_word_id, st, cnt[0]); s.down(word_val, d_word_val, st, cnt[0]); s.down(node_id, d_node_id, st, cnt[1]);
        s.down(node_off, d_node_off, st, cnt[1] + 1); s.down(node_feat, d_node_feat, st);
        if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    }
    counts[0] = cnt[0]; counts[1] = cnt[1];
    return PSLAM_OK;
}

extern "C" int pslam_bow_set_vocabulary(pslam_ctx* c, int n_nodes, int L, const uint8_t* voc_desc, const int32_t* child_off, const int32_t* child_id,
                                        const int32_t* voc_word_id, const double* voc_weight) {
    if (!c) return PSLAM_E_INVALID;
    if (n_nodes == 0) { bowvoc_free(c); return PSLAM_OK; }
    if (n_nodes < 1 || L < 1 || !voc_desc || !child_off || !child_id || !voc_word_id || !voc_weight)
        return set_error(c, PSLAM_E_INVALID, "bad vocabulary arrays");
    if (child_off[0] != 0) return set_error(c, PSLAM_E_INVALID, "child_off[0] must be 0");
    int max_k = 0;
    for (int p = 0; p < n_nodes; ++p) {
        const int nc = child_off[p + 1] - child_off[p];
        if (nc < 0) return set_error(c, PSLAM_E_INVALID, "child offsets must not decrease");
        if (nc > 32) return set_error(c, PSLAM_E_INVALID, "a vocabulary node has more than 32 children");
        max_k = std::max(max_k, nc);
        for (int q = child_off[p]; q < child_off[p + 1]; ++q)                // ids grow along every path, so a descent ends
            if (child_id[q] <= p || child_id[q] >= n_nodes) return set_error(c, PSLAM_E_INVALID, "a child id must lie in (parent id, n_nodes)");
    }
    if (child_off[1] < 1) return set_error(c, PSLAM_E_INVALID, "the root has no children");
    const int n_child = child_off[n_nodes];
    std::vector<uint8_t> cdesc((size_t)n_child * 32);
    std::vector<int4> cinfo(n_child);
    std::vector<double> cweight(n_child);
    for (int s = 0; s < n_child; ++s) {
        const int id = child_id[s];
        std::copy(voc_desc + (size_t)id * 32, voc_desc + (size_t)id * 32 + 32, cdesc.begin() + (size_t)s * 32);
        cinfo[s] = make_int4(child_off[id], child_off[id + 1] - child_off[id], id, voc_word_id[id]);
        cweight[s] = voc_weight[id];
    }
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    if (!c->bowvoc) c->bowvoc = new BowVocBuffers();
    BowVocBuffers& V = *c->bowvoc;
    bowvoc_release_vocabulary(V);
    int rc;
    if ((rc = V.d_cdesc.reserve(c, cdesc.size())) || (rc = V.d_cinfo.reserve(c, cinfo.size())) || (rc = V.d_cweight.reserve(c, cweight.size()))) {
        bowvoc_release_vocabulary(V);
        return rc;
    }
    cudaError_t e = cudaMemcpyAsync(V.d_cdesc, cdesc.data(), cdesc.size(), cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(V.d_cinfo, cinfo.data(), cinfo.size() * sizeof(int4), cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(V.d_cweight, cweight.data(), cweight.size() * 8, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { bowvoc_release_vocabulary(V); return check_cuda(c, e, "vocabulary upload"); }
    V.n_nodes = n_nodes; V.L = L; V.max_k = max_k; V.root_c0 = child_off[0]; V.root_nc = child_off[1] - child_off[0];
    return PSLAM_OK;
}

extern "C" int pslam_bow_transform_batch_dev(pslam_ctx* c, const uint8_t* d_desc, const int32_t* d_n, int cap, int nframes, int levelsup, int32_t* d_word_id,
                                             double* d_word_val, int32_t* d_node_id, int32_t* d_node_off, int32_t* d_node_feat, int32_t* d_counts) {
    if (!c) return PSLAM_E_INVALID;
    int rc = bow_batch_check(c, cap, nframes);
    if (rc != PSLAM_OK) return rc;
    if (nframes == 0) return PSLAM_OK;
    if (!d_desc || !d_n || !d_word_id || !d_word_val || !d_node_id || !d_node_off || !d_node_feat || !d_counts || ((uintptr_t)d_desc & 15))
        return set_error(c, PSLAM_E_INVALID, "bad device arrays (descriptors 16-byte aligned)");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    return bow_batch_run(c, d_desc, d_n, cap, nframes, levelsup, d_word_id, d_word_val, d_node_id, d_node_off, d_node_feat, d_counts);
}

extern "C" int pslam_bow_transform_batch(pslam_ctx* c, const uint8_t* desc, const int32_t* n, int cap, int nframes, int levelsup, int32_t* word_id,
                                         double* word_val, int32_t* node_id, int32_t* node_off, int32_t* node_feat, int32_t* counts) {
    if (!c) return PSLAM_E_INVALID;
    int rc = bow_batch_check(c, cap, nframes);
    if (rc != PSLAM_OK) return rc;
    if (nframes == 0) return PSLAM_OK;
    if (!desc || !n || !word_id || !word_val || !node_id || !node_off || !node_feat || !counts) return set_error(c, PSLAM_E_INVALID, "bad host arrays");
    for (int f = 0; f < nframes; ++f)
        if (n[f] < 0 || n[f] > cap) return set_error(c, PSLAM_E_INVALID, "n[f] must lie in [0, cap] (at most 3072 features per frame)");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const size_t nf = (size_t)nframes * cap;
    Slab s;
    const auto d_desc = s.add<uint8_t>(nf * 32);
    const auto d_n = s.add<int32_t>(nframes), d_word_id = s.add<int32_t>(nf);
    const auto d_word_val = s.add<double>(nf);
    const auto d_node_id = s.add<int32_t>(nf), d_node_off = s.add<int32_t>((size_t)nframes * (cap + 1)), d_node_feat = s.add<int32_t>(nf);
    const auto d_counts = s.add<int32_t>((size_t)nframes * 2);
    if ((rc = s.alloc(c, c->bowvoc->d_stage)) != PSLAM_OK) return rc;
    cudaStream_t st = c->stream;
    s.up(d_desc, desc, st); s.up(d_n, n, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    rc = bow_batch_run(c, s[d_desc], s[d_n], cap, nframes, levelsup, s[d_word_id], s[d_word_val], s[d_node_id], s[d_node_off], s[d_node_feat], s[d_counts]);
    if (rc != PSLAM_OK) return rc;
    s.down(word_id, d_word_id, st); s.down(word_val, d_word_val, st); s.down(node_id, d_node_id, st); s.down(node_off, d_node_off, st);
    s.down(node_feat, d_node_feat, st); s.down(counts, d_counts, st);
    return s.sync(c, st);
}
