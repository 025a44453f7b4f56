// DBoW2 vocabulary transform on sm_90a: TemplatedVocabulary<FORB::TDescriptor, FORB>::transform(features, BowVector&, FeatureVector&,
// levelsup) (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1125-1193, per-feature descent :1213-1252) as Frame::ComputeBoW /
// KeyFrame::ComputeBoW use it (TF_IDF weights, L1 normalisation, levelsup = 4).
//   k_bow_descend   one warp per feature: at every level the lanes take one child each (k <= 32), 256-bit Hamming distance, warp
//                   arg-min with "first minimum wins"; L2-resident gather of k x 32 bytes per level
//   k_bow_assemble  one CTA per feature set: stable rank of the features by word id and by node id (std::map order, insertion
//                   order inside a node), word weights accumulated by repeated addition in feature order (BowVector::addWeight),
//                   L1 norm summed in word order by one thread (BowVector::normalize)
#include <cuda_runtime.h>

#include <cstdint>

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
    const size_t sz[] = {(size_t)n_nodes * 32, (size_t)(n_nodes + 1) * 4, (size_t)n_child * 4, (size_t)n_nodes * 4, (size_t)n_nodes * 8, (size_t)n * 32,
                         (size_t)n * 4, (size_t)n * 4, (size_t)n * 8, (size_t)n * 4, (size_t)n * 8, (size_t)n * 4, (size_t)(n + 1) * 4, (size_t)n * 4, 8};
    const void* src[] = {voc_desc, child_off, child_id, voc_word_id, voc_weight, features};
    size_t off[16]; off[0] = 0;
    for (int i = 0; i < 15; ++i) off[i + 1] = (off[i] + sz[i] + 15) & ~(size_t)15;
    uint8_t* d = nullptr;
    PSLAM_CUDA(c, cudaMalloc((void**)&d, off[15]));
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 6 && e == cudaSuccess; ++i) e = cudaMemcpyAsync(d + off[i], src[i], sz[i], cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { cudaFree(d); return check_cuda(c, e, "bow transform upload"); }
    PSLAM_LAUNCH(c, "bow_descend", k_bow_descend<<<(n + 3) / 4, 128, 0, st>>>(n, L, levelsup, d + off[0], (const int32_t*)(d + off[1]), (const int32_t*)(d + off[2]),
                 (const int32_t*)(d + off[3]), (const double*)(d + off[4]), d + off[5], (int32_t*)(d + off[6]), (int32_t*)(d + off[7]), (double*)(d + off[8])));
    PSLAM_LAUNCH(c, "bow_assemble", k_bow_assemble<<<1, 256, 0, st>>>(n, (const int32_t*)(d + off[6]), (const int32_t*)(d + off[7]), (const double*)(d + off[8]),
                 (int32_t*)(d + off[9]), (double*)(d + off[10]), (int32_t*)(d + off[11]), (int32_t*)(d + off[12]), (int32_t*)(d + off[13]), (int32_t*)(d + off[14])));
    int32_t cnt[2] = {0, 0};
    e = cudaMemcpyAsync(cnt, d + off[14], 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess && cnt[0] > 0) {
        e = cudaMemcpyAsync(word_id, d + off[9], (size_t)cnt[0] * 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(word_val, d + off[10], (size_t)cnt[0] * 8, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(node_id, d + off[11], (size_t)cnt[1] * 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(node_off, d + off[12], (size_t)(cnt[1] + 1) * 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(node_feat, d + off[13], (size_t)n * 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    cudaFree(d);
    if (e != cudaSuccess) return check_cuda(c, e, "bow transform");
    counts[0] = cnt[0]; counts[1] = cnt[1];
    return PSLAM_OK;
}
