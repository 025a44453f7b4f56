// Brute-force Hamming matching of 256-bit descriptors (ORB rBRIEF, LBD) for sm_90a, batched over frames.
//
// Reference semantics: ORBmatcher::DescriptorDistance src/ORBmatcher.cc:1712-1728; ORBmatcher::MatchORBPoints :1332-1394
// (cv::BFMatcher(NORM_HAMMING).match, then keep dist < max(2*min_dist, 15)); LSDmatcher::SearchByDescriptor
// src/LSDmatcher.cpp:242-279 (knnMatch k=2).  cv::BFMatcher semantics (first minimum wins; k-NN = the k smallest in
// (distance, train index) order) are pinned against cv2 by tests/test_oracle_match.py.
//
// One warp per query descriptor; the train set streams through shared memory in tiles of 256 descriptors; each lane
// XOR-popcounts its share (8 x 32-bit words per pair) and keeps its two smallest (distance << 16 | index) keys; a
// warp-shuffle top-2 merge produces the result.  On-chip work: report pairs/s, not an HBM fraction (SURVEY.md §8d).
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <vector>

#include "pslam_internal.h"

namespace pslam {

#define MATCH_TILE 256
#define MATCH_WARPS 8

// Every warp keeps MATCH_NQ query rows in registers: a 32-byte train row read from shared memory serves four distances (the kernel with one query per warp was
// bound by its two 16-byte shared loads per distance).
#define MATCH_NQ 4
__global__ void __launch_bounds__(MATCH_WARPS * 32) k_hamming_knn2(const uint8_t* __restrict__ q, const int32_t* __restrict__ nq, int capq,
                                                                  const uint8_t* __restrict__ t, const int32_t* __restrict__ nt, int capt,
                                                                  int32_t* __restrict__ idx, int32_t* __restrict__ dist) {
    __shared__ uint4 tile[MATCH_TILE][2];
    const int frame = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int nQ = min(nq[frame], capq), nT = min(nt[frame], capt);
    const int q0 = (blockIdx.x * MATCH_WARPS + wid) * MATCH_NQ;
    uint32_t qw[MATCH_NQ][8];
#pragma unroll
    for (int u = 0; u < MATCH_NQ; ++u) {
#pragma unroll
        for (int k = 0; k < 8; ++k) qw[u][k] = 0;
        if (q0 + u < nQ) {
            const uint4* qp = reinterpret_cast<const uint4*>(q + ((size_t)frame * capq + q0 + u) * 32);
            const uint4 a = qp[0], b = qp[1];
            qw[u][0] = a.x; qw[u][1] = a.y; qw[u][2] = a.z; qw[u][3] = a.w; qw[u][4] = b.x; qw[u][5] = b.y; qw[u][6] = b.z; qw[u][7] = b.w;
        }
    }
    const uint32_t NONE = 0xffffffffu;
    uint32_t k0[MATCH_NQ], k1[MATCH_NQ];
#pragma unroll
    for (int u = 0; u < MATCH_NQ; ++u) { k0[u] = NONE; k1[u] = NONE; }
    const uint4* tp = reinterpret_cast<const uint4*>(t + (size_t)frame * capt * 32);
    for (int base = 0; base < nT; base += MATCH_TILE) {
        const int cnt = min(MATCH_TILE, nT - base);
        __syncthreads();
        for (int i = threadIdx.x; i < cnt * 2; i += MATCH_WARPS * 32) tile[i >> 1][i & 1] = tp[(size_t)(base + (i >> 1)) * 2 + (i & 1)];
        __syncthreads();
        if (q0 < nQ)
            for (int j = lane; j < cnt; j += 32) {
                const uint4 a = tile[j][0], b = tile[j][1];
#pragma unroll
                for (int u = 0; u < MATCH_NQ; ++u) {
                    const int d = __popc(qw[u][0] ^ a.x) + __popc(qw[u][1] ^ a.y) + __popc(qw[u][2] ^ a.z) + __popc(qw[u][3] ^ a.w) +
                                  __popc(qw[u][4] ^ b.x) + __popc(qw[u][5] ^ b.y) + __popc(qw[u][6] ^ b.z) + __popc(qw[u][7] ^ b.w);
                    const uint32_t key = ((uint32_t)d << 16) | (uint32_t)(base + j);
                    if (key < k0[u]) { k1[u] = k0[u]; k0[u] = key; } else if (key < k1[u]) k1[u] = key;
                }
            }
    }
#pragma unroll
    for (int u = 0; u < MATCH_NQ; ++u) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const uint32_t o0 = __shfl_xor_sync(0xffffffffu, k0[u], o), o1 = __shfl_xor_sync(0xffffffffu, k1[u], o);
            const uint32_t lo = min(k0[u], o0), hi = max(k0[u], o0);
            k1[u] = min(hi, min(k1[u], o1));
            k0[u] = lo;
        }
        if (q0 + u < nQ && lane == 0) {
            const size_t o = ((size_t)frame * capq + q0 + u) * 2;
            idx[o] = k0[u] == NONE ? -1 : (int)(k0[u] & 0xffff); dist[o] = k0[u] == NONE ? 256 : (int)(k0[u] >> 16);
            idx[o + 1] = k1[u] == NONE ? -1 : (int)(k1[u] & 0xffff); dist[o + 1] = k1[u] == NONE ? 256 : (int)(k1[u] >> 16);
        }
    }
}

// MatchORBPoints' gate: keep query i when dist < max(2 * min_dist, 15); kept query indices in ascending order.
__global__ void __launch_bounds__(256) k_match_gate(const int32_t* __restrict__ nq, int capq, const int32_t* __restrict__ idx, const int32_t* __restrict__ dist,
                                                    int32_t* __restrict__ good, int32_t* __restrict__ n_good) {
    __shared__ int s_min, s_part[256];
    const int frame = blockIdx.x, tid = threadIdx.x;
    const int nQ = min(nq[frame], capq);
    const int32_t* d = dist + (size_t)frame * capq * 2;
    if (tid == 0) s_min = 1000;
    __syncthreads();
    int m = 1000;
    const int32_t* ix = idx + (size_t)frame * capq * 2;          // rows without a neighbour (empty train set: idx -1) take no part: BFMatcher::match returns
    for (int i = tid; i < nQ; i += 256) if (ix[2 * i] >= 0) m = min(m, d[2 * i]);      // no DMatch for them (src/ORBmatcher.cc:1346-1366)
    atomicMin(&s_min, m);
    __syncthreads();
    const double th = fmax(2.0 * (double)s_min, 15.0);
    const int per = (nQ + 255) / 256, b0 = tid * per, b1 = min(nQ, b0 + per);
    int c = 0;
    for (int i = b0; i < b1; ++i) c += ix[2 * i] >= 0 && (double)d[2 * i] < th;
    s_part[tid] = c;
    __syncthreads();
    if (tid == 0) { int run = 0; for (int k = 0; k < 256; ++k) { const int v = s_part[k]; s_part[k] = run; run += v; } n_good[frame] = run; }
    __syncthreads();
    int pos = s_part[tid];
    for (int i = b0; i < b1; ++i) if (ix[2 * i] >= 0 && (double)d[2 * i] < th) good[(size_t)frame * capq + pos++] = i;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_hamming_knn2_batch_dev(pslam_ctx* c, const uint8_t* d_q, const int32_t* d_nq, int capq, const uint8_t* d_t, const int32_t* d_nt,
                                 int capt, int nframes, int32_t* d_idx, int32_t* d_dist, int32_t* d_good, int32_t* d_ngood) {
    if (!c) return PSLAM_E_INVALID;
    if (!d_q || !d_nq || !d_t || !d_nt || !d_idx || !d_dist || nframes < 1 || capq < 1 || capt < 1 || capt > 65535)
        return set_error(c, PSLAM_E_INVALID, "null pointer, nframes < 1 or capacity outside [1, 65535]");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    PSLAM_LAUNCH(c, "hamming_knn2", k_hamming_knn2<<<dim3((capq + MATCH_WARPS * MATCH_NQ - 1) / (MATCH_WARPS * MATCH_NQ), nframes), MATCH_WARPS * 32, 0, c->stream>>>(
                     d_q, d_nq, capq, d_t, d_nt, capt, d_idx, d_dist));
    if (d_good && d_ngood) PSLAM_LAUNCH(c, "match_gate", k_match_gate<<<nframes, 256, 0, c->stream>>>(d_nq, capq, d_idx, d_dist, d_good, d_ngood));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

int pslam_hamming_knn2(pslam_ctx* c, const uint8_t* q, int nq, const uint8_t* t, int nt, int32_t* idx2, int32_t* dist2, int32_t* good,
                       int32_t* n_good) {
    if (!c) return PSLAM_E_INVALID;
    if (nq < 0 || nt < 0 || nt > 65535 || (nq && !q) || (nt && !t) || !idx2 || !dist2) return set_error(c, PSLAM_E_INVALID, "bad descriptor arrays");
    if (nq == 0) { if (n_good) *n_good = 0; return PSLAM_OK; }
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    const int capt = nt > 0 ? nt : 1;
    cudaStream_t st = c->stream;
    Slab s;
    const auto dq = s.add<uint8_t>((size_t)nq * 32), dt = s.add<uint8_t>((size_t)capt * 32);
    const auto dn = s.add<int32_t>(2), dng = s.add<int32_t>(1), di = s.add<int32_t>((size_t)nq * 2), dd = s.add<int32_t>((size_t)nq * 2), dg = s.add<int32_t>(nq);
    int rc = s.alloc(c);
    if (rc != PSLAM_OK) return rc;
    const int32_t counts[2] = {nq, nt};
    s.up(dq, q, st);
    if (nt) s.up(dt, t, st);
    s.up(dn, counts, st); s.zero(dng, st);
    if ((rc = s.check(c)) != PSLAM_OK) return rc;
    rc = pslam_hamming_knn2_batch_dev(c, s[dq], s[dn], nq, s[dt], s[dn] + 1, capt, 1, s[di], s[dd], good ? s[dg] : nullptr, good ? s[dng] : nullptr);
    if (rc != PSLAM_OK) return rc;
    s.down(idx2, di, st); s.down(dist2, dd, st);
    int32_t ng = 0;
    if (good) { s.down(good, dg, st); s.down(&ng, dng, st); }
    if ((rc = s.sync(c, st)) != PSLAM_OK) return rc;
    if (n_good) *n_good = ng;
    return PSLAM_OK;
}

}  // extern "C"
