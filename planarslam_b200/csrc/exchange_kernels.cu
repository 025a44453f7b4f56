// Key-frame descriptor exchange over NVLink peer memory, fused with the brute-force Hamming matcher (SURVEY.md section 8e; the consumer is the loop-closure /
// relocalisation style query: KeyFrameDatabase::DetectLoopCandidates src/KeyFrameDatabase.cc:76-197 shortlists key frames, ORBmatcher::SearchByBoW(KF, KF)
// src/ORBmatcher.cc:526-659 / cv::BFMatcher::knnMatch compare their descriptors).
//
// One process per GPU.  Every rank owns a block of `slots` key-frame records in its OWN HBM
//     { uint32 epoch flag, int32 count, uint8 desc[cap][32], pslam_keypoint kps[cap] }
// allocated with cudaMalloc and exported as a CUDA IPC handle; the peers map it (cudaIpcOpenMemHandle, NVLink / NVSwitch P2P).  Nothing is gathered into a
// staging buffer: k_exchange_match runs one CTA per (query tile, peer); the CTA for peer p spins on p's epoch flag IN p's MEMORY (ld.acquire.sys), then
// streams p's descriptor rows over NVLink straight into shared memory and keeps each query's two best (distance, row) keys against that peer.  The last CTA
// of a query tile to finish (atomic ticket) merges the per-peer pairs in rank order, so the result is the k = 2 nearest neighbours over the concatenation
// rank 0 rows, rank 1 rows, ... with cv::BFMatcher's tie rule (lowest row first) - identical to pslam_hamming_knn2 on the concatenated set (tested).
// Publishing is a copy into the rank's own record followed by a system-scope release of the epoch flag.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "pslam_internal.h"

namespace pslam {

#define XCH_MAX_WORLD 16
#define XCH_TILE 256
#define XCH_WARPS 8

struct ExchangeBuffers {
    int cap = 0, slots = 0, world = 1, rank = 0;
    size_t slot_bytes = 0;
    DevArray<uint8_t> local;                        // this rank's block
    uint8_t* peer[XCH_MAX_WORLD] = {nullptr};       // mapped blocks (peer[rank] == local)
    bool opened[XCH_MAX_WORLD] = {false};
    DevArray<uint32_t> d_part;                      // [XCH_MAX_WORLD][capq][2] per-peer best keys
    DevArray<int32_t> d_ticket;                     // per query tile
    DevArray<int32_t> d_timeouts;                   // CTAs that gave up waiting for a peer's epoch flag (pslam_exchange_timeouts)
    int capq = 0;
};

struct ExchangePeers { const uint8_t* block[XCH_MAX_WORLD]; };

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t global_timer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
#define XCH_WAIT_NS 20000000000ull      // a peer that has not published after 20 s is treated as absent (its rows are skipped, the wait is counted)
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// record layout inside a slot
__host__ __device__ inline size_t xch_desc_off() { return 16; }
__host__ __device__ inline size_t xch_kps_off(int cap) { return 16 + (size_t)cap * 32; }
__host__ __device__ inline size_t xch_slot_bytes(int cap) { return (16 + (size_t)cap * (32 + 28) + 255) / 256 * 256; }

__global__ void __launch_bounds__(256) k_exchange_publish(uint8_t* __restrict__ slot, int cap, const uint8_t* __restrict__ desc, const pslam_keypoint* __restrict__ kps,
                                                          const int32_t* __restrict__ n_dev, uint32_t epoch) {
    const int n = min(max(*n_dev, 0), cap);
    uint4* d = reinterpret_cast<uint4*>(slot + xch_desc_off());
    const uint4* s = reinterpret_cast<const uint4*>(desc);
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n * 2; i += gridDim.x * 256) d[i] = s[i];
    if (kps) {
        uint32_t* dk = reinterpret_cast<uint32_t*>(slot + xch_kps_off(cap));
        const uint32_t* sk = reinterpret_cast<const uint32_t*>(kps);
        for (int i = blockIdx.x * 256 + threadIdx.x; i < n * 7; i += gridDim.x * 256) dk[i] = sk[i];
    }
    // single-CTA launch: the barrier orders every thread's stores before the flag; the fence + release make them visible to the peers
    __threadfence_system();
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        reinterpret_cast<int32_t*>(slot)[1] = n;
        __threadfence_system();
        st_release_sys(reinterpret_cast<uint32_t*>(slot), epoch);
    }
}

// One CTA per (tile of XCH_WARPS * XCH_NQ queries, peer).  Every warp keeps XCH_NQ queries in registers, so a CTA streams the peer's rows once for 32 queries and
// few CTAs (32 per peer for 1024 queries) sit on an SM while they wait for a peer that is behind - waiting CTAs hold registers the frame kernels of the other
// streams want (measured: 8 % of the step at 2 GPUs with 128 waiting CTAs per peer).
#define XCH_NQ 4
__global__ void __launch_bounds__(XCH_WARPS * 32) k_exchange_match(ExchangePeers P, int world, int cap, size_t slot_off, uint32_t epoch, const uint8_t* __restrict__ q,
                                                                   const int32_t* __restrict__ nq_dev, int capq, uint32_t* __restrict__ part,
                                                                   int32_t* __restrict__ ticket, int32_t* __restrict__ timeouts, int32_t* __restrict__ idx, int32_t* __restrict__ dist) {
    __shared__ uint4 tile[XCH_TILE][2];
    __shared__ int s_nt, s_last;
    const int p = blockIdx.y, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int nQ = min(*nq_dev, capq);
    const int q0 = (blockIdx.x * XCH_WARPS + wid) * XCH_NQ;
    const uint8_t* slot = P.block[p] + slot_off;
    if (threadIdx.x == 0) {
        const uint64_t t0 = global_timer_ns();
        bool there = true;
        while (ld_acquire_sys(reinterpret_cast<const uint32_t*>(slot)) != epoch) {                     // peer p has published this epoch
            __nanosleep(500);
            if (global_timer_ns() - t0 > XCH_WAIT_NS) { there = false; atomicAdd(timeouts, 1); break; }
        }
        s_nt = there ? min(max(reinterpret_cast<const volatile int32_t*>(slot)[1], 0), cap) : 0;
    }
    __syncthreads();
    const int nT = s_nt;
    uint32_t qw[XCH_NQ][8];
#pragma unroll
    for (int t = 0; t < XCH_NQ; ++t) {
#pragma unroll
        for (int k = 0; k < 8; ++k) qw[t][k] = 0;
        if (q0 + t < nQ) {
            const uint4* qp = reinterpret_cast<const uint4*>(q + (size_t)(q0 + t) * 32);
            const uint4 a = qp[0], b = qp[1];
            qw[t][0] = a.x; qw[t][1] = a.y; qw[t][2] = a.z; qw[t][3] = a.w; qw[t][4] = b.x; qw[t][5] = b.y; qw[t][6] = b.z; qw[t][7] = b.w;
        }
    }
    const uint32_t NONE = 0xffffffffu;
    uint32_t k0[XCH_NQ], k1[XCH_NQ];
#pragma unroll
    for (int t = 0; t < XCH_NQ; ++t) { k0[t] = NONE; k1[t] = NONE; }
    const uint4* tp = reinterpret_cast<const uint4*>(slot + xch_desc_off());          // peer memory: these loads cross NVLink
    for (int base = 0; base < nT; base += XCH_TILE) {
        const int cnt = min(XCH_TILE, nT - base);
        __syncthreads();
        for (int i = threadIdx.x; i < cnt * 2; i += XCH_WARPS * 32) tile[i >> 1][i & 1] = tp[(size_t)(base + (i >> 1)) * 2 + (i & 1)];
        __syncthreads();
        if (q0 < nQ)
            for (int j = lane; j < cnt; j += 32) {
                const uint4 a = tile[j][0], b = tile[j][1];
#pragma unroll
                for (int t = 0; t < XCH_NQ; ++t) {
                    const int d = __popc(qw[t][0] ^ a.x) + __popc(qw[t][1] ^ a.y) + __popc(qw[t][2] ^ a.z) + __popc(qw[t][3] ^ a.w) + __popc(qw[t][4] ^ b.x) +
                                  __popc(qw[t][5] ^ b.y) + __popc(qw[t][6] ^ b.z) + __popc(qw[t][7] ^ b.w);
                    const uint32_t key = ((uint32_t)d << 16) | (uint32_t)(base + j);
                    if (key < k0[t]) { k1[t] = k0[t]; k0[t] = key; } else if (key < k1[t]) k1[t] = key;
                }
            }
    }
#pragma unroll
    for (int t = 0; t < XCH_NQ; ++t) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const uint32_t o0 = __shfl_xor_sync(0xffffffffu, k0[t], o), o1 = __shfl_xor_sync(0xffffffffu, k1[t], o);
            const uint32_t lo = min(k0[t], o0), hi = max(k0[t], o0);
            k1[t] = min(hi, min(k1[t], o1));
            k0[t] = lo;
        }
        if (q0 + t < nQ && lane == 0) { part[((size_t)p * capq + q0 + t) * 2] = k0[t]; part[((size_t)p * capq + q0 + t) * 2 + 1] = k1[t]; }
    }
    // the last CTA of this query tile merges the per-peer pairs (rank order = concatenation order)
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&ticket[blockIdx.x], 1) == world - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (threadIdx.x == 0) ticket[blockIdx.x] = 0;                     // ready for the next call
    if (lane < XCH_NQ && q0 + lane < nQ) {
        const int qi = q0 + lane;
        uint64_t b0 = ~0ull, b1 = ~0ull;                              // (distance << 32 | row in the concatenation)
        uint32_t off = 0;
        for (int r = 0; r < world; ++r) {
            const uint8_t* sl = P.block[r] + slot_off;
            const int nr = min(max(reinterpret_cast<const volatile int32_t*>(sl)[1], 0), cap);
            for (int k = 0; k < 2; ++k) {
                const uint32_t key = __ldcg(&part[((size_t)r * capq + qi) * 2 + k]);
                if (key == NONE) continue;
                const uint64_t g = ((uint64_t)(key >> 16) << 32) | (uint64_t)(off + (key & 0xffff));
                if (g < b0) { b1 = b0; b0 = g; } else if (g < b1) b1 = g;
            }
            off += (uint32_t)nr;
        }
        idx[2 * qi] = b0 == ~0ull ? -1 : (int)(b0 & 0xffffffffu); dist[2 * qi] = b0 == ~0ull ? 256 : (int)(b0 >> 32);
        idx[2 * qi + 1] = b1 == ~0ull ? -1 : (int)(b1 & 0xffffffffu); dist[2 * qi + 1] = b1 == ~0ull ? 256 : (int)(b1 >> 32);
    }
}

void exchange_free(pslam_ctx* c) {
    if (!c->exchange) return;
    ExchangeBuffers& B = *c->exchange;
    for (int r = 0; r < B.world; ++r) if (B.opened[r] && B.peer[r]) cudaIpcCloseMemHandle(B.peer[r]);      // before the local block goes
    delete c->exchange;
    c->exchange = nullptr;
}

}  // namespace pslam

using namespace pslam;

extern "C" {

int pslam_exchange_create(pslam_ctx* c, int cap_kp, int slots, void* ipc_handle_out) {
    if (!c) return PSLAM_E_INVALID;
    if (cap_kp < 1 || cap_kp > 65535 || slots < 1 || !ipc_handle_out) return set_error(c, PSLAM_E_INVALID, "exchange: capacity outside [1, 65535], slots < 1 or null handle");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    exchange_free(c);
    c->exchange = new ExchangeBuffers();
    ExchangeBuffers& B = *c->exchange;
    B.cap = cap_kp; B.slots = slots; B.slot_bytes = xch_slot_bytes(cap_kp);
    int rc;
    if ((rc = B.local.reserve(c, B.slot_bytes * slots))) return rc;
    PSLAM_CUDA(c, cudaMemset(B.local, 0, B.slot_bytes * slots));
    if ((rc = B.d_timeouts.reserve(c, 1))) return rc;
    PSLAM_CUDA(c, cudaMemset(B.d_timeouts, 0, 4));
    B.peer[0] = B.local; B.world = 1; B.rank = 0;
    cudaIpcMemHandle_t h;
    PSLAM_CUDA(c, cudaIpcGetMemHandle(&h, B.local));
    static_assert(sizeof(cudaIpcMemHandle_t) == PSLAM_IPC_HANDLE_BYTES, "IPC handle size");
    std::memcpy(ipc_handle_out, &h, sizeof h);
    return PSLAM_OK;
}

int pslam_exchange_attach(pslam_ctx* c, int world, int rank, const void* handles) {
    if (!c) return PSLAM_E_INVALID;
    if (!c->exchange) return set_error(c, PSLAM_E_INVALID, "exchange: create first");
    if (world < 1 || world > XCH_MAX_WORLD || rank < 0 || rank >= world || (world > 1 && !handles)) return set_error(c, PSLAM_E_INVALID, "exchange: bad world / rank");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    ExchangeBuffers& B = *c->exchange;
    B.world = world; B.rank = rank;
    for (int r = 0; r < world; ++r) {
        if (r == rank) { B.peer[r] = B.local; B.opened[r] = false; continue; }
        cudaIpcMemHandle_t h;
        std::memcpy(&h, (const uint8_t*)handles + (size_t)r * sizeof h, sizeof h);
        void* p = nullptr;
        const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) { cudaGetLastError(); return set_error(c, PSLAM_E_NCCL, std::string("exchange: cannot map the block of rank ") + std::to_string(r) + ": " + cudaGetErrorString(e)); }
        B.peer[r] = (uint8_t*)p; B.opened[r] = true;
    }
    return PSLAM_OK;
}

int pslam_exchange_publish_dev(pslam_ctx* c, int slot, const uint8_t* d_desc, const pslam_keypoint* d_kps, const int32_t* d_n, uint32_t epoch) {
    if (!c) return PSLAM_E_INVALID;
    if (!c->exchange || slot < 0 || slot >= c->exchange->slots || !d_desc || !d_n || epoch == 0) return set_error(c, PSLAM_E_INVALID, "exchange publish: bad slot / null pointer / epoch 0");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    ExchangeBuffers& B = *c->exchange;
    PSLAM_LAUNCH(c, "exchange_publish", k_exchange_publish<<<1, 256, 0, c->stream>>>(B.local + (size_t)slot * B.slot_bytes, B.cap, d_desc, d_kps, d_n, epoch));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

int pslam_exchange_match_dev(pslam_ctx* c, int slot, uint32_t epoch, const uint8_t* d_qdesc, const int32_t* d_nq, int capq, int32_t* d_idx, int32_t* d_dist) {
    if (!c) return PSLAM_E_INVALID;
    if (!c->exchange || slot < 0 || slot >= c->exchange->slots || !d_qdesc || !d_nq || !d_idx || !d_dist || capq < 1 || epoch == 0)
        return set_error(c, PSLAM_E_INVALID, "exchange match: bad slot / null pointer / capacity");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    ExchangeBuffers& B = *c->exchange;
    const int tiles = (capq + XCH_WARPS * XCH_NQ - 1) / (XCH_WARPS * XCH_NQ);
    if (capq > B.capq) {
        int rc;
        if ((rc = B.d_part.reserve(c, (size_t)XCH_MAX_WORLD * capq * 2)) || (rc = B.d_ticket.reserve(c, tiles))) return rc;
        PSLAM_CUDA(c, cudaMemsetAsync(B.d_ticket, 0, (size_t)tiles * 4, c->stream));
        B.capq = capq;
    }
    ExchangePeers P;
    for (int r = 0; r < XCH_MAX_WORLD; ++r) P.block[r] = r < B.world ? B.peer[r] : nullptr;
    PSLAM_LAUNCH(c, "exchange_match", k_exchange_match<<<dim3(tiles, B.world), XCH_WARPS * 32, 0, c->stream>>>(P, B.world, B.cap, (size_t)slot * B.slot_bytes, epoch,
                 d_qdesc, d_nq, capq, B.d_part, B.d_ticket, B.d_timeouts, d_idx, d_dist));
    PSLAM_CUDA(c, cudaGetLastError());
    return PSLAM_OK;
}

int pslam_exchange_timeouts(pslam_ctx* c, int32_t* n_out) {
    if (!c) return PSLAM_E_INVALID;
    if (!c->exchange || !n_out) return set_error(c, PSLAM_E_INVALID, "exchange timeouts: create first / null pointer");
    PSLAM_CUDA(c, cudaSetDevice(c->cfg.device));
    PSLAM_CUDA(c, cudaStreamSynchronize(c->stream));
    PSLAM_CUDA(c, cudaMemcpy(n_out, c->exchange->d_timeouts, 4, cudaMemcpyDeviceToHost));
    return PSLAM_OK;
}

}  // extern "C"
