// Ownership of the library's device and page-locked host memory, and the staging of host-pointer calls through one allocation.
// Needs nothing from the library but check_cuda (abi.cu), so a host-only test can compile it against the CUDA runtime.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <cstdint>

#include "../../include/pslam_abi.h"

struct pslam_ctx;

namespace pslam {

int check_cuda(pslam_ctx* c, cudaError_t e, const char* what);

// One cudaMalloc (or, Pinned, cudaMallocHost) allocation of cap elements, freed by the destructor.  Converts to T*, so launches and pointer
// arithmetic take it as they take a raw pointer.
template <typename T, bool Pinned = false>
struct DevArray {
    T* ptr = nullptr;
    size_t cap = 0;

    DevArray() = default;
    DevArray(const DevArray&) = delete;
    DevArray& operator=(const DevArray&) = delete;
    ~DevArray() { release(); }

    operator T*() const { return ptr; }

    void release() {
        if (ptr) { if (Pinned) cudaFreeHost(ptr); else cudaFree(ptr); }
        ptr = nullptr;
        cap = 0;
    }
    // At least n elements (and at least one).  A larger request frees the old block first, so a failed allocation leaves the array empty
    // (null, cap 0) and the next request allocates again.
    int reserve(pslam_ctx* c, size_t n) {
        n = std::max<size_t>(n, 1);
        if (n <= cap) return PSLAM_OK;
        release();
        void* p = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
        if (e != cudaSuccess) return check_cuda(c, e, Pinned ? "cudaMallocHost" : "cudaMalloc");
        ptr = static_cast<T*>(p);
        cap = n;
        return PSLAM_OK;
    }
    // reserve with slack, for scratch whose size changes from call to call: 1.5x the request, at least 256 bytes
    int grow(pslam_ctx* c, size_t n) { return n <= cap ? PSLAM_OK : reserve(c, std::max(n * 3 / 2, (256 + sizeof(T) - 1) / sizeof(T))); }
};

template <typename T>
using PinnedArray = DevArray<T, true>;

// n elements of type T at byte offset off of a Slab
template <typename T>
struct Seg {
    size_t off, n;
};

// Named segments, each 256-byte aligned, laid out over one device allocation: the staging of a host-pointer call.  The allocation is owned by the
// Slab for the length of the call, or carved from a context-owned buffer.  up / down / zero queue copies on a stream and keep the first CUDA error;
// once one has failed, later ones are skipped.
class Slab {
  public:
    template <typename T>
    Seg<T> add(size_t n) {
        const Seg<T> s{bytes_, n};
        bytes_ += (n * sizeof(T) + 255) / 256 * 256;
        return s;
    }
    size_t bytes() const { return bytes_; }

    int alloc(pslam_ctx* c) { return alloc(c, own_); }
    // carve from a context-owned buffer: exact size, or with grow's slack
    int alloc(pslam_ctx* c, DevArray<uint8_t>& buf, bool slack = false) {
        const int rc = slack ? buf.grow(c, bytes_) : buf.reserve(c, bytes_);
        base_ = buf;
        return rc;
    }

    template <typename T>
    T* operator[](Seg<T> s) const { return reinterpret_cast<T*>(base_ + s.off); }

    // n elements (default: the whole segment); zero-byte copies are not queued
    template <typename T>
    void up(Seg<T> s, const T* src, cudaStream_t st, size_t n = SIZE_MAX) { copy((*this)[s], src, std::min(n, s.n) * sizeof(T), cudaMemcpyHostToDevice, st); }
    template <typename T>
    void down(T* dst, Seg<T> s, cudaStream_t st, size_t n = SIZE_MAX) { copy(dst, (*this)[s], std::min(n, s.n) * sizeof(T), cudaMemcpyDeviceToHost, st); }
    template <typename T>
    void zero(Seg<T> s, cudaStream_t st) { if (err_ == cudaSuccess) note(cudaMemsetAsync((*this)[s], 0, s.n * sizeof(T), st), "cudaMemsetAsync"); }

    // PSLAM_OK, or the first failed copy's error
    int check(pslam_ctx* c) const { return check_cuda(c, err_, what_); }
    // synchronises st unless a copy failed; PSLAM_OK or the first error
    int sync(pslam_ctx* c, cudaStream_t st) {
        if (err_ == cudaSuccess) note(cudaStreamSynchronize(st), "cudaStreamSynchronize");
        return check(c);
    }

  private:
    void note(cudaError_t e, const char* what) { if (e != cudaSuccess) { err_ = e; what_ = what; } }
    void copy(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st) {
        if (err_ == cudaSuccess && bytes) note(cudaMemcpyAsync(dst, src, bytes, kind, st), "cudaMemcpyAsync");
    }

    DevArray<uint8_t> own_;
    uint8_t* base_ = nullptr;
    size_t bytes_ = 0;
    cudaError_t err_ = cudaSuccess;
    const char* what_ = "";
};

}  // namespace pslam
