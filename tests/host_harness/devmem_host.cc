// Host build of planarslam_b200/csrc/devmem.h (the library's owning device arrays and staging slabs), for tests/test_devmem_host.py: g++ compiles the
// header the library compiles, against the CUDA runtime.  The header needs only check_cuda from the library; this one maps any error to PSLAM_E_CUDA.
#include <cstdint>

#include "devmem.h"

namespace pslam {
int check_cuda(pslam_ctx*, cudaError_t e, const char*) { return e == cudaSuccess ? PSLAM_OK : PSLAM_E_CUDA; }
}  // namespace pslam

using namespace pslam;

struct Rec28 { char b[28]; };           // the size of pslam_keypoint

template <typename T>
static Seg<T> add_seg(Slab& s, long n, long* off) { const Seg<T> g = s.add<T>((size_t)n); *off = (long)g.off; return g; }

extern "C" {

// Lays out segments of elem_bytes[i] (1, 2, 4, 8, 16 or 28) x counts[i]; writes each segment's byte offset, returns the slab size (-1: bad size).
long host_slab_layout(int n, const int* elem_bytes, const long* counts, long* offsets) {
    Slab s;
    for (int i = 0; i < n; ++i) {
        switch (elem_bytes[i]) {
            case 1: add_seg<uint8_t>(s, counts[i], offsets + i); break;
            case 2: add_seg<uint16_t>(s, counts[i], offsets + i); break;
            case 4: add_seg<float>(s, counts[i], offsets + i); break;
            case 8: add_seg<double>(s, counts[i], offsets + i); break;
            case 16: add_seg<int4>(s, counts[i], offsets + i); break;
            case 28: add_seg<Rec28>(s, counts[i], offsets + i); break;
            default: return -1;
        }
    }
    return (long)s.bytes();
}

// reserve(n) (grow(n) when slack) on an empty device (pinned = 0) or page-locked host (pinned = 1) array, twice; state[3k .. 3k + 2] = the return code,
// whether the pointer is set and the cap after call k.
void host_reserve_twice(int pinned, int slack, unsigned long long n, long long* state) {
    auto run = [&](auto& a) {
        for (int k = 0; k < 2; ++k) {
            state[3 * k] = slack ? a.grow(nullptr, n) : a.reserve(nullptr, n);
            state[3 * k + 1] = a.ptr != nullptr;
            state[3 * k + 2] = (long long)a.cap;
        }
    };
    if (pinned) { PinnedArray<uint8_t> a; run(a); } else { DevArray<uint8_t> a; run(a); }
}

// A request that the held block already covers returns PSLAM_OK without touching the CUDA runtime and keeps the block.  The "block" is host
// memory planted in the array and taken out again before the array is destroyed.  Returns 1 when reserve(0), reserve(cap), grow(cap) all kept it.
int host_reserve_within_cap() {
    static uint8_t buf[64];
    DevArray<uint8_t> a;
    a.ptr = buf; a.cap = sizeof buf;
    const bool ok = a.reserve(nullptr, 0) == PSLAM_OK && a.reserve(nullptr, sizeof buf) == PSLAM_OK && a.grow(nullptr, sizeof buf) == PSLAM_OK &&
                    a.ptr == buf && a.cap == sizeof buf;
    a.ptr = nullptr; a.cap = 0;
    return ok ? 1 : 0;
}

// Slab::alloc of a slab with one segment of n bytes, owned for the call (ctx = 0) or carved from an empty context-owned array (ctx = 1).
// Returns the code; *base_null = 1 when the slab's segment pointer is null afterwards, *buf_cap = the context-owned array's cap.
int host_slab_alloc(int ctx, unsigned long long n, int* base_null, long long* buf_cap) {
    DevArray<uint8_t> buf;
    Slab s;
    const Seg<uint8_t> g = s.add<uint8_t>(n);
    const int rc = ctx ? s.alloc(nullptr, buf) : s.alloc(nullptr);
    *base_null = s[g] == nullptr;
    *buf_cap = (long long)buf.cap;
    return rc;
}

}  // extern "C"
