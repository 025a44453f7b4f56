// Host build of planarslam_b200/csrc/lsd_alignbounds.h (the alignment word sets of the CUDA NFA validation), for tests/test_lsd_alignbounds_host.py:
// g++ compiles the very source nvcc compiles for the device.
#include <cstdint>
#include <initializer_list>

#include "lsd_alignbounds.h"

extern "C" {

// out = lo[0..2], len[0..2] of lsd_align_set(theta, prec)
void host_lsd_align_set(double theta, double prec, uint32_t* out) {
    LsdAlignSet S;
    lsd_align_set(theta, prec, S);
    for (int i = 0; i < 3; ++i) { out[i] = S.lo[i]; out[3 + i] = S.len[i]; }
}

// Words of w[0 .. n) and the words within 4 of every bound (with and without the used bit) whose set membership differs from the exact test the kernels
// made before (defined word and lsd_aligned_angle).
long host_lsd_align_mismatches(const uint32_t* w, long n, double theta, double prec) {
    LsdAlignSet S;
    lsd_align_set(theta, prec, S);
    auto exact = [&](uint32_t x) { return (x & 0x7fffffffu) < LSD_ANG_UNDEF && lsd_aligned_angle(lsd_word_angle(x), theta, prec); };
    long bad = 0;
    for (long i = 0; i < n; ++i) bad += exact(w[i]) != lsd_word_aligned(S, w[i]);
    for (int i = 0; i < 3; ++i)
        for (uint32_t b : {S.lo[i], S.lo[i] + S.len[i]})
            for (int d = -4; d <= 4; ++d)
                for (uint32_t u : {0u, 0x80000000u}) {
                    const uint32_t x = ((b + (uint32_t)d) & 0x7fffffffu) | u;
                    bad += exact(x) != lsd_word_aligned(S, x);
                }
    return bad;
}

}  // extern "C"
