// The level-line alignment test of the LSD rectangle validation as integer bounds on the angle word.
//
// lsd_aligned_angle(lsd_word_angle(w), theta, prec) is the reference's isaligned() on a pixel of the angle plane (k_lsd_gradient stores the angle in degrees as
// non-negative float bits, or LSD_ANG_UNDEF = +inf bits when the gradient is too weak).  For one (theta, prec) with 0 <= prec <= 3 pi / 2, the words it accepts are
// at most three intervals of uint32:
//   - integer order on non-negative float bits is float order, and a(w) = fl((double)deg(w) * DEG2RAD) does not decrease as w grows;
//   - e = fl(theta - a) does not increase, r = fl(a - theta) = -e does not decrease, and fl(x - 2 pi) does not decrease in x;
//   - the test accepts w when |e| <= prec (the interval around theta), or when e > 3 pi / 2 and |fl(e - 2 pi)| <= prec (around theta - 2 pi), or when
//     r > 3 pi / 2 and |fl(r - 2 pi)| <= prec (around theta + 2 pi).  Each condition is a conjunction of monotone conditions on w, hence an interval.
// lsd_align_set finds every bound with the exact test itself (a closed-form guess, then a galloping search on the monotone condition), over all non-negative
// floats below LSD_ANG_UNDEF, so that the result does not depend on the range of the angles the gradient kernel produces.  Undefined words fall outside every
// interval.  Plain IEEE double arithmetic only: nvcc (--fmad=false) and g++ (-ffp-contract=off) give the same bounds, and the CPU suite checks them for the host
// (tests/test_lsd_alignbounds_host.py).
#pragma once
#include <stdint.h>
#include <string.h>

#include "lsd_rectenum.h"

#define LSD_PI 3.14159265358979323846
#define LSD_DEG2RAD (LSD_PI / 180)
#define LSD_3_2_PI ((3 * LSD_PI) / 2)
#define LSD_2PI (2 * LSD_PI)
#define LSD_ANG_UNDEF 0x7f800000u

LSD_HD double lsd_word_angle(uint32_t w) {
    const uint32_t m = w & 0x7fffffffu;
    float deg;
    memcpy(&deg, &m, 4);
    return (double)deg * LSD_DEG2RAD;
}

LSD_HD bool lsd_aligned_angle(double a, double theta, double prec) {
    double n_theta = theta - a;
    if (n_theta < 0) n_theta = -n_theta;
    if (n_theta > LSD_3_2_PI) {
        n_theta -= LSD_2PI;
        if (n_theta < 0) n_theta = -n_theta;
    }
    return n_theta <= prec;
}

// aligned words: (w & 0x7fffffff) - lo[i] < len[i] (unsigned) for some i
struct LsdAlignSet { uint32_t lo[3], len[3]; };

LSD_HD bool lsd_word_aligned(const LsdAlignSet& S, uint32_t w) {
    const uint32_t m = w & 0x7fffffffu;
    return (m - S.lo[0] < S.len[0]) | (m - S.lo[1] < S.len[1]) | (m - S.lo[2] < S.len[2]);
}

// the word whose angle is closest to `rad` (a starting point only: the search below does not depend on it)
LSD_HD uint32_t lsd_ab_guess(double rad) {
    const double deg = rad * (180 / LSD_PI);
    if (!(deg > 0)) return 0;
    if (deg >= 3.0e38) return LSD_ANG_UNDEF - 1;
    const float f = (float)deg;
    uint32_t w;
    memcpy(&w, &f, 4);
    return w;
}

// Smallest w in [0, LSD_ANG_UNDEF) for which pred holds, pred being false then true over that range; LSD_ANG_UNDEF when it holds nowhere.  Gallops from
// `guess` to a bracket, then bisects it: a few evaluations when the guess is within a few ulps, 2 log2(distance) + 2 otherwise.
template <class Pred>
LSD_HD uint32_t lsd_ab_first(const Pred& pred, uint32_t guess) {
    uint32_t lo, hi, step = 1;                              // the answer lies in [lo, hi]
    if (guess >= LSD_ANG_UNDEF) guess = LSD_ANG_UNDEF - 1;
    if (pred(guess)) {
        hi = guess;
        while (true) {
            if (hi < step) { lo = 0; break; }
            const uint32_t t = hi - step;
            if (!pred(t)) { lo = t + 1; break; }
            hi = t;
            step *= 2;
        }
    } else {
        lo = guess + 1;
        while (true) {
            const uint32_t t = guess + step;
            if (t >= LSD_ANG_UNDEF) { hi = LSD_ANG_UNDEF; break; }
            if (pred(t)) { hi = t; break; }
            lo = t + 1;
            step *= 2;
        }
    }
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (pred(mid)) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

// The words lsd_aligned_angle(lsd_word_angle(w), theta, prec) accepts, for 0 <= prec <= 3 pi / 2 and a finite theta.
LSD_HD void lsd_align_set(double theta, double prec, LsdAlignSet& S) {
    const double neg = -prec;
    auto set = [&S](int i, uint32_t lo, uint32_t end) { S.lo[i] = lo; S.len[i] = end > lo ? end - lo : 0u; };
    // |e| <= prec: fl(theta - a) <= prec from some word on, fl(a - theta) <= prec up to some word
    set(0, lsd_ab_first([&](uint32_t w) { return theta - lsd_word_angle(w) <= prec; }, lsd_ab_guess(theta - prec)),
        lsd_ab_first([&](uint32_t w) { return !(lsd_word_angle(w) - theta <= prec); }, lsd_ab_guess(theta + prec)));
    // e > 3 pi / 2 and -prec <= fl(e - 2 pi) <= prec, e = fl(theta - a)
    set(1, lsd_ab_first([&](uint32_t w) { const double e = theta - lsd_word_angle(w); return e - LSD_2PI <= prec; }, lsd_ab_guess(theta - LSD_2PI - prec)),
        lsd_ab_first([&](uint32_t w) { const double e = theta - lsd_word_angle(w); return !(e > LSD_3_2_PI && e - LSD_2PI >= neg); },
                     lsd_ab_guess(theta - LSD_2PI + prec)));
    // r > 3 pi / 2 and -prec <= fl(r - 2 pi) <= prec, r = fl(a - theta)
    set(2, lsd_ab_first([&](uint32_t w) { const double r = lsd_word_angle(w) - theta; return r > LSD_3_2_PI && r - LSD_2PI >= neg; },
                        lsd_ab_guess(theta + LSD_2PI - prec)),
        lsd_ab_first([&](uint32_t w) { const double r = lsd_word_angle(w) - theta; return !(r - LSD_2PI <= prec); }, lsd_ab_guess(theta + LSD_2PI + prec)));
}
