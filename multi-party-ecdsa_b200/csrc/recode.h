// Sliding-window recoding of a fixed exponent (plain host code).  Exponents that are per-key constants (N, p, q, p-1, q-1)
// are recoded once at key upload; nadic_jobs_kernel then multiplies only where a digit sits, by an odd power from a table
// of x, x^3 .. x^(2^SLIDE_BITS - 1).  Against fixed 5-bit windows this saves about a quarter of the non-squaring products.
#pragma once
#include <cstdint>

namespace tecdsa {

constexpr int SLIDE_BITS = 6;       // digits < 64: the 32 odd powers fill one window table of nadic_jobs_kernel

// digits[b] for every bit b < 32 * limbs: 0, or the odd digit of the window whose lowest bit is b, so that
// sum_b digits[b] * 2^b == e.  Windows are taken greedily from the top and never overlap.
inline void slide_recode(uint8_t* digits, const uint32_t* e, int limbs) {
    const int nbits = 32 * limbs;
    auto bit = [&](int i) { return (e[i >> 5] >> (i & 31)) & 1u; };
    for (int i = 0; i < nbits; i++) digits[i] = 0;
    int i = nbits - 1;
    while (i >= 0) {
        if (!bit(i)) { i--; continue; }
        int j = i - SLIDE_BITS + 1 > 0 ? i - SLIDE_BITS + 1 : 0;
        while (!bit(j)) j++;
        uint32_t d = 0;
        for (int k = i; k >= j; k--) d = (d << 1) | bit(k);
        digits[j] = (uint8_t)d;
        i = j - 1;
    }
}

}  // namespace tecdsa
