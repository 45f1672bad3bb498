// digits.cuh -- signed c-bit window recoding of a canonical Fr scalar, shared by the Pippenger MSM (msm.cu) and the fixed-base
// comb of the SRS setup (setup.cu).
//
// Window w covers bits [c w, c (w + 1)).  A raw window value plus the carry from the window below is a digit d in [0, 2^c]; a digit
// above 2^(c-1) is replaced by d - 2^c (negative) and carries one into the next window, so every |digit| is in [0, 2^(c-1)].  For a
// scalar < r < 2^254 and ceil(255 / c) windows the top window never carries out.
#pragma once
#include <stdint.h>

namespace zkb {

// c bits of the canonical scalar (8 x u32) from `bit` on (bit < 256)
__device__ __forceinline__ uint32_t raw_window(const uint32_t s[8], uint32_t bit, uint32_t c) {
    const uint32_t limb = bit >> 5, off = bit & 31;
    uint64_t v = s[limb];
    if (limb + 1 < 8) v |= (uint64_t)s[limb + 1] << 32;
    return (uint32_t)(v >> off) & ((1u << c) - 1);
}

// |digit| of the window starting at `bit`, given the carry out of the window below; updates `carry` and sets `neg` (half = 2^(c-1))
__device__ __forceinline__ uint32_t signed_digit(const uint32_t s[8], uint32_t bit, uint32_t c, uint32_t half, uint32_t &carry, uint32_t &neg) {
    uint32_t d = (bit < 256 ? raw_window(s, bit, c) : 0) + carry;
    neg = 0;
    if (d > half) { d = (1u << c) - d; neg = 1; carry = 1; }
    else carry = 0;
    return d;
}

}  // namespace zkb
