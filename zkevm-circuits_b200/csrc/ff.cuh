// ff.cuh -- 254-bit prime-field arithmetic for BN254 (Fr and Fq), host + device, sm_90a.
//
// In-memory layout is exactly halo2curves' (scroll-tech/halo2curves @ a495a7b, src/bn256/{fr,fq}.rs):
// 4 x u64 little-endian limbs of a*R mod p with R = 2^256, i.e. 8 x u32 little-endian limbs here.  Elements
// in memory are always fully reduced (< p), so buffers can be shared with the Rust side byte for byte
// (reference boundary: prover/src/io.rs:28-34 uses Fr::to_bytes/from_repr on the same type).
//
// Device multiply: word-serial Montgomery (CIOS) on 32-bit limbs with two column-aligned accumulators
// (even/odd) so that every 32x32->64 product is one mad.lo.cc/madc.hi.cc pair on adjacent limbs of a single
// carry chain (ptxas fuses each pair into IMAD.WIDE with predicate carry): 122 IMAD.WIDE + 17 IMAD per multiply in SASS.
// The kernel class built on this is bound by the integer-multiply pipe (fmaheavy: 64 32-bit products/clk/SM), not by HBM --
// see DESIGN.md section 2.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define FF_HD __host__ __device__ __forceinline__
#define FF_D __device__ __forceinline__
#else
#define FF_HD inline
#define FF_D inline
#endif

namespace zkb {

// ---------------------------------------------------------------------------------------------------------
// field parameter packs (constants cross-checked in tests/test_oracle_golden.py against the reference fixture)
// ---------------------------------------------------------------------------------------------------------
struct FrParams {
    static constexpr uint32_t INV = 0xefffffffu;  // -p^{-1} mod 2^32
    FF_HD static constexpr uint32_t P(int i) {
        constexpr uint32_t v[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return v[i];
    }
    FF_HD static constexpr uint32_t P2(int i) {  // 2p (lazy-reduction bound of the NTT butterflies)
        constexpr uint32_t v[8] = {0xe0000002u, 0x87c3eb27u, 0xf372e122u, 0x5067d090u, 0x0302b0bau, 0x70a08b6du, 0xc2634053u, 0x60c89ce5u};
        return v[i];
    }
    FF_HD static constexpr uint32_t R1(int i) {  // R mod p
        constexpr uint32_t v[8] = {0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u, 0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return v[i];
    }
    FF_HD static constexpr uint32_t R2(int i) {  // R^2 mod p
        constexpr uint32_t v[8] = {0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u, 0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u};
        return v[i];
    }
};

struct FqParams {
    static constexpr uint32_t INV = 0xe4866389u;
    FF_HD static constexpr uint32_t P(int i) {
        constexpr uint32_t v[8] = {0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
        return v[i];
    }
    FF_HD static constexpr uint32_t P2(int i) {  // 2p
        constexpr uint32_t v[8] = {0xb0f9fa8eu, 0x7841182du, 0xd0e3951au, 0x2f02d522u, 0x0302b0bbu, 0x70a08b6du, 0xc2634053u, 0x60c89ce5u};
        return v[i];
    }
    FF_HD static constexpr uint32_t R1(int i) {
        constexpr uint32_t v[8] = {0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
        return v[i];
    }
    FF_HD static constexpr uint32_t R2(int i) {
        constexpr uint32_t v[8] = {0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u, 0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u};
        return v[i];
    }
};

template <class PR>
struct alignas(32) Fp {
    uint32_t l[8];

    FF_HD static Fp zero() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; ++i) r.l[i] = 0;
        return r;
    }
    FF_HD static Fp one() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; ++i) r.l[i] = PR::R1(i);
        return r;
    }
    FF_HD static Fp r2() {
        Fp r;
#pragma unroll
        for (int i = 0; i < 8; ++i) r.l[i] = PR::R2(i);
        return r;
    }
    FF_HD bool is_zero() const {
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) o |= l[i];
        return o == 0;
    }
    FF_HD bool operator==(const Fp &b) const {
        uint32_t o = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) o |= l[i] ^ b.l[i];
        return o == 0;
    }
    FF_HD bool operator!=(const Fp &b) const { return !(*this == b); }
};

// ---------------------------------------------------------------------------------------------------------
// add / sub
// ---------------------------------------------------------------------------------------------------------
template <class PR>
FF_HD Fp<PR> fp_add(const Fp<PR> &a, const Fp<PR> &b) {
    Fp<PR> r, t;
#if defined(__CUDA_ARCH__)
    asm("add.cc.u32 %0, %8, %16;\n\t"
        "addc.cc.u32 %1, %9, %17;\n\t"
        "addc.cc.u32 %2, %10, %18;\n\t"
        "addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t"
        "addc.cc.u32 %5, %13, %21;\n\t"
        "addc.cc.u32 %6, %14, %22;\n\t"
        "addc.u32 %7, %15, %23;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7])
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
    uint32_t borrow;
    asm("sub.cc.u32 %0, %9, %17;\n\t"
        "subc.cc.u32 %1, %10, %18;\n\t"
        "subc.cc.u32 %2, %11, %19;\n\t"
        "subc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, %21;\n\t"
        "subc.cc.u32 %5, %14, %22;\n\t"
        "subc.cc.u32 %6, %15, %23;\n\t"
        "subc.cc.u32 %7, %16, %24;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(t.l[0]), "=r"(t.l[1]), "=r"(t.l[2]), "=r"(t.l[3]), "=r"(t.l[4]), "=r"(t.l[5]), "=r"(t.l[6]), "=r"(t.l[7]), "=r"(borrow)
        : "r"(r.l[0]), "r"(r.l[1]), "r"(r.l[2]), "r"(r.l[3]), "r"(r.l[4]), "r"(r.l[5]), "r"(r.l[6]), "r"(r.l[7]),
          "r"(PR::P(0)), "r"(PR::P(1)), "r"(PR::P(2)), "r"(PR::P(3)), "r"(PR::P(4)), "r"(PR::P(5)), "r"(PR::P(6)), "r"(PR::P(7)));
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = borrow ? r.l[i] : t.l[i];
#else
    uint64_t c = 0;
    for (int i = 0; i < 8; ++i) { c += (uint64_t)a.l[i] + b.l[i]; r.l[i] = (uint32_t)c; c >>= 32; }
    int64_t br = 0;
    for (int i = 0; i < 8; ++i) { int64_t d = (int64_t)r.l[i] - PR::P(i) + br; t.l[i] = (uint32_t)d; br = d >> 32; }
    if (br == 0) r = t;
#endif
    return r;
}

template <class PR>
FF_HD Fp<PR> fp_sub(const Fp<PR> &a, const Fp<PR> &b) {
    Fp<PR> r;
#if defined(__CUDA_ARCH__)
    uint32_t borrow;
    asm("sub.cc.u32 %0, %9, %17;\n\t"
        "subc.cc.u32 %1, %10, %18;\n\t"
        "subc.cc.u32 %2, %11, %19;\n\t"
        "subc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, %21;\n\t"
        "subc.cc.u32 %5, %14, %22;\n\t"
        "subc.cc.u32 %6, %15, %23;\n\t"
        "subc.cc.u32 %7, %16, %24;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7]), "=r"(borrow)
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
    // borrow is 0 or 0xffffffff: add back p & borrow
    asm("add.cc.u32 %0, %0, %8;\n\t"
        "addc.cc.u32 %1, %1, %9;\n\t"
        "addc.cc.u32 %2, %2, %10;\n\t"
        "addc.cc.u32 %3, %3, %11;\n\t"
        "addc.cc.u32 %4, %4, %12;\n\t"
        "addc.cc.u32 %5, %5, %13;\n\t"
        "addc.cc.u32 %6, %6, %14;\n\t"
        "addc.u32 %7, %7, %15;"
        : "+r"(r.l[0]), "+r"(r.l[1]), "+r"(r.l[2]), "+r"(r.l[3]), "+r"(r.l[4]), "+r"(r.l[5]), "+r"(r.l[6]), "+r"(r.l[7])
        : "r"(PR::P(0) & borrow), "r"(PR::P(1) & borrow), "r"(PR::P(2) & borrow), "r"(PR::P(3) & borrow),
          "r"(PR::P(4) & borrow), "r"(PR::P(5) & borrow), "r"(PR::P(6) & borrow), "r"(PR::P(7) & borrow));
#else
    int64_t br = 0;
    for (int i = 0; i < 8; ++i) { int64_t d = (int64_t)a.l[i] - b.l[i] + br; r.l[i] = (uint32_t)d; br = d >> 32; }
    if (br) {
        uint64_t c = 0;
        for (int i = 0; i < 8; ++i) { c += (uint64_t)r.l[i] + PR::P(i); r.l[i] = (uint32_t)c; c >>= 32; }
    }
#endif
    return r;
}

template <class PR>
FF_HD Fp<PR> fp_neg(const Fp<PR> &a) {
    return fp_sub(Fp<PR>::zero(), a);
}
template <class PR>
FF_HD Fp<PR> fp_dbl(const Fp<PR> &a) {
    return fp_add(a, a);
}

// ---------------------------------------------------------------------------------------------------------
// Montgomery multiplication
// ---------------------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
namespace detail {
// acc[0..7] (+carry into acc8) += (e0,e1,e2,e3) * b laid out as lo/hi pairs on adjacent limbs -- one carry chain.
FF_D void chain_mad(uint32_t &c0, uint32_t &c1, uint32_t &c2, uint32_t &c3, uint32_t &c4, uint32_t &c5, uint32_t &c6, uint32_t &c7,
                    uint32_t &c8, uint32_t e0, uint32_t e1, uint32_t e2, uint32_t e3, uint32_t b) {
    asm("mad.lo.cc.u32 %0, %9, %13, %0;\n\t"
        "madc.hi.cc.u32 %1, %9, %13, %1;\n\t"
        "madc.lo.cc.u32 %2, %10, %13, %2;\n\t"
        "madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
        "madc.lo.cc.u32 %4, %11, %13, %4;\n\t"
        "madc.hi.cc.u32 %5, %11, %13, %5;\n\t"
        "madc.lo.cc.u32 %6, %12, %13, %6;\n\t"
        "madc.hi.cc.u32 %7, %12, %13, %7;\n\t"
        "addc.u32 %8, %8, 0;"
        : "+r"(c0), "+r"(c1), "+r"(c2), "+r"(c3), "+r"(c4), "+r"(c5), "+r"(c6), "+r"(c7), "+r"(c8)
        : "r"(e0), "r"(e1), "r"(e2), "r"(e3), "r"(b));
}
// same, no carry-out limb (the caller proved the chain cannot overflow)
FF_D void chain_mad_nc(uint32_t &c0, uint32_t &c1, uint32_t &c2, uint32_t &c3, uint32_t &c4, uint32_t &c5, uint32_t &c6, uint32_t &c7,
                       uint32_t e0, uint32_t e1, uint32_t e2, uint32_t e3, uint32_t b) {
    asm("mad.lo.cc.u32 %0, %8, %12, %0;\n\t"
        "madc.hi.cc.u32 %1, %8, %12, %1;\n\t"
        "madc.lo.cc.u32 %2, %9, %12, %2;\n\t"
        "madc.hi.cc.u32 %3, %9, %12, %3;\n\t"
        "madc.lo.cc.u32 %4, %10, %12, %4;\n\t"
        "madc.hi.cc.u32 %5, %10, %12, %5;\n\t"
        "madc.lo.cc.u32 %6, %11, %12, %6;\n\t"
        "madc.hi.cc.u32 %7, %11, %12, %7;"
        : "+r"(c0), "+r"(c1), "+r"(c2), "+r"(c3), "+r"(c4), "+r"(c5), "+r"(c6), "+r"(c7)
        : "r"(e0), "r"(e1), "r"(e2), "r"(e3), "r"(b));
}
// x0 += stray (carry out at the next column) ; then the column-1-aligned chain absorbs that carry
FF_D void chain_stray_mad_nc(uint32_t &x0, uint32_t stray, uint32_t &c0, uint32_t &c1, uint32_t &c2, uint32_t &c3, uint32_t &c4,
                             uint32_t &c5, uint32_t &c6, uint32_t &c7, uint32_t e0, uint32_t e1, uint32_t e2, uint32_t e3, uint32_t b) {
    asm("add.cc.u32 %0, %0, %9;\n\t"
        "madc.lo.cc.u32 %1, %10, %14, %1;\n\t"
        "madc.hi.cc.u32 %2, %10, %14, %2;\n\t"
        "madc.lo.cc.u32 %3, %11, %14, %3;\n\t"
        "madc.hi.cc.u32 %4, %11, %14, %4;\n\t"
        "madc.lo.cc.u32 %5, %12, %14, %5;\n\t"
        "madc.hi.cc.u32 %6, %12, %14, %6;\n\t"
        "madc.lo.cc.u32 %7, %13, %14, %7;\n\t"
        "madc.hi.u32 %8, %13, %14, %8;"
        : "+r"(x0), "+r"(c0), "+r"(c1), "+r"(c2), "+r"(c3), "+r"(c4), "+r"(c5), "+r"(c6), "+r"(c7)
        : "r"(stray), "r"(e0), "r"(e1), "r"(e2), "r"(e3), "r"(b));
}
}  // namespace detail
#endif

// REDUCE = false: the final conditional subtraction is skipped and the result is only guaranteed < 2p ("lazy" form, used by the NTT
// butterflies).  Bounds (word-serial CIOS): the running value stays < a + p and the result is < a*b/R + p, so with R = 2^256 > 4p the
// lazy product of a < 4p (first operand, the one that feeds the multiply chains) and b < p is < 2p and nothing overflows 8 limbs.
template <class PR, bool REDUCE>
FF_HD Fp<PR> fp_mul_t(const Fp<PR> &a, const Fp<PR> &b) {
    Fp<PR> r;
#if defined(__CUDA_ARCH__)
    using namespace detail;
    // running total S = X + Y * 2^32 ; X column-aligned at 0 (9 limbs), Y at column 1 (8 limbs)
    uint32_t x0 = 0, x1 = 0, x2 = 0, x3 = 0, x4 = 0, x5 = 0, x6 = 0, x7 = 0, x8 = 0;
    uint32_t y0 = 0, y1 = 0, y2 = 0, y3 = 0, y4 = 0, y5 = 0, y6 = 0, y7 = 0;
    constexpr uint32_t p0 = PR::P(0), p1 = PR::P(1), p2 = PR::P(2), p3 = PR::P(3), p4 = PR::P(4), p5 = PR::P(5), p6 = PR::P(6), p7 = PR::P(7);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint32_t bi = b.l[i];
        if (i == 0) {
            chain_mad_nc(y0, y1, y2, y3, y4, y5, y6, y7, a.l[1], a.l[3], a.l[5], a.l[7], bi);
        } else {
            // divide S by 2^32 : X' = Y,  Y' = X >> 64,  stray limb x1 joins column 0
            uint32_t s = x1;
            uint32_t t0 = x2, t1 = x3, t2 = x4, t3 = x5, t4 = x6, t5 = x7, t6 = x8;
            x0 = y0; x1 = y1; x2 = y2; x3 = y3; x4 = y4; x5 = y5; x6 = y6; x7 = y7; x8 = 0;
            y0 = t0; y1 = t1; y2 = t2; y3 = t3; y4 = t4; y5 = t5; y6 = t6; y7 = 0;
            chain_stray_mad_nc(x0, s, y0, y1, y2, y3, y4, y5, y6, y7, a.l[1], a.l[3], a.l[5], a.l[7], bi);
        }
        chain_mad(x0, x1, x2, x3, x4, x5, x6, x7, x8, a.l[0], a.l[2], a.l[4], a.l[6], bi);
        const uint32_t m = x0 * PR::INV;
        chain_mad(x0, x1, x2, x3, x4, x5, x6, x7, x8, p0, p2, p4, p6, m);
        chain_mad_nc(y0, y1, y2, y3, y4, y5, y6, y7, p1, p3, p5, p7, m);
    }
    // result = (X >> 32) + Y  (< 2p), then one conditional subtraction
    asm("add.cc.u32 %0, %8, %16;\n\t"
        "addc.cc.u32 %1, %9, %17;\n\t"
        "addc.cc.u32 %2, %10, %18;\n\t"
        "addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t"
        "addc.cc.u32 %5, %13, %21;\n\t"
        "addc.cc.u32 %6, %14, %22;\n\t"
        "addc.u32 %7, %15, %23;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7])
        : "r"(x1), "r"(x2), "r"(x3), "r"(x4), "r"(x5), "r"(x6), "r"(x7), "r"(x8),
          "r"(y0), "r"(y1), "r"(y2), "r"(y3), "r"(y4), "r"(y5), "r"(y6), "r"(y7));
    if (!REDUCE) return r;
    Fp<PR> t;
    uint32_t borrow;
    asm("sub.cc.u32 %0, %9, %17;\n\t"
        "subc.cc.u32 %1, %10, %18;\n\t"
        "subc.cc.u32 %2, %11, %19;\n\t"
        "subc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, %21;\n\t"
        "subc.cc.u32 %5, %14, %22;\n\t"
        "subc.cc.u32 %6, %15, %23;\n\t"
        "subc.cc.u32 %7, %16, %24;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(t.l[0]), "=r"(t.l[1]), "=r"(t.l[2]), "=r"(t.l[3]), "=r"(t.l[4]), "=r"(t.l[5]), "=r"(t.l[6]), "=r"(t.l[7]), "=r"(borrow)
        : "r"(r.l[0]), "r"(r.l[1]), "r"(r.l[2]), "r"(r.l[3]), "r"(r.l[4]), "r"(r.l[5]), "r"(r.l[6]), "r"(r.l[7]),
          "r"(p0), "r"(p1), "r"(p2), "r"(p3), "r"(p4), "r"(p5), "r"(p6), "r"(p7));
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = borrow ? r.l[i] : t.l[i];
#else
    // host: CIOS on 4 x 64-bit limbs with unsigned __int128 (same layout: limb pairs of the 32-bit view)
    uint64_t A[4], B[4], P64[4], t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; ++i) {
        A[i] = (uint64_t)a.l[2 * i] | ((uint64_t)a.l[2 * i + 1] << 32);
        B[i] = (uint64_t)b.l[2 * i] | ((uint64_t)b.l[2 * i + 1] << 32);
        P64[i] = (uint64_t)PR::P(2 * i) | ((uint64_t)PR::P(2 * i + 1) << 32);
    }
    // -p^{-1} mod 2^64 from the 32-bit constant by one Newton step: inv64 = inv32 * (2 + p0 * inv32)   (signs: INV = -p^{-1})
    uint64_t inv64 = PR::INV;
    inv64 = inv64 * (2 + P64[0] * inv64);
    typedef unsigned __int128 u128;
    for (int i = 0; i < 4; ++i) {
        u128 c = 0;
        for (int j = 0; j < 4; ++j) { c += (u128)A[j] * B[i] + t[j]; t[j] = (uint64_t)c; c >>= 64; }
        c += t[4]; t[4] = (uint64_t)c; t[5] = (uint64_t)(c >> 64);
        const uint64_t m = t[0] * inv64;
        c = (u128)m * P64[0] + t[0]; c >>= 64;
        for (int j = 1; j < 4; ++j) { c += (u128)m * P64[j] + t[j]; t[j - 1] = (uint64_t)c; c >>= 64; }
        c += t[4]; t[3] = (uint64_t)c; t[4] = t[5] + (uint64_t)(c >> 64);
    }
    uint64_t u[4];
    u128 br = 0;
    for (int i = 0; i < 4; ++i) { u128 d = (u128)t[i] - P64[i] - (uint64_t)br; u[i] = (uint64_t)d; br = (d >> 64) & 1; }
    const bool ge = t[4] != 0 || br == 0;
    for (int i = 0; i < 4; ++i) {
        const uint64_t v = ge ? u[i] : t[i];
        r.l[2 * i] = (uint32_t)v;
        r.l[2 * i + 1] = (uint32_t)(v >> 32);
    }
#endif
    return r;
}

template <class PR>
FF_HD Fp<PR> fp_mul(const Fp<PR> &a, const Fp<PR> &b) { return fp_mul_t<PR, true>(a, b); }
// a < 4p, b < p (or both < 2p)  ->  a*b/R mod p as a representative < 2p
template <class PR>
FF_HD Fp<PR> fp_mul_lazy(const Fp<PR> &a, const Fp<PR> &b) { return fp_mul_t<PR, false>(a, b); }

template <class PR>
FF_HD Fp<PR> fp_sqr(const Fp<PR> &a) {
    return fp_mul(a, a);
}

#if defined(__CUDACC__)
// ---- lazy (< 2p) arithmetic for the NTT butterflies (device only) --------------------------------------------------------
// a, b < 2p  ->  a + b reduced into [0, 2p)
template <class PR>
__device__ __forceinline__ Fp<PR> fp_add_lazy(const Fp<PR> &a, const Fp<PR> &b) {
    Fp<PR> r, t;
    asm("add.cc.u32 %0, %8, %16;\n\t"
        "addc.cc.u32 %1, %9, %17;\n\t"
        "addc.cc.u32 %2, %10, %18;\n\t"
        "addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t"
        "addc.cc.u32 %5, %13, %21;\n\t"
        "addc.cc.u32 %6, %14, %22;\n\t"
        "addc.u32 %7, %15, %23;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7])
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
    uint32_t borrow;
    asm("sub.cc.u32 %0, %9, %17;\n\t"
        "subc.cc.u32 %1, %10, %18;\n\t"
        "subc.cc.u32 %2, %11, %19;\n\t"
        "subc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, %21;\n\t"
        "subc.cc.u32 %5, %14, %22;\n\t"
        "subc.cc.u32 %6, %15, %23;\n\t"
        "subc.cc.u32 %7, %16, %24;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(t.l[0]), "=r"(t.l[1]), "=r"(t.l[2]), "=r"(t.l[3]), "=r"(t.l[4]), "=r"(t.l[5]), "=r"(t.l[6]), "=r"(t.l[7]), "=r"(borrow)
        : "r"(r.l[0]), "r"(r.l[1]), "r"(r.l[2]), "r"(r.l[3]), "r"(r.l[4]), "r"(r.l[5]), "r"(r.l[6]), "r"(r.l[7]),
          "r"(PR::P2(0)), "r"(PR::P2(1)), "r"(PR::P2(2)), "r"(PR::P2(3)), "r"(PR::P2(4)), "r"(PR::P2(5)), "r"(PR::P2(6)), "r"(PR::P2(7)));
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = borrow ? r.l[i] : t.l[i];
    return r;
}
// a, b < 2p  ->  a - b + 2p  in (0, 4p): no conditional (the wrap of a - b modulo 2^256 is undone by the addition)
template <class PR>
__device__ __forceinline__ Fp<PR> fp_sub_lazy(const Fp<PR> &a, const Fp<PR> &b) {
    Fp<PR> r;
    asm("sub.cc.u32 %0, %8, %16;\n\t"
        "subc.cc.u32 %1, %9, %17;\n\t"
        "subc.cc.u32 %2, %10, %18;\n\t"
        "subc.cc.u32 %3, %11, %19;\n\t"
        "subc.cc.u32 %4, %12, %20;\n\t"
        "subc.cc.u32 %5, %13, %21;\n\t"
        "subc.cc.u32 %6, %14, %22;\n\t"
        "subc.u32 %7, %15, %23;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7])
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
    asm("add.cc.u32 %0, %0, %8;\n\t"
        "addc.cc.u32 %1, %1, %9;\n\t"
        "addc.cc.u32 %2, %2, %10;\n\t"
        "addc.cc.u32 %3, %3, %11;\n\t"
        "addc.cc.u32 %4, %4, %12;\n\t"
        "addc.cc.u32 %5, %5, %13;\n\t"
        "addc.cc.u32 %6, %6, %14;\n\t"
        "addc.u32 %7, %7, %15;"
        : "+r"(r.l[0]), "+r"(r.l[1]), "+r"(r.l[2]), "+r"(r.l[3]), "+r"(r.l[4]), "+r"(r.l[5]), "+r"(r.l[6]), "+r"(r.l[7])
        : "r"(PR::P2(0)), "r"(PR::P2(1)), "r"(PR::P2(2)), "r"(PR::P2(3)), "r"(PR::P2(4)), "r"(PR::P2(5)), "r"(PR::P2(6)), "r"(PR::P2(7)));
    return r;
}
// x < 4p -> [0, 2p)   /   x < 2p -> [0, p): one conditional subtraction of 2p (TWO = true) or p
template <class PR, bool TWO>
__device__ __forceinline__ Fp<PR> fp_cond_sub(const Fp<PR> &x) {
    Fp<PR> t, r;
    uint32_t borrow;
    asm("sub.cc.u32 %0, %9, %17;\n\t"
        "subc.cc.u32 %1, %10, %18;\n\t"
        "subc.cc.u32 %2, %11, %19;\n\t"
        "subc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, %21;\n\t"
        "subc.cc.u32 %5, %14, %22;\n\t"
        "subc.cc.u32 %6, %15, %23;\n\t"
        "subc.cc.u32 %7, %16, %24;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(t.l[0]), "=r"(t.l[1]), "=r"(t.l[2]), "=r"(t.l[3]), "=r"(t.l[4]), "=r"(t.l[5]), "=r"(t.l[6]), "=r"(t.l[7]), "=r"(borrow)
        : "r"(x.l[0]), "r"(x.l[1]), "r"(x.l[2]), "r"(x.l[3]), "r"(x.l[4]), "r"(x.l[5]), "r"(x.l[6]), "r"(x.l[7]),
          "r"(TWO ? PR::P2(0) : PR::P(0)), "r"(TWO ? PR::P2(1) : PR::P(1)), "r"(TWO ? PR::P2(2) : PR::P(2)), "r"(TWO ? PR::P2(3) : PR::P(3)),
          "r"(TWO ? PR::P2(4) : PR::P(4)), "r"(TWO ? PR::P2(5) : PR::P(5)), "r"(TWO ? PR::P2(6) : PR::P(6)), "r"(TWO ? PR::P2(7) : PR::P(7)));
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = borrow ? x.l[i] : t.l[i];
    return r;
}
#endif

// a^e, e given as 8 x u32 little-endian (plain integer)
template <class PR>
FF_HD Fp<PR> fp_pow(const Fp<PR> &a, const uint32_t e[8]) {
    Fp<PR> acc = Fp<PR>::one(), base = a;
    for (int i = 0; i < 256; ++i) {
        if ((e[i >> 5] >> (i & 31)) & 1) acc = fp_mul(acc, base);
        base = fp_sqr(base);
    }
    return acc;
}
template <class PR>
FF_HD Fp<PR> fp_pow_u64(const Fp<PR> &a, uint64_t e) {
    Fp<PR> acc = Fp<PR>::one(), base = a;
    while (e) {
        if (e & 1) acc = fp_mul(acc, base);
        base = fp_sqr(base);
        e >>= 1;
    }
    return acc;
}

// Fermat inverse a^(p-2); inv(0) = 0 (matches ff::Field::invert().unwrap_or(0) uses in halo2's batch_invert)
template <class PR>
FF_HD Fp<PR> fp_inv(const Fp<PR> &a) {
    uint32_t e[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) e[i] = PR::P(i);
    e[0] -= 2;  // P(0) >= 2 for both fields
    Fp<PR> acc = Fp<PR>::one();
    // left-to-right so the loop is squarings + conditional multiplies by the fixed base
    for (int i = 255; i >= 0; --i) {
        acc = fp_sqr(acc);
        if ((e[i >> 5] >> (i & 31)) & 1) acc = fp_mul(acc, a);
    }
    return acc;
}

template <class PR>
FF_HD Fp<PR> fp_from_canonical(const Fp<PR> &c) {  // plain integer limbs (< p) -> Montgomery
    return fp_mul(c, Fp<PR>::r2());
}
template <class PR>
FF_HD Fp<PR> fp_to_canonical(const Fp<PR> &a) {  // Montgomery -> plain integer limbs
    Fp<PR> one = Fp<PR>::zero();
    one.l[0] = 1;
    return fp_mul(a, one);
}
template <class PR>
FF_HD Fp<PR> fp_from_u64(uint64_t v) {
    Fp<PR> c = Fp<PR>::zero();
    c.l[0] = (uint32_t)v;
    c.l[1] = (uint32_t)(v >> 32);
    return fp_from_canonical(c);
}

using Fr = Fp<FrParams>;
using Fq = Fp<FqParams>;

#if defined(__CUDACC__)
// 32-byte element load/store as two 16-byte vector accesses (element = one 32 B DRAM sector)
template <class PR>
FF_D Fp<PR> fp_load(const Fp<PR> *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 lo = q[0], hi = q[1];
    Fp<PR> r;
    r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w;
    r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
    return r;
}
// streaming variants: bypass L1 (ld.global.cg / st.global.cg) so one-touch data does not evict the L1-resident twiddle tables
template <class PR>
FF_D Fp<PR> fp_load_stream(const Fp<PR> *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 lo = __ldcg(q), hi = __ldcg(q + 1);
    Fp<PR> r;
    r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w;
    r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
    return r;
}
template <class PR>
FF_D void fp_store_stream(Fp<PR> *p, const Fp<PR> &v) {
    uint4 *q = reinterpret_cast<uint4 *>(p);
    __stcg(q, make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]));
    __stcg(q + 1, make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]));
}
template <class PR>
FF_D void fp_store(Fp<PR> *p, const Fp<PR> &v) {
    uint4 *q = reinterpret_cast<uint4 *>(p);
    q[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    q[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}
#endif

}  // namespace zkb
