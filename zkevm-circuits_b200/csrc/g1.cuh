// g1.cuh -- BN254 G1 group law for the MSM kernels (host + device).
//
// Memory types are halo2curves' (scroll-tech/halo2curves @ a495a7b src/bn256/curve.rs): G1Affine {x, y} with the
// identity stored as (0, 0); G1 {x, y, z} Jacobian.  Internally buckets are accumulated in extended Jacobian
// ("XYZZ": x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2) coordinates: a mixed addition is 8M + 2S with no inversion and a
// cheap identity test (ZZ == 0).  Formulas: EFD "madd-2008-s", "add-2008-s", "dbl-2008-s-1", "mdbl-2008-s-1"
// for short Weierstrass curves with a = 0.
// On the device the squarings use fp_sqr's dedicated square and each y3 = A*B - C*D one reduction (fp_mul_sub_mul); both
// return the same canonical elements as separate multiplies, so the points are bit-identical.
#pragma once
#include "ff.cuh"

namespace zkb {

struct alignas(32) G1Affine {
    Fq x, y;
    FF_HD bool is_identity() const { return x.is_zero() && y.is_zero(); }
};

struct alignas(32) G1Xyzz {
    Fq x, y, zz, zzz;
    FF_HD bool is_identity() const { return zz.is_zero(); }
    FF_HD static G1Xyzz identity() {
        G1Xyzz r;
        r.x = Fq::zero(); r.y = Fq::zero(); r.zz = Fq::zero(); r.zzz = Fq::zero();
        return r;
    }
    FF_HD static G1Xyzz from_affine(const G1Affine &p) {
        if (p.is_identity()) return identity();
        G1Xyzz r;
        r.x = p.x; r.y = p.y; r.zz = Fq::one(); r.zzz = Fq::one();
        return r;
    }
};

// doubling of an affine point -> XYZZ (mdbl-2008-s-1)
FF_HD G1Xyzz g1_dbl_affine(const G1Affine &p) {
    if (p.is_identity()) return G1Xyzz::identity();
    G1Xyzz r;
    Fq u = fp_dbl(p.y);
    Fq v = fp_sqr(u);
    Fq w = fp_mul(u, v);
    Fq s = fp_mul(p.x, v);
    Fq xx = fp_sqr(p.x);
    Fq m = fp_add(fp_dbl(xx), xx);
    r.x = fp_sub(fp_sqr(m), fp_dbl(s));
    r.y = fp_mul_sub_mul(m, fp_sub(s, r.x), w, p.y);
    r.zz = v;
    r.zzz = w;
    return r;
}

FF_HD G1Xyzz g1_dbl(const G1Xyzz &p) {
    if (p.is_identity()) return p;
    G1Xyzz r;
    Fq u = fp_dbl(p.y);
    Fq v = fp_sqr(u);
    Fq w = fp_mul(u, v);
    Fq s = fp_mul(p.x, v);
    Fq xx = fp_sqr(p.x);
    Fq m = fp_add(fp_dbl(xx), xx);
    r.x = fp_sub(fp_sqr(m), fp_dbl(s));
    r.y = fp_mul_sub_mul(m, fp_sub(s, r.x), w, p.y);
    r.zz = fp_mul(v, p.zz);
    r.zzz = fp_mul(w, p.zzz);
    return r;
}

// acc += q (affine), complete: handles identity operands, doubling and inverse points
FF_HD void g1_add_mixed(G1Xyzz &acc, const G1Affine &q) {
    if (q.is_identity()) return;
    if (acc.is_identity()) { acc = G1Xyzz::from_affine(q); return; }
    Fq u2 = fp_mul(q.x, acc.zz);
    Fq s2 = fp_mul(q.y, acc.zzz);
    Fq p = fp_sub(u2, acc.x);
    Fq r = fp_sub(s2, acc.y);
    if (p.is_zero()) {
        if (r.is_zero()) acc = g1_dbl_affine(q);
        else acc = G1Xyzz::identity();
        return;
    }
    Fq pp = fp_sqr(p);
    Fq ppp = fp_mul(p, pp);
    Fq qq = fp_mul(acc.x, pp);
    Fq x3 = fp_sub(fp_sub(fp_sqr(r), ppp), fp_dbl(qq));
    Fq y3 = fp_mul_sub_mul(r, fp_sub(qq, x3), acc.y, ppp);
    acc.x = x3;
    acc.y = y3;
    acc.zz = fp_mul(acc.zz, pp);
    acc.zzz = fp_mul(acc.zzz, ppp);
}

// acc += q (XYZZ), complete
FF_HD void g1_add(G1Xyzz &acc, const G1Xyzz &q) {
    if (q.is_identity()) return;
    if (acc.is_identity()) { acc = q; return; }
    Fq u1 = fp_mul(acc.x, q.zz);
    Fq u2 = fp_mul(q.x, acc.zz);
    Fq s1 = fp_mul(acc.y, q.zzz);
    Fq s2 = fp_mul(q.y, acc.zzz);
    Fq p = fp_sub(u2, u1);
    Fq r = fp_sub(s2, s1);
    if (p.is_zero()) {
        if (r.is_zero()) acc = g1_dbl(acc);
        else acc = G1Xyzz::identity();
        return;
    }
    Fq pp = fp_sqr(p);
    Fq ppp = fp_mul(p, pp);
    Fq qq = fp_mul(u1, pp);
    Fq x3 = fp_sub(fp_sub(fp_sqr(r), ppp), fp_dbl(qq));
    Fq y3 = fp_mul_sub_mul(r, fp_sub(qq, x3), s1, ppp);
    acc.x = x3;
    acc.y = y3;
    acc.zz = fp_mul(fp_mul(acc.zz, q.zz), pp);
    acc.zzz = fp_mul(fp_mul(acc.zzz, q.zzz), ppp);
}

FF_HD G1Affine g1_neg(const G1Affine &p) {
    G1Affine r;
    r.x = p.x;
    r.y = p.is_identity() ? p.y : fp_neg(p.y);
    return r;
}

// XYZZ -> affine (one field inversion)
FF_HD G1Affine g1_to_affine(const G1Xyzz &p) {
    G1Affine r;
    if (p.is_identity()) { r.x = Fq::zero(); r.y = Fq::zero(); return r; }
    // 1/ZZZ, then 1/ZZ = ZZ^2 / ZZZ^2 ... simpler: invert both through one inversion of ZZ*ZZZ
    Fq t = fp_inv(fp_mul(p.zz, p.zzz));
    Fq zz_inv = fp_mul(t, p.zzz);
    Fq zzz_inv = fp_mul(t, p.zz);
    r.x = fp_mul(p.x, zz_inv);
    r.y = fp_mul(p.y, zzz_inv);
    return r;
}

// G1Affine::to_bytes (halo2curves src/derive/curve.rs): LE canonical x, (y & 1) << 6 into byte 31; identity = zeros
inline void g1_compress(const G1Affine &p, uint8_t out[32]) {
    if (p.is_identity()) { for (int i = 0; i < 32; ++i) out[i] = 0; return; }
    Fq x = fp_to_canonical(p.x), y = fp_to_canonical(p.y);
    for (int i = 0; i < 8; ++i) {
        out[4 * i + 0] = (uint8_t)(x.l[i]);
        out[4 * i + 1] = (uint8_t)(x.l[i] >> 8);
        out[4 * i + 2] = (uint8_t)(x.l[i] >> 16);
        out[4 * i + 3] = (uint8_t)(x.l[i] >> 24);
    }
    out[31] |= (uint8_t)((y.l[0] & 1u) << 6);
}

#if defined(__CUDACC__)
FF_D G1Affine g1_load_affine(const G1Affine *p) {
    G1Affine r;
    r.x = fp_load(&p->x);
    r.y = fp_load(&p->y);
    return r;
}
FF_D void g1_store_affine(G1Affine *p, const G1Affine &v) {
    fp_store(&p->x, v.x);
    fp_store(&p->y, v.y);
}
FF_D G1Xyzz g1_load_xyzz(const G1Xyzz *p) {
    G1Xyzz r;
    r.x = fp_load(&p->x); r.y = fp_load(&p->y); r.zz = fp_load(&p->zz); r.zzz = fp_load(&p->zzz);
    return r;
}
FF_D void g1_store_xyzz(G1Xyzz *p, const G1Xyzz &v) {
    fp_store(&p->x, v.x); fp_store(&p->y, v.y); fp_store(&p->zz, v.zz); fp_store(&p->zzz, v.zzz);
}
#endif

}  // namespace zkb
