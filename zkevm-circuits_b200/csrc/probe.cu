// probe.cu -- test surface of the ff.cuh / g1.cuh primitives: one primitive applied to n records of raw operands, on the device
// (grid-stride kernel) and on the host (plain loop), both through the same dispatch, so each side runs the production templates of
// its own compilation pass.  Operands are copied limb by limb and neither reduced nor checked: the lazy forms' wider input ranges
// are reachable.  The op table is documented with zkb_arith_probe_dev in include/zkb200.h.
#include "common.cuh"

namespace zkb {
namespace {

constexpr int PROBE_G1 = 32;  // ops >= 32 are G1 routines (field must be Fq)

// field elements read per record (0: unknown op) and written per record
FF_HD int probe_arity(int op) {
    switch (op) {
    case 2: case 3: case 5: case 11: case 12: case 15: case 16: case 17: case 18: return 1;
    case 0: case 1: case 4: case 8: case 9: case 10: case 13: case 14: return 2;
    case 6: case 7: return 4;
    case 32: return 6;
    case 33: return 8;
    case 34: case 36: return 4;
    case 35: case 37: case 38: return 2;
    default: return 0;
    }
}
FF_HD int probe_width(int op) {
    switch (op) {
    case 32: case 33: case 34: case 35: case 38: return 4;
    case 36: case 37: return 2;
    default: return op < PROBE_G1 ? 1 : 0;
    }
}
// ops 8 - 12 (fp_mul_lazy, fp_add_lazy, fp_sub_lazy, fp_cond_sub) exist on the device only
inline bool probe_device_only(int op) { return op >= 8 && op <= 12; }

template <class PR>
FF_HD Fp<PR> probe_load(const uint64_t *w) {
    Fp<PR> r;
    for (int i = 0; i < 4; ++i) {
        r.l[2 * i] = (uint32_t)w[i];
        r.l[2 * i + 1] = (uint32_t)(w[i] >> 32);
    }
    return r;
}
template <class PR>
FF_HD void probe_store(uint64_t *w, const Fp<PR> &v) {
    for (int i = 0; i < 4; ++i) w[i] = (uint64_t)v.l[2 * i] | ((uint64_t)v.l[2 * i + 1] << 32);
}

template <class PR>
FF_HD Fp<PR> probe_field(int op, const Fp<PR> *x) {
    switch (op) {
    case 0: return fp_add(x[0], x[1]);
    case 1: return fp_sub(x[0], x[1]);
    case 2: return fp_neg(x[0]);
    case 3: return fp_dbl(x[0]);
    case 4: return fp_mul(x[0], x[1]);
    case 5: return fp_sqr(x[0]);
    case 6: return fp_mul_add_mul(x[0], x[1], x[2], x[3]);
    case 7: return fp_mul_sub_mul(x[0], x[1], x[2], x[3]);
#if defined(__CUDA_ARCH__)
    case 8: return fp_mul_lazy(x[0], x[1]);
    case 9: return fp_add_lazy(x[0], x[1]);
    case 10: return fp_sub_lazy(x[0], x[1]);
    case 11: return fp_cond_sub<PR, false>(x[0]);
    case 12: return fp_cond_sub<PR, true>(x[0]);
#endif
    case 13: return fp_pow(x[0], x[1].l);
    case 14: return fp_pow_u64(x[0], (uint64_t)x[1].l[0] | ((uint64_t)x[1].l[1] << 32));
    case 15: return fp_inv(x[0]);
    case 16: return fp_from_canonical(x[0]);
    case 17: return fp_to_canonical(x[0]);
    default: return fp_from_u64<PR>((uint64_t)x[0].l[0] | ((uint64_t)x[0].l[1] << 32));  // 18
    }
}

FF_HD void probe_g1(int op, const Fq *x, Fq *r) {
    G1Affine a;
    G1Xyzz p;
    switch (op) {
    case 32:  // acc XYZZ += q affine
        p = {x[0], x[1], x[2], x[3]};
        a = {x[4], x[5]};
        g1_add_mixed(p, a);
        break;
    case 33: {  // acc XYZZ += q XYZZ
        p = {x[0], x[1], x[2], x[3]};
        const G1Xyzz q = {x[4], x[5], x[6], x[7]};
        g1_add(p, q);
        break;
    }
    case 34: p = g1_dbl(G1Xyzz{x[0], x[1], x[2], x[3]}); break;
    case 35: p = g1_dbl_affine(G1Affine{x[0], x[1]}); break;
    case 36: a = g1_to_affine(G1Xyzz{x[0], x[1], x[2], x[3]}); break;
    case 37: a = g1_neg(G1Affine{x[0], x[1]}); break;
    default: p = G1Xyzz::from_affine(G1Affine{x[0], x[1]}); break;  // 38
    }
    if (op == 36 || op == 37) {
        r[0] = a.x; r[1] = a.y;
    } else {
        r[0] = p.x; r[1] = p.y; r[2] = p.zz; r[3] = p.zzz;
    }
}

// one record: in = arity x 4 limbs, out = width x 4 limbs; op and field already validated
FF_HD void probe_apply(int field, int op, const uint64_t *in, uint64_t *out) {
    const int arity = probe_arity(op);
    if (field == 0) {
        Fr x[4];
        for (int i = 0; i < arity; ++i) x[i] = probe_load<FrParams>(in + 4 * i);
        probe_store(out, probe_field(op, x));
    } else if (op < PROBE_G1) {
        Fq x[4];
        for (int i = 0; i < arity; ++i) x[i] = probe_load<FqParams>(in + 4 * i);
        probe_store(out, probe_field(op, x));
    } else {
        Fq x[8], r[4];
        for (int i = 0; i < arity; ++i) x[i] = probe_load<FqParams>(in + 4 * i);
        probe_g1(op, x, r);
        for (int i = 0; i < probe_width(op); ++i) probe_store(out + 4 * i, r[i]);
    }
}

__global__ void probe_kernel(int field, int op, const uint64_t *__restrict__ in, uint64_t *__restrict__ out, uint64_t n) {
    const int arity = probe_arity(op), width = probe_width(op);
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        probe_apply(field, op, in + i * arity * 4, out + i * width * 4);
}

bool probe_valid(int32_t field, int32_t op) {
    return (field == 0 || field == 1) && op >= 0 && probe_arity(op) > 0 && (op < PROBE_G1 || field == 1);
}

}  // namespace
}  // namespace zkb
using namespace zkb;

extern "C" int32_t zkb_arith_probe_dev(zkb_ctx *ctx, int32_t field, int32_t op, const uint64_t *in_dev, uint64_t *out_dev, uint64_t n,
                                       void *stream) {
    ZKB_ARG(ctx && probe_valid(field, op));
    if (n == 0) return ZKB_OK;
    ZKB_ARG(in_dev && out_dev);
    const uint64_t blocks = (n + 127) / 128, cap = (uint64_t)ctx->sm_count * 8;
    probe_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 128, 0, pick_stream(ctx, stream)>>>(field, op, in_dev, out_dev, n);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

extern "C" int32_t zkb_arith_probe_host(int32_t field, int32_t op, const uint64_t *in, uint64_t *out, uint64_t n) {
    ZKB_ARG(probe_valid(field, op) && !probe_device_only(op));
    if (n == 0) return ZKB_OK;
    ZKB_ARG(in && out);
    const int arity = probe_arity(op), width = probe_width(op);
    for (uint64_t i = 0; i < n; ++i) probe_apply(field, op, in + i * arity * 4, out + i * width * 4);
    return ZKB_OK;
}
