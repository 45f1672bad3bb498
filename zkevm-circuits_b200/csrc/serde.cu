// serde.cu -- the point encodings of a ParamsKZG file (halo2_proofs SerdeFormat): G1 decode / encode on the device, G2 on the host.
//
//   Processed          32 B per G1 point: LE canonical x, bit 6 of byte 31 = canonical y & 1, bit 7 = 0; identity = 32 zero bytes.
//                      Decoding takes a square root in Fq: y = (x^3 + 3)^((q+1)/4) (q = 3 mod 4), one thread per point.
//   RawBytes           64 B per G1 point, the in-memory G1Affine (Montgomery x || y): limbs < q and on the curve, then a copy.
//   RawBytesUnchecked  the same bytes, copied without a check (no kernel).
//
// A bad point is written as (0, 0) and counted; the first bad index and its reason are packed into one 64-bit word (index << 2 |
// reason) lowered with atomicMin, so the report is the same on every run whatever the schedule.  Host buffers are streamed through
// pinned double buffers in chunks of ZKB_SERDE_CHUNK_POINTS: the copy in of chunk i + 1 overlaps the kernel and the copy out of chunk i.
#include "common.cuh"
#include "serde.cuh"
#include <string.h>
#include <algorithm>

namespace zkb {

// (q + 1) / 4 = (q >> 2) + 1 (q = 3 mod 4; the + 1 cannot carry out of limb 0)
constexpr uint32_t sqrt_exp_word(int i) {
    return ((FqParams::P(i) >> 2) | (i < 7 ? FqParams::P(i + 1) << 30 : 0u)) + (i == 0 ? 1u : 0u);
}
static_assert(sqrt_exp_word(7) >> 28 == 0 && (sqrt_exp_word(7) >> 24) != 0, "(q+1)/4 has 252 bits: its top 4-bit window is bits 248..251");
__constant__ uint32_t SQRT_EXP[8] = {sqrt_exp_word(0), sqrt_exp_word(1), sqrt_exp_word(2), sqrt_exp_word(3),
                                     sqrt_exp_word(4), sqrt_exp_word(5), sqrt_exp_word(6), sqrt_exp_word(7)};

// x < q as plain integers (the check every decoded coordinate needs: halo2curves' from_repr / from_raw_bytes)
FF_HD bool fq_is_canonical(const Fq &x) {
    for (int i = 7; i >= 0; --i) {
        if (x.l[i] != FqParams::P(i)) return x.l[i] < FqParams::P(i);
    }
    return false;
}

FF_HD Fq fq_three() { return fp_add(fp_add(Fq::one(), Fq::one()), Fq::one()); }

// a^((q+1)/4) with a fixed 4-bit window: 14 multiplications for the table, then 62 windows of 4 squarings and at most one multiply
// (the exponent has 252 bits: its top window is bit 248..251) -- about 325 multiplications
__device__ Fq fq_sqrt_candidate(const Fq &a) {
    Fq tbl[16];
    tbl[0] = Fq::one();
    tbl[1] = a;
#pragma unroll 1
    for (int i = 2; i < 16; ++i) tbl[i] = fp_mul(tbl[i - 1], a);
    Fq acc = tbl[(SQRT_EXP[7] >> 24) & 15u];
#pragma unroll 1
    for (int w = 61; w >= 0; --w) {
        acc = fp_sqr(fp_sqr(fp_sqr(fp_sqr(acc))));
        const uint32_t d = (SQRT_EXP[w >> 3] >> (4 * (w & 7))) & 15u;
        if (d) acc = fp_mul(acc, tbl[d]);
    }
    return acc;
}

FF_D Fq fq_load_bytes(const uint4 *p) {
    const uint4 lo = p[0], hi = p[1];
    Fq r;
    r.l[0] = lo.x; r.l[1] = lo.y; r.l[2] = lo.z; r.l[3] = lo.w;
    r.l[4] = hi.x; r.l[5] = hi.y; r.l[6] = hi.z; r.l[7] = hi.w;
    return r;
}

// one Processed point -> affine (Montgomery); returns a ZKB_SERDE_* reason, 0 when the point is good
FF_D uint32_t g1_decompress_point(const uint4 *src, G1Affine &p) {
    Fq x = fq_load_bytes(src);
    const uint32_t top = x.l[7];
    if (top >> 31) return ZKB_SERDE_BAD_FLAGS;
    const uint32_t sign = (top >> 30) & 1u;
    x.l[7] = top & 0x3fffffffu;
    if (x.is_zero() && !sign) { p.x = Fq::zero(); p.y = Fq::zero(); return ZKB_SERDE_OK; }
    if (!fq_is_canonical(x)) return ZKB_SERDE_NON_CANONICAL;
    const Fq xm = fp_from_canonical(x);
    const Fq rhs = fp_add(fp_mul(fp_sqr(xm), xm), fq_three());
    Fq y = fq_sqrt_candidate(rhs);
    if (fp_sqr(y) != rhs) return ZKB_SERDE_NOT_ON_CURVE;
    if ((fp_to_canonical(y).l[0] & 1u) != sign) y = fp_neg(y);
    p.x = xm;
    p.y = y;
    return ZKB_SERDE_OK;
}

FF_D uint32_t g1_check_raw_point(const G1Affine &p) {
    if (!fq_is_canonical(p.x) || !fq_is_canonical(p.y)) return ZKB_SERDE_NON_CANONICAL;
    if (p.is_identity()) return ZKB_SERDE_OK;
    if (fp_sqr(p.y) != fp_add(fp_mul(fp_sqr(p.x), p.x), fq_three())) return ZKB_SERDE_NOT_ON_CURVE;
    return ZKB_SERDE_OK;
}

struct DecodeState {
    unsigned long long first;   // (index << 2) | reason of the first bad point; ~0 when none
    unsigned long long count;
};

template <int FMT>
__global__ void __launch_bounds__(SERDE_THREADS) g1_decode_kernel(const uint4 *__restrict__ in, uint64_t n, uint64_t base,
                                                                  G1Affine *__restrict__ out, DecodeState *st) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1Affine p;
    uint32_t reason;
    if (FMT == ZKB_SERDE_PROCESSED) {
        reason = g1_decompress_point(in + 2 * i, p);
    } else {
        p.x = fq_load_bytes(in + 4 * i);
        p.y = fq_load_bytes(in + 4 * i + 2);
        reason = g1_check_raw_point(p);
    }
    if (reason) {
        p.x = Fq::zero();
        p.y = Fq::zero();
        atomicMin(&st->first, (unsigned long long)(((base + i) << 2) | reason));
        atomicAdd(&st->count, 1ull);
    }
    g1_store_affine(out + i, p);
}

// Processed encoding (G1Affine::to_bytes): canonical x with the parity of canonical y in bit 6 of byte 31
__global__ void __launch_bounds__(SERDE_THREADS) g1_encode_processed_kernel(const G1Affine *__restrict__ in, uint64_t n, uint4 *__restrict__ out) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const G1Affine p = g1_load_affine(in + i);
    Fq x = Fq::zero();
    if (!p.is_identity()) {
        x = fp_to_canonical(p.x);
        x.l[7] |= (fp_to_canonical(p.y).l[0] & 1u) << 30;
    }
    out[2 * i] = make_uint4(x.l[0], x.l[1], x.l[2], x.l[3]);
    out[2 * i + 1] = make_uint4(x.l[4], x.l[5], x.l[6], x.l[7]);
}

// Runs launch(src_dev, dst_dev, count, first_index, stream) over n points of in_sz bytes in / out_sz bytes out.  Device buffers on
// both sides: one launch on st.  Otherwise host sides are staged chunk by chunk; work already queued on st is complete before the first
// chunk starts and the outputs are complete when this returns.
template <class Launch>
static int32_t run_points(zkb_ctx *ctx, const uint8_t *in, size_t in_sz, uint8_t *out, size_t out_sz, uint64_t n, cudaStream_t st, Launch launch) {
    const bool in_dev = is_device_ptr(in), out_dev = is_device_ptr(out);
    if (in_dev) ZKB_ARG(((uintptr_t)in & 15) == 0);
    if (out_dev) ZKB_ARG(((uintptr_t)out & 15) == 0);
    if (in_dev && out_dev) {
        ZKB_TRY(launch(in, out, n, 0, st));
        return ZKB_OK;
    }
    const uint64_t chunk = std::min<uint64_t>(n, ZKB_SERDE_CHUNK_POINTS);
    SerdePipe pp(ctx);
    cudaEvent_t ready;
    ZKB_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    cudaEventRecord(ready, st);
    for (int j = 0; j < 2; ++j) {
        ZKB_CUDA(cudaStreamCreateWithFlags(&pp.s[j], cudaStreamNonBlocking));
        ZKB_CUDA(cudaEventCreateWithFlags(&pp.done[j], cudaEventDisableTiming));
        ZKB_CUDA(cudaStreamWaitEvent(pp.s[j], ready, 0));
        if (!in_dev) {
            ZKB_CUDA(cudaHostAlloc((void **)&pp.h_in[j], chunk * in_sz, cudaHostAllocDefault));
            ZKB_TRY(pp.pool.alloc(chunk * in_sz, (void **)&pp.d_in[j]));
        }
        if (!out_dev) {
            ZKB_CUDA(cudaHostAlloc((void **)&pp.h_out[j], chunk * out_sz, cudaHostAllocDefault));
            ZKB_TRY(pp.pool.alloc(chunk * out_sz, (void **)&pp.d_out[j]));
        }
    }
    cudaEventDestroy(ready);
    const uint64_t nchunks = (n + chunk - 1) / chunk;
    auto drain = [&](uint64_t c) -> int32_t {   // chunk c's slot is idle: hand its output to the caller's buffer
        const int j = (int)(c & 1);
        ZKB_CUDA(cudaEventSynchronize(pp.done[j]));
        if (!out_dev) {
            const uint64_t off = c * chunk, cnt = std::min(chunk, n - off);
            memcpy(out + off * out_sz, pp.h_out[j], cnt * out_sz);
        }
        return ZKB_OK;
    };
    for (uint64_t c = 0; c < nchunks; ++c) {
        const int j = (int)(c & 1);
        if (c >= 2) ZKB_TRY(drain(c - 2));
        const uint64_t off = c * chunk, cnt = std::min(chunk, n - off);
        const uint8_t *src = in_dev ? in + off * in_sz : pp.d_in[j];
        uint8_t *dst = out_dev ? out + off * out_sz : pp.d_out[j];
        if (!in_dev) {
            memcpy(pp.h_in[j], in + off * in_sz, cnt * in_sz);
            ZKB_CUDA(cudaMemcpyAsync(pp.d_in[j], pp.h_in[j], cnt * in_sz, cudaMemcpyHostToDevice, pp.s[j]));
        }
        ZKB_TRY(launch(src, dst, cnt, off, pp.s[j]));
        if (!out_dev) ZKB_CUDA(cudaMemcpyAsync(pp.h_out[j], pp.d_out[j], cnt * out_sz, cudaMemcpyDeviceToHost, pp.s[j]));
        ZKB_CUDA(cudaEventRecord(pp.done[j], pp.s[j]));
    }
    for (uint64_t c = nchunks >= 2 ? nchunks - 2 : 0; c < nchunks; ++c) ZKB_TRY(drain(c));
    return ZKB_OK;
}

// RawBytesUnchecked decode and RawBytes* encode: the encoded point is the in-memory point
static int32_t copy_points(const void *in, void *out, size_t bytes, cudaStream_t st) {
    if (!bytes) return ZKB_OK;
    if (!is_device_ptr(in) && !is_device_ptr(out)) {
        memcpy(out, in, bytes);
        return ZKB_OK;
    }
    ZKB_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDefault, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    return ZKB_OK;
}

// ---- G2 on the host: Fq2 = Fq[i] / (i^2 + 1), twist E'(Fq2): y^2 = x^3 + 3 / (9 + i) ------------------------------------------
struct Fq2 { Fq c0, c1; };
static Fq2 f2_add(const Fq2 &a, const Fq2 &b) { return {fp_add(a.c0, b.c0), fp_add(a.c1, b.c1)}; }
static Fq2 f2_neg(const Fq2 &a) { return {fp_neg(a.c0), fp_neg(a.c1)}; }
static Fq2 f2_mul(const Fq2 &a, const Fq2 &b) {
    const Fq t0 = fp_mul(a.c0, b.c0), t1 = fp_mul(a.c1, b.c1);
    return {fp_sub(t0, t1), fp_sub(fp_sub(fp_mul(fp_add(a.c0, a.c1), fp_add(b.c0, b.c1)), t0), t1)};
}
static bool f2_eq(const Fq2 &a, const Fq2 &b) { return a.c0 == b.c0 && a.c1 == b.c1; }
static bool f2_is_zero(const Fq2 &a) { return a.c0.is_zero() && a.c1.is_zero(); }
static Fq2 f2_pow(const Fq2 &a, const uint32_t e[8]) {
    Fq2 acc = {Fq::one(), Fq::zero()};
    for (int i = 255; i >= 0; --i) {
        acc = f2_mul(acc, acc);
        if ((e[i >> 5] >> (i & 31)) & 1) acc = f2_mul(acc, a);
    }
    return acc;
}
// q >> s as 8 x u32
static void q_shifted(int s, uint32_t e[8]) {
    for (int i = 0; i < 8; ++i) e[i] = (FqParams::P(i) >> s) | (i < 7 ? FqParams::P(i + 1) << (32 - s) : 0u);
}
static Fq2 g2_b() {   // 3 / (9 + i) = (27 - 3 i) / 82
    const Fq inv82 = fp_inv(fp_from_u64<FqParams>(82));
    return {fp_mul(fp_from_u64<FqParams>(27), inv82), fp_neg(fp_mul(fp_from_u64<FqParams>(3), inv82))};
}
static Fq2 g2_rhs(const Fq2 &x) { return f2_add(f2_mul(f2_mul(x, x), x), g2_b()); }

// square root in Fq2 for q = 3 mod 4 (Adj and Rodriguez-Henriquez, "Square root computation over even extension fields", Alg. 9)
static bool f2_sqrt(const Fq2 &a, Fq2 &out) {
    uint32_t e1[8], e2[8];
    q_shifted(2, e1);   // (q - 3) / 4
    q_shifted(1, e2);   // (q - 1) / 2
    const Fq2 a1 = f2_pow(a, e1);
    const Fq2 alpha = f2_mul(a1, f2_mul(a1, a));
    const Fq2 x0 = f2_mul(a1, a);
    const Fq2 minus_one = {fp_neg(Fq::one()), Fq::zero()};
    Fq2 x;
    if (f2_eq(alpha, minus_one)) x = {fp_neg(x0.c1), x0.c0};   // i * x0
    else x = f2_mul(f2_pow(f2_add(alpha, {Fq::one(), Fq::zero()}), e2), x0);
    if (!f2_eq(f2_mul(x, x), a)) return false;
    out = x;
    return true;
}

// the sign bit of a compressed G2 point: parity of canonical y.c0, or of canonical y.c1 when y.c0 = 0 (then y and -y share c0)
static uint32_t g2_sign(const Fq2 &y) {
    const Fq c0 = fp_to_canonical(y.c0);
    return c0.is_zero() ? (fp_to_canonical(y.c1).l[0] & 1u) : (c0.l[0] & 1u);
}

// ---- [s] G2 (ParamsKZG::setup's g2 / s_g2): Jacobian coordinates x = X / Z^2, y = Y / Z^3, identity Z = 0; a = 0 ----------------
struct G2Jac { Fq2 x, y, z; };
static Fq2 f2_sub(const Fq2 &a, const Fq2 &b) { return {fp_sub(a.c0, b.c0), fp_sub(a.c1, b.c1)}; }
static Fq2 f2_dbl(const Fq2 &a) { return f2_add(a, a); }
static Fq2 f2_inv(const Fq2 &a) {   // (c0 - c1 i) / (c0^2 + c1^2); 0 -> 0
    const Fq t = fp_inv(fp_add(fp_mul(a.c0, a.c0), fp_mul(a.c1, a.c1)));
    return {fp_mul(a.c0, t), fp_neg(fp_mul(a.c1, t))};
}
// the halo2curves G2 generator (canonical limbs, 8 x u32 LE per coordinate: x.c0, x.c1, y.c0, y.c1)
static const uint32_t G2_GEN_CANON[4][8] = {
    {0xd992f6edu, 0x46debd5cu, 0xf75edaddu, 0x674322d4u, 0x5e5c4479u, 0x426a0066u, 0x121f1e76u, 0x1800deefu},
    {0xaef312c2u, 0x97e485b7u, 0x35a9e712u, 0xf1aa4933u, 0x31fb5d25u, 0x7260bfb7u, 0x920d483au, 0x198e9393u},
    {0x66fa7daau, 0x4ce6cc01u, 0x0c43d37bu, 0xe3d1e769u, 0x8dcb408fu, 0x4aab7180u, 0xdb8c6debu, 0x12c85ea5u},
    {0xd122975bu, 0x55acdadcu, 0x70b38ef3u, 0xbc4b3133u, 0x690c3395u, 0xec9e99adu, 0x585ff075u, 0x090689d0u},
};
static G2Jac g2_generator() {
    Fq c[4];
    for (int j = 0; j < 4; ++j) {
        for (int i = 0; i < 8; ++i) c[j].l[i] = G2_GEN_CANON[j][i];
        c[j] = fp_from_canonical(c[j]);
    }
    return {{c[0], c[1]}, {c[2], c[3]}, {Fq::one(), Fq::zero()}};
}
static G2Jac g2_identity() { return {{Fq::zero(), Fq::zero()}, {Fq::zero(), Fq::zero()}, {Fq::zero(), Fq::zero()}}; }
static G2Jac g2_dbl(const G2Jac &p) {   // EFD dbl-2009-l
    if (f2_is_zero(p.z)) return p;
    const Fq2 a = f2_mul(p.x, p.x), b = f2_mul(p.y, p.y), c = f2_mul(b, b);
    const Fq2 xb = f2_add(p.x, b);
    const Fq2 d = f2_dbl(f2_sub(f2_sub(f2_mul(xb, xb), a), c));
    const Fq2 e = f2_add(f2_dbl(a), a), f = f2_mul(e, e);
    G2Jac r;
    r.x = f2_sub(f, f2_dbl(d));
    r.y = f2_sub(f2_mul(e, f2_sub(d, r.x)), f2_dbl(f2_dbl(f2_dbl(c))));
    r.z = f2_dbl(f2_mul(p.y, p.z));
    return r;
}
static G2Jac g2_add(const G2Jac &p, const G2Jac &q) {   // EFD add-2007-bl, complete: identity operands, doubling, inverse points
    if (f2_is_zero(p.z)) return q;
    if (f2_is_zero(q.z)) return p;
    const Fq2 z1z1 = f2_mul(p.z, p.z), z2z2 = f2_mul(q.z, q.z);
    const Fq2 u1 = f2_mul(p.x, z2z2), u2 = f2_mul(q.x, z1z1);
    const Fq2 s1 = f2_mul(f2_mul(p.y, q.z), z2z2), s2 = f2_mul(f2_mul(q.y, p.z), z1z1);
    const Fq2 h = f2_sub(u2, u1), rr = f2_dbl(f2_sub(s2, s1));
    if (f2_is_zero(h)) return f2_is_zero(rr) ? g2_dbl(p) : g2_identity();
    const Fq2 h2 = f2_dbl(h), i = f2_mul(h2, h2), j = f2_mul(h, i), v = f2_mul(u1, i);
    G2Jac r;
    r.x = f2_sub(f2_sub(f2_mul(rr, rr), j), f2_dbl(v));
    r.y = f2_sub(f2_mul(rr, f2_sub(v, r.x)), f2_dbl(f2_mul(s1, j)));
    const Fq2 zs = f2_add(p.z, q.z);
    r.z = f2_mul(f2_sub(f2_sub(f2_mul(zs, zs), z1z1), z2z2), h);
    return r;
}
static void fq_to_le_bytes(const Fq &a, uint8_t *b);
// affine raw form (x.c0, x.c1, y.c0, y.c1, Montgomery limbs); identity = zeros
static void g2_to_raw(const G2Jac &p, uint64_t out[16]) {
    memset(out, 0, 16 * sizeof(uint64_t));
    if (f2_is_zero(p.z)) return;
    const Fq2 zi = f2_inv(p.z), zi2 = f2_mul(zi, zi), zi3 = f2_mul(zi2, zi);
    const Fq2 x = f2_mul(p.x, zi2), y = f2_mul(p.y, zi3);
    const Fq v[4] = {x.c0, x.c1, y.c0, y.c1};
    for (int i = 0; i < 4; ++i) fq_to_le_bytes(v[i], (uint8_t *)out + 32 * i);
}

static Fq fq_from_le_bytes(const uint8_t *b) {
    Fq r;
    for (int i = 0; i < 8; ++i) r.l[i] = (uint32_t)b[4 * i] | (uint32_t)b[4 * i + 1] << 8 | (uint32_t)b[4 * i + 2] << 16 | (uint32_t)b[4 * i + 3] << 24;
    return r;
}
static void fq_to_le_bytes(const Fq &a, uint8_t *b) {
    for (int i = 0; i < 32; ++i) b[i] = (uint8_t)(a.l[i >> 2] >> (8 * (i & 3)));
}

}  // namespace zkb

using namespace zkb;

extern "C" int32_t zkb_g1_decode(zkb_ctx *ctx, int32_t format, const uint8_t *in, uint64_t n, uint64_t *out_affine, zkb_decode_report *rep,
                                 void *stream) {
    ZKB_ARG(ctx && rep);
    ZKB_ARG(format == ZKB_SERDE_PROCESSED || format == ZKB_SERDE_RAW_BYTES || format == ZKB_SERDE_RAW_BYTES_UNCHECKED);
    ZKB_ARG(n == 0 || (in && out_affine));
    ZKB_ARG(n < (1ull << 62));
    rep->first_bad = UINT64_MAX;
    rep->count = 0;
    rep->reason = ZKB_SERDE_OK;
    rep->reserved = 0;
    if (n == 0) return ZKB_OK;
    ZKB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pick_stream(ctx, stream);
    if (format == ZKB_SERDE_RAW_BYTES_UNCHECKED) return copy_points(in, out_affine, n * sizeof(G1Affine), st);
    DevPool pool;
    pool.ctx = ctx;
    DecodeState *d_st = nullptr;
    ZKB_TRY(pool.alloc(sizeof(DecodeState), (void **)&d_st));
    ZKB_CUDA(cudaMemsetAsync(d_st, 0xff, 8, st));
    ZKB_CUDA(cudaMemsetAsync((uint8_t *)d_st + 8, 0, 8, st));
    auto launch = [&](const uint8_t *src, uint8_t *dst, uint64_t cnt, uint64_t base, cudaStream_t s) -> int32_t {
        const unsigned grid = (unsigned)((cnt + SERDE_THREADS - 1) / SERDE_THREADS);
        if (format == ZKB_SERDE_PROCESSED)
            g1_decode_kernel<ZKB_SERDE_PROCESSED><<<grid, SERDE_THREADS, 0, s>>>((const uint4 *)src, cnt, base, (G1Affine *)dst, d_st);
        else
            g1_decode_kernel<ZKB_SERDE_RAW_BYTES><<<grid, SERDE_THREADS, 0, s>>>((const uint4 *)src, cnt, base, (G1Affine *)dst, d_st);
        ctx->launches++;
        ZKB_CUDA(cudaGetLastError());
        return ZKB_OK;
    };
    const size_t in_sz = format == ZKB_SERDE_PROCESSED ? 32 : 64;
    ZKB_TRY(run_points(ctx, in, in_sz, (uint8_t *)out_affine, sizeof(G1Affine), n, st, launch));
    DecodeState h;
    ZKB_CUDA(cudaMemcpyAsync(&h, d_st, sizeof(h), cudaMemcpyDeviceToHost, st));   // after every chunk: run_points has joined its streams
    ZKB_CUDA(cudaStreamSynchronize(st));
    if (h.count) {
        rep->first_bad = h.first >> 2;
        rep->reason = (uint32_t)(h.first & 3);
        rep->count = h.count;
    }
    return ZKB_OK;
}

extern "C" int32_t zkb_g1_encode(zkb_ctx *ctx, int32_t format, const uint64_t *in_affine, uint64_t n, uint8_t *out, void *stream) {
    ZKB_ARG(ctx);
    ZKB_ARG(format == ZKB_SERDE_PROCESSED || format == ZKB_SERDE_RAW_BYTES || format == ZKB_SERDE_RAW_BYTES_UNCHECKED);
    ZKB_ARG(n == 0 || (in_affine && out));
    if (n == 0) return ZKB_OK;
    ZKB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pick_stream(ctx, stream);
    if (format != ZKB_SERDE_PROCESSED) return copy_points(in_affine, out, n * sizeof(G1Affine), st);
    auto launch = [&](const uint8_t *src, uint8_t *dst, uint64_t cnt, uint64_t, cudaStream_t s) -> int32_t {
        g1_encode_processed_kernel<<<(unsigned)((cnt + SERDE_THREADS - 1) / SERDE_THREADS), SERDE_THREADS, 0, s>>>((const G1Affine *)src, cnt,
                                                                                                                   (uint4 *)dst);
        ctx->launches++;
        ZKB_CUDA(cudaGetLastError());
        return ZKB_OK;
    };
    ZKB_TRY(run_points(ctx, (const uint8_t *)in_affine, sizeof(G1Affine), out, 32, n, st, launch));
    ZKB_CUDA(cudaStreamSynchronize(st));
    return ZKB_OK;
}

extern "C" int32_t zkb_g2_decode_host(int32_t format, const uint8_t *in, uint64_t out[16], int32_t *status) {
    ZKB_ARG(in && out && status);
    ZKB_ARG(format == ZKB_SERDE_PROCESSED || format == ZKB_SERDE_RAW_BYTES || format == ZKB_SERDE_RAW_BYTES_UNCHECKED);
    *status = ZKB_SERDE_OK;
    if (format != ZKB_SERDE_PROCESSED) {
        uint64_t raw[16];
        memcpy(raw, in, sizeof(raw));
        if (format == ZKB_SERDE_RAW_BYTES) {
            Fq c[4];
            bool canon = true;
            for (int i = 0; i < 4; ++i) {
                c[i] = fq_from_le_bytes(in + 32 * i);
                canon = canon && fq_is_canonical(c[i]);
            }
            const Fq2 x = {c[0], c[1]}, y = {c[2], c[3]};
            if (!canon) *status = ZKB_SERDE_NON_CANONICAL;
            else if (!(f2_is_zero(x) && f2_is_zero(y)) && !f2_eq(f2_mul(y, y), g2_rhs(x))) *status = ZKB_SERDE_NOT_ON_CURVE;
        }
        if (*status == ZKB_SERDE_OK) memcpy(out, raw, sizeof(raw));
        else memset(out, 0, 16 * sizeof(uint64_t));
        return ZKB_OK;
    }
    memset(out, 0, 16 * sizeof(uint64_t));
    if (in[63] >> 7) { *status = ZKB_SERDE_BAD_FLAGS; return ZKB_OK; }
    const uint32_t sign = (in[63] >> 6) & 1u;
    Fq c0 = fq_from_le_bytes(in), c1 = fq_from_le_bytes(in + 32);
    c1.l[7] &= 0x3fffffffu;
    if (c0.is_zero() && c1.is_zero() && !sign) return ZKB_OK;   // identity
    if (!fq_is_canonical(c0) || !fq_is_canonical(c1)) { *status = ZKB_SERDE_NON_CANONICAL; return ZKB_OK; }
    const Fq2 x = {fp_from_canonical(c0), fp_from_canonical(c1)};
    Fq2 y;
    if (!f2_sqrt(g2_rhs(x), y)) { *status = ZKB_SERDE_NOT_ON_CURVE; return ZKB_OK; }
    if (g2_sign(y) != sign) y = f2_neg(y);
    const Fq v[4] = {x.c0, x.c1, y.c0, y.c1};
    for (int i = 0; i < 4; ++i) fq_to_le_bytes(v[i], (uint8_t *)out + 32 * i);
    return ZKB_OK;
}

// g2_out = the G2 generator, s_g2_out = [s] g2 (double-and-add over the canonical bits of s); host only
extern "C" int32_t zkb_g2_setup_host(const uint64_t s[4], uint64_t g2_out[16], uint64_t s_g2_out[16]) {
    ZKB_ARG(s && g2_out && s_g2_out);
    Fr sm;
    memcpy(sm.l, s, 32);
    bool below_r = false;   // the stored integer must be < r
    for (int i = 7; i >= 0; --i) {
        if (sm.l[i] != FrParams::P(i)) { below_r = sm.l[i] < FrParams::P(i); break; }
    }
    ZKB_ARG(below_r);
    const Fr e = fp_to_canonical(sm);
    const G2Jac g = g2_generator();
    G2Jac acc = g2_identity();
    for (int bit = 255; bit >= 0; --bit) {
        acc = g2_dbl(acc);
        if ((e.l[bit >> 5] >> (bit & 31)) & 1) acc = g2_add(acc, g);
    }
    g2_to_raw(g, g2_out);
    g2_to_raw(acc, s_g2_out);
    return ZKB_OK;
}

extern "C" int32_t zkb_g2_encode_host(int32_t format, const uint64_t in[16], uint8_t *out) {
    ZKB_ARG(in && out);
    ZKB_ARG(format == ZKB_SERDE_PROCESSED || format == ZKB_SERDE_RAW_BYTES || format == ZKB_SERDE_RAW_BYTES_UNCHECKED);
    if (format != ZKB_SERDE_PROCESSED) {
        memcpy(out, in, 16 * sizeof(uint64_t));
        return ZKB_OK;
    }
    const uint8_t *b = (const uint8_t *)in;
    const Fq2 x = {fq_from_le_bytes(b), fq_from_le_bytes(b + 32)}, y = {fq_from_le_bytes(b + 64), fq_from_le_bytes(b + 96)};
    memset(out, 0, 64);
    if (f2_is_zero(x) && f2_is_zero(y)) return ZKB_OK;
    fq_to_le_bytes(fp_to_canonical(x.c0), out);
    fq_to_le_bytes(fp_to_canonical(x.c1), out + 32);
    out[63] |= (uint8_t)(g2_sign(y) << 6);
    return ZKB_OK;
}
