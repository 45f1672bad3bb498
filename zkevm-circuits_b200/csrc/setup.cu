// setup.cu -- ParamsKZG<Bn256>::setup / unsafe_setup_with_s / new on the device: g[i] = [s^i] G1 and g_lagrange[i] = [L_i(s)] G1
// for i < n = 2^k, with L_i(s) = w^i (s^n - 1) / (n (s - w^i)) (halo2_proofs src/poly/kzg/commitment.rs).  [s] G2 is host work
// (serde.cu, zkb_g2_setup_host).
//
//   1. scalars: s^i (fr_powers_device) and L_i(s) -- w^i, the n denominators s - w^i through batch_invert_device, then one
//      element-wise pass multiplying in w^i (s^n - 1) / n.  Both vectors (2n scalars) go through the comb in ONE launch.
//   2. fixed-base comb over G = (1, 2): the scalar is recoded into W = ceil(255 / c) signed c-bit digits (digits.cuh, the MSM's
//      recoder) and the point is the sum of W table entries T[w][|d|] = [|d| 2^(c w)] G, negated for a negative digit: W mixed
//      XYZZ additions and no doubling.  The table (W x 2^(c-1) affine points) is built on the device per call: one thread doubles
//      G through the window bases 2^(c w) G, then one thread per entry multiplies its window base by |d|.
//   3. normalisation: Montgomery's trick across each CTA -- one field inversion per SETUP_T points instead of one per point.  Each
//      point contributes ZZ * ZZZ (identity points contribute one and are written as (0, 0)); 1/ZZ = ZZZ / (ZZ ZZZ) and
//      1/ZZZ = ZZ / (ZZ ZZZ).  Field results are unique, so every point is bit-identical to g1_to_affine.
//
// Root of unity: if s^n = 1 then s = w^j for one j < n and every closed-form denominator ... numerator pair at j is 0 / 0.  Upstream's
// `invert().unwrap()` panics there; this entry returns the true Lagrange basis instead, L_i(s) = [i = j]: g_lagrange[j] = G and
// every other entry is the identity, which is what g_to_lagrange(g) (downsize) computes from the same g.  This covers s = 1 and
// s = r - 1 (= w^(n/2)) for every k >= 1.
//
// Window bits and table placement: c = 12 (22 additions per point) with the table (22 x 2048 points, 2.75 MiB) in global memory,
// where it stays L2-resident -- the fastest of the variants measured in DESIGN.md section 3.8.  ZKB_SETUP_WINDOW_BITS (6, 7, 8, 10,
// 12) and ZKB_SETUP_TABLE_SMEM=1 (c <= 7: the table staged into shared memory per CTA) select the others.
#include "common.cuh"
#include "digits.cuh"
#include <stdlib.h>
#include <string.h>

namespace zkb {

constexpr uint32_t SETUP_T = 256;   // points per CTA = points per shared inversion

FF_D Fq shfl_up_fq(const Fq &v, uint32_t o) {
    Fq r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = __shfl_up_sync(0xffffffffu, v.l[i], o);
    return r;
}
FF_D Fq shfl_down_fq(const Fq &v, uint32_t o) {
    Fq r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = __shfl_down_sync(0xffffffffu, v.l[i], o);
    return r;
}

// affine(p) for every thread of the CTA (all SETUP_T threads must call it) with ONE field inversion: the inverse of a_t = ZZ ZZZ
// is inv(prod a) * (prod of a below t) * (prod of a above t); the products come from warp scans in both directions and one
// thread's serial pass over the warp totals.
__device__ __forceinline__ G1Affine block_to_affine(const G1Xyzz &p) {
    constexpr uint32_t NW = SETUP_T / 32;
    __shared__ Fq s_tot[NW], s_below[NW], s_above[NW], s_inv;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const bool id = p.is_identity();
    const Fq a = id ? Fq::one() : fp_mul(p.zz, p.zzz);
    Fq pre = a, suf = a;   // inclusive products of lanes <= lane / >= lane
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const Fq u = shfl_up_fq(pre, o), v = shfl_down_fq(suf, o);
        if (lane >= o) pre = fp_mul(pre, u);
        if (lane + o < 32) suf = fp_mul(suf, v);
    }
    Fq below = shfl_up_fq(pre, 1), above = shfl_down_fq(suf, 1);
    if (lane == 0) below = Fq::one();
    if (lane == 31) above = Fq::one();
    if (lane == 31) s_tot[wid] = pre;
    __syncthreads();
    if (threadIdx.x == 0) {
        Fq acc = Fq::one();
        for (uint32_t w = 0; w < NW; ++w) { s_below[w] = acc; acc = fp_mul(acc, s_tot[w]); }
        s_inv = fp_inv(acc);
        acc = Fq::one();
        for (int w = (int)NW - 1; w >= 0; --w) { s_above[w] = acc; acc = fp_mul(acc, s_tot[w]); }
    }
    __syncthreads();
    const Fq t = fp_mul(fp_mul(s_inv, fp_mul(s_below[wid], below)), fp_mul(s_above[wid], above));
    G1Affine r;
    if (id) { r.x = Fq::zero(); r.y = Fq::zero(); return r; }
    r.x = fp_mul(p.x, fp_mul(t, p.zzz));
    r.y = fp_mul(p.y, fp_mul(t, p.zz));
    return r;
}

// ---- table -----------------------------------------------------------------------------------------------------------------
// bases[w] = [2^(c w)] G, w < windows (one thread: the doubling chain is serial)
__global__ void comb_window_bases_kernel(G1Affine gen, uint32_t c, uint32_t windows, G1Xyzz *__restrict__ bases) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    G1Xyzz b = G1Xyzz::from_affine(gen);
    for (uint32_t w = 0; w < windows; ++w) {
        g1_store_xyzz(bases + w, b);
        for (uint32_t j = 0; j < c; ++j) b = g1_dbl(b);
    }
}
// table[w * half + d - 1] = affine([d] bases[w]), d = 1 ... half
__global__ void __launch_bounds__(SETUP_T) comb_table_kernel(const G1Xyzz *__restrict__ bases, uint32_t c, uint32_t windows,
                                                             G1Affine *__restrict__ table) {
    const uint32_t half = 1u << (c - 1), t = blockIdx.x * SETUP_T + threadIdx.x;
    G1Xyzz acc = G1Xyzz::identity();
    if (t < windows * half) {
        const uint32_t d = t % half + 1;
        const G1Xyzz b = g1_load_xyzz(bases + t / half);
        for (int bit = 31 - __clz(d); bit >= 0; --bit) {
            acc = g1_dbl(acc);
            if ((d >> bit) & 1) g1_add(acc, b);
        }
    }
    const G1Affine r = block_to_affine(acc);
    if (t < windows * half) g1_store_affine(table + t, r);
}

// ---- comb: point i of the 2n scalars -> g_out[i] (i < n) or gl_out[i - n] ---------------------------------------------------------
template <uint32_t C, bool SMEM>
__global__ void __launch_bounds__(SETUP_T, 2) setup_comb_kernel(const Fr *__restrict__ scalars, uint64_t n, const G1Affine *__restrict__ table,
                                                                 G1Affine *__restrict__ g_out, G1Affine *__restrict__ gl_out) {
    constexpr uint32_t W = (255 + C - 1) / C, HALF = 1u << (C - 1);
    const G1Affine *tbl = table;
    if (SMEM) {
        extern __shared__ uint4 sm_tbl[];
        const uint4 *src = reinterpret_cast<const uint4 *>(table);
        for (uint32_t j = threadIdx.x; j < W * HALF * 4; j += SETUP_T) sm_tbl[j] = src[j];
        __syncthreads();
        tbl = reinterpret_cast<const G1Affine *>(sm_tbl);
    }
    const uint64_t i = blockIdx.x * (uint64_t)SETUP_T + threadIdx.x;
    G1Xyzz acc = G1Xyzz::identity();
    if (i < 2 * n) {
        Fr s = fp_to_canonical(fp_load(scalars + i));
        uint32_t carry = 0;
#pragma unroll 1
        for (uint32_t w = 0; w < W; ++w) {
            // window w is the low C bits once the scalar has been shifted right by C w bits: constant limb indices keep the
            // scalar in registers inside the rolled loop
            uint32_t neg;
            const uint32_t d = signed_digit(s.l, 0, C, HALF, carry, neg);
#pragma unroll
            for (int j = 0; j < 7; ++j) s.l[j] = __funnelshift_r(s.l[j], s.l[j + 1], C);
            s.l[7] >>= C;
            if (d != 0) {
                const G1Affine q = g1_load_affine(tbl + w * HALF + (d - 1));
                g1_add_mixed(acc, neg ? g1_neg(q) : q);
            }
        }
    }
    const G1Affine r = block_to_affine(acc);
    if (i < n) g1_store_affine(g_out + i, r);
    else if (i < 2 * n) g1_store_affine(gl_out + (i - n), r);
}

// ---- scalars ---------------------------------------------------------------------------------------------------------------------
__global__ void setup_den_kernel(const Fr *__restrict__ w_pow, Fr s, uint64_t n, Fr *__restrict__ den) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) fp_store(den + i, fp_sub(s, fp_load(w_pow + i)));
}
// L_i = w^i * inv_i * c1 with c1 = (s^n - 1) / n; root != 0 (s^n = 1): L_i = [w^i = s]
__global__ void setup_lagrange_kernel(const Fr *__restrict__ w_pow, Fr *__restrict__ inv_l, Fr c1, Fr s, int root, uint64_t n) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr w = fp_load(w_pow + i);
    fp_store(inv_l + i, root ? (w == s ? Fr::one() : Fr::zero()) : fp_mul(fp_mul(w, fp_load(inv_l + i)), c1));
}

struct CombChoice { uint32_t c; bool smem; };

static int32_t comb_choice(CombChoice *out) {
    const char *cb = getenv("ZKB_SETUP_WINDOW_BITS"), *sm = getenv("ZKB_SETUP_TABLE_SMEM");
    out->c = cb ? (uint32_t)atoi(cb) : 12;
    out->smem = sm && atoi(sm) != 0;
    ZKB_ARG(out->c == 6 || out->c == 7 || out->c == 8 || out->c == 10 || out->c == 12);
    ZKB_ARG(!out->smem || out->c <= 7);   // c = 8 needs 256 KiB, more than a CTA's shared memory
    return ZKB_OK;
}

template <uint32_t C, bool SMEM>
static int32_t launch_comb(zkb_ctx *ctx, const Fr *x, uint64_t n, const G1Affine *table, G1Affine *g_out, G1Affine *gl_out, cudaStream_t st) {
    constexpr uint32_t W = (255 + C - 1) / C, HALF = 1u << (C - 1);
    const size_t smem = SMEM ? (size_t)W * HALF * sizeof(G1Affine) : 0;
    if (SMEM) ZKB_CUDA(cudaFuncSetAttribute(setup_comb_kernel<C, SMEM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    setup_comb_kernel<C, SMEM><<<(unsigned)((2 * n + SETUP_T - 1) / SETUP_T), SETUP_T, smem, st>>>(x, n, table, g_out, gl_out);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

static int32_t srs_setup_run(zkb_ctx *ctx, DevPool &pool, uint32_t k, const Fr &s, const CombChoice &cc, G1Affine *g_out, G1Affine *gl_out,
                             cudaStream_t st) {
    const uint64_t n = 1ull << k;
    const uint32_t c = cc.c, windows = (255 + c - 1) / c, half = 1u << (c - 1);
    Fr *x = nullptr;
    G1Xyzz *bases = nullptr;
    G1Affine *table = nullptr;
    ZKB_TRY(pool.fr(2 * n, &x));
    ZKB_TRY(pool.alloc((size_t)windows * sizeof(G1Xyzz), (void **)&bases));
    ZKB_TRY(pool.alloc((size_t)windows * half * sizeof(G1Affine), (void **)&table));

    // table: window bases, then their multiples
    G1Affine gen;
    gen.x = Fq::one();
    gen.y = fp_add(Fq::one(), Fq::one());
    comb_window_bases_kernel<<<1, 32, 0, st>>>(gen, c, windows, bases);
    comb_table_kernel<<<(windows * half + SETUP_T - 1) / SETUP_T, SETUP_T, 0, st>>>(bases, c, windows, table);
    ctx->launches += 2;

    // scalars: x[0, n) = s^i, x[n, 2n) = L_i(s).  w^i and the denominators are staged in gl_out (n x 64 B = 2n Fr), which the comb
    // overwrites last.
    ZKB_TRY(fr_powers_device(ctx, s, n, x, st));
    Fr *w_pow = (Fr *)gl_out, *den = (Fr *)gl_out + n;
    ZKB_TRY(fr_powers_device(ctx, host_root_of_unity(k), n, w_pow, st));
    Fr sn = s;
    for (uint32_t j = 0; j < k; ++j) sn = fp_sqr(sn);
    const int root = sn == Fr::one();
    const Fr c1 = fp_mul(fp_sub(sn, Fr::one()), fp_inv(fp_from_u64<FrParams>(n)));
    const unsigned eb = (unsigned)((n + 255) / 256);
    if (!root) {
        setup_den_kernel<<<eb, 256, 0, st>>>(w_pow, s, n, den);
        ctx->launches++;
        ZKB_TRY(batch_invert_device(ctx, den, x + n, n, st));
    }
    setup_lagrange_kernel<<<eb, 256, 0, st>>>(w_pow, x + n, c1, s, root, n);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());

    switch (c * 2 + (cc.smem ? 1 : 0)) {
    case 12: return launch_comb<6, false>(ctx, x, n, table, g_out, gl_out, st);
    case 13: return launch_comb<6, true>(ctx, x, n, table, g_out, gl_out, st);
    case 14: return launch_comb<7, false>(ctx, x, n, table, g_out, gl_out, st);
    case 15: return launch_comb<7, true>(ctx, x, n, table, g_out, gl_out, st);
    case 16: return launch_comb<8, false>(ctx, x, n, table, g_out, gl_out, st);
    case 20: return launch_comb<10, false>(ctx, x, n, table, g_out, gl_out, st);
    case 24: return launch_comb<12, false>(ctx, x, n, table, g_out, gl_out, st);
    default: ZKB_ARG(false);
    }
    return ZKB_OK;
}

}  // namespace zkb
using namespace zkb;

extern "C" int32_t zkb_srs_setup_dev(zkb_ctx *ctx, uint32_t k, const uint64_t s[4], uint64_t *g_out_dev, uint64_t *g_lagrange_out_dev, void *stream) {
    ZKB_ARG(ctx && s && g_out_dev && g_lagrange_out_dev && k <= 28);
    ZKB_ARG(((uintptr_t)g_out_dev & 15) == 0 && ((uintptr_t)g_lagrange_out_dev & 15) == 0);
    Fr sm;
    memcpy(sm.l, s, 32);
    bool below_r = false;   // the stored integer must be < r
    for (int i = 7; i >= 0; --i) {
        if (sm.l[i] != FrParams::P(i)) { below_r = sm.l[i] < FrParams::P(i); break; }
    }
    ZKB_ARG(below_r);
    CombChoice cc;
    ZKB_TRY(comb_choice(&cc));
    ZKB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pick_stream(ctx, stream);
    DevPool pool;
    pool.ctx = ctx;
    const int32_t rc = srs_setup_run(ctx, pool, k, sm, cc, (G1Affine *)g_out_dev, (G1Affine *)g_lagrange_out_dev, st);
    const cudaError_t e = cudaStreamSynchronize(st);   // the scratch returns to the block cache only after the kernels using it
    if (rc != ZKB_OK) return rc;
    ZKB_CUDA(e);
    return ZKB_OK;
}
