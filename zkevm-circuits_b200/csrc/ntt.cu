// ntt.cu -- radix-2 NTT over BN254 Fr for sm_90a: persistent CTAs, TMA-staged data and twiddle tiles, mbarrier pipeline.
//
// Replaces halo2_proofs::arithmetic::best_fft (halo2_proofs 1.1.0 @ e5ddf67 src/arithmetic.rs; reached from
// circuit-benchmarks/src/super_circuit.rs:117-132 through EvaluationDomain::{lagrange_to_coeff, coeff_to_extended,
// extended_to_coeff}).  Same contract: in place, natural order in / natural order out, a'[k] = sum_j a[j] w^(jk).
//
// Design (NOT upstream's bit-reverse + log n global layers):
//   n = A1 * A2 (* A3): 1 pass up to 2^11, 2 passes up to 2^20, 3 passes above (non-final factors <= 2^9, final <= 2^11).  A pass
//   is ONE persistent kernel, TWO 256-thread CTAs per SM, each walking over TILES of 2048 elements (64 KB): a tile is C = 2048 / A
//   adjacent columns of the Cooley-Tukey index split, i.e. C independent length-A transforms whose rows are C*32 contiguous bytes
//   in HBM.  The two resident CTAs run out of phase, so while one waits for TMA data, converts layouts or streams results out, the
//   other is in its multiplier-bound butterfly rounds: the integer-multiply pipe (the bound, see DESIGN.md) stays fed.  Per tile:
//     * the data tile is fetched by TMA (cp.async.bulk.tensor.2d through a per-column tensor map: box = 256 rows x 32 B;
//       the contiguous sub-transforms of the last pass by cp.async.bulk), completion signalled on an mbarrier
//       (complete_tx::bytes); the fetch of tile i+1 is issued the moment tile i's last result left shared memory;
//     * the tile's inter-pass twiddles w_n^(j_in * k) are TMA-staged as well: the table is stored tile-major in the order the
//       store phase consumes it and streams through a ring of four 8 KB slots (one slot = the 256 elements of one store
//       iteration), refilled four iterations ahead -- across the tile boundary, so the next tile's first twiddles are already
//       resident while its butterflies run;
//     * the A/2 local twiddles of the pass sit in shared memory for the life of the CTA (one bulk copy at kernel start);
//     * decimation in frequency in radix-8 rounds held in registers (8 elements / thread / round, 256 threads), the short round
//       first and a radix-8 round last, where the unit twiddles (3 of 8 per thread, plus the whole last stage) are known at
//       compile time and cost no multiply: (A/2) log2 A - (A - 1) + A/8 multiplies per transform instead of (A/2) log2 A;
//     * two 16-byte planes with an XOR swizzle + one padding slot per column -> conflict-free 128-bit LDS/STS;
//     * results leave through 32-byte streaming stores, C adjacent threads writing C*32 contiguous bytes.
//   Scaling by 1/n (any caller scale) is folded into the last inter-pass table; zeta-coset scaling and an arbitrary
//   per-element input scale are fused into the first / last register round.
#include "common.cuh"
#include <string.h>
#include <stdlib.h>
#include <algorithm>
#include <cuda.h>  // CUtensorMap + enums only; cuTensorMapEncodeTiled is resolved at run time (no -lcuda)

namespace zkb {

// Two 256-thread CTAs per SM on 2048-element tiles: a non-final pass takes 105 KB of shared memory per CTA (header + data tile
// + twiddle ring + local twiddles), so two CTAs fit the 228 KB of an H100 SM.
constexpr int NTT_TILE_BITS = 11;        // 2048 elements = 64 KB per tile
constexpr int NTT_MAX_BITS = 11;         // largest in-CTA transform (final pass: no twiddle ring in shared memory)
constexpr int NTT_PREF_INNER_BITS = 9;   // non-final passes: <= 8 KB of local twiddles next to the 32 KB twiddle ring -> two CTAs per SM
constexpr int NTT_MAX_INNER_BITS = 9;
constexpr int NTT_THREADS = 256;         // 8 elements per thread and round
constexpr int NTT_CTAS_PER_SM = 2;
constexpr int TW_LO_BITS = 12;
constexpr uint32_t NTT_BOX_ROWS = 256;
constexpr uint32_t NTT_HDR_BYTES = 128;                                  // mbarriers: [0] data, [1] local twiddles, [2..5] ring slots
constexpr uint32_t NTT_DBUF_BYTES = 32u * ((1u << NTT_TILE_BITS) + 32u);  // two 16-byte planes of C*(A+1) <= 2048+32 slots (A >= 64 in multi-pass plans)
constexpr uint32_t NTT_TW_SLOTS = 4;
constexpr uint32_t NTT_TW_SLOT_ELEMS = NTT_THREADS;                       // one store iteration
constexpr uint32_t NTT_TW_RING_BYTES = NTT_TW_SLOTS * NTT_TW_SLOT_ELEMS * 32u;

// ZETA = 7^((r-1)/3) and ZETA^2 (Montgomery form); EvaluationDomain::g_coset / g_coset_inv (poly/domain.rs)
__device__ __constant__ uint32_t ZETA_POW[2][8];

struct PassArgs {
    uint32_t a;          // log2 of the in-CTA transform length A
    uint32_t log_c;      // log2 of the number of columns per tile (C * A = tile elements)
    uint32_t log_inner;  // log2 of the element stride S between the rows of this pass
    uint32_t log_n;
    uint32_t is_final;   // last pass: contiguous sub-transforms in, digit-reversed scatter out
    uint32_t a1, a2;     // final pass: bits of the first / middle pass (oidx = k1 + (k2 << a1) + (k << (a1 + a2)))
    uint32_t coset_in;   // multiply input i by ZETA^(i mod 3)        (first pass only)
    uint32_t coset_out;  // multiply output k by ZETA^(-(k mod 3))    (final pass only)
    uint32_t use_scale;  // multiply outputs by *scale                 (single-pass transforms only)
    uint32_t has_in_scale;
    uint32_t tiles_per_col, total_tiles;
    const Fr *loc;       // 2^(a-1) local twiddles of this pass
    const Fr *tw;        // inter-pass table of this boundary, tile-major (non-final passes)
    const Fr *scale;
    const Fr *in_scale;  // optional per-element input multiplier (first pass only): coset scaling tables
    // final pass of a domain-sharded transform (sharded.cu): output element oidx is multiplied by out_tw[oidx] and stored into the
    // receive window of rank (oidx >> peer_log_blk) at row peer_rank -- the all-to-all of the four-step NTT happens inside the
    // store phase, over NVLink peer memory, tile by tile
    const Fr *out_tw;
    uint32_t peer_routed, peer_log_blk, peer_rank;
    Fr *peers[16];
    const CUtensorMap *maps;   // per column: 2-D view [n / S rows][S * 4 u64] of the pass input (non-final passes)
    const Fr *const *src;      // per column input  (final pass: bulk copies)
    Fr *const *dst;            // per column output
};

struct TileInfo {
    uint32_t y;       // column of the batch
    uint32_t c0;      // first column of the tile (non-final: j_in block; final: k1 block)
    uint32_t outer;   // non-final: index of the enclosing outer block; final: k2
    uint32_t tw_tile;
};

__device__ __forceinline__ TileInfo decode_tile(const PassArgs &p, uint32_t gt) {
    TileInfo t;
    t.y = gt / p.tiles_per_col;
    const uint32_t tau = gt - t.y * p.tiles_per_col;
    const uint32_t lb = (p.is_final ? p.a1 : p.log_inner) - p.log_c;  // log2 (number of column blocks)
    const uint32_t blk = tau & ((1u << lb) - 1);
    t.outer = tau >> lb;
    t.c0 = blk << p.log_c;
    t.tw_tile = blk;
    return t;
}

// ---- PTX wrappers: mbarrier + TMA -----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "NTT_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra NTT_DONE;\n"
        "bra NTT_WAIT;\n"
        "NTT_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, int32_t x, int32_t y, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
                 "l"(map), "r"(x), "r"(y), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void tma_load_bulk(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
                 "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- shared-memory element access -----------------------------------------------------------------------------------------
// L0: the layout TMA leaves: element (c, r) at byte (c * A + r) * 32.
// L1: two 16-byte planes, element (c, r) at slot c * (A + 1) + (r ^ ((r >> 3) & 7)): unit-stride runs stay conflict free, the
//     stride-8 pattern of the last radix-8 round hits 8 distinct bank groups, and the +1 per column spreads the columns of a
//     row over distinct banks for the store phase.
__device__ __forceinline__ uint32_t swz(uint32_t i) { return i ^ ((i >> 3) & 7u); }
__device__ __forceinline__ Fr ld_pair(const uint4 *lo, const uint4 *hi) {
    const uint4 a = *lo, b = *hi;
    Fr r;
    r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w;
    r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}
__device__ __forceinline__ Fr ld_lin(const uint8_t *buf, uint32_t idx) {
    const uint4 *q = reinterpret_cast<const uint4 *>(buf) + 2 * (size_t)idx;
    return ld_pair(q, q + 1);
}
__device__ __forceinline__ Fr ld_l1(const uint4 *lo, const uint4 *hi, uint32_t slot) { return ld_pair(lo + slot, hi + slot); }
__device__ __forceinline__ void st_l1(uint4 *lo, uint4 *hi, uint32_t slot, const Fr &v) {
    lo[slot] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    hi[slot] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}
__device__ __forceinline__ Fr zeta_pow(int i) {  // i in {1,2}
    Fr z;
#pragma unroll
    for (int k = 0; k < 8; ++k) z.l[k] = ZETA_POW[i - 1][k];
    return z;
}

// R consecutive DIF stages (s .. s+R-1) on groups of 2^R elements held in registers: one shared-memory round trip and one
// barrier per R stages.  Every thread owns 8 element slots per round (8 / 2^R groups).  FIRST: the inputs are read from the
// TMA layout L0 (with the fused input scalings), then -- after a barrier, the conversion is in place -- written in L1.
// LAST (s + R == a): the group's elements are adjacent rows, so the twiddle exponents depend on the register index alone and the
// unit twiddles (m & (d - 1)) == 0 are dropped at compile time.
template <int R, bool FIRST, bool LAST>
__device__ __forceinline__ void ntt_round(uint8_t *dbuf, const PassArgs &p, const TileInfo &ti, uint32_t s, const uint8_t *loc_sm, uint32_t tid) {
    constexpr int E = 1 << R, NG = 8 / E;
    const uint32_t a = p.a, A = 1u << a;
    const uint32_t elems = 1u << (a + p.log_c);
    const uint32_t total_groups = elems >> R;
    const uint32_t lgpc = a - R;                     // log2 (groups per column)
    const uint32_t lq = LAST ? 0u : a - s - R;       // log2 of the spacing of a group's elements (half distance of the round's last stage)
    const uint32_t q = 1u << lq;
    uint4 *lo = reinterpret_cast<uint4 *>(dbuf);
    uint4 *hi = lo + ((A + 1) << p.log_c);
    Fr x[8];
    uint32_t cbase[NG], rbase[NG], ploc[NG];
#pragma unroll
    for (int u = 0; u < NG; ++u) {
        // a tile shorter than 8 x 256 elements (single-pass transforms below 2^11) wraps: the surplus threads redo a valid
        // group and write identical values, which keeps the register arrays free of divergent definitions
        const uint32_t G = (tid + u * NTT_THREADS) & (total_groups - 1);
        uint32_t c, ghi;
        if (FIRST || p.log_c < 3) {
            // rows fastest: adjacent lanes read adjacent 32-byte elements of the TMA layout (and, with fewer than 8 columns per
            // tile, the only mapping that keeps the 128-bit data accesses of a quarter-warp on 8 distinct bank groups)
            c = G >> lgpc;
            const uint32_t g = G & ((1u << lgpc) - 1);
            ploc[u] = g & (q - 1);
            ghi = g >> lq;
        } else {
            // columns fastest, then the block index, then the position inside the block: the lanes of a warp share ONE twiddle
            // (position), which the shared-memory load broadcasts -- with rows fastest the twiddle loads of the middle rounds are
            // strided by 2^(s+t) elements and replay up to 32 times (measured: 39 M of 80 M wavefronts per pass were replays);
            // the data stays conflict free because the column stride A + 1 is odd
            c = G & ((1u << p.log_c) - 1);
            const uint32_t rest = G >> p.log_c, lgh = lgpc - lq;
            ghi = rest & ((1u << lgh) - 1);
            ploc[u] = rest >> lgh;
        }
        rbase[u] = (ghi << (lq + R)) + ploc[u];
        cbase[u] = c;
#pragma unroll
        for (int m = 0; m < E; ++m) {
            const uint32_t r = rbase[u] + ((uint32_t)m << lq);
            if (FIRST) x[u * E + m] = ld_lin(dbuf, (c << a) + r);
            else x[u * E + m] = ld_l1(lo, hi, c * (A + 1) + swz(r));
        }
    }
    if (FIRST) {
        if (p.coset_in || p.has_in_scale) {
#pragma unroll
            for (int u = 0; u < NG; ++u) {
#pragma unroll
                for (int m = 0; m < E; ++m) {
                    const uint32_t r = rbase[u] + ((uint32_t)m << lq);
                    const uint32_t idx = (r << p.log_inner) + ti.c0 + cbase[u];   // first pass: outer == 0
                    if (p.coset_in) {
                        const uint32_t z = idx % 3;
                        if (z) x[u * E + m] = fp_mul_lazy(x[u * E + m], zeta_pow(z));
                    }
                    if (p.has_in_scale) x[u * E + m] = fp_mul_lazy(x[u * E + m], fp_load(p.in_scale + idx));
                }
            }
        }
        __syncthreads();  // every L0 read is done before the first L1 write (same bytes)
    }
#pragma unroll
    for (int u = 0; u < NG; ++u) {
#pragma unroll
        for (int t = 0; t < R; ++t) {
            const int d = E >> (t + 1);
            const bool last_trivial = ((uint32_t)d << lq) == 1u;   // half distance 1: twiddle is omega^0
#pragma unroll
            for (int m = 0; m < E; ++m) {
                if ((m & d) == 0) {
                    // lazy butterflies: every element stays a representative < 2p; u - v + 2p (< 4p, no conditional) feeds the
                    // multiply chains directly and the product comes back < 2p without the final conditional subtraction
                    const Fr uu = x[u * E + m], vv = x[u * E + m + d];
                    x[u * E + m] = fp_add_lazy(uu, vv);
                    Fr dif = fp_sub_lazy(uu, vv);
                    if (LAST) {
                        if ((m & (d - 1)) != 0) dif = fp_mul_lazy(dif, ld_lin(loc_sm, (uint32_t)(m & (d - 1)) << (s + t)));
                        else dif = fp_cond_sub<FrParams, true>(dif);
                    } else if (!last_trivial) {
                        const uint32_t pos = ploc[u] + ((uint32_t)(m & (d - 1)) << lq);
                        dif = fp_mul_lazy(dif, ld_lin(loc_sm, pos << (s + t)));
                    } else dif = fp_cond_sub<FrParams, true>(dif);
                    x[u * E + m + d] = dif;
                }
            }
        }
#pragma unroll
        for (int m = 0; m < E; ++m) {
            const uint32_t r = rbase[u] + ((uint32_t)m << lq);
            st_l1(lo, hi, cbase[u] * (A + 1) + swz(r), x[u * E + m]);
        }
    }
}

// thread 0: start the TMA traffic of one tile into data buffer `dst` (shared address), completion on `bar`
__device__ __forceinline__ void issue_data(const PassArgs &p, uint32_t gt, uint32_t dst, uint32_t bar) {
    const TileInfo t = decode_tile(p, gt);
    const uint32_t A = 1u << p.a, C = 1u << p.log_c;
    mbar_expect_tx(bar, (A << p.log_c) * 32u);
    if (!p.is_final) {
        const CUtensorMap *map = p.maps + t.y;
        const uint32_t br = A < NTT_BOX_ROWS ? A : NTT_BOX_ROWS;
        for (uint32_t c = 0; c < C; ++c)
            for (uint32_t r0 = 0; r0 < A; r0 += br)
                tma_load_2d(dst + ((c << p.a) + r0) * 32u, map, (int32_t)((t.c0 + c) * 4u), (int32_t)((t.outer << p.a) + r0), bar);
    } else {
        const Fr *src = p.src[t.y];
        for (uint32_t c = 0; c < C; ++c) {
            const uint64_t sub = ((uint64_t)(t.c0 + c) << p.a2) + t.outer;   // sub-transform (k1, k2): input is contiguous
            tma_load_bulk(dst + (c << p.a) * 32u, src + (sub << p.a), A * 32u, bar);
        }
    }
}
// thread 0: stage chunk `chunk` (chunk_elems twiddles) of tile gt's boundary-table tile into ring slot memory `dst`
__device__ __forceinline__ void issue_tw(const PassArgs &p, uint32_t gt, uint32_t chunk, uint32_t chunk_elems, uint32_t dst, uint32_t bar) {
    const TileInfo t = decode_tile(p, gt);
    const uint32_t bytes = chunk_elems * 32u;
    mbar_expect_tx(bar, bytes);
    tma_load_bulk(dst, p.tw + ((size_t)t.tw_tile << (p.a + p.log_c)) + (size_t)chunk * chunk_elems, bytes, bar);
}

__global__ void __launch_bounds__(NTT_THREADS, NTT_CTAS_PER_SM) ntt_tile_kernel(const __grid_constant__ PassArgs p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t tid = threadIdx.x;
    const uint32_t a = p.a, A = 1u << a, C = 1u << p.log_c, elems = A << p.log_c;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem);   // [0] data buffer, [1] local twiddles, [2 .. 5] twiddle ring slots
    uint8_t *d = smem + NTT_HDR_BYTES;
    uint8_t *twring = d + NTT_DBUF_BYTES;
    uint8_t *locbuf = twring + (p.is_final ? 0u : NTT_TW_RING_BYTES);
    const uint32_t bar_d = smem_u32(bars), bar_loc = smem_u32(bars + 1), bar_tw0 = smem_u32(bars + 2);
    const uint32_t stride = gridDim.x;
    uint32_t gt = blockIdx.x;
    if (gt >= p.total_tiles) return;
    // the boundary-table tile is consumed in chunks of one store iteration (256 elements; a whole short tile at once)
    const uint32_t chunk_elems = elems < NTT_TW_SLOT_ELEMS ? elems : NTT_TW_SLOT_ELEMS;
    const uint32_t nchunks = elems / chunk_elems;
    // thread 0 only: position of the next chunk to stage (walks this CTA's tile sequence), and its running number
    uint32_t is_gt = gt, is_c = 0, is_g = 0;
    uint32_t g_wait = 0;   // running number of the next chunk to consume: slot = g & 3, parity = (g >> 2) & 1

    if (tid == 0) {
        mbar_init(bar_d, 1); mbar_init(bar_loc, 1);
        for (uint32_t j = 0; j < NTT_TW_SLOTS; ++j) mbar_init(bar_tw0 + 8 * j, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
        const uint32_t loc_bytes = (a ? (A >> 1) : 1u) * 32u;
        mbar_expect_tx(bar_loc, loc_bytes);
        tma_load_bulk(smem_u32(locbuf), p.loc, loc_bytes, bar_loc);
        issue_data(p, gt, smem_u32(d), bar_d);
        if (!p.is_final) {
            for (; is_g < NTT_TW_SLOTS && is_gt < p.total_tiles; ++is_g) {
                issue_tw(p, is_gt, is_c, chunk_elems, smem_u32(twring) + (is_g & 3u) * (NTT_TW_SLOT_ELEMS * 32u), bar_tw0 + 8 * (is_g & 3u));
                if (++is_c == nchunks) { is_c = 0; is_gt += stride; }
            }
        }
    }
    mbar_wait(bar_loc, 0);

    for (uint32_t it = 0; gt < p.total_tiles; ++it, gt += stride) {
        const TileInfo ti = decode_tile(p, gt);
        mbar_wait(bar_d, it & 1);

        // decimation in frequency: natural order in, bit-reversed order out (inside shared memory); radix-8 rounds in registers,
        // the short round (a mod 3 stages) first, so that the last one is a full radix-8 round with compile-time unit twiddles
        if (a == 0) {
            ntt_round<0, true, false>(d, p, ti, 0, locbuf, tid);
            __syncthreads();
        } else {
            const uint32_t r0 = a % 3 ? a % 3 : 3;
            if (r0 == 1) ntt_round<1, true, false>(d, p, ti, 0, locbuf, tid);
            else if (r0 == 2) ntt_round<2, true, false>(d, p, ti, 0, locbuf, tid);
            else ntt_round<3, true, false>(d, p, ti, 0, locbuf, tid);
            __syncthreads();
            uint32_t s = r0;
            while (a - s > 3) { ntt_round<3, false, false>(d, p, ti, s, locbuf, tid); __syncthreads(); s += 3; }
            if (a - s == 3) { ntt_round<3, false, true>(d, p, ti, s, locbuf, tid); __syncthreads(); }
        }

        const uint4 *lo = reinterpret_cast<const uint4 *>(d);
        const uint4 *hi = lo + ((A + 1) << p.log_c);
        Fr *__restrict__ out = p.dst[ti.y];
        if (!p.is_final) {
            // slot q of a column holds output k = bitrev(q); the staged table is [q][c] in exactly this order
            for (uint32_t u = 0; u < nchunks; ++u, ++g_wait) {
                const uint32_t slot = g_wait & 3u;
                mbar_wait(bar_tw0 + 8 * slot, (g_wait >> 2) & 1u);
                const uint32_t e = tid + u * NTT_THREADS;
                if (tid < chunk_elems) {
                    const uint32_t c = e & (C - 1), q = e >> p.log_c;
                    const uint32_t k = __brev(q) >> (32 - a);   // a >= 1 in non-final passes
                    const Fr v = fp_mul_lazy(ld_l1(lo, hi, c * (A + 1) + swz(q)), ld_lin(twring + slot * (NTT_TW_SLOT_ELEMS * 32u), tid));   // < 2p: the next pass takes it lazily
                    const uint64_t oidx = ((((uint64_t)ti.outer << a) + k) << p.log_inner) + ti.c0 + c;
                    fp_store_stream(out + oidx, v);
                }
                // generic-proxy reads of this slot (and, after the last iteration, of the data buffer) are ordered before the
                // async-proxy (TMA) writes that reuse them
                fence_proxy_async();
                __syncthreads();
                if (tid == 0 && is_gt < p.total_tiles) {
                    issue_tw(p, is_gt, is_c, chunk_elems, smem_u32(twring) + (is_g & 3u) * (NTT_TW_SLOT_ELEMS * 32u), bar_tw0 + 8 * (is_g & 3u));
                    ++is_g;
                    if (++is_c == nchunks) { is_c = 0; is_gt += stride; }
                }
            }
        } else {
            const uint64_t obase = (uint64_t)ti.c0 + ((uint64_t)ti.outer << p.a1);
#pragma unroll 4
            for (uint32_t u = 0; u < 8; ++u) {
                const uint32_t e = tid + u * NTT_THREADS;
                if (e < elems) {
                    const uint32_t c = e & (C - 1), q = e >> p.log_c;
                    const uint32_t k = a ? (__brev(q) >> (32 - a)) : 0;
                    Fr v = ld_l1(lo, hi, c * (A + 1) + swz(q));
                    const uint64_t oidx = obase + c + ((uint64_t)k << (p.a1 + p.a2));
                    if (p.use_scale) v = fp_mul_lazy(v, fp_load(p.scale));
                    if (p.coset_out) {
                        const uint32_t m = (uint32_t)(oidx % 3);
                        if (m) v = fp_mul_lazy(v, zeta_pow(3 - m));  // ZETA^(-m) = ZETA^(3-m)
                    }
                    if (p.out_tw) v = fp_mul_lazy(v, fp_load(p.out_tw + oidx));   // sharded transform: omega^(rank * k2)
                    v = fp_cond_sub<FrParams, false>(v);   // leave the lazy domain: results are canonical (< p) like best_fft's
                    if (p.peer_routed) {   // ... and straight into the owner's window (peer store over NVLink)
                        Fr *w = p.peers[oidx >> p.peer_log_blk];
                        fp_store_stream(w + ((uint64_t)p.peer_rank << p.peer_log_blk) + (oidx & ((1ull << p.peer_log_blk) - 1)), v);
                    } else
                        fp_store_stream(out + oidx, v);
                }
            }
            fence_proxy_async();
            __syncthreads();
        }
        if (tid == 0 && gt + stride < p.total_tiles) issue_data(p, gt + stride, smem_u32(d), bar_d);
    }
}

// Boundary table of a non-final pass, tile-major: entry [cblk][q][c] = w_n^((j_in * bitrev_a(q)) << shift) (x scale),
// j_in = cblk * C + c, built from the two-level table lo[e & 4095] * hi[e >> 12].
__global__ void build_boundary_table_kernel(const Fr *__restrict__ lo, const Fr *__restrict__ hi, uint32_t log_n, uint32_t a, uint32_t log_c,
                                            uint32_t log_inner, uint32_t shift, const Fr *__restrict__ scale, Fr *__restrict__ out) {
    const uint64_t idx = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (idx >= (1ull << (a + log_inner))) return;
    const uint32_t c = (uint32_t)(idx & ((1u << log_c) - 1));
    const uint32_t q = (uint32_t)((idx >> log_c) & ((1u << a) - 1));
    const uint64_t cblk = idx >> (log_c + a);
    const uint64_t j_in = (cblk << log_c) + c;
    const uint64_t k = a ? (__brev(q) >> (32 - a)) : 0;
    const uint64_t e = (j_in * k) << shift;
    Fr tw = fp_load(lo + (e & ((1u << TW_LO_BITS) - 1)));
    if (log_n > TW_LO_BITS) tw = fp_mul(tw, fp_load(hi + (e >> TW_LO_BITS)));
    if (scale) tw = fp_mul(tw, fp_load(scale));
    fp_store(out + idx, tw);
}

// ---------------------------------------------------------------------------------------------------------
// host side: plans
// ---------------------------------------------------------------------------------------------------------
static const uint32_t FR_ROOT_OF_UNITY_CANON[8] = {0x60c37c9cu, 0xd34f1ed9u, 0xd39329c8u, 0x3215cf6du, 0x3dd31f74u, 0x98865ea9u, 0x166d18b7u, 0x03ddb9f5u};
static const uint32_t FR_ZETA_CANON[8] = {0xb99c90ddu, 0x8b17ea66u, 0x8d8daaa7u, 0x5bfc4108u, 0x41a91758u, 0xb3c4d79du, 0x00000000u, 0x00000000u};

Fr host_root_of_unity(uint32_t k) {
    Fr c;
    for (int i = 0; i < 8; ++i) c.l[i] = FR_ROOT_OF_UNITY_CANON[i];
    Fr w = fp_from_canonical(c);
    for (uint32_t i = k; i < 28; ++i) w = fp_sqr(w);
    return w;
}
Fr host_zeta() {
    Fr c;
    for (int i = 0; i < 8; ++i) c.l[i] = FR_ZETA_CANON[i];
    return fp_from_canonical(c);
}

static int32_t upload_powers(zkb_ctx *ctx, const Fr &w, size_t count, Fr **out) {
    std::vector<Fr> h(count);
    Fr cur = Fr::one();
    for (size_t i = 0; i < count; ++i) { h[i] = cur; cur = fp_mul(cur, w); }
    ZKB_CUDA(cudaMalloc((void **)out, count * sizeof(Fr)));
    ZKB_CUDA(cudaMemcpyAsync(*out, h.data(), count * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
    ZKB_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZKB_OK;
}

// per-pass geometry shared by the plan builder and the launcher
struct PassGeom { uint32_t a, log_inner, log_c, shift; bool is_final; };
static void pass_geometry(const NttPlan &plan, int ps, PassGeom &g) {
    uint32_t consumed = 0;
    for (int q = 0; q < ps; ++q) consumed += plan.bits[q];
    g.a = plan.bits[ps];
    g.shift = consumed;
    g.log_inner = plan.log_n - consumed - g.a;
    g.is_final = (ps == plan.npass - 1);
    uint32_t lc = NTT_TILE_BITS - g.a;                     // C * A = 2048 ...
    const uint32_t cap = g.is_final ? (plan.npass > 1 ? (uint32_t)plan.bits[0] : 0u) : g.log_inner;  // ... unless fewer columns exist
    if (lc > cap) lc = cap;
    g.log_c = lc;
}

static int32_t get_plan(zkb_ctx *ctx, uint32_t log_n, const Fr &omega, NttPlan **out) {
    std::array<uint64_t, 5> key;
    key[0] = log_n;
    for (int i = 0; i < 4; ++i) key[1 + i] = (uint64_t)omega.l[2 * i] | ((uint64_t)omega.l[2 * i + 1] << 32);
    auto it = ctx->ntt_plans.find(key);
    if (it != ctx->ntt_plans.end()) { *out = &it->second; return ZKB_OK; }

    // order check: omega^(2^log_n) == 1 and omega^(2^(log_n-1)) == -1
    {
        Fr t = omega;
        for (uint32_t i = 0; i + 1 < log_n; ++i) t = fp_sqr(t);
        if (log_n >= 1) {
            if (!(fp_add(t, Fr::one()).is_zero())) { set_error("omega does not have order 2^%u", log_n); return ZKB_ERR_ARG; }
        } else if (!(omega == Fr::one())) { set_error("omega must be 1 for log_n = 0"); return ZKB_ERR_ARG; }
    }

    NttPlan plan;
    plan.log_n = log_n;
    // factor sizes: the final pass may be as long as a tile (2^11), the others are bounded by the shared-memory budget of two
    // resident CTAs (2^9); more, shorter passes cost no extra multiplies (every pass drops its A - 1 unit twiddles, which pays
    // for the extra boundary multiply per element), only one more trip through HBM
    // ZKB_NTT_MAX_A (experiments): upper bound on every factor, e.g. 8 turns 2^20 into 7 + 7 + 6 (C >= 8 columns per tile in every pass)
    int max_final = NTT_MAX_BITS, pref_inner = NTT_PREF_INNER_BITS;
    if (const char *e = getenv("ZKB_NTT_MAX_A")) {
        const int v = atoi(e);
        if (v >= 6 && v <= NTT_MAX_BITS && 3 * v >= (int)log_n) { max_final = v; pref_inner = std::min(pref_inner, v); }
    }
    if ((int)log_n <= max_final) { plan.npass = 1; plan.bits[0] = log_n; }
    else if ((int)log_n <= pref_inner + max_final) {
        plan.npass = 2;
        plan.bits[0] = std::min<int>(pref_inner, (log_n + 1) / 2);
        plan.bits[1] = log_n - plan.bits[0];
    } else {
        const int cap = (int)log_n > 2 * pref_inner + max_final ? NTT_MAX_INNER_BITS : pref_inner;
        plan.npass = 3;
        plan.bits[0] = std::min<int>(cap, (log_n + 2) / 3);
        plan.bits[1] = std::min<int>(cap, (log_n - plan.bits[0] + 1) / 2);
        plan.bits[2] = log_n - plan.bits[0] - plan.bits[1];
    }
    if (plan.bits[plan.npass - 1] > NTT_MAX_BITS) { set_error("log_n %u exceeds the three-pass limit", log_n); return ZKB_ERR_ARG; }

    const uint32_t lo_bits = log_n < TW_LO_BITS ? log_n : TW_LO_BITS;
    ZKB_TRY(upload_powers(ctx, omega, (size_t)1 << lo_bits, &plan.tw_lo));
    if (log_n > TW_LO_BITS) {
        Fr w = omega;
        for (int i = 0; i < TW_LO_BITS; ++i) w = fp_sqr(w);
        ZKB_TRY(upload_powers(ctx, w, (size_t)1 << (log_n - TW_LO_BITS), &plan.tw_hi));
    }
    for (int ps = 0; ps < plan.npass; ++ps) {
        const int a = plan.bits[ps];
        Fr w = omega;
        for (uint32_t i = a; i < log_n; ++i) w = fp_sqr(w);  // omega^(2^(log_n - a)) : order 2^a
        ZKB_TRY(upload_powers(ctx, w, a ? ((size_t)1 << (a - 1)) : 1, &plan.loc[ps]));
    }
    // unscaled boundary tables (n entries for the first boundary, A2 * A3 for the second)
    for (int ps = 0; ps + 1 < plan.npass; ++ps) {
        PassGeom g;
        pass_geometry(plan, ps, g);
        const uint64_t entries = 1ull << (g.a + g.log_inner);
        ZKB_CUDA(cudaMalloc((void **)&plan.tw_b[ps], entries * sizeof(Fr)));
        build_boundary_table_kernel<<<(unsigned)((entries + 255) / 256), 256, 0, ctx->stream>>>(plan.tw_lo, plan.tw_hi, log_n, g.a, g.log_c, g.log_inner,
                                                                                              g.shift, nullptr, plan.tw_b[ps]);
        ctx->launches++;
    }
    ZKB_CUDA(cudaGetLastError());
    auto ins = ctx->ntt_plans.emplace(key, plan);
    *out = &ins.first->second;
    return ZKB_OK;
}

// ---- tensor maps ------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}
// 2-D view of one column for a pass with row stride S = 2^log_inner elements: dim0 = S * 4 u64 (one row of S elements), dim1 = n / S rows;
// box = one element (4 u64 = 32 B) x min(A, 256) rows
static int32_t encode_column_map(CUtensorMap *m, const Fr *base, uint32_t log_n, uint32_t log_inner, uint32_t a) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return ZKB_ERR_CUDA; }
    const cuuint64_t dims[2] = {(cuuint64_t)4 << log_inner, (cuuint64_t)1 << (log_n - log_inner)};
    const cuuint64_t strides[1] = {(cuuint64_t)32 << log_inner};
    const uint32_t A = 1u << a;
    const cuuint32_t box[2] = {4, A < NTT_BOX_ROWS ? A : NTT_BOX_ROWS};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, (void *)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) for log_n %u log_inner %u a %u", (int)r, log_n, log_inner, a); return ZKB_ERR_CUDA; }
    return ZKB_OK;
}

static uint32_t pass_smem_bytes(const PassGeom &g) {
    return NTT_HDR_BYTES + NTT_DBUF_BYTES + (g.is_final ? 0u : NTT_TW_RING_BYTES) + (g.a ? (32u << (g.a - 1)) : 32u);
}

// batch of `count` transforms: column y reads h_src[y], writes h_dst[y] (HOST arrays of device pointers; the arrays may alias,
// h_src[y] == h_dst[y] is an in-place transform).
int32_t ntt_fr_batch_device_ex(zkb_ctx *ctx, const Fr *const *h_src, Fr *const *h_dst, uint32_t count, uint32_t log_n, const Fr &omega,
                               const Fr *scale_host, int coset_zeta, const Fr *d_in_scale, const NttPeerRoute *route, cudaStream_t st);
int32_t ntt_fr_batch_device(zkb_ctx *ctx, const Fr *const *h_src, Fr *const *h_dst, uint32_t count, uint32_t log_n, const Fr &omega,
                            const Fr *scale_host, int coset_zeta, const Fr *d_in_scale, cudaStream_t st) {
    return ntt_fr_batch_device_ex(ctx, h_src, h_dst, count, log_n, omega, scale_host, coset_zeta, d_in_scale, nullptr, st);
}
int32_t ntt_fr_batch_device_ex(zkb_ctx *ctx, const Fr *const *h_src, Fr *const *h_dst, uint32_t count, uint32_t log_n, const Fr &omega,
                               const Fr *scale_host, int coset_zeta, const Fr *d_in_scale, const NttPeerRoute *route, cudaStream_t st) {
    ZKB_ARG(route == nullptr || (count == 1 && route->out_tw && route->nranks >= 1 && route->nranks <= 16));
    ZKB_ARG(log_n <= 28 && count >= 1 && h_src && h_dst);
    ZKB_ARG(coset_zeta >= 0 && coset_zeta <= 2);
    NttPlan *plan = nullptr;
    ZKB_TRY(get_plan(ctx, log_n, omega, &plan));
    if (!ctx->ntt_ready) {
        // per device (a context owns one device): opt in to the large dynamic shared-memory window, upload ZETA
        // two CTAs per SM: header + data tile + twiddle ring + <= 8 KB of local twiddles (non-final) or <= 32 KB (final, no ring)
        ZKB_CUDA(cudaFuncSetAttribute(ntt_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)(NTT_HDR_BYTES + NTT_DBUF_BYTES + NTT_TW_RING_BYTES + (32u << (NTT_MAX_INNER_BITS - 1)))));
        ZKB_CUDA(cudaFuncSetAttribute(ntt_tile_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
        Fr z = host_zeta(), z2 = fp_sqr(z);
        uint32_t h[2][8];
        for (int i = 0; i < 8; ++i) { h[0][i] = z.l[i]; h[1][i] = z2.l[i]; }
        ZKB_CUDA(cudaMemcpyToSymbol(ZETA_POW, h, sizeof(h)));
        ctx->ntt_ready = true;
    }
    const uint64_t n = 1ull << log_n;
    const int npass = plan->npass;
    Fr *scratch = nullptr;
    if (npass > 1) ZKB_TRY(scratch_get(ctx, SCR_NTT, (size_t)count * n * sizeof(Fr), (void **)&scratch));

    // scale: single pass -> multiplied at the store; otherwise folded into the last boundary table (cached per scale value)
    Fr *d_scale = nullptr;
    const Fr *last_tw = npass > 1 ? plan->tw_b[npass - 2] : nullptr;
    if (scale_host) {
        void *misc = nullptr;
        ZKB_TRY(scratch_get(ctx, SCR_MISC, sizeof(Fr), &misc));
        d_scale = (Fr *)misc;
        if (npass == 1) {
            ZKB_CUDA(cudaMemcpyAsync(d_scale, scale_host, sizeof(Fr), cudaMemcpyHostToDevice, st));
        } else {
            PassGeom g;
            pass_geometry(*plan, npass - 2, g);
            const uint64_t entries = 1ull << (g.a + g.log_inner);
            if (!plan->tw_b_scaled) ZKB_CUDA(cudaMalloc((void **)&plan->tw_b_scaled, entries * sizeof(Fr)));
            if (!plan->has_scaled || !(plan->scaled_key == *scale_host)) {
                ZKB_CUDA(cudaMemcpyAsync(d_scale, scale_host, sizeof(Fr), cudaMemcpyHostToDevice, st));
                build_boundary_table_kernel<<<(unsigned)((entries + 255) / 256), 256, 0, st>>>(plan->tw_lo, plan->tw_hi, log_n, g.a, g.log_c, g.log_inner,
                                                                                              g.shift, d_scale, plan->tw_b_scaled);
                ctx->launches++;
                plan->scaled_key = *scale_host;
                plan->has_scaled = true;
            }
            last_tw = plan->tw_b_scaled;
        }
    }

    // descriptor blob: per non-final pass `count` tensor maps, then per pass the src / dst pointer tables
    const size_t maps_bytes = (size_t)(npass - 1) * count * sizeof(CUtensorMap);
    const size_t tbl_bytes = (size_t)count * sizeof(void *);
    const size_t blob_bytes = maps_bytes + 2 * (size_t)npass * tbl_bytes;
    std::vector<uint8_t> blob(blob_bytes + 64);
    uint8_t *hb = blob.data();
    uint8_t *hb_al = hb + ((64 - ((uintptr_t)hb & 63)) & 63);   // CUtensorMap wants 64-byte alignment (also on the host side)
    uint8_t *dblob = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_NTT_DESC, blob_bytes + 64, (void **)&dblob));
    for (int ps = 0; ps < npass; ++ps) {
        PassGeom g;
        pass_geometry(*plan, ps, g);
        const Fr **srcs = (const Fr **)(hb_al + maps_bytes + (size_t)(2 * ps) * tbl_bytes);
        Fr **dsts = (Fr **)(hb_al + maps_bytes + (size_t)(2 * ps + 1) * tbl_bytes);
        for (uint32_t y = 0; y < count; ++y) {
            srcs[y] = ps == 0 ? h_src[y] : scratch + (size_t)y * n;
            dsts[y] = g.is_final ? h_dst[y] : scratch + (size_t)y * n;
            ZKB_ARG(srcs[y] != nullptr && dsts[y] != nullptr);
            if (!g.is_final) ZKB_TRY(encode_column_map((CUtensorMap *)(hb_al + ((size_t)ps * count + y) * sizeof(CUtensorMap)), srcs[y], log_n, g.log_inner, g.a));
        }
    }
    ZKB_CUDA(cudaMemcpyAsync(dblob, hb_al, blob_bytes, cudaMemcpyHostToDevice, st));

    for (int ps = 0; ps < npass; ++ps) {
        PassGeom g;
        pass_geometry(*plan, ps, g);
        PassArgs p;
        memset(&p, 0, sizeof(p));
        p.a = g.a;
        p.log_c = g.log_c;
        p.log_inner = g.log_inner;
        p.log_n = log_n;
        p.is_final = g.is_final;
        if (g.is_final && npass == 2) { p.a1 = plan->bits[0]; }
        if (g.is_final && npass == 3) { p.a1 = plan->bits[0]; p.a2 = plan->bits[1]; }
        p.coset_in = (ps == 0 && coset_zeta == 1);
        p.coset_out = (g.is_final && coset_zeta == 2);
        p.use_scale = (npass == 1 && scale_host != nullptr);
        p.has_in_scale = (ps == 0 && d_in_scale != nullptr);
        p.tiles_per_col = (uint32_t)(n >> (g.a + g.log_c));
        p.total_tiles = p.tiles_per_col * count;
        p.loc = plan->loc[ps];
        p.tw = g.is_final ? nullptr : (ps == npass - 2 ? last_tw : plan->tw_b[ps]);
        p.scale = d_scale;
        p.in_scale = d_in_scale;
        if (route && g.is_final) {
            p.out_tw = route->out_tw;
            p.peer_routed = route->routed ? 1u : 0u;
            p.peer_log_blk = route->log_blk;
            p.peer_rank = route->rank;
            for (int i = 0; i < route->nranks; ++i) p.peers[i] = route->peers[i];
        }
        p.maps = (const CUtensorMap *)(dblob + (size_t)ps * count * sizeof(CUtensorMap));
        p.src = (const Fr *const *)(dblob + maps_bytes + (size_t)(2 * ps) * tbl_bytes);
        p.dst = (Fr *const *)(dblob + maps_bytes + (size_t)(2 * ps + 1) * tbl_bytes);
        ZKB_ARG((uint64_t)p.tiles_per_col * count < (1ull << 32));
        const uint32_t max_ctas = (uint32_t)ctx->sm_count * NTT_CTAS_PER_SM;
        const uint32_t grid = p.total_tiles < max_ctas ? p.total_tiles : max_ctas;
        {
            ProfScope ps_(ctx, PROF_NTT, st);
            ntt_tile_kernel<<<grid, NTT_THREADS, pass_smem_bytes(g), st>>>(p);
        }
        ctx->launches++;
    }
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

int32_t ntt_fr_device(zkb_ctx *ctx, const Fr *src_data, Fr *data, uint32_t log_n, const Fr &omega, const Fr *scale_host, int coset_zeta,
                      const Fr *d_in_scale, cudaStream_t st) {
    return ntt_fr_batch_device(ctx, &src_data, &data, 1, log_n, omega, scale_host, coset_zeta, d_in_scale, st);
}

}  // namespace zkb

using namespace zkb;

extern "C" int32_t zkb_fr_root_of_unity(uint32_t k, uint64_t omega[4], uint64_t omega_inv[4]) {
    ZKB_ARG(k <= 28 && omega != nullptr);
    Fr w = host_root_of_unity(k);
    memcpy(omega, w.l, 32);
    if (omega_inv) {
        Fr wi = fp_inv(w);
        memcpy(omega_inv, wi.l, 32);
    }
    return ZKB_OK;
}

extern "C" int32_t zkb_ntt_fr_dev(zkb_ctx *ctx, uint64_t *data_dev, uint32_t log_n, const uint64_t omega[4], const uint64_t *scale,
                                  int32_t coset_zeta, void *stream) {
    ZKB_ARG(ctx && data_dev && omega);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    Fr w, sc;
    memcpy(w.l, omega, 32);
    if (scale) memcpy(sc.l, scale, 32);
    return ntt_fr_device(ctx, (const Fr *)data_dev, (Fr *)data_dev, log_n, w, scale ? &sc : nullptr, coset_zeta, nullptr, pick_stream(ctx, stream));
}

// `count` in-place transforms of the same size in ONE launch per pass (cols_dev: HOST array of device pointers)
extern "C" int32_t zkb_ntt_fr_batch_dev(zkb_ctx *ctx, uint64_t *const *cols_dev, uint32_t count, uint32_t log_n, const uint64_t omega[4],
                                        const uint64_t *scale, int32_t coset_zeta, void *stream) {
    ZKB_ARG(ctx && cols_dev && omega && count >= 1);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    Fr w, sc;
    memcpy(w.l, omega, 32);
    if (scale) memcpy(sc.l, scale, 32);
    cudaStream_t st = pick_stream(ctx, stream);
    // bound the scratch of multi-pass plans to ~2 GiB per launch group
    const uint64_t per = (uint64_t)32 << log_n;
    uint32_t group = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(256, (1ull << 31) / per));
    for (uint32_t done = 0; done < count; done += group) {
        const uint32_t cur = count - done < group ? count - done : group;
        ZKB_TRY(ntt_fr_batch_device(ctx, (const Fr *const *)(cols_dev + done), (Fr *const *)(cols_dev + done), cur, log_n, w, scale ? &sc : nullptr, coset_zeta,
                                    nullptr, st));
    }
    return ZKB_OK;
}

extern "C" int32_t zkb_ntt_fr_host(zkb_ctx *ctx, uint64_t *data_host, uint32_t log_n, const uint64_t omega[4], const uint64_t *scale,
                                   int32_t coset_zeta) {
    ZKB_ARG(ctx && data_host && omega && log_n <= 28);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    const size_t bytes = ((size_t)1 << log_n) * 32;
    void *d = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_HOSTIO_A, bytes, &d));
    ZKB_CUDA(cudaMemcpyAsync(d, data_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    ZKB_TRY(zkb_ntt_fr_dev(ctx, (uint64_t *)d, log_n, omega, scale, coset_zeta, ctx->stream));
    ZKB_CUDA(cudaMemcpyAsync(data_host, d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    ZKB_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZKB_OK;
}
