// msm.cu -- multi-scalar multiplication over BN254 G1 (Pippenger bucket method) for sm_90a.
//
// Replaces halo2_proofs::arithmetic::best_multiexp (halo2_proofs 1.1.0 @ e5ddf67 src/arithmetic.rs), the body of
// ParamsKZG::commit / commit_lagrange (src/poly/kzg/commitment.rs) -- every commitment of create_proof
// (circuit-benchmarks/src/super_circuit.rs:117-132).  Same contract: sum_i coeffs[i] * bases[i]; the group element is
// unique, so the normalised (affine / compressed) output is bit-identical to the CPU prover's.
//
// Design (NOT upstream's per-thread serial windows):
//   1. scalars leave Montgomery form once and are recoded into signed c-bit digits (W = ceil(255/c) windows, buckets
//      1..2^(c-1) per window) -- coalesced 32-byte loads, one thread per scalar;
//   2. a counting sort (histogram -> scan -> scatter) groups point indices by (window, |digit|): 4 bytes per
//      (point, window) pair, no 64-byte point ever moves;
//   3. the sorted (bucket-major) pair list is cut into CHUNKS of exactly 32 entries, one thread per chunk, regardless of bucket
//      boundaries: every lane of a warp performs the same 32 mixed XYZZ additions (8M + 2S, bases gathered by index, a base is
//      two 32-byte sectors) and flushes one partial sum per bucket it crossed; the partials of a bucket are then reduced by
//      levels of <= 64-entry tasks.  No step between the digit kernels and the final window sums returns to the host: task
//      arrays are sized from bounds, and the reduction levels that turn out to be unnecessary exit on a device-side flag;
//   4. each window's buckets are reduced by segmented running sums (all windows and segments in parallel), the
//      segment partials are tree-reduced per window, and the W window sums are combined by Horner doubling.
//   Work is dominated by n*W mixed additions = n*W*10 Fq multiplies: bound by the integer-multiply pipe.
#include "common.cuh"
#include "digits.cuh"
#include <string.h>
#include <algorithm>

namespace zkb {

struct MsmCfg {
    uint32_t c;         // window bits
    uint32_t windows;   // W
    uint32_t half;      // 2^(c-1) buckets per window
    uint32_t shifted;   // 1: bases array holds W copies, copy w = 2^(c w) * P_i -> ONE bucket set per column, no Horner
    uint32_t n32;       // points per copy (shifted mode)
};

// signed-digit recoding of a canonical scalar (8 x u32) by signed_digit (digits.cuh); carry chain from window 0
// mode 0: histogram; mode 1: scatter
template <int MODE>
__global__ void msm_digits_kernel(const Fr *const *__restrict__ scalar_cols, uint64_t n, MsmCfg m, uint32_t *__restrict__ counts,
                                  uint32_t *__restrict__ cursors, uint32_t *__restrict__ sorted) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t col_base = blockIdx.y * (m.shifted ? m.half : m.windows * m.half);  // one bucket set per column of the batch
    const Fr s = fp_to_canonical(fp_load(scalar_cols[blockIdx.y] + i));
    uint32_t carry = 0;
    for (uint32_t w = 0; w < m.windows; ++w) {
        uint32_t neg;
        const uint32_t d = signed_digit(s.l, w * m.c, m.c, m.half, carry, neg);
        if (d != 0) {
            const uint32_t b = col_base + (m.shifted ? 0u : w * m.half) + (d - 1);
            if (MODE == 0) atomicAdd(&counts[b], 1u);
            else {
                const uint32_t pos = atomicAdd(&cursors[b], 1u);
                sorted[pos] = ((uint32_t)i + (m.shifted ? w * m.n32 : 0u)) | (neg << 31);
            }
        }
    }
}

// ---- exclusive scan of u32 (three small kernels) -----------------------------------------------------------
constexpr int SCAN_T = 512, SCAN_PER = 4, SCAN_BLK = SCAN_T * SCAN_PER;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *total, uint32_t *sm /* SCAN_T/32 */) {
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sm[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint32_t t = lane < (blockDim.x >> 5) ? sm[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += y;
        }
        sm[lane] = t;
    }
    __syncthreads();
    const uint32_t base = wid ? sm[wid - 1] : 0;
    *total = sm[(blockDim.x >> 5) - 1];
    return base + x - v;
}

// GATED: the scans of the bucket accumulation's levels >= 1.  They do nothing unless the device-side MsmState says a level is
// needed (st_words[0] = maxlen > 1), and write toff[cur ^ 1] (st_words[1] = cur: out0 when cur == 1, out1 when cur == 0).
// Plain: out0.
template <bool GATED>
__global__ void scan_blocks_kernel(const uint32_t *__restrict__ in, uint32_t *const out0, uint32_t *const out1, const uint32_t *st_words,
                                   uint32_t *__restrict__ block_sums, uint64_t n) {
    if (GATED && st_words[0] <= 1) return;
    uint32_t *out = GATED ? (st_words[1] ? out0 : out1) : out0;
    __shared__ uint32_t sm[32];
    const uint64_t base = (uint64_t)blockIdx.x * SCAN_BLK + (uint64_t)threadIdx.x * SCAN_PER;
    uint32_t v[SCAN_PER], sum = 0;
#pragma unroll
    for (int k = 0; k < SCAN_PER; ++k) { v[k] = base + k < n ? in[base + k] : 0; sum += v[k]; }
    uint32_t total;
    uint32_t ex = block_exclusive_scan(sum, &total, sm);
#pragma unroll
    for (int k = 0; k < SCAN_PER; ++k) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}
template <bool GATED>
__global__ void scan_sums_kernel(uint32_t *__restrict__ block_sums, uint32_t nblocks, uint32_t *const out0, uint32_t *const out1,
                                 const uint32_t *st_words, uint64_t n) {
    // single block; serial over chunks of SCAN_T
    if (GATED && st_words[0] <= 1) return;
    uint32_t *out = GATED ? (st_words[1] ? out0 : out1) : out0;
    __shared__ uint32_t sm[32];
    uint32_t running = 0;
    for (uint32_t s = 0; s < nblocks; s += SCAN_T) {
        const uint32_t idx = s + threadIdx.x;
        const uint32_t v = idx < nblocks ? block_sums[idx] : 0;
        uint32_t total;
        const uint32_t ex = block_exclusive_scan(v, &total, sm);
        if (idx < nblocks) block_sums[idx] = running + ex;
        running += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) out[n] = running;
}
template <bool GATED>
__global__ void scan_add_kernel(uint32_t *const out0, uint32_t *const out1, const uint32_t *st_words, const uint32_t *__restrict__ block_sums,
                                uint64_t n) {
    if (GATED && st_words[0] <= 1) return;
    uint32_t *out = GATED ? (st_words[1] ? out0 : out1) : out0;
    const uint64_t base = (uint64_t)blockIdx.x * SCAN_BLK + (uint64_t)threadIdx.x * SCAN_PER;
    const uint32_t add = block_sums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_PER; ++k)
        if (base + k < n) out[base + k] += add;
}

// out[0..n) = exclusive scan of in, out[n] = total (out = out0 unless GATED, see above).  tmp: ceil(n / SCAN_BLK) u32
template <bool GATED>
static void exclusive_scan_u32(zkb_ctx *ctx, const uint32_t *in, uint32_t *out0, uint32_t *out1, const uint32_t *st_words, uint64_t n,
                               uint32_t *tmp, cudaStream_t st) {
    const uint32_t nblocks = (uint32_t)((n + SCAN_BLK - 1) / SCAN_BLK);
    scan_blocks_kernel<GATED><<<nblocks, SCAN_T, 0, st>>>(in, out0, out1, st_words, tmp, n);
    scan_sums_kernel<GATED><<<1, SCAN_T, 0, st>>>(tmp, nblocks, out0, out1, st_words, n);
    scan_add_kernel<GATED><<<nblocks, SCAN_T, 0, st>>>(out0, out1, st_words, tmp, n);
    ctx->launches += 3;
}

// ---- bucket accumulation: equal chunks of the sorted pair list, then levels of <= ACC_CH-entry tasks per bucket -----------
// Witness columns are highly structured (most scalars are 0, 1 or small), so bucket sizes are wildly skewed, and even for
// random scalars the lengths inside a warp differ (Poisson): one thread per bucket (or per ceil(len/64) task) leaves ~30 % of
// the lanes idle.  Level 0 therefore cuts the SORTED PAIR LIST into chunks of exactly CHUNK entries: chunk t adds entries
// [CHUNK t, CHUNK (t+1)) and flushes a partial whenever it crosses a bucket boundary; bucket b (entries [off_b, off_{b+1}))
// receives one partial from each chunk it intersects, at slot toff[b] + (t - off_b / CHUNK).  The following levels add the XYZZ
// partials of a bucket in tasks of <= ACC_CH until every bucket holds one value.  Task -> bucket by binary search in the
// exclusive scan of the per-bucket task counts.
constexpr uint32_t ACC_CH = 64;
constexpr uint32_t CHUNK = 32;

// device-side pipeline state: lets the reduction levels run (or exit immediately) without a round trip to the host
struct MsmState {
    uint32_t maxlen;      // longest partial list of any bucket after the last executed level
    uint32_t cur;         // which of the two partial / task-offset arrays holds the current lists
    uint32_t levels_run;
    uint32_t pad;
    uint64_t extra_adds;  // additions performed by levels >= 1
};

// number of chunks bucket b intersects (0 for an empty bucket) + the maximum over all buckets
__global__ void chunk_count_kernel(const uint32_t *__restrict__ seg_off, uint32_t nseg, uint32_t *__restrict__ tcount, MsmState *st) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t cnt = 0;
    if (b < nseg) {
        const uint32_t lo = seg_off[b], hi = seg_off[b + 1];
        cnt = hi > lo ? (hi - 1) / CHUNK - lo / CHUNK + 1 : 0;
        tcount[b] = cnt;
    }
    for (int o = 16; o > 0; o >>= 1) {
        const uint32_t y = __shfl_down_sync(0xffffffffu, cnt, o);
        cnt = y > cnt ? y : cnt;
    }
    if ((threadIdx.x & 31) == 0 && cnt > 1) atomicMax(&st->maxlen, cnt);
}
__device__ __forceinline__ uint32_t find_segment(const uint32_t *__restrict__ toff, uint32_t nseg, uint32_t t) {
    // largest b with toff[b] <= t   (toff has nseg + 1 entries, non-decreasing)
    uint32_t lo = 0, hi = nseg;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (toff[mid] <= t) lo = mid; else hi = mid;
    }
    return lo;
}
__global__ void __launch_bounds__(128) msm_acc_chunk_kernel(const G1Affine *__restrict__ bases, const uint32_t *__restrict__ seg_off,
                                                           const uint32_t *__restrict__ sorted, const uint32_t *__restrict__ toff,
                                                           uint32_t nseg, G1Xyzz *__restrict__ part) {
    const uint32_t total = seg_off[nseg];
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t beg = t * CHUNK;
    if (beg >= total) return;
    const uint32_t end = beg + CHUNK < total ? beg + CHUNK : total;
    uint32_t b = find_segment(seg_off, nseg, beg);   // the (non-empty) bucket holding entry `beg`
    uint32_t b_first = seg_off[b], next = seg_off[b + 1];
    G1Xyzz acc = G1Xyzz::identity();
    uint32_t e = sorted[beg];
    G1Affine p = g1_load_affine(bases + (e & 0x7fffffffu));
    for (uint32_t k = beg; k < end; ++k) {
        if (k == next) {
            g1_store_xyzz(part + toff[b] + (t - b_first / CHUNK), acc);
            acc = G1Xyzz::identity();
            do { ++b; next = seg_off[b + 1]; } while (next <= k);
            b_first = seg_off[b];
        }
        // fetch the next entry's base while this addition runs
        const uint32_t e_cur = e;
        const G1Affine p_cur = p;
        if (k + 1 < end) {
            e = sorted[k + 1];
            p = g1_load_affine(bases + (e & 0x7fffffffu));
        }
        g1_add_mixed(acc, (e_cur >> 31) ? g1_neg(p_cur) : p_cur);
    }
    g1_store_xyzz(part + toff[b] + (t - b_first / CHUNK), acc);
}

// ---- levels >= 1 (all gated on the device-side state: a level that is not needed costs one empty launch per kernel) ----------
struct LevelBufs {
    uint32_t *toff[2];      // per-bucket offsets of the partial lists (nseg + 1 entries each)
    G1Xyzz *part[2];
    uint32_t *tcount;
    MsmState *st;
};
__global__ void level_task_count_kernel(LevelBufs L, uint32_t nseg) {
    if (L.st->maxlen <= 1) return;
    const uint32_t *seg_off = L.toff[L.st->cur];
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nseg) return;
    const uint32_t len = seg_off[b + 1] - seg_off[b];
    L.tcount[b] = (len + ACC_CH - 1) / ACC_CH;
}
__global__ void __launch_bounds__(128) msm_acc_levelN_kernel(LevelBufs L, uint32_t nseg) {
    if (L.st->maxlen <= 1) return;
    const uint32_t cur = L.st->cur;
    const uint32_t *__restrict__ seg_off = L.toff[cur];
    const uint32_t *__restrict__ toff = L.toff[cur ^ 1];
    const G1Xyzz *__restrict__ in = L.part[cur];
    G1Xyzz *__restrict__ part = L.part[cur ^ 1];
    const uint32_t ntasks = toff[nseg];
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < ntasks; t += gridDim.x * blockDim.x) {
        const uint32_t b = find_segment(toff, nseg, t);
        const uint32_t beg = seg_off[b] + (t - toff[b]) * ACC_CH;
        const uint32_t lim = seg_off[b + 1];
        const uint32_t end = beg + ACC_CH < lim ? beg + ACC_CH : lim;
        G1Xyzz acc = g1_load_xyzz(in + beg);
        for (uint32_t k = beg + 1; k < end; ++k) g1_add(acc, g1_load_xyzz(in + k));
        g1_store_xyzz(part + t, acc);
    }
}
__global__ void level_advance_kernel(LevelBufs L, uint32_t nseg) {
    MsmState *st = L.st;
    if (st->maxlen <= 1) return;
    const uint32_t cur = st->cur;
    st->extra_adds += L.toff[cur][nseg];   // entries consumed by this level (one addition each, minus one per task)
    st->maxlen = (st->maxlen + ACC_CH - 1) / ACC_CH;
    st->cur = cur ^ 1;
    st->levels_run++;
}
// buckets[b] = the single remaining partial of segment b (or the identity for an empty bucket)
__global__ void msm_gather_buckets_kernel(LevelBufs L, uint32_t nseg, G1Xyzz *__restrict__ buckets) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nseg) return;
    const uint32_t cur = L.st->cur;
    const uint32_t *seg_off = L.toff[cur];
    const uint32_t beg = seg_off[b], end = seg_off[b + 1];
    g1_store_xyzz(buckets + b, end > beg ? g1_load_xyzz(L.part[cur] + beg) : G1Xyzz::identity());
}

// ---- window reduction: sum_j j * in[j] (0-based weights) by levels of length-L running sums ----------------------------
// level kernel, thread (w, s): segment s of window w (count entries per window):
//   acc_out = sum_{j=1}^{len-1} j * in[s*L + j],   run_out = sum_j in[s*L + j]
// so  sum_j j*in[j] = sum_s acc_s + L * sum_s s * run_s  -> recurse on the `run` array; no per-thread scalar multiplication.
__global__ void __launch_bounds__(128) msm_wsum_level_kernel(const G1Xyzz *__restrict__ in, uint32_t count, uint32_t log_l, uint32_t windows,
                                                            G1Xyzz *__restrict__ acc_out, G1Xyzz *__restrict__ run_out) {
    const uint32_t L = 1u << log_l;
    const uint32_t segs = (count + L - 1) >> log_l;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= windows * segs) return;
    const uint32_t w = t / segs, s = t % segs;
    const uint32_t base = s << log_l;
    const uint32_t len = count - base < L ? count - base : L;
    const G1Xyzz *p = in + (size_t)w * count + base;
    G1Xyzz running = G1Xyzz::identity(), acc = G1Xyzz::identity();
    for (int j = (int)len - 1; j >= 1; --j) {
        g1_add(running, g1_load_xyzz(p + j));
        g1_add(acc, running);
    }
    g1_add(running, g1_load_xyzz(p));
    g1_store_xyzz(acc_out + t, acc);
    g1_store_xyzz(run_out + t, running);
}
// plain sums of `segs` entries per window (one block per window); result ADDED into / written to out[w]
__global__ void __launch_bounds__(256) msm_window_sum_kernel(const G1Xyzz *__restrict__ partials, G1Xyzz *__restrict__ window_sums, uint32_t segs) {
    extern __shared__ uint4 sm4[];
    G1Xyzz *sm = reinterpret_cast<G1Xyzz *>(sm4);
    const uint32_t w = blockIdx.x;
    G1Xyzz acc = G1Xyzz::identity();
    for (uint32_t s = threadIdx.x; s < segs; s += blockDim.x) g1_add(acc, g1_load_xyzz(partials + (size_t)w * segs + s));
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (uint32_t o = blockDim.x >> 1; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            G1Xyzz a = sm[threadIdx.x];
            g1_add(a, sm[threadIdx.x + o]);
            sm[threadIdx.x] = a;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) g1_store_xyzz(window_sums + w, sm[0]);
}
// per window: result = S_all + T0, T0 = S(acc_1) + 2^l (S(acc_2) + 2^l (S(acc_3) + ...)); level sums laid out [level][window]
__global__ void msm_window_combine_kernel(const G1Xyzz *__restrict__ level_sums, const G1Xyzz *__restrict__ all_sum, uint32_t nlevels,
                                          uint32_t log_l, uint32_t windows, G1Xyzz *__restrict__ out) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= windows) return;
    G1Xyzz r = g1_load_xyzz(level_sums + (size_t)(nlevels - 1) * windows + w);
    for (int lv = (int)nlevels - 2; lv >= 0; --lv) {
        for (uint32_t d = 0; d < log_l; ++d) r = g1_dbl(r);
        g1_add(r, g1_load_xyzz(level_sums + (size_t)lv * windows + w));
    }
    g1_add(r, g1_load_xyzz(all_sum + w));
    g1_store_xyzz(out + w, r);
}

// ---- window-shifted bases: out[i] = 2^c * in[i] (affine in, affine out) --------------------------------------------------
__global__ void __launch_bounds__(128) msm_shift_bases_kernel(const G1Affine *__restrict__ in, G1Affine *__restrict__ out, uint64_t n, uint32_t c) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1Xyzz p = G1Xyzz::from_affine(g1_load_affine(in + i));
    for (uint32_t k = 0; k < c; ++k) p = g1_dbl(p);
    g1_store_affine(out + i, g1_to_affine(p));
}

// ---- fixed-base scalar multiplication: out[i] = [s_i] base (affine) ------------------------------------------
// Plain double-and-add with one inversion per point: the independent reference the SRS setup's comb (setup.cu) is tested against,
// and the source of distinct benchmark bases.
__global__ void __launch_bounds__(128) fixed_base_mul_kernel(G1Affine base, const Fr *__restrict__ scalars, uint64_t n, G1Affine *__restrict__ out) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr s = fp_to_canonical(fp_load(scalars + i));
    G1Xyzz acc = G1Xyzz::identity();
    for (int bit = 253; bit >= 0; --bit) {
        acc = g1_dbl(acc);
        if ((s.l[bit >> 5] >> (bit & 31)) & 1) g1_add_mixed(acc, base);
    }
    g1_store_affine(out + i, g1_to_affine(acc));
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static uint32_t log2_floor(uint64_t n) {
    uint32_t lg = 0;
    while ((1ull << (lg + 1)) <= n) ++lg;
    return lg;
}

// window bits used with precomputed shifted bases for n points (0 = not supported at this size)
uint32_t msm_shift_window_bits(uint64_t n) {
    const uint32_t lg = log2_floor(n);
    if (lg < 10 || lg > 22) return 0;
    return lg > 20 ? 20 : lg;
}
uint32_t msm_shift_copies(uint64_t n) {
    const uint32_t c = msm_shift_window_bits(n);
    return c ? (255 + c - 1) / c : 0;
}
// out: copies x n affine points, copy w = 2^(c w) * bases
int32_t msm_build_shifted_bases(zkb_ctx *ctx, const G1Affine *bases, uint64_t n, G1Affine *out, cudaStream_t st) {
    const uint32_t c = msm_shift_window_bits(n), copies = msm_shift_copies(n);
    ZKB_ARG(c != 0);
    ZKB_CUDA(cudaMemcpyAsync(out, bases, n * sizeof(G1Affine), cudaMemcpyDeviceToDevice, st));
    for (uint32_t w = 1; w < copies; ++w) {
        msm_shift_bases_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(out + (size_t)(w - 1) * n, out + (size_t)w * n, n, c);
        ctx->launches++;
    }
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

// window configuration for n points: c = log2(n) - 4 within [3, 20]; against shifted bases c = msm_shift_window_bits(n), which is
// 0 where no copies exist
static MsmCfg msm_cfg(uint64_t n, bool shifted) {
    MsmCfg m = {};
    m.c = shifted ? msm_shift_window_bits(n) : (uint32_t)std::clamp((int)log2_floor(n) - 4, 3, 20);
    if (m.c) {
        m.windows = (255 + m.c - 1) / m.c;
        m.half = 1u << (m.c - 1);
    }
    m.shifted = shifted;
    m.n32 = shifted ? (uint32_t)n : 0;
    return m;
}

uint32_t msm_max_batch(uint64_t n) {
    if (n == 0) return 64;
    uint64_t b = (1ull << 28) / (n * msm_cfg(n, false).windows);
    const MsmCfg s = msm_cfg(n, true);
    if (s.c) {  // shifted mode: half * batch buckets of 128 B (+ partials): keep the bucket arrays under ~2 GiB
        const uint64_t bb = (1ull << 31) / ((uint64_t)s.half * 3 * sizeof(G1Xyzz));
        if (bb < b) b = bb;
    }
    return (uint32_t)std::clamp<uint64_t>(b, 1, 64);
}

// ---- one pass: `batch` MSMs over the same bases --------------------------------------------------------------------------
// Everything a pass allocates is sized on the host from bounds, so no count returns from the device before the result does.
// tests/msm_model.py (msm_cfg, msm_max_batch, level_bound, scratch, arg_failures) restates these numbers.
struct MsmPlan {
    MsmCfg m;
    uint64_t n, pairs;     // pairs: (point, window) pairs of the pass
    uint32_t batch;
    uint32_t sets;         // bucket sets (reduction windows) per column: 1 against shifted bases, W otherwise
    uint32_t wred;         // reduction windows of the pass: sets x batch
    uint32_t nbuckets;     // wred x half
    uint32_t acc_levels;   // gated accumulation levels >= 1: enough for the partials of the fullest possible bucket
    uint32_t log_l;        // window reduction: segments of 2^log_l buckets ...
    uint32_t nlevels;      // ... reduced in this many levels
    size_t level_entries;  // G1Xyzz written by the window-reduction levels (acc and run outputs)
    size_t part0_n;        // bound of the level-0 partials: one per chunk plus one per bucket
    size_t part1_n;        // bound of every later level's partials: previous / ACC_CH plus one per bucket
    // scratch A, bytes: counts | offsets (+1) | cursors | tcount | toff[0] (+1) | toff[1] (+1), at k * cnt_bytes, then the
    // scan tmp at a_scan_tmp and the MsmState at a_state
    size_t cnt_bytes, a_scan_tmp, a_state, a_bytes;
    size_t b_bytes;        // scratch B: the sorted pair list, 4 B per pair
    // scratch C, bytes: part[0] at 0 | part[1] | buckets | window-reduction levels | level sums | all-bucket sums | window results
    size_t c_part1, c_buckets, c_lvl, c_lvl_sums, c_all_sum, c_wres, c_bytes;
};

// shifted: against msm_shift_copies(n) x n bases built by msm_build_shifted_bases.  Refuses what the 32-bit pair list and bucket
// indices cannot hold.
static int32_t msm_plan(uint64_t n, uint32_t batch, bool shifted, MsmPlan *out) {
    ZKB_ARG(n < (1ull << 31) && batch >= 1);
    MsmPlan p = {};
    p.m = msm_cfg(n, shifted);
    ZKB_ARG(p.m.c != 0);
    ZKB_ARG(!shifted || (uint64_t)p.m.windows * n < (1ull << 31));
    p.n = n;
    p.batch = batch;
    p.sets = shifted ? 1 : p.m.windows;
    p.pairs = n * p.m.windows * batch;
    ZKB_ARG(p.pairs < (1ull << 32) && (uint64_t)batch * p.sets * p.m.half < (1ull << 31));
    p.wred = p.sets * batch;
    p.nbuckets = p.wred * p.m.half;
    for (uint64_t bound = (n * (shifted ? p.m.windows : 1) + CHUNK - 1) / CHUNK + 1; bound > 1; bound = (bound + ACC_CH - 1) / ACC_CH)
        p.acc_levels++;
    // short window-reduction segments when a single column would otherwise leave the SMs empty; c >= 3, so at least one level
    p.log_l = 5;
    while (p.log_l > 3 && (uint64_t)p.wred * (p.m.half >> p.log_l) < 32768) --p.log_l;
    for (uint32_t cnt = p.m.half; cnt > 1; p.nlevels++) {
        cnt = (cnt + (1u << p.log_l) - 1) >> p.log_l;
        p.level_entries += 2ull * cnt * p.wred;
    }
    p.part0_n = (size_t)((p.pairs + CHUNK - 1) / CHUNK) + p.nbuckets + 1;
    p.part1_n = p.part0_n / ACC_CH + p.nbuckets + 1;
    ZKB_ARG(p.part0_n < (1ull << 32));

    p.cnt_bytes = align_up((size_t)(p.nbuckets + 2) * 4, 256);
    p.a_scan_tmp = 6 * p.cnt_bytes;
    p.a_state = p.a_scan_tmp + align_up(((size_t)p.nbuckets / SCAN_BLK + 2) * 4, 256);
    p.a_bytes = p.a_state + 256;
    p.b_bytes = p.pairs * 4;
    p.c_part1 = p.part0_n * sizeof(G1Xyzz);
    p.c_buckets = p.c_part1 + p.part1_n * sizeof(G1Xyzz);
    p.c_lvl = p.c_buckets + (size_t)p.nbuckets * sizeof(G1Xyzz);
    p.c_lvl_sums = p.c_lvl + p.level_entries * sizeof(G1Xyzz);
    p.c_all_sum = p.c_lvl_sums + (size_t)p.nlevels * p.wred * sizeof(G1Xyzz);
    p.c_wres = p.c_all_sum + (size_t)p.wred * sizeof(G1Xyzz);
    p.c_bytes = p.c_wres + (size_t)p.wred * sizeof(G1Xyzz);
    *out = p;
    return ZKB_OK;
}

// the plan's arrays in the context's scratch arenas
struct MsmBufs {
    uint32_t *counts, *offsets, *cursors, *tcount, *toff[2], *scan_tmp, *sorted;
    MsmState *state;
    G1Xyzz *part[2], *buckets, *lvl, *lvl_sums, *all_sum, *wres;
};
static int32_t msm_scratch(zkb_ctx *ctx, const MsmPlan &p, MsmBufs *b) {
    uint8_t *A = nullptr, *B = nullptr, *C = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_MSM_A, p.a_bytes, (void **)&A));
    ZKB_TRY(scratch_get(ctx, SCR_MSM_B, p.b_bytes, (void **)&B));
    ZKB_TRY(scratch_get(ctx, SCR_MSM_C, p.c_bytes, (void **)&C));
    auto a = [&](int k) { return (uint32_t *)(A + k * p.cnt_bytes); };
    auto c = [&](size_t off) { return (G1Xyzz *)(C + off); };
    b->counts = a(0), b->offsets = a(1), b->cursors = a(2), b->tcount = a(3), b->toff[0] = a(4), b->toff[1] = a(5);
    b->scan_tmp = (uint32_t *)(A + p.a_scan_tmp);
    b->state = (MsmState *)(A + p.a_state);
    b->sorted = (uint32_t *)B;
    b->part[0] = c(0), b->part[1] = c(p.c_part1), b->buckets = c(p.c_buckets), b->lvl = c(p.c_lvl), b->lvl_sums = c(p.c_lvl_sums);
    b->all_sum = c(p.c_all_sum), b->wres = c(p.c_wres);
    return ZKB_OK;
}

// counting sort of the (point, window) pairs by bucket: histogram, scan, scatter
static int32_t msm_sort(zkb_ctx *ctx, const MsmPlan &p, const MsmBufs &b, const Fr *const *d_cols, cudaStream_t st) {
    ZKB_CUDA(cudaMemsetAsync(b.counts, 0, p.cnt_bytes, st));
    const dim3 grid((unsigned)((p.n + 255) / 256), p.batch);
    msm_digits_kernel<0><<<grid, 256, 0, st>>>(d_cols, p.n, p.m, b.counts, nullptr, nullptr);
    exclusive_scan_u32<false>(ctx, b.counts, b.offsets, nullptr, nullptr, p.nbuckets, b.scan_tmp, st);
    ZKB_CUDA(cudaMemcpyAsync(b.cursors, b.offsets, (size_t)p.nbuckets * 4, cudaMemcpyDeviceToDevice, st));
    msm_digits_kernel<1><<<grid, 256, 0, st>>>(d_cols, p.n, p.m, nullptr, b.cursors, b.sorted);
    ctx->launches += 2;
    return ZKB_OK;
}

// bucket accumulation: level 0 over the 32-entry chunks of the sorted list, the gated levels >= 1, then one value per bucket
static int32_t msm_accumulate(zkb_ctx *ctx, const MsmPlan &p, const MsmBufs &b, const G1Affine *bases, cudaStream_t st) {
    ZKB_CUDA(cudaMemsetAsync(b.state, 0, sizeof(MsmState), st));
    const unsigned bb = (p.nbuckets + 255) / 256;
    chunk_count_kernel<<<bb, 256, 0, st>>>(b.offsets, p.nbuckets, b.tcount, b.state);
    exclusive_scan_u32<false>(ctx, b.tcount, b.toff[0], nullptr, nullptr, p.nbuckets, b.scan_tmp, st);
    {   // one thread per chunk (grid from the bound; surplus threads exit on the device-side total)
        const uint64_t max_chunks = (p.pairs + CHUNK - 1) / CHUNK;
        ProfScope ps_(ctx, PROF_MSM_ACC, st);
        msm_acc_chunk_kernel<<<(unsigned)((max_chunks + 127) / 128), 128, 0, st>>>(bases, b.offsets, b.sorted, b.toff[0], p.nbuckets, b.part[0]);
    }
    ctx->launches += 2;
    // each level >= 1 exits at once when the lists are already single
    const LevelBufs L = {{b.toff[0], b.toff[1]}, {b.part[0], b.part[1]}, b.tcount, b.state};
    const unsigned lv_blocks = (unsigned)std::min<uint64_t>((p.part0_n / ACC_CH + p.nbuckets + 127) / 128, (uint64_t)ctx->sm_count * 32);
    for (uint32_t lv = 0; lv < p.acc_levels; ++lv) {
        level_task_count_kernel<<<bb, 256, 0, st>>>(L, p.nbuckets);
        exclusive_scan_u32<true>(ctx, b.tcount, b.toff[0], b.toff[1], (const uint32_t *)b.state, p.nbuckets, b.scan_tmp, st);
        msm_acc_levelN_kernel<<<lv_blocks, 128, 0, st>>>(L, p.nbuckets);
        level_advance_kernel<<<1, 1, 0, st>>>(L, p.nbuckets);
        ctx->launches += 3;
    }
    msm_gather_buckets_kernel<<<bb, 256, 0, st>>>(L, p.nbuckets, b.buckets);
    ctx->launches++;
    return ZKB_OK;
}

// window reduction: per reduction window sum_j j * bucket_j by levels of running sums, then the combine
static int32_t msm_reduce_windows(zkb_ctx *ctx, const MsmPlan &p, const MsmBufs &b, cudaStream_t st) {
    const uint32_t W = p.wred;
    const G1Xyzz *in = b.buckets;
    uint32_t count = p.m.half;
    G1Xyzz *out = b.lvl;
    for (uint32_t lv = 0; lv < p.nlevels; ++lv) {
        const uint32_t segs = (count + (1u << p.log_l) - 1) >> p.log_l;
        G1Xyzz *acc_out = out, *run_out = out + (size_t)segs * W;
        msm_wsum_level_kernel<<<(W * segs + 127) / 128, 128, 0, st>>>(in, count, p.log_l, W, acc_out, run_out);
        uint32_t wt = 32;
        while (wt < segs && wt < 256) wt <<= 1;
        msm_window_sum_kernel<<<W, wt, wt * sizeof(G1Xyzz), st>>>(acc_out, b.lvl_sums + (size_t)lv * W, segs);
        ctx->launches += 2;
        in = run_out;
        count = segs;
        out += 2ull * segs * W;
    }
    // count == 1 now: the last level's run_out[w] is the sum of all buckets of window w
    ZKB_CUDA(cudaMemcpyAsync(b.all_sum, in, (size_t)W * sizeof(G1Xyzz), cudaMemcpyDeviceToDevice, st));
    msm_window_combine_kernel<<<(W + 31) / 32, 32, 0, st>>>(b.lvl_sums, b.all_sum, p.nlevels, p.log_l, W, b.wres);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

// on the host: Horner over each column's window sums (W * c doublings + W additions of single points), and the counters
static int32_t msm_finish(zkb_ctx *ctx, const MsmPlan &p, const MsmBufs &b, G1Affine *out_host, cudaStream_t st) {
    std::vector<G1Xyzz> h(p.wred);
    MsmState h_state;
    uint32_t total_pairs = 0;
    ZKB_CUDA(cudaMemcpyAsync(h.data(), b.wres, p.wred * sizeof(G1Xyzz), cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaMemcpyAsync(&h_state, b.state, sizeof(MsmState), cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaMemcpyAsync(&total_pairs, b.offsets + p.nbuckets, 4, cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaStreamSynchronize(st));   // the ONLY synchronisation of an MSM: its result is needed on the host (transcript)
    for (uint32_t col = 0; col < p.batch; ++col) {
        const G1Xyzz *hw = h.data() + (size_t)col * p.sets;
        G1Xyzz acc = hw[p.sets - 1];
        for (int w = (int)p.sets - 2; w >= 0; --w) {
            for (uint32_t k = 0; k < p.m.c; ++k) acc = g1_dbl(acc);
            g1_add(acc, hw[w]);
        }
        out_host[col] = g1_to_affine(acc);
    }
    ctx->msm_last_adds = (uint64_t)total_pairs + h_state.extra_adds + 2ull * p.nbuckets;
    ctx->msm_last_levels = h_state.levels_run;
    return ZKB_OK;
}

// d_cols: DEVICE array of `batch` device pointers
static int32_t msm_pass(zkb_ctx *ctx, const Fr *const *d_cols, uint32_t batch, const G1Affine *bases, uint64_t n, G1Affine *out_host,
                        bool shifted, cudaStream_t st) {
    MsmPlan p;
    MsmBufs b;
    ZKB_TRY(msm_plan(n, batch, shifted, &p));
    ZKB_TRY(msm_scratch(ctx, p, &b));
    ZKB_TRY(msm_sort(ctx, p, b, d_cols, st));
    ZKB_TRY(msm_accumulate(ctx, p, b, bases, st));
    ZKB_TRY(msm_reduce_windows(ctx, p, b, st));
    return msm_finish(ctx, p, b, out_host, st);
}

int32_t msm_g1_columns(zkb_ctx *ctx, const Fr *const *h_cols, uint32_t count, const G1Affine *bases, uint64_t n, G1Affine *out_host,
                       bool shifted, cudaStream_t st) {
    if (n == 0) {   // msm_last_levels keeps the previous MSM's value
        memset(out_host, 0, sizeof(G1Affine) * count);
        ctx->msm_last_adds = 0;
        return ZKB_OK;
    }
    const uint32_t maxb = msm_max_batch(n);
    const Fr **d_tbl = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_MSM_TBL, 64 * sizeof(Fr *), (void **)&d_tbl));
    for (uint32_t done = 0; done < count; done += maxb) {
        const uint32_t cur = std::min(count - done, maxb);
        ZKB_CUDA(cudaMemcpyAsync(d_tbl, h_cols + done, cur * sizeof(Fr *), cudaMemcpyHostToDevice, st));
        ZKB_TRY(msm_pass(ctx, d_tbl, cur, bases, n, out_host + done, shifted, st));
    }
    return ZKB_OK;
}

int32_t msm_g1_device(zkb_ctx *ctx, const Fr *scalars, const G1Affine *bases, uint64_t n, G1Affine *out_affine_host, cudaStream_t st) {
    return msm_g1_columns(ctx, &scalars, 1, bases, n, out_affine_host, false, st);
}

void g1_emit(const G1Affine &r, uint64_t out_affine[8], uint64_t *out_jacobian, uint8_t *out_compressed) {
    memcpy(out_affine, &r, 64);
    if (out_jacobian) {
        memcpy(out_jacobian, &r, 64);
        Fq z = r.is_identity() ? Fq::zero() : Fq::one();  // identity = (0, 0, 0), any z = 0 point is the identity
        memcpy(out_jacobian + 8, &z, 32);
    }
    if (out_compressed) g1_compress(r, out_compressed);
}

}  // namespace zkb
using namespace zkb;

extern "C" int32_t zkb_msm_g1_dev(zkb_ctx *ctx, const uint64_t *scalars_dev, const uint64_t *bases_dev, uint64_t n, uint64_t out_affine[8],
                                  uint64_t *out_jacobian, uint8_t *out_compressed, void *stream) {
    ZKB_ARG(ctx && out_affine && (n == 0 || (scalars_dev && bases_dev)));
    ZKB_CUDA(cudaSetDevice(ctx->device));
    G1Affine r;
    ZKB_TRY(msm_g1_device(ctx, (const Fr *)scalars_dev, (const G1Affine *)bases_dev, n, &r, pick_stream(ctx, stream)));
    g1_emit(r, out_affine, out_jacobian, out_compressed);
    return ZKB_OK;
}

extern "C" int32_t zkb_msm_g1_host(zkb_ctx *ctx, const uint64_t *scalars_host, const uint64_t *bases_host, uint64_t n, uint64_t out_affine[8],
                                   uint64_t *out_jacobian, uint8_t *out_compressed) {
    ZKB_ARG(ctx && out_affine && (n == 0 || (scalars_host && bases_host)));
    ZKB_CUDA(cudaSetDevice(ctx->device));
    void *ds = nullptr, *db = nullptr;
    if (n) {
        ZKB_TRY(scratch_get(ctx, SCR_HOSTIO_A, n * 32, &ds));
        ZKB_TRY(scratch_get(ctx, SCR_HOSTIO_B, n * 64, &db));
        ZKB_CUDA(cudaMemcpyAsync(ds, scalars_host, n * 32, cudaMemcpyHostToDevice, ctx->stream));
        ZKB_CUDA(cudaMemcpyAsync(db, bases_host, n * 64, cudaMemcpyHostToDevice, ctx->stream));
    }
    return zkb_msm_g1_dev(ctx, (const uint64_t *)ds, (const uint64_t *)db, n, out_affine, out_jacobian, out_compressed, ctx->stream);
}

extern "C" int32_t zkb_msm_g1_batch_dev(zkb_ctx *ctx, const uint64_t *const *scalar_cols_dev, uint32_t batch, const uint64_t *bases_dev, uint64_t n,
                                        uint64_t *out_affine, void *stream) {
    ZKB_ARG(ctx && scalar_cols_dev && bases_dev && out_affine && batch >= 1);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    return msm_g1_columns(ctx, (const Fr *const *)scalar_cols_dev, batch, (const G1Affine *)bases_dev, n, (G1Affine *)out_affine, false,
                          pick_stream(ctx, stream));
}

extern "C" int32_t zkb_g1_fixed_base_mul_dev(zkb_ctx *ctx, const uint64_t base_affine_host[8], const uint64_t *scalars_dev, uint64_t n,
                                             uint64_t *out_affine_dev, void *stream) {
    ZKB_ARG(ctx && base_affine_host && scalars_dev && out_affine_dev);
    if (n == 0) return ZKB_OK;
    G1Affine base;
    memcpy(&base, base_affine_host, 64);
    fixed_base_mul_kernel<<<(unsigned)((n + 127) / 128), 128, 0, pick_stream(ctx, stream)>>>(base, (const Fr *)scalars_dev, n, (G1Affine *)out_affine_dev);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}
