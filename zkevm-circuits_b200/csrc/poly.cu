// poly.cu -- polynomial utilities of the prover around MSM/NTT (SURVEY.md section 8a rows a5-a9), sm_90a.
//
//   fr_powers            : out[i] = base^i                  (coset scaling tables, omega^i for the permutation argument)
//   poly_eval (batched)  : halo2_proofs::arithmetic::eval_polynomial over many polynomials at one point (row a8)
//   kate_division        : halo2_proofs::arithmetic::kate_division, (a(X) - a(u)) / (X - u) (row a9, SHPLONK)
//   prefix product / sum : running product z (permutation/prover.rs) and running sum phi (mv_lookup/prover.rs) (a5, a6)
//   lincomb              : sum_j c_j * P_j(X)  (SHPLONK numerators; reads every committed polynomial once)
// All are exact Fr arithmetic, bit-identical to the CPU prover by construction (the results are unique field elements).
// Parallel structure: every linear recurrence x_{i+1} = m * x_i + a_i is cut into per-thread chunks, chunk summaries
// are combined with precomputed powers m^(2^j) (Hillis-Steele inside a block, a second tiny kernel across blocks),
// and the carries are applied in a final pass: ~3 multiplies per element instead of a serial chain.
#include "common.cuh"
#include <string.h>

namespace zkb {

struct Pow2Table { Fr p[40]; };  // p[j] = base^(2^j)

static Pow2Table make_pow2(const Fr &base) {
    Pow2Table t;
    t.p[0] = base;
    for (int j = 1; j < 40; ++j) t.p[j] = fp_sqr(t.p[j - 1]);
    return t;
}
__device__ __forceinline__ Fr pow_from_table(const Pow2Table &t, uint64_t e) {
    Fr acc = Fr::one();
    bool first = true;
    for (int j = 0; j < 40 && (e >> j); ++j) {
        if ((e >> j) & 1) {
            if (first) { acc = t.p[j]; first = false; }
            else acc = fp_mul(acc, t.p[j]);
        }
    }
    return acc;
}

constexpr int PL = 8;      // elements per thread
constexpr int PT = 256;    // threads per block
constexpr int PB = PL * PT;  // elements per block

// ---------------------------------------------------------------------------------------------------------- powers
__global__ void __launch_bounds__(PT) powers_kernel(Pow2Table t, uint64_t n, Fr *__restrict__ out) {
    const uint64_t s = ((uint64_t)blockIdx.x * PT + threadIdx.x) * PL;
    if (s >= n) return;
    Fr cur = pow_from_table(t, s);
#pragma unroll
    for (int j = 0; j < PL; ++j) {
        if (s + j < n) fp_store(out + s + j, cur);
        cur = fp_mul(cur, t.p[0]);
    }
}

// ---------------------------------------------------------------------------------------------------------- eval
// stage 1: grid (ceil(n / PB), num_polys); partial[p][b] = sum_{i in block b} c_i x^(i - b*PB)
__global__ void __launch_bounds__(PT) eval_stage1_kernel(const Fr *const *__restrict__ polys, uint64_t n, Pow2Table t, Fr *__restrict__ partial) {
    __shared__ uint4 sm[2 * PT];
    Fr *smf = reinterpret_cast<Fr *>(sm);
    const Fr *c = polys[blockIdx.y];
    const uint64_t s = ((uint64_t)blockIdx.x * PT + threadIdx.x) * PL;
    Fr acc = Fr::zero();
#pragma unroll
    for (int j = PL - 1; j >= 0; --j) {
        acc = fp_mul(acc, t.p[0]);
        if (s + j < n) acc = fp_add(acc, fp_load(c + s + j));
    }
    smf[threadIdx.x] = acc;
    __syncthreads();
    // tree: T_t += x^(PL * d) * T_{t+d};  x^(PL*d) = p[3 + log2 d]
    int lvl = 3;
    for (int d = 1; d < PT; d <<= 1, ++lvl) {
        if ((threadIdx.x & (2 * d - 1)) == 0) {
            Fr a = smf[threadIdx.x];
            a = fp_add(a, fp_mul(smf[threadIdx.x + d], t.p[lvl]));
            smf[threadIdx.x] = a;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) fp_store(partial + (size_t)blockIdx.y * gridDim.x + blockIdx.x, smf[0]);
}
// stage 2: one block per polynomial; result = sum_b partial[b] * x^(PB * b)
__global__ void __launch_bounds__(PT) eval_stage2_kernel(const Fr *__restrict__ partial, uint32_t nblocks, Pow2Table t, Fr *__restrict__ out) {
    __shared__ uint4 sm[2 * PT];
    Fr *smf = reinterpret_cast<Fr *>(sm);
    const Fr *pp = partial + (size_t)blockIdx.x * nblocks;
    // thread handles blocks b = tid, tid + PT, ... (Horner in x^(PB*PT) from the top)
    Fr acc = Fr::zero();
    const Fr stride = t.p[11 + 8];  // x^(PB * PT) = x^(2^11 * 2^8)
    int top = (int)((nblocks + PT - 1) / PT) - 1;
    for (int r = top; r >= 0; --r) {
        acc = fp_mul(acc, stride);
        const uint32_t b = (uint32_t)r * PT + threadIdx.x;
        if (b < nblocks) acc = fp_add(acc, fp_load(pp + b));
    }
    smf[threadIdx.x] = acc;
    __syncthreads();
    int lvl = 11;  // x^(PB * d)
    for (int d = 1; d < PT; d <<= 1, ++lvl) {
        if ((threadIdx.x & (2 * d - 1)) == 0) {
            Fr a = smf[threadIdx.x];
            a = fp_add(a, fp_mul(smf[threadIdx.x + d], t.p[lvl]));
            smf[threadIdx.x] = a;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) fp_store(out + blockIdx.x, smf[0]);
}

// ---------------------------------------------------------------------------------------------------------- scans
// generic linear recurrence, forward:  y_0 = init ; y_{i+1} = OP(y_i, in_i)   (exclusive scan, n outputs)
//   MODE 0: product (y_{i+1} = y_i * in_i)      MODE 1: sum (y_{i+1} = y_i + in_i)
template <int MODE>
__device__ __forceinline__ Fr scan_op(const Fr &a, const Fr &b) { return MODE == 0 ? fp_mul(a, b) : fp_add(a, b); }
template <int MODE>
__device__ __forceinline__ Fr scan_identity() { return MODE == 0 ? Fr::one() : Fr::zero(); }

// block-wide inclusive scan of one Fr per thread through shared memory (Hillis-Steele)
template <int MODE>
__device__ __forceinline__ Fr block_inclusive_scan(Fr v, Fr *smf) {
    smf[threadIdx.x] = v;
    __syncthreads();
    for (int d = 1; d < PT; d <<= 1) {
        Fr o = v;
        if ((int)threadIdx.x >= d) o = scan_op<MODE>(smf[threadIdx.x - d], v);
        __syncthreads();
        v = o;
        smf[threadIdx.x] = v;
        __syncthreads();
    }
    return v;
}

template <int MODE>
__global__ void __launch_bounds__(PT) scan_stage1_kernel(const Fr *__restrict__ in, uint64_t n, Fr *__restrict__ out, Fr *__restrict__ block_tot) {
    __shared__ uint4 sm[2 * PT];
    Fr *smf = reinterpret_cast<Fr *>(sm);
    const uint64_t s = ((uint64_t)blockIdx.x * PT + threadIdx.x) * PL;
    Fr v[PL];
    Fr tot = scan_identity<MODE>();
#pragma unroll
    for (int j = 0; j < PL; ++j) {
        v[j] = s + j < n ? fp_load(in + s + j) : scan_identity<MODE>();
        tot = scan_op<MODE>(tot, v[j]);
    }
    const Fr incl = block_inclusive_scan<MODE>(tot, smf);
    // exclusive prefix of this thread = inclusive of the previous thread
    Fr pre = threadIdx.x ? smf[threadIdx.x - 1] : scan_identity<MODE>();
#pragma unroll
    for (int j = 0; j < PL; ++j) {
        if (s + j < n) fp_store(out + s + j, pre);
        pre = scan_op<MODE>(pre, v[j]);
    }
    if (threadIdx.x == PT - 1) fp_store(block_tot + blockIdx.x, incl);
}
// single block: exclusive scan of the block totals, seeded with init
template <int MODE>
__global__ void __launch_bounds__(PT) scan_stage2_kernel(Fr *__restrict__ block_tot, uint32_t nblocks, Fr init) {
    __shared__ uint4 sm[2 * PT];
    Fr *smf = reinterpret_cast<Fr *>(sm);
    Fr running = init;
    for (uint32_t s = 0; s < nblocks; s += PT) {
        const uint32_t idx = s + threadIdx.x;
        const Fr v = idx < nblocks ? fp_load(block_tot + idx) : scan_identity<MODE>();
        const Fr incl = block_inclusive_scan<MODE>(v, smf);
        const Fr pre = threadIdx.x ? smf[threadIdx.x - 1] : scan_identity<MODE>();
        const Fr last = smf[PT - 1];
        if (idx < nblocks) fp_store(block_tot + idx, scan_op<MODE>(running, pre));
        running = scan_op<MODE>(running, last);
        (void)incl;
        __syncthreads();
    }
}
template <int MODE>
__global__ void __launch_bounds__(PT) scan_stage3_kernel(Fr *__restrict__ out, uint64_t n, const Fr *__restrict__ block_pre) {
    const uint64_t s = ((uint64_t)blockIdx.x * PT + threadIdx.x) * PL;
    const Fr pre = fp_load(block_pre + blockIdx.x);
#pragma unroll
    for (int j = 0; j < PL; ++j)
        if (s + j < n) fp_store(out + s + j, scan_op<MODE>(pre, fp_load(out + s + j)));
}

// ---------------------------------------------------------------------------------------------------------- kate division
// q_{i-1} = a_i + u q_i (i = n-1 .. 1), q_{n-1} := 0.  Output array has n entries (q[n-1] = 0).
// stage 1: per-thread local suffix Horner with zero carry; block suffix combine; block head value to block_tot.
__global__ void __launch_bounds__(PT) kate_stage1_kernel(const Fr *__restrict__ a, uint64_t n, Pow2Table t, Fr *__restrict__ q, Fr *__restrict__ block_tot) {
    __shared__ uint4 sm[2 * PT];
    Fr *smf = reinterpret_cast<Fr *>(sm);
    // thread owns a-indices [s, s + PL); writes q[i-1] for those i (i >= 1)
    const uint64_t s = ((uint64_t)blockIdx.x * PT + threadIdx.x) * PL;
    Fr tv = Fr::zero();
#pragma unroll
    for (int j = PL - 1; j >= 0; --j) {
        const uint64_t i = s + j;
        tv = fp_mul(tv, t.p[0]);
        if (i < n) tv = fp_add(tv, fp_load(a + i));
        if (i >= 1 && i < n) fp_store(q + i - 1, tv);
    }
    // suffix combine inside the block: Q_c = T_c + u^PL * Q_{c+1}  ->  Hillis-Steele with u^(PL * d)
    smf[threadIdx.x] = tv;
    __syncthreads();
    Fr v = tv;
    int lvl = 3;
    for (int d = 1; d < PT; d <<= 1, ++lvl) {
        Fr o = v;
        if (threadIdx.x + d < PT) o = fp_add(v, fp_mul(smf[threadIdx.x + d], t.p[lvl]));
        __syncthreads();
        v = o;
        smf[threadIdx.x] = v;
        __syncthreads();
    }
    // carry into this thread's chunk from the chunks above it *inside the block* = Q_{c+1} (block-local)
    const Fr carry = threadIdx.x + 1 < PT ? smf[threadIdx.x + 1] : Fr::zero();
    // apply block-local carry: q[i-1] += u^(s + PL - i) * carry
    if (!carry.is_zero()) {
        Fr p = t.p[0];
#pragma unroll
        for (int j = PL - 1; j >= 0; --j) {
            const uint64_t i = s + j;
            if (i >= 1 && i < n) fp_store(q + i - 1, fp_add(fp_load(q + i - 1), fp_mul(p, carry)));
            p = fp_mul(p, t.p[0]);
        }
    }
    if (threadIdx.x == 0) fp_store(block_tot + blockIdx.x, smf[0]);
}
// stage 2 (single block): suffix combine of block heads: C_b = carry INTO block b = sum_{j > b} head_j u^(PB (j - b - 1))
__global__ void __launch_bounds__(PT) kate_stage2_kernel(Fr *__restrict__ block_tot, uint32_t nblocks, Pow2Table t) {
    __shared__ uint4 sm[2 * PT];
    Fr *smf = reinterpret_cast<Fr *>(sm);
    Fr running = Fr::zero();  // value of Q at the bottom of the tile above (true suffix value entering the tile)
    const int tiles = (int)((nblocks + PT - 1) / PT);
    for (int tile = tiles - 1; tile >= 0; --tile) {
        const uint32_t idx = (uint32_t)tile * PT + threadIdx.x;
        Fr v = idx < nblocks ? fp_load(block_tot + idx) : Fr::zero();
        smf[threadIdx.x] = v;
        __syncthreads();
        int lvl = 11;
        for (int d = 1; d < PT; d <<= 1, ++lvl) {
            Fr o = v;
            if (threadIdx.x + d < PT) o = fp_add(v, fp_mul(smf[threadIdx.x + d], t.p[lvl]));
            __syncthreads();
            v = o;
            smf[threadIdx.x] = v;
            __syncthreads();
        }
        // v = suffix value of this tile alone starting at block idx ; add contribution of everything above the tile:
        // true S_idx = v + u^(PB * (PT - tid)) * running ; carry INTO block idx = S_{idx+1}
        Fr above = threadIdx.x + 1 < PT ? smf[threadIdx.x + 1] : Fr::zero();
        const uint64_t e = (uint64_t)PB * (PT - 1 - threadIdx.x);
        Fr carry_in = fp_add(above, fp_mul(pow_from_table(t, e), running));
        const Fr tile_head = fp_add(smf[0], fp_mul(pow_from_table(t, (uint64_t)PB * PT), running));
        __syncthreads();
        if (idx < nblocks) fp_store(block_tot + idx, carry_in);
        running = tile_head;
        __syncthreads();
    }
}
__global__ void __launch_bounds__(PT) kate_stage3_kernel(Fr *__restrict__ q, uint64_t n, Pow2Table t, const Fr *__restrict__ block_carry) {
    const Fr carry = fp_load(block_carry + blockIdx.x);
    if (carry.is_zero()) return;
    const uint64_t s = ((uint64_t)blockIdx.x * PT + threadIdx.x) * PL;
    // exponent for index i: distance to the top of the block: (block_top - i), block_top = (blockIdx+1)*PB
    const uint64_t top = ((uint64_t)blockIdx.x + 1) * PB;
    if (s >= n) return;
    Fr p = pow_from_table(t, top - (s + PL - 1));
#pragma unroll
    for (int j = PL - 1; j >= 0; --j) {
        const uint64_t i = s + j;
        if (i >= 1 && i < n) fp_store(q + i - 1, fp_add(fp_load(q + i - 1), fp_mul(p, carry)));
        p = fp_mul(p, t.p[0]);
    }
}

// ---------------------------------------------------------------------------------------------------------- lincomb
// out[r] = sum_j coef[j] * polys[j][r]   (+ out_prev[r] * prev_scale if accumulate)
__global__ void __launch_bounds__(256) lincomb_kernel(const Fr *const *__restrict__ polys, const Fr *__restrict__ coefs, uint32_t num, uint64_t n,
                                                      Fr *__restrict__ out, int accumulate) {
    for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
        Fr acc = accumulate ? fp_load(out + r) : Fr::zero();
        for (uint32_t j = 0; j < num; ++j) acc = fp_add(acc, fp_mul(fp_load(polys[j] + r), fp_load(coefs + j)));
        fp_store(out + r, acc);
    }
}

// ---------------------------------------------------------------------------------------------------------- host wrappers (C++)
int32_t fr_powers_device(zkb_ctx *ctx, const Fr &base, uint64_t n, Fr *out, cudaStream_t st) {
    if (n == 0) return ZKB_OK;
    Pow2Table t = make_pow2(base);
    powers_kernel<<<(unsigned)((n + PB - 1) / PB), PT, 0, st>>>(t, n, out);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

// evaluate `num` polynomials (device pointer table d_polys, device) of n coefficients at x; results to out_host (synchronises)
int32_t poly_eval_device(zkb_ctx *ctx, const Fr *const *d_polys, uint32_t num, uint64_t n, const Fr &x, Fr *out_host, cudaStream_t st) {
    if (num == 0) return ZKB_OK;
    const uint32_t nblocks = (uint32_t)((n + PB - 1) / PB);
    Fr *tmp = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_MISC2, ((size_t)nblocks * num + num) * sizeof(Fr), (void **)&tmp));
    Fr *res = tmp + (size_t)nblocks * num;
    Pow2Table t = make_pow2(x);
    eval_stage1_kernel<<<dim3(nblocks, num), PT, 0, st>>>(d_polys, n, t, tmp);
    eval_stage2_kernel<<<num, PT, 0, st>>>(tmp, nblocks, t, res);
    ctx->launches += 2;
    ZKB_CUDA(cudaGetLastError());
    ZKB_CUDA(cudaMemcpyAsync(out_host, res, num * sizeof(Fr), cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    return ZKB_OK;
}

template <int MODE>
static int32_t scan_device(zkb_ctx *ctx, const Fr *in, uint64_t n, const Fr &init, Fr *out, cudaStream_t st) {
    if (n == 0) return ZKB_OK;
    const uint32_t nblocks = (uint32_t)((n + PB - 1) / PB);
    Fr *tot = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_MISC2, (size_t)nblocks * sizeof(Fr), (void **)&tot));
    scan_stage1_kernel<MODE><<<nblocks, PT, 0, st>>>(in, n, out, tot);
    scan_stage2_kernel<MODE><<<1, PT, 0, st>>>(tot, nblocks, init);
    scan_stage3_kernel<MODE><<<nblocks, PT, 0, st>>>(out, n, tot);
    ctx->launches += 3;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}
int32_t prefix_product_device(zkb_ctx *ctx, const Fr *in, uint64_t n, const Fr &init, Fr *out, cudaStream_t st) { return scan_device<0>(ctx, in, n, init, out, st); }
int32_t prefix_sum_device(zkb_ctx *ctx, const Fr *in, uint64_t n, const Fr &init, Fr *out, cudaStream_t st) { return scan_device<1>(ctx, in, n, init, out, st); }

int32_t kate_division_device(zkb_ctx *ctx, const Fr *a, uint64_t n, const Fr &u, Fr *q, cudaStream_t st) {
    if (n == 0) return ZKB_OK;
    const uint32_t nblocks = (uint32_t)((n + PB - 1) / PB);
    Fr *tot = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_MISC2, (size_t)nblocks * sizeof(Fr), (void **)&tot));
    Pow2Table t = make_pow2(u);
    ZKB_CUDA(cudaMemsetAsync(q + n - 1, 0, sizeof(Fr), st));
    kate_stage1_kernel<<<nblocks, PT, 0, st>>>(a, n, t, q, tot);
    if (nblocks > 1) {
        kate_stage2_kernel<<<1, PT, 0, st>>>(tot, nblocks, t);
        kate_stage3_kernel<<<nblocks, PT, 0, st>>>(q, n, t, tot);
        ctx->launches += 2;
    }
    ctx->launches += 1;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

int32_t lincomb_device(zkb_ctx *ctx, const Fr *const *d_polys, const Fr *d_coefs, uint32_t num, uint64_t n, Fr *out, bool accumulate, cudaStream_t st) {
    if (n == 0) return ZKB_OK;
    uint64_t blocks = (n + 255) / 256;
    const uint64_t cap = (uint64_t)ctx->sm_count * 8;
    if (blocks > cap) blocks = cap;
    lincomb_kernel<<<(unsigned)blocks, 256, 0, st>>>(d_polys, d_coefs, num, n, out, accumulate ? 1 : 0);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

}  // namespace zkb
using namespace zkb;

static Fr load_fr(const uint64_t *p) {
    Fr r;
    memcpy(r.l, p, 32);
    return r;
}

extern "C" int32_t zkb_fr_powers_dev(zkb_ctx *ctx, const uint64_t base[4], uint64_t n, uint64_t *out_dev, void *stream) {
    ZKB_ARG(ctx && base && (out_dev || n == 0));
    return fr_powers_device(ctx, load_fr(base), n, (Fr *)out_dev, pick_stream(ctx, stream));
}

extern "C" int32_t zkb_poly_eval_dev(zkb_ctx *ctx, const uint64_t *const *polys_dev, uint32_t num_polys, uint64_t n, const uint64_t x[4],
                                     uint64_t *out_host, void *stream) {
    ZKB_ARG(ctx && polys_dev && x && out_host && n > 0);
    cudaStream_t st = pick_stream(ctx, stream);
    Fr **tbl = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_MISC, (size_t)num_polys * sizeof(Fr *), (void **)&tbl));
    ZKB_CUDA(cudaMemcpyAsync(tbl, polys_dev, (size_t)num_polys * sizeof(Fr *), cudaMemcpyHostToDevice, st));
    return poly_eval_device(ctx, (const Fr *const *)tbl, num_polys, n, load_fr(x), (Fr *)out_host, st);
}

extern "C" int32_t zkb_fr_prefix_product_dev(zkb_ctx *ctx, const uint64_t *in_dev, uint64_t n, const uint64_t init[4], uint64_t *out_dev, void *stream) {
    ZKB_ARG(ctx && in_dev && init && out_dev && in_dev != out_dev);
    return prefix_product_device(ctx, (const Fr *)in_dev, n, load_fr(init), (Fr *)out_dev, pick_stream(ctx, stream));
}
extern "C" int32_t zkb_fr_prefix_sum_dev(zkb_ctx *ctx, const uint64_t *in_dev, uint64_t n, const uint64_t init[4], uint64_t *out_dev, void *stream) {
    ZKB_ARG(ctx && in_dev && init && out_dev && in_dev != out_dev);
    return prefix_sum_device(ctx, (const Fr *)in_dev, n, load_fr(init), (Fr *)out_dev, pick_stream(ctx, stream));
}
extern "C" int32_t zkb_kate_division_dev(zkb_ctx *ctx, const uint64_t *a_dev, uint64_t n, const uint64_t u[4], uint64_t *q_dev, void *stream) {
    ZKB_ARG(ctx && a_dev && u && q_dev && a_dev != q_dev);
    return kate_division_device(ctx, (const Fr *)a_dev, n, load_fr(u), (Fr *)q_dev, pick_stream(ctx, stream));
}
