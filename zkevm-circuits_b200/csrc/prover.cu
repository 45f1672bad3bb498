// prover.cu -- device-resident create_proof: host orchestration (C++) over the CUDA kernels.
//
// Mirrors halo2_proofs 1.1.0 (scroll-tech/halo2 v1.1 @ e5ddf67) plonk/prover.rs `create_proof` for
// KZGCommitmentScheme<Bn256> + ProverSHPLONK + Blake2bWrite/Challenge255, the instantiation the reference uses at
// circuit-benchmarks/src/super_circuit.rs:117-132 and circuit-benchmarks/src/packed_multi_keccak.rs:72-87:
//   transcript order, mv-lookup (logUp) argument (plonk/mv_lookup/prover.rs), permutation argument
//   (plonk/permutation/prover.rs), vanishing argument (plonk/vanishing/prover.rs), quotient numerator term order
//   (plonk/evaluation.rs evaluate_h), evaluation order and SHPLONK multi-open (poly/kzg/multiopen/shplonk/prover.rs).
// The proof layout / evaluation order / constraint formulas are the ones visible in the reference fixture
// aggregator/data/batch-task.json (see tests/golden and SURVEY.md appendix B).
//
// What crosses the boundary (include/zkb200.h, `zkb_pk_*`, `zkb_prove_*`): the constraint system as a flat "CSF" blob,
// fixed / sigma column values, the SRS, per-phase advice columns (already blinded by the caller), blinding scalars and
// vk.transcript_repr (Rust-specific derivations, SURVEY.md hard part 1).  Everything else stays in HBM: columns,
// polynomials, coset evaluations, the quotient; only 64-byte commitments and 32-byte evaluations return to the host.
//
// Design points (not upstream's): the quotient is evaluated coset-part by coset-part (extended domain = E cosets of
// size n, SURVEY 8e) by one fused interpreter launch per degree group on the part, each group only on the parts its degree
// needs (QuotientGroups); all scans / inversions / evaluations are parallel kernels.
#include "common.cuh"
#include "csf.cuh"
#include "expr.cuh"
#include "lookup.cuh"
#include "pk.cuh"
#include "transcript.cuh"
#include <algorithm>
#include <memory>
#include <string.h>
#include <stdlib.h>
#include <time.h>

namespace zkb {

// ---------------------------------------------------------------------------------------------------------- small kernels
__global__ void set_one_kernel(Fr *a, uint64_t idx) { fp_store(a + idx, Fr::one()); }
__global__ void fill_range_one_kernel(Fr *a, uint64_t from, uint64_t to) {
    uint64_t i = from + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < to) fp_store(a + i, Fr::one());
}
__global__ void mul_arrays_kernel(const Fr *__restrict__ a, const Fr *__restrict__ b, Fr *__restrict__ out, uint64_t n) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) fp_store(out + i, fp_mul(fp_load(a + i), fp_load(b + i)));
}
// a[i] *= c
__global__ void scale_const_kernel(Fr *__restrict__ a, Fr c, uint64_t n) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) fp_store(a + i, fp_mul(fp_load(a + i), c));
}
// out[i] -= low[i] for i < k (subtract a low-degree polynomial given on the device)
__global__ void sub_low_kernel(Fr *__restrict__ out, const Fr *__restrict__ low, uint32_t k) {
    uint32_t i = threadIdx.x;   // one block of MAX_POINTS_PER_COLUMN threads: a rotation set has at most that many points
    if (i < k) fp_store(out + i, fp_sub(fp_load(out + i), fp_load(low + i)));
}

// out[j + m * i] = slab[rows[j] * n + i]  (a quotient group's coset parts gathered as rows -> its order on zeta D_{mn})
__global__ void interleave_rows_kernel(const Fr *__restrict__ slab, const uint32_t *__restrict__ rows, Fr *__restrict__ out, uint32_t log_n,
                                       uint32_t m) {
    const uint64_t idx = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (idx >= ((uint64_t)m << log_n)) return;
    const uint64_t j = idx % m, i = idx / m;
    fp_store(out + idx, fp_load(slab + ((uint64_t)rows[j] << log_n) + i));
}

// ---------------------------------------------------------------------------------------------------------- helpers
static Fr fr_from_u64(uint64_t v) { return fp_from_u64<FrParams>(v); }
static bool fr_less(const Fr &a, const Fr &b) {  // halo2curves Ord: canonical integer comparison
    Fr x = fp_to_canonical(a), y = fp_to_canonical(b);
    for (int i = 7; i >= 0; --i) {
        if (x.l[i] != y.l[i]) return x.l[i] < y.l[i];
    }
    return false;
}
static Fr fr_pow_i64(const Fr &base, const Fr &base_inv, int64_t e) { return e >= 0 ? fp_pow_u64(base, (uint64_t)e) : fp_pow_u64(base_inv, (uint64_t)(-e)); }

}  // namespace zkb
using namespace zkb;

struct zkb_session {
    zkb_pk *pk = nullptr;
    Transcript tr;   // its callback status is checked after every stage
    DevPool pool;
    std::vector<Fr *> inst_values, inst_polys, adv_values;
    // columns handed over ahead of their phase (zkb_prove_upload_advice): staged device copies, consumed by zkb_prove_advice_phase
    std::map<uint32_t, Fr *> early_cols;
    std::vector<Fr> challenges;
    uint32_t next_phase = 0;
    bool finished = false;
};

namespace zkb {

// ---------------------------------------------------------------------------------------------------------- basis changes
static int32_t lagrange_to_coeff(zkb_pk *pk, const Fr *values, Fr *poly, cudaStream_t st) {
    return ntt_fr_device(pk->ctx, values, poly, pk->k, pk->omega_inv, &pk->n_inv, 0, nullptr, st);
}
// size-n NTTs of many columns, batched in chunks that need at most 2 GiB of NTT scratch
static int32_t ntt_many(zkb_pk *pk, const std::vector<Fr *> &src, const std::vector<Fr *> &dst, const Fr &w, const Fr *scale, const Fr *in_scale,
                        cudaStream_t st) {
    const uint32_t chunk = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(256, (1ull << 31) / (pk->n * sizeof(Fr))));
    for (size_t done = 0; done < src.size(); done += chunk) {
        const uint32_t cur = (uint32_t)std::min<size_t>(chunk, src.size() - done);
        std::vector<Fr *> a(src.begin() + done, src.begin() + done + cur), b(dst.begin() + done, dst.begin() + done + cur);
        ZKB_TRY(ntt_fr_batch_device(pk->ctx, a.data(), b.data(), cur, pk->k, w, scale, 0, in_scale, st));
    }
    return ZKB_OK;
}

// multi-GPU dealing of independent units (columns, lookup arguments, coset parts): the `count` units are cut into P contiguous
// blocks of blk = ceil(count / P), rank r computes block r.  Results live in a slab of P * blk unit slots (the tail of the last
// blocks is padding), so ONE in-place ncclAllGather (every rank contributes its own block, 1/P of the slab) completes it -- no
// zero filling, no arithmetic on the wire (round 1 used an all-reduce over a zero-initialised slab: P times the bytes).
struct Deal {
    size_t count = 0, blk = 0;
    int P = 1, rank = 0;
    bool on = false;
    Deal(const zkb_ctx *c, size_t n) : count(n), P(c->nranks), rank(c->rank) {
        on = P > 1 && n >= 2;
        blk = on ? (n + P - 1) / P : n;
    }
    bool mine(size_t i) const { return !on || (int)(i / blk) == rank; }
    size_t padded() const { return on ? (size_t)P * blk : count; }
};
static int32_t deal_gather(zkb_ctx *ctx, const Deal &d, void *slab, size_t unit_bytes, cudaStream_t st) {
    if (!d.on) return ZKB_OK;
    return comm_allgather(ctx, (const uint8_t *)slab + (size_t)d.rank * d.blk * unit_bytes, slab, d.blk * unit_bytes, st);
}
// cols[i] = column i of a new slab of d.padded() columns of n elements (nothing is allocated for no columns)
static int32_t dealt_columns(DevPool &pool, const Deal &d, uint64_t n, std::vector<Fr *> &cols, Fr **slab) {
    cols.resize(d.count);
    if (!d.count) return ZKB_OK;
    ZKB_TRY(pool.fr(d.padded() * n, slab));
    for (size_t i = 0; i < d.count; ++i) cols[i] = *slab + i * n;
    return ZKB_OK;
}

// srs_commit_many's basis index: g (coefficient form, ParamsKZG::commit) / g_lagrange (values, commit_lagrange)
enum { BASIS_G = 0, BASIS_LAGRANGE = 1 };

// commit several size-n columns against one basis with batched MSMs.  With a communicator the columns are dealt in contiguous
// blocks (Deal) and the 64-byte results are all-gathered.
static int32_t commit_many(zkb_pk *pk, const std::vector<Fr *> &cols, int basis, std::vector<G1Affine> &out, cudaStream_t st) {
    zkb_ctx *ctx = pk->ctx;
    const uint64_t len = pk->n;
    if (ctx->nranks > 1 && cols.size() == 1 && len >= (1u << 14)) {
        // a single commitment (random polynomial, SHPLONK's h and the final quotient) cannot be dealt: shard it by point range instead
        // (SURVEY 8e): every rank reduces len / P points, the 64-byte partial sums are all-gathered and added on the host
        const uint64_t P = (uint64_t)ctx->nranks, lo = len * (uint64_t)ctx->rank / P, hi = len * ((uint64_t)ctx->rank + 1) / P;
        const G1Affine *bases = basis == BASIS_G ? pk->srs->g : pk->srs->g_lagrange;
        G1Affine part;
        ZKB_TRY(msm_g1_device(ctx, cols[0] + lo, bases + lo, hi - lo, &part, st));
        G1Affine *d_buf = nullptr;
        ZKB_TRY(scratch_get(ctx, SCR_COMM, 16 * sizeof(G1Affine), (void **)&d_buf));
        ZKB_CUDA(cudaMemcpyAsync(d_buf + ctx->rank, &part, sizeof(G1Affine), cudaMemcpyHostToDevice, st));
        ZKB_TRY(comm_allgather(ctx, d_buf + ctx->rank, d_buf, sizeof(G1Affine), st));
        G1Affine all[16];
        ZKB_CUDA(cudaMemcpyAsync(all, d_buf, P * sizeof(G1Affine), cudaMemcpyDeviceToHost, st));
        ZKB_CUDA(cudaStreamSynchronize(st));
        G1Xyzz acc = G1Xyzz::identity();
        for (uint64_t r = 0; r < P; ++r) g1_add_mixed(acc, all[r]);
        out.assign(1, g1_to_affine(acc));
        return ZKB_OK;
    }
    const Deal d(ctx, cols.size());
    if (!d.on) {
        out.resize(cols.size());
        return srs_commit_many(pk->srs, basis, cols.data(), (uint32_t)cols.size(), len, out.data(), st);
    }
    std::vector<Fr *> mine;
    for (size_t i = 0; i < cols.size(); ++i)
        if (d.mine(i)) mine.push_back(cols[i]);
    std::vector<G1Affine> part(mine.size());
    if (!mine.empty()) ZKB_TRY(srs_commit_many(pk->srs, basis, mine.data(), (uint32_t)mine.size(), len, part.data(), st));
    G1Affine *d_buf = nullptr;
    ZKB_TRY(scratch_get(ctx, SCR_COMM, d.padded() * sizeof(G1Affine), (void **)&d_buf));
    if (!part.empty()) ZKB_CUDA(cudaMemcpyAsync(d_buf + (size_t)d.rank * d.blk, part.data(), part.size() * sizeof(G1Affine), cudaMemcpyHostToDevice, st));
    ZKB_TRY(deal_gather(ctx, d, d_buf, sizeof(G1Affine), st));
    out.resize(d.padded());
    ZKB_CUDA(cudaMemcpyAsync(out.data(), d_buf, d.padded() * sizeof(G1Affine), cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    out.resize(cols.size());
    return ZKB_OK;
}
// commit the columns and write the commitments to the transcript in order
static int32_t commit_write(zkb_session *s, const std::vector<Fr *> &cols, int basis, cudaStream_t st) {
    std::vector<G1Affine> cms;
    ZKB_TRY(commit_many(s->pk, cols, basis, cms, st));
    for (auto &cm : cms) ZKB_TRY(s->tr.write_point(cm));
    return ZKB_OK;
}

// out (+)= sum_i coefs[i] * polys[i] over n coefficients.  `coefs` is copied asynchronously: keep it alive until the stream is synchronised.
static int32_t lincomb(zkb_pk *pk, DevPool &pool, const std::vector<Fr *> &polys, const std::vector<Fr> &coefs, Fr *out, bool accumulate, cudaStream_t st) {
    Fr **d_p = nullptr;
    Fr *d_c = nullptr;
    ZKB_TRY(upload_table(pool, polys, &d_p, st));
    ZKB_TRY(pool.fr(coefs.size(), &d_c));
    ZKB_CUDA(cudaMemcpyAsync(d_c, coefs.data(), coefs.size() * sizeof(Fr), cudaMemcpyHostToDevice, st));
    return lincomb_device(pk->ctx, d_p, d_c, (uint32_t)polys.size(), pk->n, out, accumulate, st);
}

}  // namespace zkb

// ================================================================================================ C ABI: proving key
// the quotient table's proof-independent slots in coefficient form, null elsewhere
std::vector<Fr *> zkb::pk_quotient_polys(const zkb_pk *pk) {
    const SlotMap &sm = pk->sm;
    std::vector<Fr *> t(sm.slots, nullptr);
    put_columns(t, sm.fixed0, pk->fixed_polys);
    put_columns(t, sm.sigma0, pk->sigma_polys);
    t[sm.x] = pk->xid_poly; t[sm.l0] = pk->l0_poly; t[sm.l_last] = pk->llast_poly; t[sm.l_blind] = pk->lblind_poly;
    return t;
}

// The first stage of every pk constructor: domain constants, l_0 / l_last / l_blind / X in coefficient form, omega^i.  The SRS handle
// is shared, not copied.
int32_t zkb::pk_begin(zkb_ctx *ctx, Csf &&csf, zkb_srs *srs, zkb_pk **out) {
    ZKB_CUDA(cudaSetDevice(ctx->device));
    std::unique_ptr<zkb_pk> pk(new zkb_pk());
    pk->ctx = ctx;
    pk->pool.ctx = ctx;
    pk->srs = srs;
    pk->cs = std::move(csf);
    const Csf &cs = pk->cs;
    if (srs->ctx != ctx || srs->k != cs.k) { set_error("the SRS handle is for k = %u on another context or size (circuit k = %u): downsize it first", srs->k, cs.k); return ZKB_ERR_ARG; }
    cudaStream_t st = ctx->stream;
    pk->k = cs.k;
    pk->n = 1ull << cs.k;
    const uint64_t n = pk->n;
    // EvaluationDomain::new(j = cs.degree(), k)
    pk->qdeg = cs.d - 1;
    pk->ext_k = cs.k;
    while ((1ull << pk->ext_k) < n * pk->qdeg) pk->ext_k++;
    ZKB_ARG(pk->ext_k <= 28);
    pk->N = 1ull << pk->ext_k;
    pk->E = (uint32_t)(pk->N / n);
    pk->chunk = cs.d - 2;
    pk->nsets = (uint32_t)((cs.perm.size() + pk->chunk - 1) / pk->chunk);
    pk->sm = SlotMap(cs, pk->nsets);
    pk->ext_omega = host_root_of_unity(pk->ext_k);
    pk->omega = pk->ext_omega;
    for (uint32_t i = cs.k; i < pk->ext_k; ++i) pk->omega = fp_sqr(pk->omega);
    pk->omega_inv = fp_inv(pk->omega);
    pk->ext_omega_inv = fp_inv(pk->ext_omega);
    pk->n_inv = fp_inv(fr_from_u64(n));
    pk->N_inv = fp_inv(fr_from_u64(pk->N));
    pk->zeta = host_zeta();
    pk->t_inv.resize(pk->E);
    for (uint32_t j = 0; j < pk->E; ++j) pk->t_inv[j] = fp_inv(fp_sub(fp_pow_u64(pk->coset_gen(j), n), Fr::one()));
    // l_0, l_last, l_blind (Lagrange indicator vectors -> coefficient form), X (identity polynomial), omega^i
    ZKB_TRY(pk->pool.fr(n, &pk->l0_poly));
    ZKB_TRY(pk->pool.fr(n, &pk->llast_poly));
    ZKB_TRY(pk->pool.fr(n, &pk->lblind_poly));
    ZKB_TRY(pk->pool.fr(n, &pk->xid_poly));
    ZKB_TRY(pk->pool.fr(n, &pk->omega_pows));
    ZKB_CUDA(cudaMemsetAsync(pk->l0_poly, 0, n * sizeof(Fr), st));
    ZKB_CUDA(cudaMemsetAsync(pk->llast_poly, 0, n * sizeof(Fr), st));
    ZKB_CUDA(cudaMemsetAsync(pk->lblind_poly, 0, n * sizeof(Fr), st));
    ZKB_CUDA(cudaMemsetAsync(pk->xid_poly, 0, n * sizeof(Fr), st));
    ZKB_ARG(n > cs.bf + 1);
    set_one_kernel<<<1, 1, 0, st>>>(pk->l0_poly, 0);
    set_one_kernel<<<1, 1, 0, st>>>(pk->llast_poly, n - cs.bf - 1);
    fill_range_one_kernel<<<(cs.bf + 127) / 128, 128, 0, st>>>(pk->lblind_poly, n - cs.bf, n);
    if (n > 1) set_one_kernel<<<1, 1, 0, st>>>(pk->xid_poly, 1);
    ctx->launches += 4;
    ZKB_TRY(lagrange_to_coeff(pk.get(), pk->l0_poly, pk->l0_poly, st));
    ZKB_TRY(lagrange_to_coeff(pk.get(), pk->llast_poly, pk->llast_poly, st));
    ZKB_TRY(lagrange_to_coeff(pk.get(), pk->lblind_poly, pk->lblind_poly, st));
    ZKB_TRY(fr_powers_device(ctx, pk->omega, n, pk->omega_pows, st));
    *out = pk.release();
    return ZKB_OK;
}

// fixed / sigma columns: values and coefficient form (sources on the host, or on the device)
int32_t zkb::pk_ingest(zkb_pk *pk, const void *const *src, size_t cnt, std::vector<Fr *> &vals, std::vector<Fr *> &polys) {
    const uint64_t n = pk->n;
    cudaStream_t st = pk->ctx->stream;
    vals.resize(cnt);
    polys.resize(cnt);
    for (size_t i = 0; i < cnt; ++i) {
        ZKB_TRY(pk->pool.fr(n, &vals[i]));
        ZKB_TRY(pk->pool.fr(n, &polys[i]));
        ZKB_CUDA(cudaMemcpyAsync(vals[i], src[i], n * sizeof(Fr), cudaMemcpyDefault, st));
        ZKB_TRY(lagrange_to_coeff(pk, vals[i], polys[i], st));
    }
    return ZKB_OK;
}

int32_t zkb::pk_finish(zkb_pk *pk) {
    zkb_ctx *ctx = pk->ctx;
    cudaStream_t st = ctx->stream;
    const uint64_t n = pk->n;
    {
        // cache the coset evaluations of the static polynomials unless that would take more than ZKB_COSET_CACHE_GB (default: a
        // quarter of the device memory, 20 GB on an 80 GB H100 -- the rest holds the proving session's columns and coset parts)
        const std::vector<Fr *> stat = pk_quotient_polys(pk);
        const size_t nstat = stat.size() - std::count(stat.begin(), stat.end(), nullptr);
        const char *env = getenv("ZKB_COSET_CACHE_GB");
        const double budget = env ? atof(env) * 1e9 : 0.25 * (double)ctx->mem_bytes;
        if ((double)nstat * pk->N * sizeof(Fr) <= budget) {
            Fr *pows = nullptr;
            ZKB_TRY(pk->pool.fr(n, &pows));
            pk->coset_cache.assign(pk->E, std::vector<Fr *>(stat.size(), nullptr));
            for (uint32_t j = 0; j < pk->E; ++j) {
                ZKB_TRY(fr_powers_device(ctx, pk->coset_gen(j), n, pows, st));
                for (size_t i = 0; i < stat.size(); ++i) {
                    if (!stat[i]) continue;
                    ZKB_TRY(pk->pool.fr(n, &pk->coset_cache[j][i]));
                    ZKB_TRY(ntt_fr_device(ctx, stat[i], pk->coset_cache[j][i], pk->k, pk->omega, nullptr, 0, pows, st));
                }
            }
        }
    }
    ZKB_CUDA(cudaStreamSynchronize(st));
    return ZKB_OK;
}

// Builds the device-resident proving key of a loaded CSF.  sigma columns come either from the host (sigma_values) or are already on
// the device (sigma_dev, keygen path).
static int32_t pk_build(zkb_ctx *ctx, Csf &&csf, const uint64_t *const *fixed_values, const uint64_t *const *sigma_values,
                        const std::vector<Fr *> *sigma_dev, zkb_srs *srs, bool owns_srs, zkb_pk **out) {
    ZKB_ARG((csf.nf == 0 || fixed_values) && (csf.perm.empty() || sigma_values || sigma_dev));
    if (sigma_dev) ZKB_ARG(sigma_dev->size() == csf.perm.size());
    zkb_pk *raw = nullptr;
    ZKB_TRY(pk_begin(ctx, std::move(csf), srs, &raw));
    std::unique_ptr<zkb_pk> pk(raw);   // owns_srs stays false until the key is complete: on failure the caller still owns the handle
    const Csf &cs = pk->cs;
    ZKB_TRY(pk_ingest(pk.get(), (const void *const *)fixed_values, cs.nf, pk->fixed_values, pk->fixed_polys));
    const void *const *sigma_src = sigma_dev ? (const void *const *)sigma_dev->data() : (const void *const *)sigma_values;
    ZKB_TRY(pk_ingest(pk.get(), sigma_src, cs.perm.size(), pk->sigma_values, pk->sigma_polys));
    ZKB_TRY(pk_finish(pk.get()));
    pk->owns_srs = owns_srs;
    *out = pk.release();
    return ZKB_OK;
}

extern "C" int32_t zkb_pk_create(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, const uint64_t *const *fixed_values,
                                 const uint64_t *const *sigma_values, const uint64_t *g, const uint64_t *g_lagrange, zkb_pk **out) {
    ZKB_ARG(ctx && csf && csf_words >= 18 && g && g_lagrange && out);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    Csf cs;
    ZKB_TRY(load_csf(csf, csf_words, cs));
    ZKB_TRY(check_openings(cs));
    zkb_srs *srs = nullptr;
    ZKB_TRY(srs_create(ctx, cs.k, (const G1Affine *)g, false, (const G1Affine *)g_lagrange, false, &srs));
    const int32_t r = pk_build(ctx, std::move(cs), fixed_values, sigma_values, nullptr, srs, true, out);
    if (r != ZKB_OK) zkb_srs_destroy(srs);
    return r;
}
extern "C" int32_t zkb_pk_create_with_srs(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, const uint64_t *const *fixed_values,
                                          const uint64_t *const *sigma_values, zkb_srs *srs, zkb_pk **out) {
    ZKB_ARG(ctx && csf && srs && out);
    Csf cs;
    ZKB_TRY(load_csf(csf, csf_words, cs));
    ZKB_TRY(check_openings(cs));
    return pk_build(ctx, std::move(cs), fixed_values, sigma_values, nullptr, srs, false, out);
}

// ---- keygen: permutation assembly + sigma columns (plonk/permutation/keygen.rs Assembly::copy, build_pk) -------------------
// sigma_i[j] = DELTA^(mapping column) * omega^(mapping row): the cycle structure is merged on the host exactly like upstream
// (mapping / aux / sizes with union by size -- inherently sequential), the n x P field values are produced on the device.
__global__ void sigma_from_mapping_kernel(const uint32_t *__restrict__ map_col, const uint32_t *__restrict__ map_row, const Fr *__restrict__ omega_pows,
                                          const Fr *__restrict__ delta_pows, uint64_t n, Fr *__restrict__ out) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) fp_store(out + i, fp_mul(fp_load(delta_pows + map_col[i]), fp_load(omega_pows + map_row[i])));
}

// copies: n_copies x 4 u32 = (left column, left row, right column, right row); columns are indices into the CSF's permutation column list
extern "C" int32_t zkb_keygen_pk(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, const uint64_t *const *fixed_values, const uint32_t *copies,
                                 uint64_t n_copies, zkb_srs *srs, zkb_pk **out) {
    ZKB_ARG(ctx && csf && srs && out && (copies || n_copies == 0));
    ZKB_CUDA(cudaSetDevice(ctx->device));
    Csf cs;
    ZKB_TRY(load_csf(csf, csf_words, cs));
    ZKB_TRY(check_openings(cs));
    const uint64_t n = 1ull << cs.k;
    const size_t P = cs.perm.size();
    ZKB_ARG(P * n < (1ull << 32));
    // Assembly: mapping[c][r] = next cell of the cycle, aux = cycle representative, sizes = cycle length at the representative
    std::vector<uint32_t> map_col(P * n), map_row(P * n), aux_col(P * n), aux_row(P * n), sizes(P * n, 1);
    for (size_t c = 0; c < P; ++c)
        for (uint64_t r = 0; r < n; ++r) { map_col[c * n + r] = aux_col[c * n + r] = (uint32_t)c; map_row[c * n + r] = aux_row[c * n + r] = (uint32_t)r; }
    for (uint64_t i = 0; i < n_copies; ++i) {
        const uint32_t lc = copies[4 * i], lr = copies[4 * i + 1], rc = copies[4 * i + 2], rr = copies[4 * i + 3];
        if (lc >= P || rc >= P || lr >= n || rr >= n) { set_error("copy constraint %llu is out of range", (unsigned long long)i); return ZKB_ERR_ARG; }
        const size_t a = lc * n + lr, b = rc * n + rr;
        size_t lcy = aux_col[a] * n + aux_row[a], rcy = aux_col[b] * n + aux_row[b];
        if (lcy == rcy) continue;
        if (sizes[lcy] < sizes[rcy]) std::swap(lcy, rcy);
        sizes[lcy] += sizes[rcy];
        size_t cur = rcy;
        do {   // relabel the smaller cycle
            aux_col[cur] = (uint32_t)(lcy / n);
            aux_row[cur] = (uint32_t)(lcy % n);
            cur = map_col[cur] * n + map_row[cur];
        } while (cur != rcy);
        std::swap(map_col[a], map_col[b]);
        std::swap(map_row[a], map_row[b]);
    }
    cudaStream_t st = ctx->stream;
    DevPool tmp;
    tmp.ctx = ctx;
    uint32_t *d_mc = nullptr, *d_mr = nullptr;
    Fr *d_om = nullptr, *d_dl = nullptr;
    ZKB_TRY(tmp.alloc(P * n * 4 + 4, (void **)&d_mc));
    ZKB_TRY(tmp.alloc(P * n * 4 + 4, (void **)&d_mr));
    ZKB_TRY(tmp.fr(n, &d_om));
    ZKB_TRY(tmp.fr(P + 1, &d_dl));
    ZKB_CUDA(cudaMemcpyAsync(d_mc, map_col.data(), P * n * 4, cudaMemcpyHostToDevice, st));
    ZKB_CUDA(cudaMemcpyAsync(d_mr, map_row.data(), P * n * 4, cudaMemcpyHostToDevice, st));
    Fr omega = host_root_of_unity(cs.k);
    ZKB_TRY(fr_powers_device(ctx, omega, n, d_om, st));
    ZKB_TRY(fr_powers_device(ctx, perm_delta(), P + 1, d_dl, st));
    std::vector<Fr *> sig(P);
    for (size_t c = 0; c < P; ++c) {
        ZKB_TRY(tmp.fr(n, &sig[c]));
        sigma_from_mapping_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_mc + c * n, d_mr + c * n, d_om, d_dl, n, sig[c]);
        ctx->launches++;
    }
    ZKB_CUDA(cudaGetLastError());
    ZKB_CUDA(cudaStreamSynchronize(st));   // host vectors die at return
    return pk_build(ctx, std::move(cs), fixed_values, nullptr, &sig, srs, false, out);
}
// sigma column values of a proving key (n x 32 B each, Lagrange basis) back to the host: lets a caller persist / inspect keygen output
extern "C" int32_t zkb_pk_sigma_read(zkb_pk *pk, uint32_t column, uint64_t *out_host) {
    ZKB_ARG(pk && out_host && column < pk->sigma_values.size());
    ZKB_CUDA(cudaSetDevice(pk->ctx->device));
    ZKB_CUDA(cudaMemcpyAsync(out_host, pk->sigma_values[column], pk->n * sizeof(Fr), cudaMemcpyDeviceToHost, pk->ctx->stream));
    ZKB_CUDA(cudaStreamSynchronize(pk->ctx->stream));
    return ZKB_OK;
}

int32_t zkb::pk_vk_commitments(zkb_pk *pk, std::vector<G1Affine> &out) {
    ZKB_CUDA(cudaSetDevice(pk->ctx->device));
    std::vector<Fr *> cols;
    for (auto c : pk->fixed_values) cols.push_back(c);
    for (auto c : pk->sigma_values) cols.push_back(c);
    out.clear();
    if (!cols.empty()) ZKB_TRY(commit_many(pk, cols, BASIS_LAGRANGE, out, pk->ctx->stream));
    return ZKB_OK;
}

// VerifyingKey::write(SerdeFormat::Processed) (halo2_proofs plonk.rs): u32 BE k || u32 BE num_fixed || fixed commitments ||
// permutation commitments, points compressed -- the layout of the reference fixture's `vk` (aggregator/data/batch-task.json:
// 0x19, 4, 4 + 3 points = 232 B).  Commitments = commit_lagrange of the fixed / sigma columns (keygen.rs), batched MSMs.
extern "C" int32_t zkb_pk_vk_bytes(zkb_pk *pk, uint8_t *out, uint64_t cap, uint64_t *len) {
    ZKB_ARG(pk && len);
    const Csf &cs = pk->cs;
    const uint64_t need = 8 + 32ull * (cs.nf + cs.perm.size());
    *len = need;
    if (!out) return ZKB_OK;
    ZKB_ARG(cap >= need);
    std::vector<G1Affine> cms;
    ZKB_TRY(pk_vk_commitments(pk, cms));
    auto be32 = [](uint8_t *p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; };
    be32(out, cs.k);
    be32(out + 4, cs.nf);
    for (size_t i = 0; i < cms.size(); ++i) g1_compress(cms[i], out + 8 + 32 * i);
    return ZKB_OK;
}

// host-only structural check of a CSF blob (no device needed)
extern "C" int32_t zkb_csf_validate(const uint32_t *csf, uint64_t csf_words) {
    Csf c;
    ZKB_TRY(load_csf(csf, csf_words, c));
    return check_openings(c);
}

extern "C" int32_t zkb_pk_destroy(zkb_pk *pk) {
    if (pk) {
        cudaSetDevice(pk->ctx->device);
        cudaStreamSynchronize(pk->ctx->stream);
        delete pk;
    }
    return ZKB_OK;
}

// ================================================================================================ C ABI: proof session
static int32_t prove_begin_common(zkb_pk *pk, Transcript::Kind transcript_kind, const zkb_transcript_vtable *vt, const uint64_t transcript_repr[4],
                                  const uint64_t *const *instance_values, const uint32_t *instance_lens, zkb_session **out) {
    ZKB_ARG(pk && transcript_repr && out && (pk->cs.ni == 0 || (instance_values && instance_lens)));
    ZKB_CUDA(cudaSetDevice(pk->ctx->device));
    std::unique_ptr<zkb_session> s(new zkb_session());
    s->pk = pk;
    s->tr = Transcript(transcript_kind, vt);
    s->pool.ctx = pk->ctx;
    const Csf &cs = pk->cs;
    const uint64_t n = pk->n;
    cudaStream_t st = pk->ctx->stream;
    Fr repr;
    memcpy(repr.l, transcript_repr, 32);
    s->tr.common_scalar(repr);  // vk.hash_into(transcript)
    s->inst_values.resize(cs.ni);
    s->inst_polys.resize(cs.ni);
    for (uint32_t c = 0; c < cs.ni; ++c) {
        ZKB_ARG(instance_lens[c] <= n - (cs.bf + 1));
        ZKB_TRY(s->pool.fr(n, &s->inst_values[c]));
        ZKB_TRY(s->pool.fr(n, &s->inst_polys[c]));
        ZKB_CUDA(cudaMemsetAsync(s->inst_values[c], 0, n * sizeof(Fr), st));
        for (uint32_t i = 0; i < instance_lens[c]; ++i) {  // KZG: QUERY_INSTANCE = false -> values are absorbed as scalars
            Fr v;
            memcpy(v.l, instance_values[c] + 4 * i, 32);
            s->tr.common_scalar(v);
        }
        if (instance_lens[c]) ZKB_CUDA(cudaMemcpyAsync(s->inst_values[c], instance_values[c], (size_t)instance_lens[c] * sizeof(Fr), cudaMemcpyHostToDevice, st));
        ZKB_TRY(lagrange_to_coeff(pk, s->inst_values[c], s->inst_polys[c], st));
    }
    s->adv_values.assign(cs.na, nullptr);
    s->challenges.assign(cs.nch, Fr::zero());
    ZKB_CUDA(cudaStreamSynchronize(st));
    ZKB_TRY(s->tr.status());
    *out = s.release();
    return ZKB_OK;
}

extern "C" int32_t zkb_prove_begin(zkb_pk *pk, const uint64_t transcript_repr[4], const uint64_t *const *instance_values, const uint32_t *instance_lens,
                                   zkb_session **out) {
    return zkb_prove_begin_ex(pk, Transcript::BLAKE2B, transcript_repr, instance_values, instance_lens, out);
}
extern "C" int32_t zkb_prove_begin_ex(zkb_pk *pk, int32_t transcript_kind, const uint64_t transcript_repr[4], const uint64_t *const *instance_values,
                                      const uint32_t *instance_lens, zkb_session **out) {
    ZKB_ARG(transcript_kind >= Transcript::BLAKE2B && transcript_kind <= Transcript::EVM);
    return prove_begin_common(pk, (Transcript::Kind)transcript_kind, nullptr, transcript_repr, instance_values, instance_lens, out);
}
extern "C" int32_t zkb_prove_begin_cb(zkb_pk *pk, const zkb_transcript_vtable *vt, const uint64_t transcript_repr[4],
                                      const uint64_t *const *instance_values, const uint32_t *instance_lens, zkb_session **out) {
    ZKB_ARG(vt && vt->common_scalar && vt->write_scalar && vt->write_point && vt->squeeze_challenge);
    return prove_begin_common(pk, Transcript::CALLER, vt, transcript_repr, instance_values, instance_lens, out);
}

// Witness-side overlap (SURVEY 8f row 4): `synthesize` assigns sub-circuit after sub-circuit (super_circuit.rs:714-806), so the columns
// of a phase become final one at a time.  The shim may hand each finished column over immediately: the copy runs on the copy stream
// while Rust keeps synthesising, and zkb_prove_advice_phase later finds the column already in HBM (its pointer may then be NULL).
extern "C" int32_t zkb_prove_upload_advice(zkb_session *s, uint32_t column, const uint64_t *values) {
    ZKB_ARG(s && values && column < s->pk->cs.na);
    zkb_pk *pk = s->pk;
    if (s->finished || pk->cs.adv_phase[column] < s->next_phase) { set_error("column %u belongs to a phase that is already committed", column); return ZKB_ERR_STATE; }
    ZKB_CUDA(cudaSetDevice(pk->ctx->device));
    Fr *&d = s->early_cols[column];
    if (!d) ZKB_TRY(s->pool.fr(pk->n, &d));
    ZKB_CUDA(cudaMemcpyAsync(d, values, pk->n * sizeof(Fr), cudaMemcpyDefault, pk->ctx->copy_stream));
    return ZKB_OK;
}

extern "C" int32_t zkb_prove_advice_phase(zkb_session *s, uint32_t phase, const uint64_t *const *advice_columns, uint64_t *challenges_out) {
    ZKB_ARG(s && advice_columns);
    zkb_pk *pk = s->pk;
    const Csf &cs = pk->cs;
    if (phase != s->next_phase || phase >= cs.nphases || s->finished) { set_error("advice phases must be submitted in order"); return ZKB_ERR_STATE; }
    ZKB_CUDA(cudaSetDevice(pk->ctx->device));
    cudaStream_t st = pk->ctx->stream;
    const uint64_t n = pk->n;
    // H2D on the copy stream, batch by batch; the MSM of batch b waits only for batch b's event, so the copies of the
    // following batches overlap it (pinned caller buffers; pageable ones are staged synchronously by the driver anyway).
    // Multi-GPU: a rank uploads and commits only the columns it owns, then the column data is gathered over NVLink.
    std::vector<const uint64_t *> phase_src;
    std::vector<uint32_t> phase_idx;
    for (uint32_t c = 0; c < cs.na; ++c) {
        if (cs.adv_phase[c] != phase) continue;
        auto early = s->early_cols.find(c);
        const uint64_t *src = advice_columns[c] ? advice_columns[c] : (early != s->early_cols.end() ? (const uint64_t *)early->second : nullptr);
        if (!src) { set_error("advice column %u of phase %u was neither passed nor uploaded ahead", c, phase); return ZKB_ERR_ARG; }
        phase_src.push_back(src);   // a staged copy is a device pointer: the gather into the phase slab below is then device-to-device
        phase_idx.push_back(c);
    }
    const size_t ncols = phase_src.size();
    const Deal deal(pk->ctx, ncols);
    Fr *slab = nullptr;
    ZKB_TRY(s->pool.fr(std::max<size_t>(1, deal.padded()) * n, &slab));
    std::vector<Fr *> phase_cols(ncols);
    for (size_t i = 0; i < ncols; ++i) { phase_cols[i] = slab + i * n; s->adv_values[phase_idx[i]] = phase_cols[i]; }
    const bool dealt = deal.on;
    ZKB_CUDA(cudaStreamSynchronize(st));  // the destination block may still be in use by work queued on `st`
    const uint32_t maxb = msm_max_batch(n);
    const size_t nbatch = dealt ? 1 : (ncols + maxb - 1) / maxb;
    struct EventList {   // destroyed on every exit path
        std::vector<cudaEvent_t> v;
        ~EventList() { for (auto e : v) if (e) cudaEventDestroy(e); }
    } evl;
    evl.v.assign(nbatch, nullptr);
    std::vector<cudaEvent_t> &evs = evl.v;
    for (size_t b = 0; b < nbatch; ++b) {
        ZKB_CUDA(cudaEventCreateWithFlags(&evs[b], cudaEventDisableTiming));
        const size_t lo = dealt ? 0 : b * maxb, hi = dealt ? ncols : std::min(ncols, (b + 1) * (size_t)maxb);
        for (size_t i = lo; i < hi; ++i)
            if (deal.mine(i))
                ZKB_CUDA(cudaMemcpyAsync(phase_cols[i], phase_src[i], n * sizeof(Fr), cudaMemcpyDefault, pk->ctx->copy_stream));   // host (pinned or pageable) or device-resident columns
        ZKB_CUDA(cudaEventRecord(evs[b], pk->ctx->copy_stream));
    }
    for (size_t b = 0; b < nbatch; ++b) {
        ZKB_CUDA(cudaStreamWaitEvent(st, evs[b], 0));
        const size_t lo = dealt ? 0 : b * maxb, hi = dealt ? ncols : std::min(ncols, (b + 1) * (size_t)maxb);
        // dealt: the same contiguous blocks as the uploads (same unit count)
        ZKB_TRY(commit_write(s, std::vector<Fr *>(phase_cols.begin() + lo, phase_cols.begin() + hi), BASIS_LAGRANGE, st));
    }
    ZKB_TRY(deal_gather(pk->ctx, deal, slab, n * sizeof(Fr), st));   // column data of the other ranks' blocks over NVLink
    for (uint32_t i = 0; i < cs.nch; ++i) {
        if (cs.ch_phase[i] == phase) {
            s->challenges[i] = s->tr.squeeze();
            if (challenges_out) memcpy(challenges_out + 4 * i, s->challenges[i].l, 32);
        }
    }
    s->next_phase++;
    return s->tr.status();
}

extern "C" int32_t zkb_session_destroy(zkb_session *s) {
    if (s) {
        cudaSetDevice(s->pk->ctx->device);
        cudaStreamSynchronize(s->pk->ctx->stream);
        delete s;
    }
    return ZKB_OK;
}

namespace zkb {

// stage timing (ZKB_TRACE=1): wall clock per create_proof stage after a stream synchronise, printed to stderr
struct StageTrace {
    bool on;
    cudaStream_t st;
    double t0;
    explicit StageTrace(cudaStream_t s) : st(s) {
        const char *e = getenv("ZKB_TRACE");
        on = e && e[0] == '1';
        t0 = now();
    }
    static double now() {
        timespec ts;
        clock_gettime(CLOCK_MONOTONIC, &ts);
        return ts.tv_sec + 1e-9 * ts.tv_nsec;
    }
    void mark(const char *name) {
        if (!on) return;
        cudaStreamSynchronize(st);
        const double t = now();
        fprintf(stderr, "[zkb trace] %-28s %9.3f ms\n", name, (t - t0) * 1e3);
        t0 = t;
    }
};

struct OpenQuery {
    int poly_id;        // identity of the committed polynomial
    const Fr *poly;     // device coefficients (n)
    int64_t rot;        // point = x * omega^rot
};

// what one stage of the proof hands to a later one
struct ProofState {
    Fr theta, beta, gamma, y, x;
    Fr **d_vcols = nullptr;                  // value-domain column table: the SlotMap prefix up to X (omega_pows)
    std::vector<std::vector<Fr *>> lk_f;     // compressed inputs per lookup / input set
    std::vector<Fr *> lk_t, lk_m;            // compressed table, multiplicities per lookup
    std::vector<Fr *> zs, phis;              // permutation grand products per set, lookup grand sums per lookup
    Fr *random_poly = nullptr;
    std::vector<Fr *> adv_polys, z_polys, phi_polys, m_polys;
    Fr *h_ext = nullptr;                     // h on the extended domain; after the inverse transform, qdeg pieces of n coefficients
    std::vector<Fr *> h_group;               // quotient group g's values on zeta D_{mn}, m = 2^g (the top one is h_ext; null: empty)
    std::vector<Fr *> h_pieces;
    std::map<int64_t, Fr> point_of;          // rotation mod n -> x * omega^rot
    std::map<std::pair<int, int64_t>, Fr> eval_of;   // (polynomial, rotation mod n) -> evaluation
    std::vector<OpenQuery> queries;          // multiopen queries in prover.rs order
};

// mv_lookup/prover.rs prepare: theta, compressed inputs and table (interpreter on the Lagrange domain), multiplicities m over the
// usable rows, m commitments.  Multi-GPU: the lookup arguments are dealt and the m columns, one slab, are all-gathered.
static int32_t lookup_prepare(zkb_session *s, ProofState &ps) {
    zkb_pk *pk = s->pk;
    zkb_ctx *ctx = pk->ctx;
    const Csf &cs = pk->cs;
    const uint64_t n = pk->n;
    const uint32_t usable = (uint32_t)(n - cs.bf - 1);
    const size_t nl = cs.lookups.size();
    cudaStream_t st = ctx->stream;
    DevPool &pool = s->pool;
    ps.theta = s->tr.squeeze();
    ps.lk_f.resize(nl);
    ps.lk_t.resize(nl);
    const Deal deal(ctx, nl);
    Fr *m_slab = nullptr;
    ZKB_TRY(dealt_columns(pool, deal, n, ps.lk_m, &m_slab));
    uint32_t *slots = nullptr, mask = 0;
    uint64_t lookup_errors = 0;
    for (size_t l = 0; l < nl; ++l) {
        if (!deal.mine(l)) continue;
        const size_t ns = cs.lookups[l].inputs.size();
        ps.lk_f[l].resize(ns);
        for (auto &f : ps.lk_f[l]) ZKB_TRY(pool.fr(n, &f));
        ZKB_TRY(pool.fr(n, &ps.lk_t[l]));
        ZKB_TRY(lookup_compress(ctx, cs, l, pk->sm, s->challenges, ps.theta, pool, ps.d_vcols, ps.lk_f[l], ps.lk_t[l], st));
        bool unsatisfied = false;
        ZKB_TRY(lookup_multiplicities(ctx, pool, ps.lk_f[l].data(), ns, ps.lk_t[l], n, usable, ps.lk_m[l], slots, mask, &unsatisfied, st));
        if (unsatisfied) {
            set_error("lookup %zu: an input row is not in the table (unsatisfied witness)", l);
            if (!deal.on) return ZKB_ERR_ARG;
            lookup_errors++;   // multi-GPU: every rank must learn about it before anyone leaves the collective sequence
        }
    }
    if (deal.on) {
        ZKB_TRY(deal_gather(ctx, deal, m_slab, n * sizeof(Fr), st));
        uint64_t *d_errw = nullptr;   // every rank learns about an unsatisfied lookup before anyone leaves the collective sequence
        ZKB_TRY(scratch_get(ctx, SCR_COMM_FLAG, 64, (void **)&d_errw));
        ZKB_CUDA(cudaMemcpyAsync(d_errw + 1, &lookup_errors, 8, cudaMemcpyHostToDevice, st));
        ZKB_TRY(comm_allreduce_u64(ctx, d_errw + 1, 1, st));
        uint64_t total_err = 0;
        ZKB_CUDA(cudaMemcpyAsync(&total_err, d_errw + 1, 8, cudaMemcpyDeviceToHost, st));
        ZKB_CUDA(cudaStreamSynchronize(st));
        if (total_err) {
            if (!lookup_errors) set_error("a lookup input row is not in the table (reported by another rank)");
            return ZKB_ERR_ARG;
        }
    }
    return commit_write(s, ps.lk_m, BASIS_LAGRANGE, st);
}

// permutation/prover.rs commit: beta, gamma, the grand product z of every set of `chunk` permutation columns, z commitments
static int32_t permutation_commit(zkb_session *s, ProofState &ps, const uint64_t *z_blinds) {
    zkb_pk *pk = s->pk;
    zkb_ctx *ctx = pk->ctx;
    const Csf &cs = pk->cs;
    const uint64_t n = pk->n;
    const uint32_t bf = cs.bf;
    const Fr one = Fr::one();
    cudaStream_t st = ctx->stream;
    DevPool &pool = s->pool;
    ps.beta = s->tr.squeeze();
    ps.gamma = s->tr.squeeze();
    // Multi-GPU: the sets are dealt.  Upstream chains them (z_i[0] = last value of z_{i-1}), which is sequential; here every set is
    // scanned from 1 and rescaled afterwards by c_i = product of the previous sets' last values -- the same field elements
    // (z_i = c_i * z'_i row by row), with only the nsets last values crossing the ranks before the columns are gathered.
    const Deal deal(ctx, pk->nsets);
    Fr *z_slab = nullptr;
    ZKB_TRY(pool.fr(std::max<size_t>(1, deal.padded()) * n, &z_slab));
    ps.zs.resize(pk->nsets);
    for (uint32_t si = 0; si < pk->nsets; ++si) ps.zs[si] = z_slab + (size_t)si * n;
    Fr *num, *den, *tmp;
    ZKB_TRY(pool.fr(n, &num));
    ZKB_TRY(pool.fr(n, &den));
    ZKB_TRY(pool.fr(n, &tmp));
    std::vector<Fr> lasts(std::max<size_t>(1, deal.padded()), one);
    Fr last_z = one;
    for (uint32_t si = 0; si < pk->nsets; ++si) {
        if (!deal.mine(si)) continue;
        ExprBuilder eb;
        uint32_t nnum = NO_NODE, nden = NO_NODE;
        perm_set_products(cs, pk->sm, pk->chunk, si, ps.beta, ps.gamma, eb, nnum, nden);
        ZKB_TRY(run_store_program(pk->ctx, pk->k, pool, eb, {nnum, nden}, {num, den}, ps.d_vcols, "permutation", st));
        ZKB_TRY(batch_invert_device(ctx, den, tmp, n, st));
        mul_arrays_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(num, tmp, den, n);  // den <- modified values
        ctx->launches++;
        // one GPU: chained exactly like upstream (init = previous last value); dealt: from 1, rescaled below
        ZKB_TRY(prefix_product_device(ctx, den, n, deal.on ? one : last_z, ps.zs[si], st));
        ZKB_CUDA(cudaMemcpyAsync(&last_z, ps.zs[si] + (n - bf - 1), sizeof(Fr), cudaMemcpyDeviceToHost, st));
        ZKB_CUDA(cudaStreamSynchronize(st));
        lasts[si] = last_z;
        if (!deal.on) ZKB_CUDA(cudaMemcpyAsync(ps.zs[si] + (n - bf), z_blinds + 4ull * bf * si, (size_t)bf * sizeof(Fr), cudaMemcpyHostToDevice, st));
    }
    if (deal.on) {
        Fr *d_l = nullptr;
        ZKB_TRY(scratch_get(ctx, SCR_COMM, deal.padded() * sizeof(Fr), (void **)&d_l));
        ZKB_CUDA(cudaMemcpyAsync(d_l, lasts.data(), deal.padded() * sizeof(Fr), cudaMemcpyHostToDevice, st));
        ZKB_TRY(deal_gather(ctx, deal, d_l, sizeof(Fr), st));
        ZKB_CUDA(cudaMemcpyAsync(lasts.data(), d_l, deal.padded() * sizeof(Fr), cudaMemcpyDeviceToHost, st));
        ZKB_CUDA(cudaStreamSynchronize(st));
        Fr c = one;   // c_i = prod_{j < i} last'_j
        for (uint32_t si = 0; si < pk->nsets; ++si) {
            if (deal.mine(si)) {
                if (!(c == one)) { scale_const_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ps.zs[si], c, n); ctx->launches++; }
                ZKB_CUDA(cudaMemcpyAsync(ps.zs[si] + (n - bf), z_blinds + 4ull * bf * si, (size_t)bf * sizeof(Fr), cudaMemcpyHostToDevice, st));
            }
            c = fp_mul(c, lasts[si]);
        }
        ZKB_TRY(deal_gather(ctx, deal, z_slab, n * sizeof(Fr), st));
    }
    return commit_write(s, ps.zs, BASIS_LAGRANGE, st);
}

// mv_lookup/prover.rs commit_grand_sum: phi = prefix sums of sum_j 1/(f_j + beta) - m/(t + beta), all denominators of a lookup
// inverted at once; phi commitments.  Multi-GPU: dealt like the multiplicities.
static int32_t lookup_commit_grand_sum(zkb_session *s, ProofState &ps, const uint64_t *phi_blinds) {
    zkb_pk *pk = s->pk;
    zkb_ctx *ctx = pk->ctx;
    const uint64_t n = pk->n;
    const uint32_t bf = pk->cs.bf;
    const size_t nl = pk->cs.lookups.size();
    cudaStream_t st = ctx->stream;
    DevPool &pool = s->pool;
    const Deal deal(ctx, nl);
    Fr *phi_slab = nullptr;
    ZKB_TRY(dealt_columns(pool, deal, n, ps.phis, &phi_slab));
    for (size_t l = 0; l < nl; ++l) {
        if (!deal.mine(l)) continue;
        const size_t J = ps.lk_f[l].size();
        // denominators (f_j + beta), (t + beta) into one contiguous array, inverted at once
        Fr *dens, *invs, *dterm;
        ZKB_TRY(pool.fr((J + 1) * n, &dens));
        ZKB_TRY(pool.fr((J + 1) * n, &invs));
        ZKB_TRY(pool.fr(n, &dterm));
        std::vector<Fr *> cols = ps.lk_f[l];
        cols.push_back(ps.lk_t[l]);       // slot J
        cols.push_back(ps.lk_m[l]);       // slot J + 1
        for (size_t j = 0; j <= J; ++j) cols.push_back(invs + j * n);  // slots J + 2 ..
        Fr **d_cols = nullptr;
        ZKB_TRY(upload_table(pool, cols, &d_cols, st));
        {
            ExprBuilder eb;
            std::vector<uint32_t> roots;
            std::vector<Fr *> outs;
            for (size_t j = 0; j <= J; ++j) {
                roots.push_back(eb.add(eb.col((uint32_t)j, 0), eb.constant(ps.beta)));
                outs.push_back(dens + j * n);
            }
            ZKB_TRY(run_store_program(pk->ctx, pk->k, pool, eb, roots, outs, d_cols, "lookup sum", st));
        }
        ZKB_TRY(batch_invert_device(ctx, dens, invs, (J + 1) * n, st));
        {
            ExprBuilder eb;
            uint32_t acc = eb.neg(eb.mul(eb.col((uint32_t)J + 1, 0), eb.col((uint32_t)(J + 2 + J), 0)));  // - m / (t + beta)
            for (size_t j = 0; j < J; ++j) acc = eb.add(acc, eb.col((uint32_t)(J + 2 + j), 0));
            ZKB_TRY(run_store_program(pk->ctx, pk->k, pool, eb, {acc}, {dterm}, d_cols, "lookup sum", st));
        }
        ZKB_TRY(prefix_sum_device(ctx, dterm, n, Fr::zero(), ps.phis[l], st));
        ZKB_CUDA(cudaMemcpyAsync(ps.phis[l] + (n - bf), phi_blinds + 4ull * bf * l, (size_t)bf * sizeof(Fr), cudaMemcpyHostToDevice, st));
    }
    if (nl) ZKB_TRY(deal_gather(ctx, deal, phi_slab, n * sizeof(Fr), st));
    return commit_write(s, ps.phis, BASIS_LAGRANGE, st);
}

// vanishing/prover.rs commit: the caller's random polynomial (coefficients) committed against g, then y
static int32_t vanishing_commit(zkb_session *s, ProofState &ps, const uint64_t *random_poly_host) {
    zkb_pk *pk = s->pk;
    cudaStream_t st = pk->ctx->stream;
    ZKB_TRY(s->pool.fr(pk->n, &ps.random_poly));
    ZKB_CUDA(cudaMemcpyAsync(ps.random_poly, random_poly_host, pk->n * sizeof(Fr), cudaMemcpyHostToDevice, st));
    ZKB_TRY(commit_write(s, {ps.random_poly}, BASIS_G, st));
    ps.y = s->tr.squeeze();
    return ZKB_OK;
}

// Lagrange -> coefficient form of `vals` into a new slab.  Multi-GPU: contiguous blocks of columns per rank, one all-gather.
static int32_t to_coeff_dealt(zkb_session *s, const std::vector<Fr *> &vals, std::vector<Fr *> &polys) {
    zkb_pk *pk = s->pk;
    const Deal dc(pk->ctx, vals.size());
    Fr *pslab = nullptr;
    ZKB_TRY(dealt_columns(s->pool, dc, pk->n, polys, &pslab));
    if (vals.empty()) return ZKB_OK;
    std::vector<Fr *> src, dst;
    for (size_t i = 0; i < vals.size(); ++i)
        if (dc.mine(i)) { src.push_back(vals[i]); dst.push_back(polys[i]); }
    if (!src.empty()) ZKB_TRY(ntt_many(pk, src, dst, pk->omega_inv, &pk->n_inv, nullptr, pk->ctx->stream));
    return deal_gather(pk->ctx, dc, pslab, pk->n * sizeof(Fr), pk->ctx->stream);
}
static int32_t coefficient_forms(zkb_session *s, ProofState &ps) {
    ZKB_TRY(to_coeff_dealt(s, s->adv_values, ps.adv_polys));
    ZKB_TRY(to_coeff_dealt(s, ps.zs, ps.z_polys));
    ZKB_TRY(to_coeff_dealt(s, ps.phis, ps.phi_polys));
    return to_coeff_dealt(s, ps.lk_m, ps.m_polys);
}

// The quotient numerator split by degree.  Constraint i of T contributes c_i y^(T-1-i).  A constraint of degree d vanishes on H,
// so c_i / Z_H has degree at most d (n - 1) - n < (d - 1) n: its share of h is fixed by its values on the m n points zeta D_{mn},
// m the smallest power of two >= max(d - 1, 1), at most E.  Those points are the coset parts j = 0 mod E/m (part (E/m) j' has the
// generator zeta w_{mn}^j').  Group g collects the constraints with m = 2^g into a program of its own, keeping the global y order:
// its Horner steps are y^(i - i_prev) (i_prev the group's previous constraint), and the tail y^(T-1-i_last) goes into the STOREACC
// scale.  The groups' h_g add up to h coefficient for coefficient, so the proof does not change.  Putting a constraint in a larger
// group is always correct: a folded selector run takes its highest-degree member's group.  With one group (E = 1) every gap is 1
// and the single program of before comes out unchanged.
struct QuotientGroups {
    ExprBuilder &eb;
    const Fr y;
    const uint32_t E;
    const std::vector<ProgramBuilder *> pb;     // group g (m = 2^g) writes pb[g]; log2(E) + 1 of them
    std::vector<int64_t> last;                  // global index of the group's latest constraint, -1 before its first
    std::vector<uint32_t> count;                // constraints per group
    std::vector<std::vector<uint32_t>> reads;   // per group, nodes whose columns it reads (they decide the coset NTTs)
    int64_t next = 0;                           // global index of the next constraint
    std::string error;

    QuotientGroups(ExprBuilder &eb, const Fr &y, uint32_t E, std::vector<ProgramBuilder *> pb)
        : eb(eb), y(y), E(E), pb(std::move(pb)), last(this->pb.size(), -1), count(this->pb.size(), 0), reads(this->pb.size()) {
        eb.const_slot(y);   // y is the first constant, as the Horner steps are almost all y^1
    }
    uint32_t group_of(uint32_t degree) const {
        const uint32_t need = std::max<uint32_t>(degree, 2) - 1;
        uint32_t g = 0;
        while ((1u << g) < need && (1u << g) < E) ++g;
        return g;
    }
    // y^(gap) for a group's next constraint at global index i; a group's first step multiplies a zero accumulator
    uint32_t step(uint32_t g, int64_t i) { return eb.const_slot(fp_pow_u64(y, last[g] < 0 ? 1 : (uint64_t)(i - last[g]))); }
    bool emit(uint32_t g, const std::vector<ProgramBuilder::Root> &r) {
        if (pb[g]->scope(r)) return true;
        error = pb[g]->error;
        return false;
    }
    // constraints in order, sharing one CSE scope per group (a lookup's three roots: the l_0 / l_last ones have degree 2)
    bool scope(const std::vector<uint32_t> &nodes) {
        std::vector<std::vector<ProgramBuilder::Root>> per(pb.size());
        for (uint32_t v : nodes) {
            const uint32_t g = group_of(eb.degree[v]);
            per[g].push_back({v, ProgramBuilder::HORNER, step(g, next)});
            reads[g].push_back(v);
            last[g] = next++;
            count[g]++;
        }
        for (uint32_t g = 0; g < pb.size(); ++g)
            if (!per[g].empty() && !emit(g, per[g])) return false;
        return true;
    }
    // a folded selector run sel * rests[t]: acc2 Horner-steps by y inside the run, FOLD steps acc by y^(s - i_prev - 1 + r)
    bool run(const std::vector<uint32_t> &rests, uint32_t sel) {
        uint32_t d = 0;
        for (uint32_t v : rests) d = std::max(d, eb.degree[v]);
        const uint32_t g = group_of(eb.degree[sel] + d);
        const int64_t s = next, r = (int64_t)rests.size();
        for (uint32_t v : rests)
            if (!emit(g, {{v, ProgramBuilder::HORNER2, eb.const_slot(y)}})) return false;
        const uint32_t fold = eb.const_slot(fp_pow_u64(y, (uint64_t)(last[g] < 0 ? r : s - last[g] - 1 + r)));
        if (!emit(g, {{sel, ProgramBuilder::FOLD, fold}})) return false;
        reads[g].push_back(sel);
        reads[g].insert(reads[g].end(), rests.begin(), rests.end());
        last[g] = s + r - 1;
        next += r;
        count[g] += (uint32_t)r;
        return true;
    }
    // y^(T-1-i_last) of a non-empty group, once every constraint is in
    Fr tail(uint32_t g) const { return fp_pow_u64(y, (uint64_t)(next - 1 - last[g])); }
};

// Gate polynomials of the quotient program, Horner in y in constraint-system order.  Circuits multiply whole groups of constraints
// by one selector (`q_enable * constraint`), so runs of CONSECUTIVE gates of the form fixed(col, rot) * t_j are folded exactly:
//   (..(acc y + f t_1) y + ..) y + f t_r  =  acc y^r + f (t_1 y^(r-1) + .. + t_r)
// -- the same field element (distributivity is exact mod r), one multiply per gate less than the term-by-term form.
static int32_t quotient_gates(const Csf &cs, const std::vector<Fr> &challenges, QuotientGroups &qg, const SlotMap &sm,
                              std::vector<int64_t> &memo) {
    ExprBuilder &qeb = qg.eb;
    auto selector_split = [&](uint32_t gnode, uint32_t &sel, uint32_t &rest) -> bool {
        const auto &nd = cs.nodes[gnode];
        if (nd[0] != N_MUL) return false;
        for (int side = 0; side < 2; ++side) {
            const uint32_t a = nd[1 + side], b = nd[2 - side];
            if (cs.nodes[a][0] == N_FIXED) { sel = a; rest = b; return true; }
        }
        return false;
    };
    auto same_query = [&](uint32_t a, uint32_t b) { return cs.nodes[a][1] == cs.nodes[b][1] && cs.nodes[a][2] == cs.nodes[b][2]; };
    for (size_t gi = 0; gi < cs.gates.size();) {
        uint32_t sel = 0, rest = 0;
        size_t run = 1;
        if (selector_split(cs.gates[gi], sel, rest)) {
            uint32_t s2 = 0, r2 = 0;
            while (gi + run < cs.gates.size() && run < 4096 && selector_split(cs.gates[gi + run], s2, r2) && same_query(sel, s2)) ++run;
        }
        if (run < 2) {
            if (!qg.scope({translate(cs, cs.gates[gi], qeb, sm, challenges, memo)})) { set_error("gate: %s", qg.error.c_str()); return ZKB_ERR_ARG; }
            ++gi;
            continue;
        }
        // the whole run is translated first: its degree picks the group (the selector is a column: it adds no constant)
        std::vector<uint32_t> rests(run);
        for (size_t t = 0; t < run; ++t) {
            uint32_t s2 = 0, r2 = 0;
            selector_split(cs.gates[gi + t], s2, r2);
            rests[t] = translate(cs, r2, qeb, sm, challenges, memo);
        }
        if (!qg.run(rests, translate(cs, sel, qeb, sm, challenges, memo))) { set_error("gate: %s", qg.error.c_str()); return ZKB_ERR_ARG; }
        gi += run;
    }
    return ZKB_OK;
}

// Lookup input sets combined in coefficient form.  compress_exprs makes an input set of W >= 2 expressions e_c into
// sum_c theta^(W-1-c) e_c.  When every e_c is S * a_c(w^r X) -- one advice-free cofactor S (the same hash-consed node; or no
// cofactor at all), one rotation r -- that sum is S * A(w^r X) with A = sum_c theta^(W-1-c) a_c.  A is formed once from the
// advice polynomials and the quotient reads it as one more slot: one coset NTT per part instead of W, and per row one column
// load and (with S) one product instead of W loads, W products and W - 1 theta steps.  The coset NTT is linear and field
// arithmetic exact, so the values, h and the proof do not change.  A set combines only if none of its columns is read in the quotient other than through combined sets (gates,
// the permutation, tables, sets compressed term by term): such a column keeps its coset NTTs, and A would add one.
struct InputCombos {
    struct Set { int32_t combo = -1; uint32_t cofactor = NO_NODE; int32_t rot = 0; };   // combo -1: compressed term by term
    std::vector<std::vector<Set>> sets;            // [lookup][input set]
    std::vector<std::vector<uint32_t>> columns;    // per combination, its advice columns in order: the slot sm.slots + index
};
static InputCombos lookup_input_combos(const Csf &cs, ExprBuilder &qeb, const SlotMap &sm, const std::vector<Fr> &challenges,
                                       std::vector<int64_t> &memo) {
    // nodes that read an advice or instance cell (operands come before the node that reads them)
    std::vector<char> reads_cells(cs.nodes.size(), 0);
    for (size_t i = 0; i < cs.nodes.size(); ++i) {
        const auto &nd = cs.nodes[i];
        reads_cells[i] = nd[0] == N_ADVICE || nd[0] == N_INSTANCE || (nd[0] >= N_NEG && reads_cells[nd[1]]) ||
                         ((nd[0] == N_ADD || nd[0] == N_MUL) && reads_cells[nd[2]]);
    }
    std::vector<char> elsewhere(cs.na, 0), seen(cs.nodes.size(), 0);   // advice columns read other than through combined sets
    auto read_by = [&](uint32_t root) {
        std::vector<uint32_t> stack{root};
        while (!stack.empty()) {
            const uint32_t v = stack.back();
            stack.pop_back();
            if (seen[v]) continue;
            seen[v] = 1;
            const auto &nd = cs.nodes[v];
            if (nd[0] == N_ADVICE) elsewhere[nd[1]] = 1;
            if (nd[0] >= N_NEG) stack.push_back(nd[1]);
            if (nd[0] == N_ADD || nd[0] == N_MUL) stack.push_back(nd[2]);
        }
    };
    for (uint32_t g : cs.gates) read_by(g);
    for (auto &pc : cs.perm)
        if (pc[0] == N_ADVICE) elsewhere[pc[1]] = 1;
    InputCombos out;
    std::vector<std::vector<std::vector<uint32_t>>> cols(cs.lookups.size());   // a candidate set's columns
    out.sets.resize(cs.lookups.size());
    for (size_t l = 0; l < cs.lookups.size(); ++l) {
        const CsfLookup &lk = cs.lookups[l];
        for (uint32_t v : lk.table) read_by(v);
        out.sets[l].resize(lk.inputs.size());
        cols[l].resize(lk.inputs.size());
        for (size_t i = 0; i < lk.inputs.size(); ++i) {
            const std::vector<uint32_t> &inp = lk.inputs[i];
            InputCombos::Set &set = out.sets[l][i];
            bool ok = inp.size() >= 2;
            for (size_t c = 0; c < inp.size() && ok; ++c) {
                // e_c = Advice(col, rot), or Advice(col, rot) * S / S * Advice(col, rot) with S advice- and instance-free
                const auto &nd = cs.nodes[inp[c]];
                uint32_t adv = inp[c], cof = NO_NODE;
                if (nd[0] == N_MUL) {
                    const int side = cs.nodes[nd[1]][0] == N_ADVICE && !reads_cells[nd[2]] ? 0 : 1;
                    adv = nd[1 + side];
                    cof = nd[2 - side];
                    if (reads_cells[cof]) ok = false;
                }
                if (!ok || cs.nodes[adv][0] != N_ADVICE) { ok = false; break; }
                const uint32_t s = cof == NO_NODE ? NO_NODE : translate(cs, cof, qeb, sm, challenges, memo);
                const int32_t rot = (int32_t)cs.nodes[adv][2];
                if (c == 0) { set.cofactor = s; set.rot = rot; }
                else ok = s == set.cofactor && rot == set.rot;
                cols[l][i].push_back(cs.nodes[adv][1]);
            }
            if (ok) set.combo = 0;
            else for (uint32_t v : inp) read_by(v);
        }
    }
    // a set dropped for a column read elsewhere makes its other columns read elsewhere too
    for (bool changed = true; changed;) {
        changed = false;
        for (size_t l = 0; l < cs.lookups.size(); ++l)
            for (size_t i = 0; i < cols[l].size(); ++i) {
                InputCombos::Set &set = out.sets[l][i];
                if (set.combo < 0 || std::none_of(cols[l][i].begin(), cols[l][i].end(), [&](uint32_t c) { return elsewhere[c]; })) continue;
                set.combo = -1;
                for (uint32_t c : cols[l][i]) elsewhere[c] = 1;
                changed = true;
            }
    }
    // one combination per distinct column tuple, in order of first use
    std::map<std::vector<uint32_t>, int32_t> index;
    for (size_t l = 0; l < cs.lookups.size(); ++l)
        for (size_t i = 0; i < cols[l].size(); ++i) {
            InputCombos::Set &set = out.sets[l][i];
            if (set.combo < 0) continue;
            auto it = index.emplace(cols[l][i], (int32_t)out.columns.size()).first;
            if (it->second == (int32_t)out.columns.size()) out.columns.push_back(cols[l][i]);
            set.combo = it->second;
        }
    return out;
}

// evaluation.rs evaluate_h: the quotient numerator (gates, permutation, lookups, in upstream's y-Horner order) as one program per
// degree group (QuotientGroups), then per coset part j the coset NTTs of the polynomials its groups read that the pk's coset cache
// does not hold, and one interpreter launch per group on the part, x y^(T-1-i_last) / ((zeta w^j)^n - 1)
static int32_t evaluate_h(zkb_session *s, ProofState &ps, StageTrace &trace) {
    zkb_pk *pk = s->pk;
    zkb_ctx *ctx = pk->ctx;
    const Csf &cs = pk->cs;
    const uint64_t n = pk->n;
    const uint32_t k = cs.k;
    const Fr one = Fr::one();
    cudaStream_t st = ctx->stream;
    DevPool &pool = s->pool;
    // the quotient table in coefficient form
    const SlotMap &sm = pk->sm;
    std::vector<Fr *> qpolys = pk_quotient_polys(pk);
    put_columns(qpolys, sm.advice0, ps.adv_polys);
    put_columns(qpolys, sm.instance0, s->inst_polys);
    put_columns(qpolys, sm.z0, ps.z_polys);
    put_columns(qpolys, sm.phi0, ps.phi_polys);
    put_columns(qpolys, sm.m0, ps.m_polys);

    const uint32_t E = pk->E;
    uint32_t G = 1;   // groups m = 1, 2, .., E
    while ((1u << (G - 1)) < E) ++G;
    ExprBuilder qeb;
    std::vector<ProgramBuilder> qpbs(G, ProgramBuilder(qeb));
    std::vector<ProgramBuilder *> qpb_ptrs;
    for (auto &p : qpbs) qpb_ptrs.push_back(&p);
    QuotientGroups qg(qeb, ps.y, E, qpb_ptrs);
    std::vector<int64_t> memo(cs.nodes.size(), -1);
    ZKB_TRY(quotient_gates(cs, s->challenges, qg, sm, memo));
    auto lactive = [&]() { return qeb.sub(qeb.sub(qeb.constant(one), qeb.col(sm.l_last, 0)), qeb.col(sm.l_blind, 0)); };
    if (pk->nsets) {
        const uint32_t z0 = qeb.col(sm.z0, 0), zl = qeb.col(sm.z0 + pk->nsets - 1, 0);
        if (!qg.scope({qeb.mul(qeb.sub(qeb.constant(one), z0), qeb.col(sm.l0, 0))})) return ZKB_ERR_ARG;
        if (!qg.scope({qeb.mul(qeb.sub(qeb.mul(zl, zl), zl), qeb.col(sm.l_last, 0))})) return ZKB_ERR_ARG;
        for (uint32_t i = 1; i < pk->nsets; ++i) {
            const uint32_t t = qeb.mul(qeb.sub(qeb.col(sm.z0 + i, 0), qeb.col(sm.z0 + i - 1, -(int32_t)(cs.bf + 1))), qeb.col(sm.l0, 0));
            if (!qg.scope({t})) return ZKB_ERR_ARG;
        }
        for (uint32_t si = 0; si < pk->nsets; ++si) {
            uint32_t left = qeb.col(sm.z0 + si, 1), right = qeb.col(sm.z0 + si, 0);
            perm_set_products(cs, sm, pk->chunk, si, ps.beta, ps.gamma, qeb, right, left);
            if (!qg.scope({qeb.mul(qeb.sub(left, right), lactive())})) { set_error("permutation: %s", qg.error.c_str()); return ZKB_ERR_ARG; }
        }
    }
    const InputCombos combos = lookup_input_combos(cs, qeb, sm, s->challenges, memo);
    for (size_t l = 0; l < cs.lookups.size(); ++l) {
        const CsfLookup &lk = cs.lookups[l];
        std::vector<uint32_t> fsb;
        for (size_t i = 0; i < lk.inputs.size(); ++i) {
            const InputCombos::Set &set = combos.sets[l][i];
            uint32_t f;
            if (set.combo < 0) f = compress_exprs(cs, lk.inputs[i], qeb, sm, s->challenges, memo, ps.theta);
            else {
                f = qeb.col(sm.slots + (uint32_t)set.combo, set.rot);
                if (set.cofactor != NO_NODE) f = qeb.mul(set.cofactor, f);
            }
            fsb.push_back(qeb.add(f, qeb.constant(ps.beta)));
        }
        const uint32_t tb = qeb.add(compress_exprs(cs, lk.table, qeb, sm, s->challenges, memo, ps.theta), qeb.constant(ps.beta));
        uint32_t prod = fsb[0];
        for (size_t j = 1; j < fsb.size(); ++j) prod = qeb.mul(prod, fsb[j]);
        uint32_t ssum = 0;
        bool have_sum = false;
        for (size_t i = 0; i < fsb.size(); ++i) {
            uint32_t pr = 0;
            bool have = false;
            for (size_t j = 0; j < fsb.size(); ++j) {
                if (j == i) continue;
                pr = have ? qeb.mul(pr, fsb[j]) : fsb[j];
                have = true;
            }
            if (!have) pr = qeb.constant(one);
            ssum = have_sum ? qeb.add(ssum, pr) : pr;
            have_sum = true;
        }
        const uint32_t phi = qeb.col(sm.phi0 + (uint32_t)l, 0), phi_next = qeb.col(sm.phi0 + (uint32_t)l, 1), m = qeb.col(sm.m0 + (uint32_t)l, 0);
        const uint32_t lhs = qeb.mul(qeb.mul(tb, prod), qeb.sub(phi_next, phi));
        const uint32_t rhs = qeb.sub(qeb.mul(tb, ssum), qeb.mul(m, prod));
        if (!qg.scope({qeb.mul(phi, qeb.col(sm.l0, 0)), qeb.mul(phi, qeb.col(sm.l_last, 0)), qeb.mul(qeb.sub(lhs, rhs), lactive())})) {
            set_error("lookup %zu: %s", l, qg.error.c_str());
            return ZKB_ERR_ARG;
        }
    }
    // the combined input columns A = sum_c theta^(W-1-c) a_c in coefficient form, slots sm.slots + index.  Every rank holds every
    // advice polynomial (coefficient_forms all-gathers them), so each forms all of them.  `coefs` lives until the stream is synchronised.
    std::vector<std::vector<Fr>> coefs(combos.columns.size());
    Fr *combo_polys = nullptr;
    if (!combos.columns.empty()) ZKB_TRY(pool.fr(combos.columns.size() * n, &combo_polys));
    for (size_t c = 0; c < combos.columns.size(); ++c) {
        const std::vector<uint32_t> &cols = combos.columns[c];
        std::vector<Fr *> polys(cols.size());
        coefs[c].resize(cols.size());
        Fr p = one;
        for (size_t t = cols.size(); t-- > 0;) {
            polys[t] = ps.adv_polys[cols[t]];
            coefs[c][t] = p;
            p = fp_mul(p, ps.theta);
        }
        ZKB_TRY(lincomb(pk, pool, polys, coefs[c], combo_polys + c * n, false, st));
        qpolys.push_back(combo_polys + c * n);
    }
    ZKB_ARG(qpolys.size() < 65536);
    // group g runs on the coset parts j = 0 mod E/m, m = 2^g: every group on part 0, only the top one (m = E) on the odd parts
    auto on_part = [&](uint32_t g, uint32_t j) { return j % (E >> g) == 0; };
    std::vector<uint32_t> groups;   // the non-empty ones
    for (uint32_t g = 0; g < G; ++g)
        if (qg.count[g]) groups.push_back(g);
    // one program per group.  Its device code buffer holds the body + one trailing STOREACC slot, rewritten per part with the scale
    // t_inv[j] y^(T-1-i_last)
    std::vector<std::vector<uint32_t>> scale_idx(G, std::vector<uint32_t>(E, 0));
    for (uint32_t g : groups) {
        const Fr tail = qg.tail(g);
        for (uint32_t j = 0; j < E; ++j)
            if (on_part(g, j)) scale_idx[g][j] = qeb.const_slot(fp_mul(pk->t_inv[j], tail));
    }
    std::vector<DeviceProgram> qdp(G);
    std::vector<size_t> base_len(G, 0);
    for (uint32_t g : groups) {
        base_len[g] = qpbs[g].code.size();
        qpbs[g].store_acc(0, scale_idx[g][0]);
        ZKB_TRY(upload_program(pool, qpbs[g], qeb, qdp[g], st));
    }
    // slots served from the pk's coset cache
    auto cached = [&](size_t i) { return !pk->coset_cache.empty() && i < pk->coset_cache[0].size() && pk->coset_cache[0][i]; };
    // the largest group reading each slot: a polynomial outside the cache is transformed on that group's parts (a smaller group's
    // parts are a subset of them), and not at all when no constraint reads it
    std::vector<int> reader(qpolys.size(), -1);
    {
        std::vector<char> seen(qeb.nodes.size());
        for (uint32_t g : groups) {
            std::fill(seen.begin(), seen.end(), 0);
            std::vector<char> used(qpolys.size(), 0);
            for (uint32_t v : qg.reads[g]) qeb.columns(v, seen, used);
            for (size_t i = 0; i < used.size(); ++i)
                if (used[i]) reader[i] = (int)g;
        }
    }
    if (trace.on) {
        for (uint32_t g : groups) {
            size_t instrs = 0, ntts = 0;
            for (const Instr &in : qpbs[g].code) instrs += in.op != OP_ARG;
            for (size_t i = 0; i < qpolys.size(); ++i) ntts += !cached(i) && reader[i] == (int)g;
            fprintf(stderr, "[zkb trace] quotient group m = %-2u %6u constraints %7zu instructions/row %5zu coset NTTs\n", 1u << g, qg.count[g],
                    instrs, ntts << g);
        }
    }
    trace.mark("quotient program build+upload");

    // evaluate h part by part: group g's value at zeta w_{mn}^(j' + m i) is h_g[j' + m i], part j = (E/m) j'; the top group's h_g is h_ext
    // one n-element array per polynomial that is transformed; the others are read from the coset cache or by no group
    std::vector<Fr *> qcols(qpolys.size(), nullptr);
    size_t transformed = 0;
    for (size_t i = 0; i < qpolys.size(); ++i) transformed += !cached(i) && reader[i] >= 0;
    Fr *slab, *pows;
    ZKB_TRY(pool.fr(transformed * n, &slab));
    for (size_t i = 0, t = 0; i < qpolys.size(); ++i)
        if (!cached(i) && reader[i] >= 0) qcols[i] = slab + t++ * n;
    ZKB_TRY(pool.fr(n, &pows));
    ZKB_TRY(pool.fr(pk->N, &ps.h_ext));
    ps.h_group.assign(G, nullptr);
    for (uint32_t g : groups) {
        if (g + 1 == G) ps.h_group[g] = ps.h_ext;
        else ZKB_TRY(pool.fr(n << g, &ps.h_group[g]));
    }
    // multi-GPU: coset parts are dealt in contiguous blocks.  A rank writes one n-element row of rows_slab per (part, group on it),
    // parts in order from row rank * blk_rows, so one all-gather of blk_rows rows per rank completes the slab; each group's rows are
    // then interleaved into its order h_g[j' + m i]
    const Deal dq(ctx, E);
    std::vector<std::vector<uint32_t>> row_of(G, std::vector<uint32_t>(E, 0));
    size_t blk_rows = 0;
    Fr *rows_slab = nullptr;
    if (dq.on) {
        std::vector<size_t> next_row(dq.P, 0);   // rows per rank, then the next free row of each rank
        for (uint32_t j = 0; j < E; ++j)
            for (uint32_t g : groups) next_row[j / dq.blk] += on_part(g, j);
        blk_rows = *std::max_element(next_row.begin(), next_row.end());
        for (int r = 0; r < dq.P; ++r) next_row[r] = (size_t)r * blk_rows;
        for (uint32_t j = 0; j < E; ++j)
            for (uint32_t g : groups)
                if (on_part(g, j)) row_of[g][j] = (uint32_t)next_row[j / dq.blk]++;
        ZKB_TRY(pool.fr((size_t)dq.P * blk_rows * n, &rows_slab));
    }
    std::vector<Fr **> d_hout(G, nullptr);
    for (uint32_t g : groups) ZKB_TRY(upload_table(pool, std::vector<Fr *>{dq.on ? rows_slab : ps.h_group[g]}, &d_hout[g], st));
    Fr **d_qcols = nullptr;
    ZKB_TRY(pool.alloc(qcols.size() * sizeof(Fr *) + 8, (void **)&d_qcols));
    for (uint32_t j = 0; j < E; ++j) {
        if (!dq.mine(j)) continue;
        std::vector<Fr *> ntt_src, ntt_dst;
        for (size_t i = 0; i < qpolys.size(); ++i)
            if (!cached(i) && reader[i] >= 0 && on_part((uint32_t)reader[i], j)) { ntt_src.push_back(qpolys[i]); ntt_dst.push_back(qcols[i]); }
        if (!ntt_src.empty()) {
            ZKB_TRY(fr_powers_device(ctx, pk->coset_gen(j), n, pows, st));
            ZKB_TRY(ntt_many(pk, ntt_src, ntt_dst, pk->omega, nullptr, pows, st));
        }
        std::vector<Fr *> cols_j = qcols;
        for (size_t i = 0; i < qpolys.size(); ++i)
            if (cached(i)) cols_j[i] = pk->coset_cache[j][i];
        ZKB_CUDA(cudaMemcpyAsync(d_qcols, cols_j.data(), cols_j.size() * sizeof(Fr *), cudaMemcpyHostToDevice, st));
        std::vector<Instr> tails(G);
        for (uint32_t g : groups) {
            if (!on_part(g, j)) continue;
            tails[g] = Instr{OP_STOREACC, 0, 0, 0, 0u | (scale_idx[g][j] << 8)};
            ZKB_CUDA(cudaMemcpyAsync(qdp[g].code + base_len[g], &tails[g], sizeof(Instr), cudaMemcpyHostToDevice, st));
            const DeviceProgram &dp = qdp[g];
            if (dq.on) ZKB_TRY(expr_run_device(ctx, dp.code, dp.ncode, dp.nregs, d_qcols, dp.consts, d_hout[g], k, 1, (uint32_t)(row_of[g][j] * n), st));
            else ZKB_TRY(expr_run_device(ctx, dp.code, dp.ncode, dp.nregs, d_qcols, dp.consts, d_hout[g], k, 1u << g, j / (E >> g), st));
        }
        ZKB_CUDA(cudaStreamSynchronize(st));  // `tails` and `cols_j` live on the stack
    }
    if (dq.on) {
        ZKB_TRY(comm_allgather(ctx, rows_slab + (size_t)dq.rank * blk_rows * n, rows_slab, blk_rows * n * sizeof(Fr), st));
        std::vector<std::vector<uint32_t>> rows(G);
        for (uint32_t g : groups) {
            for (uint32_t jj = 0; jj < (1u << g); ++jj) rows[g].push_back(row_of[g][jj * (E >> g)]);
            uint32_t *d_rows = nullptr;
            ZKB_TRY(pool.alloc(rows[g].size() * sizeof(uint32_t), (void **)&d_rows));
            ZKB_CUDA(cudaMemcpyAsync(d_rows, rows[g].data(), rows[g].size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
            interleave_rows_kernel<<<(unsigned)(((n << g) + 255) / 256), 256, 0, st>>>(rows_slab, d_rows, ps.h_group[g], k, 1u << g);
            ctx->launches++;
        }
        ZKB_CUDA(cudaStreamSynchronize(st));  // `rows` lives on the stack
    }
    return ZKB_OK;
}

// vanishing/prover.rs construct: extended_to_coeff (inverse NTT over the extended domain with 1/N and the zeta coset undone), the
// qdeg pieces of n coefficients committed against g, then x.  Each smaller quotient group's h_g comes back from zeta D_{mn} with an
// inverse NTT of size m n (1/(mn), zeta undone) and is added into the first m n coefficients.
static int32_t vanishing_construct(zkb_session *s, ProofState &ps) {
    zkb_pk *pk = s->pk;
    cudaStream_t st = pk->ctx->stream;
    const uint32_t G = (uint32_t)ps.h_group.size();
    if (ps.h_group[G - 1]) ZKB_TRY(ntt_fr_device(pk->ctx, ps.h_ext, ps.h_ext, pk->ext_k, pk->ext_omega_inv, &pk->N_inv, 2, nullptr, st));
    else ZKB_CUDA(cudaMemsetAsync(ps.h_ext, 0, pk->N * sizeof(Fr), st));
    std::vector<Fr> mn_inv(G);
    for (uint32_t g = 0; g + 1 < G; ++g) {
        if (!ps.h_group[g]) continue;
        const uint64_t mn = pk->n << g;
        mn_inv[g] = fp_inv(fr_from_u64(mn));
        ZKB_TRY(ntt_fr_device(pk->ctx, ps.h_group[g], ps.h_group[g], pk->k + g, fp_pow_u64(pk->ext_omega_inv, pk->E >> g), &mn_inv[g], 2, nullptr, st));
        ZKB_TRY(zkb_field_binop_dev(pk->ctx, 0, 0, (const uint64_t *)ps.h_ext, (const uint64_t *)ps.h_group[g], (uint64_t *)ps.h_ext, mn, st));
    }
    ZKB_CUDA(cudaStreamSynchronize(st));   // `mn_inv` lives on the stack
    for (uint32_t i = 0; i < pk->qdeg; ++i) ps.h_pieces.push_back(ps.h_ext + (size_t)i * pk->n);
    ZKB_TRY(commit_write(s, ps.h_pieces, BASIS_G, st));
    ps.x = s->tr.squeeze();
    return ZKB_OK;
}

// prover.rs evaluations (with permutation / mv_lookup / vanishing evaluate), batched per rotation and written in upstream's order;
// then the multiopen query list in prover.rs order
static int32_t evaluate_at_x(zkb_session *s, ProofState &ps) {
    zkb_pk *pk = s->pk;
    zkb_ctx *ctx = pk->ctx;
    const Csf &cs = pk->cs;
    const uint64_t n = pk->n;
    const size_t nl = cs.lookups.size();
    cudaStream_t st = ctx->stream;
    DevPool &pool = s->pool;
    // h(X) = sum_i x^(n i) piece_i
    Fr *h_poly;
    ZKB_TRY(pool.fr(n, &h_poly));
    {
        const Fr xn = fp_pow_u64(ps.x, n);
        std::vector<Fr> cf;
        Fr cur = Fr::one();
        for (uint32_t i = 0; i < pk->qdeg; ++i) { cf.push_back(cur); cur = fp_mul(cur, xn); }
        ZKB_TRY(lincomb(pk, pool, ps.h_pieces, cf, h_poly, false, st));
        ZKB_CUDA(cudaStreamSynchronize(st));
    }
    int next_id = 0;
    std::vector<int> adv_id(cs.na), fix_id(cs.nf), sig_id(cs.perm.size()), z_id(pk->nsets), phi_id(nl), m_id(nl);
    for (auto &v : adv_id) v = next_id++;
    for (auto &v : fix_id) v = next_id++;
    for (auto &v : sig_id) v = next_id++;
    for (auto &v : z_id) v = next_id++;
    for (auto &v : phi_id) v = next_id++;
    for (auto &v : m_id) v = next_id++;
    const int h_id = next_id++, rand_id = next_id++;
    const int64_t rot_last = -(int64_t)(cs.bf + 1);
    // rotations r and r + n open a polynomial at the same point (omega^n = 1): SHPLONK's sets are sets of points
    // (construct_intermediate_sets compares point values), so the opening side keys every rotation by r mod n
    const auto at = [n](int64_t rot) { return ((rot % (int64_t)n) + (int64_t)n) % (int64_t)n; };
    // (1) the evaluations written to the transcript, in order; `queries` is built afterwards in the multiopen order
    struct EvalReq { int poly_id; const Fr *poly; int64_t rot; };
    std::vector<EvalReq> reqs;
    for (auto &q : cs.advq) reqs.push_back({adv_id[q[0]], ps.adv_polys[q[0]], q[1]});
    for (auto &q : cs.fixq) reqs.push_back({fix_id[q[0]], pk->fixed_polys[q[0]], q[1]});
    reqs.push_back({rand_id, ps.random_poly, 0});
    for (size_t i = 0; i < cs.perm.size(); ++i) reqs.push_back({sig_id[i], pk->sigma_polys[i], 0});
    for (uint32_t i = 0; i < pk->nsets; ++i) {
        reqs.push_back({z_id[i], ps.z_polys[i], 0});
        reqs.push_back({z_id[i], ps.z_polys[i], 1});
        if (i + 1 != pk->nsets) reqs.push_back({z_id[i], ps.z_polys[i], rot_last});
    }
    for (size_t l = 0; l < nl; ++l) {
        reqs.push_back({phi_id[l], ps.phi_polys[l], 0});
        reqs.push_back({phi_id[l], ps.phi_polys[l], 1});
        reqs.push_back({m_id[l], ps.m_polys[l], 0});
    }
    const size_t n_written = reqs.size();
    reqs.push_back({h_id, h_poly, 0});  // needed by SHPLONK, not written
    // batch by rotation
    std::map<int64_t, std::vector<size_t>> by_rot;
    for (size_t i = 0; i < reqs.size(); ++i) by_rot[reqs[i].rot].push_back(i);
    std::vector<Fr> evals(reqs.size());
    for (auto &kv : by_rot) {
        const Fr pt = fp_mul(ps.x, fr_pow_i64(pk->omega, pk->omega_inv, kv.first));
        ps.point_of[at(kv.first)] = pt;
        std::vector<Fr *> ptrs;
        for (size_t i : kv.second) ptrs.push_back(const_cast<Fr *>(reqs[i].poly));
        Fr **d_p = nullptr;
        ZKB_TRY(upload_table(pool, ptrs, &d_p, st));
        // multi-GPU: the polynomials of a rotation are dealt, the 32-byte results all-gathered
        const Deal de(ctx, ptrs.size());
        std::vector<Fr> res(std::max<size_t>(1, de.padded()));
        if (!de.on) {
            ZKB_TRY(poly_eval_device(ctx, d_p, (uint32_t)ptrs.size(), n, pt, res.data(), st));
        } else {
            const size_t lo = (size_t)de.rank * de.blk, hi = std::min(ptrs.size(), lo + de.blk);
            if (hi > lo) ZKB_TRY(poly_eval_device(ctx, d_p + lo, (uint32_t)(hi - lo), n, pt, res.data() + lo, st));
            Fr *d_r = nullptr;
            ZKB_TRY(scratch_get(ctx, SCR_COMM, de.padded() * sizeof(Fr), (void **)&d_r));
            ZKB_CUDA(cudaMemcpyAsync(d_r + lo, res.data() + lo, de.blk * sizeof(Fr), cudaMemcpyHostToDevice, st));
            ZKB_TRY(deal_gather(ctx, de, d_r, sizeof(Fr), st));
            ZKB_CUDA(cudaMemcpyAsync(res.data(), d_r, de.padded() * sizeof(Fr), cudaMemcpyDeviceToHost, st));
            ZKB_CUDA(cudaStreamSynchronize(st));
        }
        for (size_t t = 0; t < kv.second.size(); ++t) evals[kv.second[t]] = res[t];
    }
    for (size_t i = 0; i < n_written; ++i) s->tr.write_scalar(evals[i]);
    for (size_t i = 0; i < reqs.size(); ++i) ps.eval_of[{reqs[i].poly_id, at(reqs[i].rot)}] = evals[i];

    // (2) multiopen queries in prover.rs order
    auto push_q = [&](int id, const Fr *poly, int64_t rot) { ps.queries.push_back({id, poly, at(rot)}); };
    for (auto &q : cs.advq) push_q(adv_id[q[0]], ps.adv_polys[q[0]], q[1]);
    for (uint32_t i = 0; i < pk->nsets; ++i) { push_q(z_id[i], ps.z_polys[i], 0); push_q(z_id[i], ps.z_polys[i], 1); }
    for (int i = (int)pk->nsets - 2; i >= 0; --i) push_q(z_id[i], ps.z_polys[i], rot_last);
    for (size_t l = 0; l < nl; ++l) { push_q(phi_id[l], ps.phi_polys[l], 0); push_q(phi_id[l], ps.phi_polys[l], 1); push_q(m_id[l], ps.m_polys[l], 0); }
    for (auto &q : cs.fixq) push_q(fix_id[q[0]], pk->fixed_polys[q[0]], q[1]);
    for (size_t i = 0; i < cs.perm.size(); ++i) push_q(sig_id[i], pk->sigma_polys[i], 0);
    push_q(h_id, h_poly, 0);
    push_q(rand_id, ps.random_poly, 0);
    return ZKB_OK;
}

// low-degree interpolant through (points, evals): coefficients, low to high
static std::vector<Fr> interpolate(const std::vector<Fr> &pts, const std::vector<Fr> &evs) {
    const size_t m = pts.size();
    std::vector<Fr> coeffs(m, Fr::zero());
    for (size_t j = 0; j < m; ++j) {
        std::vector<Fr> num{Fr::one()};
        Fr den = Fr::one();
        for (size_t t = 0; t < m; ++t) {
            if (t == j) continue;
            std::vector<Fr> nx(num.size() + 1, Fr::zero());
            for (size_t i = 0; i < num.size(); ++i) {
                nx[i + 1] = fp_add(nx[i + 1], num[i]);
                nx[i] = fp_sub(nx[i], fp_mul(pts[t], num[i]));
            }
            num.swap(nx);
            den = fp_mul(den, fp_sub(pts[j], pts[t]));
        }
        const Fr sc = fp_mul(evs[j], fp_inv(den));
        for (size_t i = 0; i < m; ++i) coeffs[i] = fp_add(coeffs[i], fp_mul(num[i], sc));
    }
    return coeffs;
}
static Fr horner_host(const std::vector<Fr> &c, const Fr &at) {
    Fr acc = Fr::zero();
    for (size_t i = c.size(); i-- > 0;) acc = fp_add(fp_mul(acc, at), c[i]);
    return acc;
}

// multiopen/shplonk/prover.rs: rotation sets (construct_intermediate_sets), numerators sum_j y^j (P_ij - R_ij) divided by each
// set's vanishing polynomial into h_x, its commitment, then the linearisation at u divided by (X - u) and the final commitment
static int32_t shplonk(zkb_session *s, ProofState &ps) {
    zkb_pk *pk = s->pk;
    zkb_ctx *ctx = pk->ctx;
    const uint64_t n = pk->n;
    const Fr one = Fr::one();
    cudaStream_t st = ctx->stream;
    DevPool &pool = s->pool;
    const Fr sy = s->tr.squeeze();
    // construct_intermediate_sets
    struct Commit { int id; const Fr *poly; std::vector<int64_t> rots; };
    std::vector<Commit> cmap;
    std::vector<int64_t> super_rots;
    for (auto &q : ps.queries) {
        if (std::find(super_rots.begin(), super_rots.end(), q.rot) == super_rots.end()) super_rots.push_back(q.rot);
        auto it = std::find_if(cmap.begin(), cmap.end(), [&](const Commit &c) { return c.id == q.poly_id; });
        if (it == cmap.end()) cmap.push_back({q.poly_id, q.poly, {q.rot}});
        else if (std::find(it->rots.begin(), it->rots.end(), q.rot) == it->rots.end()) it->rots.push_back(q.rot);
    }
    auto sort_rots = [&](std::vector<int64_t> &r) { std::sort(r.begin(), r.end(), [&](int64_t a, int64_t b) { return fr_less(ps.point_of[a], ps.point_of[b]); }); };
    sort_rots(super_rots);
    for (auto &c : cmap) sort_rots(c.rots);
    struct RSet { std::vector<int64_t> rots; std::vector<Commit *> comms; };
    std::vector<RSet> rsets;
    for (auto &c : cmap) {
        auto it = std::find_if(rsets.begin(), rsets.end(), [&](const RSet &r) { return r.rots == c.rots; });
        if (it == rsets.end()) rsets.push_back({c.rots, {&c}});
        else it->comms.push_back(&c);
    }
    const Fr sv = s->tr.squeeze();
    Fr *hx, *work, *work2, *d_small;
    ZKB_TRY(pool.fr(n, &hx));
    ZKB_TRY(pool.fr(n, &work));
    ZKB_TRY(pool.fr(n, &work2));
    ZKB_TRY(pool.fr(MAX_POINTS_PER_COLUMN, &d_small));
    ZKB_CUDA(cudaMemsetAsync(hx, 0, n * sizeof(Fr), st));
    std::vector<std::vector<std::vector<Fr>>> r_coeffs(rsets.size());   // [set][commitment] -> interpolant R_ij
    Fr vpow = one;
    for (size_t si = 0; si < rsets.size(); ++si) {
        const RSet &rs = rsets[si];
        std::vector<Fr> pts;
        for (int64_t r : rs.rots) pts.push_back(ps.point_of[r]);
        ZKB_ARG(pts.size() <= MAX_POINTS_PER_COLUMN);   // refused earlier by check_openings; Keccak's hot cell column has 56 points
        // N_i(X) = sum_j y^j (P_ij(X) - R_ij(X))
        std::vector<Fr *> ptrs;
        std::vector<Fr> cf;
        std::vector<Fr> rsum(pts.size(), Fr::zero());
        Fr ypow = one;
        for (Commit *c : rs.comms) {
            std::vector<Fr> evs;
            for (int64_t r : rs.rots) evs.push_back(ps.eval_of[{c->id, r}]);
            r_coeffs[si].push_back(interpolate(pts, evs));
            for (size_t i = 0; i < pts.size(); ++i) rsum[i] = fp_add(rsum[i], fp_mul(r_coeffs[si].back()[i], ypow));
            ptrs.push_back(const_cast<Fr *>(c->poly));
            cf.push_back(ypow);
            ypow = fp_mul(ypow, sy);
        }
        ZKB_TRY(lincomb(pk, pool, ptrs, cf, work, false, st));
        ZKB_CUDA(cudaMemcpyAsync(d_small, rsum.data(), rsum.size() * sizeof(Fr), cudaMemcpyHostToDevice, st));
        sub_low_kernel<<<1, MAX_POINTS_PER_COLUMN, 0, st>>>(work, d_small, (uint32_t)rsum.size());
        ctx->launches++;
        ZKB_CUDA(cudaStreamSynchronize(st));
        // divide by the vanishing polynomial of the set, one root at a time
        Fr *src = work, *dst = work2;
        for (const Fr &p : pts) {
            ZKB_TRY(kate_division_device(ctx, src, n, p, dst, st));
            std::swap(src, dst);
        }
        // h_x += v^i * Q_i
        const std::vector<Fr> vcoef{vpow};
        ZKB_TRY(lincomb(pk, pool, {src}, vcoef, hx, true, st));
        ZKB_CUDA(cudaStreamSynchronize(st));
        vpow = fp_mul(vpow, sv);
    }
    ZKB_TRY(commit_write(s, {hx}, BASIS_G, st));
    const Fr su = s->tr.squeeze();
    // L(X) = sum_i v^i z_i sum_j y^j (P_ij(X) - r_ij) - zt * h_x(X), scaled by 1/z_0, divided by (X - u)
    std::vector<Fr> super_pts;
    for (int64_t r : super_rots) super_pts.push_back(ps.point_of[r]);
    std::vector<Fr> zdiff(rsets.size());
    for (size_t si = 0; si < rsets.size(); ++si) {
        Fr z = one;
        for (size_t t = 0; t < super_rots.size(); ++t) {
            if (std::find(rsets[si].rots.begin(), rsets[si].rots.end(), super_rots[t]) == rsets[si].rots.end()) z = fp_mul(z, fp_sub(su, super_pts[t]));
        }
        zdiff[si] = z;
    }
    Fr zt = one;
    for (auto &p : super_pts) zt = fp_mul(zt, fp_sub(su, p));
    const Fr z0inv = fp_inv(zdiff[0]);
    std::vector<Fr *> ptrs;
    std::vector<Fr> cf;
    Fr const_term = Fr::zero();
    vpow = one;
    for (size_t si = 0; si < rsets.size(); ++si) {
        Fr ypow = one;
        for (size_t ci = 0; ci < rsets[si].comms.size(); ++ci) {
            const Fr w = fp_mul(fp_mul(fp_mul(vpow, zdiff[si]), ypow), z0inv);
            ptrs.push_back(const_cast<Fr *>(rsets[si].comms[ci]->poly));
            cf.push_back(w);
            const_term = fp_add(const_term, fp_mul(w, horner_host(r_coeffs[si][ci], su)));
            ypow = fp_mul(ypow, sy);
        }
        vpow = fp_mul(vpow, sv);
    }
    ptrs.push_back(hx);
    cf.push_back(fp_neg(fp_mul(zt, z0inv)));
    ZKB_TRY(lincomb(pk, pool, ptrs, cf, work, false, st));
    ZKB_CUDA(cudaMemcpyAsync(d_small, &const_term, sizeof(Fr), cudaMemcpyHostToDevice, st));
    sub_low_kernel<<<1, 256, 0, st>>>(work, d_small, 1);
    ctx->launches++;
    ZKB_CUDA(cudaStreamSynchronize(st));
    ZKB_TRY(kate_division_device(ctx, work, n, su, work2, st));
    return commit_write(s, {work2}, BASIS_G, st);
}

// create_proof after the advice phases (plonk/prover.rs), one function per upstream stage, in transcript order
static int32_t prove_finish_stages(zkb_session *s, const uint64_t *z_blinds, const uint64_t *phi_blinds, const uint64_t *random_poly_host) {
    zkb_pk *pk = s->pk;
    ProofState ps;
    StageTrace trace(pk->ctx->stream);
    // the value-domain column table of the lookup compression and the permutation products
    const SlotMap &sm = pk->sm;
    std::vector<Fr *> vcols(sm.x + 1);
    put_columns(vcols, sm.fixed0, pk->fixed_values);
    put_columns(vcols, sm.advice0, s->adv_values);
    put_columns(vcols, sm.instance0, s->inst_values);
    put_columns(vcols, sm.sigma0, pk->sigma_values);
    vcols[sm.x] = pk->omega_pows;
    ZKB_TRY(upload_table(s->pool, vcols, &ps.d_vcols, pk->ctx->stream));
    ZKB_TRY(lookup_prepare(s, ps));
    trace.mark("lookups: compress + m + commit");
    ZKB_TRY(permutation_commit(s, ps, z_blinds));
    trace.mark("permutation z + commit");
    ZKB_TRY(lookup_commit_grand_sum(s, ps, phi_blinds));
    trace.mark("lookup phi + commit");
    ZKB_TRY(vanishing_commit(s, ps, random_poly_host));
    trace.mark("random poly commit");
    ZKB_TRY(coefficient_forms(s, ps));
    trace.mark("lagrange_to_coeff (all columns)");
    ZKB_TRY(evaluate_h(s, ps, trace));   // marks "quotient program build+upload" between the program and the coset parts
    trace.mark("quotient: coset NTTs + fused eval");
    ZKB_TRY(vanishing_construct(s, ps));
    trace.mark("extended iNTT + h commits");
    ZKB_TRY(evaluate_at_x(s, ps));
    trace.mark("evaluations");
    ZKB_TRY(shplonk(s, ps));
    trace.mark("shplonk");
    ZKB_TRY(s->tr.status());
    s->finished = true;
    return ZKB_OK;
}

}  // namespace zkb

extern "C" int32_t zkb_prove_finish(zkb_session *s, const uint64_t *z_blinds, const uint64_t *phi_blinds, const uint64_t *random_poly,
                                    uint8_t *proof_out, uint64_t proof_cap, uint64_t *proof_len) {
    ZKB_ARG(s && proof_len);
    zkb_pk *pk = s->pk;
    if (!s->finished) {
        // first call: run the proof.  The bytes stay in the session, so a query call (proof_out == NULL) or a call with a short
        // buffer loses nothing: call again with a buffer of *proof_len bytes.
        ZKB_ARG(random_poly != nullptr);
        if (s->next_phase != pk->cs.nphases) { set_error("zkb_prove_finish: advice phases incomplete"); return ZKB_ERR_STATE; }
        ZKB_ARG((pk->nsets == 0 || z_blinds) && (pk->cs.lookups.empty() || phi_blinds));
        ZKB_CUDA(cudaSetDevice(pk->ctx->device));
        ZKB_TRY(prove_finish_stages(s, z_blinds, phi_blinds, random_poly));
    }
    const std::vector<uint8_t> &proof = s->tr.proof();
    *proof_len = proof.size();
    if (proof_out) {
        if (proof_cap < proof.size()) { set_error("zkb_prove_finish: buffer of %llu bytes, proof has %llu (kept in the session: call again)",
                                             (unsigned long long)proof_cap, (unsigned long long)proof.size()); return ZKB_ERR_ARG; }
        memcpy(proof_out, proof.data(), proof.size());
    }
    return ZKB_OK;
}

// ================================================================================================ C ABI: constraint interpreter
// The gates of a CSF evaluated over caller columns by the prover's own compiler (translate, ProgramBuilder, quotient_gates) and
// interpreter (expr_run_device): the hot kernel of a proof checked row by row against a reference evaluator.
// The gate program of zkb_expr_eval_dev / zkb_expr_program over the caller's columns, the [fixed | advice | instance] prefix of
// SlotMap.  Mode 0: every gate a STORE root of ONE CSE scope, like the lookup compression programs.  Mode 1: the gate part of
// evaluate_h's quotient program, then one STOREACC with `scale`.
static int32_t gate_program(const Csf &cs, const SlotMap &sm, int32_t mode, const uint64_t *challenges, const uint64_t y[4], const uint64_t scale[4],
                            ExprBuilder &eb, ProgramBuilder &pb) {
    ZKB_ARG(cs.nch == 0 || challenges);
    const std::vector<Fr> ch = host_challenges(challenges, cs.nch);
    std::vector<int64_t> memo(cs.nodes.size(), -1);
    if (mode == 0) {
        std::vector<ProgramBuilder::Root> roots;
        for (size_t i = 0; i < cs.gates.size(); ++i) roots.push_back({translate(cs, cs.gates[i], eb, sm, ch, memo), ProgramBuilder::STORE, (uint32_t)i});
        if (!pb.scope(roots)) { set_error("gates: %s", pb.error.c_str()); return ZKB_ERR_ARG; }
        return ZKB_OK;
    }
    Fr yv, sv;
    memcpy(yv.l, y, sizeof(Fr));
    memcpy(sv.l, scale, sizeof(Fr));
    QuotientGroups qg(eb, yv, 1, {&pb});   // one group: every Horner gap is 1
    ZKB_TRY(quotient_gates(cs, ch, qg, sm, memo));
    pb.store_acc(0, eb.const_slot(sv));
    return ZKB_OK;
}

extern "C" int32_t zkb_expr_eval_dev(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, int32_t mode, const uint64_t *challenges,
                                     const uint64_t y[4], const uint64_t scale[4], const uint64_t *const *columns_dev,
                                     uint64_t *const *outs_dev, uint32_t out_stride, uint32_t out_offset, uint32_t *nregs_out, void *stream) {
    ZKB_ARG(ctx && csf && columns_dev && outs_dev && (mode == 0 || mode == 1));
    ZKB_ARG(mode == 0 ? out_stride == 1 && out_offset == 0 : y && scale && out_stride >= 1);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    Csf cs;
    ZKB_TRY(load_csf(csf, csf_words, cs));
    const SlotMap sm(cs, 0);
    ExprBuilder eb;
    ProgramBuilder pb(eb);
    ZKB_TRY(gate_program(cs, sm, mode, challenges, y, scale, eb, pb));
    cudaStream_t st = pick_stream(ctx, stream);
    const std::vector<Fr *> cols((Fr *const *)columns_dev, (Fr *const *)columns_dev + sm.sigma0);
    std::vector<Fr *> outs(mode == 0 ? cs.gates.size() : 1);
    for (size_t i = 0; i < outs.size(); ++i) outs[i] = (Fr *)outs_dev[i];
    DevPool pool;
    pool.ctx = ctx;
    Fr **d_cols = nullptr, **d_outs = nullptr;
    DeviceProgram dp;
    ZKB_TRY(upload_table(pool, cols, &d_cols, st));
    ZKB_TRY(upload_table(pool, outs, &d_outs, st));
    ZKB_TRY(upload_program(pool, pb, eb, dp, st));
    ZKB_TRY(expr_run_device(ctx, dp.code, dp.ncode, dp.nregs, d_cols, dp.consts, d_outs, cs.k, out_stride, out_offset, st));
    ZKB_CUDA(cudaStreamSynchronize(st));   // the program buffers go back to the context's block cache on return
    if (nregs_out) *nregs_out = (uint32_t)dp.nregs;
    return ZKB_OK;
}

extern "C" int32_t zkb_expr_program(const uint32_t *csf, uint64_t csf_words, int32_t mode, const uint64_t *challenges, const uint64_t y[4],
                                    const uint64_t scale[4], uint64_t *code_out, uint64_t cap, uint64_t *ncode_out, uint32_t *nregs_out) {
    ZKB_ARG(csf && ncode_out && (mode == 0 || mode == 1) && (mode == 0 || (y && scale)) && (code_out || cap == 0));
    Csf cs;
    ZKB_TRY(load_csf(csf, csf_words, cs));
    ExprBuilder eb;
    ProgramBuilder pb(eb);
    ZKB_TRY(gate_program(cs, SlotMap(cs, 0), mode, challenges, y, scale, eb, pb));
    static_assert(sizeof(Instr) == sizeof(uint64_t), "one program word per instruction");
    *ncode_out = pb.code.size();
    if (nregs_out) *nregs_out = (uint32_t)pb.max_regs_used;
    if (cap) memcpy(code_out, pb.code.data(), std::min<uint64_t>(cap, pb.code.size()) * sizeof(Instr));
    return ZKB_OK;
}
