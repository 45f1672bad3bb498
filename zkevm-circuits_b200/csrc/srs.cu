// srs.cu -- ParamsKZG<Bn256> on the device: load once per context, commit against it, downsize it.
//
// Replaces the prover-facing part of halo2_proofs::poly::kzg::commitment::ParamsKZG (halo2_proofs 1.1.0 @ e5ddf67
// src/poly/kzg/commitment.rs): `read_custom` / `setup` products g and g_lagrange, `commit` / `commit_lagrange`
// (= best_multiexp against the stored bases) and `downsize(k)`, which the reference calls whenever a circuit is smaller than
// the loaded parameters (prover/src/common/prover.rs:54-55, aggregator/src/recursion/util.rs:156; params come from
// prover/src/utils.rs load_params).  `g_to_lagrange` (the inverse FFT over G1 that setup / downsize run) is a device kernel
// chain here: log n radix-2 stages on XYZZ points, each butterfly one scalar multiplication by a twiddle.
//
// One zkb_srs per context is shared by every proving key created from it (zkb_pk_create_with_srs): the 64-byte bases are
// uploaded once, and -- memory permitting (ZKB_MSM_SHIFT_GB, default an eighth of the device memory) -- the window-shifted copies 2^(c w) P_i used by the
// one-bucket-set Pippenger variant are built once.
#include "common.cuh"
#include <stdlib.h>
#include <string.h>
#include <memory>

namespace zkb {

// ---- scalar multiplication by a canonical scalar (plain double-and-add; used by the group FFT, not by the MSM) ------------
__device__ __forceinline__ G1Xyzz g1_scalar_mul(const G1Xyzz &p, const Fr &s_canon) {
    G1Xyzz acc = G1Xyzz::identity();
    int top = 253;
    while (top >= 0 && !((s_canon.l[top >> 5] >> (top & 31)) & 1)) --top;
    for (int bit = top; bit >= 0; --bit) {
        acc = g1_dbl(acc);
        if ((s_canon.l[bit >> 5] >> (bit & 31)) & 1) g1_add(acc, p);
    }
    return acc;
}
__device__ __forceinline__ G1Xyzz g1_neg_xyzz(const G1Xyzz &p) {
    G1Xyzz r = p;
    if (!p.is_identity()) r.y = fp_neg(p.y);
    return r;
}

__global__ void g1_affine_to_xyzz_kernel(const G1Affine *__restrict__ in, G1Xyzz *__restrict__ out, uint64_t n) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) g1_store_xyzz(out + i, G1Xyzz::from_affine(g1_load_affine(in + i)));
}
// one DIF stage of the group FFT: (u, v) -> (u + v, (u - v) * w^(j << s)), half = n >> (s + 1); tw holds w^i (canonical), i < n / 2
__global__ void __launch_bounds__(128) g1_fft_stage_kernel(G1Xyzz *__restrict__ a, uint32_t log_n, uint32_t s, const Fr *__restrict__ tw_canon) {
    const uint64_t idx = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (idx >= (1ull << (log_n - 1))) return;
    const uint32_t lh = log_n - s - 1;
    const uint64_t j = idx & ((1ull << lh) - 1), blk = idx >> lh;
    const uint64_t i0 = (blk << (lh + 1)) + j, i1 = i0 + (1ull << lh);
    G1Xyzz u = g1_load_xyzz(a + i0);
    const G1Xyzz v = g1_load_xyzz(a + i1);
    G1Xyzz d = u;
    g1_add(d, g1_neg_xyzz(v));
    g1_add(u, v);
    g1_store_xyzz(a + i0, u);
    const uint64_t e = j << s;
    if (e != 0) d = g1_scalar_mul(d, fp_load(tw_canon + e));
    g1_store_xyzz(a + i1, d);
}
// out[i] = affine(scale * a[bitrev(i)])
__global__ void __launch_bounds__(128) g1_fft_finish_kernel(const G1Xyzz *__restrict__ a, uint32_t log_n, Fr scale_canon, G1Affine *__restrict__ out) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= (1ull << log_n)) return;
    const uint64_t r = log_n ? (__brevll(i) >> (64 - log_n)) : 0;
    g1_store_affine(out + i, g1_to_affine(g1_scalar_mul(g1_load_xyzz(a + r), scale_canon)));
}
__global__ void fr_to_canonical_kernel(Fr *__restrict__ a, uint64_t n) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i < n) fp_store(a + i, fp_to_canonical(fp_load(a + i)));
}

// g_lagrange = g_to_lagrange(g, k): inverse FFT over the group with omega_k^-1, times 1/n (poly/kzg/commitment.rs)
static int32_t g_to_lagrange_device(zkb_ctx *ctx, const G1Affine *g, uint32_t k, G1Affine *out, cudaStream_t st) {
    const uint64_t n = 1ull << k;
    void *scr = nullptr;
    const size_t tw_n = n > 1 ? n / 2 : 1;
    ZKB_TRY(scratch_get(ctx, SCR_MSM_C, n * sizeof(G1Xyzz) + tw_n * sizeof(Fr), &scr));
    G1Xyzz *work = (G1Xyzz *)scr;
    Fr *tw = (Fr *)(work + n);
    const Fr w_inv = fp_inv(host_root_of_unity(k));
    ZKB_TRY(fr_powers_device(ctx, w_inv, tw_n, tw, st));
    fr_to_canonical_kernel<<<(unsigned)((tw_n + 255) / 256), 256, 0, st>>>(tw, tw_n);
    g1_affine_to_xyzz_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g, work, n);
    ctx->launches += 2;
    for (uint32_t s = 0; s < k; ++s) {
        g1_fft_stage_kernel<<<(unsigned)((n / 2 + 127) / 128), 128, 0, st>>>(work, k, s, tw);
        ctx->launches++;
    }
    const Fr n_inv = fp_to_canonical(fp_inv(fp_from_u64<FrParams>(n)));
    g1_fft_finish_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(work, k, n_inv, out);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

static int32_t srs_alloc(zkb_srs *s, size_t bytes, void **out) {
    size_t got = 0;
    ZKB_TRY(block_alloc(s->ctx, bytes, out, &got));
    s->blocks.push_back({*out, got});
    return ZKB_OK;
}
static void srs_free(zkb_srs *s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    cudaStreamSynchronize(s->ctx->stream);
    for (auto &b : s->blocks) block_free(s->ctx, b.first, b.second);
    delete s;
}
// window-shifted copies unless they would exceed ZKB_MSM_SHIFT_GB (default: an eighth of the device memory, 10 GB on an 80 GB
// H100) in total
static int32_t srs_build_shifted(zkb_srs *s, cudaStream_t st) {
    const uint32_t copies = msm_shift_copies(s->n);
    const char *env = getenv("ZKB_MSM_SHIFT_GB");
    const double budget = env ? atof(env) * 1e9 : 0.125 * (double)s->ctx->mem_bytes;
    if (copies && 2.0 * copies * s->n * sizeof(G1Affine) <= budget) {
        ZKB_TRY(srs_alloc(s, (size_t)copies * s->n * sizeof(G1Affine), (void **)&s->g_shift));
        ZKB_TRY(srs_alloc(s, (size_t)copies * s->n * sizeof(G1Affine), (void **)&s->g_lagrange_shift));
        ZKB_TRY(msm_build_shifted_bases(s->ctx, s->g, s->n, s->g_shift, st));
        ZKB_TRY(msm_build_shifted_bases(s->ctx, s->g_lagrange, s->n, s->g_lagrange_shift, st));
    }
    return ZKB_OK;
}

// host or device sources; g_lagrange == nullptr -> derived on the device
int32_t srs_create(zkb_ctx *ctx, uint32_t k, const G1Affine *g, bool g_on_device, const G1Affine *g_lagrange, bool gl_on_device, zkb_srs **out) {
    ZKB_ARG(ctx && g && out && k <= 28);
    std::unique_ptr<zkb_srs, void (*)(zkb_srs *)> s(new zkb_srs(), srs_free);
    s->ctx = ctx;
    s->k = k;
    s->n = 1ull << k;
    cudaStream_t st = ctx->stream;
    const size_t bytes = s->n * sizeof(G1Affine);
    ZKB_TRY(srs_alloc(s.get(), bytes, (void **)&s->g));
    ZKB_TRY(srs_alloc(s.get(), bytes, (void **)&s->g_lagrange));
    ZKB_CUDA(cudaMemcpyAsync(s->g, g, bytes, g_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    if (g_lagrange) ZKB_CUDA(cudaMemcpyAsync(s->g_lagrange, g_lagrange, bytes, gl_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    else ZKB_TRY(g_to_lagrange_device(ctx, s->g, k, s->g_lagrange, st));
    ZKB_TRY(srs_build_shifted(s.get(), st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    *out = s.release();
    return ZKB_OK;
}

// `batch` commitments against one basis of the SRS (ParamsKZG::commit / commit_lagrange), shifted copies when present.
// cols: HOST array of device pointers, len scalars each (len <= n; shifted copies only serve len == n).
int32_t srs_commit_many(zkb_srs *s, int basis, const Fr *const *cols, uint32_t count, uint64_t len, G1Affine *out_host, cudaStream_t st) {
    ZKB_ARG(s && (basis == 0 || basis == 1) && len <= s->n);
    zkb_ctx *ctx = s->ctx;
    const G1Affine *bases = basis == 0 ? s->g : s->g_lagrange;
    const G1Affine *shift = (len == s->n) ? (basis == 0 ? s->g_shift : s->g_lagrange_shift) : nullptr;
    const uint32_t maxb = msm_max_batch(len);
    for (uint32_t done = 0; done < count; done += maxb) {
        const uint32_t cur = count - done < maxb ? count - done : maxb;
        const Fr **d_tbl = nullptr;
        ZKB_TRY(scratch_get(ctx, SCR_MSM_TBL, 64 * sizeof(Fr *), (void **)&d_tbl));
        ZKB_CUDA(cudaMemcpyAsync(d_tbl, cols + done, cur * sizeof(Fr *), cudaMemcpyHostToDevice, st));
        ZKB_TRY(msm_g1_batch_device_ex(ctx, d_tbl, cur, shift ? shift : bases, len, out_host + done, shift != nullptr, st));
    }
    return ZKB_OK;
}

}  // namespace zkb
using namespace zkb;

extern "C" int32_t zkb_srs_load(zkb_ctx *ctx, uint32_t k, const uint64_t *g_host, const uint64_t *g_lagrange_host, zkb_srs **out) {
    ZKB_ARG(ctx && g_host && out);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    return srs_create(ctx, k, (const G1Affine *)g_host, false, (const G1Affine *)g_lagrange_host, false, out);
}
extern "C" int32_t zkb_srs_load_dev(zkb_ctx *ctx, uint32_t k, const uint64_t *g_dev, const uint64_t *g_lagrange_dev, zkb_srs **out) {
    ZKB_ARG(ctx && g_dev && out);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    return srs_create(ctx, k, (const G1Affine *)g_dev, true, (const G1Affine *)g_lagrange_dev, true, out);
}
extern "C" int32_t zkb_srs_destroy(zkb_srs *srs) {
    srs_free(srs);
    return ZKB_OK;
}
extern "C" uint32_t zkb_srs_k(const zkb_srs *srs) { return srs ? srs->k : 0; }

// ParamsKZG::downsize(new_k): g is truncated to 2^new_k points, g_lagrange is recomputed from it (g_to_lagrange)
extern "C" int32_t zkb_srs_downsize(zkb_srs *srs, uint32_t new_k, zkb_srs **out) {
    ZKB_ARG(srs && out && new_k <= srs->k);
    ZKB_CUDA(cudaSetDevice(srs->ctx->device));
    if (new_k == srs->k) return srs_create(srs->ctx, new_k, srs->g, true, srs->g_lagrange, true, out);
    return srs_create(srs->ctx, new_k, srs->g, true, nullptr, true, out);
}
// read back one basis (2^k x 64 B): 0 = g, 1 = g_lagrange
extern "C" int32_t zkb_srs_read(zkb_srs *srs, int32_t basis, uint64_t *out_host) {
    ZKB_ARG(srs && out_host && (basis == 0 || basis == 1));
    ZKB_CUDA(cudaSetDevice(srs->ctx->device));
    ZKB_CUDA(cudaMemcpyAsync(out_host, basis == 0 ? srs->g : srs->g_lagrange, srs->n * sizeof(G1Affine), cudaMemcpyDeviceToHost, srs->ctx->stream));
    ZKB_CUDA(cudaStreamSynchronize(srs->ctx->stream));
    return ZKB_OK;
}
static void srs_emit(const G1Affine &r, uint64_t out_affine[8], uint8_t *out_compressed) {
    memcpy(out_affine, &r, 64);
    if (out_compressed) g1_compress(r, out_compressed);
}
extern "C" int32_t zkb_srs_commit_dev(zkb_srs *srs, int32_t basis, const uint64_t *scalars_dev, uint64_t n, uint64_t out_affine[8], uint8_t *out_compressed,
                                      void *stream) {
    ZKB_ARG(srs && out_affine && (n == 0 || scalars_dev));
    ZKB_CUDA(cudaSetDevice(srs->ctx->device));
    G1Affine r;
    const Fr *col = (const Fr *)scalars_dev;
    if (n == 0) memset(&r, 0, sizeof(r));
    else ZKB_TRY(srs_commit_many(srs, basis, &col, 1, n, &r, pick_stream(srs->ctx, stream)));
    srs_emit(r, out_affine, out_compressed);
    return ZKB_OK;
}
extern "C" int32_t zkb_srs_commit_host(zkb_srs *srs, int32_t basis, const uint64_t *scalars_host, uint64_t n, uint64_t out_affine[8], uint8_t *out_compressed) {
    ZKB_ARG(srs && out_affine && (n == 0 || scalars_host));
    ZKB_CUDA(cudaSetDevice(srs->ctx->device));
    void *ds = nullptr;
    if (n) {
        ZKB_TRY(scratch_get(srs->ctx, SCR_HOSTIO_A, n * 32, &ds));
        ZKB_CUDA(cudaMemcpyAsync(ds, scalars_host, n * 32, cudaMemcpyHostToDevice, srs->ctx->stream));
    }
    return zkb_srs_commit_dev(srs, basis, (const uint64_t *)ds, n, out_affine, out_compressed, srs->ctx->stream);
}
// `batch` columns of n scalars each against one basis in one pass (all advice columns of a phase): scalar_cols_dev is a HOST array
// of device pointers; out_affine receives batch x 8 limbs
extern "C" int32_t zkb_srs_commit_batch_dev(zkb_srs *srs, int32_t basis, const uint64_t *const *scalar_cols_dev, uint32_t batch, uint64_t n,
                                            uint64_t *out_affine, void *stream) {
    ZKB_ARG(srs && scalar_cols_dev && out_affine && batch >= 1 && n >= 1);
    ZKB_CUDA(cudaSetDevice(srs->ctx->device));
    return srs_commit_many(srs, basis, (const Fr *const *)scalar_cols_dev, batch, n, (G1Affine *)out_affine, pick_stream(srs->ctx, stream));
}
