/*
 * zkb200.h -- C ABI of libzkb200.so, the H100 (sm_90a) Halo2/KZG proving backend.
 *
 * This is the boundary a fork-shaped `halo2_proofs` crate binds to (SURVEY.md section 8b): the reference swaps its
 * prover backend at crate level (docker/testool/gpu/Dockerfile:7, cargo `paths` override of halo2_proofs), and the
 * bodies of the upstream functions named below call these entry points instead of their rayon loops.  The
 * reference-side call sites that reach them: circuit-benchmarks/src/super_circuit.rs:117-132 (create_proof),
 * prover/src/common/prover/utils.rs:31 (gen_snark_shplonk), prover/src/common/prover/utils.rs:55 (keygen_pk2).
 *
 * Conventions (precedent: geth-utils/src/lib.rs:9-14 -- plain C types, explicit ownership):
 *   - every function returns int32_t: 0 = ok, negative = error; zkb_last_error() gives a thread-local message.
 *   - field elements / points are caller-owned buffers in halo2curves' in-memory layout (halo2curves 0.1.0 @ a495a7b):
 *       Fr, Fq   : 4 x u64 little-endian limbs, Montgomery form (a * 2^256 mod p), fully reduced, 32 B
 *       G1Affine : x || y, 64 B, identity = (0, 0)          G1 (projective) : x || y || z Jacobian, 96 B, identity z = 0
 *     so Rust passes `slice.as_ptr()` with no conversion.
 *   - `*_host` entry points take HOST pointers and include the H2D / D2H copies; `*_dev` take DEVICE pointers and a
 *     CUDA stream (as void*, NULL = the context's stream) and never synchronise unless stated.
 *   - opaque handles are created / destroyed explicitly; one proof at a time per context (the reference serialises
 *     proving behind a Mutex<Prover>: prover/src/test/inner.rs:20-30).
 *   - There is NO CPU fallback: without a CUDA device every compute entry point fails with ZKB_ERR_CUDA.
 */
#ifndef ZKB200_H
#define ZKB200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define ZKB_API __attribute__((visibility("default")))
#else
#define ZKB_API
#endif

#define ZKB_OK 0
#define ZKB_ERR_CUDA (-1)    /* CUDA runtime failure or no device */
#define ZKB_ERR_ARG (-2)     /* invalid argument */
#define ZKB_ERR_ALLOC (-3)   /* device memory exhausted */
#define ZKB_ERR_STATE (-4)   /* call sequence violated */

typedef struct zkb_ctx zkb_ctx;

/* ---- context ------------------------------------------------------------------------------------------- */
/* Create a context on CUDA device `device` (one context per GPU / per process rank). */
ZKB_API int32_t zkb_init(int32_t device, zkb_ctx **out);
ZKB_API int32_t zkb_destroy(zkb_ctx *ctx);
ZKB_API const char *zkb_last_error(void);
/* ABI version of this header: major << 16 | minor */
ZKB_API uint32_t zkb_version(void);
/* Number of kernel launches issued through this context so far (bench.py's `gpu_launches`). */
ZKB_API uint64_t zkb_launch_count(const zkb_ctx *ctx);
ZKB_API int32_t zkb_sync(zkb_ctx *ctx);
/* Device time per kernel class, measured with CUDA event pairs on the launching stream (off by default).  cls: 0 ntt_tile_kernel,
 * 1 msm_acc_chunk_kernel, 2 expr_kernel; the phases of zkb_check_witness_dev: 4 gate flags, 5 lookup flags (with the compression
 * programs, which also count under 2), 6 copy flags, 7 counting and record extraction.  zkb_prof_read synchronises on the recorded events; reset != 0 clears the counters. */
ZKB_API int32_t zkb_prof_enable(zkb_ctx *ctx, int32_t on);
ZKB_API int32_t zkb_prof_read(zkb_ctx *ctx, int32_t cls, uint64_t *launches, double *ms, int32_t reset);
/* Stream the context launches on (cudaStream_t as void*), for event timing by the caller. */
ZKB_API void *zkb_stream(zkb_ctx *ctx);

/* ---- device memory (thin wrappers so a non-CUDA host language can own device buffers) --------------------- */
ZKB_API int32_t zkb_malloc(zkb_ctx *ctx, uint64_t bytes, void **dptr);
ZKB_API int32_t zkb_free(zkb_ctx *ctx, void *dptr);
ZKB_API int32_t zkb_h2d(zkb_ctx *ctx, void *dst_dev, const void *src_host, uint64_t bytes);
ZKB_API int32_t zkb_d2h(zkb_ctx *ctx, void *dst_host, const void *src_dev, uint64_t bytes);

/* ---- NTT over Fr ------------------------------------------------------------------------------------------
 * Replaces halo2_proofs::arithmetic::best_fft(a: &mut [Fr], omega: Fr, log_n: u32)   (halo2_proofs 1.1.0 @ e5ddf67
 * src/arithmetic.rs) : in place, natural order in and out, a'[k] = sum_j a[j] * omega^(j k).  omega must have
 * order exactly 2^log_n.  If `scale` is non-NULL every output is additionally multiplied by *scale (Montgomery Fr) --
 * this fuses EvaluationDomain::ifft's `ifft_divisor` (src/poly/domain.rs `lagrange_to_coeff`, `extended_to_coeff`).
 * If `coset_zeta` != 0 the input coefficient i is first multiplied by ZETA^(i mod 3) (coset_zeta = 1) or
 * ZETA^(-(i mod 3)) applied to the OUTPUT (coset_zeta = 2), fusing `distribute_powers_zeta` of coeff_to_extended /
 * extended_to_coeff.                                                                                         */
ZKB_API int32_t zkb_ntt_fr_host(zkb_ctx *ctx, uint64_t *data_host, uint32_t log_n, const uint64_t omega[4],
                        const uint64_t *scale /* 4 limbs or NULL */, int32_t coset_zeta);
ZKB_API int32_t zkb_ntt_fr_dev(zkb_ctx *ctx, uint64_t *data_dev, uint32_t log_n, const uint64_t omega[4],
                       const uint64_t *scale /* HOST pointer, 4 limbs or NULL */, int32_t coset_zeta, void *stream);
/* `count` in-place transforms of one size through ONE kernel launch per pass (all columns of a prover stage): cols_dev is a HOST
 * array of `count` device pointers.                                                                                              */
ZKB_API int32_t zkb_ntt_fr_batch_dev(zkb_ctx *ctx, uint64_t *const *cols_dev, uint32_t count, uint32_t log_n, const uint64_t omega[4],
                                     const uint64_t *scale /* HOST pointer or NULL */, int32_t coset_zeta, void *stream);
/* omega_k = Fr::ROOT_OF_UNITY^(2^(28-k)) and its inverse (EvaluationDomain::new); host-side helper. */
ZKB_API int32_t zkb_fr_root_of_unity(uint32_t k, uint64_t omega[4], uint64_t omega_inv[4]);

/* ---- MSM over G1 -------------------------------------------------------------------------------------------
 * Replaces halo2_proofs::arithmetic::best_multiexp(coeffs: &[Fr], bases: &[G1Affine]) -> G1, the body of
 * ParamsKZG::commit / commit_lagrange (src/poly/kzg/commitment.rs).  out = sum_i coeffs[i] * bases[i].
 * The result is returned normalised: out_affine (64 B) and, if non-NULL, out_jacobian (96 B, z = 1 or identity) and
 * out_compressed (32 B, G1Affine::to_bytes: LE x with (y & 1) << 6 in byte 31; identity = zeros).               */
ZKB_API int32_t zkb_msm_g1_host(zkb_ctx *ctx, const uint64_t *scalars_host, const uint64_t *bases_host, uint64_t n,
                        uint64_t out_affine[8], uint64_t *out_jacobian, uint8_t *out_compressed);
ZKB_API int32_t zkb_msm_g1_dev(zkb_ctx *ctx, const uint64_t *scalars_dev, const uint64_t *bases_dev, uint64_t n,
                       uint64_t out_affine[8], uint64_t *out_jacobian, uint8_t *out_compressed, void *stream);
/* `batch` MSMs over the SAME bases in one pass (all advice columns of a phase are committed this way): scalar_cols_dev is a
 * HOST array of `batch` device pointers (n scalars each); out_affine receives batch x 8 limbs.                              */
ZKB_API int32_t zkb_msm_g1_batch_dev(zkb_ctx *ctx, const uint64_t *const *scalar_cols_dev, uint32_t batch,
                                     const uint64_t *bases_dev, uint64_t n, uint64_t *out_affine, void *stream);
/* Number of bucket additions + reduction additions the last MSM on this context performed (G1-adds metric). */
ZKB_API uint64_t zkb_msm_last_adds(const zkb_ctx *ctx);
/* Bucket-reduction levels beyond the first that the last MSM actually executed (decided on the device, no host round trip). */
ZKB_API uint32_t zkb_msm_last_levels(const zkb_ctx *ctx);

/* out[i] = [scalars[i]] * base, affine outputs (device buffers).  A plain double-and-add with one inversion per point: the
 * independent reference zkb_srs_setup_dev is tested against, and the source of distinct benchmark bases.  Not the setup path. */
ZKB_API int32_t zkb_g1_fixed_base_mul_dev(zkb_ctx *ctx, const uint64_t base_affine_host[8], const uint64_t *scalars_dev,
                                  uint64_t n, uint64_t *out_affine_dev, void *stream);

/* ---- SRS handle: ParamsKZG<Bn256> resident on the device ---------------------------------------------------------------
 * Replaces the prover-facing part of halo2_proofs::poly::kzg::commitment::ParamsKZG (src/poly/kzg/commitment.rs): the
 * reference loads one params file per degree (prover/src/utils.rs load_params, prover/src/common/prover.rs:37-57) and
 * `downsize`s it for smaller circuits (prover/src/common/prover.rs:54-55, aggregator/src/recursion/util.rs:156).
 * zkb_srs_load       upload g / g_lagrange (2^k x 64 B each, halo2curves G1Affine layout) ONCE per context; g_lagrange may be
 *                    NULL: it is then derived on the device by the inverse FFT over G1 (`g_to_lagrange`).  Memory permitting
 *                    (ZKB_MSM_SHIFT_GB, default 1/8 of device memory) the window-shifted copies 2^(c w) P_i of both bases are built, which turns
 *                    every commitment into ONE bucket set with no Horner pass (msm.cu).
 * zkb_srs_downsize   ParamsKZG::downsize(new_k): g truncated to 2^new_k, g_lagrange recomputed; the source handle stays valid.
 * zkb_srs_commit_*   ParamsKZG::commit (basis 0, coefficients against g) / commit_lagrange (basis 1, values against g_lagrange);
 *                    n <= 2^k scalars; the result is normalised like zkb_msm_g1_*.
 * zkb_srs_read       copy one basis back to the host (tests, writing a downsized params file).                                    */
typedef struct zkb_srs zkb_srs;
ZKB_API int32_t zkb_srs_load(zkb_ctx *ctx, uint32_t k, const uint64_t *g_host, const uint64_t *g_lagrange_host, zkb_srs **out);
ZKB_API int32_t zkb_srs_load_dev(zkb_ctx *ctx, uint32_t k, const uint64_t *g_dev, const uint64_t *g_lagrange_dev, zkb_srs **out);
ZKB_API int32_t zkb_srs_destroy(zkb_srs *srs);
ZKB_API uint32_t zkb_srs_k(const zkb_srs *srs);
ZKB_API int32_t zkb_srs_downsize(zkb_srs *srs, uint32_t new_k, zkb_srs **out);
ZKB_API int32_t zkb_srs_read(zkb_srs *srs, int32_t basis, uint64_t *out_host);
ZKB_API int32_t zkb_srs_commit_dev(zkb_srs *srs, int32_t basis, const uint64_t *scalars_dev, uint64_t n, uint64_t out_affine[8],
                                   uint8_t *out_compressed, void *stream);
ZKB_API int32_t zkb_srs_commit_host(zkb_srs *srs, int32_t basis, const uint64_t *scalars_host, uint64_t n, uint64_t out_affine[8],
                                    uint8_t *out_compressed);
ZKB_API int32_t zkb_srs_commit_batch_dev(zkb_srs *srs, int32_t basis, const uint64_t *const *scalar_cols_dev, uint32_t batch, uint64_t n,
                                         uint64_t *out_affine, void *stream);

/* ---- SRS generation: ParamsKZG::unsafe_setup_with_s (and setup / new, whose s the caller draws) --------------------------------------
 * zkb_srs_setup_dev   g[i] = [s^i] G1 and g_lagrange[i] = [L_i(s)] G1 for i < 2^k, L_i(s) = w^i (s^n - 1) / (n (s - w^i)), G1 = (1, 2),
 *                     written as 2^k x 64 B affine points to two device buffers (16-byte aligned).  s is a HOST Montgomery Fr whose
 *                     stored integer is < r; k <= 28.  A violation returns ZKB_ERR_ARG before any launch and leaves the outputs
 *                     untouched.  Scratch (2 * 2^k x 32 B of scalars and the comb table) comes from the context's block cache and is
 *                     returned before the call returns; synchronises `stream`.  The same inputs give the same bytes on every run.
 *                     Deviation from upstream: when s^n = 1 (s = w^j, e.g. s = 1 or s = r - 1), upstream's invert().unwrap() panics;
 *                     here g_lagrange is the true Lagrange basis, g_lagrange[j] = G1 and every other entry (0, 0), which equals
 *                     what downsize's group iFFT derives from g.
 * zkb_srs_setup_dev reads ZKB_SETUP_WINDOW_BITS (6, 7, 8, 10, 12 default) and ZKB_SETUP_TABLE_SMEM (1: comb table in shared memory,
 *                     c <= 7) to select a comb variant; every variant computes the same bytes.
 * zkb_g2_setup_host   g2_out = the G2 generator, s_g2_out = [s] g2, raw 128-byte points in the layout of zkb_g2_*_host (x.c0, x.c1,
 *                     y.c0, y.c1, Montgomery; identity = zeros).  Same rule for s; host only, no device needed.                        */
ZKB_API int32_t zkb_srs_setup_dev(zkb_ctx *ctx, uint32_t k, const uint64_t s[4], uint64_t *g_out_dev, uint64_t *g_lagrange_out_dev,
                                  void *stream);
ZKB_API int32_t zkb_g2_setup_host(const uint64_t s[4], uint64_t g2_out[16], uint64_t s_g2_out[16]);

/* ---- params file points: ParamsKZG::read_custom / write_custom (halo2_proofs src/poly/kzg/commitment.rs) --------------------------
 * A params file is 4 B k (u32 LE) | g: 2^k G1 | g_lagrange: 2^k G1 | g2 | s_g2, each point in the SerdeFormat the caller names (the
 * reference loader prover/src/utils.rs load_params checks the length 4 + 2 * 2^k * g1 + 2 * g2 bytes):
 *   format 0 Processed          G1 32 B: LE canonical x, bit 6 of byte 31 = canonical y & 1, bit 7 = 0, identity = 32 zero bytes (the
 *                               G1Affine::to_bytes of zkb_msm_g1_*: pinned by the reference fixture's vk and proof points).
 *                               G2 64 B: x.c0 || x.c1, LE canonical; bit 6 of byte 63 = parity of canonical y.c0 (of y.c1 when
 *                               y.c0 = 0), bit 7 = 0, identity = 64 zero bytes.  This G2 convention follows upstream halo2curves
 *                               and is NOT pinned by any fixture here; zkb_g2_decode_host and zkb_g2_encode_host share it.
 *   format 1 RawBytes           G1 64 B / G2 128 B: the in-memory point (Montgomery limbs; G2 x.c0, x.c1, y.c0, y.c1); decoding checks
 *                               every limb set < q and the curve equation ((0, 0) is the identity).
 *   format 2 RawBytesUnchecked  the same bytes, copied without a check.
 * zkb_g1_decode  n encoded points -> n G1Affine.  in and out_affine may each be host or device pointers (device pointers 16-byte
 *                aligned); host buffers are streamed in chunks of ZKB_SERDE_CHUNK_POINTS through pinned double buffers, so the whole
 *                input and output never need to be on the device.  A bad point is written as (0, 0); *rep receives the first bad
 *                index (UINT64_MAX when none), the exact number of bad points and the reason of the first one, the same on every
 *                run.  Returns ZKB_OK whether or not points are bad (bad points are data), ZKB_ERR_ARG for a bad format or pointer.
 *                Work queued on `stream` before the call is complete before it reads `in`; synchronises `stream`.
 * zkb_g1_encode  n G1Affine -> n encoded points (Processed: 32 B, raw formats: 64 B); same pointer rules; synchronises `stream`.
 * zkb_g2_decode_host / zkb_g2_encode_host   one G2 point (g2, s_g2 of a file), host memory only, no device needed; *status receives the
 *                reason code (0 = good; a bad point is written as zeros).                                                          */
#define ZKB_SERDE_PROCESSED 0
#define ZKB_SERDE_RAW_BYTES 1
#define ZKB_SERDE_RAW_BYTES_UNCHECKED 2
#define ZKB_SERDE_OK 0
#define ZKB_SERDE_BAD_FLAGS 1        /* bit 7 of the last byte set */
#define ZKB_SERDE_NON_CANONICAL 2    /* a coordinate (Processed: x; raw: any limb set) >= q */
#define ZKB_SERDE_NOT_ON_CURVE 3     /* Processed: x^3 + b has no square root; raw: y^2 != x^3 + b */
#define ZKB_SERDE_CHUNK_POINTS (1u << 20)
typedef struct zkb_decode_report {
    uint64_t first_bad;   /* index of the first bad point, UINT64_MAX when every point is good */
    uint64_t count;       /* number of bad points */
    uint32_t reason;      /* ZKB_SERDE_* reason of the first bad point */
    uint32_t reserved;
} zkb_decode_report;
ZKB_API int32_t zkb_g1_decode(zkb_ctx *ctx, int32_t format, const uint8_t *in, uint64_t n, uint64_t *out_affine, zkb_decode_report *rep,
                              void *stream);
ZKB_API int32_t zkb_g1_encode(zkb_ctx *ctx, int32_t format, const uint64_t *in_affine, uint64_t n, uint8_t *out, void *stream);
ZKB_API int32_t zkb_g2_decode_host(int32_t format, const uint8_t *in, uint64_t out[16], int32_t *status);
ZKB_API int32_t zkb_g2_encode_host(int32_t format, const uint64_t in[16], uint8_t *out);

/* ---- proving-key files: ProvingKey::write / ProvingKey::read (halo2_proofs plonk.rs, PSE line) ----------------------------------------
 * snark-verifier-sdk's gen_pk(params, circuit, Some(path)) caches keys on disk with these two functions.  A pk file is, in order:
 *   vk      u32 BE k || u32 BE num_fixed || fixed commitments || permutation commitments; points 32 B compressed (Processed) or the
 *           raw 64 B G1Affine (RawBytes, RawBytesUnchecked), as zkb_g1_encode encodes them.  No selector bytes: the CSF carries no
 *           selectors.  A caller whose halo2 appends packed selectors to the vk writes / consumes those bytes itself, between the vk
 *           section and the body.
 *   body    sections 0 l0, 1 l_last, 2 l_active_row (one polynomial each, extended form, N = 2^ext_k values), 3 fixed_values (n each),
 *           4 fixed_polys (coefficients, n each), 5 fixed_cosets (extended, N each), 6 permutation sigma values (n each), 7 their
 *           coefficient forms (n each), 8 their extended forms (N each).  Sections 3 - 8 are slices: u32 BE count, then polynomials.
 *           A polynomial is u32 BE length, then its elements.  Extended index m is the value at zeta * omega_ext^m (coeff_to_extended),
 *           i.e. coset part m mod E, row m / E of the prover's coset layout.  l_active_row = 1 - l_last - l_blind.
 *   Fr      32 B: Processed = canonical little-endian (< r); RawBytes = the Montgomery limbs, stored integer < r; RawBytesUnchecked =
 *           the Montgomery limbs, not checked.
 * I/O goes through caller callbacks, the read_exact / write_all of Rust's io::Read / io::Write: the library never seeks and never
 * holds a whole file.  read() returns 0 when all len bytes were read, ZKB_IO_EOF when the input ended first (a truncated file:
 * ZKB_ERR_ARG naming the section) and any other non-zero value on an I/O error; write() returns 0 or non-zero.  Any other non-zero
 * callback return aborts the call with ZKB_ERR_STATE.
 * zkb_pk_vk_write  the vk section in `format`; Processed gives exactly the bytes of zkb_pk_vk_bytes.  COLLECTIVE like zkb_pk_vk_bytes.
 * zkb_pk_write     sections 0 - 8.  Values and coefficient forms come from the key; extended forms from the coset cache when it holds
 *                  them, otherwise they are computed column by column into one N x 32 B scratch from the context's block cache.  The
 *                  encode kernel gathers the E coset parts in extended order and encodes chunk by chunk (ZKB_SERDE_CHUNK_POINTS
 *                  elements) through pinned double buffers.  The same key gives the same bytes on every run.  Rank-local.
 * zkb_pk_read      sections 0 - 8 of a key for `csf` (the caller has consumed the vk section and checked k and num_fixed).  Every
 *                  length prefix is checked against the CSF's n, N, num_fixed and permutation column count before anything is
 *                  allocated for it.  Fixed and sigma values are decoded on the GPU and the key is built by the same stages as
 *                  zkb_pk_create_with_srs (same coset-cache decision, same proof bytes).  The derived sections (0 - 2, 4, 5, 7, 8) are
 *                  decoded too: with check = 0 they are range-checked (per format) and discarded; with check = 1 every element is also
 *                  compared, in the decode kernel, with the form the key being built derives.  Deviation from upstream, which trusts the
 *                  file's polys and cosets: here they are never loaded, only checked or skipped.  Reading stops at the end of the
 *                  first polynomial that holds a bad element; *rep then names it: section, column (0 for sections 0 - 2), the index of
 *                  its first bad element, the number of bad elements in it and the reason of the first (ZKB_SERDE_NON_CANONICAL or
 *                  ZKB_PK_MISMATCH).  Bad elements, wrong length prefixes and truncated input return ZKB_ERR_ARG and no key; *rep is
 *                  filled on every return: after a wrong length prefix or truncated input it names where reading stopped (column
 *                  UINT32_MAX for a slice's count) with reason 0 and count 0; after success section and column are UINT32_MAX
 *                  (first_index UINT64_MAX, count 0).  The context stays usable.  COLLECTIVE on a context with a communicator: every rank reads its own copy of
 *                  the file, and when any rank fails every rank returns ZKB_ERR_ARG.                                                */
#define ZKB_IO_EOF 1
#define ZKB_PK_MISMATCH 4   /* check = 1: a derived element differs from the form the key derives */
typedef struct zkb_io_vtable {
    void *user;
    int32_t (*read)(void *user, uint8_t *buf, uint64_t len);
    int32_t (*write)(void *user, const uint8_t *buf, uint64_t len);
} zkb_io_vtable;
typedef struct zkb_pk_read_report {
    uint32_t section, column, reason, reserved;
    uint64_t first_index, count;
} zkb_pk_read_report;
ZKB_API int32_t zkb_pk_vk_write(struct zkb_pk *pk, int32_t format, const zkb_io_vtable *io);
ZKB_API int32_t zkb_pk_write(struct zkb_pk *pk, int32_t format, const zkb_io_vtable *io);
ZKB_API int32_t zkb_pk_read(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, int32_t format, const zkb_io_vtable *io, zkb_srs *srs,
                            int32_t check, zkb_pk_read_report *rep, struct zkb_pk **out);

/* ---- element-wise field kernels (device buffers); field: 0 = Fr, 1 = Fq ------------------------------------
 * op: 0 add, 1 sub, 2 mul (binary);  unary op: 0 invert (0 -> 0), 1 canonical->Montgomery, 2 Montgomery->canonical,
 * 3 square, 4 negate.  These back Polynomial +,-,* and the unit tests of the device arithmetic.                  */
ZKB_API int32_t zkb_field_binop_dev(zkb_ctx *ctx, int32_t field, int32_t op, const uint64_t *a, const uint64_t *b,
                            uint64_t *out, uint64_t n, void *stream);
ZKB_API int32_t zkb_field_unop_dev(zkb_ctx *ctx, int32_t field, int32_t op, const uint64_t *a, uint64_t *out, uint64_t n,
                           void *stream);
/* Montgomery batch inversion (halo2 `BatchInvert` / batch_invert_assigned): out[i] = a[i]^-1, zeros stay zero. */
ZKB_API int32_t zkb_fr_batch_invert_dev(zkb_ctx *ctx, const uint64_t *a, uint64_t *out, uint64_t n, void *stream);

/* Test surface: one primitive of ff.cuh / g1.cuh applied to n records of raw operands.  Operands are NOT reduced or
 * checked, so the lazy forms' wider input ranges can be reached.  in: n x arity x 4 u64, out: n x width x 4 u64.
 * field: 0 = Fr, 1 = Fq (G1 ops need 1).  Values are the stored integers (Montgomery form for field elements); the contract
 * is what each primitive is specified for -- outside it the output is unspecified.
 *   op  primitive                  operands            contract (stored integers)                 output
 *    0  fp_add                     a, b                < p                                        (a + b) mod p
 *    1  fp_sub                     a, b                < p                                        (a - b) mod p
 *    2  fp_neg                     a                   < p                                        (-a) mod p
 *    3  fp_dbl                     a                   < p                                        2a mod p
 *    4  fp_mul                     a, b                < p                                        a b / R mod p
 *    5  fp_sqr                     a                   < p                                        a^2 / R mod p
 *    6  fp_mul_add_mul             a, b, c, d          a, c <= p; b, d < p                        (a b + c d) / R mod p
 *    7  fp_mul_sub_mul             a, b, c, d          a <= p; b, c, d < p                        (a b - c d) / R mod p
 *    8  fp_mul_lazy                a, b                a < 4p and b < p, or a, b < 2p             the REDC value (a b + M p) / R < 2p
 *    9  fp_add_lazy                a, b                < 2p                                       a + b, minus 2p if >= 2p: [0, 2p)
 *   10  fp_sub_lazy                a, b                < 2p                                       a - b + 2p: (0, 4p)
 *   11  fp_cond_sub<false>         x                   < 2p                                       x, minus p if >= p: [0, p)
 *   12  fp_cond_sub<true>          x                   < 4p                                       x, minus 2p if >= 2p: [0, 2p)
 *   13  fp_pow                     a, e                a < p; e any 256-bit integer               a^e (Montgomery), a^0 = one
 *   14  fp_pow_u64                 a, e                a < p; e = limb 0 of the second operand    a^e (Montgomery)
 *   15  fp_inv                     a                   < p                                        a^-1 (Montgomery); inv(0) = 0
 *   16  fp_from_canonical          a                   < p                                        a R mod p
 *   17  fp_to_canonical            a                   < p                                        a / R mod p
 *   18  fp_from_u64                v                   limb 0, any u64                            v R mod p
 *   32  g1_add_mixed               acc XYZZ, q affine  points in Fq (Montgomery)                  acc + q, XYZZ
 *   33  g1_add                     acc XYZZ, q XYZZ                                               acc + q, XYZZ
 *   34  g1_dbl                     XYZZ                                                           2P, XYZZ
 *   35  g1_dbl_affine              affine                                                         2P, XYZZ
 *   36  g1_to_affine               XYZZ                                                           affine, identity (0, 0)
 *   37  g1_neg                     affine                                                         affine
 *   38  G1Xyzz::from_affine        affine                                                         XYZZ (x, y, one, one), identity zeros
 * R = 2^256; M = (-a b p^-1) mod R.  XYZZ is x = X / ZZ, y = Y / ZZZ with ZZ^3 = ZZZ^2, the identity when ZZ = 0.
 * zkb_arith_probe_host runs the host-compiled branches of the same templates; the device-only ops 8 - 12 return ZKB_ERR_ARG
 * there, as does an unknown op or a G1 op with field != 1 on either side.  Needs no CUDA device.                          */
ZKB_API int32_t zkb_arith_probe_dev(zkb_ctx *ctx, int32_t field, int32_t op, const uint64_t *in_dev, uint64_t *out_dev,
                                    uint64_t n, void *stream);
ZKB_API int32_t zkb_arith_probe_host(int32_t field, int32_t op, const uint64_t *in, uint64_t *out, uint64_t n);

/* ---- polynomial utilities around MSM/NTT (device buffers) ----------------------------------------------------
 * zkb_fr_powers_dev        out[i] = base^i
 * zkb_poly_eval_dev        halo2_proofs::arithmetic::eval_polynomial for `num_polys` polynomials (host array of device
 *                          pointers, n coefficients each) at one point x; results (Montgomery) to out_host; synchronises.
 *                          num_polys <= 65535, else ZKB_ERR_ARG before any launch.
 * zkb_fr_prefix_product_dev / _sum_dev   out[0] = init, out[i+1] = out[i] (*|+) in[i]  (n outputs; the running product z of
 *                          permutation/prover.rs and the running sum phi of mv_lookup/prover.rs)
 * zkb_kate_division_dev    halo2_proofs::arithmetic::kate_division: q = (a(X) - a(u)) / (X - u); q has n entries, q[n-1] = 0 */
ZKB_API int32_t zkb_fr_powers_dev(zkb_ctx *ctx, const uint64_t base[4], uint64_t n, uint64_t *out_dev, void *stream);
ZKB_API int32_t zkb_poly_eval_dev(zkb_ctx *ctx, const uint64_t *const *polys_dev, uint32_t num_polys, uint64_t n,
                                  const uint64_t x[4], uint64_t *out_host, void *stream);
ZKB_API int32_t zkb_fr_prefix_product_dev(zkb_ctx *ctx, const uint64_t *in_dev, uint64_t n, const uint64_t init[4],
                                          uint64_t *out_dev, void *stream);
ZKB_API int32_t zkb_fr_prefix_sum_dev(zkb_ctx *ctx, const uint64_t *in_dev, uint64_t n, const uint64_t init[4],
                                      uint64_t *out_dev, void *stream);
ZKB_API int32_t zkb_kate_division_dev(zkb_ctx *ctx, const uint64_t *a_dev, uint64_t n, const uint64_t u[4],
                                      uint64_t *q_dev, void *stream);

/* ---- multi-GPU building blocks (one process per GPU; collectives are issued by the host layer over NCCL) -----------------
 * zkb_ntt_cross_dev       size-p transform across ranks after the all-to-all of a domain-sharded NTT:
 *                         out[k][t] = sum_j in[j][t] * omega_p^(j k), in/out are p x len row-major, p in {1,2,4,8,16}
 * zkb_g1_sum_affine_host  sum of per-rank MSM partial results (host buffers, 64 B each); host-only, needs no device   */
ZKB_API int32_t zkb_ntt_cross_dev(zkb_ctx *ctx, const uint64_t *in_dev, uint64_t *out_dev, uint32_t p, uint64_t len,
                                  const uint64_t omega_p[4], void *stream);
ZKB_API int32_t zkb_g1_sum_affine_host(const uint64_t *points, uint64_t count, uint64_t out_affine[8], uint8_t *out_compressed);

/* zkb_ntt_fr_sharded_dev   ONE transform of size 2^log_n spread over the ranks of the communicator (north_star: "the k >= 26 domain
 *                          shards across the 8 GPUs"; zkb_comm_init first; COLLECTIVE).  n = P * M.  direction 0: in = this rank's
 *                          cyclic subsequence x[rank + P t] (M elements), out = the strip layout (row k1 * M/P + t holds
 *                          X[k1 M + rank M/P + t]); direction 1: strips in, cyclic out -- so forward (0) followed by the inverse root
 *                          and 1/n scale (1) is a round trip with no re-layout.  The twiddle multiply and the all-to-all are fused
 *                          into the store phase of the transform kernels: results go straight into the owner's window over NVLink
 *                          peer memory (cudaIpc-mapped); ZKB_SHARDED_EXCHANGE=nccl selects the ncclSend/ncclRecv baseline.
 * zkb_msm_g1_sharded_dev   point-range sharded MSM (aggregator/configs/compression_thin.config: 2^26 points over 8 GPUs): every rank
 *                          reduces its own slice, the 64-byte partial sums are all-gathered and added; same result on every rank. */
ZKB_API int32_t zkb_ntt_fr_sharded_dev(zkb_ctx *ctx, const uint64_t *in_dev, uint64_t *out_dev, uint32_t log_n, const uint64_t omega[4],
                                       const uint64_t *scale /* HOST pointer or NULL */, int32_t direction, void *stream);
ZKB_API int32_t zkb_msm_g1_sharded_dev(zkb_ctx *ctx, const uint64_t *scalars_shard_dev, const uint64_t *bases_shard_dev, uint64_t n_local,
                                       uint64_t out_affine[8], uint8_t *out_compressed, void *stream);

/* zkb_comm_*   NCCL communicator of a context for the multi-GPU create_proof (one process per GPU).  Rank 0 creates a
 * 128-byte unique id, the host layer broadcasts it, every rank calls zkb_comm_init.  With a communicator the proving session
 * stays replicated (identical transcript and proof bytes on every rank) while independent units -- columns, lookup arguments,
 * permutation sets, the quotient's coset parts -- are cut into P contiguous blocks (rank r computes block r) and each result is
 * completed by one in-place all-gather.  At most 16 ranks.                                                                    */
ZKB_API int32_t zkb_comm_unique_id(uint8_t out[128]);
ZKB_API int32_t zkb_comm_init(zkb_ctx *ctx, const uint8_t unique_id[128], int32_t rank, int32_t nranks);
/* zkb_comm_init_local   joins `nranks` contexts of ONE process on ONE device into one group (context i becomes rank i), so the
 *                       multi-rank paths run on a single GPU: each rank is then driven from its own host thread.  The collectives
 *                       stay stream-ordered (events, device-to-device copies; no host synchronisation is added).  Every collective
 *                       carries its kind and size: ranks that disagree all fail with ZKB_ERR_STATE before anything is copied.  A
 *                       meeting of the ranks that waits longer than timeout_ms poisons the group: every later collective fails at
 *                       once with ZKB_ERR_STATE.  ZKB_ERR_ARG: 1 <= nranks <= 16 violated, contexts on different devices, a context
 *                       given twice or one that already has a communicator.  zkb_comm_destroy / zkb_destroy of any member ends the
 *                       group for the others (their next collective fails).                                                        */
ZKB_API int32_t zkb_comm_init_local(zkb_ctx *const *ctxs, int32_t nranks, uint32_t timeout_ms);
ZKB_API int32_t zkb_comm_destroy(zkb_ctx *ctx);

/* ---- create_proof: device-resident proving session --------------------------------------------------------------
 * Replaces the body of halo2_proofs::plonk::create_proof::<KZGCommitmentScheme<Bn256>, ProverSHPLONK, Challenge255, R,
 * Blake2bWrite, C> (plonk/prover.rs; called at circuit-benchmarks/src/super_circuit.rs:117-132 and, through
 * snark_verifier_sdk::gen_snark_shplonk, at prover/src/common/prover/utils.rs:31).  `Circuit::synthesize`, the RNG and
 * vk.transcript_repr stay on the caller's side: advice columns arrive phase by phase already blinded (rows >= n - (bf+1)
 * random), blinding scalars for z / phi and the vanishing argument's random polynomial are passed in.
 *
 * CSF blob (little-endian u32 words) -- the flattened plonk::ConstraintSystem after selector compression and
 * chunk_lookups():  [0] magic 'ZSF1' 0x3146535a [1] k [2] num_fixed [3] num_advice [4] num_instance [5] num_challenges
 *   [6] blinding_factors [7] cs.degree() [8] num_phases [9] n_nodes [10] n_consts [11] n_gates [12] n_lookups
 *   [13] n_permutation_columns [14] n_advice_queries [15] n_fixed_queries [16] n_instance_queries [17] reserved, then
 *   advice_phase[num_advice], challenge_phase[num_challenges], nodes[n_nodes] x (op, a, b), consts[n_consts] x 8 (Fr,
 *   Montgomery), gates[n_gates] (node ids), per lookup: (n_input_sets, width, input node ids..., table node ids),
 *   permutation columns x (type, index), advice / fixed / instance queries x (column, rotation as i32).
 *   node ops: 0 CONST(a = const idx) 1 FIXED(a = col, b = rot) 2 ADVICE 3 INSTANCE 4 CHALLENGE(a = idx) 5 NEG(a)
 *   6 ADD(a, b) 7 MUL(a, b) 8 SCALED(a = node, b = const idx); children precede parents; column type codes 1/2/3.
 * zkb_pk_create      ProvingKey material: fixed and permutation-sigma column VALUES (host pointers, n x Fr each), SRS
 *                    g / g_lagrange (n x G1Affine); polynomial forms, l_0 / l_last / l_blind are derived on the device.
 * zkb_prove_begin    absorbs vk.transcript_repr and the instance values (KZG: QUERY_INSTANCE = false)
 * zkb_prove_advice_phase   commits the advice columns of `phase` (pointers of other phases are ignored), returns the
 *                    challenges squeezed after that phase in challenges_out[num_challenges][4] (Montgomery Fr)
 * zkb_prove_finish   lookups -> permutation -> vanishing -> quotient -> evaluations -> SHPLONK; z_blinds
 *                    [n_sets][bf], phi_blinds [n_lookups][bf], random_poly [n] are Montgomery Fr arrays on the host.
 *                    The first call runs the proof and keeps its bytes in the session: proof_out may be NULL (query the length) or
 *                    too short (ZKB_ERR_ARG, *proof_len set) -- call again with a buffer of *proof_len bytes; later calls only copy.
 *                    Multi-GPU sessions (zkb_comm_init): every zkb_pk_* / zkb_prove_* call, zkb_pk_vk_bytes included, is a COLLECTIVE
 *                    over the communicator and must be issued by all ranks in the same order; a rank-local failure (allocation, CUDA
 *                    error) leaves the other ranks inside a collective, so abort the job on any non-zero return.                  */
typedef struct zkb_pk zkb_pk;
typedef struct zkb_session zkb_session;
ZKB_API int32_t zkb_pk_create(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, const uint64_t *const *fixed_values,
                              const uint64_t *const *sigma_values, const uint64_t *g, const uint64_t *g_lagrange, zkb_pk **out);
/* Same against a loaded SRS handle (shared by every pk of the context; srs->k must equal the circuit's k: downsize first). */
ZKB_API int32_t zkb_pk_create_with_srs(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, const uint64_t *const *fixed_values,
                                       const uint64_t *const *sigma_values, zkb_srs *srs, zkb_pk **out);
/* keygen_pk2 / keygen_vk + keygen_pk (halo2_proofs plonk/keygen.rs; reference call site prover/src/common/prover/utils.rs:43-61,
 * :55): the caller runs Circuit::synthesize in keygen mode and hands over the fixed column values and the COPY CONSTRAINTS
 * (n_copies x 4 u32: left column, left row, right column, right row; columns index the CSF's permutation column list).  The
 * permutation Assembly (cycle merging, permutation/keygen.rs) runs on the host, the sigma columns delta^col * omega^row, every
 * polynomial / coset form and the vk commitments (zkb_pk_vk_bytes) are produced on the device.                                   */
ZKB_API int32_t zkb_keygen_pk(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, const uint64_t *const *fixed_values,
                              const uint32_t *copies, uint64_t n_copies, zkb_srs *srs, zkb_pk **out);
/* sigma column `column` of a proving key (Lagrange values, 2^k x 32 B) back to the host. */
ZKB_API int32_t zkb_pk_sigma_read(zkb_pk *pk, uint32_t column, uint64_t *out_host);
ZKB_API int32_t zkb_pk_destroy(zkb_pk *pk);
/* VerifyingKey bytes in SerdeFormat::Processed layout (u32 BE k || u32 BE num_fixed || fixed || permutation commitments,
 * compressed points; the layout of the reference fixture's vk).  out may be NULL to query the length.                     */
ZKB_API int32_t zkb_pk_vk_bytes(zkb_pk *pk, uint8_t *out, uint64_t cap, uint64_t *len);
/* Host-only structural validation of a CSF blob (no CUDA device needed); zkb_pk_create, zkb_pk_create_with_srs and
 * zkb_keygen_pk run it first.  Deviation from halo2: SHPLONK opens one advice or fixed column at the points x w^r of its
 * distinct rotations mod n, and this prover takes at most 256 such points per column (upstream has no limit).  A CSF that
 * opens a column at more fails here with ZKB_ERR_ARG, naming the column and its point count; rotations r and r -+ n count once. */
ZKB_API int32_t zkb_csf_validate(const uint32_t *csf, uint64_t csf_words);
/* The gates of a CSF evaluated over caller columns by the prover's own expression compiler and interpreter (the quotient's hot
 * kernel, exposed for row-by-row tests).  columns_dev: HOST array of device pointers in slot order fixed | advice | instance,
 * 2^k elements each; challenges: num_challenges x 4 limbs (Montgomery), may be NULL without challenges.
 *   mode 0: gate i -> outs_dev[i][row], all gates in ONE common-subexpression scope (like the lookup compression programs);
 *           out_stride must be 1 and out_offset 0.
 *   mode 1: the gates folded in y exactly as the quotient program of zkb_prove_finish (selector runs folded), times `scale`,
 *           -> outs_dev[0][row * out_stride + out_offset]; other entries are not written.
 * *nregs_out (may be NULL) receives the register count that chose the kernel build (<= 8, <= 16: shared memory; <= 64: local
 * memory).  A program needing more than 64 live registers fails with ZKB_ERR_ARG before anything is launched.  Synchronises
 * `stream`.                                                                                                                  */
ZKB_API int32_t zkb_expr_eval_dev(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, int32_t mode, const uint64_t *challenges,
                                  const uint64_t y[4], const uint64_t scale[4], const uint64_t *const *columns_dev,
                                  uint64_t *const *outs_dev, uint32_t out_stride, uint32_t out_offset, uint32_t *nregs_out, void *stream);
/* Host only (no CUDA device needed): the interpreter program zkb_expr_eval_dev would run for the same csf / mode / challenges /
 * y / scale, after operand fusion.  One 64-bit word per instruction (the Instr layout of csrc/expr.cuh: op, dst, a, b bytes,
 * then the 32-bit imm); the first min(cap, *ncode_out) words go to code_out (may be NULL when cap is 0).  *nregs_out (may be
 * NULL) receives the register count that picks the kernel build.  For instruction counts (scripts/expr_program_stats.py).    */
ZKB_API int32_t zkb_expr_program(const uint32_t *csf, uint64_t csf_words, int32_t mode, const uint64_t *challenges, const uint64_t y[4],
                                 const uint64_t scale[4], uint64_t *code_out, uint64_t cap, uint64_t *ncode_out, uint32_t *nregs_out);
/* Test surface: the mv-lookup multiplicities m exactly as zkb_prove_finish computes them (mv_lookup/prover.rs prepare), over caller
 * buffers of already-compressed values (Montgomery Fr, compared as stored bytes).  inputs_dev: HOST array of n_sets device pointers, n
 * elements each; table_dev: n elements.  m_out_dev[r] (n Fr, Montgomery) = the number of input rows i < usable over all sets whose value
 * the table holds at row r, where r is the LAST table row < usable with that value (BTreeMap collect()); every other row, rows >= usable
 * included, is zero.  Input rows >= usable are ignored.  *unsatisfied = 1 when an input row < usable is not among the table rows < usable,
 * else 0 (the prover's "unsatisfied witness" error; the rows that are found are still counted).  The table's hash set has
 * n_slots = the smallest power of two >= 2 usable u32 slots: 0 = empty, otherwise table row + 1, probed linearly from
 * key_hash(value) & (n_slots - 1) (csrc/lookup.cuh).  Which slot of its probe run a key lands in depends on the insertion schedule, so
 * the slots may differ between calls while m does not.  The first min(slots_cap, n_slots) slots go to slots_out (host, may be NULL when
 * slots_cap is 0) and n_slots to *n_slots (may be NULL).  ZKB_ERR_ARG before any launch unless 0 < usable < n <= 2^31 and
 * n_sets >= 1.  Synchronises `stream`.                                                                                          */
ZKB_API int32_t zkb_lookup_multiplicities_dev(zkb_ctx *ctx, const uint64_t *const *inputs_dev, uint32_t n_sets, const uint64_t *table_dev, uint64_t n,
                                              uint32_t usable, uint64_t *m_out_dev, int32_t *unsatisfied, uint32_t *slots_out, uint64_t slots_cap,
                                              uint64_t *n_slots, void *stream);
/* Witness check (halo2 MockProver::run + verify / assert_satisfied_par, without region information): which constraints of a CSF
 * fail on caller columns, row by row, before any proof is attempted.  A failure is what the verifier would reject:
 *   gate g          g(row) != 0 on ALL n rows (rotation r reads row (row + r) mod n): the quotient needs every gate to vanish on
 *                   all of H, blinding rows included.  sub = 1 ("poisoned", MockProver's ConstraintPoisoned) when one of the gate's
 *                   ADVICE queries reads a row >= usable = n - blinding_factors - 1 at that row: usually a selector that is not zero
 *                   in the blinding rows.  Unlike MockProver the check uses the real numbers in the cells, not poison values: a gate
 *                   that reads blinding rows but comes out numerically zero is not reported.
 *   lookup l, set j the input tuple at a row < usable is not among the table tuples at rows < usable (the rows the prover's
 *                   multiplicities cover).  Tuples are compared compressed with the caller's theta: a reported failure is always
 *                   real; a real one is missed only on a theta collision, probability at most #inputs * #table rows * (width - 1) / r
 *                   (below 2^-200 for k <= 26).  theta may be NULL only when every lookup has width 1.
 *   copy i          v[lc][lr] != v[rc][rr] for copies_dev[i] = (lc, lr, rc, rr), columns indexing the CSF's permutation column list
 *                   (the copy format of zkb_keygen_pk).
 * columns_dev: HOST array of device pointers, fixed | advice | instance, 2^k elements each (instance zero-padded; advice blinded or
 * not).  counts_out (host) receives the EXACT failure count of every gate, of every (lookup, input set) and of all copies together,
 * in that order (n_gates + sum_l n_input_sets(l) + 1 entries), also when the records are truncated.  records_out (host) receives
 * the first min(cap, total) failures in one fixed order: gates by (gate, row), then lookups by (lookup, set, row), then copies by
 * index; *n_records their number; cap = 0 returns counts only.  The output is deterministic (same inputs, same bytes).
 * Returns ZKB_OK whether or not anything fails (failures are data); ZKB_ERR_ARG for a malformed CSF, missing challenges or theta,
 * or a copy entry out of range (column >= P or row >= n; the message names the first one).  Rank-local, also on a context with a
 * communicator.  Temporary device memory comes from the context's block cache and is returned before the call returns.
 * Synchronises `stream`.                                                                                                        */
typedef struct zkb_check_record {
    uint32_t kind;    /* 0 gate, 1 lookup, 2 copy */
    uint32_t index;   /* gate index, lookup argument index, or position in the copy list */
    uint32_t sub;     /* gate: poisoned (0/1); lookup: input set; copy: 0 */
    uint32_t row;     /* the failing row; copy: the left row */
} zkb_check_record;
ZKB_API int32_t zkb_check_witness_dev(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, const uint64_t *const *columns_dev,
                                      const uint64_t *challenges, const uint64_t *theta, const uint32_t *copies_dev, uint64_t n_copies,
                                      uint64_t *counts_out, zkb_check_record *records_out, uint32_t cap, uint32_t *n_records, void *stream);
ZKB_API int32_t zkb_prove_begin(zkb_pk *pk, const uint64_t transcript_repr[4], const uint64_t *const *instance_values,
                                const uint32_t *instance_lens, zkb_session **out);
/* Same with a choice of transcript: 0 = Blake2bWrite/Challenge255 (the reference's benches, circuit-benchmarks/src/super_circuit.rs:112),
 * 1 = snark-verifier-sdk PoseidonTranscript<NativeLoader> (gen_snark_shplonk, prover/src/common/prover/utils.rs:31): Poseidon T=5,
 * RATE=4, R_F=8, R_P=60 over Fr; points absorbed as (x mod r, y mod r).  The Poseidon restatement is pinned by the reference's own
 * chunk proof (tests/test_fixture_proof.py);
 * 2 = snark-verifier EvmTranscript<G1Affine, NativeLoader> over Keccak-256 (gen_evm_proof_shplonk, prover/src/common/prover/evm.rs:67):
 * points absorbed AND written uncompressed as x || y big-endian (64 B), scalars 32 B big-endian, challenge = keccak256(buffer) mod r.   */
ZKB_API int32_t zkb_prove_begin_ex(zkb_pk *pk, int32_t transcript_kind, const uint64_t transcript_repr[4],
                                   const uint64_t *const *instance_values, const uint32_t *instance_lens, zkb_session **out);
/* 3 = THE CALLER'S transcript: create_proof is generic over `T: TranscriptWrite<G1Affine, Challenge255<G1Affine>>` (and the SDK
 * instantiates it with Blake2b, Poseidon and Keccak transcripts), and a generic type cannot cross a C ABI -- but its four
 * operations can.  The shim passes a table of extern "C" trampolines around the `&mut T` it was handed; the session then calls
 * exactly the sequence halo2's prover would (common_scalar for vk.transcript_repr and the instances, write_point per commitment,
 * squeeze_challenge, write_scalar per evaluation), so ANY transcript -- including ones this library has never seen -- produces its
 * own proof bytes on the Rust side and the RNG-free session needs no replay.  Scalars are Fr in halo2curves' Montgomery layout,
 * points G1Affine x || y; a callback returns 0 or an error code that aborts the session (ZKB_ERR_STATE).  In this mode
 * zkb_prove_finish reports proof_len = 0: the bytes live in the caller's writer.                                                */
typedef struct zkb_transcript_vtable {
    void *user;
    int32_t (*common_scalar)(void *user, const uint64_t scalar[4]);
    int32_t (*write_scalar)(void *user, const uint64_t scalar[4]);
    int32_t (*write_point)(void *user, const uint64_t point_xy[8]);
    int32_t (*squeeze_challenge)(void *user, uint64_t challenge_out[4]);
} zkb_transcript_vtable;
ZKB_API int32_t zkb_prove_begin_cb(zkb_pk *pk, const zkb_transcript_vtable *vt, const uint64_t transcript_repr[4],
                                   const uint64_t *const *instance_values, const uint32_t *instance_lens, zkb_session **out);
/* Host-only transcript primitives (no CUDA device needed; used by the CPU test-suite to pin the session's hashers):
 * zkb_poseidon_hash_host        absorb n Fr (Montgomery) into a fresh PoseidonTranscript sponge, squeeze one challenge
 * zkb_blake2b_challenge_host    feed bytes to a fresh Blake2b("Halo2-Transcript") state, squeeze one Challenge255 (mod r)
 * zkb_keccak256_host            Keccak-256 of a byte string (the EvmTranscript hash; eth-types KECCAK_CODE_HASH_EMPTY is its "" digest)
 * zkb_transcript_script_host    replay ops (0 common_scalar, 1 write_scalar, 2 write_point, 3 squeeze) through the session's transcript
 *                               code of `kind`; operands in order (scalar 4 limbs, point 8 limbs, Montgomery); returns the proof bytes
 *                               written and the squeezed challenges (4 limbs each); proof may be NULL to query the length          */
ZKB_API int32_t zkb_poseidon_hash_host(const uint64_t *inputs, uint64_t n, uint64_t out[4]);
ZKB_API int32_t zkb_blake2b_challenge_host(const uint8_t *bytes, uint64_t len, uint64_t out[4]);
ZKB_API int32_t zkb_keccak256_host(const uint8_t *bytes, uint64_t len, uint8_t out[32]);
ZKB_API int32_t zkb_transcript_script_host(int32_t kind, const uint8_t *ops, uint64_t n_ops, const uint64_t *operands, uint8_t *proof,
                                           uint64_t cap, uint64_t *proof_len, uint64_t *challenges);
ZKB_API int32_t zkb_prove_advice_phase(zkb_session *s, uint32_t phase, const uint64_t *const *advice_columns,
                                       uint64_t *challenges_out);
/* Witness-side overlap (SURVEY 8f row 4; zkevm-circuits/src/super_circuit.rs:714-806 assigns sub-circuit after sub-circuit): hand a
 * finished, blinded advice column over BEFORE its phase is submitted.  The H2D copy runs on the copy stream while the caller keeps
 * synthesising; zkb_prove_advice_phase then accepts NULL for that column.  The buffer must stay valid until the phase call.       */
ZKB_API int32_t zkb_prove_upload_advice(zkb_session *s, uint32_t column, const uint64_t *values);
ZKB_API int32_t zkb_prove_finish(zkb_session *s, const uint64_t *z_blinds, const uint64_t *phi_blinds,
                                 const uint64_t *random_poly, uint8_t *proof_out, uint64_t proof_cap, uint64_t *proof_len);
ZKB_API int32_t zkb_session_destroy(zkb_session *s);

#ifdef __cplusplus
}
#endif
#endif
