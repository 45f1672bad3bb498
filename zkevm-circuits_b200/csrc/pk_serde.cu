// pk_serde.cu -- proving-key files: ProvingKey::write / ProvingKey::read (halo2_proofs plonk.rs) streamed through the device.
//
// The file layout is documented in include/zkb200.h.  Every field element of the body passes through one of two kernels, one thread
// per element, in chunks of ZKB_SERDE_CHUNK_POINTS elements through the pinned double buffers of SerdePipe (serde.cuh):
//   fr_encode_kernel<PROCESSED>   gathers element m of a polynomial (a plain column, or extended index m = coset part m mod E, row
//                                 m / E of the prover's layout, or l_active_row = 1 - l_last - l_blind formed on the fly) and writes
//                                 it canonical (Processed) or as its Montgomery limbs (raw formats): no separate transpose pass.
//   fr_decode_kernel<FMT, CHECK>  range-checks (Processed, RawBytes), converts (Processed), optionally compares with the element the
//                                 key being built derives, gathered the same way, and stores.  The first bad element and its reason
//                                 are packed into one 64-bit word (index << 3 | reason) lowered with atomicMin, the bad elements are
//                                 counted: the report is the same on every run.
// Writing: the encode of chunk c + 1 overlaps the caller's write() of chunk c.  Reading: the caller's read() of chunk c + 1 overlaps
// the copy and decode of chunk c.  Work on the context's stream (the sources of a gather, the extended-form scratch) is ordered
// before a polynomial's chunks by an event, and the context's stream waits for the chunks before it touches those buffers again.
#include "common.cuh"
#include "serde.cuh"
#include "pk.cuh"
#include <string.h>
#include <algorithm>
#include <memory>

namespace zkb {

// element m of a polynomial: col[m] (a plain column), or parts[m mod E][m / E] (extended order over the E = 2^log_e coset parts);
// `active`: 1 - a - b with b gathered from bparts the same way (l_active_row)
struct Gather {
    const Fr *col = nullptr;
    const Fr *const *parts = nullptr;
    const Fr *const *bparts = nullptr;
    uint32_t log_e = 0;
    bool active = false;
};

FF_D Fr gather_at(const Gather &g, uint64_t m) {
    if (g.col) return fp_load(g.col + m);
    const uint64_t j = m & ((1ull << g.log_e) - 1), i = m >> g.log_e;
    Fr v = fp_load(g.parts[j] + i);
    if (g.active) v = fp_sub(fp_sub(Fr::one(), v), fp_load(g.bparts[j] + i));
    return v;
}

// stored integer < r (halo2curves' Fr::from_repr / from_raw_bytes checks)
FF_HD bool fr_is_canonical(const Fr &x) {
    for (int i = 7; i >= 0; --i) {
        if (x.l[i] != FrParams::P(i)) return x.l[i] < FrParams::P(i);
    }
    return false;
}

struct FrDecodeState {
    unsigned long long first;   // (index << 3) | reason of the first bad element; ~0 when none
    unsigned long long count;
};

template <bool PROCESSED>
__global__ void __launch_bounds__(SERDE_THREADS) fr_encode_kernel(Gather g, uint64_t base, uint64_t cnt, uint4 *__restrict__ out) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    Fr v = gather_at(g, base + i);
    if (PROCESSED) v = fp_to_canonical(v);
    out[2 * i] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    out[2 * i + 1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}

// out (may be null: the element is only checked) is the chunk's first output element
template <int FMT, bool CHECK>
__global__ void __launch_bounds__(SERDE_THREADS) fr_decode_kernel(const uint4 *__restrict__ in, uint64_t base, uint64_t cnt, Fr *__restrict__ out,
                                                                  Gather ref, FrDecodeState *st) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    const uint4 lo = in[2 * i], hi = in[2 * i + 1];
    Fr v;
    v.l[0] = lo.x; v.l[1] = lo.y; v.l[2] = lo.z; v.l[3] = lo.w;
    v.l[4] = hi.x; v.l[5] = hi.y; v.l[6] = hi.z; v.l[7] = hi.w;
    uint32_t reason = ZKB_SERDE_OK;
    if (FMT != ZKB_SERDE_RAW_BYTES_UNCHECKED && !fr_is_canonical(v)) reason = ZKB_SERDE_NON_CANONICAL;
    else if (FMT == ZKB_SERDE_PROCESSED) v = fp_from_canonical(v);
    if (CHECK && reason == ZKB_SERDE_OK && v != gather_at(ref, base + i)) reason = ZKB_PK_MISMATCH;
    if (reason != ZKB_SERDE_OK) {
        atomicMin(&st->first, (unsigned long long)(((base + i) << 3) | reason));
        atomicAdd(&st->count, 1ull);
    }
    if (out) fp_store(out + i, v);
}

// the coefficients of l_active_row = 1 - l_last - l_blind
__global__ void lactive_coeff_kernel(const Fr *__restrict__ llast, const Fr *__restrict__ lblind, uint64_t n, Fr *__restrict__ out) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr one = i == 0 ? Fr::one() : Fr::zero();
    fp_store(out + i, fp_sub(fp_sub(one, fp_load(llast + i)), fp_load(lblind + i)));
}

static_assert(sizeof(G1Affine) == 64, "the raw vk point is the 64-byte in-memory G1Affine");

static const char *const SECTION_NAMES[9] = {"l0", "l_last", "l_active_row", "fixed_values", "fixed_polys", "fixed_cosets",
                                             "permutation values", "permutation polys", "permutation cosets"};

// One pass over a pk file through the caller's callbacks: two slots of ZKB_SERDE_CHUNK_POINTS elements, each with its own stream,
// pinned staging and device staging.  Chunks alternate slots; a slot is reused only after its previous chunk is complete (writing: and
// handed to write(), in file order).
struct PkStream {
    zkb_ctx *ctx;
    const zkb_io_vtable *io;
    int32_t fmt;
    bool writing;
    SerdePipe pp;
    cudaEvent_t ready = nullptr;
    bool busy[2] = {false, false};
    uint64_t busy_cnt[2] = {0, 0};
    int next = 0;
    int section = 0;
    static constexpr uint64_t CHUNK = ZKB_SERDE_CHUNK_POINTS;

    PkStream(zkb_ctx *c, const zkb_io_vtable *v, int32_t f, bool w) : ctx(c), io(v), fmt(f), writing(w), pp(c) {}
    ~PkStream() {
        if (ready) cudaEventDestroy(ready);
    }
    int32_t init() {
        ZKB_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
        for (int j = 0; j < 2; ++j) {
            ZKB_CUDA(cudaStreamCreateWithFlags(&pp.s[j], cudaStreamNonBlocking));
            ZKB_CUDA(cudaEventCreateWithFlags(&pp.done[j], cudaEventDisableTiming));
            uint8_t **h = writing ? &pp.h_out[j] : &pp.h_in[j];
            uint8_t **d = writing ? &pp.d_out[j] : &pp.d_in[j];
            ZKB_CUDA(cudaHostAlloc((void **)h, CHUNK * sizeof(Fr), cudaHostAllocDefault));
            ZKB_TRY(pp.pool.alloc(CHUNK * sizeof(Fr), (void **)d));
        }
        return ZKB_OK;
    }
    // the slots' streams start after the work queued on the context's stream so far
    int32_t begin_poly() {
        ZKB_CUDA(cudaEventRecord(ready, ctx->stream));
        for (int j = 0; j < 2; ++j) ZKB_CUDA(cudaStreamWaitEvent(pp.s[j], ready, 0));
        return ZKB_OK;
    }
    // later work on the context's stream waits for every chunk queued so far
    int32_t end_poly() {
        for (int j = 0; j < 2; ++j) ZKB_CUDA(cudaStreamWaitEvent(ctx->stream, pp.done[j], 0));
        return ZKB_OK;
    }
    int32_t io_status(int32_t rc, const char *what) {
        if (rc == 0) return ZKB_OK;
        if (!writing && rc == ZKB_IO_EOF) {
            set_error("pk file: the input ends inside section %d (%s)", section, SECTION_NAMES[section]);
            return ZKB_ERR_ARG;
        }
        set_error("pk file: the %s callback failed (%d) in section %d (%s)", what, rc, section, SECTION_NAMES[section]);
        return ZKB_ERR_STATE;
    }

    // ---- writing
    int32_t drain(int j) {
        ZKB_CUDA(cudaEventSynchronize(pp.done[j]));
        busy[j] = false;
        return io_status(io->write(io->user, pp.h_out[j], busy_cnt[j] * sizeof(Fr)), "write");
    }
    int32_t flush() {
        for (int t = 0; t < 2; ++t, next ^= 1)   // the slot used next holds the older chunk
            if (busy[next]) ZKB_TRY(drain(next));
        return ZKB_OK;
    }
    int32_t write_bytes(const void *p, uint64_t len) {
        ZKB_TRY(flush());
        return io_status(io->write(io->user, (const uint8_t *)p, len), "write");
    }
    int32_t write_u32(uint32_t v) {
        const uint8_t b[4] = {(uint8_t)(v >> 24), (uint8_t)(v >> 16), (uint8_t)(v >> 8), (uint8_t)v};
        return write_bytes(b, 4);
    }
    // a polynomial: u32 BE length, then its n elements
    int32_t write_poly(const Gather &g, uint64_t n) {
        ZKB_TRY(write_u32((uint32_t)n));
        ZKB_TRY(begin_poly());
        for (uint64_t off = 0; off < n; off += CHUNK) {
            const int j = next;
            if (busy[j]) ZKB_TRY(drain(j));
            const uint64_t cnt = std::min(CHUNK, n - off);
            const unsigned grid = (unsigned)((cnt + SERDE_THREADS - 1) / SERDE_THREADS);
            if (fmt == ZKB_SERDE_PROCESSED) fr_encode_kernel<true><<<grid, SERDE_THREADS, 0, pp.s[j]>>>(g, off, cnt, (uint4 *)pp.d_out[j]);
            else fr_encode_kernel<false><<<grid, SERDE_THREADS, 0, pp.s[j]>>>(g, off, cnt, (uint4 *)pp.d_out[j]);
            ctx->launches++;
            ZKB_CUDA(cudaGetLastError());
            ZKB_CUDA(cudaMemcpyAsync(pp.h_out[j], pp.d_out[j], cnt * sizeof(Fr), cudaMemcpyDeviceToHost, pp.s[j]));
            ZKB_CUDA(cudaEventRecord(pp.done[j], pp.s[j]));
            busy[j] = true;
            busy_cnt[j] = cnt;
            next ^= 1;
        }
        return end_poly();
    }

    // ---- reading
    int32_t read_bytes(void *p, uint64_t len) { return io_status(io->read(io->user, (uint8_t *)p, len), "read"); }
    int32_t read_u32(uint32_t &v) {
        uint8_t b[4];
        ZKB_TRY(read_bytes(b, 4));
        v = (uint32_t)b[0] << 24 | (uint32_t)b[1] << 16 | (uint32_t)b[2] << 8 | b[3];
        return ZKB_OK;
    }
    template <int FMT, bool CHECK>
    void launch_decode(int j, uint64_t off, uint64_t cnt, Fr *out, const Gather &ref, FrDecodeState *st) {
        fr_decode_kernel<FMT, CHECK><<<(unsigned)((cnt + SERDE_THREADS - 1) / SERDE_THREADS), SERDE_THREADS, 0, pp.s[j]>>>(
            (const uint4 *)pp.d_in[j], off, cnt, out ? out + off : nullptr, ref, st);
    }
    // n elements -> out (device, may be null), compared with ref when given; bad elements are recorded in *st
    int32_t read_elems(uint64_t n, Fr *out, const Gather *ref, FrDecodeState *st) {
        // nothing to store, compare or check: the bytes are only consumed
        const bool device = out || ref || fmt != ZKB_SERDE_RAW_BYTES_UNCHECKED;
        if (device) ZKB_TRY(begin_poly());
        const Gather none;
        for (uint64_t off = 0; off < n; off += CHUNK) {
            const int j = next;
            if (busy[j]) {   // the slot's pinned buffer is free again once its previous chunk has been copied
                ZKB_CUDA(cudaEventSynchronize(pp.done[j]));
                busy[j] = false;
            }
            const uint64_t cnt = std::min(CHUNK, n - off);
            ZKB_TRY(read_bytes(pp.h_in[j], cnt * sizeof(Fr)));
            if (!device) continue;
            ZKB_CUDA(cudaMemcpyAsync(pp.d_in[j], pp.h_in[j], cnt * sizeof(Fr), cudaMemcpyHostToDevice, pp.s[j]));
            const Gather &r = ref ? *ref : none;
            switch (fmt * 2 + (ref ? 1 : 0)) {
                case 0: launch_decode<ZKB_SERDE_PROCESSED, false>(j, off, cnt, out, r, st); break;
                case 1: launch_decode<ZKB_SERDE_PROCESSED, true>(j, off, cnt, out, r, st); break;
                case 2: launch_decode<ZKB_SERDE_RAW_BYTES, false>(j, off, cnt, out, r, st); break;
                case 3: launch_decode<ZKB_SERDE_RAW_BYTES, true>(j, off, cnt, out, r, st); break;
                case 4: launch_decode<ZKB_SERDE_RAW_BYTES_UNCHECKED, false>(j, off, cnt, out, r, st); break;
                default: launch_decode<ZKB_SERDE_RAW_BYTES_UNCHECKED, true>(j, off, cnt, out, r, st); break;
            }
            ctx->launches++;
            ZKB_CUDA(cudaGetLastError());
            ZKB_CUDA(cudaEventRecord(pp.done[j], pp.s[j]));
            busy[j] = true;
            next ^= 1;
        }
        return device ? end_poly() : ZKB_OK;
    }
};

// The extended form of one size-n coefficient polynomial into `scratch` as E coset parts of n elements (part j = evaluations at
// zeta * omega_ext^j * omega^i, the layout of the coset cache); pows holds E x n coset-generator powers.
static int32_t ext_parts(zkb_pk *pk, const Fr *poly, const Fr *pows, Fr *scratch) {
    for (uint32_t j = 0; j < pk->E; ++j)
        ZKB_TRY(ntt_fr_device(pk->ctx, poly, scratch + (uint64_t)j * pk->n, pk->k, pk->omega, nullptr, 0, pows + (uint64_t)j * pk->n, pk->ctx->stream));
    return ZKB_OK;
}

// The E-part extended-form scratch of a write or a checked read: scratch + part tables, coset-generator powers.
struct ExtScratch {
    Fr *data = nullptr, *pows = nullptr, *lactive = nullptr;
    Fr **parts = nullptr;
    int32_t init(zkb_pk *pk, DevPool &pool) {
        cudaStream_t st = pk->ctx->stream;
        ZKB_TRY(pool.fr(pk->N, &data));
        ZKB_TRY(pool.fr(pk->N, &pows));
        ZKB_TRY(pool.fr(pk->n, &lactive));
        for (uint32_t j = 0; j < pk->E; ++j) ZKB_TRY(fr_powers_device(pk->ctx, pk->coset_gen(j), pk->n, pows + (uint64_t)j * pk->n, st));
        std::vector<Fr *> tbl(pk->E);
        for (uint32_t j = 0; j < pk->E; ++j) tbl[j] = data + (uint64_t)j * pk->n;
        return upload_table(pool, tbl, &parts, st);
    }
    // the gather of poly's extended form, computed into the scratch
    int32_t of(zkb_pk *pk, const Fr *poly, Gather &g) {
        ZKB_TRY(ext_parts(pk, poly, pows, data));
        g = Gather();
        g.parts = parts;
        g.log_e = (uint32_t)__builtin_ctz(pk->E);
        return ZKB_OK;
    }
    int32_t of_lactive(zkb_pk *pk, Gather &g) {
        lactive_coeff_kernel<<<(unsigned)((pk->n + 255) / 256), 256, 0, pk->ctx->stream>>>(pk->llast_poly, pk->lblind_poly, pk->n, lactive);
        pk->ctx->launches++;
        ZKB_CUDA(cudaGetLastError());
        return of(pk, lactive, g);
    }
};

static Gather plain(const Fr *col) {
    Gather g;
    g.col = col;
    return g;
}

static bool format_ok(int32_t f) { return f == ZKB_SERDE_PROCESSED || f == ZKB_SERDE_RAW_BYTES || f == ZKB_SERDE_RAW_BYTES_UNCHECKED; }

static int32_t pk_write_body(zkb_pk *pk, int32_t format, const zkb_io_vtable *io) {
    zkb_ctx *ctx = pk->ctx;
    cudaStream_t st = ctx->stream;
    const SlotMap &sm = pk->sm;
    const uint64_t n = pk->n, N = pk->N;
    const uint32_t log_e = (uint32_t)__builtin_ctz(pk->E);
    DevPool tmp;
    tmp.ctx = ctx;
    // the coset cache's parts of every cached slot, in one table: slot s at tbl[s * E]
    const bool cache = !pk->coset_cache.empty();
    Fr **cache_tbl = nullptr;
    if (cache) {
        std::vector<Fr *> tbl((size_t)sm.slots * pk->E, nullptr);
        for (uint32_t j = 0; j < pk->E; ++j)
            for (size_t s = 0; s < pk->coset_cache[j].size(); ++s) tbl[s * pk->E + j] = pk->coset_cache[j][s];
        ZKB_TRY(upload_table(tmp, tbl, &cache_tbl, st));
    }
    auto cached = [&](uint32_t slot) { return cache && slot < pk->coset_cache[0].size() && pk->coset_cache[0][slot]; };
    ExtScratch xs;
    bool xs_ready = false;
    auto extended = [&](uint32_t slot, const Fr *poly, Gather &g) -> int32_t {
        if (cached(slot)) {
            g = Gather();
            g.parts = cache_tbl + (size_t)slot * pk->E;
            g.log_e = log_e;
            return ZKB_OK;
        }
        if (!xs_ready) { ZKB_TRY(xs.init(pk, tmp)); xs_ready = true; }
        return xs.of(pk, poly, g);
    };
    PkStream ps(ctx, io, format, true);
    ZKB_TRY(ps.init());
    Gather g;
    ps.section = 0;
    ZKB_TRY(extended(sm.l0, pk->l0_poly, g));
    ZKB_TRY(ps.write_poly(g, N));
    ps.section = 1;
    ZKB_TRY(extended(sm.l_last, pk->llast_poly, g));
    ZKB_TRY(ps.write_poly(g, N));
    ps.section = 2;
    if (cached(sm.l_last) && cached(sm.l_blind)) {
        g = Gather();
        g.parts = cache_tbl + (size_t)sm.l_last * pk->E;
        g.bparts = cache_tbl + (size_t)sm.l_blind * pk->E;
        g.log_e = log_e;
        g.active = true;
    } else {
        if (!xs_ready) { ZKB_TRY(xs.init(pk, tmp)); xs_ready = true; }
        ZKB_TRY(xs.of_lactive(pk, g));
    }
    ZKB_TRY(ps.write_poly(g, N));
    // sections 3 - 5 (fixed), 6 - 8 (permutation): values, coefficients, extended forms
    auto columns = [&](int first_section, const std::vector<Fr *> &vals, const std::vector<Fr *> &polys, uint32_t slot0) -> int32_t {
        ps.section = first_section;
        ZKB_TRY(ps.write_u32((uint32_t)vals.size()));
        for (auto v : vals) ZKB_TRY(ps.write_poly(plain(v), n));
        ps.section = first_section + 1;
        ZKB_TRY(ps.write_u32((uint32_t)polys.size()));
        for (auto p : polys) ZKB_TRY(ps.write_poly(plain(p), n));
        ps.section = first_section + 2;
        ZKB_TRY(ps.write_u32((uint32_t)polys.size()));
        for (size_t c = 0; c < polys.size(); ++c) {
            ZKB_TRY(extended(slot0 + (uint32_t)c, polys[c], g));
            ZKB_TRY(ps.write_poly(g, N));
        }
        return ZKB_OK;
    };
    ZKB_TRY(columns(3, pk->fixed_values, pk->fixed_polys, sm.fixed0));
    ZKB_TRY(columns(6, pk->sigma_values, pk->sigma_polys, sm.sigma0));
    return ps.flush();
}

// Reads sections 0 - 8 into a key built by pk_begin / pk_ingest / pk_finish.  *rep is filled by the caller's defaults and here.
static int32_t pk_read_body(zkb_ctx *ctx, Csf &&csf, int32_t format, const zkb_io_vtable *io, zkb_srs *srs, bool check, zkb_pk_read_report *rep,
                            zkb_pk **out) {
    zkb_pk *raw = nullptr;
    ZKB_TRY(pk_begin(ctx, std::move(csf), srs, &raw));
    std::unique_ptr<zkb_pk> pk(raw);
    const Csf &cs = pk->cs;
    const uint64_t n = pk->n, N = pk->N;
    cudaStream_t st = ctx->stream;
    DevPool tmp;
    tmp.ctx = ctx;
    FrDecodeState *d_st = nullptr;
    ZKB_TRY(tmp.alloc(sizeof(FrDecodeState), (void **)&d_st));
    ExtScratch xs;
    if (check) ZKB_TRY(xs.init(pk.get(), tmp));
    PkStream ps(ctx, io, format, false);
    ZKB_TRY(ps.init());
    auto where = [&](uint32_t column) { rep->section = (uint32_t)ps.section; rep->column = column; };
    // one polynomial of `len` elements: its length prefix, then its elements -> out (may be null), compared with ref when given
    auto poly = [&](uint32_t column, uint64_t len, Fr *dst, const Gather *ref) -> int32_t {
        where(column);
        uint32_t got = 0;
        ZKB_TRY(ps.read_u32(got));
        if (got != len) {
            set_error("pk file: section %d (%s) column %u has length %u, the constraint system needs %llu", ps.section, SECTION_NAMES[ps.section], column,
                      got, (unsigned long long)len);
            return ZKB_ERR_ARG;
        }
        ZKB_CUDA(cudaMemsetAsync(d_st, 0xff, 8, st));
        ZKB_CUDA(cudaMemsetAsync((uint8_t *)d_st + 8, 0, 8, st));
        ZKB_TRY(ps.read_elems(len, dst, ref, d_st));
        FrDecodeState h;
        ZKB_CUDA(cudaMemcpyAsync(&h, d_st, sizeof(h), cudaMemcpyDeviceToHost, st));
        ZKB_CUDA(cudaStreamSynchronize(st));
        if (h.count) {
            rep->first_index = h.first >> 3;
            rep->reason = (uint32_t)(h.first & 7);
            rep->count = h.count;
            set_error("pk file: section %d (%s) column %u: %llu bad element(s), the first at index %llu (%s)", ps.section, SECTION_NAMES[ps.section], column,
                      (unsigned long long)h.count, (unsigned long long)rep->first_index,
                      rep->reason == ZKB_PK_MISMATCH ? "differs from the form the key derives" : "not a canonical field element");
            return ZKB_ERR_ARG;
        }
        return ZKB_OK;
    };
    auto slice = [&](uint64_t count) -> int32_t {
        where(UINT32_MAX);
        uint32_t got = 0;
        ZKB_TRY(ps.read_u32(got));
        if (got != count) {
            set_error("pk file: section %d (%s) holds %u polynomials, the constraint system has %llu", ps.section, SECTION_NAMES[ps.section], got,
                      (unsigned long long)count);
            return ZKB_ERR_ARG;
        }
        return ZKB_OK;
    };
    Gather g;
    // 0 - 2: depend on the domain and the blinding factors only
    ps.section = 0;
    if (check) ZKB_TRY(xs.of(pk.get(), pk->l0_poly, g));
    ZKB_TRY(poly(0, N, nullptr, check ? &g : nullptr));
    ps.section = 1;
    if (check) ZKB_TRY(xs.of(pk.get(), pk->llast_poly, g));
    ZKB_TRY(poly(0, N, nullptr, check ? &g : nullptr));
    ps.section = 2;
    if (check) ZKB_TRY(xs.of_lactive(pk.get(), g));
    ZKB_TRY(poly(0, N, nullptr, check ? &g : nullptr));
    // 3 - 5 fixed, 6 - 8 permutation: values decoded and ingested, then the key's derived forms checked against the file's
    auto columns = [&](int first_section, size_t cnt, std::vector<Fr *> &vals, std::vector<Fr *> &polys) -> int32_t {
        ps.section = first_section;
        ZKB_TRY(slice(cnt));
        std::vector<Fr *> decoded(cnt);
        for (size_t c = 0; c < cnt; ++c) {
            ZKB_TRY(tmp.fr(n, &decoded[c]));
            ZKB_TRY(poly((uint32_t)c, n, decoded[c], nullptr));
        }
        ZKB_TRY(pk_ingest(pk.get(), (const void *const *)decoded.data(), cnt, vals, polys));
        ps.section = first_section + 1;
        ZKB_TRY(slice(cnt));
        for (size_t c = 0; c < cnt; ++c) {
            g = plain(polys[c]);
            ZKB_TRY(poly((uint32_t)c, n, nullptr, check ? &g : nullptr));
        }
        ps.section = first_section + 2;
        ZKB_TRY(slice(cnt));
        for (size_t c = 0; c < cnt; ++c) {
            if (check) ZKB_TRY(xs.of(pk.get(), polys[c], g));
            ZKB_TRY(poly((uint32_t)c, N, nullptr, check ? &g : nullptr));
        }
        return ZKB_OK;
    };
    ZKB_TRY(columns(3, cs.nf, pk->fixed_values, pk->fixed_polys));
    ZKB_TRY(columns(6, cs.perm.size(), pk->sigma_values, pk->sigma_polys));
    rep->section = rep->column = UINT32_MAX;
    ZKB_TRY(pk_finish(pk.get()));
    *out = pk.release();
    return ZKB_OK;
}

// v summed over the context's ranks (a COLLECTIVE)
static int32_t sum_over_ranks(zkb_ctx *ctx, uint64_t v, uint64_t &sum) {
    DevPool tmp;
    tmp.ctx = ctx;
    uint64_t *d = nullptr;
    ZKB_TRY(tmp.alloc(sizeof(uint64_t), (void **)&d));
    ZKB_CUDA(cudaMemcpyAsync(d, &v, sizeof(v), cudaMemcpyHostToDevice, ctx->stream));
    ZKB_TRY(comm_allreduce_u64(ctx, d, 1, ctx->stream));
    ZKB_CUDA(cudaMemcpyAsync(&sum, d, sizeof(sum), cudaMemcpyDeviceToHost, ctx->stream));
    ZKB_CUDA(cudaStreamSynchronize(ctx->stream));
    return ZKB_OK;
}

}  // namespace zkb

using namespace zkb;

extern "C" int32_t zkb_pk_vk_write(zkb_pk *pk, int32_t format, const zkb_io_vtable *io) {
    ZKB_ARG(pk && io && io->write && format_ok(format));
    std::vector<G1Affine> cms;
    ZKB_TRY(pk_vk_commitments(pk, cms));
    const size_t pt = format == ZKB_SERDE_PROCESSED ? 32 : sizeof(G1Affine);
    std::vector<uint8_t> buf(8 + pt * cms.size());
    const uint32_t hdr[2] = {pk->cs.k, pk->cs.nf};
    for (int w = 0; w < 2; ++w)
        for (int b = 0; b < 4; ++b) buf[4 * w + b] = (uint8_t)(hdr[w] >> (24 - 8 * b));
    for (size_t i = 0; i < cms.size(); ++i) {
        if (format == ZKB_SERDE_PROCESSED) g1_compress(cms[i], buf.data() + 8 + pt * i);
        else memcpy(buf.data() + 8 + pt * i, &cms[i], sizeof(G1Affine));
    }
    const int32_t rc = io->write(io->user, buf.data(), buf.size());
    if (rc) {
        set_error("pk file: the write callback failed (%d) in the vk section", rc);
        return ZKB_ERR_STATE;
    }
    return ZKB_OK;
}

extern "C" int32_t zkb_pk_write(zkb_pk *pk, int32_t format, const zkb_io_vtable *io) {
    ZKB_ARG(pk && io && io->write && format_ok(format));
    ZKB_CUDA(cudaSetDevice(pk->ctx->device));
    return pk_write_body(pk, format, io);
}

extern "C" int32_t zkb_pk_read(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, int32_t format, const zkb_io_vtable *io, zkb_srs *srs,
                               int32_t check, zkb_pk_read_report *rep, zkb_pk **out) {
    ZKB_ARG(rep);
    rep->section = rep->column = UINT32_MAX;
    rep->reason = ZKB_SERDE_OK;
    rep->reserved = 0;
    rep->first_index = UINT64_MAX;
    rep->count = 0;
    ZKB_ARG(ctx && csf && io && io->read && srs && out && format_ok(format) && (check == 0 || check == 1));
    *out = nullptr;
    ZKB_CUDA(cudaSetDevice(ctx->device));
    Csf cs;
    ZKB_TRY(load_csf(csf, csf_words, cs));
    ZKB_TRY(check_openings(cs));
    zkb_pk *pk = nullptr;
    int32_t r = pk_read_body(ctx, std::move(cs), format, io, srs, check != 0, rep, &pk);
    if (ctx->nranks > 1) {
        // every rank returns a key or none: the ranks' failures are summed before anyone keeps its key
        const uint64_t mine = r == ZKB_OK ? 0 : 1;
        uint64_t all = 0;
        const int32_t rc = sum_over_ranks(ctx, mine, all);
        if (r == ZKB_OK && (rc != ZKB_OK || all != 0)) {
            zkb_pk_destroy(pk);
            pk = nullptr;
            if (rc == ZKB_OK) set_error("zkb_pk_read: another rank failed to read its copy of the key file");
            r = rc != ZKB_OK ? rc : ZKB_ERR_ARG;
        }
    }
    if (r == ZKB_OK) *out = pk;
    return r;
}
