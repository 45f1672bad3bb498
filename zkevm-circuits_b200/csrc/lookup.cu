// lookup.cu -- lookup compression and the table hash set (see lookup.cuh).
#include "lookup.cuh"
#include <algorithm>

namespace zkb {

__global__ void m_insert_kernel(const Fr *__restrict__ t, uint32_t usable, uint32_t *slots, uint32_t mask) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= usable) return;
    const uint32_t i = usable - 1 - tid;  // descending row order: the winning (last) duplicate tends to arrive first
    const Fr key = fp_load(t + i);
    uint32_t h = key_hash(key) & mask;
    while (true) {
        const uint32_t s = atomicCAS(&slots[h], 0u, i + 1);
        if (s == 0) return;
        if (fp_load(t + (s - 1)) == key) {   // BTreeMap collect(): the last duplicate table row wins
            if (s < i + 1) atomicMax(&slots[h], i + 1);
            return;
        }
        h = (h + 1) & mask;
    }
}

// multiplicities of the mv-lookup: input rows counted per table row through the table's hash set
__global__ void m_count_kernel(const Fr *__restrict__ f, const Fr *__restrict__ t, uint32_t usable, const uint32_t *__restrict__ slots,
                               uint32_t mask, uint32_t *counts, int *err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t target = NOT_IN_TABLE;
    if (i < usable) {
        target = m_probe(f, i, t, slots, mask);
        if (target == NOT_IN_TABLE) atomicExch(err, 1);  // input not in table: unsatisfied lookup
    }
    // most rows of a zkEVM lookup hit the same few table rows (selector off -> the all-zero row): aggregate per warp
    const uint32_t peers = __match_any_sync(0xffffffffu, target);
    if (target != NOT_IN_TABLE && (threadIdx.x & 31) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&counts[target], (uint32_t)__popc(peers));
}
__global__ void counts_to_fr_kernel(const uint32_t *__restrict__ counts, uint32_t n, Fr *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fp_store(out + i, fp_from_u64<FrParams>(counts[i]));
}

int32_t lookup_compress(zkb_ctx *ctx, const Csf &cs, size_t l, const SlotMap &sm, const std::vector<Fr> &ch, const Fr &theta, DevPool &pool,
                        const Fr *const *d_cols, std::vector<Fr *> f, Fr *t, cudaStream_t st) {
    const CsfLookup &lk = cs.lookups[l];
    ExprBuilder eb;
    std::vector<int64_t> memo(cs.nodes.size(), -1);
    std::vector<uint32_t> roots;
    for (auto &inp : lk.inputs) roots.push_back(compress_exprs(cs, inp, eb, sm, ch, memo, theta));
    roots.push_back(compress_exprs(cs, lk.table, eb, sm, ch, memo, theta));
    f.push_back(t);
    return run_store_program(ctx, cs.k, pool, eb, roots, f, d_cols, "lookup " + std::to_string(l), st);
}

int32_t table_hash_set(zkb_ctx *ctx, DevPool &pool, const Fr *t, uint32_t usable, uint32_t *&slots, uint32_t &mask, cudaStream_t st) {
    uint32_t tsize = 1;
    while (tsize < 2 * usable) tsize <<= 1;
    if (!slots) ZKB_TRY(pool.alloc((size_t)tsize * 4, (void **)&slots));
    mask = tsize - 1;
    ZKB_CUDA(cudaMemsetAsync(slots, 0, (size_t)tsize * 4, st));
    if (usable) {   // the witness check takes circuits too small to have usable rows
        m_insert_kernel<<<(usable + 255) / 256, 256, 0, st>>>(t, usable, slots, mask);
        ctx->launches++;
    }
    return ZKB_OK;
}

int32_t lookup_multiplicities(zkb_ctx *ctx, DevPool &pool, const Fr *const *f, size_t n_sets, const Fr *t, uint64_t n, uint32_t usable, Fr *m_out,
                              uint32_t *&slots, uint32_t &mask, bool *unsatisfied, cudaStream_t st) {
    ZKB_TRY(table_hash_set(ctx, pool, t, usable, slots, mask, st));
    uint32_t *counts = nullptr;
    ZKB_TRY(pool.alloc((size_t)n * 4 + 16, (void **)&counts));
    int *d_err = (int *)(counts + n);
    ZKB_CUDA(cudaMemsetAsync(counts, 0, (size_t)n * 4 + 16, st));
    for (size_t j = 0; j < n_sets; ++j) m_count_kernel<<<(usable + 255) / 256, 256, 0, st>>>(f[j], t, usable, slots, mask, counts, d_err);
    counts_to_fr_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(counts, (uint32_t)n, m_out);
    ctx->launches += 1 + n_sets;
    ZKB_CUDA(cudaGetLastError());
    int herr = 0;
    ZKB_CUDA(cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    *unsatisfied = herr != 0;
    return ZKB_OK;
}

}  // namespace zkb
using namespace zkb;

// the prover's multiplicities over caller buffers (semantics in zkb200.h)
extern "C" int32_t zkb_lookup_multiplicities_dev(zkb_ctx *ctx, const uint64_t *const *inputs_dev, uint32_t n_sets, const uint64_t *table_dev, uint64_t n,
                                                 uint32_t usable, uint64_t *m_out_dev, int32_t *unsatisfied, uint32_t *slots_out, uint64_t slots_cap,
                                                 uint64_t *n_slots, void *stream) {
    ZKB_ARG(ctx && inputs_dev && n_sets > 0 && table_dev && m_out_dev && unsatisfied && (slots_out || slots_cap == 0));
    ZKB_ARG(usable > 0 && usable < n && n <= (1ull << 31));
    for (uint32_t j = 0; j < n_sets; ++j) ZKB_ARG(inputs_dev[j]);
    ZKB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pick_stream(ctx, stream);
    DevPool pool;
    pool.ctx = ctx;
    uint32_t *slots = nullptr, mask = 0;
    bool unsat = false;
    ZKB_TRY(lookup_multiplicities(ctx, pool, (const Fr *const *)inputs_dev, n_sets, (const Fr *)table_dev, n, usable, (Fr *)m_out_dev, slots, mask,
                                  &unsat, st));
    *unsatisfied = unsat ? 1 : 0;
    const uint64_t tsize = (uint64_t)mask + 1;
    if (n_slots) *n_slots = tsize;
    if (slots_cap) {
        ZKB_CUDA(cudaMemcpyAsync(slots_out, slots, std::min<uint64_t>(slots_cap, tsize) * 4, cudaMemcpyDeviceToHost, st));
        ZKB_CUDA(cudaStreamSynchronize(st));
    }
    return ZKB_OK;
}
