// lookup.cu -- lookup compression and the table hash set (see lookup.cuh).
#include "lookup.cuh"

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

}  // namespace zkb
