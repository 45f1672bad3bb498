// lookup.cuh -- the mv-lookup's compressed values and the hash set of a compressed table, shared by the prover's multiplicities
// (lookup_multiplicities, lookup.cu) and the witness check's membership flags (m_member_kernel, check.cu).  The set is an open-addressing
// hash table keyed by the 32-byte compressed table value.
#pragma once
#include "csf.cuh"

namespace zkb {

__device__ __forceinline__ uint32_t key_hash(const Fr &k) {
    uint32_t h = 0x9e3779b9u;
#pragma unroll
    for (int i = 0; i < 8; ++i) { h ^= k.l[i]; h *= 0x85ebca6bu; h ^= h >> 13; }
    return h;
}
constexpr uint32_t NOT_IN_TABLE = 0xffffffffu;
// the table row holding input row i's value, or NOT_IN_TABLE
__device__ __forceinline__ uint32_t m_probe(const Fr *__restrict__ f, uint32_t i, const Fr *__restrict__ t, const uint32_t *__restrict__ slots,
                                            uint32_t mask) {
    const Fr key = fp_load(f + i);
    uint32_t h = key_hash(key) & mask;
    while (true) {
        const uint32_t s = slots[h];
        if (s == 0) return NOT_IN_TABLE;
        if (fp_load(t + (s - 1)) == key) return s - 1;
        h = (h + 1) & mask;
    }
}

// lookup l's compressed input sets into f[j] and its compressed table into t, over the 2^k rows of the d_cols table
int32_t lookup_compress(zkb_ctx *ctx, const Csf &cs, size_t l, const SlotMap &sm, const std::vector<Fr> &ch, const Fr &theta, DevPool &pool,
                        const Fr *const *d_cols, std::vector<Fr *> f, Fr *t, cudaStream_t st);
// the hash set of table t's usable rows that m_probe searches: the smallest power of two >= 2 usable slots, cleared, then filled.
// `slots` is allocated when null and otherwise reused (its size depends on `usable` only).
int32_t table_hash_set(zkb_ctx *ctx, DevPool &pool, const Fr *t, uint32_t usable, uint32_t *&slots, uint32_t &mask, cudaStream_t st);
// mv_lookup/prover.rs multiplicities: m_out[r] (n Fr, Montgomery) = the number of input rows i < usable, over the n_sets compressed
// input sets f[j] (a host array of device pointers), whose value is the one table t holds at row r, where r is the LAST row < usable
// holding that value (BTreeMap collect()); rows >= usable are zero.  Builds t's hash set into `slots` / `mask` (table_hash_set) and
// sets *unsatisfied when an input row < usable is not in the table.  Synchronises st.
int32_t lookup_multiplicities(zkb_ctx *ctx, DevPool &pool, const Fr *const *f, size_t n_sets, const Fr *t, uint64_t n, uint32_t usable, Fr *m_out,
                              uint32_t *&slots, uint32_t &mask, bool *unsatisfied, cudaStream_t st);

}  // namespace zkb
