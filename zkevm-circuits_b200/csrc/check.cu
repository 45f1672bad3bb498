// check.cu -- the bitmap side of the witness check (zkb_check_witness_dev, prover.cu): copy-constraint flags, exact failure counts
// and the ordered extraction of failure records.
//
// Every item (a gate, a lookup input set, the copy list) owns a bitmap with one bit per row (per copy for the copy list); bit b of
// word w stands for row 32 w + b.  Every word is written by exactly one warp with __ballot_sync, so the bitmaps, the counts and the
// records are the same bytes on every run.  Only the counts and the first `cap` records cross PCIe, never a bitmap.
#include "common.cuh"

namespace zkb {

constexpr uint32_t CHECK_THREADS = 256;

// one thread per copy (lc, lr, rc, rr); columns index the permutation column list.  An entry out of range votes 0 and lowers
// *first_bad to its index (atomicMin: the first offending entry whatever the schedule).
__global__ void copy_flag_kernel(const uint32_t *__restrict__ copies, uint64_t n_copies, const Fr *const *__restrict__ perm_cols, uint32_t P,
                                 uint32_t n, uint32_t *__restrict__ bits, unsigned long long *first_bad) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    bool differ = false;
    if (i < n_copies) {
        const uint32_t lc = copies[4 * i], lr = copies[4 * i + 1], rc = copies[4 * i + 2], rr = copies[4 * i + 3];
        if (lc >= P || rc >= P || lr >= n || rr >= n) atomicMin(first_bad, (unsigned long long)i);
        else differ = !(fp_load(perm_cols[lc] + lr) == fp_load(perm_cols[rc] + rr));
    }
    const uint32_t b = __ballot_sync(0xffffffffu, differ);
    if ((threadIdx.x & 31) == 0 && (i >> 5) < (n_copies + 31) / 32) bits[i >> 5] = b;
}

// one CTA per item: popcount of its words -> counts[item]
__global__ void __launch_bounds__(CHECK_THREADS) bitmap_count_kernel(const CheckItem *__restrict__ items, unsigned long long *counts) {
    __shared__ unsigned long long part[CHECK_THREADS / 32];
    const CheckItem it = items[blockIdx.x];
    unsigned long long c = 0;
    for (uint64_t w = threadIdx.x; w < it.words; w += CHECK_THREADS) c += __popc(it.bits[w]);
    for (int d = 16; d > 0; d >>= 1) c += __shfl_down_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (uint32_t j = 0; j < CHECK_THREADS / 32; ++j) t += part[j];
        counts[blockIdx.x] = t;
    }
}

// one CTA per item with a share: walk the item's words in order, CHECK_THREADS at a time; a block-wide exclusive scan of the
// popcounts gives each word's first record slot, and the set bits are written in ascending order until the share is filled
__global__ void __launch_bounds__(CHECK_THREADS) bitmap_extract_kernel(const CheckItem *__restrict__ items, const uint32_t *__restrict__ copies,
                                                                       zkb_check_record *__restrict__ out) {
    __shared__ uint32_t warp_sum[CHECK_THREADS / 32];
    const CheckItem it = items[blockIdx.x];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint64_t written = 0;
    for (uint64_t base = 0; base < it.words && written < it.share; base += CHECK_THREADS) {   // both conditions are block-uniform
        const uint64_t w = base + threadIdx.x;
        const uint32_t word = w < it.words ? it.bits[w] : 0u;
        const uint32_t c = __popc(word);
        uint32_t incl = c;
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= (uint32_t)d) incl += y;
        }
        if (lane == 31) warp_sum[wid] = incl;
        __syncthreads();
        uint32_t before = 0, total = 0;
        for (uint32_t j = 0; j < CHECK_THREADS / 32; ++j) {
            const uint32_t t = warp_sum[j];
            if (j < wid) before += t;
            total += t;
        }
        __syncthreads();   // warp_sum is rewritten by the next round
        uint64_t pos = written + before + (incl - c);
        for (uint32_t m = word; m && pos < it.share; m &= m - 1, ++pos) {
            const uint64_t idx = w * 32 + (uint32_t)(__ffs(m) - 1);
            zkb_check_record r;
            r.kind = it.kind;
            if (it.kind == 2) { r.index = (uint32_t)idx; r.sub = 0; r.row = copies[4 * idx + 1]; }
            else { r.index = it.index; r.sub = it.sub; r.row = (uint32_t)idx; }
            out[it.offset + pos] = r;
        }
        written += total;
    }
}

int32_t copy_flags_device(zkb_ctx *ctx, DevPool &pool, const uint32_t *copies, uint64_t n_copies, const Fr *const *d_perm_cols, uint32_t P,
                          uint32_t n, uint32_t *bits, uint64_t *first_bad, cudaStream_t st) {
    unsigned long long *d_bad = nullptr;
    ZKB_TRY(pool.alloc(8, (void **)&d_bad));
    ZKB_CUDA(cudaMemsetAsync(d_bad, 0xff, 8, st));
    if (n_copies) {
        copy_flag_kernel<<<(unsigned)((n_copies + CHECK_THREADS - 1) / CHECK_THREADS), CHECK_THREADS, 0, st>>>(copies, n_copies, d_perm_cols, P, n,
                                                                                                                bits, d_bad);
        ctx->launches++;
        ZKB_CUDA(cudaGetLastError());
    }
    unsigned long long bad = 0;
    ZKB_CUDA(cudaMemcpyAsync(&bad, d_bad, 8, cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    *first_bad = bad;
    return ZKB_OK;
}

int32_t check_collect(zkb_ctx *ctx, DevPool &pool, const std::vector<CheckItem> &items, const uint32_t *copies, uint64_t *counts_out,
                      zkb_check_record *records_out, uint32_t cap, uint32_t *n_records, cudaStream_t st) {
    ProfScope ps_(ctx, PROF_CHECK_EXTRACT, st);
    const size_t ni = items.size();
    CheckItem *d_items = nullptr;
    unsigned long long *d_counts = nullptr;
    ZKB_TRY(pool.alloc(ni * sizeof(CheckItem), (void **)&d_items));
    ZKB_TRY(pool.alloc(ni * sizeof(unsigned long long), (void **)&d_counts));
    ZKB_CUDA(cudaMemcpyAsync(d_items, items.data(), ni * sizeof(CheckItem), cudaMemcpyHostToDevice, st));
    bitmap_count_kernel<<<(unsigned)ni, CHECK_THREADS, 0, st>>>(d_items, d_counts);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    static_assert(sizeof(unsigned long long) == sizeof(uint64_t), "counts are copied as u64");
    ZKB_CUDA(cudaMemcpyAsync(counts_out, d_counts, ni * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    // each item's share of `cap`, in report order
    std::vector<CheckItem> busy;
    uint64_t left = cap, offset = 0;
    for (size_t i = 0; i < ni && left; ++i) {
        const uint64_t share = std::min<uint64_t>(counts_out[i], left);
        if (!share) continue;
        CheckItem it = items[i];
        it.share = share;
        it.offset = offset;
        busy.push_back(it);
        offset += share;
        left -= share;
    }
    *n_records = (uint32_t)offset;
    if (busy.empty()) return ZKB_OK;
    CheckItem *d_busy = nullptr;
    zkb_check_record *d_rec = nullptr;
    ZKB_TRY(pool.alloc(busy.size() * sizeof(CheckItem), (void **)&d_busy));
    ZKB_TRY(pool.alloc(offset * sizeof(zkb_check_record), (void **)&d_rec));
    ZKB_CUDA(cudaMemcpyAsync(d_busy, busy.data(), busy.size() * sizeof(CheckItem), cudaMemcpyHostToDevice, st));
    bitmap_extract_kernel<<<(unsigned)busy.size(), CHECK_THREADS, 0, st>>>(d_busy, copies, d_rec);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    ZKB_CUDA(cudaMemcpyAsync(records_out, d_rec, offset * sizeof(zkb_check_record), cudaMemcpyDeviceToHost, st));
    ZKB_CUDA(cudaStreamSynchronize(st));   // `busy` is read by the copy above
    return ZKB_OK;
}

}  // namespace zkb
