// check.cu -- the witness check (zkb_check_witness_dev): gate flags from the interpreter's flag build, lookup membership flags,
// copy-constraint flags, exact failure counts and the ordered extraction of failure records.
//
// Every item (a gate, a lookup input set, the copy list) owns a bitmap with one bit per row (per copy for the copy list); bit b of
// word w stands for row 32 w + b.  Every word is written by exactly one warp with __ballot_sync, so the bitmaps, the counts and the
// records are the same bytes on every run.  Only the counts and the first `cap` records cross PCIe, never a bitmap.
#include "lookup.cuh"

namespace zkb {

constexpr uint32_t CHECK_THREADS = 256;

struct CheckItem {
    const uint32_t *bits;   // bit b of word w: row (or copy index) 32 w + b fails
    uint64_t words;
    uint32_t kind, index, sub;   // the record fields (zkb_check_record); copies take index = copy index, row = left row
    uint64_t share, offset;      // extraction: records to write and where (filled by check_collect)
};

// the same probe as the prover's m_count_kernel, but one bit per row (word i / 32 by __ballot_sync, one writer per word) saying
// "input row i < usable is not in the table"; launched over all words of the bitmap, rows >= usable vote 0
__global__ void m_member_kernel(const Fr *__restrict__ f, const Fr *__restrict__ t, uint32_t usable, const uint32_t *__restrict__ slots,
                                uint32_t mask, uint32_t *__restrict__ bits, uint32_t words) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool missing = i < usable && m_probe(f, i, t, slots, mask) == NOT_IN_TABLE;
    const uint32_t b = __ballot_sync(0xffffffffu, missing);
    if ((threadIdx.x & 31) == 0 && (i >> 5) < words) bits[i >> 5] = b;
}

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

// bit i of bits[i / 32]: copy i's two cells differ.  Returns in *first_bad the first entry with a column >= P or a row >= n, or
// UINT64_MAX; synchronises.
static int32_t copy_flags_device(zkb_ctx *ctx, DevPool &pool, const uint32_t *copies, uint64_t n_copies, const Fr *const *d_perm_cols, uint32_t P,
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

// exact set-bit count of every item to counts_out, then the first `cap` set bits in item order to records_out (*n_records of them);
// only counts and records leave the device; synchronises
static int32_t check_collect(zkb_ctx *ctx, DevPool &pool, const std::vector<CheckItem> &items, const uint32_t *copies, uint64_t *counts_out,
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
using namespace zkb;

// MockProver::run + assert_satisfied on the device (semantics in zkb200.h): one bitmap per gate (the interpreter's flag build, one
// CSE scope per gate), per lookup input set (compression as the prover's lookup_prepare computes it, the table's hash set,
// m_member_kernel) and for the copy list, then exact counts and the first `cap` records (check_collect).
extern "C" int32_t zkb_check_witness_dev(zkb_ctx *ctx, const uint32_t *csf, uint64_t csf_words, const uint64_t *const *columns_dev,
                                         const uint64_t *challenges, const uint64_t *theta, const uint32_t *copies_dev, uint64_t n_copies,
                                         uint64_t *counts_out, zkb_check_record *records_out, uint32_t cap, uint32_t *n_records, void *stream) {
    ZKB_ARG(ctx && csf && columns_dev && counts_out && n_records && (records_out || cap == 0) && (copies_dev || n_copies == 0));
    ZKB_ARG(n_copies < (1ull << 32));
    ZKB_CUDA(cudaSetDevice(ctx->device));
    Csf cs;
    ZKB_TRY(load_csf(csf, csf_words, cs));
    if (cs.nch && !challenges) { set_error("zkb_check_witness_dev: the constraint system has %u challenges and none were given", cs.nch); return ZKB_ERR_ARG; }
    for (size_t l = 0; l < cs.lookups.size(); ++l)
        if (cs.lookups[l].table.size() > 1 && !theta) {
            set_error("zkb_check_witness_dev: lookup %zu has width %zu and needs theta", l, cs.lookups[l].table.size());
            return ZKB_ERR_ARG;
        }
    const std::vector<Fr> ch = host_challenges(challenges, cs.nch);
    Fr th = Fr::zero();
    if (theta) memcpy(th.l, theta, sizeof(Fr));
    cudaStream_t st = pick_stream(ctx, stream);
    const uint32_t n = 1u << cs.k, words = (n + 31) / 32;
    const uint32_t usable = n > cs.bf + 1 ? n - cs.bf - 1 : 0;
    const SlotMap sm(cs, 0);   // the caller's columns are its [fixed | advice | instance] prefix
    const std::vector<Fr *> cols((Fr *const *)columns_dev, (Fr *const *)columns_dev + sm.sigma0);
    size_t nsets = 0, maxsets = 0;
    for (auto &lk : cs.lookups) { nsets += lk.inputs.size(); maxsets = std::max(maxsets, lk.inputs.size()); }
    const uint64_t copy_words = (n_copies + 31) / 32;
    DevPool pool;
    pool.ctx = ctx;
    Fr **d_cols = nullptr;
    uint32_t *bits = nullptr;
    ZKB_TRY(upload_table(pool, cols, &d_cols, st));
    ZKB_TRY(pool.alloc(((cs.gates.size() + nsets) * words + copy_words) * 4, (void **)&bits));
    uint32_t *lk_bits = bits + cs.gates.size() * words, *copy_bits = lk_bits + nsets * words;
    std::vector<CheckItem> items;

    if (!cs.gates.empty()) {   // gates: one scope per gate, no selector folding
        ProfScope ps_(ctx, PROF_CHECK_GATES, st);
        ExprBuilder eb;
        ProgramBuilder pb(eb);
        std::vector<int64_t> memo(cs.nodes.size(), -1);
        for (size_t g = 0; g < cs.gates.size(); ++g)
            if (!pb.scope({{translate(cs, cs.gates[g], eb, sm, ch, memo), ProgramBuilder::FLAG, (uint32_t)g}})) {
                set_error("gate %zu: %s", g, pb.error.c_str());
                return ZKB_ERR_ARG;
            }
        DeviceProgram dp;
        ZKB_TRY(upload_program(pool, pb, eb, dp, st));
        ZKB_TRY(expr_flag_run_device(ctx, dp.code, dp.ncode, dp.nregs, d_cols, dp.consts, bits, words, cs.k, st));
    }
    for (size_t g = 0; g < cs.gates.size(); ++g) items.push_back({bits + g * words, words, 0, (uint32_t)g, 0, 0, 0});

    if (nsets) {               // lookups, one argument at a time: compressed inputs and table, the table's hash set, membership bits
        ProfScope ps_(ctx, PROF_CHECK_LOOKUPS, st);
        std::vector<Fr *> bufs(maxsets + 1);
        for (auto &b : bufs) ZKB_TRY(pool.fr(n, &b));
        uint32_t *slots = nullptr, mask = 0;
        uint32_t *out = lk_bits;
        for (size_t l = 0; l < cs.lookups.size(); ++l) {
            const size_t ns = cs.lookups[l].inputs.size();
            ZKB_TRY(lookup_compress(ctx, cs, l, sm, ch, th, pool, d_cols, std::vector<Fr *>(bufs.begin(), bufs.begin() + ns), bufs[maxsets], st));
            ZKB_TRY(table_hash_set(ctx, pool, bufs[maxsets], usable, slots, mask, st));
            for (size_t j = 0; j < ns; ++j, out += words) {
                m_member_kernel<<<(n + 255) / 256, 256, 0, st>>>(bufs[j], bufs[maxsets], usable, slots, mask, out, words);
                ctx->launches++;
                items.push_back({out, words, 1, (uint32_t)l, (uint32_t)j, 0, 0});
            }
            ZKB_CUDA(cudaGetLastError());
        }
    }

    {                          // copies
        ProfScope ps_(ctx, PROF_CHECK_COPIES, st);
        std::vector<Fr *> pc;
        for (auto &c : cs.perm) pc.push_back(cols[sm.perm(c)]);
        Fr **d_pc = nullptr;
        ZKB_TRY(upload_table(pool, pc, &d_pc, st));
        uint64_t first_bad = 0;
        ZKB_TRY(copy_flags_device(ctx, pool, copies_dev, n_copies, d_pc, (uint32_t)pc.size(), n, copy_bits, &first_bad, st));
        if (first_bad != ~0ull) {
            set_error("zkb_check_witness_dev: copy constraint %llu is out of range (column >= %zu or row >= %u)", (unsigned long long)first_bad,
                      pc.size(), n);
            return ZKB_ERR_ARG;
        }
    }
    items.push_back({copy_bits, copy_words, 2, 0, 0, 0, 0});

    ZKB_TRY(check_collect(ctx, pool, items, copies_dev, counts_out, records_out, cap, n_records, st));
    // poisoned gate failures: an advice query of the gate reads a row >= usable at the failing row
    std::vector<std::vector<int32_t>> adv_rots(cs.gates.size());
    std::vector<bool> adv_rots_done(cs.gates.size(), false);
    for (uint32_t i = 0; i < *n_records && records_out[i].kind == 0; ++i) {
        zkb_check_record &r = records_out[i];
        std::vector<int32_t> &rots = adv_rots[r.index];
        if (!adv_rots_done[r.index]) {
            std::vector<uint32_t> stack{cs.gates[r.index]};
            std::vector<bool> seen(cs.nodes.size(), false);
            while (!stack.empty()) {
                const uint32_t v = stack.back();
                stack.pop_back();
                if (seen[v]) continue;
                seen[v] = true;
                const auto &nd = cs.nodes[v];
                if (nd[0] == N_ADVICE) rots.push_back((int32_t)nd[2]);
                else if (nd[0] == N_NEG || nd[0] == N_SCALED) stack.push_back(nd[1]);
                else if (nd[0] == N_ADD || nd[0] == N_MUL) { stack.push_back(nd[1]); stack.push_back(nd[2]); }
            }
            adv_rots_done[r.index] = true;
        }
        r.sub = 0;
        for (int32_t rot : rots)
            if (((r.row + (uint32_t)rot) & (n - 1)) >= usable) { r.sub = 1; break; }
    }
    return ZKB_OK;
}
