// expr.cu -- device interpreter for constraint-expression programs (see expr.cuh).
#include <atomic>
#include <type_traits>
#include "common.cuh"
#include "expr.cuh"

namespace zkb {

struct ExprLaunch {
    const Instr *code;
    uint32_t ncode;
    const Fr *const *cols;   // column slot -> device array of (1 << log_n) elements
    const Fr *consts;
    Fr *const *outs;         // output slot -> device array
    uint32_t log_n;
    uint32_t out_stride;     // output index = row * out_stride + out_offset
    uint32_t out_offset;
};

// Register file of the interpreter.  SMEM = true: in SHARED memory, two 16-byte planes indexed [reg][thread] (adjacent lanes touch
// adjacent 16-byte slots: conflict free).  SMEM = false: local memory, 512 B per thread at NREGS = 16: with every SM full that is
// more than the L2 holds, so the "registers" and the column data evict each other and the DRAM traffic is a multiple of the
// algorithmic one.
template <int NREGS, int THREADS, bool SMEM>
struct RegFile {
    uint4 *lo, *hi;
    Fr loc[SMEM ? 1 : NREGS];
    __device__ __forceinline__ RegFile(uint4 *base) : lo(base + threadIdx.x), hi(base + NREGS * THREADS + threadIdx.x) {}
    __device__ __forceinline__ Fr get(uint32_t r) const {
        if (!SMEM) return loc[r];
        const uint4 a = lo[r * THREADS], b = hi[r * THREADS];
        Fr v;
        v.l[0] = a.x; v.l[1] = a.y; v.l[2] = a.z; v.l[3] = a.w;
        v.l[4] = b.x; v.l[5] = b.y; v.l[6] = b.z; v.l[7] = b.w;
        return v;
    }
    __device__ __forceinline__ void set(uint32_t r, const Fr &v) {
        if (!SMEM) { loc[r] = v; return; }
        lo[r * THREADS] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
        hi[r * THREADS] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
    }
};

// Flag build of the interpreter (zkb_check_witness_dev): a gate program whose roots are FLAG(gate) instructions.  FLAG sets bit
// `row` of the gate's bitmap when the value is not zero.  A warp's 32 rows make one 32-bit word, written by that warp's lane 0
// from __ballot_sync: every word has exactly one writer, no atomics, and the bitmap is the same on every run.  Lanes past the last
// row (k < 5: fewer rows than a warp) evaluate row mod n and vote 0, so the whole warp reaches every ballot.  A separate kernel
// (the accumulator and output roots compile out of it), sharing run_program with expr_kernel.
struct FlagLaunch {
    const Instr *code;
    uint32_t ncode;
    const Fr *const *cols;
    const Fr *consts;
    uint32_t *bits;          // bitmap of gate g: bits + g * words
    uint32_t words;          // (n + 31) / 32
    uint32_t log_n;
};

// The interpreter loop of both kernels for thread `tid` (row tid mod n).  Every form of one operation ends in the same field
// operation (the goto targets after the switch), so a fused form costs its operand fetches and no second copy of the arithmetic.
// The sums of two products (FOLD and the merged HORNER forms) share one tail.
template <int NREGS, int THREADS, bool SMEM, class Launch>
__device__ __forceinline__ void run_program(const Launch &L, uint32_t tid) {
    constexpr bool FLAG = std::is_same<Launch, FlagLaunch>::value;
    extern __shared__ uint4 expr_smem[];
    const uint32_t mask = (1u << L.log_n) - 1, row = tid & mask;
    RegFile<NREGS, THREADS, SMEM> regs(expr_smem);
    Fr acc = Fr::zero(), acc2 = Fr::zero();
    uint32_t pc = 0;
    auto col = [&](uint32_t imm) {   // imm = slot | rotation << 16
        const int32_t rot = (int32_t)(int16_t)(imm >> 16);
        return fp_load(L.cols[imm & 0xffffu] + ((row + (uint32_t)rot) & mask));
    };
    auto cst = [&](uint32_t i) { return fp_load(L.consts + i); };
    auto arg = [&]() { return L.code[++pc].imm; };   // the OP_ARG word after the current instruction
    for (; pc < L.ncode; ++pc) {
        const Instr in = L.code[pc];
        Fr x, y, z, w;
        switch (in.op) {
        case OP_LOADCOL: regs.set(in.dst, col(in.imm)); continue;
        case OP_LOADCONST: regs.set(in.dst, cst(in.imm)); continue;
        case OP_ADD: x = regs.get(in.a); y = regs.get(in.b); goto add;
        case OP_ADD_RC + FORM_RC: x = regs.get(in.a); y = col(in.imm); goto add;
        case OP_ADD_RC + FORM_CR: x = col(in.imm); y = regs.get(in.a); goto add;
        case OP_ADD_RC + FORM_RK: x = regs.get(in.a); y = cst(in.imm); goto add;
        case OP_ADD_RC + FORM_KR: x = cst(in.imm); y = regs.get(in.a); goto add;
        case OP_ADD_RC + FORM_CC: x = col(in.imm); y = col(arg()); goto add;
        case OP_ADD_RC + FORM_CK: x = col(in.imm); y = cst(arg()); goto add;
        case OP_ADD_RC + FORM_KC: x = cst(in.imm); y = col(arg()); goto add;
        case OP_SUB: x = regs.get(in.a); y = regs.get(in.b); goto sub;
        case OP_SUB_RC + FORM_RC: x = regs.get(in.a); y = col(in.imm); goto sub;
        case OP_SUB_RC + FORM_CR: x = col(in.imm); y = regs.get(in.a); goto sub;
        case OP_SUB_RC + FORM_RK: x = regs.get(in.a); y = cst(in.imm); goto sub;
        case OP_SUB_RC + FORM_KR: x = cst(in.imm); y = regs.get(in.a); goto sub;
        case OP_SUB_RC + FORM_CC: x = col(in.imm); y = col(arg()); goto sub;
        case OP_SUB_RC + FORM_CK: x = col(in.imm); y = cst(arg()); goto sub;
        case OP_SUB_RC + FORM_KC: x = cst(in.imm); y = col(arg()); goto sub;
        case OP_MUL: x = regs.get(in.a); y = regs.get(in.b); goto mul;
        case OP_MUL_RC + FORM_RC: x = regs.get(in.a); y = col(in.imm); goto mul;
        case OP_MUL_RC + FORM_CR: x = col(in.imm); y = regs.get(in.a); goto mul;
        case OP_MUL_RC + FORM_RK: x = regs.get(in.a); y = cst(in.imm); goto mul;
        case OP_MUL_RC + FORM_KR: x = cst(in.imm); y = regs.get(in.a); goto mul;
        case OP_MUL_RC + FORM_CC: x = col(in.imm); y = col(arg()); goto mul;
        case OP_MUL_RC + FORM_CK: x = col(in.imm); y = cst(arg()); goto mul;
        case OP_MUL_RC + FORM_KC: x = cst(in.imm); y = col(arg()); goto mul;
        case OP_NEG: regs.set(in.dst, fp_neg(regs.get(in.a))); continue;
        case OP_FLAG:
            if constexpr (FLAG) {
                const uint32_t b = __ballot_sync(0xffffffffu, tid < (1u << L.log_n) && !regs.get(in.a).is_zero());
                const uint32_t word = tid >> 5;
                if ((threadIdx.x & 31) == 0 && word < L.words) L.bits[(size_t)in.imm * L.words + word] = b;
            }
            continue;
        case OP_HORNER: case OP_HORNER_C:
            if constexpr (!FLAG) acc = fp_add(fp_mul(acc, cst(in.imm)), in.op == OP_HORNER ? regs.get(in.a) : col(arg()));
            continue;
        case OP_HORNER2: case OP_HORNER2_C:
            if constexpr (!FLAG) acc2 = fp_add(fp_mul(acc2, cst(in.imm)), in.op == OP_HORNER2 ? regs.get(in.a) : col(arg()));
            continue;
        case OP_FOLD: case OP_FOLD_C:
            if constexpr (FLAG) continue;
            else { x = acc; y = cst(in.imm); z = in.op == OP_FOLD ? regs.get(in.a) : col(arg()); w = acc2; goto mac; }
        case OP_HORNER_M: case OP_HORNER2_M:
            if constexpr (FLAG) continue;
            else if constexpr (!SMEM) {
                // the local-memory build (programs of > 16 registers) keeps its register budget: product first, then the root
                const Fr t = fp_mul(regs.get(in.a), regs.get(in.b));
                if (in.op == OP_HORNER_M) acc = fp_add(fp_mul(acc, cst(in.imm)), t);
                else acc2 = fp_add(fp_mul(acc2, cst(in.imm)), t);
                continue;
            } else { x = in.op == OP_HORNER_M ? acc : acc2; y = cst(in.imm); z = regs.get(in.a); w = regs.get(in.b); goto mac; }
        case OP_STORE:
            if constexpr (!FLAG) fp_store(L.outs[in.imm] + (size_t)row * L.out_stride + L.out_offset, regs.get(in.a));
            continue;
        case OP_STOREACC:
            if constexpr (!FLAG) fp_store(L.outs[in.imm & 0xffu] + (size_t)row * L.out_stride + L.out_offset, fp_mul(acc, cst(in.imm >> 8)));
            continue;
        case OP_CLEARACC: acc = Fr::zero(); continue;
        default: continue;
        }
    add: regs.set(in.dst, fp_add(x, y)); continue;
    sub: regs.set(in.dst, fp_sub(x, y)); continue;
    mul: regs.set(in.dst, fp_mul(x, y)); continue;
    mac: {   // x * y + z * w, one reduction: FOLD and the merged HORNER forms
        const Fr r = fp_mul_add_mul(x, y, z, w);
        if (in.op == OP_HORNER2_M) acc2 = r;
        else {
            acc = r;
            if (in.op != OP_HORNER_M) acc2 = Fr::zero();   // FOLD
        }
    }
    }
}

template <int NREGS, int THREADS, bool SMEM>
__global__ void __launch_bounds__(THREADS) expr_kernel(ExprLaunch L) {
    const uint32_t row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= (1u << L.log_n)) return;
    run_program<NREGS, THREADS, SMEM>(L, row);
}

template <int NREGS, int THREADS, bool SMEM>
__global__ void __launch_bounds__(THREADS) expr_flag_kernel(FlagLaunch L) {
    run_program<NREGS, THREADS, SMEM>(L, blockIdx.x * blockDim.x + threadIdx.x);
}

// one launch of KERNEL with its register file in dynamic shared memory (NREGS x THREADS x 32 bytes)
template <class Launch, int NREGS, int THREADS, void (*KERNEL)(Launch)>
static int32_t launch_smem(const Launch &L, uint32_t n, cudaStream_t st) {
    constexpr size_t bytes = (size_t)NREGS * THREADS * 32;
    // the opt-in is per device; contexts of one process may launch from several threads at the same time.  Setting it is
    // idempotent, so threads that both find the flag clear both set it; the flag is published only after the attribute is set
    static std::atomic<bool> attr_set[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (bytes > 48 * 1024 && dev < 64 && !attr_set[dev].load(std::memory_order_acquire)) {
        ZKB_CUDA(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        attr_set[dev].store(true, std::memory_order_release);
    }
    KERNEL<<<(n + THREADS - 1) / THREADS, THREADS, bytes, st>>>(L);
    return ZKB_OK;
}

int32_t expr_run_device(zkb_ctx *ctx, const Instr *d_code, uint32_t ncode, int nregs, const Fr *const *d_cols, const Fr *d_consts,
                        Fr *const *d_outs, uint32_t log_n, uint32_t out_stride, uint32_t out_offset, cudaStream_t st) {
    ExprLaunch L{d_code, ncode, d_cols, d_consts, d_outs, log_n, out_stride, out_offset};
    const uint32_t n = 1u << log_n;
    const unsigned blocks = (n + 127) / 128;
    ProfScope ps_(ctx, PROF_EXPR, st);
    // Register file placement: in local memory the registers and the columns compete for the 50 MB L2; in shared memory 16
    // registers take 64 KB per 128 threads, which leaves 12 warps per SM.  On an H100 (80 GB SXM, 400 W power limit) the k = 20
    // quotient program (9-16 registers) is faster from shared memory: 1.00 s instead of 1.18 s of interpreter time per proof,
    // and the lower DRAM traffic lets the power-capped card hold higher clocks.  Programs of <= 16 registers therefore run from
    // shared memory (32 KB per block for <= 8 registers), larger ones from local memory.
    if (nregs <= 8) ZKB_TRY((launch_smem<ExprLaunch, 8, 128, expr_kernel<8, 128, true>>(L, n, st)));
    else if (nregs <= 16) ZKB_TRY((launch_smem<ExprLaunch, 16, 128, expr_kernel<16, 128, true>>(L, n, st)));
    else expr_kernel<64, 128, false><<<blocks, 128, 0, st>>>(L);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

int32_t expr_flag_run_device(zkb_ctx *ctx, const Instr *d_code, uint32_t ncode, int nregs, const Fr *const *d_cols, const Fr *d_consts,
                             uint32_t *bits, uint32_t words, uint32_t log_n, cudaStream_t st) {
    FlagLaunch L{d_code, ncode, d_cols, d_consts, bits, words, log_n};
    const uint32_t n = 1u << log_n;
    if (nregs <= 8) ZKB_TRY((launch_smem<FlagLaunch, 8, 128, expr_flag_kernel<8, 128, true>>(L, n, st)));
    else if (nregs <= 16) ZKB_TRY((launch_smem<FlagLaunch, 16, 128, expr_flag_kernel<16, 128, true>>(L, n, st)));
    else expr_flag_kernel<64, 128, false><<<(n + 127) / 128, 128, 0, st>>>(L);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

}  // namespace zkb
