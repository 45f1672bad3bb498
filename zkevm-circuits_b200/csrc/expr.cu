// expr.cu -- device interpreter for constraint-expression programs (see expr.cuh).
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

template <int NREGS, int THREADS, bool SMEM>
__global__ void __launch_bounds__(THREADS) expr_kernel(ExprLaunch L) {
    extern __shared__ uint4 expr_smem[];
    const uint32_t n = 1u << L.log_n, mask = n - 1;
    const uint32_t row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    RegFile<NREGS, THREADS, SMEM> regs(expr_smem);
    Fr acc = Fr::zero(), acc2 = Fr::zero();
    for (uint32_t pc = 0; pc < L.ncode; ++pc) {
        const Instr in = L.code[pc];
        switch (in.op) {
        case OP_LOADCOL: {
            const int32_t rot = (int32_t)(int16_t)(in.imm >> 16);
            const uint32_t r = (row + (uint32_t)rot) & mask;
            regs.set(in.dst, fp_load(L.cols[in.imm & 0xffffu] + r));
        } break;
        case OP_LOADCONST: regs.set(in.dst, fp_load(L.consts + in.imm)); break;
        case OP_ADD: { Fr a = regs.get(in.a), b = regs.get(in.b); regs.set(in.dst, fp_add(a, b)); } break;
        case OP_SUB: { Fr a = regs.get(in.a), b = regs.get(in.b); regs.set(in.dst, fp_sub(a, b)); } break;
        case OP_MUL: { Fr a = regs.get(in.a), b = regs.get(in.b); regs.set(in.dst, fp_mul(a, b)); } break;
        case OP_NEG: { Fr a = regs.get(in.a); regs.set(in.dst, fp_neg(a)); } break;
        case OP_HORNER: acc = fp_add(fp_mul(acc, fp_load(L.consts + in.imm)), regs.get(in.a)); break;
        case OP_STORE: fp_store(L.outs[in.imm] + (size_t)row * L.out_stride + L.out_offset, regs.get(in.a)); break;
        case OP_STOREACC:
            fp_store(L.outs[in.imm & 0xffu] + (size_t)row * L.out_stride + L.out_offset, fp_mul(acc, fp_load(L.consts + (in.imm >> 8))));
            break;
        case OP_CLEARACC: acc = Fr::zero(); break;
        case OP_HORNER2: acc2 = fp_add(fp_mul(acc2, fp_load(L.consts + in.imm)), regs.get(in.a)); break;
        case OP_FOLD:
            acc = fp_add(fp_mul(acc, fp_load(L.consts + in.imm)), fp_mul(regs.get(in.a), acc2));
            acc2 = Fr::zero();
            break;
        default: break;
        }
    }
}

template <int NREGS, int THREADS>
static int32_t launch_smem(const ExprLaunch &L, uint32_t n, cudaStream_t st) {
    constexpr size_t bytes = (size_t)NREGS * THREADS * 32;
    static bool attr_set[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (bytes > 48 * 1024 && dev < 64 && !attr_set[dev]) {
        ZKB_CUDA(cudaFuncSetAttribute(expr_kernel<NREGS, THREADS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        attr_set[dev] = true;
    }
    expr_kernel<NREGS, THREADS, true><<<(n + THREADS - 1) / THREADS, THREADS, bytes, st>>>(L);
    return ZKB_OK;
}

// d_code / d_cols / d_consts / d_outs are device pointers
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
    if (nregs <= 8) ZKB_TRY((launch_smem<8, 128>(L, n, st)));
    else if (nregs <= 16) ZKB_TRY((launch_smem<16, 128>(L, n, st)));
    else expr_kernel<64, 128, false><<<blocks, 128, 0, st>>>(L);
    ctx->launches++;
    ZKB_CUDA(cudaGetLastError());
    return ZKB_OK;
}

}  // namespace zkb
