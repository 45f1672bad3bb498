// expr.cuh -- constraint-expression programs: host-side compiler (DAG -> linear register program) and the device
// interpreter that evaluates them row by row.
//
// Replaces halo2_proofs plonk/evaluation.rs (`GraphEvaluator`, `ValueSource`, `Calculation`, `Evaluator::evaluate_h`):
// upstream compiles every gate / lookup expression into a calculation graph and walks it per row on rayon threads.
// Here the whole quotient numerator -- custom gates, permutation argument terms and mv-lookup (logUp) terms, in
// upstream's Horner-in-y order -- is ONE program executed by ONE kernel: a thread owns a row, streams the column
// values it needs (rotations are index offsets inside the coset), keeps intermediates in a small register file and
// folds `acc = acc * y + term` after every constraint.  The same interpreter compresses lookup inputs / tables with
// theta on the Lagrange domain (mv_lookup/prover.rs `prepare`).
#pragma once
#include <stdint.h>
#include <algorithm>
#include <array>
#include <map>
#include <string>
#include <tuple>
#include <vector>
#include "common.cuh"

namespace zkb {

enum : uint8_t {
    OP_LOADCOL = 0,   // reg[dst] = cols[imm & 0xffff][(row + rot) mod n], rot = (int16)(imm >> 16)
    OP_LOADCONST = 1, // reg[dst] = consts[imm]
    OP_ADD = 2,
    OP_SUB = 3,
    OP_MUL = 4,
    OP_NEG = 5,
    OP_HORNER = 6,    // acc = acc * consts[imm] + reg[a]
    OP_STORE = 7,     // outs[imm][row] = reg[a]
    OP_STOREACC = 8,  // outs[imm][row] = acc * consts[b-as-index given in `a`]... see kernel: acc scaled by consts[a]
    OP_CLEARACC = 9,
    OP_HORNER2 = 10,  // acc2 = acc2 * consts[imm] + reg[a]            (inner Horner of a run of constraints sharing one factor)
    OP_FOLD = 11,     // acc = acc * consts[imm] + reg[a] * acc2; acc2 = 0
    OP_FLAG = 12,     // bit `row` of bitmap imm = (reg[a] != 0)     (flag build only: expr_flag_kernel, the witness check)
    OP_ARG = 13,      // not an instruction: the second 32-bit operand of the fused instruction before it
    // Fused operand forms (ProgramBuilder::fuse).  An operand is R = reg[a], C = a column at a rotation (encoded as OP_LOADCOL's
    // imm) or K = consts[index].  The first C / K operand is `imm`, a second one is the imm of the OP_ARG word that follows;
    // OP_ADD_RC + form, OP_SUB_RC + form, OP_MUL_RC + form compute  left op right  for the forms below, in that order.
    FORM_RC = 0, FORM_CR = 1, FORM_RK = 2, FORM_KR = 3, FORM_CC = 4, FORM_CK = 5, FORM_KC = 6,
    OP_ADD_RC = 16,
    OP_SUB_RC = 24,
    OP_MUL_RC = 32,
    OP_HORNER_C = 40,   // OP_HORNER / OP_HORNER2 / OP_FOLD with the term a column: consts[imm] as before, the column in OP_ARG
    OP_HORNER2_C = 41,
    OP_FOLD_C = 42,
    // Merged products (ProgramBuilder::merge_products): a register-register OP_MUL whose result is read once, by a HORNER / HORNER2
    // root, is evaluated inside the root as a sum of two products with one Montgomery reduction (fp_mul_add_mul).
    OP_HORNER_M = 43,   // acc = acc * consts[imm] + reg[a] * reg[b]
    OP_HORNER2_M = 44,  // acc2 = acc2 * consts[imm] + reg[a] * reg[b]
};

struct alignas(8) Instr {
    uint8_t op, dst, a, b;
    uint32_t imm;
};

constexpr int EXPR_MAX_REGS = 64;

// ---- host-side expression DAG with hash-consing --------------------------------------------------------------------
struct ENode {
    uint8_t kind;   // 0 col, 1 const, 2 add, 3 sub, 4 mul, 5 neg
    uint32_t a, b;  // children, or (slot, rot) for col, const index for const
};

class ExprBuilder {
public:
    std::vector<ENode> nodes;
    std::vector<Fr> consts;
    // degree of each node as a polynomial in the columns, set as the node is interned (children come first): a column 1 (X, l_0,
    // l_last and l_blind too, an upper bound), a constant 0, add / sub the larger operand's, mul the sum, neg its operand's
    std::vector<uint32_t> degree;

    uint32_t col(uint32_t slot, int32_t rot) { return intern(0, slot, (uint32_t)rot); }
    uint32_t constant(const Fr &v) {
        // constants are deduplicated by value
        std::array<uint32_t, 8> key;
        for (int i = 0; i < 8; ++i) key[i] = v.l[i];
        auto it = const_index.find(key);
        uint32_t idx;
        if (it == const_index.end()) {
            idx = (uint32_t)consts.size();
            consts.push_back(v);
            const_index.emplace(key, idx);
        } else idx = it->second;
        return intern(1, idx, 0);
    }
    uint32_t add(uint32_t x, uint32_t y) { return intern(2, x, y); }
    uint32_t sub(uint32_t x, uint32_t y) { return intern(3, x, y); }
    uint32_t mul(uint32_t x, uint32_t y) { return intern(4, x, y); }
    uint32_t neg(uint32_t x) { return intern(5, x, 0); }
    uint32_t const_slot(const Fr &v) {  // index into consts (for HORNER / STOREACC immediates)
        uint32_t n = constant(v);
        return nodes[n].a;
    }
    // set used[slot] for every column slot read under `root`; `seen` (one entry per node) carries the visited nodes across calls
    void columns(uint32_t root, std::vector<char> &seen, std::vector<char> &used) const {
        std::vector<uint32_t> stack{root};
        while (!stack.empty()) {
            const uint32_t v = stack.back();
            stack.pop_back();
            if (seen[v]) continue;
            seen[v] = 1;
            const ENode &e = nodes[v];
            if (e.kind == 0) used[e.a] = 1;
            else if (e.kind >= 2) {
                stack.push_back(e.a);
                if (e.kind != 5) stack.push_back(e.b);
            }
        }
    }

private:
    std::map<std::tuple<uint8_t, uint32_t, uint32_t>, uint32_t> index;
    std::map<std::array<uint32_t, 8>, uint32_t> const_index;
    uint32_t intern(uint8_t kind, uint32_t a, uint32_t b) {
        auto key = std::make_tuple(kind, a, b);
        auto it = index.find(key);
        if (it != index.end()) return it->second;
        nodes.push_back(ENode{kind, a, b});
        degree.push_back(kind == 0 ? 1 : kind == 1 ? 0 : kind == 4 ? degree[a] + degree[b] : kind == 5 ? degree[a] : std::max(degree[a], degree[b]));
        index.emplace(key, (uint32_t)nodes.size() - 1);
        return (uint32_t)nodes.size() - 1;
    }
};

// ---- program assembly: a sequence of "scopes"; inside a scope common subexpressions are computed once --------------
class ProgramBuilder {
public:
    explicit ProgramBuilder(ExprBuilder &eb) : eb(eb) {}
    std::vector<Instr> code;
    int max_regs_used = 0;
    std::string error;

    // evaluate `roots` (node ids) within one CSE scope and call emit_root(i, reg) after each is available
    enum RootAction { HORNER, STORE, HORNER2, FOLD, FLAG };
    struct Root { uint32_t node; RootAction action; uint32_t imm; };
    bool scope(const std::vector<Root> &roots);
    void clear_acc() { code.push_back(Instr{OP_CLEARACC, 0, 0, 0, 0}); }
    void store_acc(uint32_t out_slot, uint32_t scale_const_index) {
        code.push_back(Instr{OP_STOREACC, 0, 0, 0, out_slot | (scale_const_index << 8)});
    }

private:
    ExprBuilder &eb;
    void fuse(size_t begin);
    static void merge_products(std::vector<Instr> &code);
};

// Peephole pass over the code of one scope, code[begin..): an OP_LOADCOL / OP_LOADCONST whose register is read exactly once
// before it is written again, by an ADD / SUB / MUL or (a column only) by a HORNER / HORNER2 / FOLD root, becomes an operand of
// that reader, so the value goes from global memory straight into the field operation instead of through the register file.
// Operand order, and with it every result bit, is unchanged; registers are only dropped, so max_regs_used (which picks the
// kernel build) is the allocator's count as before.  Two constants into one instruction (no KK form): the right one stays a load.
inline void ProgramBuilder::fuse(size_t begin) {
    auto is_arith = [](uint8_t op) { return op == OP_ADD || op == OP_SUB || op == OP_MUL; };
    auto is_root = [](uint8_t op) { return op == OP_HORNER || op == OP_HORNER2 || op == OP_FOLD; };
    auto is_load = [](uint8_t op) { return op == OP_LOADCOL || op == OP_LOADCONST; };
    auto reads = [&](const Instr &in, int s) {   // does operand slot s (0: a, 1: b) of `in` read a register
        if (is_arith(in.op)) return true;
        return s == 0 && (in.op == OP_NEG || is_root(in.op) || in.op == OP_STORE || in.op == OP_FLAG);
    };
    auto writes = [&](const Instr &in) { return is_load(in.op) || is_arith(in.op) || in.op == OP_NEG; };
    const size_t end = code.size();
    std::vector<std::array<int64_t, 2>> src(end - begin, {-1, -1});   // the load feeding operand slot 0 / 1, or -1
    for (size_t i = begin; i < end; ++i) {
        if (!is_load(code[i].op)) continue;
        const uint8_t r = code[i].dst;
        int uses = 0, slot = -1;
        size_t user = 0;
        for (size_t j = i + 1; j < end && uses < 2; ++j) {
            for (int s = 0; s < 2; ++s)
                if (reads(code[j], s) && (s == 0 ? code[j].a : code[j].b) == r) { ++uses; user = j; slot = s; }
            if (writes(code[j]) && code[j].dst == r) break;
        }
        if (uses != 1) continue;
        const uint8_t op = code[user].op;
        if (is_arith(op) || (is_root(op) && code[i].op == OP_LOADCOL)) src[user - begin][slot] = (int64_t)i;
    }
    auto kind = [&](const std::array<int64_t, 2> &s, int k) { return s[k] < 0 ? 'R' : code[s[k]].op == OP_LOADCOL ? 'C' : 'K'; };
    std::vector<bool> fused(end - begin, false);
    for (auto &s : src) {
        if (kind(s, 0) == 'K' && kind(s, 1) == 'K') s[1] = -1;
        for (int k = 0; k < 2; ++k)
            if (s[k] >= 0) fused[s[k] - begin] = true;
    }
    std::vector<Instr> out;
    for (size_t i = begin; i < end; ++i) {
        const Instr in = code[i];
        const auto &s = src[i - begin];
        if (fused[i - begin]) continue;
        if (s[0] < 0 && s[1] < 0) { out.push_back(in); continue; }
        if (is_root(in.op)) {
            const uint8_t op = in.op == OP_HORNER ? OP_HORNER_C : in.op == OP_HORNER2 ? OP_HORNER2_C : OP_FOLD_C;
            out.push_back(Instr{op, 0, 0, 0, in.imm});
            out.push_back(Instr{OP_ARG, 0, 0, 0, code[s[0]].imm});
            continue;
        }
        const char ka = kind(s, 0), kb = kind(s, 1);
        const int form = ka == 'R' ? (kb == 'C' ? FORM_RC : FORM_RK)
                       : kb == 'R' ? (ka == 'C' ? FORM_CR : FORM_KR)
                       : ka == 'C' ? (kb == 'C' ? FORM_CC : FORM_CK) : FORM_KC;
        const uint8_t base = in.op == OP_ADD ? OP_ADD_RC : in.op == OP_SUB ? OP_SUB_RC : OP_MUL_RC;
        const int first = s[0] >= 0 ? 0 : 1;   // the first non-register operand goes to imm, a second one to OP_ARG
        const uint8_t reg = ka == 'R' ? in.a : in.b;
        out.push_back(Instr{(uint8_t)(base + form), in.dst, (uint8_t)(form < FORM_CC ? reg : 0), 0, code[s[first]].imm});
        if (form >= FORM_CC) out.push_back(Instr{OP_ARG, 0, 0, 0, code[s[1]].imm});
    }
    merge_products(out);
    code.resize(begin);
    code.insert(code.end(), out.begin(), out.end());
}

// Second peephole step, on the operand-fused code of one scope: a register-register OP_MUL whose register is read exactly once
// before it is written again, by a HORNER / HORNER2 root, and whose operand registers are not written before that read, moves
// into the root (OP_HORNER_M / OP_HORNER2_M): acc * y + a * b then costs one Montgomery reduction instead of two.  A product read
// twice, or read by anything else, stays an OP_MUL.  Operand order is kept and the result is the same canonical element;
// registers are only dropped, as in fuse.  (Sums of two products in ADD / SUB are not merged: their tail would keep four
// operands and both accumulators live and push the interpreter past its register budget.)
inline void ProgramBuilder::merge_products(std::vector<Instr> &code) {
    const size_t n = code.size();
    auto reg_reads = [](const Instr &in, int s) {   // does operand slot s (0: a, 1: b) of `in` read a register
        const uint8_t op = in.op;
        if (op == OP_ADD || op == OP_SUB || op == OP_MUL) return true;
        if (s != 0) return false;
        if (op == OP_NEG || op == OP_HORNER || op == OP_HORNER2 || op == OP_FOLD || op == OP_STORE || op == OP_FLAG) return true;
        return op >= OP_ADD_RC && op < OP_MUL_RC + 8 && (op & 7) < FORM_CC;
    };
    auto reg_writes = [](const Instr &in) {
        const uint8_t op = in.op;
        return op == OP_LOADCOL || op == OP_LOADCONST || op == OP_ADD || op == OP_SUB || op == OP_MUL || op == OP_NEG ||
               (op >= OP_ADD_RC && op < OP_MUL_RC + 8);
    };
    std::vector<int64_t> reader(n, -1);   // for a mergeable OP_MUL: the index of its one reader
    for (size_t i = 0; i < n; ++i) {
        const Instr &m = code[i];
        if (m.op != OP_MUL) continue;
        int uses = 0;
        size_t user = 0;
        for (size_t j = i + 1; j < n && uses < 2; ++j) {
            for (int s = 0; s < 2; ++s)
                if (reg_reads(code[j], s) && (s == 0 ? code[j].a : code[j].b) == m.dst) { ++uses; user = j; }
            if (reg_writes(code[j]) && code[j].dst == m.dst) break;
        }
        if (uses != 1) continue;
        bool intact = true;
        for (size_t j = i + 1; j < user; ++j)
            if (reg_writes(code[j]) && (code[j].dst == m.a || code[j].dst == m.b)) intact = false;
        if (intact) reader[i] = (int64_t)user;
    }
    std::vector<int64_t> prod(n, -1);   // the mergeable product read by each root
    for (size_t i = 0; i < n; ++i)
        if (reader[i] >= 0 && (code[reader[i]].op == OP_HORNER || code[reader[i]].op == OP_HORNER2)) prod[reader[i]] = (int64_t)i;
    std::vector<bool> merged(n, false);
    std::vector<Instr> out;
    for (size_t j = 0; j < n; ++j) {
        Instr in = code[j];
        if (prod[j] >= 0) {
            in = Instr{(uint8_t)(in.op == OP_HORNER ? OP_HORNER_M : OP_HORNER2_M), 0, code[prod[j]].a, code[prod[j]].b, in.imm};
            merged[prod[j]] = true;
        }
        out.push_back(in);
    }
    code.clear();
    for (size_t j = 0; j < n; ++j)
        if (!merged[j]) code.push_back(out[j]);
}

inline bool ProgramBuilder::scope(const std::vector<Root> &roots) {
    const size_t begin = code.size();
    // 1. reference counts inside the scope (number of parents + root uses)
    std::map<uint32_t, int> refs;
    std::vector<uint32_t> stack;
    std::map<uint32_t, bool> seen;
    for (auto &r : roots) {
        refs[r.node]++;
        if (!seen[r.node]) { seen[r.node] = true; stack.push_back(r.node); }
    }
    while (!stack.empty()) {
        uint32_t n = stack.back();
        stack.pop_back();
        const ENode &e = eb.nodes[n];
        if (e.kind >= 2) {
            uint32_t ch[2] = {e.a, e.b};
            int nch = e.kind == 5 ? 1 : 2;
            for (int i = 0; i < nch; ++i) {
                refs[ch[i]]++;
                if (!seen[ch[i]]) { seen[ch[i]] = true; stack.push_back(ch[i]); }
            }
        }
    }
    // 2. emit with a register pool; a node's register is released when its last use is consumed
    std::map<uint32_t, int> reg_of;
    std::vector<int> free_regs;
    for (int i = EXPR_MAX_REGS - 1; i >= 0; --i) free_regs.push_back(i);
    auto alloc = [&]() -> int {
        if (free_regs.empty()) return -1;
        int r = free_regs.back();
        free_regs.pop_back();
        if (r + 1 > max_regs_used) max_regs_used = r + 1;
        return r;
    };
    auto release_use = [&](uint32_t n) {
        if (--refs[n] == 0) {
            free_regs.push_back(reg_of[n]);
            reg_of.erase(n);
        }
    };
    // iterative post-order evaluation
    struct Frame { uint32_t node; int state; };
    for (auto &r : roots) {
        if (!reg_of.count(r.node)) {
            std::vector<Frame> st;
            st.push_back({r.node, 0});
            while (!st.empty()) {
                Frame &f = st.back();
                const ENode e = eb.nodes[f.node];
                if (reg_of.count(f.node)) { st.pop_back(); continue; }
                if (e.kind < 2) {
                    int rg = alloc();
                    if (rg < 0) { error = "expression needs more than 64 live registers"; return false; }
                    if (e.kind == 0) code.push_back(Instr{OP_LOADCOL, (uint8_t)rg, 0, 0, (e.a & 0xffffu) | ((uint32_t)(uint16_t)(int16_t)(int32_t)e.b << 16)});
                    else code.push_back(Instr{OP_LOADCONST, (uint8_t)rg, 0, 0, e.a});
                    reg_of[f.node] = rg;
                    st.pop_back();
                    continue;
                }
                const int nch = e.kind == 5 ? 1 : 2;
                if (f.state == 0) {
                    f.state = 1;
                    if (!reg_of.count(e.a)) { st.push_back({e.a, 0}); continue; }
                }
                if (f.state == 1) {
                    f.state = 2;
                    if (nch == 2 && !reg_of.count(e.b)) { st.push_back({e.b, 0}); continue; }
                }
                // children ready
                const int ra = reg_of[e.a];
                const int rb = nch == 2 ? reg_of[e.b] : 0;
                const uint32_t me = f.node;
                // consume child uses first so the destination may reuse a dying child's register
                release_use(e.a);
                if (nch == 2) release_use(e.b);
                int rg = alloc();
                if (rg < 0) { error = "expression needs more than 64 live registers"; return false; }
                uint8_t op = e.kind == 2 ? OP_ADD : e.kind == 3 ? OP_SUB : e.kind == 4 ? OP_MUL : OP_NEG;
                code.push_back(Instr{op, (uint8_t)rg, (uint8_t)ra, (uint8_t)rb, 0});
                reg_of[me] = rg;
                st.pop_back();
            }
        }
        const int rr = reg_of[r.node];
        if (r.action == HORNER) code.push_back(Instr{OP_HORNER, 0, (uint8_t)rr, 0, r.imm});
        else if (r.action == HORNER2) code.push_back(Instr{OP_HORNER2, 0, (uint8_t)rr, 0, r.imm});
        else if (r.action == FOLD) code.push_back(Instr{OP_FOLD, 0, (uint8_t)rr, 0, r.imm});
        else if (r.action == FLAG) code.push_back(Instr{OP_FLAG, 0, (uint8_t)rr, 0, r.imm});
        else code.push_back(Instr{OP_STORE, 0, (uint8_t)rr, 0, r.imm});
        release_use(r.node);
    }
    fuse(begin);
    return true;
}

// ---- running programs (expr.cu) ---------------------------------------------------------------------------------------
// d_code / d_cols / d_consts / d_outs are device pointers
int32_t expr_run_device(zkb_ctx *ctx, const Instr *d_code, uint32_t ncode, int nregs, const Fr *const *d_cols, const Fr *d_consts,
                        Fr *const *d_outs, uint32_t log_n, uint32_t out_stride, uint32_t out_offset, cudaStream_t st);
// the flag build over 2^log_n rows: FLAG(g) writes words [g * words, (g + 1) * words) of `bits` (device pointers as above); the
// register bands are those of expr_run_device
int32_t expr_flag_run_device(zkb_ctx *ctx, const Instr *d_code, uint32_t ncode, int nregs, const Fr *const *d_cols, const Fr *d_consts,
                             uint32_t *bits, uint32_t words, uint32_t log_n, cudaStream_t st);

// program bundle uploaded to the device
struct DeviceProgram {
    Instr *code = nullptr;
    uint32_t ncode = 0;
    int nregs = 0;
    Fr *consts = nullptr;
};
inline int32_t upload_program(DevPool &pool, const ProgramBuilder &pb, const ExprBuilder &eb, DeviceProgram &dp, cudaStream_t st) {
    dp.ncode = (uint32_t)pb.code.size();
    dp.nregs = pb.max_regs_used;
    ZKB_TRY(pool.alloc(pb.code.size() * sizeof(Instr) + 8, (void **)&dp.code));
    ZKB_TRY(pool.alloc(eb.consts.size() * sizeof(Fr) + 32, (void **)&dp.consts));
    ZKB_CUDA(cudaMemcpyAsync(dp.code, pb.code.data(), pb.code.size() * sizeof(Instr), cudaMemcpyHostToDevice, st));
    ZKB_CUDA(cudaMemcpyAsync(dp.consts, eb.consts.data(), eb.consts.size() * sizeof(Fr), cudaMemcpyHostToDevice, st));
    ZKB_CUDA(cudaStreamSynchronize(st));  // host vectors may die after return
    return ZKB_OK;
}
template <class T>
inline int32_t upload_table(DevPool &pool, const std::vector<T *> &host, T ***dev, cudaStream_t st) {
    ZKB_TRY(pool.alloc(host.size() * sizeof(T *) + 8, (void **)dev));
    ZKB_CUDA(cudaMemcpyAsync(*dev, host.data(), host.size() * sizeof(T *), cudaMemcpyHostToDevice, st));
    ZKB_CUDA(cudaStreamSynchronize(st));
    return ZKB_OK;
}
// one program whose root i is STOREd to outs[i], uploaded with its output table and run over the 2^log_n rows of the d_cols table
inline int32_t run_store_program(zkb_ctx *ctx, uint32_t log_n, DevPool &pool, ExprBuilder &eb, const std::vector<uint32_t> &roots,
                                 const std::vector<Fr *> &outs, const Fr *const *d_cols, const std::string &what, cudaStream_t st) {
    ProgramBuilder pb(eb);
    std::vector<ProgramBuilder::Root> stores;
    for (size_t i = 0; i < roots.size(); ++i) stores.push_back({roots[i], ProgramBuilder::STORE, (uint32_t)i});
    if (!pb.scope(stores)) { set_error("%s: %s", what.c_str(), pb.error.c_str()); return ZKB_ERR_ARG; }
    DeviceProgram dp;
    ZKB_TRY(upload_program(pool, pb, eb, dp, st));
    Fr **d_outs = nullptr;
    ZKB_TRY(upload_table(pool, outs, &d_outs, st));
    return expr_run_device(ctx, dp.code, dp.ncode, dp.nregs, d_cols, dp.consts, d_outs, log_n, 1, 0, st);
}

}  // namespace zkb
