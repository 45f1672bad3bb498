// csf.cuh -- the constraint system as it crosses the C ABI (the "CSF" blob, layout in include/zkb200.h) and its translation into
// interpreter expressions: parse and validate, the column slots of the interpreter's tables, gate / lookup / permutation terms.
// Host code, shared by the prover (prover.cu), the lookup compression (lookup.cu) and the witness check (check.cu).
#pragma once
#include <string.h>
#include <algorithm>
#include "common.cuh"
#include "expr.cuh"

namespace zkb {

enum { N_CONST = 0, N_FIXED = 1, N_ADVICE = 2, N_INSTANCE = 3, N_CHALLENGE = 4, N_NEG = 5, N_ADD = 6, N_MUL = 7, N_SCALED = 8 };
constexpr uint32_t CSF_MAGIC = 0x3146535au;

struct CsfLookup {
    std::vector<std::vector<uint32_t>> inputs;
    std::vector<uint32_t> table;
};
struct Csf {
    uint32_t k = 0, nf = 0, na = 0, ni = 0, nch = 0, bf = 0, d = 0, nphases = 0;
    std::vector<uint32_t> adv_phase, ch_phase;
    std::vector<std::array<uint32_t, 3>> nodes;
    std::vector<Fr> consts;
    std::vector<uint32_t> gates;
    std::vector<CsfLookup> lookups;
    std::vector<std::array<uint32_t, 2>> perm;
    std::vector<std::array<int32_t, 2>> advq, fixq, instq;
};

inline bool parse_csf(const uint32_t *w, uint64_t nw, Csf &c) {
    if (nw < 18 || w[0] != CSF_MAGIC) { set_error("CSF: bad magic / too short"); return false; }
    c.k = w[1]; c.nf = w[2]; c.na = w[3]; c.ni = w[4]; c.nch = w[5]; c.bf = w[6]; c.d = w[7]; c.nphases = w[8];
    const uint32_t n_nodes = w[9], n_consts = w[10], n_gates = w[11], n_lookups = w[12], n_perm = w[13], n_aq = w[14], n_fq = w[15], n_iq = w[16];
    uint64_t p = 18;
    auto need = [&](uint64_t cnt) { return p + cnt <= nw; };
    if (!need(c.na + c.nch)) { set_error("CSF: truncated"); return false; }
    c.adv_phase.assign(w + p, w + p + c.na); p += c.na;
    c.ch_phase.assign(w + p, w + p + c.nch); p += c.nch;
    if (!need(3ull * n_nodes)) { set_error("CSF: truncated nodes"); return false; }
    c.nodes.resize(n_nodes);
    for (uint32_t i = 0; i < n_nodes; ++i) { c.nodes[i] = {w[p], w[p + 1], w[p + 2]}; p += 3; }
    if (!need(8ull * n_consts)) { set_error("CSF: truncated consts"); return false; }
    c.consts.resize(n_consts);
    for (uint32_t i = 0; i < n_consts; ++i) { memcpy(c.consts[i].l, w + p, 32); p += 8; }
    if (!need(n_gates)) { set_error("CSF: truncated gates"); return false; }
    c.gates.assign(w + p, w + p + n_gates); p += n_gates;
    c.lookups.resize(n_lookups);
    for (uint32_t l = 0; l < n_lookups; ++l) {
        if (!need(2)) { set_error("CSF: truncated lookups"); return false; }
        const uint32_t nsets = w[p], width = w[p + 1];
        p += 2;
        if (nsets == 0 || width == 0 || nsets > 4096 || width > 4096) { set_error("CSF: lookup %u has an implausible shape (%u input sets x %u)", l, nsets, width); return false; }
        if (!need(((uint64_t)nsets + 1) * (uint64_t)width)) { set_error("CSF: truncated lookup body"); return false; }
        c.lookups[l].inputs.resize(nsets);
        for (uint32_t s = 0; s < nsets; ++s) { c.lookups[l].inputs[s].assign(w + p, w + p + width); p += width; }
        c.lookups[l].table.assign(w + p, w + p + width); p += width;
    }
    if (!need(2ull * (n_perm + n_aq + n_fq + n_iq))) { set_error("CSF: truncated tail"); return false; }
    c.perm.resize(n_perm);
    for (uint32_t i = 0; i < n_perm; ++i) { c.perm[i] = {w[p], w[p + 1]}; p += 2; }
    auto rdq = [&](std::vector<std::array<int32_t, 2>> &q, uint32_t cnt) {
        q.resize(cnt);
        for (uint32_t i = 0; i < cnt; ++i) { q[i] = {(int32_t)w[p], (int32_t)w[p + 1]}; p += 2; }
    };
    rdq(c.advq, n_aq); rdq(c.fixq, n_fq); rdq(c.instq, n_iq);
    for (auto &nd : c.nodes) {
        if (nd[0] > N_SCALED) { set_error("CSF: bad node op"); return false; }
    }
    if (c.k < 1 || c.k > 26 || c.d < 3 || c.bf < 5) { set_error("CSF: bad k / degree / blinding factors"); return false; }
    return true;
}

// parse a CSF blob and check it: node references point backwards, every column / challenge / constant index is in range
inline int32_t load_csf(const uint32_t *csf, uint64_t csf_words, Csf &c) {
    ZKB_ARG(csf != nullptr);
    if (!parse_csf(csf, csf_words, c)) return ZKB_ERR_ARG;
    for (size_t i = 0; i < c.nodes.size(); ++i) {
        const auto &nd = c.nodes[i];
        bool ok = true;
        switch (nd[0]) {
        case N_CONST: ok = nd[1] < c.consts.size(); break;
        case N_FIXED: ok = nd[1] < c.nf; break;
        case N_ADVICE: ok = nd[1] < c.na; break;
        case N_INSTANCE: ok = nd[1] < c.ni; break;
        case N_CHALLENGE: ok = nd[1] < c.nch; break;
        case N_NEG: ok = nd[1] < i; break;
        case N_ADD: case N_MUL: ok = nd[1] < i && nd[2] < i; break;
        case N_SCALED: ok = nd[1] < i && nd[2] < c.consts.size(); break;
        }
        if (!ok) { set_error("CSF: node %zu has an out-of-range operand", i); return ZKB_ERR_ARG; }
    }
    auto in_nodes = [&](uint32_t v) { return v < c.nodes.size(); };
    for (auto g : c.gates) if (!in_nodes(g)) { set_error("CSF: gate references a missing node"); return ZKB_ERR_ARG; }
    for (auto &lk : c.lookups) {
        if (lk.inputs.empty() || lk.table.empty()) { set_error("CSF: empty lookup"); return ZKB_ERR_ARG; }
        for (auto &inp : lk.inputs) for (auto v : inp) if (!in_nodes(v)) { set_error("CSF: lookup references a missing node"); return ZKB_ERR_ARG; }
        for (auto v : lk.table) if (!in_nodes(v)) { set_error("CSF: lookup references a missing node"); return ZKB_ERR_ARG; }
    }
    for (auto &pc : c.perm) {
        const uint32_t lim = pc[0] == N_FIXED ? c.nf : pc[0] == N_ADVICE ? c.na : pc[0] == N_INSTANCE ? c.ni : 0;
        if (pc[1] >= lim) { set_error("CSF: permutation column out of range"); return ZKB_ERR_ARG; }
    }
    // queries: column in range, rotation representable in the interpreter's 16-bit field (also for expression nodes)
    auto chkq = [&](const std::vector<std::array<int32_t, 2>> &q, uint32_t lim, const char *what) {
        for (auto &e : q) {
            if (e[0] < 0 || (uint32_t)e[0] >= lim) { set_error("CSF: %s query references column %d of %u", what, e[0], lim); return false; }
            if (e[1] < -32767 || e[1] > 32767) { set_error("CSF: %s query rotation %d does not fit 16 bits", what, e[1]); return false; }
        }
        return true;
    };
    if (!chkq(c.advq, c.na, "advice") || !chkq(c.fixq, c.nf, "fixed") || !chkq(c.instq, c.ni, "instance")) return ZKB_ERR_ARG;
    for (auto &nd : c.nodes) {
        if (nd[0] == N_FIXED || nd[0] == N_ADVICE || nd[0] == N_INSTANCE) {
            const int32_t rot = (int32_t)nd[2];
            if (rot < -32767 || rot > 32767) { set_error("CSF: node rotation %d does not fit 16 bits", rot); return ZKB_ERR_ARG; }
        }
    }
    if ((uint64_t)c.nf + c.na + c.ni + c.perm.size() + 1 >= 65536) { set_error("CSF: more than 65535 column slots"); return ZKB_ERR_ARG; }
    for (uint32_t ph : c.adv_phase) if (ph >= c.nphases) { set_error("CSF: advice phase out of range"); return ZKB_ERR_ARG; }
    for (uint32_t ph : c.ch_phase) if (ph >= c.nphases) { set_error("CSF: challenge phase out of range"); return ZKB_ERR_ARG; }
    return ZKB_OK;
}

// SHPLONK opens a column at the points x w^r of its distinct rotations mod n, and the prover takes at most MAX_POINTS_PER_COLUMN
// of them (shplonk() in prover.cu); instance columns are not opened.  The point sets are static in the CSF, so zkb_csf_validate
// and every pk constructor refuse a constraint system past the limit before any proof work.
constexpr size_t MAX_POINTS_PER_COLUMN = 256;
inline int32_t check_openings(const Csf &c) {
    const int64_t n = 1ll << c.k;
    auto chk = [&](const std::vector<std::array<int32_t, 2>> &q, uint32_t ncols, const char *what) {
        std::vector<std::vector<int64_t>> pts(ncols);
        for (auto &e : q) pts[e[0]].push_back(((e[1] % n) + n) % n);
        for (uint32_t col = 0; col < ncols; ++col) {
            std::sort(pts[col].begin(), pts[col].end());
            const size_t m = std::unique(pts[col].begin(), pts[col].end()) - pts[col].begin();
            if (m > MAX_POINTS_PER_COLUMN) {
                set_error("CSF: %s column %u is opened at %zu points (distinct rotations mod n), more than the %zu SHPLONK takes per column",
                          what, col, m, MAX_POINTS_PER_COLUMN);
                return false;
            }
        }
        return true;
    };
    return chk(c.advq, c.na, "advice") && chk(c.fixq, c.nf, "fixed") ? ZKB_OK : ZKB_ERR_ARG;
}

// the caller's `nch` challenge values (4 limbs each, Montgomery form)
inline std::vector<Fr> host_challenges(const uint64_t *limbs, uint32_t nch) {
    std::vector<Fr> ch(nch);
    for (uint32_t i = 0; i < nch; ++i) memcpy(ch[i].l, limbs + 4 * i, sizeof(Fr));
    return ch;
}

// The column slots of the interpreter's tables, in the one order every table uses:
//   [fixed | advice | instance | sigma | X | l_0 | l_last | l_blind | z | phi | m]
// The callers of the interpreter entry points pass the prefix [fixed | advice | instance].  A proof's value-domain table (lookup
// compression, permutation products) is the prefix up to X, with X = omega^i; its quotient table is all of it on a coset part, with
// X = the identity polynomial.  Fixed, sigma, X, l_0, l_last and l_blind do not depend on the proof: the pk caches their coset values.
struct SlotMap {
    uint32_t fixed0 = 0, advice0 = 0, instance0 = 0, sigma0 = 0, x = 0, l0 = 0, l_last = 0, l_blind = 0, z0 = 0, phi0 = 0, m0 = 0, slots = 0;
    SlotMap() = default;
    SlotMap(const Csf &cs, uint32_t nsets)
        : advice0(cs.nf), instance0(advice0 + cs.na), sigma0(instance0 + cs.ni), x(sigma0 + (uint32_t)cs.perm.size()), l0(x + 1), l_last(x + 2),
          l_blind(x + 3), z0(x + 4), phi0(z0 + nsets), m0(phi0 + (uint32_t)cs.lookups.size()), slots(m0 + (uint32_t)cs.lookups.size()) {}
    // slot of a permutation column (kind, index)
    uint32_t perm(const std::array<uint32_t, 2> &c) const { return c[0] == N_FIXED ? fixed0 + c[1] : c[0] == N_ADVICE ? advice0 + c[1] : instance0 + c[1]; }
};
// t[first + i] = cols[i]
inline void put_columns(std::vector<Fr *> &t, uint32_t first, const std::vector<Fr *> &cols) { std::copy(cols.begin(), cols.end(), t.begin() + first); }

// translate CSF nodes into ExprBuilder nodes
inline uint32_t translate(const Csf &cs, uint32_t node, ExprBuilder &eb, const SlotMap &sm, const std::vector<Fr> &challenges, std::vector<int64_t> &memo) {
    if (memo[node] >= 0) return (uint32_t)memo[node];
    const auto &nd = cs.nodes[node];
    uint32_t r = 0;
    switch (nd[0]) {
    case N_CONST: r = eb.constant(cs.consts[nd[1]]); break;
    case N_FIXED: r = eb.col(sm.fixed0 + nd[1], (int32_t)nd[2]); break;
    case N_ADVICE: r = eb.col(sm.advice0 + nd[1], (int32_t)nd[2]); break;
    case N_INSTANCE: r = eb.col(sm.instance0 + nd[1], (int32_t)nd[2]); break;
    case N_CHALLENGE: r = eb.constant(challenges[nd[1]]); break;
    case N_NEG: r = eb.neg(translate(cs, nd[1], eb, sm, challenges, memo)); break;
    case N_ADD: { uint32_t a = translate(cs, nd[1], eb, sm, challenges, memo), b = translate(cs, nd[2], eb, sm, challenges, memo); r = eb.add(a, b); } break;
    case N_MUL: { uint32_t a = translate(cs, nd[1], eb, sm, challenges, memo), b = translate(cs, nd[2], eb, sm, challenges, memo); r = eb.mul(a, b); } break;
    case N_SCALED: { uint32_t a = translate(cs, nd[1], eb, sm, challenges, memo); r = eb.mul(a, eb.constant(cs.consts[nd[2]])); } break;
    }
    memo[node] = r;
    return r;
}
// compressed = fold(exprs, acc * theta + e), first term taken as is (0 * theta + e0 == e0)
inline uint32_t compress_exprs(const Csf &cs, const std::vector<uint32_t> &exprs, ExprBuilder &eb, const SlotMap &sm, const std::vector<Fr> &ch,
                               std::vector<int64_t> &memo, const Fr &theta) {
    uint32_t acc = translate(cs, exprs[0], eb, sm, ch, memo);
    for (size_t i = 1; i < exprs.size(); ++i) acc = eb.add(eb.mul(acc, eb.constant(theta)), translate(cs, exprs[i], eb, sm, ch, memo));
    return acc;
}

// the permutation argument's DELTA = 7^(2^28): column i of a permutation set is labelled by DELTA^i
inline Fr perm_delta() {
    Fr d = fp_from_u64<FrParams>(7);
    for (int i = 0; i < 28; ++i) d = fp_sqr(d);
    return d;
}
constexpr uint32_t NO_NODE = 0xffffffffu;
// permutation/prover.rs: the factors of set si over its columns j, multiplied left to right onto num (v_j + beta delta^j X + gamma) and
// den (v_j + beta sigma_j + gamma); a product given as NO_NODE starts from its first factor.  X is slot sm.x in both domains.
inline void perm_set_products(const Csf &cs, const SlotMap &sm, uint32_t chunk, uint32_t si, const Fr &beta, const Fr &gamma, ExprBuilder &eb,
                              uint32_t &num, uint32_t &den) {
    const Fr delta = perm_delta();
    Fr delta_pow = fp_pow_u64(delta, (uint64_t)si * chunk);
    for (uint32_t j = si * chunk; j < std::min<size_t>((si + 1) * chunk, cs.perm.size()); ++j) {
        const uint32_t v = eb.col(sm.perm(cs.perm[j]), 0);
        const uint32_t dterm = eb.add(eb.add(v, eb.mul(eb.col(sm.sigma0 + j, 0), eb.constant(beta))), eb.constant(gamma));
        const uint32_t nterm = eb.add(eb.add(v, eb.mul(eb.col(sm.x, 0), eb.constant(fp_mul(beta, delta_pow)))), eb.constant(gamma));
        den = den == NO_NODE ? dterm : eb.mul(den, dterm);
        num = num == NO_NODE ? nterm : eb.mul(num, nterm);
        delta_pow = fp_mul(delta_pow, delta);
    }
}

}  // namespace zkb
