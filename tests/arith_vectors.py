"""Operand sets and exact references for the primitives of csrc/ff.cuh and csrc/g1.cuh as zkb_arith_probe_dev /
zkb_arith_probe_host apply them (op table: include/zkb200.h).

Every value is a stored integer: the 256-bit number in the limbs, Montgomery form for field elements (stored a means a / R).
The reference is Python integers, exact: each op's output is compared with the one integer the primitive must produce, not
only its residue, and every generated operand tuple is checked against the op's contract (`in_contract`), so a vector outside
what a primitive promises to handle can never pass or fail a test by accident.

Operand sets per field:
  boundary   0, 1, 2, p - 1, p - 2, (p -+ 1) / 2, R mod p, R^2 mod p, (R - 1) mod p, 2^k and 2^k - 1 for k in {32, 64, 128, 192,
             224, 253}, p - 2^k for k in {32, 64, 128, 192}, and the 256 values whose 32-bit limbs are each 0 or 0xffffffff,
             reduced mod p
  lazy       the boundary set shifted by p (< 2p) and by p, 2p, 3p (< 4p), plus 2p - 1 and 4p - 1
  long runs  random values made of long runs of ones and zeros (in the style of GMP's mpz_rrandomb)
  uniform    uniform random values
The unary and binary ops run the full Cartesian product of their edge sets; the 4-operand ops the product over
{0, 1, p - 1, p where allowed} plus random mixes.
"""
import itertools
import random

import numpy as np

import pyref as P

R = 1 << 256
MASK64 = (1 << 64) - 1
FIELDS = {0: P.R_MOD, 1: P.Q_MOD}

(ADD, SUB, NEG, DBL, MUL, SQR, MUL_ADD_MUL, MUL_SUB_MUL, MUL_LAZY, ADD_LAZY, SUB_LAZY, COND_SUB_P, COND_SUB_2P, POW, POW_U64, INV,
 FROM_CANONICAL, TO_CANONICAL, FROM_U64) = range(19)
G1_ADD_MIXED, G1_ADD, G1_DBL, G1_DBL_AFFINE, G1_TO_AFFINE, G1_NEG, G1_FROM_AFFINE = range(32, 39)
FIELD_OPS = list(range(19))
G1_OPS = list(range(32, 39))
DEVICE_ONLY = (MUL_LAZY, ADD_LAZY, SUB_LAZY, COND_SUB_P, COND_SUB_2P)
OP_NAMES = {ADD: "add", SUB: "sub", NEG: "neg", DBL: "dbl", MUL: "mul", SQR: "sqr", MUL_ADD_MUL: "mul_add_mul", MUL_SUB_MUL: "mul_sub_mul",
            MUL_LAZY: "mul_lazy", ADD_LAZY: "add_lazy", SUB_LAZY: "sub_lazy", COND_SUB_P: "cond_sub_p", COND_SUB_2P: "cond_sub_2p",
            POW: "pow", POW_U64: "pow_u64", INV: "inv", FROM_CANONICAL: "from_canonical", TO_CANONICAL: "to_canonical",
            FROM_U64: "from_u64", G1_ADD_MIXED: "g1_add_mixed", G1_ADD: "g1_add", G1_DBL: "g1_dbl", G1_DBL_AFFINE: "g1_dbl_affine",
            G1_TO_AFFINE: "g1_to_affine", G1_NEG: "g1_neg", G1_FROM_AFFINE: "g1_from_affine"}

N_RANDOM = 2000  # long-run and uniform tuples per op, each


def _dedup(vals):
    return list(dict.fromkeys(vals))


def boundary(p):
    v = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, R % p, R * R % p, (R - 1) % p]
    for k in (32, 64, 128, 192, 224, 253):
        v += [1 << k, (1 << k) - 1]
    v += [p - (1 << k) for k in (32, 64, 128, 192)]
    v += [sum(0xFFFFFFFF << (32 * i) for i in range(8) if (m >> i) & 1) % p for m in range(256)]
    assert all(0 <= x < p for x in v)
    return _dedup(v)


def exponents(p):
    """fp_pow exponents: the small and large edges of the boundary set and the integers past p, up to 2^256 - 1 (bit 255 set)"""
    v = [0, 1, 2, 3, p - 2, p - 1, (p - 1) // 2, (p + 1) // 2, p, p + 1, 2 * p, 4 * p - 1, R - p, 1 << 254, (1 << 255) - 1, 1 << 255,
         (1 << 255) + 1, R - 2, R - 1]
    for k in (32, 64, 128, 192, 224, 253):
        v += [1 << k, (1 << k) - 1]
    return _dedup(v)


def limb_masks():
    """the 256 integers whose 32-bit limbs are each 0 or 0xffffffff, unreduced"""
    return [sum(0xFFFFFFFF << (32 * i) for i in range(8) if (m >> i) & 1) for m in range(256)]


def u64_edges(p):
    v = [0, 1, 2, 3, (1 << 31), (1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, MASK64 - 1, MASK64,
         p & MASK64, (p - 1) & MASK64, (R % p) & MASK64, 0xFFFFFFFF00000000, 0x00000000FFFFFFFF]
    return _dedup(v)


def long_run(rnd, bound):
    """a value < bound made of runs of ones and zeros of random length (1 .. 64 bits)"""
    bits = bound.bit_length()
    while True:
        x, pos = 0, 0
        while pos < bits:
            run = rnd.randint(1, 64)
            if rnd.random() < 0.5:
                x |= ((1 << run) - 1) << pos
            pos += run
        x &= (1 << bits) - 1
        if x < bound:
            return x


class Domains:
    def __init__(self, field):
        p = self.p = FIELDS[field]
        self.canon = boundary(p)
        self.lazy2 = _dedup(self.canon + [v + p for v in self.canon] + [2 * p - 1])
        self.lazy4 = _dedup([v + k * p for k in range(4) for v in self.canon] + [2 * p - 1, 4 * p - 1])
        self.exp = exponents(p)
        self.u64 = u64_edges(p)
        self.small = [0, 1, p - 1]           # the 4-operand ops' product set; with p where the contract allows it
        self.small_p = [0, 1, p - 1, p]
        self.canon_p = self.canon + [p]


def spec(field, op):
    """-> (Cartesian products: list of per-operand value lists, random draws: list of per-operand exclusive bounds, mixes: per-operand
    value lists drawn from at random, or None)"""
    d = Domains(field)
    p = d.p
    c, c2 = d.canon, d.lazy2
    if op in (ADD, SUB, MUL):
        return [(c, c)], [(p, p)], None
    if op in (NEG, DBL, SQR, INV, FROM_CANONICAL, TO_CANONICAL):
        return [(c,)], [(p,)], None
    if op == MUL_ADD_MUL:
        return [(d.small_p, d.small, d.small_p, d.small)], [(p + 1, p, p + 1, p)], (d.canon_p, c, d.canon_p, c)
    if op == MUL_SUB_MUL:
        return [(d.small_p, d.small, d.small, d.small)], [(p + 1, p, p, p)], (d.canon_p, c, c, c)
    if op == MUL_LAZY:
        return [(d.lazy4, c), (c2, c2)], [(4 * p, p), (2 * p, 2 * p)], None
    if op in (ADD_LAZY, SUB_LAZY):
        return [(c2, c2)], [(2 * p, 2 * p)], None
    if op == COND_SUB_P:
        return [(c2,)], [(2 * p,)], None
    if op == COND_SUB_2P:
        return [(d.lazy4,)], [(4 * p,)], None
    if op == POW:
        return [(c, d.exp), ([0, 1, 2, p - 1, R % p], limb_masks())], [(p, R)], (c, c + d.exp + limb_masks())
    if op == POW_U64:
        return [(c, d.u64)], [(p, 1 << 64)], None
    if op == FROM_U64:
        return [(d.u64,)], [(1 << 64,)], None
    raise ValueError(op)


def field_cases(field, op, seed=0):
    """every operand tuple of (field, op): the edge products, random mixes of the edge sets, long-run and uniform draws"""
    products, bounds, mixes = spec(field, op)
    rnd = random.Random(1000 * seed + 100 * field + op)
    cases = []
    for prod in products:
        cases += list(itertools.product(*prod))
    if mixes is not None:
        cases += [tuple(rnd.choice(m) for m in mixes) for _ in range(4 * N_RANDOM)]
    for b in bounds:
        cases += [tuple(long_run(rnd, x) for x in b) for _ in range(N_RANDOM)]
        cases += [tuple(rnd.randrange(x) for x in b) for _ in range(N_RANDOM)]
    return cases


def in_contract(field, op, x):
    """the operand contract of include/zkb200.h's op table (stored integers)"""
    p = FIELDS[field]
    if op in (ADD, SUB, MUL, NEG, DBL, SQR, INV, FROM_CANONICAL, TO_CANONICAL):
        return all(0 <= v < p for v in x)
    if op == MUL_ADD_MUL:
        a, b, c, d = x
        return 0 <= a <= p and 0 <= c <= p and 0 <= b < p and 0 <= d < p
    if op == MUL_SUB_MUL:
        a, b, c, d = x
        return 0 <= a <= p and 0 <= b < p and 0 <= c < p and 0 <= d < p
    if op == MUL_LAZY:
        a, b = x
        return (0 <= a < 4 * p and 0 <= b < p) or (0 <= a < 2 * p and 0 <= b < 2 * p)
    if op in (ADD_LAZY, SUB_LAZY, COND_SUB_P):
        return all(0 <= v < 2 * p for v in x)
    if op == COND_SUB_2P:
        return 0 <= x[0] < 4 * p
    if op == POW:
        return 0 <= x[0] < p and 0 <= x[1] < R
    if op == POW_U64:
        return 0 <= x[0] < p and 0 <= x[1] <= MASK64
    if op == FROM_U64:
        return 0 <= x[0] <= MASK64
    raise ValueError(op)


def out_range(field, op):
    """(lo, hi): every output of op lies in [lo, hi)"""
    p = FIELDS[field]
    if op in (MUL_LAZY, ADD_LAZY, COND_SUB_2P):
        return 0, 2 * p
    if op == SUB_LAZY:
        return 1, 4 * p
    return 0, p


_RINV = {f: pow(R, -1, p) for f, p in FIELDS.items()}              # R^-1 mod p
_MINV = {f: -pow(p, -1, R) % R for f, p in FIELDS.items()}          # -p^-1 mod R (the REDC multiplier)


def expected(field, op, x):
    """the exact stored integer op must return for operands x"""
    p, ri = FIELDS[field], _RINV[field]
    if op == ADD: return (x[0] + x[1]) % p
    if op == SUB: return (x[0] - x[1]) % p
    if op == NEG: return -x[0] % p
    if op == DBL: return 2 * x[0] % p
    if op == MUL: return x[0] * x[1] * ri % p
    if op == SQR: return x[0] * x[0] * ri % p
    if op == MUL_ADD_MUL: return (x[0] * x[1] + x[2] * x[3]) * ri % p
    if op == MUL_SUB_MUL: return (x[0] * x[1] - x[2] * x[3]) * ri % p
    if op == MUL_LAZY:
        t = x[0] * x[1]
        return (t + (t * _MINV[field] % R) * p) >> 256
    if op == ADD_LAZY:
        s = x[0] + x[1]
        return s - 2 * p if s >= 2 * p else s
    if op == SUB_LAZY: return x[0] - x[1] + 2 * p
    if op == COND_SUB_P: return x[0] - p if x[0] >= p else x[0]
    if op == COND_SUB_2P: return x[0] - 2 * p if x[0] >= 2 * p else x[0]
    if op in (POW, POW_U64): return pow(x[0] * ri % p, x[1], p) * R % p
    if op == INV: return pow(x[0], -1, p) * R * R % p if x[0] else 0
    if op == FROM_CANONICAL: return x[0] * R % p
    if op == TO_CANONICAL: return x[0] * ri % p
    if op == FROM_U64: return x[0] * R % p
    raise ValueError(op)


# ---- packing ----------------------------------------------------------------------------------------------------------------
def pack(tuples, arity):
    """tuples of 256-bit ints -> numpy uint64 (n, 4 * arity), 4 little-endian limbs per value"""
    buf = b"".join(v.to_bytes(32, "little") for t in tuples for v in t)
    return np.frombuffer(buf, dtype=np.uint64).reshape(len(tuples), 4 * arity).copy()


def unpack(arr):
    """numpy uint64 (n, 4 * width) -> list of n tuples of width ints"""
    arr = np.ascontiguousarray(arr, dtype=np.uint64)
    b = arr.tobytes()
    width = arr.shape[1] // 4
    vals = [int.from_bytes(b[32 * i:32 * i + 32], "little") for i in range(arr.size // 4)]
    return [tuple(vals[r * width:(r + 1) * width]) for r in range(arr.shape[0])]


def field_mismatches(field, op, cases, outs, limit=5):
    """(number of wrong outputs, first few as readable strings): exact value and output range"""
    lo, hi = out_range(field, op)
    bad, shown = 0, []
    for x, (y,) in zip(cases, outs):
        e = expected(field, op, x)
        assert lo <= e < hi, "reference outside the op's range"
        if y != e or not lo <= y < hi:
            bad += 1
            if len(shown) < limit:
                shown.append(f"{OP_NAMES[op]}({', '.join(hex(v) for v in x)}) = {y:#x}, expected {e:#x}")
    return bad, shown


# ---- G1 ---------------------------------------------------------------------------------------------------------------------
Q = P.Q_MOD
Q_RINV = pow(R, -1, Q)


def fq_m(v):
    return v * R % Q


def fq_plain(v):
    return v * Q_RINV % Q


def g1_points(seed=0):
    """O (None), P, -P, 2P and generic points Q1, Q2 (pyref affine tuples), with their names"""
    rnd = random.Random(7000 + seed)
    g = P.G1_GEN
    p1 = P.g1_mul(g, rnd.randrange(2, P.R_MOD))
    pts = {"O": None, "P": p1, "-P": P.g1_neg(p1), "2P": P.g1_add(p1, p1),
           "Q1": P.g1_mul(g, rnd.randrange(2, P.R_MOD)), "Q2": P.g1_mul(g, rnd.randrange(2, P.R_MOD))}
    assert all(P.g1_is_on_curve(v) for v in pts.values())
    return pts


def xyzz_forms(pt, rnd, n_random=2):
    """(lambda name, plain (X, Y, ZZ, ZZZ)) = (l^2 x, l^3 y, l^2, l^3) for l = 1, -1 and random l; the identity is all zeros"""
    if pt is None:
        return [("0", (0, 0, 0, 0))]
    x, y = pt
    lams = [("1", 1), ("-1", Q - 1)] + [(f"r{i}", rnd.randrange(2, Q - 1)) for i in range(n_random)]
    return [(n, (l * l * x % Q, l ** 3 * y % Q, l * l % Q, l ** 3 % Q)) for n, l in lams]


def affine_plain(pt):
    return (0, 0) if pt is None else pt


def g1_cases(op, seed=0):
    """-> list of (label, operand tuple of stored Fq values, expected pyref point or exact stored tuple)"""
    rnd = random.Random(7100 + seed)
    pts = g1_points(seed)
    forms = {name: xyzz_forms(pt, rnd) for name, pt in pts.items()}
    mont = lambda t: tuple(fq_m(v) for v in t)
    cases = []
    if op == G1_ADD:
        for (na, a), (nb, b) in itertools.product(pts.items(), repeat=2):
            for (la, fa), (lb, fb) in itertools.product(forms[na], forms[nb]):
                cases.append((f"{na}[{la}] + {nb}[{lb}]", mont(fa) + mont(fb), P.g1_add(a, b)))
    elif op == G1_ADD_MIXED:
        for (na, a), (nb, b) in itertools.product(pts.items(), repeat=2):
            for la, fa in forms[na]:
                cases.append((f"{na}[{la}] + {nb}", mont(fa) + mont(affine_plain(b)), P.g1_add(a, b)))
    elif op == G1_DBL:
        for na, a in pts.items():
            for la, fa in forms[na]:
                cases.append((f"2 {na}[{la}]", mont(fa), P.g1_add(a, a)))
    elif op == G1_DBL_AFFINE:
        for na, a in pts.items():
            cases.append((f"2 {na}", mont(affine_plain(a)), P.g1_add(a, a)))
    elif op == G1_TO_AFFINE:
        for na, a in pts.items():
            for la, fa in forms[na]:
                cases.append((f"affine {na}[{la}]", mont(fa), mont(affine_plain(a))))
    elif op == G1_NEG:
        for na, a in pts.items():
            cases.append((f"-{na}", mont(affine_plain(a)), mont(affine_plain(P.g1_neg(a)))))
    elif op == G1_FROM_AFFINE:
        for na, a in pts.items():
            cases.append((f"xyzz {na}", mont(affine_plain(a)), (0, 0, 0, 0) if a is None else mont(a) + (R % Q, R % Q)))
    else:
        raise ValueError(op)
    return cases


G1_XYZZ_OUT = (G1_ADD_MIXED, G1_ADD, G1_DBL, G1_DBL_AFFINE)


def g1_mismatches(op, cases, outs, limit=5):
    """XYZZ results: every coordinate < q, ZZ^3 = ZZZ^2, identity exactly when ZZ = 0, and (X / ZZ, Y / ZZZ) equal to pyref's
    point; exact tuples otherwise"""
    bad, shown = 0, []
    for (label, _, want), got in zip(cases, outs):
        why = None
        if any(v >= Q for v in got):
            why = "coordinate not < q"
        elif op in G1_XYZZ_OUT:
            x, y, zz, zzz = (fq_plain(v) for v in got)
            if pow(zz, 3, Q) != zzz * zzz % Q:
                why = "ZZ^3 != ZZZ^2"
            elif (zz == 0) != (want is None):
                why = "identity flag"
            elif want is not None and (x * pow(zz, -1, Q) % Q, y * pow(zzz, -1, Q) % Q) != want:
                why = "normalises to a different point"
        elif tuple(got) != want:
            why = "not the exact result"
        if why:
            bad += 1
            if len(shown) < limit:
                shown.append(f"{OP_NAMES[op]} {label}: {why}: got {[hex(v) for v in got]}")
    return bad, shown
