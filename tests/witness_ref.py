"""CPU reference of the witness check (zkb_check_witness_dev), with exact tuple comparison and no theta, over the oracle's expression
evaluator (`Ref.eval_expr`).  Semantics, as in include/zkb200.h:
  gate g       g(row) != 0 on all n rows (rotation r reads (row + r) mod n); poisoned when one of the gate's advice queries reads a
               row >= usable at that row
  lookup l, j  the input tuple at a row < usable is not among the table tuples of the rows < usable
  copy i       v[lc][lr] != v[rc][rr], columns indexing cs.perm_columns
Returns the same counts (gates, then (lookup, set) pairs, then all copies) and the same ordered record list as the device."""
import numpy as np

import halo2_ref as H


def advice_rotations(e, out=None):
    out = set() if out is None else out
    if e.op == H.ADVICE: out.add(e.b)
    elif e.op in (H.NEG, H.SCALED): advice_rotations(e.a, out)
    elif e.op in (H.ADD, H.MUL): advice_rotations(e.a, out); advice_rotations(e.b, out)
    return out


def _tuples(ref, exprs, cols, challenges, n, rows):
    vals = [np.ascontiguousarray(ref.eval_expr(e, cols, challenges, n, 1)[:rows]) for e in exprs]
    return [b"".join(v[i].tobytes() for v in vals) for i in range(rows)]


def check_witness(ref, cs, cols, challenges, copies, usable):
    """cs: oracle ConstraintSystem; cols: {FIXED/ADVICE/INSTANCE: [(n, 4) Montgomery arrays]} (instance zero-padded); challenges: ints;
    copies: (lc, lr, rc, rr) entries.  -> (counts as uint64 array, [(kind, index, sub, row)])"""
    n = cs.n
    usable = max(0, usable)
    counts, records = [], []
    for g, e in enumerate(cs.gates):
        rows = np.nonzero(ref.eval_expr(e, cols, challenges, n, 1).any(axis=1))[0]
        rots = advice_rotations(e)
        counts.append(len(rows))
        records += [(0, g, int(any((int(r) + rot) % n >= usable for rot in rots)), int(r)) for r in rows]
    for l, lk in enumerate(cs.lookups):
        table = set(_tuples(ref, lk.table, cols, challenges, n, usable))
        for j, inp in enumerate(lk.inputs):
            bad = [r for r, t in enumerate(_tuples(ref, inp, cols, challenges, n, usable)) if t not in table]
            counts.append(len(bad))
            records += [(1, l, j, r) for r in bad]
    perm = [cols[t][i] for (t, i) in cs.perm_columns]
    bad = [i for i, (lc, lr, rc, rr) in enumerate(copies) if (perm[lc][lr] != perm[rc][rr]).any()]
    counts.append(len(bad))
    records += [(2, i, 0, int(copies[i][1])) for i in bad]
    return np.array(counts, dtype=np.uint64), records


def perm_copies(cs, copies):
    """((type, col, row), (type, col, row)) pairs of tests/circuits.py -> (lc, lr, rc, rr) over cs.perm_columns"""
    cidx = {c: i for i, c in enumerate(cs.perm_columns)}
    return [(cidx[(lt, lc)], lr, cidx[(rt, rc)], rr) for (lt, lc, lr), (rt, rc, rr) in copies]


def circuit_columns(tc, F, challenges):
    """{FIXED, ADVICE, INSTANCE} Montgomery columns of a tests/circuits.py circuit, synthesised with the given challenge ints"""
    n = tc.n
    adv = [None] * tc.cs.num_advice
    for phase in range(tc.cs.num_phases()):
        for c, v in tc.advice_ints(phase, {i: ch for i, ch in enumerate(challenges)}).items():
            if tc.cs.advice_phase[c] == phase:
                adv[c] = F.arr(v)
    inst = []
    for v in tc.instances:
        col = np.zeros((n, 4), dtype=np.uint64)
        col[: len(v)] = F.arr(v)
        inst.append(col)
    return {H.FIXED: [F.arr(c) for c in tc.fixed_ints], H.ADVICE: adv, H.INSTANCE: inst}
