"""The CPU reference of the witness check (tests/witness_ref.py): no failures on the satisfied witnesses of every circuit family, and
exactly the injected faults otherwise -- a broken advice cell, a lookup input moved out of its table, a broken permutation cell, a
selector switched on in a blinding row (poisoned).  One injected gate fault also makes the oracle verifier reject the oracle proof,
which ties the checker's notion of "fails" to the verifier's."""
import numpy as np
import pytest

import halo2_ref as H
import standin_copies
import standins
from circuits import ToyCircuit, ThinCompressionShape, GatesOnlyCircuit, DeepGateCircuit
from test_gpu_prover_wide import to_oracle_cs
from witness_ref import check_witness, perm_copies, circuit_columns

CH = [0x5EED5, 0xC0FFEE]


def run_ref(tc, cols=None):
    ref = H.Ref(tc.cs, 0, build_srs=False)
    cols = cols or circuit_columns(tc, ref.F, CH)
    return check_witness(ref, tc.cs, cols, CH, perm_copies(tc.cs, tc.copies), tc.n - ref.bf - 1), cols, ref


@pytest.mark.parametrize("make", [lambda: ToyCircuit(6, seed=1), lambda: ToyCircuit(6, seed=2, two_phase=False), lambda: ThinCompressionShape(7, seed=3),
                                  lambda: GatesOnlyCircuit(6, seed=4), lambda: DeepGateCircuit(6, seed=5)],
                         ids=["toy", "toy-one-phase", "thin", "gates-only", "deep"])
def test_satisfied_circuits_have_no_failures(make):
    tc = make()
    (counts, recs), _, _ = run_ref(tc)
    assert not counts.any() and recs == []
    assert len(counts) == len(tc.cs.gates) + sum(len(lk.inputs) for lk in tc.cs.lookups) + 1


@pytest.mark.parametrize("kind", ["keccak", "super"])
def test_satisfied_standins_have_no_failures(kind):
    ops = standins.OracleOps()
    sc = standins.keccak_shape(9, seed=1, ops=ops, scale=0.12) if kind == "keccak" else standins.super_shape(8, seed=2, ops=ops, advice=40, n_gates=60)
    cs = to_oracle_cs(sc.cs)
    ref = H.Ref(cs, 0, build_srs=False)
    F = ref.F
    ch = F.arr(CH[: len(sc.cs.challenge_phase)])
    fixed, adv, inst = standin_copies.witness(sc, list(ch))
    cols = {H.FIXED: [sc.host(t) for t in fixed], H.ADVICE: [sc.host(t) for t in adv], H.INSTANCE: [sc.host(t) for t in inst]}
    copies = standin_copies.copies(sc).numpy().astype(np.uint32)
    assert len(copies) == (sc.P - 1) * sc.usable
    counts, recs = check_witness(ref, cs, cols, CH[: len(sc.cs.challenge_phase)], copies, sc.usable)
    assert not counts.any() and recs == []
    # one broken permutation cell of column 0 breaks exactly the copies that point at it
    v = 17
    cols[H.ADVICE][sc.c_perm0] = cols[H.ADVICE][sc.c_perm0].copy()
    cols[H.ADVICE][sc.c_perm0][v] = F.arr([12345])[0]
    counts, recs = check_witness(ref, cs, cols, CH[: len(sc.cs.challenge_phase)], copies, sc.usable)
    want = [(2, int(i), 0, int(copies[i][1])) for i in np.nonzero(copies[:, 3] == v)[0]]
    assert len(want) == sc.P - 1 and recs == want


def selector(gate):
    """(fixed column, rotation) of the gate's selector factor q in q * constraint"""
    assert gate.op == H.MUL and gate.a.op == H.FIXED
    return gate.a.a, gate.a.b


def advice_queries(e, col, out=None):
    out = [] if out is None else out
    if e.op == H.ADVICE and e.a == col: out.append(e.b)
    elif e.op in (H.NEG, H.SCALED): advice_queries(e.a, col, out)
    elif e.op in (H.ADD, H.MUL): advice_queries(e.a, col, out); advice_queries(e.b, col, out)
    return out


def test_broken_advice_cell_fails_where_the_gates_read_it():
    tc = ToyCircuit(7, seed=9, lookups=False, extra_perm=False)
    (_, _), cols, ref = run_ref(tc)
    n, F = tc.n, ref.F
    c = 2                                                    # advice c is read by gate 0 at rotation 0 and gate 1 at rotation 1
    r = next(i for i in range(2, tc.usable) if tc.fixed_ints[0][i] and tc.fixed_ints[1][i - 1] == 0)
    cols[H.ADVICE][c] = cols[H.ADVICE][c].copy()
    cols[H.ADVICE][c][r] = F.arr([F.ints(cols[H.ADVICE][c][r:r + 1])[0] + 1])[0]
    counts, recs = check_witness(ref, tc.cs, cols, CH, [], tc.n - ref.bf - 1)
    want = []
    for g, gate in enumerate(tc.cs.gates):
        s, srot = selector(gate)
        rows = sorted({(r - rot) % n for rot in advice_queries(gate, c)})
        want += [(0, g, 0, i) for i in rows if tc.fixed_ints[s][(i + srot) % n]]
    assert want and [x for x in recs if x[0] == 0] == want
    assert all(x[0] != 1 for x in recs)


def test_lookup_input_out_of_table_and_its_copies():
    tc = ToyCircuit(7, seed=10)
    i = next(i for i in range(2, tc.usable) if tc.fixed_ints[2][i])
    tc.cols0[3][i] = 123456789                             # d at a q_lk row: lookups 0 (set 0) and 1 read d(0), lookup 0 set 1 reads d(1)
    (counts, recs), _, ref = run_ref(tc)
    want = [(1, 0, 0, i)] + ([(1, 0, 1, i - 1)] if tc.fixed_ints[3][i - 1] else []) + [(1, 1, 0, i)]
    assert [x for x in recs if x[0] == 1] == want
    copies = perm_copies(tc.cs, tc.copies)
    d = tc.cs.perm_columns.index((H.ADVICE, 3))
    touching = [(2, k, 0, lr) for k, (lc, lr, rc, rr) in enumerate(copies) if (lc, lr) == (d, i) or (rc, rr) == (d, i)]
    assert [x for x in recs if x[0] == 2] == touching
    assert not any(x[0] == 0 for x in recs)


def test_broken_permutation_cell_breaks_the_copies_that_touch_it():
    tc = ToyCircuit(7, seed=11)
    copies = perm_copies(tc.cs, tc.copies)
    a = tc.cs.perm_columns.index((H.ADVICE, 0))
    lc, lr, rc, rr = next(cp for cp in copies if cp[0] == a)
    tc.cols0[0][lr] = (tc.cols0[0][lr] + 5) % H.R
    (counts, recs), _, _ = run_ref(tc)
    touching = [(2, k, 0, x[1]) for k, x in enumerate(copies) if (x[0], x[1]) == (a, lr) or (x[2], x[3]) == (a, lr)]
    assert touching and [x for x in recs if x[0] == 2] == touching
    assert counts[-1] == len(touching)


def test_selector_in_a_blinding_row_is_poisoned():
    tc = GatesOnlyCircuit(6, seed=12)
    row = tc.usable + 1
    tc.fixed_ints[0][row] = 1
    (counts, recs), _, _ = run_ref(tc)
    assert recs == [(0, 0, 1, row)] and list(counts) == [1, 0]


def test_gate_fault_found_by_checker_is_rejected_by_the_verifier():
    tc = ToyCircuit(6, seed=13)
    tc.tamper()                                              # breaks one mul gate: c[i] += 1 at the first q_mul row
    i = next(i for i in range(tc.usable) if tc.fixed_ints[0][i])
    (counts, recs), _, ref = run_ref(tc)
    assert (0, 0, 0, i) in recs and counts[0] >= 1
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    pkr = ref.keygen([F.arr(c) for c in tc.fixed_ints], tc.copies)
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": F.arr(tc.blinds_ints["random_poly"])}
    proof, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, ch).items()}, blinds)
    assert not ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof)
