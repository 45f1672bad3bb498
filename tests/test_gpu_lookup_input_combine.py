"""Lookup input sets combined in coefficient form (lookup_input_combos, csrc/prover.cu).  An input set S * a_0(w^r X), ..,
S * a_{W-1}(w^r X) with one advice-free cofactor S (or none) and one rotation r is theta-compressed to S * A(w^r X), A =
sum_c theta^(W-1-c) a_c formed once from the advice polynomials: the quotient transforms A instead of the W columns.  A set
combines only when none of its columns is read in the quotient other than through combined sets.  Every proof here must be
byte-identical to the oracle prover's and accepted by its verifier, and the ZKB_TRACE line of the top degree group must show the
coset NTTs that the combinations save: E x (columns read only through combinations - combinations)."""
import random
import re

import numpy as np
import pytest

import halo2_ref as H
import pyref as P
from test_gpu_prover import first_diff, to_product_cs

pytestmark = pytest.mark.gpu
R = P.R_MOD
GROUP_LINE = re.compile(r"quotient group m = (\d+)\s+(\d+) constraints\s+(\d+) instructions/row\s+(\d+) coset NTTs")
TABLE_BASE = {2: 8, 3: 4}   # table of width W: every W-tuple of values below TABLE_BASE[W] (row 0 the zero tuple)
Q1, Q2 = 1, 2               # fixed cofactor columns (0 is the gate selector)


class CombineCircuit:
    """lookups: a list of input-set lists; a set is a list of terms (cofactor, column, rotation) into the table of its width.
    cofactor: None (a bare advice term), Q1 / Q2 (a fixed 0/1 column) or ("adv", c) (q1 * advice c, a 0/1 column).  Every
    lookup column holds values below 4 on every row, so any term of any set at any rotation is in its table.  squared: columns
    c that a gate q * (s_c - c * c) also reads, s_c a column of its own.
    fixed: 0 q, 1 q1, 2 q2, then the width-2 table, then the width-3 table;  advice: 0 .. n_cols - 1, then the s_c"""

    def __init__(self, k, lookups, squared=(), seed=0):
        rnd = random.Random(seed)
        self.k, self.n = k, 1 << k
        n = self.n
        n_cols = 1 + max(c for sets in lookups for s in sets for cof, col, _ in s for c in (col, cof[1] if isinstance(cof, tuple) else 0))
        tcol = {2: 3, 3: 5}
        nf, na = 8, n_cols + len(squared)
        cs = H.ConstraintSystem(k, nf, na, 0)
        for t, c in enumerate(squared):
            cs.gates.append(H.fixed(0) * (H.advice(n_cols + t) - H.advice(c) * H.advice(c)))

        def term(cof, col, rot):
            a = H.advice(col, rot)
            if cof is None: return a
            if isinstance(cof, tuple): return H.fixed(Q1) * H.advice(cof[1]) * a
            return H.fixed(cof) * a
        for sets in lookups:
            W = len(sets[0])
            cs.lookups.append(H.Lookup([[term(*t) for t in s] for s in sets], [H.fixed(tcol[W] + c) for c in range(W)]))
        cs.finalize()
        self.cs = cs
        bf = cs.blinding_factors()
        usable = n - (bf + 1)
        fixed = [[0] * n for _ in range(nf)]
        for i in range(usable):
            fixed[0][i] = 1 if rnd.random() < 0.7 else 0
            fixed[Q1][i] = 1 if rnd.random() < 0.6 else 0
            fixed[Q2][i] = 1 if rnd.random() < 0.6 else 0
        for W, c0 in tcol.items():
            V = TABLE_BASE[W]
            for j in range(V ** W):
                for c in range(W):
                    fixed[c0 + c][j] = j // V ** (W - 1 - c) % V
        bits = {cof[1] for sets in lookups for s in sets for cof, _, _ in s if isinstance(cof, tuple)}
        cols = [[rnd.randrange(2 if c in bits else 4) for _ in range(n)] for c in range(n_cols)]
        cols += [[v * v % R for v in cols[c]] for c in squared]
        self.fixed_ints, self.copies, self.instances, self.cols = fixed, [], [], cols
        self.blinds_ints = {"z": [], "phi": [[rnd.randrange(R) for _ in range(bf)] for _ in cs.lookups],
                            "random_poly": [rnd.randrange(R) for _ in range(n)]}
        self.transcript_repr = rnd.randrange(R)
        # advice columns the input sets read, their cofactors' included
        self.input_columns = len({c for sets in lookups for s in sets for cof, col, _ in s for c in ([col] + ([cof[1]] if isinstance(cof, tuple) else []))})

    def advice_ints(self, phase, challenges):
        return {c: list(v) for c, v in enumerate(self.cols)}

    def constraints(self):
        return len(self.cs.gates) + 3 * len(self.cs.lookups)


def prove_traced(tc, monkeypatch, capfd):
    """prove tc on the device and with the oracle, byte for byte; -> ({m: (constraints, coset NTTs)} of the device's proof, E)"""
    from zkb200 import plonk as Z
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    blinds = {"z": [], "phi": tc.blinds_ints["phi"], "random_poly": rp}
    synth = lambda phase, ch: {c: F.arr(v) for c, v in tc.advice_ints(phase, ch).items()}
    proof_ref, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, synth, blinds)
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof_ref)

    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]])
    monkeypatch.setenv("ZKB_TRACE", "1")
    capfd.readouterr()
    proof = Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [], synth, None, pb, rp)
    groups = {int(m.group(1)): (int(m.group(2)), int(m.group(4))) for m in GROUP_LINE.finditer(capfd.readouterr().err)}
    assert first_diff(proof, proof_ref) is None, f"first differing 32-byte proof item: {first_diff(proof, proof_ref)}"
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof)
    assert sum(c for c, _ in groups.values()) == tc.constraints()
    E = 1
    while E < ref.d - 1:
        E *= 2
    return groups, E


def check_top_group(tc, monkeypatch, capfd, only, combos):
    """every lookup is in the top group, which reads nothing else the coset cache does not hold: per lookup phi and m, and the input
    columns, of which the `only` read only through combinations are replaced by `combos` combined columns"""
    groups, E = prove_traced(tc, monkeypatch, capfd)
    assert E == 8 and max(groups) == 8
    assert groups[8] == (len(tc.cs.lookups), 8 * (2 * len(tc.cs.lookups) + tc.input_columns - (only - combos)))


def test_pair_at_three_rotations(monkeypatch, capfd):
    """q1 * (a, b) at rotations 0, 1 and -1: the three sets share one combination"""
    tc = CombineCircuit(8, [[[(Q1, 0, r), (Q1, 1, r)] for r in (0, 1, -1)]], seed=1)
    check_top_group(tc, monkeypatch, capfd, only=2, combos=1)


def test_width_three_with_and_without_cofactor(monkeypatch, capfd):
    """width 3: the bare (a, b, c) and q1 * (a, b, c)(w X) share a combination, q2 * (d, e, f) has its own; width 2, bare:
    (g, h) at rotations 0 and 1 and (h, g) are two combinations (the order of the columns is the order of theta's powers)"""
    tc = CombineCircuit(8, [[[(None, 0, 0), (None, 1, 0), (None, 2, 0)], [(Q1, 0, 1), (Q1, 1, 1), (Q1, 2, 1)], [(Q2, 3, 0), (Q2, 4, 0), (Q2, 5, 0)]],
                            [[(None, 6, 0), (None, 7, 0)], [(None, 6, 1), (None, 7, 1)], [(None, 7, 0), (None, 6, 0)]]], seed=2)
    check_top_group(tc, monkeypatch, capfd, only=8, combos=4)


def test_sets_that_do_not_combine(monkeypatch, capfd):
    """compressed term by term: mixed rotations (a, b(w X)); different cofactors q1 * c, q2 * d; a cofactor q1 * s that reads advice;
    g, which a gate also reads, and so its partner h, and then (h, k), which shares h.  Only the bare (i, j) combines"""
    tc = CombineCircuit(8, [[[(Q1, 0, 0), (Q1, 1, 1)], [(Q1, 2, 0), (Q2, 3, 0)], [(Q1, 6, 0), (Q1, 7, 0)]],
                            [[(("adv", 4), 5, 0), (("adv", 4), 8, 0)], [(None, 9, 0), (None, 10, 0)], [(Q1, 7, -1), (Q1, 11, -1)]]],
                        squared=(6,), seed=3)
    check_top_group(tc, monkeypatch, capfd, only=2, combos=1)


def test_super_circuit_standin(monkeypatch, capfd):
    """the k = 13 SuperCircuit stand-in byte for byte against the oracle prover; its 16 pair columns are read only by the lookups, in
    8 pairs.  The same constraint system with one more gate q_lk * (c - c) per pair column compresses every set term by term: its
    top group transforms 8 x (16 - 8) more coset columns, and the other groups' transforms are the same"""
    import standins
    import test_gpu_standins   # a module import: pytest must not collect its test a second time here
    from zkb200.params import ParamsKZG
    from zkb200.plonk import Expression as Ex

    def traced(prove):
        monkeypatch.setenv("ZKB_TRACE", "1")
        capfd.readouterr()
        prove()
        return {int(m.group(1)): (int(m.group(2)), int(m.group(4))) for m in GROUP_LINE.finditer(capfd.readouterr().err)}
    kw = dict(advice=64, scale=1.0, n_gates=120)
    combined = traced(lambda: test_gpu_standins.test_standin_proof_bytes_match_oracle("super", 13, kw))
    sc = standins.super_shape(13, seed=13, **kw)
    pairs = range(sc.c_pair0, sc.c_perm0)
    assert len(pairs) == 16 and len({pr for _, sets in sc.lk_plan for pr, _ in sets}) == 8
    # selector q_lk, which no other gate uses: the new gates form a selector run of their own, of degree 2 (group m = 1)
    sc.cs.gates += [Ex.Fixed(1) * (Ex.Advice(c) + (-Ex.Advice(c))) for c in pairs]
    separate = traced(lambda: test_gpu_standins.prove_gpu(sc, ParamsKZG.unsafe_setup_with_s(13, 4321)))
    assert sorted(combined) == sorted(separate) == [1, 2, 4, 8]
    assert separate[1] == (combined[1][0] + 16, combined[1][1])
    assert separate[8] == (combined[8][0], combined[8][1] + 8 * (16 - 8))
    assert all(separate[m] == combined[m] for m in (2, 4))
