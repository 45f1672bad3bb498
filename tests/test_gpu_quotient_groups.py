"""The quotient evaluated per degree group (QuotientGroups, csrc/prover.cu).  A constraint of degree d needs only the m n points
zeta D_{mn}, m the smallest power of two >= d - 1: the coset parts j = 0 mod E/m.  Each group is its own interpreter program; the
groups' quotients are added coefficient by coefficient, so every proof here must be byte-identical to the oracle prover's (which
evaluates everything on the full extended domain) and accepted by the oracle verifier.  ZKB_TRACE=1 prints one line per group; the
tests read it to check which groups ran, with how many constraints."""
import random
import re

import numpy as np
import pytest

import halo2_ref as H
import pyref as P
from halo2_ref import ADVICE
from test_gpu_prover import first_diff, to_product_cs

pytestmark = pytest.mark.gpu
R = P.R_MOD


class MixedDegreeCircuit:
    """gates: a list of (shared, d).  Gate t is  sel_t * (a_0 * a_1(1) * a_2 * .. (d - 1 factors) - c_t), of degree d.  Consecutive
    shared gates use the selector q (fixed 0), so the quotient folds them into one selector run; every other gate has a selector of
    its own.  Options: a permutation over a_0, a_1 and every c_t (copies a_1 <- a_0 that hold), and a logUp lookup of q_lk * a_0 into
    a fixed table (degree 5).  fixed: 0 q, 1 q_lk, 2 table, 3 + t gate t's own selector;  advice: 0..7 a_s, 8 + t c_t"""

    def __init__(self, k, gates, perm=False, lookup=False, seed=0):
        rnd = random.Random(seed)
        self.k, self.n = k, 1 << k
        n = self.n
        nf, na = 3 + len(gates), 8 + len(gates)
        cs = H.ConstraintSystem(k, nf, na, 0)
        factors = lambda d: [(s, 1 if s == 1 else 0) for s in range(d - 1)]   # (column, rotation) of each a_s
        sel_of = [0 if shared else 3 + t for t, (shared, _) in enumerate(gates)]
        for t, (_, d) in enumerate(gates):
            prod = None
            for c, r in factors(d):
                prod = H.advice(c, r) if prod is None else prod * H.advice(c, r)
            cs.gates.append(H.fixed(sel_of[t]) * (prod - H.advice(8 + t)))
        if lookup:
            cs.lookups.append(H.Lookup([[H.fixed(1) * H.advice(0)]], [H.fixed(2)]))
        if perm:
            cs.perm_columns = [(ADVICE, 0), (ADVICE, 1)] + [(ADVICE, 8 + t) for t in range(len(gates))]
        cs.finalize()
        self.cs = cs
        bf = cs.blinding_factors()
        usable = n - (bf + 1)
        T = 1 << max(1, k - 2)
        fixed = [[0] * n for _ in range(nf)]
        fixed[2][:T] = list(range(T))
        for sel in set(sel_of):
            for i in range(usable - 1):
                fixed[sel][i] = 1 if rnd.random() < 0.7 else 0
        for i in range(usable):
            fixed[1][i] = 1 if rnd.random() < 0.5 else 0
        cols = [[rnd.randrange(R) for _ in range(n)] for _ in range(na)]   # rows >= usable are the blinding rows
        if lookup:
            for i in range(usable):
                cols[0][i] = rnd.randrange(T)
        copies = []
        if perm:
            for i in rnd.sample(range(usable), max(1, usable // 8)):           # a_1[i] = a_0[j], decided before the outputs
                j = rnd.randrange(usable)
                cols[1][i] = cols[0][j]
                copies.append(((ADVICE, 1, i), (ADVICE, 0, j)))
        for t, (_, d) in enumerate(gates):
            for i in range(usable):
                if fixed[sel_of[t]][i]:
                    v = 1
                    for c, r in factors(d):
                        v = v * cols[c][i + r] % R
                    cols[8 + t][i] = v
        self.fixed_ints, self.copies, self.instances, self.cols = fixed, copies, [], cols
        self.nsets = (len(cs.perm_columns) + cs.degree() - 3) // (cs.degree() - 2) if perm else 0
        self.blinds_ints = {"z": [[rnd.randrange(R) for _ in range(bf)] for _ in range(self.nsets)],
                            "phi": [[rnd.randrange(R) for _ in range(bf)] for _ in cs.lookups],
                            "random_poly": [rnd.randrange(R) for _ in range(n)]}
        self.transcript_repr = rnd.randrange(R)

    def advice_ints(self, phase, challenges):
        return {c: list(v) for c, v in enumerate(self.cols)}

    def constraints(self):
        """quotient constraints: the gates, 2 nsets + 1 permutation terms (nsets > 0), 3 per lookup"""
        return len(self.cs.gates) + (2 * self.nsets + 1 if self.nsets else 0) + 3 * len(self.cs.lookups)


GROUP_LINE = re.compile(r"quotient group m = (\d+)\s+(\d+) constraints\s+(\d+) instructions/row\s+(\d+) coset NTTs")


def traced_groups(err):
    """{m: constraints} from the ZKB_TRACE lines of one proof"""
    return {int(m.group(1)): int(m.group(2)) for m in GROUP_LINE.finditer(err)}


def prove_and_compare(tc, monkeypatch, capfd):
    """prove tc on the device and with the oracle, byte for byte; returns the device's groups {m: constraints} and E"""
    from zkb200 import plonk as Z
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": rp}
    synth = lambda phase, ch: {c: F.arr(v) for c, v in tc.advice_ints(phase, ch).items()}
    proof_ref, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, synth, blinds)
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof_ref)

    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    zb = np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]) if tc.blinds_ints["z"] else None
    pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]) if tc.blinds_ints["phi"] else None
    monkeypatch.setenv("ZKB_TRACE", "1")
    capfd.readouterr()
    proof = Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth, zb, pb, rp)
    groups = traced_groups(capfd.readouterr().err)
    assert len(proof) == len(proof_ref)
    assert first_diff(proof, proof_ref) is None, f"first differing 32-byte proof item: {first_diff(proof, proof_ref)}"
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof)
    assert sum(groups.values()) == tc.constraints()
    E = 1
    while E < ref.d - 1:
        E *= 2
    return groups, E


S, Q = False, True   # a gate with its own selector / one of the selector run on q


def test_extended_domain_of_two(monkeypatch, capfd):
    """degree 3 (E = 2): the degree-2 gate and the permutation's l_0 terms need part 0 only; the run (2, 3), (z_l^2 - z_l) l_last
    and the set products (degree 3) need both parts"""
    tc = MixedDegreeCircuit(6, [(Q, 2), (Q, 3), (S, 2)], perm=True, seed=1)
    groups, E = prove_and_compare(tc, monkeypatch, capfd)
    assert E == 2 and tc.nsets == 5
    assert groups == {1: 1 + 1 + 4, 2: 2 + 1 + 5}


def test_extended_domain_of_four(monkeypatch, capfd):
    """degree 5 (E = 4): gates of degree 2, 3 and 5 and a degree-5 lookup whose l_0 / l_last terms have degree 2"""
    tc = MixedDegreeCircuit(6, [(S, 5), (S, 2), (S, 3)], perm=True, lookup=True, seed=2)
    groups, E = prove_and_compare(tc, monkeypatch, capfd)
    assert E == 4 and tc.nsets == 2
    # m = 1: the degree-2 gate, (1 - z_0) l_0, the set link, the lookup's l_0 / l_last terms;  m = 2: the degree-3 gate and
    # (z_l^2 - z_l) l_last;  m = 4: the degree-5 gate, the two set products (degree 5 and 4), the lookup's main constraint
    assert groups == {1: 1 + 2 + 2, 2: 1 + 1, 4: 1 + 2 + 1}


def test_degrees_two_to_nine_with_a_run_across_groups(monkeypatch, capfd):
    """degree 9 (E = 8): constraints of degree 2, 3, 5 and 9 in one circuit.  The selector run (3, 9, 2) goes whole to the group of
    its degree-9 member, so the group m = 8 folds a run; the single gates go to their own groups"""
    tc = MixedDegreeCircuit(6, [(S, 5), (Q, 3), (Q, 9), (Q, 2), (S, 2), (S, 3), (S, 5)], perm=True, lookup=True, seed=3)
    groups, E = prove_and_compare(tc, monkeypatch, capfd)
    assert E == 8 and tc.nsets == 2
    # m = 8: the run and the first set product (7 columns);  m = 4: the degree-5 gates, the second set product (2 columns, degree
    # 4) and the lookup's main constraint
    assert groups == {1: 1 + 2 + 2, 2: 1 + 1, 4: 2 + 1 + 1, 8: 3 + 1}


def test_gaps_in_y_around_a_folded_run(monkeypatch, capfd):
    """a run of degree-3 gates between degree-3 and degree-9 gates: within the group m = 2 the run follows its previous member
    after a gap (FOLD steps by y^(s - i_prev - 1 + r), not y^r) and is followed by one; m = 8 steps by y^4"""
    tc = MixedDegreeCircuit(6, [(S, 3), (S, 9), (Q, 3), (Q, 2), (Q, 3), (S, 9), (S, 3)], seed=4)
    groups, E = prove_and_compare(tc, monkeypatch, capfd)
    assert E == 8
    assert groups == {2: 5, 8: 2}


def test_empty_top_group(monkeypatch, capfd):
    """degree-2 gates only, no permutation or lookup: the constraint system's degree is 3 (E = 2), but every constraint fits
    part 0, so the top group is empty and h comes from one size-n inverse transform.  h then has degree below n while the
    quotient has qdeg = 2 pieces: the second piece is zero and its commitment the point at infinity, which no transcript can
    take.  The oracle prover refuses such a circuit, and so must the device, at the same point."""
    from zkb200 import plonk as Z
    from zkb200.lib import ZkbError
    tc = MixedDegreeCircuit(5, [(Q, 2), (Q, 2), (S, 2)], seed=5)
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    synth = lambda phase, ch: {c: F.arr(v) for c, v in tc.advice_ints(phase, ch).items()}
    with pytest.raises(AssertionError, match="points at infinity"):
        ref.create_proof(pkr, tc.transcript_repr, tc.instances, synth, {"z": [], "phi": [], "random_poly": rp})
    assert ref.d == 3
    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    monkeypatch.setenv("ZKB_TRACE", "1")
    capfd.readouterr()
    with pytest.raises(ZkbError, match="points at infinity"):
        Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [], synth, None, None, rp)
    assert traced_groups(capfd.readouterr().err) == {1: 3}


def test_super_circuit_standin(monkeypatch, capfd):
    """the k = 13 SuperCircuit-shaped stand-in, byte for byte against the oracle prover, split into the groups m = 1, 2, 4, 8"""
    import test_gpu_standins   # a module import: pytest must not collect its test a second time here
    monkeypatch.setenv("ZKB_TRACE", "1")
    capfd.readouterr()
    test_gpu_standins.test_standin_proof_bytes_match_oracle("super", 13, dict(advice=64, scale=1.0, n_gates=120))
    groups = traced_groups(capfd.readouterr().err)
    assert sorted(groups) == [1, 2, 4, 8]
    assert groups[4] > groups[8]      # the condition gates (degree 5) outnumber the degree-9 set products and lookups


@pytest.mark.parametrize("case", [test_extended_domain_of_two, test_extended_domain_of_four, test_degrees_two_to_nine_with_a_run_across_groups,
                                  test_gaps_in_y_around_a_folded_run], ids=lambda f: f.__name__[len("test_"):])
def test_without_coset_cache(case, monkeypatch, capfd):
    """the proofs above, which run with the pk's coset cache of fixed, sigma, X, l_0, l_last and l_blind, made again with the cache off
    (ZKB_COSET_CACHE_GB=0, read when the pk is built): every coset part then transforms those polynomials itself, and the bytes and
    groups must be the same"""
    monkeypatch.setenv("ZKB_COSET_CACHE_GB", "0")
    case(monkeypatch, capfd)
