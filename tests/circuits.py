"""Synthetic satisfiable PLONKish circuits for the prover parity tests (stand-ins for circuits we cannot synthesise
without Rust: SURVEY.md 8d).  Shape knobs mimic what the zkEVM circuits exercise: custom gates with rotations, a
multi-column permutation with several chunks, mv-lookups with more than one input set per table, an instance column,
and a second advice phase driven by a challenge (zkevm-circuits/src/util.rs:120-133)."""
import random
import numpy as np

import pyref as P
import halo2_ref as H
from halo2_ref import FIXED, ADVICE, INSTANCE

R = P.R_MOD


class ToyCircuit:
    """fixed: 0 q_mul, 1 q_add, 2 q_lk, 3 q_lk2, 4 t0, 5 t1, 6 q_ch, 7 konst
       advice: 0 a, 1 b, 2 c, 3 d, 4 e (phase 0), 5 f (phase 1)        instance: 0"""

    def __init__(self, k, seed=0, two_phase=True, lookups=True, n_instance=4, extra_perm=True):
        rnd = random.Random(seed)
        self.k, self.n = k, 1 << k
        n = self.n
        self.two_phase = two_phase
        adv_phase = [0, 0, 0, 0, 0, 1 if two_phase else 0]
        cs = H.ConstraintSystem(k, 8, 6, 1, adv_phase, [0] if two_phase else [])
        a, b, c, d, e, f = [lambda r=0, i=i: H.advice(i, r) for i in range(6)]
        fx = lambda i, r=0: H.fixed(i, r)
        cs.gates.append(fx(0) * (a() * b() - c()))
        cs.gates.append(fx(1) * (a() + b(1) - c(1)))
        if two_phase:
            cs.gates.append(fx(6) * (f() - H.challenge(0) * a() * b()))
        else:
            cs.gates.append(fx(6) * (f() - H.scaled(a() * b(), 5)))
        if lookups:
            cs.lookups.append(H.Lookup([[fx(2) * d(), fx(2) * e()], [fx(3) * d(1), fx(3) * e(1)]], [fx(4), fx(5)]))
            cs.lookups.append(H.Lookup([[fx(2) * d()]], [fx(4)]))
        cs.perm_columns = [(ADVICE, 0), (ADVICE, 1), (ADVICE, 2), (INSTANCE, 0), (FIXED, 7)]
        if extra_perm:
            cs.perm_columns += [(ADVICE, 3), (ADVICE, 4), (ADVICE, 5)]
        cs.finalize()
        self.cs = cs
        bf = cs.blinding_factors()
        usable = n - (bf + 1)
        self.usable = usable
        # ---- fixed columns
        T = max(2, min(usable, 1 << max(1, k - 2)))
        fixed = [[0] * n for _ in range(8)]
        for j in range(1, T):
            fixed[4][j] = j
            fixed[5][j] = (j * j + 7) % R
        for i in range(usable):
            fixed[7][i] = rnd.randrange(R) if i % 3 == 0 else (i + 1)
        q_mul, q_add, q_lk, q_lk2, q_ch = fixed[0], fixed[1], fixed[2], fixed[3], fixed[6]
        for i in range(usable - 1):
            t = rnd.random()
            if t < 0.4: q_mul[i] = 1
            elif t < 0.7: q_add[i] = 1
        for i in range(1, usable):           # an add row at i-1 fixes c[i]: row i cannot also be a mul row
            if q_add[i - 1]: q_mul[i] = 0
        for i in range(usable - 1):
            if rnd.random() < 0.5: q_lk[i] = 1
            if rnd.random() < 0.3: q_lk2[i] = 1
            if rnd.random() < 0.5: q_ch[i] = 1
        self.fixed_ints = fixed
        # ---- witness (phase 0)
        self.instances = [[rnd.randrange(R) for _ in range(n_instance)]]
        A = [rnd.randrange(R) for _ in range(n)]
        B = [rnd.randrange(R) for _ in range(n)]
        C = [rnd.randrange(R) for _ in range(n)]
        D = [0] * n
        E = [0] * n
        copies = []
        for i in range(usable):
            # copy constraints decided before the row's outputs are computed
            t = rnd.random()
            if i > 2 and t < 0.25:
                j = rnd.randrange(i)
                A[i] = C[j]; copies.append(((ADVICE, 0, i), (ADVICE, 2, j)))
            elif t < 0.35 and n_instance:
                j = rnd.randrange(n_instance)
                A[i] = self.instances[0][j]; copies.append(((ADVICE, 0, i), (INSTANCE, 0, j)))
            elif t < 0.45:
                j = rnd.randrange(usable)
                A[i] = fixed[7][j]; copies.append(((ADVICE, 0, i), (FIXED, 7, j)))
            if i > 0 and q_add[i - 1]:
                pass                                           # b[i] free, c[i] = a[i-1] + b[i]
            elif i > 2 and rnd.random() < 0.2:
                j = rnd.randrange(i)
                B[i] = B[j]; copies.append(((ADVICE, 1, i), (ADVICE, 1, j)))
            if q_mul[i]: C[i] = A[i] * B[i] % R
            if i > 0 and q_add[i - 1]: C[i] = (A[i - 1] + B[i]) % R
        # lookups: rows with q_lk (or q_lk2 at i-1) carry a table row
        for i in range(usable):
            need = q_lk[i] or (i > 0 and q_lk2[i - 1])
            j = rnd.randrange(T) if need else rnd.randrange(T)
            D[i], E[i] = fixed[4][j], fixed[5][j]
        if extra_perm:
            for _ in range(max(1, usable // 8)):
                i, j = rnd.randrange(usable), rnd.randrange(usable)
                if D[i] == D[j]: copies.append(((ADVICE, 3, i), (ADVICE, 3, j)))
                if E[i] == E[j]: copies.append(((ADVICE, 4, i), (ADVICE, 4, j)))
        self.copies = copies
        self.cols0 = [A, B, C, D, E]
        self.rnd = rnd
        self.bf = bf
        self.blind_rows = {c: [rnd.randrange(R) for _ in range(bf + 1)] for c in range(6)}
        nsets = (len(cs.perm_columns) + (cs.degree() - 2) - 1) // (cs.degree() - 2)
        self.blinds_ints = {"z": [[rnd.randrange(R) for _ in range(bf)] for _ in range(nsets)],
                            "phi": [[rnd.randrange(R) for _ in range(bf)] for _ in cs.lookups],
                            "random_poly": [rnd.randrange(R) for _ in range(n)]}
        self.transcript_repr = rnd.randrange(R)

    # column values as ints, blinded
    def advice_ints(self, phase, challenges):
        n, usable = self.n, self.usable
        out = {}
        if phase == 0:
            for ci, col in enumerate(self.cols0):
                v = list(col); v[usable:] = self.blind_rows[ci]; out[ci] = v
            if not self.two_phase:
                out[5] = self._f(5)
        if phase == 1 and self.two_phase:
            out[5] = self._f(challenges[0])
        return out

    def _f(self, ch):
        A, B = self.cols0[0], self.cols0[1]
        v = [ch * A[i] % R * B[i] % R if self.fixed_ints[6][i] else (i * 31 + 5) % R for i in range(self.n)]
        v[self.usable:] = self.blind_rows[5]
        return v

    def tamper(self):
        """break one mul gate"""
        for i in range(self.usable):
            if self.fixed_ints[0][i]:
                self.cols0[2][i] = (self.cols0[2][i] + 1) % R
                return


class ThinCompressionShape:
    """The constraint system of the reference's thin compression circuit exactly as its snark-verifier `Protocol` spells it
    (aggregator/data/batch-task.json -> chunk_proofs[0].protocol, SURVEY.md appendix B), at a small k with a synthetic witness:
      fixed: 0 lookup table, 1 constants column, 2 gate selector, 3 lookup selector;  advice: 0;  instance: 0
      gate  : q_gate * (a(0) + a(1) * a(2) - a(3))            (halo2-lib flex gate)
      lookup: (q_lookup * a(0)) in table                       (one input set, one table column)
      permutation over [fixed 1, advice 0, instance 0]         (one chunk: cs degree 5 -> chunk length 3)
    Expected proof layout (fixture): 1 advice + 1 m + z, phi, random + 4 h pieces + 17 evals + 2 = 28 items."""

    @staticmethod
    def constraint_system(k):
        cs = H.ConstraintSystem(k, 4, 1, 1)
        a = lambda r=0: H.advice(0, r)
        cs.gates.append(H.fixed(2) * (a(0) + a(1) * a(2) - a(3)))
        cs.lookups.append(H.Lookup([[H.fixed(3) * a(0)]], [H.fixed(0)]))
        cs.perm_columns = [(FIXED, 1), (ADVICE, 0), (INSTANCE, 0)]
        cs.finalize()
        # the fixture's evaluation order lists fixed column 1 (constants, from the permutation) before column 0: halo2 records
        # queries in configure() order (enable_equality on the constants column happens before the lookup table is queried)
        cs.fixed_queries = [(1, 0), (0, 0), (2, 0), (3, 0)]
        return cs

    def __init__(self, k, seed=0, n_instance=6, table=None):
        """table: optional usable -> (m, 4) uint64 array of extra table values in the stored (Montgomery) form; they follow the T small
        values, a few of them repeat at later rows and one past the usable rows, and the range-checked cells draw from the whole table."""
        rnd = random.Random(seed)
        self.k, self.n = k, 1 << k
        n = self.n
        cs = self.constraint_system(k)
        self.cs = cs
        bf = cs.blinding_factors()
        assert bf == 6 and cs.degree() == 5
        usable = n - (bf + 1)
        self.usable = usable
        T = 1 << max(2, k - 2)
        fixed = [[0] * n for _ in range(4)]
        for j in range(T): fixed[0][j] = j
        if table is not None:
            extra = [P.from_mont(P.from_limbs(v), R) for v in table(usable)]
            dups = [extra[rnd.randrange(len(extra))] for _ in range(max(1, len(extra) // 8))]
            assert T + len(extra) + len(dups) <= usable
            fixed[0][T:T + len(extra)] = extra
            fixed[0][T + len(extra):T + len(extra) + len(dups)] = dups
            fixed[0][usable] = extra[0]
            T = T + len(extra) + len(dups)          # the range-checked cells below draw from every table row set so far
        self.instances = [[rnd.randrange(R) for _ in range(n_instance)]]
        A = [rnd.randrange(T) for _ in range(n)]          # default: small values (valid lookup inputs)
        copies = []
        r = 0
        while r + 4 <= usable:
            kind = rnd.random()
            if kind < 0.5:                                 # a gate instance on rows r..r+3
                fixed[2][r] = 1
                A[r], A[r + 1], A[r + 2] = rnd.randrange(R), rnd.randrange(R), rnd.randrange(R)
                if kind < 0.1 and n_instance:
                    j = rnd.randrange(n_instance); A[r] = self.instances[0][j]; copies.append(((ADVICE, 0, r), (INSTANCE, 0, j)))
                elif kind < 0.2:
                    c = rnd.randrange(R); fixed[1][r] = c; A[r] = c; copies.append(((ADVICE, 0, r), (FIXED, 1, r)))
                A[r + 3] = (A[r] + A[r + 1] * A[r + 2]) % R
                r += 4
            else:                                          # a range-checked cell
                fixed[3][r] = 1
                A[r] = fixed[0][rnd.randrange(T)]
                r += 1
        for _ in range(usable // 8):
            i, j = rnd.randrange(usable), rnd.randrange(usable)
            if A[i] == A[j]: copies.append(((ADVICE, 0, i), (ADVICE, 0, j)))
        self.fixed_ints, self.copies, self.A = fixed, copies, A
        self.bf = bf
        self.blind = [rnd.randrange(R) for _ in range(bf + 1)]
        self.blinds_ints = {"z": [[rnd.randrange(R) for _ in range(bf)]], "phi": [[rnd.randrange(R) for _ in range(bf)]],
                            "random_poly": [rnd.randrange(R) for _ in range(n)]}
        self.transcript_repr = rnd.randrange(R)

    def advice_ints(self, phase, challenges):
        v = list(self.A)
        v[self.usable:] = self.blind
        return {0: v}


class GatesOnlyCircuit:
    """No permutation, no lookup, no instance: one fixed selector, two advice columns, one degree-3 gate with rotations."""

    def __init__(self, k, seed=0):
        rnd = random.Random(seed)
        self.k, self.n = k, 1 << k
        n = self.n
        cs = H.ConstraintSystem(k, 1, 2, 0)
        cs.gates.append(H.fixed(0) * (H.advice(0) * H.advice(1, 1) - H.advice(1, -1)))
        cs.finalize()
        self.cs = cs
        bf = cs.blinding_factors()
        usable = n - (bf + 1)
        self.usable = usable
        q = [1 if 0 < i < usable - 1 and i % 2 == 1 else 0 for i in range(n)]
        a0 = [rnd.randrange(R) for _ in range(n)]
        a1 = [rnd.randrange(R) for _ in range(n)]
        for i in range(n - 1, -1, -1):                            # descending: a1[i+1] is final when a1[i-1] is derived
            if q[i]: a1[i - 1] = a0[i] * a1[i + 1] % R           # odd rows constrain their even neighbours
        self.fixed_ints, self.copies, self.instances = [q], [], []
        self.cols = [a0, a1]
        self.blind_rows = [[rnd.randrange(R) for _ in range(bf + 1)] for _ in range(2)]
        self.blinds_ints = {"z": [], "phi": [], "random_poly": [rnd.randrange(R) for _ in range(n)]}
        self.transcript_repr = rnd.randrange(R)

    def advice_ints(self, phase, challenges):
        out = {}
        for c in range(2):
            v = list(self.cols[c]); v[self.usable:] = self.blind_rows[c]; out[c] = v
        return out


class DeepGateCircuit:
    """One deep gate whose quotient program needs more than 16 live registers, so the proof runs the interpreter's local-memory
    build: q * (a_0 * a_0(1) * a_1 * a_1(1) * ... * a_{m-1}(1) - a_m), the product nested to the right (2m queries live at
    once next to q), plus a permutation over a_0 and a_1 with copies that hold.  fixed: 0 q;  advice: 0 .. m."""

    def __init__(self, k, seed=0, m=8):
        rnd = random.Random(seed)
        self.k, self.n = k, 1 << k
        n = self.n
        cs = H.ConstraintSystem(k, 1, m + 1, 0)
        queries = [H.advice(c, r) for c in range(m) for r in (0, 1)]
        prod = queries[-1]
        for e in reversed(queries[:-1]):
            prod = e * prod
        cs.gates.append(H.fixed(0) * (prod - H.advice(m)))
        cs.perm_columns = [(ADVICE, 0), (ADVICE, 1)]
        cs.finalize()
        self.cs = cs
        bf = cs.blinding_factors()
        usable = n - (bf + 1)
        self.usable = usable
        cols = [[rnd.randrange(R) for _ in range(n)] for _ in range(m + 1)]   # rows >= usable are the blinding rows
        copies = []
        for i in rnd.sample(range(usable), max(1, usable // 8)):             # a_1[i] = a_0[j]: decided before the product
            j = rnd.randrange(usable)
            cols[1][i] = cols[0][j]; copies.append(((ADVICE, 1, i), (ADVICE, 0, j)))
        q = [1 if i < usable - 1 and rnd.random() < 0.8 else 0 for i in range(n)]
        for i in range(n):
            if q[i]:
                v = 1
                for c in range(m):
                    v = v * cols[c][i] % R * cols[c][i + 1] % R
                cols[m][i] = v
        self.fixed_ints, self.copies, self.instances = [q], copies, []
        self.cols = cols
        nsets = (len(cs.perm_columns) + (cs.degree() - 2) - 1) // (cs.degree() - 2)
        self.blinds_ints = {"z": [[rnd.randrange(R) for _ in range(bf)] for _ in range(nsets)], "phi": [],
                            "random_poly": [rnd.randrange(R) for _ in range(n)]}
        self.transcript_repr = rnd.randrange(R)

    def advice_ints(self, phase, challenges):
        return {c: list(v) for c, v in enumerate(self.cols)}
