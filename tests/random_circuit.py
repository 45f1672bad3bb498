"""Seeded random constraint systems with witnesses that satisfy them by construction, for proof parity between the CUDA prover
and the oracle prover on shapes nobody wrote down (DESIGN.md §6, item 2b).

`RandomCircuit(seed, **overrides)` has the interface of tests/circuits.py's ToyCircuit (cs, fixed_ints, copies, instances,
blinds_ints, transcript_repr, advice_ints(phase, challenges)) plus `transcript`, `features()` and `describe()`.  Every draw comes
from random.Random(seed); witness values are Python ints mod r, computed by the plain integer evaluator `eval_column` below.

Column roles:
  fixed    selectors (0 on rows >= usable), free columns (random, may sit in the permutation), table columns, table selectors
  advice   free (random on all n rows, copy targets), table columns, lookup columns (filled from a table through per-column
           offsets), derived columns (each defined by exactly one gate q * (d - P) or d - P, P a random DAG)
  instance random cells, or one 0/1 column used as a lookup cofactor
Lookup group: columns a_c with offsets o_c; for every anchor row j, a_c[(j + o_c) mod n] = T_c[idx_j], so an input set that reads
a_c at o_c + s for one shift s lands on a table row at every row.  Rows where a set's cofactor is 0 give the zero tuple, which
every table holds at a usable row.  Identity gates are two differently structured, algebraically equal DAGs."""
import dataclasses
import random

import halo2_ref as H
import pyref as P
from halo2_ref import CONST, FIXED, ADVICE, INSTANCE, CHALLENGE, NEG, ADD, MUL, SCALED

R = P.R_MOD
TRANSCRIPTS = ("blake2b", "poseidon", "evm")
MAX_ROT = 9                 # |rotation| of gates and lookups, except the occasional +-(n - 1)
MAX_ROTS_PER_COLUMN = 5     # distinct rotations of one advice column: blinding factors <= 7, usable >= n - 8
MAX_DEPTH = 4               # DAG depth of a random expression: its program stays far below the interpreter's 64 registers
MAX_DEGREE = 17             # cs.degree() <= 17: extended factor E <= 16
MAX_ROT_BITS = 32767        # the interpreter keeps a rotation in 16 bits (csrc/csf.cuh)
MAX_POINTS_PER_COLUMN = 256  # SHPLONK opens one column at most at this many points (zkb_csf_validate)


@dataclasses.dataclass
class Shape:
    """Every size knob of a random circuit; the structure inside these sizes is drawn from the seed."""
    k: int
    degree: int             # degree of the top gate (cs.degree() is at least this; a lookup can raise it)
    phases: int
    n_instance: int
    n_free: int             # free advice columns (>= phases: each phase gets one)
    n_derived: int
    n_identity: int
    n_lookups: int
    max_sets: int
    max_width: int
    n_perm: int             # permutation columns (0: no permutation)
    n_cycles: int           # copy cycles
    far_rotation: bool      # gates read rotations +-(n - 1); one column is read at both r and r -+ n (r = +-1)
    transcript: str
    # ((kind, points, rotations), ...): one gate reads a free "fixed" or "advice" column at `rotations` rotation numbers that
    # make `points` distinct points mod n (rotations - points of them are r -+ n of another); the columns' point sets are
    # disjoint.  An advice column's blinding factors become its query count + 2.  Never drawn: only overrides set it.
    wide_columns: tuple = ()

    @staticmethod
    def draw(rnd):
        phases = rnd.choice([1, 1, 2, 2, 3])
        return Shape(k=rnd.randint(5, 8), degree=rnd.randint(10, MAX_DEGREE) if rnd.random() < 0.2 else rnd.randint(3, 9),
                     phases=phases, n_instance=rnd.choice([0, 1, 1, 2]), n_free=rnd.randint(phases, 4), n_derived=rnd.randint(1, 5),
                     n_identity=rnd.randint(0, 2), n_lookups=rnd.choice([0, 1, 2, 2, 3, 4]), max_sets=rnd.randint(1, 4),
                     max_width=rnd.randint(1, 3), n_perm=rnd.choice([0, 2, 3, 4, 5, 6, 8]), n_cycles=rnd.randint(1, 8),
                     far_rotation=rnd.random() < 0.2, transcript=rnd.choice(TRANSCRIPTS))


def eval_column(e, cols, challenges, n, memo=None):
    """values of expression e on all n rows (ints mod r); cols: {FIXED / ADVICE / INSTANCE: [n-length int lists]}; rotation r
    reads row (i + r) mod n.  Shared nodes are evaluated once."""
    memo = {} if memo is None else memo
    key = id(e)
    if key in memo:
        return memo[key]
    op = e.op
    if op == CONST: v = [e.a % R] * n
    elif op == CHALLENGE: v = [challenges[e.a] % R] * n
    elif op in (FIXED, ADVICE, INSTANCE):
        c, r = cols[op][e.a], e.b
        v = [c[(i + r) % n] for i in range(n)]
    elif op == NEG: v = [(R - x) % R for x in eval_column(e.a, cols, challenges, n, memo)]
    elif op == SCALED: v = [x * e.b % R for x in eval_column(e.a, cols, challenges, n, memo)]
    elif op == ADD: v = [(x + y) % R for x, y in zip(eval_column(e.a, cols, challenges, n, memo), eval_column(e.b, cols, challenges, n, memo))]
    elif op == MUL: v = [x * y % R for x, y in zip(eval_column(e.a, cols, challenges, n, memo), eval_column(e.b, cols, challenges, n, memo))]
    else: raise ValueError(op)
    memo[key] = v
    return v


def leaves(e, out=None):
    """(op, column, rotation) of every column query and ("ch", index) of every challenge in e"""
    out = set() if out is None else out
    if e.op in (FIXED, ADVICE, INSTANCE): out.add((e.op, e.a, e.b))
    elif e.op == CHALLENGE: out.add(("ch", e.a))
    elif e.op in (NEG, SCALED): leaves(e.a, out)
    elif e.op in (ADD, MUL): leaves(e.a, out); leaves(e.b, out)
    return out


def transcript_layout(cs, kind):
    """[(item name, byte length)] of a proof of the oracle ConstraintSystem cs in transcript `kind`, in the order plonk/prover.rs
    writes it (Ref.create_proof): advice commitments per phase, m, z, phi, random, h pieces, the evaluations by (column, rotation),
    then the two SHPLONK points.  Points take 64 bytes in the EVM transcript (uncompressed), 32 otherwise; scalars 32."""
    pt, sc = (64 if kind == "evm" else 32), 32
    d = cs.degree()
    chunk = d - 2
    nsets = (len(cs.perm_columns) + chunk - 1) // chunk
    out = []
    for phase in range(cs.num_phases()):
        out += [(f"advice {c} (phase {phase})", pt) for c in range(cs.num_advice) if cs.advice_phase[c] == phase]
    out += [(f"m {l}", pt) for l in range(len(cs.lookups))]
    out += [(f"z {i}", pt) for i in range(nsets)]
    out += [(f"phi {l}", pt) for l in range(len(cs.lookups))]
    out += [("random", pt)]
    out += [(f"h piece {i}", pt) for i in range(d - 1)]
    out += [(f"advice {c} at rotation {r}", sc) for c, r in cs.advice_queries]
    out += [(f"fixed {c} at rotation {r}", sc) for c, r in cs.fixed_queries]
    out += [("random eval", sc)]
    out += [(f"sigma {i} eval", sc) for i in range(len(cs.perm_columns))]
    for i in range(nsets):
        out += [(f"z {i} at x", sc), (f"z {i} at wx", sc)] + ([(f"z {i} at x_last", sc)] if i != nsets - 1 else [])
    for l in range(len(cs.lookups)):
        out += [(f"phi {l} at x", sc), (f"phi {l} at wx", sc), (f"m {l} at x", sc)]
    out += [("shplonk h", pt), ("shplonk q", pt)]
    return out


def item_at(layout, offset):
    """name of the layout item that holds byte `offset` (None past the end)"""
    pos = 0
    for name, size in layout:
        if offset < pos + size:
            return name
        pos += size
    return None


class _Group:
    """a lookup's columns and table values; several lookups may share one"""
    def __init__(self):
        self.kind = self.form = None
        self.base = []          # table base columns: (FIXED or ADVICE, index), rotation 0
        self.cols = []          # lookup advice columns a_c
        self.offsets = []
        self.qt = None          # table selector column of form "q"
        self.ch = None          # challenge index of form "ch"
        self.source = None      # group whose lookup columns the table reads (kind "other")
        self.twin = False       # table (t_0, t_0, ...)
        self.shifts = []
        self.zero_row = None    # a usable row where every base column is 0
        self.all_zero_row = None   # a usable row where every lookup column is 0


class RandomCircuit:
    def __init__(self, seed, **overrides):
        self.seed = seed
        rnd = self.rnd = random.Random(seed)
        shape = Shape.draw(rnd)
        self.shape = sh = dataclasses.replace(shape, **overrides)
        self.k, self.n = sh.k, 1 << sh.k
        n = self.n
        if sh.far_rotation and n - 1 > MAX_ROT_BITS:
            raise ValueError(f"far_rotation reads rotations +-(n - 1) = +-{n - 1} at k = {sh.k}: the interpreter keeps a rotation "
                             f"in 16 bits (|rotation| <= {MAX_ROT_BITS}), so far_rotation needs k <= 15")
        self.transcript = sh.transcript
        self.fixed_role, self.adv_role, self.adv_phase, self._rots = [], [], [], []
        self.challenge_phase = [p for p in range(sh.phases - 1) for _ in range(rnd.randint(1, 2))]
        self.sel_instance = sh.n_instance > 0 and rnd.random() < 0.5          # instance 0 holds 0 / 1 cells
        self.selectors = [self._fixed("sel") for _ in range(rnd.randint(1, 3))]
        self.free_fixed = [self._fixed("free") for _ in range(rnd.randint(1, 2))]
        self.free = [self._advice("free", p if p < sh.phases else rnd.randrange(sh.phases)) for p in range(sh.n_free)]
        self.groups, self.lookup_groups, self.set_info = [], [], []
        lookups = [self._lookup(l) for l in range(sh.n_lookups)]
        self.derived = []       # (advice column, gate, selector column or None, P)
        self.identities = []
        gates = self._gates()
        cs = H.ConstraintSystem(self.k, len(self.fixed_role), len(self.adv_role), sh.n_instance, list(self.adv_phase), list(self.challenge_phase))
        cs.gates, cs.lookups = gates, lookups
        pool = [(ADVICE, c) for c in self.free] * 2 + [(FIXED, c) for c in self.free_fixed] + [(INSTANCE, i) for i in range(sh.n_instance)] \
            + [(ADVICE, c) for c in range(len(self.adv_role)) if c not in self.free and self.adv_role[c] != "wide"]
        perm = []
        for col in rnd.sample(pool, len(pool)):
            if len(perm) < sh.n_perm and col not in perm:
                perm.append(col)
        cs.perm_columns = perm
        cs.finalize()
        self.cs = cs
        self.degree = cs.degree()
        assert 3 <= self.degree <= MAX_DEGREE, self.degree
        self.bf = bf = cs.blinding_factors()
        self.usable = usable = n - (bf + 1)
        assert bf <= max([MAX_ROTS_PER_COLUMN] + [rots for kind, _, rots in sh.wide_columns if kind == "advice"]) + 2
        self._values()
        chunk = self.degree - 2
        nsets = (len(perm) + chunk - 1) // chunk
        self.blinds_ints = {"z": [[rnd.randrange(R) for _ in range(bf)] for _ in range(nsets)],
                            "phi": [[rnd.randrange(R) for _ in range(bf)] for _ in cs.lookups],
                            "random_poly": [rnd.randrange(R) for _ in range(n)]}
        self.transcript_repr = rnd.randrange(R)

    # ------------------------------------------------------------------------------------------------ structure
    def _fixed(self, role):
        self.fixed_role.append(role)
        return len(self.fixed_role) - 1

    def _advice(self, role, phase=None):
        self.adv_role.append(role)
        self.adv_phase.append(self.rnd.randrange(self.shape.phases) if phase is None else phase)
        self._rots.append({0})
        return len(self.adv_role) - 1

    def _value(self):
        """a random cell value: small (so that tables repeat), an edge, or uniform"""
        t = self.rnd.random()
        return self.rnd.randrange(6) if t < 0.4 else (R - 1 - self.rnd.randrange(2)) if t < 0.5 else self.rnd.randrange(R)

    def _const(self):
        return self.rnd.choice([0, 1, R - 1, 2, self.rnd.randrange(R)])

    def _rot_ok(self, col, rot):
        return rot in self._rots[col] or len(self._rots[col]) < MAX_ROTS_PER_COLUMN

    def _rotation(self, kind, col):
        rnd, n = self.rnd, self.n
        if rnd.random() < 0.4:
            r = 0
        elif self.shape.far_rotation and rnd.random() < 0.15:
            r = rnd.choice([n - 1, -(n - 1)])
        else:
            r = rnd.randint(-MAX_ROT, MAX_ROT)
        if kind == ADVICE:
            if not self._rot_ok(col, r):
                r = rnd.choice(sorted(self._rots[col]))
            self._rots[col].add(r)
        return r

    def _lookup(self, l):
        rnd, sh = self.rnd, self.shape
        if self.groups and rnd.random() < 0.2:
            g = rnd.choice(self.groups)                      # the same column tuple in a second lookup
            shared = True
        else:
            shared = False
            g = _Group()
            kinds = ["fixed", "fixed", "advice", "advice"] + (["other", "other"] if self.groups else [])
            g.kind = rnd.choice(kinds)
            g.form = rnd.choice(["plain", "plain", "q"] + (["ch", "ch"] if self.challenge_phase else []))
            W = rnd.randint(1, sh.max_width)
            twin = W >= 2 and rnd.random() < 0.3             # table (t_0, t_0, ...): a set may read one column twice
            if g.kind == "other":
                g.source = rnd.choice(self.groups)
                src = g.source.cols
                W = min(W, len(src))
                base = [(ADVICE, c) for c in rnd.sample(src, W)]
            elif g.kind == "fixed":
                base = [(FIXED, self._fixed("table")) for _ in range(W)]
            else:
                base = [(ADVICE, self._advice("table")) for _ in range(W)]
            if twin and W >= 2:
                base[1] = base[0]
            g.base = base
            g.twin = W >= 2 and base[1] == base[0]
            if g.form == "q":
                g.qt = self._fixed("qt")
            if g.form == "ch":
                g.ch = rnd.randrange(len(self.challenge_phase))
            g.cols = [self._advice("lk") for _ in range(W)]
            g.offsets = [0] * W if rnd.random() < 0.5 else [rnd.randint(-2, 2) for _ in range(W)]
            self.groups.append(g)
        W = len(g.cols)

        def table_entry(t, c):
            e = H.Expr(t, c, 0)
            if g.form == "q":
                return H.fixed(g.qt) * e if rnd.random() < 0.5 else e * H.fixed(g.qt)
            if g.form == "ch":
                return H.challenge(g.ch) * e if rnd.random() < 0.5 else e * H.challenge(g.ch)
            return e
        table = [table_entry(t, c) for t, c in g.base]
        sets = []
        for j in range(rnd.randint(1, sh.max_sets)):
            s = 0 if rnd.random() < 0.3 else rnd.randint(-(MAX_ROT - 2), MAX_ROT - 2)
            if not all(self._rot_ok(a, o + s) for a, o in zip(g.cols, g.offsets)):
                s = rnd.choice(g.shifts) if g.shifts else 0
            if s not in g.shifts:
                g.shifts.append(s)
            for a, o in zip(g.cols, g.offsets):
                self._rots[a].add(o + s)
            q = H.fixed(rnd.choice(self.selectors))
            if g.form == "ch":
                chx = H.challenge(g.ch)
                cof = rnd.choice([chx, q * chx, chx * q])
            else:
                opts = [None, None, q, q]
                if self.sel_instance:
                    opts += [H.instance(0, 0), q * H.instance(0, 0)]
                cof = rnd.choice(opts)
            side = rnd.choice(["left", "left", "right", "mixed"])
            one_node = rnd.random() < 0.5                  # every entry's cofactor is one shared node, or a copy per entry
            entries, info, rights = [], [], []
            for c in range(W):
                col, rot = g.cols[c], g.offsets[c] + s
                if g.twin and c == 1 and rnd.random() < 0.5:
                    col, rot = g.cols[0], g.offsets[0] + s  # the same column twice in one set
                a = H.advice(col, rot)
                info.append((col, rot))
                if cof is None:
                    entries.append(a)
                    continue
                S = cof if one_node else _copy(cof)
                right = side == "right" or (side == "mixed" and rnd.random() < 0.5)
                rights.append(right)
                entries.append(a * S if right else S * a)
            sets.append(entries)
            self.set_info.append(dict(lookup=l, set=j, entries=info, cof=cof, right=any(rights)))
        self.lookup_groups.append((g, shared))
        return H.Lookup(sets, table)

    def _leaf(self, budget, phase, upto):
        """a column query (degree 1) or, with no degree left or by chance, a constant or a challenge readable in `phase`"""
        rnd = self.rnd
        chs = [i for i, p in enumerate(self.challenge_phase) if p < phase]
        if budget == 0 or rnd.random() < 0.15:
            if chs and rnd.random() < 0.5:
                return H.challenge(rnd.choice(chs))
            return H.const(self._const())
        advs = [c for c, role in enumerate(self.adv_role) if role != "derived"] + \
               [d for d, _, _, _ in self.derived[:upto] if self.adv_phase[d] <= phase]
        t = rnd.random()
        if t < 0.6 or (t >= 0.85 and not self.shape.n_instance):
            col = rnd.choice(advs)
            return H.advice(col, self._rotation(ADVICE, col))
        if t < 0.85:
            col = rnd.randrange(len(self.fixed_role))
            return H.fixed(col, self._rotation(FIXED, col))
        col = rnd.randrange(self.shape.n_instance)
        return H.instance(col, self._rotation(INSTANCE, col))

    def _dag(self, budget, depth, phase, upto, shared):
        """a random expression of degree <= budget; sub-expressions in `shared` may be reused"""
        rnd = self.rnd
        if depth >= MAX_DEPTH or rnd.random() < 0.25:
            return self._leaf(budget, phase, upto)
        if shared and rnd.random() < 0.2:
            cands = [e for e in shared if e.degree() <= budget]
            if cands:
                return rnd.choice(cands)
        op = rnd.choices(["add", "sub", "mul", "neg", "scaled"], [3, 2, 4, 1, 1])[0]
        sub = lambda b: self._dag(b, depth + 1, phase, upto, shared)
        if op == "add": e = sub(budget) + sub(budget)
        elif op == "sub": e = sub(budget) - sub(budget)
        elif op == "mul":
            b1 = rnd.randint(0, budget)
            e = sub(b1) * sub(budget - b1)
        elif op == "neg": e = -sub(budget)
        else: e = H.scaled(sub(budget), self._const())
        shared.append(e)
        return e

    def _product(self, m, phase, upto):
        """a product of m column queries, nested left, right or balanced"""
        fs = []
        while len(fs) < m:
            f = self._leaf(1, phase, upto)
            if f.degree() == 1:
                fs.append(f)
        how = self.rnd.choice(["left", "right", "balanced"])

        def nest(xs):
            if len(xs) == 1: return xs[0]
            if how == "left": return nest(xs[:-1]) * xs[-1]
            if how == "right": return xs[0] * nest(xs[1:])
            return nest(xs[: len(xs) // 2]) * nest(xs[len(xs) // 2:])
        return nest(fs)

    def _gates(self):
        rnd, sh = self.rnd, self.shape
        D = sh.degree
        top = rnd.randrange(sh.n_derived)
        gates = []
        if sh.far_rotation:                                    # one free column read at r and r -+ n: two queries, one opening point
            col = rnd.choice(self.free)
            r = rnd.choice([-1, 1])
            wrapped = r - self.n if r > 0 else r + self.n
            self._rots[col] |= {r, wrapped}
            sel = rnd.choice(self.selectors) if rnd.random() < 0.5 else None
            body = (H.advice(col, r) - H.advice(col, wrapped)) * self._leaf(1, sh.phases, 0)
            self.identities.append(len(gates))
            gates.append(H.fixed(sel) * body if sel is not None else body)
        for i in range(sh.n_derived):
            phase = rnd.randrange(sh.phases)
            d = self._advice("derived", phase)
            sel = rnd.choice(self.selectors) if rnd.random() < 0.6 else None
            budget = D - (sel is not None)
            if i == top:
                p = self._product(budget, phase, i)
                if rnd.random() < 0.5:
                    p = p + self._dag(min(budget, 3), 1, phase, i, [])
            else:
                p = self._dag(rnd.randint(1, min(budget, 4)), 0, phase, i, [])
            if sel is None:                                    # d = P on every row: a free column keeps d from being all zero
                col = rnd.choice(self.free)
                p = p + H.advice(col, self._rotation(ADVICE, col)) if rnd.random() < 0.5 else H.advice(col, self._rotation(ADVICE, col)) + p
            body = H.advice(d) - p
            gate = H.fixed(sel) * body if sel is not None else body
            self.derived.append((d, len(gates), sel, p))
            gates.append(gate)
        for _ in range(sh.n_identity):
            sel = rnd.choice(self.selectors) if rnd.random() < 0.5 else None
            budget = rnd.randint(2, max(2, D - (sel is not None)))
            if rnd.random() < 0.4:                             # (a + b)^2 - (a^2 + 2ab + b^2)
                a, b = self._leaf(1, sh.phases, len(self.derived)), self._leaf(1, sh.phases, len(self.derived))
                body = (a + b) * (a + b) - (a * a + H.scaled(a * b, 2) + b * b)
            else:
                x = self._dag(budget, 0, sh.phases, len(self.derived), [])
                body = x - _rewrite(x, rnd)
            self.identities.append(len(gates))
            gates.append(H.fixed(sel) * body if sel is not None else body)
        used = set()
        for kind, points, rotations in sh.wide_columns:
            gates.append(self._wide_gate(kind, points, rotations, used, len(gates)))
        order = list(range(len(gates)))
        rnd.shuffle(order)
        where = {g: i for i, g in enumerate(order)}
        self.derived = [(d, where[g], sel, p) for d, g, sel, p in self.derived]
        self.identities = [where[g] for g in self.identities]
        return [gates[g] for g in order]

    def _wide_gate(self, kind, points, rotations, used, gate):
        """q * (d - sum_i c_i col(r_i)) over a fresh column read at `rotations` rotation numbers that make `points` points mod n,
        none of them in `used`; d is a derived column"""
        rnd, n = self.rnd, self.n
        assert kind in ("fixed", "advice") and 1 <= points <= rotations < 2 * points, (kind, points, rotations)
        rots = rnd.sample([r for r in range(-(n // 2) + 1, n // 2 + 1) if r % n not in used], points)
        used.update(r % n for r in rots)
        rots += [r - n if r > 0 else r + n for r in rnd.sample([r for r in rots if r], rotations - points)]
        assert all(abs(r) <= MAX_ROT_BITS for r in rots)
        phase = rnd.randrange(self.shape.phases)
        if kind == "advice":
            col = self._advice("wide", phase)
            self._rots[col] = set(rots)
            read = H.advice
        else:
            col = self._fixed("wide")
            read = H.fixed

        def total(xs):
            return xs[0] if len(xs) == 1 else total(xs[: len(xs) // 2]) + total(xs[len(xs) // 2:])
        p = total([H.scaled(read(col, r), rnd.randrange(1, R)) for r in rots])
        d = self._advice("derived", phase)
        sel = rnd.choice(self.selectors)
        self.derived.append((d, gate, sel, p))
        return H.fixed(sel) * (H.advice(d) - p)

    # ------------------------------------------------------------------------------------------------ values
    def _values(self):
        rnd, n, usable, sh = self.rnd, self.n, self.usable, self.shape
        fixed = [[0] * n for _ in self.fixed_role]
        for c, role in enumerate(self.fixed_role):
            if role == "sel":
                fixed[c] = [int(rnd.random() < 0.6) if i < usable else 0 for i in range(n)]
            elif role == "qt":
                fixed[c] = [int(rnd.random() < 0.7) for i in range(n)]
                fixed[c][rnd.randrange(usable)] = 0           # the zero tuple is a table row
            elif role in ("free", "wide"):
                fixed[c] = [self._value() for _ in range(n)]
        adv = [None] * len(self.adv_role)
        for c, role in enumerate(self.adv_role):
            if role in ("free", "table", "wide"):
                adv[c] = [self._value() for _ in range(n)]
        self.instances = []
        for i in range(sh.n_instance):
            L = rnd.randint(1, min(12, usable))
            self.instances.append([int(rnd.random() < 0.6) for _ in range(L)] if i == 0 and self.sel_instance else [self._value() for _ in range(L)])
        cols = {FIXED: fixed, ADVICE: adv}
        for g in self.groups:
            self._fill_group(g, cols)
        self._copies(fixed, adv)
        self.fixed_ints = fixed
        self.cols = adv
        self._dinit = {d: [rnd.randrange(R) for _ in range(n)] for d, _, _, _ in self.derived}

    def _fill_group(self, g, cols):
        rnd, n, usable = self.rnd, self.n, self.usable
        W = len(g.cols)
        if g.kind == "other":
            g.zero_row = g.source.all_zero_row
        else:
            g.zero_row = rnd.randrange(usable)
            done = set()
            for t, c in g.base:
                if (t, c) in done:
                    continue
                done.add((t, c))
                v = [self._value() for _ in range(n)]
                for i in range(usable):
                    if rnd.random() < 0.2 and i:
                        v[i] = v[rnd.randrange(i)]           # duplicate table rows
                cols[t][c] = v
            for i in range(usable):                           # whole duplicate tuples
                if rnd.random() < 0.1 and i:
                    j = rnd.randrange(i)
                    for t, c in done:
                        cols[t][c][i] = cols[t][c][j]
            for t, c in done:
                cols[t][c][g.zero_row] = 0
        T = [cols[t][c] for t, c in g.base]
        qt = cols[FIXED][g.qt] if g.qt is not None else None
        valid = [i for i in range(usable) if qt is None or qt[i] or not any(col[i] for col in T)]
        idx = [rnd.choice(valid) for _ in range(n)]
        i0 = rnd.randrange(usable)                            # a usable row where every lookup column is 0: the zero row of tables reading them
        for o in g.offsets:
            idx[(i0 - o) % n] = g.zero_row
        g.all_zero_row = i0
        for a, o, col in zip(g.cols, g.offsets, T):
            v = [0] * n
            for j in range(n):
                v[(j + o) % n] = col[idx[j]]
            cols[ADVICE][a] = v

    def _copies(self, fixed, adv):
        rnd, usable, cs = self.rnd, self.usable, self.cs
        cells = []
        for (t, c) in cs.perm_columns:
            if t == ADVICE and self.adv_role[c] == "free":
                cells += [(ADVICE, c, r) for r in range(usable)]
            elif t == FIXED and self.fixed_role[c] == "free":
                cells += [(FIXED, c, r) for r in range(usable)]
            elif t == INSTANCE and not (c == 0 and self.sel_instance):
                cells += [(INSTANCE, c, r) for r in range(len(self.instances[c]))]
        store = {FIXED: fixed, ADVICE: adv, INSTANCE: self.instances}
        copies, used = [], set()
        for _ in range(self.shape.n_cycles if len(cells) >= 2 else 0):
            cyc = [x for x in rnd.sample(cells, min(len(cells), rnd.randint(2, 4))) if x not in used]
            if len(cyc) < 2:
                continue
            used.update(cyc)
            v = store[cyc[0][0]][cyc[0][1]][cyc[0][2]]
            for t, c, r in cyc[1:]:
                store[t][c][r] = v
            pairs = []
            for i in range(1, len(cyc)):
                a, b = (cyc[i - 1], cyc[i]) if rnd.random() < 0.5 else (cyc[0], cyc[i])
                pairs.append((a, b) if rnd.random() < 0.5 else (b, a))
            if rnd.random() < 0.2:
                pairs.append((cyc[-1], cyc[0]))                # a copy inside one cycle: the assembly skips it
            copies += pairs
        rnd.shuffle(copies)
        self.copies = copies

    # ------------------------------------------------------------------------------------------------ witness
    def columns(self, challenges):
        """every advice column (derived ones computed from `challenges`, {index: int}) as n-length int lists"""
        n = self.n
        adv = list(self.cols)
        inst = [list(v) + [0] * (n - len(v)) for v in self.instances]
        cols = {FIXED: self.fixed_ints, ADVICE: adv, INSTANCE: inst}
        for d, _, sel, p in self.derived:
            needed = [i for i, ph in enumerate(self.challenge_phase) if ph < self.adv_phase[d]]
            if any(i not in challenges for i in needed):
                continue
            pv = eval_column(p, cols, challenges, n)
            if sel is None:
                adv[d] = pv
            else:
                q = self.fixed_ints[sel]
                adv[d] = [pv[i] if q[i] else self._dinit[d][i] for i in range(n)]
        return adv

    def advice_ints(self, phase, challenges):
        chs = {i: int(v) % R for i, v in challenges.items() if self.challenge_phase[i] < phase}
        adv = self.columns(chs)
        return {c: list(adv[c]) for c in range(len(adv)) if self.adv_phase[c] == phase}

    # ------------------------------------------------------------------------------------------------ reports
    def features(self):
        cs, n = self.cs, self.n
        f = dict.fromkeys(["E16", "advice_table", "table_expression", "table_challenge", "input_challenge", "cofactor_right",
                           "same_column_twice", "instance_in_set", "shared_tuple", "table_read_column", "combinable_set",
                           "unselected_gate", "identity_gate", "three_phases", "instance_in_perm", "no_permutation", "no_lookup",
                           "perm_chunks", "rotation_beyond_blinding", "far_rotation", "rotations_equal_mod_n", "copies"], 0)
        f["E16"] = int(self.degree >= 10)
        table_read = set()
        for g, shared in self.lookup_groups:
            f["shared_tuple"] += shared
            if shared:
                continue
            f["advice_table"] += g.base[0][0] == ADVICE
            f["table_expression"] += g.form != "plain"
            f["table_challenge"] += g.form == "ch"
        for lk in cs.lookups:
            for e in lk.table:
                table_read |= {c for t, c, _ in (x for x in leaves(e) if x[0] != "ch") if t == ADVICE}
        for s in self.set_info:
            lv = leaves(s["cof"]) if s["cof"] is not None else set()
            f["input_challenge"] += any(x[0] == "ch" for x in lv)
            f["instance_in_set"] += any(x[0] == INSTANCE for x in lv)
            f["cofactor_right"] += s["right"]
            f["same_column_twice"] += len({c for c, _ in s["entries"]}) < len(s["entries"])
            f["table_read_column"] += any(c in table_read for c, _ in s["entries"])
            f["combinable_set"] += len(s["entries"]) >= 2 and len({r for _, r in s["entries"]}) == 1
        f["unselected_gate"] = sum(sel is None for _, _, sel, _ in self.derived)
        f["identity_gate"] = len(self.identities)
        f["three_phases"] = int(cs.num_phases() == 3)
        f["instance_in_perm"] = int(any(t == INSTANCE for t, _ in cs.perm_columns))
        f["no_permutation"] = int(not cs.perm_columns)
        f["no_lookup"] = int(not cs.lookups)
        f["perm_chunks"] = int(len(cs.perm_columns) > self.degree - 2)
        rots = [r for _, r in cs.advice_queries] + [r for _, r in cs.fixed_queries] + [r for _, r in cs.instance_queries]
        f["rotation_beyond_blinding"] = int(any(self.bf < abs(r) < n - 1 for r in rots))
        f["far_rotation"] = int(any(abs(r) == n - 1 for r in rots))
        f["rotations_equal_mod_n"] = int(any((c, r + n) in cs.advice_queries or (c, r - n) in cs.advice_queries for c, r in cs.advice_queries))
        f["copies"] = len(self.copies)
        return f

    def describe(self):
        cs = self.cs
        chunk = self.degree - 2
        lks = " ".join(f"{len(lk.inputs)}x{len(lk.table)}{g.kind[0]}{g.form[0]}{'s' if sh else ''}"
                       for lk, (g, sh) in zip(cs.lookups, self.lookup_groups))
        return (f"seed {self.seed}: k={self.k} d={self.degree} E={H.Domain(self.k, self.degree).E} phases={cs.num_phases()} "
                f"fixed={cs.num_fixed} advice={cs.num_advice} instance={cs.num_instance} gates={len(cs.gates)} "
                f"(derived {len(self.derived)}, unselected {sum(s is None for _, _, s, _ in self.derived)}, identity {len(self.identities)}) "
                f"lookups=[{lks}] perm={len(cs.perm_columns)} cols/{-(-len(cs.perm_columns) // chunk)} sets copies={len(self.copies)} "
                f"bf={self.bf} transcript={self.transcript}" + (f" wide={list(self.shape.wide_columns)}" if self.shape.wide_columns else ""))


def _copy(e):
    if e.op in (NEG, SCALED): return H.Expr(e.op, _copy(e.a), e.b)
    if e.op in (ADD, MUL): return H.Expr(e.op, _copy(e.a), _copy(e.b))
    return H.Expr(e.op, e.a, e.b)


def _rewrite(e, rnd):
    """an expression equal to e as a polynomial, built differently: operands swapped, products distributed over sums, NEG as a
    scaling by r - 1, SCALED as a product with a constant, columns times 1 or plus 0"""
    op = e.op
    rw = lambda x: _rewrite(x, rnd)
    if op in (CONST, CHALLENGE, FIXED, ADVICE, INSTANCE):
        t = rnd.random()
        leaf = H.Expr(op, e.a, e.b)
        return leaf * H.const(1) if t < 0.15 else leaf + H.const(0) if t < 0.25 else leaf
    if op == NEG:
        return H.scaled(rw(e.a), R - 1) if rnd.random() < 0.5 else -rw(e.a)
    if op == SCALED:
        return H.const(e.b) * rw(e.a) if rnd.random() < 0.5 else H.scaled(rw(e.a), e.b)
    if op == ADD:
        return rw(e.b) + rw(e.a) if rnd.random() < 0.5 else rw(e.a) + rw(e.b)
    if op == MUL:
        if e.b.op == ADD and rnd.random() < 0.4:
            return rw(e.a) * rw(e.b.a) + rw(e.a) * rw(e.b.b)
        if e.a.op == ADD and rnd.random() < 0.4:
            return rw(e.a.a) * rw(e.b) + rw(e.a.b) * rw(e.b)
        return rw(e.b) * rw(e.a) if rnd.random() < 0.5 else rw(e.a) * rw(e.b)
    raise ValueError(op)
