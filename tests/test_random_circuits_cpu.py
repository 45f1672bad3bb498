"""The random circuit corpus of tests/random_circuit.py on the CPU: every seed's witness satisfies its constraint system (and a changed
cell does not), the oracle proves and verifies a sample in every transcript, seeds are deterministic, proof layouts match the
oracle's bytes, and the seeds that tests/test_gpu_random_circuits.py proves cover every shape feature a stated number of times."""
import collections

import numpy as np
import pytest

import halo2_ref as H
import keccak_ref as K
import pyref as P
from random_circuit import RandomCircuit, TRANSCRIPTS, transcript_layout, eval_column
from test_gpu_prover import to_product_cs
from witness_ref import check_witness, perm_copies, circuit_columns

R = P.R_MOD
CPU_SEEDS = range(200)
GPU_SEEDS = range(96)       # the seeds tests/test_gpu_random_circuits.py proves on the device

# each feature at least this many times across GPU_SEEDS (counts per seed: circuits, lookups or input sets)
COVERAGE = {
    "E16": 12,                   # cs.degree() >= 10: extended factor 16, >= 9 h pieces
    "advice_table": 20,          # a table over advice columns
    "table_expression": 20,      # q * t or ch * t
    "table_challenge": 8,
    "input_challenge": 15,       # an input set whose cofactor reads a challenge
    "cofactor_right": 15,        # a(r) * S
    "same_column_twice": 5,
    "instance_in_set": 8,
    "shared_tuple": 8,           # one column tuple in two lookups
    "table_read_column": 10,     # an input set whose column a table reads
    "combinable_set": 15,        # width >= 2 at one rotation
    "unselected_gate": 40,
    "identity_gate": 40,
    "three_phases": 10,
    "instance_in_perm": 10,
    "no_permutation": 5,
    "no_lookup": 5,
    "perm_chunks": 10,           # more permutation columns than d - 2
    "rotation_beyond_blinding": 40,
    "far_rotation": 8,           # +-(n - 1)
    "rotations_equal_mod_n": 8,  # one column read at r and r -+ n: one opening point
}


def challenges_for(tc):
    rnd = np.random.default_rng(tc.seed)
    return [int(x) for x in rnd.integers(1, 1 << 62, len(tc.cs.challenge_phase))]


def oracle_check(tc, cols=None):
    ref = H.Ref(tc.cs, 0, build_srs=False)
    ch = challenges_for(tc)
    cols = cols if cols is not None else circuit_columns(tc, ref.F, ch)
    return check_witness(ref, tc.cs, cols, ch, perm_copies(tc.cs, tc.copies), tc.usable)


def oracle_prove(tc, kind):
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": rp}
    synth = lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, ch).items()}
    writer = {"blake2b": None, "poseidon": H.Ref.PoseidonTranscript(ref), "evm": K.EvmTranscript(ref)}[kind]
    proof, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, synth, blinds, transcript=writer)
    reader = {"blake2b": None, "poseidon": H.Ref.PoseidonReader(proof), "evm": K.EvmTranscript(proof=proof)}[kind]
    return ref, pkr, proof, ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof, reader=reader)


def test_every_seed_is_satisfied():
    bad = []
    for seed in CPU_SEEDS:
        tc = RandomCircuit(seed)
        counts, recs = oracle_check(tc)
        if recs:
            bad.append(f"{tc.describe()}: {recs[:4]}")
    assert not bad, "\n".join(bad)


def test_registers_and_rotations_stay_inside_the_limits():
    """every seed's gates compile into one program of at most 64 registers; rotations fit 16 bits; instances and tables lie in the
    usable rows"""
    from zkb200 import plonk as Z
    for seed in CPU_SEEDS:
        tc = RandomCircuit(seed)
        zcs = to_product_cs(tc.cs, tc.bf, tc.degree)
        _, nregs = Z.expr_program(zcs, mode=1, challenges=[[1, 0, 0, 0]] * len(tc.cs.challenge_phase), y=[5, 0, 0, 0], scale=[1, 0, 0, 0])
        assert nregs <= 64, tc.describe()
        Z.validate_csf(zcs.to_csf())
        assert all(len(v) <= tc.usable for v in tc.instances)
        rots = [r for q in (tc.cs.advice_queries, tc.cs.fixed_queries, tc.cs.instance_queries) for _, r in q]
        assert all(abs(r) < min(tc.n, 1 << 15) for r in rots)


@pytest.mark.parametrize("seed", [0, 2, 3, 5, 6, 7, 9, 12])
def test_oracle_proves_and_verifies(seed):
    tc = RandomCircuit(seed)
    _, _, proof, ok = oracle_prove(tc, tc.transcript)
    assert ok, tc.describe()
    assert len(proof) == sum(size for _, size in transcript_layout(tc.cs, tc.transcript))


def test_sample_covers_every_transcript():
    kinds = {RandomCircuit(s).transcript for s in [0, 2, 3, 5, 6, 7, 9, 12]}
    assert kinds == set(TRANSCRIPTS)


@pytest.mark.parametrize("kind", TRANSCRIPTS)
def test_layout_length_in_every_transcript(kind):
    """the same circuit proved in each transcript kind: the layout's total is the proof's length"""
    tc = RandomCircuit(11)
    _, _, proof, ok = oracle_prove(tc, kind)
    assert ok
    layout = transcript_layout(tc.cs, kind)
    assert len(proof) == sum(size for _, size in layout)
    assert layout[-1] == ("shplonk q", 64 if kind == "evm" else 32)


def test_changed_cells_are_reported():
    """one derived cell at a row where its gate is on, then one lookup column cell at a row where a set reads it with a nonzero
    cofactor: the reference check reports the defining gate, then that input set"""
    tried = 0
    for seed in range(40):
        tc = RandomCircuit(seed)
        ref = H.Ref(tc.cs, 0, build_srs=False)
        F = ref.F
        ch = challenges_for(tc)
        cols = circuit_columns(tc, F, ch)
        d, g, sel, _ = tc.derived[0]
        rows = [i for i in range(tc.usable) if sel is None or tc.fixed_ints[sel][i]]
        if not rows:
            continue
        r = rows[len(rows) // 2]
        broken = {t: list(v) for t, v in cols.items()}
        broken[H.ADVICE][d] = cols[H.ADVICE][d].copy()
        broken[H.ADVICE][d][r] = F.arr([(F.ints(cols[H.ADVICE][d][r:r + 1])[0] + 1) % R])[0]
        counts, recs = oracle_check(tc, broken)
        assert (0, g, 0, r) in [(k, i, 0, row) for k, i, _, row in recs], tc.describe()
        if tc.set_info:
            s = tc.set_info[0]
            n = tc.n
            ints = {H.FIXED: tc.fixed_ints, H.ADVICE: tc.columns({i: c for i, c in enumerate(ch)}),
                    H.INSTANCE: [list(v) + [0] * (n - len(v)) for v in tc.instances]}
            cof = eval_column(s["cof"], ints, dict(enumerate(ch)), n) if s["cof"] is not None else [1] * n
            row = next((i for i in range(tc.usable) if cof[i]), None)
            if row is not None:
                col, rot = s["entries"][0]
                broken = {t: list(v) for t, v in cols.items()}
                broken[H.ADVICE][col] = cols[H.ADVICE][col].copy()
                broken[H.ADVICE][col][(row + rot) % n] = F.arr([0xBAD0BAD0BAD])[0]
                counts, recs = oracle_check(tc, broken)
                assert (1, s["lookup"], s["set"], row) in recs, tc.describe()
                tried += 1
    assert tried >= 10


def test_same_seed_same_bytes():
    for seed in (0, 1, 6, 33):
        a, b = RandomCircuit(seed), RandomCircuit(seed)
        assert (to_product_cs(a.cs, a.bf, a.degree).to_csf() == to_product_cs(b.cs, b.bf, b.degree).to_csf()).all()
        ch = challenges_for(a)
        for ph in range(a.cs.num_phases()):
            assert a.advice_ints(ph, dict(enumerate(ch))) == b.advice_ints(ph, dict(enumerate(ch)))
        assert (a.fixed_ints, a.copies, a.instances, a.blinds_ints, a.transcript_repr) == (b.fixed_ints, b.copies, b.instances, b.blinds_ints, b.transcript_repr)


def test_overrides_pin_a_shape():
    tc = RandomCircuit(5, k=6, degree=12, n_lookups=3, phases=3, transcript="evm")
    assert (tc.k, tc.transcript, tc.cs.num_phases(), len(tc.cs.lookups)) == (6, "evm", 3, 3) and tc.degree >= 12
    counts, recs = oracle_check(tc)
    assert not recs


def test_coverage_of_the_gpu_seeds():
    total = collections.Counter()
    for seed in GPU_SEEDS:
        total.update(RandomCircuit(seed).features())
    short = {f: (total[f], want) for f, want in COVERAGE.items() if total[f] < want}
    assert not short, f"features below their stated count (have, want): {short}"
    degrees = [RandomCircuit(s).degree for s in GPU_SEEDS]
    assert sum(d > 9 for d in degrees) >= len(degrees) // 10 and max(degrees) <= 17 and min(degrees) >= 3
    assert {RandomCircuit(s).transcript for s in GPU_SEEDS} == set(TRANSCRIPTS)
