"""GPU parity on random circuits at the sizes real circuits have, and on SHPLONK rotation sets up to the prover's 256-point limit.

The corpus of tests/test_gpu_random_circuits.py draws k = 5 ... 8, where every size-n transform is one NTT pass and every scan
and carry of csrc/poly.cu (2048 elements per block) fits one block.  LARGE_CASES pins k = 12 ... 17 through overrides, so a
byte-compared proof runs the 2- and 3-pass NTT plans (the 3-pass extended iNTT at k = 17 with E = 16: 2^21 points), the
permutation products, phi's prefix sum, eval_polynomial and kate_division across blocks, the MSM configurations of 2^12 ... 2^17
points through the SRS handle, rotation +-32767 at k = 15, and device keygen's sigma columns at large n.  Each case is proved once
by the oracle; prove_and_compare checks the device proof, the oracle verifier, device keygen, the witness check, and the proof
with columns uploaded ahead and without the coset cache against that one proof; the k = 12 ... 14 cases are also proved on 2 and
3 in-process ranks.

ROTATION_CASES read one column at up to 256 distinct points (one SHPLONK rotation set of that size); a column at 257 points is
refused by every pk constructor before any proof work, and the context proves the next circuit."""
import pytest

from random_circuit import RandomCircuit
from test_gpu_random_circuits import prove_and_compare
from test_gpu_ranks_one_device import oracle_prove_columns, prove_on_ranks, check_ranks

pytestmark = pytest.mark.gpu

# (seed, overrides, why); every case is byte-compared with the oracle
LARGE_CASES = [
    (100, dict(k=12, degree=7, transcript="blake2b"), "k = 12: size-n NTTs take 2 passes, scans cross two 2048-element blocks"),
    (101, dict(k=12, degree=12, phases=3, transcript="poseidon"), "E = 16 at k = 12 with 3 phases: extended iNTT of 2^16 points"),
    (102, dict(k=12, degree=5, n_lookups=3, max_sets=4, max_width=3, transcript="evm"), "lookups with several input sets of width 3, hash set beyond one CTA"),
    (103, dict(k=13, degree=5, n_perm=8, n_cycles=8, transcript="blake2b"), "k = 13: 8 permutation columns in 3 sets chained across blocks"),
    (104, dict(k=13, degree=11, n_lookups=2, transcript="evm"), "E = 16 at k = 13 in the EVM transcript"),
    (105, dict(k=13, degree=6, phases=3, n_lookups=2, max_sets=3, max_width=3, transcript="poseidon"), "3 phases and multi-set lookups at k = 13"),
    (106, dict(k=14, degree=9, n_lookups=2, max_sets=2, max_width=2, transcript="blake2b"), "k = 14, E = 8: the largest size also proved on ranks"),
    (107, dict(k=14, degree=5, n_perm=8, n_cycles=8, transcript="evm"), "8 permutation columns in 3 sets at k = 14, chained across 8 blocks"),
    (108, dict(k=14, degree=10, phases=2, n_lookups=2, transcript="poseidon"), "E = 16 at k = 14"),
    (109, dict(k=15, far_rotation=True, degree=5, transcript="blake2b"), "k = 15 far_rotation: rotations +-32767, the 16-bit limit"),
    (110, dict(k=15, far_rotation=True, degree=8, n_lookups=2, transcript="evm"), "far_rotation again at k = 15 with lookups, EVM transcript"),
    (111, dict(k=15, degree=6, phases=3, n_perm=6, transcript="poseidon"), "k = 15 with 3 phases and 2 permutation sets"),
    (112, dict(k=16, degree=6, n_lookups=2, max_sets=2, max_width=2, transcript="poseidon"), "k = 16: size-n transforms in 2 passes at 2^16"),
    (113, dict(k=16, degree=5, n_perm=5, n_lookups=1, transcript="blake2b"), "k = 16: 5 permutation columns in 2 sets, E = 4"),
    (114, dict(k=17, degree=12, n_lookups=2, transcript="blake2b"), "k = 17, E = 16: the 3-pass extended iNTT of 2^21 points and 2^20 group iNTTs"),
]
RANK_K = (12, 13, 14)     # cases of these sizes are also proved on 2 and 3 in-process ranks

# (seed, overrides, why); k = 10 or 11, one SHPLONK rotation set per wide column
ROTATION_CASES = [
    (200, dict(k=10, wide_columns=(("fixed", 57, 57),)), "a fixed column at 57 points, past Keccak's 56"),
    (201, dict(k=11, wide_columns=(("fixed", 128, 128),)), "a fixed column at 128 points: half the interpolant block"),
    (202, dict(k=11, wide_columns=(("fixed", 255, 255),)), "a fixed column at 255 points"),
    (203, dict(k=10, wide_columns=(("fixed", 256, 256),)), "a fixed column at 256 points: the limit"),
    (204, dict(k=10, wide_columns=(("fixed", 256, 257),)), "257 rotation numbers, two equal mod n: 256 points, accepted"),
    (205, dict(k=11, wide_columns=(("fixed", 200, 200), ("fixed", 200, 200))), "two disjoint 200-point sets: a 400-point super-set"),
    (206, dict(k=10, wide_columns=(("advice", 256, 256),)), "an advice column at 256 points: blinding factors 258"),
]


def case_id(case):
    seed, kw, _ = case
    return f"seed{seed}-k{kw['k']}"


@pytest.mark.parametrize("case", LARGE_CASES, ids=case_id)
def test_large_random_circuit_matches_oracle(case, monkeypatch):
    seed, kw, _ = case
    tc = RandomCircuit(seed, **kw)
    ref, pkr, proof_ref, ok, cols = oracle_prove_columns(tc)
    prove_and_compare(tc, monkeypatch, again=True, oracle=(ref, pkr, proof_ref, ok))
    if tc.k in RANK_K:
        for P in (2, 3):
            check_ranks(tc, ref, pkr, proof_ref, prove_on_ranks(tc, ref, pkr, cols, P, keygen=P == 3), P)


@pytest.mark.parametrize("case", ROTATION_CASES, ids=case_id)
def test_rotation_set_matches_oracle(case, monkeypatch):
    seed, kw, _ = case
    prove_and_compare(RandomCircuit(seed, **kw), monkeypatch, again=True)


def test_column_at_257_points_is_refused_then_the_context_proves(monkeypatch):
    """a fixed column opened at 257 points: zkb_pk_create, zkb_pk_create_with_srs and zkb_keygen_pk all fail with ZKB_ERR_ARG
    naming the column and its count, before any device work; the same context then proves a corpus circuit byte for byte"""
    import halo2_ref as H
    import zkb200
    from zkb200 import plonk as Z
    from zkb200.params import ParamsKZG
    from test_gpu_prover import to_product_cs
    from witness_ref import perm_copies
    tc = RandomCircuit(207, k=10, wide_columns=(("fixed", 257, 257),))
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    zcs = to_product_cs(tc.cs, ref.bf, ref.d)
    col = next(c for c, role in enumerate(tc.fixed_role) if role == "wide")
    match = f"fixed column {col} is opened at 257 points"
    with pytest.raises(zkb200.ZkbError, match=match):
        Z.ProvingKey(zcs, fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    srs = ParamsKZG(tc.k, ref.g, ref.g_lagrange).load()
    with pytest.raises(zkb200.ZkbError, match=match):
        Z.ProvingKey(zcs, fixed, pkr["sigma_values"], srs=srs)
    with pytest.raises(zkb200.ZkbError, match=match):
        Z.ProvingKey(zcs, fixed, None, srs=srs, copies=perm_copies(tc.cs, tc.copies))
    srs.close()
    prove_and_compare(RandomCircuit(0), monkeypatch)
