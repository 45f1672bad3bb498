"""GPU parity on the random circuit corpus (tests/random_circuit.py): for every seed the CUDA prover's proof is byte-identical to the
oracle prover's in the seed's transcript and the oracle verifier accepts it; keygen on the device gives the oracle's sigma columns
and vk bytes; the device witness check finds nothing on the satisfied witness and, with one changed advice cell, reports exactly
what tests/witness_ref.py reports.  Every eighth seed is proved again without the pk's coset cache and with its columns uploaded
ahead of their phase calls, with the same bytes."""
import numpy as np
import pytest

import halo2_ref as H
import keccak_ref as K
from random_circuit import RandomCircuit, transcript_layout, item_at
from test_gpu_prover import first_diff, to_product_cs
from test_gpu_witness_check import assert_same, gpu_check
from test_random_circuits_cpu import GPU_SEEDS, challenges_for, oracle_prove
from witness_ref import check_witness as ref_check, perm_copies, circuit_columns

pytestmark = pytest.mark.gpu


def gpu_prove(tc, ref, pk, **kw):
    from zkb200 import plonk as Z
    F = ref.F
    synth = lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, {i: F.ints(v[None])[0] for i, v in ch.items()}).items()}
    zb = np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]) if tc.blinds_ints["z"] else None
    pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]) if tc.blinds_ints["phi"] else None
    return Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth, zb, pb,
                          F.arr(tc.blinds_ints["random_poly"]), transcript=tc.transcript, **kw)


def assert_same_proof(tc, proof, proof_ref, what="proof"):
    if proof == proof_ref:
        return
    layout = transcript_layout(tc.cs, tc.transcript)
    i = next((b for b in range(min(len(proof), len(proof_ref))) if proof[b] != proof_ref[b]), min(len(proof), len(proof_ref)))
    pytest.fail(f"{what} differs from the oracle's ({len(proof)} vs {len(proof_ref)} bytes) first at byte {i}, item "
                f"'{item_at(layout, i)}' (32-byte word {first_diff(proof, proof_ref)}); {tc.describe()}")


def prove_and_compare(tc, monkeypatch, again=False, oracle=None):
    """oracle: (ref, pkr, proof, verified) of oracle_prove(tc, tc.transcript) when the caller has it already"""
    from zkb200 import plonk as Z
    from zkb200.params import ParamsKZG
    ref, pkr, proof_ref, ok = oracle if oracle is not None else oracle_prove(tc, tc.transcript)
    assert ok, f"the oracle rejects its own proof: {tc.describe()}"
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    zcs = to_product_cs(tc.cs, ref.bf, ref.d)
    pk = Z.ProvingKey(zcs, fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    proof = gpu_prove(tc, ref, pk)
    assert_same_proof(tc, proof, proof_ref)
    reader = {"blake2b": None, "poseidon": H.Ref.PoseidonReader(proof), "evm": K.EvmTranscript(proof=proof)}[tc.transcript]
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof, reader=reader)
    if again:
        assert_same_proof(tc, gpu_prove(tc, ref, pk, upload_ahead=True), proof_ref, "proof with columns uploaded ahead")
        monkeypatch.setenv("ZKB_COSET_CACHE_GB", "0")
        pk_nc = Z.ProvingKey(zcs, fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
        monkeypatch.delenv("ZKB_COSET_CACHE_GB")
        assert_same_proof(tc, gpu_prove(tc, ref, pk_nc), proof_ref, "proof without the coset cache")
        pk_nc.close()
    pk.close()
    # keygen on the device: permutation assembly from the copies, sigma columns and vk bytes
    srs = ParamsKZG(tc.k, ref.g, ref.g_lagrange).load()
    pk_kg = Z.ProvingKey(zcs, fixed, None, srs=srs, copies=perm_copies(tc.cs, tc.copies))
    for i in range(len(tc.cs.perm_columns)):
        assert (pk_kg.sigma_values(i) == pkr["sigma_values"][i]).all(), f"sigma column {i}: {tc.describe()}"
    exp_vk = tc.k.to_bytes(4, "big") + len(fixed).to_bytes(4, "big") + \
        b"".join(ref.o.g1_compress(c) for c in pkr["fixed_commitments"] + pkr["sigma_commitments"])
    assert pk_kg.vk_bytes() == exp_vk, tc.describe()
    pk_kg.close()
    # the witness check: nothing on the satisfied witness, the reference's exact report with one changed advice cell
    ch = challenges_for(tc)
    cols = circuit_columns(tc, F, ch)
    copies = perm_copies(tc.cs, tc.copies)
    rep = gpu_check(zcs, cols, F, ch, copies)
    assert rep.ok and rep.failures == [], f"{rep.summary()}; {tc.describe()}"
    rnd = np.random.default_rng(tc.seed)
    c = int(rnd.integers(tc.cs.num_advice))
    r = int(rnd.integers(tc.usable))
    cols[H.ADVICE][c] = cols[H.ADVICE][c].copy()
    cols[H.ADVICE][c][r] = F.arr([int(rnd.integers(1 << 62))])[0]
    want = ref_check(ref, tc.cs, cols, ch, copies, tc.usable)
    assert_same(gpu_check(zcs, cols, F, ch, copies), want)


@pytest.mark.parametrize("seed", GPU_SEEDS)
def test_random_circuit_matches_oracle(seed, monkeypatch):
    prove_and_compare(RandomCircuit(seed), monkeypatch, again=seed % 8 == 0)


@pytest.mark.parametrize("k,transcript", [(5, "blake2b"), (7, "poseidon"), (8, "evm")])
def test_one_column_opened_at_rotations_equal_mod_n(k, transcript, monkeypatch):
    """a column read at rotation r and at r -+ n is two queries with two evaluations in the transcript, but one opening point x w^r:
    SHPLONK's rotation sets are sets of points (construct_intermediate_sets), so that column's set holds the point once, and a
    column read at {0, 1 - n} shares the permutation's set {x, w x}.  The prover once grouped openings by rotation number and wrote
    a different first SHPLONK commitment for such circuits."""
    tc = RandomCircuit(1, k=k, far_rotation=True, transcript=transcript)
    assert tc.features()["rotations_equal_mod_n"]
    prove_and_compare(tc, monkeypatch, again=True)
