"""The prover's mv-lookup multiplicities (zkb_lookup_multiplicities_dev, the code lookup_prepare runs) row by row against a plain
reference, with the table's hash set checked slot by slot (lookup_hash_model.py): sizes at warp / CTA / load-factor edges, duplicate
table rows across CTAs and past the usable rows, a probe chain of 300+ colliding keys wrapping through slot 0, warp-aggregated
counts, unsatisfied inputs, and a proof whose table carries the collisions, byte-identical to the oracle prover's."""
import numpy as np
import pytest

import lookup_hash_model as LH
from util import to_dev, to_host

pytestmark = pytest.mark.gpu


def run(oracle, inputs, table, usable, expect_unsat=False, ref=None):
    """m, the flag and the slots on the device == the reference (`ref`: (counts, flag) when the caller has it); slot invariants hold;
    returns the slots"""
    from zkb200 import plonk as Z
    m, unsat, slots = Z.lookup_multiplicities([to_dev(f) for f in inputs], to_dev(table), usable, slots=True)
    ref, ref_unsat = ref if ref is not None else LH.multiplicities(inputs, table, usable)
    assert ref_unsat == expect_unsat, "the test's own inputs are not what it meant to build"
    assert unsat == ref_unsat
    canon = np.zeros((table.shape[0], 4), dtype=np.uint64)
    canon[:, 0] = ref
    got = to_host(m)
    exp = oracle.fr_from_canonical(canon)
    bad = np.nonzero((got != exp).any(axis=1))[0]
    assert len(bad) == 0, f"{len(bad)} rows of m differ, first {bad[:8].tolist()}"
    if table.shape[0] <= 1 << 20:
        LH.check_slots(slots, table, usable)
    return slots


def junk_past_usable(table, usable, seed):
    """rows >= usable: values in no usable table row (the input rows there must be ignored)"""
    table[usable:] = LH.random_values(table.shape[0] - usable, seed)


SIZES = [(1, 2), (31, 32), (32, 64), (33, 64), (255, 256), (256, 512), (257, 512), (1 << 12, 1 << 13), ((1 << 12) + 1, 1 << 13),
         (1 << 16, 1 << 17), ((1 << 16) + 1, 1 << 17), ((1 << 20) - 7, 1 << 20), (1 << 19, 1 << 20)]


@pytest.mark.parametrize("usable,n", SIZES)
def test_sizes(oracle, usable, n):
    rng = np.random.default_rng(usable)
    pool = LH.random_values(max(1, usable // 2), usable)          # about two table rows per value: duplicates everywhere
    table = pool[rng.integers(0, len(pool), size=n)]
    junk_past_usable(table, usable, usable + 1)
    inputs = []
    for j in range(2):
        f = table[rng.integers(0, usable, size=n)]
        f[usable:] = LH.random_values(n - usable, 7 * usable + j)
        inputs.append(f)
    run(oracle, inputs, table, usable)


def test_size_2_24(oracle):
    """2^24 rows; the reference works on pool indices (the pool's and the junk's 254-bit random values are distinct)"""
    n, usable = 1 << 24, (1 << 24) - 7
    rng = np.random.default_rng(24)
    pool = LH.random_values(1 << 22, 24)
    tid = rng.integers(0, len(pool), size=n)
    table = pool[tid]
    junk_past_usable(table, usable, 25)
    fid = tid[rng.integers(0, usable, size=n)]
    f = pool[fid]
    last = np.full(len(pool), -1, dtype=np.int64)
    np.maximum.at(last, tid[:usable], np.arange(usable))
    assert (last[fid[:usable]] >= 0).all()
    run(oracle, [f], table, usable, ref=(np.bincount(last[fid[:usable]], minlength=n), False))


def test_all_table_rows_equal(oracle):
    n, usable = 4096, 4089
    table = np.repeat(LH.random_values(1, 1), n, axis=0)
    inputs = [table.copy(), table.copy()]
    run(oracle, inputs, table, usable)
    from zkb200 import plonk as Z
    m, _ = Z.lookup_multiplicities([to_dev(f) for f in inputs], to_dev(table), usable)
    assert (to_host(m)[usable - 1] == oracle.fr_from_canonical(np.array([[2 * usable, 0, 0, 0]], dtype=np.uint64))[0]).all()


def test_duplicates_far_apart_and_past_usable(oracle):
    n, usable = 1 << 14, (1 << 14) - 9
    rng = np.random.default_rng(3)
    table = LH.random_values(n, 3)
    for r in (0, 5, 200, 255):                                    # row r repeated at r + 256 j: one copy per CTA of the insert
        for j in (1, 7, 30, 63):
            table[r + 256 * j] = table[r]
    table[usable] = table[17]                                     # a duplicate at a row >= usable must not win
    table[n - 1] = table[usable - 1]
    table[usable + 2] = LH.random_values(1, 99)[0]
    f = table[rng.integers(0, usable, size=n)]
    f[:4] = table[[0, 5, 200, 255]]
    f[4] = table[17]
    f[usable:] = LH.random_values(n - usable, 4)
    run(oracle, [f], table, usable)
    bad = f.copy()
    bad[9] = table[usable + 2]                                    # present only past the usable rows: unsatisfied
    run(oracle, [bad], table, usable, expect_unsat=True)


@pytest.mark.parametrize("usable", [1000, 4097])
def test_collision_chain_wraps(oracle, usable):
    n = 1 << (usable.bit_length() + 1)
    tsize = LH.slot_count(usable)
    home = tsize - 4                                               # a few slots below the mask: the chain wraps through slot 0
    chain = LH.colliding_values(320, home, usable, seed=usable)
    rng = np.random.default_rng(usable)
    table = LH.random_values(n, usable + 1)
    rows = rng.permutation(usable)[:320]
    table[rows] = chain
    dup_rows = rng.permutation(np.setdiff1d(np.arange(usable), rows))[:64]
    table[dup_rows] = chain[rng.integers(0, 320, size=64)]        # duplicates interleaved into the chain, in either row order
    table[usable:usable + 16] = chain[:16]                         # and past the usable rows
    f = table[rng.integers(0, usable, size=n)]
    f[:320] = chain                                                # every key of the chain is hit
    f[usable:] = LH.random_values(n - usable, 5)
    slots = run(oracle, [f, chain[rng.integers(0, 320, size=n)]], table, usable)
    assert (LH.home_slot(table[:usable], usable) == home).sum() >= 320 + 64
    run_len = LH.probe_run(slots, home)
    assert run_len >= 300 and home + run_len > tsize, f"the probe chain is {run_len} slots from {home} of {tsize}"


@pytest.mark.parametrize("n_sets", [1, 2, 5])
def test_input_shapes(oracle, n_sets):
    n, usable = 1 << 13, (1 << 13) - 10
    table = LH.random_values(n, 11)
    junk_past_usable(table, usable, 12)
    same = [np.repeat(table[37:38], n, axis=0) for _ in range(n_sets)]     # one value everywhere: whole warps aggregate
    for f in same:
        f[usable:] = LH.random_values(n - usable, 13)
    run(oracle, same, table, usable)
    distinct = [table[np.random.default_rng(j).permutation(n) % usable] for j in range(n_sets)]
    run(oracle, distinct, table, usable)
    alt = [np.where((np.arange(n) % 2 == 0)[:, None], table[3], table[usable - 1]) for _ in range(n_sets)]
    for j, f in enumerate(alt):
        if j % 2:
            f[::3] = table[100]                                               # three values interleaved inside each warp
    run(oracle, alt, table, usable)


@pytest.mark.parametrize("row,flagged", [(0, True), (-1, True), ("past", False)])
def test_unsatisfied(oracle, row, flagged):
    n, usable = 1 << 12, (1 << 12) - 10
    table = LH.random_values(n, 21)
    f = table[np.random.default_rng(21).integers(0, usable, size=n)]
    r = {0: 0, -1: usable - 1, "past": usable}[row]
    f[r] = LH.random_values(1, 22)[0]
    run(oracle, [table[:].copy(), f], table, usable, expect_unsat=flagged)


def test_deterministic(oracle):
    from zkb200 import plonk as Z
    n, usable = 1 << 16, (1 << 16) - 3
    rng = np.random.default_rng(31)
    pool = LH.random_values(5000, 31)
    table = pool[rng.integers(0, 5000, size=n)]
    ins = [to_dev(pool[rng.integers(0, 5000, size=n)]) for _ in range(2)]
    a = Z.lookup_multiplicities(ins, to_dev(table), usable, slots=True)
    b = Z.lookup_multiplicities(ins, to_dev(table), usable, slots=True)
    # which slot of a probe run a key lands in depends on the insertion schedule; m does not
    assert (to_host(a[0]) == to_host(b[0])).all() and a[1] == b[1]
    LH.check_slots(a[2], table, usable)
    LH.check_slots(b[2], table, usable)


@pytest.mark.parametrize("usable,n", [(0, 64), (64, 64), (65, 64)])
def test_arguments_rejected_before_launch(usable, n):
    from zkb200 import plonk as Z, ZkbError, default_context
    t = to_dev(LH.random_values(n, 1))
    before = default_context().launch_count
    with pytest.raises(ZkbError):
        Z.lookup_multiplicities([t], t, usable)
    assert default_context().launch_count == before


def test_proof_with_colliding_table_matches_oracle():
    """A width-1 lookup whose fixed table holds a wrapping collision chain and duplicates: the device proof (lookup_prepare through
    lookup_multiplicities) is byte-identical to the oracle prover's."""
    import halo2_ref as H
    from circuits import ThinCompressionShape
    from test_gpu_prover import to_product_cs, first_diff
    from zkb200 import plonk as Z
    k = 10
    tc = ThinCompressionShape(k, seed=5, table=lambda usable: LH.colliding_values(300, LH.slot_count(usable) - 3, usable, seed=k))
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    usable = tc.usable
    homes = LH.home_slot(fixed[0][:usable], usable)
    assert (homes == LH.slot_count(usable) - 3).sum() >= 300    # the compressed width-1 table is the fixed column itself
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": rp}
    synth = lambda phase, ch: {c: F.arr(v) for c, v in tc.advice_ints(phase, ch).items()}
    proof_ref, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, synth, blinds)
    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    proof = Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth,
                           np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]), np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]), rp)
    assert first_diff(proof, proof_ref) is None
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof)
