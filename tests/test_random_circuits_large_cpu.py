"""The large-k and rotation-set cases of tests/test_gpu_random_circuits_large.py on the CPU: the case list covers the sizes, degree
groups, transcripts and shapes it states; far_rotation reads +-32767 at k = 15 and is refused at k = 16; the wide-column knob
reads exactly the points it asks for; the oracle proves and verifies a 256-point case and a 257-rotation, 256-point case."""
import halo2_ref as H
import pytest

from random_circuit import RandomCircuit, MAX_POINTS_PER_COLUMN, transcript_layout
from test_gpu_prover import to_product_cs
from test_gpu_random_circuits_large import LARGE_CASES, ROTATION_CASES, RANK_K
from test_random_circuits_cpu import oracle_prove


def large(k_max=17):
    return [RandomCircuit(seed, **kw) for seed, kw, _ in LARGE_CASES if kw["k"] <= k_max]


def points(tc, kind):
    """{column: number of distinct points mod n} of the fixed or advice queries"""
    qs = tc.cs.fixed_queries if kind == "fixed" else tc.cs.advice_queries
    out = {}
    for c, r in qs:
        out.setdefault(c, set()).add(r % tc.n)
    return {c: len(p) for c, p in out.items()}


def test_large_cases_cover_what_they_state():
    cases = large()
    ks = [tc.k for tc in cases]
    assert set(ks) == {12, 13, 14, 15, 16, 17}
    e16 = {tc.k for tc in cases if H.Domain(tc.k, tc.degree).E == 16}
    assert len(e16) >= 3 and 17 in e16, e16
    assert {tc.transcript for tc in cases} == {"blake2b", "poseidon", "evm"}
    assert any(tc.cs.num_phases() == 3 for tc in cases)
    assert any(-(-len(tc.cs.perm_columns) // (tc.degree - 2)) >= 3 for tc in cases)
    assert sum(-(-len(tc.cs.perm_columns) // (tc.degree - 2)) >= 2 for tc in cases) >= 3
    assert any(len(lk.inputs) >= 2 and len(lk.table) >= 2 for tc in cases for lk in tc.cs.lookups)
    assert sum(any(len(lk.inputs) >= 2 and len(lk.table) >= 2 for lk in tc.cs.lookups) for tc in cases) >= 3
    assert any(tc.k == 15 and tc.features()["far_rotation"] and tc.features()["rotations_equal_mod_n"] for tc in cases)
    assert {tc.k for tc in cases} >= set(RANK_K)
    assert len({seed for seed, _, _ in LARGE_CASES}) == len(LARGE_CASES)
    for tc in cases:
        assert tc.bf <= 7 and max(points(tc, "advice").values()) <= 5, tc.describe()


def test_far_rotation_at_k15_reads_the_16_bit_limit():
    """far_rotation at k = 15 reads rotations +-32767 and one column at r and r -+ n; every pinned k = 15 case does"""
    from zkb200 import plonk as Z
    for seed, kw, _ in LARGE_CASES:
        if kw["k"] != 15 or not kw.get("far_rotation"):
            continue
        tc = RandomCircuit(seed, **kw)
        rots = {r for q in (tc.cs.advice_queries, tc.cs.fixed_queries, tc.cs.instance_queries) for _, r in q}
        assert rots & {32767, -32767}, tc.describe()
        assert any((c, r - tc.n) in tc.cs.advice_queries for c, r in tc.cs.advice_queries if r > 0), tc.describe()
        Z.validate_csf(to_product_cs(tc.cs, tc.bf, tc.degree).to_csf())


def test_far_rotation_at_k16_is_refused():
    with pytest.raises(ValueError, match="16 bits"):
        RandomCircuit(112, k=16, far_rotation=True)
    RandomCircuit(112, k=16, far_rotation=False)


@pytest.mark.parametrize("case", ROTATION_CASES, ids=lambda c: f"seed{c[0]}")
def test_wide_columns_read_the_stated_points(case):
    """each wide column is read at exactly its rotation count and point count, and the point sets of two wide columns are disjoint;
    an advice column's blinding factors are its query count + 2, fixed ones leave them as drawn; the CSF passes zkb_csf_validate"""
    from zkb200 import plonk as Z
    seed, kw, _ = case
    tc = RandomCircuit(seed, **kw)
    assert tc.k in (10, 11)
    wide = {"fixed": [c for c, r in enumerate(tc.fixed_role) if r == "wide"], "advice": [c for c, r in enumerate(tc.adv_role) if r == "wide"]}
    queries = {"fixed": tc.cs.fixed_queries, "advice": tc.cs.advice_queries}
    sets = []
    for kind, want_pts, want_rots in kw["wide_columns"]:
        col = wide[kind].pop(0)
        rots = [r for c, r in queries[kind] if c == col]
        sets.append({r % tc.n for r in rots})
        assert (len(rots), len(sets[-1])) == (want_rots, want_pts), tc.describe()
    assert len(set().union(*sets)) == sum(map(len, sets))
    advice_rots = [rots for kind, _, rots in kw["wide_columns"] if kind == "advice"]
    assert tc.bf == max(advice_rots) + 2 if advice_rots else tc.bf <= 7
    assert max(points(tc, "fixed").values()) <= MAX_POINTS_PER_COLUMN and max(points(tc, "advice").values()) <= MAX_POINTS_PER_COLUMN
    Z.validate_csf(to_product_cs(tc.cs, tc.bf, tc.degree).to_csf())


def test_wide_column_knob_is_off_by_default():
    assert RandomCircuit(3).shape.wide_columns == ()
    assert "wide" not in RandomCircuit(3).fixed_role + RandomCircuit(3).adv_role


@pytest.mark.parametrize("seed", [203, 204])
def test_oracle_proves_and_verifies_wide_sets(seed):
    """the oracle prover and verifier on a 256-point set and on 257 rotations that make 256 points"""
    seed, kw, _ = next(c for c in ROTATION_CASES if c[0] == seed)
    tc = RandomCircuit(seed, **kw)
    _, _, proof, ok = oracle_prove(tc, tc.transcript)
    assert ok, tc.describe()
    assert len(proof) == sum(size for _, size in transcript_layout(tc.cs, tc.transcript))
