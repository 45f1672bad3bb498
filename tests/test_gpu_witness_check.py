"""GPU: the witness check (zkb_check_witness_dev, plonk.check_witness) against the CPU reference of tests/witness_ref.py.

Counts per item and the full ordered record list must be equal, on satisfied witnesses and with seeded random faults, for every
circuit family: hand-built CSFs at k = 1, 3, 4 (partial warps), two-phase circuits with challenges, lookups of width 1 and 2, the
instance column inside the permutation.  Also: the record cap, determinism, argument errors, no effect on a later proof, and the
k = 20 SuperCircuit stand-in with single broken cells whose records are derived from the circuit's structure."""
import ctypes

import numpy as np
import pytest

import halo2_ref as H
import standin_copies
import standins
from circuits import ToyCircuit, ThinCompressionShape, GatesOnlyCircuit, DeepGateCircuit
from test_gpu_prover import to_product_cs
from test_gpu_prover_wide import to_oracle_cs
from witness_ref import check_witness as ref_check, perm_copies, circuit_columns

pytestmark = pytest.mark.gpu

CH = [0x5EED5, 0xC0FFEE]


def gpu_check(zcs, cols, F, challenges, copies, cap=1 << 20, theta=None):
    from zkb200 import plonk as Z
    rep = Z.check_witness(zcs, cols[H.FIXED], cols[H.ADVICE], cols[H.INSTANCE], challenges=F.arr(challenges) if challenges else (),
                          copies=copies, theta=theta, cap=cap)
    return rep


def assert_same(rep, want):
    counts, recs = want
    assert list(rep.counts) == list(counts), "counts differ"
    assert [tuple(f) for f in rep.failures] == recs[: len(rep.failures)] and len(rep.failures) == len(recs), "records differ"


def faults(cols, F, rng, count, kinds=(H.ADVICE,)):
    """`count` random cells of the given column kinds set to random values (in place, on copies of the columns)"""
    for _ in range(count):
        t = kinds[rng.integers(len(kinds))]
        if not cols[t]:
            continue
        c = int(rng.integers(len(cols[t])))
        r = int(rng.integers(cols[t][c].shape[0]))
        cols[t][c] = cols[t][c].copy()
        cols[t][c][r] = F.arr([int(rng.integers(1 << 62))])[0]


FAMILIES = [("toy", 5, {}), ("toy", 8, {}), ("toy", 6, dict(two_phase=False)), ("thin", 7, {}), ("gates", 5, {}), ("deep", 6, {})]


@pytest.mark.parametrize("kind,k,kw", FAMILIES)
@pytest.mark.parametrize("n_faults", [0, 1, 50])
def test_circuits_match_reference(kind, k, kw, n_faults):
    tc = {"toy": ToyCircuit, "thin": ThinCompressionShape, "gates": GatesOnlyCircuit, "deep": DeepGateCircuit}[kind](k, seed=40 + k, **kw)
    ref = H.Ref(tc.cs, 0, build_srs=False)
    F = ref.F
    cols = circuit_columns(tc, F, CH)
    faults(cols, F, np.random.default_rng(k * 100 + n_faults), n_faults, (H.ADVICE, H.FIXED, H.INSTANCE))
    copies = perm_copies(tc.cs, tc.copies)
    want = ref_check(ref, tc.cs, cols, CH, copies, tc.n - ref.bf - 1)
    rep = gpu_check(to_product_cs(tc.cs, ref.bf, ref.d), cols, F, CH[: len(tc.cs.challenge_phase)], copies)
    assert_same(rep, want)
    assert rep.ok == (not want[1])              # a random cell may be one no constraint reads
    if n_faults == 0:
        assert rep.ok
        rep.assert_satisfied()


def small_cs(k):
    """hand-built: two gates with rotations, a width-1 and a width-2 lookup, the instance column in the permutation"""
    cs = H.ConstraintSystem(k, 3, 3, 1)
    a, b, c = (lambda r=0, i=i: H.advice(i, r) for i in range(3))
    cs.gates = [H.fixed(0) * (a() * b(1) - c(-1)), H.fixed(1) * (a(3) + H.instance(0, 1)), c(2) * c()]
    cs.lookups = [H.Lookup([[a()]], [H.fixed(2)]), H.Lookup([[a(), b()], [b(1), c()]], [H.fixed(2), H.fixed(0)])]
    cs.perm_columns = [(H.ADVICE, 0), (H.INSTANCE, 0), (H.FIXED, 1)]
    return cs.finalize()


@pytest.mark.parametrize("k", [1, 3, 4])
def test_tiny_domains(k):
    """fewer rows than a warp: every lane past the last row must still vote 0 in the ballots"""
    cs = small_cs(k)
    ref = H.Ref(cs, 0, build_srs=False)
    F = ref.F
    n, bf = cs.n, 5
    rng = np.random.default_rng(k)
    small = lambda: F.arr([int(x) for x in rng.integers(0, 3, n)])
    cols = {H.FIXED: [small() for _ in range(3)], H.ADVICE: [small() for _ in range(3)], H.INSTANCE: [small()]}
    copies = [(int(rng.integers(3)), int(rng.integers(n)), int(rng.integers(3)), int(rng.integers(n))) for _ in range(40)]
    want = ref_check(ref, cs, cols, [], copies, n - bf - 1)
    assert sum(want[0]) > 0
    rep = gpu_check(to_product_cs(cs, bf, 5), cols, F, [], copies)
    assert_same(rep, want)


@pytest.mark.parametrize("kind", ["keccak", "super"])
def test_standins_match_reference(kind):
    sc = standins.keccak_shape(9, seed=1, scale=0.12) if kind == "keccak" else standins.super_shape(8, seed=2, advice=40, n_gates=60)
    cs = to_oracle_cs(sc.cs)
    ref = H.Ref(cs, 0, build_srs=False)
    F = ref.F
    nch = len(sc.cs.challenge_phase)
    fixed, adv, inst = standin_copies.witness(sc, list(F.arr(CH[:nch])))
    copies = standin_copies.copies(sc)
    cols = {H.FIXED: [sc.host(t) for t in fixed], H.ADVICE: [sc.host(t) for t in adv], H.INSTANCE: [sc.host(t) for t in inst]}
    hcopies = copies.cpu().numpy().astype(np.uint32)
    for n_faults in (0, 50):
        faults(cols, F, np.random.default_rng(n_faults), n_faults)
        want = ref_check(ref, cs, cols, CH[:nch], hcopies, sc.usable)
        rep = gpu_check(sc.cs, cols, F, CH[:nch], copies)
        assert_same(rep, want)
        assert rep.ok == (not want[1]) and (rep.ok or n_faults)


def test_cap_prefix_and_determinism():
    tc = ToyCircuit(8, seed=7)
    ref = H.Ref(tc.cs, 0, build_srs=False)
    F = ref.F
    cols = circuit_columns(tc, F, CH)
    faults(cols, F, np.random.default_rng(3), 60, (H.ADVICE,))
    copies = perm_copies(tc.cs, tc.copies)
    counts, recs = ref_check(ref, tc.cs, cols, CH, copies, tc.n - ref.bf - 1)
    assert len({(r[0], r[1], r[2] if r[0] == 1 else 0) for r in recs}) >= 3      # failures in several items
    zcs = to_product_cs(tc.cs, ref.bf, ref.d)
    theta = F.arr([0x7E7A])[0]
    for cap in (0, 1, len(recs) // 2, len(recs) + 10):
        rep = gpu_check(zcs, cols, F, CH[:1], copies, cap=cap, theta=theta)
        assert list(rep.counts) == list(counts)
        assert [tuple(f) for f in rep.failures] == recs[:cap]
    a = gpu_check(zcs, cols, F, CH[:1], copies, cap=len(recs), theta=theta)
    b = gpu_check(zcs, cols, F, CH[:1], copies, cap=len(recs), theta=theta)
    assert a.counts.tobytes() == b.counts.tobytes() and a.failures == b.failures
    from zkb200 import ZkbError
    with pytest.raises(ZkbError, match=r"gate \d+ not satisfied at row"):
        a.assert_satisfied()


def test_invalid_arguments():
    from zkb200 import ZkbError, plonk as Z, default_context
    tc = ToyCircuit(5, seed=8)
    ref = H.Ref(tc.cs, 0, build_srs=False)
    F = ref.F
    cols = circuit_columns(tc, F, CH)
    zcs = to_product_cs(tc.cs, ref.bf, ref.d)
    P, n = len(tc.cs.perm_columns), tc.n
    for bad in [(P, 0, 0, 0), (0, 0, 0, n)]:
        with pytest.raises(ZkbError, match="copy constraint 1 is out of range"):
            gpu_check(zcs, cols, F, CH[:1], [(0, 0, 0, 0), bad, bad])
    with pytest.raises(ZkbError, match="challenges"):
        gpu_check(zcs, cols, F, [], [])
    # theta = NULL with width-2 lookups, through the C ABI directly (the Python wrapper always passes one)
    import torch
    ctx = default_context()
    dcols = [torch.from_numpy(np.ascontiguousarray(c).view(np.int64)).cuda() for t in (H.FIXED, H.ADVICE, H.INSTANCE) for c in cols[t]]
    blob = zcs.to_csf()
    ch = np.ascontiguousarray(F.arr(CH[:1]))
    tbl = (ctypes.c_void_p * len(dcols))(*[c.data_ptr() for c in dcols])
    counts = np.zeros(64, dtype=np.uint64)
    nrec = ctypes.c_uint32(0)
    rc = ctx.lib.zkb_check_witness_dev(ctx.handle, ctypes.c_void_p(blob.ctypes.data), blob.size, ctypes.cast(tbl, ctypes.c_void_p),
                                       ctypes.c_void_p(ch.ctypes.data), None, None, 0, ctypes.c_void_p(counts.ctypes.data), None, 0,
                                       ctypes.byref(nrec), None)
    assert rc == -2 and b"needs theta" in ctx.lib.zkb_last_error()


def test_check_then_prove_gives_the_oracle_proof():
    from zkb200 import plonk as Z
    tc = ToyCircuit(6, seed=21)
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    zcs = to_product_cs(tc.cs, ref.bf, ref.d)
    pk = Z.ProvingKey(zcs, fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    cols = circuit_columns(tc, F, CH)
    faults(cols, F, np.random.default_rng(5), 10)
    assert not gpu_check(zcs, cols, F, CH[:1], perm_copies(tc.cs, tc.copies)).ok
    rp = F.arr(tc.blinds_ints["random_poly"])
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": rp}
    proof_ref, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, ch).items()}, blinds)
    synth = lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, {i: F.ints(v[None])[0] for i, v in ch.items()}).items()}
    proof = Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth,
                           np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]), np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]), rp)
    assert proof == proof_ref


# ---------------------------------------------------------------------------------------------------- k = 20 bench shape
def zero_part(e):
    """the constraint difference (A + (-B)) inside a stand-in gate: the factor that vanishes on a satisfied witness"""
    if e.op == H.ADD and e.b.op == H.NEG:
        return e
    for ch in ((e.a, e.b) if e.op in (H.ADD, H.MUL) else (e.a,) if e.op in (H.NEG, H.SCALED) else ()):
        z = zero_part(ch)
        if z is not None:
            return z
    return None


def queries(e, kind, col, out):
    if e.op == kind and e.a == col: out.add(e.b)
    elif e.op in (H.NEG, H.SCALED): queries(e.a, kind, col, out)
    elif e.op in (H.ADD, H.MUL): queries(e.a, kind, col, out); queries(e.b, kind, col, out)
    return out


def test_super_shape_k20():
    import torch
    from zkb200 import plonk as Z
    sc = standins.super_shape(20, advice=128, seed=5)
    assert sc.shape["gates"] >= 600
    cs = to_oracle_cs(sc.cs)
    F = H.FA()
    n, usable = sc.n, sc.usable
    ch = F.arr(CH)
    fixed, adv, inst = standin_copies.witness(sc, list(ch))
    pis = standin_copies.permutations(sc)
    copies = standin_copies.copies(sc, pis)
    run = lambda a: Z.check_witness(sc.cs, fixed, a, inst, challenges=ch, copies=copies, cap=4096)
    rep = run(adv)
    assert rep.ok and not rep.counts.any() and rep.failures == []
    sel_rows = {0: usable, 2: len(sc.instances[0])}            # q_gate is 1 on the usable rows, q_pi on the instance cells
    junk = torch.from_numpy(F.arr([0xDEADBEEF12345])[0].view(np.int64)).cuda()

    def broken(c, r):
        a = list(adv)
        a[c] = adv[c].clone()
        a[c][r] = junk
        return a
    # a gate-read column (the hot base column): the gates whose constraint difference reads it, at row r - rot
    c, r = 0, 1000
    want = []
    for g, gate in enumerate(cs.gates):
        z = zero_part(gate)
        sel = gate.a.a
        rows = sorted({(r - rot) % n for rot in queries(z, H.ADVICE, c, set())})
        want += [(0, g, 0, i) for i in rows if i < sel_rows[sel]]
    assert want
    got = run(broken(c, r))
    assert [tuple(f) for f in got.failures] == want and got.total == len(want)
    # a lookup-pair column: the input sets that read it, at rows where the lookup selector is on
    c, r = sc.c_pair0 + 1, 2000
    q_lk = sc.host(sc.fixed[1])
    want = []
    for l, lk in enumerate(cs.lookups):
        for j, inp in enumerate(lk.inputs):
            rows = sorted({(r - rot) % n for e in inp for rot in queries(e, H.ADVICE, c, set())})
            want += [(1, l, j, i) for i in rows if i < usable and q_lk[i].any()]
    assert want
    got = run(broken(c, r))
    assert [tuple(f) for f in got.failures] == want and got.total == len(want)
    # a permutation column: column 0 cell v is the target of one copy per other column; column j >= 1 cell r of exactly one
    v = 3000
    idx = [(j - 1) * usable + int(torch.nonzero(pis[j] == v)[0]) for j in range(1, sc.P)]
    got = run(broken(sc.c_perm0, v))
    assert [tuple(f) for f in got.failures] == sorted((2, i, 0, i % usable) for i in idx)
    j, r = 3, 4000
    got = run(broken(sc.c_perm0 + j, r))
    assert [tuple(f) for f in got.failures] == [(2, (j - 1) * usable + r, 0, r)]
