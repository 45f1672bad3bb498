"""The multi-rank paths on ONE GPU: P contexts of this process joined into one group by the in-process communicator
(zkb_comm_init_local), every rank driven from its own thread under its own torch stream.  NCCL refuses two ranks on one device, so
without this group the code that runs only when a context has nranks > 1 -- the dealt stages of create_proof, the point-range
single commitments, the sharded NTT's window and exchanges, the sharded MSM's host sum -- would run only on machines with several
GPUs.  Every result is compared with a single-rank reference: the oracle prover's bytes, best_fft on the whole array, the
trapdoor's [sum c_i s^i] G.  The NCCL transport, cudaIpc windows and peer stores across devices stay with test_gpu_multi.py."""
import collections
import random
import threading
import time

import numpy as np
import pytest

import halo2_ref as H
import pyref as PR
from random_circuit import RandomCircuit
from test_gpu_prover import to_product_cs
from test_gpu_random_circuits import assert_same_proof
from test_random_circuits_cpu import challenges_for, oracle_check
from witness_ref import circuit_columns, perm_copies

pytestmark = pytest.mark.gpu
R = PR.R_MOD
ZKB_ERR_ARG, ZKB_ERR_STATE = -2, -4
DEADLINE_S = 900          # every thread of one on_ranks call has returned by then (a group times out long before)
TIMEOUT_MS = 120000       # a rank waits this long for the others at one meeting


def on_ranks(P, fn, timeout_ms=TIMEOUT_MS):
    """P contexts on device 0 joined into one group; fn(rank, ctx) runs in P threads, each under its own torch stream.  Returns the
    list of results by rank; raises the first exception, tagged with its rank."""
    import torch
    import zkb200
    ctxs = [zkb200.Context(0) for _ in range(P)]
    zkb200.init_comm_local(ctxs, timeout_ms=timeout_ms)
    torch.cuda.synchronize()     # inputs the caller prepared on its own stream are complete
    results, errors = [None] * P, [None] * P

    def run(r):
        try:
            torch.cuda.set_device(0)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                results[r] = fn(r, ctxs[r])
            s.synchronize()
        except BaseException as e:   # noqa: B036 -- reported below with its rank
            errors[r] = e
    threads = [threading.Thread(target=run, args=(r,), name=f"rank {r} of {P}") for r in range(P)]
    for t in threads:
        t.start()
    end = time.monotonic() + DEADLINE_S
    for t in threads:
        t.join(max(0.0, end - time.monotonic()))
    stuck = [r for r, t in enumerate(threads) if t.is_alive()]
    assert not stuck, f"ranks {stuck} of {P} still running after {DEADLINE_S} s"
    for c in ctxs:
        c.close()
    for r, e in enumerate(errors):
        if e is not None:
            raise AssertionError(f"rank {r} of {P}: {type(e).__name__}: {e}") from e
    return results


def error_code(e):
    """the return code of a ZkbError ('libzkb200 error -4: ...')"""
    return int(str(e).split("libzkb200 error ")[1].split(":")[0])


def mont(v):
    return np.array(PR.limbs(PR.to_mont(v % R, R)), dtype=np.uint64)


def dev_scalars(vals):
    import torch
    a = np.array([PR.limbs(PR.to_mont(v % R, R)) for v in vals], dtype=np.uint64).reshape(-1, 4)
    return torch.from_numpy(a.view(np.int64)).cuda()


# ---------------------------------------------------------------------------------------------------- sharded NTT
_fft_cases = {}


def fft_case(log_n):
    """(x, best_fft(x)) of a seeded array of 2^log_n elements, the transform by the CPU oracle (numpy uint64 (n, 4))"""
    import oracle_lib
    from zkb200 import arithmetic as A
    if log_n not in _fft_cases:
        x = A.random_fr_dev(1 << log_n, 1000 + log_n).cpu().numpy().view(np.uint64)
        _fft_cases[log_n] = (x, oracle_lib.load().best_fft(x, A.root_of_unity(log_n)[0], log_n))
    return _fft_cases[log_n]


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("P", [2, 4, 8, 16])
def test_sharded_ntt_matches_best_fft(P, mode, monkeypatch):
    """zkb_ntt_fr_sharded_dev, forward (cyclic in, strips out) and inverse with the 1/n scale (strips in, cyclic out), for every log_n
    from 2 log2 P to 20, then 16 again (the window grows at every size and is reused at the last), in the fused peer-store exchange
    and in the all-to-all one.  The inverse is fed the exact strips, so each direction is checked on its own."""
    import torch
    from zkb200 import arithmetic as A, parallel
    monkeypatch.setenv("ZKB_SHARDED_EXCHANGE", mode)
    log_p = P.bit_length() - 1
    sizes = list(range(2 * log_p, 21)) + [16]
    cases = {}
    for log_n in sorted(set(sizes)):
        x, X = fft_case(log_n)
        cases[log_n] = (torch.from_numpy(x.view(np.int64)).cuda(), torch.from_numpy(X.view(np.int64)).cuda())

    def fn(r, ctx):
        bad = []
        for log_n in sizes:
            n = 1 << log_n
            M, blk = n // P, n // P // P
            x, X = cases[log_n]
            w, wi = A.root_of_unity(log_n)
            cyclic = x[r::P].contiguous()
            strips = torch.cat([X[k * M + r * blk: k * M + (r + 1) * blk] for k in range(P)])
            fwd = parallel.ntt_sharded_dev(cyclic, log_n, w, 0, ctx=ctx)
            inv = parallel.ntt_sharded_dev(strips, log_n, wi, 1, scale=mont(pow(n, -1, R)), ctx=ctx)
            for what, got, want in (("forward", fwd, strips), ("inverse", inv, cyclic)):
                if not torch.equal(got, want):
                    row = int((got != want).any(dim=1).nonzero()[0])
                    bad.append(f"{what} 2^{log_n}: first wrong row {row} of {got.shape[0]}")
        return bad
    for r, bad in enumerate(on_ranks(P, fn)):
        assert not bad, f"rank {r} of {P} ({mode}): {bad}"


# ---------------------------------------------------------------------------------------------------- sharded MSM
# per rank: "rand" random terms, "neg0" / "neg3" the negated terms of rank 0 / 3 (the partial sums cancel), "same0" / "same3" rank
# 0's / 3's terms again (equal partial sums: the host sum doubles), "empty" n_local = 0
MSM_PATTERNS = {
    2: ["rand", "neg0"],
    3: ["rand", "same0", "empty"],
    5: ["empty", "rand", "rand", "same2", "neg1"],
    16: ["rand", "neg0", "empty", "rand", "same3", "rand", "empty", "rand", "rand", "empty", "rand", "neg3", "rand", "empty", "same5", "rand"],
}


@pytest.mark.parametrize("P", sorted(MSM_PATTERNS))
def test_sharded_msm_partial_sums(P):
    """zkb_msm_g1_sharded_dev with ranks that hold no points, partial sums that cancel across ranks and equal partial sums, over the
    SRS of a known trapdoor s: every rank's result == [sum c_i s^(e_i)] G == the single-rank MSM of all terms"""
    import torch
    from zkb200 import arithmetic as A, parallel
    from zkb200.params import ParamsKZG
    k, s = 10, 0x5EED5EED5EED
    params = ParamsKZG.unsafe_setup_with_s(k, s)
    rnd = random.Random(P)
    terms = []
    for pat in MSM_PATTERNS[P]:
        if pat == "rand":
            m = rnd.choice([1, 2, 37, 300])
            terms.append(([rnd.randrange(1 << k) for _ in range(m)], [rnd.randrange(R) for _ in range(m)]))
        elif pat == "empty":
            terms.append(([], []))
        else:
            e, c = terms[int(pat[-1])]
            terms.append((list(e), [(-v) % R for v in c] if pat.startswith("neg") else list(c)))
    total = sum(c * pow(s, e, R) for es, cs in terms for e, c in zip(es, cs)) % R
    want = PR.g1_compress(PR.g1_mul(PR.G1_GEN, total))
    shards = []
    for es, cs in terms:
        idx = torch.tensor(es, dtype=torch.int64, device="cuda")
        shards.append((dev_scalars(cs).contiguous() if cs else torch.empty((0, 4), dtype=torch.int64, device="cuda"),
                       params.g[idx].contiguous() if es else torch.empty((0, 8), dtype=torch.int64, device="cuda")))
    single = A.best_multiexp_dev(torch.cat([a for a, _ in shards]), torch.cat([b for _, b in shards])).compressed
    assert single == want, "the single-rank MSM differs from the trapdoor's value"
    got = on_ranks(P, lambda r, ctx: parallel.msm_sharded_dev(shards[r][0], shards[r][1], ctx=ctx)[1])
    for r, comp in enumerate(got):
        assert comp == want, f"rank {r} of {P}: {comp.hex()} != {want.hex()} (patterns {MSM_PATTERNS[P]})"


# ---------------------------------------------------------------------------------------------------- proofs
def oracle_prove_columns(tc):
    """oracle_prove, also returning the advice columns of every phase as the oracle synthesised them (Montgomery arrays): the
    rank threads prove from these, so they only read shared data; a prover that squeezes other challenges writes other bytes"""
    import keccak_ref as K
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": F.arr(tc.blinds_ints["random_poly"])}
    cols = {}

    def synth(ph, ch):
        cols[ph] = {c: F.arr(v) for c, v in tc.advice_ints(ph, ch).items()}
        return cols[ph]
    writer = {"blake2b": None, "poseidon": H.Ref.PoseidonTranscript(ref), "evm": K.EvmTranscript(ref)}[tc.transcript]
    proof, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, synth, blinds, transcript=writer)
    reader = {"blake2b": None, "poseidon": H.Ref.PoseidonReader(proof), "evm": K.EvmTranscript(proof=proof)}[tc.transcript]
    return ref, pkr, proof, ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof, reader=reader), cols


def prove_with(tc, ref, pk, cols, **kw):
    from zkb200 import plonk as Z
    F = ref.F
    zb = np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]) if tc.blinds_ints["z"] else None
    pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]) if tc.blinds_ints["phi"] else None
    return Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], lambda ph, ch: cols[ph], zb, pb,
                          F.arr(tc.blinds_ints["random_poly"]), transcript=tc.transcript, **kw)


def prove_on_ranks(tc, ref, pkr, cols, P, keygen=False, again=False):
    """every rank builds its pk and proves tc (again: also with the columns uploaded ahead); keygen: device keygen's sigma columns
    and vk bytes too.  -> one dict per rank"""
    from zkb200 import plonk as Z
    from zkb200.params import ParamsKZG
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    zcs = to_product_cs(tc.cs, ref.bf, ref.d)

    def fn(r, ctx):
        out = {}
        pk = Z.ProvingKey(zcs, fixed, pkr["sigma_values"], ref.g, ref.g_lagrange, ctx=ctx)
        try:
            out["proof"] = prove_with(tc, ref, pk, cols)
            if again:
                out["proof uploaded ahead"] = prove_with(tc, ref, pk, cols, upload_ahead=True)
        finally:
            pk.close()
        if keygen:
            srs = ParamsKZG(tc.k, ref.g, ref.g_lagrange).load(ctx=ctx)
            pk_kg = Z.ProvingKey(zcs, fixed, None, srs=srs, copies=perm_copies(tc.cs, tc.copies))
            try:
                out["sigma"] = [pk_kg.sigma_values(i) for i in range(len(tc.cs.perm_columns))]
                out["vk"] = pk_kg.vk_bytes()
            finally:
                pk_kg.close()
                srs.close()
        return out
    return on_ranks(P, fn)


def check_ranks(tc, ref, pkr, proof_ref, outs, P):
    for r, out in enumerate(outs):
        for what in ("proof", "proof uploaded ahead"):
            if what in out:
                assert_same_proof(tc, out[what], proof_ref, f"rank {r} of {P}: {what}")
        if "vk" in out:
            for i, sig in enumerate(out["sigma"]):
                assert (sig == pkr["sigma_values"][i]).all(), f"rank {r} of {P}: keygen sigma column {i}; {tc.describe()}"
            fixed = [ref.F.arr(c) for c in tc.fixed_ints]
            exp_vk = tc.k.to_bytes(4, "big") + len(fixed).to_bytes(4, "big") + \
                b"".join(ref.o.g1_compress(c) for c in pkr["fixed_commitments"] + pkr["sigma_commitments"])
            assert out["vk"] == exp_vk, f"rank {r} of {P}: vk bytes; {tc.describe()}"


RANDOM_SEEDS = range(32)


def ranks_for(seed):
    return (2, 3, 4, 16) if seed % 8 == 0 else (2, 3, 4)


@pytest.mark.parametrize("seed", RANDOM_SEEDS)
def test_random_circuit_on_ranks(seed, monkeypatch):
    """the random corpus proved by groups of 2, 3 and 4 ranks (16 for every eighth seed): every rank's bytes == the oracle's.  With 3
    ranks also device keygen (sigma columns, vk bytes); every eighth seed again with the columns uploaded ahead and without the coset
    cache."""
    tc = RandomCircuit(seed)
    ref, pkr, proof_ref, ok, cols = oracle_prove_columns(tc)
    assert ok, f"the oracle rejects its own proof: {tc.describe()}"
    for P in ranks_for(seed):
        outs = prove_on_ranks(tc, ref, pkr, cols, P, keygen=P == 3, again=P == 3 and seed % 8 == 0)
        check_ranks(tc, ref, pkr, proof_ref, outs, P)
    if seed % 8 == 0:
        monkeypatch.setenv("ZKB_COSET_CACHE_GB", "0")
        check_ranks(tc, ref, pkr, proof_ref, prove_on_ranks(tc, ref, pkr, cols, 3), 3)


K14_SEEDS = (1, 3)    # blake2b and poseidon transcripts


@pytest.mark.parametrize("seed", K14_SEEDS)
def test_point_range_single_commitments(seed):
    """at n = 2^14 a single commitment is sharded by point range across the ranks: the random polynomial and both SHPLONK
    commitments of every proof, and the vk commitment of a circuit with one fixed column and no permutation"""
    from zkb200 import plonk as Z
    tc = RandomCircuit(seed, k=14)
    assert tc.n == 1 << 14
    ref, pkr, proof_ref, ok, cols = oracle_prove_columns(tc)
    assert ok, tc.describe()
    for P in (2, 3):
        check_ranks(tc, ref, pkr, proof_ref, prove_on_ranks(tc, ref, pkr, cols, P), P)
    # one fixed column, no sigma: zkb_pk_vk_bytes commits exactly one column
    F = ref.F
    cs = Z.ConstraintSystem(14, 1, 1, 0, [0], [], 5, 3)
    cs.gates = [Z.Expression.Fixed(0) * Z.Expression.Advice(0)]
    cs.advice_queries, cs.fixed_queries = [(0, 0)], [(0, 0)]
    rnd = random.Random(seed)
    fixed = F.arr([rnd.randrange(R) for _ in range(tc.n)])
    want = tc.k.to_bytes(4, "big") + (1).to_bytes(4, "big") + bytes(ref.o.g1_compress(ref.commit_lagrange(fixed)))
    for P in (2, 3):
        def fn(r, ctx):
            pk = Z.ProvingKey(cs, [fixed], [], ref.g, ref.g_lagrange, ctx=ctx)
            try:
                return pk.vk_bytes()
            finally:
                pk.close()
        for r, vk in enumerate(on_ranks(P, fn)):
            assert vk == want, f"rank {r} of {P}: vk of the one-column circuit"


def test_super_standin_k13_on_four_ranks():
    """the k = 13 SuperCircuit stand-in (3 phases, the instance column in the permutation) proved by 4 ranks == the oracle's bytes"""
    import standins
    from zkb200 import plonk as Z
    from test_gpu_prover_wide import to_oracle_cs
    k = 13
    sc = standins.super_shape(k, seed=k, advice=64, scale=1.0, n_gates=120)
    assert sc.cs.num_phases() == 3 and sc.cs.num_instance == 1 and any(t == 3 for t, _ in sc.cs.perm_columns)
    cs = to_oracle_cs(sc.cs)
    ref = H.Ref(cs, 4321)
    F, h, n, bf = ref.F, sc.host, sc.n, sc.bf
    fixed = [h(t) for t in sc.fixed]
    sigma = [h(t) for t in sc.sigma]
    inst = [h(t) for t in sc.instances]
    pkr = {"fixed_values": fixed, "fixed_polys": [ref.lagrange_to_coeff(v) for v in fixed], "sigma_values": sigma,
           "sigma_polys": [ref.lagrange_to_coeff(v) for v in sigma]}
    l0 = np.zeros((n, 4), dtype=np.uint64); l0[0] = ref.w_arr(1)
    lb = np.zeros((n, 4), dtype=np.uint64); lb[n - bf:] = ref.w_arr(1)
    ll = np.zeros((n, 4), dtype=np.uint64); ll[n - bf - 1] = ref.w_arr(1)
    pkr["l0"], pkr["l_last"], pkr["l_blind"] = [ref.lagrange_to_coeff(v) for v in (l0, ll, lb)]
    pkr["fixed_commitments"] = [ref.commit_lagrange(v) for v in fixed]
    pkr["sigma_commitments"] = [ref.commit_lagrange(v) for v in sigma]
    zb, pb, rp = h(sc.z_blinds), h(sc.phi_blinds), h(sc.random_poly)
    blinds = {"z": [F.ints(zb[i * bf:(i + 1) * bf]) for i in range(sc.nsets)], "phi": [F.ints(pb[i * bf:(i + 1) * bf]) for i in range(sc.L)],
              "random_poly": rp}
    trep = F.ints(h(sc.transcript_repr[None]))[0]

    columns = {}

    def synth_ref_cached(phase, ch):
        columns[phase] = {c: h(t) for c, t in sc.synthesize_dev(phase, {i: F.arr([v])[0] for i, v in ch.items()}).items()}
        return columns[phase]
    proof_ref, _ = ref.create_proof(pkr, trep, [F.ints(a) for a in inst], synth_ref_cached, blinds)
    tr = h(sc.transcript_repr[None])[0]

    def fn(r, ctx):
        # every rank squeezes the oracle's challenges (or its proof differs anyway): it is handed the columns the oracle proved
        pk = Z.ProvingKey(sc.cs, fixed, sigma, ref.g, ref.g_lagrange, ctx=ctx)
        try:
            return Z.create_proof(pk, tr, inst, lambda phase, ch: columns[phase], zb, pb, rp)
        finally:
            pk.close()
    for r, proof in enumerate(on_ranks(4, fn)):
        assert proof == proof_ref, f"rank {r} of 4: the k = 13 stand-in's proof differs from the oracle's"


# ---------------------------------------------------------------------------------------------------- what the cases deal
def dealt_shapes():
    """(name, P, {unit kind: count}, E) of every group the proof cases above run"""
    import standins
    out = []

    def add(name, cs, degree, k, P):
        E = H.Domain(k, degree).E
        nsets = -(-len(cs.perm_columns) // (degree - 2)) if cs.perm_columns else 0
        units = {"lookup": len(cs.lookups), "set": nsets, "part": E}
        for ph, cnt in collections.Counter(cs.advice_phase).items():
            units[f"phase {ph} column"] = cnt
        out.append((name, P, units, E))
    for seed in RANDOM_SEEDS:
        tc = RandomCircuit(seed)
        for P in ranks_for(seed):
            add(f"seed {seed}", tc.cs, tc.degree, tc.k, P)
    for seed in K14_SEEDS:
        tc = RandomCircuit(seed, k=14)
        for P in (2, 3):
            add(f"k = 14 seed {seed}", tc.cs, tc.degree, tc.k, P)
    return out


def test_cases_cover_the_dealing_edges():
    """computed from the shapes with parallel.Deal (the host mirror of prover.cu's Deal): across the proof cases a rank owns no unit
    of each dealt kind, a count of 1 turns dealing off, E = 16 is dealt over 3 ranks and there are more ranks than coset parts"""
    from zkb200.parallel import Deal
    seen = collections.Counter()
    for name, P, units, E in dealt_shapes():
        for kind, count in units.items():
            kind = "phase column" if kind.startswith("phase") else kind
            if count == 0:
                continue
            if count == 1:
                seen[f"one {kind}: not dealt"] += 1
                assert not Deal(count, 0, P).on
                continue
            if any(not any(Deal(count, r, P).mine(i) for i in range(count)) for r in range(P)):
                seen[f"a rank without a {kind}"] += 1
        seen["E = 16 over 3 ranks"] += E == 16 and P == 3
        seen["more ranks than coset parts"] += P > E
    want = ["a rank without a lookup", "a rank without a set", "a rank without a part", "a rank without a phase column",
            "one lookup: not dealt", "one set: not dealt", "one phase column: not dealt", "E = 16 over 3 ranks",
            "more ranks than coset parts"]
    missing = [w for w in want if not seen[w]]
    assert not missing, f"no case has: {missing}; have {dict(seen)}"


# ---------------------------------------------------------------------------------------------------- errors
def unsatisfied_cell(tc, lookup):
    """(phase-0 advice column, row, value) such that changing that cell leaves exactly lookup `lookup` unsatisfied, or None"""
    F = H.Ref(tc.cs, 0, build_srs=False).F
    ch = challenges_for(tc)
    cols = circuit_columns(tc, F, ch)
    for s in tc.set_info:
        if s["lookup"] != lookup:
            continue
        for col, rot in s["entries"]:
            if tc.cs.advice_phase[col] != 0:
                continue
            for row in range(0, tc.usable, 7):
                cell = (row + rot) % tc.n
                broken = {t: list(v) for t, v in cols.items()}
                broken[H.ADVICE][col] = cols[H.ADVICE][col].copy()
                broken[H.ADVICE][col][cell] = F.arr([0xBAD0BAD0BAD])[0]
                _, recs = oracle_check(tc, broken)
                failing = {rec[1] for rec in recs if rec[0] == 1}
                if failing == {lookup}:
                    return col, cell, 0xBAD0BAD0BAD
    return None


def test_unsatisfied_lookup_fails_on_every_rank():
    """one lookup input row outside the table, in a lookup of rank 0 and then in one of rank P - 1: every rank raises ZKB_ERR_ARG well
    within the timeout, the ranks that do not own it say that another rank reported it, and the same contexts then prove the
    satisfied circuit"""
    from zkb200 import lib, plonk as Z
    from zkb200.parallel import Deal
    P = 3
    tc = next(t for t in (RandomCircuit(s) for s in range(64)) if len(t.cs.lookups) >= 2 and Deal(len(t.cs.lookups), P - 1, P).mine(len(t.cs.lookups) - 1)
              and unsatisfied_cell(t, 0) and unsatisfied_cell(t, len(t.cs.lookups) - 1))
    nl = len(tc.cs.lookups)
    ref, pkr, proof_ref, ok, cols = oracle_prove_columns(tc)
    assert ok
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    zcs = to_product_cs(tc.cs, ref.bf, ref.d)
    for lookup, owner in ((0, 0), (nl - 1, P - 1)):
        assert Deal(nl, owner, P).mine(lookup)
        col, cell, value = unsatisfied_cell(tc, lookup)

        def synth_bad(ph, ch):
            ints = tc.advice_ints(ph, {i: F.ints(v[None])[0] for i, v in ch.items()})
            if col in ints:
                ints[col] = list(ints[col])
                ints[col][cell] = value
            return {c: F.arr(v) for c, v in ints.items()}

        def fn(r, ctx):
            pk = Z.ProvingKey(zcs, fixed, pkr["sigma_values"], ref.g, ref.g_lagrange, ctx=ctx)
            try:
                t0 = time.monotonic()
                try:
                    Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth_bad,
                                   np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]) if tc.blinds_ints["z"] else None,
                                   np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]), F.arr(tc.blinds_ints["random_poly"]),
                                   transcript=tc.transcript)
                    err = None
                except lib.ZkbError as e:
                    err = e
                return err, time.monotonic() - t0, prove_with(tc, ref, pk, cols)
            finally:
                pk.close()
        for r, (err, secs, proof) in enumerate(on_ranks(P, fn, timeout_ms=60000)):
            assert err is not None, f"rank {r}: a proof of an unsatisfied lookup {lookup} (rank {owner}'s) succeeded"
            assert error_code(err) == ZKB_ERR_ARG, f"rank {r}: {err}"
            assert secs < 30, f"rank {r} took {secs:.1f} s to fail"
            if r == owner:
                assert f"lookup {lookup}:" in str(err), f"rank {r}: {err}"
            else:
                assert "reported by another rank" in str(err), f"rank {r}: {err}"
            assert_same_proof(tc, proof, proof_ref, f"rank {r} of {P}: the satisfied proof after the failed one")


def test_missing_rank_times_out_and_poisons_the_group():
    """rank 0 runs a sharded MSM and rank 1 nothing: rank 0's first meeting waits 2 s and fails with ZKB_ERR_STATE; after that every
    collective of the group fails at once.  Only the host waits: no device work waits for rank 1."""
    from zkb200 import arithmetic as A, lib, parallel
    from zkb200.params import g1_generator
    scal, bases = A.random_fr_dev(64, 1), A.g1_fixed_base_mul_dev(g1_generator(), A.random_fr_dev(64, 2))

    def fn(r, ctx):
        if r == 1:
            return None
        out = []
        for _ in range(2):
            t0 = time.monotonic()
            try:
                parallel.msm_sharded_dev(scal, bases, ctx=ctx)
                out.append((None, time.monotonic() - t0))
            except lib.ZkbError as e:
                out.append((e, time.monotonic() - t0))
        return out
    (e1, s1), (e2, s2) = on_ranks(2, fn, timeout_ms=2000)[0]
    assert e1 is not None and error_code(e1) == ZKB_ERR_STATE and "waited more than 2000 ms" in str(e1), e1
    assert 1.5 < s1 < 30, s1
    assert e2 is not None and error_code(e2) == ZKB_ERR_STATE and s2 < 1.0, (e2, s2)


def test_ranks_calling_different_collectives_all_fail():
    """rank 0 all-gathers 64 bytes (sharded MSM), rank 1 all-reduces 8 bytes (the barrier before the sharded NTT's window): both fail
    with ZKB_ERR_STATE at that collective, before any copy is queued, and the message names both calls"""
    import torch
    from zkb200 import arithmetic as A, lib, parallel
    from zkb200.params import g1_generator
    scal, bases = A.random_fr_dev(64, 1), A.g1_fixed_base_mul_dev(g1_generator(), A.random_fr_dev(64, 2))
    x = A.random_fr_dev(8, 3)

    def fn(r, ctx):
        try:
            if r == 0:
                parallel.msm_sharded_dev(scal, bases, ctx=ctx)
            else:
                parallel.ntt_sharded_dev(x, 4, A.root_of_unity(4)[0], 0, ctx=ctx)
        except lib.ZkbError as e:
            return e
        return None
    for r, e in enumerate(on_ranks(2, fn, timeout_ms=30000)):
        assert e is not None and error_code(e) == ZKB_ERR_STATE, f"rank {r}: {e}"
        msg = str(e)
        assert "disagree at collective #0" in msg and "all-gather of 64 bytes" in msg and "u64 all-reduce of 8 bytes" in msg, msg
    torch.cuda.synchronize()


def test_init_comm_local_arguments():
    import zkb200
    from zkb200 import lib
    ctxs = [zkb200.Context(0) for _ in range(17)]
    try:
        with pytest.raises(lib.ZkbError) as ei:
            zkb200.init_comm_local(ctxs)
        assert error_code(ei.value) == ZKB_ERR_ARG
        with pytest.raises(lib.ZkbError) as ei:
            zkb200.init_comm_local([ctxs[0], ctxs[0]])
        assert error_code(ei.value) == ZKB_ERR_ARG
        zkb200.init_comm_local(ctxs[:2])
        for group in ([ctxs[2], ctxs[0]], [ctxs[1]]):
            with pytest.raises(lib.ZkbError) as ei:
                zkb200.init_comm_local(group)
            assert error_code(ei.value) == ZKB_ERR_ARG and "already has a communicator" in str(ei.value)
        zkb200.init_comm_local(ctxs[2:18])     # 15 fresh contexts still form a group
    finally:
        for c in ctxs:
            c.close()


def test_init_comm_local_rejects_two_devices():
    import torch
    import zkb200
    from zkb200 import lib
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two devices")
    ctxs = [zkb200.Context(0), zkb200.Context(1)]
    try:
        with pytest.raises(lib.ZkbError) as ei:
            zkb200.init_comm_local(ctxs)
        assert error_code(ei.value) == ZKB_ERR_ARG
    finally:
        for c in ctxs:
            c.close()
