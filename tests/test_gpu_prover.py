"""GPU parity for create_proof: the CUDA proving session must emit byte-identical proofs to the CPU oracle's restated
halo2 prover on the same witness / blinding / transcript_repr, and the oracle verifier must accept them."""
import numpy as np
import pytest

import halo2_ref as H
from circuits import ToyCircuit, ThinCompressionShape, GatesOnlyCircuit, DeepGateCircuit

pytestmark = pytest.mark.gpu


def to_product_cs(cs, bf, degree):
    from zkb200 import plonk as Z

    def conv(e, F):
        op = e.op
        if op == H.CONST: return Z.Expression.Constant(F.arr([e.a])[0])
        if op == H.FIXED: return Z.Expression.Fixed(e.a, e.b)
        if op == H.ADVICE: return Z.Expression.Advice(e.a, e.b)
        if op == H.INSTANCE: return Z.Expression.Instance(e.a, e.b)
        if op == H.CHALLENGE: return Z.Expression.Challenge(e.a)
        if op == H.NEG: return -conv(e.a, F)
        if op == H.ADD: return conv(e.a, F) + conv(e.b, F)
        if op == H.MUL: return conv(e.a, F) * conv(e.b, F)
        if op == H.SCALED: return conv(e.a, F).scaled(F.arr([e.b])[0])
        raise ValueError
    F = H.FA()
    z = Z.ConstraintSystem(cs.k, cs.num_fixed, cs.num_advice, cs.num_instance, cs.advice_phase, cs.challenge_phase, bf, degree)
    z.gates = [conv(g, F) for g in cs.gates]
    z.lookups = [([[conv(e, F) for e in inp] for inp in lk.inputs], [conv(e, F) for e in lk.table]) for lk in cs.lookups]
    z.perm_columns = list(cs.perm_columns)
    z.advice_queries, z.fixed_queries, z.instance_queries = list(cs.advice_queries), list(cs.fixed_queries), list(cs.instance_queries)
    return z


def first_diff(a, b):
    for i in range(0, min(len(a), len(b)), 32):
        if a[i:i + 32] != b[i:i + 32]: return i // 32
    return None if len(a) == len(b) else min(len(a), len(b)) // 32


CASES = [("toy", 5, {}), ("toy", 6, dict(two_phase=False)), ("toy", 6, dict(lookups=False, extra_perm=False)), ("toy", 8, {}), ("toy", 11, {}),
         ("thin", 7, {}), ("thin", 10, {}), ("gates", 5, {}), ("gates", 9, {}), ("deep", 6, {}), ("deep", 9, {})]


@pytest.mark.parametrize("kind,k,kw", CASES)
def test_create_proof_matches_oracle(kind, k, kw):
    from zkb200 import plonk as Z
    tc = {"toy": ToyCircuit, "thin": ThinCompressionShape, "gates": GatesOnlyCircuit, "deep": DeepGateCircuit}[kind](k, seed=100 + k, **kw)
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": rp}
    synth_ref = lambda phase, ch: {c: F.arr(v) for c, v in tc.advice_ints(phase, ch).items()}
    proof_ref, dbg = ref.create_proof(pkr, tc.transcript_repr, tc.instances, synth_ref, blinds)
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof_ref)

    zcs = to_product_cs(tc.cs, ref.bf, ref.d)
    pk = Z.ProvingKey(zcs, fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)

    def synth(phase, ch):
        chi = {i: F.ints(v[None])[0] for i, v in ch.items()}
        return {c: F.arr(v) for c, v in tc.advice_ints(phase, chi).items()}
    zb = np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]) if tc.blinds_ints["z"] else None
    pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]) if tc.blinds_ints["phi"] else None
    proof = Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth, zb, pb, rp)
    assert len(proof) == len(proof_ref)
    assert first_diff(proof, proof_ref) is None, f"first differing 32-byte proof item: {first_diff(proof, proof_ref)}"
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof)
    if kind == "deep":
        # the quotient program's register count is the maximum over its scopes: its gate part alone needs the local-memory build
        # (> 16 registers), so the proof above ran expr_kernel<64, 128, false>.  On the satisfied witness the folded gate is zero.
        import torch
        cols = [torch.from_numpy(np.ascontiguousarray(c).view(np.int64)).cuda() for c in fixed + [F.arr(v) for v in tc.advice_ints(0, {}).values()]]
        (h,), nregs = Z.expr_eval(zcs, cols, mode=1, y=F.arr([5])[0], scale=F.arr([1])[0])
        assert nregs >= 17
        assert not h.cpu().numpy().any()


def test_unsatisfied_lookup_is_reported():
    from zkb200 import plonk as Z, ZkbError
    tc = ToyCircuit(6, seed=7)
    # break a lookup input: d at a q_lk row gets a value outside the table
    for i in range(tc.usable):
        if tc.fixed_ints[2][i]:
            tc.cols0[3][i] = 123456789
            break
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    synth = lambda phase, ch: {c: F.arr(v) for c, v in tc.advice_ints(phase, {i: F.ints(v[None])[0] for i, v in ch.items()}).items()}
    zb = np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]); pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]])
    with pytest.raises(ZkbError):
        Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth, zb, pb, F.arr(tc.blinds_ints["random_poly"]))


def test_vk_bytes_processed_format():
    """keygen commitments on the GPU in the reference's SerdeFormat::Processed vk layout (fixture: u32 BE k, u32 BE #fixed, points)."""
    import pyref as P
    from zkb200 import plonk as Z
    tc = ToyCircuit(6, seed=3)
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    vk = pk.vk_bytes()
    assert int.from_bytes(vk[:4], "big") == 6 and int.from_bytes(vk[4:8], "big") == len(fixed)
    pts = pkr["fixed_commitments"] + pkr["sigma_commitments"]
    assert len(vk) == 8 + 32 * len(pts)
    for i, aff in enumerate(pts):
        assert vk[8 + 32 * i: 40 + 32 * i] == ref.o.g1_compress(aff)


@pytest.mark.parametrize("kind,k", [("toy", 6), ("thin", 8)])
def test_create_proof_poseidon_transcript_matches_oracle(kind, k):
    """gen_snark_shplonk's transcript: the CUDA session with the Poseidon transcript == the oracle's Poseidon prover byte for byte,
    and the fixture-pinned verifier (Poseidon reader) accepts it."""
    from zkb200 import plonk as Z
    tc = (ToyCircuit if kind == "toy" else ThinCompressionShape)(k, seed=200 + k)
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": rp}
    synth_ref = lambda phase, ch: {c: F.arr(v) for c, v in tc.advice_ints(phase, ch).items()}
    proof_ref, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, synth_ref, blinds, transcript=H.Ref.PoseidonTranscript(ref))
    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    synth = lambda phase, ch: {c: F.arr(v) for c, v in tc.advice_ints(phase, {i: F.ints(v[None])[0] for i, v in ch.items()}).items()}
    zb = np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]); pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]])
    proof = Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth, zb, pb, rp, transcript="poseidon")
    assert first_diff(proof, proof_ref) is None, f"first differing 32-byte proof item: {first_diff(proof, proof_ref)}"
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof, reader=H.Ref.PoseidonReader(proof))


@pytest.mark.parametrize("k", [5, 8])
def test_keygen_pk_matches_oracle_keygen(k):
    """zkb_keygen_pk: permutation assembly from the copy constraints + sigma columns on the device == the oracle's restated
    keygen (plonk/permutation/keygen.rs), vk bytes identical to the host-sigma path, and the pk proves byte-identically."""
    from zkb200 import plonk as Z
    from zkb200.params import ParamsKZG
    tc = ToyCircuit(k, seed=300 + k)
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    cidx = {c: i for i, c in enumerate(tc.cs.perm_columns)}
    copies = [(cidx[(lt, lc)], lr, cidx[(rt, rc)], rr) for (lt, lc, lr), (rt, rc, rr) in tc.copies]
    srs = ParamsKZG(k, ref.g, ref.g_lagrange).load()
    zcs = to_product_cs(tc.cs, ref.bf, ref.d)
    pk = Z.ProvingKey(zcs, fixed, None, srs=srs, copies=copies)
    for i in range(len(tc.cs.perm_columns)):
        assert (pk.sigma_values(i) == pkr["sigma_values"][i]).all(), f"sigma column {i}"
    pk_host = Z.ProvingKey(zcs, fixed, pkr["sigma_values"], srs=srs)        # two keys share one SRS handle
    assert pk.vk_bytes() == pk_host.vk_bytes()
    exp_vk = k.to_bytes(4, "big") + len(fixed).to_bytes(4, "big") + b"".join(ref.o.g1_compress(c) for c in pkr["fixed_commitments"] + pkr["sigma_commitments"])
    assert pk.vk_bytes() == exp_vk
    rp = F.arr(tc.blinds_ints["random_poly"])
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": rp}
    proof_ref, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, ch).items()}, blinds)

    def synth(phase, ch):
        chi = {i: F.ints(v[None])[0] for i, v in ch.items()}
        return {c: F.arr(v) for c, v in tc.advice_ints(phase, chi).items()}
    zb = np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]) if tc.blinds_ints["z"] else None
    pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]) if tc.blinds_ints["phi"] else None
    proof = Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth, zb, pb, rp)
    assert proof == proof_ref


def test_prove_finish_query_then_fetch():
    """header contract: proof_out == NULL queries the length, a short buffer fails WITHOUT losing the proof, a second call copies it"""
    import ctypes
    from zkb200 import plonk as Z
    from zkb200.lib import check
    tc = GatesOnlyCircuit(5, seed=3)
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    lib = pk.ctx.lib
    tr = np.ascontiguousarray(F.arr([tc.transcript_repr])[0])
    sess = ctypes.c_void_p()
    check(lib.zkb_prove_begin(pk.handle, ctypes.c_void_p(tr.ctypes.data), None, None, ctypes.byref(sess)))
    cols = {c: np.ascontiguousarray(F.arr(v)) for c, v in tc.advice_ints(0, {}).items()}
    tbl = (ctypes.c_void_p * tc.cs.num_advice)(*[cols[c].ctypes.data for c in range(tc.cs.num_advice)])
    check(lib.zkb_prove_advice_phase(sess, 0, ctypes.cast(tbl, ctypes.c_void_p), None))
    rp = np.ascontiguousarray(F.arr(tc.blinds_ints["random_poly"]))
    zb = np.ascontiguousarray(np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]])) if tc.blinds_ints["z"] else None
    n = ctypes.c_uint64(0)
    check(lib.zkb_prove_finish(sess, ctypes.c_void_p(zb.ctypes.data) if zb is not None else None, None, ctypes.c_void_p(rp.ctypes.data), None, 0, ctypes.byref(n)))
    assert n.value > 0
    small = (ctypes.c_uint8 * 8)()
    assert lib.zkb_prove_finish(sess, None, None, None, ctypes.cast(small, ctypes.c_void_p), 8, ctypes.byref(n)) != 0
    out = (ctypes.c_uint8 * n.value)()
    check(lib.zkb_prove_finish(sess, None, None, None, ctypes.cast(out, ctypes.c_void_p), n.value, ctypes.byref(n)))
    lib.zkb_session_destroy(sess)
    blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": F.arr(tc.blinds_ints["random_poly"])}
    proof_ref, _ = ref.create_proof(pkr, tc.transcript_repr, tc.instances, lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, ch).items()}, blinds)
    assert bytes(out) == proof_ref


def test_callers_transcript_through_callbacks_writes_the_same_proof():
    """create_proof's generic `T: TranscriptWrite` (SURVEY 8b): the session drives a transcript object that lives on the CALLER's side
    through zkb_transcript_vtable.  Here that object is the oracle's Blake2b transcript (hashlib): the bytes it writes must equal the
    proof of the in-library Blake2b session, and an exception raised inside a callback must surface as an error, not a crash."""
    from zkb200 import plonk as Z
    from zkb200.lib import ZkbError
    tc = ToyCircuit(7, seed=321)
    ref = H.Ref(tc.cs, 1234)
    F = ref.F
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], ref.g, ref.g_lagrange)
    synth = lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, {i: F.ints(v[None])[0] for i, v in ch.items()}).items()}
    args = (pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth,
            np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]), np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]), rp)
    proof_lib = Z.create_proof(*args)

    class Mine:
        def __init__(self): self.t = H.Ref.Transcript(ref); self.ops = 0
        def common_scalar(self, l): self.ops += 1; self.t.common_scalar(F.ints(l[None])[0])
        def write_scalar(self, l): self.ops += 1; self.t.write_scalar(F.ints(l[None])[0])
        def write_point(self, l): self.ops += 1; self.t.write_point(l)
        def squeeze_challenge(self): self.ops += 1; return F.arr([self.t.squeeze()])[0]
    # columns handed over one by one ahead of their phase (zkb_prove_upload_advice): same proof
    assert Z.create_proof(*args, upload_ahead=True) == proof_lib
    mine = Mine()
    out = Z.create_proof(*args, transcript=Z.CallbackTranscript(mine))
    assert out == b"" and bytes(mine.t.buf) == proof_lib and mine.ops > 20

    class Broken(Mine):
        def write_point(self, l): raise RuntimeError("writer full")
    cbt = Z.CallbackTranscript(Broken())
    with pytest.raises(ZkbError):
        Z.create_proof(*args, transcript=cbt)
    assert isinstance(cbt.error, RuntimeError)
