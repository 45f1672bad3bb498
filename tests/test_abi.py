"""CPU: the C-ABI library loads, exports every symbol include/zkb200.h declares, and fails loudly without a GPU."""
import os, re
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "zkb200.h")).read()
    return sorted(set(re.findall(r"ZKB_API[^;(]*?\b(zkb_\w+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    import zkb200
    from zkb200 import lib as zl
    names = declared_symbols()
    assert len(names) >= 20
    cdll = zkb200.load_library()
    for n in names:
        assert hasattr(cdll, n), f"{n} declared in include/zkb200.h but not exported"
        assert n in zl.SIGNATURES, f"{n} has no ctypes signature"
    assert sorted(zl.SIGNATURES) == names


def test_version():
    import zkb200
    assert zkb200.load_library().zkb_version() >> 16 == 1


def test_handles_outliving_their_context_are_not_destroyed():
    """Finalisers of garbage run in no fixed order: at interpreter exit the traceback of a failed proof test can keep a proving key
    alive past its context.  A key or SRS whose context is already destroyed must not reach zkb_pk_destroy / zkb_srs_destroy,
    which would read the freed context (a crash at exit)."""
    from zkb200 import lib as zl, plonk as Z, params
    calls = []

    class Lib:
        def __getattr__(self, name): return lambda *a: calls.append(name)
    ctx = zl.Context.__new__(zl.Context)
    ctx.lib, ctx.handle = Lib(), 1
    objs = [Z.ProvingKey.__new__(Z.ProvingKey), params.Srs.__new__(params.Srs), Z.ProvingKey.__new__(Z.ProvingKey)]
    for o in objs:
        o.ctx, o.handle = ctx, 2
    objs[0].close()
    ctx.close()
    objs[1].close(); objs[2].close()
    assert calls == ["zkb_pk_destroy", "zkb_destroy"]
    assert all(o.handle is None for o in objs)


def test_root_of_unity_matches_fixture(golden):
    import numpy as np
    from zkb200 import arithmetic
    w, wi = arithmetic.root_of_unity(golden["domain"]["k"])
    assert (w == np.array(golden["domain"]["gen"], dtype=np.uint64)).all()
    assert (wi == np.array(golden["domain"]["gen_inv"], dtype=np.uint64)).all()


def test_no_cpu_fallback():
    import torch, zkb200
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(zkb200.ZkbError):
        zkb200.Context(0)


def _toy_cs():
    from zkb200 import plonk as Z
    E = Z.Expression
    cs = Z.ConstraintSystem(5, 2, 2, 1, [0, 0], [], 5, 4)
    one = (0xac96341c4ffffffb, 0x36fc76959f60cd29, 0x666ea36f7879462e, 0x0e0a77c19a07df2f)
    cs.gates = [E.Fixed(0) * (E.Advice(0) * E.Advice(1, 1) + (-E.Instance(0))), (E.Advice(0) + E.Constant(one)).scaled(one)]
    cs.lookups = [([[E.Fixed(0) * E.Advice(1)]], [E.Fixed(1)])]
    cs.perm_columns = [(Z.ADVICE, 0), (Z.INSTANCE, 0)]
    cs.advice_queries, cs.fixed_queries, cs.instance_queries = [(0, 0), (1, 1), (1, 0)], [(0, 0), (1, 0)], [(0, 0)]
    return cs


def test_csf_roundtrip_and_validation():
    """The CSF blob (constraint system across the C ABI) is validated host-side: well-formed accepted, corrupt rejected."""
    import numpy as np
    import zkb200
    from zkb200 import plonk as Z
    blob = _toy_cs().to_csf()
    Z.validate_csf(blob)
    assert blob[0] == Z.CSF_MAGIC and blob[1] == 5 and blob[11] == 2 and blob[12] == 1 and blob[13] == 2
    for mutate in (lambda b: b.__setitem__(0, 0x12345678),          # bad magic
                   lambda b: b.__setitem__(3, 1),                    # fewer advice columns than the nodes reference
                   lambda b: b.__setitem__(9, int(b[9]) + 50),       # node count beyond the blob
                   lambda b: b.__setitem__(7, 2)):                   # degree below the permutation argument's
        bad = blob.copy()
        mutate(bad)
        with pytest.raises(zkb200.ZkbError):
            Z.validate_csf(bad)
    with pytest.raises(zkb200.ZkbError):
        Z.validate_csf(blob[:20])


def test_csf_rotation_limit():
    """The interpreter keeps a rotation in 16 bits: +-32767 is accepted, +-32768 is rejected, in a gate and in the query list."""
    import zkb200
    from zkb200 import plonk as Z
    E = Z.Expression
    for rot in (32767, -32767, 32768, -32768):
        for in_gate in (True, False):
            cs = Z.ConstraintSystem(3, 1, 1, 0, [0], [], 5, 3)
            cs.gates = [E.Fixed(0) * E.Advice(0, rot if in_gate else 0)]
            cs.advice_queries = [(0, 0 if in_gate else rot)]
            if abs(rot) <= 32767:
                Z.validate_csf(cs.to_csf())
            else:
                with pytest.raises(zkb200.ZkbError, match="16 bits"):
                    Z.validate_csf(cs.to_csf())



@pytest.mark.parametrize("kind", ["fixed", "advice"])
def test_csf_opening_point_limit(kind):
    """SHPLONK opens one column at most at 256 points x w^r (distinct rotations mod n): 256 are accepted, 257 are refused with the
    column and its count, 257 rotations of which two are equal mod n (r and r - n) make 256 points and are accepted."""
    import zkb200
    from zkb200 import plonk as Z
    E = Z.Expression
    k = 10
    n = 1 << k
    for rots, ok in ((list(range(-128, 128)), True), (list(range(-128, 129)), False), (list(range(-128, 128)) + [100 - n], True)):
        cs = Z.ConstraintSystem(k, 2, 2, 0, [0, 0], [], len(rots) + 2 if kind == "advice" else 5, 3)
        read = E.Fixed if kind == "fixed" else E.Advice
        body = read(1, rots[0])
        for r in rots[1:]:
            body = body + read(1, r)
        cs.gates = [E.Fixed(0) * (E.Advice(0) + body)]
        queries = [(0, 0), (1, 0)] + [(1, r) for r in rots if r != 0]
        cs.advice_queries, cs.fixed_queries = ([(0, 0)] + queries[1:], [(0, 0)]) if kind == "advice" else ([(0, 0)], queries)
        if ok:
            Z.validate_csf(cs.to_csf())
        else:
            with pytest.raises(zkb200.ZkbError, match=f"{kind} column 1 is opened at 257 points"):
                Z.validate_csf(cs.to_csf())

def test_params_file_roundtrip(tmp_path, oracle):
    """ParamsKZG file layout of the reference loader (prover/src/utils.rs:56-75): 4 B k | g | g_lagrange | g2 | s_g2, RawBytes."""
    import numpy as np
    import halo2_ref as H
    from zkb200.params import ParamsKZG
    k = 4
    ref = H.Ref(H.ConstraintSystem(k, 0, 1, 0).finalize(), 777)
    p = ParamsKZG(k, ref.g.copy(), ref.g_lagrange.copy(), bytes(range(128)), bytes(range(128, 256)))
    path = tmp_path / "params4"
    p.write_custom(str(path))
    assert path.stat().st_size == ParamsKZG.expected_file_len(k) == 4 + 2 * 16 * 64 + 2 * 128
    q = ParamsKZG.read_custom(str(path), to_device=False)
    assert q.k == k and (q.g == ref.g).all() and (q.g_lagrange == ref.g_lagrange).all()
    assert q.g2 == bytes(range(128)) and q.s_g2 == bytes(range(128, 256))
    # every stored point is a valid raw G1Affine (Montgomery x || y on the curve)
    assert all(oracle.g1_is_on_curve(pt) for pt in q.g)
    with open(path, "ab") as f:
        f.write(b"x")
    with pytest.raises(ValueError):
        ParamsKZG.read_custom(str(path), to_device=False)


def test_proof_container_matches_fixture(golden, tmp_path):
    """prover::Proof container (prover/src/proof.rs): the fixture's own chunk proof round-trips byte for byte, instances are
    32-byte big-endian words."""
    import base64
    from zkb200.proof_io import Proof, serialize_instances
    proof, inst, vk = bytes.fromhex(golden["proof_hex"]), bytes.fromhex(golden["instances_hex"]), bytes.fromhex(golden["vk_hex"])
    p = Proof(proof, inst, vk, golden["git_version"])
    vals = p.instances()
    assert len(vals) == 1 and len(vals[0]) == golden["num_instance"][0] == 44
    assert all(v < 21888242871839275222246405745257275088548364400416034343698204186575808495617 for v in vals[0])
    # the 32 public-input bytes of the chunk sit in the last 32 instance cells, each < 256 (SURVEY appendix B)
    assert all(v < 256 for v in vals[0][12:])
    assert serialize_instances(vals) == inst
    o = p.to_json_obj()
    assert base64.b64decode(o["proof"]) == proof and base64.b64decode(o["instances"]) == inst and base64.b64decode(o["vk"]) == vk
    p.dump(str(tmp_path), "chunk_0")
    q = Proof.from_json_file(str(tmp_path), "chunk_0")
    assert (q.proof, q.instances_raw, q.vk, q.git_version) == (proof, inst, vk, golden["git_version"])
    assert (tmp_path / "vk_chunk_0.vkey").read_bytes() == vk


def test_product_never_imports_the_oracle():
    """The product path must not route through oracle/ (only tests, smoke() and bench.py's baseline legs may)."""
    import re
    bad = re.compile(r"^\s*(import|from)\s+(oracle_lib|pyref|halo2_ref|oracle)\b", re.M)
    pkg = os.path.join(ROOT, "zkevm-circuits_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, fn), errors="ignore").read()
                assert not bad.search(src), fn
                assert "libzkoracle" not in src and "zko_" not in src, fn
    src = open(os.path.join(ROOT, "scripts", "proof_bench.py")).read()
    assert not bad.search(src)


def test_session_hashers_host_side(oracle):
    """The two transcripts of the proving session, pinned on the CPU: Poseidon vs the fixture-pinned restatement
    (oracle/poseidon_ref.py), Blake2b challenge vs hashlib."""
    import ctypes, hashlib, random
    import numpy as np
    import zkb200
    import pyref as P
    import poseidon_ref as PO
    lib = zkb200.load_library()
    rnd = random.Random(9)
    spec = PO.Spec(5, 8, 60)
    for n in (0, 1, 3, 4, 5, 8, 13):
        vals = [rnd.randrange(P.R_MOD) for _ in range(n)]
        a = np.array([P.limbs(P.to_mont(v, P.R_MOD)) for v in vals], dtype=np.uint64).reshape(-1, 4)
        out = np.zeros(4, dtype=np.uint64)
        assert lib.zkb_poseidon_hash_host(ctypes.c_void_p(a.ctypes.data) if n else None, n, ctypes.c_void_p(out.ctypes.data)) == 0
        sp = PO.Poseidon(spec)
        sp.update(vals)
        assert P.from_mont(P.from_limbs(out), P.R_MOD) == sp.squeeze()
    for ln in (0, 1, 32, 127, 128, 129, 300):
        data = bytes(rnd.randrange(256) for _ in range(ln))
        out = np.zeros(4, dtype=np.uint64)
        buf = (ctypes.c_uint8 * max(1, ln)).from_buffer_copy(data or b"\0")
        assert lib.zkb_blake2b_challenge_host(ctypes.cast(buf, ctypes.c_void_p) if ln else None, ln, ctypes.c_void_p(out.ctypes.data)) == 0
        h = hashlib.blake2b(digest_size=64, person=b"Halo2-Transcript")
        h.update(data + b"\x00")
        assert P.from_mont(P.from_limbs(out), P.R_MOD) == int.from_bytes(h.digest(), "little") % P.R_MOD


def test_transcript_framing_all_kinds(oracle):
    """The session's own transcript code (zkb_transcript_script_host replays it without a device) against the oracle's three
    transcripts on a scripted create_proof-like sequence: same proof bytes, same challenges.  Blake2b and Poseidon framing are also
    covered end to end by the GPU proof tests; the EVM/Keccak framing is pinned by KECCAK_CODE_HASH_EMPTY + this."""
    import ctypes, random
    import numpy as np
    import zkb200
    import pyref as P
    import halo2_ref as H
    import keccak_ref as K
    lib = zkb200.load_library()
    rnd = random.Random(77)
    vp = ctypes.c_void_p
    for ln in (0, 1, 135, 136, 137, 500):                                        # the hash itself
        data = bytes(rnd.randrange(256) for _ in range(ln))
        out = (ctypes.c_uint8 * 32)()
        buf = (ctypes.c_uint8 * max(1, ln)).from_buffer_copy(data or b"\0")
        assert lib.zkb_keccak256_host(ctypes.cast(buf, vp) if ln else None, ln, ctypes.cast(out, vp)) == 0
        assert bytes(out) == K.keccak256(data)
    # script: repr, instances, then rounds of points / squeezes / scalars, with back-to-back squeezes (beta, gamma) as in create_proof
    g = (1, 2)
    def aff_limbs(pt):
        return P.limbs(P.to_mont(pt[0], P.Q_MOD)) + P.limbs(P.to_mont(pt[1], P.Q_MOD))
    pts = [aff_limbs(P.g1_mul(g, rnd.randrange(1, P.R_MOD))) for _ in range(9)]
    ops, operands, script = [], [], []
    def sc(kind):
        v = rnd.randrange(P.R_MOD); ops.append(kind); operands.extend(P.limbs(P.to_mont(v, P.R_MOD))); script.append((kind, v))
    def pt(i):
        ops.append(2); operands.extend(int(x) for x in pts[i]); script.append((2, pts[i]))
    def sq():
        ops.append(3); script.append((3, None))
    sc(0); sc(0); sc(0)
    pt(0); pt(1); sq()
    pt(2); sq(); sq()
    pt(3); pt(4); pt(5); sq()
    for _ in range(7): sc(1)
    sq(); sq(); pt(6); sq(); sc(1); pt(7); sq(); sq(); sq(); pt(8)
    n_sq = sum(1 for o in ops if o == 3)
    opa = np.array(ops, dtype=np.uint8)
    opd = np.array(operands, dtype=np.uint64)

    class _O:                                                                     # the oracle transcripts only need g1_compress
        def __init__(self, o): self.o = o
    for kind, mk in ((0, lambda: H.Ref.Transcript(_O(oracle))), (1, lambda: H.Ref.PoseidonTranscript(_O(oracle))), (2, lambda: K.EvmTranscript())):
        t = mk()
        want_ch = []
        for k, v in script:
            if k == 0: t.common_scalar(v)
            elif k == 1: t.write_scalar(v)
            elif k == 2: t.write_point(np.array(v, dtype=np.uint64))
            else: want_ch.append(t.squeeze())
        plen = ctypes.c_uint64(0)
        ch = np.zeros((n_sq, 4), dtype=np.uint64)
        proof = (ctypes.c_uint8 * 4096)()
        rc = lib.zkb_transcript_script_host(kind, vp(opa.ctypes.data), len(ops), vp(opd.ctypes.data), ctypes.cast(proof, vp), 4096,
                                            ctypes.byref(plen), vp(ch.ctypes.data))
        assert rc == 0
        assert bytes(proof[: plen.value]) == bytes(t.buf), kind
        assert [P.from_mont(P.from_limbs(c), P.R_MOD) for c in ch] == want_ch, kind
    # identity points are refused by every kind, unknown kinds / ops too
    bad = np.zeros(8, dtype=np.uint64)
    one = np.array([2], dtype=np.uint8)
    plen = ctypes.c_uint64(0)
    for kind in (0, 1, 2):
        assert lib.zkb_transcript_script_host(kind, vp(one.ctypes.data), 1, vp(bad.ctypes.data), None, 0, ctypes.byref(plen), None) != 0
    assert lib.zkb_transcript_script_host(3, vp(one.ctypes.data), 0, None, None, 0, ctypes.byref(plen), None) != 0
