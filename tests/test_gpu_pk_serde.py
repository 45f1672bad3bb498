"""GPU: proving-key files (zkb_pk_vk_write, zkb_pk_write, zkb_pk_read; ProvingKey.write / ProvingKey.read).

- The bytes of every format equal the oracle's restated ProvingKey::write (pk_serde_ref.py), for keys made by device keygen and from
  host sigma columns, with and without the coset cache.
- A file read back (check on and off) gives the same vk and sigma columns, proves the original key's bytes and writes the same file;
  Processed -> RawBytes equals a direct RawBytes write.
- The k = 17, E = 16 case writes 2^21-element polynomials: chunk boundaries of ZKB_SERDE_CHUNK_POINTS.
- Faults are data: non-canonical elements in every section, derived elements that differ, wrong length prefixes, truncated input
  and a failing writer, each with its report and code, and the context proves afterwards.
- Two in-process ranks read one file and prove the same bytes."""
import io
import struct

import numpy as np
import pytest

import halo2_ref as H
import pyref as P
import pk_serde_ref as S
from circuits import ToyCircuit, ThinCompressionShape, GatesOnlyCircuit
from random_circuit import RandomCircuit
from test_gpu_prover import to_product_cs
from test_gpu_random_circuits_large import LARGE_CASES
from test_gpu_ranks_one_device import on_ranks
from witness_ref import perm_copies

pytestmark = pytest.mark.gpu

FORMATS = [S.PROCESSED, S.RAW_BYTES, S.RAW_BYTES_UNCHECKED]
ERR_ARG, ERR_STATE = -2, -4

CIRCUITS = {
    "toy6": lambda: ToyCircuit(6, seed=3),
    "thin8": lambda: ThinCompressionShape(8, seed=208),
    "thin10": lambda: ThinCompressionShape(10, seed=210),
    "gates6": lambda: GatesOnlyCircuit(6, seed=4),
}
CIRCUITS.update({f"random{s}": (lambda s=s: RandomCircuit(s)) for s in range(0, 96, 12)})


class Case:
    """a circuit, its oracle keygen / proof / advice columns, the oracle's file bodies and the device-side handles"""

    def __init__(self, tc, prove=True):
        import keccak_ref as K
        from zkb200.params import ParamsKZG
        self.tc = tc
        self.transcript = getattr(tc, "transcript", "blake2b")
        ref = self.ref = H.Ref(tc.cs, 1234)
        F = ref.F
        self.fixed = [F.arr(c) for c in tc.fixed_ints]
        self.pkr = ref.keygen(self.fixed, tc.copies)
        self.zcs = to_product_cs(tc.cs, ref.bf, ref.d)
        self.items = S.body_polys(ref, self.pkr)
        self.cols = {}
        self.proof_ref = None
        if prove:
            blinds = {"z": tc.blinds_ints["z"], "phi": tc.blinds_ints["phi"], "random_poly": F.arr(tc.blinds_ints["random_poly"])}

            def synth(ph, ch):
                self.cols[ph] = {c: F.arr(v) for c, v in tc.advice_ints(ph, ch).items()}
                return self.cols[ph]
            writer = {"blake2b": None, "poseidon": H.Ref.PoseidonTranscript(ref), "evm": K.EvmTranscript(ref)}[self.transcript]
            self.proof_ref, _ = ref.create_proof(self.pkr, tc.transcript_repr, tc.instances, synth, blinds, transcript=writer)
            reader = {"blake2b": None, "poseidon": H.Ref.PoseidonReader(self.proof_ref), "evm": K.EvmTranscript(proof=self.proof_ref)}[self.transcript]
            assert ref.verify_proof(self.pkr, tc.transcript_repr, tc.instances, self.proof_ref, reader=reader)
        self.params = ParamsKZG(tc.cs.k, ref.g, ref.g_lagrange)
        self.srs = self.params.load()

    def expected(self, fmt):
        return S.pk_write(self.ref, self.pkr, fmt, self.items)

    def key(self, keygen=False, srs=None, ctx=None):
        from zkb200 import plonk as Z
        srs = srs or self.srs
        if keygen:
            return Z.ProvingKey(self.zcs, self.fixed, None, srs=srs, copies=perm_copies(self.tc.cs, self.tc.copies))
        return Z.ProvingKey(self.zcs, self.fixed, self.pkr["sigma_values"], srs=srs)

    def prove(self, pk):
        from zkb200 import plonk as Z
        F, tc = self.ref.F, self.tc
        zb = np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]) if tc.blinds_ints["z"] else None
        pb = np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]) if tc.blinds_ints["phi"] else None
        return Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], lambda ph, ch: self.cols[ph], zb, pb,
                              F.arr(tc.blinds_ints["random_poly"]), transcript=self.transcript)

    def offset(self, fmt, section, column, index):
        return S.element_offset(self.tc.cs.k, self.ref.dom.extended_k, self.tc.cs.num_fixed, len(self.tc.cs.perm_columns), fmt, section,
                                column, index)

    def columns(self, section):
        return 1 if section < 3 else (self.tc.cs.num_fixed if section < 6 else len(self.tc.cs.perm_columns))

    def length(self, section):
        return self.tc.cs.n if S.SECTIONS[section][1] == "n" else self.ref.dom.N


def write(pk, fmt):
    buf = io.BytesIO()
    pk.write(buf, fmt)
    return buf.getvalue()


def read(case, data, fmt, check, srs=None):
    from zkb200 import plonk as Z
    return Z.ProvingKey.read(io.BytesIO(data), case.zcs, srs or case.srs, fmt, check=check)


def assert_same_key(case, pk, pk0, what):
    assert pk.vk_bytes() == pk0.vk_bytes(), what
    for i in range(len(case.tc.cs.perm_columns)):
        assert (pk.sigma_values(i) == case.pkr["sigma_values"][i]).all(), f"{what}: sigma column {i}"


@pytest.mark.parametrize("name", list(CIRCUITS))
def test_bytes_equal_oracle_and_round_trip(name):
    case = Case(CIRCUITS[name]())
    pk_kg, pk = case.key(keygen=True), case.key()
    try:
        files = {}
        for fmt in FORMATS:
            exp = files[fmt] = case.expected(fmt)
            assert write(pk_kg, fmt) == exp, f"{name}: keygen key, format {fmt}"
            assert write(pk, fmt) == exp, f"{name}: key from sigma values, format {fmt}"
            assert pk.vk_write(fmt) == exp[: len(pk.vk_write(fmt))]
        assert pk.vk_write(S.PROCESSED) == pk.vk_bytes()
        assert case.prove(pk) == case.proof_ref
        for fmt in FORMATS:
            for check in (False, True):
                what = f"{name}: format {fmt}, check {check}"
                pk2 = read(case, files[fmt], fmt, check)
                try:
                    assert_same_key(case, pk2, pk, what)
                    assert case.prove(pk2) == case.proof_ref, what
                    assert write(pk2, fmt) == files[fmt], what
                    if fmt == S.PROCESSED:
                        assert write(pk2, S.RAW_BYTES) == files[S.RAW_BYTES], what
                finally:
                    pk2.close()
    finally:
        pk_kg.close()
        pk.close()


@pytest.mark.parametrize("name", ["toy6", "random36"])
def test_without_the_coset_cache(name, monkeypatch):
    """extended forms computed per column into the scratch (write) and against it (checked read) give the same bytes and proofs"""
    case = Case(CIRCUITS[name]())
    monkeypatch.setenv("ZKB_COSET_CACHE_GB", "0")
    pk = case.key()
    try:
        for fmt in FORMATS:
            data = write(pk, fmt)
            assert data == case.expected(fmt), fmt
            pk2 = read(case, data, fmt, True)
            try:
                assert case.prove(pk2) == case.proof_ref
            finally:
                pk2.close()
    finally:
        pk.close()


def test_chunk_boundaries_k17():
    """k = 17, E = 16: every extended polynomial has 2^21 > ZKB_SERDE_CHUNK_POINTS elements"""
    seed, kw, _ = next(c for c in LARGE_CASES if c[1]["k"] == 17)
    case = Case(RandomCircuit(seed, **kw), prove=False)
    assert case.ref.dom.E == 16 and case.ref.dom.N == 1 << 21
    pk = case.key()
    try:
        data = write(pk, S.RAW_BYTES)
        assert data == case.expected(S.RAW_BYTES)
        pk2 = read(case, data, S.RAW_BYTES, True)
        try:
            assert_same_key(case, pk2, pk, "k = 17")
            assert write(pk2, S.RAW_BYTES) == data
        finally:
            pk2.close()
    finally:
        pk.close()


@pytest.fixture(scope="module")
def toy():
    return Case(CIRCUITS["toy6"]())


def read_error(case, data, fmt, check):
    from zkb200.lib import ZkbError
    with pytest.raises(ZkbError) as ei:
        read(case, data, fmt, check).close()
    return ei.value


def put(data, off, raw):
    b = bytearray(data)
    b[off: off + 32] = raw
    return bytes(b)


@pytest.mark.parametrize("fmt", [S.PROCESSED, S.RAW_BYTES])
def test_non_canonical_element_in_every_section(toy, fmt):
    case = toy
    good = case.expected(fmt)
    bad_value = P.R_MOD.to_bytes(32, "little")          # r: canonical form and stored integer both >= r
    for section in range(9):
        cols = case.columns(section)
        if not cols:
            continue
        col, length = cols - 1, case.length(section)
        first = length // 3 + 1
        data = put(put(good, case.offset(fmt, section, col, first), bad_value), case.offset(fmt, section, col, length - 1), bad_value)
        for check in (False, True):
            e = read_error(case, data, fmt, check)
            assert f"error {ERR_ARG}" in str(e)
            assert e.report == (section, col, 2, first, 2), (section, check, e.report, str(e))
        if fmt == S.RAW_BYTES:   # the same bytes are accepted unchecked
            read(case, data, S.RAW_BYTES_UNCHECKED, False).close()


def test_mismatching_derived_elements(toy):
    from zkb200.lib import ZkbError
    case = toy
    fmt = S.RAW_BYTES
    good = case.expected(fmt)
    for section, col, idx in ((4, 0, 5), (5, case.columns(5) - 1, case.length(5) - 1), (8, 0, 0), (8, case.columns(8) - 1, 12345 % case.length(8)),
                              (0, 0, 1), (2, 0, 7)):
        off = case.offset(fmt, section, col, idx)
        v = P.from_limbs(np.frombuffer(good[off: off + 32], dtype="<u8"))
        data = put(good, off, ((v + 1) % P.R_MOD).to_bytes(32, "little"))
        e = read_error(case, data, fmt, True)
        assert e.report == (section, col, 4, idx, 1), (section, e.report, str(e))
        pk = read(case, data, fmt, False)    # unchecked: the file's derived forms are not used
        try:
            assert case.prove(pk) == case.proof_ref
            assert write(pk, fmt) == good
        finally:
            pk.close()


def test_bad_lengths_truncation_and_writer_errors(toy):
    from zkb200.lib import ZkbError
    case = toy
    fmt = S.PROCESSED
    good = case.expected(fmt)
    # a wrong polynomial length and a wrong slice count
    off = case.offset(fmt, 5, 0, 0) - 4
    data = good[:off] + struct.pack(">I", case.length(5) // 2) + good[off + 4:]
    e = read_error(case, data, fmt, False)
    assert f"error {ERR_ARG}" in str(e) and "fixed_cosets" in str(e) and e.report[:2] == (5, 0)
    off = case.offset(fmt, 6, 0, 0) - 8
    data = good[:off] + struct.pack(">I", case.columns(6) + 1) + good[off + 4:]
    e = read_error(case, data, fmt, False)
    assert f"error {ERR_ARG}" in str(e) and "permutation values" in str(e) and e.report[0] == 6
    # truncated inside section 7, and inside the vk
    e = read_error(case, good[: case.offset(fmt, 7, 0, 3) + 5], fmt, True)
    assert f"error {ERR_ARG}" in str(e) and "ends inside section 7" in str(e)
    e = read_error(case, good[:20], fmt, False)
    assert "vk" in str(e)
    # a vk for another circuit
    e = read_error(case, struct.pack(">I", case.tc.cs.k + 1) + good[4:], fmt, False)
    assert "k = " in str(e)

    # a writer that fails part-way
    class Failing(io.RawIOBase):
        def __init__(self, limit):
            self.n, self.limit = 0, limit

        def write(self, b):
            self.n += len(b)
            if self.n > self.limit:
                raise OSError("disk full")
            return len(b)
    pk = case.key()
    try:
        with pytest.raises(ZkbError) as ei:
            pk.write(Failing(len(good) // 2), fmt)
        assert f"error {ERR_STATE}" in str(ei.value) and isinstance(ei.value.__cause__, OSError)
        # the same context proves afterwards, from a file read back
        pk2 = read(case, good, fmt, True)
        try:
            assert case.prove(pk2) == case.proof_ref
        finally:
            pk2.close()
        assert case.prove(pk) == case.proof_ref
    finally:
        pk.close()
    nxt = Case(CIRCUITS["thin8"]())
    pk3 = read(nxt, nxt.expected(S.RAW_BYTES_UNCHECKED), S.RAW_BYTES_UNCHECKED, False)
    try:
        assert nxt.prove(pk3) == nxt.proof_ref
    finally:
        pk3.close()


def test_two_ranks_read_one_file():
    """zkb_pk_read is collective: two in-process ranks read the same bytes and prove the oracle's proof; a bad copy on one rank fails
    both"""
    from zkb200 import plonk as Z
    from zkb200.lib import ZkbError
    case = Case(CIRCUITS["random24"]())
    fmt = S.PROCESSED
    data = case.expected(fmt)
    bad = put(data, case.offset(fmt, 3, 0, 2), P.R_MOD.to_bytes(32, "little"))

    def fn(r, ctx, blob):
        srs = case.params.load(ctx=ctx)
        try:
            pk = Z.ProvingKey.read(io.BytesIO(blob(r)), case.zcs, srs, fmt, check=True)
            try:
                return case.prove(pk)
            finally:
                pk.close()
        except ZkbError as e:
            return e
        finally:
            srs.close()
    outs = on_ranks(2, lambda r, ctx: fn(r, ctx, lambda _: data))
    assert outs == [case.proof_ref, case.proof_ref]
    outs = on_ranks(2, lambda r, ctx: fn(r, ctx, lambda r: bad if r == 0 else data))
    assert all(isinstance(o, ZkbError) for o in outs), outs
    assert outs[0].report == (3, 0, 2, 2, 1) and "another rank" in str(outs[1])
