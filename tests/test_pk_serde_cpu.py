"""CPU: the proving-key file layout restated in pk_serde_ref.py (ProvingKey::write) -- its lengths in every format, its vk prefix
against the oracle's vk bytes and the reference fixture's vk, its Fr encodings against pyref -- and the C ABI's new symbols."""
import random
import struct

import numpy as np
import pytest

import halo2_ref as H
import pyref as P
import pk_serde_ref as S
from circuits import ToyCircuit, GatesOnlyCircuit

FORMATS = [S.PROCESSED, S.RAW_BYTES, S.RAW_BYTES_UNCHECKED]


@pytest.fixture(scope="module")
def toy():
    tc = ToyCircuit(5, seed=11)
    ref = H.Ref(tc.cs, 1234)
    pk = ref.keygen([ref.F.arr(c) for c in tc.fixed_ints], tc.copies)
    return tc, ref, pk, S.body_polys(ref, pk)


def test_empty_slices_keep_their_count():
    """a circuit without permutation columns still writes the three permutation slice counts (0)"""
    tc = GatesOnlyCircuit(5, seed=4)
    assert not tc.cs.perm_columns
    ref = H.Ref(tc.cs, 1234)
    pk = ref.keygen([ref.F.arr(c) for c in tc.fixed_ints], tc.copies)
    data = S.pk_write(ref, pk, S.PROCESSED)
    _, total = S.layout(tc.cs.k, ref.dom.extended_k, tc.cs.num_fixed, 0, S.PROCESSED)
    assert len(data) == total and data[-12:] == bytes(12)


@pytest.mark.parametrize("fmt", FORMATS)
def test_oracle_layout_lengths(toy, fmt):
    """every length prefix sits where layout() puts it and says what the constraint system needs; the file ends after section 8"""
    tc, ref, pk, items = toy
    data = S.pk_write(ref, pk, fmt, items)
    nf, npm = tc.cs.num_fixed, len(tc.cs.perm_columns)
    entries, total = S.layout(tc.cs.k, ref.dom.extended_k, nf, npm, fmt)
    assert len(data) == total
    assert len(entries) == 3 + 3 * nf + 3 * npm
    for sec, col, pos, length in entries:
        assert struct.unpack(">I", data[pos - 4: pos])[0] == length, (sec, col)
        assert length == (tc.cs.n if S.SECTIONS[sec][1] == "n" else ref.dom.N)
        if col == 0 and sec >= 3:
            assert struct.unpack(">I", data[pos - 8: pos - 4])[0] == (nf if sec < 6 else npm), sec
    for (sec, col, pos, length), (sec2, col2, arr) in zip(entries, items):
        assert (sec, col) == (sec2, col2)
        assert data[pos: pos + 32 * length] == S.fr_bytes(arr, fmt, ref)


def test_processed_vk_prefix_is_the_oracle_vk(toy):
    tc, ref, pk, items = toy
    exp = tc.cs.k.to_bytes(4, "big") + len(tc.fixed_ints).to_bytes(4, "big") + b"".join(
        ref.o.g1_compress(c) for c in pk["fixed_commitments"] + pk["sigma_commitments"])
    assert S.pk_write(ref, pk, S.PROCESSED, items)[: len(exp)] == exp
    raw = S.pk_write(ref, pk, S.RAW_BYTES, items)
    pts = pk["fixed_commitments"] + pk["sigma_commitments"]
    assert raw[:8] == exp[:8]
    for i, aff in enumerate(pts):
        assert raw[8 + 64 * i: 72 + 64 * i] == np.ascontiguousarray(aff, dtype="<u8").tobytes()


def test_vk_prefix_length_matches_the_fixture(golden):
    """the reference's vk (k = 25, 4 fixed and 3 permutation commitments: 232 B) is the layout's vk prefix"""
    vk = bytes.fromhex(golden["vk_hex"])
    k, nf = struct.unpack(">II", vk[:8])
    npm = (len(vk) - 8) // 32 - nf
    assert (len(vk), k, nf, npm) == (232, 25, 4, 3)
    entries, _ = S.layout(k, k + 3, nf, npm, S.PROCESSED)
    assert entries[0][2] == len(vk) + 4


def test_fr_encodings_against_pyref(toy):
    _, ref, _, _ = toy
    rng = random.Random(5)
    vals = [0, 1, 2, P.R_MOD - 1, P.FR_ZETA, P.FR_DELTA] + [rng.randrange(P.R_MOD) for _ in range(64)]
    arr = ref.F.arr(vals)
    proc = S.fr_bytes(arr, S.PROCESSED, ref)
    raw = S.fr_bytes(arr, S.RAW_BYTES, ref)
    assert S.fr_bytes(arr, S.RAW_BYTES_UNCHECKED, ref) == raw
    for i, v in enumerate(vals):
        assert proc[32 * i: 32 * i + 32] == v.to_bytes(32, "little")
        assert raw[32 * i: 32 * i + 32] == S.montgomery_bytes(v)
        assert raw[32 * i: 32 * i + 32] == np.array(P.limbs(P.to_mont(v, P.R_MOD)), dtype="<u8").tobytes()


def test_extended_order_is_coset_part_major_by_index():
    """extended index m = the value at zeta * w_ext^m: part j = m mod E, row i = m / E (part j's generator is zeta * w_ext^j)"""
    tc = GatesOnlyCircuit(4, seed=1)
    ref = H.Ref(tc.cs, 99, build_srs=False)
    dom = ref.dom
    rng = random.Random(1)
    coeffs = [rng.randrange(P.R_MOD) for _ in range(tc.cs.n)]
    ext = ref.F.ints(ref.coeff_to_extended(ref.F.arr(coeffs)))

    def ev(x):
        acc = 0
        for c in reversed(coeffs):
            acc = (acc * x + c) % P.R_MOD
        return acc
    for m in (0, 1, dom.E - 1, dom.E, dom.N - 1, rng.randrange(dom.N)):
        j, i = m % dom.E, m // dom.E
        x = P.FR_ZETA * pow(dom.extended_omega, j, P.R_MOD) * pow(dom.omega, i, P.R_MOD) % P.R_MOD
        assert ext[m] == ev(x)


def test_abi_symbols_exported():
    import zkb200
    from zkb200 import lib as zl
    lib = zkb200.load_library()
    for name in ("zkb_pk_vk_write", "zkb_pk_write", "zkb_pk_read"):
        assert hasattr(lib, name) and name in zl.SIGNATURES
    assert lib.zkb_version() == (1 << 16) | 7
