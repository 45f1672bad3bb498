"""CPU: [s]G2 of the SRS setup (zkb_g2_setup_host) against the oracle's affine G2 arithmetic, its encodings, and the
recoding model of the setup's fixed-base comb (tests/fixed_base_model.py)."""
import numpy as np
import pytest

import msm_model as M
import pairing_ref as E
import pyref as P
import fixed_base_model as FB

R, Q = P.R_MOD, P.Q_MOD
EDGE_S = [0, 1, 2, R - 1, R - 2, (1 << 253) + 1]
RANDOM_S = [sum(int(x) << (62 * j) for j, x in enumerate(row)) % R for row in np.random.default_rng(2024).integers(0, 1 << 62, size=(16, 5))]


def s_mont(s):
    return np.array(P.limbs(P.to_mont(s, R)), dtype=np.uint64)


def raw_to_point(raw):
    """raw 128-byte G2 point (Montgomery x.c0, x.c1, y.c0, y.c1) -> pairing_ref affine point, None for the identity"""
    v = np.frombuffer(raw, dtype=np.uint64).reshape(4, 4)
    c = [P.from_mont(P.from_limbs(row), Q) for row in v]
    if not any(c):
        return None
    return E.FQ2([c[0], c[1]]), E.FQ2([c[2], c[3]])


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return all(int(x) == int(y) for p, q in zip(a, b) for x, y in zip(p.c, q.c))


@pytest.mark.parametrize("s", EDGE_S + RANDOM_S)
def test_s_g2_matches_reference(s):
    from zkb200.params import g2_setup
    g2, s_g2 = g2_setup(s_mont(s))
    assert same(raw_to_point(g2), E.G2)
    assert same(raw_to_point(s_g2), E.g2_mul(E.G2, s))
    if s == 0:
        assert s_g2 == bytes(128)
    else:
        assert E.g2_is_on_curve(raw_to_point(s_g2))


@pytest.mark.parametrize("s", [3, R - 1, 0x1234567890ABCDEF ** 3 % R])
@pytest.mark.parametrize("fmt", ["Processed", "RawBytes"])
def test_g2_encoding_round_trip(s, fmt):
    from zkb200.params import SerdeFormat, g2_decode, g2_encode, g2_setup
    f = SerdeFormat[fmt]
    for raw in g2_setup(s_mont(s)):
        enc = g2_encode(f, raw)
        assert len(enc) == 2 * f.g1_len
        back, status = g2_decode(f, enc)
        assert status == 0 and back == raw


def test_s_outside_the_field_is_rejected():
    import ctypes
    import zkb200
    lib = zkb200.load_library()
    g2, s_g2 = np.full(16, 7, dtype=np.uint64), np.full(16, 7, dtype=np.uint64)
    for v in (R, (1 << 256) - 1):   # stored integers >= r
        s = np.array(P.limbs(v), dtype=np.uint64)
        rc = lib.zkb_g2_setup_host(ctypes.c_void_p(s.ctypes.data), ctypes.c_void_p(g2.ctypes.data), ctypes.c_void_p(s_g2.ctypes.data))
        assert rc == -2
        assert (g2 == 7).all() and (s_g2 == 7).all()


def _model_scalars(c):
    rng = np.random.default_rng(c)
    rand = [sum(int(x) << (62 * j) for j, x in enumerate(row)) % R for row in rng.integers(0, 1 << 62, size=(2000, 5))]
    return M.edge_scalars(c) + [0, 1, R - 1, FB.top_carry_scalar(c)] + rand


@pytest.mark.parametrize("c", sorted({c for c, _ in FB.COMB_VARIANTS}))
def test_comb_recoding_reconstructs_every_scalar(c):
    vals = _model_scalars(c)
    digits, idx, carry = FB.digits_and_indices(vals, c)
    g = FB.cfg(c)
    assert not carry.any(), "a carry left the top window"
    assert (np.abs(digits) <= g.half).all()
    assert FB.reconstruct(digits, c) == vals
    assert idx.max() < FB.table_size(c) == g.windows * g.half
    assert ((idx == -1) == (digits == 0)).all()


def test_top_carry_scalar_carries_into_the_top_window():
    c = FB.COMB_C
    g = FB.cfg(c)
    digits, idx, _ = FB.digits_and_indices([FB.top_carry_scalar(c)], c)
    assert digits[0, g.windows - 2] < 0 and digits[0, g.windows - 1] == 1
    assert idx[0, g.windows - 1] == (g.windows - 1) * g.half
