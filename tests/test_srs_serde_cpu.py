"""CPU: params file lengths per SerdeFormat, and the host G2 encodings (zkb_g2_decode_host / zkb_g2_encode_host) against the
oracle's Fq2 arithmetic (oracle/pairing_ref.py)."""
import numpy as np
import pytest

import pyref as P
import pairing_ref as PR

Q = P.Q_MOD


def raw_g2(pt):
    """(FQ2 x, FQ2 y) or None -> the raw 128-byte G2Affine (x.c0, x.c1, y.c0, y.c1 Montgomery limbs)"""
    if pt is None:
        return bytes(128)
    x, y = pt
    return np.array(sum((P.limbs(P.to_mont(c, Q)) for c in x.c + y.c), []), dtype=np.uint64).tobytes()


def g2_of_raw(raw):
    l = np.frombuffer(raw, dtype=np.uint64)
    c = [P.from_mont(P.from_limbs(l[4 * i: 4 * i + 4]), Q) for i in range(4)]
    return None if not any(l) else (PR.FQ2(c[:2]), PR.FQ2(c[2:]))


def is_square_fq2(a):
    """a is a square in Fq2 iff its norm a0^2 + a1^2 is a square in Fq"""
    nrm = (a.c[0] ** 2 + a.c[1] ** 2) % Q
    return nrm == 0 or pow(nrm, (Q - 1) // 2, Q) == 1


@pytest.mark.parametrize("k", range(1, 27))
def test_expected_file_len_matches_reference_formula(k):
    """prover/src/utils.rs:56-75: 4 + 2 * 2^k * g1 + 2 * g2, g1 = 32 (Processed) or 64, g2 = 2 * g1."""
    from zkb200.params import ParamsKZG, SerdeFormat
    for fmt, g1 in ((SerdeFormat.Processed, 32), (SerdeFormat.RawBytes, 64), (SerdeFormat.RawBytesUnchecked, 64)):
        assert ParamsKZG.expected_file_len(k, fmt) == 4 + 2 * (1 << k) * g1 + 2 * (2 * g1)
    assert ParamsKZG.expected_file_len(k) == ParamsKZG.expected_file_len(k, SerdeFormat.RawBytesUnchecked)


def test_secret_power_constant_is_the_reference_point():
    """PARAMS_G2_SECRET_POWER is the point prover/src/utils.rs:36 prints (canonical hex, Fq2 { c0, c1 }), on the twist."""
    from zkb200.params import PARAMS_G2_SECRET_POWER
    ref = (PR.FQ2([0x17944351223333f260ddc3b4af45191b856689eda9eab5cbcddbbe570ce860d2, 0x186282957db913abd99f91db59fe69922e95040603ef44c0bd7aa3adeef8f5ac]),
           PR.FQ2([0x297772d34bc9aa8ae56162486363ffe417b02dc7e8c207fc2cc20203e67a02ad, 0x298adc7396bd3865cbf6d6df91bae406694e6d2215baa893bdeadb63052895f4]))
    raw = np.array(PARAMS_G2_SECRET_POWER, dtype=np.uint64).tobytes()
    assert raw == raw_g2(ref)
    assert PR.g2_is_on_curve(g2_of_raw(raw))


def test_g2_roundtrip_and_reasons():
    from zkb200.params import PARAMS_G2_SECRET_POWER, SerdeFormat as SF, g2_decode, g2_encode
    pts = [PR.G2, g2_of_raw(np.array(PARAMS_G2_SECRET_POWER, dtype=np.uint64).tobytes()), PR.g2_mul(PR.G2, 987654321)]
    for pt in pts:
        raw = raw_g2(pt)
        for fmt in SF:
            enc = g2_encode(fmt, raw)
            assert len(enc) == 2 * fmt.g1_len
            dec, status = g2_decode(fmt, enc)
            assert status == 0 and dec == raw
            assert PR.g2_is_on_curve(g2_of_raw(dec))
        enc = bytearray(g2_encode(SF.Processed, raw))
        x, y = pt
        assert bytes(enc[:32]) == x.c[0].to_bytes(32, "little")
        assert (enc[63] >> 6) & 1 == y.c[0] & 1 and enc[63] >> 7 == 0
        enc[63] ^= 0x40                                              # the other root: -y
        dec, status = g2_decode(SF.Processed, bytes(enc))
        assert status == 0 and g2_of_raw(dec) == (x, -y)
        enc[63] |= 0x80
        assert g2_decode(SF.Processed, bytes(enc))[1] == 1
    # the identity in every format
    for fmt in SF:
        assert g2_encode(fmt, bytes(128)) == bytes(2 * fmt.g1_len)
        assert g2_decode(fmt, bytes(2 * fmt.g1_len)) == (bytes(128), 0)
    # an x whose x^3 + b has no square root
    t = 1
    while is_square_fq2(PR.FQ2([t, 1]) ** 3 + PR.B2):
        t += 1
    enc = t.to_bytes(32, "little") + (1).to_bytes(32, "little")
    assert g2_decode(SF.Processed, enc) == (bytes(128), 3)
    # x.c1 >= q
    assert g2_decode(SF.Processed, bytes(32) + Q.to_bytes(32, "little"))[1] == 2
    # raw: a limb set >= q, and a point off the curve
    raw = bytearray(raw_g2(PR.G2))
    bad = bytes(raw[:64]) + (Q + 1).to_bytes(32, "little") + bytes(raw[96:])
    assert g2_decode(SF.RawBytes, bad) == (bytes(128), 2)
    raw[0] ^= 1
    assert g2_decode(SF.RawBytes, bytes(raw)) == (bytes(128), 3)
    assert g2_decode(SF.RawBytesUnchecked, bytes(raw)) == (bytes(raw), 0)


def test_check_s_g2():
    from zkb200.params import PARAMS_G2_SECRET_POWER, ParamsKZG
    p = ParamsKZG(1, None, None, raw_g2(PR.G2), np.array(PARAMS_G2_SECRET_POWER, dtype=np.uint64).tobytes())
    p.check_s_g2()
    p.s_g2 = raw_g2(PR.g2_mul(PR.G2, 2))
    with pytest.raises(ValueError, match="Wrong params file of degree 1"):
        p.check_s_g2()


def test_truncated_file_names_the_position(tmp_path):
    """The length check runs before any decoding: a short file names the first element it cuts."""
    from zkb200.params import ParamsKZG, SerdeFormat as SF
    k = 3
    for fmt in SF:
        full = ParamsKZG.expected_file_len(k, fmt)
        for cut, where in ((4 + 5 * fmt.g1_len + 1, r"g\[5\]"), (4 + 8 * fmt.g1_len + 3 * fmt.g1_len, r"g_lagrange\[3\]"),
                           (full - 1, "s_g2")):
            path = tmp_path / f"p{int(fmt)}_{cut}"
            path.write_bytes(k.to_bytes(4, "little") + bytes(cut - 4))
            with pytest.raises(ValueError, match=where):
                ParamsKZG.read_custom(str(path), fmt, to_device=False)
        path.write_bytes(k.to_bytes(4, "little") + bytes(full))
        with pytest.raises(ValueError, match="4 trailing bytes"):
            ParamsKZG.read_custom(str(path), fmt, to_device=False)
