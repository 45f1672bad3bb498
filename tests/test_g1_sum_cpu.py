"""zkb_g1_sum_affine_host (the host-side sum of per-rank MSM partial results) against pyref's affine group law, affine limbs and
compressed bytes.  Pure host code: no device needed."""
import random

import numpy as np
import pytest

import pyref as P


def enc(points):
    """pyref affine points (None = identity) -> (m, 8) uint64 Montgomery Fq limbs, identity (0, 0)"""
    out = np.zeros((len(points), 8), dtype=np.uint64)
    for i, pt in enumerate(points):
        if pt is not None:
            out[i, :4] = P.limbs(P.to_mont(pt[0], P.Q_MOD))
            out[i, 4:] = P.limbs(P.to_mont(pt[1], P.Q_MOD))
    return out


def dec(aff):
    if not aff.any():
        return None
    return (P.from_mont(P.from_limbs(aff[:4]), P.Q_MOD), P.from_mont(P.from_limbs(aff[4:]), P.Q_MOD))


def summed(points):
    from zkb200.parallel import g1_sum_affine
    aff, comp = g1_sum_affine(enc(points) if points else np.zeros((0, 8), dtype=np.uint64))
    exp = None
    for pt in points:
        exp = P.g1_add(exp, pt)
    assert dec(aff) == exp
    assert comp == P.g1_compress(exp)
    return exp


G = P.G1_GEN
A = P.g1_mul(G, 0x1234567890ABCDEF1234567890ABCDEF)


def test_empty_is_identity():
    assert summed([]) is None


def test_one_point():
    assert summed([A]) == A


def test_point_plus_its_negation_is_identity():
    assert summed([A, P.g1_neg(A)]) is None
    assert summed([A, G, P.g1_neg(A)]) == G


def test_doubling_inside_the_mixed_add():
    assert summed([A, A]) == P.g1_add(A, A)
    assert summed([G, G, G]) == P.g1_mul(G, 3)


def test_identity_entries():
    assert summed([None, A, None, None, G, None]) == P.g1_add(A, G)
    assert summed([None, None]) is None


def test_thousand_points():
    rnd = random.Random(7)
    ks = [rnd.randrange(1, 1 << 64) for _ in range(1000)]
    pts = [P.g1_mul(G, k) for k in ks]
    assert summed(pts) == P.g1_mul(G, sum(ks))


def test_argument_check():
    from zkb200 import ZkbError
    from zkb200.lib import check, load_library
    with pytest.raises(ZkbError):
        check(load_library().zkb_g1_sum_affine_host(None, 1, None, None))
