"""The polynomial utilities of poly.cu at their tile edges.  Every scan and evaluation cuts the input into blocks of 2048 elements
and walks the block totals in tiles of 256 blocks (2^19 elements), carrying one value from tile to tile; kate_division skips the
blocks whose carry is zero.  So the sizes here are one tile and its neighbours (2^19 - 1, 2^19, 2^19 + 1), 9 tiles (2^22 + 2049) and
the 128 tiles of a 2^26 domain; the points are 0, 1, -1, a root of unity with u^2048 = 1 and a random one; the inputs are zero
everywhere, zero but for the last or the first coefficient, a zero run across a tile boundary, p - 1 everywhere, and random.  Large
outputs are checked as exact recurrences with the oracle's vectorised Fr arithmetic; evaluations as sums of canonical limbs."""
import numpy as np
import pytest

import pyref as P
from util import rand_field, to_dev, to_host

pytestmark = pytest.mark.gpu
R = P.R_MOD
TILE = 256 * 2048
SIZES = [TILE - 1, TILE, TILE + 1, (1 << 22) + 2049]
CHUNK = 1 << 22


def mont(oracle, vals):
    return oracle.fr_from_canonical(np.array([P.limbs(v % R) for v in vals], dtype=np.uint64).reshape(-1, 4))


def points(oracle):
    return {"zero": 0, "one": 1, "minus_one": R - 1, "omega_2^11": P.omega(11), "random": P.from_limbs(rand_field(1, 91)[0]) % R}


def inputs(oracle, n):
    """name -> (n, 4) Montgomery array"""
    out = {"random": rand_field(n, n % 1000)}
    z = np.zeros((n, 4), dtype=np.uint64)
    out["zero"] = z
    last = z.copy(); last[n - 1] = mont(oracle, [7])[0]
    first = z.copy(); first[0] = mont(oracle, [5])[0]
    run = rand_field(n, 3)
    lo, hi = max(0, TILE - 3 * 2048 - 5), min(n, TILE + 2 * 2048 + 7)   # zero across the first tile boundary (or to the end)
    run[lo:hi] = 0
    out.update(last_only=last, first_only=first, zero_run=run, p_minus_1=np.repeat(mont(oracle, [R - 1]), n, axis=0))
    return out


def check_rec(oracle, out, first, op, a, b):
    """out[0] == first and out[1:] == op(a, b) chunk by chunk (a, b arrays aligned with out[1:], or one element broadcast)"""
    assert (out[0] == first).all(), "first element"
    m = out.shape[0] - 1
    for s in range(0, m, CHUNK):
        e = min(m, s + CHUNK)
        aa = a[s:e] if a.shape[0] > 1 else np.repeat(a, e - s, axis=0)
        bb = b[s:e] if b.shape[0] > 1 else np.repeat(b, e - s, axis=0)
        exp = op(np.ascontiguousarray(aa), np.ascontiguousarray(bb))
        bad = np.nonzero((out[1 + s:1 + e] != exp).any(axis=1))[0]
        assert len(bad) == 0, f"{len(bad)} elements break the recurrence, first at {1 + s + bad[0]}"


def canonical_sum(oracle, a):
    """sum of the canonical values of the Montgomery rows of a, exact (32-bit column sums in uint64), mod r"""
    tot = 0
    for s in range(0, a.shape[0], CHUNK):
        c = oracle.fr_to_canonical(np.ascontiguousarray(a[s:s + CHUNK])).view(np.uint32).reshape(-1, 8).astype(np.uint64)
        tot += sum(int(v) << (32 * i) for i, v in enumerate(c.sum(axis=0)))
    return tot % R


def check_scans(oracle, a, init):
    from zkb200 import poly
    d = to_dev(a)
    gp = to_host(poly.prefix_product_dev(d, init))
    check_rec(oracle, gp, init, oracle.fr_mul, gp[:-1], a[:-1])
    gs = to_host(poly.prefix_sum_dev(d, init))
    check_rec(oracle, gs, init, oracle.fr_add, gs[:-1], a[:-1])


def check_kate(oracle, a, u):
    from zkb200 import poly
    q = to_host(poly.kate_division_dev(to_dev(a), u))
    assert not q[-1].any(), "q[n - 1] must be zero"
    # q[i] = a[i + 1] + u q[i + 1] for i < n - 1, checked as out = q reversed: out[0] = 0, out[j] = a[n - j] + u out[j - 1]
    rq, ra = q[::-1], a[::-1]
    mul_add = lambda x, y: oracle.fr_add(y, oracle.fr_mul(x, np.repeat(u[None], x.shape[0], axis=0)))
    check_rec(oracle, np.ascontiguousarray(rq), rq[0], mul_add, rq[:-1], ra[:-1])


def check_powers_and_eval(oracle, polys, base):
    """fr_powers(base) as a recurrence, then every polynomial's eval_polynomial(base) from those powers"""
    from zkb200 import poly
    n = polys[0].shape[0]
    pw = to_host(poly.fr_powers_dev(base, n))
    check_rec(oracle, pw, mont(oracle, [1])[0], oracle.fr_mul, pw[:-1], base[None])
    got = poly.eval_polynomial_dev([to_dev(p) for p in polys], base)
    for p, g in zip(polys, got):
        exp = 0
        for s in range(0, n, CHUNK):
            exp += canonical_sum(oracle, oracle.fr_mul(np.ascontiguousarray(p[s:s + CHUNK]), np.ascontiguousarray(pw[s:s + CHUNK])))
        assert P.from_limbs(oracle.fr_to_canonical(g[None])[0]) == exp % R


@pytest.mark.parametrize("n", SIZES)
def test_scans_at_tile_edges(oracle, n):
    ins = inputs(oracle, n)
    rnd = rand_field(1, 5)[0]
    for name, a in ins.items():
        check_scans(oracle, a, rnd)
    a = ins["random"].copy()
    a[TILE - 1 if n > TILE else n // 2] = 0                        # a zero factor: the product is zero from there on
    check_scans(oracle, a, rnd)
    check_scans(oracle, ins["random"], np.zeros(4, dtype=np.uint64))   # init = 0
    check_scans(oracle, ins["p_minus_1"], mont(oracle, [1])[0])


@pytest.mark.parametrize("point", ["zero", "one", "minus_one", "omega_2^11", "random"])
@pytest.mark.parametrize("n", SIZES)
def test_kate_division_at_tile_edges(oracle, n, point):
    u = mont(oracle, [points(oracle)[point]])[0]
    for name, a in inputs(oracle, n).items():
        check_kate(oracle, a, u)


@pytest.mark.parametrize("point", ["zero", "one", "minus_one", "omega_2^11", "random"])
@pytest.mark.parametrize("n", SIZES)
def test_powers_and_eval_at_tile_edges(oracle, n, point):
    x = mont(oracle, [points(oracle)[point]])[0]
    check_powers_and_eval(oracle, list(inputs(oracle, n).values()), x)


def test_domain_2_26(oracle):
    """the 128 tile-to-tile carries of a 2^26 domain"""
    n = 1 << 26
    a = rand_field(n, 26)
    u = rand_field(1, 27)[0]
    check_scans(oracle, a, u)
    check_kate(oracle, a, u)
    check_powers_and_eval(oracle, [a], u)


@pytest.mark.parametrize("num,n", [(1, 2049), (300, 5), (65535, 3)])
def test_eval_many_polynomials(oracle, num, n):
    """one grid row per polynomial, up to the 65535 rows of gridDim.y"""
    import torch
    from zkb200 import poly
    allp = rand_field(num * n, num)
    x = rand_field(1, 3)[0]
    t = to_dev(allp)
    got = poly.eval_polynomial_dev([t[i * n:(i + 1) * n] for i in range(num)], x)
    cols = allp.reshape(num, n, 4)
    xs = np.repeat(x[None], num, axis=0)
    exp = np.zeros((num, 4), dtype=np.uint64)
    for i in range(n - 1, -1, -1):                                  # Horner over all polynomials at once
        exp = oracle.fr_add(oracle.fr_mul(exp, xs), np.ascontiguousarray(cols[:, i]))
    assert (got == exp).all()


def test_eval_rejects_too_many_polynomials():
    from zkb200 import poly, ZkbError, default_context
    t = to_dev(rand_field(65536, 1))
    before = default_context().launch_count
    with pytest.raises(ZkbError):
        poly.eval_polynomial_dev([t[i:i + 1] for i in range(65536)], rand_field(1, 2)[0])
    assert default_context().launch_count == before
