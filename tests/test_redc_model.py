"""Big-integer models of csrc/ff.cuh's dedicated square and one-reduction sum of products, limb for limb with 32-bit words:
   the column-aligned square (detail::wide_sqr): every carry chain ends in a limb that holds no product limb yet;
   REDC (detail::redc): its running frame fits X (9 limbs at column 0) + Y (8 limbs at column 1), its m * p_odd chain cannot
   overflow, and T < R p gives < 2p before the conditional subtraction;
   fp_mul_add_mul (both products' rows added before each word-serial round): the same frame bounds, and a*b + c*d and
   a*b - c*d (as a*b + (p - c)*d) equal the separately reduced products, for both BN254 fields.
Inputs: random elements and 0, 1, p - 1 in every operand position."""
import itertools
import random

P_FR = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
P_FQ = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
R = 1 << 256
W = 1 << 32
M32 = W - 1


def limbs(x, n=8):
    return [(x >> (32 * i)) & M32 for i in range(n)]


def value(ls):
    return sum(v << (32 * i) for i, v in enumerate(ls))


def mad_row(c, at, e, b, holds_product):
    """c[at .. at + 2K) += e * b as lo/hi pairs, the carry out added to c[at + 2K], which must hold no product limb"""
    k = len(e)
    assert not holds_product[at + 2 * k], "carry limb already holds a product limb"
    acc = value(c[at:at + 2 * k]) + sum(ej * b << (64 * j) for j, ej in enumerate(e))
    for j in range(2 * k):
        c[at + j] = (acc >> (32 * j)) & M32
        holds_product[at + j] = True
    c[at + 2 * k] += acc >> (64 * k)
    assert c[at + 2 * k] < W, "carry limb overflow"


class Wide:
    def __init__(self):
        self.E, self.O = [0] * 17, [0] * 17
        self.hE, self.hO = [False] * 17, [False] * 17

    def sum(self):
        assert self.O[16] == 0 and self.E[16] == 0
        t = value(self.E[:16]) + value(self.O[:16])
        assert t < 1 << 512
        return t


def mul_add_mul(pairs, p):
    """fp_mul_add_mul: X (9 limbs, column 0) and Y (8 limbs, column 1); each round adds the rows of every product, then m * p"""
    inv = (-pow(p, -1, W)) % W
    pe, po = limbs(p)[0::2], limbs(p)[1::2]
    X, Y = [0] * 9, [0] * 8

    def add(acc, n, e, b):
        v = value(acc) + sum(ej * b << (64 * j) for j, ej in enumerate(e))
        assert v < 1 << (32 * n), "chain overflows its accumulator"
        return limbs(v, n)

    for i in range(8):
        carry = 0
        if i:
            s = X[1]
            X, Y = Y + [0], X[2:9] + [0]
            x0 = X[0] + s
            X[0], carry = x0 & M32, x0 >> 32
        Y = limbs(value(Y) + carry, 8)
        assert value(Y) < R
        for a, b in pairs:
            Y = add(Y, 8, limbs(a)[1::2], limbs(b)[i])
            X = add(X, 9, limbs(a)[0::2], limbs(b)[i])
        m = X[0] * inv % W
        X = add(X, 9, pe, m)
        Y = add(Y, 8, po, m)
        assert X[0] == 0
    r = value(X[1:9]) + value(Y)
    assert r < 2 * p, "result must be < 2p"
    return r - p if r >= p else r


def wide_sqr(a):
    x = limbs(a)
    w = Wide()
    for i in range(7):
        od, ev = x[i + 1::2], x[i + 2::2]
        mad_row(w.O, 2 * i + 1, od, x[i], w.hO)
        if ev:
            mad_row(w.E, 2 * i + 2, ev, x[i], w.hE)
    t = 2 * w.sum() + sum(v * v << (64 * i) for i, v in enumerate(x))
    assert t < 1 << 512
    return t


def redc(t, p):
    """the frame of detail::redc: total S = X + Y * 2^32 relative to the current column; returns the value before the final
    conditional subtraction"""
    inv = (-pow(p, -1, W)) % W
    pe, po = limbs(p)[0::2], limbs(p)[1::2]
    tl = limbs(t, 16)
    X, Y = tl[:8] + [0], [0] * 8
    for i in range(8):
        if i:
            s = X[1]
            X, Y = Y + [0], X[2:9] + [0]
            x0 = X[0] + s
            X[0] = x0 & M32
            carry = x0 >> 32
        else:
            carry = 0
        m = X[0] * inv % W
        yv = value(Y) + carry + sum(v * m << (64 * j) for j, v in enumerate(po))
        assert yv < R, "m * p_odd chain overflows Y"
        Y = limbs(yv)
        xv = value(X) + sum(v * m << (64 * j) for j, v in enumerate(pe))
        assert xv < 1 << 288, "X overflows its 9 limbs"
        X = limbs(xv, 9)
        assert X[0] == 0
    r = value(X[1:9]) + value(Y) + value(tl[8:16])
    assert r < 2 * p, "REDC output must be < 2p"
    assert r % p == t * pow(R, -1, p) % p
    return r - p if r >= p else r


def mont_mul(a, b, p):
    return a * b * pow(R, -1, p) % p


def operands(p, rnd, n):
    ext = [0, 1, p - 1]
    vals = [rnd.randrange(p) for _ in range(n)]
    return ext, vals


def test_square_and_redc_match_python():
    rnd = random.Random(3)
    for p in (P_FR, P_FQ):
        ext, vals = operands(p, rnd, 300)
        for a in ext + vals:
            assert wide_sqr(a) == a * a
            assert redc(wide_sqr(a), p) == mont_mul(a, a, p)
        for a, b in itertools.product(ext, ext):
            assert redc(a * b, p) == mont_mul(a, b, p)
        for a, b in zip(vals, reversed(vals)):
            assert redc(a * b, p) == mont_mul(a, b, p)


def test_merged_sum_and_difference_extremes():
    """0, 1, p - 1 in every one of the four operand positions, for a*b + c*d and a*b - c*d"""
    for p in (P_FR, P_FQ):
        ext = [0, 1, p - 1]
        for a, b, c, d in itertools.product(ext, repeat=4):
            t = a * b + c * d
            assert t < 2 * p * p
            assert mul_add_mul([(a, b), (c, d)], p) == (mont_mul(a, b, p) + mont_mul(c, d, p)) % p
            nc = p - c                     # in (0, p]: c = 0 gives p itself
            assert a * b + nc * d < 2 * p * p
            assert mul_add_mul([(a, b), (nc, d)], p) == (mont_mul(a, b, p) - mont_mul(c, d, p)) % p


def test_merged_sum_and_difference_random():
    rnd = random.Random(11)
    for p in (P_FR, P_FQ):
        ext = [0, 1, p - 1]
        for _ in range(400):
            a, b, c, d = (rnd.choice(ext) if rnd.random() < 0.25 else rnd.randrange(p) for _ in range(4))
            assert mul_add_mul([(a, b), (c, d)], p) == (mont_mul(a, b, p) + mont_mul(c, d, p)) % p
            assert mul_add_mul([(a, b), (p - c, d)], p) == (mont_mul(a, b, p) - mont_mul(c, d, p)) % p


def test_redc_bound_is_tight_enough():
    """a T far above any square still gives < 2p (T < R p is what REDC needs)"""
    for p in (P_FR, P_FQ):
        t = 2 * (p - 1) * (p - 1) + (p - 1)
        assert t < R * p
        redc(t, p)
