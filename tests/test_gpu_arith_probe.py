"""GPU: every primitive of ff.cuh and g1.cuh on the device, through zkb_arith_probe_dev, exactly against Python integers at the
contract edges of tests/arith_vectors.py (lazy operands up to 4p - 1, c = 0 in fp_mul_sub_mul, exponents with bit 255 set,
inv(0), one point in several XYZZ representations, P + (-P) ...); the host-compiled branch of each op byte for byte equal to the
device's; the dedicated square and the Fermat inverse on random elements through the probe and through zkb_field_unop_dev; and
the batch inversion at its 32-element chunk structure."""
import numpy as np
import pytest

import arith_vectors as V
import pyref as P
from util import rand_field, to_dev, to_host

pytestmark = pytest.mark.gpu

R = V.R


@pytest.fixture(scope="module")
def A():
    from zkb200 import arithmetic
    return arithmetic


@pytest.mark.parametrize("field", [0, 1])
@pytest.mark.parametrize("op", V.FIELD_OPS)
def test_field_op(A, field, op):
    cases = V.field_cases(field, op)
    arity, _ = A.PROBE_SHAPE[op]
    ins = V.pack(cases, arity)
    got = to_host(A.arith_probe_dev(field, op, to_dev(ins)))
    bad, shown = V.field_mismatches(field, op, cases, V.unpack(got))
    assert bad == 0, f"{bad} of {len(cases)} wrong: " + "; ".join(shown)
    if op not in V.DEVICE_ONLY:
        host = A.arith_probe_host(field, op, ins)
        assert host.tobytes() == got.tobytes(), "host and device branches differ"


@pytest.mark.parametrize("op", V.G1_OPS)
def test_g1_op(A, op):
    """O, P, -P, 2P and generic points, each XYZZ operand under lambda = 1, -1 and random lambda: O + O, O + P, P + O, P + P and
    P + (-P) in the same and in different representations, P + 2P, generic sums, doublings, normalisation"""
    cases = V.g1_cases(op)
    arity, _ = A.PROBE_SHAPE[op]
    ins = V.pack([c[1] for c in cases], arity)
    got = to_host(A.arith_probe_dev(1, op, to_dev(ins)))
    bad, shown = V.g1_mismatches(op, cases, V.unpack(got))
    assert bad == 0, f"{bad} of {len(cases)} wrong: " + "; ".join(shown)
    assert A.arith_probe_host(1, op, ins).tobytes() == got.tobytes(), "host and device branches differ"


@pytest.mark.parametrize("name", ["fr", "fq"])
def test_square_and_inverse(A, name):
    """fp_sqr (wide square + REDC) and fp_inv on 0, 1, p - 1, p - 2, (R - 1) mod p and 4096 random elements, through the probe and
    through zkb_field_unop_dev (Montgomery form in, Montgomery form out)"""
    field = 0 if name == "fr" else 1
    p = V.FIELDS[field]
    rng = np.random.default_rng(5)
    vals = [0, 1, p - 1, p - 2, (R - 1) % p] + [int.from_bytes(rng.bytes(32), "little") % p for _ in range(4096)]
    dev = to_dev(V.pack([(v,) for v in vals], 1))
    rinv = pow(R, -1, p)
    sqr = [v * v * rinv % p for v in vals]
    assert [y for (y,) in V.unpack(to_host(A.arith_probe_dev(field, V.SQR, dev)))] == sqr
    assert [y for (y,) in V.unpack(to_host(A.field_unop_dev(field, A.UOP_SQR, dev)))] == sqr
    # a R -> (a R)^-1 R^2 = a^-1 R; inv(0) = 0
    inv = [pow(v, -1, p) * R * R % p if v else 0 for v in vals[:64]]
    assert [y for (y,) in V.unpack(to_host(A.arith_probe_dev(field, V.INV, dev[:64])))] == inv
    assert [y for (y,) in V.unpack(to_host(A.field_unop_dev(field, A.UOP_INV, dev[:64])))] == inv


def test_probe_device_arguments(A):
    """the device entry refuses what the host entry refuses; the device-only ops are accepted there"""
    import ctypes
    import torch
    from zkb200 import ZkbError
    from zkb200.lib import default_context
    buf = torch.zeros((1, 32), dtype=torch.int64, device="cuda")
    vp = ctypes.c_void_p(buf.data_ptr())
    ctx = default_context()
    for field, op in [(0, -1), (0, 19), (1, 31), (1, 39), (0, V.G1_ADD), (2, V.ADD), (-1, V.ADD)]:
        assert ctx.lib.zkb_arith_probe_dev(ctx.handle, field, op, vp, vp, 1, None) == -2, (field, op)
    for op in V.DEVICE_ONLY:
        assert ctx.lib.zkb_arith_probe_dev(ctx.handle, 0, op, vp, vp, 0, None) == 0
    with pytest.raises(ZkbError):
        A.arith_probe_host(0, V.MUL_LAZY, np.zeros((1, 8), dtype=np.uint64))


# ---- batch inversion (fieldops.cu: one thread per 32-element chunk, zeros skipped) ------------------------------------------------
BI_CHUNK = 32
FR = V.FIELDS[0]


def batch_inverse_ref(vals):
    """Montgomery a R -> a^-1 R = R^2 / (a R); zeros stay zero"""
    cache = {}
    r2 = R * R % FR
    out = []
    for v in vals:
        if v not in cache:
            cache[v] = pow(v, -1, FR) * r2 % FR if v else 0
        out.append(cache[v])
    return out


def batch_patterns(n, seed):
    """name -> stored Fr values (uint64 (n, 4))"""
    base = rand_field(n, seed)
    pats = {"all zero": np.zeros((n, 4), dtype=np.uint64)}
    z = base.copy()
    idx = np.arange(n)
    z[(idx % BI_CHUNK == 0) | (idx % BI_CHUNK == BI_CHUNK - 1) | (idx == n - 1)] = 0
    pats["zero at every chunk start and end"] = z
    w = base.copy()
    c = 1 if n > 2 * BI_CHUNK else 0          # a whole chunk of zeros except one element
    lo, hi = c * BI_CHUNK, min(n, (c + 1) * BI_CHUNK)
    w[lo:hi] = 0
    w[lo + (hi - lo) // 2] = base[lo + (hi - lo) // 2]
    pats["one non-zero in a zero chunk"] = w
    ones = V.pack([(v,) for v in [1, FR - 1, R % FR, (R - 1) % FR]], 1)
    pats["1 and p - 1"] = ones[idx % 4]
    return pats


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4097, (1 << 20) + 7])
def test_batch_invert_chunks(A, oracle, n):
    for name, a in batch_patterns(n, 900 + n).items():
        got = to_host(A.fr_batch_invert_dev(to_dev(a)))
        if n <= 4097 or name in ("all zero", "1 and p - 1"):
            exp = V.pack([(v,) for v in batch_inverse_ref([x for (x,) in V.unpack(a)])], 1)
        else:
            exp = oracle.fr_inv(a)
        assert (got == exp).all(), f"n = {n}, {name}: first wrong index {int(np.argmax((got != exp).any(axis=1)))}"
