"""The device square (fp_sqr: dedicated wide square + REDC) and the Fermat inverse built on it, against Python integers, for both
BN254 fields, at 0, 1, p - 1 and random elements (Montgomery form in, Montgomery form out)."""
import numpy as np
import pytest

from test_redc_model import P_FQ, P_FR, R

FIELDS = {"fr": P_FR, "fq": P_FQ}


def to_limbs(vals):
    return np.array([[(v >> (64 * i)) & ((1 << 64) - 1) for i in range(4)] for v in vals], dtype=np.uint64)


def from_limbs(arr):
    return [sum(int(x) << (64 * i) for i, x in enumerate(row)) for row in arr]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FIELDS))
def test_device_square_and_inverse(name):
    import torch
    from zkb200 import arithmetic as A
    p = FIELDS[name]
    field = A.FR if name == "fr" else A.FQ
    rng = np.random.default_rng(5)
    vals = [0, 1, p - 1, p - 2, (R - 1) % p] + [int.from_bytes(rng.bytes(32), "little") % p for _ in range(4096)]
    dev = torch.from_numpy(to_limbs(vals).view(np.int64)).cuda()
    rinv = pow(R, -1, p)
    got = from_limbs(A.field_unop_dev(field, A.UOP_SQR, dev).cpu().numpy().view(np.uint64))
    assert got == [v * v * rinv % p for v in vals]
    inv = from_limbs(A.field_unop_dev(field, A.UOP_INV, dev[:64]).cpu().numpy().view(np.uint64))
    # Montgomery a*R -> (a*R)^-1 * R^2 = a^-1 * R; inv(0) = 0
    assert inv == [pow(v, -1, p) * R * R % p if v else 0 for v in vals[:64]]
