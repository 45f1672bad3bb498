"""The cross-rank transform of the domain-sharded NTT (zkb_ntt_cross_dev) against its definition, and the whole sharded NTT's
arithmetic (local transforms, twiddles, cross transform, as zkb200.parallel.ntt_distributed runs them) on one device with the
all-to-all done as a host reshuffle, against best_fft of the whole input."""
import ctypes

import numpy as np
import pytest

import pyref as P
from util import rand_field, to_dev, to_host

pytestmark = pytest.mark.gpu
R = P.R_MOD


def mont(oracle, v):
    return oracle.fr_from_canonical(np.array([P.limbs(v % R)], dtype=np.uint64))[0]


def omega_p(oracle, p):
    return mont(oracle, P.omega(p.bit_length() - 1))


def cross(x, p, w):
    from zkb200 import parallel
    return parallel.DeviceOps().cross(x, p, w)


def reference(oracle, x, p, w):
    """out[k] = sum_j in[j] w^(j k), rows of length len"""
    ln = x.shape[0] // p
    rows = [np.ascontiguousarray(x[j * ln:(j + 1) * ln]) for j in range(p)]
    out = []
    for k in range(p):
        acc = np.zeros((ln, 4), dtype=np.uint64)
        for j in range(p):
            wjk = oracle.fr_pow(w, j * k)
            acc = oracle.fr_add(acc, oracle.fr_mul(rows[j], np.repeat(wjk[None], ln, axis=0)))
        out.append(acc)
    return np.concatenate(out)


@pytest.mark.parametrize("ln", [1, 127, 128, 129, (1 << 20) + 3])
@pytest.mark.parametrize("p", [1, 2, 4, 8, 16])
def test_cross_transform_definition(oracle, p, ln):
    w = omega_p(oracle, p)
    top = mont(oracle, R - 1)
    for x in (rand_field(p * ln, p * 1000 + ln % 1000), np.repeat(top[None], p * ln, axis=0)):
        got = to_host(cross(to_dev(x), p, w))
        if (x == top).all():   # every column is the same: one column of the reference, repeated
            exp = np.repeat(reference(oracle, np.repeat(top[None], p, axis=0), p, w), ln, axis=0)
        else:
            exp = reference(oracle, x, p, w)
        bad = np.nonzero((got != exp).any(axis=1))[0]
        assert len(bad) == 0, f"{len(bad)} outputs differ, first at row {bad[0] // ln}, column {bad[0] % ln}"


@pytest.mark.parametrize("case", ["p3", "order_too_high", "order_too_low", "in_is_out"])
def test_cross_transform_rejects(oracle, case):
    from zkb200 import ZkbError, default_context
    from zkb200.lib import check
    ctx = default_context()
    x = to_dev(rand_field(4 * 16, 1))
    out = x.clone()
    p, w = 4, omega_p(oracle, 4)
    if case == "p3":
        p = 3
    elif case == "order_too_high":
        w = omega_p(oracle, 8)
    elif case == "order_too_low":
        w = omega_p(oracle, 2)
    w = np.ascontiguousarray(w)
    dst = x if case == "in_is_out" else out
    before = ctx.launch_count
    with pytest.raises(ZkbError):
        check(ctx.lib.zkb_ntt_cross_dev(ctx.handle, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(dst.data_ptr()), p, x.shape[0] // 4,
                                        ctypes.c_void_p(w.ctypes.data), None))
    assert ctx.launch_count == before


@pytest.mark.parametrize("world", [2, 4, 8, 16])
def test_sharded_ntt_arithmetic_on_one_device(oracle, world):
    import torch
    from zkb200.parallel import DeviceOps, cyclic_shard, strips_to_natural
    ops = DeviceOps()
    log_n = 14
    n = 1 << log_n
    log_p = world.bit_length() - 1
    M = n // world
    x = rand_field(n, world)
    omega = mont(oracle, P.omega(log_n))
    omega_m = ops.pow_omega(omega, world)
    z = []
    for r in range(world):
        zr = ops.local_ntt(to_dev(np.ascontiguousarray(cyclic_shard(x, r, world))), omega_m, log_n - log_p)
        if r:
            zr = ops.mul(zr, ops.powers(ops.pow_omega(omega, r), M, zr))
        z.append(zr)
    blk = M // world
    strips = []
    for s in range(world):
        recv = torch.cat([z[j][s * blk:(s + 1) * blk] for j in range(world)]).contiguous()   # the all-to-all, block s of every rank
        strips.append(to_host(ops.cross(recv, world, ops.pow_omega(omega, M))))
    got = strips_to_natural(strips, world)
    assert (got == oracle.best_fft(x, omega, log_n)).all()
