"""The NTT tile kernel's double-buffered tile walk, limb for limb against the oracle's best_fft: batches whose tile count leaves
CTAs with an odd number of tiles (the buffer parity wraps), exactly one tile per CTA, fewer tiles than CTAs, the zeta coset on
the input and on the output of 1-, 2- and 3-pass plans, inputs at the top of the field, and launches queued back to back on one
stream into the same buffers."""
import numpy as np
import pytest

import pyref as P
from util import rand_field, to_dev, to_host

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def A():
    from zkb200 import arithmetic
    return arithmetic


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def zeta_tables(oracle, n):
    """per-element ZETA^(i mod 3) and ZETA^(-(i mod 3)) (Montgomery limbs)"""
    zeta = oracle.fr_from_canonical(np.array([P.limbs(P.FR_ZETA)], dtype=np.uint64))[0]
    zeta2 = oracle.fr_mul(zeta[None], zeta[None])[0]
    one = oracle.fr_from_canonical(np.array([[1, 0, 0, 0]], dtype=np.uint64))[0]
    idx = np.arange(n) % 3
    return np.stack([one, zeta, zeta2])[idx], np.stack([one, zeta2, zeta])[idx]


def check_batch(A, oracle, log_n, count, seed, inverse=False, coset_zeta=0, cols=None):
    from zkb200 import poly as Pz
    n = 1 << log_n
    w, wi = A.root_of_unity(log_n)
    if cols is None:
        cols = [rand_field(n, seed + i) for i in range(count)]
    count = len(cols)
    scale = None
    if inverse:
        scale = oracle.fr_inv(oracle.fr_from_canonical(np.array([[n, 0, 0, 0]], dtype=np.uint64)))[0]
    got = Pz.ntt_batch_dev([to_dev(c) for c in cols], wi if inverse else w, log_n, scale=scale, coset_zeta=coset_zeta)
    zin, zout = zeta_tables(oracle, n) if coset_zeta else (None, None)
    for y, (c, g) in enumerate(zip(cols, got)):
        x = oracle.fr_mul(c, zin) if coset_zeta == 1 else c
        exp = oracle.best_fft(x, wi if inverse else w, log_n)
        if inverse:
            exp = oracle.fr_mul(exp, np.repeat(scale[None], n, axis=0))
        if coset_zeta == 2:
            exp = oracle.fr_mul(exp, zout)
        assert (to_host(g) == exp).all(), f"column {y} of {count}, 2^{log_n}"


@pytest.mark.parametrize("log_n,count", [(18, 3), (17, 5), (20, 1)])
def test_tile_count_not_a_multiple_of_the_grid(A, oracle, log_n, count):
    """2^18 x 3 = 384 tiles per pass on 132 SMs: CTAs run 2 or 3 tiles, so both buffers and both parities of each are used"""
    assert (count << (log_n - 11)) % sm_count() != 0
    check_batch(A, oracle, log_n, count, 7000 + log_n)
    check_batch(A, oracle, log_n, count, 7100 + log_n, inverse=True)


def test_one_tile_per_cta(A, oracle):
    """as many single-tile transforms (2^11, one pass) as the grid has CTAs, and a two-pass batch of the same tile count"""
    sms = sm_count()
    check_batch(A, oracle, 11, sms, 7200)
    if sms % 4 == 0:
        check_batch(A, oracle, 13, sms // 4, 7300)   # 2^13 = 4 tiles per column in each pass


@pytest.mark.parametrize("log_n", [12, 14])
def test_fewer_tiles_than_ctas(A, oracle, log_n):
    check_batch(A, oracle, log_n, 1, 7400 + log_n)
    check_batch(A, oracle, log_n, 1, 7500 + log_n, inverse=True)


@pytest.mark.parametrize("log_n", [10, 16, 21])   # 1-, 2- and 3-pass plans
def test_coset_in_and_out(A, oracle, log_n):
    check_batch(A, oracle, log_n, 2, 7600 + log_n, coset_zeta=1)
    check_batch(A, oracle, log_n, 2, 7700 + log_n, inverse=True, coset_zeta=2)


@pytest.mark.parametrize("log_n", [10, 16, 21])   # 1-, 2- and 3-pass plans
def test_extreme_inputs(A, oracle, log_n):
    """inputs that drive the lazy (< 2p) butterflies to the top of their ranges: every element p - 1, 0 and p - 1 alternating, and
    p - 1 only at index 0 and at n - 1 (stored integers), through the forward transform, the inverse with the fused 1/n, and the zeta
    coset on the input and on the output"""
    n = 1 << log_n
    top = np.array(P.limbs(P.R_MOD - 1), dtype=np.uint64)
    full = np.repeat(top[None], n, axis=0)
    alt = full.copy()
    alt[0::2] = 0
    ends = np.zeros((n, 4), dtype=np.uint64)
    ends[0] = ends[-1] = top
    cols = [full, alt, ends]
    check_batch(A, oracle, log_n, 0, 0, cols=cols)
    check_batch(A, oracle, log_n, 0, 0, inverse=True, cols=cols)
    check_batch(A, oracle, log_n, 0, 0, coset_zeta=1, cols=cols)
    check_batch(A, oracle, log_n, 0, 0, inverse=True, coset_zeta=2, cols=cols)


@pytest.mark.parametrize("log_n", [11, 15, 21])
def test_back_to_back_launches(A, oracle, log_n):
    """two batches queued on one stream without a synchronisation in between, the second on the first one's output"""
    from zkb200 import poly as Pz
    n = 1 << log_n
    w, _ = A.root_of_unity(log_n)
    cols = [rand_field(n, 7800 + log_n + i) for i in range(3)]
    dev = [to_dev(c) for c in cols]
    Pz.ntt_batch_dev(dev, w, log_n)
    Pz.ntt_batch_dev(dev, w, log_n, coset_zeta=1)
    zin, _ = zeta_tables(oracle, n)
    for c, g in zip(cols, dev):
        exp = oracle.best_fft(oracle.fr_mul(oracle.best_fft(c, w, log_n), zin), w, log_n)
        assert (to_host(g) == exp).all()
