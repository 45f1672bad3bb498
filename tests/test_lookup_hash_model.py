"""CPU checks of the lookup hash-set model (lookup_hash_model.py) that the GPU multiplicity tests build their inputs and references on."""
import numpy as np
import pytest

import lookup_hash_model as LH


def test_slot_count():
    assert [LH.slot_count(u) for u in (1, 2, 3, 31, 32, 33, 256, 257)] == [2, 4, 8, 64, 64, 128, 512, 1024]


@pytest.mark.parametrize("usable,home", [(33, 0), (1000, 2047), (4097, 16383 - 3), (1 << 16, 12345)])
def test_colliding_values_share_one_home_slot(usable, home):
    v = LH.colliding_values(300, home, usable, seed=home)
    assert v.shape == (300, 4)
    assert len(np.unique(v, axis=0)) == 300
    assert (v[:, 3] < np.uint64(LH.FR_TOP)).all()
    assert (LH.home_slot(v, usable) == home).all()
    # the solved top word is what the forward hash sees: flipping it moves the key off its home slot
    w = v.copy()
    w[:, 3] ^= np.uint64(1 << 32)
    assert (LH.home_slot(w, usable) != home).any()


def test_key_hash_rounds_invert():
    rng = np.random.default_rng(1)
    h = rng.integers(0, 1 << 32, size=10000, dtype=np.uint64)
    assert (LH._round(LH._unround(h), np.zeros_like(h)) == h).all()


def test_vectorised_reference_equals_dict():
    rng = np.random.default_rng(2)
    n, usable = 512, 500
    pool = LH.random_values(40, 3)
    table = pool[rng.integers(0, 40, size=n)]
    table[usable:] = LH.random_values(n - usable, 4)       # values only past the usable rows
    ins = [pool[rng.integers(0, 40, size=n)] for _ in range(3)]
    ins[1][7] = table[usable + 3]                            # present only at a row >= usable: unsatisfied
    ins[2][usable + 1] = LH.random_values(1, 5)[0]          # not in the table, but at a row >= usable: ignored
    for inputs in (ins[:1], [ins[0], ins[2]], ins):
        m, un = LH.multiplicities(inputs, table, usable)
        md, und = LH.multiplicities_dict(inputs, table, usable)
        assert (m == md).all() and un == und
    assert LH.multiplicities(ins, table, usable)[1]
    assert not LH.multiplicities([ins[0], ins[2]], table, usable)[1]
