"""CPU checks of csrc/msm.cu's configuration and recoding through tests/msm_model.py: the signed digits reconstruct every
scalar at every window size, the top window never carries out, no argument limit trips at any size up to 2^28, the scratch
the MSM allocates from bounds holds the worst-case partial lists, and the configuration table is pinned."""
import random

import numpy as np
import pytest

import msm_model as M

WINDOW_BITS = list(range(3, 21))


def reconstruct(digits, c):
    return [sum(int(d) << (c * w) for w, d in enumerate(row)) for row in digits.tolist()]


@pytest.mark.parametrize("c", WINDOW_BITS)
def test_recode_round_trip(c):
    """sum_w +-d_w 2^(c w) == s with 0 <= d_w <= half and no carry out of the top window, for the edge scalars and 3000
    random ones.  Catches a dropped or doubled carry, a digit equal to half sent negative (or half + 1 kept positive), and a
    window read across a 32-bit limb boundary from the wrong limb."""
    cfg = M.Cfg(c)
    rnd = random.Random(c)
    vals = M.edge_scalars(c) + [rnd.randrange(M.R_MOD) for _ in range(3000)] + [rnd.randrange(1 << 64) for _ in range(100)]
    assert all(0 <= v < M.R_MOD for v in vals)
    digits, carry = M.recode(M.ints_to_canon(vals), cfg)
    assert not carry.any()
    assert (np.abs(digits) <= cfg.half).all() and (digits != -cfg.half).all()
    assert reconstruct(digits, c) == vals


@pytest.mark.parametrize("c", WINDOW_BITS)
def test_top_window_never_carries(c):
    """msm_digits_kernel drops the carry out of the top window; that is exact only while the top raw window plus a carry of 1
    stays <= half for every s < r.  c * W == 255 exactly at c = 3, 5, 15 and 17, where the margin is tightest."""
    cfg = M.Cfg(c)
    assert c * cfg.windows >= 255
    top = (M.R_MOD - 1) >> (c * (cfg.windows - 1))
    assert top + 1 <= cfg.half


def sizes_up_to_2_28():
    for lg in range(0, 29):
        yield 1 << lg
        if lg < 28:
            yield (1 << (lg + 1)) - 1


def test_argument_limits():
    """For every n <= 2^28 (the largest SRS) and every batch up to msm_max_batch(n), none of msm_plan's
    argument checks refuses the call, plain or against shifted copies.  Catches a batch limit that lets a pass overflow
    the 32-bit pair list or bucket index.  (A plain MSM of more than 2^32 / 13 points is refused: pairs >= 2^32.)"""
    for n in sizes_up_to_2_28():
        mb = M.msm_max_batch(n)
        for batch in sorted({1, mb}):
            assert M.arg_failures(n, batch, False) == [], (n, batch)
            if M.msm_shift_window_bits(n):
                assert M.arg_failures(n, batch, True) == [], (n, batch)
    assert M.arg_failures((1 << 29) - 1, 1, False) == ["pairs < 2^32"]


def one_bucket_counts(sc, n, batch):
    """every scalar in one bucket of each column (plain: one bucket per window, n entries each; shifted: a digit of 1 in
    every window, n * W entries in one bucket, the last of its set); 31 of the first column's entries go to bucket 0 so that
    the big buckets start mid-chunk"""
    cfg = sc["cfg"]
    per = cfg.half if cfg.shifted else cfg.windows * cfg.half
    counts = np.zeros(sc["nbuckets"], dtype=np.int64)
    for col in range(batch):
        if cfg.shifted:
            counts[col * per + cfg.half - 1] = n * cfg.windows
        else:
            for w in range(cfg.windows):
                counts[col * per + w * cfg.half + cfg.half - 1] = n
    moved = min(31, n - 1)
    counts[cfg.half - 1] -= moved
    counts[0] += moved
    return counts


def straddling_counts(sc, n):
    """every nonempty bucket straddles chunk boundaries: equal sizes, a multiple of 32, shifted by one entry"""
    cfg = sc["cfg"]
    cap = n * cfg.windows if cfg.shifted else n
    q = min(cap, max(M.CHUNK, (sc["pairs"] // sc["nbuckets"]) // M.CHUNK * M.CHUNK))
    k = min(sc["nbuckets"], sc["pairs"] // q)
    counts = np.zeros(sc["nbuckets"], dtype=np.int64)
    counts[:k] = q
    counts[0] -= 1
    return counts


@pytest.mark.parametrize("shifted", [False, True])
def test_worst_case_scratch(shifted):
    """The level-0 partials, the outputs of every later level (written alternately to part[1] and part[0]) and the number of
    levels stay within what msm_plan allocates from its bounds, for all scalars in one bucket and for every
    bucket straddling chunk boundaries, at every size 2^3 ... 2^28 with one column and with msm_max_batch columns.
    Catches a partial buffer sized without the one-extra-partial-per-bucket term, or a missing reduction level."""
    for lg in range(3, 29):
        n = 1 << lg
        if shifted and not M.msm_shift_window_bits(n):
            continue
        for batch in sorted({1, M.msm_max_batch(n)}):
            sc = M.scratch(n, batch, shifted)
            for counts in (one_bucket_counts(sc, n, batch), straddling_counts(sc, n)):
                assert counts.sum() <= sc["pairs"]
                lens = M.level0_partials(counts)
                assert lens.sum() <= sc["part0_n"], (n, batch)
                extra, run, totals, maxlen = M.reduce_levels(lens, sc["levels"])
                assert maxlen <= 1 and run <= sc["levels"], (n, batch)
                outs = totals[1:] + [int(np.count_nonzero(counts))] if run else []
                for j, t in enumerate(outs):
                    assert t <= (sc["part1_n"] if j % 2 == 0 else sc["part0_n"]), (n, batch, j)
    # the straddling pattern reaches the level-0 bound up to the one spare slot: the bound is tight
    sc = M.scratch(1 << 20, 1, False)
    assert M.level0_partials(straddling_counts(sc, 1 << 20)).sum() >= sc["part0_n"] - sc["nbuckets"]


def test_accounting_matches_the_device_levels_already_pinned(oracle):
    """test_gpu_parity.py::test_msm_reduction_levels_decided_on_device observes 2 levels for random and all-equal scalars at
    2^16 and 1 level for all-equal scalars at 2^11; the model predicts the same, and a single scalar 1 costs one pair plus
    the 2 * nbuckets of the window reduction."""
    from util import rand_field
    n = 1 << 16
    cfg = M.choose_cfg(n)
    rnd = oracle.fr_to_canonical(rand_field(n, 778))
    assert M.predict([M.bucket_counts(rnd, cfg)], n, cfg)[1] == 2
    same = oracle.fr_to_canonical(rand_field(1, 779))
    assert M.predict([M.bucket_counts(same, cfg, mult=[n])], n, cfg)[1] == 2
    m = 1 << 11
    assert M.predict([M.bucket_counts(same, M.choose_cfg(m), mult=[m])], m, M.choose_cfg(m))[1] == 1
    one = M.Cfg(3)
    assert M.predict([M.bucket_counts(M.ints_to_canon([1]), one)], 1, one) == (1 + 2 * 85 * 4, 0)


def test_bucket_index_and_entries():
    """bucket and sorted-list entry of a digit, plain and shifted, for column 2 of a batch"""
    plain, shifted = M.Cfg(10), M.Cfg(14, shifted=True)
    assert M.bucket_index(3, 7, plain, col=2) == 2 * 26 * 512 + 3 * 512 + 6
    assert M.bucket_index(3, 7, shifted, col=2) == 2 * 8192 + 6
    assert M.sorted_entry(5, 3, True, plain, 1 << 14) == 5 | (1 << 31)
    assert M.sorted_entry(5, 3, False, shifted, 1 << 14) == 5 + 3 * (1 << 14)


# (c, W, shifted c, shifted copies, msm_max_batch) for n = 2^10 ... 2^28
PINNED = {
    10: (6, 43, 10, 26, 64), 11: (7, 37, 11, 24, 64), 12: (8, 32, 12, 22, 64), 13: (9, 29, 13, 20, 64),
    14: (10, 26, 14, 19, 64), 15: (11, 24, 15, 17, 64), 16: (12, 22, 16, 16, 64), 17: (13, 20, 17, 15, 64),
    18: (14, 19, 18, 15, 42), 19: (15, 17, 19, 14, 21), 20: (16, 16, 20, 13, 10), 21: (17, 15, 20, 13, 8),
    22: (18, 15, 20, 13, 4), 23: (19, 14, 0, 0, 2), 24: (20, 13, 0, 0, 1), 25: (20, 13, 0, 0, 1), 26: (20, 13, 0, 0, 1),
    27: (20, 13, 0, 0, 1), 28: (20, 13, 0, 0, 1),
}


def test_pinned_configuration_table():
    """The window sizes, shifted copies and per-pass batch limits of every SRS size, pinned as documentation: a change to
    choose_cfg, msm_shift_window_bits or msm_max_batch shows up here and in the GPU tests' coverage of each c."""
    for lg, row in PINNED.items():
        n = 1 << lg
        cfg = M.choose_cfg(n)
        assert (cfg.c, cfg.windows, M.msm_shift_window_bits(n), M.msm_shift_copies(n), M.msm_max_batch(n)) == row, lg
