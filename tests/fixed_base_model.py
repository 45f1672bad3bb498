"""Model of the fixed-base comb of csrc/setup.cu (zkb_srs_setup_dev): the window size, the table layout and the signed-digit
recoding it shares with the MSM (digits.cuh, modelled by msm_model.window_digits).  A scalar s < r becomes W = ceil(255 / c)
digits d_w with |d_w| <= 2^(c-1) and s = sum_w d_w 2^(c w); the point is the sum of the table entries T[w][|d_w|] = [|d_w| 2^(c w)] G,
negated where d_w < 0, at table index w 2^(c-1) + |d_w| - 1.  tests/test_srs_setup_cpu.py checks the model; the GPU tests use its
edge scalars."""
import numpy as np

import msm_model as M

COMB_C = 12         # the default window size of setup_comb_kernel
COMB_T = 256        # points per CTA (SETUP_T): one shared inversion each
COMB_VARIANTS = [(6, False), (6, True), (7, False), (7, True), (8, False), (10, False), (12, False)]   # (c, table in shared memory)


def cfg(c=COMB_C):
    return M.Cfg(c)


def table_size(c=COMB_C):
    g = cfg(c)
    return g.windows * g.half


def digits_and_indices(vals, c=COMB_C):
    """-> (signed digits (m, W), table index per digit (m, W), -1 where the digit is 0, carry out of the top window (m,))"""
    g = cfg(c)
    digits, carry = M.recode(M.ints_to_canon(vals), g)
    w = np.arange(g.windows)[None, :]
    idx = np.where(digits != 0, w * g.half + np.abs(digits) - 1, -1)
    return digits, idx, carry


def reconstruct(digits, c=COMB_C):
    return [sum(int(d) << (c * w) for w, d in enumerate(row)) for row in digits]


def top_carry_scalar(c=COMB_C):
    """a scalar < r whose window W - 2 is half + 1: negative there, so its recoding carries into the top window"""
    g = cfg(c)
    v = (g.half + 1) << (c * (g.windows - 2))
    assert v < M.R_MOD
    return v
