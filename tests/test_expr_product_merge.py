"""The interpreter's product merging (ProgramBuilder::merge_products, csrc/expr.cuh): a register-register MUL read once, by a
HORNER / HORNER2 root, becomes OP_HORNER_M / OP_HORNER2_M (acc * y + a * b with one Montgomery reduction).  The program is read
on the host to see which products were merged and which were not; the GPU case evaluates the same gates, bit for bit against
`Ref.eval_expr`."""
import pytest

import halo2_ref as H
from test_gpu_expr import R, check_mode1, make_cols, make_cs, ref  # noqa: F401  (ref is a fixture)
from test_gpu_expr_fusion import OP_HORNER, OP_HORNER2, OP_MUL, program

OP_HORNER_M, OP_HORNER2_M = 43, 44


def merge_gates():
    a, b, c, d = (H.advice(i, i - 1) for i in range(4))
    q = H.fixed(0)
    x = (a + b) * (c + d)
    return [
        (a + b) * (c + d),                 # a bare gate: its product feeds the HORNER root
        x * x,                             # x is read twice and stays a MUL; x * x is read once by the root
        q * ((a + c) * (b + d)),           # selector run: the product feeds HORNER2
        q * ((a - b) * (c - d)),
        (a + b) * c,                       # a column operand: MUL_RC, not a register-register MUL, is not merged
    ]


def test_single_read_products_are_merged():
    ops, _ = program(make_cs(4, merge_gates()[:1]), 1)
    assert OP_HORNER_M in ops and OP_HORNER not in ops and OP_MUL not in ops


def test_product_read_twice_stays_a_mul():
    ops, _ = program(make_cs(4, merge_gates()[1:2]), 1)
    assert ops.count(OP_MUL) == 1          # x = (a + b) * (c + d), read twice
    assert ops.count(OP_HORNER_M) == 1     # x * x, read once by its root


def test_selector_run_products_merge_into_horner2():
    ops, _ = program(make_cs(4, merge_gates()[2:4]), 1)
    assert ops.count(OP_HORNER2_M) == 2 and OP_HORNER2 not in ops


def test_store_programs_are_unchanged():
    """mode 0 stores each gate: no accumulator root, nothing to merge"""
    ops, _ = program(make_cs(4, merge_gates()), 0)
    assert OP_HORNER_M not in ops and OP_HORNER2_M not in ops and OP_MUL in ops


@pytest.mark.gpu
@pytest.mark.parametrize("k", [3, 7])
def test_merged_values(ref, k):
    cs = make_cs(k, merge_gates(), na=4)
    cols = make_cols(ref, cs, seed=k + 20)
    check_mode1(ref, cs, cols, [], y=0x3E5, scale=R - 1)
