"""The interpreter's operand fusion (ProgramBuilder::fuse, csrc/expr.cuh): a column or constant load whose register is read once
becomes an operand of its reader.  The program the compiler emits is read on the host (zkb_expr_program) to see which loads were
fused and which were not, and every case is then run by the interpreter and compared bit for bit with `Ref.eval_expr`, as in
test_gpu_expr.py."""
import numpy as np
import pytest

import halo2_ref as H
from test_gpu_expr import R, check_mode0, check_mode1, make_cols, make_cs, ref  # noqa: F401  (ref is a fixture)
from test_gpu_prover import to_product_cs

OP_LOADCOL, OP_LOADCONST, OP_ADD, OP_MUL, OP_HORNER, OP_HORNER2, OP_FOLD = 0, 1, 2, 4, 6, 10, 11
OP_ADD_RC, OP_SUB_RC, OP_MUL_RC = 16, 24, 32
FORM_RC, FORM_CR, FORM_RK, FORM_KR, FORM_CC, FORM_CK, FORM_KC = range(7)
OP_HORNER_C, OP_HORNER2_C, OP_FOLD_C = 40, 41, 42


def program(cs, mode, challenges=()):
    """opcodes of the dispatched instructions (OP_ARG words dropped) and the register count"""
    from zkb200 import plonk as Z
    ch = [[c, 0, 0, 0] for c in challenges]
    one = np.array([1, 0, 0, 0], dtype=np.uint64)
    code, nregs = Z.expr_program(to_product_cs(cs, 5, 3), mode=mode, challenges=ch, y=one, scale=one)
    ops = [int(w) & 0xFF for w in code]
    return [o for o in ops if o != 13], nregs


def test_two_uses_are_not_fused():
    """a * b + a: `a` is read twice, so it stays an OP_LOADCOL and both readers take its register; `b` is fused"""
    a, b = H.advice(0), H.advice(1, 1)
    ops, _ = program(make_cs(4, [a * b + a]), 0)
    assert ops.count(OP_LOADCOL) == 1
    assert OP_MUL_RC + FORM_RC in ops and OP_ADD in ops


def test_reloaded_register_is_fused_per_load():
    """(a * b) * (c * d): a's register is loaded again for c after its one read, b's is overwritten by a * b.  Each load's reads
    are counted up to the next write of its register, so a, b, c and d are all fused and no load is left"""
    a, b, c, d = (H.advice(i) for i in range(4))
    ops, nregs = program(make_cs(4, [(a * b) * (c * d)]), 0)
    assert OP_LOADCOL not in ops
    assert ops.count(OP_MUL_RC + FORM_CC) == 2 and OP_MUL in ops
    assert nregs == 3                              # the allocator's count, not the fused program's


def test_constants_and_columns_in_every_form():
    a, b = H.advice(0), H.advice(1)
    gates = [a + H.const(5), H.const(7) + (a * b), (a * b) * H.const(R - 1), H.const(3) * a, a * H.const(2),
             H.const(4) + H.const(6), H.challenge(0) * a, (a * b) + b * b]
    ops, _ = program(make_cs(4, gates, nch=1), 1, challenges=[9])   # mode 1: one scope per gate, so `a` is not shared
    for op in (OP_ADD_RC + FORM_CK, OP_ADD_RC + FORM_KR, OP_MUL_RC + FORM_RK, OP_MUL_RC + FORM_KC, OP_MUL_RC + FORM_CK):
        assert op in ops, op
    assert OP_LOADCONST in ops                     # const + const: no KK form, the right constant stays a load


@pytest.mark.gpu
@pytest.mark.parametrize("k", [3, 7])
def test_fused_values(ref, k):
    """the gates of the structural tests above, evaluated"""
    a, b, c, d = (H.advice(i, i - 1) for i in range(4))
    gates = [a * b + a, (a * b) * (c * d), a + H.const(5), H.const(7) + (a * b), (a * b) * H.const(R - 1), H.const(3) * a,
             H.const(4) + H.const(6), H.challenge(0) * a, (a * b) + b * b, -(a * b) + c, a + (-b), H.scaled(c, R - 2)]
    cs = make_cs(k, gates, na=4, nch=1)
    cols = make_cols(ref, cs, seed=k)
    check_mode0(ref, cs, cols, [R - 1])
    check_mode1(ref, cs, cols, [R - 1], y=0x3E5, scale=R - 1)


def fold_root_gates(rot):
    """runs of q(rot) * column (HORNER2 and FOLD roots that are plain queries), a bare column gate (a HORNER root), and a run
    whose terms are composite"""
    q = H.fixed(0, rot)
    gates = [q * H.advice(0, -rot), q * H.advice(1, rot), H.advice(2) * q,
             H.advice(0, rot),
             H.fixed(1) * (H.advice(0) * H.advice(1, -rot)), H.fixed(1) * (H.advice(2, rot) + H.const(3))]
    return gates


def test_fold_roots_take_columns():
    ops, _ = program(make_cs(4, fold_root_gates(1), na=3), 1)
    assert ops.count(OP_HORNER2_C) == 3 and ops.count(OP_FOLD_C) == 2 and ops.count(OP_HORNER_C) == 1
    assert OP_HORNER2 in ops                       # the composite terms keep the register form


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 4, 10, 17])
def test_fused_rotations_wrap(ref, k):
    """rotations 0, +-1, +-(n-1) and +-32767 through fused column operands of every kind: CC, CK / KC, RC / CR and the
    HORNER / HORNER2 / FOLD roots; every row is compared, so the reads that wrap at row 0 and row n-1 are checked"""
    n = 1 << k
    rots = sorted(r for r in {0, 1, -1, n - 1, -(n - 1), 32767, -32767} if abs(r) <= 32767)
    gates = []
    for r in rots:
        gates += [H.advice(1, r) * H.advice(2, -r), H.advice(0, r) + H.const(11), H.const(R - 2) * H.fixed(1, -r),
                  (H.advice(0) * H.advice(1)) * H.instance(0, r), H.instance(0, -r) + (H.advice(1) * H.advice(2))]
        gates += fold_root_gates(r)
    cs = make_cs(k, gates, na=3)
    ops, _ = program(cs, 1)
    for op in (OP_MUL_RC + FORM_CC, OP_ADD_RC + FORM_CK, OP_MUL_RC + FORM_KC, OP_MUL_RC + FORM_RC, OP_ADD_RC + FORM_CR,
               OP_HORNER_C, OP_HORNER2_C, OP_FOLD_C):
        assert op in ops, op
    cols = make_cols(ref, cs, seed=40 + k)
    check_mode0(ref, cs, cols)
    check_mode1(ref, cs, cols, (), y=0xF01D, scale=5)
