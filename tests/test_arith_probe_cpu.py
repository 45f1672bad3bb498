"""CPU: the host-compiled branches of ff.cuh and g1.cuh (the `#else` of __CUDA_ARCH__ that computes challenges, pow tables, coset
generators, vk values and serde constants) through zkb_arith_probe_host, exactly against Python integers at the contract edges
of every primitive (tests/arith_vectors.py); the operand vectors themselves checked against each op's contract; and the probe's
argument checks."""
import ctypes

import pytest

import arith_vectors as V

HOST_FIELD_OPS = [op for op in V.FIELD_OPS if op not in V.DEVICE_ONLY]


@pytest.fixture(scope="module")
def A():
    from zkb200 import arithmetic
    return arithmetic


@pytest.mark.parametrize("field", [0, 1])
@pytest.mark.parametrize("op", V.FIELD_OPS)
def test_vectors_inside_contract(field, op):
    """every generated tuple lies inside its op's contract, and the edges the contract names are among them"""
    cases = V.field_cases(field, op)
    bad = [x for x in cases if not V.in_contract(field, op, x)]
    assert not bad, f"{V.OP_NAMES[op]}: {len(bad)} tuples outside the contract, first {[hex(v) for v in bad[0]]}"
    p = V.FIELDS[field]
    flat = {v for x in cases for v in x}
    must = {V.MUL_LAZY: (4 * p - 1, 2 * p - 1), V.COND_SUB_2P: (4 * p - 1, 2 * p, 2 * p - 1), V.COND_SUB_P: (2 * p - 1, p),
            V.ADD_LAZY: (2 * p - 1,), V.SUB_LAZY: (2 * p - 1,), V.POW: (0, p - 1, p, V.R - 1, 1 << 255), V.POW_U64: (0, 1, V.MASK64),
            V.MUL_ADD_MUL: (p,), V.MUL_SUB_MUL: (p,), V.INV: (0,), V.FROM_U64: (V.MASK64,)}
    assert set(must.get(op, (0, 1, p - 1))) <= flat
    if op == V.MUL_SUB_MUL:
        assert any(x[2] == 0 for x in cases)      # c = 0: the inner p - c is p
    # the contract check itself rejects the first value past each bound
    over = {V.ADD: (p, 0), V.MUL_LAZY: (4 * p, 0), V.ADD_LAZY: (2 * p, 0), V.COND_SUB_2P: (4 * p,), V.COND_SUB_P: (2 * p,),
            V.MUL_ADD_MUL: (p + 1, 0, 0, 0), V.MUL_SUB_MUL: (0, 0, p, 0), V.POW_U64: (0, 1 << 64), V.FROM_U64: (1 << 64,)}
    if op in over:
        assert not V.in_contract(field, op, over[op])


@pytest.mark.parametrize("field", [0, 1])
@pytest.mark.parametrize("op", HOST_FIELD_OPS)
def test_host_field_op(A, field, op):
    cases = V.field_cases(field, op)
    arity, _ = A.PROBE_SHAPE[op]
    outs = V.unpack(A.arith_probe_host(field, op, V.pack(cases, arity)))
    bad, shown = V.field_mismatches(field, op, cases, outs)
    assert bad == 0, f"{bad} of {len(cases)} wrong: " + "; ".join(shown)


@pytest.mark.parametrize("op", V.G1_OPS)
def test_host_g1_op(A, op):
    cases = V.g1_cases(op)
    arity, _ = A.PROBE_SHAPE[op]
    outs = V.unpack(A.arith_probe_host(1, op, V.pack([c[1] for c in cases], arity)))
    bad, shown = V.g1_mismatches(op, cases, outs)
    assert bad == 0, f"{bad} of {len(cases)} wrong: " + "; ".join(shown)


def test_probe_arguments():
    """device-only ops, unknown ops, G1 ops outside Fq and unknown fields are refused on the host; the device entry refuses
    a missing context"""
    import zkb200
    lib = zkb200.load_library()
    vp = ctypes.c_void_p
    buf = (ctypes.c_uint64 * 32)()
    p = ctypes.cast(buf, vp)
    for op in V.DEVICE_ONLY + (-1, 19, 31, 39, 1000):
        assert lib.zkb_arith_probe_host(0, op, p, p, 1) == -2, op
    for op in V.G1_OPS:
        assert lib.zkb_arith_probe_host(0, op, p, p, 1) == -2, op
    for field in (-1, 2):
        assert lib.zkb_arith_probe_host(field, V.ADD, p, p, 1) == -2
    assert lib.zkb_arith_probe_host(0, V.ADD, None, None, 1) == -2
    assert lib.zkb_arith_probe_host(0, V.ADD, None, None, 0) == 0
    assert lib.zkb_arith_probe_dev(None, 0, V.ADD, p, p, 1, None) == -2
