"""GPU: the constraint interpreter (`expr_kernel`, csrc/expr.cu) row by row against the oracle's expression evaluator.

Every program here goes through the prover's own compiler and interpreter (zkb_expr_eval_dev: translate, one ProgramBuilder
scope per gate set or quotient_gates' selector-run folding, upload_program, expr_run_device) and is compared bit for bit with
`Ref.eval_expr` of oracle/halo2_ref.py, where rotation r reads row (i + r) mod n.  Mode 1 is compared with the plain Horner
fold acc = acc * y + gate_i, times `scale`.  The register count the entry point reports picks the kernel build, and the tests
assert it: <= 8 registers expr_kernel<8, 128, true>, 9-16 expr_kernel<16, 128, true> (both with the register file in shared
memory), 17-64 expr_kernel<64, 128, false> (local memory); a program needing more than 64 is an error.
"""
import numpy as np
import pytest

import halo2_ref as H
import pyref as P
from test_gpu_prover import to_product_cs

pytestmark = pytest.mark.gpu

R = P.R_MOD
TOP_LIMB = 0x30644E72E131A029                 # r's top limb: limbs drawn below it form a value < r (a valid Montgomery form)
EDGES = [0, 1, R - 1, R - 2, (R - 1) // 2]
SENTINEL = np.uint64(0xFFFFFFFFFFFFFFFF)      # all-ones limbs: not a reduced field element, so never a kernel result


@pytest.fixture(scope="module")
def ref():
    return H.Ref(H.ConstraintSystem(1, 0, 1, 0), 0, build_srs=False)


def columns(ref, n, count, seed):
    """`count` columns of n Montgomery values: uniform below r, with the field edges on about a quarter of the rows"""
    rng = np.random.default_rng(seed)
    edges = ref.F.arr(EDGES)
    out = []
    for _ in range(count):
        a = rng.integers(0, 1 << 64, size=(n, 4), dtype=np.uint64)
        a[:, 3] = rng.integers(0, TOP_LIMB, size=n, dtype=np.uint64)
        rows = rng.random(n) < 0.25
        a[rows] = edges[rng.integers(0, len(EDGES), size=int(rows.sum()))]
        out.append(a)
    return out


def make_cs(k, gates, nf=2, na=8, ni=1, nch=0):
    cs = H.ConstraintSystem(k, nf, na, ni, [0] * na, [0] * nch)
    cs.gates = list(gates)
    return cs


def make_cols(ref, cs, seed):
    return {H.FIXED: columns(ref, cs.n, cs.num_fixed, seed), H.ADVICE: columns(ref, cs.n, cs.num_advice, seed + 1),
            H.INSTANCE: columns(ref, cs.n, cs.num_instance, seed + 2)}


def run(ref, cs, cols, challenges=(), mode=0, y=None, scale=None, out=None, out_stride=1, out_offset=0):
    """the device side: (outputs as host arrays, register count)"""
    import torch
    from zkb200 import plonk as Z
    F = ref.F
    dev = [torch.from_numpy(c.view(np.int64)).cuda() for t in (H.FIXED, H.ADVICE, H.INSTANCE) for c in cols[t]]
    kw = {}
    if mode == 1:
        kw = dict(y=F.arr([y])[0], scale=F.arr([scale])[0], out_stride=out_stride, out_offset=out_offset,
                  out=None if out is None else torch.from_numpy(out.view(np.int64)).cuda())
    outs, nregs = Z.expr_eval(to_product_cs(cs, 5, 3), dev, mode=mode, challenges=F.arr(challenges) if challenges else (), **kw)
    return [o.cpu().numpy().view(np.uint64) for o in outs], nregs


def gate_values(ref, cs, cols, challenges=()):
    return [ref.eval_expr(g, cols, list(challenges), cs.n, 1) for g in cs.gates]


def folded(ref, cs, cols, challenges, y, scale):
    F = ref.F
    acc = np.zeros((cs.n, 4), dtype=np.uint64)
    for v in gate_values(ref, cs, cols, challenges):
        acc = F.add(F.scal(acc, y), v)
    return F.scal(acc, scale)


def assert_rows(got, want, what):
    bad = np.nonzero((got != want).any(axis=1))[0]
    if bad.size:
        i = bad[0]
        pytest.fail(f"{what}: {bad.size} of {len(want)} rows differ; first at row {i}: got limbs {[hex(x) for x in got[i]]}, "
                    f"want {[hex(x) for x in want[i]]}")


def check_mode0(ref, cs, cols, challenges=()):
    outs, nregs = run(ref, cs, cols, challenges)
    for gi, (got, want) in enumerate(zip(outs, gate_values(ref, cs, cols, challenges))):
        assert_rows(got, want, f"gate {gi}")
    return nregs


def check_mode1(ref, cs, cols, challenges, y, scale):
    (got,), nregs = run(ref, cs, cols, challenges, mode=1, y=y, scale=scale)
    assert_rows(got, folded(ref, cs, cols, challenges, y, scale), "folded gates")
    return nregs


def nested_product(r, width=8):
    """a right-nested product of r distinct queries (advice column j mod width at rotation j // width - 4): r live registers"""
    qs = [H.advice(j % width, j // width - 4) for j in range(r)]
    e = qs[-1]
    for q in reversed(qs[:-1]):
        e = q * e
    return e


# ---------------------------------------------------------------------------------------------------- register-file bands
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("r", [1, 8, 9, 16, 17, 44, 64])
def test_register_band(ref, r, mode):
    """Band edges 8/9 and 16/17 and the 64-register limit: the reported count is exactly r, and the values match."""
    cs = make_cs(7, [nested_product(r)], nf=0, ni=0)
    cols = make_cols(ref, cs, seed=r)
    nregs = check_mode0(ref, cs, cols) if mode == 0 else check_mode1(ref, cs, cols, (), y=0x1234567, scale=R - 3)
    assert nregs == r


@pytest.mark.parametrize("mode", [0, 1])
def test_more_than_64_registers_is_an_error(ref, mode):
    from zkb200 import ZkbError
    cs = make_cs(3, [nested_product(65)], nf=0, ni=0)
    with pytest.raises(ZkbError, match="more than 64 live registers"):
        run(ref, cs, make_cols(ref, cs, seed=65), mode=mode, y=5, scale=1)


@pytest.mark.parametrize("r", [8, 16, 44])
def test_register_band_at_k20(ref, r):
    """The production row count, once per build: 2^20 rows, 8192 blocks."""
    cs = make_cs(20, [nested_product(r)], nf=0, ni=0)
    assert check_mode0(ref, cs, make_cols(ref, cs, seed=100 + r)) == r


# ---------------------------------------------------------------------------------------------------- rotations and sizes
@pytest.mark.parametrize("k", [1, 3, 6, 7, 10, 17])
def test_rotations_wrap(ref, k):
    """Rotations 0, +-1, +-(n-1) and the 16-bit limit +-32767 (many wraps at small k); every row is compared, so the reads that
    wrap at row 0 and at row n-1 are checked.  k = 1 and 3 are less than one 128-thread block."""
    n = 1 << k
    rots = sorted(r for r in {0, 1, -1, n - 1, -(n - 1), 32767, -32767} if abs(r) <= 32767)
    gates = []
    for r in rots:
        gates += [H.advice(0, r), H.fixed(0, r), H.instance(0, r), H.advice(1, r) * H.advice(2, -r) + H.fixed(1, r)]
    cs = make_cs(k, gates, na=3)
    cols = make_cols(ref, cs, seed=k)
    assert check_mode0(ref, cs, cols) <= 8
    assert check_mode1(ref, cs, cols, (), y=0xABCDEF, scale=7) <= 8


# ---------------------------------------------------------------------------------------------------- DAG shapes and field edges
def dag_gates():
    a, b, c, d = (H.advice(i) for i in range(4))
    s = a * b + H.advice(2, 1)                      # shared inside the scope: its register lives until its last use
    t = -(s * s) + H.scaled(s, 5)
    x = a
    for _ in range(6):                               # x_{i+1} = x_i * x_i + b(-1): every level used twice
        x = x * x + H.advice(1, -1)
    return [s * H.advice(3, -1), s * s, (s + c) * s,
            t, t,                                    # one node as two roots
            H.advice(4, 2), H.const(0), H.const(R - 1),   # roots that are a bare column or a bare constant
            -(-a) + (-b), a + (-a),
            H.scaled(a, 5) + H.const(5) * b,         # duplicate constants are deduplicated by value
            H.challenge(0) * a + H.challenge(1),
            H.const(7) * c + H.challenge(2) * d,     # challenge 2 equals the constant 7
            x, x * s,
            H.instance(0, -1) * H.fixed(1, 3)] + [H.const(e) * a + H.scaled(b, e) for e in EDGES]


@pytest.mark.parametrize("k", [3, 7])
def test_dag_shapes(ref, k):
    cs = make_cs(k, dag_gates(), nch=3)
    cols = make_cols(ref, cs, seed=11 * k)
    ch = [0x5EED, R - 1, 7]
    assert 1 <= check_mode0(ref, cs, cols, ch) <= 64
    assert 1 <= check_mode1(ref, cs, cols, ch, y=0x77777, scale=R - 1) <= 64


def test_field_edge_values(ref):
    """Every ordered pair of the edge values 0, 1, p-1, p-2, (p-1)/2 through add, negate, multiply and constants."""
    F = ref.F
    cs = make_cs(5, [], na=2, nf=1, ni=0)
    cols = make_cols(ref, cs, seed=5)
    e = F.arr(EDGES)
    m = len(EDGES)
    cols[H.ADVICE][0][: m * m] = np.repeat(e, m, axis=0)
    cols[H.ADVICE][1][: m * m] = np.tile(e, (m, 1))
    a, b = H.advice(0), H.advice(1)
    cs.gates = [a * b, a + b, -a, a + (-b), a * b * b, H.scaled(a, R - 1), a * H.const(R - 1) + H.const(R - 2),
                H.const((R - 1) // 2) * b + a * a]
    check_mode0(ref, cs, cols)
    check_mode1(ref, cs, cols, (), y=R - 1, scale=R - 2)


# ---------------------------------------------------------------------------------------------------- mode 1: selector runs
def fold_gates(long_run):
    q, q_rot = H.fixed(0), H.fixed(0, 1)

    def t(j):
        return H.advice(j % 4, j % 3 - 1) * H.advice((j + 1) % 4) + H.const(j + 2)
    gates = [q * t(0), q * t(1), q * t(2),
             t(3) * q, q * t(4),                     # the selector on the right-hand side continues the run
             q_rot * t(5), q_rot * t(6),             # same column at another rotation: a new run
             H.advice(0) * H.advice(1),              # a single gate without selector between runs
             q * t(7),                               # a run of one
             H.fixed(1) * t(8), q * H.fixed(1), H.fixed(1) * q,   # both sides fixed
             q * t(9), H.advice(2) + H.const(3), q * t(10)]
    gates += [q * t(11 + j) for j in range(long_run)]     # longer than the 4096-gate cap of a run
    gates += [q * t(1)]
    return gates


@pytest.mark.parametrize("y", [0x1D1CE, R - 1, 0], ids=["random", "p-1", "zero"])
def test_selector_run_folding(ref, y):
    """quotient_gates' rewrite (HORNER2 / FOLD) against the term-by-term Horner fold: runs broken by rotation, selectors on
    either side, single gates between runs, and a run past the 4096 cap."""
    cs = make_cs(4, fold_gates(4100), na=4, ni=0)
    cols = make_cols(ref, cs, seed=y & 0xFFFF)
    assert check_mode1(ref, cs, cols, (), y=y, scale=0x5CA1E) <= 8


@pytest.mark.parametrize("stride,offset", [(1, 0), (1, 7), (8, 0), (8, 7)])
def test_coset_part_output(ref, stride, offset):
    """Strided output of a coset part (row i -> out[i * stride + offset]): written entries match, all others keep the sentinel."""
    cs = make_cs(6, fold_gates(20) + dag_gates(), na=5, nch=3)
    cols = make_cols(ref, cs, seed=stride * 10 + offset)
    ch = [3, 1, 7]
    n = cs.n
    buf = np.full((n * stride + offset + stride, 4), SENTINEL, dtype=np.uint64)
    (got,), nregs = run(ref, cs, cols, ch, mode=1, y=0xC05E7, scale=0xBEEF, out=buf, out_stride=stride, out_offset=offset)
    rows = np.arange(n) * stride + offset
    assert_rows(got[rows], folded(ref, cs, cols, ch, 0xC05E7, 0xBEEF), f"stride {stride} offset {offset}")
    untouched = np.ones(len(got), dtype=bool)
    untouched[rows] = False
    assert (got[untouched] == SENTINEL).all(), "an entry outside row * stride + offset was written"
    assert 1 <= nregs <= 64
