"""GPU: ParamsKZG::setup on the device (zkb_srs_setup_dev, csrc/setup.cu) against three independent routes:
  - the previous composition (fr_powers_dev, the closed form with fr_batch_invert_dev, then the double-and-add kernel
    g1_fixed_base_mul_dev), byte for byte over whole arrays up to k = 20;
  - Python-integer scalars s^i and w^i (s^n - 1) / (n (s - w^i)) through the oracle's fixed-base multiplication (and through
    g1_fixed_base_mul_dev at every CTA boundary of the comb launch), sampled at k = 23 and 26;
  - the group iFFT of g (zkb_srs_load with g_lagrange NULL, downsize's route), including s a root of unity.
The file round trip, the argument errors and a proof decided by a real pairing against the returned g2 / s_g2 close it."""
import ctypes

import numpy as np
import pytest

import fixed_base_model as FB
import pairing_ref as E
import pyref as P
from util import to_dev, to_host

pytestmark = pytest.mark.gpu

R = P.R_MOD


def old_composition(k, s):
    """the previous Python body of unsafe_setup_with_s, kept as a reference"""
    from zkb200 import arithmetic as A, poly
    from zkb200.params import bcast, fr_pow2k_dev, fr_scalar_dev, g1_generator
    n = 1 << k
    gen = g1_generator()
    s_t = fr_scalar_dev(s)
    pw = poly.fr_powers_dev(s_t.cpu().numpy().view(np.uint64)[0], n)
    g = A.g1_fixed_base_mul_dev(gen, pw)
    omega, _ = A.root_of_unity(k)
    W = poly.fr_powers_dev(omega, n)
    inv = A.fr_batch_invert_dev(A.field_binop_dev(A.FR, A.OP_SUB, bcast(s_t, n), W))
    one = fr_scalar_dev(1)
    c1 = A.field_binop_dev(A.FR, A.OP_MUL, A.field_binop_dev(A.FR, A.OP_SUB, fr_pow2k_dev(s_t, k), one),
                           A.field_unop_dev(A.FR, A.UOP_INV, fr_scalar_dev(n)))
    L = A.field_binop_dev(A.FR, A.OP_MUL, A.field_binop_dev(A.FR, A.OP_MUL, W, inv), bcast(c1, n))
    return g, A.g1_fixed_base_mul_dev(gen, L)


def setup(k, s):
    from zkb200.params import ParamsKZG
    return ParamsKZG.setup(k, s)


def mont_limbs(vals):
    return np.array([P.limbs(P.to_mont(v % R, R)) for v in vals], dtype=np.uint64).reshape(-1, 4)


def lagrange_ints(k, s, idx):
    n, w = 1 << k, P.omega(k)
    c1 = (pow(s, n, R) - 1) * pow(n, -1, R) % R
    out = []
    for i in idx:
        wi = pow(w, int(i), R)
        out.append(wi * c1 * pow((s - wi) % R, -1, R) % R)
    return out


def sample_indices(k, rng):
    n = 1 << k
    ends = np.concatenate([np.arange(64), np.arange(n - 64, n)])
    return np.unique(np.concatenate([ends, rng.integers(0, n, 4096)]))


def cta_boundaries(k):
    """both sides of every CTA boundary of the comb launch (2n points, CTAs of FB.COMB_T) as indices into g and g_lagrange"""
    n = 1 << k
    b = np.arange(FB.COMB_T, n + 1, FB.COMB_T)
    return np.unique(np.concatenate([b - 1, b[b < n]]))


@pytest.mark.parametrize("k", [0, 1, 2, 3, 5, 10, 11, 16, 20])
def test_whole_arrays_equal_the_previous_composition(k):
    s = 0x5EED0000 + 7 * k
    p = setup(k, s)
    g, gl = old_composition(k, s)
    assert p.g.shape == (1 << k, 8) and p.g_lagrange.shape == (1 << k, 8)
    assert (to_host(p.g) == to_host(g)).all()
    assert (to_host(p.g_lagrange) == to_host(gl)).all()


@pytest.mark.parametrize("k", [23, 26])
def test_sampled_indices_at_large_k(oracle, k):
    import torch
    from zkb200 import arithmetic as A
    s = 0xC0FFEE0000 + k
    p = setup(k, s)
    G = oracle.g1_generator()
    rng = np.random.default_rng(k)
    idx = sample_indices(k, rng)
    bnd = cta_boundaries(k)
    every = np.unique(np.concatenate([idx, bnd]))
    pw = mont_limbs([pow(s, int(i), R) for i in every])
    lag = mont_limbs(lagrange_ints(k, s, every))
    it = torch.from_numpy(every).cuda()
    got_g, got_l = to_host(p.g[it]), to_host(p.g_lagrange[it])
    # every index against the double-and-add kernel, the sampled ones also against the oracle
    assert (got_g == to_host(A.g1_fixed_base_mul_dev(G, to_dev(pw)))).all()
    assert (got_l == to_host(A.g1_fixed_base_mul_dev(G, to_dev(lag)))).all()
    sel = np.isin(every, idx)
    assert (got_g[sel] == oracle.g1_fixed_base_mul(G, np.ascontiguousarray(pw[sel]))).all()
    assert (got_l[sel] == oracle.g1_fixed_base_mul(G, np.ascontiguousarray(lag[sel]))).all()


def group_ifft_lagrange(p):
    from zkb200.params import ParamsKZG
    srs = ParamsKZG(p.k, np.ascontiguousarray(to_host(p.g)), None).load(derive_lagrange=True)
    try:
        return srs.read(1)
    finally:
        srs.close()


@pytest.mark.parametrize("k", [4, 9, 12])
def test_group_ifft_route(oracle, k):
    n, w = 1 << k, P.omega(k)
    G = oracle.g1_generator()
    p = setup(k, 0xAB5EED + k)
    assert (to_host(p.g_lagrange) == group_ifft_lagrange(p)).all()
    for j, s in [(0, 1), (n // 2, R - 1), (3, pow(w, 3, R)), (n - 1, pow(w, n - 1, R))]:
        p = setup(k, s)
        gl = to_host(p.g_lagrange)
        assert (gl == group_ifft_lagrange(p)).all(), f"s = w^{j}"
        nz = np.flatnonzero(gl.any(axis=1))
        assert list(nz) == [j] and (gl[j] == G).all()


def test_edge_s(oracle):
    k, n = 10, 1 << 10
    G = oracle.g1_generator()
    p = setup(k, 0)
    g = to_host(p.g)
    assert (g[0] == G).all() and not g[1:].any()
    inv_n = oracle.g1_fixed_base_mul(G, mont_limbs([pow(n, -1, R)]))[0]
    assert (to_host(p.g_lagrange) == inv_n[None, :]).all()
    for s in (R - 2, FB.top_carry_scalar()):
        p = setup(k, s)
        g, gl = old_composition(k, s)
        assert (to_host(p.g) == to_host(g)).all() and (to_host(p.g_lagrange) == to_host(gl)).all()
        assert (to_host(p.g[1:2]) == oracle.g1_fixed_base_mul(G, mont_limbs([s]))).all()


def _call(k, s_limbs, g, gl, stream=None):
    from zkb200.lib import default_context
    ctx = default_context()
    s_h = np.ascontiguousarray(np.asarray(s_limbs, dtype=np.uint64))
    ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    return ctx.lib.zkb_srs_setup_dev(ctx.handle, k, ctypes.c_void_p(s_h.ctypes.data), ptr(g), ptr(gl), stream)


def test_repeat_and_stream_give_the_same_bytes():
    import torch
    k, s = 14, 0x5151
    a, b = setup(k, s), setup(k, s)
    assert (to_host(a.g) == to_host(b.g)).all() and (to_host(a.g_lagrange) == to_host(b.g_lagrange)).all()
    st = torch.cuda.Stream()
    g = torch.empty((1 << k, 8), dtype=torch.int64, device="cuda")
    gl = torch.empty_like(g)
    torch.cuda.synchronize()
    assert _call(k, mont_limbs([s])[0], g, gl, ctypes.c_void_p(st.cuda_stream)) == 0
    assert (to_host(g) == to_host(a.g)).all() and (to_host(gl) == to_host(a.g_lagrange)).all()


def test_argument_errors_leave_outputs_untouched():
    import torch
    k = 4
    g = torch.full((1 << k, 8), 7, dtype=torch.int64, device="cuda")
    gl = torch.full((1 << k, 8), 7, dtype=torch.int64, device="cuda")
    good = mont_limbs([5])[0]
    cases = [(29, good, g, gl), (k, np.array(P.limbs(R), dtype=np.uint64), g, gl),
             (k, np.array(P.limbs((1 << 256) - 1), dtype=np.uint64), g, gl), (k, good, None, gl), (k, good, g, None)]
    for kk, s, a, b in cases:
        assert _call(kk, s, a, b) == -2
        torch.cuda.synchronize()
        assert (g == 7).all() and (gl == 7).all()


@pytest.mark.parametrize("fmt", ["Processed", "RawBytes", "RawBytesUnchecked"])
def test_file_round_trip(tmp_path, fmt):
    from zkb200.params import ParamsKZG, SerdeFormat
    f = SerdeFormat[fmt]
    p = setup(10, 0xF11E)
    path = tmp_path / "params.bin"
    p.write_custom(str(path), f)
    assert path.stat().st_size == ParamsKZG.expected_file_len(10, f)
    q = ParamsKZG.read_custom(str(path), f)
    assert (to_host(q.g) == to_host(p.g)).all() and (to_host(q.g_lagrange) == to_host(p.g_lagrange)).all()
    assert q.g2 == p.g2 and q.s_g2 == p.s_g2 and p.s_g2 != bytes(128)


def raw_g2(raw):
    v = np.frombuffer(raw, dtype=np.uint64).reshape(4, 4)
    c = [P.from_mont(P.from_limbs(row), P.Q_MOD) for row in v]
    return E.FQ2([c[0], c[1]]), E.FQ2([c[2], c[3]])


def test_proof_against_the_setup_verifies_with_a_pairing():
    """A k = 10 proof made against ParamsKZG.setup(k, s).load() is accepted by the oracle verifier whose final check is a
    real pairing against the g2 / s_g2 the setup returned, and a flipped proof byte is rejected."""
    import halo2_ref as H
    from circuits import ToyCircuit
    from test_gpu_prover import to_product_cs
    from zkb200 import plonk as Z
    k, s = 10, 0x5E7C0DE
    p = setup(k, s)
    tc = ToyCircuit(k, seed=21)
    ref = H.Ref(tc.cs, s)
    F = ref.F
    assert (to_host(p.g) == ref.g).all() and (to_host(p.g_lagrange) == ref.g_lagrange).all()
    fixed = [F.arr(c) for c in tc.fixed_ints]
    pkr = ref.keygen(fixed, tc.copies)
    rp = F.arr(tc.blinds_ints["random_poly"])
    pk = Z.ProvingKey(to_product_cs(tc.cs, ref.bf, ref.d), fixed, pkr["sigma_values"], srs=p.load())
    synth = lambda ph, ch: {c: F.arr(v) for c, v in tc.advice_ints(ph, {i: F.ints(v[None])[0] for i, v in ch.items()}).items()}
    proof = Z.create_proof(pk, F.arr([tc.transcript_repr])[0], [F.arr(c) for c in tc.instances], synth,
                           np.concatenate([F.arr(b) for b in tc.blinds_ints["z"]]), np.concatenate([F.arr(b) for b in tc.blinds_ints["phi"]]), rp)
    g2, s_g2 = raw_g2(p.g2), raw_g2(p.s_g2)
    assert E.g2_is_on_curve(g2) and E.g2_is_on_curve(s_g2)
    decide = lambda lhs, rhs: E.pairing_product_is_one([(lhs, g2), (P.g1_neg(rhs), s_g2)])   # e(lhs, g2) == e(rhs, [s]g2)
    assert ref.verify_proof(pkr, tc.transcript_repr, tc.instances, proof, decide=decide)
    bad = bytearray(proof)
    bad[len(bad) // 2] ^= 1
    try:   # rejected: the verifier returns False, or refuses a point that no longer decodes
        accepted = ref.verify_proof(pkr, tc.transcript_repr, tc.instances, bytes(bad), decide=decide)
    except Exception:
        accepted = False
    assert not accepted
