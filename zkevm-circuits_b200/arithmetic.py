"""Host-side mirror of halo2_proofs::arithmetic for the accelerated path (names and argument meaning follow
halo2_proofs 1.1.0 @ e5ddf67 src/arithmetic.rs: `best_fft(a, omega, log_n)`, `best_multiexp(coeffs, bases)`).

Array conventions (halo2curves in-memory layout): Fr/Fq = 4 little-endian u64 limbs in Montgomery form.
  host   : numpy uint64 arrays, shape (n, 4) for scalars, (n, 8) for G1Affine
  device : torch int64 CUDA tensors of the same shapes (torch has no uint64 arithmetic; only storage is used)
Every function drives the CUDA kernels through the C ABI; nothing here computes on the CPU (arith_probe_host runs the library's
own host-compiled primitives, for tests).
"""
import ctypes
import numpy as np

from .lib import check, default_context

_vp = ctypes.c_void_p


def _np_ptr(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"], "need a C-contiguous uint64 array"
    return _vp(a.ctypes.data)


def _limbs_ptr(x):
    """4-limb Fr given as numpy uint64[4] -> (keepalive, pointer)."""
    a = np.ascontiguousarray(np.asarray(x, dtype=np.uint64).reshape(4))
    return a, _vp(a.ctypes.data)


def _cur_stream():
    """torch's current stream as a cudaStream_t.  torch reports the legacy default stream as 0, which the C ABI reads
    as "use the context's own stream"; pass cudaStreamLegacy (0x1) instead so launches stay ordered with torch's work."""
    import torch
    s = torch.cuda.current_stream().cuda_stream
    return _vp(s if s else 1)


def sync_current_stream():
    """wait for torch's current stream (entry points that work on the context's own stream read tensors torch produced)"""
    import torch
    torch.cuda.current_stream().synchronize()


def root_of_unity(k):
    """(omega, omega_inv) of the 2^k domain: Fr::ROOT_OF_UNITY^(2^(28-k)) (EvaluationDomain::new)."""
    from .lib import load_library
    w = np.zeros(4, dtype=np.uint64)
    wi = np.zeros(4, dtype=np.uint64)
    check(load_library().zkb_fr_root_of_unity(int(k), _np_ptr(w), _np_ptr(wi)))
    return w, wi


def best_fft(a, omega, log_n, scale=None, coset_zeta=0, ctx=None):
    """In-place NTT of a host array (H2D + kernels + D2H inside).  a: numpy uint64 (2^log_n, 4)."""
    ctx = ctx or default_context()
    assert a.shape == (1 << log_n, 4)
    wk, wp = _limbs_ptr(omega)
    if scale is not None:
        sk, sp = _limbs_ptr(scale)
    else:
        sk, sp = None, None
    check(ctx.lib.zkb_ntt_fr_host(ctx.handle, _np_ptr(a), int(log_n), wp, sp, int(coset_zeta)))
    return a


def best_fft_pinned(t, omega, log_n, scale=None, coset_zeta=0, ctx=None):
    """Same as best_fft for a pinned CPU torch tensor (int64, (n,4)) -- the end-to-end benchmark path."""
    ctx = ctx or default_context()
    assert (not t.is_cuda) and t.is_contiguous() and t.numel() == 4 << log_n
    wk, wp = _limbs_ptr(omega)
    sk, sp = _limbs_ptr(scale) if scale is not None else (None, None)
    check(ctx.lib.zkb_ntt_fr_host(ctx.handle, _vp(t.data_ptr()), int(log_n), wp, sp, int(coset_zeta)))
    return t


def best_fft_dev(t, omega, log_n, scale=None, coset_zeta=0, ctx=None):
    """In-place NTT of a device tensor on torch's current stream (no synchronisation)."""
    ctx = ctx or default_context(t.device.index)
    assert t.is_cuda and t.is_contiguous() and t.numel() == 4 << log_n
    wk, wp = _limbs_ptr(omega)
    sk, sp = _limbs_ptr(scale) if scale is not None else (None, None)
    check(ctx.lib.zkb_ntt_fr_dev(ctx.handle, _vp(t.data_ptr()), int(log_n), wp, sp, int(coset_zeta), _cur_stream()))
    return t


class MsmResult:
    def __init__(self, affine, jacobian, compressed):
        self.affine = affine          # numpy uint64[8]  (x, y) Montgomery; identity = zeros
        self.jacobian = jacobian      # numpy uint64[12] (x, y, z) with z = 1 (or 0 for the identity)
        self.compressed = compressed  # bytes, G1Affine::to_bytes


def _msm_out():
    aff = np.zeros(8, dtype=np.uint64)
    jac = np.zeros(12, dtype=np.uint64)
    comp = (ctypes.c_uint8 * 32)()
    return aff, jac, comp


def best_multiexp(coeffs, bases, ctx=None):
    """sum_i coeffs[i] * bases[i] for host arrays (H2D inside).  coeffs: (n,4) uint64, bases: (n,8) uint64."""
    ctx = ctx or default_context()
    n = coeffs.shape[0]
    assert coeffs.shape == (n, 4) and bases.shape == (n, 8)
    aff, jac, comp = _msm_out()
    cp = _np_ptr(coeffs) if n else None
    bp = _np_ptr(bases) if n else None
    check(ctx.lib.zkb_msm_g1_host(ctx.handle, cp, bp, n, _np_ptr(aff), _np_ptr(jac), ctypes.cast(comp, _vp)))
    return MsmResult(aff, jac, bytes(comp))


def best_multiexp_pinned(coeffs_t, bases_t, ctx=None):
    """End-to-end path with pinned CPU torch tensors."""
    ctx = ctx or default_context()
    n = coeffs_t.shape[0]
    aff, jac, comp = _msm_out()
    check(ctx.lib.zkb_msm_g1_host(ctx.handle, _vp(coeffs_t.data_ptr()), _vp(bases_t.data_ptr()), n,
                                  _np_ptr(aff), _np_ptr(jac), ctypes.cast(comp, _vp)))
    return MsmResult(aff, jac, bytes(comp))


def best_multiexp_dev(coeffs_t, bases_t, ctx=None):
    """Device-resident inputs (torch int64 CUDA tensors (n,4), (n,8)); synchronises to return the point."""
    ctx = ctx or default_context(coeffs_t.device.index)
    n = coeffs_t.shape[0]
    assert coeffs_t.is_cuda and bases_t.is_cuda and coeffs_t.is_contiguous() and bases_t.is_contiguous()
    aff, jac, comp = _msm_out()
    check(ctx.lib.zkb_msm_g1_dev(ctx.handle, _vp(coeffs_t.data_ptr()), _vp(bases_t.data_ptr()), n,
                                 _np_ptr(aff), _np_ptr(jac), ctypes.cast(comp, _vp), _cur_stream()))
    return MsmResult(aff, jac, bytes(comp))


def best_multiexp_batch_dev(coeff_cols, bases_t, ctx=None):
    """Commit several scalar columns (list of device tensors (n,4)) against the same bases in one batched pass.
    Returns numpy uint64 (len(cols), 8) affine points."""
    ctx = ctx or default_context(bases_t.device.index)
    n = coeff_cols[0].shape[0]
    ptrs = (ctypes.c_void_p * len(coeff_cols))(*[c.data_ptr() for c in coeff_cols])
    out = np.zeros((len(coeff_cols), 8), dtype=np.uint64)
    check(ctx.lib.zkb_msm_g1_batch_dev(ctx.handle, ctypes.cast(ptrs, _vp), len(coeff_cols), _vp(bases_t.data_ptr()), n, _np_ptr(out), _cur_stream()))
    return out


def msm_last_adds(ctx=None):
    ctx = ctx or default_context()
    return int(ctx.lib.zkb_msm_last_adds(ctx.handle))


def g1_fixed_base_mul_dev(base_affine, scalars_t, ctx=None):
    """out[i] = [scalars[i]] base -> torch int64 CUDA tensor (n, 8).  Plain double-and-add: the independent
    reference of the SRS setup tests and the source of benchmark bases."""
    import torch
    ctx = ctx or default_context(scalars_t.device.index)
    n = scalars_t.shape[0]
    out = torch.empty((n, 8), dtype=torch.int64, device=scalars_t.device)
    b = np.ascontiguousarray(np.asarray(base_affine, dtype=np.uint64).reshape(8))
    check(ctx.lib.zkb_g1_fixed_base_mul_dev(ctx.handle, _np_ptr(b), _vp(scalars_t.data_ptr()), n, _vp(out.data_ptr()), _cur_stream()))
    return out


# ---- element-wise field kernels --------------------------------------------------------------------------------
FR, FQ = 0, 1
OP_ADD, OP_SUB, OP_MUL = 0, 1, 2
UOP_INV, UOP_TO_MONT, UOP_FROM_MONT, UOP_SQR, UOP_NEG = 0, 1, 2, 3, 4


def field_binop_dev(field, op, a, b, ctx=None):
    import torch
    ctx = ctx or default_context(a.device.index)
    out = torch.empty_like(a)
    check(ctx.lib.zkb_field_binop_dev(ctx.handle, field, op, _vp(a.data_ptr()), _vp(b.data_ptr()), _vp(out.data_ptr()),
                                      a.shape[0], _cur_stream()))
    return out


def field_unop_dev(field, op, a, ctx=None):
    import torch
    ctx = ctx or default_context(a.device.index)
    out = torch.empty_like(a)
    check(ctx.lib.zkb_field_unop_dev(ctx.handle, field, op, _vp(a.data_ptr()), _vp(out.data_ptr()), a.shape[0], _cur_stream()))
    return out


def fr_batch_invert_dev(a, ctx=None):
    import torch
    ctx = ctx or default_context(a.device.index)
    out = torch.empty_like(a)
    check(ctx.lib.zkb_fr_batch_invert_dev(ctx.handle, _vp(a.data_ptr()), _vp(out.data_ptr()), a.shape[0], _cur_stream()))
    return out


# ---- primitive probe (test surface of ff.cuh / g1.cuh, include/zkb200.h zkb_arith_probe_*) --------------------------------
# op -> (field elements read per record, field elements written per record)
PROBE_SHAPE = {0: (2, 1), 1: (2, 1), 2: (1, 1), 3: (1, 1), 4: (2, 1), 5: (1, 1), 6: (4, 1), 7: (4, 1), 8: (2, 1), 9: (2, 1),
               10: (2, 1), 11: (1, 1), 12: (1, 1), 13: (2, 1), 14: (2, 1), 15: (1, 1), 16: (1, 1), 17: (1, 1), 18: (1, 1),
               32: (6, 4), 33: (8, 4), 34: (4, 4), 35: (2, 4), 36: (4, 2), 37: (2, 2), 38: (2, 4)}


def arith_probe_dev(field, op, a, ctx=None):
    """Primitive `op` on every record of a (torch int64 CUDA tensor (n, arity * 4)) -> (n, width * 4), torch's current stream."""
    import torch
    ctx = ctx or default_context(a.device.index)
    arity, width = PROBE_SHAPE[op]
    assert a.is_cuda and a.is_contiguous() and a.dim() == 2 and a.shape[1] == 4 * arity
    out = torch.empty((a.shape[0], 4 * width), dtype=torch.int64, device=a.device)
    check(ctx.lib.zkb_arith_probe_dev(ctx.handle, field, op, _vp(a.data_ptr()), _vp(out.data_ptr()), a.shape[0], _cur_stream()))
    return out


def arith_probe_host(field, op, a):
    """The host-compiled branch of the same primitive: a numpy uint64 (n, arity * 4) -> (n, width * 4).  Needs no device."""
    from .lib import load_library
    arity, width = PROBE_SHAPE[op]
    a = np.ascontiguousarray(a, dtype=np.uint64)
    assert a.ndim == 2 and a.shape[1] == 4 * arity
    out = np.zeros((a.shape[0], 4 * width), dtype=np.uint64)
    check(load_library().zkb_arith_probe_host(field, op, _np_ptr(a), _np_ptr(out), a.shape[0]))
    return out


# ---- synthetic inputs (device-side, no oracle involved) ---------------------------------------------------------
FR_TOP_LIMB = 0x30644E72E131A029


def random_fr_dev(n, seed, device="cuda"):
    """n uniform-looking Fr elements as Montgomery limbs: the top limb is drawn below r's top limb so every value
    is < r; any bit pattern < r is the Montgomery form of some field element."""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    lo = torch.randint(-(1 << 63), (1 << 63) - 1, (n, 3), dtype=torch.int64, device=device, generator=g)
    hi = torch.randint(0, FR_TOP_LIMB, (n, 1), dtype=torch.int64, device=device, generator=g)
    return torch.cat([lo, hi], dim=1).contiguous()
