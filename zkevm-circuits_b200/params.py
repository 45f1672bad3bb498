"""Host mirror of halo2_proofs::poly::kzg::commitment::ParamsKZG<Bn256> (the prover-side fields) built on the GPU.

`unsafe_setup_with_s` follows ParamsKZG::unsafe_setup_with_s (used by the reference at
zkevm-circuits/src/super_circuit/test.rs:74): g[i] = [s^i] G1, g_lagrange[i] = [L_i(s)] G1 with
L_i(s) = w^i (s^n - 1) / (n (s - w^i)).  All arithmetic runs through the CUDA kernels (no CPU field code here).
"""
import numpy as np

from . import arithmetic as A
from . import poly


def fr_scalar_dev(v, device="cuda"):
    """python int -> 1-element device tensor holding the Montgomery form (conversion done by the device kernel)."""
    import torch
    limbs = [(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)]
    t = torch.from_numpy(np.array([limbs], dtype=np.uint64).view(np.int64)).to(device)
    return A.field_unop_dev(A.FR, A.UOP_TO_MONT, t)


def fr_ints_to_dev(vals_int64, device="cuda"):
    """int64 tensor of small non-negative values (n,) -> (n,4) Montgomery tensor."""
    import torch
    z = torch.zeros((vals_int64.shape[0], 4), dtype=torch.int64, device=device)
    z[:, 0] = vals_int64
    return A.field_unop_dev(A.FR, A.UOP_TO_MONT, z)


def bcast(scalar_t, n):
    return scalar_t.expand(n, 4).contiguous()


def fr_pow2k_dev(t, k):
    for _ in range(k):
        t = A.field_unop_dev(A.FR, A.UOP_SQR, t)
    return t


def g1_generator():
    import torch
    g_can = torch.tensor([[1, 0, 0, 0], [2, 0, 0, 0]], dtype=torch.int64, device="cuda")
    return A.field_unop_dev(A.FQ, A.UOP_TO_MONT, g_can).cpu().numpy().view(np.uint64).reshape(8)


class ParamsKZG:
    def __init__(self, k, g, g_lagrange, g2=None, s_g2=None):
        self.k, self.n = k, 1 << k
        self.g, self.g_lagrange = g, g_lagrange          # (n, 8) device tensors (or host numpy arrays when read without a GPU)
        self.g2, self.s_g2 = g2, s_g2                    # opaque 128-byte raw G2 points (only the verifier uses them)

    # ---- params file I/O: ParamsKZG::read_custom / write_custom with SerdeFormat::RawBytes[Unchecked] --------------------
    # Layout checked by the reference loader prover/src/utils.rs:56-75: 4 B k (LE u32) | g: 2^k x 64 B | g_lagrange: 2^k x 64 B |
    # g2: 128 B | s_g2: 128 B, i.e. 4 + 2 * 2^k * 64 + 2 * 128 bytes; a raw G1 point is x || y as 4 x u64 LE Montgomery limbs
    # each -- byte for byte the in-memory G1Affine the kernels consume, so loading is a copy.
    @staticmethod
    def expected_file_len(k):
        return 4 + 2 * (1 << k) * 64 + 2 * 128

    @staticmethod
    def read_custom(path, to_device=True):
        import os
        with open(path, "rb") as f:
            raw = f.read()
        k = int.from_bytes(raw[:4], "little")
        if len(raw) != ParamsKZG.expected_file_len(k):
            raise ValueError(f"invalid params file len {len(raw)} for degree {k}")
        n = 1 << k
        g = np.frombuffer(raw, dtype=np.uint64, count=n * 8, offset=4).reshape(n, 8).copy()
        gl = np.frombuffer(raw, dtype=np.uint64, count=n * 8, offset=4 + n * 64).reshape(n, 8).copy()
        g2 = raw[4 + 2 * n * 64: 4 + 2 * n * 64 + 128]
        s_g2 = raw[4 + 2 * n * 64 + 128:]
        if to_device:
            import torch
            g = torch.from_numpy(g.view(np.int64)).cuda()
            gl = torch.from_numpy(gl.view(np.int64)).cuda()
        return ParamsKZG(k, g, gl, g2, s_g2)

    def write_custom(self, path):
        def host(a):
            return a if isinstance(a, np.ndarray) else a.cpu().numpy().view(np.uint64)
        with open(path, "wb") as f:
            f.write(int(self.k).to_bytes(4, "little"))
            f.write(np.ascontiguousarray(host(self.g)).tobytes())
            f.write(np.ascontiguousarray(host(self.g_lagrange)).tobytes())
            f.write(self.g2 if self.g2 is not None else bytes(128))
            f.write(self.s_g2 if self.s_g2 is not None else bytes(128))

    @staticmethod
    def unsafe_setup_with_s(k, s):
        n = 1 << k
        gen = g1_generator()
        s_t = fr_scalar_dev(s)
        s_host = s_t.cpu().numpy().view(np.uint64)[0]
        pw = poly.fr_powers_dev(s_host, n)
        g = A.g1_fixed_base_mul_dev(gen, pw)
        omega, _ = A.root_of_unity(k)
        W = poly.fr_powers_dev(omega, n)
        den = A.field_binop_dev(A.FR, A.OP_SUB, bcast(s_t, n), W)
        inv = A.fr_batch_invert_dev(den)
        one = fr_scalar_dev(1)
        c1 = A.field_binop_dev(A.FR, A.OP_MUL, A.field_binop_dev(A.FR, A.OP_SUB, fr_pow2k_dev(s_t, k), one),
                               A.field_unop_dev(A.FR, A.UOP_INV, fr_scalar_dev(n)))
        L = A.field_binop_dev(A.FR, A.OP_MUL, A.field_binop_dev(A.FR, A.OP_MUL, W, inv), bcast(c1, n))
        gl = A.g1_fixed_base_mul_dev(gen, L)
        return ParamsKZG(k, g, gl)

    def commit_lagrange(self, values_dev):
        return A.best_multiexp_dev(values_dev, self.g_lagrange)

    def commit(self, coeffs_dev):
        return A.best_multiexp_dev(coeffs_dev, self.g[: coeffs_dev.shape[0]].contiguous())

    def load(self, ctx=None, derive_lagrange=False):
        """-> Srs: the device-resident handle (zkb_srs_load); shared by every ProvingKey created from it."""
        return Srs.from_params(self, ctx=ctx, derive_lagrange=derive_lagrange)


class Srs:
    """zkb_srs handle: ParamsKZG resident on one GPU (prover/src/common/prover.rs:37-57 keeps one per degree and downsizes)."""

    def __init__(self, ctx, handle):
        self.ctx, self.handle = ctx, handle

    @staticmethod
    def from_params(params, ctx=None, derive_lagrange=False):
        import ctypes
        from .lib import check, default_context
        ctx = ctx or default_context()
        h = ctypes.c_void_p()
        g, gl = params.g, (None if derive_lagrange else params.g_lagrange)
        if isinstance(g, np.ndarray):
            g = np.ascontiguousarray(g)
            glp = np.ascontiguousarray(gl) if gl is not None else None
            check(ctx.lib.zkb_srs_load(ctx.handle, params.k, ctypes.c_void_p(g.ctypes.data), ctypes.c_void_p(glp.ctypes.data) if glp is not None else None,
                                       ctypes.byref(h)))
        else:
            A.sync_current_stream()
            check(ctx.lib.zkb_srs_load_dev(ctx.handle, params.k, ctypes.c_void_p(g.data_ptr()), ctypes.c_void_p(gl.data_ptr()) if gl is not None else None,
                                           ctypes.byref(h)))
        return Srs(ctx, h)

    @property
    def k(self):
        return int(self.ctx.lib.zkb_srs_k(self.handle))

    def downsize(self, new_k):
        """ParamsKZG::downsize: g truncated, g_lagrange recomputed by the group iFFT on the device."""
        import ctypes
        from .lib import check
        h = ctypes.c_void_p()
        check(self.ctx.lib.zkb_srs_downsize(self.handle, int(new_k), ctypes.byref(h)))
        return Srs(self.ctx, h)

    def read(self, basis):
        """basis 0 = g, 1 = g_lagrange -> uint64 (n, 8) host array."""
        import ctypes
        from .lib import check
        out = np.empty((1 << self.k, 8), dtype=np.uint64)
        check(self.ctx.lib.zkb_srs_read(self.handle, int(basis), ctypes.c_void_p(out.ctypes.data)))
        return out

    def _commit(self, basis, scalars_dev):
        import ctypes
        from .lib import check
        out = np.zeros(8, dtype=np.uint64)
        comp = (ctypes.c_uint8 * 32)()
        check(self.ctx.lib.zkb_srs_commit_dev(self.handle, basis, ctypes.c_void_p(scalars_dev.data_ptr()), scalars_dev.shape[0],
                                              ctypes.c_void_p(out.ctypes.data), ctypes.cast(comp, ctypes.c_void_p), A._cur_stream()))
        return A.MsmResult(out, None, bytes(comp))

    def commit(self, coeffs_dev):
        return self._commit(0, coeffs_dev)

    def commit_lagrange(self, values_dev):
        return self._commit(1, values_dev)

    def commit_batch(self, basis, cols_dev):
        """zkb_srs_commit_batch_dev: several device columns of equal length against basis 0 = g / 1 = g_lagrange, in passes of
        msm_max_batch columns (how the prover commits a phase) -> uint64 (len(cols_dev), 8) affine points."""
        import ctypes
        from .lib import check
        ptrs = (ctypes.c_void_p * len(cols_dev))(*[c.data_ptr() for c in cols_dev])
        out = np.zeros((len(cols_dev), 8), dtype=np.uint64)
        check(self.ctx.lib.zkb_srs_commit_batch_dev(self.handle, int(basis), ctypes.cast(ptrs, ctypes.c_void_p), len(cols_dev), cols_dev[0].shape[0],
                                                    ctypes.c_void_p(out.ctypes.data), A._cur_stream()))
        return out

    def close(self):
        if self.handle and self.ctx.handle:   # not after its context: see plonk.ProvingKey.close
            self.ctx.lib.zkb_srs_destroy(self.handle)
        self.handle = None

    def __del__(self):
        try: self.close()
        except Exception: pass
