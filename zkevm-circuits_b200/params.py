"""Host mirror of halo2_proofs::poly::kzg::commitment::ParamsKZG<Bn256> (the prover-side fields) built on the GPU.

`setup` / `unsafe_setup_with_s` follow ParamsKZG::setup / unsafe_setup_with_s (used by the reference at
zkevm-circuits/src/super_circuit/test.rs:74): g[i] = [s^i] G1, g_lagrange[i] = [L_i(s)] G1 with
L_i(s) = w^i (s^n - 1) / (n (s - w^i)) through zkb_srs_setup_dev, g2 and s_g2 = [s] g2 through zkb_g2_setup_host.  All field
arithmetic runs in libzkb200 (no CPU field code here).
"""
import ctypes
import enum
from collections import namedtuple

import numpy as np

from . import arithmetic as A


class SerdeFormat(enum.IntEnum):
    """halo2_proofs::SerdeFormat, with the codes of zkb_g1_decode / zkb_g1_encode (include/zkb200.h)."""
    Processed = 0           # compressed: G1 32 B, G2 64 B; reading takes a square root per point
    RawBytes = 1            # the in-memory points (Montgomery limbs): G1 64 B, G2 128 B; reading checks limbs < q and the curve
    RawBytesUnchecked = 2   # the same bytes, read without a check (the reference prover's default, prover/src/utils.rs:33)

    @property
    def g1_len(self):
        return 32 if self is SerdeFormat.Processed else 64


DECODE_REASONS = {1: "has flag bit 7 set", 2: "has a coordinate >= q", 3: "is not on the curve"}
DecodeReport = namedtuple("DecodeReport", "first_bad count reason")   # first_bad is None when every point is good

# [s]G2 of the production setup (prover/src/utils.rs:36, PARAMS_G2_SECRET_POWER) in the raw 128-byte form: x.c0, x.c1, y.c0, y.c1,
# 4 x u64 LE Montgomery limbs each
PARAMS_G2_SECRET_POWER = (
    0xa911be278d071a14, 0xa66ec680042958fb, 0x7d2102725a5ed2fb, 0x2fb482eed95a462c,
    0xe81e349c63a38a7a, 0x18e6583e831884b4, 0x921b073b146926d1, 0x2b325d32a24da9ad,
    0xf0f4ae3615096f63, 0x51f0a3146f3c0c02, 0xa3c6c2623c4e999e, 0x209512c9d2d1086d,
    0xd8bcba5b3d674d1f, 0xf05e7d77bc27ef19, 0xa6323002e07b9911, 0x28fda6e0e2f6801f,
)


class _Report(ctypes.Structure):
    _fields_ = [("first_bad", ctypes.c_uint64), ("count", ctypes.c_uint64), ("reason", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


def _nbytes(a):
    return a.numel() * a.element_size() if hasattr(a, "data_ptr") else a.nbytes


def _ptr(a):
    if hasattr(a, "data_ptr"):
        assert a.is_contiguous()
        return ctypes.c_void_p(a.data_ptr())
    assert a.flags["C_CONTIGUOUS"]
    return ctypes.c_void_p(a.ctypes.data)


def g1_decode(fmt, src, n, out, ctx=None):
    """zkb_g1_decode: n G1 points encoded in `fmt` (src: uint8 numpy array or CUDA tensor) -> out ((n, 8) uint64 numpy array or
    int64 CUDA tensor; a bad point is written as (0, 0)).  Returns the DecodeReport."""
    from .lib import check, default_context
    fmt = SerdeFormat(fmt)
    assert _nbytes(src) >= n * fmt.g1_len and _nbytes(out) >= n * 64
    ctx = ctx or default_context()
    rep = _Report()
    check(ctx.lib.zkb_g1_decode(ctx.handle, int(fmt), _ptr(src) if n else None, n, _ptr(out) if n else None, ctypes.byref(rep),
                                A._cur_stream()))
    return DecodeReport(int(rep.first_bad) if rep.count else None, int(rep.count), int(rep.reason))


def g1_encode(fmt, points, out, ctx=None):
    """zkb_g1_encode: (n, 8) points (numpy uint64 or CUDA int64) -> out (uint8 numpy array or CUDA tensor of n * fmt.g1_len bytes)."""
    from .lib import check, default_context
    fmt = SerdeFormat(fmt)
    n = points.shape[0]
    assert _nbytes(points) == n * 64 and _nbytes(out) >= n * fmt.g1_len
    ctx = ctx or default_context()
    check(ctx.lib.zkb_g1_encode(ctx.handle, int(fmt), _ptr(points) if n else None, n, _ptr(out) if n else None, A._cur_stream()))
    return out


def g2_decode(fmt, data):
    """zkb_g2_decode_host: one encoded G2 point -> (raw 128 bytes, reason code; 0 = good).  Host only."""
    from .lib import check, load_library
    fmt = SerdeFormat(fmt)
    src = np.frombuffer(bytes(data), dtype=np.uint8)
    assert src.nbytes == 2 * fmt.g1_len
    out = np.zeros(16, dtype=np.uint64)
    status = ctypes.c_int32(0)
    check(load_library().zkb_g2_decode_host(int(fmt), _ptr(src), _ptr(out), ctypes.byref(status)))
    return out.tobytes(), int(status.value)


def g2_encode(fmt, raw):
    """zkb_g2_encode_host: a raw 128-byte G2 point -> its encoding in `fmt` (64 or 128 bytes).  Host only."""
    from .lib import check, load_library
    fmt = SerdeFormat(fmt)
    src = np.frombuffer(bytes(raw), dtype=np.uint64)
    assert src.size == 16
    out = np.zeros(2 * fmt.g1_len, dtype=np.uint8)
    check(load_library().zkb_g2_encode_host(int(fmt), _ptr(src), _ptr(out)))
    return out.tobytes()


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


def srs_setup_dev(k, s_mont, ctx=None):
    """zkb_srs_setup_dev: s_mont (4 Montgomery limbs, stored integer < r) -> (g, g_lagrange), (2^k, 8) int64 CUDA tensors."""
    import torch
    from .lib import check, default_context
    ctx = ctx or default_context()
    n = 1 << k
    s_h = np.ascontiguousarray(np.asarray(s_mont, dtype=np.uint64).reshape(4))
    g = torch.empty((n, 8), dtype=torch.int64, device=f"cuda:{ctx.device}")
    gl = torch.empty((n, 8), dtype=torch.int64, device=f"cuda:{ctx.device}")
    check(ctx.lib.zkb_srs_setup_dev(ctx.handle, int(k), _ptr(s_h), _ptr(g), _ptr(gl), A._cur_stream()))
    return g, gl


def g2_setup(s_mont):
    """zkb_g2_setup_host: -> (g2, [s] g2) as raw 128-byte points.  Host only."""
    from .lib import check, load_library
    s_h = np.ascontiguousarray(np.asarray(s_mont, dtype=np.uint64).reshape(4))
    g2, s_g2 = np.zeros(16, dtype=np.uint64), np.zeros(16, dtype=np.uint64)
    check(load_library().zkb_g2_setup_host(_ptr(s_h), _ptr(g2), _ptr(s_g2)))
    return g2.tobytes(), s_g2.tobytes()


def g1_generator():
    import torch
    g_can = torch.tensor([[1, 0, 0, 0], [2, 0, 0, 0]], dtype=torch.int64, device="cuda")
    return A.field_unop_dev(A.FQ, A.UOP_TO_MONT, g_can).cpu().numpy().view(np.uint64).reshape(8)


class ParamsKZG:
    def __init__(self, k, g, g_lagrange, g2=None, s_g2=None):
        self.k, self.n = k, 1 << k
        self.g, self.g_lagrange = g, g_lagrange          # (n, 8) device tensors (or host numpy arrays when read without a GPU)
        self.g2, self.s_g2 = g2, s_g2                    # raw 128-byte G2 points whatever the file format (only the verifier uses them)

    # ---- params file I/O: ParamsKZG::read_custom / write_custom ----------------------------------------------------------------
    # Layout checked by the reference loader prover/src/utils.rs:56-75: 4 B k (LE u32) | g: 2^k G1 | g_lagrange: 2^k G1 | g2 | s_g2,
    # i.e. 4 + 2 * 2^k * g1 + 2 * g2 bytes with g1 = 32 (Processed) or 64 (raw) and g2 = 2 * g1.  A raw G1 point is byte for byte
    # the in-memory G1Affine the kernels consume, so RawBytesUnchecked loading is a copy; the checked formats are decoded on the
    # GPU (zkb_g1_decode).  g2 / s_g2 are kept in the raw form, so a file converts between formats losslessly.
    @staticmethod
    def expected_file_len(k, fmt=SerdeFormat.RawBytesUnchecked):
        g1 = SerdeFormat(fmt).g1_len
        return 4 + 2 * (1 << k) * g1 + 2 * 2 * g1

    @staticmethod
    def _file_position(offset, k, g1):
        """the array element a byte offset of a params file falls in"""
        if offset < 4:
            return "the degree"
        n = 1 << k
        for name, size, count in (("g", g1, n), ("g_lagrange", g1, n), ("g2", 2 * g1, 1), ("s_g2", 2 * g1, 1)):
            if offset < 4 + size * count:
                return name if count == 1 else f"{name}[{(offset - 4) // size}]"
            offset -= size * count
        return "the end"

    @staticmethod
    def read_custom(path, fmt=SerdeFormat.RawBytesUnchecked, to_device=True):
        """ParamsKZG::read_custom.  A bad point in a checked format raises ValueError naming the array, the first bad index, the
        reason and the number of bad points in that array."""
        fmt = SerdeFormat(fmt)
        with open(path, "rb") as f:
            raw = f.read()
        k = int.from_bytes(raw[:4], "little")
        if k > 28:   # Fr's two-adicity: no domain, hence no params file, is larger
            raise ValueError(f"invalid params file: degree {k} > 28")
        want = ParamsKZG.expected_file_len(k, fmt)
        if len(raw) != want:
            where = (f"truncated at {ParamsKZG._file_position(len(raw), k, fmt.g1_len)}" if len(raw) < want
                     else f"{len(raw) - want} trailing bytes")
            raise ValueError(f"invalid params file len {len(raw)} for degree {k} ({fmt.name} expects {want}: {where})")
        n, g1 = 1 << k, fmt.g1_len
        off_g2 = 4 + 2 * n * g1
        if fmt is SerdeFormat.RawBytesUnchecked:
            g = np.frombuffer(raw, dtype=np.uint64, count=n * 8, offset=4).reshape(n, 8).copy()
            gl = np.frombuffer(raw, dtype=np.uint64, count=n * 8, offset=4 + n * 64).reshape(n, 8).copy()
            if to_device:
                import torch
                g = torch.from_numpy(g.view(np.int64)).cuda()
                gl = torch.from_numpy(gl.view(np.int64)).cuda()
            return ParamsKZG(k, g, gl, raw[off_g2: off_g2 + 128], raw[off_g2 + 128:])
        buf = np.frombuffer(raw, dtype=np.uint8)
        g = ParamsKZG._read_g1("g", fmt, buf[4: 4 + n * g1], n, to_device)
        gl = ParamsKZG._read_g1("g_lagrange", fmt, buf[4 + n * g1: off_g2], n, to_device)
        g2 = ParamsKZG._read_g2("g2", fmt, raw[off_g2: off_g2 + 2 * g1])
        s_g2 = ParamsKZG._read_g2("s_g2", fmt, raw[off_g2 + 2 * g1:])
        return ParamsKZG(k, g, gl, g2, s_g2)

    @staticmethod
    def _read_g1(name, fmt, src, n, to_device):
        if to_device:
            import torch
            out = torch.empty((n, 8), dtype=torch.int64, device="cuda")
        else:
            out = np.empty((n, 8), dtype=np.uint64)
        rep = g1_decode(fmt, src, n, out)
        if rep.count:
            raise ValueError(f"params file ({fmt.name}): {name}[{rep.first_bad}] {DECODE_REASONS[rep.reason]}; "
                             f"{rep.count} bad point(s) in {name}")
        return out

    @staticmethod
    def _read_g2(name, fmt, data):
        raw, status = g2_decode(fmt, data)
        if status:
            raise ValueError(f"params file ({fmt.name}): {name} {DECODE_REASONS[status]}")
        return raw

    def write_custom(self, path, fmt=SerdeFormat.RawBytesUnchecked):
        """ParamsKZG::write_custom; Processed points are encoded on the GPU (zkb_g1_encode)."""
        fmt = SerdeFormat(fmt)

        def host(a):
            return a if isinstance(a, np.ndarray) else a.cpu().numpy().view(np.uint64)

        def g1(a):
            if fmt is not SerdeFormat.Processed:
                return np.ascontiguousarray(host(a)).tobytes()
            out = np.empty(a.shape[0] * 32, dtype=np.uint8)
            return g1_encode(fmt, a if not isinstance(a, np.ndarray) else np.ascontiguousarray(a), out)

        def g2(raw):
            raw = raw if raw is not None else bytes(128)
            return raw if fmt is not SerdeFormat.Processed else g2_encode(fmt, raw)
        with open(path, "wb") as f:
            f.write(int(self.k).to_bytes(4, "little"))
            f.write(g1(self.g))
            f.write(g1(self.g_lagrange))
            f.write(g2(self.g2))
            f.write(g2(self.s_g2))

    def check_s_g2(self):
        """load_params' "Wrong params file" check (prover/src/utils.rs:78-80) as a point comparison: s_g2 must be the production
        [s]G2.  Raises ValueError otherwise."""
        if self.s_g2 != np.array(PARAMS_G2_SECRET_POWER, dtype=np.uint64).tobytes():
            raise ValueError(f"Wrong params file of degree {self.k}")

    @staticmethod
    def setup(k, s, ctx=None):
        """ParamsKZG::setup / new with the caller's trapdoor s (a python int; setup's random s is drawn by the caller): g and
        g_lagrange as (2^k, 8) device tensors (zkb_srs_setup_dev), g2 / s_g2 as raw 128-byte points (zkb_g2_setup_host).  When
        s^n = 1 g_lagrange is the true Lagrange basis (see include/zkb200.h), where upstream panics."""
        s_mont = fr_scalar_dev(s).cpu().numpy().view(np.uint64)[0].copy()
        g, gl = srs_setup_dev(k, s_mont, ctx=ctx)
        g2, s_g2 = g2_setup(s_mont)
        return ParamsKZG(k, g, gl, g2, s_g2)

    @staticmethod
    def unsafe_setup_with_s(k, s):
        return ParamsKZG.setup(k, s)

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
