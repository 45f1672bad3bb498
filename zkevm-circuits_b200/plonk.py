"""Host mirror of the prover-facing surface of halo2_proofs::plonk (names follow the crate: `Expression`,
`ConstraintSystem`, `ProvingKey`, `create_proof`) on top of the C ABI's proving session (`zkb_pk_*`, `zkb_prove_*`).

The reference reaches this surface at circuit-benchmarks/src/super_circuit.rs:109-132 (`keygen_pk`, `create_proof`).
Here a constraint system is described by plain Python objects (the Rust shim would serialise halo2's own
`ConstraintSystem` the same way, see INTEGRATION.md) and flattened into the CSF blob documented in include/zkb200.h.
Nothing in this module computes field arithmetic on the CPU; it only marshals buffers.
"""
import contextlib
import ctypes
import os
import struct
from collections import namedtuple

import numpy as np

from .lib import ZkbError, check, default_context

_vp = ctypes.c_void_p
CONST, FIXED, ADVICE, INSTANCE, CHALLENGE, NEG, ADD, MUL, SCALED = range(9)
CSF_MAGIC = 0x3146535A


class Expression:
    """plonk::Expression<Fr> (selectors already compiled into fixed columns)."""
    __slots__ = ("op", "a", "b")

    def __init__(self, op, a=None, b=None):
        self.op, self.a, self.b = op, a, b

    @staticmethod
    def Constant(limbs):               # limbs: 4 x u64 Montgomery
        return Expression(CONST, tuple(int(x) for x in limbs))

    @staticmethod
    def Fixed(col, rot=0): return Expression(FIXED, col, rot)
    @staticmethod
    def Advice(col, rot=0): return Expression(ADVICE, col, rot)
    @staticmethod
    def Instance(col, rot=0): return Expression(INSTANCE, col, rot)
    @staticmethod
    def Challenge(i): return Expression(CHALLENGE, i)
    def __neg__(self): return Expression(NEG, self)
    def __add__(self, o): return Expression(ADD, self, o)
    def __mul__(self, o): return Expression(MUL, self, o)
    def scaled(self, limbs): return Expression(SCALED, self, tuple(int(x) for x in limbs))


class ConstraintSystem:
    """The fields of plonk::ConstraintSystem the prover reads."""

    def __init__(self, k, num_fixed, num_advice, num_instance, advice_phase, challenge_phase, blinding_factors, degree):
        self.k, self.n = k, 1 << k
        self.num_fixed, self.num_advice, self.num_instance = num_fixed, num_advice, num_instance
        self.advice_phase, self.challenge_phase = list(advice_phase), list(challenge_phase)
        self.blinding_factors, self.degree = blinding_factors, degree
        self.gates, self.lookups, self.perm_columns = [], [], []      # lookups: (list of input-expression lists, table list)
        self.advice_queries, self.fixed_queries, self.instance_queries = [], [], []

    def num_phases(self):
        return max(self.advice_phase + self.challenge_phase + [0]) + 1

    def to_csf(self):
        nodes, consts, memo, cmemo = [], [], {}, {}

        def cidx(limbs):
            if limbs not in cmemo:
                cmemo[limbs] = len(consts)
                consts.append(limbs)
            return cmemo[limbs]

        def visit(e):
            key = id(e)
            if key in memo: return memo[key]
            if e.op == CONST: nd = (CONST, cidx(e.a), 0)
            elif e.op in (FIXED, ADVICE, INSTANCE): nd = (e.op, e.a, e.b & 0xFFFFFFFF)
            elif e.op == CHALLENGE: nd = (CHALLENGE, e.a, 0)
            elif e.op == NEG: nd = (NEG, visit(e.a), 0)
            elif e.op in (ADD, MUL): nd = (e.op, visit(e.a), visit(e.b))
            elif e.op == SCALED: nd = (SCALED, visit(e.a), cidx(e.b))
            else: raise ValueError(e.op)
            nodes.append(nd)
            memo[key] = len(nodes) - 1
            return memo[key]
        gates = [visit(g) for g in self.gates]
        lks = []
        for inputs, table in self.lookups:
            lks.append(([[visit(e) for e in inp] for inp in inputs], [visit(e) for e in table]))
        w = [CSF_MAGIC, self.k, self.num_fixed, self.num_advice, self.num_instance, len(self.challenge_phase), self.blinding_factors, self.degree,
             self.num_phases(), len(nodes), len(consts), len(gates), len(lks), len(self.perm_columns), len(self.advice_queries),
             len(self.fixed_queries), len(self.instance_queries), 0]
        w += self.advice_phase + self.challenge_phase
        for nd in nodes: w += list(nd)
        for c in consts:
            for limb in c: w += [limb & 0xFFFFFFFF, limb >> 32]
        w += gates
        for inputs, table in lks:
            w += [len(inputs), len(table)]
            for inp in inputs: w += inp
            w += table
        for (t, i) in self.perm_columns: w += [t, i]
        for q in (self.advice_queries, self.fixed_queries, self.instance_queries):
            for (c, r) in q: w += [c, r & 0xFFFFFFFF]
        return np.array(w, dtype=np.uint32)


def validate_csf(blob):
    """host-only structural check of a CSF blob (raises ZkbError)."""
    from .lib import load_library
    b = np.ascontiguousarray(blob, dtype=np.uint32)
    check(load_library().zkb_csf_validate(_vp(b.ctypes.data), b.size))


def expr_eval(cs, columns, mode=0, challenges=(), y=None, scale=None, out=None, out_stride=1, out_offset=0, ctx=None):
    """The gates of `cs` evaluated by the prover's own expression compiler and interpreter (zkb_expr_eval_dev), on torch's current stream.

    columns: torch int64 CUDA tensors (n, 4) in slot order fixed | advice | instance.  challenges: 4-limb Montgomery values.
    mode 0 -> one (n, 4) tensor per gate.  mode 1 -> [out]: scale * (the gates folded in y as the quotient program folds them) at
    rows i * out_stride + out_offset of `out` (allocated zeroed, n * out_stride rows, when None); other rows are left as they were.
    Returns (outputs, register count of the program)."""
    import torch
    from .arithmetic import _cur_stream
    ctx = ctx or default_context(columns[0].device.index)
    n = cs.n
    assert len(columns) == cs.num_fixed + cs.num_advice + cs.num_instance
    assert all(c.is_cuda and c.dtype == torch.int64 and c.is_contiguous() and c.shape == (n, 4) for c in columns)
    blob = cs.to_csf()
    if mode == 0:
        outs = [torch.empty((n, 4), dtype=torch.int64, device=columns[0].device) for _ in cs.gates]
    else:
        if out is None:
            out = torch.zeros((n * out_stride, 4), dtype=torch.int64, device=columns[0].device)
        assert out.is_cuda and out.dtype == torch.int64 and out.is_contiguous() and out.shape[0] > (n - 1) * out_stride + out_offset
        outs = [out]
    ch = np.ascontiguousarray(np.asarray(challenges, dtype=np.uint64).reshape(-1, 4))
    yl = np.ascontiguousarray(np.asarray(y if y is not None else [0] * 4, dtype=np.uint64).reshape(4))
    sl = np.ascontiguousarray(np.asarray(scale if scale is not None else [0] * 4, dtype=np.uint64).reshape(4))
    ctbl = (ctypes.c_void_p * len(columns))(*[c.data_ptr() for c in columns])
    otbl = (ctypes.c_void_p * max(1, len(outs)))(*[o.data_ptr() for o in outs])
    nregs = ctypes.c_uint32(0)
    check(ctx.lib.zkb_expr_eval_dev(ctx.handle, _vp(blob.ctypes.data), blob.size, int(mode), _vp(ch.ctypes.data) if ch.size else None,
                                    _vp(yl.ctypes.data) if y is not None else None, _vp(sl.ctypes.data) if scale is not None else None,
                                    ctypes.cast(ctbl, _vp), ctypes.cast(otbl, _vp), int(out_stride), int(out_offset), ctypes.byref(nregs),
                                    _cur_stream()))
    return outs, int(nregs.value)


def lookup_multiplicities(inputs, table, usable, slots=False, ctx=None):
    """The prover's mv-lookup multiplicities (zkb_lookup_multiplicities_dev) on torch's current stream.

    inputs: list of torch int64 CUDA tensors (n, 4), compressed input sets; table: the compressed table (n, 4).  Returns
    (m: (n, 4) CUDA tensor, Montgomery Fr; unsatisfied: bool), plus the table's hash-set slots as a numpy uint32 array when `slots`."""
    import torch
    from .arithmetic import _cur_stream
    ctx = ctx or default_context(table.device.index)
    n = table.shape[0]
    assert all(t.is_cuda and t.dtype == torch.int64 and t.is_contiguous() and t.shape == (n, 4) for t in list(inputs) + [table])
    m = torch.empty((n, 4), dtype=torch.int64, device=table.device)
    itbl = (ctypes.c_void_p * max(1, len(inputs)))(*[t.data_ptr() for t in inputs])
    unsat = ctypes.c_int32(0)
    nslots = ctypes.c_uint64(0)
    tsize = 1
    while tsize < 2 * usable:
        tsize <<= 1
    sl = np.zeros(tsize if slots else 0, dtype=np.uint32)
    check(ctx.lib.zkb_lookup_multiplicities_dev(ctx.handle, ctypes.cast(itbl, _vp), len(inputs), _vp(table.data_ptr()), n, int(usable),
                                                _vp(m.data_ptr()), ctypes.byref(unsat), _vp(sl.ctypes.data) if slots else None, sl.size,
                                                ctypes.byref(nslots), _cur_stream()))
    if slots:
        assert nslots.value == tsize
        return m, bool(unsat.value), sl
    return m, bool(unsat.value)


def expr_program(cs, mode=0, challenges=(), y=None, scale=None):
    """Host only: the interpreter program expr_eval would run (zkb_expr_program), as (uint64 array, one word per instruction:
    op | dst << 8 | a << 16 | b << 24 | imm << 32, register count)."""
    from .lib import load_library
    lib = load_library()
    blob = cs.to_csf()
    ch = np.ascontiguousarray(np.asarray(challenges, dtype=np.uint64).reshape(-1, 4))
    yl = np.ascontiguousarray(np.asarray(y if y is not None else [0] * 4, dtype=np.uint64).reshape(4))
    sl = np.ascontiguousarray(np.asarray(scale if scale is not None else [0] * 4, dtype=np.uint64).reshape(4))
    args = [_vp(blob.ctypes.data), blob.size, int(mode), _vp(ch.ctypes.data) if ch.size else None,
            _vp(yl.ctypes.data) if y is not None else None, _vp(sl.ctypes.data) if scale is not None else None]
    ncode, nregs = ctypes.c_uint64(0), ctypes.c_uint32(0)
    check(lib.zkb_expr_program(*args, None, 0, ctypes.byref(ncode), None))
    code = np.zeros(ncode.value, dtype=np.uint64)
    check(lib.zkb_expr_program(*args, _vp(code.ctypes.data), code.size, ctypes.byref(ncode), ctypes.byref(nregs)))
    return code, int(nregs.value)


R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
GATE, LOOKUP, COPY = 0, 1, 2
Failure = namedtuple("Failure", "kind index sub row")   # zkb_check_record: sub = poisoned (gate) / input set (lookup) / 0 (copy)


class _CheckRecord(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_uint32), ("index", ctypes.c_uint32), ("sub", ctypes.c_uint32), ("row", ctypes.c_uint32)]


class WitnessReport:
    """What check_witness found: `counts` holds the exact failure count of every gate, every (lookup, input set) and of all copies
    together, in that order (also as `gate_counts`, `lookup_counts` {(lookup, set): count} and `copy_count`); `failures` holds the
    first `cap` failures as Failure tuples, gates by (gate, row), then lookups by (lookup, set, row), then copies by index."""

    def __init__(self, cs, counts, failures, copies):
        self.counts = counts
        self.failures = failures
        self._copies = copies
        ng = len(cs.gates)
        self.gate_counts = [int(c) for c in counts[:ng]]
        keys = [(l, j) for l, (inputs, _) in enumerate(cs.lookups) for j in range(len(inputs))]
        self.lookup_counts = {key: int(c) for key, c in zip(keys, counts[ng:ng + len(keys)])}
        self.copy_count = int(counts[-1])
        self.total = int(counts.sum())
        self.ok = self.total == 0

    def __repr__(self):
        return f"WitnessReport(ok={self.ok}, total={self.total}, records={len(self.failures)})"

    def summary(self, rows_shown=8):
        """one line per failing item, e.g. 'gate 17 not satisfied at rows 5, 6 (and 1021 more)'"""
        by_item = {}
        for f in self.failures:
            by_item.setdefault((f.kind, f.index, f.sub if f.kind == LOOKUP else 0), []).append(f)
        lines = []

        def rows_text(fs, count):
            shown = [str(f.row) for f in fs[:rows_shown]]
            if not shown:
                return f"at {count} rows (not listed: the record cap was reached)"
            more = count - len(shown)
            return f"at row{'s' if len(shown) > 1 else ''} {', '.join(shown)}" + (f" (and {more} more)" if more else "")
        for g, c in enumerate(self.gate_counts):
            if c:
                fs = by_item.get((GATE, g, 0), [])
                poisoned = sum(f.sub for f in fs)
                lines.append(f"gate {g} not satisfied {rows_text(fs, c)}" + (f"; {poisoned} listed rows read blinding rows (poisoned)" if poisoned else ""))
        for (l, j), c in self.lookup_counts.items():
            if c:
                lines.append(f"lookup {l} set {j} {rows_text(by_item.get((LOOKUP, l, j), []), c)}")
        copy_fs = [f for f in self.failures if f.kind == COPY]
        for f in copy_fs[:rows_shown]:
            lc, lr, rc, rr = (int(x) for x in self._copies(f.index))
            lines.append(f"copy {f.index}: (col {lc}, row {lr}) != (col {rc}, row {rr})")
        if self.copy_count > min(len(copy_fs), rows_shown):
            lines.append(f"(and {self.copy_count - min(len(copy_fs), rows_shown)} more copy failures)")
        return lines

    def assert_satisfied(self):
        """raise ZkbError with a readable summary unless every constraint holds (MockProver::assert_satisfied)"""
        if not self.ok:
            raise ZkbError(f"witness does not satisfy the constraint system ({self.total} failures):\n  " + "\n  ".join(self.summary()))


def check_witness(cs, fixed, advice, instances, challenges=(), copies=(), theta=None, cap=1024, ctx=None):
    """MockProver::run + verify on the GPU (zkb_check_witness_dev): which gates, lookups and copy constraints of `cs` fail on this
    witness, by row.  fixed / advice: one column per entry, n rows each, numpy uint64 (n, 4) Montgomery arrays or int64 CUDA tensors;
    instances: columns of at most n cells (zero-padded here).  challenges: the 4-limb values used for synthesis.  copies: (left perm
    column, left row, right perm column, right row) entries -- columns index cs.perm_columns as for ProvingKey(copies=...) -- or an
    int32 CUDA tensor of shape (m, 4).  theta: the lookup compression challenge (4 Montgomery limbs); None draws a fresh random one.
    Runs on torch's current stream of the columns' device; returns a WitnessReport with at most `cap` failure records."""
    import os
    import torch
    from .arithmetic import _cur_stream
    n = cs.n
    cols = list(fixed) + list(advice) + list(instances)
    devs = [c.device for c in cols if isinstance(c, torch.Tensor) and c.is_cuda]
    device = devs[0] if devs else torch.device("cuda", torch.cuda.current_device())
    ctx = ctx or default_context(device.index)
    assert len(fixed) == cs.num_fixed and len(advice) == cs.num_advice and len(instances) == cs.num_instance

    def dev_col(c, pad=False):
        t = c if isinstance(c, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(c, dtype=np.uint64).view(np.int64))
        t = t.to(device=device, dtype=torch.int64).reshape(-1, 4)
        if pad and t.shape[0] < n:
            t = torch.cat([t, torch.zeros((n - t.shape[0], 4), dtype=torch.int64, device=device)])
        assert t.shape == (n, 4), f"a column has {t.shape[0]} rows, expected {n}"
        return t.contiguous()
    dcols = [dev_col(c) for c in list(fixed) + list(advice)] + [dev_col(c, pad=True) for c in instances]
    if isinstance(copies, torch.Tensor):
        cp = copies.to(device=device, dtype=torch.int32).reshape(-1, 4).contiguous()
    else:
        cp = torch.from_numpy(np.ascontiguousarray(np.asarray(copies, dtype=np.uint32).reshape(-1, 4)).view(np.int32)).to(device)
    if theta is None:
        th = int.from_bytes(os.urandom(40), "little") % R_MOD   # a uniform reduced value is the Montgomery form of a uniform element
        theta = [(th >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)]
    th = np.ascontiguousarray(np.asarray(theta, dtype=np.uint64).reshape(4))
    ch = np.ascontiguousarray(np.asarray(challenges, dtype=np.uint64).reshape(-1, 4))
    blob = cs.to_csf()
    n_items = len(cs.gates) + sum(len(inputs) for inputs, _ in cs.lookups) + 1
    counts = np.zeros(n_items, dtype=np.uint64)
    recs = (_CheckRecord * max(1, cap))()
    n_rec = ctypes.c_uint32(0)
    ctbl = (ctypes.c_void_p * max(1, len(dcols)))(*[c.data_ptr() for c in dcols])
    check(ctx.lib.zkb_check_witness_dev(ctx.handle, _vp(blob.ctypes.data), blob.size, ctypes.cast(ctbl, _vp),
                                        _vp(ch.ctypes.data) if ch.size else None, _vp(th.ctypes.data), _vp(cp.data_ptr()) if cp.shape[0] else None,
                                        cp.shape[0], _vp(counts.ctypes.data), ctypes.cast(recs, _vp), int(cap), ctypes.byref(n_rec), _cur_stream()))
    failures = [Failure(r.kind, r.index, r.sub, r.row) for r in recs[: n_rec.value]]
    return WitnessReport(cs, counts, failures, lambda i: cp[i].cpu().numpy().view(np.uint32))


def _ptr_array(arrs):
    """host numpy arrays, device buffers (objects with a `device_ptr` attribute) or None -> (keepalive list, void** as c_void_p array)."""
    keep, ptrs = [], []
    for a in arrs:
        if a is None:
            keep.append(None); ptrs.append(None)
        elif hasattr(a, "device_ptr"):
            keep.append(a); ptrs.append(int(a.device_ptr))
        else:
            c = np.ascontiguousarray(a)
            keep.append(c); ptrs.append(c.ctypes.data)
    tbl = (ctypes.c_void_p * max(1, len(keep)))(*ptrs)
    return keep, tbl


class DeviceColumn:
    """a witness column that already lives in HBM (torch tensor or raw pointer): zkb_prove_advice_phase copies it device-to-device"""
    def __init__(self, tensor):
        self.tensor = tensor
        self.device_ptr = tensor.data_ptr()
        self.shape = tuple(tensor.shape)
        self.dtype = np.dtype(np.uint64)


class ProvingKey:
    """plonk::ProvingKey<G1Affine> material resident on the GPU (keygen itself stays with the caller: SURVEY 8f row 3)."""

    def __init__(self, cs, fixed_values, sigma_values, g=None, g_lagrange=None, ctx=None, srs=None, copies=None):
        """Either (g, g_lagrange) host arrays [legacy: the pk uploads its own SRS] or srs = params.Srs handle (shared).
        copies != None: keygen path (zkb_keygen_pk) -- sigma_values is ignored and the permutation is assembled from the copy
        constraints [(left perm column, left row, right perm column, right row), ...]."""
        self.ctx = ctx or (srs.ctx if srs is not None else default_context())
        self.cs = cs
        self.srs = srs
        n = cs.n
        blob = cs.to_csf()
        kf, ftbl = _ptr_array(fixed_values)
        h = _vp()
        if copies is not None:
            assert srs is not None
            cp = np.ascontiguousarray(np.asarray(copies, dtype=np.uint32).reshape(-1, 4))
            check(self.ctx.lib.zkb_keygen_pk(self.ctx.handle, _vp(blob.ctypes.data), blob.size, ctypes.cast(ftbl, _vp), _vp(cp.ctypes.data), cp.shape[0],
                                             srs.handle, ctypes.byref(h)))
        elif srs is not None:
            ks, stbl = _ptr_array(sigma_values)
            check(self.ctx.lib.zkb_pk_create_with_srs(self.ctx.handle, _vp(blob.ctypes.data), blob.size, ctypes.cast(ftbl, _vp), ctypes.cast(stbl, _vp),
                                                      srs.handle, ctypes.byref(h)))
        else:
            assert g.shape == (n, 8) and g_lagrange.shape == (n, 8)
            ks, stbl = _ptr_array(sigma_values)
            g = np.ascontiguousarray(g); gl = np.ascontiguousarray(g_lagrange)
            check(self.ctx.lib.zkb_pk_create(self.ctx.handle, _vp(blob.ctypes.data), blob.size, ctypes.cast(ftbl, _vp), ctypes.cast(stbl, _vp),
                                             _vp(g.ctypes.data), _vp(gl.ctypes.data), ctypes.byref(h)))
        self.handle = h

    def sigma_values(self, column):
        out = np.empty((self.cs.n, 4), dtype=np.uint64)
        check(self.ctx.lib.zkb_pk_sigma_read(self.handle, int(column), _vp(out.ctypes.data)))
        return out

    def vk_bytes(self):
        """VerifyingKey::to_bytes(SerdeFormat::Processed): fixed + permutation commitments computed on the GPU."""
        n = ctypes.c_uint64(0)
        check(self.ctx.lib.zkb_pk_vk_bytes(self.handle, None, 0, ctypes.byref(n)))
        out = (ctypes.c_uint8 * n.value)()
        check(self.ctx.lib.zkb_pk_vk_bytes(self.handle, ctypes.cast(out, _vp), n.value, ctypes.byref(n)))
        return bytes(out)

    def vk_write(self, fmt=None):
        """VerifyingKey::write(fmt) without selectors (zkb_pk_vk_write) -> bytes; Processed equals vk_bytes()."""
        from .params import SerdeFormat
        fmt = SerdeFormat.RawBytesUnchecked if fmt is None else SerdeFormat(fmt)
        out = []
        io = _CallbackIo(writer=lambda b: out.append(bytes(b)))
        check(self.ctx.lib.zkb_pk_vk_write(self.handle, int(fmt), ctypes.cast(ctypes.pointer(io.vt), _vp)))
        return b"".join(out)

    def write(self, path_or_file, fmt=None):
        """ProvingKey::write(writer, fmt): the vk section, then l0, l_last, l_active_row, the fixed values / polys / cosets and the
        permutation values / polys / cosets (layout: include/zkb200.h).  path_or_file: a path, or a binary file object with write().
        The default format is snark-verifier-sdk gen_pk's RawBytesUnchecked."""
        from .params import SerdeFormat
        fmt = SerdeFormat.RawBytesUnchecked if fmt is None else SerdeFormat(fmt)
        with _binary_file(path_or_file, "wb") as f:
            f.write(self.vk_write(fmt))
            io = _CallbackIo(writer=f.write)
            io.run(self.ctx.lib.zkb_pk_write(self.handle, int(fmt), ctypes.cast(ctypes.pointer(io.vt), _vp)))

    @classmethod
    def read(cls, path_or_file, cs, srs, fmt=None, check=False):
        """ProvingKey::read(reader, fmt) for constraint system `cs` against the SRS handle `srs` (params.Srs of degree cs.k).

        The vk header (k, num_fixed) is checked against cs; the vk commitments are recomputed from the values, and with check=True they
        must equal the file's.  The file's polys and cosets are never loaded: with check=False they are only range-checked, with
        check=True every element must equal the form the key derives.  Raises ZkbError; when the body is at fault the error carries
        .report, a PkReadReport naming the section, column, first bad index, count and reason."""
        from .params import SerdeFormat
        fmt = SerdeFormat.RawBytesUnchecked if fmt is None else SerdeFormat(fmt)
        ctx = srs.ctx
        npts = cs.num_fixed + len(cs.perm_columns)
        with _binary_file(path_or_file, "rb") as f:
            head = _read_exact(f, 8 + npts * fmt.g1_len, "the vk section")
            k, nf = struct.unpack(">II", head[:8])
            if (k, nf) != (cs.k, cs.num_fixed):
                raise ZkbError(f"pk file: the vk is for k = {k} with {nf} fixed columns, the constraint system has k = {cs.k} and {cs.num_fixed}")
            blob = cs.to_csf()
            rep = _PkReadReport()
            io = _CallbackIo(reader=f)
            h = _vp()
            rc = ctx.lib.zkb_pk_read(ctx.handle, _vp(blob.ctypes.data), blob.size, int(fmt), ctypes.cast(ctypes.pointer(io.vt), _vp), srs.handle,
                                     1 if check else 0, ctypes.byref(rep), ctypes.byref(h))
            report = None if rep.count == 0 and rep.section == 0xFFFFFFFF else PkReadReport(
                int(rep.section), int(rep.column), int(rep.reason), int(rep.first_index), int(rep.count))
            try:
                io.run(rc)
            except ZkbError as e:
                e.report = report
                raise
        pk = cls.__new__(cls)
        pk.ctx, pk.cs, pk.srs, pk.handle = ctx, cs, srs, h
        if check and pk.vk_write(fmt) != head:
            pk.close()
            raise ZkbError("pk file: the vk commitments differ from the ones the key's values give")
        return pk

    def close(self):
        # finalisers of garbage run in no fixed order (at interpreter exit a failed test's traceback can hold the last key): once
        # the context is destroyed the key's C state points into freed memory, so it is dropped, not destroyed
        if self.handle and self.ctx.handle:
            self.ctx.lib.zkb_pk_destroy(self.handle)
        self.handle = None

    def __del__(self):
        try: self.close()
        except Exception: pass


PK_SECTIONS = ("l0", "l_last", "l_active_row", "fixed_values", "fixed_polys", "fixed_cosets", "permutation values", "permutation polys",
               "permutation cosets")
PK_MISMATCH = 4         # ZKB_PK_MISMATCH; ZKB_SERDE_NON_CANONICAL = 2 is the other reason
_IO_EOF = 1             # ZKB_IO_EOF
PkReadReport = namedtuple("PkReadReport", "section column reason first_index count")   # zkb_pk_read_report


class _PkReadReport(ctypes.Structure):
    _fields_ = [("section", ctypes.c_uint32), ("column", ctypes.c_uint32), ("reason", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
                ("first_index", ctypes.c_uint64), ("count", ctypes.c_uint64)]


_IO_READ = ctypes.CFUNCTYPE(ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64)
_IO_WRITE = ctypes.CFUNCTYPE(ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64)


class _IoVtable(ctypes.Structure):
    _fields_ = [("user", ctypes.c_void_p), ("read", _IO_READ), ("write", _IO_WRITE)]


@contextlib.contextmanager
def _binary_file(path_or_file, mode):
    if isinstance(path_or_file, (str, bytes, os.PathLike)):
        with open(path_or_file, mode) as f:
            yield f
    else:
        yield path_or_file


def _read_exact(f, n, what):
    data = f.read(n)
    if len(data) != n:
        raise ZkbError(f"pk file: the input ends inside {what}")
    return data


class _CallbackIo:
    """zkb_io_vtable over a binary reader (readinto) or a writer callable: read_exact / write_all.  The writer gets a memoryview of
    the library's buffer, valid only during the call (file.write and BytesIO.write copy it)."""

    def __init__(self, reader=None, writer=None):
        self.error = None

        def rd(_user, buf, n):
            try:
                view = memoryview((ctypes.c_uint8 * n).from_address(buf)).cast("B")
                got = 0
                while got < n:
                    r = reader.readinto(view[got:])
                    if not r:
                        return _IO_EOF
                    got += r
                return 0
            except Exception as e:   # never let a Python exception unwind through C
                self.error = e
                return 2

        def wr(_user, buf, n):
            try:
                writer(memoryview((ctypes.c_uint8 * n).from_address(buf)).cast("B") if n else b"")
                return 0
            except Exception as e:
                self.error = e
                return 2
        self._keep = (_IO_READ(rd), _IO_WRITE(wr))
        self.vt = _IoVtable(None, *self._keep)

    def run(self, rc):
        """check(rc), chaining the exception a callback raised"""
        try:
            check(rc)
        except ZkbError as e:
            if self.error is not None:
                raise e from self.error
            raise


TRANSCRIPTS = {"blake2b": 0, "poseidon": 1, "evm": 2}

_CB_SCALAR = ctypes.CFUNCTYPE(ctypes.c_int32, ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64))


class _TranscriptVtable(ctypes.Structure):
    _fields_ = [("user", ctypes.c_void_p), ("common_scalar", _CB_SCALAR), ("write_scalar", _CB_SCALAR), ("write_point", _CB_SCALAR),
                ("squeeze_challenge", _CB_SCALAR)]


class CallbackTranscript:
    """zkb_transcript_vtable around a caller-side transcript object (the stand-in for create_proof's generic `T: TranscriptWrite`, which
    the Rust shim forwards the same way).  `obj` implements common_scalar(limbs), write_scalar(limbs), write_point(limbs8) and
    squeeze_challenge() -> 4 Montgomery limbs; limbs are numpy uint64 arrays in halo2curves' in-memory layout."""

    def __init__(self, obj):
        self.obj = obj
        self.error = None

        def wrap(fn, n_in):
            def cb(_user, ptr):
                try:
                    fn(np.ctypeslib.as_array(ptr, shape=(n_in,)).copy())
                    return 0
                except Exception as e:   # never let a Python exception unwind through C
                    self.error = e
                    return 1
            return _CB_SCALAR(cb)

        def squeeze(_user, ptr):
            try:
                out = np.ascontiguousarray(obj.squeeze_challenge(), dtype=np.uint64)
                for i in range(4): ptr[i] = int(out[i])
                return 0
            except Exception as e:
                self.error = e
                return 1
        self._keep = (wrap(obj.common_scalar, 4), wrap(obj.write_scalar, 4), wrap(obj.write_point, 8), _CB_SCALAR(squeeze))
        self.vt = _TranscriptVtable(None, *self._keep)


def create_proof(pk, transcript_repr, instances, synthesize, z_blinds, phi_blinds, random_poly, transcript="blake2b", upload_ahead=False):
    """Mirror of plonk::create_proof for one circuit; transcript = "blake2b" (Blake2bWrite, the reference's benches) or "poseidon"
    (snark-verifier-sdk's PoseidonTranscript, what gen_snark_shplonk uses) or "evm" (snark-verifier's EvmTranscript over Keccak-256,
    what gen_evm_proof_shplonk uses; proof items uncompressed big-endian) or a CallbackTranscript around the caller's own transcript
    object (create_proof's generic `T`): then the returned bytes are empty and the proof is whatever that object wrote.

    transcript_repr: uint64[4] (Montgomery Fr).   instances: list of uint64 (len, 4) arrays (one per instance column).
    synthesize(phase, challenges) -> dict {advice column: uint64 (n,4) array, already blinded} for that phase's columns,
      where challenges is a dict {index: uint64[4]} of the challenges available so far (Circuit::synthesize stand-in).
    z_blinds (n_sets*bf, 4), phi_blinds (n_lookups*bf, 4), random_poly (n, 4): uint64 Montgomery arrays.
    Returns the proof bytes."""
    cs, lib, ctx = pk.cs, pk.ctx.lib, pk.ctx
    tr = np.ascontiguousarray(np.asarray(transcript_repr, dtype=np.uint64).reshape(4))
    ki, itbl = _ptr_array(instances)
    lens = (ctypes.c_uint32 * max(1, len(instances)))(*[a.shape[0] for a in instances])
    sess = _vp()
    if isinstance(transcript, CallbackTranscript):   # the caller's own transcript object: proof bytes are written on its side
        check(lib.zkb_prove_begin_cb(pk.handle, ctypes.cast(ctypes.pointer(transcript.vt), _vp), _vp(tr.ctypes.data), ctypes.cast(itbl, _vp),
                                     ctypes.cast(lens, _vp), ctypes.byref(sess)))
    else:
        check(lib.zkb_prove_begin_ex(pk.handle, TRANSCRIPTS[transcript], _vp(tr.ctypes.data), ctypes.cast(itbl, _vp), ctypes.cast(lens, _vp), ctypes.byref(sess)))
    try:
        nch = len(cs.challenge_phase)
        ch_buf = np.zeros((max(1, nch), 4), dtype=np.uint64)
        challenges = {}
        for phase in range(cs.num_phases()):
            cols = synthesize(phase, dict(challenges))
            arrs = [cols.get(c) if cs.advice_phase[c] == phase else None for c in range(cs.num_advice)]
            for c, a in enumerate(arrs):
                if cs.advice_phase[c] == phase:
                    assert a is not None and a.shape == (cs.n, 4) and a.dtype == np.uint64
            if upload_ahead:   # column by column ahead of the phase call (zkb_prove_upload_advice), then NULL pointers in the phase call
                idx = [c for c, a in enumerate(arrs) if a is not None]
                keep_up, utbl = _ptr_array([arrs[c] for c in idx])      # keep_up holds the (contiguous) buffers alive until the phase call returns
                for t, c in enumerate(idx):
                    check(lib.zkb_prove_upload_advice(sess, c, _vp(utbl[t])))
                arrs = [None] * len(arrs)
            ka, atbl = _ptr_array(arrs)
            check(lib.zkb_prove_advice_phase(sess, phase, ctypes.cast(atbl, _vp), _vp(ch_buf.ctypes.data)))
            for i, ph in enumerate(cs.challenge_phase):
                if ph == phase: challenges[i] = ch_buf[i].copy()
        zb = np.ascontiguousarray(z_blinds) if z_blinds is not None and len(z_blinds) else None
        pb = np.ascontiguousarray(phi_blinds) if phi_blinds is not None and len(phi_blinds) else None
        rp = np.ascontiguousarray(random_poly)
        plen = ctypes.c_uint64(0)
        # first call runs the proof and reports its length (bytes stay in the session); second call copies them out
        check(lib.zkb_prove_finish(sess, _vp(zb.ctypes.data) if zb is not None else None, _vp(pb.ctypes.data) if pb is not None else None,
                                   _vp(rp.ctypes.data), None, 0, ctypes.byref(plen)))
        out = (ctypes.c_uint8 * max(1, plen.value))()
        check(lib.zkb_prove_finish(sess, None, None, None, ctypes.cast(out, _vp), plen.value, ctypes.byref(plen)))
        return bytes(out[: plen.value])
    finally:
        lib.zkb_session_destroy(sess)
