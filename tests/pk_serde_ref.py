"""ProvingKey::write restated over the oracle keygen's dict (TEST INFRASTRUCTURE ONLY, never imported by the product).

The file layout of halo2_proofs' `ProvingKey::write(writer, format)` (plonk.rs, PSE line, which scroll-tech/halo2 v1.1 forks) as this
repository reads it.  What the reference's fixture pins: the vk prefix (aggregator/data/batch-task.json, checked by
tests/test_oracle_golden.py), the Processed Fr encoding (the proof's scalars), the Montgomery raw layout and the domain constants.
What it does NOT pin: the section order below and the u32 big-endian length prefixes (`Polynomial::write`,
`write_polynomial_slice` in helpers.rs) are restated from upstream without a Rust toolchain to check them against.  This is the one
place they are restated; a machine with cargo can diff `SECTIONS` and `pk_write` against upstream's bytes.
"""
import struct

import numpy as np

import pyref as P

PROCESSED, RAW_BYTES, RAW_BYTES_UNCHECKED = 0, 1, 2

# (name, kind): "ext" = one polynomial in extended Lagrange form (N values), "n" / "N" slices of polynomials of n / N values
SECTIONS = [
    ("l0", "ext"),
    ("l_last", "ext"),
    ("l_active_row", "ext"),
    ("fixed_values", "n"),
    ("fixed_polys", "n"),
    ("fixed_cosets", "N"),
    ("permutation values", "n"),
    ("permutation polys", "n"),
    ("permutation cosets", "N"),
]


def fr_bytes(arr, fmt, ref):
    """(m, 4) Montgomery limbs -> 32 B per element: canonical LE (Processed) or the Montgomery limbs (raw formats)."""
    a = np.ascontiguousarray(arr, dtype=np.uint64)
    if fmt == PROCESSED:
        a = ref.o.fr_to_canonical(a)
    return np.ascontiguousarray(a, dtype="<u8").tobytes()


def vk_bytes(ref, pk, fmt):
    """u32 BE k || u32 BE num_fixed || fixed commitments || permutation commitments (no selectors)."""
    pts = list(pk["fixed_commitments"]) + list(pk["sigma_commitments"])
    out = struct.pack(">II", ref.cs.k, len(pk["fixed_values"]))
    for aff in pts:
        out += ref.o.g1_compress(aff) if fmt == PROCESSED else np.ascontiguousarray(aff, dtype="<u8").tobytes()
    return out


def body_polys(ref, pk):
    """[(section index, column, (m, 4) array)] in file order."""
    F, n = ref.F, ref.cs.n
    ext = ref.coeff_to_extended
    bf = ref.bf
    l_active = np.zeros((n, 4), dtype=np.uint64)
    l_active[: n - bf - 1] = ref.w_arr(1)        # 1 - l_last - l_blind on the rows: the usable rows
    items = [(0, 0, ext(pk["l0"])), (1, 0, ext(pk["l_last"])), (2, 0, ext(ref.lagrange_to_coeff(l_active)))]
    for base, vals, polys in ((3, pk["fixed_values"], pk["fixed_polys"]), (6, pk["sigma_values"], pk["sigma_polys"])):
        items += [(base, c, v) for c, v in enumerate(vals)]
        items += [(base + 1, c, p) for c, p in enumerate(polys)]
        items += [(base + 2, c, ext(p)) for c, p in enumerate(polys)]
    return items


def pk_write(ref, pk, fmt, items=None):
    """ProvingKey::write(fmt) of the oracle keygen's pk dict (Ref.keygen) -> bytes.  items: body_polys(ref, pk), when already made."""
    items = body_polys(ref, pk) if items is None else items
    out = [vk_bytes(ref, pk, fmt)]
    for sec, (_, kind) in enumerate(SECTIONS):
        polys = [arr for s, _, arr in items if s == sec]
        if kind != "ext":                        # a slice: its count, also when it is empty
            out.append(struct.pack(">I", len(polys)))
        for arr in polys:
            out.append(struct.pack(">I", arr.shape[0]))
            out.append(fr_bytes(arr, fmt, ref))
    return b"".join(out)


def layout(k, ext_k, num_fixed, num_perm, fmt):
    """[(section, column, offset of its first element, length)] of a pk file's body, and the total file length."""
    n, N = 1 << k, 1 << ext_k
    pos = 8 + (num_fixed + num_perm) * (32 if fmt == PROCESSED else 64)
    out = []
    for sec, (name, kind) in enumerate(SECTIONS):
        cols = 1 if kind == "ext" else (num_fixed if sec < 6 else num_perm)
        if kind != "ext":
            pos += 4
        length = n if kind == "n" else N
        for c in range(cols):
            pos += 4
            out.append((sec, c, pos, length))
            pos += 32 * length
    return out, pos


def element_offset(k, ext_k, num_fixed, num_perm, fmt, section, column, index):
    """byte offset of one element of a pk file"""
    entries, _ = layout(k, ext_k, num_fixed, num_perm, fmt)
    for sec, c, pos, length in entries:
        if (sec, c) == (section, column):
            assert index < length
            return pos + 32 * index
    raise KeyError((section, column))


def montgomery_bytes(v):
    """the RawBytes encoding of the integer v < r: v * 2^256 mod r as 4 little-endian u64 limbs"""
    return (v * (1 << 256) % P.R_MOD).to_bytes(32, "little")
