"""numpy model of the mv-lookup table hash set (csrc/lookup.cuh) and the multiplicities built on it (zkb_lookup_multiplicities_dev).

Values are Fr in the stored (Montgomery) form, numpy uint64 (n, 4).  key_hash folds the eight little-endian 32-bit words of a stored value;
a key's home slot is key_hash & mask over a slot array of the smallest power of two >= 2 usable entries.  colliding_values builds distinct
values that share one home slot by inverting the hash's last round, so long probe chains can be built on purpose."""
import numpy as np

FR_TOP = 0x30644E72E131A029          # top limb of r: a value whose top limb is below it is < r
_H0, _C = 0x9E3779B9, 0x85EBCA6B
_C_INV = pow(_C, -1, 1 << 32)
M32 = np.uint64(0xFFFFFFFF)


def _words(v):
    """(n, 4) uint64 -> (n, 8) uint64 holding the little-endian 32-bit words"""
    v = np.ascontiguousarray(v, dtype=np.uint64)
    return np.ascontiguousarray(v).view(np.uint32).reshape(-1, 8).astype(np.uint64)


def _round(h, w):
    h = (h ^ w) & M32
    h = (h * np.uint64(_C)) & M32
    return h ^ (h >> np.uint64(13))


def key_hash(v):
    """lookup.cuh key_hash of every row of v -> uint64 array of 32-bit hashes"""
    w = _words(v)
    h = np.full(w.shape[0], _H0, dtype=np.uint64)
    for i in range(8):
        h = _round(h, w[:, i])
    return h


def slot_count(usable):
    t = 1
    while t < 2 * usable:
        t <<= 1
    return t


def home_slot(v, usable):
    return key_hash(v) & np.uint64(slot_count(usable) - 1)


def _unround(h):
    """the value before the last round's multiply-xorshift, given its output h (both bijections of u32)"""
    x = h ^ (h >> np.uint64(13)) ^ (h >> np.uint64(26))
    return (x * np.uint64(_C_INV)) & M32


def colliding_values(count, home, usable, seed):
    """`count` distinct Fr values (stored form, all < r) whose home slot is `home` for a table of `usable` rows.  Words 0..6 are
    random; word 7 is solved so that the hash lands on `home`, with random high hash bits until the top limb is below r's."""
    rng = np.random.default_rng(seed)
    mask = slot_count(usable) - 1
    out = []
    got = 0
    while got < count:
        m = 4 * (count - got) + 64
        v = rng.integers(0, 1 << 64, size=(m, 4), dtype=np.uint64)
        w = _words(v)
        h = np.full(m, _H0, dtype=np.uint64)
        for i in range(7):
            h = _round(h, w[:, i])
        target = (rng.integers(0, 1 << 32, size=m, dtype=np.uint64) & ~np.uint64(mask)) | np.uint64(home)
        w7 = _unround(target) ^ h
        v[:, 3] = (v[:, 3] & M32) | (w7 << np.uint64(32))
        ok = v[:, 3] < np.uint64(FR_TOP)
        out.append(v[ok])
        got += int(ok.sum())
    v = np.unique(np.concatenate(out), axis=0)[:count]
    assert v.shape[0] == count and (home_slot(v, usable) == home).all()
    return np.ascontiguousarray(v)


def random_values(n, seed):
    rng = np.random.default_rng(seed)
    v = rng.integers(0, 1 << 64, size=(n, 4), dtype=np.uint64)
    v[:, 3] = rng.integers(0, FR_TOP, size=n, dtype=np.uint64)
    return v


def _keys(v):
    return np.ascontiguousarray(v, dtype=np.uint64).view(np.dtype((np.void, 32))).ravel()


def multiplicities(inputs, table, usable):
    """Reference m (python-int counts, numpy int64 (n,)) and the unsatisfied flag: the table rows < usable with the LAST row of each
    value winning (BTreeMap collect()), input rows < usable counted on their value's winning row; rows that are not in the table set
    the flag and are not counted."""
    n = table.shape[0]
    tk = _keys(table[:usable])
    uniq, first_rev = np.unique(tk[::-1], return_index=True)
    last_row = usable - 1 - first_rev
    m = np.zeros(n, dtype=np.int64)
    unsat = False
    for f in inputs:
        fk = _keys(f[:usable])
        pos = np.minimum(np.searchsorted(uniq, fk), len(uniq) - 1)
        found = uniq[pos] == fk
        unsat |= not found.all()
        m += np.bincount(last_row[pos[found]], minlength=n)
    return m, unsat


def multiplicities_dict(inputs, table, usable):
    """The same as a plain dict over the rows, as oracle/halo2_ref.py writes it (small sizes)"""
    index = {}
    for i in range(usable):
        index[table[i].tobytes()] = i
    m = [0] * table.shape[0]
    unsat = False
    for f in inputs:
        for r in f[:usable]:
            i = index.get(r.tobytes())
            if i is None:
                unsat = True
            else:
                m[i] += 1
    return np.array(m, dtype=np.int64), unsat


def check_slots(slots, table, usable):
    """Assert every structural invariant of the filled hash set."""
    tsize = slot_count(usable)
    mask = tsize - 1
    assert slots.shape == (tsize,)
    occ = np.nonzero(slots)[0]
    rows = slots[occ].astype(np.int64) - 1
    assert (rows >= 0).all() and (rows < usable).all(), "a slot holds a row outside the usable table rows"
    # each distinct key occupies exactly one slot, holding its last row
    tk = _keys(table[:usable])
    uniq, first_rev = np.unique(tk[::-1], return_index=True)
    last_row = usable - 1 - first_rev
    sk = tk[rows]
    assert len(np.unique(sk)) == len(sk), "a key occupies more than one slot"
    assert len(occ) == len(uniq), "occupied slots != distinct keys"
    pos = np.searchsorted(uniq, sk)
    assert (uniq[pos] == sk).all() and (last_row[pos] == rows).all(), "a slot does not hold its key's last row"
    # every occupied slot is reached from its key's home slot without crossing an empty slot
    home = home_slot(table[rows], usable).astype(np.int64)
    dist = (occ - home) & mask
    empty = slots == 0
    # distance from each slot back to the nearest empty slot (cyclic), so "no empty slot in [home, s]" is dist < back[s]
    e = np.nonzero(empty)[0]
    assert len(e), "a full slot array"
    idx = np.arange(tsize)
    prev_e = e[np.searchsorted(e, idx, side="right") - 1]   # the last empty slot at or before idx (wraps via index -1)
    back = (idx - prev_e) & mask
    assert (dist < back[occ]).all(), "an empty slot lies between a key's home slot and its slot"


def probe_run(slots, start):
    """number of occupied slots from `start` up to the first empty one (wrapping at the mask)"""
    mask = slots.shape[0] - 1
    s, length = start, 0
    while slots[s]:
        length += 1
        s = (s + 1) & mask
    return length
