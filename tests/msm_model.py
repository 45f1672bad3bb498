"""Model of the configuration choices and the work accounting of csrc/msm.cu, in vectorised numpy: the window size
(`msm_cfg`, whose plain branch is `choose_cfg`), the shifted-SRS window size and copy count, the per-pass batch limit, the
signed-digit recoding of `msm_digits_kernel` (32-bit limbs, carry chain from window 0), the bucket index of a digit, the
scratch bounds and argument checks of `msm_plan`, and what `zkb_msm_last_adds` / `zkb_msm_last_levels` report after an
MSM.  Names follow the kernel.  tests/test_msm_model.py checks it on the CPU; the GPU tests compare the library's counters
with it, which proves which configuration an MSM ran.  It is a check of the host logic and the accounting -- not a product
path."""
import numpy as np

R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
CHUNK = 32      # entries per level-0 chunk (msm_acc_chunk_kernel)
ACC_CH = 64     # partials per task of the levels >= 1 (msm_acc_levelN_kernel)
G1_XYZZ_BYTES = 128


def log2_floor(n):
    return int(n).bit_length() - 1


class Cfg:
    """MsmCfg: c window bits, `windows` digit windows, `half` buckets per bucket set; shifted: one bucket set per column."""

    def __init__(self, c, shifted=False):
        self.c = c
        self.windows = (255 + c - 1) // c
        self.half = 1 << (c - 1)
        self.shifted = shifted

    def __repr__(self):
        return f"Cfg(c={self.c}, W={self.windows}, shifted={self.shifted})"


def choose_cfg(n):
    return Cfg(min(max(log2_floor(n) - 4, 3), 20))


def msm_shift_window_bits(n):
    lg = log2_floor(n)
    return 0 if lg < 10 or lg > 22 else min(lg, 20)


def msm_shift_copies(n):
    c = msm_shift_window_bits(n)
    return (255 + c - 1) // c if c else 0


def msm_max_batch(n):
    if n == 0:
        return 64
    b = (1 << 28) // (n * choose_cfg(n).windows)
    cs = msm_shift_window_bits(n)
    if cs:
        b = min(b, (1 << 31) // ((1 << (cs - 1)) * 3 * G1_XYZZ_BYTES))
    return max(1, min(64, b))


def msm_cfg(n, shifted):
    """the configuration a pass runs for n points (shifted: against msm_shift_copies(n) copies of the bases)"""
    if not shifted:
        return choose_cfg(n)
    c = msm_shift_window_bits(n)
    assert c, f"no shifted copies at n = {n}"
    return Cfg(c, shifted=True)


def srs_uses_shift(n, mem_bytes, shift_gb=None):
    """srs_build_shifted: copies exist at this size and both bases' copies fit the budget (ZKB_MSM_SHIFT_GB, default 1/8 of
    the device memory)"""
    copies = msm_shift_copies(n)
    budget = shift_gb * 1e9 if shift_gb is not None else 0.125 * mem_bytes
    return bool(copies) and 2.0 * copies * n * 64 <= budget


# ---- signed-digit recoding ---------------------------------------------------------------------------------------------
def raw_window(s32, bit, c):
    """c bits of the canonical scalars from `bit` on; s32: (m, 8) uint32 limbs"""
    limb, off = bit >> 5, bit & 31
    v = s32[:, limb].astype(np.uint64)
    if limb + 1 < 8:
        v |= s32[:, limb + 1].astype(np.uint64) << np.uint64(32)
    return ((v >> np.uint64(off)) & np.uint64((1 << c) - 1)).astype(np.int64)


def window_digits(canon, cfg):
    """yields (w, |digit|, negative) per window for canonical scalars (m, 4) uint64, then ('carry', carry out of the top
    window, None): what msm_digits_kernel computes (it drops that last carry)."""
    s32 = np.ascontiguousarray(canon).view(np.uint32).reshape(-1, 8)
    carry = np.zeros(s32.shape[0], dtype=np.int64)
    for w in range(cfg.windows):
        bit = w * cfg.c
        d = (raw_window(s32, bit, cfg.c) if bit < 256 else 0) + carry
        neg = d > cfg.half
        d = np.where(neg, (1 << cfg.c) - d, d)
        carry = neg.astype(np.int64)
        yield w, d, neg
    yield "carry", carry, None


def recode(canon, cfg):
    """-> (signed digits (m, W) int64, carry out of the top window (m,))"""
    out = np.zeros((canon.shape[0], cfg.windows), dtype=np.int64)
    for w, d, neg in window_digits(canon, cfg):
        if w == "carry":
            return out, d
        out[:, w] = np.where(neg, -d, d)


def bucket_index(w, d, cfg, col=0):
    """bucket of a nonzero |digit| d in window w of column `col` of a batch"""
    col_base = col * (cfg.half if cfg.shifted else cfg.windows * cfg.half)
    return col_base + (0 if cfg.shifted else w * cfg.half) + (d - 1)


def sorted_entry(i, w, neg, cfg, n):
    """the u32 a point contributes to the sorted pair list: its base index (in the w-th copy when shifted), sign in bit 31"""
    return (i + (w * n if cfg.shifted else 0)) | (int(neg) << 31)


def bucket_counts(canon, cfg, mult=None):
    """entries per bucket of ONE column's bucket set(s); mult: multiplicity of each row (structured columns given by their
    distinct values).  Chunks of a column may be counted separately and added."""
    nb = cfg.half if cfg.shifted else cfg.windows * cfg.half
    counts = np.zeros(nb, dtype=np.int64)
    for w, d, _ in window_digits(canon, cfg):
        if w == "carry":
            assert not d.any(), "a carry left the top window"
            break
        nz = d != 0
        base = bucket_index(w, 1, cfg)
        wt = None if mult is None else np.asarray(mult, dtype=np.float64)[nz]
        counts[base:base + cfg.half] += np.bincount(d[nz] - 1, weights=wt, minlength=cfg.half).astype(np.int64)
    return counts


# ---- bucket accumulation accounting ------------------------------------------------------------------------------------
def level0_partials(counts):
    """chunk_count_kernel: partials each bucket receives from the 32-entry chunks of the sorted list (0 for an empty bucket)"""
    off = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)])
    lo, hi = off[:-1], off[1:]
    return np.where(hi > lo, (hi - 1) // CHUNK - lo // CHUNK + 1, 0)


def level_bound(n, cfg):
    """msm_plan's bound: partials of the fullest possible bucket (n entries, n * W when shifted), and the
    number of reduction levels it launches for it"""
    bound = (n * (cfg.windows if cfg.shifted else 1) + CHUNK - 1) // CHUNK + 1
    b, launched = bound, 0
    while b > 1:
        b = (b + ACC_CH - 1) // ACC_CH
        launched += 1
    return bound, launched


def reduce_levels(lens, launched):
    """levels >= 1 as the gated kernels run them -> (extra additions, levels executed, per-level totals, longest list left)"""
    lens = np.asarray(lens, dtype=np.int64)
    maxlen = int(lens.max()) if lens.size else 0
    extra, run, totals = 0, 0, []
    for _ in range(launched):
        if maxlen <= 1:
            break
        totals.append(int(lens.sum()))
        extra += totals[-1]
        lens = (lens + ACC_CH - 1) // ACC_CH
        maxlen = (maxlen + ACC_CH - 1) // ACC_CH
        run += 1
    return extra, run, totals, maxlen


def predict(col_counts, n, cfg):
    """(zkb_msm_last_adds, zkb_msm_last_levels) of one pass over the columns whose bucket counts are given"""
    counts = np.concatenate(col_counts)
    extra, run, _, maxlen = reduce_levels(level0_partials(counts), level_bound(n, cfg)[1])
    assert maxlen <= 1, "the launched levels do not reduce every bucket to one partial"
    return int(counts.sum()) + extra + 2 * counts.size, run


# ---- scratch bounds and argument limits of msm_plan ------------------------------------------------------------------
def scratch(n, batch, shifted):
    cfg = msm_cfg(n, shifted)
    rwin1 = 1 if shifted else cfg.windows
    nbuckets = batch * rwin1 * cfg.half
    pairs = n * cfg.windows * batch
    part0_n = (pairs + CHUNK - 1) // CHUNK + nbuckets + 1
    part1_n = part0_n // ACC_CH + nbuckets + 1
    bound, launched = level_bound(n, cfg)
    return dict(cfg=cfg, nbuckets=nbuckets, pairs=pairs, part0_n=part0_n, part1_n=part1_n, bound=bound, levels=launched)


def arg_failures(n, batch, shifted):
    """the ZKB_ARG checks of msm_plan that would refuse this call (empty: it runs)"""
    sc = scratch(n, batch, shifted)
    cfg, bad = sc["cfg"], []
    if not n < (1 << 31):
        bad.append("n < 2^31")
    if shifted and not cfg.windows * n < (1 << 31):
        bad.append("W * n < 2^31")
    if not sc["pairs"] < (1 << 32):
        bad.append("pairs < 2^32")
    if not sc["nbuckets"] < (1 << 31):
        bad.append("buckets < 2^31")
    if not sc["part0_n"] < (1 << 32):
        bad.append("part0_n < 2^32")
    return bad


# ---- scalars that sit on the recoding's edges --------------------------------------------------------------------------
def edge_scalars(c):
    """canonical ints for window size c, each < r: the field's ends, every digit equal to half / half + 1 (the largest
    positive digit, the smallest negative one), a digit of 1 in every window, one full window, the top window alone, and
    every window below the top full (a carry that runs through all windows)"""
    cfg = Cfg(c)
    W, half = cfg.windows, cfg.half
    every = lambda d: sum(d << (c * w) for w in range(W))
    below_r = lambda v: v if v < R_MOD else v % (1 << 253)
    return [0, 1, R_MOD - 1, R_MOD - 2, (R_MOD - 1) // 2,
            below_r(every(half)), below_r(every(half + 1)), below_r(every(1)),
            (1 << c) - 1, 1 << (c * (W - 1)), (1 << (c * (W - 1))) - 1]


def ints_to_canon(vals):
    return np.array([[(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] for v in vals], dtype=np.uint64).reshape(-1, 4)
