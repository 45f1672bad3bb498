"""Every MSM window size of csrc/msm.cu, exactly, up to 2^26 points, against a reference that needs no Pippenger: the bases
are B_i = [k_i] G from known discrete logs k_i (zkb_g1_fixed_base_mul_dev, a separate double-and-add kernel), so
sum_i s_i B_i = [sum_i s_i k_i mod r] G -- one vectorised field multiplication, an exact integer sum and one scalar
multiplication on the CPU.  Each MSM's `zkb_msm_last_adds` / `zkb_msm_last_levels` must equal tests/msm_model.py's
prediction, which proves which configuration ran.

One pool of 2^26 bases (4 GB) lives on the device for the module, under a context of its own whose scratch is freed with
it; every size takes a prefix.  Scalars are generated on the device and streamed to the host in 2^22-row chunks."""
import time

import numpy as np
import pytest

import msm_model as M
import pyref as P
from util import rand_field, to_dev, to_host

pytestmark = pytest.mark.gpu

POOL_LOG = 26
CH = 1 << 22


@pytest.fixture(scope="module")
def A():
    from zkb200 import arithmetic
    return arithmetic


class Pool:
    """bases[i] = [K[i]] G on the device; K (Montgomery limbs) on the host"""

    def __init__(self, ctx, A, oracle):
        import torch
        self.ctx, self.A, self.o = ctx, A, oracle
        self.G = oracle.g1_generator()
        self.free_min = torch.cuda.mem_get_info()[0]
        n = 1 << POOL_LOG
        self.K = np.empty((n, 4), dtype=np.uint64)
        self.bases = torch.empty((n, 8), dtype=torch.int64, device="cuda")
        t0 = time.perf_counter()
        for a in range(0, n, CH):
            self.K[a:a + CH] = rand_field(CH, 7000 + a // CH)
            self.bases[a:a + CH] = A.g1_fixed_base_mul_dev(self.G, to_dev(self.K[a:a + CH]), ctx=ctx)
        torch.cuda.synchronize()
        self.build_s = time.perf_counter() - t0
        self.note()

    def note(self):
        import torch
        self.free_min = min(self.free_min, torch.cuda.mem_get_info()[0])

    def msm(self, s_t):
        r = self.A.best_multiexp_dev(s_t, self.bases[: s_t.shape[0]], ctx=self.ctx)
        self.note()
        return r, self.A.msm_last_adds(self.ctx), int(self.ctx.lib.zkb_msm_last_levels(self.ctx.handle))

    def host_pass(self, s_t, K=None, cfg=None):
        """one streaming pass over a device column: the discrete-log reference [sum s_i K_i] G (affine limbs) and, with cfg,
        the model's bucket counts"""
        o, n = self.o, s_t.shape[0]
        K = self.K if K is None else K
        acc = np.zeros(8, dtype=np.uint64)
        counts = None
        for a in range(0, n, CH):
            sc = np.ascontiguousarray(to_host(s_t[a:a + CH]))
            can = o.fr_to_canonical(o.fr_mul(sc, np.ascontiguousarray(K[a:a + sc.shape[0]])))
            acc += can.view(np.uint32).reshape(-1, 8).sum(axis=0, dtype=np.uint64)   # < 2^32 * 2^26 per half-limb
            if cfg is not None:
                bc = M.bucket_counts(o.fr_to_canonical(sc), cfg)
                counts = bc if counts is None else counts + bc
        e = sum(int(v) << (32 * j) for j, v in enumerate(acc)) % P.R_MOD
        return fbm(o, self.G, e), counts


def fbm(o, G, e):
    """[e] G affine (identity = zeros) through the oracle's fixed-base multiplication"""
    return o.g1_fixed_base_mul(G, o.fr_from_canonical(M.ints_to_canon([e])))[0]


def mont(o, vals):
    return o.fr_from_canonical(M.ints_to_canon(vals))


@pytest.fixture(scope="module")
def pool(A, oracle):
    import torch
    from zkb200.lib import Context
    free0, total = torch.cuda.mem_get_info()
    ctx = Context(torch.cuda.current_device())
    p = Pool(ctx, A, oracle)
    # the pool against the oracle: first and last 64 points and 1024 random ones
    n = 1 << POOL_LOG
    idx = np.concatenate([np.arange(64), np.arange(n - 64, n), np.random.default_rng(1).integers(0, n, 1024)])
    got = to_host(p.bases[torch.from_numpy(idx).cuda()])
    assert (got == oracle.g1_fixed_base_mul(p.G, np.ascontiguousarray(p.K[idx]))).all(), "fixed-base multiplication differs from the oracle"
    yield p
    p.note()
    print(f"\nmsm windows: pool of 2^{POOL_LOG} bases built in {p.build_s:.2f} s; device memory in use (all processes) "
          f"{(total - free0) / 2**30:.2f} GiB before, peak {(total - p.free_min) / 2**30:.2f} GiB")
    del p.bases
    ctx.close()
    torch.cuda.empty_cache()


def random_col(A, n, seed):
    """random device column, generated in chunks so that a 2^26 column needs no column-sized temporaries"""
    import torch
    t = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    for a in range(0, n, CH):
        t[a:a + CH] = A.random_fr_dev(min(CH, n - a), 1000 * seed + a // CH)
    return t


def device_col(A, n, seed, rows=()):
    """random device column with rows[(index, Montgomery limbs)] written in"""
    t = random_col(A, n, seed)
    for i, v in rows:
        t[i] = to_dev(np.ascontiguousarray(v.reshape(1, 4)))[0]
    return t


def check(pool, s_t, n, dist=None):
    """MSM of s_t over the first n pool bases == the discrete-log reference, and the device's additions and reduction levels
    == the model's; dist = (distinct values, multiplicities) of a structured column saves the model a pass over it"""
    cfg = M.choose_cfg(n)
    r, adds, levels = pool.msm(s_t)
    exp, counts = pool.host_pass(s_t, cfg=cfg if dist is None else None)
    if dist is not None:
        counts = M.bucket_counts(M.ints_to_canon(dist[0]), cfg, mult=dist[1])
    assert (r.affine == exp).all(), f"MSM of {n} points differs from the discrete-log reference"
    assert r.compressed == pool.o.g1_compress(exp)
    assert (adds, levels) == M.predict([counts], n, cfg), f"n = {n}: the device did not run {cfg}"
    return r, adds, levels


# one n per window size, inside [2^(c+4), 2^(c+5)) and not a power of two; c = 3 also covers the sizes below 2^7
PLAIN = [(3, n) for n in (1, 2, 5, 33, 127)] + [(c, (1 << (c + 4)) + (1 << (c + 2)) + 2 * c + 1) for c in range(4, 21)]


class EditedBases:
    """a few pool rows overwritten for one test (restored afterwards): bases[i0] = identity (k = 0), bases[i1] = -bases[a]
    (k = r - k_a), bases[i2] = bases[b] (k = k_b); the scalars at i1 and i2 copy those at a and b, so that P and -P, and P
    and P, land in the same bucket of every window"""

    def __init__(self, pool, n, i0, i1, i2, a, b):
        self.pool, self.rows = pool, [i0, i1, i2]
        self.saved_b = pool.bases[self.rows].clone()
        self.saved_k = pool.K[self.rows].copy()
        o = pool.o
        pb = to_host(pool.bases[[a]])[0].copy()
        neg = pb.copy()
        neg[4:] = o.field_unop(1, 4, np.ascontiguousarray(pb[4:].reshape(1, 4)))[0]
        pool.bases[i0] = 0
        pool.bases[i1] = to_dev(neg.reshape(1, 8))[0]
        pool.bases[i2] = pool.bases[b].clone()
        pool.K[i0] = 0
        pool.K[i1] = o.fr_sub(np.zeros((1, 4), dtype=np.uint64), np.ascontiguousarray(pool.K[a:a + 1]))[0]
        pool.K[i2] = pool.K[b]
        self.copies = [(i1, a), (i2, b)]

    def apply_scalars(self, s_t):
        for dst, src in self.copies:
            s_t[dst] = s_t[src]

    def restore(self):
        self.pool.bases[self.rows] = self.saved_b
        self.pool.K[self.rows] = self.saved_k


@pytest.mark.parametrize("c,n", PLAIN, ids=[f"c{c}-n{n}" for c, n in PLAIN])
def test_plain_window(A, pool, oracle, c, n):
    """Random scalars with the edge scalars of this c (0, 1, r - 1, r - 2, (r - 1)/2, every digit half, every digit half + 1,
    a digit of 1 in every window, 2^c - 1, 2^(c(W-1)), 2^(c(W-1)) - 1) at index 0, at the middle and at n - 1, over bases
    that include the identity, a negated point and a duplicate.  Catches a dropped top carry, a digit equal to half sent to the
    wrong sign, an index-0 or last-index point lost by the scatter, the identity base mishandled by the mixed addition, and
    P + (-P) / P + P inside one bucket (the exceptional cases of the addition formulas)."""
    cfg = M.choose_cfg(n)
    assert cfg.c == c
    edges = mont(oracle, M.edge_scalars(c))
    E = len(edges)
    if n < 64:
        # a few points: the edge scalars three at a time at 0, n // 2, n - 1, then the edited bases on their own
        for j in range(0, E, 3):
            rows = [(i, edges[min(j + t, E - 1)]) for t, i in enumerate((0, n // 2, n - 1))]
            check(pool, device_col(A, n, 10 * n + j, rows), n)
        if n >= 5:
            ed = EditedBases(pool, n, 1, 2, 3, 0, n - 1)
            try:
                s_t = device_col(A, n, 11 * n)
                ed.apply_scalars(s_t)
                check(pool, s_t, n)
            finally:
                ed.restore()
        return
    mid = n // 2 - E // 2
    rows = [(i, edges[i]) for i in range(E)] + [(mid + i, edges[i]) for i in range(E)] + [(n - E + i, edges[i]) for i in range(E)]
    ed = EditedBases(pool, n, n // 4, n // 4 + 1, n // 4 + 2, 3 * n // 4, 3 * n // 4 + 1)
    try:
        s_t = device_col(A, n, 100 + c, rows)
        ed.apply_scalars(s_t)
        check(pool, s_t, n)
    finally:
        ed.restore()


def test_reference_matches_oracle_pippenger(A, pool, oracle):
    """the discrete-log reference equals the oracle's own best_multiexp once, at 40 000 points"""
    n = 40000
    s_t = random_col(A, n, 5)
    exp, _ = pool.host_pass(s_t)
    assert (exp == oracle.g1_to_affine(oracle.best_multiexp(to_host(s_t), to_host(pool.bases[:n])))).all()


SKEW_C = [8, 16, 19, 20]
SKEW_KINDS = ["zero", "selector", "small", "all_equal", "last_only", "digit_one"]


def skewed_col(A, oracle, kind, n, c):
    """-> (device column, (distinct values, multiplicities))"""
    import torch
    from zkb200 import arithmetic as AR
    g = torch.Generator(device="cuda")
    g.manual_seed(n + len(kind))

    def small(hi):
        ints = torch.randint(0, hi, (n,), dtype=torch.int64, device="cuda", generator=g)
        t = AR.field_unop_dev(AR.FR, AR.UOP_TO_MONT, torch.nn.functional.pad(ints[:, None], (0, 3)).contiguous())
        return t, (list(range(hi)), torch.bincount(ints, minlength=hi).cpu().tolist())

    def const(v):
        return to_dev(mont(oracle, [v])).expand(n, 4).contiguous(), ([v], [n])

    if kind == "zero":
        return torch.zeros((n, 4), dtype=torch.int64, device="cuda"), ([0], [n])
    if kind == "selector":
        return small(2)
    if kind == "small":
        return small(16)
    if kind == "all_equal":
        return const(0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF1234567890ABCDE % P.R_MOD)
    if kind == "last_only":
        t = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
        t[n - 1] = to_dev(mont(oracle, [M.R_MOD - 3]))[0]
        return t, ([0, M.R_MOD - 3], [n - 1, 1])
    return const(M.edge_scalars(c)[7])   # a digit of 1 in every window


@pytest.mark.parametrize("c", SKEW_C)
@pytest.mark.parametrize("kind", SKEW_KINDS)
def test_skewed_columns(A, pool, oracle, kind, c):
    """Witness-shaped columns at c = 8, 16, 19, 20: all zero (must be the identity: catches an empty bucket that is not the
    identity, or skipped in the chunk kernel), 0/1 selectors and integers below 16 (two or a few giant buckets in window 0,
    all others empty), one value repeated (one bucket per window, the most reduction levels: catches a missing level), a
    single nonzero scalar at n - 1 (catches the last chunk or the last bucket dropped), a digit of 1 in every window (the
    same bucket index in every window)."""
    n = dict(PLAIN)[c]
    s_t, dist = skewed_col(A, oracle, kind, n, c)
    r, adds, levels = check(pool, s_t, n, dist)
    if kind == "zero":
        assert r.compressed == bytes(32) and not r.affine.any()
    if kind in ("all_equal", "digit_one"):
        assert levels == M.level_bound(n, M.choose_cfg(n))[1]


@pytest.mark.parametrize("lg", [23, 24, 25, 26])
def test_production_sizes(A, pool, oracle, lg):
    """dense random scalars at 2^23 ... 2^26 (the compression layer's commitments are 2^26 points), exact; at 2^26 also one
    repeated value (each window's n entries in one bucket: the deepest reduction the largest MSM can need)"""
    import torch
    torch.cuda.empty_cache()
    n = 1 << lg
    check(pool, random_col(A, n, 4000 + lg), n)
    if lg == 26:
        s_t, dist = skewed_col(A, oracle, "all_equal", n, 20)
        _, _, levels = check(pool, s_t, n, dist)
        assert levels == M.level_bound(n, M.choose_cfg(n))[1]


@pytest.mark.parametrize("lg", [20, 23])
def test_batch_across_pass_split(A, pool, oracle, lg):
    """zkb_msm_g1_batch_dev with msm_max_batch(n) + 1 columns (11 at 2^20, 3 at 2^23), so the last column runs in a pass of
    its own, including an all-zero and an all-equal column: every result equals its single-column MSM and the reference.
    Catches a column lost or shifted at the split, or bucket sets of neighbouring columns that overlap."""
    n = 1 << lg
    nb = M.msm_max_batch(n) + 1
    cols = [random_col(A, n, 6000 + i) for i in range(nb)]
    cols[0] = skewed_col(A, oracle, "all_equal", n, 0)[0]
    cols[1] = skewed_col(A, oracle, "zero", n, 0)[0]
    got = A.best_multiexp_batch_dev(cols, pool.bases[:n], ctx=pool.ctx)
    pool.note()
    cfg = M.choose_cfg(n)
    last_counts = None
    for i, col in enumerate(cols):
        exp, counts = pool.host_pass(col, cfg=cfg if i == nb - 1 else None)
        assert (got[i] == exp).all(), f"column {i} of {nb}"
        if i == nb - 1:
            last_counts = counts
    adds_batch = A.msm_last_adds(pool.ctx)
    assert adds_batch == M.predict([last_counts], n, cfg)[0]   # the last pass held the last column alone
    for i, col in enumerate(cols):
        assert (pool.msm(col)[0].affine == got[i]).all()
