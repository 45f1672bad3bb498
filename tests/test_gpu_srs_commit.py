"""The SRS handle's commitment paths (csrc/srs.cu), exactly, at k = 10 ... 23, against the trapdoor: with
g[i] = [s^i] G and g_lagrange[i] = [L_i(s)] G, commit(v) = [v(s)] G and commit_lagrange(v) = [sum_i v_i L_i(s)] G.  The
vectors (s^i) and (L_i(s)) come from the oracle -- L(s) = (1/n) DFT_{w^-1}(s^i), one FFT per size -- so each reference is a
field multiplication, an exact sum and one scalar multiplication, independent of any Pippenger.

Every k runs under a context of its own, closed at the end, so the shifted copies and the MSM scratch of one size are freed
before the next.  Which path ran (window-shifted copies or the plain MSM) is asserted through tests/msm_model.py: the
device's `zkb_msm_last_adds` / `zkb_msm_last_levels` must equal the model's for that path."""
import numpy as np
import pytest

import msm_model as M
import pyref as P
from util import to_dev, to_host

pytestmark = pytest.mark.gpu

CH = 1 << 22
KS = [10, 11, 12, 14, 15, 17, 18, 20, 21, 22, 23]


def mont(o, vals):
    return o.fr_from_canonical(M.ints_to_canon(vals))


def trapdoor_vectors(o, s, k):
    """(s^i), (L_i(s)) for i < 2^k as Montgomery limbs"""
    n = 1 << k
    pw = o.fr_powers(mont(o, [s])[0], n)
    w_inv = o.fr_inv(o.fr_omega(k).reshape(1, 4))[0]
    lag = o.fr_mul(o.best_fft(pw, w_inv, k), np.repeat(o.fr_inv(mont(o, [n])), n, axis=0))
    return pw, lag


def trapdoor_commit(o, col_t, vec):
    """[sum_i col_i vec_i] G: col on the device, streamed in chunks; the sum is exact over 32-bit halves of canonical limbs"""
    acc = np.zeros(8, dtype=np.uint64)
    for a in range(0, col_t.shape[0], CH):
        sc = np.ascontiguousarray(to_host(col_t[a:a + CH]))
        can = o.fr_to_canonical(o.fr_mul(sc, np.ascontiguousarray(vec[a:a + sc.shape[0]])))
        acc += can.view(np.uint32).reshape(-1, 8).sum(axis=0, dtype=np.uint64)
    e = sum(int(v) << (32 * j) for j, v in enumerate(acc)) % P.R_MOD
    return o.g1_fixed_base_mul(o.g1_generator(), mont(o, [e]))[0]


def model_counts(o, col_t, cfg):
    counts = np.zeros(cfg.half if cfg.shifted else cfg.windows * cfg.half, dtype=np.int64)
    for a in range(0, col_t.shape[0], CH):
        counts += M.bucket_counts(o.fr_to_canonical(np.ascontiguousarray(to_host(col_t[a:a + CH]))), cfg)
    return counts


def columns(A, oracle, n, k):
    """a random column and the witness shapes: 0/1 selectors, one repeated value, a single nonzero scalar at n - 1, all zero"""
    import torch
    sel = A.field_unop_dev(A.FR, A.UOP_TO_MONT, torch.nn.functional.pad(
        (torch.arange(n, device="cuda", dtype=torch.int64) % 3 == 1).to(torch.int64)[:, None], (0, 3)).contiguous())
    last = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
    last[n - 1] = to_dev(mont(oracle, [P.R_MOD - 1]))[0]
    return {"random": A.random_fr_dev(n, 300 + k), "selector": sel,
            "all_equal": to_dev(mont(oracle, [0xC0FFEE ** 9 % P.R_MOD])).expand(n, 4).contiguous(), "last_only": last,
            "zero": torch.zeros((n, 4), dtype=torch.int64, device="cuda")}


@pytest.mark.parametrize("k", KS)
def test_srs_commit_paths(oracle, monkeypatch, k):
    """At each k: the setup's bases against the trapdoor (sampled); commit and commit_lagrange of a random column and of
    witness-shaped ones; an (n - 5)-scalar commit (the plain MSM at c = k - 5 against g's prefix); zkb_srs_commit_batch_dev
    with msm_max_batch(n) + 1 columns; the same params loaded again with ZKB_MSM_SHIFT_GB=0 (the plain path at full length);
    downsize(k - 1) and a commit against it.  Catches a wrong shifted-copy index (copy w of point i read for another w or i),
    a shifted copy built with the wrong number of doublings, a basis mix-up between g and g_lagrange, a column lost at a
    batch pass split, a fallback to the plain path that computes something else, and a wrong group iFFT in downsize."""
    import torch
    from zkb200 import arithmetic as A
    from zkb200.lib import Context
    from zkb200.params import ParamsKZG, Srs
    n = 1 << k
    s = 0x5EED0000 + k
    free0, total = torch.cuda.mem_get_info()
    mem_bytes = torch.cuda.get_device_properties(torch.cuda.current_device()).total_memory   # what the shift budget is read against
    free_min = [free0]
    note = lambda: free_min.__setitem__(0, min(free_min[0], torch.cuda.mem_get_info()[0]))
    ctx = Context(torch.cuda.current_device())
    handles = []
    last = lambda: (A.msm_last_adds(ctx), int(ctx.lib.zkb_msm_last_levels(ctx.handle)))
    try:
        params = ParamsKZG.unsafe_setup_with_s(k, s)
        pw, lag = trapdoor_vectors(oracle, s, k)
        G = oracle.g1_generator()
        idx = np.unique(np.concatenate([np.arange(32), np.arange(n - 32, n), np.random.default_rng(k).integers(0, n, 256)]))
        it = torch.from_numpy(idx).cuda()
        assert (to_host(params.g[it]) == oracle.g1_fixed_base_mul(G, np.ascontiguousarray(pw[idx]))).all()
        assert (to_host(params.g_lagrange[it]) == oracle.g1_fixed_base_mul(G, np.ascontiguousarray(lag[idx]))).all()
        if k <= 14:
            # the FFT route to L_i(s) against the closed form w^i (s^n - 1) / (n (s - w^i))
            wi = oracle.fr_powers(oracle.fr_omega(k), n)
            sn1 = mont(oracle, [(pow(s, n, P.R_MOD) - 1) % P.R_MOD])
            den = oracle.fr_mul(oracle.fr_sub(np.repeat(mont(oracle, [s]), n, axis=0), wi), np.repeat(mont(oracle, [n]), n, axis=0))
            assert (oracle.fr_mul(oracle.fr_mul(wi, np.repeat(sn1, n, axis=0)), oracle.fr_inv(den)) == lag).all()

        monkeypatch.delenv("ZKB_MSM_SHIFT_GB", raising=False)
        srs = Srs.from_params(params, ctx=ctx)
        handles.append(srs)
        assert srs.k == k
        shifted = M.srs_uses_shift(n, mem_bytes)
        assert shifted == (k <= 22), "an 80 GB device holds the shifted copies of every k <= 22 under the default budget"
        cfg = M.msm_cfg(n, shifted)
        cols = columns(A, oracle, n, k)
        exp, pred = {}, {}
        for name, col in cols.items():
            exp[name] = (trapdoor_commit(oracle, col, pw), trapdoor_commit(oracle, col, lag))
            pred[name] = model_counts(oracle, col, cfg)
            for basis, commit in enumerate((srs.commit, srs.commit_lagrange)):
                r = commit(col)
                note()
                assert (r.affine == exp[name][basis]).all(), f"k = {k}, {name} column, basis {basis}"
                assert last() == M.predict([pred[name]], n, cfg), f"k = {k}: the commit did not run {cfg}"
        assert not exp["zero"][0].any() and not exp["zero"][1].any()

        short = cols["random"][: n - 5]
        plain_short = M.choose_cfg(n - 5)
        assert plain_short.c == k - 5
        r = srs.commit(short)
        assert (r.affine == trapdoor_commit(oracle, short, pw)).all()
        assert last() == M.predict([model_counts(oracle, short, plain_short)], n - 5, plain_short)

        nb = M.msm_max_batch(n) + 1
        batch = [A.random_fr_dev(n, 1000 * k + i) for i in range(nb - 2)] + [cols["all_equal"], cols["zero"]]
        for basis in (0, 1):
            got = srs.commit_batch(basis, batch)
            note()
            assert got.shape == (nb, 8)
            for i, col in enumerate(batch):
                assert (got[i] == trapdoor_commit(oracle, col, (pw, lag)[basis])).all(), f"k = {k}, basis {basis}: column {i} of {nb}"

        # the plain path at full length: no shifted copies under a zero budget (read when the handle is created)
        monkeypatch.setenv("ZKB_MSM_SHIFT_GB", "0")
        srs0 = Srs.from_params(params, ctx=ctx)
        handles.append(srs0)
        plain = M.choose_cfg(n)
        for name in ("random", "all_equal"):
            for basis, commit in enumerate((srs0.commit, srs0.commit_lagrange)):
                assert (commit(cols[name]).affine == exp[name][basis]).all(), f"k = {k}, {name} column, basis {basis}, no shifted copies"
                assert last() == M.predict([model_counts(oracle, cols[name], plain)], n, plain)
        got0 = srs0.commit_batch(1, batch)
        assert (got0 == got).all()
        note()
        srs0.close()
        monkeypatch.delenv("ZKB_MSM_SHIFT_GB")

        small = srs.downsize(k - 1)
        handles.append(small)
        assert small.k == k - 1
        h = n // 2
        pw_h, lag_h = trapdoor_vectors(oracle, s, k - 1)
        assert (pw_h == pw[:h]).all()
        v = A.random_fr_dev(h, 77 + k)
        cfg_h = M.msm_cfg(h, M.srs_uses_shift(h, mem_bytes))
        for basis, (commit, vec) in enumerate(((small.commit, pw_h), (small.commit_lagrange, lag_h))):
            assert (commit(v).affine == trapdoor_commit(oracle, v, vec)).all(), f"downsize({k - 1}), basis {basis}"
            assert last() == M.predict([model_counts(oracle, v, cfg_h)], h, cfg_h)
        note()
    finally:
        for hd in handles:
            hd.close()
        ctx.close()
        params = None
        torch.cuda.empty_cache()
    print(f"\nsrs k = {k}: shifted copies {shifted}; device memory in use (all processes) {(total - free0) / 2**30:.2f} GiB before, "
          f"peak {(total - free_min[0]) / 2**30:.2f} GiB")
