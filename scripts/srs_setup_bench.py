"""Time of ParamsKZG::setup on the device (zkb_srs_setup_dev) against the previous composition, and of [s]G2 on the host.

    python scripts/srs_setup_bench.py [--ks 20 23 26] [--reps 5] [--sweep-k 23] [--out FILE]

For each k the two device paths run alternately, --reps times each after one warm-up call of each:
  - setup: zkb_srs_setup_dev (g and g_lagrange, 2 * 2^k points, through the fixed-base comb);
  - previous: the element-wise composition around the double-and-add kernel zkb_g1_fixed_base_mul_dev that unsafe_setup_with_s used
    before (restated below).
Each call ends in a device synchronise and is timed with the host clock around it; best and median are reported, and the two paths'
outputs are compared byte for byte.  zkb_g2_setup_host is timed on the host.  With --sweep-k the comb variants (window bits c and the
table in global or shared memory, ZKB_SETUP_WINDOW_BITS / ZKB_SETUP_TABLE_SMEM) are timed the same way at that k and checked to give
the default's bytes.  Every line carries the card name and its power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = [(6, 0), (6, 1), (7, 0), (7, 1), (8, 0), (10, 0), (12, 0)]


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(), pl


def previous_composition(k, s):
    import numpy as np
    from zkb200 import arithmetic as A, poly
    from zkb200.params import bcast, fr_pow2k_dev, fr_scalar_dev, g1_generator
    n = 1 << k
    gen = g1_generator()
    s_t = fr_scalar_dev(s)
    pw = poly.fr_powers_dev(s_t.cpu().numpy().view(np.uint64)[0], n)
    g = A.g1_fixed_base_mul_dev(gen, pw)
    del pw
    omega, _ = A.root_of_unity(k)
    W = poly.fr_powers_dev(omega, n)
    inv = A.fr_batch_invert_dev(A.field_binop_dev(A.FR, A.OP_SUB, bcast(s_t, n), W))
    one = fr_scalar_dev(1)
    c1 = A.field_binop_dev(A.FR, A.OP_MUL, A.field_binop_dev(A.FR, A.OP_SUB, fr_pow2k_dev(s_t, k), one),
                           A.field_unop_dev(A.FR, A.UOP_INV, fr_scalar_dev(n)))
    L = A.field_binop_dev(A.FR, A.OP_MUL, A.field_binop_dev(A.FR, A.OP_MUL, W, inv), bcast(c1, n))
    del W, inv
    return g, A.g1_fixed_base_mul_dev(gen, L)


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def summary(ts):
    return {"best_ms": round(1e3 * min(ts), 3), "median_ms": round(1e3 * statistics.median(ts), 3), "runs": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="+", default=[20, 23, 26])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sweep-k", type=int, default=0)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    import torch
    from zkb200.params import fr_scalar_dev, g2_setup, srs_setup_dev
    assert torch.cuda.is_available(), "the setup benchmark needs a GPU"
    name, power = card()
    s = 0x5EED5EED
    s_mont = fr_scalar_dev(s).cpu().numpy().view(np.uint64)[0].copy()
    lines = []

    def emit(rec):
        rec.update(card=name, power_limit=power)
        lines.append(rec)
        print(json.dumps(rec), flush=True)

    ts = []
    for _ in range(args.reps + 1):
        t0 = time.perf_counter()
        g2_setup(s_mont)
        ts.append(time.perf_counter() - t0)
    emit({"what": "zkb_g2_setup_host", **summary(ts[1:])})

    for k in args.ks:
        new_t, old_t = [], []
        same = True
        for rep in range(args.reps + 1):
            dt_new, (g, gl) = timed(lambda: srs_setup_dev(k, s_mont))
            dt_old, (g0, gl0) = timed(lambda: previous_composition(k, s))
            same = same and bool(torch.equal(g, g0)) and bool(torch.equal(gl, gl0))
            del g, gl, g0, gl0
            if rep:
                new_t.append(dt_new)
                old_t.append(dt_old)
        emit({"what": "setup_vs_previous", "k": k, "points": 2 << k, "setup": summary(new_t), "previous": summary(old_t),
              "speedup_median": round(statistics.median(old_t) / statistics.median(new_t), 2), "same_bytes": same})

    if args.sweep_k:
        k = args.sweep_k
        ref_g, ref_gl = srs_setup_dev(k, s_mont)
        times = {v: [] for v in VARIANTS}
        same = {v: True for v in VARIANTS}
        try:
            for rep in range(args.reps + 1):
                for c, sm in VARIANTS:
                    os.environ["ZKB_SETUP_WINDOW_BITS"], os.environ["ZKB_SETUP_TABLE_SMEM"] = str(c), str(sm)
                    dt, (g, gl) = timed(lambda: srs_setup_dev(k, s_mont))
                    same[(c, sm)] = same[(c, sm)] and bool(torch.equal(g, ref_g)) and bool(torch.equal(gl, ref_gl))
                    del g, gl
                    if rep:
                        times[(c, sm)].append(dt)
        finally:
            os.environ.pop("ZKB_SETUP_WINDOW_BITS", None)
            os.environ.pop("ZKB_SETUP_TABLE_SMEM", None)
        for (c, sm), ts in times.items():
            emit({"what": "comb_variant", "k": k, "c": c, "table": "shared" if sm else "global", **summary(ts), "same_bytes": same[(c, sm)]})

    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
