"""Throughput of the params file point codecs (zkb_g1_decode / zkb_g1_encode) in points/s, for every SerdeFormat, device-resident
and host-to-host, on the 2^(k+1) G1 points (g and g_lagrange) of a params file of degree k.

    python scripts/srs_serde_bench.py [--ks 20 23 26] [--reps 3]

The points are 2^16 distinct SRS points tiled to size (the codecs do the same work for every point, whatever its value).  Each
call synchronises, so a call is timed with the host clock around it, best of --reps after one warm-up call.  Every line carries
the card name and its power limit.  decode(encode(points)) is checked against the points for every format and size.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(), pl


def best_of(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="+", default=[20, 23, 26])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    from zkb200.params import ParamsKZG, SerdeFormat, g1_decode, g1_encode
    assert torch.cuda.is_available(), "the codec benchmark needs a GPU"
    name, power = card()
    base = ParamsKZG.unsafe_setup_with_s(16, 4321).g
    for k in args.ks:
        n = 2 << k
        pts_dev = base.repeat((n + base.shape[0] - 1) // base.shape[0], 1)[:n].contiguous()
        pts_host = pts_dev.cpu().numpy().view(np.uint64)
        for fmt in SerdeFormat:
            nb = n * fmt.g1_len
            enc_dev = torch.empty(nb, dtype=torch.uint8, device="cuda")
            enc_host = np.empty(nb, dtype=np.uint8)
            out_dev = torch.empty((n, 8), dtype=torch.int64, device="cuda")
            out_host = np.empty((n, 8), dtype=np.uint64)
            cases = {
                ("encode", "device"): lambda: g1_encode(fmt, pts_dev, enc_dev),
                ("encode", "host"): lambda: g1_encode(fmt, pts_host, enc_host),
                ("decode", "device"): lambda: g1_decode(fmt, enc_dev, n, out_dev),
                ("decode", "host"): lambda: g1_decode(fmt, enc_host, n, out_host),
            }
            for (op, where), fn in cases.items():
                t = best_of(fn, args.reps)
                print(json.dumps({"k": k, "points": n, "format": fmt.name, "op": op, "path": where, "seconds": round(t, 4),
                                  "points_per_s": round(n / t), "gpu": name, "power_limit": power}), flush=True)
            assert torch.equal(out_dev, pts_dev) and (out_host == pts_host).all(), f"decode(encode(points)) differs: {fmt.name} k={k}"
            del enc_dev, enc_host, out_dev, out_host
        del pts_dev, pts_host
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
