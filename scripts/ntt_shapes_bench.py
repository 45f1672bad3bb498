"""Time of ntt_tile_kernel on the transform shapes one k = 20 proof is made of, in ms per transform and butterflies/s.

    python scripts/ntt_shapes_bench.py [--cols 16] [--reps 10]

Shapes (all device-resident, through the batched entry point, one launch per pass for the whole batch):
  * coset_2^20   --cols forward 2^20 transforms with the coset input scaling fused into the first pass (coeff_to_extended);
                 the proof scales by a per-element power table instead, which the C ABI does not expose; the fused
                 multiply sits in the same first round
  * intt_2^20    --cols inverse 2^20 transforms scaled by 1/n (lagrange_to_coeff)
  * intt_2^23    one inverse 2^23 transform scaled by 1/n (extended_to_coeff of the quotient)
Each shape is warmed up, then timed with CUDA events over --reps launches of the batch.  Every line carries the card name and
its power limit.  A butterfly is one of the (n / 2) log2 n of a radix-2 transform of size n.
"""
import argparse
import json
import os
import subprocess
import sys

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


def inv_n(A, log_n):
    import numpy as np
    import torch
    n_can = torch.tensor([[1 << log_n, 0, 0, 0]], dtype=torch.int64, device="cuda")
    return A.field_unop_dev(A.FR, A.UOP_INV, A.field_unop_dev(A.FR, A.UOP_TO_MONT, n_can)).cpu().numpy().view(np.uint64)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cols", type=int, default=16)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    from zkb200 import arithmetic as A
    from zkb200.poly import ntt_batch_dev
    assert torch.cuda.is_available(), "the NTT benchmark needs a GPU"
    name, power = card()
    shapes = [("coset_2^20", 20, args.cols, False), ("intt_2^20", 20, args.cols, True), ("intt_2^23", 23, 1, True)]
    for label, log_n, cols, inverse in shapes:
        w, wi = A.root_of_unity(log_n)
        data = [A.random_fr_dev(1 << log_n, 100 + i) for i in range(cols)]
        if inverse:
            ninv = inv_n(A, log_n)
            step = lambda: ntt_batch_dev(data, wi, log_n, scale=ninv)
        else:
            step = lambda: ntt_batch_dev(data, w, log_n, coset_zeta=1)
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / (args.reps * cols)
        bfly = (1 << (log_n - 1)) * log_n
        print(json.dumps({"shape": label, "log_n": log_n, "batch": cols, "ms_per_transform": round(ms, 4),
                          "butterflies_per_s": round(bfly / (ms * 1e-3)), "gpu": name, "power_limit": power}), flush=True)
        del data
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
