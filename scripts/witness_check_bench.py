"""Time the witness check (zkb_check_witness_dev) on the k = 20 SuperCircuit stand-in and the k = 17 Keccak stand-in, with
device-resident witnesses and the full copy list, next to one create_proof of the same shape.
usage: python scripts/witness_check_bench.py [--reps R] [--out FILE]   (JSON to stdout and to FILE if given)"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

PHASES = {"gates": 4, "lookups": 5, "copies": 6, "extract": 7}   # zkb_prof_read classes of the check's phases


def card():
    """name and power limit of GPU 0 (query only)"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:   # the numbers are still worth printing; say why the card is unknown
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def run(kind, reps):
    import zkb200
    import standin_copies
    import standins
    from zkb200 import plonk as Z
    from zkb200.params import ParamsKZG
    ctx = zkb200.default_context()
    sc = standins.super_shape(20, advice=128, seed=5) if kind == "super" else standins.keccak_shape(17, seed=3)
    nch = len(sc.cs.challenge_phase)
    ch = np.array([[0x5EED5 + i, 0, 0, 0] for i in range(nch)], dtype=np.uint64)   # any reduced values stand for the challenges
    fixed, adv, inst = standin_copies.witness(sc, list(ch))
    copies = standin_copies.copies(sc)
    theta = np.array([0x7E7A, 1, 2, 3], dtype=np.uint64)
    check = lambda: Z.check_witness(sc.cs, fixed, adv, inst, challenges=ch, copies=copies, theta=theta, cap=1024)
    for _ in range(2):
        assert check().ok
    ctx.prof_enable(True)
    for cls in PHASES.values():
        ctx.prof_read(cls, reset=True)
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    phases = {name: ctx.prof_read(cls)[1] / reps / 1e3 for name, cls in PHASES.items()}
    ctx.prof_enable(False)
    # one create_proof of the same shape with the witness resident in HBM (bench.py's `value` path)
    h = sc.host
    params = ParamsKZG.unsafe_setup_with_s(sc.k, 1234)
    srs = params.load()
    pk = Z.ProvingKey(sc.cs, [h(t) for t in sc.fixed], [h(t) for t in sc.sigma], srs=srs)
    synth = lambda phase, c: {i: Z.DeviceColumn(t) for i, t in sc.synthesize_dev(phase, c).items()}
    prove = lambda: Z.create_proof(pk, h(sc.transcript_repr[None])[0], [h(t) for t in sc.instances], synth, h(sc.z_blinds), h(sc.phi_blinds),
                                   h(sc.random_poly))
    prove()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    prove()
    torch.cuda.synchronize()
    t_proof = time.perf_counter() - t0
    pk.close()
    med = sorted(times)[len(times) // 2]
    return {"shape": kind, "k": sc.k, "gates": sc.shape["gates"], "lookup_input_sets": sc.shape["lookup_input_sets"],
            "permutation_columns": sc.shape["permutation_columns"], "copies": int(copies.shape[0]), "check_seconds_median": med,
            "check_seconds_best": min(times), "phase_device_seconds": phases, "create_proof_seconds": t_proof, "check_over_proof": med / t_proof}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card(), results=[run("super", a.reps), run("keccak", a.reps)])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
