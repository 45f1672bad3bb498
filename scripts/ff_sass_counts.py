"""Integer-multiply instructions per field and group primitive, counted in the sm_90a SASS.

Each primitive of csrc/ff.cuh and csrc/g1.cuh is compiled into a probe kernel of its own (load the operands, one call, store
the result) and the IMAD* instructions of that kernel are counted in `cuobjdump -sass`.  A Montgomery multiply, square and the
sum of two products with one reduction (fp_mul_add_mul) are the field's units of cost on the integer-multiply pipe; the group
operations show what the MSM kernels pay per bucket addition.  Needs nvcc and cuobjdump, no GPU.

    python scripts/ff_sass_counts.py [--json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zkevm-circuits_b200", "csrc")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")

PROBES = {
    "fp_mul": "Fq a = fp_load(in), b = fp_load(in + 1); fp_store(out, fp_mul(a, b));",
    "fp_sqr": "Fq a = fp_load(in); fp_store(out, fp_sqr(a));",
    "fp_mul_add_mul": "Fq a = fp_load(in), b = fp_load(in + 1), c = fp_load(in + 2), d = fp_load(in + 3);"
                      " fp_store(out, fp_mul_add_mul(a, b, c, d));",
    "fp_mul_sub_mul": "Fq a = fp_load(in), b = fp_load(in + 1), c = fp_load(in + 2), d = fp_load(in + 3);"
                      " fp_store(out, fp_mul_sub_mul(a, b, c, d));",
    "g1_add_mixed": "G1Xyzz acc = g1_load_xyzz((const G1Xyzz *)in); G1Affine q = g1_load_affine((const G1Affine *)(in + 4));"
                    " g1_add_mixed(acc, q); g1_store_xyzz((G1Xyzz *)out, acc);",
    "g1_add": "G1Xyzz acc = g1_load_xyzz((const G1Xyzz *)in), q = g1_load_xyzz((const G1Xyzz *)(in + 4));"
              " g1_add(acc, q); g1_store_xyzz((G1Xyzz *)out, acc);",
    "g1_dbl": "G1Xyzz p = g1_load_xyzz((const G1Xyzz *)in); g1_store_xyzz((G1Xyzz *)out, g1_dbl(p));",
}


def probe_source():
    lines = ['#include "g1.cuh"', "using namespace zkb;"]
    for name, body in PROBES.items():
        lines.append(f'extern "C" __global__ void probe_{name}(const Fq *__restrict__ in, Fq *__restrict__ out) {{ {body} }}')
    return "\n".join(lines) + "\n"


def count(sass):
    """per probe kernel: IMAD.WIDE (one 32x32->64 product), IMAD.HI, and every other IMAD form (IMAD, IMAD.X, IMAD.MOV, ..)"""
    res, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : probe_(\w+)", line)
        if m:
            cur = res.setdefault(m.group(1), {"IMAD.WIDE": 0, "IMAD.HI": 0, "IMAD other": 0})
            continue
        if cur is None:
            continue
        m = re.search(r"\b(IMAD(?:\.[A-Z0-9]+)*)\b", line)
        if not m:
            continue
        op = m.group(1)
        key = "IMAD.WIDE" if op.startswith("IMAD.WIDE") else "IMAD.HI" if op.startswith("IMAD.HI") else "IMAD other"
        cur[key] += 1
    for v in res.values():
        v["total"] = v["IMAD.WIDE"] + v["IMAD.HI"] + v["IMAD other"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "probe.cu")
        with open(src, "w") as f:
            f.write(probe_source())
        cubin = os.path.join(tmp, "probe.cubin")
        subprocess.check_call([os.path.join(CUDA, "bin", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                               "--expt-relaxed-constexpr", "-cubin", "-I", CSRC, src, "-o", cubin])
        sass = subprocess.check_output([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], text=True)
    res = {k: count(sass)[k] for k in PROBES}
    if args.json:
        print(json.dumps(res, indent=1))
        return
    print(f"{'primitive':16s} {'IMAD.WIDE':>9s} {'IMAD.HI':>8s} {'other':>6s} {'total':>6s}")
    for k, v in res.items():
        print(f"{k:16s} {v['IMAD.WIDE']:9d} {v['IMAD.HI']:8d} {v['IMAD other']:6d} {v['total']:6d}")


if __name__ == "__main__":
    sys.exit(main())
