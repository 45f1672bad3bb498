"""Per-row instruction counts of the constraint interpreter's program for the gates of a stand-in circuit, before and after
operand fusion (csrc/expr.cuh, ProgramBuilder::fuse).  Host only: the program comes from zkb_expr_program, exactly as
zkb_expr_eval_dev would upload it.  Mode 1 (default) is the gate part of the quotient program (selector runs folded with
HORNER2 / FOLD); the permutation and lookup scopes of a proof's quotient program come on top.

The unfused program is rebuilt from the fused one: every column (C) or constant (K) operand of a fused form was one
OP_LOADCOL / OP_LOADCONST into a register that the plain form then read.  Per row it prints
  - interpreted instructions (dispatches) by opcode, and program words fetched (a fused form with two C / K operands is two words);
  - register-file accesses: an access moves one 32-byte field element, two 16-byte LDS / STS in the shared-memory builds;
  - global field-element loads: columns, constants (including the y powers of HORNER / FOLD and STOREACC's scale);
  - Montgomery products and reductions: MUL, HORNER, HORNER2 and STOREACC are one product and one reduction each; FOLD
    (acc * y^r + f * acc2) and the merged HORNER_M / HORNER2_M (acc * y + a * b) two products with one reduction.
usage: python scripts/expr_program_stats.py [--shape super|keccak] [--k K] [--mode 0|1] [--json]"""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import numpy as np

# opcodes of csrc/expr.cuh
BASE = {0: "LOADCOL", 1: "LOADCONST", 2: "ADD", 3: "SUB", 4: "MUL", 5: "NEG", 6: "HORNER", 7: "STORE", 8: "STOREACC",
        9: "CLEARACC", 10: "HORNER2", 11: "FOLD", 12: "FLAG", 43: "HORNER_M", 44: "HORNER2_M"}
ARG = 13
FORMS = ["RC", "CR", "RK", "KR", "CC", "CK", "KC"]
FUSED = {16 + f: ("ADD", FORMS[f]) for f in range(7)}
FUSED.update({24 + f: ("SUB", FORMS[f]) for f in range(7)})
FUSED.update({32 + f: ("MUL", FORMS[f]) for f in range(7)})
FUSED.update({40: ("HORNER", "C"), 41: ("HORNER2", "C"), 42: ("FOLD", "C")})


def decode(code):
    """-> list of opcode bytes of the dispatched instructions (OP_ARG words are skipped) and the word count"""
    ops = [int(w) & 0xFF for w in code]
    return [o for o in ops if o != ARG], len(ops)


def counts(ops, words):
    """(dispatches by name, register-file reads, writes, global loads, words) for the fused program and its unfused original"""
    fused, plain = collections.Counter(), collections.Counter()
    rf = {"fused": [0, 0], "plain": [0, 0]}       # [reads, writes]
    loads = {"fused": 0, "plain": 0}
    for o in ops:
        if o in FUSED:
            base, form = FUSED[o]
            fused[f"{base}_{form}"] += 1
            plain[base] += 1
            ncol, nconst = form.count("C"), form.count("K")
            plain["LOADCOL"] += ncol
            plain["LOADCONST"] += nconst
            nreg = form.count("R") if base in ("ADD", "SUB", "MUL") else 0
            rf["fused"][0] += nreg
            rf["plain"][0] += nreg + ncol + nconst
            rf["plain"][1] += ncol + nconst
            if base in ("ADD", "SUB", "MUL"):
                rf["fused"][1] += 1
                rf["plain"][1] += 1
            extra = 1 if base in ("HORNER", "HORNER2", "FOLD") else 0   # the y-power constant
            loads["fused"] += ncol + nconst + extra
            loads["plain"] += ncol + nconst + extra
            continue
        name = BASE[o]
        fused[name] += 1
        if name in ("HORNER_M", "HORNER2_M"):        # merged: unfused it is a MUL (2 reads, 1 write) and the root (1 read)
            plain["MUL"] += 1
            plain[name[:-2]] += 1
            rf["fused"][0] += 2
            rf["plain"][0] += 3
            rf["plain"][1] += 1
            loads["fused"] += 1
            loads["plain"] += 1
            continue
        plain[name] += 1
        reads = {"ADD": 2, "SUB": 2, "MUL": 2, "NEG": 1, "HORNER": 1, "HORNER2": 1, "FOLD": 1, "STORE": 1, "FLAG": 1}.get(name, 0)
        writes = 1 if name in ("LOADCOL", "LOADCONST", "ADD", "SUB", "MUL", "NEG") else 0
        gl = 1 if name in ("LOADCOL", "LOADCONST", "HORNER", "HORNER2", "FOLD", "STOREACC") else 0
        for key in ("fused", "plain"):
            rf[key][0] += reads
            rf[key][1] += writes
            loads[key] += gl
    # Montgomery multiplies per row: (products, reductions) of the program as it runs
    cost = {"MUL": (1, 1), "HORNER": (1, 1), "HORNER2": (1, 1), "STOREACC": (1, 1), "FOLD": (2, 1), "HORNER_M": (2, 1),
            "HORNER2_M": (2, 1)}
    by = collections.Counter()
    for k, v in fused.items():
        by[k.split("_")[0] if k.split("_")[-1] in FORMS or k.endswith("_C") else k] += v
    products = sum(cost.get(k, (0, 0))[0] * v for k, v in by.items())
    reductions = sum(cost.get(k, (0, 0))[1] * v for k, v in by.items())
    return {"products": products, "reductions": reductions,
            "fused": {"dispatches": sum(fused.values()), "words": words, "by_op": dict(sorted(fused.items())),
                      "regfile_reads": rf["fused"][0], "regfile_writes": rf["fused"][1], "global_loads": loads["fused"]},
            "unfused": {"dispatches": sum(plain.values()), "words": sum(plain.values()), "by_op": dict(sorted(plain.items())),
                        "regfile_reads": rf["plain"][0], "regfile_writes": rf["plain"][1], "global_loads": loads["plain"]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", choices=["super", "keccak"], default="super")
    ap.add_argument("--k", type=int, default=17, help="row count exponent of the stand-in (default 17)")
    ap.add_argument("--mode", type=int, choices=[0, 1], default=1)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    import standins
    from zkb200 import plonk as Z
    # Only the constraint system is used.  From k = 17 up the stand-ins' gates, lookups and table sizes no longer change with k,
    # and rotations are row offsets, so the k = 17 program is the one the k = 20 benchmark proof runs; the witness the
    # constructor also builds (on the CPU here) is smaller at 17.
    k = args.k
    ops = standins.OracleOps()
    cs = (standins.super_shape(k, advice=128, seed=5, ops=ops) if args.shape == "super" else standins.keccak_shape(k, seed=3, ops=ops)).cs
    nch = len(cs.challenge_phase)
    ch = np.array([[0x5EED5 + i, 0, 0, 0] for i in range(nch)], dtype=np.uint64)   # any reduced values stand for the challenges
    one = np.array([1, 0, 0, 0], dtype=np.uint64)
    code, nregs = Z.expr_program(cs, mode=args.mode, challenges=ch, y=np.array([0x1D1CE, 0, 0, 0], dtype=np.uint64), scale=one)
    ops, words = decode(code)
    res = {"shape": args.shape, "k": k, "mode": args.mode, "gates": len(cs.gates), "registers": nregs, **counts(ops, words)}
    if args.json:
        print(json.dumps(res))
        return
    print(f"{args.shape} stand-in, k = {k}, mode {args.mode}: {len(cs.gates)} gates, {nregs} registers (per row)")
    f, p = res["fused"], res["unfused"]
    print(f"{'':24}{'unfused':>10}{'fused':>10}")
    for key in ("dispatches", "words", "regfile_reads", "regfile_writes", "global_loads"):
        print(f"{key:24}{p[key]:>10}{f[key]:>10}")
    print(f"Montgomery products {res['products']}, reductions {res['reductions']} per row")
    print("dispatches by opcode:")
    for name in sorted(set(f["by_op"]) | set(p["by_op"])):
        print(f"  {name:22}{p['by_op'].get(name, 0):>10}{f['by_op'].get(name, 0):>10}")


if __name__ == "__main__":
    main()
