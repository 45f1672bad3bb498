"""Throughput of proving-key files (ProvingKey.write / ProvingKey.read: zkb_pk_write, zkb_pk_read) for the SuperCircuit-shaped
stand-in's key (tests/standins.py, the shape bench.py proves), through an in-memory writer and reader.

    python scripts/pk_serde_bench.py [--k 20] [--advice 128] [--reps 3] [--formats RawBytesUnchecked Processed]

For every format: write (vk + body) and read with check off and on, best of --reps after one warm-up call, timed with the host
clock around the call (every call synchronises).  One JSON line per (format, op) with the file's bytes and GB/s of file bytes, the
card name and its power limit.  Every file read back is written again and compared with the original bytes.  The
file lives in one preallocated buffer: the k = 20 key is about 21 GB in every raw format.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


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


class Counter:
    """a writer that keeps only the length of what it is given"""
    def __init__(self):
        self.n = 0

    def write(self, b):
        self.n += len(b)
        return len(b)


class Compare:
    """a writer that checks what it is given against the bytes of `view`"""
    def __init__(self, view):
        self.view, self.pos, self.same = view, 0, True

    def write(self, b):
        self.same = self.same and self.view[self.pos: self.pos + len(b)] == b
        self.pos += len(b)
        return len(b)


class Memory:
    """an in-memory file of a known size, written and read in place (no growth, no copies beyond the writes and reads themselves)"""
    def __init__(self, size):
        self.buf, self.pos = bytearray(size), 0
        self.view = memoryview(self.buf)

    def write(self, b):
        self.view[self.pos: self.pos + len(b)] = b
        self.pos += len(b)
        return len(b)

    def read(self, n):
        out = bytes(self.view[self.pos: self.pos + n])
        self.pos += len(out)
        return out

    def readinto(self, b):
        n = min(len(b), len(self.buf) - self.pos)
        b[:n] = self.view[self.pos: self.pos + n]
        self.pos += n
        return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--advice", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--formats", nargs="+", default=["RawBytesUnchecked", "RawBytes", "Processed"])
    args = ap.parse_args()
    import torch
    import standins
    from zkb200 import plonk as Z
    from zkb200.params import ParamsKZG, SerdeFormat
    assert torch.cuda.is_available(), "the pk file benchmark needs a GPU"
    name, power = card()
    sc = standins.super_shape(args.k, advice=args.advice, seed=5)
    srs = ParamsKZG.unsafe_setup_with_s(args.k, 1234).load()
    pk = Z.ProvingKey(sc.cs, [sc.host(t) for t in sc.fixed], [sc.host(t) for t in sc.sigma], srs=srs)
    vk = pk.vk_bytes()
    for fname in args.formats:
        fmt = SerdeFormat[fname]
        ref = Counter()
        pk.write(ref, fmt)
        mem = Memory(ref.n)

        def write():
            mem.pos = 0
            pk.write(mem, fmt)
        t = best_of(write, args.reps)
        line = {"k": args.k, "format": fname, "bytes": ref.n, "gpu": name, "power_limit": power}
        print(json.dumps({**line, "op": "write", "seconds": round(t, 4), "GB_per_s": round(ref.n / t / 1e9, 3)}), flush=True)
        for check in (False, True):
            def read():
                mem.pos = 0
                Z.ProvingKey.read(mem, sc.cs, srs, fmt, check=check).close()
            t = best_of(read, args.reps)
            print(json.dumps({**line, "op": f"read check={int(check)}", "seconds": round(t, 4), "GB_per_s": round(ref.n / t / 1e9, 3)}), flush=True)
        mem.pos = 0
        key = Z.ProvingKey.read(mem, sc.cs, srs, fmt, check=True)
        try:
            again = Compare(mem.view)
            key.write(again, fmt)
            assert key.vk_bytes() == vk and again.same and again.pos == ref.n, f"{fname}: the key read back writes other bytes"
        finally:
            key.close()
        del mem

if __name__ == "__main__":
    main()
