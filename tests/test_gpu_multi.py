"""Multi-GPU paths on real GPUs (skipped on a single-GPU box): domain-sharded NTT, point-range sharded MSM and the
multi-GPU create_proof must reproduce the single-GPU results exactly.  Run on a machine with at least two GPUs."""
import json
import os
import subprocess
import sys
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpu():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(script, args, nproc, port=None):
    port = port or _free_port()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "scripts", script)] + [str(a) for a in args]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    return json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_sharded_ntt_and_msm_match_single_gpu():
    r = _torchrun("multi_gpu_check.py", [], 2)
    assert r["all_ranks_ok"]
    assert all(v["ok"] for k, v in r.items() if isinstance(v, dict))


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_multi_gpu_create_proof_identical():
    r = _torchrun("multi_gpu_proof.py", [12, 12, 2, 10], 2)
    assert r["identical_proof_on_all_ranks"]
