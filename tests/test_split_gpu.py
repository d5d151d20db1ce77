"""Real multi-GPU batch split (needs >= 2 GPUs; skipped on a single-GPU machine): the gathered
batch of a request sharded with pfd_b200/parallel.py equals the single-GPU result for the same seed."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_gpu_split_equals_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tools", "split_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("SPLIT_RESULT ")]
    assert r.returncode == 0 and lines, (r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(lines[-1][len("SPLIT_RESULT "):])
    print(res)
    assert res["noise_slice_equals_single_gpu_randn"] and res["rel_rms_gathered_vs_single_gpu"] < 3e-3
