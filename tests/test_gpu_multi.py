"""2-GPU sharded engine vs the single-GPU engine (needs >= 2 GPUs; skipped otherwise)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_two_rank_sharded_matches_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "mg_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0 and "MG_CHECK_OK" in r.stdout
