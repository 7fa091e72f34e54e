"""-m gpu test of the runtime filter across ranks: launches tests/runtime_filter_worker.py with one process per GPU (2 when
the box has at least two, else the same program with a single rank so that the code path still runs)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_runtime_filter_merge_shuffled_join_q3_across_ranks():
    import torch
    n = min(torch.cuda.device_count(), int(os.environ.get("GSQL_TEST_GPUS", "2")))
    assert n >= 1, "no CUDA device"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(27500 + os.getpid() % 2000), os.path.join(ROOT, "tests", "runtime_filter_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and "RUNTIME_FILTER_MULTIGPU_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-6000:])
    print(r.stdout.strip().splitlines()[-1])
