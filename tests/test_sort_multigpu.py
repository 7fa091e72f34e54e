"""-m gpu test of Q3's ORDER BY across ranks: launches tests/sort_worker.py with one process per GPU on 2 GPUs.  With a
single rank the pipeline returns before the gather to rank 0, so on a box with fewer than two GPUs the test is skipped
rather than passing without running the path it is named for (the one-rank ordered Q3 is tests/test_sort_q3_gpu.py)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_q3_order_by_gathered_to_rank0_across_ranks():
    import torch
    n = min(torch.cuda.device_count(), int(os.environ.get("GSQL_TEST_GPUS", "2")))
    assert n >= 1, "no CUDA device"
    if n < 2:
        pytest.skip("the gather of sorted runs to rank 0 needs at least 2 GPUs; with one rank it is never reached")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(29500 + os.getpid() % 2000), os.path.join(ROOT, "tests", "sort_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and "SORT_MULTIGPU_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-6000:])
    print(r.stdout.strip().splitlines()[-1])
