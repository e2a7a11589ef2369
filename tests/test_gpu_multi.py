"""Multi-GPU (NCCL) check of the population-sharded CEM: needs >= 2 GPUs; skipped otherwise.
The single-GPU equivalent of the same property (two shards in one process) is tests/test_gpu_shuffle.py::
test_sharded_cem_equals_unsharded_plan."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_sharded_cem_over_nccl_equals_single_gpu_plan():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "multi_worker.py")]
    res = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    lines = [l for l in res.stdout.splitlines() if l.startswith("{")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-2000:]
    rep = json.loads(lines[-1])
    assert rep["multi_gpu_check"] == "ok", rep
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "multi_gpu_check.json"), "w") as f:
        json.dump(rep, f)
