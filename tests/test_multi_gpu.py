"""N > 1 on real GPUs (needs >= 2 visible devices; the round-end single-GPU box skips it with a
reason): the hand-written NVLink P2P observation all-gathers -- the synchronous stand-alone kernel and the
pipelined push / wait pair that runs beside the chained HP1 steps -- equal NCCL's bit for bit."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_p2p_allgather_equals_nccl():
    env = dict(os.environ, N_ENVS="4096", ITERS="50", NCCL_DEBUG="WARN")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                        "127.0.0.1", "--master-port", "29533", os.path.join(ROOT, "tools", "check_p2p_allgather.py")],
                       capture_output=True, text=True, env=env, timeout=240)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("P2P_ALLGATHER")][-1]
    assert "equal_to_nccl=True" in line, line
    assert "pipelined_sync_equal=True" in line, line   # the gather beside the chained HP1 steps, awaited every step
    assert "pipelined_free_equal=True" in line, line   # ... and free running (pushes overlap the next steps)
