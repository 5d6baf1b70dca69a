"""GPU, world_size 2 (needs two GPUs on the box; skipped on a single-GPU box): the row-sharded step of config 5 through
torchrun, both forms of the exchange -- "p2p" (kernels storing into the peers' symmetric-memory buffers, signal-pad
barriers, no NCCL on the data path) and "nccl" (the collective baseline).  tools/shard_bench.py --check verifies on every
rank: scores against the all-gathered tables (<= 1e-5) and the SGD step of its shard against the autograd step of the
GLOBAL objective on the gathered tables."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs on one box (gpurun --gpus 2)")]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_two_rank_sharded_step_matches_the_global_objective(exchange):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tools", "shard_bench.py"), "--check", "--n_items", "200000",
           "--n_users", "50000", "--emb", "128", "--B", "512", "--K", "31", "--steps", "3", "--warmup", "1", "--optimizer", "SGD",
           "--exchange", exchange]
    env = dict(os.environ, PYTHONPATH=ROOT)
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    checks = [json.loads(ln) for ln in res.stdout.splitlines() if ln.startswith("{") and "check_max_abs_err" in ln]
    assert len(checks) == 2
    for c in checks:
        assert c["check_max_abs_err"] <= 1e-5 and c["update_ok"], c
