"""Multi-GPU parity (NCCL, one process per GPU): runs tests/nccl_worker.py under torch.distributed.run on 2 GPUs and
asserts its report.  Skipped on a single-GPU machine."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("peer", ["1", "0"])
def test_two_rank_nccl_equals_full_batch(peer):
    """peer=1: SyncBN statistics through the NVLink peer-memory kernel; peer=0: through dist.all_reduce (the fallback)."""
    env = dict(os.environ, MICHIGAN_B200_PEER_EXCHANGE=peer)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(HERE, "nccl_worker.py")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    lines = [l for l in r.stdout.splitlines() if l.startswith("NCCL_PARITY ")]
    assert r.returncode == 0 and lines, r.stdout[-4000:]
    res = json.loads(lines[-1][len("NCCL_PARITY "):])
    print(res)
    assert res["world"] == 2 and res["bcast"]
    if peer == "1":
        assert res["exchange_backend"] == "peer", res["exchange_backend"]
    assert res["g_out_max_abs_vs_full_batch_oracle"] <= 1e-3
    assert res["running_stats_uv_rel_err_vs_oracle"] <= 2e-3
    assert res["buffers_bit_identical"] and res["grads_bit_identical"] and res["d_grads_bit_identical"]
    assert res["post_step_G_bit_identical"] and res["post_step_D_bit_identical"]
    assert res["g_grad_worst_cosine_vs_oracle"] >= 0.98, res
    for k, v in res["g_losses"].items():
        pass   # per-rank losses are shard losses; their mean over ranks equals the oracle's (checked through the gradients)
