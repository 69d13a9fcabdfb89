"""The sharded mdev re-scan delta (kvg_dev_scan_mdev_shard_fetch_delta) on the H100s of the box: one process per GPU
(world = min(GPU count, 8); on a single-GPU box world 1, where the owned lists equal the local list but the exchange
and the three delta kernels still run), over both transports, at 10,000 mdevs per rank (classify and send fused in one
kernel over peer windows) and at 2 Mi + 1000 (past FUSED_SEND_MAX: the standalone send).  tests/_mdev_shard_delta_worker.py
holds the checks; tests/test_gpu_exchange_one_device.py runs it at P > 1 with the ranks sharing one GPU.
Every test here needs an H100 (`-m gpu`)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

Mi = 1 << 20


def _gpu_count():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("n", [10_000, 2 * Mi + 1000])
def test_sharded_mdev_delta_sequence(n, mode):
    world = max(1, min(_gpu_count(), 8))
    here = os.path.dirname(os.path.abspath(__file__))
    port = 30250 + (n % 97) + (0 if mode == "p2p" else 100)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(here, "_mdev_shard_delta_worker.py"), str(n), mode]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "mdev-shard-delta-ok world=%d n=%d" % (world, n) in r.stdout
