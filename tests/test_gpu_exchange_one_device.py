"""The sharded scan's exchange at P = 2 to 16 ranks on ONE H100: P processes share device 0 and store into each other's
peer windows (CUDA IPC between processes of one device), over a gloo group (tests/_one_device.py).  This runs every
multi-rank path of the peer-window exchange on a single GPU: ranks running concurrently and waiting on each other's
flags and acknowledgements, every k_classify_send instantiation (C = 1 + 2P counters: CW4 = 2 up to P = 3, 4 up to 7,
5 up to 9, 9 up to 16), owners that are not powers of two, ranks taking different send kernels in one step, and owned
lists far longer than the orderings were shaped for.  The checks are exact (tests/_one_device_exchange_worker.py).

The worlds are the two ends of every CW4: C = 5 / 7 -> 2, 9 / 15 -> 4, 17 / 19 -> 5, 21 / 33 -> 9.  The same transport
also runs the multi-GPU workers of test_gpu_parity, test_gpu_shard_delta and test_gpu_mdev_shard_delta at P > 1.

Contexts of one device time-slice: nothing here measures speed.  Several processes on one device need the Default
compute mode; it is read (never changed) and the tests skip under any other.  Every test here needs an H100 (`-m gpu`)."""
import os
import subprocess
import sys

import pytest

import _one_device

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
Mi = 1 << 20
WORLDS = [2, 3, 4, 7, 8, 9, 10, 16]


def _launch(world, script, args, timeout):
    mode = _one_device.compute_mode(0)
    if mode != _one_device.COMPUTE_MODE_DEFAULT:
        pytest.skip("device 0 is not in the Default compute mode (%r): its processes cannot share it" % mode)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(world),
           os.path.join(HERE, script)] + [str(a) for a in args]
    env = dict(os.environ, KVG_WORKER_STALL_S=str(timeout - 30), OMP_NUM_THREADS="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    return r.stdout


@pytest.mark.parametrize("world", WORLDS)
def test_exchange_steps(world):
    """Twelve scans on the same windows: tile edges, one owner, nothing home, empty, sparse dictionary, wide keys."""
    out = _launch(world, "_one_device_exchange_worker.py", ["steps"], 600)
    assert "exchange-ok job=steps world=%d" % world in out, out[-2000:]


def test_mixed_send_kernels():
    """P = 2 at FUSED_SEND_MAX - 1 and + 1 records: one rank fuses classify and send, the other sends standalone."""
    out = _launch(2, "_one_device_exchange_worker.py", ["mixed"], 900)
    assert "exchange-ok job=mixed world=2" in out, out[-2000:]


@pytest.mark.parametrize("world,n", [(2, 1_500_000), (4, 1_000_000)])
def test_owned_lists_past_expected_shape(world, n):
    """One owner takes every key: its owned lists are P x n records, the orderings were shaped for about n."""
    out = _launch(world, "_one_device_exchange_worker.py", ["big", n], 900)
    assert "exchange-ok job=big world=%d" % world in out, out[-2000:]


@pytest.mark.parametrize("world", [3, 8])
def test_sharded_scan_matches_oracle(world):
    """tests/_nccl_worker.py: PCI and mdev parts of every rank, merged, against the oracle over four steps."""
    out = _launch(world, "_nccl_worker.py", [200_003, "one-device"], 600)
    assert "nccl-ok world=%d n=200003" % world in out and "exchange=p2p" in out, out[-2000:]


@pytest.mark.parametrize("world,n", [(3, 10_000), (2, 2 * Mi + 1000)])
def test_sharded_delta_sequence(world, n):
    """tests/_shard_delta_worker.py: the sharded PCI re-scan delta at P > 1."""
    out = _launch(world, "_shard_delta_worker.py", [n, "one-device"], 900)
    assert "shard-delta-ok world=%d n=%d exchange=p2p" % (world, n) in out, out[-2000:]


@pytest.mark.parametrize("world,n", [(3, 10_000), (2, 2 * Mi + 1000)])
def test_sharded_mdev_delta_sequence(world, n):
    """tests/_mdev_shard_delta_worker.py: the sharded mdev re-scan delta at P > 1."""
    out = _launch(world, "_mdev_shard_delta_worker.py", [n, "one-device"], 900)
    assert "mdev-shard-delta-ok world=%d n=%d exchange=p2p" % (world, n) in out, out[-2000:]
