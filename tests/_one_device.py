"""Several ranks of a sharded scan on ONE GPU: every process a rank on CUDA device 0, a gloo process group, and the
byte collectives ShardedScan needs on CPU tensors.  The peer windows work between processes that share a device
(CUDA IPC opens a handle exported by another process of the same device) while NCCL refuses two ranks on one GPU,
so this transport is p2p only.  Contexts of one device time-slice instead of running at once: it tests the exchange
at any world size up to 16, it says nothing about its speed.

Launched by torch.distributed.run (RANK / WORLD_SIZE in the environment)."""
import ctypes
import os

CU_DEVICE_ATTRIBUTE_COMPUTE_MODE = 20
COMPUTE_MODE_DEFAULT = 0


def compute_mode(device: int = 0):
    """The compute mode of a device, read through the driver API (read only), or None without a driver.  Several
    processes on one device need the Default mode."""
    try:
        cuda = ctypes.CDLL("libcuda.so.1")
    except OSError:
        return None
    dev, mode = ctypes.c_int(0), ctypes.c_int(-1)
    if cuda.cuInit(0) or cuda.cuDeviceGet(ctypes.byref(dev), device):
        return None
    if cuda.cuDeviceGetAttribute(ctypes.byref(mode), CU_DEVICE_ATTRIBUTE_COMPUTE_MODE, dev):
        return None
    return mode.value


def init():
    """Join the gloo group on device 0 -> (rank, world, device)."""
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo")
    return int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), 0


def broadcast(b, src):
    """The 128-byte broadcast of ShardedScan (NCCL unique id; unused when the peer windows work)."""
    import torch
    import torch.distributed as dist
    t = torch.zeros(128, dtype=torch.uint8)
    if dist.get_rank() == src:
        t[:len(b)].copy_(torch.frombuffer(bytearray(b), dtype=torch.uint8))
    dist.broadcast(t, src)
    return bytes(t.numpy().tobytes())


def allgather(b):
    """Every rank's bytes (all of the same length), in rank order."""
    import torch
    import torch.distributed as dist
    t = torch.frombuffer(bytearray(b), dtype=torch.uint8)
    outs = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(outs, t)
    return [bytes(o.numpy().tobytes()) for o in outs]


def gather(obj):
    """Every rank's object, in rank order."""
    import torch.distributed as dist
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj)
    return out
