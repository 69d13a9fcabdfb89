"""Worker for the multi-GPU parity test: rank r scans its shard on GPU r (PCI records, then mdev records);
the union of the ranks' parts — every rank holds the keys it owns, with ALL their members — must equal the
oracle on the unsharded snapshot, byte for byte, for several back-to-back steps (window reuse, acks).

Arguments: n [mode [m_total [table]]]; table "long-names" scans against util.long_name_pciids() with the
type names of util.long_name_types() (vGPU resource names of up to 60,000 bytes) instead of the shipped
pci.ids and the synthetic type names."""
import hashlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "kubevirt-gpu-device-plugin_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch
import torch.distributed as dist

import kvgpu
import util
from oracle import oracle as O


def main():
    n = int(sys.argv[1])
    mode = sys.argv[2] if len(sys.argv) > 2 else "p2p"
    m_total = int(sys.argv[3]) if len(sys.argv) > 3 else max(n // 8, 3)
    long_names = len(sys.argv) > 4 and sys.argv[4] == "long-names"
    rank, world, local_rank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    text = util.long_name_pciids() if long_names else util.pciids_text()
    ids = O.nv_ids(text)
    ctx = kvgpu.Context(local_rank)
    ctx.pciids_load(text)
    # device-resident copy of the image: reps 1 and 3 re-parse it right before the scan, which then runs beside the
    # parse (side stream) and joins the names late
    pad = ctx.text_pad(len(text))
    h_text = np.full(pad + 16, 10, dtype=np.uint8)
    h_text[:len(text)] = np.frombuffer(text, dtype=np.uint8)
    d_text = torch.from_numpy(h_text).cuda()
    ctx.dev_pciids_parse(d_text.data_ptr(), len(text), pad + 16, 1)

    def bcast(b, src):
        t = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == src:
            t.copy_(torch.frombuffer(bytearray(b), dtype=torch.uint8))
        dist.broadcast(t, src)
        return bytes(t.cpu().numpy().tobytes())

    def allgather(b):
        t = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
        outs = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(outs, t)
        return [bytes(o.cpu().numpy().tobytes()) for o in outs]

    lo, hi = kvgpu.shard_range(n, rank, world)
    mlo, mhi = kvgpu.shard_range(m_total, rank, world)
    cap = max((n + world - 1) // world + 1, 2 * ((m_total + world - 1) // world + 1))
    sh = kvgpu.ShardedScan(ctx, rank, world, bcast, allgather if mode == "p2p" else None, cap)
    if mode == "p2p" and sh.mode != "p2p" and rank == 0:
        print("note: peer windows unavailable, fell back to NCCL")
    buf = torch.empty(max(hi - lo, 1) * 16, dtype=torch.uint8, device="cuda")
    mbuf = torch.empty(max(mhi - mlo, 1) * 32, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx.dev_gen_pci(buf.data_ptr(), lo, hi - lo, ids, 17)
    ctx.dev_gen_mdev(mbuf.data_ptr(), mlo, mhi - mlo)
    types = util.long_name_types() if long_names else O.gen_type_names(256)
    want_m = O.Maps()
    want_m.create_iommu_device_map_flat(O.gen_pci(0, n, ids, 17))
    want_m.create_vgpu_id_map_flat(O.gen_mdev(0, m_total), types)
    want = want_m.dump(text)
    trace = os.environ.get("KVG_WORKER_TRACE") == "1"
    for rep in range(4):   # > 2: exercises window reuse and the consumed-acks
        if trace:
            print("rank %d rep %d scan" % (rank, rep), file=sys.stderr, flush=True)
        if rep & 1:
            ctx.dev_pciids_parse(d_text.data_ptr(), len(text), pad + 16, 1)
        sh.scan_device_shard(buf.data_ptr(), hi - lo)
        res = sh.fetch()
        part = kvgpu.pci_maps_from_shard(res)
        # the maps are partitioned by key: rank r owns the keys with key % world == r
        assert all(int(k, 16) % world == rank for k in part.deviceMap), "foreign device key"
        assert all(int(k) % world == rank for k in part.iommuMap), "foreign iommu group"
        sh.scan_device_mdev_shard(mbuf.data_ptr(), mhi - mlo, types)
        mres = sh.fetch_mdev()
        mpart = kvgpu.mdev_maps_from_shard(mres)
        assert all(int(k) % world == rank for k in mres.by_type.type_keys), "foreign mdev type"
        assert all(int(k) % world == rank for k in mres.by_parent.par_keys), "foreign parent"
        part.vGpuMap, part.gpuVgpuMap = mpart.vGpuMap, mpart.gpuVgpuMap
        part.deviceNames.update(mpart.deviceNames)
        parts = [None] * world
        dist.all_gather_object(parts, part)
        got = kvgpu.canonical_dump(kvgpu.merge_parts(parts))      # raises if a key is owned twice
        assert got == want, "rank %d rep %d: sharded dump differs (%s vs %s)" % (
            rank, rep, hashlib.sha256(got).hexdigest()[:12], hashlib.sha256(want).hexdigest()[:12])
    dist.barrier()
    if rank == 0:
        print("nccl-ok world=%d n=%d sha=%s exchange=%s" % (world, n, hashlib.sha256(got).hexdigest()[:16], sh.mode))
    sh.close()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    # a failing rank must take the job down instead of hanging in collective teardown: dump where
    # every thread is if the run stalls, and leave without running destructors on an exception
    import faulthandler
    import traceback
    faulthandler.dump_traceback_later(int(os.environ.get("KVG_WORKER_STALL_S", "150")), exit=True)
    try:
        main()
    except BaseException:
        traceback.print_exc()
        sys.stderr.flush()
        os._exit(1)
