"""CPU: how ShardedScan chooses its transport.  The peer windows are tried first and the NCCL communicator is created
only when they fail on some rank, and then on every rank.  P ranks run as threads over fake contexts that record
their calls, joined by byte collectives on a barrier."""
import threading

import pytest

import kvgpu
from kvgpu import _lib as L


class FakeCtx:
    def __init__(self, rank, export_ok=True, import_ok=True):
        self.rank, self.export_ok, self.import_ok = rank, export_ok, import_ok
        self.calls = []

    def comm_unique_id(self):
        self.calls.append(("comm_unique_id",))
        return b"u" * 128

    def comm_init(self, rank, world, uid):
        self.calls.append(("comm_init", rank, world, uid))

    def comm_p2p_export(self, rank, world, cap):
        self.calls.append(("comm_p2p_export", rank, world, cap))
        if not self.export_ok:
            raise L.KvgError(-2, "export refused")      # KVG_ECUDA
        return bytes([0x40 + rank]) * 64

    def comm_p2p_import(self, handles):
        self.calls.append(("comm_p2p_import", handles))
        if not self.import_ok:
            raise L.KvgError(-2, "import refused")      # KVG_ECUDA

    def comm_p2p_enable(self, on):
        self.calls.append(("comm_p2p_enable", on))

    def comm_destroy(self):
        self.calls.append(("comm_destroy",))

    def names(self):
        return [c[0] for c in self.calls]


class Collectives:
    """Byte broadcast / all-gather among `world` threads (rank order)."""

    def __init__(self, world):
        self.barrier = threading.Barrier(world, timeout=20)
        self.slots = [None] * world

    def allgather(self, rank, b):
        self.slots[rank] = bytes(b)
        self.barrier.wait()
        out = list(self.slots)
        self.barrier.wait()
        return out

    def broadcast(self, rank, b, src):
        if rank == src:
            self.slots[src] = bytes(b)
        self.barrier.wait()
        out = self.slots[src]
        self.barrier.wait()
        return out


def _run(world, ctxs, with_allgather=True, cap=1000):
    col = Collectives(world)
    out, errs = [None] * world, []

    def rank_main(r):
        try:
            sh = kvgpu.ShardedScan(ctxs[r], r, world, lambda b, src: col.broadcast(r, b, src),
                                   (lambda b: col.allgather(r, b)) if with_allgather else None, cap)
            sh.close()
            out[r] = sh
        except BaseException as e:    # noqa: BLE001 - reported below
            errs.append(e)
            col.barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(30)
    assert not errs, errs
    return out


@pytest.mark.parametrize("world", [1, 2, 5])
def test_peer_windows_everywhere_no_nccl(world):
    ctxs = [FakeCtx(r) for r in range(world)]
    shs = _run(world, ctxs)
    handles = b"".join(bytes([0x40 + r]) * 64 for r in range(world))
    for r, (sh, c) in enumerate(zip(shs, ctxs)):
        assert sh.mode == "p2p"
        assert c.names() == ["comm_p2p_export", "comm_p2p_import", "comm_p2p_enable", "comm_destroy"], c.calls
        assert c.calls[0] == ("comm_p2p_export", r, world, 1000)
        assert c.calls[1] == ("comm_p2p_import", handles)
        assert c.calls[2] == ("comm_p2p_enable", True)


@pytest.mark.parametrize("failing", ["export", "import"])
@pytest.mark.parametrize("world", [2, 4])
def test_one_rank_fails_every_rank_uses_nccl(world, failing):
    bad = world - 1
    ctxs = [FakeCtx(r, export_ok=not (failing == "export" and r == bad),
                    import_ok=not (failing == "import" and r == bad)) for r in range(world)]
    shs = _run(world, ctxs)
    for r, (sh, c) in enumerate(zip(shs, ctxs)):
        assert sh.mode == "nccl"
        n = c.names()
        assert "comm_p2p_enable" not in n, c.calls
        assert ("comm_p2p_import" in n) == (failing == "import"), c.calls    # no import after a failed export
        inits = [x for x in c.calls if x[0] == "comm_init"]
        assert inits == [("comm_init", r, world, b"u" * 128)], c.calls       # rank 0's unique id on every rank
        assert n.count("comm_unique_id") == (r == 0)
        assert n[-1] == "comm_destroy"


def test_without_allgather_nccl_as_before():
    world = 3
    ctxs = [FakeCtx(r) for r in range(world)]
    shs = _run(world, ctxs, with_allgather=False)
    for r, (sh, c) in enumerate(zip(shs, ctxs)):
        assert sh.mode == "nccl"
        want = ([("comm_unique_id",)] if r == 0 else []) + [("comm_init", r, world, b"u" * 128), ("comm_destroy",)]
        assert c.calls == want
