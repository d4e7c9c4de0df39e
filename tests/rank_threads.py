"""Ranks emulated by threads of one process on one GPU, for the collective host calls (sharded.rebalance): an in-process stand-in for
sharded.ProcessGroupTransport and a runner that starts one thread per rank."""
import threading
import types


class InProcessTransport:
    """rebalance()'s transport for rank `rank` of `world` ranks emulated by threads of one process, all on the same stream; `hub` is
    the state the ranks share (a barrier and one slot per rank)."""

    def __init__(self, hub, rank: int):
        self.hub, self.rank, self.world = hub, rank, len(hub.slot)

    def all_gather(self, t):
        h = self.hub
        h.slot[self.rank] = t.clone()
        h.barrier.wait()
        out = list(h.slot)
        h.barrier.wait()
        return out

    def exchange(self, sends, recvs):
        h = self.hub
        h.slot[self.rank] = dict(sends)
        h.barrier.wait()  # every rank's pack is enqueued before any copy out of its buffers
        for s, buf in recvs.items():
            buf.copy_(h.slot[s][self.rank])
        h.barrier.wait()


def run_ranks(world, fn):
    """fn(rank, transport) on `world` threads; re-raises the first failure."""
    hub = types.SimpleNamespace(barrier=threading.Barrier(world, timeout=300), slot=[None] * world)
    out, errs = [None] * world, [None] * world

    def body(r):
        try:
            out[r] = fn(r, InProcessTransport(hub, r))
        except BaseException as e:  # noqa: BLE001 - handed to the main thread
            errs[r] = e
            hub.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in errs:
        if e is not None and not isinstance(e, threading.BrokenBarrierError):
            raise e
    assert not any(errs), errs
    return out
