"""Rank harnesses of the multi-rank tests and tools.

- ThreadDist / run_ranks: the part of torch.distributed that infidex_b200.dist uses, for ranks that are threads of one process (CPU tensors,
  or CUDA tensors on one device).
- free_port / spawn_gloo: ranks that are processes of one gloo group on this host."""
import os
import socket
import threading

import torch


class _Group:
    def __init__(self, world):
        self.world = world; self.slots = [None] * world; self.bar = threading.Barrier(world, timeout=600)


class ThreadDist:
    """torch.distributed's collectives for ranks that are threads of one process."""

    class ReduceOp:
        SUM, MAX = "sum", "max"

    def __init__(self, group, rank):
        self.g, self.rank = group, rank

    def get_rank(self):
        return self.rank

    def get_world_size(self):
        return self.g.world

    def _exchange(self, value):
        self.g.slots[self.rank] = value
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        self.g.bar.wait(); vals = list(self.g.slots); self.g.bar.wait()
        return vals

    def barrier(self):
        self.g.bar.wait()

    def all_gather(self, out, t):
        for o, v in zip(out, self._exchange(t.clone())):
            o.copy_(v)

    def all_reduce(self, t, op=ReduceOp.SUM):
        vals = self._exchange(t.clone()); r = vals[0].clone()
        for v in vals[1:]:
            r = r + v if op == self.ReduceOp.SUM else torch.maximum(r, v)
        t.copy_(r)

    def all_gather_object(self, out, obj):
        out[:] = self._exchange(obj)


def run_ranks(world, fn):
    """fn(dist, rank) on `world` threads that form one group; returns the results by rank."""
    g = _Group(world); res = [None] * world; err = []

    def body(r):
        try:
            res[r] = fn(ThreadDist(g, r), r)
        except BaseException as e:      # the other ranks would wait at the barrier forever
            err.append(e); g.bar.abort()
    ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if err:
        raise err[0]
    return res


def free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _gloo_rank(rank, world, port, worker, args):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    worker(rank, world, *args)
    dist.barrier(); dist.destroy_process_group()


def spawn_gloo(worker, world, *args):
    """worker(rank, world, *args) in `world` processes that form one gloo group (torch.distributed is initialised when it runs). `worker` is
    a top-level function, so that the spawned processes can import it."""
    import torch.multiprocessing as mp
    mp.spawn(_gloo_rank, args=(world, free_port(), worker, args), nprocs=world, join=True)
