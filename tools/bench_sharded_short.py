"""Cost of answering short queries (no word of >= 3 characters) on doc-id-range shards.

1. Build time (CPU, host builder only): the champion exchange of a corpus split 2 and 8 ways -- bytes all-gathered and the seconds of one
   shard's ifx_builder_export_champions and ifx_builder_globalize_champions (shards export in parallel on their own hosts).
2. Search (GPU): ms per batch of a short-heavy batch, two shards on one device through the in-process harness (each rank a thread,
   exchanging through CUDA tensors), against the unsharded engine on the same corpus. Under torchrun with >= 2 GPUs the shards run one per
   GPU over NCCL instead.

    python tools/bench_sharded_short.py --build-docs 10000000 --gpu-docs 2000000
    torchrun --nproc-per-node 2 tools/bench_sharded_short.py --skip-build
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import infidex_b200 as ib                      # noqa: E402
from infidex_b200 import dist as ifxd          # noqa: E402
from infidex_b200 import synth                 # noqa: E402

SHORT = ["a", "e", "s", "t", "x", "st", "an", "re", "a b", "s t", "on", "in", "m", "p", "de", "ra"]


def short_batch(n_ngram_texts):
    qs = [ib.Query(t, 10) for t in SHORT * 4] + [ib.Query(t, 10) for t in n_ngram_texts]
    return qs


def build_exchange(n_docs, world, threads):
    """Bytes and seconds of the champion exchange at `world` shards (one shard's builder timed; blobs of all shards)."""
    vocab = synth.make_vocab(100_000)
    schema = [ib.Field("title", None, ib.Weight.Med)]
    blobs, t_export, keep = [], [], None
    for r, (lo, hi) in enumerate(ifxd.shard_ranges(n_docs, world)):
        docs = synth.gen_docs(hi - lo, vocab, start=lo)
        e = ib.SearchEngine(); e.IndexColumns(docs["keys"], schema, [docs["title"]], threads=threads, upload=False)
        ln = C.c_size_t(0); e._host.ifx_builder_export_champions.restype = C.c_void_p
        t0 = time.perf_counter(); p = e._host.ifx_builder_export_champions(C.c_void_p(e._builder), C.byref(ln)); t_export.append(time.perf_counter() - t0)
        blobs.append(np.ctypeslib.as_array((C.c_uint8 * ln.value).from_address(p)).copy())
        if r == 0:
            keep = e
        else:
            e.Dispose()
    arr = (C.c_void_p * world)(*[b.ctypes.data for b in blobs])
    t0 = time.perf_counter(); rc = keep._host.ifx_builder_globalize_champions(C.c_void_p(keep._builder), world, 0, arr); t_glob = time.perf_counter() - t0
    assert rc == 0
    keep.Dispose()
    return {"docs": n_docs, "shards": world, "exchange_bytes": int(sum(len(b) for b in blobs)), "export_s_max": round(max(t_export), 3),
            "globalize_s": round(t_glob, 3)}


class _Group:
    def __init__(self, world):
        self.world = world; self.slots = [None] * world; self.bar = threading.Barrier(world, timeout=600)


class ThreadDist:
    """torch.distributed's collectives for ranks that are threads of one process (CUDA tensors on one device)."""

    class ReduceOp:
        SUM, MAX = "sum", "max"

    def __init__(self, group, rank):
        self.g, self.rank = group, rank

    def get_rank(self):
        return self.rank

    def get_world_size(self):
        return self.g.world

    def _exchange(self, value):
        import torch
        self.g.slots[self.rank] = value; torch.cuda.synchronize()
        self.g.bar.wait(); vals = list(self.g.slots); self.g.bar.wait()
        return vals

    def barrier(self):
        self.g.bar.wait()

    def all_gather(self, out, t):
        for o, v in zip(out, self._exchange(t.clone())):
            o.copy_(v)

    def all_reduce(self, t, op=ReduceOp.SUM):
        import torch
        vals = self._exchange(t.clone()); r = vals[0].clone()
        for v in vals[1:]:
            r = r + v if op == self.ReduceOp.SUM else torch.maximum(r, v)
        t.copy_(r)

    def all_gather_object(self, out, obj):
        out[:] = self._exchange(obj)


def run_ranks(world, fn):
    g = _Group(world); res = [None] * world; err = []

    def body(r):
        try:
            res[r] = fn(ThreadDist(g, r), r)
        except BaseException as e:
            err.append(e); g.bar.abort()
    ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if err:
        raise err[0]
    return res


def time_batches(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def gpu_in_process(n_docs, steps, warmup):
    vocab = synth.make_vocab(100_000); docs = synth.gen_docs(n_docs, vocab)
    schema = [ib.Field("title", None, ib.Weight.Med)]
    queries = short_batch(synth.gen_queries(64, docs, vocab))
    whole = ib.SearchEngine(); whole.IndexColumns(docs["keys"], schema, [docs["title"]])
    ms_whole = time_batches(lambda: whole.SearchBatch(queries), steps, warmup)
    whole.Dispose()
    ranges = ifxd.shard_ranges(n_docs, 2); blob, off = docs["title"]

    def build(d, r):
        lo, hi = ranges[r]
        col = (np.ascontiguousarray(blob[int(off[lo]): int(off[hi])]), np.ascontiguousarray(off[lo: hi + 1] - off[lo]))
        eng = ifxd.ShardedSearchEngine(d, device_index=0); eng.IndexShard(docs["keys"][lo:hi], schema, [col]); return eng
    engines = run_ranks(2, build)

    def one():
        def fn(d, r):
            engines[r].dist = d; engines[r].SearchBatch(queries)
        run_ranks(2, fn)
    ms_sh = time_batches(one, steps, warmup)
    short_ms = engines[0].exchange_ms.get("short", 0.0) / (steps + warmup)
    for e in engines:
        e.Close()
    return {"docs": n_docs, "queries": len(queries), "short_queries": len(SHORT) * 4, "ms_per_batch_unsharded": round(ms_whole, 2),
            "ms_per_batch_2_shards_one_gpu": round(ms_sh, 2), "short_rounds_ms_per_batch": round(short_ms, 2)}


def gpu_nccl(n_docs, steps, warmup):
    import torch
    import torch.distributed as dist
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local); dist.init_process_group("nccl")
    vocab = synth.make_vocab(100_000); lo, hi = ifxd.shard_ranges(n_docs, world)[rank]
    docs = synth.gen_docs(hi - lo, vocab, start=lo)
    schema = [ib.Field("title", None, ib.Weight.Med)]
    queries = short_batch(synth.gen_queries(64, synth.corpus_ref(n_docs), vocab))
    eng = ifxd.ShardedSearchEngine(dist, device_index=local); eng.IndexShard(docs["keys"], schema, [docs["title"]])
    ms = time_batches(lambda: eng.SearchBatch(queries), steps, warmup)
    eng.Close(); dist.destroy_process_group()
    return rank, {"docs": n_docs, "gpus": world, "queries": len(queries), "ms_per_batch": round(ms, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-docs", type=int, default=10_000_000)
    ap.add_argument("--gpu-docs", type=int, default=2_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--threads", type=int, default=None)
    ap.add_argument("--skip-build", action="store_true")
    ap.add_argument("--skip-gpu", action="store_true")
    a = ap.parse_args()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        rank, r = gpu_nccl(a.gpu_docs, a.steps, a.warmup)
        if rank == 0:
            print(json.dumps({"nccl": r}))
        return
    out = {}
    if not a.skip_build:
        out["champion_exchange"] = [build_exchange(a.build_docs, w, a.threads) for w in (2, 8)]
    if not a.skip_gpu:
        import torch
        out["gpu_in_process"] = gpu_in_process(a.gpu_docs, a.steps, a.warmup)
        out["gpu"] = torch.cuda.get_device_name(0)
        out["multi_gpu"] = "not measured: one process on one GPU (run under torchrun with >= 2 GPUs for the NCCL time)"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
