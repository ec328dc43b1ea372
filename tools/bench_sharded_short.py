"""Cost of answering short queries (no word of >= 3 characters) on doc-id-range shards.

1. Build time (CPU, host builder only): the champion exchange of a corpus split 2 and 8 ways -- bytes all-gathered and the seconds of the
   slowest shard's ifx_builder_export_champions, all-gather and ifx_builder_globalize_champions (every shard's builder a thread of this
   process, so the shards share this host's cores).
2. Search (GPU): ms per batch of a short-heavy batch, two shards on one device through the in-process harness (each rank a thread,
   exchanging through CUDA tensors), against the unsharded engine on the same corpus. Under torchrun with >= 2 GPUs the shards run one per
   GPU over NCCL instead.

    python tools/bench_sharded_short.py --build-docs 10000000 --gpu-docs 2000000
    torchrun --nproc-per-node 2 tools/bench_sharded_short.py --skip-build
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

import infidex_b200 as ib                      # noqa: E402
from dist_util import run_ranks                # noqa: E402
from infidex_b200 import dist as ifxd          # noqa: E402
from infidex_b200 import synth                 # noqa: E402

SHORT = ["a", "e", "s", "t", "x", "st", "an", "re", "a b", "s t", "on", "in", "m", "p", "de", "ra"]


def short_batch(n_ngram_texts):
    qs = [ib.Query(t, 10) for t in SHORT * 4] + [ib.Query(t, 10) for t in n_ngram_texts]
    return qs


def build_exchange(n_docs, world, threads):
    """Bytes and seconds of the champion exchange at `world` shards (all shards' builders at once, the slowest shard timed)."""
    vocab = synth.make_vocab(100_000)
    schema = [ib.Field("title", None, ib.Weight.Med)]
    shards = []
    for lo, hi in ifxd.shard_ranges(n_docs, world):
        docs = synth.gen_docs(hi - lo, vocab, start=lo)
        e = ib.SearchEngine(); e.IndexColumns(docs["keys"], schema, [docs["title"]], threads=threads, upload=False); shards.append(e)

    def fn(d, r):
        t0 = time.perf_counter()
        blobs = ifxd.exchange_builder(d, shards[r], "ifx_builder_export_champions", "ifx_builder_globalize_champions")
        return time.perf_counter() - t0, sum(len(b) for b in blobs)
    res = run_ranks(world, fn)
    for e in shards:
        e.Dispose()
    return {"docs": n_docs, "shards": world, "exchange_bytes": int(res[0][1]), "exchange_s_max": round(max(t for t, _ in res), 3)}


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
