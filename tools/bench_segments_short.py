"""Cost of short queries (no word of >= 3 characters) when documents share a DocumentKey (segments). The same synthetic titles are indexed
twice, with unique keys and with about a third of the keys spread over runs of 2-3 consecutive documents, and a short-heavy batch (64 short
+ 64 n-gram queries) is timed on each, one index after the other, alternating, in one process. Prints one JSON line: ms per batch, ms per
short query (the batch's time less the same n-gram queries alone, over 64), the device and its power limit.

    python tools/bench_segments_short.py --docs 1000000 --steps 5 --warmup 2
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import infidex_b200 as ib                      # noqa: E402
from infidex_b200 import synth                 # noqa: E402

SHORT = ["a", "e", "s", "t", "x", "st", "an", "re", "a b", "s t", "on", "in", "m", "p", "de", "ra"]


def repeated_keys(n, seed=5):
    """Keys of n documents: two thirds of the keys hold one document, the rest runs of 2 or 3."""
    rng = np.random.Generator(np.random.PCG64(seed))
    keys = np.empty(n, np.int64); k = 0; i = 0
    while i < n:
        run = 1 if rng.random() < 2 / 3 else int(rng.integers(2, 4))
        keys[i: i + run] = k; k += 1; i += run
    return keys, k


def time_batch(eng, qs, steps, warmup):
    import torch
    for _ in range(warmup):
        eng.SearchBatch(qs)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(steps):
        eng.SearchBatch(qs)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_segments_short: needs a CUDA device")
    vocab = synth.make_vocab(100_000)
    docs = synth.gen_docs(a.docs, vocab)
    schema = [ib.Field("title", None, ib.Weight.Med)]
    rep, n_keys = repeated_keys(a.docs)
    engines = {}
    for name, keys in (("unique", docs["keys"]), ("segments", rep)):
        e = ib.SearchEngine(); e.IndexColumns(keys, schema, [docs["title"]]); engines[name] = e
    ngram = [ib.Query(t, 10) for t in synth.gen_queries(64, docs, vocab)]
    short = [ib.Query(t, 10) for t in SHORT * 4]
    flagged = {n: sum(1 for r in e.SearchBatch(short) if r.Status & ~8) for n, e in engines.items()}
    res = {n: {"batch_ms": [], "ngram_ms": []} for n in engines}
    for _ in range(a.rounds):
        for n, e in engines.items():
            res[n]["batch_ms"].append(time_batch(e, short + ngram, a.steps, a.warmup))
            res[n]["ngram_ms"].append(time_batch(e, ngram, a.steps, a.warmup))
    out = {"docs": a.docs, "keys_segments": int(n_keys), "batch": "64 short + 64 n-gram", "flagged": flagged}
    for n, r in res.items():
        b, g = min(r["batch_ms"]), min(r["ngram_ms"])
        out[n] = {"batch_ms": round(b, 2), "ngram_only_ms": round(g, 2), "ms_per_short_query": round((b - g) / 64, 3),
                  "batch_ms_all": [round(x, 2) for x in r["batch_ms"]]}
    out["device"] = torch.cuda.get_device_name(0)
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                                            timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        out["power_limit"] = "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
