"""Boosts + SortBy next to the plain C4 workload, on one index, in one process.

  python tools/bench_post.py [--steps 3 --warmup 1 --n-docs 10000000 --nq 10000 --sample 512]

c4     = bench.py --workload c4: 10 M multi-field docs, Filter.Parse('year >= 2000 AND rating > 7.0') + EnableFacets, top-10
c4post = c4 + Query.EnableBoost with Boosts [genre = 'drama' High, year >= 2015 Low] + SortBy rating descending

Both batch kinds are uploaded once (device-resident, as bench.py's `value`) and run alternately, with the L2 flushed before every run;
the device time comes from the library's CUDA events (ms_total, and ms_final = k_finalize, where boosts and sort run). Parity: the first
`--sample` queries of the first timed c4post batch are answered by the oracle with its post-processing extension (tests/oracle_post.py)
and compared bit for bit. Prints one JSON line with the card's name and power limit; exits 1 on a parity mismatch.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import bench  # noqa: E402
import infidex_b200 as ib  # noqa: E402
import oracle_post  # noqa: E402

BOOSTS = [("genre = 'drama'", ib.BoostStrength.High), ("year >= 2015", ib.BoostStrength.Low)]
SORT = ("rating", False)


def make_batch(texts, flt, post):
    out = []
    for t in texts:
        x = ib.Query(t, 10); x.Filter = flt; x.EnableFacets = True
        if post:
            x.EnableBoost = True; x.Boosts = [ib.Boost(ib.Filter.Parse(f), k) for f, k in BOOSTS]
            x.SortBy, x.SortAscending = SORT
        out.append(x)
    return out


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n-docs", type=int, default=10_000_000); ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--sample", type=int, default=512)
    args = ap.parse_args()
    wl = dict(bench.WORKLOADS["c4"], n_docs=args.n_docs, nq=args.nq)
    vocab, docs, schema, cols = bench.make_corpus(wl)
    eng = ib.SearchEngine.CreateDefault()
    eng.IndexColumns(docs["keys"], schema, cols)
    flt = ib.Filter.Parse(bench.C4_FILTER)
    n_total = args.warmup + args.steps
    texts = [bench.batch_queries(wl, docs, vocab, s) for s in range(n_total)]
    kinds = ("c4", "c4post")
    handles = {k: [eng.UploadBatch(make_batch(texts[s], flt, k == "c4post")) for s in range(n_total)] for k in kinds}
    ms = {k: 0.0 for k in kinds}; fin = {k: 0.0 for k in kinds}
    for s in range(n_total):
        for k in (kinds if s % 2 == 0 else kinds[::-1]):      # alternate which kind runs first
            eng.FlushL2(); st = eng.RunBatch(handles[k][s])
            if s >= args.warmup:
                ms[k] += st.ms_total; fin[k] += st.ms_final
    for k in kinds:
        for h in handles[k]:
            eng.FreeBatch(h)
    # parity of c4post: the first timed batch through the C-ABI call, against the oracle over the same image
    s0 = args.warmup; sample = min(args.sample, wl["nq"])
    packed = eng.PackBatch(make_batch(texts[s0][:sample], flt, True)); eng.SearchPacked(packed); g = packed["bufs"]
    orc = bench.oracle_from_image(eng, schema)
    for f, col in zip(schema, cols):       # the image holds column values as text: SortBy compares the int64 / double values
        if isinstance(col, np.ndarray) and (f.Filterable or f.Facetable or f.Sortable):
            oracle_post.set_field_kind(orc, f.Name, 2 if col.dtype.kind in "iu" else 3)
    ok, osc, ot, on, ost = oracle_post.search_batch(orc, texts[s0][:sample], 10, 500, True, flt.bytecode(), threads=bench.effective_cpus(),
                                                    boosts=[(ib.Filter.Parse(f).bytecode(), k) for f, k in BOOSTS], sort=SORT)
    bad = []
    for i in range(sample):
        st = int(g["status"][i]) & ~8
        if ost[i] != 0 or st != 0:
            if (ost[i] != 0) != (st != 0):
                bad.append((texts[s0][i], "status", int(ost[i]), st))
            continue
        n = int(on[i])
        if not (n == int(g["n"][i]) and np.array_equal(g["keys"][i, :n], ok[i, :n]) and np.array_equal(g["scores"][i, :n].view(np.uint32), osc[i, :n].view(np.uint32))
                and np.array_equal(g["ties"][i, :n], ot[i, :n])):
            bad.append((texts[s0][i], g["keys"][i, :3].tolist(), ok[i, :3].tolist()))
    line = {"gpu": gpu_info(), "n_docs": wl["n_docs"], "batch": wl["nq"], "steps": args.steps, "warmup": args.warmup,
            "queries_per_s": {k: wl["nq"] * args.steps / (ms[k] / 1e3) for k in kinds},
            "ms_per_batch": {k: ms[k] / args.steps for k in kinds}, "k_finalize_ms_per_batch": {k: fin[k] / args.steps for k in kinds},
            "c4post_parity": {"checked": sample, "mismatches": len(bad), "what": "DocumentId order, float32 Score bits, Tiebreaker bytes vs the oracle"}}
    print(json.dumps(line), flush=True)
    if bad:
        print("PARITY FAILURE: %r" % bad[:3], file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
