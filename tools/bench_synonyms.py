"""SearchEngine with a SynonymMap against the same engine without one, on BASELINE.json configs[2] (10M multi-field documents, 10k-query
batches, top-10, coverage depth 500).

The map is seeded over the synthetic vocabulary (synth.make_synonym_pairs: 5 000 groups of 2-4 words, the first groups made of the most
frequent words). The plain index and the synonym index are built and timed one at a time, alternately (two 10M indexes do not fit on one
card together). For each: index build time, the k_canon stage of ifx_index_create, device bytes of the index, queries/s over
device-resident batches (CUDA events), Stage-1 waves. The synonym index is then checked against the oracle with the same map over its
image on 512 queries (half of them made of the map's surface forms): the run fails unless all 512 match (ids, Score bits, ties).

    python tools/bench_synonyms.py [--steps 3 --warmup 1 --rounds 1 --out DIR]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

import infidex_b200 as ib  # noqa: E402
from infidex_b200 import dist as ifxd  # noqa: E402
from infidex_b200 import synth  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the measurement itself needs no nvidia-smi
        return "unknown (%s)" % e


class CaptureStderr:
    """The native IFX_CREATE_TIMING lines go to fd 2: keep them to read the stage times and device bytes."""
    def __enter__(self):
        self.f = tempfile.TemporaryFile(mode="w+b"); sys.stderr.flush(); self.saved = os.dup(2); os.dup2(self.f.fileno(), 2); return self

    def __exit__(self, *a):
        sys.stderr.flush(); os.dup2(self.saved, 2); os.close(self.saved); self.f.seek(0); self.text = self.f.read().decode(errors="replace"); self.f.close()


def run_one(label, synonym_map, docs, schema, cols, batches, args):
    os.environ["IFX_CREATE_TIMING"] = "1"
    eng = ib.SearchEngine(synonymMap=synonym_map)
    with CaptureStderr() as cap:
        t0 = time.time(); eng.IndexColumns(docs["keys"], schema, cols); t_index = time.time() - t0
    del os.environ["IFX_CREATE_TIMING"]
    m = re.search(r"device memory: index ([\d.]+) MB", cap.text)
    k = re.search(r"synonym coverage text \(k_canon\)\s+([\d.]+) s", cap.text)
    kb = re.search(r"synonym coverage text: (\d+) keys, (\d+) chars, ([\d.]+) MB", cap.text)
    handles = [eng.UploadBatch(b) for b in batches]
    ms = 0.0; nq = 0; waves = 0
    for s, h in enumerate(handles):
        eng.FlushL2()
        st = eng.RunBatch(h)
        if s >= args.warmup:
            ms += st.ms_total; nq += len(batches[s]); waves = max(waves, st.s1_waves)
    for h in handles:
        eng.FreeBatch(h)
    out = {"index": label, "queries_per_s": round(nq / (ms / 1e3), 1) if ms > 0 else None, "ms_per_batch": round(ms / max(len(batches) - args.warmup, 1), 2),
           "index_build_s": round(t_index, 1), "index_device_mb": float(m.group(1)) if m else None,
           "k_canon_s": float(k.group(1)) if k else None, "cov_text_mb": float(kb.group(3)) if kb else None, "s1_waves": int(waves)}
    return eng, out


def parity(eng, schema, pairs, docs, vocab, n=512):
    from oracle.oracle import Field as OField
    from oracle_syn import SynOracleEngine
    orc = SynOracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema], pairs)
    orc.load_image(eng.image_ptr())
    rng = np.random.Generator(np.random.PCG64(1234))
    words = sorted({w for p in pairs for w in p})
    qs = synth.gen_queries(n // 2, docs, vocab, seed=99) + [" ".join(rng.choice(words, int(rng.integers(1, 3)))) for _ in range(n - n // 2)]
    res = eng.SearchBatch([ib.Query(q, 10) for q in qs])
    ok, os_, ot, on, ost = orc.search_batch(qs, 10, 500, True, None, threads=os.cpu_count() or 1)
    bad = 0
    for i, r in enumerate(res):
        k = [t.DocumentId for t in r.Records]; s = np.array([t.Score for t in r.Records], np.float32); ti = [t.Tiebreaker for t in r.Records]
        m = int(on[i])
        same = (r.Status & ~8) == 0 and ost[i] == 0 and k == ok[i, :m].tolist() and np.array_equal(s.view(np.uint32), os_[i, :m].view(np.uint32)) and ti == ot[i, :m].tolist()
        bad += 0 if same else 1
    return len(qs) - bad, len(qs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=1, help="plain / synonym builds, alternated")
    ap.add_argument("--n-docs", type=int, default=10_000_000); ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--groups", type=int, default=5000)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    t0 = time.time()
    vocab = synth.make_vocab(400_000)
    docs = synth.gen_docs(args.n_docs, vocab, with_description=True)
    schema, cols = synth.schema_and_columns(docs, True)
    pairs = synth.make_synonym_pairs(vocab, args.groups)
    smap = ib.SynonymMap()
    for a, b in pairs:
        smap.AddSynonym(a, b)
    batches = [[ib.Query(t, 10) for t in synth.gen_queries(args.nq, docs, vocab, seed=ifxd.rank_batch_seed(synth.SEED, s, 0))] for s in range(args.warmup + args.steps)]
    t_setup = time.time() - t0
    runs = []
    for r in range(args.rounds):
        for label, m in (("plain", None), ("synonyms", smap)):
            eng, out = run_one(label, m, docs, schema, cols, batches, args); out["round"] = r
            if label == "synonyms" and r == args.rounds - 1:
                good, total = parity(eng, schema, pairs, docs, vocab); out["parity"] = "%d / %d" % (good, total)
            eng.Dispose(); del eng
            runs.append(out); print(json.dumps(out), flush=True)
    res = {"workload": "configs[2]: %d multi-field docs, %d-query batches, top-10, coverage depth 500" % (args.n_docs, args.nq),
           "synonym_map": "%d groups, %d AddSynonym calls, %d keys" % (args.groups, len(pairs), len(smap.canonical_table())),
           "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "setup_s": round(t_setup, 1), "runs": runs}
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_synonyms.json"), "w") as f:
            json.dump(res, f, indent=1)
    p = [x["parity"] for x in runs if "parity" in x][-1]
    good, total = (int(v) for v in p.split(" / "))
    if good != total:
        sys.exit("parity: %s" % p)


if __name__ == "__main__":
    main()
