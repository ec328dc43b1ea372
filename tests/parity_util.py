"""Shared helpers: compare the product (CUDA, or the kernel emulation in CPU tests) with the oracle, bit for bit."""
import os

import numpy as np

import infidex_b200 as ib
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_LIB = os.path.join(ROOT, "tests", "emu", "libifx_emu.so")


def emu_lib():
    import __graft_entry__ as g
    return g.build_emu()


def build_pair(keys, schema, cols, gpu_lib=None):
    eng = ib.SearchEngine(_gpu_lib=gpu_lib) if gpu_lib else ib.SearchEngine.CreateDefault()
    eng.IndexColumns(keys, schema, cols)
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema])
    orc.index_columns(keys, cols)
    return eng, orc


def compare_stage1(eng, orc, queries, depth=500, stats=None):
    keys, scores, n, status = eng.Stage1Batch(queries, depth, stats)
    bad = []
    for i, q in enumerate(queries):
        r = orc.stage1(q, depth)
        st = int(status[i]) & ~8          # IFX_Q_EMPTY (blank query -> empty result) is not an error
        if r["status"] != 0 or st != 0:
            if (r["status"] != 0) != (st != 0):
                bad.append((q, "status", r["status"], int(status[i])))
            continue
        ok = n[i] == len(r["keys"]) and np.array_equal(keys[i, : n[i]], r["keys"]) and \
            np.array_equal(scores[i, : n[i]].view(np.uint32), r["scores"].view(np.uint32))
        if not ok:
            m = min(int(n[i]), len(r["keys"]))
            d = [k for k in range(m) if keys[i, k] != r["keys"][k] or scores[i, k] != r["scores"][k]][:3]
            bad.append((q, int(n[i]), len(r["keys"]), "path", r["path"], "cands", r["candidates"], "first diffs", d,
                        keys[i, d].tolist(), r["keys"][d].tolist(), scores[i, d].tolist(), r["scores"][d].tolist()))
    return bad


def compare_search(eng, orc, queries, max_results=10, flt=None, facets=False, depth=500, coverage=True):
    """Identical DocumentId order, Score bits (stricter than the 1e-5 relative tolerance of the north star),
    Tiebreaker bytes, TotalCandidates and facet tables."""
    qs = []
    for q in queries:
        x = ib.Query(q, max_results); x.Filter = flt; x.EnableFacets = facets; x.CoverageDepth = depth; x.EnableCoverage = coverage; qs.append(x)
    res = eng.SearchBatch(qs)
    bad = []
    for q, r in zip(queries, res):
        x = orc.search(q, max_results, depth=depth, coverage=coverage, filter_bytes=flt.bytecode() if flt else None, facets=facets)
        k = [t.DocumentId for t in r.Records]; s = np.array([t.Score for t in r.Records], np.float32); ti = [t.Tiebreaker for t in r.Records]
        st = r.Status & ~8
        if x["status"] != 0 or st != 0:
            if (x["status"] != 0) != (st != 0):
                bad.append((q, "status", x["status"], r.Status))
            continue
        ok = k == x["keys"] and np.array_equal(s.view(np.uint32), x["scores"].view(np.uint32)) and ti == x["ties"] and r.TotalCandidates == x["total"]
        if facets:
            fo = {}
            for f, v, c in x["facets"]:
                fo.setdefault(f, []).append((v, c))
            ok = ok and (r.Facets or {}) == fo
        if not ok:
            bad.append((q, k[:5], x["keys"][:5], s[:3].tolist(), x["scores"][:3].tolist(), ti[:3], x["ties"][:3], r.TotalCandidates, x["total"]))
    return bad


def compare_search_batch(eng, orc, queries, max_results=10, flt=None, depth=500, threads=None):
    """compare_search for large batches: the oracle runs the whole batch on all host threads (ids, Score bits, tie bytes, counts);
    TotalCandidates / facets are covered by compare_search on a subset."""
    qs = []
    for q in queries:
        x = ib.Query(q, max_results); x.Filter = flt; x.CoverageDepth = depth; qs.append(x)
    res = eng.SearchBatch(qs)
    ok, os_, ot, on, ost = orc.search_batch(queries, max_results, depth, True, flt.bytecode() if flt else None, threads=threads or (os.cpu_count() or 1))
    bad = []
    for i, (q, r) in enumerate(zip(queries, res)):
        st = r.Status & ~8
        if ost[i] != 0 or st != 0:
            if (ost[i] != 0) != (st != 0):
                bad.append((q, "status", int(ost[i]), r.Status))
            continue
        n = int(on[i]); k = [t.DocumentId for t in r.Records]; s = np.array([t.Score for t in r.Records], np.float32); ti = [t.Tiebreaker for t in r.Records]
        if not (k == ok[i, :n].tolist() and np.array_equal(s.view(np.uint32), os_[i, :n].view(np.uint32)) and ti == ot[i, :n].tolist()):
            bad.append((q, k[:5], ok[i, :n].tolist()[:5], s[:3].tolist(), os_[i, :3].tolist(), ti[:3], ot[i, :3].tolist()))
    return bad
