"""Boosts / SortBy parity helpers: the product (CUDA, or the kernel emulation in CPU tests) against the oracle, bit for bit."""
import numpy as np

import infidex_b200 as ib
import oracle_post


def make_query(text, max_results=10, flt=None, facets=False, depth=500, coverage=True, boosts=None, sort=None):
    """boosts: [(Filter, strength)]; sort: (field name, ascending) or None."""
    x = ib.Query(text, max_results); x.Filter = flt; x.EnableFacets = facets; x.CoverageDepth = depth; x.EnableCoverage = coverage
    if boosts is not None:
        x.EnableBoost = True; x.Boosts = [ib.Boost(f, k) for f, k in boosts]
    if sort is not None:
        x.SortBy, x.SortAscending = sort
    return x


def _oracle_args(boosts, sort):
    b = None if boosts is None else [(f.bytecode(), int(k)) for f, k in boosts if f is not None]
    return b, sort


def compare_post(eng, orc, queries, max_results=10, flt=None, facets=False, depth=500, coverage=True, boosts=None, sort=None):
    """compare_search with boosts / SortBy: identical DocumentId order, Score bits, Tiebreaker bytes, TotalCandidates and facet tables.
    Returns (mismatches, overflowed): a query the device answers with IFX_Q_OVERFLOW (it holds only part of the list to reorder) is
    listed in `overflowed` instead of being compared."""
    qs = [make_query(q, max_results, flt, facets, depth, coverage, boosts, sort) for q in queries]
    res = eng.SearchBatch(qs)
    ob, osort = _oracle_args(boosts, sort)
    bad, over = [], []
    for q, r in zip(queries, res):
        x = oracle_post.search(orc, q, max_results, depth=depth, coverage=coverage, filter_bytes=flt.bytecode() if flt else None, facets=facets,
                               boosts=ob, sort=osort)
        st = r.Status & ~8
        if st == 4 and x["status"] == 0:
            over.append(q); continue
        if x["status"] != 0 or st != 0:
            if (x["status"] != 0) != (st != 0):
                bad.append((q, "status", x["status"], r.Status))
            continue
        k = [t.DocumentId for t in r.Records]; s = np.array([t.Score for t in r.Records], np.float32); ti = [t.Tiebreaker for t in r.Records]
        ok = k == x["keys"] and np.array_equal(s.view(np.uint32), x["scores"].view(np.uint32)) and ti == x["ties"] and r.TotalCandidates == x["total"]
        if facets:
            fo = {}
            for f, v, c in x["facets"]:
                fo.setdefault(f, []).append((v, c))
            ok = ok and (r.Facets or {}) == fo
        if not ok:
            bad.append((q, k[:5], x["keys"][:5], s[:3].tolist(), x["scores"][:3].tolist(), ti[:3], x["ties"][:3], r.TotalCandidates, x["total"]))
    return bad, over


def random_posts(rng, n, filters, sort_fields):
    """n random (boosts, sort) combinations over the given boost filters and SortBy field names (either may be absent)."""
    out = []
    for _ in range(n):
        nb = int(rng.integers(0, 4))
        boosts = [(filters[int(rng.integers(0, len(filters)))], int(rng.integers(1, 4))) for _ in range(nb)] if nb else None
        sort = (sort_fields[int(rng.integers(0, len(sort_fields)))], bool(rng.integers(0, 2))) if rng.integers(0, 3) else None
        if boosts is None and sort is None:
            sort = (sort_fields[0], True)
        out.append((boosts, sort))
    return out
