"""Short queries on an index whose documents share a DocumentKey, on the GPU: segments_short_util's corpus at 120 000 documents (about a
third of the keys in runs of 2-3 segments, others scattered), so the per-block selection of the scan runs over many blocks and runs of
segments straddle block boundaries -- ids, Score bits, Tiebreakers, TotalCandidates and facets against the oracle; batches of more short
queries than one group holds through SearchBatch and Stage1Batch; and doc-id-range shards, which still flag these queries."""
import numpy as np
import pytest

import infidex_b200 as ib
import segments_short_util as U
from dist_util import run_ranks
from parity_util import build_pair, compare_search, compare_search_batch, compare_stage1

pytestmark = pytest.mark.gpu
N = 120_000
MORE = ["ка", "ма", "по", "ра", "то", "к м", "о а", "р", "т", "к", "м", "п", "zo", "ba", "ko", "mi", "b", "z", "o", "i"]


@pytest.fixture(scope="module")
def seg():
    keys, schema, cols = U.corpus(N)
    assert len(np.unique(keys)) < N * 0.85
    eng, orc = build_pair(keys, schema, cols)
    return eng, orc


@pytest.mark.parametrize("max_results", [10, 64, 100])
def test_search_matches_the_oracle(seg, max_results):
    eng, orc = seg
    res = eng.SearchBatch([ib.Query(q, max_results) for q in U.SHORT])
    assert all(r.Status & ~8 == 0 for r in res)
    bad = compare_search(eng, orc, U.SHORT + MORE, max_results=max_results)
    assert not bad, bad[:3]


def test_coverage_off_filter_and_facets(seg):
    eng, orc = seg
    bad = compare_search(eng, orc, U.SHORT, max_results=100, coverage=False)
    assert not bad, bad[:3]
    qs = [q for q in U.SHORT + MORE if orc.search(q, 10)["total"] <= 500]      # whole-list answers within the list the device keeps
    assert len(qs) >= 8
    bad = compare_search(eng, orc, qs, max_results=20, flt=ib.Filter.Parse(U.C4_FILTER), facets=True)
    assert not bad, bad[:3]


def test_batches_of_many_short_queries(seg):
    """More short queries than one group holds (32 at this size), through SearchBatch and Stage1Batch."""
    eng, orc = seg
    qs = (U.SHORT + MORE) * 2
    assert len(qs) >= 64
    bad = compare_search_batch(eng, orc, qs, max_results=50)
    assert not bad, bad[:3]
    bad = compare_stage1(eng, orc, qs, depth=64)
    assert not bad, bad[:3]


def test_two_shards_still_flag_short_queries():
    """A key's segments may sit on two doc-id-range shards, and nothing exchanges per-key partial sums: short queries stay flagged
    IFX_Q_UNSUPPORTED_OP there (the sharded short-query corpus with every key held by two consecutive documents); n-gram queries are answered."""
    import short_shard_util as S
    from infidex_b200 import dist as ifxd
    keys, schema, cols, _ = S.corpus()
    keys = keys // 2
    ranges = ifxd.shard_ranges(S.N, 2)
    qs = [ib.Query(q, 10) for q in ["a", "st", "a b", "ж", "бо", "x y"]] + [ib.Query("бор", 10), ib.Query("жук", 10)]

    def fn(d, r):
        lo, hi = ranges[r]
        eng = ifxd.ShardedSearchEngine(d, device_index=0)
        eng.IndexShard(keys[lo:hi], schema, [cols[0][lo:hi], cols[1][lo:hi]])
        return [int(x.Status) for x in eng.SearchBatch(qs)], eng
    (a, e0), (b, e1) = run_ranks(2, fn)
    e0.Close(); e1.Close()
    assert a == b
    assert all(s & 2 for s in a[:6]), a
    assert all(s & ~8 == 0 for s in a[6:]), a
