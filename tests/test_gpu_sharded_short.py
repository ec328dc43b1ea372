"""Short queries on doc-id-range shards, on the GPU: two shard indexes in one process on one device, each rank's ShardedSearchEngine in its
own thread, exchanging through dist_util's stand-in for torch.distributed (CUDA tensors, a barrier). The same cases as the CPU test, a
batch large enough to take several groups of short queries, against the unsharded oracle; and the n-gram queries of a mixed batch against
the same queries alone (the path without short queries)."""
import pytest

import infidex_b200 as ib

import short_shard_util as U
from dist_util import run_ranks

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sharded():
    from infidex_b200 import dist as ifxd
    keys, schema, cols, vocab = U.corpus()
    ranges = ifxd.shard_ranges(U.N, 2)

    def build(d, r):
        lo, hi = ranges[r]
        eng = ifxd.ShardedSearchEngine(d, device_index=0)
        eng.IndexShard(keys[lo:hi], schema, [cols[0][lo:hi], cols[1][lo:hi]])
        return eng
    engines = run_ranks(2, build)
    yield engines, U.oracle_engine(keys, schema, cols), vocab
    for e in engines:
        e.Close()


def _search_with(engines, queries):
    def fn(d, r):
        engines[r].dist = d
        return [U.signature(x) for x in engines[r].SearchBatch(queries)]
    a, b = run_ranks(2, fn)
    assert a == b          # every rank merges the same answer
    return a


def test_short_queries_on_two_gpu_shards_match_the_unsharded_oracle(sharded):
    engines, orc, vocab = sharded
    ngram = [ib.Query(t, 10) for t in U.ngram_texts(vocab)]
    alone = _search_with(engines, ngram)
    mixed = _search_with(engines, [U.make_query(c) for c in U.SHORT_CASES] + ngram)
    ns = len(U.SHORT_CASES)
    assert mixed[ns:] == alone
    U.check_shard_facts(U.SHORT_CASES, [c.cpu().numpy() for c in engines[0].last_s1_counts], engines[0].last_shard_info.cpu().numpy())
    bad = U.compare_with_oracle(orc, U.SHORT_CASES, mixed[:ns])
    assert not bad, bad


def test_a_batch_of_several_short_query_groups(sharded):
    engines, orc, _ = sharded
    cases = U.SHORT_CASES * 3                   # more short queries than one group holds (32 at this corpus size)
    assert len(cases) > 2 * 32
    got = _search_with(engines, [U.make_query(c) for c in cases])
    ns = len(U.SHORT_CASES)
    assert got[:ns] == got[ns:2 * ns] == got[2 * ns:]
    bad = U.compare_with_oracle(orc, U.SHORT_CASES, got[:ns])
    assert not bad, bad
