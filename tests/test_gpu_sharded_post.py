"""Filters and facets on doc-id-range shards, on the GPU: two shard indexes in one process on one device, each rank's ShardedSearchEngine in its
own thread, exchanging through dist_util's stand-in for torch.distributed (CUDA tensors, a barrier). About a million multi-field documents
and a 2 000-query batch with the C4 filter and facets (and the other variants of sharded_post_util), against the unsharded oracle with the
acceptance rule; the uploaded and the packed paths of SearchBatch give identical answers."""
import time

import numpy as np
import pytest
import torch

import infidex_b200 as ib

import sharded_post_util as P
import short_shard_util as U
from dist_util import run_ranks

pytestmark = pytest.mark.gpu

N = 1_000_000
NQ = 500          # texts; every one in the four variants of sharded_post_util: a batch of 2 003 queries


def _docs(lo, hi, vocab):
    from infidex_b200 import synth
    docs = synth.gen_docs(hi - lo, vocab, with_description=True, start=lo)
    schema, cols = synth.schema_and_columns(docs, True)
    return P.keys_for(np.arange(lo, hi), N), schema, cols


@pytest.fixture(scope="module")
def sharded():
    from infidex_b200 import dist as ifxd
    from infidex_b200 import synth
    from oracle.oracle import Field as OField
    from oracle.oracle import OracleEngine
    vocab = synth.make_vocab(100_000); ranges = ifxd.shard_ranges(N, 2)

    def build(d, r):
        keys, schema, cols = _docs(*ranges[r], vocab)
        eng = ifxd.ShardedSearchEngine(d, device_index=0); eng.IndexShard(keys, schema, cols)
        return eng
    engines = run_ranks(2, build)
    keys, schema, cols = _docs(0, N, vocab)          # the unsharded oracle: the host builder's image of the whole corpus
    he = ib.SearchEngine.__new__(ib.SearchEngine); he._host = ib.engine._load_host(); he._builder = None; he._index = None; he._gpu = None
    he.IndexColumns(keys, schema, cols, upload=False)
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema]); orc.load_image(he.image_ptr())
    yield engines, orc, he, synth.gen_queries(NQ, synth.corpus_ref(N), vocab)
    for e in engines:
        e.Close()


def test_filters_and_facets_on_two_gpu_shards_match_the_unsharded_oracle(sharded):
    engines, orc, _, texts = sharded
    flt = ib.Filter.Parse(P.C4_FILTER); qs = P.batch(texts, flt)
    timing = {}

    def fn(d, r):
        engines[r].dist = d
        engines[r].SearchBatch(qs)            # warm-up (the batch handle is kept)
        torch.cuda.synchronize(); t0 = time.perf_counter()
        res = engines[r].SearchBatch(qs)
        torch.cuda.synchronize(); timing[r] = time.perf_counter() - t0
        return [U.signature(x, ignore_status=8) for x in res]
    a, b = run_ranks(2, fn)
    assert a == b          # every rank merges the same answer
    plain_bad, ids_bad, checked, bad = P.check(orc, qs, a, flt.bytecode())
    print("\n%s, two shards on one device: %d queries, %.1f ms per SearchBatch (both ranks' threads, exchanges and merge included); unfiltered "
          "records differ from the oracle for %d of %d texts (%d in DocumentId order); %d filtered / faceted answers checked"
          % (torch.cuda.get_device_name(0), len(qs), 1e3 * max(timing.values()), plain_bad, NQ, ids_bad, checked))
    assert not bad, bad[:3]
    assert ids_bad <= NQ // 10 and checked >= 3 * NQ * 3 // 4
    assert sum(1 for s in a if s[3]) > NQ      # facet tables are not empty


def test_whole_stage1_lists_on_two_gpu_shards_match_the_unsharded_oracle(sharded):
    """EnableCoverage off and 3-character queries over frequent prefixes: the whole Stage-1 list is filtered on the shards (TotalCandidates
    and facet rows summed), a list cut at max by the <= 3-character rule is filtered by the hosts."""
    engines, orc, _, texts = sharded
    from infidex_b200 import synth
    flt = ib.Filter.Parse(P.C4_FILTER); qs = P.whole_list_batch(texts[:40], P.three_char_texts(synth.make_vocab(100_000)), flt)

    def fn(d, r):
        engines[r].dist = d
        return [U.signature(x, ignore_status=8) for x in engines[r].SearchBatch(qs)]
    a, b = run_ranks(2, fn)
    assert a == b
    plain_bad, ids_bad, checked, bad = P.check(orc, qs, a, flt.bytecode())
    print("\nwhole-list queries: unfiltered records differ for %d of %d texts; %d filtered / faceted answers checked" % (plain_bad, len(qs) // 4, checked))
    assert not bad, bad[:3]
    assert checked >= 3 * len(qs) // 4 // 2


def test_uploaded_and_packed_batches_give_the_same_answers(sharded):
    engines, _, _, texts = sharded
    qs = P.batch(texts[:200], ib.Filter.Parse(P.C4_FILTER))

    def fn(d, r):
        e = engines[r]; e.dist = d
        up = e.UploadBatch(qs)
        try:
            merged = e.SearchBatch(None, raw=True, uploaded=up)
            assert len(merged) == 7          # (keys, scores, ties, n, total, status, facet tables)
            via_upload = e._results(qs, merged)
        finally:
            e.FreeBatch(up)
        via_packed = e.SearchBatch(qs, packed=e.eng.PackBatch(qs))
        return [U.signature(x, ignore_status=8) for x in via_upload], [U.signature(x, ignore_status=8) for x in via_packed]
    (u0, p0), (u1, p1) = run_ranks(2, fn)
    assert u0 == p0 == u1 == p1
    assert any(s[3] for s in u0)
