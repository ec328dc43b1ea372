"""Short queries (no word of >= 3 characters) on an index whose documents share a DocumentKey, on the kernel emulation against the oracle:
scores accumulated per key (ShortQueryProcessor.SearchShortQuery), the single-character scan and the champion lists consolidated per key
(SegmentProcessor.ConsolidateSegments) -- ids, Score bits, Tiebreakers, TotalCandidates and facet tables. The corpus is
segments_short_util's: contiguous and scattered repeated keys, hand-placed titles for each branch of the path."""
import numpy as np
import pytest

import infidex_b200 as ib
import segments_short_util as U
from parity_util import build_pair, compare_search, compare_stage1, emu_lib

N = 4_000


@pytest.fixture(scope="module")
def seg():
    keys, schema, cols = U.corpus(N)
    assert len(np.unique(keys)) < N
    eng, orc = build_pair(keys, schema, cols, gpu_lib=emu_lib())
    return eng, orc, keys


@pytest.fixture(scope="module")
def uniq():
    keys, schema, cols = U.corpus(N, repeated=False)
    assert len(np.unique(keys)) == N
    return build_pair(keys, schema, cols, gpu_lib=emu_lib())


def _answered(eng, qs, mx=10):
    res = eng.SearchBatch([ib.Query(q, mx) for q in qs])
    assert all(r.Status & ~8 == 0 for r in res), [(q, r.Status) for q, r in zip(qs, res) if r.Status & ~8]
    return res


@pytest.mark.parametrize("max_results", [5, 10, 30, 64, 100, 300])
def test_search_matches_the_oracle(seg, max_results):
    eng, orc, _ = seg
    _answered(eng, U.SHORT, max_results)
    bad = compare_search(eng, orc, U.SHORT, max_results=max_results)
    assert not bad, bad[:3]


@pytest.mark.parametrize("depth", [500, 64, 20])
def test_stage1_matches_the_oracle(seg, depth):
    eng, orc, _ = seg
    bad = compare_stage1(eng, orc, U.SHORT, depth=depth)
    assert not bad, bad[:3]


def test_champions_consolidated_to_fewer_than_max(seg):
    """"ж": the first `max` champions hold two segments of several keys, so the list the reference returns is shorter than max."""
    eng, orc, _ = seg
    for mx in (10, 30, 64):
        want = orc.search("ж", mx)
        assert 0 < len(want["keys"]) < mx, (mx, len(want["keys"]))
        got = eng.Search(ib.Query("ж", mx))
        assert [e.DocumentId for e in got.Records] == want["keys"] and got.TotalCandidates == want["total"]


def test_first_token_prefix_from_a_later_segment(seg):
    """"ле": keys whose first document does not start with the query (or does not match it at all) but a later segment does take the
    first-token-prefix bit (2) of ComputePrecedence; the score is still read from the key's first document."""
    eng, orc, keys = seg
    run = keys[4 * (N // 8): 4 * (N // 8) + 40]
    want = orc.search("ле", 300, coverage=False)
    got = eng.Search(_no_cov("ле", 300))
    by_key = dict(zip(want["keys"], want["scores"].tolist()))
    assert all(int(by_key[int(k)]) & 2 for k in run), "the case lost its shape"
    assert [e.DocumentId for e in got.Records] == want["keys"]
    assert np.array_equal(np.array([e.Score for e in got.Records], np.float32).view(np.uint32), want["scores"].view(np.uint32))


def _no_cov(text, mx):
    q = ib.Query(text, mx); q.EnableCoverage = False
    return q


@pytest.mark.parametrize("coverage", [True, False])
def test_coverage_on_and_off(seg, coverage):
    """Coverage over the consolidated list, and the <= 3-character rule on both sides of 500 prefix documents ("бо": 180; "a", "s": more)."""
    eng, orc, _ = seg
    for mx in (10, 100, 300):
        bad = compare_search(eng, orc, U.SHORT, max_results=mx, coverage=coverage, depth=mx if mx > 10 else 500)
        assert not bad, (mx, bad[:3])


def test_filter_and_facets(seg):
    """The C4 filter with facets. A query answered by its whole Stage-1 list filters and counts the list the device keeps (up to the
    coverage depth), so queries matching more keys than that are left out here, as they would be with unique keys."""
    eng, orc, _ = seg
    flt = ib.Filter.Parse(U.C4_FILTER)
    qs = [q for q in U.SHORT if orc.search(q, 10)["total"] <= 500]
    assert len(qs) >= len(U.SHORT) - 3
    for mx in (10, 64, 100):
        bad = compare_search(eng, orc, qs, max_results=mx, flt=flt, facets=True)
        assert not bad, (mx, bad[:3])
        bad = compare_search(eng, orc, qs, max_results=mx, facets=True)
        assert not bad, (mx, bad[:3])


def test_mixed_batch(seg):
    """Segmented short queries, n-gram queries and short queries whose every key is unique ("щ") in one batch; each n-gram answer equals the
    same query alone."""
    eng, orc, _ = seg
    ngram = ["бор", "лето тёплое", "старый лес", "гол 12", "щука", "море юг", "вечер"]
    qs = [x for pair in zip(U.SHORT, ngram * 3) for x in pair]
    bad = compare_search(eng, orc, qs, max_results=20)
    assert not bad, bad[:3]
    alone = eng.SearchBatch([ib.Query(q, 20) for q in ngram])
    mixed = eng.SearchBatch([ib.Query(q, 20) for q in ngram + U.SHORT])[: len(ngram)]
    assert [[(e.DocumentId, e.Score) for e in r.Records] for r in alone] == [[(e.DocumentId, e.Score) for e in r.Records] for r in mixed]


@pytest.mark.parametrize("max_results", [10, 100])
def test_unique_key_control(uniq, max_results):
    """The same titles with unique keys (no key_first): the path is the one that ran before keys could repeat."""
    eng, orc = uniq
    _answered(eng, U.SHORT, max_results)
    bad = compare_search(eng, orc, U.SHORT, max_results=max_results)
    assert not bad, bad[:3]
    bad = compare_stage1(eng, orc, U.SHORT)
    assert not bad, bad[:3]


def test_ngram_filter_and_facets_read_the_keys_first_document(seg):
    """Coverage records of n-gram queries too: the filter and the facet table read the key's first live document, whichever segment the
    record came from (the oracle's GetDocumentByPublicKey)."""
    eng, orc, keys = seg
    _, _, cols = U.corpus(N)
    qs = ["дым", "бор", "лето", "вечер", "море юг", "гол", "щука"] + [cols[0][i].split()[0] for i in range(0, N, 100)]
    flt = ib.Filter.Parse(U.C4_FILTER)
    for mx in (10, 100):
        assert not compare_search(eng, orc, qs, max_results=mx, facets=True)
        assert not compare_search(eng, orc, qs, max_results=mx, flt=flt, facets=True)
