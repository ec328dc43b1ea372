"""Boosts and SortBy on the GPU at scale: the multi-field slice of test_gpu_at_scale (100 k documents), the C4 filter + facets with
boosts and sorts on every column type, max_results 10 and 100, coverage on and off, tie-heavy cases -- bit-identical to the oracle."""
import numpy as np
import pytest

import infidex_b200 as ib
from infidex_b200 import synth
from parity_util import build_pair, compare_search
from post_util import compare_post, make_query, random_posts

pytestmark = pytest.mark.gpu
F = ib.Filter
C4_FILTER = "year >= 2000 AND rating > 7.0"


@pytest.fixture(scope="module")
def multi():
    vocab = synth.make_vocab(100_000)
    docs = synth.gen_docs(100_000, vocab, with_description=True)
    schema, cols = synth.schema_and_columns(docs, True)
    eng, orc = build_pair(docs["keys"], schema, cols)
    return eng, orc, synth.gen_queries(400, docs, vocab)


@pytest.mark.parametrize("max_results", [10, 100])
@pytest.mark.parametrize("coverage", [True, False])
def test_c4_boosts_and_sort(multi, max_results, coverage):
    eng, orc, qs = multi
    flt = F.Parse(C4_FILTER)
    boosts = [(F.Parse("genre = 'drama'"), ib.BoostStrength.High), (F.Parse("year >= 2015"), ib.BoostStrength.Low)]
    for b, s in ((boosts, ("rating", False)), (boosts, None), (None, ("genre", True)), (None, ("year", False))):
        bad, over = compare_post(eng, orc, qs[:150], max_results=max_results, flt=flt, facets=True, coverage=coverage, boosts=b, sort=s)
        assert not bad and not over, (b is not None, s, bad[:3])


def test_random_mixes(multi):
    eng, orc, qs = multi
    rng = np.random.Generator(np.random.PCG64(23))
    filters = [F.Parse("genre = 'drama'"), F.Parse("year >= 2015"), F.Parse("rating > 7.5"), F.Parse("genre IN ('comedy', 'horror')"), F.Parse("year < 1990")]
    short = ["a", "th", "x"]
    for i, (b, s) in enumerate(random_posts(rng, 16, filters, ["genre", "year", "rating", "nonexistent"])):
        bad, over = compare_post(eng, orc, qs[i * 20:i * 20 + 20] + short + [""], max_results=(10, 100)[i % 2], facets=i % 2 == 0,
                                 coverage=i % 3 != 0, flt=F.Parse(C4_FILTER) if i % 4 == 1 else None, boosts=b, sort=s)
        assert not bad, (i, bad[:3])
        assert set(over) <= set(short), over


def test_default_path_unchanged_after_post_queries(multi):
    """A batch with boosts / SortBy, then the plain batch on the same cached handle: the plain answers are the oracle's."""
    eng, orc, qs = multi
    eng.SearchBatch([make_query(q, 10, boosts=[(F.Parse("genre = 'drama'"), 3)], sort=("rating", True)) for q in qs[:50]])
    assert not compare_search(eng, orc, qs[:50])


def test_twenty_identical_documents_tie_order():
    texts = ["batman saves the day"] * 20; tags = ["x"] * 20
    schema = [ib.Field("content"), ib.Field("tag", None, ib.Weight.Med, indexable=False, filterable=True)]
    eng, orc = build_pair(np.arange(20), schema, [texts, tags])
    for mr in (20, 50):
        for b, s in (([(F.Parse("tag = 'nobody'"), 3)], None), (None, ("tag", True)), ([(F.Parse("tag = 'x'"), 1)], ("tag", False))):
            bad, over = compare_post(eng, orc, ["batman", "saves the day", "batmen"], max_results=mr, boosts=b, sort=s)
            assert not bad and not over, (mr, bad[:2])
