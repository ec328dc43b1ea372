"""SearchEngine with a SynonymMap on the GPU against the oracle with the same map (tests/oracle_syn.py): DocumentId order, float32 Score
bits, Tiebreaker bytes, TotalCandidates, facets. The tiebreaker |Q| / |doc| of every multi-token result reads the length of the coverage
text the device derives (k_canon_*), so parity checks that text directly."""
import numpy as np
import pytest

import infidex_b200 as ib
from infidex_b200 import synth
from oracle.oracle import Field as OField
from oracle_syn import SynOracleEngine
from parity_util import compare_search, compare_search_batch

pytestmark = pytest.mark.gpu


def _map(pairs):
    m = ib.SynonymMap()
    for a, b in pairs:
        m.AddSynonym(a, b)
    return m


def _surface_queries(pairs, rng, n):
    words = sorted({w for p in pairs for w in p})
    return [" ".join(rng.choice(words, int(rng.integers(1, 3)))) for _ in range(n)]


def _oschema(schema):
    return [OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema]


def test_synthetic_100k_against_oracle_build():
    vocab = synth.make_vocab(100_000)
    docs = synth.gen_docs(100_000, vocab)
    pairs = synth.make_synonym_pairs(vocab, 2000)
    schema, cols = synth.schema_and_columns(docs, False)
    eng = ib.SearchEngine(synonymMap=_map(pairs)); eng.IndexColumns(docs["keys"], schema, cols)
    orc = SynOracleEngine(_oschema(schema), pairs); orc.index_columns(docs["keys"], cols)
    rng = np.random.Generator(np.random.PCG64(7))
    qs = synth.gen_queries(300, docs, vocab) + _surface_queries(pairs, rng, 200)
    bad = compare_search(eng, orc, qs)
    assert not bad, bad[:5]


def test_synthetic_1m_against_oracle_over_image():
    vocab = synth.make_vocab(400_000)
    docs = synth.gen_docs(1_000_000, vocab)
    pairs = synth.make_synonym_pairs(vocab, 5000)
    schema, cols = synth.schema_and_columns(docs, False)
    eng = ib.SearchEngine(synonymMap=_map(pairs)); eng.IndexColumns(docs["keys"], schema, cols)
    orc = SynOracleEngine(_oschema(schema), pairs); orc.load_image(eng.image_ptr())
    rng = np.random.Generator(np.random.PCG64(8))
    qs = synth.gen_queries(1000, docs, vocab) + _surface_queries(pairs, rng, 500)
    qs = [q for q in qs if any(len(w) >= 3 for w in q.split())]      # an image carries no champion lists: short queries are the 100 k test's
    bad = compare_search_batch(eng, orc, qs)
    assert not bad, bad[:5]


def test_multi_field_filter_facets():
    vocab = synth.make_vocab(50_000)
    docs = synth.gen_docs(50_000, vocab, with_description=True)
    pairs = synth.make_synonym_pairs(vocab, 1000)
    schema, cols = synth.schema_and_columns(docs, True)
    eng = ib.SearchEngine(synonymMap=_map(pairs)); eng.IndexColumns(docs["keys"], schema, cols)
    orc = SynOracleEngine(_oschema(schema), pairs); orc.index_columns(docs["keys"], cols)
    rng = np.random.Generator(np.random.PCG64(9))
    qs = synth.gen_queries(150, docs, vocab) + _surface_queries(pairs, rng, 100)
    bad = compare_search(eng, orc, qs, flt=ib.Filter.Parse("year >= 2000 AND rating > 7.0"), facets=True)
    assert not bad, bad[:5]


# k_canon_* at its edges: one thread per document in blocks of 256, so N = 1, 255, 256, 257; empty and delimiter-only documents;
# documents that grow more than 8x (a 2-character key with a long canonical form); the last document of the grid
@pytest.mark.parametrize("n", [1, 255, 256, 257])
def test_k_canon_edges(n):
    pairs = [("zs", "zakladniskola"), ("qq", "queryquestionqualifier"), ("nyc", "new york"), ("Ab", "ABBA")]
    base = ["zs zs zs zs", "", "-- .. //", "qq", "nyc zs", "plain words only", "    ", "x§zs§qq"]
    texts = [base[i % len(base)] for i in range(n)]
    texts[-1] = "zs-qq-zs nyc"                     # the last document, grown more than 8x
    keys = np.arange(1, n + 1, dtype=np.int64)
    eng = ib.SearchEngine(synonymMap=_map(pairs)); eng.IndexDocuments([ib.Document(int(k), t) for k, t in zip(keys, texts)])
    orc = SynOracleEngine(synonyms=pairs); orc.index_columns(keys, [texts])
    bad = compare_search(eng, orc, ["zakladniskola words", "zs qq", "queryquestionqualifier", "new york zs", "plain words", "abba zs"], max_results=50)
    assert not bad, bad[:5]
