"""SearchEngine with a SynonymMap through the kernel emulation against the oracle with the same map (tests/oracle_syn.py): DocumentId order,
Score bits, Tiebreaker bytes, TotalCandidates, facets. Corpora: the 18 books, the movie titles with a map over their words, the school-name
fixture (tests/golden/czech_schools.json) with the school search suite's three pairs, seeded random maps over synthetic documents."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import infidex_b200 as ib
from infidex_b200 import synth
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from oracle_syn import SynOracleEngine
from parity_util import compare_search, emu_lib
from test_book_library import BOOKS, _columns as book_columns, _schema as book_schema
from test_host_builder import _Image, _strings

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SCHOOL_PAIRS = [("zs", "zakladni"), ("ss", "stredni"), ("gympl", "gymnazium")]     # SchoolSearchParityTests.BuildSchoolEngine
WS_QUERIES = ["a b", "x y", " ", "-  -", "§ ", "zs  ss"]                # U+00A0 / U+2003: whitespace the normaliser keeps


def _map(pairs):
    m = ib.SynonymMap()
    for a, b in pairs:
        m.AddSynonym(a, b)
    return m


def _oschema(schema):
    return [OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema]


def _pair(keys, schema, cols, pairs):
    eng = ib.SearchEngine(_gpu_lib=emu_lib(), synonymMap=_map(pairs)); eng.IndexColumns(keys, schema, cols)
    orc = SynOracleEngine(_oschema(schema), pairs); orc.index_columns(keys, cols)
    return eng, orc


def _texts(keys, texts, pairs):
    return _pair(np.asarray(keys, np.int64), [ib.Field("content", None, ib.Weight.Med)], [list(texts)], pairs)


def test_known_answers_car_automobile():
    """Search_WithSynonyms_FindsBothTerms / _WorksBothDirections (SynonymTests.cs), on config 400."""
    eng, orc = _texts([1, 2, 3], ["I drive a car to work", "The automobile industry is growing", "Bicycles are eco-friendly"], [("car", "automobile")])
    for q in ("car", "automobile"):
        keys = [r.DocumentId for r in eng.Search(ib.Query(q, 10)).Records]
        assert 1 in keys and 2 in keys, (q, keys)
    assert not compare_search(eng, orc, ["car", "automobile", "bicycle", "cars", "automobiles"])


def test_school_fixture():
    rows = json.load(open(os.path.join(GOLDEN, "czech_schools.json"), encoding="utf-8"))
    schema = [ib.Field("name", None, ib.Weight.High), ib.Field("city", None, ib.Weight.Low, facetable=True, filterable=True)]
    cols = [[r[1] for r in rows], [r[2] for r in rows]]
    eng, orc = _pair(np.array([r[0] for r in rows], np.int64), schema, cols, SCHOOL_PAIRS)
    qs = ["zs", "ss", "gympl", "zs brno", "základní škola", "zakladni skola brno", "gymnazium", "stredni skola", "ZŠ", "SŠ Pardubice",
          "zs§ss", "gympl olomouc", "skola", "obchodni akademie", "a", "zs ss gympl"] + WS_QUERIES
    assert not compare_search(eng, orc, qs, max_results=20)
    assert not compare_search(eng, orc, qs, max_results=20, facets=True)
    assert not compare_search(eng, orc, qs[:10], max_results=20, flt=ib.Filter.Parse("city = 'Brno' OR city = 'Praha'"), facets=True)
    r = eng.Search(ib.Query("zs", 20))           # a 2-character query whose canonical form is long leaves the short-query path
    assert r.Records and {1, 3, 10, 11, 14} & {x.DocumentId for x in r.Records}


def test_books():
    pairs = [("hp", "harry potter"), ("lotr", "lord of the rings"), ("magic", "sorcery"), ("wizard", "mage")]
    keys = np.array([b[0] for b in BOOKS], np.int64)
    eng, orc = _pair(keys, book_schema(), book_columns(), pairs)
    qs = ["hp", "harry potter", "lotr", "lord rings", "sorcery", "magic school", "mage", "wizard hogwarts", "tolkien", "the"]
    assert not compare_search(eng, orc, qs, max_results=20, facets=True)


def test_movies_with_map(movie_titles):
    rng = np.random.Generator(np.random.PCG64(5))
    words = sorted({w.lower() for t in movie_titles[:3000] for w in t.split() if w.isalpha() and len(w) >= 3})
    pick = [str(w) for w in rng.choice(words, 120, replace=False)]
    pairs = [(pick[i], pick[i + 1]) for i in range(0, 120, 2)] + [("nyc", "new york"), ("lotr", "lord of the rings")]
    titles = movie_titles[:20000]
    eng, orc = _texts(np.arange(len(titles)), titles, pairs)
    qs = pick[:60] + ["nyc", "new york", "lotr", "lord rings", "star wars", "the godfather"]
    bad = compare_search(eng, orc, qs)
    assert not bad, bad[:5]


def test_edge_cases():
    pairs = [("nyc", "new york"), ("zs", "základní"), ("qqq", "neverseenanywhere"), ("colour", "COLOR"), ("x y", "zzz")]
    texts = ["NYC marathon", "New York, New York", "zs Brno§základní škola", "colour of magic", "color television", "nyc§zs§qqq glued",
             "a b c", "non breaking", "", "--", "New York", "nyc nyc nyc nyc"]
    eng, orc = _texts(np.arange(1, len(texts) + 1), texts, pairs)
    qs = ["nyc", "new york", "zs", "základní", "zakladni", "qqq", "neverseenanywhere", "colour", "COLOR tv", "nyc zs qqq", "x y",
          "marathon", "glued"] + WS_QUERIES
    assert not compare_search(eng, orc, qs, max_results=20)
    assert not compare_search(eng, orc, qs, max_results=20, facets=True)


def test_duplicate_document_keys():
    """Segments of one document share a DocumentKey (queries with a word of >= 3 characters: the device flags short queries over such an
    index as unsupported, with or without a map)."""
    pairs = [("nyc", "new york"), ("zs", "zakladni")]
    texts = ["NYC marathon", "New York, New York", "zs Brno", "zakladni skola", "nyc again", "marathon zs"]
    eng, orc = _texts([1, 2, 3, 2, 1, 4], texts, pairs)
    assert not compare_search(eng, orc, ["nyc", "new york", "zakladni", "marathon", "skola zs", "york again"], max_results=20, facets=True)


@pytest.mark.parametrize("seed", range(4))
def test_fuzz_random_maps(seed):
    rng = np.random.Generator(np.random.PCG64(100 + seed))
    vocab = synth.make_vocab(3000, seed=seed)
    docs = synth.gen_docs(3000, vocab, seed=seed, with_description=seed % 2 == 1)
    schema, cols = synth.schema_and_columns(docs, seed % 2 == 1)
    pairs = synth.make_synonym_pairs(vocab, 300, seed=seed, n_frequent=20)
    pairs += [(str(rng.choice(vocab["words"])), "%s %s" % tuple(rng.choice(vocab["words"], 2))) for _ in range(10)]   # multi-word canonicals
    eng, orc = _pair(docs["keys"], schema, cols, pairs)
    words = sorted({w for p in pairs for w in p})
    qs = synth.gen_queries(100, docs, vocab, seed=seed) + [" ".join(rng.choice(words, int(rng.integers(1, 3)))) for _ in range(100)]
    bad = compare_search(eng, orc, qs)
    assert not bad, bad[:5]
    if seed % 2:
        bad = compare_search(eng, orc, qs[:80], flt=ib.Filter.Parse("year >= 2000 AND rating > 7.0"), facets=True)
        assert not bad, bad[:5]


def _image_arrays(eng):
    img = C.cast(eng.image_ptr(), C.POINTER(_Image)).contents
    n, T = img.n_docs, img.terms.n
    P = int(np.ctypeslib.as_array(img.row_ptr, shape=(T + 1,))[T])
    return {"text": np.ctypeslib.as_array(img.text_chars, shape=(max(int(img.text_off[n]), 1),)).copy(),
            "terms": [_strings(img.terms, t) for t in range(T)], "df": np.ctypeslib.as_array(img.df, shape=(T,)).copy(),
            "post_doc": np.ctypeslib.as_array(img.post_doc, shape=(max(P, 1),)).copy(), "post_tf": np.ctypeslib.as_array(img.post_tf, shape=(max(P, 1),)).copy(),
            "doc_len": np.ctypeslib.as_array(img.doc_len, shape=(n,)).copy(), "first_token": [_strings(img.first_token, d) for d in range(n)],
            "token_count": np.ctypeslib.as_array(img.token_count, shape=(n,)).copy(), "words": [_strings(img.words, i) for i in range(img.words.n)],
            "word_idf": np.ctypeslib.as_array(img.word_idf, shape=(max(img.words.n, 1),)).copy()}


def test_empty_map_is_no_map():
    vocab = synth.make_vocab(2000); docs = synth.gen_docs(2000, vocab, with_description=True)
    schema, cols = synth.schema_and_columns(docs, True)
    plain = ib.SearchEngine(_gpu_lib=emu_lib()); plain.IndexColumns(docs["keys"], schema, cols)
    empty = ib.SearchEngine(_gpu_lib=emu_lib(), synonymMap=ib.SynonymMap()); empty.IndexColumns(docs["keys"], schema, cols)
    a, b = _image_arrays(plain), _image_arrays(empty)
    for k in a:
        assert (np.array_equal(a[k], b[k]) if isinstance(a[k], np.ndarray) else a[k] == b[k]), k
    qs = synth.gen_queries(100, docs, vocab) + ["a", "zz"]
    ra, rb = plain.SearchBatch([ib.Query(q, 10) for q in qs]), empty.SearchBatch([ib.Query(q, 10) for q in qs])
    for x, y in zip(ra, rb):
        assert [(r.DocumentId, np.float32(r.Score).view(np.uint32), r.Tiebreaker) for r in x.Records] == \
               [(r.DocumentId, np.float32(r.Score).view(np.uint32), r.Tiebreaker) for r in y.Records] and x.TotalCandidates == y.TotalCandidates
    orc = OracleEngine(_oschema(schema)); orc.index_columns(docs["keys"], cols)
    assert not compare_search(empty, orc, qs[:50])


def test_wordmatcher_and_word_idf_read_the_raw_text():
    """WordMatcher and the word-idf cache are built from the text as it is; the index text, the metadata and the coverage text are not."""
    texts = ["nyc lights", "car wash", "automobile club"]
    pairs = [("nyc", "new york"), ("car", "automobile")]
    eng, orc = _texts([1, 2, 3], texts, pairs)
    plain = ib.SearchEngine(_gpu_lib=emu_lib()); plain.IndexDocuments([ib.Document(k, t) for k, t in zip([1, 2, 3], texts)])
    a, b = _image_arrays(plain), _image_arrays(eng)
    assert a["words"] == b["words"] and np.array_equal(a["word_idf"], b["word_idf"]) and np.array_equal(a["text"], b["text"])
    assert "york" in b["terms"] and "york" not in a["terms"] and "nyc" not in b["terms"]
    assert b["first_token"] == ["new", "automobile", "automobile"] and list(b["token_count"]) == [3, 2, 2]
    assert orc.word_idf("york") == -1.0 and orc.word_idf("nyc") > 0        # a canonical form in no raw text has no word idf
    assert not compare_search(eng, orc, ["new york", "york", "nyc", "car", "club automobile"])


def test_multi_field_tf_bytes_match_the_oracle():
    """Field weights are looked up by token position in the canonical text against the boundaries of the raw concatenation: tf bytes
    shift when the canonical forms change lengths."""
    schema = [ib.Field("title", None, ib.Weight.High), ib.Field("body", None, ib.Weight.Low)]
    titles = ["nyc zs", "a b c d e f", "zs"]; bodies = ["zs zs nyc", "nyc", "long body words here nyc"]
    pairs = [("nyc", "new york city"), ("zs", "zakladniskola")]
    eng, orc = _pair(np.array([1, 2, 3], np.int64), schema, [titles, bodies], pairs)
    b = _image_arrays(eng); img = C.cast(eng.image_ptr(), C.POINTER(_Image)).contents
    row = np.ctypeslib.as_array(img.row_ptr, shape=(img.terms.n + 1,))
    assert len(b["terms"]) == orc.num_terms()
    for t in range(len(b["terms"])):
        text, df, docs, w = orc.term(t)
        assert b["terms"][t] == text and int(b["df"][t]) == df
        assert np.array_equal(b["post_doc"][row[t]:row[t + 1]], docs) and np.array_equal(b["post_tf"][row[t]:row[t + 1]], w), text
    assert not compare_search(eng, orc, ["nyc", "zs", "new york city", "zakladniskola body", "words"])


def test_changing_the_map_after_indexing_raises():
    m = _map([("car", "automobile")])
    eng = ib.SearchEngine(_gpu_lib=emu_lib(), synonymMap=m)
    eng.IndexDocuments([ib.Document(1, "car"), ib.Document(2, "automobile")])
    assert eng.SynonymMap is m and eng.Search("car").Records
    m.AddSynonym("bike", "bicycle")
    with pytest.raises(RuntimeError):
        eng.Search("car")
    eng.IndexDocuments([ib.Document(1, "car"), ib.Document(2, "bike")])      # indexing again takes the new map
    assert eng.Search("bicycle").Records
    m.Clear()
    with pytest.raises(RuntimeError):
        eng.Search("car")
    e2 = ib.SearchEngine(_gpu_lib=emu_lib(), synonymMap=ib.SynonymMap())     # a map that gains its first mapping after indexing
    e2.IndexDocuments([ib.Document(1, "car")]); e2.SynonymMap.AddSynonym("car", "auto")
    with pytest.raises(RuntimeError):
        e2.Search("car")
