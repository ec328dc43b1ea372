"""The host index builder with a SynonymMap against the oracle's index with the same map, structure by structure: term dictionary in
TermCollection order, df, posting lists with their tf bytes (the field-weight shift of multi-field documents), document lengths, prefix
docsets; the word-idf cache and the document text equal to the builder's image WITHOUT a map (they read the raw text; WordMatcher's
dictionaries do too, checked through search parity in test_emu_synonyms.py). No GPU involved."""
import ctypes as C

import numpy as np
import pytest

import infidex_b200 as ib
from infidex_b200 import synth
from oracle.oracle import Field as OField
from oracle_syn import SynOracleEngine
from parity_util import emu_lib
from test_host_builder import _Image, _strings


@pytest.mark.parametrize("multi", [False, True])
def test_image_with_map_matches_oracle_index(multi):
    vocab = synth.make_vocab(20_000)
    docs = synth.gen_docs(4_000, vocab, with_description=multi)
    schema, cols = synth.schema_and_columns(docs, multi)
    pairs = synth.make_synonym_pairs(vocab, 800, n_frequent=40) + [(vocab["words"][3], "%s %s" % (vocab["words"][5], vocab["words"][7]))]
    m = ib.SynonymMap()
    for a, b in pairs:
        m.AddSynonym(a, b)
    eng = ib.SearchEngine(_gpu_lib=emu_lib(), synonymMap=m); eng.IndexColumns(docs["keys"], schema, cols, upload=False)
    plain = ib.SearchEngine(_gpu_lib=emu_lib()); plain.IndexColumns(docs["keys"], schema, cols, upload=False)
    orc = SynOracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema], pairs); orc.index_columns(docs["keys"], cols)
    img = C.cast(eng.image_ptr(), C.POINTER(_Image)).contents; pim = C.cast(plain.image_ptr(), C.POINTER(_Image)).contents
    n = img.n_docs
    assert np.float32(img.avgdl).view(np.uint32) == np.float32(orc.avgdl()).view(np.uint32)
    assert np.array_equal(np.ctypeslib.as_array(img.doc_len, shape=(n,)).view(np.uint32), orc.doc_lens().view(np.uint32))
    T = img.terms.n
    assert T == orc.num_terms()
    row = np.ctypeslib.as_array(img.row_ptr, shape=(T + 1,)); P = int(row[T])
    pd = np.ctypeslib.as_array(img.post_doc, shape=(max(P, 1),)); pt = np.ctypeslib.as_array(img.post_tf, shape=(max(P, 1),))
    df = np.ctypeslib.as_array(img.df, shape=(T,))
    rng = np.random.Generator(np.random.PCG64(12))
    for t in list(range(min(T, 300))) + rng.integers(0, T, 700).tolist():
        text, odf, odocs, ow = orc.term(int(t))
        assert _strings(img.terms, t) == text and int(df[t]) == odf, (t, text)
        a, b = int(row[t]), int(row[t + 1])
        assert np.array_equal(pd[a:b], odocs) and np.array_equal(pt[a:b], ow), (t, text)
    pk = img.prefix.keys; prow = np.ctypeslib.as_array(img.prefix.row_ptr, shape=(pk.n + 1,))
    pdoc = np.ctypeslib.as_array(img.prefix.doc_id, shape=(max(int(prow[pk.n]), 1),))
    for k in list(range(min(pk.n, 200))) + rng.integers(0, pk.n, 300).tolist():
        assert pdoc[prow[k]:prow[k + 1]].tolist() == orc.dict_docs(0, _strings(pk, int(k))), _strings(pk, int(k))
    # the word-idf cache and the document text are those of the raw text
    assert [_strings(img.words, i) for i in range(img.words.n)] == [_strings(pim.words, i) for i in range(pim.words.n)]
    assert np.array_equal(np.ctypeslib.as_array(img.word_idf, shape=(img.words.n,)), np.ctypeslib.as_array(pim.word_idf, shape=(pim.words.n,)))
    assert np.array_equal(np.ctypeslib.as_array(img.text_chars, shape=(int(img.text_off[n]),)), np.ctypeslib.as_array(pim.text_chars, shape=(int(pim.text_off[n]),)))
