"""Short queries (no word of >= 3 characters) on doc-id-range shards.

The champion exchange at build time: the global lists of 2 and 3 shard builders, mapped to global ids, equal the unsharded builder's lists.
The search path on CPU: two processes (gloo, world size 2), each holding one shard (kernel emulation build), against the unsharded oracle
built from its own index: ids, score bits, tiebreakers, TotalCandidates and status (a shard's batch carries no facet tables)."""
import ctypes as C
import os

import numpy as np
import pytest

import infidex_b200 as ib
from infidex_b200 import synth
from infidex_b200.engine import Field, Weight

import short_shard_util as U
from dist_util import run_ranks, spawn_gloo


class _Strings(C.Structure):
    _fields_ = [("chars", C.POINTER(C.c_uint16)), ("off", C.POINTER(C.c_uint32)), ("n", C.c_int32)]


class _Docset(C.Structure):
    _fields_ = [("keys", _Strings), ("row_ptr", C.POINTER(C.c_int64)), ("doc_id", C.POINTER(C.c_int32))]


class _Image(C.Structure):      # include/infidex_gpu.h: ifx_index_image up to the champion lists
    _fields_ = [("n_docs", C.c_int32), ("n_live", C.c_int32), ("avgdl", C.c_float),
                ("doc_key", C.c_void_p), ("deleted", C.c_void_p), ("doc_len", C.c_void_p), ("text_chars", C.c_void_p), ("text_off", C.c_void_p),
                ("first_token", _Strings), ("token_count", C.c_void_p), ("terms", _Strings), ("df", C.c_void_p), ("row_ptr", C.c_void_p),
                ("post_doc", C.c_void_p), ("post_tf", C.c_void_p), ("words", _Strings), ("word_idf", C.c_void_p),
                ("prefix", _Docset), ("wm_exact", _Docset), ("wm_ld1", _Docset), ("affix_words", _Strings), ("affix_last_doc", C.c_void_p),
                ("n_columns", C.c_int32), ("columns", C.c_void_p),
                ("n_champ_chars", C.c_int32), ("champ_chars", C.POINTER(C.c_uint16)), ("champ_off", C.POINTER(C.c_int32)),
                ("champ_doc", C.POINTER(C.c_int32)), ("champ_score", C.POINTER(C.c_float))]


def _champions(eng):
    img = C.cast(eng.image_ptr(), C.POINTER(_Image)).contents
    nc = img.n_champ_chars; off = np.ctypeslib.as_array(img.champ_off, shape=(nc + 1,)).copy(); ne = int(off[nc])
    chars = np.ctypeslib.as_array(img.champ_chars, shape=(max(nc, 1),))[:nc].copy()
    doc = np.ctypeslib.as_array(img.champ_doc, shape=(max(ne, 1),))[:ne].copy(); score = np.ctypeslib.as_array(img.champ_score, shape=(max(ne, 1),))[:ne].copy()
    return {int(chars[i]): (doc[off[i]:off[i + 1]], score[off[i]:off[i + 1]]) for i in range(nc)}


def _tie_corpus():
    """Synthetic titles plus runs of identical titles (equal champion scores) straddling the shard cuts used below."""
    vocab = synth.make_vocab(5_000); n = 9_000
    docs = synth.gen_docs(n, vocab); blob, off = docs["title"]
    titles = [blob[int(off[i]): int(off[i + 1])].tobytes().decode("utf-16-le") for i in range(n)]
    for c0, texts in [(2_950, ["жук", "жук лес", "x жук", "ж"]), (5_980, ["щит", "щит стал", "a щит"])]:
        for i in range(90):
            titles[c0 + i] = texts[(i * 7) % len(texts)] if i % 3 else texts[0]
    for i in range(0, n, 97):
        titles[i] = "ёж " + titles[i]
    return np.arange(n, dtype=np.int64) + 10, titles


@pytest.mark.parametrize("cuts", [[3_000], [3_000, 6_000], [2_980, 6_010]])
def test_globalized_champions_equal_the_unsharded_lists(cuts):
    from infidex_b200.dist import exchange_builder
    keys, titles = _tie_corpus(); n = len(keys)
    schema = [Field("title", None, Weight.High)]
    whole = ib.SearchEngine(); whole.IndexColumns(keys, schema, [titles], upload=False)
    want = _champions(whole)
    bounds = [0] + cuts + [n]; W = len(bounds) - 1
    shards = []
    for s in range(W):
        e = ib.SearchEngine(); e.IndexColumns(keys[bounds[s]:bounds[s + 1]], schema, [titles[bounds[s]:bounds[s + 1]]], upload=False); shards.append(e)
    run_ranks(W, lambda d, s: exchange_builder(d, shards[s], "ifx_builder_export_champions", "ifx_builder_globalize_champions"))
    got = [_champions(e) for e in shards]
    tied = 0
    for ch, (doc, score) in want.items():
        glob = np.full(len(doc), -1, np.int64)
        for s in range(W):
            d, sc = got[s][ch]
            assert len(d) == len(doc) and np.array_equal(sc.view(np.uint32), score.view(np.uint32)), chr(ch)
            own = d >= 0; assert (glob[own] < 0).all(); glob[own] = d[own] + bounds[s]
        assert np.array_equal(glob, doc), chr(ch)
        tied += len(doc) == 64 and len(np.unique(score)) < 8
    assert tied >= 2      # the tie-heavy characters were in play
    for s in range(W):
        assert set(got[s]) == set(want)


def _worker(rank, world, emu, outdir):
    import pickle
    import torch.distributed as dist
    from infidex_b200 import dist as ifxd
    keys, schema, cols, vocab = U.corpus()
    lo, hi = ifxd.shard_ranges(U.N, world)[rank]
    eng = ifxd.ShardedSearchEngine(dist, _gpu_lib=emu)
    eng.IndexShard(keys[lo:hi], schema, [cols[0][lo:hi], cols[1][lo:hi]], threads=2)
    ngram = [ib.Query(t, 10) for t in U.ngram_texts(vocab)]
    alone = [U.signature(r) for r in eng.SearchBatch(ngram)]                                   # no short query: the parent's path
    mixed = [U.signature(r) for r in eng.SearchBatch([U.make_query(c) for c in U.SHORT_CASES] + ngram)]
    counts = [c.cpu().numpy() for c in eng.last_s1_counts]; info = eng.last_shard_info.cpu().numpy()
    eng.Close()
    if rank == 0:
        pickle.dump({"alone": alone, "mixed": mixed, "counts": counts, "info": info}, open(os.path.join(outdir, "out.pkl"), "wb"))


def test_two_shards_answer_short_queries_as_the_unsharded_oracle(tmp_path):
    import pickle
    from parity_util import emu_lib
    spawn_gloo(_worker, 2, emu_lib(), str(tmp_path))
    out = pickle.load(open(tmp_path / "out.pkl", "rb"))
    ns = len(U.SHORT_CASES)
    assert out["mixed"][ns:] == out["alone"]                    # the n-gram queries of a mixed batch are untouched
    U.check_shard_facts(U.SHORT_CASES, out["counts"], out["info"])
    keys, schema, cols, _ = U.corpus()
    bad = U.compare_with_oracle(U.oracle_engine(keys, schema, cols), U.SHORT_CASES, out["mixed"][:ns])
    assert not bad, bad
