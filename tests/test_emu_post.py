"""Query boosts and SortBy (ResultProcessor.ApplyBoosts / ApplySort): hand-written known answers on the 18-book library, the kernel
emulation against the oracle on tie-heavy and random cases, the three restatements of .NET's introsort against each other, and the
rejections. The `-m gpu` twin is tests/test_gpu_post.py."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import infidex_b200 as ib
import oracle_post
from infidex_b200 import synth
from oracle import oracle as O
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from parity_util import build_pair, emu_lib
from post_util import compare_post, make_query, random_posts

HERE = os.path.dirname(os.path.abspath(__file__))
BOOKS = json.load(open(os.path.join(HERE, "golden", "books.json"), encoding="utf-8"))
F = ib.Filter


@pytest.fixture(scope="module")
def emu():
    return emu_lib()


def _book_schema():
    return [ib.Field("title", None, ib.Weight.High), ib.Field("author", None, ib.Weight.Med, facetable=True),
            ib.Field("year", None, ib.Weight.Low, indexable=False, facetable=True, sortable=True),
            ib.Field("genre", None, ib.Weight.Low, filterable=True, facetable=True), ib.Field("description", None, ib.Weight.Med)]


def _book_columns():
    return [[b[1] for b in BOOKS], [b[2] for b in BOOKS], np.array([int(b[3]) for b in BOOKS], np.int64), [b[4] for b in BOOKS], [b[5] for b in BOOKS]]


@pytest.fixture(scope="module")
def books(emu):
    keys = np.array([b[0] for b in BOOKS], np.int64)
    return build_pair(keys, _book_schema(), _book_columns(), gpu_lib=emu)


def _recs(r):
    return [(e.DocumentId, np.float32(e.Score)) for e in r.Records]


def _book(k):
    return next(b for b in BOOKS if b[0] == k)


QUERIES = ["harry potter", "the", "lord", "wizard", "king"]


def test_boost_adds_strength_once_in_float32_and_sums(books):
    """Score + (int)BoostStrength, one float32 add per record; several matching boosts add up; then a stable re-sort by score (<= 16 records)."""
    eng, orc = books
    boosts = [(F.Parse("genre = 'Fantasy'"), ib.BoostStrength.High), (F.Parse("year >= 1998"), ib.BoostStrength.Low), (F.Parse("author = 'J.R.R. Tolkien'"), ib.BoostStrength.Med)]
    for q in QUERIES:
        base = _recs(eng.Search(make_query(q, 10)))
        assert len(base) <= 16
        want = []
        for k, s in base:
            b = _book(k); total = (3 if b[4] == "Fantasy" else 0) + (1 if int(b[3]) >= 1998 else 0) + (2 if b[2] == "J.R.R. Tolkien" else 0)
            want.append((k, np.float32(s + np.float32(total)) if total > 0 else s))
        want = sorted(want, key=lambda t: -t[1])           # Python's sort is stable, like .NET's insertion sort for n <= 16
        got = _recs(eng.Search(make_query(q, 10, boosts=boosts)))
        assert [k for k, _ in got] == [k for k, _ in want], q
        assert np.array_equal(np.array([s for _, s in got], np.float32).view(np.uint32), np.array([s for _, s in want], np.float32).view(np.uint32)), q
    bad, over = compare_post(eng, orc, QUERIES, boosts=boosts)
    assert not bad and not over, bad[:3]


def test_boost_matching_nothing_keeps_the_list(books):
    eng, orc = books
    for q in QUERIES:
        base = _recs(eng.Search(make_query(q, 10)))
        got = _recs(eng.Search(make_query(q, 10, boosts=[(F.Parse("genre = 'Cookbook'"), ib.BoostStrength.High)])))
        assert got == base, q
    assert compare_post(eng, orc, QUERIES, boosts=[(F.Parse("genre = 'Cookbook'"), 3)]) == ([], [])


@pytest.mark.parametrize("ascending", [True, False])
def test_sort_by_year(books, ascending):
    eng, orc = books
    for q in QUERIES:
        base = _recs(eng.Search(make_query(q, 10)))
        want = sorted(base, key=lambda t: int(_book(t[0])[3]), reverse=not ascending)
        if not ascending:      # a stable descending sort keeps equal years in their original order
            want = sorted(base, key=lambda t: -int(_book(t[0])[3]))
        got = _recs(eng.Search(make_query(q, 10, sort=("year", ascending))))
        assert got == want, (q, got, want)
    assert compare_post(eng, orc, QUERIES, sort=("year", ascending)) == ([], [])


def test_sort_with_null_values_first_or_last(emu):
    """Books 1-9 carry a year, books 10-18 have none (null): ascending puts the nulls first, descending last."""
    keys = np.array([b[0] for b in BOOKS], np.int64)
    cols = _book_columns(); h = 9
    chunk = lambda a, b: [c[a:b] if c is not None else None for c in cols]
    first, second = chunk(0, h), chunk(h, len(BOOKS)); second[2] = None
    eng = ib.SearchEngine(_gpu_lib=emu); eng.IndexChunks(_book_schema(), [(keys[:h], first), (keys[h:], second)])
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in _book_schema()])
    L = O.lib()
    for ks, cc in ((keys[:h], first), (keys[h:], second)):       # two add_docs calls, one build: the second has no year column (kind 0)
        kinds = np.zeros(len(cc), np.int32); cp, op, keep = (C.c_void_p * len(cc))(), (C.c_void_p * len(cc))(), []
        for i, col in enumerate(cc):
            if col is None:
                continue
            if isinstance(col, np.ndarray):
                a = np.ascontiguousarray(col, np.int64); kinds[i] = 2; cp[i] = a.ctypes.data; keep.append(a)
            else:
                blob, o = O.pack_strings(col); kinds[i] = 1; cp[i] = blob.ctypes.data; op[i] = o.ctypes.data; keep += [blob, o]
        ka = np.ascontiguousarray(ks, np.int64); L.ifxo_add_docs(orc.h, len(ks), O._p(ka), O._p(kinds), cp, op)
    L.ifxo_build(orc.h)
    for asc in (True, False):
        for q in ("the", "harry", "lord king"):
            got = _recs(eng.Search(make_query(q, 10, sort=("year", asc))))
            years = [int(_book(k)[3]) if k <= h else None for k, _ in got]
            nulls = [y is None for y in years]
            assert nulls == sorted(nulls, reverse=asc), (q, asc, years)
        assert compare_post(eng, orc, ["the", "harry", "lord king", "of"], sort=("year", asc)) == ([], [])


def test_filter_boost_sort_leave_facets_and_total(books):
    eng, orc = books
    flt = F.Parse("genre != 'Science Fiction'")
    boosts = [(F.Parse("year < 1960"), ib.BoostStrength.High)]
    for q in QUERIES:
        plain = eng.Search(make_query(q, 3, flt=flt, facets=True))
        post = eng.Search(make_query(q, 3, flt=flt, facets=True, boosts=boosts, sort=("genre", False)))
        assert post.TotalCandidates == plain.TotalCandidates and post.Facets == plain.Facets, q
    bad, over = compare_post(eng, orc, QUERIES, max_results=3, flt=flt, facets=True, boosts=boosts, sort=("genre", False))
    assert not bad and not over, bad[:3]


def test_sort_on_a_field_no_document_has(books):
    """Every value null: the sort still runs (a no-op below 17 records); ordinal, case-sensitive name match ('Year' is not 'year')."""
    eng, orc = books
    for name in ("publisher", "Year"):
        for q in QUERIES:
            assert _recs(eng.Search(make_query(q, 10, sort=(name, True)))) == _recs(eng.Search(make_query(q, 10)))
        assert compare_post(eng, orc, QUERIES, sort=(name, True)) == ([], [])


def test_twenty_identical_documents_tie_order(emu):
    """Every score ties: above 16 records the introsort's partitioning decides the order, for a boost that matches nobody and for a
    sort over one value."""
    texts = ["batman saves the day"] * 20; tags = ["x"] * 20
    schema = [ib.Field("content"), ib.Field("tag", None, ib.Weight.Med, indexable=False, filterable=True)]
    eng, orc = build_pair(np.arange(20), schema, [texts, tags], gpu_lib=emu)
    qs = ["batman", "saves the day", "batmen"]
    for mr in (20, 50):
        for boosts, sort in (([(F.Parse("tag = 'nobody'"), 3)], None), (None, ("tag", True)), ([(F.Parse("tag = 'x'"), 1)], ("tag", False))):
            bad, over = compare_post(eng, orc, qs, max_results=mr, boosts=boosts, sort=sort)
            assert not bad and not over, (mr, boosts, sort, bad[:2])
        assert [e.DocumentId for e in eng.Search(make_query("batman", mr, boosts=[(F.Parse("tag = 'nobody'"), 3)])).Records] != \
            [e.DocumentId for e in eng.Search(make_query("batman", mr)).Records]       # the unstable sort reorders equal scores


@pytest.fixture(scope="module")
def multi(emu):
    vocab = synth.make_vocab(20_000)
    docs = synth.gen_docs(12_000, vocab, with_description=True)
    schema, cols = synth.schema_and_columns(docs, True)
    eng, orc = build_pair(docs["keys"], schema, cols, gpu_lib=emu)
    return eng, orc, synth.gen_queries(60, docs, vocab)


def test_sort_decides_what_is_taken(multi):
    """Coverage off and the Stage-1 fallback return up to CoverageDepth records: the boosts and the sort pick the ten that survive Take;
    sort on the 20-value genre column over hundreds of records (tie-heavy), on int64 year and float64 rating."""
    eng, orc, qs = multi
    for cov in (False, True):
        for boosts, sort in ((None, ("genre", True)), (None, ("year", False)), (None, ("rating", True)),
                             ([(F.Parse("genre = 'drama'"), 3), (F.Parse("year >= 2015"), 1)], ("rating", False)),
                             ([(F.Parse("rating > 8.0"), 2)], None)):
            bad, over = compare_post(eng, orc, qs[:30], max_results=10, depth=500, coverage=cov, boosts=boosts, sort=sort)
            assert not bad and not over, (cov, boosts, sort, bad[:2])


def test_random_mixes(multi):
    eng, orc, qs = multi
    rng = np.random.Generator(np.random.PCG64(11))
    filters = [F.Parse("genre = 'drama'"), F.Parse("year >= 2015"), F.Parse("rating > 7.5"), F.Parse("genre IN ('comedy', 'horror')"), F.Parse("year < 1990")]
    flt = F.Parse("year >= 2000 AND rating > 7.0")
    short = ["a", "th", "x", "zz"]
    for i, (boosts, sort) in enumerate(random_posts(rng, 12, filters, ["genre", "year", "rating", "nonexistent"])):
        mr = (10, 100)[i % 2]; cov = i % 3 != 0; f = flt if i % 4 == 1 else None
        bad, over = compare_post(eng, orc, qs[i * 4:i * 4 + 12] + short + [""], max_results=mr, flt=f, facets=i % 2 == 0, coverage=cov, boosts=boosts, sort=sort)
        assert not bad, (i, boosts, sort, bad[:2])
        assert set(over) <= set(short), over          # only the short-query path can hold a part of its list


def test_blank_query_with_facets_ignores_boosts_and_sort(multi):
    eng, orc, _ = multi
    plain = eng.Search(make_query("", 20, facets=True))
    post = eng.Search(make_query("", 20, facets=True, boosts=[(F.Parse("genre = 'drama'"), 3)], sort=("rating", True)))
    assert _recs(post) == _recs(plain) and post.Facets == plain.Facets
    assert compare_post(eng, orc, [""], 20, facets=True, boosts=[(F.Parse("genre = 'drama'"), 3)], sort=("rating", True)) == ([], [])


def test_rejections(books, emu):
    eng, orc = books
    r = eng.Search(make_query("harry", 10, boosts=[(F.Parse("genre MATCHES 'F.*'"), 2)]))
    assert r.Status & 2                                             # MATCHES inside a boost: unsupported, never answered partially
    x = oracle_post.search(orc, "harry", 10, boosts=[(F.Parse("genre MATCHES 'F.*'").bytecode(), 2)])
    assert x["status"] != 0
    with pytest.raises(ValueError):                                 # a schema field without a device column
        eng.Search(make_query("harry", 10, sort=("title", True)))
    with pytest.raises(ValueError):
        eng.Search(make_query("harry", 10, boosts=[(F.Parse("description = 'x'"), 1)]))
    with pytest.raises(ValueError):
        eng.Search(make_query("harry", 10, boosts=[(F.Parse("genre = 'Fantasy'"), 1)] * 17))
    # the C-ABI validates what the mirror cannot: an order of the wrong size, a sort on a column without an order, an unknown boost filter
    g = eng._gpu; rank = np.zeros(3, np.int32)
    assert g.ifx_column_set_order(eng._index, 0, rank.ctypes.data_as(C.c_void_p), 3) != 0
    assert g.ifx_column_set_order(eng._index, 99, rank.ctypes.data_as(C.c_void_p), 3) != 0
    arr, keep = eng._pack_queries([ib.Query("harry", 10)])
    post = (ib.engine._QueryPost * 1)(); post[0].sort_column = eng._columns.index("genre"); post[0].n_boosts = 0
    fresh = ib.SearchEngine(_gpu_lib=emu); fresh.IndexColumns(np.array([b[0] for b in BOOKS], np.int64), _book_schema(), _book_columns())
    arr2, keep2 = fresh._pack_queries([ib.Query("harry", 10)])
    packed = fresh.PackBatch([ib.Query("harry", 10)])
    assert fresh._gpu.ifx_search_batch_post(fresh._index, arr2, post, 1, C.byref(packed["out"]), None) != 0      # no order registered
    post[0].sort_column = -1; post[0].n_boosts = 1; post[0].boost_filter[0] = 57
    assert fresh._gpu.ifx_search_batch_post(fresh._index, arr2, post, 1, C.byref(packed["out"]), None) == 0
    assert packed["bufs"]["status"][0] & 2                          # unknown boost filter id: like an unknown filter_id
    post[0].n_boosts = 17
    assert fresh._gpu.ifx_search_batch_post(fresh._index, arr2, post, 1, C.byref(packed["out"]), None) != 0


def test_host_builder_column_order(emu):
    """CompareValues ranks: int64 exact beyond 2**53, doubles numerically, strings ordinally; mixed runtime types have no order."""
    big = 2 ** 53
    ints = np.array([big + 1, big, -5, big + 1, 0], np.int64)
    dbl = np.array([2.5, -0.0, 0.0, 10.0, -1e300], np.float64)
    strs = ["b", "B", "a", "", "b"]
    schema = [ib.Field("content"), ib.Field("i", None, indexable=False, sortable=True), ib.Field("d", None, indexable=False, sortable=True),
              ib.Field("s", None, indexable=False, sortable=True)]
    eng = ib.SearchEngine(_gpu_lib=emu); eng.IndexColumns(np.arange(5), schema, [["x"] * 5, ints, dbl, strs])
    b = C.c_void_p(eng._builder); h = eng._host

    def ranks(c):
        n = h.ifx_builder_column_dict_size(b, c); r = np.zeros(n, np.int32); assert h.ifx_builder_column_order(b, c, r.ctypes.data_as(C.c_void_p)) == 0
        vals = [eng._facet_value(c, i) for i in range(n)]
        return dict(zip(vals, r.tolist()))
    ri = ranks(eng._columns.index("i")); assert ri[str(-5)] < ri["0"] < ri[str(big)] < ri[str(big + 1)]
    rd = ranks(eng._columns.index("d")); assert rd["-1e+300"] < rd["-0"] == rd["0"] < rd["2.5"] < rd["10"]
    rs = ranks(eng._columns.index("s")); assert rs[""] < rs["B"] < rs["a"] < rs["b"]
    mixed = ib.SearchEngine(_gpu_lib=emu)
    mixed.IndexChunks([ib.Field("content"), ib.Field("v", None, indexable=False, sortable=True)],
                      [(np.arange(2), [["x", "y"], np.array([1, 2], np.int64)]), (np.arange(2, 4), [["z", "w"], ["a", "b"]])])
    with pytest.raises(ValueError):
        mixed.Search(make_query("x", 10, sort=("v", True)))


def _shard_worker(rank, world, port, emu, outdir):
    import pickle
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from infidex_b200 import dist as ifxd
    N = 140_000; vocab = synth.make_vocab(20_000)
    lo, hi = ifxd.shard_ranges(N, world)[rank]
    docs = synth.gen_docs(hi - lo, vocab, with_description=True, start=lo)
    schema, cols = synth.schema_and_columns(docs, True)
    eng = ifxd.ShardedSearchEngine(dist, _gpu_lib=emu); eng.IndexShard(docs["keys"], schema, cols, threads=2)
    qs = synth.gen_queries(6, synth.corpus_ref(N), vocab)
    plain = eng.SearchBatch([make_query(q) for q in qs])
    boosted = eng.SearchBatch([make_query(q, boosts=[(F.Parse("genre = 'drama'"), 3)]) for q in qs])
    sorted_ = eng.SearchBatch([make_query(q, sort=("rating", False)) for q in qs[:3]] + [make_query(q) for q in qs[3:]])
    again = eng.SearchBatch([make_query(q) for q in qs])          # the refilled handle no longer carries the post-processing
    eng.Close()
    if rank == 0:
        st = lambda rr: [r.Status for r in rr]
        pickle.dump((st(plain), st(boosted), st(sorted_), st(again)), open(os.path.join(outdir, "status.pkl"), "wb"))
    dist.barrier(); dist.destroy_process_group()


def test_sharded_index_flags_boosts_and_sort(tmp_path, emu):
    """Post-processing belongs after the hosts' merge of the shards, which is not built: on a 2-shard (gloo) index a query with boosts or a
    SortBy carries IFX_Q_UNSUPPORTED_OP; the others in the same batch do not."""
    import pickle
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    mp.spawn(_shard_worker, args=(2, port, emu, str(tmp_path)), nprocs=2, join=True)
    plain, boosted, sorted_, again = pickle.load(open(tmp_path / "status.pkl", "rb"))
    assert not any(x & 2 for x in plain) and not any(x & 2 for x in again)
    assert all(x & 2 for x in boosted)
    assert all(x & 2 for x in sorted_[:3]) and not any(x & 2 for x in sorted_[3:])


def _harness(tmp_path, src):
    exe = str(tmp_path / ("introsort_%d" % src))
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-DSRC=%d" % src, "-o", exe, os.path.join(HERE, "introsort_harness.cpp")])
    return exe


def test_introsort_restatements_agree(tmp_path):
    """The device's IntroSort (emulation build), the host builder's DotnetIntroSort and the oracle's DotnetSort give the same permutation
    on tie-heavy arrays, n = 2..1024 (insertion sort, median-of-three partitions, the heapsort fallback at the depth limit)."""
    exes = [_harness(tmp_path, s) for s in (1, 2, 3)]
    rng = np.random.Generator(np.random.PCG64(5))
    sizes = list(range(2, 40)) + [63, 64, 65, 100, 127, 128, 200, 255, 256, 500, 511, 512, 777, 1000, 1023, 1024]
    for n in sizes:
        for distinct in (1, 2, 3, 7, n):
            vals = rng.integers(0, distinct, n)
            if distinct == n and n % 3 == 0:
                vals = np.sort(vals)[::-1].copy()                 # descending runs: degenerate pivots -> heapsort
            inp = ("%d\n" % n + " ".join(str(int(v)) for v in vals) + "\n").encode()
            outs = [subprocess.run([e], input=inp, capture_output=True, check=True).stdout for e in exes]
            assert outs[0] == outs[1] == outs[2], (n, distinct)
            perm = [int(x) for x in outs[0].split()]
            assert sorted(perm) == list(range(n)) and all(vals[perm[i]] <= vals[perm[i + 1]] for i in range(n - 1))
