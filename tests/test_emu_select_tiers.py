"""The AND tiers of the candidate selection of Stage 1 in the kernel emulation, against the oracle bit for bit. Tier 1 (every list of
the query but the lowest-idf one) is either taken from tier 0's intersection -- the id array before its last step, when the held-out
list sorts last by length and that step ran on the array -- or recomputed; the per-query debug record says which (slot 18: 1 saved,
2 recomputed because a list is longer than the held-out one, 3 recomputed because tier 0's last step ran on the bitset). Every query's
candidate count is compared with the oracle's as well as its records: after tier 1 the selection unions the highest-idf lists only
while tier 0 + tier 1 hold fewer than 5K documents, and those lists contain tier 1, so a wrong tier-1 set shows in the records only
through that decision -- at depth 10 (K = 10) it decides for most queries. The corpus is the three-container one of
test_emu_lookup_containers (the last container partial, deleted documents at container edges and among the dense candidates).
A second corpus has a word in every document: its lists are as long as the id arrays (the seed at exactly buf_cap, the longest
list of the index and at least the shard size). A longer seed cannot occur -- no list is longer than the shard."""
import ctypes as C

import numpy as np
import pytest

import infidex_b200 as ib
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from parity_util import compare_search, compare_stage1, emu_lib
from test_emu_lookup_containers import N, _ImageHead, _corpus

QDBG = 24


@pytest.fixture(scope="module")
def pair():
    texts, common, medium, rare, gap = _corpus()
    keys = np.arange(N, dtype=np.int64); schema = [ib.Field("content")]
    eng = ib.SearchEngine(_gpu_lib=emu_lib()); eng.IndexColumns(keys, schema, [texts], upload=False)
    img = C.cast(eng.image_ptr(), C.POINTER(_ImageHead)).contents
    deleted = np.ctypeslib.as_array(img.deleted, shape=(N,))
    edges = np.concatenate([np.arange(65_536 - 40, 65_536 + 40), np.arange(131_072 - 40, 131_072 + 40), np.arange(N - 40, N)])      # container edges, the end of the partial last one
    gone = np.random.Generator(np.random.PCG64(7)).choice(N, 1500, replace=False)
    deleted[np.unique(np.concatenate([gone, edges[::3], np.arange(131_072, 131_072 + 4096, 37)]))] = 1
    img.n_live = int(N - deleted.sum())
    eng._upload(eng.image_ptr())
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema])
    orc.load_image(eng.image_ptr())
    typo = medium[5][:2] + ("z" if medium[5][2] != "z" else "y") + medium[5][3:]          # an LD1 union: streamed against the container window
    qs = [common + " " + medium[a] for a in (0, 1, 8, 13)] + [common + " " + rare[r] for r in (0, 3, 9, 17, 40)] + \
         [gap + " " + medium[a] for a in (1, 2, 3, 8)] + [gap + " " + rare[r] for r in (3, 5, 9)] + \
         [common + " " + medium[1] + " " + rare[r] for r in (3, 9, 17)] + [common + " " + gap, gap + " " + common] + \
         [medium[a] + " " + rare[r] for a in (0, 2) for r in (3, 40)] + [medium[1] + " " + medium[2], rare[3] + " " + rare[4],
         typo + " " + common, common + " " + typo, gap + " " + typo]
    return eng, orc, qs


def _dbg(eng, qs, depth):
    qq = []
    for q in qs:
        x = ib.Query(q, 10); x.CoverageDepth = depth; qq.append(x)
    h = eng.UploadBatch(qq)
    try:
        eng.RunBatch(h)
        dbg = np.zeros((len(qs), QDBG), np.int64); eng._gpu.ifx_debug_stage1_queries(h, dbg.ctypes.data_as(C.c_void_p))
    finally:
        eng.FreeBatch(h)
    return dbg


@pytest.mark.parametrize("mode", ["0", "2"])
def test_emu_select_tiers(pair, monkeypatch, mode):
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, qs = pair
    assert not compare_stage1(eng, orc, qs)
    assert not compare_stage1(eng, orc, qs, depth=10)
    assert not compare_search(eng, orc, qs)
    routes = {}
    for depth in (500, 10):
        dbg = _dbg(eng, qs, depth)
        assert [int(d[0]) for d in dbg] == [orc.stage1(q, depth)["candidates"] for q in qs], depth
        route, path, terms = dbg[:, 18], dbg[:, 3], dbg[:, 1]
        assert (route[path != 3] == 0).all() and (route[terms < 3] == 0).all()      # tier 1 only on the AND path, and only with >= 3 lists
        routes[depth] = np.bincount(route, minlength=4)
    assert routes[500][1] >= 10 and routes[10][1] >= 10, routes      # tier 1 from tier 0's saved id array
    assert routes[500][3] >= 1, routes                                # tier 0 ended on the bitset: recomputed


def test_emu_select_tiers_seed_at_buf_cap(monkeypatch):
    """Every document holds `qyxqyx`, so its lists (the word and its 3-grams) are N long, the workspace's id-array capacity."""
    n = 12_000      # more documents than the prefix shortcut takes at depth 500 (K * 20)
    rng = np.random.Generator(np.random.PCG64(13)); words = []
    while len(words) < 60:
        w = "".join(rng.choice(list("bcdfgh")) + rng.choice(list("ae")) for _ in range(3))
        if w not in words:
            words.append(w)
    texts = ["%s %s qyxqyx" % (words[i % 60], words[(i * 7) % 59]) for i in range(n)]
    schema = [ib.Field("content")]
    eng = ib.SearchEngine(_gpu_lib=emu_lib()); eng.IndexColumns(np.arange(n, dtype=np.int64), schema, [texts])
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema]); orc.load_image(eng.image_ptr())
    qs = ["qyxqyx", "qyxqyx " + words[3], words[5] + " qyxqyx", "qyxqyx " + words[7] + " " + words[11]]
    for mode in ("0", "2"):
        monkeypatch.setenv("IFX_S1_LOOKUP", mode)
        assert not compare_stage1(eng, orc, qs)
        assert not compare_stage1(eng, orc, qs, depth=10)
        dbg = _dbg(eng, qs, 500)
        assert dbg[0, 3] == 3 and dbg[0, 0] == n                       # the AND path over lists of exactly buf_cap ids, no overflow
        assert [int(d[0]) for d in dbg] == [orc.stage1(q, 500)["candidates"] for q in qs]


@pytest.mark.parametrize("n, n_b_only, route", [(100_000, 150, 1), (20_000, 2400, 3)])
def test_emu_select_tiers_held_out_list_removes_documents(monkeypatch, n, n_b_only, route):
    """Tier 1 differs from tier 0. In the query `qyqyqx zwzwzw` the lowest-idf list is the 3-gram `x z` across the word boundary, which 6
    000 documents hold through the filler pair `bax zab`; of the 600 documents with both words only the 100 where they are adjacent
    hold it. So tier 0 has 100 documents and tier 1 600, and at depth 100 tier 0 + tier 1 reach 5K: the candidates are exactly tier 0
    + tier 1, and a wrong tier-1 set changes them (`zwzwzw` alone holds more). With 100 000 documents the seed list (`zwzwzw`, 750) is
    short against the shard, so tier 0 runs on the id array and tier 1 is the array saved before its last step; with 20 000 documents
    and 3 000 of `zwzwzw` the intersection stays on the bitset to the end and tier 1 is recomputed."""
    texts = ["bax zab" if i < 6000 else "dob fek" for i in range(n)]
    both = np.arange(6000, 6600); a_only = np.arange(7000, 9400); b_only = np.arange(10_000, 10_000 + n_b_only)
    for k, i in enumerate(both):
        texts[i] = ("fek qyqyqx zwzwzw dob" if k < 100 else "fek zwzwzw dob qyqyqx dob")
    for i in a_only:
        texts[i] += " qyqyqx dob"
    for i in b_only:
        texts[i] = "fek zwzwzw " + texts[i]
    schema = [ib.Field("content")]
    eng = ib.SearchEngine(_gpu_lib=emu_lib()); eng.IndexColumns(np.arange(n, dtype=np.int64), schema, [texts])
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema]); orc.load_image(eng.image_ptr())
    qs = ["qyqyqx zwzwzw"]
    for mode in ("0", "2"):
        monkeypatch.setenv("IFX_S1_LOOKUP", mode)
        assert not compare_stage1(eng, orc, qs, depth=100)
        dbg = _dbg(eng, qs, 100)
        assert dbg[0, 3] == 3 and dbg[0, 18] == route, dbg[0]
        assert dbg[0, 0] == orc.stage1(qs[0], 100)["candidates"] == 600
