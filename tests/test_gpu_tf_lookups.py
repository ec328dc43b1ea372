"""Stage 1's term-major tf lookups (k_tf_count / k_tf_scan / k_tf_fill / k_tf_terms) and the forward / streamed lookups of
stage1_lookup on the GPU, against the oracle, at the edges the one-thread kernel emulation cannot reach: tf_terms_item's thread
partitions (fewer queries than warps, one warp per query, groups of more than TF_QCAP = 256 queries in several metadata chunks),
k_tf_scan over more than one 1 024-list tile, rows on either side of the skip-table threshold (511 / 512 / 513 postings), a
partial last container and a short last work item (6 containers, TF_CRANGE = 4), every lookup mode forced, staging-pool waves
with up to 4 x SMs selection CTAs racing for the pool, and a batch handle run twice.

The corpus (340 025 documents, 5 full containers and a partial one) is built from pseudo-words over disjoint letter sets, so a
query's candidates are the documents planted for it:
  filler     one per document (letters b c d f g h a e)
  common     every 8th document
  med[k]     every 40th document (k = 0, 1, 2): rows with a skip table
  r511/512/513  exactly 511 / 512 / 513 postings over all containers, including documents 0, 31, 65 535, 65 536 and N - 1
  sparse     every 12th document of containers 0, 4 and 5: > CHUNK candidates per container for the single-word query (sub-chunks)
  few        5 documents
  rare_a[j]  1 500 words of ~145 documents in containers 0-4 (letters j k l m i o)
  rare_b[j]  40 words of ~205 documents in container 5 only (letters n p r s u)
Deleted documents sit at the container edges and among the dense candidates.

The batch is groups of queries that share one dictionary list, `shared + " " + rare word`: a rare word is the query's highest-idf
list, so its candidates are (mostly) that word's documents. Group sizes 1 and 7 (the whole CTA on one query after another), 8 and 9
(a warp per query), 255 / 256 / 257 (TF_QCAP) and 600 (three metadata chunks). Only five queries of the 600 group (`common` +
rare_b) have candidates in container 5, and they are the group's cheapest, so the LPT order of the selection puts them at the end
of the group, inside the last metadata chunk and not first in it: that chunk's first query has no candidates in container 5, and
the container is looked up only because a later query of the chunk has some. (`common` alone would have candidates there, so it is
not in the batch; the typo below selects the same candidates.) All in all the wave holds more than 1 024 distinct lists. Plus each
other shared word alone, r511 with a word of 5 documents (more candidates than the row), and typos of `common`, whose LD1 unions
hold >= 2 048 postings per container (the LONG range of the union walk)."""
import ctypes as C

import numpy as np
import pytest

import infidex_b200 as ib
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from parity_util import compare_search, compare_search_batch, compare_stage1

pytestmark = pytest.mark.gpu

N = 5 * 65536 + 12345
GROUPS = (("common", 600), ("med0", 257), ("med1", 256), ("med2", 255), ("r512", 9), ("r513", 8), ("r511", 7), ("sparse", 1))


class _ImageHead(C.Structure):      # include/infidex_gpu.h: the leading fields of ifx_index_image
    _fields_ = [("n_docs", C.c_int32), ("n_live", C.c_int32), ("avgdl", C.c_float),
                ("doc_key", C.POINTER(C.c_int64)), ("deleted", C.POINTER(C.c_uint8))]


def _words(rng, cons, vows, syl, n, taken=()):
    seen, out = set(taken), []
    while len(out) < n:
        w = "".join(rng.choice(list(cons)) + rng.choice(list(vows)) for _ in range(syl))
        if w not in seen:
            seen.add(w); out.append(w)
    return out


def corpus(big=600):
    """(texts, deleted doc ids, queries, subset of the queries for the full-search comparisons, {group: query indices},
    indices of the queries of the `common` group with candidates in container 5). `big`: size of the largest group (the emulation
    may use a smaller one)."""
    rng = np.random.Generator(np.random.PCG64(23))
    filler = _words(rng, "bcdfgh", "ae", 3, 1500)
    med = _words(rng, "bcdfgh", "ae", 4, 3)
    rare_a = _words(rng, "jklm", "io", 4, 1500)
    rare_b = _words(rng, "nprs", "u", 4, 40)
    W = {"common": "qyxqyx", "r511": "tvtvtv", "r512": "wzwzwz", "r513": "tztztz", "sparse": "vwvwvw", "few": "yqyqy",
         "med0": med[0], "med1": med[1], "med2": med[2]}
    docs = {k: [] for k in W}
    i = np.arange(N)
    docs["common"] = i[i % 8 == 0]
    for k in range(3):
        docs["med%d" % k] = i[i % 40 == 7 + k]
    docs["sparse"] = i[(i % 12 == 3) & np.isin(i >> 16, [0, 4, 5])]
    docs["few"] = np.array([100, 70_001, 140_002, 200_003, 330_004])
    edges = np.array([0, 31, 65535, 65536, N - 1])
    for name, n in (("r511", 511), ("r512", 512), ("r513", 513)):
        rest = np.setdiff1d(np.arange(N), edges)
        docs[name] = np.sort(np.concatenate([edges, rng.choice(rest, n - len(edges), replace=False)]))
    texts = [[filler[(d * 7919) % 1500]] for d in range(N)]
    for d in range(N):      # two documents in three, so that a rare word's documents hold the shared words too
        if d % 3 != 2:
            texts[d].append(rare_a[((d // 3) * 7) % 1500] if d < 5 * 65536 else rare_b[((d // 3) * 7) % 40])
    for name in sorted(docs, key=lambda k: k == "common"):      # `common` last: no 3-gram runs from it into a following word
        for d in docs[name]:
            texts[d].append(W[name])
    texts = [" ".join(t) for t in texts]
    deleted = np.unique(np.concatenate([rng.choice(N, 2000, replace=False), [31, 65535, N - 1], np.arange(0, 3000, 89),
                                        np.arange(262_144, 262_144 + 4096, 53), np.arange(5 * 65536, 5 * 65536 + 2000, 41)]))

    typo = "qyxqyz"      # LD1: `common`
    ra = iter(range(1500))
    qs, subset, gidx = [], [], {}
    for name, size in GROUPS:
        size = big if name == "common" else size
        w = W[name]
        g = [w] if name != "common" else []                                # the shared word alone
        if name == "common":
            late = range(len(qs) + size - 5, len(qs) + size)
            g += [w + " " + rare_a[next(ra)] for _ in range(size - 5)] + [w + " " + rb for rb in rare_b[:5]]
        if name == "r511":
            g += [W["few"] + " " + w]      # a word in 5 documents: a disjunctive query with more candidates than the row (the other
                                           # queries of the group take the prefix shortcut: exactly the row's documents)
        while len(g) < size:
            g.append(w + " " + rare_a[next(ra)])
        gidx[name] = range(len(qs), len(qs) + len(g))
        qs += g
        subset += g if size <= 9 else g[:6] + g[-8:]
    extra = [typo, typo + " " + rare_a[next(ra)], rare_b[7], rare_a[next(ra)] + " " + rare_a[next(ra)]]
    qs += extra; subset += extra
    return texts, deleted, qs, subset, gidx, late


def _upload(eng, pool_mb=None):
    """(Re)create the device index from the host image; `pool_mb`: Stage-1 staging pool in MB (read when the index is created)."""
    if eng._index:
        eng._gpu.ifx_index_destroy(eng._index); eng._index = C.c_void_p()
    mp = pytest.MonkeyPatch()
    if pool_mb is None:
        mp.delenv("IFX_S1_POOL_MB", raising=False)
    else:
        mp.setenv("IFX_S1_POOL_MB", str(pool_mb))
    try:
        eng._upload(eng.image_ptr())
    finally:
        mp.undo()


def build(gpu_lib=None, big=600):
    texts, deleted, qs, subset, gidx, late = corpus(big)
    keys = np.arange(N, dtype=np.int64); schema = [ib.Field("content")]
    eng = ib.SearchEngine(_gpu_lib=gpu_lib) if gpu_lib else ib.SearchEngine.CreateDefault()
    eng.IndexColumns(keys, schema, [texts], upload=False)
    img = C.cast(eng.image_ptr(), C.POINTER(_ImageHead)).contents
    flags = np.ctypeslib.as_array(img.deleted, shape=(N,)); flags[deleted] = 1
    img.n_live = int(N - flags.sum())
    _upload(eng)
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema])
    orc.load_image(eng.image_ptr())
    return eng, orc, qs, subset, (gidx, late)


def reach(eng, qs, shape):
    """Run the batch once in stream mode through a batch handle and read what Stage 1 did from its debug records; returns the
    facts the tests rely on (the caller has set IFX_S1_LOOKUP=2). The records are the query plans and the per-query lookup
    records, not k_tf_count's groups: a group here is the set of queries with candidates whose plan scores a dictionary list
    (every such list is streamed in stream mode), and the list count is the number of distinct such lists. The position of a
    query in its group follows from the LPT order of k_order, recomputed from the plans' list lengths."""
    gidx, late = shape
    h = eng.UploadBatch([ib.Query(q, 10) for q in qs])
    try:
        st = eng.RunBatch(h)
        dbg = np.zeros((len(qs), 24), np.int64); eng._gpu.ifx_debug_stage1_queries(h, dbg.ctypes.data_as(C.c_void_p))
        tt = np.zeros((len(qs), 128, 3), np.int32); eng._gpu.ifx_debug_stage1_terms(h, tt.ctypes.data_as(C.c_void_p))
    finally:
        eng.FreeBatch(h)
    has = dbg[:, 0] > 0
    sel = has[:, None] & (tt[:, :, 0] >= 0) & (tt[:, :, 2] != 0)       # the streamed dictionary lists of every query
    ids, cnt = np.unique(tt[:, :, 0][sel], return_counts=True)
    count = dict(zip(ids.tolist(), cnt.tolist()))
    lens = {int(t): int(n) for t, n in zip(tt[:, :, 0][sel], tt[:, :, 1][sel])}
    group, row = {}, {}
    for name, idx in gidx.items():      # the lists every query of the group streams (its shared word, some of the word's 3-grams)
        shared = set.intersection(*[set(tt[q, :, 0][sel[q]].tolist()) for q in idx])
        group[name] = min(count[t] for t in shared) if shared else 0      # the word's own list: only this group's queries stream it
        row[name] = min(lens[t] for t in shared) if shared else 0         # ... and its row is the shortest of them
    # k_order's bucket of every query (no prefix shortcut on these queries): 8 buckets per power of two of 8 + the plan's list lengths
    w = 8 + np.where(tt[:, :, 0] != -2, tt[:, :, 1], 0).astype(np.int64).sum(1)
    msb = np.floor(np.log2(w)).astype(np.int64); bucket = msb * 8 + ((w >> (msb - 3)) & 7)
    common = list(gidx["common"]); rest = [q for q in common if q not in late]
    n_before = min(int((bucket[rest] > bucket[q]).sum()) for q in late)     # group members LPT puts before every late query
    return dict(waves=st.s1_waves, modes=dbg[has, 6], n_lists=len(count), group=group, row=row, n_before=n_before,
                late_path=dbg[list(late), 3], late_chunks=dbg[list(late), 7])


def check_reach(r, sizes):
    assert r["waves"] == 1
    assert (r["modes"] == 2).all()                        # every query with candidates took stream mode
    assert r["n_lists"] > 1024                           # k_tf_scan over more than one tile
    assert r["group"] == sizes, r["group"]               # tf_terms_item's partitions: wide, a warp per query, TF_QCAP chunks
    assert [r["row"][n] for n in ("r511", "r512", "r513")] == [511, 512, 513]
    # the `common` group's queries with candidates in container 5 (one container each: a single chunk) come after all the others,
    # so they sit in a later TF_QCAP chunk and none of them first in it
    assert (r["late_path"] != 1).all() and (r["late_chunks"] == 1).all()
    assert r["n_before"] == sizes["common"] - 5 and r["n_before"] >= 256 and r["n_before"] % 256 != 0, r["n_before"]


@pytest.fixture(scope="module")
def gpu_pair():
    eng, orc, qs, subset, shape = build()
    yield eng, orc, qs, subset, shape
    eng.Dispose()


@pytest.mark.parametrize("mode", ["0", "1", "2"])
def test_tf_lookups_parity(gpu_pair, monkeypatch, mode):
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, qs, subset, shape = gpu_pair
    assert not compare_stage1(eng, orc, qs)
    assert not compare_search(eng, orc, subset)
    assert not compare_stage1(eng, orc, qs[::7], depth=50)
    assert not compare_search_batch(eng, orc, qs[::5], depth=50)


def test_tf_lookups_reach(gpu_pair, monkeypatch):
    monkeypatch.setenv("IFX_S1_LOOKUP", "2")
    eng, orc, qs, subset, shape = gpu_pair
    check_reach(reach(eng, qs, shape), dict(GROUPS))


def test_tf_lookups_reused_handle(gpu_pair, monkeypatch):
    """A second run of the same batch handle returns the first run's records bit for bit (the per-wave state -- pair and group
    counts, the per-term counts k_tf_terms zeroes -- is clean between runs)."""
    monkeypatch.setenv("IFX_S1_LOOKUP", "2")
    eng, orc, qs, subset, shape = gpu_pair
    qq = [ib.Query(q, 10) for q in qs]
    h = eng.UploadBatch(qq)
    try:
        runs = []
        for _ in range(2):
            eng.RunBatch(h); p = eng.PackBatch(qq); b = eng.DownloadBatch(h, p)
            runs.append({k: b[k].copy() for k in ("keys", "scores", "ties", "n", "total", "status")})
    finally:
        eng.FreeBatch(h)
    assert runs[0]["n"].sum() > 0
    for k in runs[0]:
        assert np.array_equal(runs[0][k].view(np.uint8), runs[1][k].view(np.uint8)), k


@pytest.mark.parametrize("pool_mb", [60, 100])
def test_tf_lookups_waves(gpu_pair, monkeypatch, pool_mb):
    """The same batch through a smaller staging pool (the batch takes ~280 MB in one wave): several waves, up to 4 x SMs selection
    CTAs racing for the pool, the wave state reset between waves; bit-exact in the cost model's choice and in stream mode. The
    one-CTA emulation finishes the batch in 5 waves at 60 MB and 3 at 100 MB."""
    eng, orc, qs, subset, shape = gpu_pair
    _upload(eng, pool_mb)
    try:
        for mode in ("0", "2"):
            monkeypatch.setenv("IFX_S1_LOOKUP", mode)
            st = ib.Stats(); bad = compare_stage1(eng, orc, qs, stats=st)
            print("pool %d MB, IFX_S1_LOOKUP=%s: %d waves" % (pool_mb, mode, st.s1_waves))
            assert 1 < st.s1_waves < 64
            assert not bad
            assert not compare_search_batch(eng, orc, qs)
    finally:
        _upload(eng)
