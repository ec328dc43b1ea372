"""Stage 1's staging-pool waves at their limits, in the kernel emulation and on the GPU, against the oracle.

A query makes two pool allocations that both live until its wave ends: its candidates + document lengths, then its chunk table +
tf matrix. A query whose two allocations each fit the pool but do not fit it together can never be staged, and a batch that needs
more waves than Stage 1 runs leaves queries unfinished. Either query must come back flagged IFX_Q_OVERFLOW -- from ifx_stage1_batch
and from ifx_search_batch -- and never with status 0 and an empty or different list; every other query of the batch stays bit-exact.

The corpus: 80 000 documents, the first `n_hot` of them holding five co-occurring words, a 1 MB pool. The five-word query scores
36 terms (the words and their n-grams) over `n_hot` candidates: with 22 000 it fits the pool (one query per wave), with 26 000
each allocation fits but not both, with 30 000 the tf matrix alone is larger than the pool."""
import ctypes as C

import numpy as np
import pytest

import infidex_b200 as ib
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from parity_util import emu_lib

N = 80_000
WORDS = "alpha bravo charly delta echoes"
POOL_MB = 1
OVERFLOW = 4            # IFX_Q_OVERFLOW

LIBS = [pytest.param("emu", id="emu"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]


def _fillers():
    """3 000 pseudo-words over letters the five words never use: a filler shares no n-gram with the query."""
    rng = np.random.Generator(np.random.PCG64(7)); seen, out = set(), []
    while len(out) < 3000:
        w = "".join(rng.choice(list("fgjkmnqwxz")) + rng.choice(list("iu")) for _ in range(3))
        if w not in seen:
            seen.add(w); out.append(w)
    return out


def _engine(lib, n_hot):
    f = _fillers()
    texts = [(WORDS + " " if i < n_hot else "") + f[(i * 7919) % 3000] for i in range(N)]
    schema = [ib.Field("content")]
    eng = ib.SearchEngine(_gpu_lib=emu_lib()) if lib == "emu" else ib.SearchEngine.CreateDefault()
    eng.IndexColumns(np.arange(N, dtype=np.int64), schema, [texts], upload=False)
    orc = OracleEngine([OField(x.Name, x.Weight, x.Indexable, x.Filterable, x.Facetable) for x in schema])
    orc.load_image(eng.image_ptr())
    return eng, orc, f


def _upload(eng, pool_mb):
    """(Re)create the device index from the host image with a staging pool of `pool_mb` MB (the pool size is read at creation)."""
    if eng._index:
        eng._gpu.ifx_index_destroy(eng._index); eng._index = C.c_void_p()
    mp = pytest.MonkeyPatch(); mp.setenv("IFX_S1_POOL_MB", str(pool_mb))
    try:
        eng._upload(eng.image_ptr())
    finally:
        mp.undo()


def _allocations(eng):
    """(candidates, scored terms, a1, a2) of the five-word query, measured alone on a pool large enough for it: a1 from the
    candidate count, a2 = what the query took from the pool beyond a1 (both rounded to 256 B, as the pool hands them out)."""
    _upload(eng, 8)
    h = eng.UploadBatch([ib.Query(WORDS, 10)])
    try:
        st = eng.RunBatch(h); dbg = np.zeros((1, 24), np.int64)
        eng._gpu.ifx_debug_stage1_queries(h, dbg.ctypes.data_as(C.c_void_p))
    finally:
        eng.FreeBatch(h)
    assert st.s1_waves == 1
    n_cand, ta = int(dbg[0, 0]), int(dbg[0, 9])
    a1 = (8 * n_cand + 64 + 255) & ~255
    return n_cand, ta, a1, int(st.s1_pool_bytes) - a1


def _check(eng, orc, qs, flagged, may_flag=(), st=None):
    """Stage-1 lists and search records of one batch: queries in `flagged` carry IFX_Q_OVERFLOW (and no Stage-1 list), queries in
    `may_flag` either that or the oracle's answer, every other query is bit-exact against the oracle with status 0.
    Returns the disagreements and the indices of the queries flagged in Stage 1 and in the search."""
    bad = []; flag = (set(), set()); memo = {}
    keys, scores, n, status = eng.Stage1Batch(qs, 500, st)
    res = eng.SearchBatch([ib.Query(q, 10) for q in qs])
    for i, q in enumerate(qs):
        if q not in memo:
            memo[q] = orc.stage1(q, 500), orc.search(q, 10)
            assert memo[q][0]["status"] == 0 and memo[q][1]["status"] == 0
        r, x = memo[q]
        # Stage 1
        if status[i] & OVERFLOW and (i in flagged or i in may_flag):
            flag[0].add(i)
            if n[i] != 0:
                bad.append(("stage1 flagged with a list", i, q, int(n[i])))
        elif i in flagged:
            bad.append(("stage1 not flagged", i, q, int(n[i]), int(status[i])))
        elif not (status[i] == 0 and n[i] == len(r["keys"]) and np.array_equal(keys[i, : n[i]], r["keys"])
                  and np.array_equal(scores[i, : n[i]].view(np.uint32), r["scores"].view(np.uint32))):
            bad.append(("stage1", i, q, int(n[i]), len(r["keys"]), int(status[i])))
        # the whole search
        got = res[i]; s = np.array([t.Score for t in got.Records], np.float32)
        if got.Status & OVERFLOW and (i in flagged or i in may_flag):
            flag[1].add(i)      # (its records, if any, come from the later stages alone: the flag says they are incomplete)
        elif i in flagged:
            bad.append(("search not flagged", i, q, len(got.Records), got.Status))
        elif not (got.Status == 0 and [t.DocumentId for t in got.Records] == x["keys"] and np.array_equal(s.view(np.uint32), x["scores"].view(np.uint32))
                  and [t.Tiebreaker for t in got.Records] == x["ties"] and got.TotalCandidates == x["total"]):
            bad.append(("search", i, q, [t.DocumentId for t in got.Records][:5], x["keys"][:5], got.Status))
    return bad, flag


@pytest.mark.parametrize("lib", LIBS)
def test_pool_pair_overflow(lib):
    """22 000 candidates fit a 1 MB pool, 26 000 fit it only one allocation at a time, 30 000 not even the tf matrix alone: the
    first is answered exactly, the other two are flagged, and the rest of their batch is answered exactly."""
    pool = POOL_MB << 20
    for n_hot, fits in ((22_000, True), (26_000, False), (30_000, False)):
        eng, orc, f = _engine(lib, n_hot)
        n_cand, ta, a1, a2 = _allocations(eng)
        assert n_cand == n_hot and ta >= 30, (n_hot, n_cand, ta)
        if n_hot == 22_000:
            assert a1 + a2 <= pool, (a1, a2)
        elif n_hot == 26_000:
            assert a1 <= pool and a2 <= pool < a1 + a2, (a1, a2)         # the case a per-allocation check cannot see
        else:
            assert a2 > pool, (a1, a2)
        _upload(eng, POOL_MB)
        qs = ["alpha", WORDS, "delta charly", f[5], "echoes " + f[(5 * 7919) % 3000], f[11] + " " + f[12], "bravo"]
        bad, _ = _check(eng, orc, qs, set() if fits else {1})
        assert not bad, (n_hot, bad)
        eng.Dispose()


@pytest.mark.parametrize("lib", LIBS)
def test_wave_limit(lib):
    """70 copies of the 22 000-candidate query: each takes ~0.97 MB of the 1 MB pool, so a wave finishes at most one of them and
    the batch needs more waves than Stage 1 runs. Every query is either answered exactly or flagged (the two small ones included:
    the larger queries go first and take the pool of every wave). With several selection CTAs racing for the pool, a wave can
    finish none: CTAs each hold a first allocation and none finds room for its second. The waves after such a wave run with one
    selection CTA, so at most one wave is lost. Measured on an H100: without that fallback 2 of the 72 queries were answered in
    64 waves (the copies' first allocations filled the pool in nearly every wave); with it 64, as in the one-CTA emulation."""
    eng, orc, f = _engine(lib, 22_000)
    _upload(eng, POOL_MB)
    qs = [WORDS] * 70 + [f[5], "alpha"]
    st = ib.Stats(); bad, (f1, f2) = _check(eng, orc, qs, set(), range(len(qs)), st)
    print("wave limit (%s): %d waves; queries flagged: %d of %d in Stage 1, %d in the search" % (lib, st.s1_waves, len(f1), len(qs), len(f2)))
    assert st.s1_waves == 64
    assert not bad, bad
    for f in (f1, f2):
        assert len(f & set(range(70))) >= 70 - 64     # a wave finishes at most one copy
        # ... and at least one query, but for at most one wave: when racing selection CTAs each hold a first allocation and none
        # finds room for its second, the wave finishes nothing and the rest of the batch runs with one selection CTA. (The two
        # small queries may be answered in a wave that also finishes a copy.)
        assert len(qs) - len(f) >= 63, len(f)
    eng.Dispose()
