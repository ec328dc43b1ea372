"""Stage 1's AND tiers on the GPU, against the oracle: tier 1 taken from the id array that tier 0's intersection leaves before its last
step (debug slot 18 = 1), checked through the candidate count of every query as well as its records. The corpus also puts the
unchanged count + expand of the candidate bitset at the edges the one-thread kernel emulation cannot reach: a container whose 65 536
documents are all candidates, one with 65 535, one with a single candidate, and a partial last container whose candidates sit on warp
and CTA boundaries (documents 0, 31, 32, 255, 256, 257, 2 047 and 2 048 of the container, the last one of the corpus). Deleted documents
sit at container edges and among the full containers' candidates; a typo of the dense word is an LD1 union. The dense word with each of
the filler words (about 130 documents each) holds fewer than 1 000 documents, so those queries reach AND tier 1. Parity in lookup
modes 0 and 2 at depths 500 and 10, and a reused batch handle."""
import ctypes as C

import numpy as np
import pytest

import infidex_b200 as ib
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from parity_util import compare_search, compare_stage1

pytestmark = pytest.mark.gpu

N = 3 * 65536 + 2049
EDGE = [0, 31, 32, 255, 256, 257, 2047, 2048]


class _ImageHead(C.Structure):      # include/infidex_gpu.h: the leading fields of ifx_index_image
    _fields_ = [("n_docs", C.c_int32), ("n_live", C.c_int32), ("avgdl", C.c_float),
                ("doc_key", C.POINTER(C.c_int64)), ("deleted", C.POINTER(C.c_uint8))]


def corpus():
    rng = np.random.Generator(np.random.PCG64(31)); seen, filler = set(), []
    while len(filler) < 1500:
        w = "".join(rng.choice(list("bcdfgh")) + rng.choice(list("ae")) for _ in range(3))
        if w not in seen:
            seen.add(w); filler.append(w)
    dense = "qyxqyx"
    i = np.arange(N)
    c0, c1, c2, c3 = (i >> 16) == 0, (i >> 16) == 1, (i >> 16) == 2, (i >> 16) == 3
    has = c0 | (c1 & (i != 65536 + 4097)) | (i == 2 * 65536 + 5000) | (c3 & np.isin(i - 3 * 65536, EDGE))
    texts = [filler[(d * 7919) % 1500] + (" " + dense if has[d] else "") for d in range(N)]
    deleted = np.unique(np.concatenate([rng.choice(N, 1500, replace=False), [0, 65535, 65536, 3 * 65536 + 31, N - 1],
                                        np.arange(1000, 1000 + 4096, 37)]))
    qs = [dense, "qyxqyz", dense + " " + filler[3]] + [dense + " " + filler[j] for j in range(10, 40, 3)] + [filler[j] + " " + dense for j in (5, 6)]
    return texts, deleted, qs


@pytest.fixture(scope="module")
def gpu_pair():
    texts, deleted, qs = corpus()
    schema = [ib.Field("content")]
    eng = ib.SearchEngine(); eng.IndexColumns(np.arange(N, dtype=np.int64), schema, [texts], upload=False)
    img = C.cast(eng.image_ptr(), C.POINTER(_ImageHead)).contents
    dl = np.ctypeslib.as_array(img.deleted, shape=(N,)); dl[deleted] = 1
    img.n_live = int(N - dl.sum())
    eng._upload(eng.image_ptr())
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema])
    orc.load_image(eng.image_ptr())
    return eng, orc, qs


@pytest.mark.parametrize("mode", ["0", "2"])
def test_select_tiers_parity(gpu_pair, monkeypatch, mode):
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, qs = gpu_pair
    assert not compare_stage1(eng, orc, qs)
    assert not compare_stage1(eng, orc, qs, depth=10)
    assert not compare_search(eng, orc, qs)
    for depth in (500, 10):
        qq = []
        for q in qs:
            x = ib.Query(q, 10); x.CoverageDepth = depth; qq.append(x)
        h = eng.UploadBatch(qq)
        try:
            eng.RunBatch(h)
            dbg = np.zeros((len(qs), 24), np.int64); eng._gpu.ifx_debug_stage1_queries(h, dbg.ctypes.data_as(C.c_void_p))
        finally:
            eng.FreeBatch(h)
        assert [int(d[0]) for d in dbg] == [orc.stage1(q, depth)["candidates"] for q in qs]      # the candidate sets' sizes
        assert dbg[0, 0] == 65536 + 65535 + 1 + len(EDGE)          # the dense word alone: every candidate expanded, deleted ones included
        if depth == 500:
            assert (dbg[:, 18] == 1).sum() >= 5                     # tier 1 from tier 0's saved id array (at depth 10 tier 0 alone is enough)


def test_select_tiers_reused_handle(gpu_pair):
    eng, orc, qs = gpu_pair
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
