"""The term-major tf lookups of Stage 1 (k_tf_count / k_tf_scan / k_tf_fill / k_tf_terms) in the kernel emulation, against the oracle.
The corpus of test_emu_lookup_containers (three 65 536-doc containers, deleted documents) with a 1 MB staging pool, so the batch runs
in several waves. The batch shares lists between many queries: a long list with a skip table (`common`, a medium word), a short row
without one (a rare word), a shared list in which one query has no candidates in a container (`gap common`: no candidates in
container 1), LD1 unions next to shared dictionary lists, and queries that the cost model sends to the forward index."""
import ctypes as C

import numpy as np
import pytest

import infidex_b200 as ib
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from parity_util import compare_search, compare_stage1, emu_lib
from test_emu_lookup_containers import N, _ImageHead, _corpus


@pytest.fixture(scope="module")
def pair():
    mp = pytest.MonkeyPatch()
    mp.setenv("IFX_S1_POOL_MB", "1")      # read when the index is created
    try:
        texts, common, medium, rare, gap = _corpus()
        keys = np.arange(N, dtype=np.int64); schema = [ib.Field("content")]
        eng = ib.SearchEngine(_gpu_lib=emu_lib()); eng.IndexColumns(keys, schema, [texts], upload=False)
        img = C.cast(eng.image_ptr(), C.POINTER(_ImageHead)).contents
        deleted = np.ctypeslib.as_array(img.deleted, shape=(N,))
        gone = np.random.Generator(np.random.PCG64(11)).choice(N, 2000, replace=False)
        deleted[np.unique(np.concatenate([gone, np.arange(0, 3000, 89), np.arange(131_072, 131_072 + 4096, 53)]))] = 1
        img.n_live = int(N - deleted.sum())
        eng._upload(eng.image_ptr())
    finally:
        mp.undo()
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema])
    orc.load_image(eng.image_ptr())
    typo = medium[5][:2] + ("z" if medium[5][2] != "z" else "y") + medium[5][3:]
    qs = [common, gap, gap + " " + common, common + " " + gap, rare[3], rare[3] + " " + medium[1], rare[3] + " " + common,
          rare[3] + " " + rare[4], medium[1], medium[1] + " " + medium[2], medium[2] + " " + common, typo, typo + " " + common,
          typo + " " + medium[5], rare[17] + " " + medium[2], rare[18] + " " + medium[1] + " " + common]
    qs += [common + " " + rare[i] for i in range(30, 42)] + [medium[1] + " " + rare[i] for i in range(50, 56)]
    return eng, orc, qs


@pytest.mark.parametrize("mode", ["0", "2"])
def test_emu_term_major(pair, monkeypatch, mode):
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, qs = pair
    st = ib.Stats(); eng.SearchBatch([ib.Query(q, 10) for q in qs], st)
    assert st.s1_waves > 1
    assert not compare_stage1(eng, orc, qs)
    assert not compare_search(eng, orc, qs)
