"""The container-major tf lookups of Stage 1 (stage1_lookup) in the kernel emulation, against the oracle: a corpus of three
65 536-doc containers with deleted documents, both lookup modes forced (IFX_S1_LOOKUP=2 streams every list container by container,
=1 reads forward lists and streams only the LD1 unions), and queries whose candidates exercise every kind of (list, container) range."""
import ctypes as C

import numpy as np
import pytest

import infidex_b200 as ib
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from parity_util import compare_search, compare_stage1, emu_lib

N = 150_000


class _ImageHead(C.Structure):      # include/infidex_gpu.h: the leading fields of ifx_index_image
    _fields_ = [("n_docs", C.c_int32), ("n_live", C.c_int32), ("avgdl", C.c_float),
                ("doc_key", C.POINTER(C.c_int64)), ("deleted", C.POINTER(C.c_uint8))]


def _corpus():
    """Short documents over pseudo-words: `common` in every 8th document (> 4096 candidates per container: sub-chunks), 40 medium
    words (~3 750 documents each: rows with a skip table), 1 500 rare words (100 documents each: rows below 512 postings, no skip
    table), and `gap` only in containers 0 and 2 (a container without candidates between two with candidates)."""
    rng = np.random.Generator(np.random.PCG64(3)); seen, vocab = set(), []
    while len(vocab) < 23_000:
        w = "".join(rng.choice(list("bcdfghjklmnprstvw")) + rng.choice(list("aeiou")) for _ in range(3))
        if w not in seen:
            seen.add(w); vocab.append(w)
    medium, rare, filler = vocab[1:41], vocab[100:1600], vocab[3000:23000]
    common, gap = "qyxqyx", "zyqzyq"        # letters the other words never use: the candidates are exactly these words' documents
    texts = []
    for i in range(N):
        w = [medium[i % 40], rare[(i * 7) % 1500], filler[(i * 7919) % 20000]]
        if i % 8 == 0:
            w.append(common)
        if i < 3000 or 131_072 <= i < 134_000:
            w.append(gap)
        texts.append(" ".join(w))
    return texts, common, medium, rare, gap


def _build(emu):
    texts, common, medium, rare, gap = _corpus()
    keys = np.arange(N, dtype=np.int64)
    schema = [ib.Field("content")]
    eng = ib.SearchEngine(_gpu_lib=emu)
    eng.IndexColumns(keys, schema, [texts], upload=False)
    img = C.cast(eng.image_ptr(), C.POINTER(_ImageHead)).contents
    deleted = np.ctypeslib.as_array(img.deleted, shape=(N,))
    gone = np.random.Generator(np.random.PCG64(5)).choice(N, 1500, replace=False)
    gone = np.concatenate([gone, np.arange(0, 3000, 97), np.arange(131_072, 131_072 + 4096, 61)])      # some of them among the dense candidates
    deleted[np.unique(gone)] = 1
    img.n_live = int(N - deleted.sum())
    eng._upload(eng.image_ptr())
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema])
    orc.load_image(eng.image_ptr())
    typo = medium[5][:2] + ("z" if medium[5][2] != "z" else "y") + medium[5][3:]          # an unknown word: its LD1 expansion is a union list
    qs = [common, gap, rare[3], rare[17] + " " + medium[2], medium[7], gap + " " + common, typo, typo + " " + rare[9],
          medium[1] + " " + medium[2], common + " " + rare[40]]
    return eng, orc, qs


@pytest.fixture(scope="module")
def pair():
    return _build(emu_lib())


@pytest.mark.parametrize("mode", ["2", "1"])
def test_emu_lookup_containers(pair, monkeypatch, mode):
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, qs = pair
    assert not compare_stage1(eng, orc, qs)
    assert not compare_search(eng, orc, qs)
