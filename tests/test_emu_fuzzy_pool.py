"""The LD1 expansion when a batch's unions outgrow the fuzzy pool, in the kernel emulation. Every unknown word of >= 4 characters is
expanded into the union of its edit-distance-1 matches' posting lists, and the unions of a batch share one pool of at least 1 << 20
ids. A union that does not fit raises IFX_Q_OVERFLOW on its query instead of being cut. The corpus here has 16 five-letter words,
each in about 70 % of the documents, and every query holds a one-letter variant of each of them: 16 unions of ~1 400 documents per
query, so 80 queries need ~1.8 M ids and the later ones do not fit. The expansion works through the CTA's candidate bitset, which
must be left all-zero whichever way a union ends; a plain batch after the overflowing one shows that it was."""
import numpy as np

import infidex_b200 as ib
from oracle.oracle import Field as OField
from oracle.oracle import OracleEngine
from parity_util import compare_search, compare_stage1, emu_lib

N = 2000
OVERFLOW = 4            # IFX_Q_OVERFLOW
FIELDS = ("keys", "scores", "ties", "n", "total", "status")


def _corpus():
    rng = np.random.Generator(np.random.PCG64(21))
    base = ["bacde", "fghij", "klmno", "prstu", "vwxyb", "cdfgh", "jklmp", "nortv", "wxybc", "dfhjl", "mnprs", "tvwxy", "bdfhk",
            "lnpst", "vxzbd", "gjmos"]
    texts = []
    for _ in range(N):
        words = [w for w in base if rng.random() < 0.7] or [base[0]]
        texts.append(" ".join(rng.permutation(words)))
    queries = []
    for _ in range(80):
        ws = []
        for w in rng.permutation(base):
            p = int(rng.integers(0, 5)); ws.append(w[:p] + "q" + w[p + 1:])      # 'q' is in no word: an unknown word one substitution away
        queries.append(" ".join(ws))
    return base, texts, queries


def _run_twice(eng, qq):
    h = eng.UploadBatch(qq)
    try:
        runs = []
        for _ in range(2):
            eng.RunBatch(h); b = eng.DownloadBatch(h, eng.PackBatch(qq))
            runs.append({k: b[k].copy() for k in FIELDS})
    finally:
        eng.FreeBatch(h)
    return runs


def test_emu_fuzzy_pool_overflow():
    base, texts, queries = _corpus()
    schema = [ib.Field("content")]
    eng = ib.SearchEngine(_gpu_lib=emu_lib()); eng.IndexColumns(np.arange(N, dtype=np.int64), schema, [texts])
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema]); orc.load_image(eng.image_ptr())
    qq = [ib.Query(q, 10) for q in queries]
    runs = _run_twice(eng, qq)
    for k in FIELDS:      # the same handle again: the same records
        assert np.array_equal(runs[0][k].view(np.uint8), runs[1][k].view(np.uint8)), k
    r = runs[0]; kinds = {"exact": 0, "overflow": 0}; bad = []
    for i, q in enumerate(queries):
        if r["status"][i] & OVERFLOW:
            kinds["overflow"] += 1
            continue
        x = orc.search(q, 10); n = int(r["n"][i])
        ok = r["status"][i] == 0 and x["status"] == 0 and r["keys"][i, :n].tolist() == x["keys"] and \
            np.array_equal(r["scores"][i, :n].view(np.uint32), x["scores"].view(np.uint32)) and r["ties"][i, :n].tolist() == x["ties"] and \
            r["total"][i] == x["total"]
        if ok:
            kinds["exact"] += 1
        else:
            bad.append((i, q, int(r["status"][i]), r["keys"][i, :n].tolist(), x["keys"]))
    assert not bad, bad[:3]
    assert kinds["exact"] >= 10 and kinds["overflow"] >= 10, kinds
    # a plain batch next on the same index: known words, and unknown words whose unions fit the pool now
    plain = base[:4] + [base[0] + " " + base[5], base[3] + " " + base[9] + " " + base[12]] + queries[:8] + \
        [queries[40].split()[0] + " " + base[2], base[7][:2] + "q" + base[7][3:]]
    assert not compare_stage1(eng, orc, plain)
    assert not compare_search(eng, orc, plain)
