"""The fixture of test_gpu_scorers / test_emu_scorers: a corpus whose queries reach every edge of Stage 1's three scorers
(score_warp<256> "light", score_warp<512> "mid", score_cta) and of k_s1_finish, with every query's candidate set known exactly.

Containers are 65 536 documents; the corpus has 12 full ones and a partial 13th. Words live on disjoint character sets, so a word's
3-grams occur only in the documents planted with it:
  filler      1-13 words over b c d a e, from 60 texts: documents with the same planted words and the same filler text are
              identical (score ties inside a chunk and across containers), and the lengths spread so that avgdl is not round
  light[n]    exactly n documents in every container, n = 1, 7, 8, 9, 31, 32, 33, 255, 256 (letters g-n, two per word)
  w257 ... w8195   257 / 512 / 513 / 4 095 / 4 096 / 4 097 / 8 195 documents in one or two containers
  w300        300 documents in each of the 12 full containers: a mid query with many chunks behind a full heap
  lc          every 300th document (~218 per container): `light word + lc` stays a light (or mid) query
  common      every 5th document: in `rare word + common` the common word's low-idf terms are skipped once the threshold rises
  hosts       the same sequence of 3-4 character words in every document of a host set: 250 per container ("hl", light),
              500 ("hm", mid) or 1 000 ("hc", CTA); a query made of runs of that sequence has the host's candidates and a
              scored-term count Ta that the runs set (each word, the 3-grams inside it and across the space to its neighbour)
Deleted documents sit at chunk slots 0, 255, 256, 511, 512 and 4 095 of some planted words (the slot of a single-word query's
candidate is its rank among the word's documents in the container), plus a random 0.3 %. DocumentKeys are a permutation of the
document ids, so the (score desc, key asc) order of the final list is not the document order."""
import ctypes as C

import numpy as np

import infidex_b200 as ib
from oracle import oracle as O

CONT = 65536
NC = 12
N = NC * CONT + 20000
LIGHT = (1, 7, 8, 9, 31, 32, 33, 255, 256)
BOUND = {"w257": {2: 257}, "w512": {3: 512, 9: 512}, "w513": {4: 513}, "w4095": {5: 4095}, "w4096": {6: 4096},
         "w4097": {7: 4097}, "w8195": {8: 8195}, "w300": {c: 300 for c in range(NC)}}
HOSTS = {"hl": ({c: 250 for c in range(6)}, "0123456", 20), "hm": ({1: 500, 10: 500}, "789pr", 6), "hc": ({3: 1000, 11: 1000}, "stuvwz", 5)}
# long queries: {host_Ta: indices of the host's words}; the scored-term count Ta each one reaches is read back from the device by
# the reach test (6 / 7 exercise S1_TILE in the CTA scorer, 12 / 13 the 12-row tile of a 512-slot chunk, 24 / 25
# the 24-row tile of a 256-slot chunk, 64 the largest light query and 65 the CTA)
LONG = {"hl_24": [6, 11, 12, 14, 16, 17], "hl_25": [1, 2, 3, 14, 15, 16], "hl_63": [0, 1, 2, 3, 5, 6, 7, 8, 9, 11, 12, 13, 14, 18],
        "hl_64": [0, 1, 2, 5, 6, 7, 8, 9, 10, 11, 13, 14, 16, 17], "hl_65": [0, 1, 3, 4, 5, 6, 9, 11, 12, 13, 14, 15, 17, 18, 19],
        "hm_12": [1, 4, 5], "hm_13": [0, 1, 2], "hc_6": [2, 4], "hc_7": [2, 3]}
DEPTHS = (1, 2, 3, 4, 5, 10, 500, 512, 513, 1024)
# chunk slots of deleted candidates: {word: {container: [ranks among the word's documents there]}}
DELETED_SLOTS = {"light256": {1: [0, 255], 12: [0]}, "light255": {4: [254]}, "w512": {3: [0, 255, 256, 511]}, "w513": {4: [0, 512]},
                 "w4096": {6: [0, 255, 256, 511, 512, 4095]}, "w8195": {8: [0, 4095, 4096, 8191, 8192]}, "w257": {2: [256]}}


class _ImageHead(C.Structure):      # include/infidex_gpu.h: the leading fields of ifx_index_image
    _fields_ = [("n_docs", C.c_int32), ("n_live", C.c_int32), ("avgdl", C.c_float),
                ("doc_key", C.POINTER(C.c_int64)), ("deleted", C.POINTER(C.c_uint8))]


def _alternation(a, b):
    return (a + b) * 3


def _host_words(rng, chars, n):
    """n words of 3-4 distinct characters whose 3-grams, first two and last two characters are all distinct (so every word adds
    its own terms to a query)."""
    grams, firsts, lasts, out = set(), set(), set(), []
    while len(out) < n:
        w = "".join(rng.choice(list(chars), size=int(rng.integers(3, 5)), replace=False))
        g = {w[i:i + 3] for i in range(len(w) - 2)} | {w}
        if g & grams or w[:2] in firsts or w[-2:] in lasts:
            continue
        grams |= g; firsts.add(w[:2]); lasts.add(w[-2:]); out.append(w)
    return out


def words():
    """{name: text} of every planted word and each host's word sequence."""
    rng = np.random.Generator(np.random.PCG64(71))
    pool = "ghijklmn"
    pairs = [(pool[i], pool[j]) for i in range(len(pool)) for j in range(i + 1, len(pool))]
    W = {}
    for k, n in enumerate(LIGHT):
        W["light%d" % n] = _alternation(*pairs[k])
    for k, name in enumerate(BOUND):
        W[name] = _alternation(*pairs[len(LIGHT) + k])
    W["lc"] = "fofofo"; W["common"] = "qyxqyx"
    seqs = {h: _host_words(rng, chars, n) for h, (_, chars, n) in HOSTS.items()}
    return W, seqs


def corpus():
    """(texts, keys, deleted doc ids, {word: its documents})."""
    rng = np.random.Generator(np.random.PCG64(19))
    W, seqs = words()
    fil = ["".join(rng.choice(list("bcd")) + rng.choice(list("ae")) for _ in range(3)) for _ in range(400)]
    ftexts = [" ".join(fil[(7 * k + 3 * i) % 400] for i in range(1 + (5 * k) % 13)) for k in range(60)]
    docs = {}
    for c in range(NC + 1):      # per container, disjoint pieces of a random permutation: planted words and hosts never share documents
        size = min(CONT, N - c * CONT); perm = rng.permutation(size) + c * CONT; at = 0
        want = [("light%d" % n, n) for n in LIGHT] + [(name, m[c]) for name, m in BOUND.items() if c in m] + \
               [(h, m[c]) for h, (m, _, _) in HOSTS.items() if c in m]
        for name, n in want:
            docs.setdefault(name, []).append(np.sort(perm[at:at + n])); at += n
    docs = {k: np.concatenate(v) for k, v in docs.items()}
    i = np.arange(N)
    docs["lc"] = i[i % 300 == 17]; docs["common"] = i[i % 5 == 2]
    fsel = rng.integers(0, len(ftexts), N)
    texts = [[ftexts[f]] for f in fsel]
    for name, ds in docs.items():
        if name in ("lc", "common"):
            continue
        t = " ".join(seqs[name]) if name in seqs else W[name]
        for d in ds:
            texts[d].append(t)
    for name in ("lc", "common"):      # `common` last: no 3-gram runs from it into a following word
        for d in docs[name]:
            texts[d].append(W[name])
    texts = [" ".join(t) for t in texts]
    dead = [rng.choice(N, N // 300, replace=False)]
    for name, per in DELETED_SLOTS.items():
        for c, ranks in per.items():
            ds = docs[name][(docs[name] >> 16) == c]
            dead.append(ds[ranks])
    deleted = np.unique(np.concatenate(dead))
    keys = rng.permutation(N).astype(np.int64) * 3 + 11
    return texts, keys, deleted, docs


def queries():
    """[(text, name)]: each planted word alone, rare + common, light / mid words + lc, typos, and the long host queries."""
    W, seqs = words()
    q = [(W["light%d" % n], "light%d" % n) for n in LIGHT] + [(W[name], name) for name in BOUND]
    q += [(W[a] + " " + W["common"], a + "+common") for a in ("light1", "light33", "w257", "w4095")]
    q += [(W[a] + " " + W["lc"], a + "+lc") for a in ("light1", "light8", "light33", "w257", "light255")]
    q += [(W["lc"], "lc")]
    q += [(W["light256"][:-1] + "n", "typo256"), (W["w512"][:-1] + "g", "typo512"), (W["light33"][:-1] + "m", "typo33"),
          (W["light9"][:-1] + "k" + " " + W["common"], "typo9+common")]
    for name, picks in LONG.items():
        h = name.split("_")[0]
        q.append((" ".join(seqs[h][k] for k in picks), name))
    return q


def mixed_batch():
    """[(text, name, depth)]: every query at 512, 513 and 1 024 and at one of 1-5 / 10, in one batch."""
    small = (1, 2, 3, 4, 5, 10)
    return [(q, name, d) for i, (q, name) in enumerate(queries()) for d in (small[i % len(small)], 512, 513, 1024)]


def compare_mixed(eng, orc, batch, max_results=10):
    """The batch through one UploadBatch / RunBatch, each query at its own CoverageDepth, against orc.search_batch at that depth:
    DocumentKeys, Score bits, Tiebreaker bytes and counts."""
    qq = []
    for q, _, d in batch:
        x = ib.Query(q, max_results); x.CoverageDepth = d; qq.append(x)
    h = eng.UploadBatch(qq)
    try:
        eng.RunBatch(h); b = eng.DownloadBatch(h, eng.PackBatch(qq))
    finally:
        eng.FreeBatch(h)
    bad = []
    for d in sorted({d for _, _, d in batch}):
        idx = [i for i, (_, _, dd) in enumerate(batch) if dd == d]
        ok, os_, ot, on, ost = orc.search_batch([batch[i][0] for i in idx], max_results, d, True, None, threads=8)
        for j, i in enumerate(idx):
            n = int(on[j])
            if ost[j] != 0 or b["status"][i] & ~8:
                bad.append((batch[i][1], d, "status", int(ost[j]), int(b["status"][i])))
                continue
            if not (b["n"][i] == n and np.array_equal(b["keys"][i, :n], ok[j, :n])
                    and np.array_equal(b["scores"][i, :n].view(np.uint32), os_[j, :n].view(np.uint32)) and np.array_equal(b["ties"][i, :n], ot[j, :n])):
                bad.append((batch[i][1], d, b["keys"][i, :3].tolist(), ok[j, :3].tolist(), b["scores"][i, :3].tolist(), os_[j, :3].tolist()))
    return bad


def scorer_class(max_cnt, Ta, depth):
    """The scorer stage1_lookup queues a query for (ifx_stage1_score.h): 0 nothing to score, 1 light, 2 mid, 3 CTA."""
    if Ta == 0:
        return 0
    warp_ok = Ta <= 64 and depth <= 512
    return 1 if warp_ok and max_cnt <= 256 else 2 if warp_ok and max_cnt <= 512 else 3


def reach(eng, batch):
    """Run the batch once and read, per query, what Stage 1 did: n_cand, n_chunks, max_cnt, Ta, the class the rule gives at its
    depth; and the run's Stats."""
    qq = []
    for q, _, d in batch:
        x = ib.Query(q, 10); x.CoverageDepth = d; qq.append(x)
    h = eng.UploadBatch(qq)
    try:
        st = eng.RunBatch(h)
        dbg = np.zeros((len(qq), 24), np.int64); eng._gpu.ifx_debug_stage1_queries(h, dbg.ctypes.data_as(C.c_void_p))
    finally:
        eng.FreeBatch(h)
    rows = []
    for (q, name, d), r in zip(batch, dbg):
        n_cand, n_chunks, max_cnt, Ta = (int(r[k]) for k in (0, 7, 8, 9))
        rows.append(dict(name=name, depth=d, n_cand=n_cand, n_chunks=n_chunks, max_cnt=max_cnt, Ta=Ta,
                         cls=scorer_class(max_cnt, Ta, d) if n_cand > 0 else 0))
    return rows, st


def check_reach(rows, st, docs):
    """The fixture still reaches the edges the parity tests are meant to cover, and the routing counts match the rule."""
    assert st.s1_waves == 1            # the class counts of Stats cover the last wave only
    cls = np.array([r["cls"] for r in rows])
    assert (int((cls == 1).sum()), int((cls == 2).sum()), int((cls == 3).sum())) == (st.s1_light, st.s1_mid, st.s1_heavy)
    by = {k: [r for r in rows if r["cls"] == k] for k in (1, 2, 3)}
    got = lambda k, key: {r[key] for r in by[k]}
    # a single planted word's candidates are exactly its documents, a long query's exactly its host's
    for r in rows:
        name = r["name"].split("_")[0]
        if name in docs and name not in ("lc", "common"):
            assert r["n_cand"] == len(docs[name]), r
    # light: full 256-slot chunks, 64 terms, depth 512, and both sides of the 24-row tile of a 256-slot chunk
    assert 256 in got(1, "max_cnt") and 64 in got(1, "Ta") and 512 in got(1, "depth")
    assert {24, 25} <= {r["Ta"] for r in by[1] if 241 <= r["max_cnt"] <= 256}
    # mid: 257- and 512-slot chunks, both sides of the 12-row tile of a 512-slot chunk
    assert {257, 512} <= got(2, "max_cnt")
    assert {12, 13} <= {r["Ta"] for r in by[2] if 497 <= r["max_cnt"] <= 512}
    # CTA: 513 / 4 095 / 4 096-slot chunks; reached through Ta = 65 and through depth 513 with light-sized chunks; 6 / 7 terms (S1_TILE)
    assert {513, 4095, 4096} <= got(3, "max_cnt")
    assert any(r["Ta"] == 65 and r["max_cnt"] <= 256 and r["depth"] <= 512 for r in by[3])
    assert any(r["depth"] == 513 and r["max_cnt"] <= 256 and r["Ta"] <= 64 for r in by[3])
    assert {6, 7} <= got(3, "Ta")
    assert 1024 in got(3, "depth") and {1, 2, 3, 4, 5} <= got(1, "depth") | got(2, "depth") | got(3, "depth")


def trace(orc, text, depth):
    """The oracle's per-chunk MaxScore trace: rows [threshold at chunk start, candidates, matched pairs, skipped pairs, max bound of
    the skipped, heap updates]."""
    a = O.u16(text); out = np.zeros((8192, 6)); st = np.zeros(5, np.int64)
    n = O.lib().ifxo_stage1_trace(orc.h, O._p(a), len(a), depth, O._p(out), 8192, O._p(st))
    return out[:min(n, 8192)]


def check_trace(orc, rows, batch):
    """Per class: chunks where MaxScore skipped pairs while most matched pairs were scored, queries with many chunks behind a full
    heap, and a CTA chunk at depth 1 024 with more heap updates than SURV_CAP = 512 (its survivors spill to global memory)."""
    seen = {k: dict(skip=False, behind=0, updates=0) for k in (1, 2, 3)}
    for (q, _, d), r in zip(batch, rows):
        if r["cls"] == 0:
            continue
        tr = trace(orc, q, d); s = seen[r["cls"]]
        assert len(tr) == r["n_chunks"], (r, len(tr))
        s["skip"] |= bool(((tr[:, 3] > 0) & (tr[:, 2] > tr[:, 3])).any())
        s["behind"] = max(s["behind"], int((tr[:, 0] > 0).sum()))
        if d == 1024:
            s["updates"] = max(s["updates"], int(tr[:, 5].max()))
    for k in (1, 2, 3):
        assert seen[k]["skip"], k
        assert seen[k]["behind"] >= 10, (k, seen[k])
    assert seen[3]["updates"] > 512, seen[3]


def vector_scalar_differ(orc, docs):
    """Share of the planted candidates whose BM25+ term score (tf 1 and 2) differs between the Vector256 form (B / avgdl) * dl and
    the scalar form B * (dl / avgdl), in float32. Only these candidates show a wrong rank or a wrong vec_end in a score bit."""
    f = np.float32; K1, B, one = f(1.2), f(0.75), f(1)
    avgdl = f(orc.avgdl()); dl = orc.doc_lens()[np.concatenate([v for k, v in docs.items() if k not in ("lc", "common")])].astype(f)
    differ = np.zeros(len(dl), bool)
    for tf in (f(1), f(2)):
        nv = K1 * ((one - B) + (B / avgdl) * dl); ns = K1 * (one - B + B * (dl / avgdl))
        differ |= (tf * (K1 + one)) / (tf + nv) != (tf * (K1 + one)) / (tf + ns)
    return float(differ.mean())


def build(gpu_lib=None):
    texts, keys, deleted, docs = corpus()
    schema = [ib.Field("content")]
    eng = ib.SearchEngine(_gpu_lib=gpu_lib) if gpu_lib else ib.SearchEngine.CreateDefault()
    eng.IndexColumns(keys, schema, [texts], upload=False)
    img = C.cast(eng.image_ptr(), C.POINTER(_ImageHead)).contents
    flags = np.ctypeslib.as_array(img.deleted, shape=(N,)); flags[deleted] = 1
    img.n_live = int(N - flags.sum())
    eng._upload(eng.image_ptr())
    orc = O.OracleEngine([O.Field(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema])
    orc.load_image(eng.image_ptr())
    return eng, orc, docs
