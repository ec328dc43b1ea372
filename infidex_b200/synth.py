"""Deterministic synthetic corpus + query generator for the benchmark configs (SURVEY.md 8d / BASELINE.md 2).

Vocabulary: V lower-case ASCII pseudo-words (3-12 chars, syllable generator), rank-frequency Zipf(s=1.07).
Docs     : title = 1 + Poisson(2.7) words (cap 12); description = 8 + Poisson(7) words; year U{1950..2024};
           rating U{1.0..10.0} step 0.1; genre in 20 categories (Zipf).
Queries  : 1-3 consecutive title words of a random doc; p=0.30 one edit (sub/ins/del/transpose) in a word of len >= 4;
           p=0.20 last word cut to a prefix of >= 3 chars; p=0.05 a word absent from the doc prepended.
Documents come from csrc/ifx_synth.cpp (multi-threaded; one SplitMix64 stream per document, seed 0x1F1DEC5); the vocabulary and the
queries from numpy Generator(PCG64(seed)).
"""
import numpy as np

SEED = 0x1F1DEC5
GENRES = ["drama", "comedy", "action", "thriller", "romance", "horror", "documentary", "crime", "adventure", "family",
          "fantasy", "mystery", "animation", "biography", "history", "music", "war", "western", "sport", "musical"]
_CONS = "bcdfghjklmnprstvwz"
_VOW = "aeiou"


def make_vocab(V=400_000, seed=SEED):
    rng = np.random.Generator(np.random.PCG64(seed ^ 0xA5A5))
    words, seen = [], set()
    cons, vow = np.array(list(_CONS)), np.array(list(_VOW))
    while len(words) < V:
        n = (V - len(words)) * 2 + 1000
        nsyl = rng.integers(1, 5, n)
        c1 = cons[rng.integers(0, len(cons), (n, 4))]; v1 = vow[rng.integers(0, len(vow), (n, 4))]; c2 = cons[rng.integers(0, len(cons), (n, 4))]
        tail = rng.random((n, 4)) < 0.35
        for i in range(n):
            w = "".join(c1[i, k] + v1[i, k] + (c2[i, k] if tail[i, k] else "") for k in range(nsyl[i]))
            if 3 <= len(w) <= 12 and w not in seen:
                seen.add(w); words.append(w)
                if len(words) == V:
                    break
    lens = np.array([len(w) for w in words], np.int32)
    offs = np.zeros(V + 1, np.int64); np.cumsum(lens, out=offs[1:])
    blob = np.frombuffer("".join(words).encode("ascii"), np.uint8).astype(np.uint16)
    ranks = np.arange(1, V + 1, dtype=np.float64)
    cdf = np.cumsum(ranks ** -1.07); cdf /= cdf[-1]
    return {"words": words, "blob": blob, "offs": offs, "lens": lens, "cdf": cdf}


_hostlib = None


def _host():
    global _hostlib
    if _hostlib is None:
        import ctypes as C
        from . import _build
        _hostlib = C.CDLL(_build.build_host())
    return _hostlib


def _p(a):
    import ctypes as C
    return a.ctypes.data_as(C.c_void_p)


def gen_docs(n, vocab, seed=SEED, with_description=False, start=0, threads=None):
    """Columns for docs [start, start+n) of the corpus `seed` (csrc/ifx_synth.cpp: every document has its own SplitMix64 stream, so any
    range / thread count / shard split yields the same documents)."""
    import ctypes as C
    import os
    lib = _host(); th = threads or min(os.cpu_count() or 1, 64); multi = 1 if with_description else 0
    V = len(vocab["lens"]); lens = np.ascontiguousarray(vocab["lens"], np.int32); cdf = np.ascontiguousarray(vocab["cdf"], np.float64)
    twoff = np.zeros(n + 1, np.int64); tcoff = np.zeros(n + 1, np.int64)
    dwoff = np.zeros(n + 1 if multi else 1, np.int64); dcoff = np.zeros(n + 1 if multi else 1, np.int64)
    lib.ifx_synth_sizes(C.c_int64(n), C.c_int64(start), C.c_uint64(seed), multi, th, _p(lens), _p(cdf), V, _p(twoff), _p(tcoff), _p(dwoff), _p(dcoff))
    tids = np.zeros(max(int(twoff[-1]), 1), np.int32); tblob = np.zeros(max(int(tcoff[-1]), 1), np.uint16)
    dblob = np.zeros(max(int(dcoff[-1]), 1) if multi else 1, np.uint16)
    year = np.zeros(n, np.int64); rating = np.zeros(n, np.float64); genre = np.zeros(n, np.int64)
    blob = np.ascontiguousarray(vocab["blob"], np.uint16); offs = np.ascontiguousarray(vocab["offs"], np.int64)
    lib.ifx_synth_fill(C.c_int64(n), C.c_int64(start), C.c_uint64(seed), multi, th, _p(blob), _p(offs), _p(lens), _p(cdf), V,
                       _p(twoff), _p(tcoff), _p(dwoff), _p(dcoff), _p(tids), _p(tblob), _p(dblob), _p(year), _p(rating), _p(genre))
    out = {"n": n, "start": start, "seed": seed, "keys": np.arange(start, start + n, dtype=np.int64), "title": (tblob, tcoff), "title_ids": tids[: int(twoff[-1])], "title_off": twoff,
           "year": year, "rating": rating, "genre_id": genre}
    if multi:
        out["description"] = (dblob, dcoff)
    return out


def corpus_ref(n, seed=SEED):
    """A handle on the corpus `seed` of n documents that holds no documents: enough for gen_queries (titles are regenerated on demand)."""
    return {"n": n, "seed": seed, "virtual": True}


def _title_ids(docs, vocab, d):
    if not docs.get("virtual"):
        return docs["title_ids"][int(docs["title_off"][d]): int(docs["title_off"][d + 1])]
    import ctypes as C
    out = np.zeros(12, np.int32); cdf = vocab["cdf"]
    k = _host().ifx_synth_title_ids(C.c_int64(d), C.c_uint64(docs["seed"]), _p(cdf), len(cdf), _p(out))
    return out[:k]


def gen_queries(nq, docs, vocab, seed=SEED):
    """Query strings sampled from the titles of `docs` (a gen_docs result)."""
    rng = np.random.Generator(np.random.PCG64([seed, 0x51]))
    words = vocab["words"]; out = []
    alpha = "abcdefghijklmnopqrstuvwxyz"
    for _ in range(nq):
        d = int(rng.integers(0, docs["n"]))
        tid = _title_ids(docs, vocab, d); nt = len(tid)
        k = int(min(rng.integers(1, 4), nt)); s = int(rng.integers(0, nt - k + 1))
        ws = [words[i] for i in tid[s:s + k]]
        if rng.random() < 0.30:
            cand = [i for i, w in enumerate(ws) if len(w) >= 4]
            if cand:
                i = cand[int(rng.integers(0, len(cand)))]; w = ws[i]; p = int(rng.integers(0, len(w))); kind = int(rng.integers(0, 4))
                c = alpha[int(rng.integers(0, 26))]
                if kind == 0: w = w[:p] + c + w[p + 1:]
                elif kind == 1: w = w[:p] + c + w[p:]
                elif kind == 2: w = w[:p] + w[p + 1:]
                else:
                    p = min(p, len(w) - 2); w = w[:p] + w[p + 1] + w[p] + w[p + 2:]
                ws[i] = w
        if rng.random() < 0.20 and len(ws[-1]) > 3:
            ws[-1] = ws[-1][: int(rng.integers(3, len(ws[-1])))]
        if rng.random() < 0.05:
            title_set = set(int(x) for x in tid)
            while True:
                x = int(min(np.searchsorted(vocab["cdf"], rng.random()), len(words) - 1))
                if x not in title_set:
                    break
            ws.insert(0, words[x])
        out.append(" ".join(ws))
    return out


def _pack_choice(options, ids):
    """Pre-packed (uint16 blob, int64 offsets) string column whose row i is options[ids[i]] (no per-row Python objects)."""
    ids = np.asarray(ids, np.int64)
    ol = np.array([len(o) for o in options], np.int64); oo = np.zeros(len(options) + 1, np.int64); np.cumsum(ol, out=oo[1:])
    ob = np.frombuffer("".join(options).encode("utf-16-le"), np.uint16)
    wl = ol[ids]; offs = np.zeros(len(ids) + 1, np.int64); np.cumsum(wl, out=offs[1:])
    within = np.arange(int(offs[-1]), dtype=np.int64) - np.repeat(offs[:-1], wl)
    blob = ob[np.repeat(oo[ids], wl) + within] if len(within) else np.zeros(1, np.uint16)
    return np.ascontiguousarray(blob), offs


def schema_and_columns(docs, multi_field):
    """(schema, columns) for SearchEngine.IndexColumns / the oracle, per BASELINE.json configs."""
    from .engine import Field, Weight
    if not multi_field:      # configs[1]: new Document(i, title) -> single field "content", Weight.Med
        return [Field("content", None, Weight.Med)], [docs["title"]]
    genre = _pack_choice(GENRES, docs["genre_id"])
    schema = [Field("title", None, Weight.High), Field("description", None, Weight.Low),
              Field("year", None, Weight.Med, indexable=False, filterable=True, facetable=True),
              Field("rating", None, Weight.Med, indexable=False, filterable=True),
              Field("genre", None, Weight.Med, indexable=False, filterable=True, facetable=True)]
    return schema, [docs["title"], docs["description"], docs["year"], docs["rating"], genre]


def make_synonym_pairs(vocab, n_groups=5000, seed=SEED, n_frequent=50):
    """Seeded SynonymMap over the vocabulary: `n_groups` disjoint groups of 2-4 words of mixed lengths; the first groups take the
    `n_frequent` most frequent words, the rest random ones. Returns the ordered AddSynonym(a, b) calls AddSynonymGroup(group) makes."""
    rng = np.random.Generator(np.random.PCG64(seed ^ 0x5E5E))
    words = vocab["words"]; V = len(words)
    order = np.concatenate([np.arange(min(n_frequent, V)), rng.permutation(np.arange(min(n_frequent, V), V))])
    pairs, k = [], 0
    for g in range(n_groups):
        size = int(rng.integers(2, 5))
        grp = [words[int(i)] for i in order[k:k + size]]; k += size
        if len(grp) < 2:
            break
        for i in range(len(grp)):
            for j in range(i + 1, len(grp)):
                pairs.append((grp[i], grp[j]))
    return pairs
