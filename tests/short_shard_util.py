"""Shared pieces of the sharded short-query tests (CPU: gloo + the kernel emulation; GPU: two shards on one device): a synthetic corpus of
131 072 documents, split into two doc-id-range shards at 65 536, with hand-placed documents on both sides of the boundary, the queries
that reach every branch of the short-query path, and the comparison with the unsharded oracle."""
import numpy as np

import infidex_b200 as ib
from infidex_b200 import synth
from infidex_b200.engine import Field, Weight

N = 131_072
BOUNDARY = 65_536


def _place(titles, start, texts):
    for i, t in enumerate(texts):
        titles[start + i] = t


def corpus():
    """(keys, schema, columns) of the whole corpus. Cyrillic letters appear only in the hand-placed titles, so each case owns its letters."""
    vocab = synth.make_vocab(20_000)
    docs = synth.gen_docs(N, vocab)
    blob, off = docs["title"]
    titles = [blob[int(off[i]): int(off[i + 1])].tobytes().decode("utf-16-le") for i in range(N)]
    lo, hi = 1_000, BOUNDARY + 1_000          # hand-placed runs on shard 0 / shard 1
    # champions split across shards, tie-heavy (> 16 equal scores on both sides, so the introsort order matters)
    _place(titles, lo, ["жук лес%d" % (i % 3) if i % 5 else "старый жук" for i in range(40)])
    _place(titles, hi, ["жук лес%d" % (i % 3) if i % 7 else "ж" for i in range(40)])
    # a character with fewer champions than max_results
    _place(titles, lo + 100, ["юла", "юг", "море юла"]); _place(titles, hi + 100, ["юла юла", "юрта"])
    # every match on one shard
    _place(titles, hi + 200, ["щука %d" % i for i in range(7)])
    # two characters: >= 100 matches globally, < 100 on one shard -- and the reverse
    _place(titles, lo + 300, ["бор %d" % i for i in range(130)]); _place(titles, hi + 300, ["бор тихий %d" % i for i in range(30)])
    _place(titles, lo + 500, ["гол %d" % i for i in range(30)]); _place(titles, hi + 500, ["гол мяч %d" % i for i in range(130)])
    # the fuzzy fallback (< 100 matches)
    _place(titles, lo + 700, ["дым %d" % i for i in range(20)] + ["одно дело"] * 10); _place(titles, hi + 700, ["дым густой"] * 25 + ["поход"] * 10)
    # the max integer score lives on the other shard
    _place(titles, lo + 800, ["лень %d" % i for i in range(20)]); _place(titles, hi + 800, ["лень лень лень лень ленивый"])
    # "ми": 6 + 6 matches, the fuzzy fallback adds every title with an м or и
    _place(titles, lo + 900, ["мир %d" % i for i in range(6)]); _place(titles, hi + 900, ["мир вокруг %d" % i for i in range(6)])
    # mode 2 reached only globally: 6 + 6 matches of letters no other title holds (so the fuzzy fallback adds nothing), max_results 10
    _place(titles, lo + 1000, ["эфир %d" % i for i in range(6)]); _place(titles, hi + 1000, ["эфир тут %d" % i for i in range(6)])
    # coverage word hits on one shard only: "βγ" starts words on shard 0; shard 1 holds only fuzzy matches (β / γ deep inside long words)
    _place(titles, lo + 1100, ["βγ", "βγαλε", "βγω"]); _place(titles, hi + 1100, ["αλφαβητο", "καλοβολος"])
    # mode 0: 0 < prefix cardinality <= 500 and fewer matches than max_results
    _place(titles, lo + 950, ["пух %d" % i for i in range(5)]); _place(titles, hi + 950, ["пух белый", "пушок пух", "пух", "тёплый пух", "пух 9"])
    schema = [Field("title", None, Weight.High), Field("year", None, Weight.Med, indexable=False, filterable=True, facetable=True)]
    return np.arange(N, dtype=np.int64), schema, [titles, docs["year"]], vocab


YEAR_MIN = 1990


def year_filter():
    return ib.Filter.Range("year", min=YEAR_MIN)


# (text, max_results, filter?, facets?, coverage?)
SHORT_CASES = [
    ("ж", 10, False, False, True), ("ж", 64, False, False, True), ("ж", 100, False, False, True), ("ж", 5, True, True, True),
    ("ю", 10, False, False, True), ("щ", 10, False, False, True), ("щу", 10, False, False, True),
    ("бо", 10, False, False, True), ("го", 10, False, False, True), ("б г", 10, False, False, True), ("г б", 20, False, False, True),
    ("бо", 20, True, True, True), ("б г", 10, True, True, True),
    ("ды", 10, False, False, True), ("ле", 10, False, False, True), ("ми", 10, False, False, True), ("ми", 20, False, False, True),
    ("пу", 50, False, False, True), ("пу", 50, False, False, False), ("эф", 10, False, False, True), ("βγ", 100, False, False, True),
    ("a", 10, False, False, True), ("s", 100, False, False, True), ("e", 10, True, True, True), ("st", 10, False, False, True),
    ("a b", 10, False, False, True), ("an", 25, False, False, True), ("x", 3, False, False, True),
]


def make_query(case):
    text, mx, flt, facets, cov = case
    q = ib.Query(text, mx); q.EnableFacets = facets; q.EnableCoverage = cov
    if flt:
        q.Filter = year_filter()
    return q


def ngram_texts(vocab, n=24):
    return synth.gen_queries(n, synth.corpus_ref(N), vocab)


def signature(r, ignore_status=0):
    """(records, TotalCandidates, status without the flags `ignore_status`, facets) of a Result."""
    return ([(e.DocumentId, int(np.float32(e.Score).view(np.uint32)), int(e.Tiebreaker)) for e in r.Records], int(r.TotalCandidates), int(r.Status) & ~ignore_status,
            None if r.Facets is None else {f: [(v, int(c)) for v, c in vs] for f, vs in r.Facets.items()})


def oracle_engine(keys, schema, cols):
    from oracle.oracle import Field as OField
    from oracle.oracle import OracleEngine
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema]); orc.index_columns(keys, cols)
    return orc


def check_shard_facts(cases, counts, info):
    """The cases hold the per-shard situations they are named for. counts: [W][nq] every shard's Stage-1 list length; info: [nq][W][8]
    every shard's truncation facts (info[.., 0]: max coverage word hits) -- ShardedSearchEngine.last_s1_counts / last_shard_info."""
    at = {c[:2]: i for i, c in enumerate(cases)}
    n = lambda key: [int(counts[r][at[key]]) for r in range(len(counts))]
    assert max(n(("эф", 10))) < 10 <= sum(n(("эф", 10))), n(("эф", 10))          # mode 2 only on the global count
    assert n(("бо", 10))[1] < 100 <= sum(n(("бо", 10))), n(("бо", 10))          # >= 100 matched globally, < 100 on shard 1
    assert n(("го", 10))[0] < 100 <= sum(n(("го", 10))), n(("го", 10))          # and the reverse
    hits = [int(x) for x in info[at[("βγ", 100)], :, 0]]
    assert max(hits) > 0 and min(hits) == 0, hits                                  # word hits on one shard, none on the other


def compare_with_oracle(orc, cases, sigs):
    """Mismatches between the merged sharded answers and the unsharded oracle: ids, score bits, tiebreakers, TotalCandidates, status. (Facet
    tables are not compared: a shard's batch reports none.)"""
    bad = []
    for case, (recs, total, status, facets) in zip(cases, sigs):
        text, mx, flt, fac, cov = case
        x = orc.search(text, mx, coverage=cov, filter_bytes=year_filter().bytecode() if flt else None, facets=fac)
        want = list(zip(x["keys"], x["scores"].view(np.uint32).tolist(), x["ties"]))
        if recs != want or total != x["total"] or status != x["status"]:
            bad.append((case, "records" if recs != want else ("total %d != %d" % (total, x["total"]) if total != x["total"] else "status %d != %d" % (status, x["status"]))))
    return bad
