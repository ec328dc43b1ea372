"""Shared pieces of the sharded filter / facet tests (CPU: gloo + the kernel emulation; GPU: two shards on one device): the query variants,
the corpus keys (not monotone in the internal id, so the blank browse query's internal-id order differs from DocumentId order), and the
acceptance rule against the unsharded oracle.

The rule: the hosts filter after the merged list was truncated to <= max records, so whenever a query's UNFILTERED sharded records equal the
oracle's, its filtered answer must equal the oracle's exactly -- records, score bits, tiebreakers, TotalCandidates, status and facet tables.
The unfiltered mismatches themselves come from the Stage-1 tie waiver and are held to test_sharded.py's ceiling."""
import numpy as np

import infidex_b200 as ib

C4_FILTER = "year >= 2000 AND rating > 7.0"
VARIANTS = ("plain", "filter+facets", "facets", "filter")


def keys_for(ids, n):
    """DocumentKeys of internal ids `ids` in a corpus of n documents: a bijection that is not monotone (n is not a multiple of 7919)."""
    return (np.asarray(ids, np.int64) * 7919 + 13) % n


def make(text, mx, variant, flt, coverage=True):
    q = ib.Query(text, mx)
    q.Filter = flt if "filter" in variant else None
    q.EnableFacets = "facets" in variant
    q.EnableCoverage = coverage
    return q


def batch(texts, flt, mx=10, coverage=True, blanks=True):
    """Every text in every variant, then (blanks) blank browse queries, with and without the filter."""
    qs = [make(t, mx, v, flt, coverage) for t in texts for v in VARIANTS]
    if blanks:
        qs += [make("", 10, "filter+facets", flt), make("", 25, "facets", flt), make("", 3, "filter+facets", flt)]
    return qs


def three_char_texts(vocab, n=24):
    """3-character queries over the prefixes of the most frequent words (prefix docsets of > 500 documents at the test corpus sizes): with
    max_results 10 the <= 3-character rule cuts their Stage-1 list at max; with a max_results above the coverage depth they skip the
    coverage stage and return the whole list."""
    out = []
    for w in vocab["words"]:
        if w[:3] not in out:
            out.append(w[:3])
        if len(out) == n:
            break
    return out


def whole_list_batch(texts, three, flt):
    """Queries answered with their whole Stage-1 list or a list cut at max: EnableCoverage off, and 3-character queries. The whole-list
    queries ask for max_results >= the list's length (the coverage depth, 500), so the unfiltered records ARE the list, and the acceptance
    rule's gate covers every record the filter and the facets see (documents tied at the Stage-1 cut may differ: the waiver)."""
    return batch(texts, flt, mx=500, coverage=False, blanks=False) + batch(three, flt, blanks=False) + batch(three[: len(three) // 2], flt, mx=600, blanks=False)


def oracle_signature(orc, q, flt_bytes):
    x = orc.search(q.Text, q.MaxNumberOfRecordsToReturn, coverage=q.EnableCoverage, filter_bytes=flt_bytes if q.Filter is not None else None, facets=q.EnableFacets)
    fo = None
    if q.EnableFacets:
        fo = {}
        for f, v, c in x["facets"]:
            fo.setdefault(f, []).append((v, c))
    return (list(zip(x["keys"], x["scores"].view(np.uint32).tolist(), x["ties"])), x["total"], x["status"], fo)


def check(orc, queries, sigs, flt_bytes):
    """Applies the acceptance rule to the output of batch(). Returns (unfiltered mismatches, their DocumentId-order mismatches, number of
    filtered / faceted answers checked exactly, failures)."""
    want = [oracle_signature(orc, q, flt_bytes) for q in queries]
    nv = len(VARIANTS); plain_bad = ids_bad = checked = 0; bad = []; i0 = 0
    while i0 < len(queries):
        if queries[i0].Text == "":      # a blank browse query: no waiver applies
            checked += 1
            if sigs[i0] != want[i0]:
                bad.append(("<blank>", queries[i0].MaxNumberOfRecordsToReturn, sigs[i0], want[i0]))
            i0 += 1; continue
        if sigs[i0][0] != want[i0][0]:
            plain_bad += 1; ids_bad += [r[0] for r in sigs[i0][0]] != [r[0] for r in want[i0][0]]
        else:
            if sigs[i0] != want[i0]:
                bad.append((queries[i0].Text, "plain", sigs[i0], want[i0]))
            for k in range(1, nv):
                checked += 1
                if sigs[i0 + k] != want[i0 + k]:
                    bad.append((queries[i0].Text, queries[i0].EnableCoverage, queries[i0].MaxNumberOfRecordsToReturn, VARIANTS[k], sigs[i0 + k], want[i0 + k]))
        i0 += nv
    return plain_bad, ids_bad, checked, bad
