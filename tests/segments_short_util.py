"""Shared pieces of the short-query tests on indexes whose documents share a DocumentKey (segments): a synthetic multi-field corpus whose keys
repeat -- contiguous runs of 2-3 segments for about a third of the keys, plus keys scattered far apart -- with hand-placed titles for each
branch of the short-query path, and the queries that reach them. Keys are a permutation, so their order is not the documents' order."""
import numpy as np

from infidex_b200 import synth

C4_FILTER = "year >= 2000 AND rating > 7.0"


def _place(titles, keys, start, texts, key_of):
    for i, t in enumerate(texts):
        titles[start + i] = t
        keys[start + i] = key_of(i)


def corpus(n, seed=11, repeated=True):
    """(keys, schema, columns). repeated=False: the same columns with unique keys (the control)."""
    vocab = synth.make_vocab(20_000)
    docs = synth.gen_docs(n, vocab, with_description=True)
    schema, cols = synth.schema_and_columns(docs, True)
    blob, off = cols[0]
    titles = [blob[int(off[i]): int(off[i + 1])].tobytes().decode("utf-16-le") for i in range(n)]
    rng = np.random.Generator(np.random.PCG64(seed))
    slot = np.empty(n, np.int64); k = 0; i = 0
    while i < n:                                    # about a third of the keys take 2 or 3 contiguous segments
        run = 1 if rng.random() < 2 / 3 else int(rng.integers(2, 4))
        slot[i: i + run] = k; k += 1; i += run
    far = rng.choice(np.arange(n // 2, n), size=max(n // 100, 4), replace=False)      # scattered: a late document takes an early key
    slot[far] = slot[far - n // 2]
    slot[n - 1] = slot[3]                           # the same key at doc 3 and at the last doc
    nxt = [int(slot.max()) + 1]

    def fresh(run):                                  # a new key for every `run` consecutive hand-placed documents
        base = nxt[0]; nxt[0] += 10_000
        return lambda j: base + j // run
    h = n // 8
    # one character, champion list (64 entries) with duplicate keys among the first max: pairs of segments, tie-heavy
    _place(titles, slot, h, ["ж лес%d" % (j % 3) if j % 5 else "ж" for j in range(90)], fresh(2))
    # one character, scan: more than 64 champions' worth of matches, three segments per key, one key scattered
    _place(titles, slot, 2 * h, ["ю%d юла" % j if j % 4 else "море юг" for j in range(300)], fresh(3))
    slot[n - 2] = slot[2 * h]; titles[n - 2] = "ю"
    # two characters, 60 keys x 3 segments = 180 matched documents but < 100 matched keys: the fuzzy fallback runs
    _place(titles, slot, 3 * h, ["бор %d" % (j // 3) for j in range(180)], fresh(3))
    # two characters, 150 single-segment keys: no fallback
    _place(titles, slot, 3 * h + 400, ["гол %d" % j for j in range(150)], fresh(1))
    # two characters, 120 documents in 40 keys: >= 100 documents, < 100 keys
    _place(titles, slot, 3 * h + 600, ["дым %d" % j for j in range(120)], fresh(3))
    # the first-token prefix holds for a later segment only: the key's first document does not start with the query (or does not match at all)
    _place(titles, slot, 4 * h, [("тёмный вечер", "лето тёплое")[j % 2] if j < 20 else ("старый лес", "лес густой")[j % 2] for j in range(40)], fresh(2))
    _place(titles, slot, 4 * h + 100, ["лес %d" % j for j in range(6)], fresh(1))
    slot[5] = slot[4 * h]; titles[5] = "вечер без лета"       # and a scattered key whose first document is doc 5
    # a character whose every key is unique (the unique-key queries of a mixed batch)
    _place(titles, slot, 5 * h, ["щука %d" % j for j in range(30)], fresh(1))
    # several short words
    _place(titles, slot, 5 * h + 100, ["мы и вы %d" % (j // 2) for j in range(40)], fresh(2))
    perm = np.random.Generator(np.random.PCG64(seed + 1)).permutation(int(slot.max()) + 1).astype(np.int64)
    keys = perm[slot] if repeated else np.arange(n, dtype=np.int64)[rng.permutation(n)]
    cols = [titles] + list(cols[1:])
    return keys, schema, cols


SHORT = ["ж", "ю", "щ", "бо", "го", "ды", "ле", "ло", "ми", "мы и", "и вы", "м в", "a", "s", "st", "an", "x", "th", "e r"]
