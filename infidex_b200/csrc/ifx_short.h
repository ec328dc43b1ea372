// infidex_b200 -- Stage 1 of queries WITHOUT a word of >= 3 characters (SURVEY.md 8f-1): the reference routes them past the n-gram index
// (Scoring/SearchPipeline.cs:208-297) to
//   ShortQueryResolver champion lists            Indexing/ShortQuery/ShortQueryResolver.cs:83-160,233-311   (one character, small result sizes)
//   ShortQueryProcessor.SearchSingleCharacter     Scoring/ShortQueryProcessor.cs:19-150                     (one character: scan of every document)
//   ShortQueryProcessor.SearchShortQuery          Scoring/ShortQueryProcessor.cs:152-435                    (prefix patterns over the term dictionary,
//                                                                                                           fuzzy fallback over ALL terms, final scores)
// Such queries are rare and touch the whole corpus by construction, so each one runs as a few grid-wide launches over per-index scratch arrays
// (an int and a float per document) instead of inside the per-CTA pipeline; the result is the same Stage-1 list (doc, score, key; score
// descending, key ascending) the rest of the pipeline consumes, plus the number of matched documents (Result.TotalCandidates). Where
// DocumentKeys repeat, all of it is per key (sq_slot).
// Written against ifx::Ctx like everything else: `blk` / `nblk` stand for blockIdx / gridDim so the test build can run the same code.
#pragma once
#include "ifx_stage1.h"
#include "ifx_cov.h"

namespace ifx {

constexpr int SQ_KB = 1024;           // top-K capacity of the selection (>= depth and >= max_results of the query)
constexpr int SQ_TERMS = 4096;        // ShortQueryProcessor: terms collected per prefix pattern
constexpr int SQ_PATTERNS = 4;

struct SqScratch { int32_t* vi; float* vf; int32_t* terms; int32_t* tmult; int32_t* counters;       // counters: [0] matched keys, [1] term-list length, [2] max int score, [3] total with score > 0
                   float* cand_score; int64_t* cand_key; int32_t* cand_doc; int32_t* cand_n;      // [nblk][SQ_KB] per-block survivors of the selection
                   uint32_t* seen; uint32_t* kpre; };     // repeated keys only (null otherwise): bit per document "in a processed posting list",
                                                          // bit per key slot "some matched segment's text starts with the query"
// Repeated DocumentKeys (ix.key_first non-null): the reference accumulates SearchShortQuery per KEY and consolidates the other paths per key
// (ShortQueryProcessor.cs:281-296,355-380, SegmentProcessor.cs:15-37). Every per-key quantity lives in the slot of the key's first live
// document, key_first[d]; the other documents' slots stay 0, so the selection below never sees two entries of one key.
IFX_FN int sq_slot(const DevIndex& ix, int doc) { return ix.key_first ? ix.key_first[doc] : doc; }
IFX_FN bool sq_bit(const uint32_t* b, int i) { return (b[i >> 5] >> (i & 31)) & 1u; }
// vf[slot] = max(vf[slot], s) for s > 0: positive floats order as their bit patterns
IFX_FN void sq_max_into(float* p, float s) {
#ifdef IFX_EMU
    int v; memcpy(&v, &s, 4); atomic_max(reinterpret_cast<int*>(p), v);
#else
    atomic_max(reinterpret_cast<int*>(p), __float_as_int(s));
#endif
}

// ToLowerInvariant(IndexedText) of one document: the raw text where it differs from the normalised one, else the normalised text
IFX_FN void sq_doc_text(const DevIndex& ix, int doc, const uint16_t*& p, int& n) {
    if (ix.n_raw > 0) { int64_t i = lower_bound_i32(ix.raw_doc, 0, ix.n_raw, doc); if (i < ix.n_raw && ix.raw_doc[i] == doc) { p = ix.raw_chars + ix.raw_off[i]; n = (int)(ix.raw_off[i + 1] - ix.raw_off[i]); return; } }
    const int64_t t0 = ix.text_off[doc]; p = ix.text + t0; n = (int)(ix.text_off[doc + 1] - t0);
}
IFX_FN bool sq_is_ws(const DevIndex& ix, uint16_t c) { return ix.cflags[c] & 2; }

// ---- one character: ShortQueryProcessor.SearchSingleCharacter, one document per thread ------------------------------------------------------
IFX_FN float sq_single_char_score(const DevIndex& ix, int doc, uint16_t ch) {
    const uint16_t* t; int n; sq_doc_text(ix, doc, t, n);
    int char_count = 0, first_char = -1, n_words = 0, ws_count = 0, first_word = 0x7fffffff; bool any_exact = false, first_exact = false;
    for (int i = 0; i < n;) {
        while (i < n && delim_c(ix, lo_c(ix, t[i]))) { if (lo_c(ix, t[i]) == ch) { char_count++; if (first_char < 0) first_char = i; } i++; }
        if (i >= n) break;
        const int b = i; while (i < n && !delim_c(ix, lo_c(ix, t[i]))) { if (lo_c(ix, t[i]) == ch) { char_count++; if (first_char < 0) first_char = i; } i++; }
        if (lo_c(ix, t[b]) == ch) { ws_count++; if (n_words < first_word) first_word = n_words; if (i - b == 1) { any_exact = true; if (n_words == 0) first_exact = true; } }
        n_words++;
    }
    if (char_count == 0) return 0.f;
    const bool word_start = ws_count > 0; const bool title_eq = n == 1 && lo_c(ix, t[0]) == ch;
    int prec = 0; if (word_start) { prec |= 128; if (first_word == 0) prec |= 64; } if (any_exact) prec |= 32; if (first_exact) prec |= 16; if (title_eq) prec |= 8; if (n_words <= 3) prec |= 32;
    float base;
    if (word_start) { int pc = 255 - (first_word * 16 < 240 ? first_word * 16 : 240), dc = ws_count * 8 < 32 ? ws_count * 8 : 32; int r = pc + dc; r = r < 0 ? 0 : (r > 255 ? 255 : r); base = (float)r / 255.f; }
    else { int fc = first_char > 0 ? first_char : 0; int pc = 200 - (fc * 4 < 180 ? fc * 4 : 180), dc = char_count * 4 < 40 ? char_count * 4 : 40; int r = pc + dc; r = r < 0 ? 0 : (r > 200 ? 200 : r); base = (float)(r > 1 ? r : 1) / 255.f; }
    return (float)prec + base;
}

// ---- several short words / two characters: ShortQueryProcessor.SearchShortQuery --------------------------------------------------------------
struct SqPatterns { uint16_t pat[SQ_PATTERNS][MAX_QLEN + 2]; int len[SQ_PATTERNS]; int n; };
IFX_FN void sq_build_patterns(const uint16_t* q, int qlen, SqPatterns& P) {       // BuildPrefixPatterns(searchLower, 3, 2) + " " + searchLower
    P.n = 0; const int pad = 2, mis = 3;
    for (int i = 0; i < mis && i < pad + qlen; i++) { const int pc = pad - i > 0 ? pad - i : 0; int qc = mis - pc; if (qc > qlen) qc = qlen;
        if (qc > 0) { int L = 0; for (int k = 0; k < pc; k++) P.pat[P.n][L++] = PAD; for (int k = 0; k < qc; k++) P.pat[P.n][L++] = q[k]; P.len[P.n++] = L; } }
    { int L = 0; P.pat[P.n][L++] = u' '; for (int k = 0; k < qlen; k++) P.pat[P.n][L++] = q[k]; P.len[P.n++] = L; }
}
IFX_FN int sq_cmp_term_prefix(const DevIndex& ix, int sorted_pos, const uint16_t* pat, int plen) {   // term (first plen units) vs pattern: <0, 0 (term starts with it), >0
    const int ord = ix.term_sorted[sorted_pos]; const uint16_t* s = ix.terms.chars + ix.terms.off[ord]; const int L = (int)(ix.terms.off[ord + 1] - ix.terms.off[ord]);
    const int n = L < plen ? L : plen; for (int i = 0; i < n; i++) if (s[i] != pat[i]) return s[i] < pat[i] ? -1 : 1;
    return L >= plen ? 0 : -1;
}
// thread 0 of one block: the first min(count, 4096) dictionary terms under every pattern, in trie DFS (= ordinal-lexicographic) order, weight 10
IFX_FN void sq_collect_pattern_terms(const DevIndex& ix, const SqPatterns& P, SqScratch S) {
    int nt = 0;
    for (int k = 0; k < P.n; k++) {
        int lo = 0, hi = ix.terms.n; while (lo < hi) { int mid = (lo + hi) >> 1; if (sq_cmp_term_prefix(ix, mid, P.pat[k], P.len[k]) < 0) lo = mid + 1; else hi = mid; }
        int b = lo; hi = ix.terms.n; while (lo < hi) { int mid = (lo + hi) >> 1; if (sq_cmp_term_prefix(ix, mid, P.pat[k], P.len[k]) <= 0) lo = mid + 1; else hi = mid; }
        int cnt = lo - b; if (cnt > SQ_TERMS) cnt = SQ_TERMS;
        for (int i = 0; i < cnt; i++) { S.terms[nt] = ix.term_sorted[b + i]; S.tmult[nt] = 10; nt++; }
    }
    S.counters[1] = nt;
}
// ProcessTermMatches over one term: score[key] += weight * mult for every live document of its posting list (one warp per term)
IFX_FN void sq_process_term(const Ctx& c, const DevIndex& ix, int ord, int mult, SqScratch S) {
    if (ix.df[ord] <= 0) return;
    const int64_t r0 = ix.row_ptr[ord], r1 = ix.row_ptr[ord + 1];
    for (int64_t i = r0 + c.lane(); i < r1; i += Ctx::WS) { const int d = ix.post_doc[i]; if (ix.deleted[d]) continue;
        const int old = atomic_add(&S.vi[sq_slot(ix, d)], (int)ix.post_tf[i] * mult); if (old == 0) atomic_add(&S.counters[0], 1);
        if (S.seen && !sq_bit(S.seen, d)) atomic_or(&S.seen[d >> 5], 1u << (d & 31)); }
}
// ToLowerInvariant(IndexedText).StartsWith(searchLower) of one document (ProcessTermMatches, ShortQueryProcessor.cs:281-296)
IFX_FN bool sq_first_prefix(const DevIndex& ix, int doc, const uint16_t* q, int qlen) {
    const uint16_t* t; int n; sq_doc_text(ix, doc, t, n);
    if (n < qlen) return false;
    for (int k = 0; k < qlen; k++) if (lo_c(ix, t[k]) != q[k]) return false;
    return true;
}
// ProcessFuzzyFallback (matched < 100): every dictionary term that does not start with a pattern and holds a query character
IFX_FN int sq_fuzzy_weight(const DevIndex& ix, int ord, const SqPatterns& P, const uint16_t* q, int qlen) {
    const uint16_t* s = ix.terms.chars + ix.terms.off[ord]; const int L = (int)(ix.terms.off[ord + 1] - ix.terms.off[ord]);
    for (int k = 0; k < P.n; k++) { if (L >= P.len[k]) { bool eq = true; for (int i = 0; i < P.len[k]; i++) if (s[i] != P.pat[k][i]) { eq = false; break; } if (eq) return 0; } }
    bool boundary = false; int cm = 0;
    for (int j = 0; j < qlen; j++) { const uint16_t qc = q[j]; bool wb = false, any = false;
        for (int i = 0; i < L; i++) { if (s[i] == qc) { any = true; if (i > 0 && s[i - 1] == u' ') { wb = true; break; } } }
        if (wb) { boundary = true; cm++; } else if (any) cm++; }
    return (boundary || cm > 0) ? (boundary ? 2 : 1) : 0;
}
// BuildFinalScores / ComputePrecedence for one matched key, read from its first live document `doc`. `key_prefix`: the key's first-token-prefix
// flag when keys repeat (taken from whichever segment matched), -1 to read it from `doc` itself
IFX_FN float sq_final_score(const DevIndex& ix, int doc, int v, int vmax, const uint16_t* q, int qlen, int key_prefix) {
    const float normalized = vmax > 0 ? (float)v / (float)vmax : (float)v / 255.f;
    const uint16_t* t; int n; sq_doc_text(ix, doc, t, n);
    // query tokens
    int qb[MAX_QLEN / 2 + 1], qe[MAX_QLEN / 2 + 1], nq = 0;
    for (int i = 0; i < qlen;) { while (i < qlen && delim_c(ix, q[i])) i++; if (i >= qlen) break; qb[nq] = i; while (i < qlen && !delim_c(ix, q[i])) i++; qe[nq++] = i; }
    auto word_eq = [&](int b, int e, const uint16_t* w, int wl) { if (e - b != wl) return false; for (int k = 0; k < wl; k++) if (lo_c(ix, t[b + k]) != w[k]) return false; return true; };
    int prec = 0, n_words = 0;
    if (nq >= 2) {
        unsigned long long seen = 0;       // which query tokens (first 64) equal some word
        for (int i = 0; i < n;) { while (i < n && delim_c(ix, lo_c(ix, t[i]))) i++; if (i >= n) break; const int b = i; while (i < n && !delim_c(ix, lo_c(ix, t[i]))) i++;
            for (int k = 0; k < nq && k < 64; k++) if (!((seen >> k) & 1ULL) && word_eq(b, i, q + qb[k], qe[k] - qb[k])) seen |= 1ULL << k;
            n_words++; }
        int tm = 0; for (int k = 0; k < nq && k < 64; k++) if ((seen >> k) & 1ULL) tm++;
        const bool all = tm == nq;
        if (all) { prec |= 8; if (n_words <= nq + 1) prec |= 2; } else if (tm > 0) prec |= 4;
    } else {
        bool any_exact = false, first_exact = false;
        for (int i = 0; i < n;) { while (i < n && delim_c(ix, lo_c(ix, t[i]))) i++; if (i >= n) break; const int b = i; while (i < n && !delim_c(ix, lo_c(ix, t[i]))) i++;
            if (word_eq(b, i, q, qlen)) { any_exact = true; if (n_words == 0) first_exact = true; }
            n_words++; }
        int tb = 0, te = n; while (tb < te && sq_is_ws(ix, lo_c(ix, t[tb]))) tb++; while (te > tb && sq_is_ws(ix, lo_c(ix, t[te - 1]))) te--;
        const bool title_eq = word_eq(tb, te, q, qlen);
        const bool first_prefix = key_prefix >= 0 ? key_prefix != 0 : sq_first_prefix(ix, doc, q, qlen);
        if (any_exact) prec |= 1; if (first_prefix) prec |= 2; if (first_exact) prec |= 4; if (title_eq) prec |= 8;
    }
    return (float)prec + normalized;
}

// ---- exact top-K by (score descending, key ascending) over the per-document float scores (0 = not matched) --------------------------------------
struct SqTopShared { float score[2 * SQ_KB]; int64_t key[2 * SQ_KB]; int32_t doc[2 * SQ_KB]; ScanTmp scan; int bcast[4]; };
IFX_FN bool sq_before(const SqTopShared& sh, int a, int b) { if (sh.score[a] != sh.score[b]) return sh.score[a] > sh.score[b]; if (sh.key[a] != sh.key[b]) return sh.key[a] < sh.key[b]; return sh.doc[a] < sh.doc[b]; }
IFX_FN void sq_sort_desc(const Ctx& c, SqTopShared& sh, int n2) {      // bitonic over the first n2 (power of two) entries
    const int NT = c.nthreads();
    for (int k = 2; k <= n2; k <<= 1) for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = c.tid(); i < n2; i += NT) { int l = i ^ j; if (l > i) { bool up = (i & k) == 0; bool sw = up ? sq_before(sh, l, i) : sq_before(sh, i, l);
            if (sw) { float x = sh.score[i]; sh.score[i] = sh.score[l]; sh.score[l] = x; int64_t y = sh.key[i]; sh.key[i] = sh.key[l]; sh.key[l] = y; int z = sh.doc[i]; sh.doc[i] = sh.doc[l]; sh.doc[l] = z; } } }
        c.sync();
    }
}
IFX_FN void sq_clear(const Ctx& c, SqTopShared& sh, int from, int to) { for (int i = from + c.tid(); i < to; i += c.nthreads()) { sh.score[i] = -1.f; sh.key[i] = 0x7fffffffffffffffLL; sh.doc[i] = 0x7fffffff; } c.sync(); }
// block `blk` of `nblk`: best SQ_KB of its slice of documents -> S.cand_*[blk]
IFX_FN void sq_topk_stage1(const Ctx& c, const DevIndex& ix, SqScratch S, SqTopShared& sh, int blk, int nblk) {
    const int NT = c.nthreads(); const int64_t per = ((int64_t)ix.n_docs + nblk - 1) / nblk; const int64_t d0 = per * blk, d1 = d0 + per < ix.n_docs ? d0 + per : ix.n_docs;
    sq_clear(c, sh, 0, 2 * SQ_KB); int ntile = 0, total = 0;
    for (int64_t base = d0; base < d1; base += NT) {
        const int64_t d = base + c.tid(); const bool m = d < d1 && S.vf[d] > 0.f;
        int tot; const int off = block_excl_scan(c, m ? 1 : 0, sh.scan, tot);
        if (m) { const int at = SQ_KB + ntile + off; sh.score[at] = S.vf[d]; sh.key[at] = ix.doc_key[d]; sh.doc[at] = (int)d; }
        ntile += tot; total += tot; c.sync();
        if (ntile + NT > SQ_KB) { sq_sort_desc(c, sh, 2 * SQ_KB); sq_clear(c, sh, SQ_KB, 2 * SQ_KB); ntile = 0; }      // the tile is full: keep the best SQ_KB of (best so far, tile)
    }
    if (ntile > 0) { sq_sort_desc(c, sh, 2 * SQ_KB); sq_clear(c, sh, SQ_KB, 2 * SQ_KB); }
    for (int i = c.tid(); i < SQ_KB; i += NT) { const size_t o = (size_t)blk * SQ_KB + i; S.cand_score[o] = sh.score[i]; S.cand_key[o] = sh.key[i]; S.cand_doc[o] = sh.doc[i]; }
    if (c.tid() == 0) { S.cand_n[blk] = total < SQ_KB ? total : SQ_KB; atomic_add(&S.counters[3], total); }
    c.sync();
}
// one block: merge of the per-block survivors -> the query's Stage-1 list (first `keep` entries) and its total
IFX_FN void sq_topk_stage2(const Ctx& c, SqScratch S, SqTopShared& sh, int nblk, int keep, int64_t* out_key, int32_t* out_doc, float* out_score, int32_t* out_n, int32_t* out_total) {
    const int NT = c.nthreads(); sq_clear(c, sh, 0, 2 * SQ_KB);
    for (int b = 0; b < nblk; b++) {
        const int nb = S.cand_n[b]; if (nb == 0) continue;
        for (int i = c.tid(); i < nb; i += NT) { const size_t o = (size_t)b * SQ_KB + i; sh.score[SQ_KB + i] = S.cand_score[o]; sh.key[SQ_KB + i] = S.cand_key[o]; sh.doc[SQ_KB + i] = S.cand_doc[o]; }
        c.sync(); sq_sort_desc(c, sh, 2 * SQ_KB); sq_clear(c, sh, SQ_KB, 2 * SQ_KB);
    }
    const int total = S.counters[3]; const int n = total < keep ? total : keep;
    for (int i = c.tid(); i < n; i += NT) { out_key[i] = sh.key[i]; out_doc[i] = sh.doc[i]; out_score[i] = sh.score[i]; }
    if (c.tid() == 0) { out_n[0] = n; out_total[0] = total; }
    c.sync();
}
// champion path (one character, max_results <= 64, list long enough): TopKHeap(max) over the first `max` champions, consolidated order.
// On a doc-id-range shard the lists are the global ones and another shard's entries are -1: only this shard's entries among the first `max`
// are written (the hosts' global cut merges them). Repeated keys: the champions are documents, so the best entry per key is kept
// (ConsolidateSegments after Take(max): the list can be shorter than `max`) and it hands the key's first live document on.
IFX_FN void sq_champions(const Ctx& c, const DevIndex& ix, SqTopShared& sh, int ci, int m, int64_t* out_key, int32_t* out_doc, float* out_score, int32_t* out_n, int32_t* out_total) {
    sq_clear(c, sh, 0, 128); const int b = ix.champ_off[ci];
    for (int i = c.tid(); i < m; i += c.nthreads()) { const int d = ix.champ_doc[b + i]; if (d < 0) continue; sh.score[i] = ix.champ_score[b + i]; sh.doc[i] = d; sh.key[i] = ix.doc_key[d]; }
    c.sync();
    if (c.tid() == 0) { int own = 0; for (int i = 0; i < m; i++) own += ix.champ_doc[b + i] >= 0; sh.bcast[0] = own; }
    sq_sort_desc(c, sh, 128);
    if (ix.key_first && c.tid() == 0) { int kept = 0;
        for (int i = 0; i < sh.bcast[0]; i++) { bool seen = false; for (int j = 0; j < kept && !seen; j++) seen = sh.key[j] == sh.key[i];
            if (!seen) { sh.score[kept] = sh.score[i]; sh.key[kept] = sh.key[i]; sh.doc[kept] = ix.key_first[sh.doc[i]]; kept++; } }
        sh.bcast[0] = kept; }
    c.sync();
    const int own = sh.bcast[0];
    for (int i = c.tid(); i < own; i += c.nthreads()) { out_key[i] = sh.key[i]; out_doc[i] = sh.doc[i]; out_score[i] = sh.score[i]; }
    if (c.tid() == 0) { out_n[0] = own; out_total[0] = own; }
    c.sync();
}

}  // namespace ifx
