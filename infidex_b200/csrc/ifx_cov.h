// infidex_b200 -- per-candidate lexical coverage, fusion signals and fusion score (one thread per candidate).
//
// Replaces, for one (query, document) pair (src/Infidex/...):
//   Coverage/CoverageEngine.cs:222-382 (CalculateCoverageInternal), CoverageTokenizer.cs:7-107
//   Coverage/WholeWordMatcher.cs, JoinedWordMatcher.cs, PrefixSuffixMatcher.cs, FuzzyWordMatcher.cs
//   Coverage/CoverageScorer.cs:5-198, Coverage/FusionSignalComputer.cs:53-568, Scoring/FusionScorer.cs:19-396
//   Metrics/LevenshteinDistance.cs:181-341, Metrics/StringMetrics.cs:12-36 (Lcs)
#pragma once
#include "ifx_base.h"

namespace ifx {

constexpr int MAX_DTOK = 192;        // document tokens handled on chip; longer documents raise IFX_Q_OVERFLOW

struct Str { const uint16_t* p; int n; };

IFX_FN uint16_t up_c(const DevIndex& ix, uint16_t c) { return c < 128 ? (uint16_t)((c >= 'a' && c <= 'z') ? c - 32 : c) : ix.upper[c]; }
IFX_FN uint16_t lo_c(const DevIndex& ix, uint16_t c) { return c < 128 ? (uint16_t)((c >= 'A' && c <= 'Z') ? c + 32 : c) : ix.lower[c]; }
IFX_FN bool delim_c(const DevIndex& ix, uint16_t c) { return c < 128 ? ((ix.delim_ascii[c >> 5] >> (c & 31)) & 1u) != 0 : (ix.cflags[c] & 4) != 0; }

IFX_FN bool eq_ic(const DevIndex& ix, Str a, Str b) {
    if (a.n != b.n) return false;
    for (int i = 0; i < a.n; i++) {
        const unsigned x = a.p[i], y = b.p[i]; if (x == y) continue;
        if ((x | y) < 128u) { const unsigned l = x | 0x20u; if ((x ^ y) != 0x20u || l < 'a' || l > 'z') return false; }   // ASCII: equal ignoring case = same letter, other case
        else if (up_c(ix, (uint16_t)x) != up_c(ix, (uint16_t)y)) return false;
    }
    return true;
}
IFX_FN Str sub(Str s, int off, int n) { Str r; r.p = s.p + off; r.n = n; return r; }
IFX_FN bool starts_ic(const DevIndex& ix, Str s, Str p) { return s.n >= p.n && eq_ic(ix, sub(s, 0, p.n), p); }
IFX_FN bool ends_ic(const DevIndex& ix, Str s, Str p) { return s.n >= p.n && eq_ic(ix, sub(s, s.n - p.n, p.n), p); }
IFX_FN int index_of_ic(const DevIndex& ix, Str s, Str p) {
    if (p.n == 0) return 0;
    for (int i = 0; i + p.n <= s.n; i++) if (eq_ic(ix, sub(s, i, p.n), p)) return i;
    return -1;
}
IFX_FN bool contains_ic(const DevIndex& ix, Str s, Str p) { return index_of_ic(ix, s, p) >= 0; }

// LevenshteinDistance.Calculate
IFX_FN int lev(const DevIndex& ix, Str pattern, Str text, int max_errors, bool ic) {
    if (pattern.n == 0) return text.n;
    if (text.n == 0) return pattern.n;
    if (pattern.n > text.n) { Str t = pattern; pattern = text; text = t; }
    int m = pattern.n, n = text.n;
    if (m > MAX_TOKLEN) return max_errors + 1;
    int costs[MAX_TOKLEN + 1]; uint16_t pat[MAX_TOKLEN];          // the (case-folded) pattern is read n times: fold it once
    for (int i = 0; i <= m; i++) costs[i] = i;
    for (int i = 0; i < m; i++) pat[i] = ic ? up_c(ix, pattern.p[i]) : pattern.p[i];
    for (int j = 0; j < n; j++) {
        uint16_t tv = ic ? up_c(ix, text.p[j]) : text.p[j];
        int diag = costs[0]; costs[0] = j + 1; int minc = costs[0];
        for (int i = 0; i < m; i++) {
            int left = costs[i + 1], upv = costs[i]; uint16_t pv = pat[i]; int cost;
            if (tv == pv) cost = diag; else { cost = upv + 1; if (left + 1 < cost) cost = left + 1; if (diag + 1 < cost) cost = diag + 1; }
            diag = left; costs[i + 1] = cost; if (cost < minc) minc = cost;
        }
        if (minc > max_errors) return max_errors + 1;
    }
    return costs[m];
}
// LevenshteinDistance.CalculateDamerau
IFX_FN_OUTLINED int damerau(const DevIndex& ix, Str s, Str t, int maxd, bool ic) {
    int ld = s.n - t.n; if (ld < 0) ld = -ld;
    if (ld > maxd) return maxd + 1;
    int dist = lev(ix, s, t, maxd + 1, ic);
    if (dist <= maxd) return dist;
    if (dist <= maxd + 1) {
        for (int i = 0; i < s.n - 1; i++) {
            if (i >= t.n) break;
            uint16_t s1 = ic ? lo_c(ix, s.p[i]) : s.p[i], t1 = ic ? lo_c(ix, t.p[i]) : t.p[i];
            if (s1 != t1) {
                if (i + 1 >= t.n) break;
                uint16_t s2 = ic ? lo_c(ix, s.p[i + 1]) : s.p[i + 1], t2 = ic ? lo_c(ix, t.p[i + 1]) : t.p[i + 1];
                if (s1 == t2 && s2 == t1) {
                    int rem = maxd - 1; if (rem < 0) return maxd + 1;
                    Str sr = (i + 2 < s.n) ? sub(s, i + 2, s.n - i - 2) : Str{s.p, 0}; Str tr = (i + 2 < t.n) ? sub(t, i + 2, t.n - i - 2) : Str{t.p, 0};
                    int rd = lev(ix, sr, tr, rem, ic);
                    if (rd <= rem) return 1 + rd;
                }
                break;
            }
        }
    }
    return dist;
}
// ---- exact shortcuts around the Levenshtein row (same results as damerau(), far fewer instructions on the ~99 % of token pairs that do not match)
// ASCII fold-equality (both units < 128): same letter in either case
IFX_FN bool eq_fold_ascii(unsigned x, unsigned y) { if (x == y) return true; const unsigned l = x | 0x20u; return (x ^ y) == 0x20u && l >= 'a' && l <= 'z'; }
// damerau(s, t, 1, ic = true) for strings whose units are all < 128 (there ToUpperInvariant and ToLowerInvariant induce the same
// equivalence, so the two folds the reference mixes agree): the value when it is <= 1, else 2. Distance <= 1 means: equal; one
// substitution; one adjacent transposition at the first mismatch with equal rests (CalculateDamerau's only transposition site,
// LevenshteinDistance.cs:300-341); or, lengths one apart, one deletion. Linear time, no DP row.
IFX_FN int damerau1_ascii(Str s, Str t) {
    int d = s.n - t.n; if (d > 1 || d < -1) return 2;
    if (d < 0) { Str x = s; s = t; t = x; }            // s is the longer one
    int p = 0; while (p < t.n && eq_fold_ascii(s.p[p], t.p[p])) p++;
    if (d == 0) {
        if (p == s.n) return 0;
        int k = p + 1; while (k < s.n && eq_fold_ascii(s.p[k], t.p[k])) k++;
        if (k == s.n) return 1;
        if (k == p + 1 && eq_fold_ascii(s.p[p], t.p[p + 1]) && eq_fold_ascii(s.p[p + 1], t.p[p])) { k = p + 2; while (k < s.n && eq_fold_ascii(s.p[k], t.p[k])) k++; if (k == s.n) return 1; }
        return 2;
    }
    int k = p; while (k < t.n && eq_fold_ascii(s.p[k + 1], t.p[k])) k++;
    return k == t.n ? 1 : 2;
}
// character-set signature of the case-folded token (one bit per hashed unit). damerau(s, t, maxd) <= maxd implies a Levenshtein
// distance <= maxd + 1 under the ToUpperInvariant fold (<= maxd when every unit is ASCII: the transposition branch then keeps the
// character multiset), and k edits change at most k characters of either set -- so more than k one-sided signature bits is a proof
// of "no match" and the row is never started.
IFX_FN unsigned fold_sig(const DevIndex& ix, Str s) { unsigned g = 0; for (int i = 0; i < s.n; i++) g |= 1u << ((up_c(ix, s.p[i]) * 0x9E37u >> 4) & 31); return g; }
IFX_FN bool sig_far(unsigned a, unsigned b, int k) { return popc(a & ~b) > k || popc(b & ~a) > k; }

// SegmentProcessor.CalculateLcs -> StringMetrics.Lcs on lower-cased inputs (query is already lower case)
IFX_FN int lcs_metric(const DevIndex& ix, Str q, Str r, int tol) {
    if (q.n == 0 || r.n == 0) return 0;
    bool contains = false;
    for (int i = 0; i + q.n <= r.n && !contains; i++) { bool e = true; for (int k = 0; k < q.n; k++) if (lo_c(ix, r.p[i + k]) != q.p[k]) { e = false; break; } contains = e; }
    if (contains) return q.n;
    int pl = 0, len = q.n < r.n ? q.n : r.n;
    for (int i = 0; i < len; i++) { if (q.p[i] != lo_c(ix, r.p[i])) break; pl++; }
    if (pl == 0) return 0;
    return pl + tol < len ? pl + tol : len;
}

struct Tok { uint16_t off, len; };

// query-side context shared by all candidates of a query (CoverageEngine.PrepareQuery)
struct CovQuery {
    int qlen; int n_tok; int n_ftok;           // deduped tokens (len >= 2); unfiltered fusion tokens (len >= 1)
    Tok tok[MAX_QTOK]; float term_idf[MAX_QTOK]; float word_idf[MAX_QTOK];
    Tok ftok[MAX_QTOK * 2];
    int overflow;
    int ascii;                                 // every unit of the query < 128 (enables the exact ASCII shortcuts)
    unsigned tsig[MAX_QTOK];                   // fold_sig of tok[i]
};

IFX_FN int tokenize(const DevIndex& ix, Str s, int min_size, Tok* out, int cap, bool& overflow) {   // CoverageTokenizer.TokenizeToSpan
    int n = 0, i = 0; int maxtok = s.n / 2 + 1;
    while (i < s.n) {
        while (i < s.n && delim_c(ix, s.p[i])) i++;
        if (i >= s.n) break;
        int b = i; while (i < s.n && !delim_c(ix, s.p[i])) i++;
        if (i - b >= min_size && n < maxtok) { if (n < cap) { out[n].off = (uint16_t)b; out[n].len = (uint16_t)(i - b); } else overflow = true; n++; }
    }
    return n < cap ? n : cap;
}

IFX_FN void prepare_cov_query(const DevIndex& ix, const uint16_t* q, int qlen, CovQuery& c) {
    c.qlen = qlen; c.overflow = 0; bool ovf = false;
    Str qs{q, qlen};
    Tok raw[MAX_QTOK * 2];
    int nr = tokenize(ix, qs, 2, raw, MAX_QTOK * 2, ovf);
    int nu = 0;
    for (int i = 0; i < nr; i++) {   // DeduplicateQueryTokens
        bool dup = false;
        for (int j = 0; j < nu; j++) if (c.tok[j].len == raw[i].len && eq_ic(ix, sub(qs, c.tok[j].off, c.tok[j].len), sub(qs, raw[i].off, raw[i].len))) { dup = true; break; }
        if (!dup) { if (nu < MAX_QTOK) c.tok[nu++] = raw[i]; else ovf = true; }
    }
    c.n_tok = nu;
    for (int i = 0; i < nu; i++) {   // ComputeTermIdf: mean idf of the token's unpadded 3-grams with df > 0, else log2(len + 1)
        Str t = sub(qs, c.tok[i].off, c.tok[i].len); float sum = 0.f; int cnt = 0;
        if (ix.n_live > 0) for (int k = 0; k + 3 <= t.n; k++) { int id = dict_lookup(ix.terms, t.p + k, 3); if (id >= 0 && ix.df[id] > 0) { sum += compute_idf(ix, ix.df[id]); cnt++; } }
        c.term_idf[i] = cnt > 0 ? sum / (float)cnt : ix.log2_len[t.n < 1023 ? t.n : 1023];
        int w = dict_lookup(ix.words, t.p, t.n);        // query is lower case == cache key case
        c.word_idf[i] = w >= 0 ? ix.word_idf[w] : 0.f;
    }
    c.n_ftok = tokenize(ix, qs, 0, c.ftok, MAX_QTOK * 2, ovf);
    { unsigned o = 0; for (int i = 0; i < qlen; i++) o |= q[i]; c.ascii = o < 128u ? 1 : 0; }
    for (int i = 0; i < nu; i++) c.tsig[i] = fold_sig(ix, sub(qs, c.tok[i].off, c.tok[i].len));
    c.overflow = ovf ? 1 : 0;
}

// ---- document token table (derived once per index, ifx_index_create): what CalculateCoverageInternal / ComputeSignals tokenise
// again for every (query, candidate) pair is a pure function of the document text, so it is stored. Per document, 32-bit words:
//   [0] unfiltered tokens fd | deduplicated tokens dc << 16      [1] raw count of tokens of >= 2 units (24 bits) | ascii << 30 | overflow << 31
//   [2 .. 2 + fd)            every token (CoverageTokenizer.TokenizeToSpan with minWordSize 0), Tok = off | len << 16
//   [2 + fd .. 2 + fd + dc)  tokens of >= 2 units, first occurrence only (case-insensitive), in document order
// Returns the number of words; `out` may be null (count pass).
IFX_FN int doc_tokens_emit(const DevIndex& ix, int doc, uint32_t* out) {
    const int64_t t0 = ix.cov_text_off[doc]; const Str d{ix.cov_text + t0, (int)(ix.cov_text_off[doc + 1] - t0)};
    Tok dt[MAX_DTOK]; bool ovf = false; int draw = 0, dc = 0, fd = 0; unsigned tok_or = 0;
    int i = 0; const int maxtok = d.n / 2 + 1;
    while (i < d.n) {
        while (i < d.n && delim_c(ix, d.p[i])) i++;
        if (i >= d.n) break;
        const int b = i; while (i < d.n && !delim_c(ix, d.p[i])) { tok_or |= d.p[i]; i++; }
        const int len = i - b;
        if (fd < maxtok) { if (fd < MAX_DTOK && b < 65536) { if (out) out[2 + fd] = (uint32_t)b | ((uint32_t)(uint16_t)len << 16); fd++; } else ovf = true; }
        if (len >= 2 && draw < maxtok) {
            draw++;
            bool dup = false;
            for (int j = 0; j < dc; j++) if (dt[j].len == len && eq_ic(ix, sub(d, dt[j].off, dt[j].len), sub(d, b, len))) { dup = true; break; }
            if (!dup) { if (dc < MAX_DTOK && b < 65536 && len < 65536) { dt[dc].off = (uint16_t)b; dt[dc].len = (uint16_t)len; dc++; } else ovf = true; }
        }
    }
    if (draw > 0xFFFFFF) { draw = 0xFFFFFF; ovf = true; }
    if (out) {
        for (int j = 0; j < dc; j++) out[2 + fd + j] = (uint32_t)dt[j].off | ((uint32_t)dt[j].len << 16);
        out[0] = (uint32_t)fd | ((uint32_t)dc << 16);
        out[1] = (uint32_t)draw | (tok_or < 128u ? 1u << 30 : 0u) | (ovf ? 1u << 31 : 0u);
    }
    return 2 + fd + dc;
}

struct CovResult { float score; float score0; uint8_t tie; int word_hits; int overflow; };   // score0: the same evaluation with a Stage-1 base of 0 (the WordMatcher twin of a top candidate)

// One (query, document) evaluation: coverage features -> fusion score. `lcs` as cached by the pipeline (0 unless docIndex < 2).
IFX_FN CovResult coverage_fusion(const DevIndex& ix, const CovQuery& c, const uint16_t* qtext, int doc, int lcs, float bm25) {
    CovResult R; R.score = 0.f; R.score0 = 0.f; R.tie = 0; R.word_hits = 0; R.overflow = 0;
    const Str q{qtext, c.qlen};
    const int64_t t0 = ix.cov_text_off[doc]; const Str d{ix.cov_text + t0, (int)(ix.cov_text_off[doc + 1] - t0)};
    const int qc = c.n_tok;
    // ---- doc tokens from the index's token table: every token (fdt), and the deduplicated tokens of >= 2 units (dt)
    const uint32_t* tt = ix.tok_tab + ix.tok_ptr[doc];
    const uint32_t h0 = tt[0], h1 = tt[1];
    const int fd = (int)(h0 & 0xFFFFu), dc = (int)(h0 >> 16);
    const Tok* fdt = (const Tok*)(tt + 2); const Tok* dt = fdt + fd;
    const bool ovf = (h1 >> 31) != 0;
    const int doc_tokens = (int)(h1 & 0xFFFFFFu);
    const bool ascii = c.ascii && ((h1 >> 30) & 1u);   // query and every document token are ASCII
    int word_hits = 0; double num_whole = 0, num_joined = 0, num_fuzzy = 0, num_ps = 0; int penalty = 0;
    float matched[MAX_QTOK]; int first_pos[MAX_QTOK]; uint8_t qa[MAX_QTOK], hw[MAX_QTOK], hj[MAX_QTOK], hp[MAX_QTOK]; uint8_t da[MAX_DTOK];
    for (int i = 0; i < qc; i++) { matched[i] = 0.f; first_pos[i] = -1; qa[i] = 1; hw[i] = hj[i] = hp[i] = 0; }
    for (int j = 0; j < dc; j++) da[j] = 1;
#define QT(i) sub(q, c.tok[i].off, c.tok[i].len)
#define DT(j) sub(d, dt[j].off, dt[j].len)
#define POSMIN(i, pos) do { if (first_pos[i] == -1 || (pos) < first_pos[i]) first_pos[i] = (pos); } while (0)
    if (qc > 0) {
        // ---- WholeWordMatcher
        { int pinc = qc > 1 ? 1 : 0;
          for (int i = 0; i < qc; i++) {
              int mi = -1; for (int j = 0; j < dc; j++) if (da[j] && dt[j].len == c.tok[i].len && eq_ic(ix, QT(i), DT(j))) { mi = j; break; }
              if (mi == -1) continue;
              int ql = c.tok[i].len; word_hits++; num_whole += ql; matched[i] += (float)ql; hw[i] = 1; hp[i] = 1; POSMIN(i, (int)dt[mi].off);
              if (dc > i) { if (dt[i].len != ql || !eq_ic(ix, QT(i), DT(i))) penalty++; } else penalty++;
              if (i < qc - 1) num_whole += pinc;
              qa[i] = 0; da[mi] = 0;
          } }
        // ---- JoinedWordMatcher
        for (int i = 0; i < qc - 1; i++) {
            if (!qa[i] || !qa[i + 1]) continue;
            int nx = i + 1; int jl = c.tok[i].len + c.tok[nx].len; int mi = -1;
            for (int j = 0; j < dc; j++) if (da[j] && dt[j].len == jl && starts_ic(ix, DT(j), QT(i)) && ends_ic(ix, DT(j), QT(nx))) { mi = j; break; }
            if (mi == -1) continue;
            num_joined += jl; word_hits += 2;
            matched[i] += (float)c.tok[i].len; hj[i] = 1; hp[i] = 1; int pos = dt[mi].off; POSMIN(i, pos);
            matched[nx] += (float)c.tok[nx].len; hj[nx] = 1; POSMIN(nx, pos);
            qa[i] = 0; qa[nx] = 0; da[mi] = 0;
        }
        for (int i = 0; i < dc - 1; i++) {
            if (!da[i]) continue;
            int nx = -1; for (int k = i + 1; k < dc; k++) if (da[k]) { nx = k; break; }
            if (nx == -1) break;
            int jl = dt[i].len + dt[nx].len; int mi = -1;
            for (int j = 0; j < qc; j++) if (qa[j] && c.tok[j].len == jl && starts_ic(ix, QT(j), DT(i)) && ends_ic(ix, QT(j), DT(nx))) { mi = j; break; }
            if (mi == -1) continue;
            num_joined += jl; word_hits += 1; matched[mi] += (float)jl; hj[mi] = 1; hp[mi] = 1; POSMIN(mi, (int)dt[i].off);
            qa[mi] = 0; da[i] = 0; da[nx] = 0;
        }
        // ---- PrefixSuffixMatcher: active indices, stable-sorted by length descending
        {
            uint8_t qi[MAX_QTOK]; uint8_t di[MAX_DTOK]; int nq = 0, nd = 0;
            for (int i = 0; i < qc; i++) if (qa[i]) qi[nq++] = (uint8_t)i;
            for (int j = 0; j < dc; j++) if (da[j]) di[nd++] = (uint8_t)j;
            for (int i = 1; i < nq; i++) { uint8_t cur = qi[i]; int cl = c.tok[cur].len; int j = i - 1; while (j >= 0 && c.tok[qi[j]].len < cl) { qi[j + 1] = qi[j]; j--; } qi[j + 1] = cur; }
            for (int i = 1; i < nd; i++) { uint8_t cur = di[i]; int cl = dt[cur].len; int j = i - 1; while (j >= 0 && dt[di[j]].len < cl) { di[j + 1] = di[j]; j--; } di[j + 1] = cur; }
            for (int a = 0; a < nq; a++) {   // MatchExact
                int i = qi[a]; if (!qa[i]) continue;
                int ql = c.tok[i].len; Str qt = QT(i);
                for (int b = 0; b < nd; b++) {
                    int j = di[b]; if (!da[j]) continue;
                    int dl = dt[j].len; if (ql == dl) continue;
                    Str dtx = DT(j); bool m = false, pre = false; double sc = 0;
                    if (ql < dl) {
                        if (starts_ic(ix, dtx, qt)) { sc = ql; m = true; pre = true; }
                        else if (ends_ic(ix, dtx, qt)) { int h = ql / 2; sc = h > 1 ? h : 1; m = true; }
                        else if (ql >= 4 && contains_ic(ix, dtx, qt)) { sc = ql * 0.6; m = true; }
                    } else if (ends_ic(ix, qt, dtx)) { sc = dl; m = true; }
                    if (m) { num_ps += sc; word_hits++; matched[i] += (float)sc; if (pre) hp[i] = 1; POSMIN(i, (int)dt[j].off); qa[i] = 0; da[j] = 0; break; }
                }
            }
            for (int a = 0; a < nq; a++) {   // MatchFuzzyPrefix
                int i = qi[a]; if (!qa[i]) continue;
                int ql = c.tok[i].len; Str qt = QT(i);
                if (!(ql >= 4 || (i == qc - 1 && ql >= 2))) continue;
                for (int b = 0; b < nd; b++) {
                    int j = di[b]; if (!da[j]) continue;
                    int dl = dt[j].len; if (ql >= dl) continue;
                    Str dtx = DT(j); bool m = false; double sc = 0;
                    int dist = ascii ? damerau1_ascii(qt, sub(dtx, 0, ql)) : damerau(ix, qt, sub(dtx, 0, ql), 1, true);
                    if (dist <= 1) { sc = ql - dist; if (sc < 0.1) sc = 0.1; m = true; }
                    else if (dl > ql) {
                        dist = ascii ? damerau1_ascii(qt, sub(dtx, 0, ql + 1)) : damerau(ix, qt, sub(dtx, 0, ql + 1), 1, true);
                        if (dist <= 1) { sc = ql - dist; if (sc < 0.1) sc = 0.1; m = true; }
                        else if (ql > 1) { dist = ascii ? damerau1_ascii(qt, sub(dtx, 0, ql - 1)) : damerau(ix, qt, sub(dtx, 0, ql - 1), 1, true); if (dist <= 1) { sc = ql - 1 - dist; if (sc < 0.1) sc = 0.1; m = true; } }
                    }
                    if (m) { num_ps += sc; word_hits++; matched[i] += (float)sc; POSMIN(i, (int)dt[j].off); qa[i] = 0; da[j] = 0; break; }
                }
            }
        }
        // ---- FuzzyWordMatcher (CoverageSetup defaults: MinWordSize 2, NumTypos 2, one typo from len 3, two from len 7, max word 20)
        {
            bool all_full = true; for (int i = 0; i < qc; i++) if (c.tok[i].len > 0 && matched[i] < (float)c.tok[i].len) { all_full = false; break; }
            if (!all_full) {
                int maxq = 0; for (int i = 0; i < qc; i++) if (qa[i] && c.tok[i].len > maxq) maxq = c.tok[i].len;
                int maxe = maxq >= 7 ? 2 : (maxq >= 3 ? 1 : 0); if (maxq == 2 && maxe == 0) maxe = 1; if (maxe > 2) maxe = 2;
                if (maxq > 0) for (int e = 1; e <= maxe; e++) {
                    bool any = false; for (int i = 0; i < qc; i++) if (qa[i]) any = true;
                    if (!any) break;
                    for (int i = 0; i < qc; i++) {
                        if (!qa[i]) continue;
                        int ql = c.tok[i].len; if (ql < 2) continue;
                        int tme = ql >= 7 ? 2 : (ql >= 3 ? 1 : 0); bool special = false;
                        if (ql == 2 && tme == 0) { tme = 1; special = true; }
                        if (e > tme) continue; if (special && e != 1) continue;
                        int minl = ql - e > 2 ? ql - e : 2, maxl = ql + e < 20 ? ql + e : 20; if (maxl > 63) maxl = 63;
                        Str qt = QT(i);
                        for (int j = 0; j < dc; j++) {
                            if (!da[j]) continue;
                            int dl = dt[j].len; if (dl > maxl || dl < minl) continue;
                            Str dtx = DT(j);
                            if (special && (dtx.n == 0 || lo_c(ix, dtx.p[0]) != lo_c(ix, qt.p[0]))) continue;
                            int dist;
                            if (e == 1 && ascii) dist = damerau1_ascii(qt, dtx);
                            else { if (sig_far(c.tsig[i], fold_sig(ix, dtx), ascii ? e : e + 1)) continue; dist = damerau(ix, qt, dtx, e, true); }
                            if (dist <= e) { word_hits++; num_fuzzy += (ql - dist); matched[i] += (float)(ql - dist); POSMIN(i, (int)dt[j].off); qa[i] = 0; da[j] = 0; break; }
                        }
                    }
                }
            }
        }
    }
    // ---- CoverageScorer.CalculateFinalScore
    int any_match = 0, fully = 0, strict = 0, prefix_matched = 0, first_match = -1, longest_run = 0, suffix_run = 0, preceding_strict = 0;
    float sum_ci = 0, idfw = 0, tidf = 0, midf = 0, last_idf = 0; bool last_has_prefix = false, last_typeahead = false;
    float term_ci[MAX_QTOK];
    double lcs_sum = (double)lcs;
    double num = num_joined + num_whole + num_fuzzy + num_ps - (double)(penalty & 255);
    if (num == 0.0 && lcs_sum > 2.0) num = lcs_sum - 2.0;
    (void)num;   // coverage byte is not consumed by the fusion scorer
    for (int i = 0; i < qc; i++) {
        term_ci[i] = 0.f;
        int mc = c.tok[i].len; if (mc <= 0) continue;
        float ci = matched[i] / (float)mc; if (ci > 1.0f) ci = 1.0f;
        sum_ci += ci; term_ci[i] = ci; if (ci > 0) any_match++;
        float idf = c.term_idf[i]; tidf += idf; idfw += ci * idf;
        if (ci < 1.0f) midf += (1.0f - ci) * idf;
        if (i == qc - 1) last_idf = idf;
        bool full = matched[i] >= ((float)mc - 0.01f);
        if (full) fully++;
        if ((hw[i] || hj[i]) && full) strict++;
        if (hp[i]) prefix_matched++;
        if (first_pos[i] >= 0 && (first_match == -1 || first_pos[i] < first_match)) first_match = first_pos[i];
    }
    float idf_cov = tidf > 0.f ? idfw / tidf : 0.f;
    if (qc > 0 && tidf > 0.f) { float share = last_idf / tidf; float th = 1.f / (float)(qc + 1); last_typeahead = share <= th; }
    if (qc == 1 && c.qlen > 0 && lcs_sum > 0.0) { double r = lcs_sum / c.qlen; float cl = (float)(r < 1.0 ? r : 1.0); if (cl > sum_ci) sum_ci = cl; }
    { int run = 0; for (int i = 0; i < qc; i++) { bool ph = hp[i] && c.tok[i].len > 0 && matched[i] > 0; if (ph) { run++; if (run > longest_run) longest_run = run; } else run = 0; }
      for (int i = qc - 1; i >= 0; i--) { bool ph = hp[i] && c.tok[i].len > 0 && matched[i] > 0; if (ph) suffix_run++; else break; } }
    if (qc >= 1) { last_has_prefix = hp[qc - 1] && matched[qc - 1] > 0;
        if (qc >= 2) for (int i = 0; i < qc - 1; i++) if ((hw[i] || hj[i]) && matched[i] >= ((float)c.tok[i].len - 0.01f)) preceding_strict++; }
    (void)fully;
    // ---- FusionSignalComputer.ComputeSignals: unfiltered tokens (len >= 1), no dedupe; minStemLength = MinWordSize (2)
    const int fq = c.n_ftok;
    bool lex_prefix_last = false, perfect_doc = false, stem_evidence = false, anchor_stem = false; int trailing_density = 0, single_sim = 0, single_char_boost = 0;
#define FQ(i) sub(q, c.ftok[i].off, c.ftok[i].len)
#define FD(j) sub(d, fdt[j].off, fdt[j].len)
    if (fq > 0 && fd > 0) {
        if (fq == 1) { for (int i = 0; i < fd; i++) if (starts_ic(ix, FD(i), FQ(0))) { lex_prefix_last = true; break; } }
        else {
            bool all = true;
            for (int i = 0; i < fq - 1; i++) { bool fe = false; for (int j = 0; j < fd; j++) if (eq_ic(ix, FD(j), FQ(i))) { fe = true; break; } if (!fe) { all = false; break; } }
            if (all) { Str last = FQ(fq - 1); for (int i = 0; i < fd; i++) if (starts_ic(ix, FD(i), last)) { lex_prefix_last = true; break; } }
        }
        { bool ok = true; for (int j = 0; j < fd && ok; j++) { bool ex = false; for (int i = 0; i < fq; i++) if (starts_ic(ix, FD(j), FQ(i)) || starts_ic(ix, FQ(i), FD(j))) { ex = true; break; } if (!ex) ok = false; } perfect_doc = ok; }
        if (fq >= 2) {
            int unmatched = 0, evidence = 0;
            for (int qi2 = 0; qi2 < fq; qi2++) {
                Str qq = FQ(qi2); if (qq.n < 2) continue;
                bool wm = false; for (int j = 0; j < fd; j++) { Str dd = FD(j); if (dd.n == 0) continue; if (starts_ic(ix, dd, qq)) { wm = true; break; } }
                if (wm) continue;
                unmatched++;
                for (int j = 0; j < fd; j++) {
                    Str dd = FD(j); if (dd.n < 2) continue;
                    if (starts_ic(ix, qq, dd)) { evidence++; break; }
                    int mc = qq.n < dd.n ? qq.n : dd.n;
                    if (mc >= 2) { int pl = 0; for (int i = 0; i < mc; i++) { if (lo_c(ix, qq.p[i]) == lo_c(ix, dd.p[i])) pl++; else break; } if (pl >= 2) { evidence++; break; } }
                }
            }
            stem_evidence = unmatched > 0 && evidence == unmatched;
        }
        if (c.ftok[0].len >= 3) {   // HasAnchorStem with DocumentMetadata.FirstToken
            Str stem = sub(FQ(0), 0, 3);
            bool has_tokens = ix.token_count[doc] > 0;
            Str ft{ix.first_token.chars + ix.first_token.off[doc], (int)(ix.first_token.off[doc + 1] - ix.first_token.off[doc])};
            if (has_tokens && ft.n >= 3) {
                if (starts_ic(ix, ft, stem)) anchor_stem = true;
                else for (int i = 1; i < fd; i++) if (FD(i).n >= 3 && starts_ic(ix, FD(i), stem)) { anchor_stem = true; break; }
            } else if (!has_tokens) { for (int i = 0; i < fd; i++) if (FD(i).n >= 3 && starts_ic(ix, FD(i), stem)) { anchor_stem = true; break; } }
        }
        if (fq >= 2 && c.ftok[fq - 1].len >= 1 && c.ftok[fq - 1].len <= 2) {
            Str last = FQ(fq - 1); int cnt = 0;
            for (int i = 0; i < fd; i++) if (starts_ic(ix, FD(i), last) || (FD(i).n > last.n && contains_ic(ix, FD(i), last))) cnt++;
            if (cnt > 0) { float dens = (float)cnt / (float)fd; float v = dens * 255.f; v = v < 0.f ? 0.f : (v > 255.f ? 255.f : v); trailing_density = (int)(uint8_t)v; }
        }
        if (fq == 1) {   // ComputeSingleTermLexicalSimilarity (query already lower case)
            Str qt = FQ(0); int ql = qt.n; float best = 0.f; const unsigned qsig = fold_sig(ix, qt);
            if (ql >= 3) {
                for (int t = 0; t < fd; t++) {
                    Str tk = FD(t); if (tk.n < 2) continue;
                    int idx = -1;   // qLower.IndexOf(tLower) (ordinal on lower-cased text)
                    for (int i = 0; i + tk.n <= ql && idx < 0; i++) { bool e = true; for (int k = 0; k < tk.n; k++) if (qt.p[i + k] != lo_c(ix, tk.p[k])) { e = false; break; } if (e) idx = i; }
                    if (idx >= 0) { float lf = (float)tk.n / (float)ql; float pf = 1.f - (float)idx / (float)ql; float sc = lf * pf; if (sc > best) best = sc; continue; }
                    int maxk = ql < tk.n ? ql : tk.n, bestk = 0;
                    for (int len = maxk; len >= 2; len--) { bool e = true; for (int k = 0; k < len; k++) if (qt.p[ql - len + k] != lo_c(ix, tk.p[k])) { e = false; break; } if (e) { bestk = len; break; } }
                    float ps = bestk > 0 ? (float)bestk / (float)ql : 0.f, fz = 0.f;
                    if (tk.n <= 32 && !sig_far(qsig, fold_sig(ix, tk), ascii ? 2 : 3)) { int dist = damerau(ix, qt, tk, 2, true); if (dist <= 2) fz = (float)(ql - dist) / (float)ql; }   // both sides lower-cased in the reference; case-folded compare is identical
                    float comb = ps > fz ? ps : fz; if (comb > best) best = comb;
                }
                if (ql >= 6) {
                    int seg = ql / 2 < 6 ? ql / 2 : 6; int pi = -1, si = -1;
                    for (int t = 0; t < fd; t++) {
                        Str tk = FD(t); if (tk.n < 3) continue;
                        auto pre = [&](bool tok_longer) { int n = tok_longer ? seg : tk.n; if (tok_longer ? tk.n < seg : seg < tk.n) return false; for (int k = 0; k < n; k++) if (qt.p[k] != lo_c(ix, tk.p[k])) return false; return true; };
                        auto suf = [&](bool tok_longer) { int n = tok_longer ? seg : tk.n; if (tok_longer ? tk.n < seg : seg < tk.n) return false; for (int k = 0; k < n; k++) if (qt.p[ql - 1 - k] != lo_c(ix, tk.p[tk.n - 1 - k])) return false; return true; };
                        if (pi == -1 && (pre(true) || pre(false))) pi = t;
                        if (si == -1 && (suf(true) || suf(false))) si = t;
                        if (pi != -1 && si != -1) break;
                    }
                    if (pi != -1 && si != -1 && pi != si) { float ts = (float)(seg + seg) / (float)ql; if (ts > 1.f) ts = 1.f; if (ts > best) best = ts; }
                }
            }
            float v = best * 255.f; v = v < 0.f ? 0.f : (v > 255.f ? 255.f : v); single_sim = (int)(uint8_t)v;
        }
        if (fq >= 2 && c.ftok[fq - 1].len == 1) {   // ComputeSingleCharLastTokenMatch
            uint16_t target = lo_c(ix, q.p[c.ftok[fq - 1].off]);
            if (ix.cflags[target] & 1) {
                int di2 = 0, first = -1; bool okc = true;
                for (int i = 0; i < fq - 1 && okc; i++) { bool found = false; while (di2 < fd) { if (index_of_ic(ix, FD(di2), FQ(i)) >= 0) { found = true; if (first == -1) first = di2; break; } di2++; } if (!found) okc = false; }
                if (okc && di2 + 1 < fd) {
                    Tok nx = fdt[di2 + 1];
                    if (nx.len > 0 && lo_c(ix, d.p[nx.off]) == target) {
                        int end = fdt[di2].off + fdt[di2].len; bool broken = false;
                        for (int p2 = end; p2 < nx.off; p2++) if (!(ix.cflags[d.p[p2]] & 2)) { broken = true; break; }
                        if (!broken) { int boost = 8 + (16 - first > 0 ? 16 - first : 0); if (nx.len == 1) boost += 4; single_char_boost = boost; }
                    }
                }
            }
        }
    }
    // ---- FusionScorer.Calculate
    const int terms = qc; const int n = fq > 0 ? fq : terms;
    const bool single = n <= 1;
    const bool complete = terms > 0 && any_match == terms, clean = terms > 0 && prefix_matched == terms, exact = terms > 0 && strict == terms, at_start = first_match == 0;
    const int preceding = terms - 1 > 0 ? terms - 1 : 0;
    const bool cpl = terms >= 1 && preceding_strict == preceding && last_has_prefix;
    const bool strong = lex_prefix_last && cpl;
    int prec = 0, tier = 0;
    if (!single && terms > 0) { int m = any_match; tier = m >= terms ? 3 : (m == terms - 1 ? 2 : (m * 2 >= terms ? 1 : 0)); }
    if (!single && tier > 0) prec |= (tier & 3) << 16;
    if (!single && clean && at_start && lex_prefix_last && complete) prec |= 1 << 15;
    if (!single && doc_tokens > 0 && word_hits == doc_tokens) prec |= 1 << 14;
    float avg_idf = 0.f;
    if (!single && terms >= 2) {
        bool dominant = false;
        avg_idf = tidf > 0.f ? tidf / (float)terms : 0.f;
        for (int k = 0; k < terms; k++) {
            float power = c.word_idf[k] * term_ci[k];
            if (term_ci[k] <= 0.1f || c.word_idf[k] <= 0.f || c.word_idf[k] < avg_idf) continue;
            float other = 0.f; for (int i = 0; i < terms; i++) if (i != k) other += c.word_idf[i] * term_ci[i];
            if (power >= other) { dominant = true; break; }
        }
        bool anchor = anchor_stem && c.word_idf[0] >= avg_idf;
        if (dominant || anchor) prec |= 1 << 13;
        if (dominant && terms - any_match == 1) prec |= 8;
    }
    if (single) {
        if (complete) prec |= 1 << 17;
        if (clean && terms > 0) prec |= 1 << 16;
        int t = 0; if (complete) { if (at_start) { if (exact) t = 4; else if (clean) t = 3; } else { if (exact) t = 2; else if (clean) t = 1; } }
        prec |= t << 3;
    } else {
        bool anchor_run = anchor_stem && longest_run >= 2;
        int mt = strong ? 3 : (lex_prefix_last ? 2 : ((perfect_doc || anchor_run) ? 1 : 0));
        if (fq > terms) mt += single_char_boost;
        prec |= mt;
    }
    float ratio = terms > 0 ? (float)any_match / (float)terms : 0.f;
    bool partial = ratio > 0.f && ratio < 1.f;
    if (partial && n >= 2) {
        if (stem_evidence) prec |= 8;
        else {
            int unmatched = terms - any_match; bool last_matched = last_has_prefix || (terms > 0 && any_match == terms);
            bool can = (last_matched || !last_typeahead) && tidf > 0.f;
            if (unmatched == 1 && can) { float mr = midf / tidf; float gap = 1.f - ratio; if (mr < gap) prec |= 8; }
        }
    }
    float avg_ci = terms > 0 ? sum_ci / (float)terms : 0.f, sem;
    if (single) { float ls = (float)single_sim / 255.f; sem = (avg_ci + ls) / 2.f; }
    else if (doc_tokens == 0) sem = avg_ci;
    else {
        int unmatched = terms - any_match; bool last_matched = last_has_prefix || (terms > 0 && any_match == terms);
        bool can = (last_matched || !last_typeahead) && tidf > 0.f;
        bool use_idf = partial && unmatched == 1 && can && idf_cov > ratio;
        float base = use_idf ? idf_cov : avg_ci;
        float density = (float)word_hits / (float)doc_tokens;
        sem = base * density;
        if (terms >= 3) { int sc = (anchor_stem ? 1 : 0) + (suffix_run >= 2 ? 1 : 0); if (sc > 0) { float bonus = 0.15f * (float)sc; sem = sem + bonus; if (sem > 1.f) sem = 1.f; } }
        if (terms >= 2) { float md = (float)trailing_density / 255.f; if (md > 0.f) { float head = 1.f - sem; sem += head * md; } }
    }
    float gap = 1.f - ratio;
    float sem0 = sem;                                      // base 0: `partial` means gap > 0, so the mix below never applies
    if (partial && bm25 >= gap) sem = ratio * sem + gap * bm25;
    sem = sem < 0.f ? 0.f : (sem > 0.999f ? 0.999f : sem);
    sem0 = sem0 < 0.f ? 0.f : (sem0 > 0.999f ? 0.999f : sem0);
    uint8_t tie = 0;
    if (n >= 2 && d.n > 0) { float focus = (float)c.qlen / (float)d.n; if (focus > 1.f) focus = 1.f; tie = (uint8_t)(focus * 255.f); }
    R.score = (float)prec + sem; R.score0 = (float)prec + sem0; R.tie = tie; R.word_hits = word_hits; R.overflow = ovf ? 1 : 0;
#undef QT
#undef DT
#undef FQ
#undef FD
#undef POSMIN
    return R;
}

}  // namespace ifx
