// infidex_b200 -- Stage 2 on device: WordMatcher candidate generation, per-candidate coverage + fusion, final
// top-K / consolidation / truncation, Infiscript filter VM and facet counting.
//
// Replaces (src/Infidex/...):
//   wm_query        Scoring/WordMatcherLookup.cs:11-69, WordMatcher/WordMatcher.cs:201-354, Scoring/SearchPipeline.cs:110-170,298-397,524-576
//   cov_eval        Scoring/SearchPipeline.cs:449-522 (ProcessCandidate) -> ifx_cov.h
//   finalize_query  Scoring/SearchPipeline.cs:418-440, Scoring/ResultProcessor.cs:35-70,146-178, Core/FacetBuilder.cs:19-105,
//                   Filtering/FilterVM.cs:26-357, SearchEngine.cs:304-316
#pragma once
#include "ifx_stage1.h"
#include "ifx_cov.h"
#include "../../include/infidex_gpu.h"

namespace ifx {

// ---- filter program (device view; built by ifx_filter_register from INFISCRIPT-V1 bytecode) -----------------------------
struct FConst { int32_t kind; int32_t off, len; int32_t col; int32_t is_num; int32_t arr_start, arr_len; double num; };   // kind 1 string, 2 number, 3 array
struct FInstr { int32_t op; int32_t a; };
struct FilterProg { const FConst* consts; const FInstr* code; const uint16_t* chars; int32_t n_consts, n_code; };

struct Stage2Buffers {
    int32_t* ent_doc; float* ent_base; int32_t* ent_twin; int32_t* ent_n;     // [nq][ent_cap]
    float* ent_score; uint8_t* ent_tie; int32_t* ent_hits; uint8_t* ent_lcs;   // [nq][ent_cap]
    int32_t* di_doc;      // [nq][2] documents holding docIndex 0 / 1 (SearchPipeline.cs:524-545), -1 if none
    int32_t* wm_any;      // [nq] WordMatcher union non-empty
    int32_t* mode;        // [nq] 0 coverage stage ran, 1 return the Stage-1 list, 2 Stage-1 list cut to max_results
    CovQuery* covq;       // [nq]
    int32_t* wm_cnt;      // [nq][4] per shard: top docs that are also WordMatcher docs, WordMatcher-only entries taken, union non-empty, index of the first such entry
    const int32_t* g_di;  // doc-id-range shards: [nq][2] local id of the document at global Stage-1 rank 0 / 1 (-1: another shard's, -2: fewer than two ranks exist)
    const int32_t* s1_total;   // [nq] short-query path: documents matched by Stage 1 (the list itself is cut to the depth); null / 0 otherwise
    const int32_t* s1_nglob;   // doc-id-range shards: [nq] Stage-1 list length over ALL shards (the mode decision of short queries); null otherwise
    const int32_t* g_hits;     // doc-id-range shards: [nq] max coverage word hits over ALL shards of each short query (its fallback decision); null otherwise
    const float* gmax;    // doc-id-range shards: top Stage-1 score over ALL shards per query (normBm25, SearchPipeline.cs:411-413); null: the local list's first
    int32_t ent_cap;
};

struct FinalOut { int64_t* key; float* score; uint8_t* tie; int32_t* n; int32_t* total; int32_t* status; int32_t* facet_col; int32_t* facet_val; int32_t* facet_cnt; int32_t* n_facets; int32_t cap, fcap;
                  int32_t* shard_info; int64_t* shard_dkey;      // doc-id-range shards (non-null): no local truncation, [nq][8] / [nq][2] facts for the hosts' merge
                  int32_t* rec_post; int32_t rec_stride; };      // shards: [nq][cap][rec_stride] per record: filter pass, value id of every facetable column (-1 null / empty)

struct WmList { const int32_t* p; int32_t n; };

struct WmShared {
    WmList lists[MAX_WM_WORDS * 18];
    WmList affix[MAX_WM_WORDS * 2];
    Tok words[MAX_WM_WORDS]; int n_words;
    int32_t top_sorted[MAX_K]; uint16_t top_rank[MAX_K]; alignas(4) uint8_t in_wm[MAX_K];     // Stage-1 docs ascending, their Stage-1 rank, WordMatcher membership
    uint16_t nz[MAX_WM_WORDS * 18]; int n_nz;                                      // the non-empty dictionary lists
    uint8_t dirty[MAX_CONTAINERS];
    ScanTmp scan; int bcast[8]; int first_live[2];
};

// compare the first |w| units of a (affix word) with w: <0, 0 (a has w as prefix), >0
IFX_FN int cmp_prefix(const uint16_t* a, int na, const uint16_t* w, int nw) {
    int n = na < nw ? na : nw;
    for (int i = 0; i < n; i++) if (a[i] != w[i]) return a[i] < w[i] ? -1 : 1;
    return na >= nw ? 0 : -1;
}
IFX_FN int cmp_prefix_rev(const uint16_t* a, int na, const uint16_t* w, int nw) {   // same on reversed strings
    int n = na < nw ? na : nw;
    for (int i = 0; i < n; i++) { uint16_t x = a[na - 1 - i], y = w[nw - 1 - i]; if (x != y) return x < y ? -1 : 1; }
    return na >= nw ? 0 : -1;
}

IFX_FN bool sorted_contains(const int32_t* a, int n, int32_t v) { int64_t i = lower_bound_i32(a, 0, n, v); return i < n && a[i] == v; }

// ---------------------------------------------------------------------------------------------------------------------
IFX_FN void wm_query(const Ctx& c, const DevIndex& ix, const QueryPlan& p, const int32_t* s1_doc, const float* s1_score, int n1_in,
                     S1Workspace& ws, WmShared& sh, const Stage2Buffers& B, int q) {
    const int NT = c.nthreads(); const int K = p.depth; const int cap = B.ent_cap;
    int32_t* e_doc = B.ent_doc + (size_t)q * cap; float* e_base = B.ent_base + (size_t)q * cap; int32_t* e_twin = B.ent_twin + (size_t)q * cap;
    if (c.tid() == 0) {
        int mode = 0; int n1 = n1_in < 0 ? 0 : n1_in;
        if ((p.short_kind != 0 || p.is_short3) && B.s1_nglob) n1 = B.s1_nglob[q];    // shards: the <= 3-character rule reads the list length over ALL shards, so every shard takes the same mode
        if (p.status != 0) mode = 1;
        else if (p.is_short3 && n1 >= p.max_results) mode = 2;                       // SearchPipeline.cs:114-120
        else if (!p.enable_coverage || p.short_skip_coverage || p.short_no_cov) mode = 1;              // SearchPipeline.cs:157-170
        B.mode[q] = mode; B.ent_n[q] = 0; B.wm_any[q] = 0; B.di_doc[q * 2] = -1; B.di_doc[q * 2 + 1] = -1;
        sh.bcast[0] = mode;
    }
    c.sync();
    if (sh.bcast[0] != 0) return;
    const int nt = n1_in < K ? n1_in : K;            // topCandidates.Take(coverageDepth)
    // ---- query words (len >= 2) -> dictionary lists
    if (c.tid() == 0) {
        int nw = 0; const uint16_t* t = p.qtext; int len = p.qlen;
        for (int i = 0; i < len;) {
            while (i < len && is_delim(ix, t[i])) i++;
            if (i >= len) break;
            int b = i; while (i < len && !is_delim(ix, t[i])) i++;
            bool blank = true; for (int k = b; k < i; k++) if (!is_space(ix, t[k])) blank = false;
            if (blank || i - b < 2) continue;
            if (nw < MAX_WM_WORDS) { sh.words[nw].off = (uint16_t)b; sh.words[nw].len = (uint16_t)(i - b); nw++; }
        }
        sh.n_words = nw; sh.first_live[0] = sh.first_live[1] = -1;
    }
    c.sync();
    const int nw = sh.n_words; const int n_lists = nw * 18;
    for (int it = c.tid(); it < n_lists; it += NT) {     // WordMatcher.Lookup: exact, ld1, and per single deletion ld1 + exact
        int w = it / 18, v = it % 18; const uint16_t* s = p.qtext + sh.words[w].off; int len = sh.words[w].len;
        WmList L; L.p = nullptr; L.n = 0;
        const DocsetDict* dd = nullptr; uint16_t buf[MAX_QLEN]; const uint16_t* key = s; int klen = len;
        bool ld1_ok = len >= 3 && len <= 8;
        if (v == 0) dd = &ix.wm_exact;
        else if (v == 1) { if (ld1_ok) dd = &ix.wm_ld1; }
        else if (ld1_ok) { int k = (v - 2) >> 1; if (k < len) { int o = 0; for (int i = 0; i < len; i++) if (i != k) buf[o++] = s[i]; key = buf; klen = len - 1; dd = ((v - 2) & 1) ? &ix.wm_exact : &ix.wm_ld1; } }
        if (dd) { int id = dict_lookup(dd->keys, key, klen); if (id >= 0) { L.p = dd->doc_id + dd->row_ptr[id]; L.n = (int32_t)(dd->row_ptr[id + 1] - dd->row_ptr[id]); } }
        sh.lists[it] = L;
    }
    for (int w = c.tid(); w < nw; w += NT) {             // WordMatcher.LookupAffix: prefix matches first, then suffix matches, budget 4096
        const uint16_t* s = p.qtext + sh.words[w].off; int len = sh.words[w].len; const StrDict& A = ix.affix;
        auto aw = [&](int i, const uint16_t*& ptr, int& n) { ptr = A.chars + A.off[i]; n = (int)(A.off[i + 1] - A.off[i]); };
        int lo = 0, hi = A.n;
        while (lo < hi) { int mid = (lo + hi) >> 1; const uint16_t* ap; int an; aw(mid, ap, an); if (cmp_prefix(ap, an, s, len) < 0) lo = mid + 1; else hi = mid; }
        int p0 = lo; hi = A.n;
        while (lo < hi) { int mid = (lo + hi) >> 1; const uint16_t* ap; int an; aw(mid, ap, an); if (cmp_prefix(ap, an, s, len) <= 0) lo = mid + 1; else hi = mid; }
        int pc = lo - p0;
        lo = 0; hi = A.n;
        while (lo < hi) { int mid = (lo + hi) >> 1; const uint16_t* ap; int an; aw(ix.affix_rev[mid], ap, an); if (cmp_prefix_rev(ap, an, s, len) < 0) lo = mid + 1; else hi = mid; }
        int s0 = lo; hi = A.n;
        while (lo < hi) { int mid = (lo + hi) >> 1; const uint16_t* ap; int an; aw(ix.affix_rev[mid], ap, an); if (cmp_prefix_rev(ap, an, s, len) <= 0) lo = mid + 1; else hi = mid; }
        int sc = lo - s0; int budget = AFFIX_CAP;
        int tp = pc < budget ? pc : budget; budget -= tp; int ts = budget > 0 ? (sc < budget ? sc : budget) : 0;
        sh.affix[w * 2].p = ix.affix_fwd_doc + p0; sh.affix[w * 2].n = tp;
        sh.affix[w * 2 + 1].p = ix.affix_rev_doc + s0; sh.affix[w * 2 + 1].n = ts;
    }
    // ---- top docs ascending (with their Stage-1 rank)
    int n2 = 1; while (n2 < nt) n2 <<= 1;
    for (int i = c.tid(); i < n2; i += NT) { sh.top_sorted[i] = i < nt ? s1_doc[i] : 0x7fffffff; sh.top_rank[i] = (uint16_t)i; if (i < MAX_K) sh.in_wm[i] = 0; }
    c.sync();
    for (int k = 2; k <= n2; k <<= 1) for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = c.tid(); i < n2; i += NT) { int l = i ^ j; if (l > i) { bool up = (i & k) == 0; int a = sh.top_sorted[i], b = sh.top_sorted[l];
            if (up ? a > b : a < b) { sh.top_sorted[i] = b; sh.top_sorted[l] = a; uint16_t ra = sh.top_rank[i]; sh.top_rank[i] = sh.top_rank[l]; sh.top_rank[l] = ra; } } }
        c.sync();
    }
    // ---- affix docs -> candidate set (every touched word also in the summary ws.wm_sum: one bit per word); membership of the top docs
    auto add = [&](int d) { cand_add(ws, sh.dirty, d); if (!((ws.wm_sum[d >> 10] >> ((d >> 5) & 31)) & 1u)) atomic_or(&ws.wm_sum[d >> 10], 1u << ((d >> 5) & 31)); };
    int any = 0;
    for (int a = 0; a < nw * 2; a++) { WmList L = sh.affix[a]; if (L.n > 0) any = 1;
        for (int i = c.tid(); i < L.n; i += NT) { int d = L.p[i]; if (d >= 0) add(d); } }      // d < 0 (doc-id-range shards): the word's document lives on another shard
    if (c.tid() == 0) { int n = 0; for (int l = 0; l < n_lists; l++) if (sh.lists[l].n > 0) sh.nz[n++] = (uint16_t)l; sh.n_nz = n; }
    c.sync();
    const int nnz = sh.n_nz; if (nnz > 0) any = 1;
    for (int k = c.tid(); k < nt; k += NT) { int d = sh.top_sorted[k]; sh.in_wm[k] = (uint8_t)((ws.bits[d >> 5] >> (d & 31)) & 1u); }
    c.sync();
    // one (list, top doc) probe per thread and step: consecutive threads search the same list for consecutive (ascending) documents
    for (int it = c.tid(); it < nnz * nt; it += NT) { const int k = it % nt;
        const WmList L = sh.lists[sh.nz[it / nt]]; const int d = sh.top_sorted[k];
        if (d >= L.p[0] && d <= L.p[L.n - 1] && sorted_contains(L.p, L.n, d)) atomic_or(reinterpret_cast<unsigned*>(sh.in_wm) + (k >> 2), 1u << ((k & 3) * 8)); }      // several lists may hold the same document
    c.sync();
    int my = 0; for (int k = c.tid(); k < nt; k += NT) my += sh.in_wm[k];
    const int n_overlap = block_sum(c, my, sh.scan);
    const int wm_limit = K - n_overlap > 0 ? K - n_overlap : 0;
    // ---- leading elements of every list -> candidate set (the first M elements of the union lie within the first M of each list)
    const int M = K + nt + 2;
    for (int z = 0; z < nnz; z++) { WmList L = sh.lists[sh.nz[z]]; int m = L.n < M ? L.n : M;
        for (int i = c.tid(); i < m; i += NT) add(L.p[i]); }
    c.sync();
    // ---- entries: (a) WM ∩ top ascending, base 0; the twin field holds the Stage-1 rank until group (c) is placed
    int ne = 0;
    for (int k0 = 0; k0 < nt; k0 += NT) { int k = k0 + c.tid(); int f = (k < nt && sh.in_wm[k]) ? 1 : 0; int tot; int off = block_excl_scan(c, f, sh.scan, tot);
        if (f && ne + off < cap) { e_doc[ne + off] = sh.top_sorted[k]; e_base[ne + off] = 0.f; e_twin[ne + off] = (int)sh.top_rank[k]; } ne += tot; }
    // ---- (b) WM \ top ascending, first wm_limit; also the first two live WM docs overall (docIndex assignment). Containers are walked in
    //      order while the quota or the two live documents are still open -- the summary bits say which words of the container to read at
    //      all -- and whatever is left afterwards is only cleared, through the summary, strided over the block.
    {
        const int ncont = (ix.n_docs + 65535) >> 16; const int64_t nwords = ((int64_t)ix.n_docs + 31) >> 5; const int64_t nsum = (nwords + 31) >> 5;
        int taken = 0, seen_live = 0, kdone = 0;
        for (int k = 0; k < ncont; k++) {
            if (!(taken < wm_limit || seen_live < 2)) break;      // uniform
            kdone = k + 1;
            if (!sh.dirty[k]) continue;
            int64_t w0 = (int64_t)k * 2048, w1 = w0 + 2048; if (w1 > nwords) w1 = nwords;
            int per = (int)((w1 - w0 + NT - 1) / NT); int64_t my0 = w0 + (int64_t)c.tid() * per, my1 = my0 + per; if (my1 > w1) my1 = w1;
            int cnt = 0, live = 0;
            for (int64_t w = my0; w < my1; w++) { if (!((ws.wm_sum[w >> 5] >> (w & 31)) & 1u)) continue;
                unsigned v = ws.bits[w]; while (v) { int b = ffs32(v) - 1; v &= v - 1; int d = (int)((w << 5) | b); if (!ix.deleted[d]) live++; if (!sorted_contains(sh.top_sorted, nt, d)) cnt++; } }
            int tot; int off = block_excl_scan(c, cnt, sh.scan, tot);
            int ltot; int loff = block_excl_scan(c, live, sh.scan, ltot);
            int o = off, lo2 = loff;
            for (int64_t w = my0; w < my1; w++) { if (!((ws.wm_sum[w >> 5] >> (w & 31)) & 1u)) continue;
                unsigned v = ws.bits[w]; ws.bits[w] = 0;
                while (v) { int b = ffs32(v) - 1; v &= v - 1; int d = (int)((w << 5) | b);
                    if (!ix.deleted[d]) { if (seen_live + lo2 < 2) sh.first_live[seen_live + lo2] = d; lo2++; }
                    if (!sorted_contains(sh.top_sorted, nt, d)) { if (taken + o < wm_limit && ne + o < cap) { e_doc[ne + o] = d; e_base[ne + o] = 0.f; e_twin[ne + o] = -1; } o++; } } }
            int add = tot; if (taken + add > wm_limit) add = wm_limit - taken;
            taken += add; ne += add; seen_live += ltot;
            c.sync();                                              // every thread has read this container's summary words
            for (int64_t sw = (w0 >> 5) + c.tid(); sw < ((w1 + 31) >> 5); sw += NT) ws.wm_sum[sw] = 0;
        }
        for (int64_t sw = (((int64_t)kdone * 2048) >> 5) + c.tid(); sw < nsum; sw += NT) { unsigned m = ws.wm_sum[sw]; if (!m) continue; ws.wm_sum[sw] = 0; while (m) { ws.bits[(sw << 5) | (ffs32(m) - 1)] = 0; m &= m - 1; } }
        cand_clear(c, ix, ws, sh.dirty, true);
    }
    if (c.tid() == 0 && B.wm_cnt) { B.wm_cnt[q * 4 + 0] = n_overlap; B.wm_cnt[q * 4 + 1] = ne - n_overlap; B.wm_cnt[q * 4 + 2] = any; B.wm_cnt[q * 4 + 3] = n_overlap; }
    // ---- (c) every top candidate in rank order, base = score / top score; link twins with group (a)
    const int na = n_overlap;
    for (int r = c.tid(); r < nt; r += NT) {
        int d = s1_doc[r]; float mx = B.gmax ? B.gmax[q] : s1_score[0]; float nb = mx > 0.f ? s1_score[r] / mx : 0.f;
        if (ne + r < cap) { e_doc[ne + r] = d; e_base[ne + r] = nb; e_twin[ne + r] = -1; }
    }
    c.sync();
    for (int a = c.tid(); a < na && a < cap; a += NT) {           // group (a) entry a <-> its rank-order twin
        const int r = e_twin[a];
        if (ne + r < cap) { e_twin[a] = ne + r; e_twin[ne + r] = a; } else e_twin[a] = -2;
    }
    ne += nt;
    c.sync();
    if (c.tid() == 0) {
        B.ent_n[q] = ne < cap ? ne : cap; B.wm_any[q] = any;
        // BuildDocumentKeyIndex: keys of the top list in rank order, then live WordMatcher docs ascending
        int d0 = -1, d1 = -1;
        if (B.g_di && B.g_di[q * 2] != -2) { d0 = B.g_di[q * 2]; d1 = B.g_di[q * 2 + 1]; }      // shards: docIndex 0 / 1 are the documents at GLOBAL rank 0 / 1 (possibly on another shard)
        else {
            if (nt >= 1) d0 = s1_doc[0];
            if (nt >= 2) d1 = s1_doc[1];
            for (int i = 0; i < 2; i++) { int f = sh.first_live[i]; if (f < 0) continue; if (d0 < 0) d0 = f; else if (d1 < 0 && f != d0) d1 = f; }
        }
        B.di_doc[q * 2] = d0; B.di_doc[q * 2 + 1] = d1;
    }
    c.sync();
}

// ---------------------------------------------------------------------------------------------------------------------
// one thread per (query, entry)
IFX_FN void cov_eval_entry(const DevIndex& ix, const QueryPlan& p, const Stage2Buffers& B, int q, int e) {
    const size_t o = (size_t)q * B.ent_cap + e;
    const int doc = B.ent_doc[o];
    // A top candidate that is also a WordMatcher document appears twice (group (a) with base 0 and in rank order with its normalised
    // Stage-1 score): the evaluation differs in the last mix only, so the rank-order entry computes both and the group-(a) entry --
    // those are the leading entries of a query, whole warps of them -- does nothing.
    const int tw = B.ent_twin[o];
    if (tw > e) return;
    const size_t o2 = tw >= 0 ? (size_t)q * B.ent_cap + tw : o;
    if (ix.deleted[doc] || tw == -3) { B.ent_hits[o] = -1; B.ent_score[o] = -1.f; B.ent_tie[o] = 0; B.ent_lcs[o] = 0;      // ProcessCandidate returns early
        if (tw >= 0) { B.ent_hits[o2] = -1; B.ent_score[o2] = -1.f; B.ent_tie[o2] = 0; B.ent_lcs[o2] = 0; } return; }
    const CovQuery& cq = B.covq[q];
    int lcs = 0;
    if (doc == B.di_doc[q * 2] || doc == B.di_doc[q * 2 + 1]) {
        int tol = cq.qlen >= 5 ? (int)((double)cq.qlen * 0.2) : 0;
        int64_t t0 = ix.cov_text_off[doc]; Str d{ix.cov_text + t0, (int)(ix.cov_text_off[doc + 1] - t0)};
        lcs = lcs_metric(ix, Str{p.qtext, cq.qlen}, d, tol); if (lcs > 255) lcs = 255;
    }
    CovResult r = coverage_fusion(ix, cq, p.qtext, doc, lcs, B.ent_base[o]);
    const int hits = r.word_hits | (r.overflow ? 0x40000000 : 0);
    B.ent_score[o] = r.score; B.ent_tie[o] = r.tie; B.ent_hits[o] = hits; B.ent_lcs[o] = (uint8_t)lcs;
    if (tw >= 0) { B.ent_score[o2] = r.score0; B.ent_tie[o2] = r.tie; B.ent_hits[o2] = hits; B.ent_lcs[o2] = (uint8_t)lcs; }
}

// ---------------------------------------------------------------------------------------------------------------------
// filter VM (FilterVM.Execute) over dictionary-encoded columns
struct FVal { int kind; int a, b; };   // 0 null, 1 column string (col a, id b), 2 const (idx a), 3 bool (a), 5 array const (idx a)

IFX_FN Str fval_str(const DevIndex& ix, const FilterProg& fp, const FVal& v, bool& is_num, double& num) {
    is_num = false; num = 0;
    if (v.kind == 1) { const Column& c = ix.columns[v.a]; is_num = c.dict_is_num[v.b]; num = c.dict_num[v.b]; return Str{c.dict.chars + c.dict.off[v.b], (int)(c.dict.off[v.b + 1] - c.dict.off[v.b])}; }
    if (v.kind == 2) { const FConst& k = fp.consts[v.a]; is_num = k.is_num; num = k.num; return Str{fp.chars + k.off, k.len}; }
    if (v.kind == 3) { static const uint16_t T[] = {'T', 'r', 'u', 'e'}, F[] = {'F', 'a', 'l', 's', 'e'}; return v.a ? Str{T, 4} : Str{F, 5}; }
    return Str{nullptr, 0};
}
IFX_FN int cmp_ic_str(const DevIndex& ix, Str a, Str b) {
    int n = a.n < b.n ? a.n : b.n;
    for (int i = 0; i < n; i++) { uint16_t x = up_c(ix, a.p[i]), y = up_c(ix, b.p[i]); if (x != y) return x < y ? -1 : 1; }
    return a.n == b.n ? 0 : (a.n < b.n ? -1 : 1);
}
IFX_FN bool like_match(const DevIndex& ix, Str t, Str p) {   // ^escape(p) with % -> .*, _ -> .$, IgnoreCase ('.' does not match \n)
    int ti = 0, pi = 0, star_p = -1, star_t = 0;
    while (ti < t.n) {
        if (pi < p.n && p.p[pi] == '%') { star_p = pi++; star_t = ti; }
        else if (pi < p.n && ((p.p[pi] == '_' && t.p[ti] != '\n') || (p.p[pi] != '_' && up_c(ix, p.p[pi]) == up_c(ix, t.p[ti])))) { pi++; ti++; }
        else if (star_p >= 0 && t.p[star_t] != '\n') { pi = star_p + 1; ti = ++star_t; }
        else return false;
    }
    while (pi < p.n && p.p[pi] == '%') pi++;
    return pi == p.n;
}
IFX_FN bool filter_exec(const DevIndex& ix, const FilterProg& fp, int doc, bool& unsupported) {
    FVal st[24]; int sp = 0; int ip = 0;
    auto is_null = [&](const FVal& v) { return v.kind == 0; };
    auto are_equal = [&](const FVal& l, const FVal& r) { if (is_null(l) && is_null(r)) return true; if (is_null(l) || is_null(r)) return false; if (l.kind == 5 || r.kind == 5) { unsupported = true; return false; }
        bool n1, n2; double d1, d2; Str a = fval_str(ix, fp, l, n1, d1), b = fval_str(ix, fp, r, n2, d2); return eq_ic(ix, a, b); };
    auto compare = [&](const FVal& l, const FVal& r) { if (is_null(l) && is_null(r)) return 0; if (is_null(l)) return -1; if (is_null(r)) return 1; if (l.kind == 5 || r.kind == 5) { unsupported = true; return 0; }
        bool n1, n2; double d1, d2; Str a = fval_str(ix, fp, l, n1, d1), b = fval_str(ix, fp, r, n2, d2);
        if (n1 && n2) return d1 < d2 ? -1 : (d1 > d2 ? 1 : 0);
        return cmp_ic_str(ix, a, b); };
    auto push_b = [&](bool b) { st[sp].kind = 3; st[sp].a = b ? 1 : 0; st[sp].b = 0; sp++; };
    auto as_bool = [&](const FVal& v) { return v.kind == 3 && v.a; };
    auto sstr = [&](const FVal& v) { bool n; double d; return v.kind == 0 || v.kind == 5 ? Str{nullptr, 0} : fval_str(ix, fp, v, n, d); };
    while (ip < fp.n_code) {
        const FInstr in = fp.code[ip];
        if (sp >= 22) { unsupported = true; return false; }
        switch (in.op) {
            case 0x01: { const FConst& k = fp.consts[in.a]; FVal v; v.kind = 0; v.a = v.b = 0; if (k.col >= 0) { int id = ix.columns[k.col].value_id[doc]; if (id >= 0) { v.kind = 1; v.a = k.col; v.b = id; } } st[sp++] = v; break; }
            case 0x02: { const FConst& k = fp.consts[in.a]; FVal v; v.a = in.a; v.b = 0; v.kind = k.kind == 3 ? 5 : 2; if (k.kind == 2) unsupported = true; st[sp++] = v; break; }
            case 0x03: if (sp > 0) sp--; break;
            case 0x04: if (sp > 0) { st[sp] = st[sp - 1]; sp++; } break;
            case 0x10: case 0x11: case 0x12: case 0x13: case 0x14: case 0x15: {
                if (sp < 2) { unsupported = true; return false; }
                FVal r = st[--sp], l = st[--sp]; bool res;
                if (in.op == 0x10) res = are_equal(l, r); else if (in.op == 0x11) res = !are_equal(l, r);
                else { int cv = compare(l, r); res = in.op == 0x12 ? cv < 0 : (in.op == 0x13 ? cv <= 0 : (in.op == 0x14 ? cv > 0 : cv >= 0)); }
                push_b(res); break; }
            case 0x20: case 0x21: { if (sp < 2) { unsupported = true; return false; } bool r = as_bool(st[--sp]), l = as_bool(st[--sp]); push_b(in.op == 0x20 ? (l && r) : (l || r)); break; }
            case 0x22: { if (sp < 1) { unsupported = true; return false; } bool v = as_bool(st[--sp]); push_b(!v); break; }
            case 0x30: case 0x31: case 0x32: case 0x33: {
                if (sp < 2) { unsupported = true; return false; }
                Str pat = sstr(st[--sp]), txt = sstr(st[--sp]);
                bool res = in.op == 0x30 ? contains_ic(ix, txt, pat) : (in.op == 0x31 ? starts_ic(ix, txt, pat) : (in.op == 0x32 ? ends_ic(ix, txt, pat) : like_match(ix, txt, pat)));
                push_b(res); break; }
            case 0x34: { sp -= 2; if (sp < 0) sp = 0; unsupported = true; push_b(false); break; }    // MATCHES (regex): SURVEY 8(f) "next"
            case 0x40: { if (sp < 2) { unsupported = true; return false; } FVal a = st[--sp], v = st[--sp]; bool found = false;
                if (a.kind == 5 && v.kind != 0) { const FConst& k = fp.consts[a.a]; bool n; double d; Str vs = fval_str(ix, fp, v, n, d);
                    for (int i = 0; i < k.arr_len && !found; i++) { const FConst& el = fp.consts[k.arr_start + i]; if (eq_ic(ix, vs, Str{fp.chars + el.off, el.len})) found = true; } }
                push_b(found); break; }
            case 0x41: { if (sp < 3) { unsupported = true; return false; } FVal mx = st[--sp], mn = st[--sp], v = st[--sp]; push_b(compare(v, mn) >= 0 && compare(v, mx) <= 0); break; }
            case 0x50: case 0x51: { if (sp < 1) { unsupported = true; return false; } FVal v = st[--sp]; bool n; double d; bool isn = v.kind == 0 || ((v.kind == 1 || v.kind == 2) && fval_str(ix, fp, v, n, d).n == 0); push_b(in.op == 0x50 ? isn : !isn); break; }
            case 0x60: ip = in.a - 1; break;
            case 0x61: if (sp > 0 && st[sp - 1].kind == 3 && !st[sp - 1].a) ip = in.a - 1; break;
            case 0x62: if (sp > 0 && st[sp - 1].kind == 3 && st[sp - 1].a) ip = in.a - 1; break;
            case 0xFF: ip = fp.n_code; break;
            default: unsupported = true; return false;
        }
        ip++;
    }
    if (sp == 0) return false;
    return as_bool(st[sp - 1]);
}

// ---------------------------------------------------------------------------------------------------------------------
struct FinShared {
    float score[2 * MAX_K]; int32_t idx[2 * MAX_K]; int32_t pos[2 * MAX_K];
    int32_t keep_doc[MAX_K]; float keep_score[MAX_K]; uint8_t keep_tie[MAX_K];
    int n_keep; int bcast[8]; ScanTmp scan;
    union {                                                   // never live at the same time: sort keys vs. facet scratch
        struct { int64_t ekey[2 * MAX_K]; uint8_t etie[2 * MAX_K]; };   // per entry: document key and tiebreaker (the sort's comparator reads them on score ties)
        struct { int32_t fv[MAX_K]; int32_t fc[MAX_K]; };
    };
};

// ---- ResultProcessor.ApplyBoosts / ApplySort (ResultProcessor.cs) over the filtered records sh.keep_*[0, nk): every (record, boost) pair
// runs the filter VM on its own thread, the strengths are summed per record, Score + totalBoost is one float add; then the .NET introsort is
// replayed on one thread, over record indices, first by boosted score (b.Score.CompareTo(a.Score), whenever a boost had a filter), then by
// the caller-registered rank of the SortBy value (null lowest). Facets, TotalCandidates and Take follow on the permuted list.
struct ScoreDescCmp {
    const float* s;
    IFX_FN int operator()(int a, int b) const { float x = s[b], y = s[a]; return x < y ? -1 : (x > y ? 1 : 0); }
};
struct RankCmp {      // CompareValues(a, b) ascending, CompareValues(b, a) descending
    const int32_t* r; int asc;
    IFX_FN int operator()(int a, int b) const { int x = asc ? r[a] : r[b], y = asc ? r[b] : r[a]; return x < y ? -1 : (x > y ? 1 : 0); }
};
IFX_FN float add_boost(float score, int total) {
#ifdef IFX_EMU
    return score + (float)total;
#else
    return __fadd_rn(score, (float)total);
#endif
}
IFX_FN void post_process(const Ctx& c, const DevIndex& ix, const ifx_query_post& P, const FilterProg* filters, FinShared& sh, int nk) {
    const int NT = c.nthreads(); const int nb = P.n_boosts; const bool sort = P.sort_column != IFX_SORT_NONE;
    int32_t* acc = sh.pos; int32_t* perm = sh.idx;       // (free once the records are compacted into sh.keep_*)
    if (nb > 0) {
        for (int i = c.tid(); i < nk; i += NT) acc[i] = 0;
        c.sync();
        bool unsup = false;
        for (int it = c.tid(); it < nk * nb; it += NT) { const int i = it / nb, k = it - i * nb;
            if (filter_exec(ix, filters[P.boost_filter[k]], sh.keep_doc[i], unsup)) atomic_add(&acc[i], P.boost_strength[k]); }
        if (unsup) sh.bcast[5] = 1;
        c.sync();
        for (int i = c.tid(); i < nk; i += NT) if (acc[i] > 0) sh.keep_score[i] = add_boost(sh.keep_score[i], acc[i]);
        c.sync();
    }
    if (sort) {
        const int col = P.sort_column;
        for (int i = c.tid(); i < nk; i += NT) { int r = -1;
            if (col >= 0) { const Column& C = ix.columns[col]; const int id = C.value_id[sh.keep_doc[i]]; if (id >= 0) r = C.rank[id]; }
            acc[i] = r; }
    }
    for (int i = c.tid(); i < nk; i += NT) perm[i] = i;
    c.sync();
    if (c.tid() == 0) {
        if (nb > 0) { IntroSort<ScoreDescCmp> s{{sh.keep_score}}; s.sort(perm, nk); }
        if (sort) { IntroSort<RankCmp> s{{acc, P.sort_ascending ? 1 : 0}}; s.sort(perm, nk); }
    }
    c.sync();
    for (int i = c.tid(); i < nk; i += NT) { const int j = perm[i]; sh.fv[i] = sh.keep_doc[j]; sh.score[i] = sh.keep_score[j]; sh.fc[i] = sh.keep_tie[j]; }
    c.sync();
    for (int i = c.tid(); i < nk; i += NT) { sh.keep_doc[i] = sh.fv[i]; sh.keep_score[i] = sh.score[i]; sh.keep_tie[i] = (uint8_t)sh.fc[i]; }
    c.sync();
}

// ---- FacetBuilder.BuildFacets over n items, one thread: per facetable column the value ids id_of(col, i) (< 0: none) with weight cnt_of(i) are
// summed per id -- empty strings are not counted --, ordered by OrderByDescending(count).ThenBy(key) (a stable insertion sort; key order =
// case-insensitive, then lower-case first, SURVEY Q12), and the first `per_col` of every column become rows (col, id, count) of `row`; rows
// beyond `fcap` set IFX_Q_OVERFLOW in `status`. fv / fc: scratch of n entries. Returns the number of rows written.
template <class IdOf, class CntOf>
IFX_FN int facet_table(const DevIndex& ix, int n, IdOf id_of, CntOf cnt_of, int per_col, int32_t* fv, int32_t* fc,
                       int32_t* row_col, int32_t* row_val, int32_t* row_cnt, int fcap, int& status) {
    int nf = 0;
    for (int col = 0; col < ix.n_columns; col++) {
        const Column& C = ix.columns[col]; if (!(C.flags & 2)) continue;
        int nu = 0;
        for (int i = 0; i < n; i++) { const int id = id_of(col, i); const int w = cnt_of(i); if (id < 0 || w <= 0) continue; if (C.dict.off[id + 1] == C.dict.off[id]) continue;
            int u = 0; for (; u < nu; u++) if (fv[u] == id) { fc[u] += w; break; } if (u == nu) { fv[nu] = id; fc[nu] = w; nu++; } }
        for (int a = 1; a < nu; a++) { int v = fv[a], cn = fc[a]; int b = a - 1;
            while (b >= 0) { bool gt;
                if (fc[b] != cn) gt = fc[b] < cn;
                else { Str x{C.dict.chars + C.dict.off[fv[b]], (int)(C.dict.off[fv[b] + 1] - C.dict.off[fv[b]])}, y{C.dict.chars + C.dict.off[v], (int)(C.dict.off[v + 1] - C.dict.off[v])};
                    int cv = cmp_ic_str(ix, x, y); if (cv == 0) cv = -cmp_ordinal(x.p, x.n, y.p, y.n); gt = cv > 0; }
                if (!gt) break; fv[b + 1] = fv[b]; fc[b + 1] = fc[b]; b--; }
            fv[b + 1] = v; fc[b + 1] = cn; }
        const int lim = nu < per_col ? nu : per_col;
        for (int u = 0; u < lim; u++) { if (nf < fcap) { row_col[nf] = col; row_val[nf] = fv[u]; row_cnt[nf] = fc[u]; nf++; } else status |= 4; }
    }
    return nf;
}

// `post`: [nq] boosts / SortBy per query, or null (no post-processing: exactly the plain search)
IFX_FN void finalize_query(const Ctx& c, const DevIndex& ix, const QueryPlan& p, const int32_t* s1_doc, const float* s1_score, int n1,
                           const Stage2Buffers& B, const FilterProg* filters, int n_filters, const ifx_query_post* post, FinShared& sh, const FinalOut& O, int q) {
    const int NT = c.nthreads(); const int K = p.depth; const int cap = B.ent_cap;
    const size_t eo = (size_t)q * cap;
    int mode = B.mode[q]; int status = p.status;
    if (n1 < 0) { n1 = 0; status |= 4; }
    int n_rec = 0;
    if (mode == 0) {
        const int ne = B.ent_n[q];
        int n2 = 1; while (n2 < ne) n2 <<= 1;
        int mh = 0, ovf = 0;
        for (int i = c.tid(); i < n2; i += NT) {
            if (i < ne) { int h = B.ent_hits[eo + i]; sh.etie[i] = B.ent_tie[eo + i]; sh.ekey[i] = ix.doc_key[B.ent_doc[eo + i]]; sh.idx[i] = h < 0 ? -1 : i; sh.score[i] = h < 0 ? -2.f : B.ent_score[eo + i]; if (h >= 0) { if (h & 0x40000000) ovf = 1; h &= 0x3fffffff; if (h > mh) mh = h; } }
            else { sh.idx[i] = -1; sh.score[i] = -2.f; }
        }
        c.sync();
        // max word hits / overflow (block max via scan of flags is overkill: use shared atomics-free reduction through sorted pass below)
        int tmh = mh, tovf = ovf;
#ifndef IFX_EMU
        for (int d = 16; d > 0; d >>= 1) { int o = __shfl_xor_sync(0xffffffffu, tmh, d); tmh = tmh > o ? tmh : o; tovf |= __shfl_xor_sync(0xffffffffu, tovf, d); }
#endif
        if (c.lane() == 0) { sh.scan.w[c.warp()] = tmh; }
        c.sync();
        int max_hits = 0; for (int w = 0; w < c.nwarps(); w++) max_hits = max_hits > sh.scan.w[w] ? max_hits : sh.scan.w[w];
        c.sync();
        if (c.lane() == 0) sh.scan.w[c.warp()] = tovf;
        c.sync();
        for (int w = 0; w < c.nwarps(); w++) if (sh.scan.w[w]) status |= 4;
        c.sync();
        // order entries by ScoreEntry.CompareTo descending: (score, tie, key ascending); entry index breaks exact ties
        auto before = [&](int a, int b) -> bool {
            int ia = sh.idx[a], ib = sh.idx[b];
            if (ia < 0 || ib < 0) return ia >= 0 && ib < 0;
            float sa = sh.score[a], sb = sh.score[b]; if (sa != sb) return sa > sb;
            uint8_t ta = sh.etie[ia], tb = sh.etie[ib]; if (ta != tb) return ta > tb;
            int64_t ka = sh.ekey[ia], kb = sh.ekey[ib]; if (ka != kb) return ka < kb;
            return ia < ib;
        };
        for (int k = 2; k <= n2; k <<= 1) for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = c.tid(); i < n2; i += NT) { int l = i ^ j; if (l > i) { bool up = (i & k) == 0; bool sw = up ? before(l, i) : before(i, l); if (sw) { float x = sh.score[i]; sh.score[i] = sh.score[l]; sh.score[l] = x; int y = sh.idx[i]; sh.idx[i] = sh.idx[l]; sh.idx[l] = y; } } }
            c.sync();
        }
        for (int i = c.tid(); i < ne; i += NT) sh.pos[i] = 0x7fffffff;
        c.sync();
        for (int i = c.tid(); i < n2; i += NT) if (sh.idx[i] >= 0) sh.pos[sh.idx[i]] = i;
        c.sync();
        // TopKHeap(K) keeps the K best entries; ConsolidateSegments keeps the better of two entries with the same key, and the filter, boosts,
        // SortBy and facets read the key's first live document (GetDocumentByPublicKey), whichever segment the entry came from.
        // Valid entries sort in front of the invalid ones, so "the first K valid positions" is a prefix: per-position keep flags
        // and an ordered compaction, round by round.
        const int lim = n2 < K ? n2 : K; int nk = 0;
        for (int base = 0; base < lim; base += NT) {
            const int i = base + c.tid(); int e = -1; bool keep = false;
            if (i < lim) { e = sh.idx[i]; if (e >= 0) { int tw = B.ent_twin[eo + e]; keep = !(tw >= 0 && sh.pos[tw] < i);
                if (keep && ix.key_first) { const int64_t k = sh.ekey[e]; for (int j = 0; j < i && keep; j++) { const int ej = sh.idx[j]; if (ej >= 0 && sh.ekey[ej] == k) keep = false; } } } }      // duplicate keys: the better entry of a key wins
            int tot; int off = block_excl_scan(c, keep ? 1 : 0, sh.scan, tot);
            if (keep) { const int d = B.ent_doc[eo + e]; sh.keep_doc[nk + off] = ix.key_first ? ix.key_first[d] : d; sh.keep_score[nk + off] = sh.score[i]; sh.keep_tie[nk + off] = sh.etie[e]; }
            nk += tot;
        }
        // ResultProcessor.CalculateTruncationIndex: only docIndex 0/1 have stored word hits / lcs (Span2D height-2 quirk): for each of
        // the two docs, the word hits of its first entry with non-zero hits and the lcs of its last entry (in entry order)
        const int d0 = B.di_doc[q * 2], d1 = B.di_doc[q * 2 + 1];
        if (c.tid() == 0) { sh.bcast[0] = 0x7fffffff; sh.bcast[1] = -1; sh.bcast[2] = 0x7fffffff; sh.bcast[3] = -1; sh.bcast[4] = -1; }
        c.sync();
        auto clamp_hits = [&](int e) { int h = B.ent_hits[eo + e] & 0x3fffffff; return h > 255 ? 255 : h; };
        for (int e = c.tid(); e < ne; e += NT) {
            if (B.ent_hits[eo + e] < 0) continue;
            const int dd = B.ent_doc[eo + e];
            if (dd == d0) { if (clamp_hits(e) != 0) atomic_min(&sh.bcast[0], e); atomic_max(&sh.bcast[1], e); }
            else if (dd == d1) { if (clamp_hits(e) != 0) atomic_min(&sh.bcast[2], e); atomic_max(&sh.bcast[3], e); }
        }
        c.sync();
        const int wh0 = sh.bcast[0] != 0x7fffffff ? clamp_hits(sh.bcast[0]) : 0, l0 = sh.bcast[1] >= 0 ? (int)B.ent_lcs[eo + sh.bcast[1]] : 0;
        const int wh1 = sh.bcast[2] != 0x7fffffff ? clamp_hits(sh.bcast[2]) : 0, l1 = sh.bcast[3] >= 0 ? (int)B.ent_lcs[eo + sh.bcast[3]] : 0;
        const int min_hits = max_hits > 1 ? max_hits : 1;
        for (int i = c.tid(); i < nk; i += NT) {                     // last kept record that clears the truncation test
            int dd = sh.keep_doc[i]; int wh = dd == d0 ? wh0 : (dd == d1 ? wh1 : 0); int lb = dd == d0 ? l0 : (dd == d1 ? l1 : 0);
            if (wh >= min_hits || lb > 0 || sh.keep_score[i] >= 254.f) atomic_max(&sh.bcast[4], i);
        }
        c.sync();
        if (O.shard_info) {      // shards: the truncation index is a property of the MERGED list -- report the facts, cut only to max_results
            int ge = 0; for (int i = c.tid(); i < nk; i += NT) if (sh.keep_score[i] >= 254.f) ge++;
            ge = block_sum(c, ge, sh.scan);
            if (c.tid() == 0) { int32_t* inf = O.shard_info + (size_t)q * 8; inf[0] = max_hits; inf[1] = ge; inf[2] = d0 >= 0 ? wh0 : -1; inf[3] = d0 >= 0 ? l0 : -1; inf[4] = d1 >= 0 ? wh1 : -1; inf[5] = d1 >= 0 ? l1 : -1; inf[6] = nk; inf[7] = B.wm_any[q];
                O.shard_dkey[q * 2] = d0 >= 0 ? ix.doc_key[d0] : -1; O.shard_dkey[q * 2 + 1] = d1 >= 0 ? ix.doc_key[d1] : -1; }
        }
        if (c.tid() == 0) {
            int result = nk;
            // SearchPipeline.cs:418-419: coverage returned [] -> the Stage-1 list. On shards a short query decides it on the word hits and the
            // WordMatcher flag of ALL shards (g_hits, wm_any), so every shard takes the same branch; an n-gram query keeps the coverage records.
            const bool none = (O.shard_info ? (p.short_kind != 0 && B.g_hits && B.g_hits[q] == 0) : max_hits == 0) && !B.wm_any[q];
            if (none) result = -1;
            else if (O.shard_info) { if (result > p.max_results) result = p.max_results; }
            else if (nk > 0) {
                const int trunc = sh.bcast[4];
                int count = trunc == -1 ? p.max_results : (trunc + 1 < p.max_results ? trunc + 1 : p.max_results);
                if (result > count) result = count;
            }
            sh.n_keep = result;
        }
        c.sync();
        n_rec = sh.n_keep;
        if (n_rec < 0) { if (n1 > 0 || O.shard_info) mode = 1; else n_rec = 0; }      // SearchPipeline.cs:184-197 fallback to the TF-IDF backbone (a shard: whatever part of it is here)
    }
    if (mode != 0) {
        n_rec = mode == 2 ? (n1 < p.max_results ? n1 : p.max_results) : n1;
        if (n_rec > MAX_K) n_rec = MAX_K;
        if (O.shard_info && c.tid() == 0) {      // shards: no truncation facts; inf[6] = -1 tells the hosts the records are the WHOLE Stage-1 list (filtered
            int32_t* inf = O.shard_info + (size_t)q * 8;      // here; TotalCandidates and facet rows summed over the shards), 0 a list the hosts cut at max before they filter
            inf[0] = 0; inf[1] = 0; inf[2] = -1; inf[3] = -1; inf[4] = -1; inf[5] = -1; inf[6] = (mode == 1 || p.short_kind != 0) ? -1 : 0; inf[7] = 0; O.shard_dkey[q * 2] = -1; O.shard_dkey[q * 2 + 1] = -1;
        }
        for (int i = c.tid(); i < n_rec; i += NT) { sh.keep_doc[i] = s1_doc[i]; sh.keep_score[i] = s1_score[i]; sh.keep_tie[i] = 0; }
        c.sync();
    }
    // ---- SearchEngine.HandleEmptyQueryWithFacets (SearchEngine.cs:321-346): a blank query with EnableFacets browses the corpus -- every live
    // document in id order with score ushort.MaxValue, the filter, Take(max), facets over what was taken
    const bool browse = p.status == 8 && p.enable_facets && p.filter_id < n_filters;
    if (browse) {
        int have = 0; const int want = p.max_results < MAX_K ? p.max_results : MAX_K; bool unsup = false;
        if (c.tid() == 0) sh.bcast[5] = 0;
        c.sync();
        for (int base = 0; base < ix.n_docs && have < want; base += NT) {
            const int d = base + c.tid(); bool pass = d < ix.n_docs && !ix.deleted[d];
            if (pass && p.filter_id >= 0) pass = filter_exec(ix, filters[p.filter_id], d, unsup);
            int tot; const int off = block_excl_scan(c, pass ? 1 : 0, sh.scan, tot);
            if (pass && have + off < want) { sh.keep_doc[have + off] = d; sh.keep_score[have + off] = 65535.f; sh.keep_tie[have + off] = 0; }
            have += tot;
        }
        if (unsup) sh.bcast[5] = 1;
        c.sync();
        if (sh.bcast[5]) status |= 2;
        n_rec = have < want ? have : want;
        if (O.shard_info && c.tid() == 0) O.shard_info[(size_t)q * 8 + 6] = -2;      // shards: the hosts take the shards' records in shard order
    }
    // Shards: the hosts truncate the merged coverage records (mode 0) and cut a list of the <= 3-character rule at max (mode 2), then filter:
    // such a shard reports its records unfiltered, with their filter outcomes and facet value ids (O.rec_post). A whole Stage-1 list (mode 1;
    // a short query's list in any mode: the global cut already kept it at max) is filtered here, and the blank query's browse above.
    const bool host_filter = O.shard_info && !browse && !(mode == 1 || (mode != 0 && p.short_kind != 0));
    // ---- ApplyFilter (ResultProcessor.cs:56-69), ApplyBoosts / ApplySort, facets over the post-processed records, Take(max)
    if (c.tid() == 0) {
        int nk = n_rec; bool unsupported = false;
        if (browse) { /* filtered above */ }
        else if (p.filter_id >= 0 && p.filter_id < n_filters) {
            const FilterProg fp = filters[p.filter_id]; int w = 0;
            if (!host_filter) for (int i = 0; i < nk; i++) if (filter_exec(ix, fp, sh.keep_doc[i], unsupported)) { sh.keep_doc[w] = sh.keep_doc[i]; sh.keep_score[w] = sh.keep_score[i]; sh.keep_tie[w] = sh.keep_tie[i]; w++; }
            if (!host_filter) nk = w;
        } else if (p.filter_id >= n_filters) status |= 2;
        if (unsupported) status |= 2;
        sh.bcast[5] = 0; sh.bcast[6] = nk; sh.bcast[7] = status;
    }
    c.sync();
    status = sh.bcast[7];
    if (post && !browse && (post[q].n_boosts > 0 || post[q].sort_column != IFX_SORT_NONE)) {
        const ifx_query_post& P = post[q]; bool run = true;
        for (int k = 0; k < P.n_boosts; k++) if (P.boost_filter[k] < 0 || P.boost_filter[k] >= n_filters) { status |= 2; run = false; }      // unknown filter id
        if (O.shard_info) { status |= 2; run = false; }                 // post-processing belongs after the hosts' merge of the shards
        if (mode == 1 && p.short_kind != 0 && B.s1_total && B.s1_total[q] > n_rec) { status |= 4; run = false; }      // only a prefix of the short-query list is here
        if (run) { post_process(c, ix, P, filters, sh, sh.bcast[6]); if (sh.bcast[5]) status |= 2; }
    }
    if (c.tid() == 0) {
        int nk = sh.bcast[6];
        int nf = 0;
        // shards: the hosts count the facets of the records they keep; a whole Stage-1 list is counted here in full (no cut at 100 values per
        // column), for the hosts to sum over the shards -- at most fcap rows (more sets IFX_Q_OVERFLOW, as an unsharded table over fcap does)
        if (p.enable_facets && O.fcap > 0 && nk > 0 && !(O.shard_info && (browse || host_filter))) {
            const int32_t* kd = sh.keep_doc;
            nf = facet_table(ix, nk, [&](int col, int i) { return ix.columns[col].value_id[kd[i]]; }, [](int) { return 1; }, O.shard_info ? 0x7fffffff : 100,
                             sh.fv, sh.fc, O.facet_col + (size_t)q * O.fcap, O.facet_val + (size_t)q * O.fcap, O.facet_cnt + (size_t)q * O.fcap, O.fcap, status);
        }
        if (mode == 1 && p.short_kind != 0 && p.filter_id < 0 && B.s1_total && B.s1_total[q] > nk) nk = B.s1_total[q];      // the reference returns the WHOLE short-query list: TotalCandidates counts it
        O.n_facets[q] = nf; O.total[q] = browse ? 0 : nk;       // (TotalCandidates is not set on the browse path)
        int nout = nk < p.max_results ? nk : p.max_results; if (nout > O.cap) nout = O.cap; if (nout > n_rec && !browse && p.filter_id < 0) nout = n_rec;
        for (int i = 0; i < nout; i++) { size_t oo = (size_t)q * O.cap + i; O.key[oo] = ix.doc_key[sh.keep_doc[i]]; O.score[oo] = sh.keep_score[i]; O.tie[oo] = sh.keep_tie[i]; }
        if (O.rec_post) {      // shards: per record the filter outcome (evaluated by the shard that owns the document) and its facet value ids
            const bool flt = host_filter && p.filter_id >= 0 && p.filter_id < n_filters; bool unsupported = false;
            for (int i = 0; i < nout; i++) { int32_t* r = O.rec_post + ((size_t)q * O.cap + i) * O.rec_stride; const int d = sh.keep_doc[i];
                r[0] = flt ? (filter_exec(ix, filters[p.filter_id], d, unsupported) ? 1 : 0) : 1;
                int k = 1;
                for (int col = 0; col < ix.n_columns; col++) { const Column& C = ix.columns[col]; if (!(C.flags & 2)) continue;
                    const int id = C.value_id[d]; r[k++] = (id >= 0 && C.dict.off[id + 1] != C.dict.off[id]) ? id : -1; } }
            if (unsupported) status |= 2;
        }
        O.n[q] = nout; O.status[q] = status;
    }
    c.sync();
}

}  // namespace ifx
