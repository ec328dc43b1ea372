// infidex_b200 -- device-side construction of the index's derived structures (SURVEY.md 8f-3, the part that follows the CSR):
// forward index (doc -> (term, tf) pairs), container skip tables, dense-term bitmaps + rank directories. They are pure functions
// of the uploaded CSR postings, so ifx_index_create derives them on the GPU right after the upload instead of looping over
// 10^9 postings on one host thread. Written against ifx::Ctx like the search kernels, so the host emulation of the
// test suite runs these same kernels through the launch shim.
#pragma once
#include "ifx_stage1.h"

namespace ifx {

// ---- exclusive scan of u32 counts into i64 offsets (n + 1 outputs): tile sums -> one-block scan of the tile sums -> final pass ----
// Every block covers SCAN_TILE entries whatever its size (SCAN_THREADS or a divisor of it), in slices of SCAN_PER entries per
// thread: one slice with SCAN_THREADS threads.
constexpr int SCAN_TILE = 4096, SCAN_THREADS = 256, SCAN_PER = SCAN_TILE / SCAN_THREADS;

IFX_GLOBAL void IFX_BOUNDS(SCAN_THREADS) k_scan_tile_sums(const unsigned* cnt, int64_t n, unsigned long long* tile_sum) {
    IFX_SHARED ScanTmpT<unsigned long long> wt; Ctx c; unsigned long long s = 0;
    for (int s0 = 0; s0 < SCAN_TILE; s0 += SCAN_PER * c.nthreads()) {
        const int64_t base = (int64_t)c.block() * SCAN_TILE + s0 + c.tid();
        for (int k = 0; k < SCAN_PER; k++) { int64_t i = base + (int64_t)k * c.nthreads(); if (i < n) s += cnt[i]; }
    }
    unsigned long long tot; block_excl_scan(c, s, wt, tot);
    if (c.tid() == 0) tile_sum[c.block()] = tot;
}
IFX_GLOBAL void IFX_BOUNDS(1024) k_scan_tiles(unsigned long long* tile_sum, int64_t n_tiles) {   // in place -> exclusive; one block
    IFX_SHARED ScanTmpT<unsigned long long> wt; Ctx c; unsigned long long run = 0;
    for (int64_t b0 = 0; b0 < n_tiles; b0 += c.nthreads()) {
        int64_t i = b0 + c.tid(); unsigned long long v = i < n_tiles ? tile_sum[i] : 0ULL, tot;
        unsigned long long ex = block_excl_scan(c, v, wt, tot);
        if (i < n_tiles) tile_sum[i] = run + ex;
        run += tot;
    }
}
IFX_GLOBAL void IFX_BOUNDS(SCAN_THREADS) k_scan_final(const unsigned* cnt, int64_t n, const unsigned long long* tile_excl, int64_t* out /* n + 1 */) {
    IFX_SHARED ScanTmpT<unsigned long long> wt; Ctx c; unsigned long long run = tile_excl[c.block()];
    for (int s0 = 0; s0 < SCAN_TILE; s0 += SCAN_PER * c.nthreads()) {
        const int64_t base = (int64_t)c.block() * SCAN_TILE + s0 + (int64_t)c.tid() * SCAN_PER; unsigned v[SCAN_PER]; unsigned long long s = 0;
        for (int k = 0; k < SCAN_PER; k++) { int64_t i = base + k; v[k] = i < n ? cnt[i] : 0u; s += v[k]; }
        unsigned long long tot; unsigned long long ex = run + block_excl_scan(c, s, wt, tot);
        for (int k = 0; k < SCAN_PER; k++) { int64_t i = base + k; if (i < n) out[i] = (int64_t)ex; ex += v[k]; }
        run += tot;
    }
    if (c.block() == c.nblocks() - 1 && c.tid() == c.nthreads() - 1) out[n] = (int64_t)run;
}

// ---- forward index: one warp per live term row (grid-stride), 4 postings per lane in flight ------------------------------------
IFX_GLOBAL void IFX_BOUNDS(256) k_fwd_count(const int64_t* row_ptr, const int32_t* df, int T, const int32_t* post_doc, unsigned* cnt) {
    Ctx c;
    for (int64_t t = c.gwarp(); t < T; t += c.gwarps()) {
        if (df[t] <= 0) continue;
        const int64_t r0 = row_ptr[t], r1 = row_ptr[t + 1];
        for (int64_t i = r0 + c.lane(); i < r1; i += c.WS) atomic_add(&cnt[post_doc[i]], 1u);
    }
}
IFX_GLOBAL void IFX_BOUNDS(256) k_fwd_scatter(const int64_t* row_ptr, const int32_t* df, int T, const int32_t* post_doc, const uint8_t* post_tf,
                                              const int64_t* fwd_ptr, unsigned* cursor, int32_t* fwd_term, uint8_t* fwd_tf) {
    Ctx c;
    for (int64_t t = c.gwarp(); t < T; t += c.gwarps()) {
        if (df[t] <= 0) continue;
        const int64_t r0 = row_ptr[t], r1 = row_ptr[t + 1];
        for (int64_t i0 = r0 + c.lane(); i0 < r1; i0 += 4 * c.WS) {
            int d[4]; uint8_t w[4]; unsigned at[4];
            for (int u = 0; u < 4; u++) { int64_t i = i0 + c.WS * u; d[u] = i < r1 ? post_doc[i] : -1; w[u] = i < r1 ? post_tf[i] : (uint8_t)0; }
            for (int u = 0; u < 4; u++) if (d[u] >= 0) at[u] = atomic_add(&cursor[d[u]], 1u);
            for (int u = 0; u < 4; u++) if (d[u] >= 0) { const int64_t o = fwd_ptr[d[u]] + at[u]; fwd_term[o] = (int32_t)t; fwd_tf[o] = w[u]; }
        }
    }
}

// ---- container skip tables: one thread per (skip row, container boundary) ---------------------------------------------------
IFX_GLOBAL void IFX_BOUNDS(256) k_skip_table(const int64_t* row_ptr, const int32_t* skip_terms, int n_skip, int n_cont, const int32_t* post_doc, int32_t* skip_ptr) {
    Ctx c; const int64_t idx = c.gtid(), per = n_cont + 1;
    if (idx >= (int64_t)n_skip * per) return;
    const int t = skip_terms[idx / per], cb = (int)(idx % per);
    skip_ptr[idx] = (int32_t)(lower_bound_i32(post_doc, row_ptr[t], row_ptr[t + 1], cb << 16) - row_ptr[t]);
}

// ---- dense-term bitmaps + rank directories: one block per dense row ---------------------------------------------------------
IFX_GLOBAL void IFX_BOUNDS(512) k_bitmap_fill(const int64_t* row_ptr, const int32_t* bm_terms, int bm_words, const int32_t* post_doc, unsigned* bm_bits) {
    Ctx c; const int t = bm_terms[c.block()]; unsigned* b = bm_bits + (size_t)c.block() * bm_words;
    const int64_t r0 = row_ptr[t], r1 = row_ptr[t + 1];
    for (int64_t i = r0 + c.tid(); i < r1; i += (unsigned)c.nthreads()) { int d = post_doc[i]; atomic_or(&b[d >> 5], 1u << (d & 31)); }
}
IFX_GLOBAL void IFX_BOUNDS(512) k_bitmap_rank(int bm_words, const unsigned* bm_bits, int32_t* bm_rank) {
    IFX_SHARED ScanTmpT<unsigned long long> wt; Ctx c;
    const unsigned* b = bm_bits + (size_t)c.block() * bm_words; int32_t* r = bm_rank + (size_t)c.block() * bm_words; unsigned long long run = 0;
    for (int w0 = 0; w0 < bm_words; w0 += 4 * c.nthreads()) {
        const int wb = w0 + c.tid() * 4; unsigned v[4]; unsigned long long s = 0;
        for (int u = 0; u < 4; u++) { v[u] = wb + u < bm_words ? b[wb + u] : 0u; s += popc(v[u]); }
        unsigned long long tot; unsigned long long ex = run + block_excl_scan(c, s, wt, tot);
        for (int u = 0; u < 4; u++) { if (wb + u < bm_words) r[wb + u] = (int32_t)ex; ex += popc(v[u]); }
        run += tot;
    }
}

}  // namespace ifx
