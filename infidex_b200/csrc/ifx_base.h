// infidex_b200 -- shared POD layout + execution-context abstraction.
//
// The search kernels and their __global__ wrappers are written once against `Ctx` (a cooperative group of threads):
//   * CUDA build (nvcc, sm_90a): Ctx == one CTA; sync() is __syncthreads, ballot() is __ballot_sync, atomics are
//     the hardware ones. This is the product.
//   * IFX_EMU build (g++, tests only): Ctx == one host thread (group size 1, warp size 1). The kernels are host functions
//     and the launch shim of ifx_api.inl calls them once per block, so the CPU test suite runs the product's host driver
//     and kernels, the index build's included, and checks them against the oracle without a GPU. It is never loaded by the product.
#pragma once
#include <stdint.h>
#include <stddef.h>

#ifdef IFX_EMU
#include <cstring>
#include <cmath>
#include <algorithm>
#define IFX_FN inline
#define IFX_FN_OUTLINED inline
#define IFX_GLOBAL
#define IFX_BOUNDS(...)
#define IFX_SHARED static thread_local                  // static shared memory: one instance, reused by the blocks run in turn
#define IFX_DYN_SHARED(name) unsigned char* name = ifx::emu_grid().smem
#else
#include <cuda_runtime.h>
#define IFX_GLOBAL __global__
#define IFX_BOUNDS(...) __launch_bounds__(__VA_ARGS__)
#define IFX_SHARED __shared__
#define IFX_DYN_SHARED(name) extern __shared__ __align__(16) unsigned char name[]
#define IFX_FN __device__ __forceinline__
// large helpers with several call sites inside one kernel: one shared body keeps the instruction footprint (and the i-cache
// miss rate of divergent warps) down
#ifdef IFX_COV_INLINE_ALL
#define IFX_FN_OUTLINED __device__ __forceinline__
#else
#define IFX_FN_OUTLINED __device__ __noinline__
#endif
#endif

namespace ifx {

constexpr int MAX_QLEN = 256;        // UTF-16 units of a (normalised) query; longer -> IFX_Q_OVERFLOW
constexpr int MAX_RAW_TOKENS = 128;  // VectorModel.cs:381 (ArrayPool rent of 128 RawToken)
constexpr int MAX_TERMS = 128;
constexpr int MAX_FUZZY = 16;        // unknown words (len >= 4) expanded per query
#define IFX_QDBG 24                   // int64 slots of the per-query Stage-1 debug record (ifx_debug_stage1_queries)
constexpr int LD1_CAP = 1024;        // VectorModel.cs:662 stackalloc int[1024]
constexpr int CHUNK = 4096;          // Bm25Scorer.cs:209 blockSize
constexpr int MAX_K = 1024;          // coverage depth supported by the on-chip heap
constexpr int AFFIX_CAP = 4096;      // WordMatcher.cs:41 MaxFstAffixTermsPerQuery
constexpr int MAX_QTOK = 64;         // coverage query tokens (len >= 2, deduped)
constexpr int MAX_WM_WORDS = 32;     // query words (len >= 2) looked up in the WordMatcher
constexpr int MAX_TOKLEN = 96;       // Levenshtein row length of the coverage kernel; a query word longer than this raises IFX_Q_OVERFLOW
constexpr int MAX_CONTAINERS = 8192; // 65536-doc containers per shard (N <= 536M)
constexpr char16_t PAD = 0xFFFF;

struct StrDict {                     // n strings + open-addressing hash (key = hash64 of the UTF-16 units)
    const uint16_t* chars; const uint32_t* off; int32_t n;
    const uint64_t* hkeys; const int32_t* hvals; uint32_t hmask;
};

struct DocsetDict { StrDict keys; const int64_t* row_ptr; const int32_t* doc_id; };

struct Column { const int32_t* value_id; StrDict dict; const double* dict_num; const uint8_t* dict_is_num; int32_t flags; int32_t name_const_hash_lo;
                const int32_t* rank; };     // SortBy order per dictionary entry (ifx_column_set_order), null until registered

struct DevIndex {
    int32_t n_docs, n_live; float avgdl; int32_t stop_term_limit;
    const int64_t* doc_key; const uint8_t* deleted; const float* doc_len;
    const int32_t* key_first;        // null when every DocumentKey is unique; else per doc the first live document with the same key (DocumentCollection.GetDocumentByPublicKey,
                                     // Core/DocumentCollection.cs:60-82): segments of one document share a key and are consolidated per key (SegmentProcessor.cs:15-37)
    const uint16_t* text; const int64_t* text_off;
    const int64_t* tok_ptr; const uint32_t* tok_tab;   // per document: its tokens as the coverage stage needs them (ifx_cov.h doc_tokens_emit), derived at index creation
    StrDict first_token; const uint16_t* token_count;
    StrDict terms; const int32_t* df; const int64_t* row_ptr; const int32_t* post_doc; const uint8_t* post_tf;
    const int32_t* term_sorted;      // term ordinals in ordinal-lexicographic order (trie DFS order)
    const unsigned long long* term_sig;   // per sorted position: 64-bit character-set signature (LD1 pre-filter)
    // forward index (doc -> its (term, tf) pairs, terms with df > 0 only): one lookup latency per candidate for the sparse chunks
    const int64_t* fwd_ptr; const int32_t* fwd_term; const uint8_t* fwd_tf;
    // the same dictionary grouped by term length (stable, so lexicographic inside a group): LD1 scans touch lengths m-1..m+1 only
    const int32_t* len_ptr;          // [257] group start per length (255 = 255 or longer), [256] = n terms
    const unsigned long long* len_sig;   // signature per grouped position
    const int32_t* len_ord;          // term ordinal per grouped position
    const int32_t* skip_id;          // per term: row of the container skip table, or -1 (short lists)
    const int32_t* skip_ptr;         // [n_skip][n_cont + 1] offset (relative to the row start) of the first posting with doc >= c << 16
    int32_t n_cont;                  // 65536-doc containers in this shard
    const int32_t* bm_id;            // per term: row of the dense-term bitmap table, or -1
    const unsigned* bm_bits;         // [n_bm][bm_words] membership bitmap of the posting list (dense terms: df >= n_docs / 32)
    const int32_t* bm_rank;          // [n_bm][bm_words] postings before doc (w << 5): posting index = rank[w] + popc(bits[w] & (bit - 1))
    int32_t bm_words;
    StrDict words; const float* word_idf;
    DocsetDict prefix, wm_exact, wm_ld1;
    const int32_t* prefix_gcard;     // doc-id-range shards: DocSet cardinality over ALL shards per prefix key (null: unsharded, the local row length)
    StrDict affix;                   // affix words in ordinal-lexicographic order
    const int32_t* affix_fwd_doc;    // last doc per affix word (forward order)
    const int32_t* affix_rev;        // indices into `affix`, ordered by the reversed string
    const int32_t* affix_rev_doc;    // last doc, in reverse-trie order
    const uint16_t* lower; const uint16_t* upper; const uint8_t* cflags;   // 65536-entry tables
    unsigned delim_ascii[4];         // bit c set: ASCII char c is a token delimiter (cflags[c] & 4), kept in the kernel parameters
    int32_t fwd_avg_bytes;           // average bytes of one document's forward list (+ its pointers): cost model of the per-candidate lookup mode
    const float* log2_len;           // MathF.Log2(len + 1) for len < 1024 (host glibc)
    const float* idf_table;          // Bm25Scorer.ComputeIdf(n_live, df) for df in [0, idf_table_n): evaluated on the host with the
    int32_t idf_table_n;             // C runtime's logf (what MathF.Log calls), so device scores cannot drift from the reference by an ulp
    int32_t n_columns; const Column* columns;
    // short-query path (ifx_short.h): champion lists of the 1-character prefixes, raw IndexedText of the documents that normalisation changed
    int32_t n_champ; const uint16_t* champ_chars; const int32_t* champ_off; const int32_t* champ_doc; const float* champ_score;
    int32_t n_raw; const int32_t* raw_doc; const int64_t* raw_off; const uint16_t* raw_chars;
};

IFX_FN uint64_t hash64(const uint16_t* s, int n) {
    uint64_t h = 0xcbf29ce484222325ULL ^ (uint64_t)n;
    for (int i = 0; i < n; i++) { h ^= s[i]; h *= 0x100000001b3ULL; }
    h ^= h >> 29; h *= 0xbf58476d1ce4e5b9ULL; h ^= h >> 32;
    return h | 1ULL;                 // 0 marks an empty slot
}

IFX_FN unsigned long long char_sig(const uint16_t* s, int n) {   // one bit per (hashed) character present
    unsigned long long g = 0; for (int i = 0; i < n; i++) g |= 1ULL << ((s[i] * 0x9E37u >> 4) & 63); return g;
}

IFX_FN int dict_lookup(const StrDict& d, const uint16_t* s, int n) {
    if (d.n == 0) return -1;
    uint64_t h = hash64(s, n); uint32_t slot = (uint32_t)(h >> 7) & d.hmask;
    for (;;) {
        uint64_t k = d.hkeys[slot];
        if (k == 0) return -1;
        if (k == h) {
            int idx = d.hvals[slot]; uint32_t b = d.off[idx], e = d.off[idx + 1];
            if ((int)(e - b) == n) { bool eq = true; for (int i = 0; i < n; i++) if (d.chars[b + i] != s[i]) { eq = false; break; } if (eq) return idx; }
        }
        slot = (slot + 1) & d.hmask;
    }
}

// ---- execution context ------------------------------------------------------------------------------------------
// block() / nblocks() are blockIdx.x / gridDim.x; gtid() / gthreads() and gwarp() / gwarps() number the threads and the warps of the
// whole grid. A block-strided loop of a kernel wrapper adds `(unsigned)c.nthreads()`: wrap-around arithmetic like blockDim.x,
// so nvcc emits the plain loop instead of computing a trip count.
#ifdef IFX_EMU
// The block the launch shim is running (one host thread per block) and its dynamic shared memory.
struct EmuGrid { unsigned block = 0, nblocks = 1; unsigned char* smem = nullptr; };
inline EmuGrid& emu_grid() { static thread_local EmuGrid g; return g; }
struct Ctx {
    static constexpr int WS = 1;
    unsigned b_ = emu_grid().block, nb_ = emu_grid().nblocks;
    int tid() const { return 0; } int nthreads() const { return 1; } int lane() const { return 0; } int warp() const { return 0; } int nwarps() const { return 1; }
    unsigned block() const { return b_; } unsigned nblocks() const { return nb_; }
    int64_t gtid() const { return b_; } int64_t gthreads() const { return nb_; } int64_t gwarp() const { return b_; } int64_t gwarps() const { return nb_; }
    void sync() const {}
    void sync_workers(int) const {}
    void sync_team(int) const {}
    void syncwarp() const {}
    unsigned ballot(bool p) const { return p ? 1u : 0u; }
    unsigned lanemask_lt() const { return 0u; }
    template <class T> T shfl(T v, int) const { return v; }
};
inline unsigned atomic_or(unsigned* p, unsigned v) { unsigned o = *p; *p = o | v; return o; }
inline int atomic_add(int* p, int v) { int o = *p; *p = o + v; return o; }
inline unsigned atomic_add(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
inline unsigned atomic_and(unsigned* p, unsigned v) { unsigned o = *p; *p = o & v; return o; }
inline int atomic_min(int* p, int v) { int o = *p; if (v < o) *p = v; return o; }
inline int atomic_max(int* p, int v) { int o = *p; if (v > o) *p = v; return o; }
inline unsigned long long atomic_max(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; if (v > o) *p = v; return o; }
inline unsigned long long atomic_add64(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; *p = o + v; return o; }
inline int popc(unsigned v) { return __builtin_popcount(v); }
inline int ffs32(unsigned v) { return __builtin_ffs((int)v); }
inline int popc64(unsigned long long v) { return __builtin_popcountll(v); }
inline int clz64(long long v) { return v ? __builtin_clzll((unsigned long long)v) : 64; }
inline float dev_logf_exact(float x) { return std::log(x); }
inline unsigned long long globaltimer() { return 0; }
#else
struct Ctx {
    static constexpr int WS = 32;
    __device__ int tid() const { return threadIdx.x; } __device__ int nthreads() const { return blockDim.x; }
    __device__ int lane() const { return threadIdx.x & 31; } __device__ int warp() const { return threadIdx.x >> 5; } __device__ int nwarps() const { return blockDim.x >> 5; }
    __device__ unsigned block() const { return blockIdx.x; } __device__ unsigned nblocks() const { return gridDim.x; }
    __device__ int64_t gtid() const { return (int64_t)blockIdx.x * blockDim.x + threadIdx.x; } __device__ int64_t gthreads() const { return (int64_t)gridDim.x * blockDim.x; }
    __device__ int64_t gwarp() const { return gtid() >> 5; } __device__ int64_t gwarps() const { return gthreads() >> 5; }
    __device__ void sync() const { __syncthreads(); }
    // named barrier 1 over the `n` worker threads of a warp-specialised region (n: multiple of 32; every worker warp calls it)
    __device__ void sync_workers(int n) const { asm volatile("bar.sync 1, %0;" :: "r"(n) : "memory"); }
    // named barrier 2 over the `n` threads of the small-chunk team
    __device__ void sync_team(int n) const { asm volatile("bar.sync 2, %0;" :: "r"(n) : "memory"); }
    __device__ void syncwarp() const { __syncwarp(); }
    __device__ unsigned ballot(bool p) const { return __ballot_sync(0xffffffffu, p); }
    __device__ unsigned lanemask_lt() const { return (1u << (threadIdx.x & 31)) - 1u; }
    template <class T> __device__ T shfl(T v, int src) const { return __shfl_sync(0xffffffffu, v, src); }
};
__device__ __forceinline__ unsigned atomic_or(unsigned* p, unsigned v) { return atomicOr(p, v); }
__device__ __forceinline__ int atomic_add(int* p, int v) { return atomicAdd(p, v); }
__device__ __forceinline__ unsigned atomic_add(unsigned* p, unsigned v) { return atomicAdd(p, v); }
__device__ __forceinline__ unsigned atomic_and(unsigned* p, unsigned v) { return atomicAnd(p, v); }
__device__ __forceinline__ int atomic_min(int* p, int v) { return atomicMin(p, v); }
__device__ __forceinline__ int atomic_max(int* p, int v) { return atomicMax(p, v); }
__device__ __forceinline__ unsigned long long atomic_max(unsigned long long* p, unsigned long long v) { return atomicMax(p, v); }
__device__ __forceinline__ unsigned long long atomic_add64(unsigned long long* p, unsigned long long v) { return atomicAdd(p, v); }
__device__ __forceinline__ int popc(unsigned v) { return __popc(v); }
__device__ __forceinline__ int ffs32(unsigned v) { return __ffs((int)v); }
__device__ __forceinline__ int popc64(unsigned long long v) { return __popcll(v); }
__device__ __forceinline__ int clz64(long long v) { return __clzll(v); }
// MathF.Log on the reference host is glibc logf (<1 ulp, effectively correctly rounded); evaluate in fp64 and round once.
__device__ __forceinline__ float dev_logf_exact(float x) { return (float)log((double)x); }
__device__ __forceinline__ unsigned long long globaltimer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#endif

// Bm25Scorer.ComputeIdf (src/Infidex/Indexing/Bm25Scorer.cs:686-695) -- table lookup, see DevIndex::idf_table
IFX_FN float compute_idf(const DevIndex& ix, int df) {
    if (df <= 0 || ix.n_live <= 0) return 0.f;
    if (df < ix.idf_table_n) return ix.idf_table[df];
    float d = (float)df, N = (float)ix.n_live;          // df > stop-term limit: the term is dropped by the caller anyway
    float ratio = (N - d + 0.5f) / (d + 0.5f);
    return ratio <= 0.f ? 0.f : dev_logf_exact(ratio + 1.f);
}

// ---- per-query plan written by k_prepare, completed by k_expand, consumed by k_stage1 / k_wm / k_stage2 -----------
struct QTerm {
    int64_t list_off;     // offset into post_doc/post_tf (known term) or into the fuzzy pool (fuzzy term)
    int32_t list_len;     // postings in the list (== df for live lists)
    int32_t df;
    int32_t term_id;      // >= 0 known term; -1 fuzzy union
    float idf, max_score;
};

struct FuzzyReq { uint16_t off, len; int32_t term_slot; };

struct CovToken { uint16_t off, len; };

struct QueryPlan {
    int32_t status;
    int32_t qlen;                          // full normalised lower query (Stage 2 text)
    int32_t tlen;                          // Stage-1 text (short words removed when mixed)
    int32_t n_terms;                       // slots used in `terms` (reference order; df filter applied later)
    int32_t n_fuzzy;
    int32_t depth, max_results, enable_coverage, filter_id, enable_facets;
    int32_t short_skip_coverage;           // SearchPipeline.cs:139-142 (3-char query whose prefix docset > 500)
    int32_t is_short3;                     // SearchPipeline.cs:110-112
    int32_t short_kind;                    // 0: n-gram path; 1 / 2: no word of >= 3 characters -- one character / ShortQueryProcessor.SearchShortQuery (ifx_short.h)
    int32_t short_no_cov;                  // short-query path and the coverage stage is not allowed (SearchPipeline.cs:133-170)
    uint16_t qtext[MAX_QLEN];
    uint16_t ttext[MAX_QLEN];
    QTerm terms[MAX_TERMS];
    FuzzyReq fuzzy[MAX_FUZZY];
};

struct BatchCounters { int32_t n_fuzzy_items; int32_t overflow; unsigned long long fuzzy_pool_used; unsigned long long algo_bytes; unsigned long long s1_ns_sum; unsigned long long s1_ns_max; unsigned long long s1_cand_sum;
                       unsigned long long s1_pool_used; int32_t s1_deferred, s1_n_light, s1_n_heavy, s1_wave, s1_n_mid, n_short; };

struct FuzzyItem { int32_t query; int32_t slot; };

}  // namespace ifx
