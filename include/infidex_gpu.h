/* infidex_gpu.h -- C-ABI of the H100-native Infidex search path (libinfidex_gpu.so).
 *
 * Drop-in boundary (SURVEY.md 8b): the reference (lofcz/Infidex, C#) has no FFI of its own; this ABI is what a
 * P/Invoke shim behind `SearchEngine` binds (see INTEGRATION.md):
 *   ifx_index_create   <- end of SearchEngine.IndexDocumentsInternal (src/Infidex/SearchEngine.cs:183-185) and
 *                         SearchEngine.Load (:426-441): marshal the immutable in-memory index once.
 *   ifx_filter_register<- ResultProcessor.ApplyFilter's compile-once cache (src/Infidex/Scoring/ResultProcessor.cs:37),
 *                         fed with BytecodeSerializer.Serialize output (src/Infidex/Filtering/BytecodeSerializer.cs:16-62).
 *   ifx_search_batch   <- the body of SearchEngine.Search between the read lock and `new Result(...)`
 *                         (src/Infidex/SearchEngine.cs:298-316): SearchPipeline.Execute + ApplyPostProcessing(filter)
 *                         + FacetBuilder.BuildFacets + Take(max).
 *   ifx_index_destroy  <- SearchEngine.Dispose (src/Infidex/SearchEngine.cs:477).
 * All pointers are borrowed for the duration of the call; outputs are caller-allocated; the handle owns device memory.
 * Strings are UTF-16 code units (C# `char`), little-endian. No CPU fallback exists: every call fails with
 * IFX_ERR_NO_DEVICE when no CUDA device is usable.
 */
#ifndef INFIDEX_GPU_H
#define INFIDEX_GPU_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    IFX_OK = 0,
    IFX_ERR_INVALID = 1,      /* bad argument / malformed image or bytecode */
    IFX_ERR_NO_DEVICE = 2,    /* no CUDA device / driver failure */
    IFX_ERR_OOM = 3,          /* device or workspace memory exhausted */
    IFX_ERR_UNSUPPORTED = 4,  /* feature outside the built path (see per-query status) */
    IFX_ERR_CUDA = 5
};

/* per-query status bits in ifx_batch_result.status */
enum {
    IFX_Q_OK = 0,
    IFX_Q_UNSUPPORTED_OP = 2, /* MATCHES (regex) opcode; a query without a word of >= 3 characters on a doc-id-range shard whose documents
                                 share a DocumentKey (one GPU answers those) */
    IFX_Q_OVERFLOW = 4,       /* a fixed device buffer was too small for this query */
    IFX_Q_EMPTY = 8           /* blank query -> empty result (SearchEngine.cs:295-296) */
};

typedef struct ifx_strings {          /* n strings: chars[off[i] .. off[i+1]) */
    const uint16_t* chars;
    const uint32_t* off;              /* n + 1 entries */
    int32_t n;
} ifx_strings;

typedef struct ifx_docset_dict {      /* string key -> ascending doc-id list (CSR) */
    ifx_strings keys;
    const int64_t* row_ptr;           /* keys.n + 1 */
    const int32_t* doc_id;
} ifx_docset_dict;

enum { IFX_COL_FILTERABLE = 1, IFX_COL_FACETABLE = 2, IFX_COL_SORTABLE = 4 };   /* SORTABLE: emitted because the field is Field.Sortable */

typedef struct ifx_column {           /* Field.Value.ToString() dictionary-encoded per document */
    const uint16_t* name; int32_t name_len;
    int32_t flags;
    const int32_t* value_id;          /* [n_docs], -1 = null / missing field */
    ifx_strings dict;                 /* distinct ToString() values */
} ifx_column;

/* The immutable in-memory index of the reference, flattened (SURVEY.md 8b / App. A1). Internal doc ids are the
 * insertion indices of DocumentCollection (Core/DocumentCollection.cs:21). */
typedef struct ifx_index_image {
    int32_t n_docs;                   /* _documents.Count (incl. deleted) */
    int32_t n_live;                   /* DocumentCollection.Count */
    float avgdl;                      /* VectorModel._avgDocLength */
    const int64_t* doc_key;           /* Document.DocumentKey */
    const uint8_t* deleted;           /* Document.Deleted */
    const float* doc_len;             /* VectorModel._docLengths */
    const uint16_t* text_chars;       /* TextNormalizer.Normalize(Document.IndexedText), original case */
    const int64_t* text_off;          /* n_docs + 1 */
    ifx_strings first_token;          /* DocumentMetadata.FirstToken per doc (n = n_docs) */
    const uint16_t* token_count;      /* DocumentMetadata.TokenCount */
    ifx_strings terms;                /* TermCollection, ordinal order */
    const int32_t* df;                /* Term.DocumentFrequency (-1 = stop term) */
    const int64_t* row_ptr;           /* terms.n + 1; empty row for df <= 0 */
    const int32_t* post_doc;          /* Term._documentIds */
    const uint8_t* post_tf;           /* Term._weights */
    ifx_strings words;                /* VectorModel.WordIdfCache keys (lower case) */
    const float* word_idf;
    ifx_docset_dict prefix;           /* PositionalPrefixIndex DocSet per 1..3-char prefix */
    ifx_docset_dict wm_exact;         /* WordMatcher._exactIndex */
    ifx_docset_dict wm_ld1;           /* WordMatcher._ld1Index */
    ifx_strings affix_words;          /* WordMatcher FST terms (any order) */
    const int32_t* affix_last_doc;    /* the single doc its trie output resolves to (WordMatcher.cs:166-196) */
    int32_t n_columns;
    const ifx_column* columns;        /* filterable / facetable fields, schema order of the first document */
    /* short-query path (queries without a word of >= 3 characters; Scoring/ShortQueryProcessor.cs, Indexing/ShortQuery/ShortQueryResolver.cs) */
    int32_t n_champ_chars;            /* ShortQueryResolver champion lists of the 1-character prefixes: */
    const uint16_t* champ_chars;      /*   the character, */
    const int32_t* champ_off;         /*   [n_champ_chars + 1] */
    const int32_t* champ_doc;         /*   internal doc ids, in the order BuildChampionLists leaves them (List.Sort by score descending, first 64); a shard: the global lists, another shard's entries -1 */
    const float* champ_score;         /*   (precedence << 8) | base */
    int32_t n_raw;                    /* documents whose IndexedText differs from its normalised form (the short-query scorers read ToLowerInvariant(IndexedText)): */
    const int32_t* raw_doc;           /*   ascending internal ids, */
    const int64_t* raw_off;           /*   [n_raw + 1] */
    const uint16_t* raw_chars;        /*   raw IndexedText, original case */
    /* doc-id-range shards (SURVEY 8e): zero / NULL for an unsharded index. A shard image holds its own documents (local ids from 0) and the
     * statistics of the WHOLE corpus: terms / df / idf ordinals, n_live, avgdl, word idf, the global prefix key set and affix dictionary. */
    const int32_t* prefix_global_card;/* [prefix.keys.n] DocSet cardinality over all shards (the selector's prefix rules are global) */
    int32_t shard_index, n_shards;
    int64_t doc_base;                 /* global internal id of this shard's document 0 */
    /* SynonymMap (Synonyms/SynonymMap.cs): zero / NULL = no map, or a map without mappings (HasCanonicalMappings false). Otherwise one
     * entry per key of the map's union-find (_parent): syn_keys[i] is the key (lower case, keys unique under OrdinalIgnoreCase) and
     * syn_canon[i] = GetCanonical(key), non-empty. The device derives the coverage text CanonicalizeText(Normalize(IndexedText)) from
     * text_chars with it. The rest of the image must have been built with the same map (the index text, metadata and prefix index are
     * canonicalised; WordMatcher and the word idf are not), and ifx_query.text must be canonicalised with it too: an index is re-created
     * whenever the map changes. */
    ifx_strings syn_keys;
    ifx_strings syn_canon;
} ifx_index_image;

typedef struct ifx_params {           /* ConfigurationParameters[400] + CoverageSetup defaults when zero-initialised via ifx_params_default */
    int32_t stop_term_limit;          /* 1 250 000 */
    int32_t device;                   /* CUDA device ordinal */
    int32_t max_batch;                /* queries per internal wave (workspace sizing) */
    int32_t reserved;
} ifx_params;

typedef struct ifx_query {
    const uint16_t* text;             /* after Trim + TextNormalizer.Normalize + ToLowerInvariant (SearchEngine.cs:264-274); with a SynonymMap
                                       * (image syn_keys.n > 0) then SynonymMap.CanonicalizeText and TextNormalizer.Normalize once more
                                       * (SearchPipeline.Execute), i.e. the text the pipeline works on */
    int32_t len;
    int32_t max_results;              /* Query.MaxNumberOfRecordsToReturn */
    int32_t coverage_depth;           /* Query.CoverageDepth (<= 1024) */
    int32_t enable_coverage;
    int32_t filter_id;                /* from ifx_filter_register, or -1 */
    int32_t enable_facets;
} ifx_query;

/* Query.EnableBoost + Query.Boosts and Query.SortBy + Query.SortAscending (ResultProcessor.ApplyBoosts / ApplySort, run after the filter
 * and before facets and Take). Optional per-query companion of ifx_query; a zero-filled entry with sort_column = IFX_SORT_NONE is "none".
 *   n_boosts          boosts whose Filter is not null (0 = no boosts, no re-sort by score); at most IFX_MAX_BOOSTS, more is IFX_ERR_INVALID
 *   boost_filter[i]   ifx_filter_register id of Boost[i].Filter; an unknown id sets IFX_Q_UNSUPPORTED_OP, as an unknown filter_id does
 *   boost_strength[i] (int)Boost[i].BoostStrength
 *   sort_column       column index (needs ifx_column_set_order first), IFX_SORT_NONE, or IFX_SORT_ALL_NULL for a SortBy field no
 *                     document has (every value null: the sort still runs and permutes equal values)
 * Records of a doc-id-range SHARD get IFX_Q_UNSUPPORTED_OP (post-processing belongs after the hosts' merge, which applies the filter and
 * builds the facets but has no boosts or SortBy yet: see ifx_batch_shard_records); a list the device holds only
 * in part (the short-query path returns its whole list) gets IFX_Q_OVERFLOW instead of a sorted prefix. The blank query ignores both. */
enum { IFX_MAX_BOOSTS = 16, IFX_SORT_NONE = -1, IFX_SORT_ALL_NULL = -2 };
typedef struct ifx_query_post {
    int32_t n_boosts;
    int32_t boost_filter[IFX_MAX_BOOSTS];
    int32_t boost_strength[IFX_MAX_BOOSTS];
    int32_t sort_column;
    int32_t sort_ascending;
} ifx_query_post;

typedef struct ifx_batch_result {     /* caller-allocated, row-major [nq][cap] */
    int32_t cap;                      /* >= max over queries of max_results */
    int32_t facet_cap;                /* facet rows per query (0 = none) */
    int64_t* doc_key;                 /* ScoreEntry.DocumentId */
    float* score;                     /* ScoreEntry.Score */
    uint8_t* tie;                     /* ScoreEntry.Tiebreaker */
    int32_t* n;                       /* [nq] records returned */
    int32_t* total_candidates;        /* [nq] Result.TotalCandidates */
    int32_t* status;                  /* [nq] IFX_Q_* bits */
    int32_t* facet_column;            /* [nq][facet_cap] column index */
    int32_t* facet_value;             /* [nq][facet_cap] dictionary id in that column */
    int32_t* facet_count;             /* [nq][facet_cap] */
    int32_t* n_facets;                /* [nq] */
} ifx_batch_result;

typedef struct ifx_stats {            /* filled by ifx_search_batch / ifx_batch_run when non-NULL */
    float ms_total;                   /* device time of the batch (CUDA events) */
    float ms_prepare, ms_expand, ms_stage1, ms_wordmatch, ms_stage2, ms_final;
    int64_t algo_bytes_stage1;        /* algorithmic bytes (SURVEY 8d B_q terms 1-3) summed over the batch */
    int64_t kernel_launches;
    int64_t h2d_bytes, d2h_bytes;
    float s1_query_ms_max;            /* longest single query inside k_select_lookup (device globaltimer) */
    float s1_query_ms_sum;            /* sum over queries of their time inside k_select_lookup */
    float ms_s1_select, ms_s1_score_warp, ms_s1_score_cta, ms_s1_finish;   /* the four Stage-1 launches that make up ms_stage1 */
    int32_t s1_light, s1_heavy;       /* queries scored one per warp (8 slots per lane) / one per CTA (last wave) */
    int32_t s1_waves;                 /* > 1: the batch outgrew the Stage-1 staging pool and was finished in waves */
    int32_t s1_mid;                   /* queries scored one per warp with 32 slots per lane (last wave) */
    int64_t s1_pool_bytes;            /* staging pool bytes used (last wave) */
} ifx_stats;

typedef struct ifx_index ifx_index;   /* opaque: device-resident index + workspaces */
typedef struct ifx_batch ifx_batch;   /* opaque: a query batch resident in device memory */

void ifx_params_default(ifx_params* p);
int  ifx_index_create(const ifx_index_image* img, const ifx_params* p, ifx_index** out);
void ifx_index_destroy(ifx_index* idx);
int  ifx_filter_register(ifx_index* idx, const uint8_t* infiscript_v1, size_t len, int* out_filter_id);
/* The order ResultProcessor.CompareValues gives the values of a column: rank[i] for dictionary entry i (n = dict.n), equal ranks <=>
 * CompareTo == 0, null / missing sorts lowest. The caller computes it (the C# shim with .NET's own comparer, so culture-dependent string
 * order never has to be decided on the device). A column may be registered again; a sort on a column without an order is IFX_ERR_INVALID. */
int  ifx_column_set_order(ifx_index* idx, int32_t column, const int32_t* rank, int32_t n);

/* host buffers in, host buffers out (the call SearchEngine.Search makes) */
int  ifx_search_batch(ifx_index* idx, const ifx_query* q, int nq, ifx_batch_result* out, ifx_stats* st);
/* the same with boosts / SortBy: post = [nq] or NULL (NULL is exactly ifx_search_batch) */
int  ifx_search_batch_post(ifx_index* idx, const ifx_query* q, const ifx_query_post* post, int nq, ifx_batch_result* out, ifx_stats* st);

/* split form: upload once, run on device (timed), read back */
int  ifx_batch_upload(ifx_index* idx, const ifx_query* q, int nq, ifx_batch** out);
int  ifx_batch_refill(ifx_batch* b, const ifx_query* q, int nq);      /* the same handle for the next batch: device buffers are kept while they fit; clears the boosts / SortBy */
int  ifx_batch_set_post(ifx_batch* b, const ifx_query_post* post);    /* [nq] boosts / SortBy of the uploaded queries, NULL = none; kept until the next refill */
int  ifx_batch_run(ifx_batch* b, ifx_stats* st);
int  ifx_batch_download(ifx_batch* b, ifx_batch_result* out);
void ifx_batch_free(ifx_batch* b);

/* doc-id-range shards (SURVEY.md 8e): one index handle per shard (ifx_index_image.n_shards > 1), the batch run split where the shards' hosts
 * exchange data. phase 1: query preparation + LD1 expansion; then all-reduce(sum) of ifx_batch_fuzzy_df (document frequency of every LD1
 * union: its idf is a corpus-level quantity). phase 2: count pass of the candidate selection; all-reduce(sum) of ifx_batch_select_counts (the tier
 * rules compare corpus-level cardinalities). phase 3: selection, tf lookups, scoring; then all-gather of ifx_batch_stage1_lists and
 * ifx_batch_stage1_restrict (global top-`depth` cut, global top score for normBm25). phase 4: WordMatcher lookups; ifx_batch_wm_counts
 * and ifx_batch_wm_apply. phase 5: coverage / fusion, truncation, filter, facets; ifx_batch_download gives the shard's records, which every
 * host merges after an all-gather. Phase 1, like ifx_batch_run, starts the run from the state of one GPU: nothing the exchange calls or
 * phase 5 set for the previous batch carries over, so a handle run as a shard and then by ifx_batch_run answers as one GPU.
 * buf / key / score / n / keep / gmax are DEVICE pointers. */
int  ifx_batch_run_phase(ifx_batch* b, int phase, ifx_stats* st);
int  ifx_batch_fuzzy_df(ifx_batch* b, int32_t* buf /* [nq * 16] */, int set);
int  ifx_batch_select_counts(ifx_batch* b, int32_t* buf /* [nq * 40] */, int set);
int  ifx_batch_stage1_lists(ifx_batch* b, int64_t* key, float* score, int32_t* n);
int  ifx_batch_stage1_restrict(ifx_batch* b, const uint8_t* keep /* [nq * depth]: 0 drop, 1 keep, 2 / 3 keep = global rank 0 / 1 */, const float* gmax /* [nq] */, const int32_t* n_global /* [nq] entries of the global list */);
int  ifx_batch_wm_counts(ifx_batch* b, int32_t* buf /* [nq * 4] */);                 /* after phase 4 (WordMatcher lookups) */
int  ifx_batch_wm_apply(ifx_batch* b, const int32_t* allowed /* [nq] */, const int32_t* any /* [nq] */);   /* then phase 5: coverage, fusion, finalize */
int  ifx_batch_shard_info(ifx_batch* b, int32_t* info /* [nq * 8], HOST */, int64_t* dkey /* [nq * 2], HOST */);
/* Short queries (no word of >= 3 characters) on shards, between phase 3 and ifx_batch_stage1_lists. ifx_batch_short_groups gives the number of
 * groups (0: the batch holds no short query, nothing to do) and the group size G, the same on every shard; kind (HOST [nq], may be NULL):
 * 0 not short, 1 one character, 2 several, | 4 when the <= 3-character rule of SearchPipeline applies. Then for every group g:
 *   ifx_batch_short_step(b, 0, g, buf) -> all-reduce(sum) of buf -> step 1 -> all-reduce(max) of buf -> step 2
 * buf: DEVICE int32[G] -- matched documents of each query of the group (ProcessFuzzyFallback below 100), then its largest integer score
 * (BuildFinalScores normalises by it). Step 2 leaves the shard's exact Stage-1 list of every query of the group. */
int  ifx_batch_short_groups(ifx_batch* b, int32_t* kind, int32_t* n_groups, int32_t* group_size);
int  ifx_batch_short_step(ifx_batch* b, int step, int group, int32_t* buf);
/* Then, after ifx_batch_wm_apply and before phase 5 (only when n_groups > 0): ifx_batch_short_hits(b, buf, 0) evaluates the coverage stage
 * (phase 5 does not repeat it) and leaves each short query's largest coverage word hits on this shard in buf (DEVICE int32[nq]);
 * all-reduce(max); ifx_batch_short_hits(b, buf, 1). A short query whose coverage found no word hit on any shard (and no WordMatcher
 * document) falls back to its Stage-1 list on every shard, as SearchPipeline does. Steps out of order give IFX_ERR_INVALID. */
int  ifx_batch_short_hits(ifx_batch* b, int32_t* buf, int set);
/* Filters and facets on shards. The hosts truncate the merged coverage records (CalculateTruncationIndex) and cut a list answered by the
 * <= 3-character rule at max_results (shard_info[6] == 0 for both), and the filter runs after that, as in SearchEngine.Search. So a shard
 * reports those records UNFILTERED, and ifx_batch_shard_records (after phase 5; out: DEVICE int32 [nq][cap][stride], stride = 1 + F, F =
 * facetable columns, cap = the batch's max_results; another stride is IFX_ERR_INVALID) gives per record its filter outcome (1 pass / 0 fail,
 * evaluated by the shard that owns the document) and the value id of each facetable column in column order (-1: null or empty).
 * A query answered with its WHOLE Stage-1 list (shard_info[6] == -1: EnableCoverage off, a 3-character query over a prefix of > 500
 * documents, a short query) keeps its filter on the shard: TotalCandidates is the sum of the shards' totals, and its facet rows (over the
 * shard's filtered part of the list, no cut at 100 values per column, at most facet_cap rows: more sets IFX_Q_OVERFLOW) come with
 * ifx_batch_download for the hosts to sum. The blank query with EnableFacets (shard_info[6] == -2): the shards' records in shard order, then
 * Take(max). Value ids are the same on every shard once the columns were globalized (ifx_builder_globalize_columns).
 * ifx_batch_set_facet_cap: facet rows per query of the batch's outputs (an uploaded batch starts with 0: no facet rows).
 * ifx_batch_facet_table: the facet table of every query with enable_facets from rows = DEVICE int32 [nq][m][3] (column, value id, count;
 * count 0 = no row), e.g. the records the hosts kept, one row per facetable column: counts summed per value id, ordered by count descending,
 * then by value as FacetBuilder orders keys, the first 100 per column, at most facet_cap rows (more sets IFX_Q_OVERFLOW in status). Outputs:
 * DEVICE [nq][facet_cap] column / value / count as in ifx_batch_result, n_facets [nq]; status [nq] is read and updated. */
int  ifx_batch_shard_records(ifx_batch* b, int32_t* out, int32_t stride);
int  ifx_batch_set_facet_cap(ifx_batch* b, int32_t facet_cap);
int  ifx_batch_facet_table(ifx_batch* b, const int32_t* rows, int32_t m, int32_t* column, int32_t* value, int32_t* count, int32_t* n_facets, int32_t* status);

/* Stage-1 only (Bm25Scorer.Search + ConsolidateSegments, src/Infidex/Indexing/Bm25Scorer.cs:56-193): row-major
 * [nq][depth] keys / scores, n[nq]. Used for intermediate parity checks and kernel-level measurement. */
int  ifx_stage1_batch(ifx_index* idx, const ifx_query* q, int nq, int depth, int64_t* doc_key, float* score, int32_t* n,
                      int32_t* status, ifx_stats* st);

/* benchmark hygiene: overwrite a 256 MiB scratch buffer so the next run starts with a cold L2 */
int  ifx_flush_l2(ifx_index* idx);

const char* ifx_last_error(void);     /* thread-local description of the last failure */
int  ifx_device_count(void);

#ifdef __cplusplus
}
#endif
#endif
