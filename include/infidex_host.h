/* infidex_host.h -- host-side index builder of infidex_b200 (libinfidex_host.so, no CUDA dependency).
 *
 * Stands in for the C# host's indexing half (SearchEngine.IndexDocuments, src/Infidex/SearchEngine.cs:96-192):
 * documents in, the flattened immutable index (ifx_index_image, see infidex_gpu.h) out. With the real C# host the
 * image is marshalled from its own in-memory structures instead (INTEGRATION.md); the search path is identical.
 */
#ifndef INFIDEX_HOST_H
#define INFIDEX_HOST_H
#include "infidex_gpu.h"
#ifdef __cplusplus
extern "C" {
#endif

enum { IFX_FIELD_INDEXABLE = 1, IFX_FIELD_FILTERABLE = 2, IFX_FIELD_FACETABLE = 4, IFX_FIELD_SORTABLE = 8 };   /* Field.Indexable / Filterable / Facetable / Sortable */

typedef struct ifx_builder ifx_builder;

/* schema = DocumentFields of the documents (Api/DocumentFields.cs); weight: 0 High, 1 Med, 2 Low (Api/Weight.cs) */
ifx_builder* ifx_builder_create(int nfields, const uint16_t* names, const int32_t* name_off, const int32_t* weight, const int32_t* flags);
void ifx_builder_destroy(ifx_builder* b);
/* columnar documents; kinds[f]: 0 null, 1 string (cols[f] = UTF-16 blob, offs[f] = int64[n+1]), 2 int64[n], 3 double[n] */
int ifx_builder_add_docs(ifx_builder* b, int n, const int64_t* keys, const int32_t* kinds, const void* const* cols, const long long* const* offs);
int ifx_builder_finish(ifx_builder* b, int threads);
const ifx_index_image* ifx_builder_image(ifx_builder* b);   /* valid until ifx_builder_destroy */

/* doc-id-range shards: every shard's host builds its own document range, then the shards exchange their local statistics (export ->
 * all-gather between the hosts -> globalize) so that each image carries the term ordinals, df, N, avgdl, word idf, prefix cardinalities
 * and affix dictionary of the whole corpus (infidex_gpu.h, ifx_index_image). */
const uint8_t* ifx_builder_export_stats(ifx_builder* b, size_t* len);      /* valid until the next export on this thread */
int ifx_builder_globalize(ifx_builder* b, int n_shards, int shard, const uint8_t* const* blobs);
const float* ifx_builder_doc_lengths(ifx_builder* b, int* n);              /* after globalize: second exchange ... */
int ifx_builder_set_global_lengths(ifx_builder* b, int n_shards, const float* const* lens, const int* counts);   /* ... avgdl over the whole corpus */

/* SearchEngine.Search step 1 (src/Infidex/SearchEngine.cs:264-274): Trim + TextNormalizer.Normalize + ToLowerInvariant. Returns the output length. */
int ifx_host_prepare_query(const uint16_t* in, int n, uint16_t* out, int cap);

/* filter / facet columns of the finished image (index = ifx_batch_result.facet_column) */
int ifx_builder_num_columns(ifx_builder* b);
int ifx_builder_column_name(ifx_builder* b, int c, uint16_t* buf, int cap);
int ifx_builder_column_dict_size(ifx_builder* b, int c);
int ifx_builder_column_value(ifx_builder* b, int c, int id, uint16_t* buf, int cap);
/* ResultProcessor.CompareValues ranks of column c's dictionary entries (rank[ifx_builder_column_dict_size]) for ifx_column_set_order:
 * int64 / double values compared as numbers of their own type, strings ordinally; IFX_ERR_UNSUPPORTED when the field mixes runtime types */
int ifx_builder_column_order(ifx_builder* b, int c, int32_t* rank);

#ifdef __cplusplus
}
#endif
#endif
