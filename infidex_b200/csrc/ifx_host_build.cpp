// infidex_b200 -- host-side index builder (libinfidex_host.so): documents -> ifx_index_image.
//
// This is the product's stand-in for the part of the C# host that runs *before* the search path
// (SearchEngine.IndexDocuments, src/Infidex/SearchEngine.cs:96-192): it produces exactly the state the reference
// holds after IndexDocumentsInternal, flattened into the image that ifx_index_create uploads. Bulk / sort-based and
// multi-threaded (doc-range partitions, flat posting records, counting-sort into CSR), not a per-term dictionary of lists.
//
// Index-time semantics reproduced (SURVEY.md App. A1):
//   DocumentFields.GetSearchableTexts ('§' join, High->Low)      Api/DocumentFields.cs:124-170
//   Tokenizer.EnumerateTokensForIndexing (padded 3-grams + words) Tokenization/Tokenizer.cs:89-139
//   Term.FirstCycleAdd / TermCollection.CountTermUsage            Core/Term.cs:71-121, Core/TermCollection.cs:75-138
//   VectorModel.BuildInvertedLists / BuildWordIdfCache / metadata Indexing/VectorModel.cs:130-220,250-313,864-908
//   PositionalPrefixIndex / WordMatcher.Load                      Indexing/ShortQuery/PositionalPrefixIndex.cs:55-119, WordMatcher/WordMatcher.cs:82-196
#include "../../include/infidex_gpu.h"
#include "../../include/infidex_host.h"
#include <vector>
#include <string>
#include <string_view>
#include <thread>
#include <algorithm>
#include <numeric>
#include <cmath>
#include <cstring>
#include <charconv>
#include <memory>
#include <chrono>
#include <cstdio>
#include <cstdlib>

namespace {
#include "chartables.inc"

using sv = std::u16string_view; using str = std::u16string;

struct Tables {
    std::vector<uint16_t> lower, norm; std::vector<uint8_t> flags;
    Tables() : lower(65536), norm(65536), flags(65536, 0) {
        for (int i = 0; i < 65536; i++) lower[i] = norm[i] = (uint16_t)i;
        for (int i = 0; i < IFX_LOWER_PAIRS_N; i++) lower[IFX_LOWER_PAIRS[i][0]] = IFX_LOWER_PAIRS[i][1];
        for (int i = 0; i < IFX_NORM_PAIRS_N; i++) norm[IFX_NORM_PAIRS[i][0]] = IFX_NORM_PAIRS[i][1];
        const uint16_t d[] = {' ', '-', '/', '.', ',', ':', ';', '\'', '`', 0x2013, 0x2014, '*', '&', '\\', '_', '(', ')', '{', '}', '[', ']', '\t'};
        for (uint16_t c : d) flags[c] |= 4;
    }
};
const Tables& TB() { static Tables t; return t; }
inline bool is_delim(char16_t c) { return TB().flags[c] & 4; }
void normalize_into(sv in, str& out) {   // TextNormalizer.Normalize (default map + whitespace collapse)
    out.clear(); bool prev = false;
    for (char16_t c : in) { char16_t m = (c == u'\t' || c == u'\n' || c == u'\r') ? u' ' : (char16_t)TB().norm[c]; bool sp = m == u' '; if (sp && prev) continue; out.push_back(m); prev = sp; }
}
void lower_inplace(str& s) { for (auto& c : s) c = (char16_t)TB().lower[c]; }

inline uint64_t hash64(const char16_t* s, size_t n) {
    uint64_t h = 0xcbf29ce484222325ULL ^ (uint64_t)n;
    for (size_t i = 0; i < n; i++) { h ^= s[i]; h *= 0x100000001b3ULL; }
    h ^= h >> 29; h *= 0xbf58476d1ce4e5b9ULL; h ^= h >> 32; return h | 1ULL;
}

// .NET ArraySortHelper<T>.IntrospectiveSort (List<T>.Sort(Comparison)): unstable, and the tie order is observable in the champion lists
// (ShortQueryResolver.BuildChampionLists keeps the first 64 after the sort) -- the same rules as the device's IdfSorter.
template <class T, class Cmp> struct DotnetIntroSort {
    Cmp cmp;
    void swap_if_greater(T* k, int i, int j) { if (cmp(k[i], k[j]) > 0) std::swap(k[i], k[j]); }
    void insertion(T* k, int n) { for (int i = 0; i < n - 1; i++) { T t = k[i + 1]; int j = i; while (j >= 0 && cmp(t, k[j]) < 0) { k[j + 1] = k[j]; j--; } k[j + 1] = t; } }
    void down_heap(T* k, int i, int n) { T d = k[i - 1]; while (i <= n / 2) { int ch = 2 * i; if (ch < n && cmp(k[ch - 1], k[ch]) < 0) ch++; if (!(cmp(d, k[ch - 1]) < 0)) break; k[i - 1] = k[ch - 1]; i = ch; } k[i - 1] = d; }
    void heap_sort(T* k, int n) { for (int i = n >> 1; i >= 1; i--) down_heap(k, i, n); for (int i = n; i > 1; i--) { std::swap(k[0], k[i - 1]); down_heap(k, 1, i - 1); } }
    int partition(T* k, int n) {
        int hi = n - 1, mid = hi >> 1;
        swap_if_greater(k, 0, mid); swap_if_greater(k, 0, hi); swap_if_greater(k, mid, hi);
        T pivot = k[mid]; std::swap(k[mid], k[hi - 1]);
        int left = 0, right = hi - 1;
        while (left < right) { while (cmp(k[++left], pivot) < 0) {} while (cmp(pivot, k[--right]) < 0) {} if (left >= right) break; std::swap(k[left], k[right]); }
        if (left != hi - 1) std::swap(k[left], k[hi - 1]);
        return left;
    }
    void intro(T* k, int n, int depth) {
        while (n > 1) {
            if (n <= 16) { if (n == 2) swap_if_greater(k, 0, 1); else if (n == 3) { swap_if_greater(k, 0, 1); swap_if_greater(k, 0, 2); swap_if_greater(k, 1, 2); } else insertion(k, n); return; }
            if (depth == 0) { heap_sort(k, n); return; }
            depth--; int p = partition(k, n); intro(k + p + 1, n - (p + 1), depth); n = p;
        }
    }
    void sort(T* k, int n) { if (n < 2) return; int lg = 0; for (unsigned v = (unsigned)n; v >>= 1;) lg++; intro(k, n, 2 * (lg + 1)); }
};
inline bool is_ws(char16_t c) { static std::vector<uint8_t> ws = [] { std::vector<uint8_t> w(65536, 0); for (int i = 0; i < IFX_SPACE_LIST_N; i++) w[IFX_SPACE_LIST[i]] = 1; return w; }(); return ws[c] != 0; }

// string interner: open addressing over a char arena; ids in first-insertion order
struct Interner {
    std::vector<char16_t> arena; std::vector<uint32_t> off{0}; std::vector<uint64_t> hk; std::vector<int32_t> hv; size_t mask = 0;
    Interner() { rehash(1024); }
    int size() const { return (int)off.size() - 1; }
    sv get(int id) const { return sv(arena.data() + off[id], off[id + 1] - off[id]); }
    void rehash(size_t cap) { std::vector<uint64_t> k(cap, 0); std::vector<int32_t> v(cap, -1); for (size_t i = 0; i < hk.size(); i++) if (hk[i]) { size_t s = (hk[i] >> 7) & (cap - 1); while (k[s]) s = (s + 1) & (cap - 1); k[s] = hk[i]; v[s] = hv[i]; } hk.swap(k); hv.swap(v); mask = cap - 1; }
    int find(sv s) const { uint64_t h = hash64(s.data(), s.size()); size_t slot = (h >> 7) & mask; for (;;) { if (!hk[slot]) return -1; if (hk[slot] == h && get(hv[slot]) == s) return hv[slot]; slot = (slot + 1) & mask; } }
    int intern(sv s, bool* is_new = nullptr) {
        uint64_t h = hash64(s.data(), s.size()); size_t slot = (h >> 7) & mask;
        for (;;) { if (!hk[slot]) break; if (hk[slot] == h && get(hv[slot]) == s) { if (is_new) *is_new = false; return hv[slot]; } slot = (slot + 1) & mask; }
        int id = size(); arena.insert(arena.end(), s.begin(), s.end()); off.push_back((uint32_t)arena.size());
        hk[slot] = h; hv[slot] = id; if (is_new) *is_new = true;
        if ((size_t)size() * 2 > mask) rehash((mask + 1) * 2);
        return id;
    }
};

// key -> ascending doc list with optional byte weight, as flat records (thread-local), merged into CSR later
struct KeyedRecords {
    Interner keys; std::vector<int32_t> rec_key, rec_doc; std::vector<uint8_t> rec_w; std::vector<int32_t> last_rec; std::vector<uint8_t> extra;   // extra: saturated repeats (df not decremented)
    bool weighted;
    explicit KeyedRecords(bool w) : weighted(w) {}
    int key(sv s) { bool nw; int k = keys.intern(s, &nw); if (nw) { last_rec.push_back(-1); rec_rep_last.push_back(0); } return k; }
    void add_doc(int k, int doc) { int lr = last_rec[k]; if (lr >= 0 && rec_doc[lr] == doc) return; last_rec[k] = (int)rec_doc.size(); rec_key.push_back(k); rec_doc.push_back(doc); }
    int sat_count = 0; std::vector<int32_t> sat_keys;
    void add_weighted(int k, int doc, float fw) {   // Term.FirstCycleAdd (Core/Term.cs:71-121) without the stop rule (applied globally)
        int lr = last_rec[k];
        if (lr >= 0 && rec_doc[lr] == doc) {
            float nw = (float)rec_w[lr] + fw;
            if (nw <= 255.f) rec_w[lr] = (uint8_t)std::nearbyint((double)nw); else sat_keys.push_back(k);
            rec_rep_last[k] = 1;
            return;
        }
        last_rec[k] = (int)rec_doc.size(); rec_key.push_back(k); rec_doc.push_back(doc);
        rec_w.push_back((uint8_t)std::min(std::nearbyint((double)fw), 255.0));
        rec_rep_last[k] = 0;
    }
    std::vector<uint8_t> rec_rep_last;   // did the key's latest posting see a repeat occurrence (stop-term edge rule)
};

// big flat array without the zero fill of std::vector::resize (the scatter that follows touches every element, in parallel)
template <class T> struct RawVec {
    T* p = nullptr; size_t n = 0;
    RawVec() = default; RawVec(const RawVec&) = delete; RawVec& operator=(const RawVec&) = delete;
    ~RawVec() { free(p); }
    void resize(size_t m) { free(p); p = (T*)malloc(std::max<size_t>(m, 1) * sizeof(T)); if (!p) throw std::bad_alloc(); n = m; }
    T* data() { return p; } const T* data() const { return p; } size_t size() const { return n; }
    T& operator[](size_t i) { return p[i]; } const T& operator[](size_t i) const { return p[i]; }
};

template <class F> void par_for(int64_t n, int threads, F f) {       // f(begin, end, thread index)
    threads = (int)std::max<int64_t>(1, std::min<int64_t>(threads, n));
    if (threads == 1) { f((int64_t)0, n, 0); return; }
    std::vector<std::thread> ts;
    for (int t = 0; t < threads; t++) ts.emplace_back([=] { f(n * t / threads, n * (t + 1) / threads, t); });
    for (auto& th : ts) th.join();
}

struct Csr { std::vector<char16_t> chars; std::vector<uint32_t> off; std::vector<int64_t> row; RawVec<int32_t> docs; RawVec<uint8_t> w; std::vector<int32_t> extra; std::vector<uint8_t> rep_last; int n = 0; };

// merge thread-local KeyedRecords (threads own ascending doc ranges) -> global keys in first-occurrence order + CSR
void merge_records(std::vector<std::unique_ptr<KeyedRecords>>& parts, Csr& out, bool weighted, const char* name = "") {
    const bool timing = getenv("IFX_CREATE_TIMING") != nullptr; auto t_last = std::chrono::steady_clock::now();
    auto stage = [&](const char* what) { if (!timing) return; auto now = std::chrono::steady_clock::now(); fprintf(stderr, "[merge %-6s] %-24s %.2f s\n", name, what, std::chrono::duration<double>(now - t_last).count()); t_last = now; };
    Interner g; std::vector<std::vector<int32_t>> l2g(parts.size());
    for (size_t t = 0; t < parts.size(); t++) { auto& p = *parts[t]; l2g[t].resize(p.keys.size()); for (int k = 0; k < p.keys.size(); k++) l2g[t][k] = g.intern(p.keys.get(k)); }
    stage("global keys");
    int G = g.size(); out.n = G; out.chars.assign(g.arena.begin(), g.arena.end()); out.off = g.off; if (out.chars.empty()) out.chars.push_back(0);
    // per-part per-key counts -> row pointers -> every part scatters its records in parallel (parts own ascending doc ranges,
    // so placing part t's records after those of parts < t keeps every row ascending)
    const size_t NP = parts.size();
    std::vector<std::vector<int32_t>> cnt(NP);
    { std::vector<std::thread> ts; for (size_t t = 0; t < NP; t++) ts.emplace_back([&, t] { cnt[t].assign(G, 0); for (int32_t k : parts[t]->rec_key) cnt[t][l2g[t][k]]++; }); for (auto& th : ts) th.join(); }
    stage("count");
    out.row.assign((size_t)G + 1, 0);
    for (int g2 = 0; g2 < G; g2++) { int64_t c = 0; for (size_t t = 0; t < NP; t++) c += cnt[t][g2]; out.row[g2 + 1] = out.row[g2] + c; }
    out.docs.resize((size_t)out.row[G]); if (weighted) out.w.resize(out.docs.size());
    std::vector<std::vector<int64_t>> start(NP);
    for (size_t t = 0; t < NP; t++) start[t].resize(G);
    for (int g2 = 0; g2 < G; g2++) { int64_t o = out.row[g2]; for (size_t t = 0; t < NP; t++) { start[t][g2] = o; o += cnt[t][g2]; } }
    stage("rows + starts");
    { std::vector<std::thread> ts; for (size_t t = 0; t < NP; t++) ts.emplace_back([&, t] { auto& p = *parts[t]; auto& pos = start[t];
          for (size_t r = 0; r < p.rec_key.size(); r++) { int64_t o = pos[l2g[t][p.rec_key[r]]]++; out.docs[o] = p.rec_doc[r]; if (weighted) out.w[o] = p.rec_w[r]; } });
      for (auto& th : ts) th.join(); }
    stage("scatter");
    if (weighted) {
        out.extra.assign(G, 0); out.rep_last.assign(G, 0);
        for (size_t t = 0; t < parts.size(); t++) { auto& p = *parts[t]; for (int32_t k : p.sat_keys) out.extra[l2g[t][k]]++;
            for (int k = 0; k < p.keys.size(); k++) if (p.last_rec[k] >= 0) out.rep_last[l2g[t][k]] = p.rec_rep_last[k]; }   // later threads overwrite: state of the globally last posting
    }
}

struct FieldSpec { str name; int weight; int flags; };

str value_to_string(int kind, const void* col, const long long* offs, int d) {
    char buf[64];
    if (kind == 1) { const char16_t* b = (const char16_t*)col; return str(b + offs[d], (size_t)(offs[d + 1] - offs[d])); }
    if (kind == 2) { auto r = std::to_chars(buf, buf + 64, ((const long long*)col)[d]); return str(buf, r.ptr); }
    if (kind == 3) { auto r = std::to_chars(buf, buf + 64, ((const double*)col)[d]); return str(buf, r.ptr); }
    return str();
}

}  // namespace

struct ifx_builder {
    std::vector<FieldSpec> schema; float field_weights[3] = {1.5f, 1.25f, 1.0f}; int stop_term_limit = 1250000;
    // documents (columnar, appended per add_docs call)
    std::vector<int64_t> keys; std::vector<std::vector<str>> values;   // values[f][d] = ToString(), kind 0 -> null flag
    std::vector<std::vector<uint8_t>> is_null;
    std::vector<int> kind;                                             // per field: runtime type of its values (add_docs kinds), 0 none yet, -1 mixed
    // image storage
    ifx_index_image img{}; bool finished = false;
    std::vector<uint8_t> deleted; std::vector<float> doc_len; std::vector<char16_t> text; std::vector<int64_t> text_off;
    std::vector<char16_t> ft_chars; std::vector<uint32_t> ft_off; std::vector<uint16_t> tok_count;
    Csr terms, prefix, wm_exact, wm_ld1; std::vector<int32_t> df;
    std::vector<char16_t> word_chars; std::vector<uint32_t> word_off; std::vector<float> word_idf; std::vector<int32_t> word_df;
    std::vector<char16_t> affix_chars; std::vector<uint32_t> affix_off; std::vector<int32_t> affix_last;
    std::vector<uint16_t> champ_chars; std::vector<int32_t> champ_off, champ_doc; std::vector<float> champ_score;
    std::vector<int32_t> raw_doc; std::vector<char16_t> raw_chars; std::vector<int64_t> raw_off;
    std::vector<ifx_column> cols; std::vector<std::vector<int32_t>> col_ids; std::vector<std::vector<char16_t>> col_chars; std::vector<std::vector<uint32_t>> col_off; std::vector<str> col_names;
    std::vector<int> col_kind;                                         // kind of the column's field
};

static float compute_idf_host(int total, int df) {   // Bm25Scorer.ComputeIdf
    if (df <= 0 || total <= 0) return 0.f;
    float d = (float)df, N = (float)total; float ratio = (N - d + 0.5f) / (d + 0.5f);
    return ratio <= 0.f ? 0.f : std::log(ratio + 1.f);
}

extern "C" {

ifx_builder* ifx_builder_create(int nfields, const uint16_t* names, const int32_t* name_off, const int32_t* weight, const int32_t* flags) {
    ifx_builder* b = new ifx_builder();
    for (int i = 0; i < nfields; i++) b->schema.push_back({str((const char16_t*)names + name_off[i], name_off[i + 1] - name_off[i]), weight[i], flags[i]});
    b->values.resize(nfields); b->is_null.resize(nfields); b->kind.assign(nfields, 0);
    return b;
}
void ifx_builder_destroy(ifx_builder* b);

int ifx_builder_add_docs(ifx_builder* b, int n, const int64_t* keys, const int32_t* kinds, const void* const* cols, const long long* const* offs) {
    if (b->finished) return IFX_ERR_INVALID;
    int F = (int)b->schema.size();
    b->keys.insert(b->keys.end(), keys, keys + n);
    for (int f = 0; f < F; f++) if (kinds[f] != 0) b->kind[f] = (b->kind[f] == 0 || b->kind[f] == kinds[f]) ? kinds[f] : -1;
    const int hw = (int)std::max(1u, std::min(std::thread::hardware_concurrency(), 64u));
    for (int f = 0; f < F; f++) { auto& v = b->values[f]; auto& nl = b->is_null[f]; const size_t base = v.size(); v.resize(base + n); nl.resize(base + n, kinds[f] == 0 ? 1 : 0);
        if (kinds[f] != 0) par_for(n, n >= 100000 ? hw : 1, [&, f](int64_t a, int64_t e, int) { for (int64_t d = a; d < e; d++) v[base + d] = value_to_string(kinds[f], cols[f], offs ? offs[f] : nullptr, (int)d); }); }
    return IFX_OK;
}

int ifx_builder_finish(ifx_builder* b, int threads) {
    if (b->finished) return IFX_OK;
    const int N = (int)b->keys.size(); const int F = (int)b->schema.size();
    if (threads < 1) threads = 1; if (threads > N) threads = std::max(1, N);
    const bool timing = getenv("IFX_CREATE_TIMING") != nullptr; auto t_last = std::chrono::steady_clock::now();
    auto stage = [&](const char* what) { if (!timing) return; auto now = std::chrono::steady_clock::now(); fprintf(stderr, "[ifx_builder_finish] %-28s %.2f s\n", what, std::chrono::duration<double>(now - t_last).count()); t_last = now; };
    // indexable fields ordered by Weight (stable): GetSearchAbleFieldList
    std::vector<int> order; for (int w = 0; w < 3; w++) for (int f = 0; f < F; f++) if ((b->schema[f].flags & IFX_FIELD_INDEXABLE) && b->schema[f].weight == w) order.push_back(f);
    struct Part {
        std::unique_ptr<KeyedRecords> terms, prefix, exact, ld1; Interner words; std::vector<int32_t> word_df; Interner affix; std::vector<int32_t> affix_last;
        std::vector<char16_t> text; std::vector<int64_t> text_len; std::vector<char16_t> ft; std::vector<uint32_t> ft_len; std::vector<uint16_t> tokc;
        struct Champ { char16_t ch; uint16_t score; int32_t doc; }; std::vector<Champ> champs;      // ShortQueryResolver: one record per (first character of a word, document)
        std::vector<int32_t> raw_doc; std::vector<char16_t> raw_chars; std::vector<int64_t> raw_len;   // documents whose raw IndexedText differs from its normalised form
    };
    std::vector<Part> parts(threads);
    auto work = [&](int t) {
        Part& P = parts[t]; P.terms.reset(new KeyedRecords(true)); P.prefix.reset(new KeyedRecords(false)); P.exact.reset(new KeyedRecords(false)); P.ld1.reset(new KeyedRecords(false));
        int d0 = (int)((int64_t)N * t / threads), d1 = (int)((int64_t)N * (t + 1) / threads);
        str raw, nrm, idx, padded, wm, tmp; std::vector<std::pair<int, int>> bounds; std::vector<int> seen_words; std::vector<sv> tok_scratch;
        for (int d = d0; d < d1; d++) {
            raw.clear(); bounds.clear();
            for (size_t k = 0; k < order.size(); k++) { bounds.emplace_back((int)(uint16_t)raw.size(), b->schema[order[k]].weight); raw += b->values[order[k]][d]; if (k + 1 < order.size()) raw.push_back(u'§'); }
            normalize_into(raw, nrm);                       // normalize(IndexedText): coverage doc text
            P.text.insert(P.text.end(), nrm.begin(), nrm.end()); P.text_len.push_back((int64_t)nrm.size());
            idx = nrm; lower_inplace(idx);                  // VectorModel.IndexDocument: Normalize then ToLowerInvariant
            // 3-grams of PAD PAD + text, then words (len >= 3)
            padded.assign(2, (char16_t)0xFFFF); padded += idx;
            auto fw_at = [&](int pos) { if (bounds.empty()) return 1.0f; int wi = 0; for (auto& bd : bounds) { if (bd.first <= pos) wi = bd.second; else break; } return wi < 3 ? b->field_weights[wi] : 1.0f; };
            if (padded.size() >= 3) for (size_t i = 0; i + 3 <= padded.size(); i++) { sv g(padded.data() + i, 3); if (g[0] == 0xFFFF && g[1] == 0xFFFF && g[2] == 0xFFFF) continue; P.terms->add_weighted(P.terms->key(g), d, fw_at((int)i)); }
            for (size_t i = 0; i < idx.size();) { while (i < idx.size() && is_delim(idx[i])) i++; if (i >= idx.size()) break; size_t s = i; while (i < idx.size() && !is_delim(idx[i])) i++;
                if (i - s >= 3) P.terms->add_weighted(P.terms->key(sv(idx.data() + s, i - s)), d, fw_at(2 + (int)s)); }
            // prefix docsets (PositionalPrefixIndex over the index text)
            for (size_t i = 0; i < idx.size();) { while (i < idx.size() && is_delim(idx[i])) i++; if (i >= idx.size()) break; size_t s = i; while (i < idx.size() && !is_delim(idx[i])) i++;
                size_t ml = std::min<size_t>(3, i - s); for (size_t l = 1; l <= ml; l++) P.prefix->add_doc(P.prefix->key(sv(idx.data() + s, l)), d); }
            // short-query structures (Indexing/ShortQuery/ShortQueryResolver.cs:83-160,268-311): per first character of a word of the index text,
            // (first token index, number of such word starts) -> precedence / base score against the document's lower-cased RAW title
            {   tmp = raw; lower_inplace(tmp);                                // ToLowerInvariant(IndexedText), not normalised
                if (nrm != raw) { P.raw_doc.push_back(d); P.raw_chars.insert(P.raw_chars.end(), raw.begin(), raw.end()); P.raw_len.push_back((int64_t)raw.size()); }
                // title tokens (split on the delimiters, empty entries removed) and trim
                int n_tok = 0; sv first_tok; std::vector<sv>& toks = tok_scratch; toks.clear();
                for (size_t i = 0; i < tmp.size();) { while (i < tmp.size() && is_delim(tmp[i])) i++; if (i >= tmp.size()) break; size_t s0 = i; while (i < tmp.size() && !is_delim(tmp[i])) i++; toks.emplace_back(tmp.data() + s0, i - s0); }
                n_tok = (int)toks.size(); if (n_tok) first_tok = toks[0];
                size_t tb = 0, te = tmp.size(); while (tb < te && is_ws(tmp[tb])) tb++; while (te > tb && is_ws(tmp[te - 1])) te--;
                struct Acc { char16_t ch; int first_pos, n; }; Acc acc[64]; int na = 0; int ti = 0;
                for (size_t i = 0; i < idx.size();) { while (i < idx.size() && is_delim(idx[i])) i++; if (i >= idx.size()) break; size_t s0 = i; while (i < idx.size() && !is_delim(idx[i])) i++;
                    const char16_t ch = idx[s0]; int a = 0; for (; a < na; a++) if (acc[a].ch == ch) break;
                    if (a == na) { if (na < 64) { acc[na].ch = ch; acc[na].first_pos = ti; acc[na].n = 1; na++; } } else acc[a].n++;
                    ti++; }
                for (int a = 0; a < na; a++) {
                    const char16_t ch = acc[a].ch; int prec = 128; if (acc[a].first_pos == 0) prec |= 64;
                    bool any = false, first = false; for (int i = 0; i < n_tok; i++) if (toks[i].size() == 1 && toks[i][0] == ch) { any = true; if (i == 0) first = true; break; }
                    if (any) prec |= 32; if (first) prec |= 16; if (te - tb == 1 && tmp[tb] == ch) prec |= 8; if (n_tok <= 3) prec |= 32;
                    const int pos_c = 255 - std::min(acc[a].first_pos * 16, 240), dens = std::min(acc[a].n * 8, 32); const int base = std::max(0, std::min(255, pos_c + dens));
                    P.champs.push_back({ch, (uint16_t)((prec << 8) | base), d});
                }
            }
            // WordMatcher.Load / word-idf / metadata work on normalize(lower(IndexedText))
            tmp = raw; lower_inplace(tmp); normalize_into(tmp, wm);
            int ntok = 0; bool first = true; seen_words.clear();
            for (size_t i = 0; i < wm.size();) { while (i < wm.size() && is_delim(wm[i])) i++; if (i >= wm.size()) break; size_t s = i; while (i < wm.size() && !is_delim(wm[i])) i++;
                sv w(wm.data() + s, i - s); int len = (int)w.size(); ntok++;
                if (first) { P.ft.insert(P.ft.end(), w.begin(), w.end()); P.ft_len.push_back((uint32_t)len); first = false; }
                if (len >= 2 && len <= 8) P.exact->add_doc(P.exact->key(w), d);
                if (len >= 3 && len <= 8) for (int k = 0; k < len; k++) { tmp.assign(w); tmp.erase(k, 1); P.ld1->add_doc(P.ld1->key(tmp), d); }
                if (len >= 3) { bool nw; int a = P.affix.intern(w, &nw); if (nw) P.affix_last.push_back(d); else P.affix_last[a] = d; }
                bool nw2; int wid = P.words.intern(w, &nw2); if (nw2) P.word_df.push_back(0);
                if (std::find(seen_words.begin(), seen_words.end(), wid) == seen_words.end()) { seen_words.push_back(wid); P.word_df[wid]++; }
            }
            if (first) P.ft_len.push_back(0);
            P.tokc.push_back((uint16_t)std::min(ntok, 65535));
        }
    };
    { std::vector<std::thread> ts; for (int t = 0; t < threads; t++) ts.emplace_back(work, t); for (auto& t : ts) t.join(); }
    stage("tokenise (parallel)");
    // ---- merge
    b->deleted.assign(N, 0);
    {   std::vector<size_t> tbase(threads + 1, 0), fbase(threads + 1, 0), dbase(threads + 1, 0);
        for (int t = 0; t < threads; t++) { tbase[t + 1] = tbase[t] + parts[t].text.size(); fbase[t + 1] = fbase[t] + parts[t].ft.size(); dbase[t + 1] = dbase[t] + parts[t].text_len.size(); }
        b->text.resize(std::max<size_t>(tbase[threads], 1)); b->ft_chars.resize(std::max<size_t>(fbase[threads], 1)); b->text_off.resize((size_t)N + 1); b->ft_off.resize((size_t)N + 1); b->tok_count.resize(N);
        par_for(threads, threads, [&](int64_t a, int64_t e, int) { for (int64_t t = a; t < e; t++) { Part& P = parts[t];
            if (!P.text.empty()) std::memcpy(b->text.data() + tbase[t], P.text.data(), P.text.size() * 2); if (!P.ft.empty()) std::memcpy(b->ft_chars.data() + fbase[t], P.ft.data(), P.ft.size() * 2);
            int64_t to = (int64_t)tbase[t]; uint32_t fo = (uint32_t)fbase[t];
            for (size_t i = 0; i < P.text_len.size(); i++) { to += P.text_len[i]; fo += P.ft_len[i]; b->text_off[dbase[t] + i + 1] = to; b->ft_off[dbase[t] + i + 1] = fo; b->tok_count[dbase[t] + i] = P.tokc[i]; }
            std::vector<char16_t>().swap(P.text); std::vector<char16_t>().swap(P.ft); } });
    }
    stage("text concat");
    auto small_dicts = [&] {
        {   // champion lists: per first character the documents in ascending id order, List.Sort by score descending (unstable, reproduced), first 64
            std::vector<std::vector<std::pair<uint16_t, int32_t>>> by_ch(65536);
            for (auto& P : parts) for (auto& cr : P.champs) by_ch[cr.ch].emplace_back(cr.score, cr.doc);
            b->champ_off.assign(1, 0);
            for (int ch = 0; ch < 65536; ch++) { auto& v = by_ch[ch]; if (v.empty()) continue;
                auto cmpf = [](const std::pair<uint16_t, int32_t>& x, const std::pair<uint16_t, int32_t>& y) { return y.first < x.first ? -1 : (y.first > x.first ? 1 : 0); };
                DotnetIntroSort<std::pair<uint16_t, int32_t>, decltype(cmpf)> srt{cmpf}; srt.sort(v.data(), (int)v.size());
                const size_t keep = std::min<size_t>(v.size(), 64);
                b->champ_chars.push_back((uint16_t)ch); for (size_t i = 0; i < keep; i++) { b->champ_doc.push_back(v[i].second); b->champ_score.push_back((float)v[i].first); } b->champ_off.push_back((int32_t)b->champ_doc.size()); }
            if (b->champ_chars.empty()) b->champ_chars.push_back(0); if (b->champ_doc.empty()) { b->champ_doc.push_back(0); b->champ_score.push_back(0.f); }
            b->raw_off.assign(1, 0); for (auto& P : parts) { b->raw_doc.insert(b->raw_doc.end(), P.raw_doc.begin(), P.raw_doc.end()); b->raw_chars.insert(b->raw_chars.end(), P.raw_chars.begin(), P.raw_chars.end()); for (auto l : P.raw_len) b->raw_off.push_back(b->raw_off.back() + l); }
            if (b->raw_doc.empty()) b->raw_doc.push_back(-1); if (b->raw_chars.empty()) b->raw_chars.push_back(0);
        }
    // word idf
        { Interner g; std::vector<int32_t> gdf; for (auto& P : parts) for (int k = 0; k < P.words.size(); k++) { bool nw; int id = g.intern(P.words.get(k), &nw); if (nw) gdf.push_back(0); gdf[id] += P.word_df[k]; }
          b->word_chars.assign(g.arena.begin(), g.arena.end()); if (b->word_chars.empty()) b->word_chars.push_back(0); b->word_off = g.off; b->word_idf.resize(gdf.size()); b->word_df = gdf;
          for (size_t i = 0; i < gdf.size(); i++) b->word_idf[i] = (gdf[i] > 0 && gdf[i] <= N) ? compute_idf_host(N, gdf[i]) : 0.f; }
        // affix words: last doc wins (WordMatcher.IndexWordInFst quirk Q4)
        { Interner g; for (auto& P : parts) for (int k = 0; k < P.affix.size(); k++) { bool nw; int id = g.intern(P.affix.get(k), &nw); if (nw) b->affix_last.push_back(P.affix_last[k]); else b->affix_last[id] = P.affix_last[k]; }
          b->affix_chars.assign(g.arena.begin(), g.arena.end()); if (b->affix_chars.empty()) b->affix_chars.push_back(0); b->affix_off = g.off; if (b->affix_last.empty()) b->affix_last.push_back(0); }
        // filter / facet columns
        for (int f = 0; f < F; f++) {
            if (!(b->schema[f].flags & (IFX_FIELD_FILTERABLE | IFX_FIELD_FACETABLE | IFX_FIELD_SORTABLE))) continue;
            Interner g; std::vector<int32_t> ids(N);
            for (int d = 0; d < N; d++) ids[d] = b->is_null[f][d] ? -1 : g.intern(b->values[f][d]);
            b->col_ids.push_back(std::move(ids)); b->col_chars.emplace_back(g.arena.begin(), g.arena.end()); if (b->col_chars.back().empty()) b->col_chars.back().push_back(0); b->col_off.push_back(g.off); b->col_names.push_back(b->schema[f].name); b->col_kind.push_back(b->kind[f]);
        }
    };
    {   // the four keyed-record sets merge independently; the small dictionaries (word idf, affix words, columns) alongside
        std::vector<std::unique_ptr<KeyedRecords>> v0, v1, v2, v3;
        for (auto& P : parts) { v0.push_back(std::move(P.terms)); v1.push_back(std::move(P.prefix)); v2.push_back(std::move(P.exact)); v3.push_back(std::move(P.ld1)); }
        std::thread t0([&] { merge_records(v0, b->terms, true, "terms"); }), t1([&] { merge_records(v1, b->prefix, false, "prefix"); }), t2([&] { merge_records(v2, b->wm_exact, false, "exact"); }), t3([&] { merge_records(v3, b->wm_ld1, false, "ld1"); });
        std::thread t4(small_dicts);
        t0.join(); t1.join(); t2.join(); t3.join(); t4.join();
    }
    stage("merge records -> CSR");
    // stop terms + df (Term.IncrementTermUsageCounter / FirstCycleAdd): df = postings + saturated repeats; a term dies when df would exceed the limit
    const int T = b->terms.n; b->df.assign(T, 0);
    std::vector<int64_t> new_row((size_t)T + 1, 0); int64_t wpos = 0;
    for (int t = 0; t < T; t++) {
        int64_t r0 = b->terms.row[t], r1 = b->terms.row[t + 1]; int64_t cnt = r1 - r0; int64_t dfv = cnt + b->terms.extra[t];
        bool stop = dfv > b->stop_term_limit || (cnt == b->stop_term_limit && b->terms.rep_last[t]);
        new_row[t] = wpos;
        if (stop) { b->df[t] = -1; continue; }
        b->df[t] = (int32_t)dfv;
        if (wpos != r0) { std::memmove(b->terms.docs.data() + wpos, b->terms.docs.data() + r0, (size_t)cnt * 4); std::memmove(b->terms.w.data() + wpos, b->terms.w.data() + r0, (size_t)cnt); }
        wpos += cnt;
    }
    new_row[T] = wpos; b->terms.row.swap(new_row);
    stage("stop terms");
    // doc lengths (integer sums) and avgdl (sequential float sum, VectorModel.cs:212-216)
    std::vector<uint32_t> dl(N, 0);
    par_for(wpos, threads, [&](int64_t a, int64_t e, int) { for (int64_t i = a; i < e; i++) __atomic_fetch_add(&dl[b->terms.docs[i]], (uint32_t)b->terms.w[i], __ATOMIC_RELAXED); });   // integer sums: order-free
    b->doc_len.resize(N); float total = 0.f; for (int d = 0; d < N; d++) { b->doc_len[d] = (float)dl[d]; total += b->doc_len[d]; }
    float avgdl = N > 0 ? total / (float)N : 0.f;
    stage("doc lengths");
    b->cols.resize(b->col_ids.size());
    { int ci = 0; for (int f = 0; f < F; f++) { if (!(b->schema[f].flags & (IFX_FIELD_FILTERABLE | IFX_FIELD_FACETABLE | IFX_FIELD_SORTABLE))) continue; ifx_column& c = b->cols[ci];
        c.name = (const uint16_t*)b->col_names[ci].data(); c.name_len = (int)b->col_names[ci].size(); c.flags = ((b->schema[f].flags & IFX_FIELD_FILTERABLE) ? IFX_COL_FILTERABLE : 0) | ((b->schema[f].flags & IFX_FIELD_FACETABLE) ? IFX_COL_FACETABLE : 0)
            | (!(b->schema[f].flags & (IFX_FIELD_FILTERABLE | IFX_FIELD_FACETABLE)) ? IFX_COL_SORTABLE : 0);
        c.value_id = b->col_ids[ci].data(); c.dict = {(const uint16_t*)b->col_chars[ci].data(), b->col_off[ci].data(), (int)b->col_off[ci].size() - 1}; ci++; } }
    stage("columns");
    // ---- image
    ifx_index_image& I = b->img; auto S = [](std::vector<char16_t>& c, std::vector<uint32_t>& o) { return ifx_strings{(const uint16_t*)c.data(), o.data(), (int)o.size() - 1}; };
    I.n_docs = N; I.n_live = N; I.avgdl = avgdl; I.doc_key = b->keys.data(); I.deleted = b->deleted.data(); I.doc_len = b->doc_len.data();
    I.text_chars = (const uint16_t*)b->text.data(); I.text_off = b->text_off.data(); I.first_token = S(b->ft_chars, b->ft_off); I.token_count = b->tok_count.data();
    I.terms = S(b->terms.chars, b->terms.off); I.df = b->df.data(); I.row_ptr = b->terms.row.data(); I.post_doc = b->terms.docs.data(); I.post_tf = b->terms.w.data();
    I.words = S(b->word_chars, b->word_off); I.word_idf = b->word_idf.data();
    I.prefix = {S(b->prefix.chars, b->prefix.off), b->prefix.row.data(), b->prefix.docs.data()};
    I.wm_exact = {S(b->wm_exact.chars, b->wm_exact.off), b->wm_exact.row.data(), b->wm_exact.docs.data()};
    I.wm_ld1 = {S(b->wm_ld1.chars, b->wm_ld1.off), b->wm_ld1.row.data(), b->wm_ld1.docs.data()};
    I.affix_words = S(b->affix_chars, b->affix_off); I.affix_last_doc = b->affix_last.data();
    I.n_columns = (int)b->cols.size(); I.columns = b->cols.data();
    I.n_champ_chars = (int)b->champ_off.size() - 1; I.champ_chars = b->champ_chars.data(); I.champ_off = b->champ_off.data(); I.champ_doc = b->champ_doc.data(); I.champ_score = b->champ_score.data();
    I.n_raw = (int)b->raw_off.size() - 1; I.raw_doc = b->raw_doc.data(); I.raw_off = b->raw_off.data(); I.raw_chars = (const uint16_t*)b->raw_chars.data();
    // free the raw documents
    b->values.clear(); b->values.shrink_to_fit(); b->is_null.clear();
    b->finished = true; return IFX_OK;
}

const ifx_index_image* ifx_builder_image(ifx_builder* b) { return b->finished ? &b->img : nullptr; }

// ---- doc-id-range shards (SURVEY.md 8e): a shard's builder indexes its own document range; the statistics the search path reads as
// GLOBAL quantities are exchanged between the shards' hosts (ifx_builder_export_stats -> all-gather -> ifx_builder_globalize) so that
// every shard scores with the term ordinals, df / idf, N, avgdl, word idf, prefix cardinalities and affix dictionary of the whole corpus.
}  // extern "C"
namespace {
struct Blob { std::vector<uint8_t> d;
    template <class T> void put(const T& v) { const uint8_t* p = (const uint8_t*)&v; d.insert(d.end(), p, p + sizeof(T)); }
    void bytes(const void* p, size_t n) { const uint8_t* q = (const uint8_t*)p; d.insert(d.end(), q, q + n); }
    void strings(const char16_t* chars, const uint32_t* off, int n) { put<int32_t>(n); bytes(off, ((size_t)n + 1) * 4); bytes(chars, (size_t)off[n] * 2); } };
struct Rd { const uint8_t* p; template <class T> T get() { T v; std::memcpy(&v, p, sizeof(T)); p += sizeof(T); return v; }
    const void* take(size_t n) { const void* r = p; p += n; return r; } };
struct StrView { int n; const uint32_t* off; const char16_t* chars; sv at(int i) const { return sv(chars + off[i], off[i + 1] - off[i]); } };
StrView rd_strings(Rd& r) { StrView v; v.n = r.get<int32_t>(); v.off = (const uint32_t*)r.take(((size_t)v.n + 1) * 4); v.chars = (const char16_t*)r.take((size_t)v.off[v.n] * 2); return v; }
}  // namespace

struct ifx_builder_shard { std::vector<int32_t> prefix_card; };       // extra image storage of a globalized shard
static std::vector<std::pair<ifx_builder*, ifx_builder_shard*>> g_shard_extra;
extern "C" {

// Serialised local statistics of a finished shard builder. The caller owns nothing: the blob lives until the next export / destroy.
const uint8_t* ifx_builder_export_stats(ifx_builder* b, size_t* len) {
    static thread_local Blob out; out.d.clear();
    const int N = (int)b->keys.size(); const int T = b->terms.n;
    out.put<int32_t>(N);
    out.strings(b->terms.chars.data(), b->terms.off.data(), T);
    { std::vector<int64_t> dfv(T); for (int t = 0; t < T; t++) dfv[t] = b->df[t] < 0 ? (int64_t)b->stop_term_limit + 1 : b->df[t]; out.bytes(dfv.data(), (size_t)T * 8); }
    out.strings(b->word_chars.data(), b->word_off.data(), (int)b->word_off.size() - 1);
    out.bytes(b->word_df.data(), b->word_df.size() * 4);
    out.strings(b->prefix.chars.data(), b->prefix.off.data(), b->prefix.n);
    { std::vector<int32_t> card(b->prefix.n); for (int k = 0; k < b->prefix.n; k++) card[k] = (int32_t)(b->prefix.row[k + 1] - b->prefix.row[k]); out.bytes(card.data(), card.size() * 4); }
    out.strings(b->affix_chars.data(), b->affix_off.data(), (int)b->affix_off.size() - 1);
    out.bytes(b->affix_last.data(), ((size_t)b->affix_off.size() - 1) * 4);
    out.bytes(b->doc_len.data(), (size_t)N * 4);
    *len = out.d.size(); return out.d.data();
}

// The document lengths of this shard after ifx_builder_globalize (terms that are stop terms only by their corpus-wide df are gone).
const float* ifx_builder_doc_lengths(ifx_builder* b, int* n) { *n = (int)b->doc_len.size(); return b->doc_len.data(); }
// lens[s] = ifx_builder_doc_lengths of shard s, all shards in doc order: avgdl as the reference computes it, one sequential float sum over
// all documents (VectorModel.cs:212-216).
int ifx_builder_set_global_lengths(ifx_builder* b, int n_shards, const float* const* lens, const int* counts) {
    float total = 0.f; int64_t N_all = 0;
    for (int s = 0; s < n_shards; s++) { for (int d = 0; d < counts[s]; d++) total += lens[s][d]; N_all += counts[s]; }
    b->img.avgdl = N_all > 0 ? total / (float)N_all : 0.f;
    return IFX_OK;
}

// blobs[s] = export of shard s (all shards, in doc-range order). Rewrites this builder's image so that it is shard `shard` of the
// global index. `prefix_card_out`: see ifx_builder_prefix_cardinalities.
int ifx_builder_globalize(ifx_builder* b, int n_shards, int shard, const uint8_t* const* blobs) {
    if (!b->finished || n_shards < 1 || shard < 0 || shard >= n_shards) return IFX_ERR_INVALID;
    std::vector<int> shard_docs(n_shards); int64_t N_all = 0;
    struct In { int N; StrView terms; const int64_t* df; StrView words; const int32_t* wdf; StrView prefix; const int32_t* pcard; StrView affix; const int32_t* alast; const float* dl; };
    std::vector<In> in(n_shards);
    for (int s = 0; s < n_shards; s++) { Rd r{blobs[s]}; In& x = in[s]; x.N = r.get<int32_t>(); x.terms = rd_strings(r); x.df = (const int64_t*)r.take((size_t)x.terms.n * 8);
        x.words = rd_strings(r); x.wdf = (const int32_t*)r.take((size_t)x.words.n * 4); x.prefix = rd_strings(r); x.pcard = (const int32_t*)r.take((size_t)x.prefix.n * 4);
        x.affix = rd_strings(r); x.alast = (const int32_t*)r.take((size_t)x.affix.n * 4); x.dl = (const float*)r.take((size_t)x.N * 4); shard_docs[s] = x.N; N_all += x.N; }
    if (N_all > 0x7fffffffLL) return IFX_ERR_INVALID;
    int64_t doc_base = 0; for (int s = 0; s < shard; s++) doc_base += shard_docs[s];
    const int N = (int)b->keys.size();
    // ---- terms: global ordinals = first occurrence over the shards in doc order (TermCollection order of the whole corpus), df summed
    Interner g; std::vector<int64_t> gdf; std::vector<int32_t> l2g(b->terms.n, -1);
    for (int s = 0; s < n_shards; s++) for (int t = 0; t < in[s].terms.n; t++) { bool nw; int id = g.intern(in[s].terms.at(t), &nw); if (nw) gdf.push_back(0); gdf[id] += in[s].df[t]; if (s == shard) l2g[t] = id; }
    const int TG = g.size();
    {   Csr nt; nt.n = TG; nt.chars.assign(g.arena.begin(), g.arena.end()); if (nt.chars.empty()) nt.chars.push_back(0); nt.off = g.off; nt.row.assign((size_t)TG + 1, 0);
        std::vector<int32_t> g2l(TG, -1); for (int t = 0; t < b->terms.n; t++) g2l[l2g[t]] = t;
        std::vector<int32_t> ndf(TG);
        for (int gt = 0; gt < TG; gt++) { const bool stop = gdf[gt] > b->stop_term_limit; ndf[gt] = stop ? -1 : (int32_t)gdf[gt]; const int lt = g2l[gt];
            nt.row[gt + 1] = nt.row[gt] + ((lt >= 0 && !stop && b->df[lt] > 0) ? b->terms.row[lt + 1] - b->terms.row[lt] : 0); }
        nt.docs.resize((size_t)nt.row[TG]); nt.w.resize((size_t)nt.row[TG]);
        par_for(TG, 16, [&](int64_t a, int64_t e, int) { for (int64_t gt = a; gt < e; gt++) { const int lt = g2l[gt]; const int64_t n = nt.row[gt + 1] - nt.row[gt]; if (n <= 0) continue;
            std::memcpy(nt.docs.data() + nt.row[gt], b->terms.docs.data() + b->terms.row[lt], (size_t)n * 4); std::memcpy(nt.w.data() + nt.row[gt], b->terms.w.data() + b->terms.row[lt], (size_t)n); } });
        // a term that became a stop term globally no longer contributes to the document lengths of this shard
        std::vector<uint32_t> dl(N, 0); for (int64_t i = 0; i < nt.row[TG]; i++) dl[nt.docs[i]] += nt.w[i];
        for (int d = 0; d < N; d++) b->doc_len[d] = (float)dl[d];
        std::swap(b->terms.chars, nt.chars); std::swap(b->terms.off, nt.off); std::swap(b->terms.row, nt.row); std::swap(b->terms.docs.p, nt.docs.p); std::swap(b->terms.docs.n, nt.docs.n); std::swap(b->terms.w.p, nt.w.p); std::swap(b->terms.w.n, nt.w.n);
        b->terms.n = TG; b->df.swap(ndf);
    }
    // ---- avgdl: needs every shard's lengths AFTER the global stop terms were dropped: second exchange, ifx_builder_set_global_lengths
    const float avgdl = 0.f;
    // ---- word idf over the whole corpus
    { Interner gw; std::vector<int64_t> wdf; for (int s = 0; s < n_shards; s++) for (int k = 0; k < in[s].words.n; k++) { bool nw; int id = gw.intern(in[s].words.at(k), &nw); if (nw) wdf.push_back(0); wdf[id] += in[s].wdf[k]; }
      b->word_chars.assign(gw.arena.begin(), gw.arena.end()); if (b->word_chars.empty()) b->word_chars.push_back(0); b->word_off = gw.off; b->word_idf.resize(wdf.size());
      for (size_t i = 0; i < wdf.size(); i++) b->word_idf[i] = (wdf[i] > 0 && wdf[i] <= N_all) ? compute_idf_host((int)N_all, (int)wdf[i]) : 0.f; }
    // ---- prefix docsets: global key set with global cardinalities, local rows
    ifx_builder_shard* ex = new ifx_builder_shard();
    { Interner gp; std::vector<int64_t> card; std::vector<int32_t> pl2g(b->prefix.n, -1);
      for (int s = 0; s < n_shards; s++) for (int k = 0; k < in[s].prefix.n; k++) { bool nw; int id = gp.intern(in[s].prefix.at(k), &nw); if (nw) card.push_back(0); card[id] += in[s].pcard[k]; if (s == shard) pl2g[k] = id; }
      const int PG = gp.size(); std::vector<int32_t> g2l(PG, -1); for (int k = 0; k < b->prefix.n; k++) g2l[pl2g[k]] = k;
      Csr np; np.n = PG; np.chars.assign(gp.arena.begin(), gp.arena.end()); if (np.chars.empty()) np.chars.push_back(0); np.off = gp.off; np.row.assign((size_t)PG + 1, 0);
      for (int k = 0; k < PG; k++) np.row[k + 1] = np.row[k] + (g2l[k] >= 0 ? b->prefix.row[g2l[k] + 1] - b->prefix.row[g2l[k]] : 0);
      np.docs.resize((size_t)np.row[PG]);
      for (int k = 0; k < PG; k++) if (g2l[k] >= 0) std::memcpy(np.docs.data() + np.row[k], b->prefix.docs.data() + b->prefix.row[g2l[k]], (size_t)(np.row[k + 1] - np.row[k]) * 4);
      std::swap(b->prefix.chars, np.chars); std::swap(b->prefix.off, np.off); std::swap(b->prefix.row, np.row); std::swap(b->prefix.docs.p, np.docs.p); std::swap(b->prefix.docs.n, np.docs.n); b->prefix.n = PG;
      ex->prefix_card.resize(PG); for (int k = 0; k < PG; k++) ex->prefix_card[k] = (int32_t)std::min<int64_t>(card[k], 0x7fffffff); }
    // ---- affix words: global dictionary, last document wins (Q4) -- kept as a LOCAL id when this shard owns that document, else -1
    { Interner ga; std::vector<int64_t> last; int64_t base = 0;
      for (int s = 0; s < n_shards; s++) { for (int k = 0; k < in[s].affix.n; k++) { bool nw; int id = ga.intern(in[s].affix.at(k), &nw); if (nw) last.push_back(-1); last[id] = base + in[s].alast[k]; } base += in[s].N; }
      b->affix_chars.assign(ga.arena.begin(), ga.arena.end()); if (b->affix_chars.empty()) b->affix_chars.push_back(0); b->affix_off = ga.off; b->affix_last.assign(std::max<size_t>(last.size(), 1), -1);
      for (size_t i = 0; i < last.size(); i++) { const int64_t l = last[i] - doc_base; b->affix_last[i] = (l >= 0 && l < N) ? (int32_t)l : -1; } }
    // ---- image
    ifx_index_image& I = b->img; auto S = [](std::vector<char16_t>& c, std::vector<uint32_t>& o) { return ifx_strings{(const uint16_t*)c.data(), o.data(), (int)o.size() - 1}; };
    I.n_live = (int32_t)N_all; I.avgdl = avgdl; I.doc_len = b->doc_len.data();
    I.terms = S(b->terms.chars, b->terms.off); I.df = b->df.data(); I.row_ptr = b->terms.row.data(); I.post_doc = b->terms.docs.data(); I.post_tf = b->terms.w.data();
    I.words = S(b->word_chars, b->word_off); I.word_idf = b->word_idf.data();
    I.prefix = {S(b->prefix.chars, b->prefix.off), b->prefix.row.data(), b->prefix.docs.data()};
    I.affix_words = S(b->affix_chars, b->affix_off); I.affix_last_doc = b->affix_last.data();
    I.prefix_global_card = ex->prefix_card.data(); I.shard_index = shard; I.n_shards = n_shards; I.doc_base = doc_base;
    g_shard_extra.emplace_back(b, ex);
    return IFX_OK;
}


}  // extern "C"

extern "C" void ifx_builder_destroy(ifx_builder* b) { for (size_t i = 0; i < g_shard_extra.size(); i++) if (g_shard_extra[i].first == b) { delete g_shard_extra[i].second; g_shard_extra.erase(g_shard_extra.begin() + i); break; } delete b; }

// SearchEngine.Search step 1 (src/Infidex/SearchEngine.cs:264-274): Trim, TextNormalizer.Normalize, ToLowerInvariant.
extern "C" int ifx_host_prepare_query(const uint16_t* in, int n, uint16_t* out, int cap) {
    static std::vector<uint8_t> ws = [] { std::vector<uint8_t> w(65536, 0); for (int i = 0; i < IFX_SPACE_LIST_N; i++) w[IFX_SPACE_LIST[i]] = 1; return w; }();
    int b = 0, e = n; while (b < e && ws[in[b]]) b++; while (e > b && ws[in[e - 1]]) e--;
    str nrm; normalize_into(sv((const char16_t*)in + b, (size_t)(e - b)), nrm); lower_inplace(nrm);
    int m = (int)std::min<size_t>(nrm.size(), (size_t)cap); std::memcpy(out, nrm.data(), (size_t)m * 2);
    return (int)nrm.size();
}

// accessors used by the host mirror to turn facet (column, value id) pairs back into strings
extern "C" int ifx_builder_num_columns(ifx_builder* b) { return (int)b->cols.size(); }
extern "C" int ifx_builder_column_name(ifx_builder* b, int c, uint16_t* buf, int cap) { const str& s = b->col_names[c]; int n = (int)std::min<size_t>(s.size(), (size_t)cap); std::memcpy(buf, s.data(), (size_t)n * 2); return (int)s.size(); }
extern "C" int ifx_builder_column_dict_size(ifx_builder* b, int c) { return (int)b->col_off[c].size() - 1; }
extern "C" int ifx_builder_column_value(ifx_builder* b, int c, int id, uint16_t* buf, int cap) {
    uint32_t o = b->col_off[c][id], e = b->col_off[c][id + 1]; int n = (int)std::min<size_t>(e - o, (size_t)cap); std::memcpy(buf, b->col_chars[c].data() + o, (size_t)n * 2); return (int)(e - o);
}

// ResultProcessor.CompareValues over the distinct values of column c, from the field's own runtime type: int64 as int64 (the dictionary holds
// the exact decimal text), double as double (shortest round-trip text; double.CompareTo: NaN lowest, -0 == 0), strings ordinally (this
// project's restatement of the culture-dependent string.CompareTo; a C# host ranks with .NET's own comparer instead). Dense ranks from 0.
extern "C" int ifx_builder_column_order(ifx_builder* b, int c, int32_t* rank) {
    if (!b || !b->finished || !rank || c < 0 || c >= (int)b->col_off.size()) return IFX_ERR_INVALID;
    const int kind = b->col_kind[c]; if (kind < 0) return IFX_ERR_UNSUPPORTED;      // values of several runtime types: no total order
    const int n = (int)b->col_off[c].size() - 1;
    auto at = [&](int i) { return sv(b->col_chars[c].data() + b->col_off[c][i], b->col_off[c][i + 1] - b->col_off[c][i]); };
    auto ascii = [&](int i, char* buf) { sv v = at(i); size_t m = std::min<size_t>(v.size(), 63); for (size_t k = 0; k < m; k++) buf[k] = (char)v[k]; return m; };
    std::vector<int64_t> iv; std::vector<double> dv;
    if (kind == 2) { iv.resize(n); for (int i = 0; i < n; i++) { char buf[64]; size_t m = ascii(i, buf); std::from_chars(buf, buf + m, iv[i]); } }
    if (kind == 3) { dv.resize(n); for (int i = 0; i < n; i++) { char buf[64]; size_t m = ascii(i, buf); std::from_chars(buf, buf + m, dv[i]); } }
    auto cmp = [&](int x, int y) -> int {
        if (kind == 2) return iv[x] < iv[y] ? -1 : (iv[x] > iv[y] ? 1 : 0);
        if (kind == 3) { double a = dv[x], e = dv[y]; if (a < e) return -1; if (a > e) return 1; if (a == e) return 0; return std::isnan(a) ? (std::isnan(e) ? 0 : -1) : 1; }
        sv a = at(x), e = at(y); return a < e ? -1 : (a > e ? 1 : 0);
    };
    std::vector<int32_t> ord(n); std::iota(ord.begin(), ord.end(), 0);
    std::sort(ord.begin(), ord.end(), [&](int x, int y) { return cmp(x, y) < 0; });
    for (int i = 0, r = 0; i < n; i++) { if (i > 0 && cmp(ord[i - 1], ord[i]) != 0) r++; rank[ord[i]] = r; }
    return IFX_OK;
}
