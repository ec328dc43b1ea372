// ORACLE EXTENSION (test infrastructure, NOT product code): Query.EnableBoost / Boosts and Query.SortBy / SortAscending
// (ResultProcessor.ApplyBoosts / ApplySort, run by ApplyPostProcessing after the filter) on top of the CPU restatement in oracle/.
// The oracle sources are included unchanged; this file only adds the post-processing step and its entry points, which take the
// Engine handle an OracleEngine (oracle/oracle.py) created -- the same capi.cpp compiled with the same flags, so the same layout.
// Built and loaded by tests/oracle_post.py.
#include "../oracle/capi.cpp"
#include <cmath>
#include <charconv>

namespace {

// Query.EnableBoost + Boosts (the boosts whose Filter is not null) and Query.SortBy + SortAscending
struct PostSpec { std::vector<CompiledFilter> boosts; std::vector<int> strength; bool sort = false; str sort_field; bool ascending = true; };

// ResultProcessor.CompareValues: null == null, null first; same runtime type -> IComparable.CompareTo; else ordinal compare of ToString().
// string.CompareTo is culture-dependent in .NET: this restatement compares strings ordinally (DESIGN.md section 5).
int compare_values(const Value& a, const Value& b) {
    if (a.is_null() && b.is_null()) return 0; if (a.is_null()) return -1; if (b.is_null()) return 1;
    if (a.kind == b.kind) switch (a.kind) {
        case 1: return a.s < b.s ? -1 : (a.s > b.s ? 1 : 0);
        case 2: return a.i < b.i ? -1 : (a.i > b.i ? 1 : 0);
        case 3: if (a.d < b.d) return -1; if (a.d > b.d) return 1; if (a.d == b.d) return 0; return std::isnan(a.d) ? (std::isnan(b.d) ? 0 : -1) : 1;   // double.CompareTo
        case 4: return a.b == b.b ? 0 : (a.b ? 1 : -1);
    }
    str x = a.to_string(), y = b.to_string(); return x < y ? -1 : (x > y ? 1 : 0);
}

// ResultProcessor.ApplyBoosts then ApplySort. Both end in Array.Sort(Comparison): the .NET introsort (oracle/text.hpp dotnet_sort).
void apply_post(const Index& ix, const PostSpec& P, std::vector<ScoreEntry>& res, int& status) {
    if (!P.boosts.empty()) {
        FilterVM vm;
        for (auto& s : res) {
            int id = ix.doc_by_key(s.key); if (id < 0) continue;       // GetDocumentByPublicKey
            int total = 0; for (size_t k = 0; k < P.boosts.size(); k++) if (vm.execute(P.boosts[k], ix, id)) total += P.strength[k];
            if (total > 0) s.score = s.score + (float)total;
        }
        if (vm.unsupported) status = 1;
        dotnet_sort(res, [](const ScoreEntry& a, const ScoreEntry& b) { return b.score < a.score ? -1 : (b.score > a.score ? 1 : 0); });   // b.Score.CompareTo(a.Score)
    }
    if (P.sort) {
        int f = -1; for (size_t k = 0; k < ix.schema.size(); k++) if (ix.schema[k].name == P.sort_field) { f = (int)k; break; }   // GetField: ordinal name match
        static const Value null_value;
        std::vector<std::pair<ScoreEntry, const Value*>> v;
        for (auto& s : res) { int id = ix.doc_by_key(s.key); v.emplace_back(s, (f >= 0 && id >= 0) ? &ix.docs[id].values[f] : &null_value); }
        const bool asc = P.ascending;
        dotnet_sort(v, [asc](const std::pair<ScoreEntry, const Value*>& a, const std::pair<ScoreEntry, const Value*>& b) { return asc ? compare_values(*a.second, *b.second) : compare_values(*b.second, *a.second); });
        for (size_t i = 0; i < v.size(); i++) res[i] = v[i].first;
    }
}

// SearchEngine.Search (SearchEngine.cs:256-319) with the post-processing step: the flow of do_search in oracle/capi.cpp, with
// ApplyBoosts / ApplySort between the filter and the facets. The blank query (empty result, or the facet browse) ignores both.
SearchResult search_post(const Engine& e, sv raw, int max_results, int depth, bool enable_cov, const CompiledFilter* filt, bool facets, const PostSpec& post) {
    str q = to_lower(normalize(trim(raw)));
    if (!e.ix.built || is_blank(q)) return do_search(e, raw, max_results, depth, enable_cov, filt, facets);
    SearchResult r;
    SearchOut o = e.pipe->execute(q, enable_cov, depth, max_results, nullptr, nullptr);
    if (o.unsupported) { r.status = 1; return r; }
    std::vector<ScoreEntry> res = std::move(o.records);
    if (filt) {
        FilterVM vm; std::vector<ScoreEntry> kept;
        for (auto& s : res) { int id = e.ix.doc_by_key(s.key); if (id < 0) continue; if (vm.execute(*filt, e.ix, id)) kept.push_back(s); }
        if (vm.unsupported) r.status = 1;
        res.swap(kept);
    }
    apply_post(e.ix, post, res, r.status);
    if (facets) r.facets = build_facets(e.ix, res);
    r.total = (int)res.size();
    if ((int)res.size() > max_results) res.resize(max_results);
    r.recs = std::move(res);
    return r;
}

// boosts: n_boosts INFISCRIPT-V1 programs (boost_code[i], boost_len[i]) with their (int)BoostStrength; sort_len < 0: no SortBy
bool make_post(PostSpec& P, const uint8_t* const* boost_code, const int* boost_len, const int* strength, int n_boosts,
               const uint16_t* sort_field, int sort_len, int sort_asc) {
    for (int i = 0; i < n_boosts; i++) { CompiledFilter cf = deserialize_filter(boost_code[i], (size_t)boost_len[i]); if (!cf.ok) return false; P.boosts.push_back(std::move(cf)); P.strength.push_back(strength[i]); }
    P.sort = sort_len >= 0; if (P.sort) P.sort_field = str((const char16_t*)sort_field, (size_t)sort_len); P.ascending = sort_asc != 0;
    return true;
}

}  // namespace

extern "C" {

// ifxo_search + boosts / SortBy (see make_post); status: 0 ok, 1 unsupported, 2 malformed bytecode
int ifxo_post_search(void* h, const uint16_t* q, int qlen, int max_results, int depth, int enable_cov,
                     const uint8_t* filter, int filter_len, int enable_facets,
                     const uint8_t* const* boost_code, const int* boost_len, const int* strength, int n_boosts, const uint16_t* sort_field, int sort_len, int sort_asc,
                     long long* out_keys, float* out_scores, uint8_t* out_ties, int cap, int* out_n, int* out_total,
                     char* facet_buf, int facet_cap, int* facet_len) {
    Engine* e = (Engine*)h; CompiledFilter cf; const CompiledFilter* pf = nullptr; PostSpec P;
    if (!make_post(P, boost_code, boost_len, strength, n_boosts, sort_field, sort_len, sort_asc)) return 2;
    if (filter && filter_len > 0) { cf = deserialize_filter(filter, (size_t)filter_len); if (!cf.ok) return 2; pf = &cf; }
    SearchResult r = search_post(*e, sv((const char16_t*)q, (size_t)qlen), max_results, depth, enable_cov != 0, pf, enable_facets != 0, P);
    int n = std::min((int)r.recs.size(), cap);
    for (int i = 0; i < n; i++) { out_keys[i] = r.recs[i].key; out_scores[i] = r.recs[i].score; out_ties[i] = r.recs[i].tie; }
    *out_n = n; if (out_total) *out_total = r.total;
    if (facet_len) {
        std::string fb; for (auto& f : r.facets) { fb += utf16_to_utf8(f.field); fb.push_back('\t'); fb += utf16_to_utf8(f.value); fb.push_back('\t'); fb += std::to_string(f.count); fb.push_back('\n'); }
        int m = std::min((int)fb.size(), facet_cap); if (facet_buf && m > 0) std::memcpy(facet_buf, fb.data(), m); *facet_len = m;
    }
    return r.status;
}

// ifxo_search_batch with the same boosts / SortBy on every query, over `threads` host threads
int ifxo_post_search_batch(void* h, const uint16_t* qblob, const long long* qoff, int nq, int max_results, int depth, int enable_cov,
                           const uint8_t* filter, int filter_len,
                           const uint8_t* const* boost_code, const int* boost_len, const int* strength, int n_boosts, const uint16_t* sort_field, int sort_len, int sort_asc,
                           int threads, long long* out_keys, float* out_scores, uint8_t* out_ties, int cap, int* out_n, int* status) {
    Engine* e = (Engine*)h; CompiledFilter cf; const CompiledFilter* pf = nullptr; PostSpec P;
    if (!make_post(P, boost_code, boost_len, strength, n_boosts, sort_field, sort_len, sort_asc)) return 2;
    if (filter && filter_len > 0) { cf = deserialize_filter(filter, (size_t)filter_len); if (!cf.ok) return 2; pf = &cf; }
    std::atomic<int> next{0};
    auto work = [&]() {
        for (;;) { int i = next.fetch_add(1); if (i >= nq) break;
            SearchResult r = search_post(*e, sv((const char16_t*)qblob + qoff[i], (size_t)(qoff[i + 1] - qoff[i])), max_results, depth, enable_cov != 0, pf, false, P);
            int n = std::min((int)r.recs.size(), cap);
            for (int k = 0; k < n; k++) { out_keys[(size_t)i * cap + k] = r.recs[k].key; out_scores[(size_t)i * cap + k] = r.recs[k].score; out_ties[(size_t)i * cap + k] = r.recs[k].tie; }
            out_n[i] = n; if (status) status[i] = r.status; }
    };
    if (threads <= 1) work(); else { std::vector<std::thread> ts; for (int t = 0; t < threads; t++) ts.emplace_back(work); for (auto& t : ts) t.join(); }
    return 0;
}

// An index loaded from a flattened image (ifxo_load_image) holds column values as their ToString() text. Restores the runtime type of
// field `name` (2 int64, 3 double) by parsing that text back -- exact: it is the shortest round-trip form -- so that SortBy compares the
// values as the documents hold them (10 after 9.9). ToString(), filters and facets are unchanged. Returns the number of values converted,
// -1 if the field is unknown or a value does not parse.
int ifxo_post_set_field_kind(void* h, const uint16_t* name, int n, int kind) {
    Engine* e = (Engine*)h; str nm((const char16_t*)name, (size_t)n); int f = -1;
    for (size_t k = 0; k < e->ix.schema.size(); k++) if (e->ix.schema[k].name == nm) { f = (int)k; break; }
    if (f < 0 || (kind != 2 && kind != 3)) return -1;
    int conv = 0;
    for (auto& d : e->ix.docs) { Value& v = d.values[f]; if (v.kind != 1) continue;
        std::string a(v.s.begin(), v.s.end()); std::from_chars_result r;
        if (kind == 2) r = std::from_chars(a.data(), a.data() + a.size(), v.i); else r = std::from_chars(a.data(), a.data() + a.size(), v.d);
        if (r.ec != std::errc() || r.ptr != a.data() + a.size()) return -1;
        v.kind = kind; v.s.clear(); conv++; }
    return conv;
}

}  // extern "C"
