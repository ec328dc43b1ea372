// ORACLE EXTENSION (test infrastructure, NOT product code): SearchEngine with a SynonymMap (Synonyms/SynonymMap.cs) on top of the CPU
// restatement in oracle/. The oracle sources are included unchanged; this file restates the map (its union-find replayed from the ordered
// AddSynonym calls) and the places the reference canonicalises text, each where the reference does it:
//   index text      Normalize -> ToLowerInvariant -> CanonicalizeText          VectorModel.cs:83-93 (n-grams, words, field weights, prefix index)
//   metadata        ToLowerInvariant -> Normalize -> CanonicalizeText          VectorModel.cs:268-281
//   query           Trim -> Normalize -> ToLowerInvariant -> CanonicalizeText  SearchEngine.cs:264-288 (then SearchPipeline normalises again)
//   coverage text   CanonicalizeText(Normalize(IndexedText)) on every ProcessCandidate call, SearchPipeline.cs:470-489
// WordMatcher, the word-idf cache and the short-query scorers read the text as it is. Built and loaded by tests/oracle_syn.py; the entry
// points take the Engine handle an OracleEngine (oracle/oracle.py) created.
#include "../oracle/capi.cpp"
#include <mutex>

namespace {

str fold(sv s) { str r(s); for (auto& c : r) c = up(c); return r; }        // StringComparer.OrdinalIgnoreCase

// Dictionary<string, string>(StringComparer.OrdinalIgnoreCase): the key stays the first string inserted for its fold
struct ICDict {
    std::vector<str> keys; std::vector<str> vals; StrMap<int> at;
    int find(sv k) const { auto it = at.find(fold(k)); return it == at.end() ? -1 : it->second; }
    void set(sv k, const str& v) { int i = find(k); if (i >= 0) { vals[i] = v; return; } at.emplace(fold(k), (int)keys.size()); keys.emplace_back(k); vals.push_back(v); }
};

struct SynMap {
    ICDict parent;
    StrMap<str> frozen; bool is_frozen = false;      // fold(key) -> root, once the index is built (search threads only read)
    bool has_mappings() const { return is_frozen ? !frozen.empty() : !parent.keys.empty(); }

    void add(sv a, sv b) {                                                   // AddSynonym
        if (is_blank(a) || is_blank(b)) return;
        str t1 = to_lower(trim(a)), t2 = to_lower(trim(b));
        if (t1 == t2) return;
        unite(t1, t2);
    }
    void ensure(const str& t) { if (parent.find(t) < 0) parent.set(t, t); }
    str find_root(const str& t) {
        ensure(t); str p = parent.vals[parent.find(t)];
        if (fold(p) != fold(t)) parent.set(t, find_root(p));
        return parent.vals[parent.find(t)];
    }
    void unite(const str& a, const str& b) {
        ensure(a); ensure(b);
        str r1 = find_root(a), r2 = find_root(b);
        if (fold(r1) == fold(r2)) return;
        str canon, other;
        if (r1.size() != r2.size()) { bool first = r1.size() >= r2.size(); canon = first ? r1 : r2; other = first ? r2 : r1; }
        else { canon = r1 <= r2 ? r1 : r2; other = fold(canon) == fold(r1) ? r2 : r1; }   // CompareOrdinal on UTF-16 units
        parent.set(other, canon);
    }
    str canonical(sv tok) {                                                  // GetCanonical
        if (is_blank(tok)) return str();
        str t = to_lower(trim(tok));
        if (is_frozen) { auto it = frozen.find(fold(t)); return it == frozen.end() ? t : it->second; }
        if (parent.find(t) < 0) return t;
        return find_root(t);
    }
    str canonicalize(sv text) {                                              // CanonicalizeText(text, TokenizerSetup.Delimiters)
        if (text.empty() || !has_mappings()) return str(text);
        str out;
        for (size_t i = 0; i < text.size();) {
            if (is_delim(text[i])) { out.push_back(text[i++]); continue; }
            size_t s = i; while (i < text.size() && !is_delim(text[i])) i++;
            out += canonical(text.substr(s, i - s));
        }
        return out;
    }
    void freeze() { for (size_t i = 0; i < parent.keys.size(); i++) frozen[fold(parent.keys[i])] = find_root(parent.keys[i]); is_frozen = true; }
};

std::mutex g_mu; std::unordered_map<const void*, SynMap> g_maps;
SynMap& map_of(const void* h) { std::lock_guard<std::mutex> l(g_mu); return g_maps[h]; }

// VectorModel.IndexDocument with the canonical index text (oracle/index.hpp Index::add_document, canonicalisation added)
void add_document_syn(Index& ix, SynMap& m, long long key, const std::vector<Value>& values) {
    int id = (int)ix.docs.size();
    ix.docs.emplace_back(); Doc& d = ix.docs.back(); d.key = key; d.values = values;
    ix.live_count++;
    ix.key_to_ids[key].push_back(id);
    std::vector<int> order;
    for (int w = 0; w < 3; w++) for (size_t f = 0; f < ix.schema.size(); f++) if (ix.schema[f].indexable && ix.schema[f].weight == w) order.push_back((int)f);
    std::vector<std::pair<int, int>> bounds; str text;
    for (size_t k = 0; k < order.size(); k++) {
        bounds.emplace_back((int)(uint16_t)text.size(), ix.schema[order[k]].weight);
        text += values[order[k]].to_string();
        if (k + 1 < order.size()) text.push_back(u'§');
    }
    std::stable_sort(bounds.begin(), bounds.end(), [](auto& a, auto& b) { return a.first < b.first; });
    d.indexed_text = text;
    str index_text = m.canonicalize(to_lower(normalize(text)));     // field-weight positions: canonical padded text against the raw boundaries
    tokens_for_indexing(index_text, [&](sv tok, int pos) {
        float fw = 1.0f;
        if (!bounds.empty()) { int wi = 0; for (auto& b : bounds) { if (b.first <= pos) wi = b.second; else break; } fw = wi < 3 ? ix.field_weights[wi] : 1.0f; }
        str key_s(tok);
        auto it = ix.term_ids.find(key_s); int tid;
        if (it == ix.term_ids.end()) { tid = (int)ix.terms.size(); ix.term_ids.emplace(key_s, tid); ix.terms.emplace_back(); ix.terms[tid].text = key_s; }
        else tid = it->second;
        Term& t = ix.terms[tid];
        if (t.df != -1) { t.df++; if (t.df > ix.stop_term_limit) t.df = -1; }
        if (t.df < 0) return;
        if ((int)t.w.size() < ix.stop_term_limit) {
            if (t.docs.empty() || t.docs.back() != id) { t.w.push_back(Index::round_w(fw)); t.docs.push_back(id); }
            else { float nw = (float)t.w.back() + fw; if (nw <= 255.f) { t.w.back() = (uint8_t)std::nearbyint((double)nw); t.df--; } }
        } else { t.df = -1; t.w.clear(); t.docs.clear(); }
    });
    {   int token_index = 0;
        for (sv w : split_words(index_text)) {
            int ml = std::min<int>(3, (int)w.size());
            for (int l = 1; l <= ml; l++) { str k(w.substr(0, l)); auto& v = ix.prefix_docs[k]; if (v.empty() || v.back() != id) v.push_back(id); ix.prefix_post[k].push_back({id, (uint16_t)token_index}); }
            token_index++;
        }
    }
    str wm_text = normalize(to_lower(text));                        // WordMatcher.Load: not canonicalised
    for (sv w : split_words(wm_text)) {
        int len = (int)w.size();
        auto add = [&](StrMap<std::vector<int>>& mm, const str& k) { auto& v = mm[k]; if (v.empty() || v.back() != id) v.push_back(id); };
        if (len >= 2 && len <= 8) add(ix.wm_exact, str(w));
        if (len >= 3 && len <= 8) for (int i = 0; i < len; i++) { str v(w); v.erase(i, 1); add(ix.wm_ld1, v); }
        if (len >= 3) ix.wm_affix_last[str(w)] = id;
    }
}

// BuildDocumentMetadataCache with the map (VectorModel.cs:268-281): ToLowerInvariant, Normalize, then CanonicalizeText
void metadata_syn(Index& ix, SynMap& m) {
    for (size_t d = 0; d < ix.docs.size(); d++) {
        if (ix.docs[d].deleted || ix.docs[d].indexed_text.empty()) continue;
        str t = m.canonicalize(normalize(to_lower(ix.docs[d].indexed_text)));
        auto ws = split_words(t);
        ix.first_token[d] = ws.empty() ? str() : str(ws[0]);
        ix.token_count[d] = (uint16_t)std::min<size_t>(ws.size(), 65535);
    }
}

// SearchPipeline.Execute / the coverage stage of oracle/stage2.hpp, with the document text of every ProcessCandidate call canonicalised
std::vector<ScoreEntry> coverage_stage_syn(const Pipeline& P, SynMap& m, const str& search, int depth, int max_results, std::vector<ScoreEntry> top) {
    const Index& ix = P.ix; const CoverageSetup& cs = P.cov.setup;
    if ((int)top.size() > depth) top.resize(depth);
    std::vector<int> wm = P.wm_execute(search);
    std::unordered_map<long long, int> key_idx; int next = 0;
    for (auto& e : top) if (!key_idx.count(e.key)) key_idx[e.key] = next++;
    for (int id : wm) if (!ix.docs[id].deleted && !key_idx.count(ix.docs[id].key)) key_idx[ix.docs[id].key] = next++;
    std::vector<uint8_t> lcs_row(2, 0), hits_row(2, 0);
    TopKHeap final_scores(depth); int max_hits = 0;
    QueryCtx ctx = P.cov.prepare(search);
    std::vector<int> top_ids; for (auto& e : top) { int id = ix.doc_by_key(e.key); if (id >= 0) top_ids.push_back(id); }
    std::sort(top_ids.begin(), top_ids.end());
    std::vector<int> overlap, uniq; for (int id : wm) (std::binary_search(top_ids.begin(), top_ids.end(), id) ? overlap : uniq).push_back(id);
    int wm_limit = std::max(0, depth - (int)overlap.size());
    auto process = [&](int id, float base) {
        const Doc& d = ix.docs[id]; if (d.deleted) return;
        auto it = key_idx.find(d.key); if (it == key_idx.end()) return; int di = it->second;
        str text = m.canonicalize(normalize(d.indexed_text));
        int lcs = 0;
        if (di < 2) {
            lcs = lcs_row[di];
            if (lcs == 0) { int tol = 0; if ((int)ctx.query.size() >= cs.qlimit_tol) tol = (int)((double)ctx.query.size() * cs.lcs_tol_rel); lcs = lcs_metric(ctx.query, text, tol); lcs_row[di] = (uint8_t)std::min(lcs, 255); }
        }
        Features f = P.cov.features(ctx, text, (double)lcs, id);
        auto [score, tie] = fusion_score(ctx.query, text, f, base);
        if (di < 2 && hits_row[di] == 0) hits_row[di] = (uint8_t)std::min(f.word_hits, 255);
        max_hits = std::max(max_hits, f.word_hits);
        final_scores.add({score, d.key, tie});
    };
    for (int id : overlap) process(id, 0.f);
    int pu = 0; for (int id : uniq) { if (pu >= wm_limit) break; process(id, 0.f); pu++; }
    for (auto& c : top) {
        int id = ix.doc_by_key(c.key); if (id < 0) continue;
        float mx = !top.empty() ? top[0].score : 1.f; float nb = mx > 0 ? c.score / mx : 0.f;
        process(id, nb);
    }
    if (max_hits == 0 && wm.empty()) return {};
    std::vector<ScoreEntry> fin = consolidate(final_scores.get_top_k());
    int trunc = -1;
    if (cs.truncate && !fin.empty()) {
        int min_hits = std::max(cs.min_hits_abs, max_hits - cs.min_hits_rel);
        for (int i = (int)fin.size() - 1; i >= 0; i--) {
            auto it = key_idx.find(fin[i].key); if (it == key_idx.end()) continue; int di = it->second;
            uint8_t wh = di < 2 ? hits_row[di] : 0, lb = di < 2 ? lcs_row[di] : 0;
            if (wh >= min_hits || lb > 0 || fin[i].score >= (float)cs.truncation_score) { trunc = i; break; }
        }
    }
    int count = (trunc == -1 || !cs.truncate) ? max_results : std::min(std::max(0, trunc) + 1, max_results);
    if ((int)fin.size() > count) fin.resize(count);
    return fin;
}

SearchOut execute_syn(const Pipeline& P, SynMap& m, sv search_in, bool enable_coverage, int depth, int max_results) {
    const Index& ix = P.ix; SearchOut out;
    if (is_blank(search_in)) return out;
    str search = normalize(search_in);                                       // SearchPipeline.cs:68-71: the second Normalize
    QueryAnalysis qa = analyze_query(search);
    std::vector<ScoreEntry> stage1;
    if (!qa.can_use_ngrams && ix.from_image) { out.unsupported = true; return out; }
    if (!qa.can_use_ngrams) { out.short_path = true; stage1 = P.sq.stage1(search, max_results); }
    else { str tfidf_q = qa.mixed ? qa.long_words : search; if (is_blank(tfidf_q)) tfidf_q = search; stage1 = P.s1.search(tfidf_q, depth, nullptr); }
    bool short_q = !search.empty() && search.size() <= 3; for (char16_t c : search) if (is_delim(c)) short_q = false;
    if (short_q && (long long)stage1.size() >= max_results && max_results < INT32_MAX) { stage1.resize(max_results); out.records = stage1; out.stage = 1; return out; }
    int sq_count = 0; bool sq_known = false;
    if (short_q) { auto it = ix.prefix_docs.find(search); sq_count = it == ix.prefix_docs.end() ? 0 : (int)it->second.size(); sq_known = true; }
    bool skip_cap = short_q && sq_known && sq_count > 500;
    bool allow_short_cov = short_q && sq_known && sq_count > 0 && sq_count <= 500;
    if (!enable_coverage || skip_cap || (!qa.can_use_ngrams && !allow_short_cov)) { out.records = stage1; out.stage = 1; return out; }
    std::vector<ScoreEntry> covr = coverage_stage_syn(P, m, search, depth, max_results, stage1);
    if (covr.empty() && !stage1.empty()) { out.records = stage1; out.stage = 1; return out; }
    out.records = covr; out.stage = 2; return out;
}

// SearchEngine.Search with the map: the query is canonicalised before the blank / facet decision (do_search of oracle/capi.cpp otherwise)
SearchResult search_syn(const Engine& e, SynMap& m, sv raw, int max_results, int depth, bool enable_cov, const CompiledFilter* filt, bool facets) {
    if (!m.has_mappings()) return do_search(e, raw, max_results, depth, enable_cov, filt, facets);
    SearchResult r;
    if (!e.ix.built) return r;
    str q = m.canonicalize(to_lower(normalize(trim(raw))));
    if (is_blank(q)) return do_search(e, sv(), max_results, depth, enable_cov, filt, facets);   // the empty result / the facet browse
    SearchOut o = execute_syn(*e.pipe, m, q, enable_cov, depth, max_results);
    if (o.unsupported) { r.status = 1; return r; }
    std::vector<ScoreEntry> res = std::move(o.records);
    if (filt) {
        FilterVM vm; std::vector<ScoreEntry> kept;
        for (auto& s : res) { int id = e.ix.doc_by_key(s.key); if (id < 0) continue; if (vm.execute(*filt, e.ix, id)) kept.push_back(s); }
        if (vm.unsupported) r.status = 1;
        res.swap(kept);
    }
    if (facets) r.facets = build_facets(e.ix, res);
    r.total = (int)res.size();
    if ((int)res.size() > max_results) res.resize(max_results);
    r.recs = std::move(res);
    return r;
}

}  // namespace

extern "C" {

// AddSynonym(a, b) for each pair, in order (before indexing)
int ifxo_syn_add(void* h, const uint16_t* a, int na, const uint16_t* b, int nb) {
    map_of(h).add(sv((const char16_t*)a, (size_t)na), sv((const char16_t*)b, (size_t)nb)); return 0;
}
void ifxo_syn_forget(void* h) { std::lock_guard<std::mutex> l(g_mu); g_maps.erase(h); }
// the table (key, GetCanonical(key)) over the union-find's keys in insertion order, as "key\tcanonical\n" UTF-8 lines
int ifxo_syn_table(void* h, char* buf, int cap) {
    SynMap& m = map_of(h); std::string s;
    for (size_t i = 0; i < m.parent.keys.size(); i++) { s += utf16_to_utf8(m.parent.keys[i]); s.push_back('\t'); s += utf16_to_utf8(m.find_root(m.parent.keys[i])); s.push_back('\n'); }
    int n = std::min((int)s.size(), cap); if (buf && n > 0) std::memcpy(buf, s.data(), n); return (int)s.size();
}
int ifxo_syn_canonicalize(void* h, const uint16_t* t, int n, uint16_t* out, int cap) {
    str r = map_of(h).canonicalize(sv((const char16_t*)t, (size_t)n)); int m = std::min((int)r.size(), cap); if (m > 0) std::memcpy(out, r.data(), (size_t)m * 2); return (int)r.size();
}
int ifxo_syn_add_docs(void* h, int n, const long long* keys, const int* kinds, const void* const* cols, const long long* const* offs) {
    Engine* e = (Engine*)h; SynMap& m = map_of(h); int F = (int)e->ix.schema.size();
    for (int d = 0; d < n; d++) {
        std::vector<Value> vals(F);
        for (int f = 0; f < F; f++) {
            Value& v = vals[f];
            if (kinds[f] == 1) { v.kind = 1; const char16_t* b = (const char16_t*)cols[f]; v.s = str(b + offs[f][d], (size_t)(offs[f][d + 1] - offs[f][d])); }
            else if (kinds[f] == 2) { v.kind = 2; v.i = ((const long long*)cols[f])[d]; }
            else if (kinds[f] == 3) { v.kind = 3; v.d = ((const double*)cols[f])[d]; }
        }
        add_document_syn(e->ix, m, keys[d], vals);
    }
    return 0;
}
int ifxo_syn_build(void* h) {
    Engine* e = (Engine*)h; SynMap& m = map_of(h);
    e->ix.build(); if (m.has_mappings()) metadata_syn(e->ix, m);
    m.freeze(); delete e->pipe; e->pipe = new Pipeline(e->ix); return 0;
}
// index state from an image: the map is the image's table (syn_keys -> syn_canon)
int ifxo_syn_load_image(void* h, const ifx_index_image* img) {
    ifxo_load_image(h, img); SynMap& m = map_of(h); m.frozen.clear();
    for (int i = 0; i < img->syn_keys.n; i++) {
        str k((const char16_t*)img->syn_keys.chars + img->syn_keys.off[i], img->syn_keys.off[i + 1] - img->syn_keys.off[i]);
        m.frozen[fold(k)] = str((const char16_t*)img->syn_canon.chars + img->syn_canon.off[i], img->syn_canon.off[i + 1] - img->syn_canon.off[i]);
    }
    m.is_frozen = true; return 0;
}
int ifxo_syn_search(void* h, const uint16_t* q, int qlen, int max_results, int depth, int enable_cov,
                    const uint8_t* filter, int filter_len, int enable_facets,
                    long long* out_keys, float* out_scores, uint8_t* out_ties, int cap, int* out_n, int* out_total,
                    char* facet_buf, int facet_cap, int* facet_len) {
    Engine* e = (Engine*)h; SynMap& m = map_of(h); CompiledFilter cf; const CompiledFilter* pf = nullptr;
    if (filter && filter_len > 0) { cf = deserialize_filter(filter, (size_t)filter_len); if (!cf.ok) return 2; pf = &cf; }
    SearchResult r = search_syn(*e, m, sv((const char16_t*)q, (size_t)qlen), max_results, depth, enable_cov != 0, pf, enable_facets != 0);
    int n = std::min((int)r.recs.size(), cap);
    for (int i = 0; i < n; i++) { out_keys[i] = r.recs[i].key; out_scores[i] = r.recs[i].score; out_ties[i] = r.recs[i].tie; }
    *out_n = n; if (out_total) *out_total = r.total;
    if (facet_len) {
        std::string fb; for (auto& f : r.facets) { fb += utf16_to_utf8(f.field); fb.push_back('\t'); fb += utf16_to_utf8(f.value); fb.push_back('\t'); fb += std::to_string(f.count); fb.push_back('\n'); }
        int mm = std::min((int)fb.size(), facet_cap); if (facet_buf && mm > 0) std::memcpy(facet_buf, fb.data(), mm); *facet_len = mm;
    }
    return r.status;
}
int ifxo_syn_search_batch(void* h, const uint16_t* qblob, const long long* qoff, int nq, int max_results, int depth, int enable_cov,
                          const uint8_t* filter, int filter_len, int threads,
                          long long* out_keys, float* out_scores, uint8_t* out_ties, int cap, int* out_n, int* status) {
    Engine* e = (Engine*)h; SynMap& m = map_of(h); CompiledFilter cf; const CompiledFilter* pf = nullptr;
    if (filter && filter_len > 0) { cf = deserialize_filter(filter, (size_t)filter_len); if (!cf.ok) return 2; pf = &cf; }
    std::atomic<int> next{0};
    auto work = [&]() {
        for (;;) { int i = next.fetch_add(1); if (i >= nq) break;
            SearchResult r = search_syn(*e, m, sv((const char16_t*)qblob + qoff[i], (size_t)(qoff[i + 1] - qoff[i])), max_results, depth, enable_cov != 0, pf, false);
            int n = std::min((int)r.recs.size(), cap);
            for (int k = 0; k < n; k++) { out_keys[(size_t)i * cap + k] = r.recs[k].key; out_scores[(size_t)i * cap + k] = r.recs[k].score; out_ties[(size_t)i * cap + k] = r.recs[k].tie; }
            out_n[i] = n; if (status) status[i] = r.status; }
    };
    if (threads <= 1) work(); else { std::vector<std::thread> ts; for (int t = 0; t < threads; t++) ts.emplace_back(work); for (auto& t : ts) t.join(); }
    return 0;
}

}  // extern "C"
