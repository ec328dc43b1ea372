"""Doc-id-range sharding of ONE index over the ranks of a torch.distributed job (one process per GPU; NCCL on GPUs, gloo in the CPU tests).

Layout (SURVEY.md 8e, DESIGN.md "multi-GPU"): rank r indexes the contiguous document range [r*N/R, (r+1)*N/R) rounded to multiples of
65 536 (the reference's container size, so no 4096-chunk of Bm25Scorer is ever split). The statistics the search path reads as global
quantities -- term ordinals, df / idf, N, avgdl, word idf, prefix-set cardinalities, the affix dictionary -- are exchanged once at build
time (ifx_builder_export_stats -> all_gather -> ifx_builder_globalize), and so are the champion lists of the one-character queries
(ifx_builder_export_champions -> all_gather -> ifx_builder_globalize_champions), and so are the filter / facet / sort column dictionaries
(ifx_builder_export_columns -> all_gather -> ifx_builder_globalize_columns: a value id means the same on every shard). Every batch then
runs on every shard, with these exchanges:
    all-reduce(sum)  document frequency of every LD1 union (its idf is a corpus-level quantity)                 16 int32 per query
    all-reduce(sum)  the selector's cardinalities                                                               40 int32 per query
    all-reduce(sum)  matched documents of every short query (only when the batch holds one)                     1 int32 per short query
    all-reduce(max)  largest integer score of every short query (BuildFinalScores)                              1 int32 per short query
    all-reduce(max)  largest coverage word hits per query (only with short queries: their fallback to Stage 1)   1 int32 per query
    all-gather       per-shard Stage-1 top-`depth` (key, score): global cut + global top score (normBm25)      depth * 12 B per query and shard
    all-gather       per-shard final records (key, score, tie, counts): merged identically on every rank, truncated, then filtered
    all-gather       per record: filter outcome + facet value ids (only when a query filters or counts facets)  4 * (1 + F) B per record
    all-gather       facet rows of queries answered with their whole Stage-1 list (only those with facets)   12 * facet_cap B per query
What is NOT exchanged (counted, never hidden -- `parity` in the bench line is the number of sampled queries whose merged records differ
from the unsharded oracle): the selector's tier rules and the MaxScore threshold chain run on shard-local counts / heaps, the WordMatcher
quota, docIndex-0/1 rule and truncation index are evaluated per shard.
"""
import contextlib
import ctypes as C
import time

import numpy as np

from . import engine as E

CONTAINER = 65536


def rank_batch_seed(base_seed, step, rank):
    """Deterministic, distinct batch per (step, rank)."""
    return base_seed + step + 1000 * rank


def max_over_ranks(dist, values, device="cpu"):
    import torch
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return [float(x) for x in t]


def gather_results(dist, keys, device="cpu"):
    """All-gather the [nq, cap] int64 key block of every rank; returns a list indexed by rank (numpy arrays)."""
    import torch
    payload = torch.from_numpy(np.ascontiguousarray(keys)).to(device)
    out = [torch.empty_like(payload) for _ in range(dist.get_world_size())]
    dist.all_gather(out, payload)
    return [o.cpu().numpy() for o in out]


def all_gather_blob(dist, mine, device="cpu"):
    """Every rank's byte blob (sizes differ): the sizes, then one all-gather padded to the largest."""
    import torch
    world = dist.get_world_size()
    sizes = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([len(mine)], dtype=torch.int64, device=device))
    sizes = [int(s.item()) for s in sizes]; cap = max(max(sizes), 1)
    pad = np.zeros(cap, np.uint8); pad[: len(mine)] = mine
    bufs = [torch.empty(cap, dtype=torch.uint8, device=device) for _ in range(world)]
    dist.all_gather(bufs, torch.from_numpy(pad).to(device))
    return [b.cpu().numpy()[: sizes[i]].copy() for i, b in enumerate(bufs)]


def exchange_builder(dist, eng, export, globalize, device="cpu"):
    """One build-time exchange between the shards' host builders: this shard's blob from the entry `export`, every shard's blob
    (all_gather_blob), then the entry `globalize` over them, in rank order. Returns the blobs."""
    n = C.c_size_t(0); ex = getattr(eng._host, export); ex.restype = C.c_void_p
    p = ex(C.c_void_p(eng._builder), C.byref(n))
    blobs = all_gather_blob(dist, np.ctypeslib.as_array((C.c_uint8 * n.value).from_address(p)).copy(), device)
    arr = (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])
    rc = getattr(eng._host, globalize)(C.c_void_p(eng._builder), len(blobs), dist.get_rank(), arr)
    if rc:
        raise E.NativeError("%s failed (%d)" % (globalize, rc))
    return blobs


def shard_ranges(n_docs, world):
    """Contiguous doc-id ranges on 65 536-document boundaries (every shard non-empty when n_docs >= world * 65 536)."""
    nc = (n_docs + CONTAINER - 1) // CONTAINER
    cuts = [min(n_docs, ((nc * r) // world) * CONTAINER) for r in range(world)] + [n_docs]
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


class ShardedSearchEngine:
    """SearchEngine over one doc-id-range shard per rank. `device`: "cuda" (NCCL) or "cpu" (gloo + the kernel emulation, tests only)."""

    def __init__(self, dist, device_index=0, _gpu_lib=None, synonymMap=None):
        import torch
        self.dist, self.torch = dist, torch
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.eng = E.SearchEngine(device=device_index, _gpu_lib=_gpu_lib, synonymMap=synonymMap)      # every shard's builder gets the map's table
        self.dev = torch.device("cpu") if _gpu_lib else torch.device("cuda", device_index)
        self.exchange_ms = {"fuzzy_df": 0.0, "stage1": 0.0, "final": 0.0}
        self.host_ms = {}          # wall time of the phased C-ABI calls of this rank (kernels + their host side), download, merge pieces

    # ---- build -------------------------------------------------------------------------------------------------------------------------
    def IndexShard(self, keys, schema, columns, threads=None):
        """`keys` / `columns`: this rank's document range only (ranks in doc order)."""
        eng, dist = self.eng, self.dist
        eng.IndexColumns(keys, schema, columns, threads=threads, upload=False)
        exchange_builder(dist, eng, "ifx_builder_export_stats", "ifx_builder_globalize", self.dev)
        # document lengths after the corpus-level stop terms were dropped -> avgdl (one sequential float sum, as the reference)
        cnt = C.c_int(0); eng._host.ifx_builder_doc_lengths.restype = C.c_void_p
        lp = eng._host.ifx_builder_doc_lengths(C.c_void_p(eng._builder), C.byref(cnt))
        mine = np.ctypeslib.as_array((C.c_float * max(cnt.value, 1)).from_address(lp))[: cnt.value].copy()
        lens = [b.view(np.float32) for b in all_gather_blob(dist, mine.view(np.uint8), self.dev)]
        larr = (C.c_void_p * self.world)(*[x.ctypes.data for x in lens]); carr = (C.c_int * self.world)(*[len(x) for x in lens])
        eng._host.ifx_builder_set_global_lengths(C.c_void_p(eng._builder), self.world, larr, carr)
        exchange_builder(dist, eng, "ifx_builder_export_champions", "ifx_builder_globalize_champions", self.dev)      # the one-character queries' champion lists
        exchange_builder(dist, eng, "ifx_builder_export_columns", "ifx_builder_globalize_columns", self.dev)          # a value id means the same on every shard
        colf = [f for f in schema if f.Filterable or f.Facetable or getattr(f, "Sortable", False)]      # the image's columns, schema order
        self._fcols = [c for c, f in enumerate(colf) if f.Facetable]
        eng._upload(eng._host.ifx_builder_image(C.c_void_p(eng._builder)))

    # ---- search ------------------------------------------------------------------------------------------------------------------------
    def UploadBatch(self, queries):
        """Marshal + upload a batch once (bench `value`: inputs resident in HBM before the timed region); run it with SearchBatch(uploaded=...)."""
        eng = self.eng; packed = eng.PackBatch(queries); h = C.c_void_p()
        eng._check(eng._gpu.ifx_batch_upload(eng._index, packed["arr"], len(queries), C.byref(h)), "ifx_batch_upload")
        self._setup_handle(h, packed)
        return {"packed": packed, "h": h, "queries": queries}

    def _setup_handle(self, h, packed):
        """The batch's facet capacity, and its boosts / SortBy (a refill clears them), which the device flags IFX_Q_UNSUPPORTED_OP on shards."""
        eng = self.eng
        eng._check(eng._gpu.ifx_batch_set_facet_cap(h, packed["out"].facet_cap), "ifx_batch_set_facet_cap")
        if packed["post"] is not None:
            eng._check(eng._gpu.ifx_batch_set_post(h, packed["post"]), "ifx_batch_set_post")

    def FreeBatch(self, up):
        self.eng._gpu.ifx_batch_free(up["h"])

    def Close(self):
        """Release the batch handle SearchBatch keeps between calls (must happen before the index is destroyed)."""
        h = getattr(self, "_cached_h", None)
        if h is not None:
            self.eng._gpu.ifx_batch_free(h); self._cached_h = None

    def SearchBatch(self, queries, stats=None, raw=False, uploaded=None, packed=None):
        """Every rank passes the SAME queries; every rank returns the same merged Results (Records, TotalCandidates, Facets by string)."""
        eng, torch, dist, g = self.eng, self.torch, self.dist, self.eng._gpu
        if uploaded is not None:
            queries = uploaded["queries"]
        cap = max(1, max(q.MaxNumberOfRecordsToReturn for q in queries)); nq = len(queries); K = max(max(q.CoverageDepth for q in queries), min(cap, 1024))      # row length of the Stage-1 lists
        if uploaded is not None:
            packed, h = uploaded["packed"], uploaded["h"]
        else:
            packed = packed or eng.PackBatch(queries); h = getattr(self, "_cached_h", None)      # `packed`: host-side marshalling done beforehand (what the C# shim's pinned buffers are)
            if h is not None and g.ifx_batch_refill(h, packed["arr"], nq) != 0:      # the handle of the previous call is reused (no device allocation per batch), like ifx_search_batch does
                g.ifx_batch_free(h); h = None
            if h is None:
                h = C.c_void_p(); eng._check(g.ifx_batch_upload(eng._index, packed["arr"], nq, C.byref(h)), "ifx_batch_upload")
            self._cached_h = h
            self._setup_handle(h, packed)
        st = stats if stats is not None else E.Stats()

        def phase(k):
            with self._timed(self.host_ms, "phase%d" % k):
                eng._check(g.ifx_batch_run_phase(h, k, C.byref(st)), "phase %d" % k)
        try:
            phase(1)
            self._round(h, "fuzzy_df", g.ifx_batch_fuzzy_df, nq * 16)
            phase(2)
            self._round(h, "select_counts", g.ifx_batch_select_counts, nq * 40)
            phase(3)
            kind = self._short_queries(h, nq)
            with self._timed(self.exchange_ms, "stage1"):
                key = torch.zeros(nq * K, dtype=torch.int64, device=self.dev); score = torch.zeros(nq * K, dtype=torch.float32, device=self.dev); n = torch.zeros(nq, dtype=torch.int32, device=self.dev)
                eng._check(g.ifx_batch_stage1_lists(h, C.c_void_p(key.data_ptr()), C.c_void_p(score.data_ptr()), C.c_void_p(n.data_ptr())), "stage1 lists")
                W = self.world
                ks = [torch.empty_like(key) for _ in range(W)]; ss = [torch.empty_like(score) for _ in range(W)]; ns = [torch.empty_like(n) for _ in range(W)]
                dist.all_gather(ks, key); dist.all_gather(ss, score); dist.all_gather(ns, n)
                self.last_s1_counts = ns          # every shard's Stage-1 list lengths of the last batch ([W] tensors of [nq]; diagnostics, tests)
                # the global list is cut where the unsharded one is: an n-gram query's at its CoverageDepth (the row length K may be longer when
                # another query's max_results is), a short query's at max_results when it is one character or is_short3
                lim = torch.tensor([q.CoverageDepth for q in queries], dtype=torch.int64, device=self.dev).clamp(max=K)
                if kind is not None:
                    mx = torch.tensor([q.MaxNumberOfRecordsToReturn for q in queries], dtype=torch.int64, device=self.dev).clamp(max=K)
                    kd = torch.from_numpy(kind).to(self.dev)
                    lim = torch.where(kd == 0, lim, torch.where(((kd & 3) == 1) | ((kd & 4) != 0), mx, torch.full_like(mx, K)))
                keep, gmax, nglob = self._global_cut(ks, ss, ns, nq, K, lim)
                self._keep, self._gmax = keep, gmax          # borrowed by the library until the last phase has run
                eng._check(g.ifx_batch_stage1_restrict(h, C.c_void_p(keep.data_ptr()), C.c_void_p(gmax.data_ptr()), C.c_void_p(nglob.data_ptr())), "stage1 restrict"); self._sync()
            phase(4)
            with self._timed(self.exchange_ms, "wm"):
                wc = torch.zeros(nq * 4, dtype=torch.int32, device=self.dev)
                eng._check(g.ifx_batch_wm_counts(h, C.c_void_p(wc.data_ptr())), "wm counts")
                wcs = [torch.empty_like(wc) for _ in range(W)]; dist.all_gather(wcs, wc)
                WC = torch.stack([x.view(nq, 4) for x in wcs], 1)                                # [nq, W, 4]
                depth = torch.tensor([q.CoverageDepth for q in queries], dtype=torch.int32, device=self.dev)
                limit = (depth - WC[:, :, 0].sum(1)).clamp(min=0)                                 # wmLimit = coverageDepth - overlap over all shards
                before = torch.cumsum(WC[:, :, 1], 1) - WC[:, :, 1]                               # WordMatcher-only documents of the lower shards come first (ascending ids)
                allowed = (limit.view(nq, 1) - before).clamp(min=0)[:, self.rank].to(torch.int32).contiguous()
                anyg = (WC[:, :, 2].sum(1) > 0).to(torch.int32).contiguous()
                eng._check(g.ifx_batch_wm_apply(h, C.c_void_p(allowed.data_ptr()), C.c_void_p(anyg.data_ptr())), "wm apply"); self._sync()
            if kind is not None:      # short queries: coverage word hits over all shards decide the fallback to the Stage-1 list on every shard alike
                self._round(h, "short", g.ifx_batch_short_hits, nq, dist.ReduceOp.MAX)
            phase(5)
            with self._timed(self.host_ms, "download"):
                eng._check(g.ifx_batch_download(h, C.byref(packed["out"])), "ifx_batch_download")
                info = np.zeros((nq, 8), np.int32); dkey = np.zeros((nq, 2), np.int64)
                eng._check(g.ifx_batch_shard_info(h, E._p(info), E._p(dkey)), "shard info")
                packed["bufs"]["info"], packed["bufs"]["dkey"] = info, dkey
                post = None
                if any(q.Filter is not None or q.EnableFacets for q in queries):      # per record: filter outcome and facet value ids, gathered as they are
                    post = torch.empty((nq, cap, 1 + len(self._fcols)), dtype=torch.int32, device=self.dev)
                    eng._check(g.ifx_batch_shard_records(h, C.c_void_p(post.data_ptr()), post.shape[2]), "shard records")
            with self._timed(self.exchange_ms, "final"):
                merged = self._merge(queries, packed["bufs"], cap, post, h)
        except Exception:
            if uploaded is None:
                g.ifx_batch_free(h); self._cached_h = None
            raise
        return merged if raw else self._results(queries, merged)

    def _results(self, queries, merged):
        """The Results (facets by string) of SearchBatch(raw=True)'s merged buffers."""
        return self.eng._results(queries, *merged)

    def _sync(self):
        if self.dev.type == "cuda":
            self.torch.cuda.synchronize(self.dev)

    @contextlib.contextmanager
    def _timed(self, acc, name):
        """Adds the wall time of the block to acc[name] (ms)."""
        t0 = time.perf_counter()
        yield
        acc[name] = acc.get(name, 0.0) + 1e3 * (time.perf_counter() - t0)

    def _round(self, h, name, entry, n, op=None):
        """One per-batch round: `entry` gets n int32 per shard into a device tensor, the hosts all-reduce it (sum unless `op`), `entry` sets it."""
        with self._timed(self.exchange_ms, name):
            buf = self.torch.zeros(n, dtype=self.torch.int32, device=self.dev); ptr = C.c_void_p(buf.data_ptr())
            self.eng._check(entry(h, ptr, 0), "%s get" % name)
            self.dist.all_reduce(buf, op=self.dist.ReduceOp.SUM if op is None else op)
            self.eng._check(entry(h, ptr, 1), "%s set" % name); self._sync()

    def _short_queries(self, h, nq):
        """The short queries of the batch (no word of >= 3 characters), group by group: matched documents summed over the shards (fuzzy
        fallback below 100), then the largest integer score (BuildFinalScores). Returns the per-query kinds, or None when there is none --
        the device counts them from the texts, so every rank takes the same branch."""
        eng, torch, dist, g = self.eng, self.torch, self.dist, self.eng._gpu
        ng = C.c_int(0); gs = C.c_int(0); kind = np.zeros(nq, np.int32)
        eng._check(g.ifx_batch_short_groups(h, E._p(kind), C.byref(ng), C.byref(gs)), "short groups")
        if ng.value == 0:
            return None
        with self._timed(self.exchange_ms, "short"):
            buf = torch.zeros(gs.value, dtype=torch.int32, device=self.dev); ptr = C.c_void_p(buf.data_ptr())
            for grp in range(ng.value):
                eng._check(g.ifx_batch_short_step(h, 0, grp, ptr), "short step 0"); dist.all_reduce(buf)
                eng._check(g.ifx_batch_short_step(h, 1, grp, ptr), "short step 1"); dist.all_reduce(buf, op=dist.ReduceOp.MAX)
                eng._check(g.ifx_batch_short_step(h, 2, grp, ptr), "short step 2")
        return kind

    def _global_cut(self, ks, ss, ns, nq, K, lim=None):
        """Membership of this rank's Stage-1 entries in the global top-K by (score desc, key asc), and the global top score per query.
        Every shard's list is already in that order, so an entry's global rank is its local rank plus, per other shard, the number of
        entries ahead of it -- W - 1 binary searches over packed (score bits, inverted key) words instead of a sort of all W * K entries.
        `lim` ([nq]): the global list length of every query (its CoverageDepth; short queries may be cut at max_results); None: K for all."""
        torch = self.torch; W = self.world; dev = ss[0].device
        if lim is None:
            lim = torch.full((nq,), K, dtype=torch.int64, device=dev)
        N = torch.stack(ns, 1).clamp(min=0, max=K)                                             # [nq, W]
        slot = torch.arange(K, device=dev).view(1, K)
        big = torch.iinfo(torch.int64).max
        negc = []
        fits = True
        for r in range(W):
            k = ks[r].view(nq, K); v = slot < N[:, r].view(nq, 1)
            if not bool((((k >= 0) & (k < 2 ** 32)) | ~v).all()):
                fits = False; break
            comp = (ss[r].view(nq, K).view(torch.int32).to(torch.int64) << 32) | (0xFFFFFFFF - k)      # larger = earlier in the list order
            negc.append(torch.where(v, -comp, torch.full_like(comp, big)).contiguous())           # ascending along the list; invalid slots last
        if not fits:
            return self._global_cut_sort(ks, ss, ns, nq, K, lim)
        mine = negc[self.rank]; grank = slot.expand(nq, K).clone()
        for o in range(W):
            if o != self.rank:
                grank += torch.searchsorted(negc[o], mine, right=False)
        valid = slot < N[:, self.rank].view(nq, 1)
        keep = torch.where(valid & (grank < lim.view(nq, 1)), torch.where(grank == 0, 2, torch.where(grank == 1, 3, 1)), 0).to(torch.uint8).contiguous().view(-1)      # 2 / 3: global rank 0 / 1 (docIndex 0 / 1)
        first = torch.stack([torch.where(N[:, r] > 0, ss[r].view(nq, K)[:, 0], torch.zeros((), dtype=ss[r].dtype, device=dev)) for r in range(W)], 1)
        gmax = first.max(dim=1).values.clamp(min=0).contiguous()
        nglob = torch.minimum(N.sum(1), lim).to(torch.int32).contiguous()
        return keep, gmax, nglob

    def _global_cut_sort(self, ks, ss, ns, nq, K, lim=None):
        """General form (keys beyond 32 bits): two stable sorts over all W * K entries."""
        torch = self.torch; W = self.world
        if lim is None:
            lim = torch.full((nq,), K, dtype=torch.int64, device=ss[0].device)
        S = torch.stack([s.view(nq, K) for s in ss], 1).reshape(nq, W * K); Kk = torch.stack([k.view(nq, K) for k in ks], 1).reshape(nq, W * K)
        N = torch.stack(ns, 1).clamp(min=0)                                                    # [nq, W]
        slot = torch.arange(K, device=S.device).view(1, 1, K).expand(nq, W, K)
        valid = (slot < N.view(nq, W, 1)).reshape(nq, W * K)
        S = torch.where(valid, S, torch.full_like(S, -1.0)); Kk = torch.where(valid, Kk, torch.full_like(Kk, 2 ** 62))
        i1 = torch.argsort(Kk, dim=1, stable=True); S1 = torch.gather(S, 1, i1)
        i2 = torch.argsort(S1, dim=1, descending=True, stable=True)
        order = torch.gather(i1, 1, i2)[:, :K]                                                 # flat positions of the global top-K
        top_valid = torch.gather(valid, 1, order)
        top_valid = top_valid & (torch.arange(K, device=S.device).view(1, K) < lim.view(nq, 1))
        mark = torch.zeros(nq, W * K, dtype=torch.uint8, device=S.device)
        flag = top_valid.to(torch.uint8); flag[:, 0] *= 2                                     # 2: global rank 0, 3: global rank 1 (docIndex 0 / 1)
        if K > 1:
            flag[:, 1] *= 3
        mark.scatter_(1, order, flag)
        keep = mark.view(nq, W, K)[:, self.rank, :].contiguous().view(-1)
        gmax = S.max(dim=1).values.clamp(min=0).contiguous()
        nglob = torch.minimum(valid.sum(1), lim).to(torch.int32).contiguous()
        return keep, gmax, nglob

    def _merge(self, queries, bufs, cap, post=None, h=None):
        """All-gather of every shard's records; merged by ScoreEntry order (Score desc, Tiebreaker desc, DocumentId asc), truncated
        (CalculateTruncationIndex), filtered, and the facet table built over what is left -- the order of SearchEngine.Search.
        `post` ([nq, cap, 1 + facetable columns], device): per record of this shard its filter outcome and facet value ids, or None when no
        query filters or counts facets. `h`: the batch handle (its device entry builds the facet tables)."""
        torch, dist, W = self.torch, self.dist, self.world
        nq = len(queries); eng = self.eng
        with self._timed(self.host_ms, "merge_pack"):
            rec = np.zeros((nq, cap, 3), np.float64)          # key, score bits (exact in f64), tie
            rec[:, :, 0] = bufs["keys"]; rec[:, :, 1] = bufs["scores"].view(np.uint32).astype(np.float64); rec[:, :, 2] = bufs["ties"]
            meta = np.concatenate([np.stack([bufs["n"], bufs["total"], bufs["status"], bufs["nf"]], 1).astype(np.int64), bufs["info"].astype(np.int64), bufs["dkey"]], 1)      # [nq, 4 + 8 + 2]
            t_rec = torch.from_numpy(rec).to(self.dev); t_meta = torch.from_numpy(meta).to(self.dev)
            recs = [torch.empty_like(t_rec) for _ in range(W)]; metas = [torch.empty_like(t_meta) for _ in range(W)]
            fq = np.array([q.EnableFacets for q in queries]); facets = bool(fq.any())
        with self._timed(self.host_ms, "merge_gather"):
            dist.all_gather(recs, t_rec); dist.all_gather(metas, t_meta)
            if post is not None:
                posts = [torch.empty_like(post) for _ in range(W)]; dist.all_gather(posts, post)
            M = torch.stack(metas, 1)                                                                                                    # [nq, W, 14]
            # a query answered with its WHOLE Stage-1 list (shard_info[6] == -1) was filtered on the shards: TotalCandidates and facet rows are summed
            lst = (M[:, :, 10] == -1).cpu().numpy(); whole = lst.any(1)
            sel = np.nonzero(whole & fq)[0]          # the same on every rank (from the gathered facts): each shard's facet rows of those queries
            if len(sel):
                fr = np.stack([bufs["fcol"][sel], bufs["fval"][sel], np.where(np.arange(bufs["fcnt"].shape[1])[None, :] < bufs["nf"][sel, None], bufs["fcnt"][sel], 0)], 2).astype(np.int32)
                mine = torch.from_numpy(np.ascontiguousarray(fr)).to(self.dev); srows = [torch.empty_like(mine) for _ in range(W)]; dist.all_gather(srows, mine)
            self._sync()
        with self._timed(self.host_ms, "merge_sort_cut"):
            # merge on the device: ScoreEntry order (Score desc, Tiebreaker desc, DocumentId asc) = three stable sorts, least significant key first
            R = torch.stack(recs, 1).reshape(nq, W * cap, 3)                                                                             # [nq, W*cap, 3]
            valid = (torch.arange(cap, device=self.dev).view(1, 1, cap) < M[:, :, 0:1]).reshape(nq, W * cap)
            key = R[:, :, 0].to(torch.int64); sbits = R[:, :, 1].to(torch.int64); tie = R[:, :, 2].to(torch.int64)
            score = torch.where(valid, sbits.to(torch.int32).view(torch.float32).to(torch.float64), torch.full((), float("-inf"), dtype=torch.float64, device=self.dev))
            o1 = torch.argsort(key, dim=1, stable=True)
            o2 = torch.gather(o1, 1, torch.argsort(torch.gather(-tie, 1, o1), dim=1, stable=True))
            order = torch.gather(o2, 1, torch.argsort(torch.gather(-score, 1, o2), dim=1, stable=True))[:, :cap]
            # the blank query with EnableFacets (shard_info[6] == -2) browses the corpus in internal-id order: the shards' records in shard order
            browse = (M[:, :, 10] == -2).any(1)
            if bool(browse.any()):
                order = torch.where(browse.view(nq, 1), torch.argsort((~valid).to(torch.int8), dim=1, stable=True)[:, :cap], order)
            t_key = torch.gather(key, 1, order); t_sbits = torch.gather(sbits, 1, order); t_tie = torch.gather(tie, 1, order); nvalid = valid.sum(1)
            maxr = torch.tensor([q.MaxNumberOfRecordsToReturn for q in queries], dtype=torch.int64, device=self.dev)
            # ResultProcessor.CalculateTruncationIndex over the merged list: the last record with Score >= 254 (records are sorted: the first n_ge),
            # or a docIndex-0/1 document whose word hits reach max(1, max word hits over all shards) or whose lcs is non-zero
            info = M[:, :, 4:12]; dk = M[:, :, 12:14]
            min_hits = info[:, :, 0].max(1).values.clamp(min=1); trunc = info[:, :, 1].sum(1) - 1
            pos_idx = torch.arange(cap, device=self.dev).view(1, cap)
            for j in range(2):
                wh = info[:, :, 2 + 2 * j].max(1).values; lc = info[:, :, 3 + 2 * j].max(1).values; dkj = dk[:, :, j].max(1).values      # the owner reports >= 0, the others -1
                qual = (wh >= 0) & ((wh >= min_hits) | (lc > 0))
                hit = (t_key == dkj.view(nq, 1)) & (pos_idx < nvalid.clamp(max=cap).view(nq, 1))
                pos = torch.where(hit.any(1), hit.to(torch.int64).argmax(1), torch.full((), cap, dtype=torch.int64, device=self.dev))      # beyond the merged top: at least `cap`
                trunc = torch.where(qual, torch.maximum(trunc, pos), trunc)
            count = torch.where(trunc < 0, maxr, torch.minimum(trunc + 1, maxr))
            t_n = torch.minimum(torch.minimum(nvalid, count), maxr)
            status_t = M[:, 0, 2].clone()
            for r in range(1, W):
                status_t |= M[:, r, 2]
            P = None
            if post is not None:      # ApplyFilter after the truncation: the records that fail leave, TotalCandidates counts the rest (Take(max) is then a no-op)
                S = post.shape[2]
                P = torch.gather(torch.stack(posts, 1).reshape(nq, W * cap, S), 1, order.unsqueeze(2).expand(nq, cap, S))
                kept = (P[:, :, 0] == 1) & (pos_idx < t_n.view(nq, 1))
                ko = torch.argsort((~kept).to(torch.int8), dim=1, stable=True)
                t_key = torch.gather(t_key, 1, ko); t_sbits = torch.gather(t_sbits, 1, ko); t_tie = torch.gather(t_tie, 1, ko); P = torch.gather(P, 1, ko.unsqueeze(2).expand(nq, cap, S))
                t_n = kept.sum(1)
            o_key = t_key.cpu().numpy(); o_score = t_sbits.to(torch.int32).cpu().numpy().view(np.float32); o_tie = t_tie.to(torch.uint8).cpu().numpy(); o_n = t_n.cpu().numpy()
            total = np.where(browse.cpu().numpy(), 0, o_n)          # (TotalCandidates is not set on the browse path)
        with self._timed(self.host_ms, "merge_facets"):
            self.last_shard_info = M[:, :, 4:12]          # every shard's truncation facts of the last batch ([nq, W, 8]; diagnostics, tests)
            total = np.where(whole, M[:, :, 1].sum(1).cpu().numpy(), total)      # TotalCandidates counts the whole list
            facet_out = None
            if facets:      # FacetBuilder over the records kept (one row per record and facetable column), or the summed rows of a whole Stage-1 list
                nfc = len(self._fcols); fc = max(int(bufs["fcol"].shape[1]), 1)
                cols = torch.tensor(self._fcols, dtype=torch.int32, device=self.dev).view(1, 1, nfc).expand(nq, cap, nfc)
                ids = P[:, :, 1:]; cnt = ((pos_idx < t_n.view(nq, 1)).view(nq, cap, 1) & (ids >= 0)).to(torch.int32)
                rows = torch.stack([cols, ids, cnt], 3).reshape(nq, cap * nfc, 3)
                if len(sel):
                    sr = torch.stack(srows, 1).reshape(len(sel), W * mine.shape[1], 3); m = max(rows.shape[1], sr.shape[1])
                    rows = torch.nn.functional.pad(rows, (0, 0, 0, m - rows.shape[1])).clone()
                    rows[torch.from_numpy(sel).to(self.dev)] = torch.nn.functional.pad(sr, (0, 0, 0, m - sr.shape[1]))
                rows = rows.contiguous(); m = rows.shape[1]
                f_col = torch.zeros((nq, fc), dtype=torch.int32, device=self.dev); f_val = torch.zeros_like(f_col); f_cnt = torch.zeros_like(f_col)
                f_n = torch.zeros(nq, dtype=torch.int32, device=self.dev); st32 = status_t.to(torch.int32).contiguous()
                p_ = lambda t: C.c_void_p(t.data_ptr())
                eng._check(eng._gpu.ifx_batch_facet_table(h, p_(rows), m, p_(f_col), p_(f_val), p_(f_cnt), p_(f_n), p_(st32)), "ifx_batch_facet_table")
                status_t = st32.to(torch.int64)
                facet_out = (f_col.cpu().numpy(), f_val.cpu().numpy(), f_cnt.cpu().numpy(), f_n.cpu().numpy())
            status = status_t.cpu().numpy()
            status = np.where(whole & ~lst.all(1), status | 2, status)      # shards that disagree on the answer's kind: flagged, never mixed
        self.last_raw = (o_key, o_score, o_tie, o_n, total, status)
        return o_key, o_score, o_tie, o_n, total, status, facet_out

