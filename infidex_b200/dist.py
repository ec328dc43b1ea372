"""Doc-id-range sharding of ONE index over the ranks of a torch.distributed job (one process per GPU; NCCL on GPUs, gloo in the CPU tests).

Layout (SURVEY.md 8e, DESIGN.md "multi-GPU"): rank r indexes the contiguous document range [r*N/R, (r+1)*N/R) rounded to multiples of
65 536 (the reference's container size, so no 4096-chunk of Bm25Scorer is ever split). The statistics the search path reads as global
quantities -- term ordinals, df / idf, N, avgdl, word idf, prefix-set cardinalities, the affix dictionary -- are exchanged once at build
time (ifx_builder_export_stats -> all_gather -> ifx_builder_globalize). Every batch then runs on every shard, with three exchanges:
    all-reduce(sum)  document frequency of every LD1 union (its idf is a corpus-level quantity)                 16 int32 per query
    all-gather       per-shard Stage-1 top-`depth` (key, score): global cut + global top score (normBm25)      depth * 12 B per query and shard
    all-gather       per-shard final records (key, score, tie, counts, facet rows): merged identically on every rank
What is NOT exchanged (counted, never hidden -- `parity` in the bench line is the number of sampled queries whose merged records differ
from the unsharded oracle): the selector's tier rules and the MaxScore threshold chain run on shard-local counts / heaps, the WordMatcher
quota, docIndex-0/1 rule and truncation index are evaluated per shard.
"""
import ctypes as C
import os

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


def shard_ranges(n_docs, world):
    """Contiguous doc-id ranges on 65 536-document boundaries (every shard non-empty when n_docs >= world * 65 536)."""
    nc = (n_docs + CONTAINER - 1) // CONTAINER
    cuts = [min(n_docs, ((nc * r) // world) * CONTAINER) for r in range(world)] + [n_docs]
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


class ShardedSearchEngine:
    """SearchEngine over one doc-id-range shard per rank. `device`: "cuda" (NCCL) or "cpu" (gloo + the kernel emulation, tests only)."""

    def __init__(self, dist, device_index=0, _gpu_lib=None):
        import torch
        self.dist, self.torch = dist, torch
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.eng = E.SearchEngine(device=device_index, _gpu_lib=_gpu_lib)
        self.dev = torch.device("cpu") if _gpu_lib else torch.device("cuda", device_index)
        self.exchange_ms = {"fuzzy_df": 0.0, "stage1": 0.0, "final": 0.0}
        self.host_ms = {}          # wall time of the phased C-ABI calls of this rank (kernels + their host side), download, merge pieces

    # ---- build -------------------------------------------------------------------------------------------------------------------------
    def IndexShard(self, keys, schema, columns, threads=None):
        """`keys` / `columns`: this rank's document range only (ranks in doc order)."""
        eng, torch, dist = self.eng, self.torch, self.dist
        eng.IndexColumns(keys, schema, columns, threads=threads, upload=False)
        n = C.c_size_t(0)
        eng._host.ifx_builder_export_stats.restype = C.c_void_p
        p = eng._host.ifx_builder_export_stats(C.c_void_p(eng._builder), C.byref(n))
        mine = np.ctypeslib.as_array((C.c_uint8 * n.value).from_address(p)).copy()
        sizes = [torch.zeros(1, dtype=torch.int64, device=self.dev) for _ in range(self.world)]
        dist.all_gather(sizes, torch.tensor([len(mine)], dtype=torch.int64, device=self.dev))
        sizes = [int(s.item()) for s in sizes]; cap = max(sizes)
        pad = np.zeros(cap, np.uint8); pad[: len(mine)] = mine
        bufs = [torch.empty(cap, dtype=torch.uint8, device=self.dev) for _ in range(self.world)]
        dist.all_gather(bufs, torch.from_numpy(pad).to(self.dev))
        blobs = [b.cpu().numpy()[: sizes[i]].copy() for i, b in enumerate(bufs)]
        arr = (C.c_void_p * self.world)(*[bl.ctypes.data for bl in blobs])
        rc = eng._host.ifx_builder_globalize(C.c_void_p(eng._builder), self.world, self.rank, arr)
        if rc:
            raise E.NativeError("ifx_builder_globalize failed (%d)" % rc)
        # second exchange: document lengths after the corpus-level stop terms were dropped -> avgdl (one sequential float sum, as the reference)
        cnt = C.c_int(0); eng._host.ifx_builder_doc_lengths.restype = C.c_void_p
        lp = eng._host.ifx_builder_doc_lengths(C.c_void_p(eng._builder), C.byref(cnt))
        mine_l = np.ctypeslib.as_array((C.c_float * max(cnt.value, 1)).from_address(lp))[: cnt.value].copy()
        nsz = [torch.zeros(1, dtype=torch.int64, device=self.dev) for _ in range(self.world)]
        dist.all_gather(nsz, torch.tensor([cnt.value], dtype=torch.int64, device=self.dev)); nsz = [int(x.item()) for x in nsz]; capl = max(max(nsz), 1)
        padl = np.zeros(capl, np.float32); padl[: cnt.value] = mine_l
        lb = [torch.empty(capl, dtype=torch.float32, device=self.dev) for _ in range(self.world)]
        dist.all_gather(lb, torch.from_numpy(padl).to(self.dev))
        lens = [np.ascontiguousarray(x.cpu().numpy()[: nsz[i]]) for i, x in enumerate(lb)]
        larr = (C.c_void_p * self.world)(*[x.ctypes.data for x in lens]); carr = (C.c_int * self.world)(*nsz)
        eng._host.ifx_builder_set_global_lengths(C.c_void_p(eng._builder), self.world, larr, carr)
        eng._upload(eng._host.ifx_builder_image(C.c_void_p(eng._builder)))

    # ---- search ------------------------------------------------------------------------------------------------------------------------
    def UploadBatch(self, queries):
        """Marshal + upload a batch once (bench `value`: inputs resident in HBM before the timed region); run it with SearchBatch(uploaded=...)."""
        eng = self.eng; packed = eng.PackBatch(queries); h = C.c_void_p()
        eng._check(eng._gpu.ifx_batch_upload(eng._index, packed["arr"], len(queries), C.byref(h)), "ifx_batch_upload")
        if packed["post"] is not None:      # boosts / SortBy on shards: the device flags those queries IFX_Q_UNSUPPORTED_OP
            eng._check(eng._gpu.ifx_batch_set_post(h, packed["post"]), "ifx_batch_set_post")
        return {"packed": packed, "h": h, "queries": queries}

    def FreeBatch(self, up):
        self.eng._gpu.ifx_batch_free(up["h"])

    def Close(self):
        """Release the batch handle SearchBatch keeps between calls (must happen before the index is destroyed)."""
        h = getattr(self, "_cached_h", None)
        if h is not None:
            self.eng._gpu.ifx_batch_free(h); self._cached_h = None

    def SearchBatch(self, queries, stats=None, raw=False, uploaded=None, packed=None):
        """Every rank passes the SAME queries; every rank returns the same merged Results (Records, TotalCandidates, Facets by string)."""
        import time
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
            if packed.get("post") is not None:      # (a refill clears it) boosts / SortBy on shards: flagged IFX_Q_UNSUPPORTED_OP by the device
                eng._check(g.ifx_batch_set_post(h, packed["post"]), "ifx_batch_set_post")
        st = stats if stats is not None else E.Stats()

        def sync():
            if self.dev.type == "cuda":
                torch.cuda.synchronize(self.dev)
        try:
            tp = time.perf_counter(); eng._check(g.ifx_batch_run_phase(h, 1, C.byref(st)), "phase 1"); self._acc("phase1", tp)
            t0 = time.perf_counter()
            fdf = torch.zeros(nq * 16, dtype=torch.int32, device=self.dev)
            eng._check(g.ifx_batch_fuzzy_df(h, C.c_void_p(fdf.data_ptr()), 0), "fuzzy df get")
            dist.all_reduce(fdf)
            eng._check(g.ifx_batch_fuzzy_df(h, C.c_void_p(fdf.data_ptr()), 1), "fuzzy df set"); sync()
            self.exchange_ms["fuzzy_df"] += 1e3 * (time.perf_counter() - t0)
            tp = time.perf_counter(); eng._check(g.ifx_batch_run_phase(h, 2, C.byref(st)), "phase 2"); self._acc("phase2", tp)
            t0 = time.perf_counter()
            sc = torch.zeros(nq * 40, dtype=torch.int32, device=self.dev)
            eng._check(g.ifx_batch_select_counts(h, C.c_void_p(sc.data_ptr()), 0), "select counts get")
            dist.all_reduce(sc)
            eng._check(g.ifx_batch_select_counts(h, C.c_void_p(sc.data_ptr()), 1), "select counts set"); sync()
            self.exchange_ms["select_counts"] = self.exchange_ms.get("select_counts", 0.0) + 1e3 * (time.perf_counter() - t0)
            tp = time.perf_counter(); eng._check(g.ifx_batch_run_phase(h, 3, C.byref(st)), "phase 3"); self._acc("phase3", tp)
            t0 = time.perf_counter()
            key = torch.zeros(nq * K, dtype=torch.int64, device=self.dev); score = torch.zeros(nq * K, dtype=torch.float32, device=self.dev); n = torch.zeros(nq, dtype=torch.int32, device=self.dev)
            eng._check(g.ifx_batch_stage1_lists(h, C.c_void_p(key.data_ptr()), C.c_void_p(score.data_ptr()), C.c_void_p(n.data_ptr())), "stage1 lists")
            W = self.world
            ks = [torch.empty_like(key) for _ in range(W)]; ss = [torch.empty_like(score) for _ in range(W)]; ns = [torch.empty_like(n) for _ in range(W)]
            dist.all_gather(ks, key); dist.all_gather(ss, score); dist.all_gather(ns, n)
            keep, gmax, nglob = self._global_cut(ks, ss, ns, nq, K)
            self._keep, self._gmax = keep, gmax          # borrowed by the library until the last phase has run
            eng._check(g.ifx_batch_stage1_restrict(h, C.c_void_p(keep.data_ptr()), C.c_void_p(gmax.data_ptr()), C.c_void_p(nglob.data_ptr())), "stage1 restrict"); sync()
            self.exchange_ms["stage1"] += 1e3 * (time.perf_counter() - t0)
            tp = time.perf_counter(); eng._check(g.ifx_batch_run_phase(h, 4, C.byref(st)), "phase 4"); self._acc("phase4", tp)
            t0 = time.perf_counter()
            wc = torch.zeros(nq * 4, dtype=torch.int32, device=self.dev)
            eng._check(g.ifx_batch_wm_counts(h, C.c_void_p(wc.data_ptr())), "wm counts")
            wcs = [torch.empty_like(wc) for _ in range(W)]; dist.all_gather(wcs, wc)
            WC = torch.stack([x.view(nq, 4) for x in wcs], 1)                                # [nq, W, 4]
            depth = torch.tensor([q.CoverageDepth for q in queries], dtype=torch.int32, device=self.dev)
            limit = (depth - WC[:, :, 0].sum(1)).clamp(min=0)                                 # wmLimit = coverageDepth - overlap over all shards
            before = torch.cumsum(WC[:, :, 1], 1) - WC[:, :, 1]                               # WordMatcher-only documents of the lower shards come first (ascending ids)
            allowed = (limit.view(nq, 1) - before).clamp(min=0)[:, self.rank].to(torch.int32).contiguous()
            anyg = (WC[:, :, 2].sum(1) > 0).to(torch.int32).contiguous()
            eng._check(g.ifx_batch_wm_apply(h, C.c_void_p(allowed.data_ptr()), C.c_void_p(anyg.data_ptr())), "wm apply"); sync()
            self.exchange_ms["wm"] = self.exchange_ms.get("wm", 0.0) + 1e3 * (time.perf_counter() - t0)
            tp = time.perf_counter(); eng._check(g.ifx_batch_run_phase(h, 5, C.byref(st)), "phase 5"); self._acc("phase5", tp)
            tp = time.perf_counter(); eng._check(g.ifx_batch_download(h, C.byref(packed["out"])), "ifx_batch_download")
            info = np.zeros((nq, 8), np.int32); dkey = np.zeros((nq, 2), np.int64)
            eng._check(g.ifx_batch_shard_info(h, E._p(info), E._p(dkey)), "shard info")
            packed["bufs"]["info"], packed["bufs"]["dkey"] = info, dkey; self._acc("download", tp)
        except Exception:
            if uploaded is None:
                g.ifx_batch_free(h); self._cached_h = None
            raise
        t0 = time.perf_counter()
        merged = self._merge(queries, packed["bufs"], cap)
        self.exchange_ms["final"] += 1e3 * (time.perf_counter() - t0)
        return merged if raw else self._results(queries, merged)

    def _acc(self, name, t0):
        import time
        self.host_ms[name] = self.host_ms.get(name, 0.0) + 1e3 * (time.perf_counter() - t0)

    def _global_cut(self, ks, ss, ns, nq, K):
        """Membership of this rank's Stage-1 entries in the global top-K by (score desc, key asc), and the global top score per query.
        Every shard's list is already in that order, so an entry's global rank is its local rank plus, per other shard, the number of
        entries ahead of it -- W - 1 binary searches over packed (score bits, inverted key) words instead of a sort of all W * K entries."""
        torch = self.torch; W = self.world; dev = ss[0].device
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
            return self._global_cut_sort(ks, ss, ns, nq, K)
        mine = negc[self.rank]; grank = slot.expand(nq, K).clone()
        for o in range(W):
            if o != self.rank:
                grank += torch.searchsorted(negc[o], mine, right=False)
        valid = slot < N[:, self.rank].view(nq, 1)
        keep = torch.where(valid & (grank < K), torch.where(grank == 0, 2, torch.where(grank == 1, 3, 1)), 0).to(torch.uint8).contiguous().view(-1)      # 2 / 3: global rank 0 / 1 (docIndex 0 / 1)
        first = torch.stack([torch.where(N[:, r] > 0, ss[r].view(nq, K)[:, 0], torch.zeros((), dtype=ss[r].dtype, device=dev)) for r in range(W)], 1)
        gmax = first.max(dim=1).values.clamp(min=0).contiguous()
        nglob = N.sum(1).clamp(max=K).to(torch.int32).contiguous()
        return keep, gmax, nglob

    def _global_cut_sort(self, ks, ss, ns, nq, K):
        """General form (keys beyond 32 bits): two stable sorts over all W * K entries."""
        torch = self.torch; W = self.world
        S = torch.stack([s.view(nq, K) for s in ss], 1).reshape(nq, W * K); Kk = torch.stack([k.view(nq, K) for k in ks], 1).reshape(nq, W * K)
        N = torch.stack(ns, 1).clamp(min=0)                                                    # [nq, W]
        slot = torch.arange(K, device=S.device).view(1, 1, K).expand(nq, W, K)
        valid = (slot < N.view(nq, W, 1)).reshape(nq, W * K)
        S = torch.where(valid, S, torch.full_like(S, -1.0)); Kk = torch.where(valid, Kk, torch.full_like(Kk, 2 ** 62))
        i1 = torch.argsort(Kk, dim=1, stable=True); S1 = torch.gather(S, 1, i1)
        i2 = torch.argsort(S1, dim=1, descending=True, stable=True)
        order = torch.gather(i1, 1, i2)[:, :K]                                                 # flat positions of the global top-K
        top_valid = torch.gather(valid, 1, order)
        mark = torch.zeros(nq, W * K, dtype=torch.uint8, device=S.device)
        flag = top_valid.to(torch.uint8); flag[:, 0] *= 2                                     # 2: global rank 0, 3: global rank 1 (docIndex 0 / 1)
        if K > 1:
            flag[:, 1] *= 3
        mark.scatter_(1, order, flag)
        keep = mark.view(nq, W, K)[:, self.rank, :].contiguous().view(-1)
        gmax = S.max(dim=1).values.clamp(min=0).contiguous()
        nglob = valid.sum(1).clamp(max=K).to(torch.int32).contiguous()
        return keep, gmax, nglob

    def _merge(self, queries, bufs, cap):
        """All-gather of every shard's records; merged by ScoreEntry order (Score desc, Tiebreaker desc, DocumentId asc) and cut to max."""
        torch, dist, W = self.torch, self.dist, self.world
        import time
        nq = len(queries); eng = self.eng; tp = time.perf_counter()
        rec = np.zeros((nq, cap, 3), np.float64)          # key, score bits (exact in f64), tie
        rec[:, :, 0] = bufs["keys"]; rec[:, :, 1] = bufs["scores"].view(np.uint32).astype(np.float64); rec[:, :, 2] = bufs["ties"]
        meta = np.concatenate([np.stack([bufs["n"], bufs["total"], bufs["status"], bufs["nf"]], 1).astype(np.int64), bufs["info"].astype(np.int64), bufs["dkey"]], 1)      # [nq, 4 + 8 + 2]
        t_rec = torch.from_numpy(rec).to(self.dev); t_meta = torch.from_numpy(meta).to(self.dev)
        recs = [torch.empty_like(t_rec) for _ in range(W)]; metas = [torch.empty_like(t_meta) for _ in range(W)]
        self._acc("merge_pack", tp); tp = time.perf_counter()
        dist.all_gather(recs, t_rec); dist.all_gather(metas, t_meta)
        if self.dev.type == "cuda":
            torch.cuda.synchronize(self.dev)
        self._acc("merge_gather", tp); tp = time.perf_counter()
        # merge on the device: ScoreEntry order (Score desc, Tiebreaker desc, DocumentId asc) = three stable sorts, least significant key first
        R = torch.stack(recs, 1).reshape(nq, W * cap, 3); M = torch.stack(metas, 1)                                                   # [nq, W*cap, 3], [nq, W, 14]
        valid = (torch.arange(cap, device=self.dev).view(1, 1, cap) < M[:, :, 0:1]).reshape(nq, W * cap)
        key = R[:, :, 0].to(torch.int64); sbits = R[:, :, 1].to(torch.int64); tie = R[:, :, 2].to(torch.int64)
        score = torch.where(valid, sbits.to(torch.int32).view(torch.float32).to(torch.float64), torch.full((), float("-inf"), dtype=torch.float64, device=self.dev))
        o1 = torch.argsort(key, dim=1, stable=True)
        o2 = torch.gather(o1, 1, torch.argsort(torch.gather(-tie, 1, o1), dim=1, stable=True))
        order = torch.gather(o2, 1, torch.argsort(torch.gather(-score, 1, o2), dim=1, stable=True))[:, :cap]
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
        o_key = t_key.cpu().numpy(); o_score = t_sbits.to(torch.int32).cpu().numpy().view(np.float32); o_tie = t_tie.to(torch.uint8).cpu().numpy(); o_n = t_n.cpu().numpy()
        total = o_n.copy(); status = status_t.cpu().numpy(); self._acc("merge_sort_cut", tp)
        self.last_raw = (o_key, o_score, o_tie, o_n, total, status)
        facets_all = None
        if any(q.EnableFacets for q in queries):          # facet rows travel as strings (value ids are per-shard dictionaries)
            mine = []
            for i in range(nq):
                rows = []
                for k in range(int(bufs["nf"][i])):
                    col = int(bufs["fcol"][i, k]); rows.append((eng._columns[col], eng._facet_value(col, int(bufs["fval"][i, k])), int(bufs["fcnt"][i, k])))
                mine.append(rows)
            facets_all = [None] * W
            dist.all_gather_object(facets_all, mine)
        return o_key, o_score, o_tie, o_n, total, status, facets_all

    def _results(self, queries, merged):
        o_key, o_score, o_tie, o_n, total, status, facets_all = merged; out = []
        for i, q in enumerate(queries):
            records = [E.ScoreEntry(o_score[i, k], o_key[i, k], o_tie[i, k]) for k in range(int(o_n[i]))]
            facets = None
            if q.EnableFacets:
                acc = {}
                for r in range(self.world):
                    for f, v, cnt in facets_all[r][i]:
                        acc.setdefault(f, {}); acc[f][v] = acc[f].get(v, 0) + cnt
                facets = {f: sorted(vs.items(), key=lambda kv: (-kv[1], kv[0].lower(), kv[0]))[:100] for f, vs in acc.items()}
            out.append(E.Result(records, facets, int(total[i]), int(status[i])))
        return out
