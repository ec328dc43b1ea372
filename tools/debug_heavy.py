# Scratch: per-query Stage-1 diagnostics. For the phase columns run with IFX_LIB=<library built with -DIFX_S1_TIMERS>.
import sys, os, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import infidex_b200 as ib
from infidex_b200 import synth
ND = int(os.environ.get("IFX_DBG_DOCS", "1000000")); MULTI = os.environ.get("IFX_DBG_MULTI", "0") == "1"; NQ = int(os.environ.get("IFX_DBG_NQ", "1000"))
vocab = synth.make_vocab(400_000); docs = synth.gen_docs(ND, vocab, with_description=MULTI); qs = synth.gen_queries(NQ, docs, vocab)
schema, cols = synth.schema_and_columns(docs, MULTI)
e = ib.SearchEngine.CreateDefault(_gpu_lib=os.environ.get('IFX_LIB')); e.IndexColumns(docs["keys"], schema, cols)
h = e.UploadBatch([ib.Query(q, 10) for q in qs])
for r in range(3): st = e.RunBatch(h)
print({k: round(v, 2) if isinstance(v, float) else v for k, v in st.as_dict().items()})
dbg = np.zeros((NQ, 24), np.int64); e._gpu.ifx_debug_stage1_queries(h, dbg.ctypes.data_as(C.c_void_p))
order = np.argsort(-dbg[:, 4])
print("total ms by path:", {p: round(dbg[dbg[:, 3] == p, 4].sum() / 1e6, 1) for p in (0, 1, 2, 3)}, "counts", {p: int((dbg[:, 3] == p).sum()) for p in (0, 1, 2, 3)})
print("selection share: %.1f%%" % (100 * dbg[:, 2].clip(0).sum() / dbg[:, 4].sum()))
for i in order[:12]:
    print("%-40s cand=%8d T=%3d path=%d sel=%.2fms total=%.2fms cta=%d" % (qs[i][:40], dbg[i, 0], dbg[i, 1], dbg[i, 3], dbg[i, 2] / 1e6, dbg[i, 4] / 1e6, dbg[i, 5]))
ph = dbg[:, 6:11].sum(0); print("scoring cycles share (thread 0 = heap warp): wait-for-workers %.1f%% eligibility+compaction %.1f%% phaseA(later tiles) %.1f%% phaseB %.1f%% heap drain %.1f%%" % tuple(100 * ph / ph.sum()), "| scoring cycles total %.0f M" % (ph.sum() / 1e6))
for i in order[:8]: print("   ", qs[i][:30], (dbg[i, 6:11] / 1e3).astype(int), "kcycles", "eligible", dbg[i, 11] & 0xFFFFF, "heap updates", dbg[i, 11] >> 20)
dbg[:, 18] = 0      # slot 18 is the AND tier-1 route code (ifx_base.h IFX_QDBG), not a timing
wp = dbg[:, 12:20].sum(0); print("worker-view cycles share: ids+norms %.1f%% bounds %.1f%% bitmap %.1f%% phaseA0 %.1f%% join-wait %.1f%% phaseA-later %.1f%% its-barrier %.1f%% post-join(B+elig) %.1f%%" % tuple(100 * wp / wp.sum()))
for i in order[:8]: print("   W", qs[i][:30], (dbg[i, 12:20] / 1e3).astype(int), "kcycles")
for i in order[:8]: print("   S", qs[i][:30], (dbg[i, 20:24] / 1e3).astype(int), "kcycles [prefix+sort, tier0/unions, tier1, compact]")
print("total eligible", int((dbg[:, 11] & 0xFFFFF).sum()), "total heap updates", int((dbg[:, 11] >> 20).sum()))
for pth in (1, 2, 3):
    sel = dbg[:, 3] == pth
    if sel.any(): print("path", pth, "n", int(sel.sum()), "mean cand", int(dbg[sel, 0].mean()), "mean T %.1f" % dbg[sel, 1].mean(), "mean total kcyc", int(dbg[sel, 4].mean() * 1.92e-3 * 1e3 / 1e3), "| heap-warp view kcyc", (dbg[sel, 6:11].mean(0) / 1e3).astype(int), "| worker view kcyc", (dbg[sel, 12:20].mean(0) / 1e3).astype(int), "| sel kcyc", (dbg[sel, 20:24].mean(0) / 1e3).astype(int))
np.save(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out", "qdbg_%d.npy" % ND), dbg)
ncont = (ND + 65535) // 65536; cpc = dbg[:, 0] / ncont
print("candidates per container: percentiles 10/50/90/99", np.percentile(cpc, [10, 50, 90, 99]).astype(int), "| share of queries <= 512 per container: %.1f%%, <= 1024: %.1f%%" % (100 * (cpc <= 512).mean(), 100 * (cpc <= 1024).mean()))
print("time share of queries with <= 512 cands/container: %.1f%%; <= 1024: %.1f%%" % (100 * dbg[cpc <= 512, 4].sum() / dbg[:, 4].sum(), 100 * dbg[cpc <= 1024, 4].sum() / dbg[:, 4].sum()))
c = dbg[:, 0]; print("cand percentiles", np.percentile(c, [50, 90, 99, 100]).astype(int), "mean", int(c.mean()))
# per-CTA busy time
busy = {}
for i in range(NQ): busy[dbg[i, 5]] = busy.get(dbg[i, 5], 0) + dbg[i, 4]
b = np.array(list(busy.values())) / 1e6; print("CTAs used", len(b), "busy ms max %.2f mean %.2f" % (b.max(), b.mean()))
