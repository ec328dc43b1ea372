"""A batch handle that ran through the doc-id-range phases answers like a fresh one when it is refilled and run with ifx_batch_run (kernel
emulation build, one rank of ShardedSearchEngine on a thread stand-in for torch.distributed). Every run starts from the same per-run state:
nothing a shard's phases set -- the global selection counts, the shard outputs of k_finalize -- carries over into the next run."""
import numpy as np

import infidex_b200 as ib
from infidex_b200 import synth

from dist_util import run_ranks
from parity_util import emu_lib

N = 70_000


def test_a_handle_run_as_a_shard_then_by_ifx_batch_run_answers_as_a_fresh_one():
    from infidex_b200 import dist as ifxd
    emu = emu_lib()
    vocab = synth.make_vocab(20_000); docs = synth.gen_docs(N, vocab)
    schema, cols = synth.schema_and_columns(docs, False)
    texts = synth.gen_queries(128, docs, vocab)
    first, second = [ib.Query(t, 10) for t in texts[:64]], [ib.Query(t, 10) for t in texts[64:]]

    def fn(d, r):
        eng = ifxd.ShardedSearchEngine(d, _gpu_lib=emu); eng.IndexShard(docs["keys"], schema, cols, threads=2)
        try:
            eng.SearchBatch(first)
            e = eng.eng; h = eng._cached_h; reused = e.PackBatch(second)
            e._check(e._gpu.ifx_batch_refill(h, reused["arr"], len(second)), "ifx_batch_refill")
            e.RunBatch(h); e.DownloadBatch(h, reused)
            fresh = e.PackBatch(second); e.SearchPacked(fresh)
            return reused["bufs"], fresh["bufs"]
        finally:
            eng.Close()
    (reused, fresh), = run_ranks(1, fn)

    def answer(b, i):
        n = int(b["n"][i])
        return b["keys"][i, :n].tolist(), b["scores"][i, :n].view(np.uint32).tolist(), b["ties"][i, :n].tolist(), n, int(b["total"][i]), int(b["status"][i])
    bad = [i for i in range(len(second)) if answer(reused, i) != answer(fresh, i)]
    assert not bad, (len(bad), answer(reused, bad[0]), answer(fresh, bad[0]))
