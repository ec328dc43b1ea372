"""N > 1 host logic on CPU: two processes (gloo, world size 2), each with a replica of the index (kernel emulation build),
rank-local query batches, max-over-ranks timing and the all-gather of result blocks."""
import os

import numpy as np

from dist_util import spawn_gloo


def _worker(rank, world, emu, outdir):
    import torch.distributed as dist
    import infidex_b200 as ib
    from infidex_b200 import dist as ifxd
    from infidex_b200 import synth
    vocab = synth.make_vocab(5000); docs = synth.gen_docs(4000, vocab)
    schema, cols = synth.schema_and_columns(docs, False)
    eng = ib.SearchEngine(_gpu_lib=emu); eng.IndexColumns(docs["keys"], schema, cols)
    qs = synth.gen_queries(16, docs, vocab, seed=ifxd.rank_batch_seed(synth.SEED, 0, rank))
    packed = eng.PackBatch([ib.Query(q, 10) for q in qs]); eng.SearchPacked(packed)
    keys = packed["bufs"]["keys"]
    gathered = ifxd.gather_results(dist, keys)
    tmax = ifxd.max_over_ranks(dist, [float(rank + 1), 5.0 - rank])
    np.save(os.path.join(outdir, "local_%d.npy" % rank), keys)
    if rank == 0:
        np.save(os.path.join(outdir, "gathered.npy"), np.stack(gathered)); np.save(os.path.join(outdir, "tmax.npy"), np.array(tmax))


def test_two_rank_replicas(tmp_path):
    from parity_util import emu_lib
    spawn_gloo(_worker, 2, emu_lib(), str(tmp_path))
    g = np.load(tmp_path / "gathered.npy"); l0 = np.load(tmp_path / "local_0.npy"); l1 = np.load(tmp_path / "local_1.npy")
    assert np.array_equal(g[0], l0) and np.array_equal(g[1], l1)
    assert not np.array_equal(l0, l1)                      # distinct batches per rank
    assert np.load(tmp_path / "tmax.npy").tolist() == [2.0, 5.0]
