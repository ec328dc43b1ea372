"""Doc-id-range sharding on CPU: two processes (gloo, world size 2), each holding one shard of ONE index (kernel emulation build), the three
exchanges of infidex_b200.dist.ShardedSearchEngine, and the merged result compared with the UNSHARDED oracle. Stage-1-level couplings that are
not exchanged (tier rules, threshold chain on shard-local counts; WordMatcher quota / truncation per shard) are allowed to show up as a small,
counted number of differing queries -- the test pins that number's ceiling and that everything exchanged is exact."""
import os

import numpy as np
import pytest

from dist_util import spawn_gloo


def _worker(rank, world, emu, outdir, multi):
    import torch.distributed as dist
    import infidex_b200 as ib
    from infidex_b200 import dist as ifxd
    from infidex_b200 import synth
    N = 180_000 if not multi else 140_000
    vocab = synth.make_vocab(30_000)
    lo, hi = ifxd.shard_ranges(N, world)[rank]
    docs = synth.gen_docs(hi - lo, vocab, with_description=multi, start=lo)
    schema, cols = synth.schema_and_columns(docs, multi)
    eng = ifxd.ShardedSearchEngine(dist, _gpu_lib=emu); eng.IndexShard(docs["keys"], schema, cols, threads=2)
    qs = synth.gen_queries(160, synth.corpus_ref(N), vocab)
    res = eng.SearchBatch([ib.Query(q, 10) for q in qs])
    # the engine keeps its batch handle between calls (ifx_batch_refill): a smaller batch, then the full one again, must reproduce the first answer
    sig = lambda rr: [[(e.DocumentId, np.float32(e.Score).view(np.uint32).item(), e.Tiebreaker) for e in r.Records] for r in rr]
    part = eng.SearchBatch([ib.Query(q, 10) for q in qs[:50]]); again = eng.SearchBatch([ib.Query(q, 10) for q in qs])
    assert sig(part) == sig(res)[:50] and sig(again) == sig(res)
    eng.Close()
    if rank == 0:
        import pickle
        pickle.dump([[(e.DocumentId, np.float32(e.Score).view(np.uint32).item(), e.Tiebreaker) for e in r.Records] for r in res], open(os.path.join(outdir, "merged.pkl"), "wb"))


@pytest.mark.parametrize("multi", [False, True])
def test_two_shards_against_the_unsharded_oracle(tmp_path, multi):
    import pickle
    from infidex_b200 import synth
    from oracle.oracle import Field as OField
    from oracle.oracle import OracleEngine
    from parity_util import emu_lib
    spawn_gloo(_worker, 2, emu_lib(), str(tmp_path), multi)
    merged = pickle.load(open(tmp_path / "merged.pkl", "rb"))
    N = 180_000 if not multi else 140_000
    vocab = synth.make_vocab(30_000); docs = synth.gen_docs(N, vocab, with_description=multi)
    schema, cols = synth.schema_and_columns(docs, multi)
    orc = OracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema]); orc.index_columns(docs["keys"], cols)
    qs = synth.gen_queries(160, docs, vocab)
    diff = ids_diff = 0
    for q, got in zip(qs, merged):
        x = orc.search(q, 10)
        want = list(zip(x["keys"], x["scores"].view(np.uint32).tolist(), x["ties"]))
        if got != want:
            diff += 1
            if [g[0] for g in got] != x["keys"]:
                ids_diff += 1
    print("sharded vs unsharded oracle: %d of %d queries differ (%d in DocumentId order)" % (diff, len(qs), ids_diff))
    assert ids_diff <= len(qs) // 10, (diff, ids_diff)
