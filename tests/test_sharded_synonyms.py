"""Doc-id-range sharding with a SynonymMap on CPU: two gloo processes (kernel emulation build), each shard's builder given the map's table,
the merged result against the UNSHARDED oracle with the same map. The allowance for the Stage-1 couplings that are not exchanged is
test_sharded.py's."""
import os
import pickle

import numpy as np

from dist_util import spawn_gloo

N = 160_000


def _worker(rank, world, emu, outdir):
    import torch.distributed as dist
    import infidex_b200 as ib
    from infidex_b200 import dist as ifxd
    from infidex_b200 import synth
    vocab = synth.make_vocab(30_000)
    m = ib.SynonymMap()
    for a, b in synth.make_synonym_pairs(vocab, 1500):
        m.AddSynonym(a, b)
    lo, hi = ifxd.shard_ranges(N, world)[rank]
    docs = synth.gen_docs(hi - lo, vocab, start=lo)
    schema, cols = synth.schema_and_columns(docs, False)
    eng = ifxd.ShardedSearchEngine(dist, _gpu_lib=emu, synonymMap=m); eng.IndexShard(docs["keys"], schema, cols, threads=2)
    res = eng.SearchBatch([ib.Query(q, 10) for q in _queries(vocab)])
    eng.Close()
    if rank == 0:
        pickle.dump([[(e.DocumentId, np.float32(e.Score).view(np.uint32).item(), e.Tiebreaker) for e in r.Records] for r in res], open(os.path.join(outdir, "merged.pkl"), "wb"))


def _queries(vocab):
    from infidex_b200 import synth
    pairs = synth.make_synonym_pairs(vocab, 1500)
    rng = np.random.Generator(np.random.PCG64(21)); words = sorted({w for p in pairs for w in p})
    return synth.gen_queries(100, synth.corpus_ref(N), vocab) + [" ".join(rng.choice(words, int(rng.integers(1, 3)))) for _ in range(60)]


def test_two_shards_with_a_map_against_the_unsharded_oracle(tmp_path):
    from infidex_b200 import synth
    from oracle.oracle import Field as OField
    from oracle_syn import SynOracleEngine
    from parity_util import emu_lib
    spawn_gloo(_worker, 2, emu_lib(), str(tmp_path))
    merged = pickle.load(open(tmp_path / "merged.pkl", "rb"))
    vocab = synth.make_vocab(30_000); docs = synth.gen_docs(N, vocab)
    schema, cols = synth.schema_and_columns(docs, False)
    orc = SynOracleEngine([OField(f.Name, f.Weight, f.Indexable, f.Filterable, f.Facetable) for f in schema], synth.make_synonym_pairs(vocab, 1500))
    orc.index_columns(docs["keys"], cols)
    qs = _queries(vocab)
    diff = ids_diff = 0
    for q, got in zip(qs, merged):
        x = orc.search(q, 10)
        if got != list(zip(x["keys"], x["scores"].view(np.uint32).tolist(), x["ties"])):
            diff += 1
            ids_diff += [g[0] for g in got] != x["keys"]
    print("sharded (with a map) vs unsharded oracle: %d of %d queries differ (%d in DocumentId order)" % (diff, len(qs), ids_diff))
    assert ids_diff <= len(qs) // 10, (diff, ids_diff)
