"""The fixture of test_gpu_scorers in the kernel emulation (one thread per block), against the oracle: the scorer routing, the class
edges, the heap depths 1-5 / 512 / 513 / 1 024 and the score ties at the threshold and the depth cut, without a GPU. Plus what the
fixture itself must give for the GPU parity checks to mean anything: the oracle's MaxScore trace (skipped pairs in every class,
chunks behind a full heap, a flush with more than SURV_CAP survivors) and candidates whose Vector256 and scalar BM25+ forms round
differently. The emulation cannot reach score_cta's fast path and packed rank scan (compiled out) or score_warp's 32-lane layout
(one lane holds all slots): only the GPU file covers those."""
import pytest

import scorer_corpus as S
from parity_util import compare_stage1, emu_lib


@pytest.fixture(scope="module")
def pair():
    eng, orc, docs = S.build(emu_lib())
    yield eng, orc, docs
    eng.Dispose()


@pytest.mark.parametrize("mode", ["0", "2"])
def test_emu_scorers(pair, monkeypatch, mode):
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, _ = pair
    qs = [q for q, _ in S.queries()]
    for depth in S.DEPTHS:
        bad = compare_stage1(eng, orc, qs, depth=depth)
        assert not bad, (depth, bad[:3])
    bad = S.compare_mixed(eng, orc, S.mixed_batch())
    assert not bad, bad[:3]


def test_emu_scorers_reach(pair, monkeypatch):
    monkeypatch.setenv("IFX_S1_LOOKUP", "2")
    eng, orc, docs = pair
    batch = S.mixed_batch()
    rows, st = S.reach(eng, batch)
    S.check_reach(rows, st, docs)
    S.check_trace(orc, rows, batch)


def test_emu_scorers_sensitivity(pair):
    """A wrong rank or vec_end changes a score bit only where the two forms round differently: enough candidates must."""
    _, orc, docs = pair
    share = S.vector_scalar_differ(orc, docs)
    print("avgdl %.4f: the forms differ on %.1f %% of the candidates" % (orc.avgdl(), 100 * share))
    assert share >= 0.05
