"""Stage 1's scorers on the GPU -- score_warp<256> (light), score_warp<512> (mid), score_cta and k_s1_finish -- against the oracle,
bit for bit, at the class, tile and heap edges (fixture: scorer_corpus.py). What only this file reaches:
  - score_cta's fast path (a thread's 8 slots in registers, 8-byte tf and float4 score / norm loads) and the packed 16-bit rank
    scan of a tile's unskippable terms (both compiled out of the emulation, which takes the scalar loop and one scan per term);
  - score_warp's layout (slot j in lane j % 32, register j / 32) with ranks from ballots: the emulation keeps every slot in one lane;
  - every scorer run by many warps / CTAs at once, pulling queries of one batch from the class queues.
Lookup modes 0 (the cost model's choice) and 2 (streamed lists) both run: the scorers must not depend on how the tf bytes arrived.
The routing, heap-depth and tie edges, the oracle's MaxScore trace and the fixture's sensitivity to the Vector256 / scalar split
are checked by test_emu_scorers.py on the CPU."""
import pytest

import scorer_corpus as S
from parity_util import compare_stage1

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pair():
    eng, orc, docs = S.build()
    yield eng, orc, docs
    eng.Dispose()


@pytest.mark.parametrize("mode", ["0", "2"])
def test_scorers_stage1(pair, monkeypatch, mode):
    """Every query at each depth: a 4-ary heap of 1-5 nodes, the warp heap full (512), the smallest depth sent to the CTA whatever
    the chunk size (513), and the CTA heap full with k_s1_finish over 1 024 entries (1 024)."""
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, _ = pair
    qs = [q for q, _ in S.queries()]
    for depth in S.DEPTHS:
        bad = compare_stage1(eng, orc, qs, depth=depth)
        assert not bad, (depth, bad[:3])


@pytest.mark.parametrize("mode", ["0", "2"])
def test_scorers_mixed_depth(pair, monkeypatch, mode):
    """One batch whose queries carry different CoverageDepth values, so the classes and heap sizes mix in every launch."""
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, _ = pair
    bad = S.compare_mixed(eng, orc, S.mixed_batch())
    assert not bad, bad[:3]


def test_scorers_reach(pair, monkeypatch):
    """Which scorer each query of the mixed batch reached, read back from the device: the class counts match Stats, and each class
    reaches its chunk-size, term-count and depth edges."""
    monkeypatch.setenv("IFX_S1_LOOKUP", "2")
    eng, orc, docs = pair
    rows, st = S.reach(eng, S.mixed_batch())
    print("light / mid / CTA: %d / %d / %d" % (st.s1_light, st.s1_mid, st.s1_heavy))
    S.check_reach(rows, st, docs)
