"""The corpus and batch of test_gpu_tf_lookups in the kernel emulation (one thread per block, one selection CTA), against the
oracle: it proves the fixture and its expected answers without a GPU, so a failure of the GPU tests points at thread- or CTA-level
behaviour. The largest group is smaller here (300 queries: still two TF_QCAP metadata chunks, the queries
with candidates in container 5 in the second) to keep the run short."""
import pytest

import infidex_b200 as ib
from parity_util import compare_search, compare_stage1, emu_lib
from test_gpu_tf_lookups import GROUPS, _upload, build, check_reach, reach

BIG = 300


@pytest.fixture(scope="module")
def pair():
    eng, orc, qs, subset, shape = build(emu_lib(), big=BIG)
    yield eng, orc, qs, subset, shape
    eng.Dispose()


@pytest.mark.parametrize("mode", ["0", "2"])
def test_emu_tf_lookups(pair, monkeypatch, mode):
    monkeypatch.setenv("IFX_S1_LOOKUP", mode)
    eng, orc, qs, subset, shape = pair
    assert not compare_stage1(eng, orc, qs)
    assert not compare_search(eng, orc, subset)
    if mode == "2":
        check_reach(reach(eng, qs, shape), dict(GROUPS, common=BIG))


def test_emu_tf_lookups_waves(pair, monkeypatch):
    """The batch through a 60 MB staging pool: several waves (5 with the 600-query group of the GPU test)."""
    monkeypatch.setenv("IFX_S1_LOOKUP", "2")
    eng, orc, qs, subset, shape = pair
    _upload(eng, 60)
    try:
        st = ib.Stats()
        assert not compare_stage1(eng, orc, qs, stats=st)
        assert st.s1_waves > 1
    finally:
        _upload(eng)
