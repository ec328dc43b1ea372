"""GPU parity tests, Stage 1 (BM25 backbone): the CUDA path through the C-ABI vs the oracle, bit-exact
(DocumentId order and float32 score bits). Run on an H100 with `pytest -m gpu`."""
import numpy as np
import pytest

import infidex_b200 as ib
from infidex_b200 import synth
from parity_util import build_pair, compare_stage1

pytestmark = pytest.mark.gpu

MOVIE_QUERIES = ["redemption sh", "Shawshank", "Shaaawshank", "the amtrix", "star", "the hear", "fellowship of the ring", "te matri", "san a",
                 "batman", "the", "love", "new york", "harry potter and the", "x-men", "zzzzqqq", "matrix reloaded", "lord of the rings",
                 "the lord of the rings the return of the king", "a", "  ", "spider-man", "o'brien", "Música", "amelie"]


def test_stage1_movies(movie_titles, oracle_movies):
    eng = ib.SearchEngine.CreateDefault()
    eng.IndexColumns(np.arange(len(movie_titles)), [ib.Field("content")], [movie_titles])
    bad = compare_stage1(eng, oracle_movies, MOVIE_QUERIES)
    assert not bad, bad[:5]
