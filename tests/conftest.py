import gzip
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _have_gpu():
    try:
        import ctypes
        from infidex_b200 import _build
        if not os.path.exists(_build.GPU_LIB):
            return False
        lib = ctypes.CDLL(_build.GPU_LIB); lib.ifx_device_count.restype = ctypes.c_int
        return lib.ifx_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need a CUDA device: on a box without one they are skipped (never silently run on a CPU path -- there is none)."""
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device (run on an H100 with -m gpu)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def load_movie_titles():
    p = os.path.join(ROOT, "tests", "golden", "movies_titles.txt.gz")
    return [l.rstrip("\n").replace("\\n", "\n").replace("\\\\", "\\") for l in gzip.open(p, "rt", encoding="utf-8")]


REFERENCE_10 = [
    "The quick brown fox jumps over the lazy dog", "A journey of a thousand miles begins with a single step",
    "To be or not to be, that is the question", "All that glitters is not gold", "The fox was quick and clever in the forest",
    "Batman and Robin fight crime in Gotham City", "Superman flies faster than a speeding bullet",
    "Spider-Man swings through New York City", "Wonder Woman protects the innocent", "The Flash runs at incredible speeds",
]


@pytest.fixture(scope="session")
def movie_titles():
    return load_movie_titles()


@pytest.fixture(scope="session")
def oracle_movies(movie_titles):
    from oracle.oracle import OracleEngine
    e = OracleEngine()
    e.index_texts(movie_titles)
    return e


@pytest.fixture(scope="session")
def oracle_ref10():
    import numpy as np
    from oracle.oracle import OracleEngine
    e = OracleEngine()
    e.index_texts(REFERENCE_10, keys=np.arange(1, 11))
    return e
