"""ctypes binding of tests/oracle_post.cpp: the oracle's search with Query.EnableBoost / Boosts and SortBy / SortAscending.

Test infrastructure only (tests/ and tools/bench_post.py). The library is compiled on first use, with the flags of oracle/Makefile,
into the system temporary directory (keyed by the hash of its sources), so the repository tree is never written. Its entry points
take the handle of an oracle.oracle.OracleEngine.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_post.cpp")
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_FLAGS = ["-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-shared"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [_SRC] + sorted(os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".cpp", ".hpp", ".inc")))
        h = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs) + " ".join(_FLAGS).encode()).hexdigest()[:16]
        path = os.path.join(tempfile.gettempdir(), "ifx_oracle_post_%d_%s.so" % (os.getuid(), h))
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["g++"] + _FLAGS + ["-o", tmp, _SRC])
            os.replace(tmp, path)
        _lib = C.CDLL(path)
    return _lib


def _post_args(boosts, sort):
    """boosts: [(INFISCRIPT-V1 bytes, int strength)] (the boosts whose Filter is not null); sort: (field name, ascending) or None."""
    boosts = list(boosts or [])
    codes = [np.frombuffer(b, np.uint8).copy() for b, _ in boosts]
    ptrs = (C.c_void_p * max(len(codes), 1))(*[c.ctypes.data for c in codes])
    lens = np.array([len(c) for c in codes] or [0], np.int32); strength = np.array([int(k) for _, k in boosts] or [0], np.int32)
    field = O.u16(sort[0]) if sort else np.zeros(1, np.uint16)
    keep = (codes, ptrs, lens, strength, field)
    args = (ptrs, O._p(lens), O._p(strength), len(codes), O._p(field), len(sort[0]) if sort else -1, int(bool(sort[1])) if sort else 1)
    return keep, args


def search(orc, text, max_results=10, depth=500, coverage=True, filter_bytes=None, facets=False, boosts=None, sort=None, cap=None):
    """OracleEngine.search with boosts / SortBy: the same result dict."""
    cap = cap or max(max_results, 1)
    q = O.u16(text)
    keys = np.zeros(cap, np.int64); scores = np.zeros(cap, np.float32); ties = np.zeros(cap, np.uint8)
    n = C.c_int(0); total = C.c_int(0); fb = C.create_string_buffer(1 << 16); fl = C.c_int(0)
    fbytes = np.frombuffer(filter_bytes, np.uint8).copy() if filter_bytes else None
    keep, post = _post_args(boosts, sort)
    st = lib().ifxo_post_search(orc.h, O._p(q), len(q), max_results, depth, int(coverage),
                                O._p(fbytes) if fbytes is not None else None, len(fbytes) if fbytes is not None else 0, int(facets), *post,
                                O._p(keys), O._p(scores), O._p(ties), cap, C.byref(n), C.byref(total), fb, len(fb), C.byref(fl))
    facet_list = []
    if facets:
        for line in fb.raw[: fl.value].decode("utf-8").splitlines():
            f, v, c = line.split("\t"); facet_list.append((f, v, int(c)))
    return {"status": st, "keys": keys[: n.value].tolist(), "scores": scores[: n.value].copy(), "ties": ties[: n.value].tolist(),
            "total": total.value, "facets": facet_list}


def search_batch(orc, queries, max_results=10, depth=500, coverage=True, filter_bytes=None, threads=1, boosts=None, sort=None):
    """OracleEngine.search_batch with the same boosts / SortBy on every query: (keys, scores, ties, n, status)."""
    blob, offs = O.pack_strings(queries); nq = len(queries); cap = max_results
    keys = np.zeros((nq, cap), np.int64); scores = np.zeros((nq, cap), np.float32); ties = np.zeros((nq, cap), np.uint8)
    ns = np.zeros(nq, np.int32); status = np.zeros(nq, np.int32)
    fbytes = np.frombuffer(filter_bytes, np.uint8).copy() if filter_bytes else None
    keep, post = _post_args(boosts, sort)
    lib().ifxo_post_search_batch(orc.h, O._p(blob), O._p(offs), nq, max_results, depth, int(coverage),
                                 O._p(fbytes) if fbytes is not None else None, len(fbytes) if fbytes is not None else 0, *post,
                                 threads, O._p(keys), O._p(scores), O._p(ties), cap, O._p(ns), O._p(status))
    return keys, scores, ties, ns, status


def set_field_kind(orc, name, kind):
    """After OracleEngine.load_image: field `name` holds int64 (kind 2) or double (kind 3) values, not their text."""
    a = O.u16(name); n = lib().ifxo_post_set_field_kind(orc.h, O._p(a), len(a), kind)
    if n < 0:
        raise ValueError("field %r: values do not parse as kind %d" % (name, kind))
    return n
