"""ctypes binding of tests/oracle_syn.cpp: the oracle with a SynonymMap.

Test infrastructure only (tests/ and tools/bench_synonyms.py). The library is compiled on first use, with the flags of oracle/Makefile,
into the system temporary directory (keyed by the hash of its sources), so the repository tree is never written.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oracle_syn.cpp")
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_FLAGS = ["-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-shared"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [_SRC] + sorted(os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".cpp", ".hpp", ".inc")))
        srcs.append(os.path.join(os.path.dirname(_HERE), "include", "infidex_gpu.h"))
        h = hashlib.sha1(b"".join(open(s, "rb").read() for s in srcs) + " ".join(_FLAGS).encode()).hexdigest()[:16]
        path = os.path.join(tempfile.gettempdir(), "ifx_oracle_syn_%d_%s.so" % (os.getuid(), h))
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call(["g++"] + _FLAGS + ["-o", tmp, _SRC])
            os.replace(tmp, path)
        _lib = C.CDLL(path)
        _lib.ifxo_create.restype = C.c_void_p
    return _lib


class SynOracleEngine(O.OracleEngine):
    """OracleEngine (SearchEngine.CreateDefault restated) built with a SynonymMap: `synonyms` is the ordered list of AddSynonym(a, b)
    calls, replayed by the oracle's own union-find. The engine's handle lives in this library (the same capi.cpp, compiled apart)."""

    def __init__(self, schema=None, synonyms=()):
        L = lib()
        self.h = C.c_void_p(L.ifxo_create())
        self.schema = schema or [O.Field("content", 1)]
        blob, offs = O.pack_strings([f.name for f in self.schema])
        w = np.array([f.weight for f in self.schema], np.int32)
        fl = np.array([(1 if f.indexable else 0) | (2 if f.filterable else 0) | (4 if f.facetable else 0) for f in self.schema], np.int32)
        L.ifxo_set_schema(self.h, len(self.schema), O._p(blob), O._p(offs.astype(np.int32)), O._p(w), O._p(fl))
        for a, b in synonyms:
            x, y = O.u16(a), O.u16(b)
            L.ifxo_syn_add(self.h, O._p(x), len(x), O._p(y), len(y))

    def __del__(self):
        try:
            lib().ifxo_syn_forget(self.h); lib().ifxo_destroy(self.h)
        except Exception:
            pass

    def table(self):
        """[(key, GetCanonical(key))] of the replayed map, in key insertion order."""
        n = lib().ifxo_syn_table(self.h, None, 0); buf = C.create_string_buffer(max(n, 1)); lib().ifxo_syn_table(self.h, buf, n)
        return [tuple(l.split("\t")) for l in buf.raw[:n].decode("utf-8").splitlines()]

    def canonicalize(self, text):
        a = O.u16(text); out = np.zeros(max(4 * len(a) + 64, 1), np.uint16)
        n = lib().ifxo_syn_canonicalize(self.h, O._p(a), len(a), O._p(out), len(out))
        if n > len(out):
            out = np.zeros(n, np.uint16); lib().ifxo_syn_canonicalize(self.h, O._p(a), len(a), O._p(out), len(out))
        return O.from_u16(out[:n])

    def index_columns(self, keys, columns):
        n = len(keys)
        keys = np.ascontiguousarray(keys, np.int64)
        kinds = np.zeros(len(columns), np.int32)
        keep, cols, offs = [], (C.c_void_p * len(columns))(), (C.c_void_p * len(columns))()
        for i, col in enumerate(columns):
            if isinstance(col, np.ndarray) and col.dtype.kind in "iu":
                a = np.ascontiguousarray(col, np.int64); kinds[i] = 2; cols[i] = a.ctypes.data; keep.append(a)
            elif isinstance(col, np.ndarray) and col.dtype.kind == "f":
                a = np.ascontiguousarray(col, np.float64); kinds[i] = 3; cols[i] = a.ctypes.data; keep.append(a)
            elif isinstance(col, tuple):                 # pre-packed (uint16 blob, int64 offsets)
                blob, o = col; kinds[i] = 1; cols[i] = blob.ctypes.data; offs[i] = o.ctypes.data; keep += [blob, o]
            else:
                blob, o = O.pack_strings(col); kinds[i] = 1; cols[i] = blob.ctypes.data; offs[i] = o.ctypes.data; keep += [blob, o]
        lib().ifxo_syn_add_docs(self.h, n, O._p(keys), O._p(kinds), cols, offs)
        lib().ifxo_syn_build(self.h)

    def load_image(self, image_ptr):
        lib().ifxo_syn_load_image(self.h, C.c_void_p(image_ptr))

    def search(self, text, max_results=10, depth=500, coverage=True, filter_bytes=None, facets=False, cap=None):
        cap = cap or max(max_results, 1)
        q = O.u16(text)
        keys = np.zeros(cap, np.int64); scores = np.zeros(cap, np.float32); ties = np.zeros(cap, np.uint8)
        n = C.c_int(0); total = C.c_int(0); fb = C.create_string_buffer(1 << 16); fl = C.c_int(0)
        fbytes = np.frombuffer(filter_bytes, np.uint8).copy() if filter_bytes else None
        st = lib().ifxo_syn_search(self.h, O._p(q), len(q), max_results, depth, int(coverage),
                                   O._p(fbytes) if fbytes is not None else None, len(fbytes) if fbytes is not None else 0, int(facets),
                                   O._p(keys), O._p(scores), O._p(ties), cap, C.byref(n), C.byref(total), fb, len(fb), C.byref(fl))
        facet_list = []
        if facets:
            for line in fb.raw[: fl.value].decode("utf-8").splitlines():
                f, v, c = line.split("\t"); facet_list.append((f, v, int(c)))
        return {"status": st, "keys": keys[: n.value].tolist(), "scores": scores[: n.value].copy(), "ties": ties[: n.value].tolist(),
                "total": total.value, "facets": facet_list}

    def search_batch(self, queries, max_results=10, depth=500, coverage=True, filter_bytes=None, threads=1):
        blob, offs = O.pack_strings(queries); nq = len(queries); cap = max_results
        keys = np.zeros((nq, cap), np.int64); scores = np.zeros((nq, cap), np.float32); ties = np.zeros((nq, cap), np.uint8)
        ns = np.zeros(nq, np.int32); status = np.zeros(nq, np.int32)
        fbytes = np.frombuffer(filter_bytes, np.uint8).copy() if filter_bytes else None
        lib().ifxo_syn_search_batch(self.h, O._p(blob), O._p(offs), nq, max_results, depth, int(coverage),
                                    O._p(fbytes) if fbytes is not None else None, len(fbytes) if fbytes is not None else 0, threads,
                                    O._p(keys), O._p(scores), O._p(ties), cap, O._p(ns), O._p(status))
        return keys, scores, ties, ns, status

    # introspection entry points of capi.cpp, bound to this library (the handle is one of its engines)
    def num_terms(self):
        return lib().ifxo_num_terms(self.h)

    def term(self, t):
        L = lib(); buf = np.zeros(256, np.uint16); n = L.ifxo_term_text(self.h, t, O._p(buf), 256)
        df = L.ifxo_term_df(self.h, t); npost = L.ifxo_term_npost(self.h, t)
        docs = np.zeros(max(npost, 1), np.int32); w = np.zeros(max(npost, 1), np.uint8)
        if npost:
            L.ifxo_term_postings(self.h, t, O._p(docs), O._p(w))
        return O.from_u16(buf[:n]), df, docs[:npost], w[:npost]

    def word_idf(self, word):
        L = lib(); L.ifxo_word_idf.restype = C.c_float; a = O.u16(word); return float(L.ifxo_word_idf(self.h, O._p(a), len(a)))

    def dict_docs(self, kind, key):
        a = O.u16(key); out = np.zeros(1 << 16, np.int32); n = lib().ifxo_dict_docs(self.h, kind, O._p(a), len(a), O._p(out), len(out))
        return None if n < 0 else out[:n].tolist()
