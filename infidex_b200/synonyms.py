"""SynonymMap of the reference (src/Infidex/Synonyms/SynonymMap.cs), restated for the host mirror.

A union-find over lower-cased terms: every group of synonyms collapses to one canonical root, the longest member (ties: the ordinal-
smaller root), so the canonical form depends on the order of the AddSynonym calls. The dictionaries of the reference compare keys
with StringComparer.OrdinalIgnoreCase: here a dictionary keyed by the upper-invariant fold of the key holds (first key inserted for
that fold, value). Whitespace is .NET char.IsWhiteSpace and case mapping is ToLowerInvariant / ToUpperInvariant, from the same
character tables the native code uses (csrc/chartables.inc).

An engine built with a map (SearchEngine(synonymMap=...)) hands the table of `canonical_table()` to the native builder.
"""
import os
import re

_TABLES = None

# TokenizerSetup.Delimiters of config 400 (the delimiter set of the native code)
DELIMITERS = frozenset(" -/.,:;'`–—*&\\_(){}[]\t")


def _tables():
    global _TABLES
    if _TABLES is None:
        src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "chartables.inc")).read()

        def arr(name):
            m = re.search(r"\b%s\b[^=]*=\s*\{(.*?)\};" % name, src, re.S)
            return [int(x) for x in re.findall(r"\d+", m.group(1))]
        lo, up = arr("IFX_LOWER_PAIRS"), arr("IFX_UPPER_PAIRS")
        _TABLES = ({lo[i]: lo[i + 1] for i in range(0, len(lo), 2)}, {up[i]: up[i + 1] for i in range(0, len(up), 2)},
                   frozenset(chr(c) for c in arr("IFX_SPACE_LIST")))
    return _TABLES


def _map(s, table):
    return "".join(chr(table.get(ord(c), ord(c))) for c in s)


def to_lower_invariant(s):
    return _map(s, _tables()[0])


def fold(s):
    """The key StringComparer.OrdinalIgnoreCase compares: ToUpperInvariant per UTF-16 unit."""
    return _map(s, _tables()[1])


def is_white_space(c):
    return c in _tables()[2]


def is_null_or_white_space(s):
    return s is None or all(is_white_space(c) for c in s)


def trim(s):
    b, e = 0, len(s)
    while b < e and is_white_space(s[b]):
        b += 1
    while e > b and is_white_space(s[e - 1]):
        e -= 1
    return s[b:e]


class _IgnoreCaseDict:
    """Dictionary<string, V>(StringComparer.OrdinalIgnoreCase): the key stays the first string inserted for its fold."""

    def __init__(self):
        self._d = {}

    def __contains__(self, k):
        return fold(k) in self._d

    def __getitem__(self, k):
        return self._d[fold(k)][1]

    def __setitem__(self, k, v):
        f = fold(k)
        self._d[f] = (self._d[f][0] if f in self._d else k, v)

    def __len__(self):
        return len(self._d)

    def keys(self):
        return [k for k, _ in self._d.values()]

    def clear(self):
        self._d.clear()


class SynonymMap:
    def __init__(self):
        self._synonyms = _IgnoreCaseDict()      # term -> _IgnoreCaseDict used as HashSet<string>(OrdinalIgnoreCase)
        self._parent = _IgnoreCaseDict()
        self._rank = _IgnoreCaseDict()
        self._version = 0                       # bumped by every change of the mappings (an engine's index snapshots it)

    def AddSynonym(self, term1, term2):
        if is_null_or_white_space(term1) or is_null_or_white_space(term2):
            return
        term1 = to_lower_invariant(trim(term1)); term2 = to_lower_invariant(trim(term2))
        if term1 == term2:
            return
        self._version += 1
        for a, b in ((term1, term2), (term2, term1)):
            if a not in self._synonyms:
                self._synonyms[a] = _IgnoreCaseDict()
            s = self._synonyms[a]
            if b not in s:
                s[b] = True
        self._union(term1, term2)

    def AddSynonymGroup(self, *terms):
        if len(terms) == 1 and isinstance(terms[0], (list, tuple)):
            terms = tuple(terms[0])
        if len(terms) < 2:
            return
        for i in range(len(terms)):
            for j in range(i + 1, len(terms)):
                self.AddSynonym(terms[i], terms[j])

    def GetSynonyms(self, term):
        if is_null_or_white_space(term):
            return set()
        term = to_lower_invariant(trim(term))
        return set(self._synonyms[term].keys()) if term in self._synonyms else set()

    def HasSynonyms(self, term):
        if is_null_or_white_space(term):
            return False
        return to_lower_invariant(trim(term)) in self._synonyms

    @property
    def Count(self):
        return len(self._synonyms)

    def Clear(self):
        self._version += 1
        self._synonyms.clear(); self._parent.clear(); self._rank.clear()

    def GetCanonical(self, term):
        if is_null_or_white_space(term):
            return ""
        term = to_lower_invariant(trim(term))
        if term not in self._parent:
            return term
        return self._find(term)

    def CanonicalizeText(self, text, delimiters=DELIMITERS):
        if not text or not delimiters or len(self._parent) == 0:
            return text
        out, i, n = [], 0, len(text)
        while i < n:
            if text[i] in delimiters:
                out.append(text[i]); i += 1
                continue
            s = i
            while i < n and text[i] not in delimiters:
                i += 1
            out.append(self.GetCanonical(text[s:i]))
        return "".join(out)

    @property
    def HasCanonicalMappings(self):
        return len(self._parent) > 0

    def canonical_table(self):
        """[(key, GetCanonical(key))] for every key of the union-find, in insertion order: the table an index is built with
        (ifx_builder_set_synonyms / ifx_index_image.syn_keys, syn_canon)."""
        return [(k, self.GetCanonical(k)) for k in self._parent.keys()]

    # ---- union-find (SynonymMap.cs:190-250) ----------------------------------------------------------------------------------------
    def _ensure(self, term):
        if term not in self._parent:
            self._parent[term] = term; self._rank[term] = 0

    def _find(self, term):
        self._ensure(term)
        parent = self._parent[term]
        if fold(parent) != fold(term):
            self._parent[term] = self._find(parent)
        return self._parent[term]

    def _union(self, term1, term2):
        self._ensure(term1); self._ensure(term2)
        root1, root2 = self._find(term1), self._find(term2)
        if fold(root1) == fold(root2):
            return
        l1, l2 = len(_u16(root1)) // 2, len(_u16(root2)) // 2      # string.Length: UTF-16 units
        if l1 != l2:
            canon, other = (root1, root2) if l1 >= l2 else (root2, root1)
        else:
            canon = root1 if _compare_ordinal(root1, root2) <= 0 else root2
            other = root2 if fold(canon) == fold(root1) else root1
        self._parent[other] = canon


def _u16(s):
    return s.encode("utf-16-le", "surrogatepass")


def _compare_ordinal(a, b):
    """string.CompareOrdinal: UTF-16 code units."""
    x, y = _u16(a), _u16(b)
    ux = [int.from_bytes(x[i:i + 2], "little") for i in range(0, len(x), 2)]
    uy = [int.from_bytes(y[i:i + 2], "little") for i in range(0, len(y), 2)]
    return (ux > uy) - (ux < uy)
