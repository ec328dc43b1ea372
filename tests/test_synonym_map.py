"""SynonymMap (infidex_b200/synonyms.py) against SynonymMap.cs: the SynonymTests.cs API cases, union-find roots derived by hand from
SynonymMap.cs, the table an index is built with (mirror == the oracle's own union-find, tests/oracle_syn.cpp), and the native
canonicalisation of the host builder's query preparation."""
import numpy as np
import pytest

import infidex_b200 as ib
from infidex_b200 import synonyms as S
from oracle import oracle as O
from oracle_syn import SynOracleEngine


def _map(pairs):
    m = ib.SynonymMap()
    for a, b in pairs:
        m.AddSynonym(a, b)
    return m


def test_bidirectional_pair():
    m = _map([("car", "automobile")])
    assert m.GetSynonyms("car") == {"automobile"} and m.GetSynonyms("automobile") == {"car"}
    assert m.HasSynonyms("car") and m.HasSynonyms("automobile") and m.Count == 2


def test_group_is_a_full_mesh():
    m = ib.SynonymMap(); m.AddSynonymGroup("car", "automobile", "vehicle")
    assert m.GetSynonyms("car") == {"automobile", "vehicle"}
    assert m.GetSynonyms("vehicle") == {"car", "automobile"} and m.Count == 3


def test_case_insensitive_and_unknown_and_clear():
    m = _map([("Car", "AUTOMOBILE")])
    assert m.GetSynonyms("CAR") == {"automobile"} and m.HasSynonyms("  Automobile ")
    assert m.GetSynonyms("bicycle") == set() and not m.HasSynonyms("bicycle") and m.GetSynonyms("   ") == set()
    m.Clear()
    assert m.Count == 0 and not m.HasCanonicalMappings and m.GetSynonyms("car") == set()


def test_skips_blank_and_equal_terms():
    m = _map([("", "x"), ("  ", "y"), ("Same", "same ")])
    assert m.Count == 0 and not m.HasCanonicalMappings


def test_roots_longer_wins_ties_ordinal_and_chains():
    m = _map([("ab", "abc")])                        # longer root wins
    assert m.GetCanonical("ab") == "abc"
    m = _map([("xyz", "abc")])                       # equal length: ordinal-smaller root
    assert m.GetCanonical("xyz") == "abc" and m.GetCanonical("abc") == "abc"
    m = _map([("a", "bb"), ("bb", "ccc"), ("ccc", "dd")])    # chain: every member collapses to the longest root
    assert {m.GetCanonical(t) for t in ("a", "bb", "ccc", "dd")} == {"ccc"}
    assert m.GetCanonical("unrelated Word ") == "unrelated word" and m.GetCanonical("  ") == ""


def test_roots_depend_on_call_order():
    # union of two groups: the roots are compared, not the members -- the order of the calls decides which roots meet
    m1 = _map([("aa", "bbbb"), ("cccc", "dd"), ("aa", "dd")])       # roots bbbb / cccc: equal length, ordinal -> bbbb
    m2 = _map([("aa", "dd"), ("aa", "bbbb"), ("cccc", "dd")])       # roots: {aa,dd}->aa then bbbb; cccc joins bbbb -> bbbb
    assert m1.GetCanonical("cccc") == "bbbb" and m2.GetCanonical("cccc") == "bbbb"
    m3 = _map([("cccc", "dd"), ("aa", "dd"), ("aa", "bbbb")])       # cccc is the root of {cccc, dd, aa}; bbbb ties with it -> bbbb
    m4 = _map([("zzzz", "dd"), ("aa", "dd"), ("aa", "bbbb")])       # root zzzz vs bbbb -> bbbb
    m5 = _map([("zzzzz", "dd"), ("aa", "dd"), ("aa", "bbbb")])      # a longer root survives
    assert m3.GetCanonical("dd") == "bbbb" and m4.GetCanonical("zzzz") == "bbbb" and m5.GetCanonical("bbbb") == "zzzzz"


def test_case_fold_key_collision():
    # U+017F (long s) and 's' are both lower case and fold to the same upper-case 'S': one key of the OrdinalIgnoreCase dictionary
    assert S.fold("ſ") == S.fold("s") and S.to_lower_invariant("ſ") == "ſ"
    m = _map([("ſx", "long1"), ("sx", "longer2")])
    keys = [k for k, _ in m.canonical_table()]
    assert "sx" not in keys and "ſx" in keys                   # the first string inserted stays the key
    assert m.GetCanonical("SX") == m.GetCanonical("ſx") == "longer2"


def test_whitespace_is_dotnet_not_python():
    assert "\x1c".isspace() and not S.is_white_space("\x1c")      # Python accepts U+001C-U+001F, char.IsWhiteSpace does not
    assert S.is_white_space(" ") and S.is_white_space(" ")
    m = _map([("a", "bbb")])
    assert m.CanonicalizeText("\x1ca\x1c") == "\x1ca\x1c"          # not trimmed: not a key
    assert m.CanonicalizeText("x  a  y") == "x bbb y"    # trimmed, then the key
    assert m.CanonicalizeText("x   y") == "x  y"              # a whitespace-only token becomes ""


def test_canonicalize_text_keeps_delimiters_and_lowercases_every_token():
    m = _map([("nyc", "New York")])
    assert m.CanonicalizeText("I ♥ NYC, Paris§Rome") == "i ♥ new york, paris§rome"
    assert ib.SynonymMap().CanonicalizeText("Untouched TEXT") == "Untouched TEXT"   # no mappings: the text as it is


RANDOM_WORDS = ["car", "Auto", "automobile", "nyc", "new york", "ZS", "základní", "ss", "stredni", "gympl", "gymnazium", "ſx", "sx",
                "ab", "abc", "xyz", "  pad  ", "Ärger", "ärger", "q"]


@pytest.mark.parametrize("seed", range(8))
def test_table_equals_oracle_union_find(seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    pairs = [(RANDOM_WORDS[i], RANDOM_WORDS[j]) for i, j in rng.integers(0, len(RANDOM_WORDS), (30, 2))]
    m = _map(pairs); orc = SynOracleEngine(synonyms=pairs)
    assert m.canonical_table() == orc.table()
    for t in ["I drive a CAR in NYC", "zs    ss§gympl", "-SX- ab/xyz ſx", ""]:
        assert m.CanonicalizeText(t) == orc.canonicalize(t)


def test_canon_of_normalized_equals_canon_of_lowered_normalized():
    """Coverage text vs index text: CanonicalizeText(Normalize(x)) == CanonicalizeText(ToLowerInvariant(Normalize(x))) (every token is
    lower-cased by GetCanonical, delimiters have no case) -- checked, not assumed."""
    pairs = [("nyc", "New York"), ("zs", "základní"), ("ſx", "SXX")]
    orc = SynOracleEngine(synonyms=pairs); L = O.lib()

    def normalize(s):
        a = O.u16(s); out = np.zeros(4 * len(a) + 8, np.uint16); n = L.ifxo_normalize(O._p(a), len(a), O._p(out), len(out)); return O.from_u16(out[:n])
    rng = np.random.Generator(np.random.PCG64(3))
    alphabet = list("aAbZzsS ÁáÄäSsſx-§.,  \tNnYyCc")
    for _ in range(500):
        x = "".join(rng.choice(alphabet, int(rng.integers(0, 20))))
        nx = normalize(x)
        assert orc.canonicalize(nx) == orc.canonicalize(S.to_lower_invariant(nx)), repr(x)


def test_builder_prepare_query():
    """The host builder's query preparation with a map: Trim, Normalize, ToLowerInvariant, CanonicalizeText, Normalize."""
    from infidex_b200 import engine as E                # no device needed: only the host library
    host = E._load_host()
    m = _map([("zs", "Základní"), ("nyc", "new york")])
    table = m.canonical_table()
    kb, ko = E.pack_strings([k for k, _ in table]); cb, co = E.pack_strings([c for _, c in table])
    ko32, co32 = ko.astype(np.uint32), co.astype(np.uint32)
    b = E.C.c_void_p(host.ifx_builder_create(0, None, None, None, None))
    keys = E._Strings(kb.ctypes.data, ko32.ctypes.data, len(table)); canon = E._Strings(cb.ctypes.data, co32.ctypes.data, len(table))
    assert host.ifx_builder_set_synonyms(b, E.C.byref(keys), E.C.byref(canon)) == 0

    def prep(t):
        a = O.u16(t); out = np.zeros(256, np.uint16); n = host.ifx_builder_prepare_query(b, O._p(a), len(a), O._p(out), len(out)); return O.from_u16(out[:n])
    assert prep("  ZS Brno ") == "zakladni brno"                  # the canonical form is normalised in the query only
    assert prep("x   NYC") == "x new york"                     # the whitespace token vanishes, the second Normalize collapses
    out = np.zeros(2, np.uint16); a = O.u16("zs")
    assert host.ifx_builder_prepare_query(b, O._p(a), 2, O._p(out), 2) == len("zakladni")   # the needed length, beyond the input's
    b2 = E.C.c_void_p(host.ifx_builder_create(0, None, None, None, None))
    bad_keys, bad_off = E.pack_strings(["ab", "AB"]); bo = bad_off.astype(np.uint32)
    cc, coo = E.pack_strings(["x", "y"]); c32 = coo.astype(np.uint32)
    assert host.ifx_builder_set_synonyms(b2, E.C.byref(E._Strings(bad_keys.ctypes.data, bo.ctypes.data, 2)), E.C.byref(E._Strings(cc.ctypes.data, c32.ctypes.data, 2))) != 0
    empty, eo = E.pack_strings(["ab", "cd"]); ce, ceo = E.pack_strings(["x", ""])
    assert host.ifx_builder_set_synonyms(b2, E.C.byref(E._Strings(empty.ctypes.data, eo.astype(np.uint32).ctypes.data, 2)),
                                         E.C.byref(E._Strings(ce.ctypes.data, ceo.astype(np.uint32).ctypes.data, 2))) != 0
    host.ifx_builder_destroy(b); host.ifx_builder_destroy(b2)
