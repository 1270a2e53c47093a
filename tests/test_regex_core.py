"""The regular-expression compiler and DFA walk of PQ_OP_REGEX on the CPU (tools/libregex_host.so), and the SQL front end.

* random patterns of the supported grammar without Perl classes against RE2 (pyarrow.compute.match_substring_regex);
* \\d \\s \\w over every scalar value against perl's \\p{Nd}, \\p{XPerlSpace}, \\p{Word}, and every simple case folding orbit;
* a known-answer table for the Unicode behaviour where RE2 differs from the regex crate;
* every refusal, the size caps, and random bytes as patterns: always a status code, never a crash or a hang."""
import ctypes as C
import os
import shutil
import subprocess
import time

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from parseable_b200 import _lib as L
from parseable_b200.query import Query, QueryError, _Desc, col

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rx(built):
    lib = C.CDLL(os.path.join(ROOT, "tools", "libregex_host.so"))
    lib.rx_compile.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_char_p, C.c_uint64]
    lib.rx_match_many.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


def compile_(lib, pat, ci=False):
    b = pat.encode() if isinstance(pat, str) else pat
    cap = 4 << 20
    blob = C.create_string_buffer(cap)
    n = C.c_uint64()
    err = C.create_string_buffer(512)
    st_ = lib.rx_compile(b, len(b), int(ci), blob, cap, C.byref(n), err, 512)
    return st_, blob.raw[:n.value] if st_ == 0 else b"", err.value.decode()


def match_all(lib, pat, hays, ci=False):
    st_, blob, err = compile_(lib, pat, ci)
    assert st_ == 0, (pat, err)
    enc = [h.encode() for h in hays]
    off = np.zeros(len(enc) + 1, np.int64)
    off[1:] = np.cumsum([len(e) for e in enc])
    data = np.frombuffer(b"".join(enc) + b"\0", np.uint8)
    out = np.zeros(len(enc), np.uint8)
    lib.rx_match_many(blob, data.ctypes.data, off.ctypes.data, len(enc), out.ctypes.data)
    return out.astype(bool).tolist()


# ---- random patterns vs RE2 -------------------------------------------------------------------------------------
ALPHABET = ["a", "b", "c", "A", "B", "x", "0", "1", " ", "-", "\n", "é", "É", "δ", "Δ", "K", "k", "s", "S", "ſ", "\u212a", "日", "本", "🙂"]
LITS = ["a", "b", "c", "A", "x", "0", "1", " ", "-", "é", "É", "δ", "Δ", "K", "k", "s", "S", "ſ", "\u212a", "日", "🙂", r"\.", r"\-",
        r"\n", r"\t", r"\x61", r"\x{e9}", "."]
CLASSES = ["[abc]", "[^a]", "[a-c]", "[A-Za-z]", "[0-9]", "[éδ]", "[^\\n]", "[Δ-Ω]", "[k]", "[s-t]", "[-a]", "[a-]", "[^x-z0]"]


def _atoms():
    return st.sampled_from(LITS + CLASSES + ["^", "$", r"\A", r"\z"])


def _regex():
    def extend(inner):
        rep = st.tuples(inner, st.sampled_from(["*", "+", "?", "{2}", "{1,2}", "{0,}", "{2,3}", "*?", "+?", "??", "{1,2}?"])).map(
            lambda t: f"(?:{t[0]}){t[1]}")
        cat = st.lists(inner, min_size=2, max_size=4).map("".join)
        alt = st.lists(inner, min_size=2, max_size=3).map(lambda xs: "(" + "|".join(xs) + ")")
        flg = st.tuples(st.sampled_from(["i", "m", "s", "is", "im", "ms", "-i", "i-s", "U"]), inner).map(lambda t: f"(?{t[0]}:{t[1]})")
        named = inner.map(lambda x: f"(?P<g>{x})")
        return st.one_of(rep, cat, alt, flg, named)
    body = st.recursive(_atoms(), extend, max_leaves=8)
    return st.tuples(st.sampled_from(["", "(?i)", "(?m)", "(?s)", "(?im)", "(?is)"]), body).map("".join)


HAYS = st.lists(st.text(alphabet=st.sampled_from(ALPHABET), min_size=0, max_size=10), min_size=25, max_size=40)
AGREED = []


@settings(max_examples=1500, deadline=None, suppress_health_check=list(HealthCheck))
@given(pat=_regex(), hays=HAYS)
def test_random_patterns_agree_with_re2(rx, pat, hays):
    hays = hays + ["", "a\nb", "\u212a", "ſ"]
    st_, _, err = compile_(rx, pat)
    if st_ != 0:   # a pattern past the DFA caps is refused, never guessed at; nested groups may repeat the name `g`
        assert (st_ == L.PQ_ERR_UNSUPPORTED and "too large" in err) or "duplicate capture group name" in err, (pat, err)
        return
    want = pc.match_substring_regex(pa.array(hays, pa.string()), pat).to_pylist()
    got = match_all(rx, pat, hays)
    assert got == want, (pat, [h for h, g, w in zip(hays, got, want) if g != w])
    AGREED.append(len(hays))


def test_random_patterns_count(rx):
    """The random comparison above covered at least 20 000 (pattern, haystack) pairs."""
    if not AGREED:
        pytest.skip("runs after test_random_patterns_agree_with_re2")
    assert sum(AGREED) >= 20_000, sum(AGREED)


# ---- Unicode tables vs perl ---------------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("perl") is None, reason="perl is not installed")
def test_perl_classes_and_fold_orbits_over_every_scalar_value(rx):
    perl = ("for my $c (0 .. 0x10FFFF) { next if $c >= 0xD800 && $c <= 0xDFFF; my $s = chr($c);"
            " print(($s =~ /\\p{Nd}/ ? 1 : 0), ($s =~ /\\p{XPerlSpace}/ ? 1 : 0), ($s =~ /\\p{Word}/ ? 1 : 0)); }")
    bits = subprocess.check_output(["perl", "-e", perl])
    cps = [c for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]
    want = np.frombuffer(bits, np.uint8).reshape(-1, 3) - ord("0")
    hays = [chr(c) for c in cps]
    for j, pat in enumerate([r"^\d$", r"^\s$", r"^\w$"]):
        got = np.array(match_all(rx, pat, hays), np.uint8)
        bad = np.flatnonzero(got != want[:, j])
        assert bad.size == 0, (pat, [hex(cps[i]) for i in bad[:10]])
    # every simple case folding orbit: each member matches each other under (?i)
    perl = ("use Unicode::UCD qw(all_casefolds); my $h = all_casefolds();"
            " for my $k (keys %$h) { my $r = $h->{$k}; next if $r->{simple} eq ''; print hex($r->{code}), ' ', hex($r->{simple}), \"\\n\"; }")
    orbits = {}
    for line in subprocess.check_output(["perl", "-e", perl]).decode().split("\n"):
        if line:
            a, b = map(int, line.split())
            orbits.setdefault(b, {b}).add(a)
    for members in orbits.values():
        for m in members:
            pat = "^" + "\\x{%x}" % m + "$"
            assert all(match_all(rx, pat, [chr(o) for o in members], ci=True)), [hex(o) for o in members]


# ---- known answers ----------------------------------------------------------------------------------------------
KNOWN = [
    ("١٢", r"\d", True), ("\v", r"\s", True), ("\u0085", r"\s", True), ("é", r"^\w+$", True), ("\u200d", r"\w", True),
    ("\u212a", "(?i)k", True), ("\u017f", "(?i)S", True), ("a\nb", "a$", False), ("a\nb", "(?m)a$", True),
    ("a\nb", "(?m)^b", True), ("a\nb", "^b", False), ("a\r\nb", "(?m)a$", False), ("", "", True), ("x", "", True),
    ("\n", ".", False), ("\n", "(?s).", True), ("\n", "[^a]", True), ("日本", "^..$", True), ("a\nb", r"\Aa", True),
    ("a\nb", r"(?m)b\z", True), ("a\nb", r"(?m)a\z", False), ("ab", "(?i)(?-i:A)b", False), ("Ab", "(?i:a)B", False),
    ("ß", "(?i)ẞ", True), ("Σ", "(?i)ς", True), ("x1", r"\D\d", True), ("a b", r"\S\s\S", True), ("é", r"\W", False),
    ("-", r"\W", True), ("a+b", r"a\+b", True), ("a b", r"a\ b", True), ("Ω", r"[Α-Ω]", True), ("ω", r"(?i)[Α-Ω]", True),
    ("ab", "a|", True), ("", "a|", True), ("aaa", "a{3}", True), ("aa", "^a{3,}$", False), ("\u00e9", r"\x{e9}", True),
    ("\u00e9", r"\u00e9", True), ("🙂", r"\U0001F642", True), ("🙂", r"\u{1F642}", True), ("\x07", r"\a", True),
]


@pytest.mark.parametrize("hay,pat,want", KNOWN)
def test_known_answers(rx, hay, pat, want):
    assert match_all(rx, pat, [hay]) == [want]


# ---- refusals and caps ------------------------------------------------------------------------------------------
INVALID = ["(", "a)", "(a", "[a", "[]", "[^]", "*", "+a", "a{2,1}", "[z-a]", r"\q", r"\1", r"\0", "(?=a)", "(?!a)", "(?<=a)",
           "(?<!a)", "(?z)", "(?ii)", "(?i-)", "(?)", "(?P<n>a)(?P<n>b)", "(?P<>a)", "(?P<1a>a)", "a{", "a{x}", "a{1",
           r"\x{110000}", r"\x{d800}", r"\xZZ", "\\", r"[a-\d]", "(?i)*", r"\Z", r"\e"]
UNSUPPORTED = [r"\b", r"\B", r"\<", r"\>", r"\b{start}", r"\pL", r"\p{Greek}", r"\PL", "[[:alpha:]]", "[a[b]]", "[a&&b]",
               "[a--b]", "[a~~b]", "(?x)a", "(?R)a", "(?-u)a", "a{,3}", "(" * 300 + ")" * 300]


@pytest.mark.parametrize("pat", INVALID)
def test_invalid_patterns(rx, pat):
    st_, _, err = compile_(rx, pat)
    assert st_ == L.PQ_ERR_INVALID_ARG, (pat, st_, err)
    assert "at byte" in err


@pytest.mark.parametrize("pat", UNSUPPORTED)
def test_unsupported_patterns(rx, pat):
    st_, _, err = compile_(rx, pat)
    assert st_ == L.PQ_ERR_UNSUPPORTED, (pat, st_, err)


@pytest.mark.parametrize("pat,what", [("(a|b){1000}{1000}", "NFA"), ("(a|b)*a(a|b){20}", "DFA states"),
                                      ("a" * (64 * 1024 + 1), "64 KiB"), (r"(\w|\s|\d){3000}", "NFA")])
def test_caps(rx, pat, what):
    t = time.time()
    st_, _, err = compile_(rx, pat)
    assert st_ == L.PQ_ERR_UNSUPPORTED and "too large for the device DFA" in err and what in err, err
    assert time.time() - t < 30


def test_random_bytes_as_patterns(rx):
    rng = np.random.default_rng(7)
    meta = list(b"()[]{}|*+?.^$\\-,:<>=!iPmsux0123456789dDwWsSbBApz") + [0xC3, 0xA9, 0xFF]
    for k in range(3000):
        n = int(rng.integers(0, 24))
        src = rng.integers(0, 256, n) if k % 2 else np.array(meta)[rng.integers(0, len(meta), n)]
        st_, _, _ = compile_(rx, bytes(int(b) for b in src))
        assert st_ in (0, L.PQ_ERR_INVALID_ARG, L.PQ_ERR_UNSUPPORTED)


def test_invalid_utf8_pattern(rx):
    assert compile_(rx, b"a\xffb")[0] == L.PQ_ERR_INVALID_ARG


# ---- SQL ----------------------------------------------------------------------------------------------------------
def ops_of(sql):
    q = Query(sql)
    d = _Desc()
    ops = []
    d.compile_pred(q.where, ops)
    return ops


def test_sql_regex_operators(built):
    kinds = lambda ops: [o.kind for o in ops]   # noqa: E731
    for op, flags in (("~", 0), ("~*", L.PQ_REGEX_CASE_INSENSITIVE), ("!~", L.PQ_REGEX_NEGATED),
                      ("!~*", L.PQ_REGEX_NEGATED | L.PQ_REGEX_CASE_INSENSITIVE)):
        ops = ops_of(f"SELECT * FROM s WHERE message {op} 'timeout after \\d+ ms' AND level = 'ERROR'")
        assert kinds(ops) == [L.PQ_OP_REGEX, L.PQ_OP_CMP, L.PQ_OP_AND]
        assert ops[0].flags == flags and ops[0].lit.str[:ops[0].lit.str_len] == b"timeout after \\d+ ms"
    ops = ops_of("SELECT * FROM s WHERE regexp_like(host, '^web-0[0-9]$')")
    assert kinds(ops) == [L.PQ_OP_REGEX] and ops[0].flags == 0 and ops[0].lit.str[:ops[0].lit.str_len] == b"^web-0[0-9]$"
    ops = ops_of("SELECT * FROM s WHERE regexp_like(host, 'WEB', 'im')")
    assert ops[0].lit.str[:ops[0].lit.str_len] == b"(?im)WEB"
    ops = ops_of("SELECT * FROM s WHERE NOT regexp_like(host, 'it''s') OR level ~ ''")
    assert kinds(ops) == [L.PQ_OP_REGEX, L.PQ_OP_NOT, L.PQ_OP_REGEX, L.PQ_OP_OR]
    assert ops[0].lit.str[:ops[0].lit.str_len] == b"it's" and ops[2].lit.str_len == 0
    e = col("path").regex("^/api/v[12]/", negated=True, case_insensitive=True)
    assert e.kind == "regex" and e.flags == 3


@pytest.mark.parametrize("sql,code", [
    ("SELECT * FROM s WHERE message ~ level", L.PQ_ERR_UNSUPPORTED),
    ("SELECT * FROM s WHERE regexp_like(host, level)", L.PQ_ERR_UNSUPPORTED),
    ("SELECT * FROM s WHERE regexp_like(host, 'a', 'g')", L.PQ_ERR_INVALID_ARG),
    ("SELECT * FROM s WHERE regexp_match(host, 'a')", L.PQ_ERR_UNSUPPORTED),
    ("SELECT regexp_replace(host, 'a', 'b') FROM s", L.PQ_ERR_UNSUPPORTED),
])
def test_sql_regex_refusals(built, sql, code):
    with pytest.raises(QueryError) as ei:
        ops_of(sql)
    assert ei.value.code == code, ei.value
