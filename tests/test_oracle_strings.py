"""The Utf8 oracle (oracle/string_oracle.py) against the reference's known answers and against pyarrow.compute."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from blaze_b200 import exprs as E, types as T
from oracle import string_oracle as S
from string_kat_cases import STRING_MATCH_KATS, STRING_TO_BIGINT_KAT, TO_LONG_EDGE_CASES


def _eval(expr, values, name="s"):
    schema = T.Schema([T.Field(name, T.utf8, True)])
    cols = {name: [None if v is None else v.encode() for v in values]}
    return S.evaluate(expr, cols, schema, len(values))


@pytest.mark.parametrize("case", STRING_MATCH_KATS, ids=[c[0] for c in STRING_MATCH_KATS])
def test_string_match_kats(case):
    _, values, kind, pattern, scalar, expected = case
    operand = E.Column("s") if scalar is None else E.Literal(scalar, T.utf8)
    assert _eval(E.StringMatch(kind, operand, pattern), values) == expected


def test_string_to_bigint_kat():
    got = _eval(E.TryCast(E.Column("s"), T.int64), [v for v, _ in STRING_TO_BIGINT_KAT])
    assert got == [e for _, e in STRING_TO_BIGINT_KAT]


@pytest.mark.parametrize("case", TO_LONG_EDGE_CASES, ids=[f"{c[0]!r}-{c[1]}" for c in TO_LONG_EDGE_CASES])
def test_to_long_edge_cases(case):
    s, bits, expected = case
    assert S.to_long(s.encode(), bits) == expected


def random_strings(rng, n, null_frac=0.1):
    """empty strings, NULLs, mutual prefixes, bytes >= 0x80 (multi-byte UTF-8) and one long string"""
    alphabet = ["a", "b", "ab", "é", "ß", "€", "\U0001F600", "z", "\x7f", " "]
    out = []
    for i in range(n):
        r = rng.random()
        if r < null_frac:
            out.append(None)
        elif r < null_frac + 0.05:
            out.append("")
        else:
            out.append("".join(rng.choice(alphabet, rng.integers(1, 6))))
    out[n // 2] = "ab" * 3000
    return out


PATTERNS = ["", "a", "ab", "é", "€z", "\U0001F600", "abab"]


@pytest.mark.parametrize("seed", [0, 1])
def test_comparisons_against_pyarrow(seed):
    rng = np.random.default_rng(seed)
    a, b = random_strings(rng, 400), random_strings(rng, 400)
    schema = T.Schema([T.Field("a", T.utf8), T.Field("b", T.utf8)])
    cols = {"a": [None if v is None else v.encode() for v in a], "b": [None if v is None else v.encode() for v in b]}
    pa_a, pa_b = pa.array(a, pa.string()), pa.array(b, pa.string())
    for op, fn in [("Eq", pc.equal), ("NotEq", pc.not_equal), ("Lt", pc.less), ("LtEq", pc.less_equal), ("Gt", pc.greater), ("GtEq", pc.greater_equal)]:
        assert S.evaluate(E.BinaryExpr(E.Column("a"), op, E.Column("b")), cols, schema, 400) == fn(pa_a, pa_b).to_pylist(), op
        for lit in ["", "ab", "é", "b"]:
            got = S.evaluate(E.BinaryExpr(E.Column("a"), op, E.Literal(lit, T.utf8)), cols, schema, 400)
            assert got == fn(pa_a, pa.scalar(lit, pa.string())).to_pylist(), (op, lit)


@pytest.mark.parametrize("seed", [0, 1])
def test_matches_and_in_list_against_pyarrow(seed):
    rng = np.random.default_rng(seed)
    a = random_strings(rng, 500)
    pa_a = pa.array(a, pa.string())
    for p in PATTERNS:
        assert _eval(E.StartsWith(E.Column("s"), p), a) == pc.starts_with(pa_a, p).to_pylist(), p
        assert _eval(E.EndsWith(E.Column("s"), p), a) == pc.ends_with(pa_a, p).to_pylist(), p
        assert _eval(E.Contains(E.Column("s"), p), a) == pc.match_substring(pa_a, p).to_pylist(), p
    items = ["", "ab", "é", "b"]
    expected_in = [None if v is None else v in items for v in a]
    assert _eval(E.InList(E.Column("s"), [E.Literal(x, T.utf8) for x in items]), a) == expected_in
    assert pc.is_in(pa_a, value_set=pa.array(items)).to_pylist() == [False if v is None else v for v in expected_in]
    assert _eval(E.InList(E.Column("s"), [E.Literal(x, T.utf8) for x in items], negated=True), a) == [None if v is None else not v for v in expected_in]
    with_null = _eval(E.InList(E.Column("s"), [E.Literal("ab", T.utf8), E.Literal(None, T.utf8)]), a)
    assert with_null == [None if v is None else (True if v == "ab" else None) for v in a]
    assert _eval(E.IsNull(E.Column("s")), a) == [v is None for v in a]
    assert _eval(E.IsNotNull(E.Column("s")), a) == [v is not None for v in a]
