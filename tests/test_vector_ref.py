"""tests/vector_ref.py against the row-at-a-time oracles (oracle/join_oracle.py, oracle/sort_oracle.py) on the reference's
join goldens and on small seeded inputs with NULLs, duplicates, NaNs of both signs and with payloads, ±0 and ties — the
role tests/test_exact_agg_reference.py plays for tests/exact_agg.py.  No GPU."""
import numpy as np
import pyarrow as pa
import pytest

from blaze_b200 import plans as PL, types as T
from oracle import blaze_oracle as O
from oracle import join_oracle as J
from oracle import sort_oracle as S
from join_goldens import CASES, arrow_batches
import vector_ref as V

WIRE_TO_ORACLE = {PL.JOIN_INNER: J.INNER, PL.JOIN_LEFT: J.LEFT, PL.JOIN_RIGHT: J.RIGHT, PL.JOIN_FULL: J.FULL, PL.JOIN_SEMI: J.LEFT_SEMI,
                  PL.JOIN_ANTI: J.LEFT_ANTI, PL.JOIN_EXISTENCE: J.EXISTENCE}
ORACLE_TO_WIRE = {v: k for k, v in WIRE_TO_ORACLE.items()}
ALL_JOINS = list(WIRE_TO_ORACLE)


def _oracle_join(lb, rb, on_idx, jt, map_side):
    oj = J.HashJoin(T.from_arrow_schema(lb[0].schema), T.from_arrow_schema(rb[0].schema), on_idx, WIRE_TO_ORACLE[jt], "left" if map_side == V.LEFT_SIDE else "right")
    out = oj.execute([O.batch_from_arrow(b) for b in lb], [O.batch_from_arrow(b) for b in rb])
    return V.from_batches([O.batch_to_arrow(b) for b in out], len(oj.schema))


def _vector_join(lb, rb, on_idx, jt, map_side):
    return V.join(V.from_batches(lb), V.from_batches(rb), on_idx, jt, map_side)


@pytest.mark.parametrize("map_side", [V.LEFT_SIDE, V.RIGHT_SIDE])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_join_goldens(case, map_side):
    name, left, right, on, jt, expected = case[:6]
    lb, rb = arrow_batches(left, case[6] if len(case) > 6 else "int32"), arrow_batches(right, case[6] if len(case) > 6 else "int32")
    on_idx = [(lb[0].schema.names.index(a), rb[0].schema.names.index(b)) for a, b in on]
    got = _vector_join(lb, rb, on_idx, ORACLE_TO_WIRE[jt], map_side)
    assert len(got[0]) == len(expected)
    V.assert_same_rows(got, _oracle_join(lb, rb, on_idx, ORACLE_TO_WIRE[jt], map_side))


def _random_side(rng, n, tag, key_type, krange, null_frac):
    def nulls():
        return rng.random(n) >= null_frac
    k = rng.integers(-krange, krange, n)
    cols = [V.to_arrow(key_type, k.astype(key_type.to_pandas_dtype()), nulls()),
            V.to_arrow(pa.int8(), rng.integers(-2, 2, n).astype(np.int8), nulls()),
            V.to_arrow(pa.float64(), rng.normal(size=n), nulls()),
            V.to_arrow(pa.decimal128(38, 0), rng.integers(-2**62, 2**62, (n, 2)).view(np.uint64), nulls()),
            V.to_arrow(pa.int16(), rng.integers(-500, 500, n).astype(np.int16))]
    return pa.RecordBatch.from_arrays(cols, names=[f"k{tag}", f"j{tag}", f"x{tag}", f"d{tag}", f"s{tag}"])


@pytest.mark.parametrize("map_side", [V.LEFT_SIDE, V.RIGHT_SIDE])
@pytest.mark.parametrize("jt", ALL_JOINS, ids=lambda j: J.NAMES[WIRE_TO_ORACLE[j]])
@pytest.mark.parametrize("variant", ["int32 key", "int8 x int64 keys", "two keys + nulls"])
def test_random_joins(jt, map_side, variant):
    rng = np.random.default_rng(7 + jt)
    two = variant.startswith("two")
    lt, rt = (pa.int8(), pa.int64()) if variant.startswith("int8") else (pa.int32(), pa.int32())
    l = _random_side(rng, 700, "l", lt, 60, 0.1 if two else 0.02)
    r = _random_side(rng, 400, "r", rt, 80 if not variant.startswith("int8") else 300, 0.1 if two else 0.0)
    on_idx = [(0, 0)] + ([(1, 1)] if two else [])
    lb, rb = [l.slice(0, 301), l.slice(301)], [r.slice(0, 5), r.slice(5)]
    V.assert_same_rows(_vector_join(lb, rb, on_idx, jt, map_side), _oracle_join(lb, rb, on_idx, jt, map_side))


def test_join_keys_compare_by_value_across_widths():
    """int8 -1 meets int64 -1 (not 255), and int64 256 + 5 does not meet int8 5"""
    l = pa.RecordBatch.from_arrays([pa.array([-1, 5, -128, 127, 0], pa.int8())], names=["a"])
    r = pa.RecordBatch.from_arrays([pa.array([255, -1, 261, 5, -128, 127, 128, -129], pa.int64())], names=["b"])
    got = V.join(V.from_batches([l]), V.from_batches([r]), [(0, 0)], V.INNER, V.RIGHT_SIDE)
    assert sorted(zip(got[0].values.tolist(), got[1].values.tolist())) == [(-128, -128), (-1, -1), (5, 5), (127, 127)]


# ---- sort ----------------------------------------------------------------------------------------------------------

F64_SPECIAL = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF00000DEADBEEF, 0x7FF0000000000000, 0xFFF0000000000000,
                        0, 1 << 63, 1, (1 << 63) | 1, 0x3FF0000000000000, 0xBFF0000000000000], np.uint64)
# f32 NaN payloads are quiet here: the oracle widens an f32 to a Python float, which sets the quiet bit of a signalling NaN
F32_SPECIAL = np.array([0x7FC00000, 0xFFC00000, 0x7FC00001, 0xFFC12345,0x7F800000, 0xFF800000, 0, 1 << 31, 1, (1 << 31) | 1, 0x3F800000, 0xBF800000], np.uint32)


def _sort_table(rng, n):
    def pick(special, random_bits):
        v = random_bits.copy()
        m = rng.random(n) < 0.5
        v[m] = special[rng.integers(0, len(special), int(m.sum()))]
        return v
    dec = rng.integers(-3, 3, (n, 2)).view(np.uint64)
    dec[::7] = [(2**64 - 1, 2**63 - 1)]
    cols = [V.to_arrow(pa.int8(), rng.integers(-128, 128, n).astype(np.int8), rng.random(n) > 0.1),
            V.to_arrow(pa.int16(), rng.choice(np.array([-2**15, 2**15 - 1, -1, 0, 7], np.int16), n)),
            V.to_arrow(pa.int64(), rng.choice(np.array([-2**63, 2**63 - 1, -1, 0], np.int64), n), rng.random(n) > 0.2),
            V.to_arrow(pa.float64(), pick(F64_SPECIAL, rng.normal(size=n).view(np.uint64)), rng.random(n) > 0.1),
            V.to_arrow(pa.float32(), pick(F32_SPECIAL, rng.normal(size=n).astype(np.float32).view(np.uint32)), rng.random(n) > 0.1),
            V.to_arrow(pa.decimal128(38, 0), dec, rng.random(n) > 0.1),
            V.to_arrow(pa.date32(), rng.integers(-3, 3, n).astype(np.int32)),
            V.to_arrow(pa.int64(), np.arange(n, dtype=np.int64))]
    return pa.RecordBatch.from_arrays(cols, names=["i8", "i16", "i64", "f64", "f32", "dec", "d", "row"])


SORTS = {
    "f64 asc nulls last": [(3, False, False)],
    "f64 desc nulls first": [(3, True, True)],
    "f32 asc nulls first": [(4, False, True)],
    "f32 desc nulls last": [(4, True, False)],
    "decimal asc": [(5, False, True)],
    "decimal desc nulls last": [(5, True, False)],
    "int16 desc, int64 asc nulls last": [(1, True, True), (2, False, False)],
    "date asc, int8 desc, f64 asc": [(6, False, True), (0, True, False), (3, False, True)],
    "int8 asc (ties)": [(0, False, True)],
}


@pytest.mark.parametrize("case", list(SORTS))
def test_sort_matches_the_oracle_row_for_row(case):
    rb = _sort_table(np.random.default_rng(11), 1500)
    batches = [rb.slice(0, 600), rb.slice(600)]
    exprs = SORTS[case]
    exp = S.sort_exec([O.batch_from_arrow(b) for b in batches], exprs)
    perm = V.sort_permutation(V.from_batches(batches), exprs)
    assert perm.tolist() == [int(x) for x in exp.cols[7].values]              # the same stable permutation
    got = V.sort(V.from_batches(batches), exprs)
    V.assert_same_columns(got, V.from_batches([O.batch_to_arrow(exp)]))
    assert V.sort(V.from_batches(batches), exprs, fetch=17)[7].values.tolist() == perm[:17].tolist()


def test_total_order_of_the_float_specials():
    x = V.col_from_arrow(V.to_arrow(pa.float64(), F64_SPECIAL))
    order = V.sort_permutation([x], [(0, False, True)])
    assert [hex(int(F64_SPECIAL[i])) for i in order] == [hex(v) for v in (0xFFF8000000000000, 0xFFF00000DEADBEEF, 0xFFF0000000000000, 0xBFF0000000000000,
                                                                          (1 << 63) | 1, 1 << 63, 0, 1, 0x3FF0000000000000, 0x7FF0000000000000, 0x7FF0000000000001,
                                                                          0x7FF8000000000000)]


def test_total_order_of_f32_signalling_nans():
    """raw f32 bits keep a signalling NaN's payload: 0x7F800001 sorts below the quiet 0x7FC00000"""
    bits = np.array([0x7FC00000, 0x7F800001, 0xFFC00000, 0xFF800001, 0x7F800000, 0x00000001, 0x80000001], np.uint32)
    x = V.col_from_arrow(V.to_arrow(pa.float32(), bits))
    assert V.sort_permutation([x], [(0, False, True)]).tolist() == [2, 3, 6, 5, 4, 1, 0]


def test_decimal_words():
    """the high word decides first and is signed; the low word is unsigned: -1 < 0 < 2^63 - 1 < 2^63 < 2^64 < 10^38 - 1"""
    vals = [10**38 - 1, 2**64, 2**63, 2**63 - 1, 0, -1, -(2**64), -(10**38 - 1)]
    raw = np.array([[v & (2**64 - 1), (v >> 64) & (2**64 - 1)] for v in vals], np.uint64)
    c = V.col_from_arrow(V.to_arrow(pa.decimal128(38, 0), raw))
    assert V.sort_permutation([c], [(0, False, True)]).tolist() == [7, 6, 5, 4, 3, 2, 1, 0]
    assert V.sort_permutation([c], [(0, True, True)]).tolist() == list(range(8))


def test_comparator_is_bit_exact():
    a = V.col_from_arrow(pa.array([0.0, float("nan")], pa.float64()))
    b = V.col_from_arrow(pa.array([-0.0, float("nan")], pa.float64()))
    with pytest.raises(AssertionError):
        V.assert_same_columns([a], [b])
    c = V.col_from_arrow(V.to_arrow(pa.float64(), np.array([0, 0xFFF8000000000000], np.uint64)))
    with pytest.raises(AssertionError):
        V.assert_same_columns([V.col_from_arrow(pa.array([0.0, float("nan")], pa.float64()))], [c])
    V.assert_same_rows([a, V.col_from_arrow(pa.array([1, None]))], [a.take([1, 0]), V.col_from_arrow(pa.array([None, 1]))])
