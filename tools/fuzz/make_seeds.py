"""Seeds for tools/fuzz: plans with every node / expression kind the decoder accepts (plan_decode_fuzz.cc); LZ4 frames written by the
library and by liblz4 (pyarrow) and batch_serde record streams over random schemas written by the oracle (ipc_fuzz.cc)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from blaze_b200 import exprs as E, plans as PL, types as T


def seed_plans():
    s = T.Schema([T.Field("a", T.int64, True), T.Field("b", T.int32, False), T.Field("d", T.decimal128(17, 2), True), T.Field("x", T.float64, True),
                  T.Field("t", T.date32, True), T.Field("o", T.bool_, True)])
    leaf = PL.MemoryExec(s)
    A, B, D, X, Dt, O = (E.Column(n) for n in "abdxto")
    f = PL.FilterExec([E.BinaryExpr(A, "Lt", E.Literal(5, T.int64)), E.IsNotNull(X), E.SCAnd(O, E.Not(E.IsNull(Dt))),
                       E.InList(B, [E.Literal(1, T.int32), E.Literal(None, T.int32), E.Literal(7, T.int32)], False)], leaf)
    proj = PL.ProjectExec([(E.BinaryExpr(A, "Plus", E.Cast(B, T.int64)), "c"),
                           (E.Case(None, [(E.BinaryExpr(X, "Gt", E.Literal(0.5, T.float64)), A)], E.Literal(None, T.int64)), "k"),
                           (E.TryCast(X, T.int32), "xi"), (E.Negative(A), "n"), (E.SCOr(O, E.Literal(True, T.bool_)), "oo"),
                           (E.ScalarFunction("UnscaledValue", [D], T.int64), "u"),
                           (E.ScalarFunction("CheckOverflow", [D, E.Literal(10, T.int32), E.Literal(1, T.int32)], T.decimal128(10, 1)), "co"),
                           (E.BinaryExpr(Dt, "GtEq", E.Literal(1000, T.date32)), "dd")], f)
    aggs = [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [D], s, T.decimal128(27, 2))), E.AggExpr("c", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [X], s, T.int64)),
            E.AggExpr("m", E.PARTIAL, PL.create_agg(E.AGG_MAX, [X], s, T.float64)), E.AggExpr("v", E.PARTIAL, PL.create_agg(E.AGG_AVG, [A], s, T.float64)),
            E.AggExpr("mn", E.PARTIAL, PL.create_agg(E.AGG_MIN, [B], s, T.int32))]
    partial = PL.AggExec(PL.HashAgg, [E.GroupingExpr("a", A), E.GroupingExpr("b", B)], aggs, True, f)
    specs = [(E.AGG_SUM, D, T.decimal128(27, 2)), (E.AGG_COUNT, X, T.int64), (E.AGG_MAX, X, T.float64), (E.AGG_AVG, A, T.float64), (E.AGG_MIN, B, T.int32)]
    fin = [E.AggExpr(a.field_name, E.FINAL, PL.create_agg(fn, [E.placeholder(ch.data_type(s))], partial.schema(), rt)) for a, (fn, ch, rt) in zip(aggs, specs)]
    final = PL.AggExec(PL.HashAgg, [E.GroupingExpr("a", A), E.GroupingExpr("b", B)], fin, False, partial)
    # Utf8: string nodes, comparisons, IN lists, TryCast(Utf8 -> int), COUNT / SUM(TryCast) over a string column
    su = T.Schema([T.Field("k", T.int64, False), T.Field("s", T.utf8, True), T.Field("t", T.utf8, True)])
    S_, T_ = E.Column("s"), E.Column("t")
    fs = PL.FilterExec([E.StartsWith(S_, "ab"), E.SCOr(E.EndsWith(S_, "é"), E.Contains(T_, "")), E.BinaryExpr(S_, "LtEq", T_),
                        E.InList(S_, [E.Literal("x", T.utf8), E.Literal(None, T.utf8), E.Literal("", T.utf8)], True),
                        E.BinaryExpr(E.Literal("b", T.utf8), "NotEq", S_), E.IsNotNull(T_)], PL.MemoryExec(su))
    ps = PL.ProjectExec([(E.Column("k"), "k"), (S_, "s"), (E.TryCast(T_, T.int32), "ti")], fs)
    sa = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))],
                    [E.AggExpr("c", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [S_], su, T.int64)),
                     E.AggExpr("n", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.TryCast(T_, T.int64)], su, T.int64))], False, fs)
    # ExpandExec: ROLLUP(a, b) below AggExec(Partial) (rolled-up keys as typed NULLs, the grouping id as a literal)
    xs = T.Schema([T.Field("a", T.int64, True), T.Field("b", T.int32, True), T.Field("d", T.decimal128(17, 2), True), T.Field("gid", T.int64, False)])
    n64, n32 = E.Literal(None, T.int64), E.Literal(None, T.int32)
    ex = PL.ExpandExec(xs, [[A, B, D, E.Literal(0, T.int64)], [A, n32, D, E.Literal(1, T.int64)], [n64, n32, D, E.Literal(3, T.int64)]], f)
    xa = PL.AggExec(PL.HashAgg, [E.GroupingExpr(n, E.Column(n)) for n in ("a", "b", "gid")],
                    [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("d")], xs, T.decimal128(27, 2)))], False, ex)
    return [proj.plan_bytes(), partial.plan_bytes(), final.plan_bytes(), ps.plan_bytes(), sa.plan_bytes(), xa.plan_bytes()]


if __name__ == "__main__":
    out = sys.argv[1]
    os.makedirs(out, exist_ok=True)
    for i, b in enumerate(seed_plans()):
        open(os.path.join(out, "seed%d.bin" % i), "wb").write(b)
    import decimal
    from blaze_b200 import proto
    lits = [(5, T.int64), (None, T.int32), (-3, T.int8), (1.5, T.float64), (2.5, T.float32), (True, T.bool_), (1000, T.date32), (7, T.int16),
            (decimal.Decimal("123.45"), T.decimal128(17, 2)), (None, T.null), (10**15, T.timestamp_us),
            ("abc", T.utf8), ("", T.utf8), (None, T.utf8), ("h\u00e9\u20ac\U0001F600" * 9, T.utf8)]
    for i, (v, dt) in enumerate(lits):
        open(os.path.join(out, "lit%d.bin" % i), "wb").write(proto.literal_ipc_bytes(v, dt))
    # LZ4 frames (ipc_fuzz --lz4): the library's encoder and liblz4 over byte planes, text, zeros and noise
    import numpy as np
    import pyarrow as pa
    from blaze_b200 import native
    rng = np.random.default_rng(3)
    datas = [b"", b"x", b"abcabcabcabca" * 9, np.frombuffer(rng.integers(-10**6, 10**6, 4000, dtype=np.int64).tobytes(), np.uint8).reshape(-1, 8).T.tobytes(),
             bytes(70_000), rng.integers(0, 256, 3000, dtype=np.uint8).tobytes()]
    for i, d in enumerate(datas):
        open(os.path.join(out, "lz4_lib%d.bin" % i), "wb").write(native.lz4_frame_compress(d))
        open(os.path.join(out, "lz4_pa%d.bin" % i), "wb").write(pa.Codec("lz4").compress(d, asbytes=True))
    # record streams (ipc_fuzz --records): [ncols][type ids][records], every type, with and without NULLs
    from oracle import blaze_oracle as O, shuffle_oracle as S
    cases = [[("a", pa.int64(), T.INT64), ("b", pa.binary(), T.BINARY)], [("c", pa.bool_(), T.BOOL), ("d", pa.int16(), T.INT16), ("e", pa.float64(), T.FLOAT64)],
             [("f", pa.decimal128(20, 2), T.DECIMAL128), ("g", pa.int32(), T.INT32), ("h", pa.binary(), T.BINARY), ("i", pa.int8(), T.INT8)]]
    for i, cols in enumerate(cases):
        raw = b""
        for n in (1, 7, 33):
            arrays = []
            for name, pt, tid in cols:
                mask = rng.random(n) < 0.3
                if tid == T.BINARY:
                    arrays.append(pa.array([None if m else bytes(rng.integers(0, 256, int(rng.integers(0, 9)), dtype=np.uint8)) for m in mask], pt))
                elif tid == T.BOOL:
                    arrays.append(pa.array(rng.random(n) < 0.5, pt, mask=mask))
                elif tid == T.DECIMAL128:
                    import decimal
                    arrays.append(pa.array([None if m else decimal.Decimal(int(rng.integers(-10**9, 10**9))).scaleb(-2) for m in mask], pt))
                else:
                    arrays.append(pa.array(np.where(mask, 0, rng.integers(-100, 100, n)).astype(pt.to_pandas_dtype()), pt, mask=mask))
            b = O.batch_from_arrow(pa.RecordBatch.from_arrays(arrays, names=[c[0] for c in cols]))
            raw += S.write_batch(n, b.cols)
        open(os.path.join(out, "rec_%d.bin" % i), "wb").write(bytes([len(cols)] + [c[2] for c in cols]) + raw)
