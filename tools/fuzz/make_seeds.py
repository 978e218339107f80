"""Seed plans for tools/fuzz/plan_decode_fuzz.cc: every node / expression kind the decoder accepts."""
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
