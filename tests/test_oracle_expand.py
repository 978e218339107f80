"""The oracle's ExpandExec against the reference's KATs (tests/golden/expand_kats.json), and its try_new checks."""
import pytest

from blaze_b200 import exprs as E, types as T
from blaze_b200.types import Field, Schema
from oracle import blaze_oracle as O
from oracle import expand_oracle as X

from expand_cases import KATS, kat_input, kat_projections, kat_text


@pytest.mark.parametrize("case", KATS, ids=[c["name"] for c in KATS])
def test_oracle_kats(case):
    schema, rb = kat_input(case)
    ex = X.ExpandExec(schema, kat_projections(case), schema)
    out = ex.execute([O.batch_from_arrow(rb)])
    assert len(out) == len(case["expected"])                              # one batch per projection, in order
    for b, exp in zip(out, case["expected"]):
        assert b.cols[0].valid.all()
        assert kat_text(case, b.cols[0].values.tolist()) == exp


def test_oracle_type_mismatch_and_short_projection():
    s = Schema([Field("a", T.int32, False)])
    with pytest.raises(X.OracleError, match="ExpandExec data type not matches"):
        X.ExpandExec(Schema([Field("a", T.int64, False)]), [[E.Column("a")]], s)
    with pytest.raises(X.OracleError, match="ExpandExec data type not matches"):
        X.ExpandExec(Schema([Field("a", T.int32, False), Field("b", T.int32, False)]), [[E.Column("a")]], s)


def test_oracle_extra_expressions_and_zero_projections():
    schema, rb = kat_input(KATS[0])
    ex = X.ExpandExec(schema, [[E.Column("a"), E.Literal(7, T.int64)]], schema)
    (b,) = ex.execute([O.batch_from_arrow(rb)])
    assert len(b.cols) == 1 and b.cols[0].values.tolist() == [-1, -2, 0, 3]
    assert X.ExpandExec(schema, [], schema).execute([O.batch_from_arrow(rb)]) == []
