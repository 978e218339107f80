"""CPU restatement of the reference's hash join (BroadcastJoinExec / HashJoinExec, SURVEY.md §8(f) rank 2) — TEST
INFRASTRUCTURE ONLY (tests/, smoke and bench's cpu_baseline may import it; the product never does).

Paths relative to the reference's native-engine/datafusion-ext-plans/src/:
  JoinHashMap / Table::create_from_key_columns / lookup_many      joins/join_hash_map.rs:91-275 (rows whose key has a NULL
                                                                  are left out of the map :119-128; duplicates of a key sit in
                                                                  one `mapped_indices` range in row order :129-143)
  FullJoiner (Inner / Left / Right / Full, probe side L or R)      joins/bhj/full_join.rs:90-379
  SemiJoiner (LeftSemi / LeftAnti / RightSemi / RightAnti /       joins/bhj/semi_join.rs:100-327
              Existence)
  joiner selection by (broadcast side, join type)                 broadcast_join_exec.rs:317-385
  output schema                                                   joins/test.rs:163-176 + DataFusion build_join_schema: left ++ right
                                                                  with the non-preserved side made nullable; Existence =
                                                                  left ++ `exists#0: Boolean not null`
The slot placement hash (foldhash, join_hash_map.rs:441-457) only decides where a key sits in the table: unobservable.
Key equality is value equality per column (EqComparator); a NULL in any key column never matches (full_join.rs:262-267).

Pinned by the reference's own goldens: all 18 tests of joins/test.rs:275-985 for the four hash-join drivers
(BHJLeftProbed / BHJRightProbed / SHJLeftProbed / SHJRightProbed) — tests/test_join_oracle.py.  Like the reference's
`assert_batches_sorted_eq!`, the comparison is on the multiset of rows.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from blaze_b200 import types as T
from blaze_b200.types import Field, Schema
from oracle import blaze_oracle as O
from oracle.blaze_oracle import Batch, Col

INNER, LEFT, RIGHT, FULL, LEFT_ANTI, RIGHT_ANTI, LEFT_SEMI, RIGHT_SEMI, EXISTENCE = range(9)     # joins/join_utils.rs:18-29
NAMES = ["Inner", "Left", "Right", "Full", "LeftAnti", "RightAnti", "LeftSemi", "RightSemi", "Existence"]


def join_schema(left: Schema, right: Schema, join_type: int) -> Schema:
    if join_type == EXISTENCE:
        return Schema(list(left) + [Field("exists#0", T.bool_, False)])
    if join_type in (LEFT_SEMI, LEFT_ANTI):
        return Schema(list(left))
    if join_type in (RIGHT_SEMI, RIGHT_ANTI):
        return Schema(list(right))
    ln = join_type in (RIGHT, FULL)          # left side becomes nullable
    rn = join_type in (LEFT, FULL)
    return Schema([Field(f.name, f.dtype, f.nullable or ln) for f in left] + [Field(f.name, f.dtype, f.nullable or rn) for f in right])


def _key(cols: Sequence[Col], r: int) -> Optional[tuple]:
    k = []
    for c in cols:
        if not c.valid[r]:
            return None
        v = c.values[r]
        k.append(v.item() if hasattr(v, "item") else v)
    return tuple(k)


def _take_nullable(b: Batch, idx: Sequence[Optional[int]]) -> List[Col]:
    """take_cols with Option<u32> indices: None -> NULL row (full_join.rs:147-152,197)"""
    n = len(idx)
    sel = np.array([0 if i is None else i for i in idx], np.int64)
    isnull = np.array([i is None for i in idx], bool)
    out = []
    for c in b.cols:
        if b.num_rows == 0:
            out.append(Col.nulls(c.dtype, n))
            continue
        vals = c.values[sel] if n else c.values[:0]
        valid = (c.valid[sel] & ~isnull) if n else c.valid[:0]
        if n and c.dtype.id in (T.DECIMAL128, T.BINARY):
            vals = vals.copy()
        out.append(Col(c.dtype, vals, valid))
    return out


class HashJoin:
    """BroadcastJoinExec::execute with a built map (broadcast_join_exec.rs:317-385, 496-560): `build_side` is the side
    whose rows are in the hash map ("left" | "right"), the other side is probed batch by batch."""

    def __init__(self, left_schema: Schema, right_schema: Schema, on: Sequence[Tuple[int, int]], join_type: int, build_side: str):
        self.ls, self.rs, self.on, self.jt, self.build_side = left_schema, right_schema, list(on), join_type, build_side
        self.schema = join_schema(left_schema, right_schema, join_type)

    def execute(self, left: Sequence[Batch], right: Sequence[Batch]) -> List[Batch]:
        build_is_left = self.build_side == "left"
        bschema, pschema = (self.ls, self.rs) if build_is_left else (self.rs, self.ls)
        build = O.concat_batches(bschema, list(left if build_is_left else right))
        probes = list(right if build_is_left else left)
        bkeys = [build.cols[(l if build_is_left else r)] for l, r in self.on]
        table = {}
        for i in range(build.num_rows):                                  # join_hash_map.rs:119-143: NULL keys are not inserted
            k = _key(bkeys, i)
            if k is not None:
                table.setdefault(k, []).append(i)
        jt = self.jt
        probe_is_left = not build_is_left
        # which side's rows the output is made of, and the outer flags (full_join.rs:71-79, semi_join.rs:78-87)
        probe_outer = (jt == FULL) or (jt == LEFT and probe_is_left) or (jt == RIGHT and not probe_is_left)
        build_outer = (jt == FULL) or (jt == LEFT and not probe_is_left) or (jt == RIGHT and probe_is_left)
        semi_like = jt in (LEFT_SEMI, LEFT_ANTI, RIGHT_SEMI, RIGHT_ANTI, EXISTENCE)
        probe_is_join_side = (jt in (LEFT_SEMI, LEFT_ANTI, EXISTENCE) and probe_is_left) or (jt in (RIGHT_SEMI, RIGHT_ANTI) and not probe_is_left)
        map_joined = np.zeros(build.num_rows, bool)
        out: List[Batch] = []

        def emit(pcols: List[Col], bcols: List[Col], n: int):
            cols = (pcols + bcols) if probe_is_left else (bcols + pcols)
            out.append(Batch(self.schema, [Col(f.dtype, c.values, c.valid) for f, c in zip(self.schema, cols)], n))

        for pb in probes:
            pkeys = [pb.cols[(r if build_is_left else l)] for l, r in self.on]
            if not semi_like:
                pi, bi = [], []
                for r in range(pb.num_rows):
                    k = _key(pkeys, r)
                    matches = table.get(k, []) if k is not None else []
                    for m in matches:
                        pi.append(r); bi.append(m)
                    if probe_outer and not matches:
                        pi.append(r); bi.append(None)
                if build_outer:
                    for m in bi:
                        if m is not None:
                            map_joined[m] = True
                if pi:
                    emit(_take_nullable(pb, pi), _take_nullable(build, bi), len(pi))
            else:
                joined = np.zeros(pb.num_rows, bool)
                for r in range(pb.num_rows):
                    k = _key(pkeys, r)
                    matches = table.get(k, []) if k is not None else []
                    if matches:
                        if probe_is_join_side:
                            joined[r] = True
                        else:
                            map_joined[matches] = True
                if probe_is_join_side:
                    if jt == EXISTENCE:
                        cols = [Col(c.dtype, c.values, c.valid) for c in pb.cols] + [Col(T.bool_, joined.copy(), np.ones(pb.num_rows, bool))]
                        out.append(Batch(self.schema, cols, pb.num_rows))
                    else:
                        keep = np.nonzero(joined if jt in (LEFT_SEMI, RIGHT_SEMI) else ~joined)[0]
                        out.append(Batch(self.schema, [c.take(keep) for c in pb.cols], len(keep)))
        # finish (full_join.rs:322-362, semi_join.rs:276-312)
        if not semi_like and build_outer:
            un = [int(i) for i in np.nonzero(~map_joined)[0]]
            if un:
                pnull = Batch(pschema, [Col.nulls(f.dtype, 0) for f in pschema], 0)
                emit(_take_nullable(pnull, [None] * len(un)), _take_nullable(build, un), len(un))
        if semi_like and not probe_is_join_side:
            if jt == EXISTENCE:
                cols = [Col(c.dtype, c.values, c.valid) for c in build.cols] + [Col(T.bool_, map_joined.copy(), np.ones(build.num_rows, bool))]
                out.append(Batch(self.schema, cols, build.num_rows))
            else:
                keep = np.nonzero(map_joined if jt in (LEFT_SEMI, RIGHT_SEMI) else ~map_joined)[0]
                out.append(Batch(self.schema, [c.take(keep) for c in build.cols], len(keep)))
        return [b for b in out if b.num_rows > 0]
