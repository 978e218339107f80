"""Host-side mirror of the reference's operator interface for the hot path.

Same names, argument meaning and error behaviour as the Rust constructors the plan-serde layer
calls (SURVEY.md §8b):

    FilterExec.try_new(predicates, input)                       datafusion-ext-plans/src/filter_exec.rs:52-73
    ProjectExec.try_new([(expr, name)], input)                  datafusion-ext-plans/src/project_exec.rs:57-81
    AggExec.try_new(exec_mode, groupings, aggs, supports_partial_skipping, input)
                                                                datafusion-ext-plans/src/agg_exec.rs:67-98
    create_agg(function, children, input_schema, return_type)   datafusion-ext-plans/src/agg/agg.rs:171-205
    plan.execute() / collect(plan)                              ExecutionPlan::execute + physical_plan::collect

Each plan object serialises itself to the reference's protobuf (`blaze_b200.proto`) and executes
through the C ABI (`blaze_b200.native`): the whole subtree becomes ONE fused GPU pipeline.
Constructors validate by decoding the plan in the native library (no GPU needed), so the errors are
the library's own (`FilterExec.try_new` with a non-boolean predicate raises like the reference does).
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence, Tuple

from . import exprs as E
from . import native
from . import proto as P
from . import types as T
from .exprs import AggExpr, AggFunctionExpr, GroupingExpr
from .types import Field, Schema

HashAgg, SortAgg = E.HASH_AGG, E.SORT_AGG
Partial, PartialMerge, Final = E.PARTIAL, E.PARTIAL_MERGE, E.FINAL


class ExecutionPlan:
    def schema(self) -> Schema:
        raise NotImplementedError

    def children(self) -> List["ExecutionPlan"]:
        return []

    def node(self):
        """-> plan.protobuf.PhysicalPlanNode"""
        raise NotImplementedError

    def leaf(self) -> "MemoryExec":
        p = self
        while p.children():
            p = p.children()[0]
        return p

    def plan_bytes(self) -> bytes:
        return self.node().SerializeToString()

    def explain(self) -> str:
        return native.plan_explain(self.plan_bytes())

    def _validate(self):
        native.plan_explain(self.plan_bytes())

    def execute(self, conf: Optional[native.Conf] = None, device: int = 0):
        """Run the subtree on the GPU over the leaf's batches; yields pyarrow RecordBatches."""
        leaf = self.leaf()
        with native.NativeOp(self.plan_bytes(), conf, device) as op:
            for rb in leaf.batches:
                op.push(rb)
                while True:
                    out = op.pull()
                    if out is None:
                        break
                    yield out
            op.finish()
            while True:
                out = op.pull()
                if out is None:
                    break
                yield out
            self.last_metrics = op.metrics()


def collect(plan: ExecutionPlan, conf: Optional[native.Conf] = None, device: int = 0) -> List:
    return list(plan.execute(conf, device))


class MemoryExec(ExecutionPlan):
    """In-memory source = the reference tests' `TestMemoryExec` (agg_exec.rs:490); on the wire it is an
    FFIReaderExecNode leaf, i.e. batches arrive through the Arrow C Data Interface exactly like
    FFIReaderExec's input (ffi_reader_exec.rs:163-194)."""

    def __init__(self, schema: Schema, batches: Sequence = (), resource_id: str = "mem"):
        self._schema = schema
        self.batches = list(batches)
        self.resource_id = resource_id

    @staticmethod
    def from_arrow(batches: Sequence, schema=None) -> "MemoryExec":
        import pyarrow as pa
        if schema is None:
            schema = batches[0].schema
        return MemoryExec(T.from_arrow_schema(schema), batches)

    def schema(self):
        return self._schema

    def node(self):
        return P.ffi_reader_node(self._schema, self.resource_id)


class FilterExec(ExecutionPlan):
    def __init__(self, predicates: Sequence[E.Expr], input: ExecutionPlan):
        self.predicates = list(predicates)
        self.input = input
        self._validate()

    try_new = classmethod(lambda cls, predicates, input: cls(predicates, input))

    def schema(self):
        return self.input.schema()                                      # filter_exec.rs:99-101

    def children(self):
        return [self.input]

    def node(self):
        return P.filter_node(self.input.node(), self.predicates)


class ProjectExec(ExecutionPlan):
    def __init__(self, exprs: Sequence[Tuple[E.Expr, str]], input: ExecutionPlan):
        self.exprs = [(e, n) for e, n in exprs]
        self.input = input
        ins = input.schema()
        self._schema = Schema(Field(n, e.data_type(ins), e.nullable(ins)) for e, n in self.exprs)   # project_exec.rs:62-72
        self._validate()

    try_new = classmethod(lambda cls, exprs, input: cls(exprs, input))

    def schema(self):
        return self._schema

    def children(self):
        return [self.input]

    def node(self):
        ins = self.input.schema()
        return P.projection_node(self.input.node(), [e for e, _ in self.exprs], [n for _, n in self.exprs],
                                 [e.data_type(ins) for e, _ in self.exprs])


class ExpandExec(ExecutionPlan):
    """ExpandExec::try_new(schema, projections, input) (expand_exec.rs:49-77): every input batch yields one output batch per
    projection, in order.  Each projection needs an expression of the field's exact type for every schema field; expressions
    beyond the field count are ignored.  Spark plans it below the partial aggregate of ROLLUP / CUBE / GROUPING SETS and of
    aggregates over several DISTINCT column sets."""

    def __init__(self, schema: Schema, projections: Sequence[Sequence[E.Expr]], input: ExecutionPlan):
        self._schema = schema
        self.projections = [list(p) for p in projections]
        self.input = input
        self._validate()                                                # the native decoder applies try_new's type checks

    try_new = classmethod(lambda cls, schema, projections, input: cls(schema, projections, input))

    def schema(self):
        return self._schema

    def children(self):
        return [self.input]

    def node(self):
        return P.expand_node(self.input.node(), self._schema, self.projections)


def create_agg(function: int, children: Sequence[E.Expr], input_schema: Schema, return_type: T.DataType) -> AggFunctionExpr:
    """`create_agg` (agg/agg.rs:171-205).  The Count/Sum/Avg rewrites (drop non-nullable count
    children, wrap Sum/Avg children in TryCast(return_type)) happen natively at decode time, exactly
    where the reference does them."""
    return AggFunctionExpr(function, children, return_type)


class AggExec(ExecutionPlan):
    def __init__(self, exec_mode: int, groupings: Sequence[GroupingExpr], aggs: Sequence[AggExpr],
                 supports_partial_skipping: bool, input: ExecutionPlan, columnar_state: bool = False):
        self.exec_mode = exec_mode
        self.groupings = list(groupings)
        self.aggs = list(aggs)
        self.supports_partial_skipping = supports_partial_skipping
        self.input = input
        self.columnar_state = columnar_state
        ins = input.schema()
        fields = [Field(g.field_name, g.expr.data_type(ins), g.expr.nullable(ins)) for g in self.groupings]
        final = any(a.mode == Final for a in self.aggs)
        if final:
            for a in self.aggs:
                fields.append(Field(a.field_name, _agg_final_type(a.agg, ins), a.agg.function != E.AGG_COUNT))
        elif columnar_state:
            for a in self.aggs:
                fields += _state_fields(a, ins)
        else:
            fields.append(Field(E.AGG_BUF_COLUMN_NAME, T.binary, False))                             # agg_ctx.rs:139-141
        self._schema = Schema(fields)
        self._validate()

    try_new = classmethod(lambda cls, exec_mode, groupings, aggs, supports_partial_skipping, input:
                          cls(exec_mode, groupings, aggs, supports_partial_skipping, input))

    def schema(self):
        return self._schema

    def children(self):
        return [self.input]

    def node(self):
        return P.agg_node(self.input.node(), self.exec_mode, self.groupings, self.aggs, self.supports_partial_skipping)


class ParquetScanExec(ExecutionPlan):
    """ParquetExec::new(base_conf, fs_resource_id, predicate) (datafusion-ext-plans/src/parquet_exec.rs:77-110): a LEAF that is its own
    source — files = [(path, size, (range_start, range_end) | None)], projection = indices into file_schema."""

    def __init__(self, file_schema: Schema, files, projection=None, pruning_predicates=(), limit=None):
        import os
        self.file_schema, self.projection = file_schema, list(projection) if projection is not None else list(range(len(file_schema)))
        self.files = [(p, s if s else os.path.getsize(p), r) for p, s, r in files]
        self.pruning, self.limit = list(pruning_predicates), limit
        self.batches = []
        self._validate()

    def schema(self):
        return Schema([self.file_schema[i] for i in self.projection])

    def node(self):
        return P.parquet_scan_node(self.file_schema, self.files, self.projection, self.pruning, self.limit)


class SortExec(ExecutionPlan):
    """SortExec::new(input, exprs, fetch) (sort_exec.rs:97-112); exprs = [(expr, descending, nulls_first)] like arrow's
    PhysicalSortExpr{expr, SortOptions{descending, nulls_first}} (SortOptions::default() = ascending, NULLs first)."""

    def __init__(self, input: ExecutionPlan, exprs, fetch: Optional[int] = None):
        self.input, self.exprs, self.fetch = input, [(e, bool(d), bool(nf)) for e, d, nf in exprs], fetch
        self._validate()

    new = classmethod(lambda cls, input, exprs, fetch=None: cls(input, exprs, fetch))

    def schema(self):
        return self.input.schema()

    def children(self):
        return [self.input]

    def node(self):
        return P.sort_node(self.input.node(), [(e, not d, nf) for e, d, nf in self.exprs], self.fetch)      # wire: asc = !descending (from_proto.rs:240-246)


class WindowExec(ExecutionPlan):
    """WindowExec::try_new(input, window_exprs, partition_spec, order_spec, group_limit, output_window_cols)
    (window_exec.rs:65-87): running row_number / rank / dense_rank and SUM / AVG / MIN / MAX / COUNT over ROWS BETWEEN UNBOUNDED
    PRECEDING AND CURRENT ROW of input sorted by (partition_spec, order_spec).  order_spec = [(expr, descending, nulls_first)] as
    in SortExec.  A group limit k (WindowGroupLimitExec) keeps the rows whose one window column is <= k as i32."""

    def __init__(self, input: ExecutionPlan, window_exprs: Sequence[E.WindowExpr], partition_spec: Sequence[E.Expr], order_spec,
                 group_limit: Optional[int] = None, output_window_cols: bool = True):
        self.input, self.window_exprs, self.partition_spec = input, list(window_exprs), list(partition_spec)
        self.order_spec = [(e, bool(d), bool(nf)) for e, d, nf in order_spec]
        self.group_limit, self.output_window_cols = group_limit, bool(output_window_cols)
        self._validate()

    try_new = classmethod(lambda cls, *a, **k: cls(*a, **k))

    def schema(self):
        fields = list(self.input.schema())
        if self.output_window_cols:
            fields += [w.field for w in self.window_exprs]
        return Schema(fields)

    def children(self):
        return [self.input]

    def node(self):
        return P.window_node(self.input.node(), self.window_exprs, self.partition_spec, [(e, not d, nf) for e, d, nf in self.order_spec],
                             self.group_limit, self.output_window_cols)


# protobuf JoinType (auron.proto:475-483): SEMI / ANTI are the Left forms (auron-serde/src/lib.rs:104-116)
JOIN_INNER, JOIN_LEFT, JOIN_RIGHT, JOIN_FULL, JOIN_SEMI, JOIN_ANTI, JOIN_EXISTENCE = range(7)
LEFT_SIDE, RIGHT_SIDE = 0, 1


def build_join_schema(left: Schema, right: Schema, join_type: int) -> Schema:
    """the schema the Spark side sends with the node (joins/test.rs:163-176 for the tests): left ++ right with the
    non-preserved side nullable; Semi / Anti = left; Existence = left ++ `exists#0: Boolean not null`"""
    if join_type == JOIN_EXISTENCE:
        return Schema(list(left) + [Field("exists#0", T.bool_, False)])
    if join_type in (JOIN_SEMI, JOIN_ANTI):
        return Schema(list(left))
    ln, rn = join_type in (JOIN_RIGHT, JOIN_FULL), join_type in (JOIN_LEFT, JOIN_FULL)
    return Schema([Field(f.name, f.dtype, f.nullable or ln) for f in left] + [Field(f.name, f.dtype, f.nullable or rn) for f in right])


class BroadcastJoinBuildHashMapExec(ExecutionPlan):
    """BroadcastJoinBuildHashMapExec::new(input, keys) (broadcast_join_build_hash_map_exec.rs:60-75): the map side of a join."""

    def __init__(self, input: ExecutionPlan, keys: Sequence[E.Expr]):
        self.input, self.keys = input, list(keys)
        self._validate()

    def schema(self):
        return Schema([Field(f.name, f.dtype, True) for f in self.input.schema()] + [Field("~TABLE", T.binary, True)])    # join_hash_map.rs:409-431

    def children(self):
        return [self.input]

    def node(self):
        return P.join_build_node(self.input.node(), self.keys)


class BroadcastJoinExec(ExecutionPlan):
    """BroadcastJoinExec::try_new(schema, left, right, on, join_type, broadcast_side, is_built, cached_build_hash_map_id)
    (broadcast_join_exec.rs:96-121).  is_built=True serialises as BroadcastJoinExecNode (the map side arrives as a
    BroadcastJoinBuildHashMapExec), False as HashJoinExecNode (shuffled hash join, from_proto.rs:187-223).
    execute(): the map side runs as its own op (BroadcastJoinBuildHashMapExec over that child), the other side is probed."""

    def __init__(self, schema: Schema, left: ExecutionPlan, right: ExecutionPlan, on, join_type: int, broadcast_side: int, is_built: bool = False,
                 cached_build_hash_map_id: Optional[str] = None):
        self._schema, self.left, self.right, self.on = schema, left, right, list(on)
        self.join_type, self.broadcast_side, self.is_built, self.cached_id = join_type, broadcast_side, is_built, cached_build_hash_map_id or ""
        self._validate()

    try_new = classmethod(lambda cls, *a, **k: cls(*a, **k))

    def schema(self):
        return self._schema

    def children(self):
        return [self.left, self.right]

    def _sides(self):
        build, probe = (self.left, self.right) if self.broadcast_side == LEFT_SIDE else (self.right, self.left)
        keys = [l if self.broadcast_side == LEFT_SIDE else r for l, r in self.on]
        data = build.input if isinstance(build, BroadcastJoinBuildHashMapExec) else build
        return data, keys, probe

    def node(self):
        return P.join_node(self._schema, self.left.node(), self.right.node(), self.on, self.join_type, self.broadcast_side, self.is_built, self.cached_id)

    def execute(self, conf: Optional[native.Conf] = None, device: int = 0):
        data, keys, probe = self._sides()
        build_plan = BroadcastJoinBuildHashMapExec(data, keys)
        with native.NativeOp(build_plan.plan_bytes(), conf, device) as bop:
            for rb in data.leaf().batches:
                bop.push(rb)
            bop.finish()
            self.build_metrics = bop.metrics()
            with native.NativeOp(self.plan_bytes(), conf, device) as op:
                op.attach_build(bop)
                for rb in probe.leaf().batches:
                    op.push(rb)
                    yield from op.pull_all()
                op.finish()
                yield from op.pull_all()
                self.last_metrics = op.metrics()


class ShuffleWriterExec(ExecutionPlan):
    """ShuffleWriterExec::try_new(input, partitioning, output_data_file, output_index_file)
    (datafusion-ext-plans/src/shuffle_writer_exec.rs:180-197).  partitioning: ("single",) | ("hash", [exprs], n) |
    ("round_robin", n) — the reference's `Partitioning` enum (shuffle/mod.rs:108-132).  execute() yields nothing, like the
    reference's stream; the result is the two files (and `last_chunks`, the per-partition bytes before compression)."""

    def __init__(self, input: ExecutionPlan, partitioning, output_data_file: str, output_index_file: str):
        self.input = input
        self.partitioning = tuple(partitioning)
        self.output_data_file, self.output_index_file = output_data_file, output_index_file
        self._validate()

    try_new = classmethod(lambda cls, input, partitioning, data_file, index_file: cls(input, partitioning, data_file, index_file))

    def schema(self):
        return self.input.schema()                                      # shuffle_writer_exec.rs:76-78

    def children(self):
        return [self.input]

    def node(self):
        return P.shuffle_writer_node(self.input.node(), self.partitioning, self.output_data_file, self.output_index_file)

    def execute(self, conf: Optional[native.Conf] = None, device: int = 0):
        leaf = self.leaf()
        with native.NativeOp(self.plan_bytes(), conf, device) as op:
            for rb in leaf.batches:
                op.push(rb)
            op.finish()
            self.last_chunks = op.shuffle_chunks()
            self.last_metrics = op.metrics()
        return iter(())


def _agg_data_type(f: AggFunctionExpr, ins: Schema) -> T.DataType:
    if f.function == E.AGG_COUNT:
        return T.int64
    if f.function in (E.AGG_SUM, E.AGG_AVG):
        return f.return_type
    return f.children[0].data_type(ins)


def _agg_final_type(f: AggFunctionExpr, ins: Schema) -> T.DataType:
    dt = _agg_data_type(f, ins)
    if f.function == E.AGG_AVG and not dt.is_decimal:
        return T.float64                                                                              # avg.rs:166-171
    return dt


def _state_fields(a: AggExpr, ins: Schema) -> List[Field]:
    dt = _agg_data_type(a.agg, ins)
    if a.agg.function == E.AGG_COUNT:
        return [Field(a.field_name, T.int64, False)]
    if a.agg.function == E.AGG_AVG:
        return [Field(a.field_name + "#sum", dt, True), Field(a.field_name + "#count", T.int64, False)]
    return [Field(a.field_name, dt, True)]
