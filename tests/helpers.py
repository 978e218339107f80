"""Shared helpers of the parity tests: seeded inputs, oracle runs, multiset comparison."""
import numpy as np
import pyarrow as pa

from blaze_b200 import exprs as E, plans as PL, types as T
from oracle import blaze_oracle as O


def rb_from_cols(names, arrays):
    return pa.RecordBatch.from_arrays(arrays, names=names)


def with_nulls(rng, values: np.ndarray, null_frac: float, pa_type=None):
    if null_frac <= 0:
        return pa.array(values, type=pa_type)
    mask = rng.random(len(values)) < null_frac
    return pa.array(values, mask=mask, type=pa_type)


def split_batches(rb: pa.RecordBatch, batch_rows: int):
    return [rb.slice(i, min(batch_rows, rb.num_rows - i)) for i in range(0, rb.num_rows, batch_rows)] or [rb]


def oracle_batches(batches):
    return [O.batch_from_arrow(b) for b in batches]


def gpu_multiset(out_batches):
    return O.rows_multiset([O.batch_from_arrow(b) for b in out_batches])


def assert_same_rows_ordered(gpu_batches, oracle_out, schema):
    """FilterExec/ProjectExec preserve row order: compare the concatenations exactly (values + validity)."""
    got = O.concat_batches(schema, [O.batch_from_arrow(b) for b in gpu_batches])
    exp = O.concat_batches(schema, oracle_out)
    assert got.num_rows == exp.num_rows, f"row count {got.num_rows} != {exp.num_rows}"
    for i, (g, e) in enumerate(zip(got.cols, exp.cols)):
        assert g.dtype == e.dtype, f"col {i}: dtype {g.dtype} != {e.dtype}"
        assert np.array_equal(g.valid, e.valid), f"col {i}: validity differs"
        gv, ev = g.values[g.valid], e.values[e.valid]
        if g.dtype.is_float:
            assert np.array_equal(gv.view(np.int64 if g.dtype.id == T.FLOAT64 else np.int32),
                                  ev.view(np.int64 if g.dtype.id == T.FLOAT64 else np.int32)), f"col {i}: float bits differ"
        else:
            assert np.array_equal(gv, ev), f"col {i}: values differ"


def parquet_scan(path, table_schema, **kw):
    """ParquetScanExec over one file; `range=(lo, hi)` scans one byte-range split of it."""
    return PL.ParquetScanExec(T.from_arrow_schema(table_schema), [(path, 0, kw.pop("range", None))], **kw)


def value_slots(a: pa.Array) -> np.ndarray:
    """the value bits of every slot of a fixed-width array: one bit per row (Boolean), else one row of bytes per row"""
    buf = np.frombuffer(a.buffers()[1], np.uint8)
    if a.type == pa.bool_():
        return np.unpackbits(buf, bitorder="little")[a.offset: a.offset + len(a)]
    w = a.type.byte_width
    return buf[a.offset * w: (a.offset + len(a)) * w].reshape(len(a), w)


def assert_same_table(got_batches, exp: pa.Table):
    """The scan's output against libparquet's reading of the same file: same types and validity, and the same bits in every
    non-NULL slot (float bits too: NaN payloads, -0.0).  libparquet leaves unspecified values under a NULL; the scan writes
    zero there, and that is checked too."""
    got = pa.Table.from_batches(got_batches, schema=got_batches[0].schema) if got_batches else exp.slice(0, 0)
    assert got.num_rows == exp.num_rows, (got.num_rows, exp.num_rows)
    if not exp.num_rows:
        return
    for name in exp.schema.names:
        g, e = got.column(name).combine_chunks(), exp.column(name).combine_chunks()
        assert g.type == e.type, (name, g.type, e.type)
        valid = e.is_valid().to_numpy(zero_copy_only=False)
        assert np.array_equal(g.is_valid().to_numpy(zero_copy_only=False), valid), f"{name}: validity differs"
        if g.null_count == len(g) and g.buffers()[1] is None:
            continue
        gv, ev = value_slots(g), value_slots(e) if e.null_count < len(e) else None
        if ev is not None and valid.any():
            bad = np.flatnonzero(np.any((gv[valid] != ev[valid]).reshape(int(valid.sum()), -1), axis=1))
            assert not len(bad), f"{name}: {len(bad)} values differ, first at non-NULL ordinal {bad[0]}: {g.filter(e.is_valid())[int(bad[0])]} vs {e.filter(e.is_valid())[int(bad[0])]}"
        assert not np.any(gv[~valid]), f"{name}: a NULL slot holds a nonzero value"


def assert_multiset_equal(gpu_batches, oracle_out, float_cols=(), rtol=1e-6):
    """HashAgg parity = equality of the multiset of rows (assert_batches_sorted_eq!, agg_exec.rs:679);
    columns listed in float_cols are compared within rtol (fp64 SUM/AVG contract), all others bit-exactly."""
    g = [O.batch_from_arrow(b) for b in gpu_batches]
    if not float_cols:
        ms_g, ms_e = O.rows_multiset(g), O.rows_multiset(oracle_out)
        if ms_g != ms_e:
            only_g = {k: v for k, v in ms_g.items() if ms_e.get(k) != v}
            only_e = {k: v for k, v in ms_e.items() if ms_g.get(k) != v}
            raise AssertionError(f"row multisets differ: {len(only_g)} rows only/more on GPU, {len(only_e)} only/more in oracle; "
                                 f"samples gpu={list(only_g.items())[:3]} oracle={list(only_e.items())[:3]}")
        return

    def keyed(batches):
        out = {}
        for b in batches:
            for r in range(b.num_rows):
                key, fl = [], []
                for ci, c in enumerate(b.cols):
                    v = None if not c.valid[r] else (c.values[r].item() if hasattr(c.values[r], "item") else c.values[r])
                    (fl if ci in float_cols else key).append(v)
                key = tuple(key)
                assert key not in out, f"duplicate group {key}"
                out[key] = fl
        return out
    kg, ke = keyed(g), keyed(oracle_out)
    assert kg.keys() == ke.keys(), f"group sets differ: {len(kg)} vs {len(ke)}"
    for k, fe in ke.items():
        for a, b in zip(kg[k], fe):
            if a is None or b is None:
                assert a is None and b is None, f"group {k}: NULL mismatch {a} vs {b}"
            elif b != b:
                assert a != a
            else:
                assert abs(a - b) <= rtol * max(abs(a), abs(b)) + 1e-300, f"group {k}: {a} vs {b}"
