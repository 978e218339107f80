"""Device-resident throughput of the other SURVEY §8d shapes (M0 filter+project, M2 q1-shaped fused
filter->agg, M1 through the hash path) — kernel-only numbers from b200q_metrics.hot_kernel_ns."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from blaze_b200 import exprs as E, native, plans as PL, types as T

rows = int(os.environ.get("ROWS", 1 << 28))
dev = torch.device("cuda", 0)
g = torch.Generator(device=dev); g.manual_seed(42)
peak = 3350.0                         # GB/s: H100 SXM data-sheet HBM3 bandwidth

REPS = int(os.environ.get("REPS", 0))      # override the repetitions of every shape (profiling)
ONLY = os.environ.get("SHAPES")       # comma-separated substrings of shape names to run

def run(name, plan_bytes, cols, alg_bytes_per_row, conf=None, reps=3, steady=False, valid=None):
    if ONLY and not any(t in name for t in ONLY.split(",")): return
    valid = valid or [None] * len(cols)
    reps = REPS or reps
    spec = [(c.data_ptr(), (vb.data_ptr() if vb is not None else 0), rows) for c, vb in zip(cols, valid)]
    keep = list(cols) + [vb for vb in valid if vb is not None]
    best = None; steady_ns = None
    for _ in range(reps):
        with native.NativeOp(plan_bytes, conf or native.default_conf(), 0) as op:
            op.push_device(native.DeviceBatch(spec, rows, 0, keepalive=keep))
            if steady:      # second pass over the same rows: every group already exists (steady-state cost, no inserts)
                op.sync(); m0 = op.metrics()
                op.push_device(native.DeviceBatch(spec, rows, 0, keepalive=keep))
                op.sync(); m1 = op.metrics()
                steady_ns = m1["hot_kernel_ns"] - m0["hot_kernel_ns"]
            op.finish()
            n_out = 0
            while True:
                o = op.pull_device()
                if o is None: break
                n_out += o.array.length; native.release_device_array(o)
            m = op.metrics()
        t = m["hot_kernel_ns"] / max(1, m["hot_kernel_launches"]) * m["hot_kernel_launches"]
        if best is None or t < best[0]: best = (t, m, n_out)
    t, m, n_out = best
    if steady:
        print(json.dumps({"shape": name + " [steady state, 2nd pass]", "rows": rows, "hot_kernel_ms": steady_ns / 1e6, "rows_per_s": rows / (steady_ns * 1e-9),
                          "alg_GBps": alg_bytes_per_row * rows / steady_ns, "frac_of_hbm_peak": alg_bytes_per_row * rows / steady_ns / peak}), flush=True)
        return
    gbs = alg_bytes_per_row * m["hot_kernel_rows"] / t
    print(json.dumps({"shape": name, "rows": rows, "out_rows": n_out, "hot_kernel_ms": t / 1e6, "rows_per_s": m["hot_kernel_rows"] / (t * 1e-9),
                      "alg_GBps": gbs, "frac_of_hbm_peak": gbs / peak, "fast_path_launches": m["fast_path_launches"], "launches": m["gpu_kernel_launches"]}), flush=True)

# M0: Filter[a < 500] -> Project[a, a + b]   (24 B/row at s = 0.5)
a = torch.randint(0, 1000, (rows,), dtype=torch.int64, device=dev, generator=g)
b = torch.randint(-2**31, 2**31, (rows,), dtype=torch.int64, device=dev, generator=g)
s0 = T.Schema([T.Field("a", T.int64, False), T.Field("b", T.int64, False)])
A, B = E.Column("a"), E.Column("b")
m0 = PL.ProjectExec([(A, "a"), (E.BinaryExpr(A, "Plus", B), "c")], PL.FilterExec([E.BinaryExpr(A, "Lt", E.Literal(500, T.int64))], PL.MemoryExec(s0)))
run("M0 filter+project s=0.5", m0.plan_bytes(), [a, b], 24.0)
del a, b
# M1 via hash path (dense disabled) and via the generic VM kernel
k = torch.randint(0, 1 << 20, (rows,), dtype=torch.int64, device=dev, generator=g)
v = torch.randint(-10**6, 10**6, (rows,), dtype=torch.int64, device=dev, generator=g)
s1 = T.Schema([T.Field("k", T.int64, False), T.Field("v", T.int64, False)])
aggs = [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("v")], s1, T.int64)), E.AggExpr("c", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [E.Column("v")], s1, T.int64))]
m1 = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], aggs, True, PL.MemoryExec(s1))
run("M1 dense (lean, global table)", m1.plan_bytes(), [k, v], 16.0, native.default_conf(agg_initial_groups=1 << 20))
run("M1 hash (lean, compacted probes; first pass incl. 1M inserts)", m1.plan_bytes(), [k, v], 16.0, native.default_conf(agg_initial_groups=1 << 20, agg_dense_keys=0))
run("M1 hash", m1.plan_bytes(), [k, v], 16.0, native.default_conf(agg_initial_groups=1 << 20, agg_dense_keys=0), reps=1, steady=True)
for ig in (1 << 21, 1 << 22):
    run("M1 hash initial_groups=%d" % ig, m1.plan_bytes(), [k, v], 16.0, native.default_conf(agg_initial_groups=ig, agg_dense_keys=0), reps=1, steady=True)
# typed / nullable inputs through the hashed path: int32 key, 10 % NULL values (validity bitmaps)  (12.25 B/row)
k32 = k.to(torch.int32)
vbits = torch.full(((rows + 7) // 8,), 0xFF, dtype=torch.uint8, device=dev); vbits[::10] = 0
s1t = T.Schema([T.Field("k", T.int32, False), T.Field("v", T.int64, True)])
aggs_t = [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("v")], s1t, T.int64)), E.AggExpr("c", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [E.Column("v")], s1t, T.int64))]
m1t = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], aggs_t, True, PL.MemoryExec(s1t))
run("M1 typed hash (int32 key, nullable v)", m1t.plan_bytes(), [k32, v], 12.125, native.default_conf(agg_initial_groups=1 << 20, agg_dense_keys=0), reps=1, steady=True, valid=[None, vbits])
run("M1 typed dense (int32 key, nullable v)", m1t.plan_bytes(), [k32, v], 12.125, native.default_conf(agg_initial_groups=1 << 20), reps=2, valid=[None, vbits])
del k32, vbits
# low cardinality: 64 groups (every RED of a warp lands on a handful of sectors)
klow = torch.randint(0, 64, (rows,), dtype=torch.int64, device=dev, generator=g)
run("M1 low cardinality (64 groups) dense", m1.plan_bytes(), [klow, v], 16.0, native.default_conf())
run("M1 low cardinality (64 groups) hash", m1.plan_bytes(), [klow, v], 16.0, native.default_conf(agg_dense_keys=0), reps=1, steady=True)
del klow
# skewed keys: Zipf(1.1) ranks over 2^20 keys (continuous inverse-CDF approximation), rank r -> key (r * 2654435761) mod 2^20
u = torch.rand(rows, device=dev, generator=g, dtype=torch.float64)
nk, sz = float(1 << 20), 1.1
ranks = torch.clamp(((u * (nk ** (1 - sz) - 1) + 1) ** (1 / (1 - sz))).floor().to(torch.int64), 1, 1 << 20) - 1
kz = (ranks * 2654435761) % (1 << 20)
del u, ranks
run("M1 Zipf(1.1) keys, dense, hot-key cache off", m1.plan_bytes(), [kz, v], 16.0, native.default_conf(agg_initial_groups=1 << 20, agg_hot_key_cache=0), reps=1)
run("M1 Zipf(1.1) keys, dense + hot-key cache", m1.plan_bytes(), [kz, v], 16.0, native.default_conf(agg_initial_groups=1 << 20, agg_hot_key_cache=1), reps=1)
run("M1 Zipf(1.1) keys, hash", m1.plan_bytes(), [kz, v], 16.0, native.default_conf(agg_initial_groups=1 << 20, agg_dense_keys=0), reps=1, steady=True)
del kz
# the "fp64 SUM/AVG", "decimal128(17,2)" and MIN/MAX halves of the north_star target: wide tile kernels (kernels_tile.cu)
vf = v.to(torch.float64)
s1f = T.Schema([T.Field("k", T.int64, False), T.Field("v", T.float64, False)])
mkp = lambda sch, specs: PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))],
                                    [E.AggExpr(nm, E.PARTIAL, PL.create_agg(fn, [E.Column("v")], sch, rt)) for nm, fn, rt in specs], True, PL.MemoryExec(sch))
run("M1 f64 SUM+COUNT (wide tile)", mkp(s1f, [("s", E.AGG_SUM, T.float64), ("c", E.AGG_COUNT, T.int64)]).plan_bytes(), [k, vf], 16.0, native.default_conf(agg_initial_groups=1 << 20))
run("M1 f64 AVG (wide tile)", mkp(s1f, [("a", E.AGG_AVG, T.float64)]).plan_bytes(), [k, vf], 16.0, native.default_conf(agg_initial_groups=1 << 20))
run("M1 f64 SUM+COUNT generic VM", mkp(s1f, [("s", E.AGG_SUM, T.float64), ("c", E.AGG_COUNT, T.int64)]).plan_bytes(), [k, vf], 16.0, native.default_conf(agg_initial_groups=1 << 20, force_generic_kernels=1), reps=1)
del vf
run("M1 int64 MIN+MAX (wide tile)", mkp(s1, [("mn", E.AGG_MIN, T.int64), ("mx", E.AGG_MAX, T.int64)]).plan_bytes(), [k, v], 16.0, native.default_conf(agg_initial_groups=1 << 20))
vd = torch.stack([v, v >> 63], dim=1).contiguous()          # decimal128(17,2): little-endian {lo, hi} pairs, sign-extended
s1d = T.Schema([T.Field("k", T.int64, False), T.Field("v", T.decimal128(17, 2), False)])
run("M1 decimal128(17,2) SUM+COUNT (wide tile)", mkp(s1d, [("s", E.AGG_SUM, T.decimal128(27, 2)), ("c", E.AGG_COUNT, T.int64)]).plan_bytes(), [k, vd], 24.0, native.default_conf(agg_initial_groups=1 << 20))
run("M1 decimal128(17,2) SUM+COUNT generic VM", mkp(s1d, [("s", E.AGG_SUM, T.decimal128(27, 2)), ("c", E.AGG_COUNT, T.int64)]).plan_bytes(), [k, vd], 24.0, native.default_conf(agg_initial_groups=1 << 20, force_generic_kernels=1), reps=1)
del vd
run("M1 generic VM kernel", m1.plan_bytes(), [k, v], 16.0, native.default_conf(agg_initial_groups=1 << 20, force_generic_kernels=1), reps=1)
del k
# M2: q1-shaped: f BETWEEN lo AND hi (s = 0.2), keys (k1 ~ U[0,2^17), k2 ~ U[0,8)), SUM(v)   (32 B/row)
f = torch.randint(0, 1000, (rows,), dtype=torch.int64, device=dev, generator=g)
k1 = torch.randint(0, 1 << 17, (rows,), dtype=torch.int64, device=dev, generator=g)
k2 = torch.randint(0, 8, (rows,), dtype=torch.int64, device=dev, generator=g)
s2 = T.Schema([T.Field(n, T.int64, False) for n in ("f", "k1", "k2", "v")])
preds = [E.BinaryExpr(E.Column("f"), "GtEq", E.Literal(200, T.int64)), E.BinaryExpr(E.Column("f"), "LtEq", E.Literal(399, T.int64))]
m2 = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k1", E.Column("k1")), E.GroupingExpr("k2", E.Column("k2"))],
                [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("v")], s2, T.int64))], True, PL.FilterExec(preds, PL.MemoryExec(s2)))
run("M2 q1-shaped fused filter->agg (2 keys)", m2.plan_bytes(), [f, k1, k2, v], 32.0, native.default_conf(agg_initial_groups=1 << 20))
run("M2 q1-shaped", m2.plan_bytes(), [f, k1, k2, v], 32.0, native.default_conf(agg_initial_groups=1 << 20), reps=1, steady=True)
# M2 selectivity sweep: the tile kernel reads k1, k2 and v only for the rows that pass, so s = 1.0 guards against that costing
# more than reading every column at once
m2s = lambda sch, lo, hi: PL.AggExec(PL.HashAgg, [E.GroupingExpr("k1", E.Column("k1")), E.GroupingExpr("k2", E.Column("k2"))],
                                     [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("v")], sch, T.int64))], True,
                                     PL.FilterExec([E.BinaryExpr(E.Column("f"), "GtEq", E.Literal(lo, T.int64)), E.BinaryExpr(E.Column("f"), "LtEq", E.Literal(hi, T.int64))], PL.MemoryExec(sch)))
for sel in (0.01, 0.2, 0.5, 1.0):
    run("M2 selectivity s=%.2f" % sel, m2s(s2, 0, int(1000 * sel) - 1).plan_bytes(), [f, k1, k2, v], 32.0, native.default_conf(agg_initial_groups=1 << 20))
# M2 with an int32 key and a nullable value (10 % NULL)  (28.125 B/row)
k1_32 = k1.to(torch.int32)
vbits = torch.full(((rows + 7) // 8,), 0xFF, dtype=torch.uint8, device=dev); vbits[::10] = 0
s2t = T.Schema([T.Field("f", T.int64, False), T.Field("k1", T.int32, False), T.Field("k2", T.int64, False), T.Field("v", T.int64, True)])
run("M2 int32 key, nullable v", m2s(s2t, 200, 399).plan_bytes(), [f, k1_32, k2, v], 28.125, native.default_conf(agg_initial_groups=1 << 20), valid=[None, None, None, vbits])
del k1_32, vbits
# M3: ShuffleWriterExec 200-way hash partition + batch_serde encode (BASELINE configs[3] map side): 32 B/row read + 32 B/row of byte planes written
m3 = PL.ShuffleWriterExec(PL.MemoryExec(s2), ("hash", [E.Column("k1")], 200), "", "")
run("M3 shuffle write 200-way (4 int64 columns, hash on k1)", m3.plan_bytes(), [f, k1, k2, v], 64.0, native.default_conf(shuffle_output_on_device=1), reps=2)
m3b = PL.ShuffleWriterExec(PL.MemoryExec(s2), ("hash", [E.Column("k1"), E.Column("k2")], 2000), "", "")
run("M3 shuffle write 2000-way (hash on k1,k2)", m3b.plan_bytes(), [f, k1, k2, v], 64.0, native.default_conf(shuffle_output_on_device=1), reps=2)


# M4: HashJoinExec store_sales JOIN date_dim (BASELINE configs[3] probe side): the map side is its own op, the probed side streams.
def run_join(name, n_build_keep, alg_bytes_per_row):
    if ONLY and not any(t in name for t in ONLY.split(",")): return
    ND = 73049                                                     # rows of TPC-DS date_dim
    d_sk = torch.arange(ND, dtype=torch.int64, device=dev)
    d_year = 1900 + d_sk // 366
    d_moy = (d_sk // 30) % 12 + 1
    keep = d_sk < n_build_keep                                      # the dimension filter (e.g. one year) already applied to the map side
    bcols = [d_sk[keep].contiguous(), d_year[keep].contiguous(), d_moy[keep].contiguous()]
    sk = torch.randint(0, ND, (rows,), dtype=torch.int64, device=dev, generator=g)
    sd = T.Schema([T.Field(n, T.int64, False) for n in ("d_date_sk", "d_year", "d_moy")])
    ss = T.Schema([T.Field(n, T.int64, False) for n in ("ss_sold_date_sk", "ss_item_sk", "ss_quantity", "ss_net_paid")])
    build = PL.BroadcastJoinBuildHashMapExec(PL.MemoryExec(sd), [E.Column("d_date_sk")])
    join = PL.BroadcastJoinExec(PL.build_join_schema(ss, sd, PL.JOIN_INNER), PL.MemoryExec(ss), build, [(E.Column("ss_sold_date_sk"), E.Column("d_date_sk"))], PL.JOIN_INNER, PL.RIGHT_SIDE, True, "m")
    nb = int(bcols[0].numel())
    best = None
    for _ in range(REPS or 3):
        with native.NativeOp(build.plan_bytes(), native.default_conf(), 0) as bop:
            bop.push_device(native.DeviceBatch([(c.data_ptr(), 0, nb) for c in bcols], nb, 0, keepalive=tuple(bcols)))
            bop.finish()
            with native.NativeOp(join.plan_bytes(), native.default_conf(), 0) as op:
                op.attach_build(bop)
                pc = [sk, k1, k2, v]
                op.push_device(native.DeviceBatch([(c.data_ptr(), 0, rows) for c in pc], rows, 0, keepalive=tuple(pc)))
                op.finish()
                n_out = 0
                while True:
                    o = op.pull_device()
                    if o is None: break
                    n_out += o.array.length; native.release_device_array(o)
                m = op.metrics()
        if best is None or m["hot_kernel_ns"] < best[0]: best = (m["hot_kernel_ns"], m, n_out)
    t, m, n_out = best
    gbs = alg_bytes_per_row * rows / t
    print(json.dumps({"shape": name, "rows": rows, "build_rows": nb, "out_rows": n_out, "probe_ms": t / 1e6, "rows_per_s": rows / (t * 1e-9), "alg_GBps": gbs, "frac_of_hbm_peak": gbs / peak,
                      "launches": m["gpu_kernel_launches"]}), flush=True)

run_join("M4 hash join store_sales x date_dim, every row matches (32 B read + 56 B written per probe row)", 73049, 88.0)
run_join("M4 hash join store_sales x date_dim filtered to one year (0.5 % match; 32 B read per probe row)", 366, 32.0 + 0.005 * 56)


# M5: SortExec ORDER BY one int64 key (full 64-bit range: all eight radix passes) over (key, payload), and a 20-bit key (three passes)
def run_sort(name, key, n_sort):
    if ONLY and not any(t in name for t in ONLY.split(",")): return
    ssch = T.Schema([T.Field("k", T.int64, False), T.Field("p", T.int64, False)])
    plan = PL.SortExec(PL.MemoryExec(ssch), [(E.Column("k"), False, True)])
    kk, pp = key[:n_sort].contiguous(), v[:n_sort].contiguous()
    best = None
    for _ in range(REPS or 2):
        with native.NativeOp(plan.plan_bytes(), native.default_conf(), 0) as op:
            op.push_device(native.DeviceBatch([(kk.data_ptr(), 0, n_sort), (pp.data_ptr(), 0, n_sort)], n_sort, 0, keepalive=(kk, pp)))
            op.finish()
            o = op.pull_device()
            srt = torch.as_tensor(__import__("bench").CudaView(o.array.children[0].contents.buffers[1], n_sort * 8, o), device="cuda").view(torch.int64)
            ok = bool((srt[1:] >= srt[:-1]).all())
            native.release_device_array(o)
            m = op.metrics()
        if best is None or m["hot_kernel_ns"] < best[0]: best = (m["hot_kernel_ns"], m, ok)
    t, m, ok = best
    print(json.dumps({"shape": name, "rows": n_sort, "sorted": ok, "sort_ms": t / 1e6, "rows_per_s": n_sort / (t * 1e-9), "launches": m["gpu_kernel_launches"]}), flush=True)

run_sort("M5 sort int64 key, full range (8 radix passes) + 8-byte payload", (k1 * 2654435761 * 40503 + f * 2**40) ^ (v << 20), min(rows, 1 << 26))
run_sort("M5 sort int64 key in [0, 2^17) (3 radix passes) + 8-byte payload", k1, min(rows, 1 << 26))


# M6: ParquetScanExec (BASELINE configs[2] shape): store_sales-like synthetic columns written by pyarrow, scanned (decode on the GPU) with a
# pushed-down predicate on the sorted date key; host work (file read, Thrift, Snappy) is inside the measured time
def run_parquet(name, compression, n_pq):
    if ONLY and not any(t in name for t in ONLY.split(",")): return
    import time, tempfile, numpy as np, pyarrow as pa, pyarrow.parquet as pq
    rng = np.random.default_rng(7)
    tbl = pa.table({"ss_sold_date_sk": pa.array(np.sort(rng.integers(2450816, 2452642, n_pq)).astype(np.int32), pa.int32()),
                    "ss_item_sk": pa.array(rng.integers(1, 204000, n_pq).astype(np.int32), pa.int32()),
                    "ss_quantity": pa.array(rng.integers(1, 100, n_pq).astype(np.int32), pa.int32()),
                    "ss_net_paid": pa.array(rng.integers(0, 2000000, n_pq, dtype=np.int64))})
    tbl = tbl.cast(pa.schema([pa.field(f.name, f.type, False) for f in tbl.schema]))
    path = os.path.join(tempfile.gettempdir(), f"b200q_store_sales_{compression}.parquet")
    pq.write_table(tbl, path, compression=compression, row_group_size=1 << 20)
    fsz = os.path.getsize(path)
    sch = T.from_arrow_schema(tbl.schema)
    pred = E.BinaryExpr(E.Column("ss_sold_date_sk"), "GtEq", E.Literal(2452000, T.int32))
    for label, preds in (("full scan", []), ("pushdown ss_sold_date_sk >= 2452000", [pred])):
        scan = PL.ParquetScanExec(sch, [(path, fsz, None)], pruning_predicates=preds)
        plan = PL.FilterExec(preds, scan) if preds else scan
        best = None
        for _ in range(3):
            pb = plan.plan_bytes()
            t0 = time.perf_counter()
            with native.NativeOp(pb, native.default_conf(), 0) as op:
                t1 = time.perf_counter()
                op.finish()
                t2 = time.perf_counter()
                n_out = 0
                while True:
                    o = op.pull_device()
                    if o is None: break
                    n_out += o.array.length; native.release_device_array(o)
                m = op.metrics()
                t3 = time.perf_counter()
            dt = time.perf_counter() - t0
            m["phases_ms"] = {"create": (t1 - t0) * 1e3, "finish (the scan)": (t2 - t1) * 1e3, "pull_device + release": (t3 - t2) * 1e3, "destroy": (t0 + dt - t3) * 1e3}
            if best is None or dt < best[0]: best = (dt, n_out, m)
        dt, n_out, m = best
        print(json.dumps({"shape": f"{name} [{label}]", "rows": n_pq, "file_bytes": fsz, "out_rows": n_out, "wall_ms": dt * 1e3, "rows_per_s": n_pq / dt, "file_GBps": fsz / dt / 1e9,
                          "gpu_ms": m["elapsed_compute_ns"] / 1e6, "row_groups_decoded": m["input_batches"], "row_groups_pruned": m["fast_path_launches"], "launches": m["gpu_kernel_launches"], "phases_ms": m["phases_ms"]}), flush=True)
    t0 = time.perf_counter(); pq.read_table(path); print(json.dumps({"shape": f"{name} [pyarrow.parquet.read_table on the host, all cores]", "wall_ms": (time.perf_counter() - t0) * 1e3}), flush=True)

run_parquet("M6 parquet scan store_sales-like 4 columns, snappy + dictionary", "snappy", 1 << 24)
run_parquet("M6 parquet scan store_sales-like 4 columns, uncompressed", "none", 1 << 24)


# S1-S3: Utf8 columns (device-resident, generated from the seed: lengths -> cumsum offsets, bytes from a table); 2^26 rows unless ROWS is
# set: one batch of a Utf8 column holds at most 2 GiB (32-bit Arrow offsets), and 2^26 rows of nm (mean 20 B) are 1.3 GB.  Algorithmic bytes are counted from the generated buffers: every input byte read once (values, offsets, data) plus every output byte
# written once (offsets included), so they follow the data rather than a per-row constant.
srows = int(os.environ.get("ROWS", 1 << 26))


def utf8_column(lengths, lo, span):
    """offsets from the lengths; bytes uniform in [lo, lo + span)"""
    offs = torch.zeros(lengths.numel() + 1, dtype=torch.int32, device=dev)
    offs[1:] = torch.cumsum(lengths, 0).to(torch.int32)
    data = torch.randint(lo, lo + span, (int(offs[-1].item()),), dtype=torch.uint8, device=dev, generator=g)
    return data, offs


def run_strings(name, plan, cols, in_bytes, check):
    """cols: [tensor] for fixed width, [(data, offsets)] for Utf8; check(out_batches_on_host) verifies and returns the output bytes.
    Timed: push_device -> finish -> sync (every kernel of the op, no host export)."""
    if ONLY and not any(t in name for t in ONLY.split(",")): return
    import time
    spec, keep = [], []
    for c in cols:
        if isinstance(c, tuple): spec.append((c[0].data_ptr(), 0, srows, c[1].data_ptr())); keep += list(c)
        else: spec.append((c.data_ptr(), 0, srows)); keep.append(c)
    best = None
    for _ in range(REPS or 3):
        with native.NativeOp(plan.plan_bytes(), native.default_conf(agg_initial_groups=1 << 20), 0) as op:
            torch.cuda.synchronize(); t0 = time.perf_counter()
            op.push_device(native.DeviceBatch(spec, srows, 0, keepalive=keep))
            op.finish(); op.sync()
            dt = time.perf_counter() - t0
            m = op.metrics()
            outs = op.pull_all()
        if best is None or dt < best[0]: best = (dt, m, outs)
        del outs
    dt, m, outs = best
    out_bytes = check(outs)
    gbs = (in_bytes + out_bytes) / dt / 1e9
    print(json.dumps({"shape": name, "rows": srows, "out_rows": sum(b.num_rows for b in outs), "wall_ms_push_to_sync": dt * 1e3, "rows_per_s": srows / dt,
                      "alg_bytes": in_bytes + out_bytes, "alg_GBps": gbs, "frac_of_hbm_peak": gbs / peak, "launches": m["gpu_kernel_launches"]}), flush=True)


def contains_rows(data, offs, pat):
    """per row: does the string hold `pat` (torch; positions of the first byte, then a search over the offsets)"""
    hit = torch.ones(data.numel() - len(pat) + 1, dtype=torch.bool, device=dev)
    for j, ch in enumerate(pat.encode()):
        hit &= data[j: data.numel() - len(pat) + 1 + j] == ch
    at = hit.nonzero().squeeze(1)
    row = torch.searchsorted(offs.long(), at, right=True) - 1
    ok = at + len(pat) <= offs.long()[row + 1]
    out = torch.zeros(offs.numel() - 1, dtype=torch.bool, device=dev)
    out[row[ok]] = True
    return out


if any(t in (ONLY or "S1,S2,S3") for t in ("S1", "S2", "S3")):
    import numpy as np
    codes = [a + b for a in "abcdefghij" for b in "abcde"]                   # 50 two-letter codes
    pick = torch.randint(0, 50, (srows,), device=dev, generator=g)
    code_bytes = torch.tensor([[ord(c[0]), ord(c[1])] for c in codes], dtype=torch.uint8, device=dev)
    st_data, st_offs = code_bytes[pick].reshape(-1).contiguous(), torch.arange(0, 2 * srows + 1, 2, dtype=torch.int32, device=dev)
    nm_len = torch.randint(8, 33, (srows,), device=dev, generator=g)
    nm_data, nm_offs = utf8_column(nm_len, ord("a"), 26)
    kk = torch.arange(srows, dtype=torch.int64, device=dev)
    s_sch = T.Schema([T.Field("k", T.int64, False), T.Field("st", T.utf8, False), T.Field("nm", T.utf8, False)])

    def carried_check(mask):
        def check(outs):
            want_rows = int(mask.sum().item())
            assert sum(b.num_rows for b in outs) == want_rows, "row count differs from the torch computation"
            got_k = np.concatenate([b.column("k").to_numpy() for b in outs]) if outs else np.zeros(0, np.int64)
            assert np.array_equal(got_k, kk[mask].cpu().numpy()), "carried keys differ"
            got_sum = 0
            for b in outs:
                c = b.column("nm")
                o = np.frombuffer(c.buffers()[1], np.int32)[c.offset: c.offset + len(c) + 1]
                got_sum += int(np.frombuffer(c.buffers()[2], np.uint8)[o[0]:o[-1]].astype(np.int64).sum())
            assert got_sum == int(nm_data[torch.repeat_interleave(mask, nm_len)].to(torch.int64).sum().item()), "checksum of the carried bytes differs"
            return 8 * want_rows + 4 * (want_rows + 1) + int(nm_len[mask].sum().item())
        return check

    in_s12 = 8 * srows + (st_offs.numel() + nm_offs.numel()) * 4 + st_data.numel() + nm_data.numel()
    chosen = ["ab", "cd", "fa", "je"]
    s1 = PL.ProjectExec([(E.Column("k"), "k"), (E.Column("nm"), "nm")],
                        PL.FilterExec([E.InList(E.Column("st"), [E.Literal(c, T.utf8) for c in chosen])], PL.MemoryExec(s_sch)))
    run_strings("S1 Filter[st IN (4 of 50)] -> Project[k, nm]", s1, [kk, (st_data, st_offs), (nm_data, nm_offs)], in_s12,
                carried_check(torch.isin(pick, torch.tensor([codes.index(c) for c in chosen], device=dev))))
    s2 = PL.ProjectExec([(E.Column("k"), "k"), (E.Column("nm"), "nm")],
                        PL.FilterExec([E.BinaryExpr(E.StartsWith(E.Column("nm"), "ab"), "Or", E.Contains(E.Column("nm"), "xyz"))], PL.MemoryExec(s_sch)))
    starts = (nm_data[nm_offs[:-1].long()] == ord("a")) & (nm_data[nm_offs[:-1].long() + 1] == ord("b"))
    run_strings("S2 Filter[StartsWith(nm,'ab') OR Contains(nm,'xyz')] -> Project[k, nm]", s2, [kk, (st_data, st_offs), (nm_data, nm_offs)], in_s12,
                carried_check(starts | contains_rows(nm_data, nm_offs, "xyz")))
    del st_data, st_offs, nm_data, nm_offs, pick, kk, starts
    # S3: SUM(TryCast(ns AS BIGINT)) GROUP BY k over 1-12-digit numeric strings, 1 % junk (a letter as the first byte)
    ns_len = torch.randint(1, 13, (srows,), device=dev, generator=g)
    ns_data, ns_offs = utf8_column(ns_len, ord("0"), 10)
    junk = torch.rand(srows, device=dev, generator=g) < 0.01
    ns_data[ns_offs[:-1].long()[junk]] = ord("q")
    kg = torch.randint(0, 1 << 16, (srows,), dtype=torch.int64, device=dev, generator=g)
    s3_sch = T.Schema([T.Field("k", T.int64, False), T.Field("ns", T.utf8, False)])
    sum_of = lambda mode: [E.AggExpr("s", mode, PL.create_agg(E.AGG_SUM, [E.TryCast(E.Column("ns"), T.int64) if mode == E.PARTIAL else E.placeholder(T.int64)], s3_sch, T.int64))]
    s3 = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], sum_of(E.FINAL), False,
                    PL.AggExec(PL.HashAgg, [E.GroupingExpr("k", E.Column("k"))], sum_of(E.PARTIAL), False, PL.MemoryExec(s3_sch)))
    val = torch.zeros(srows, dtype=torch.int64, device=dev)                      # torch reference: the decimal value of each string
    start = ns_offs[:-1].long()
    for p in range(12):
        live = ns_len > p
        val = torch.where(live, val * 10 + (ns_data[torch.where(live, start + p, start)].to(torch.int64) - ord("0")), val)
    val[junk] = 0
    want = torch.zeros(1 << 16, dtype=torch.int64, device=dev).index_add_(0, kg, val).cpu().numpy()
    groups = int((torch.bincount(kg, minlength=1 << 16) > 0).sum().item())
    del val, start

    def s3_check(outs):
        got = {int(k): int(s) for b in outs for k, s in zip(b.column("k").to_numpy(), b.column("s").to_numpy())}
        assert len(got) == groups and all(got[k] == int(want[k]) for k in got), "S3 sums differ from the torch computation"
        return 16 * len(got)
    run_strings("S3 SUM(TryCast(ns AS BIGINT)) GROUP BY k", s3, [kg, (ns_data, ns_offs)], 8 * srows + ns_offs.numel() * 4 + ns_data.numel(), s3_check)


# B1-B2: Binary columns through ShuffleWriterExec (the reference-format AggExec(Partial) output carries one Binary column of frozen
# accumulator rows).  Timed like S1-S3: push_device -> finish -> sync, chunks kept on the device.
def run_shuffle_wall(name, plan, spec, keep, conf, n, alg_bytes=None):
    if ONLY and not any(t in name for t in ONLY.split(",")): return
    import time
    best = None
    for _ in range(REPS or 3):
        with native.NativeOp(plan.plan_bytes(), conf, 0) as op:
            torch.cuda.synchronize(); t0 = time.perf_counter()
            op.push_device(native.DeviceBatch(spec, n, 0, keepalive=keep))
            op.finish(); op.sync()
            dt = time.perf_counter() - t0
            m = op.metrics(); chunks = op.shuffle_chunks()
        if best is None or dt < best[0]: best = (dt, m, chunks)
    dt, m, chunks = best
    out = {"shape": name, "rows": n, "wall_ms_push_to_sync": dt * 1e3, "rows_per_s": n / dt, "shuffle_chunk_rows": sum(sum(c["part_rows"]) for c in chunks),
           "encoded_bytes": sum(c["part_off"][-1] for c in chunks), "hot_kernel_ms": m["hot_kernel_ns"] / 1e6, "launches": m["gpu_kernel_launches"]}
    if alg_bytes:
        out.update(alg_bytes=alg_bytes, alg_GBps=alg_bytes / dt / 1e9, frac_of_hbm_peak=alg_bytes / dt / 1e9 / peak)
    print(json.dumps(out), flush=True)


brows = int(os.environ.get("ROWS", 1 << 26))
if any(t in (ONLY or "B1,B2") for t in ("B1", "B2")):
    # B1: 200-way shuffle of [k int64, b Binary] with 10-14-byte values (the size of a SUM+COUNT frozen row); algorithmic bytes from
    # the generated buffers: read 8 + 4 + data bytes, write 8 + 4 + data bytes per row
    bk = torch.randint(-2**62, 2**62, (brows,), dtype=torch.int64, device=dev, generator=g)
    bl = torch.randint(10, 15, (brows,), device=dev, generator=g)
    bdata, boffs = utf8_column(bl, 0, 256)
    b_sch = T.Schema([T.Field("k", T.int64, False), T.Field("b", T.binary, False)])
    b1 = PL.ShuffleWriterExec(PL.MemoryExec(b_sch), ("hash", [E.Column("k")], 200), "", "")
    run_shuffle_wall("B1 shuffle write 200-way [k int64, b Binary 10-14 B]", b1, [(bk.data_ptr(), 0, brows), (bdata.data_ptr(), 0, brows, boffs.data_ptr())],
                     [bk, bdata, boffs], native.default_conf(shuffle_output_on_device=1), brows, alg_bytes=2 * (12 * brows + bdata.numel()))
    del bk, bl, bdata, boffs
    # B2: the q1 map side as Spark plans it: Filter (s = 0.2) -> AggExec(Partial, SUM + COUNT GROUP BY k1, k2) -> ShuffleWriterExec 200-way
    # on (k1, k2); the reference-format partial state (one Binary column) against the columnar partial state of the same plan
    bf = torch.randint(0, 1000, (brows,), dtype=torch.int64, device=dev, generator=g)
    bk1 = torch.randint(0, 1 << 17, (brows,), dtype=torch.int64, device=dev, generator=g)
    bk2 = torch.randint(0, 8, (brows,), dtype=torch.int64, device=dev, generator=g)
    bv = torch.randint(-10**6, 10**6, (brows,), dtype=torch.int64, device=dev, generator=g)
    q_sch = T.Schema([T.Field(nm, T.int64, False) for nm in ("f", "k1", "k2", "v")])
    q_preds = [E.BinaryExpr(E.Column("f"), "GtEq", E.Literal(200, T.int64)), E.BinaryExpr(E.Column("f"), "LtEq", E.Literal(399, T.int64))]
    q_aggs = [E.AggExpr("s", E.PARTIAL, PL.create_agg(E.AGG_SUM, [E.Column("v")], q_sch, T.int64)), E.AggExpr("c", E.PARTIAL, PL.create_agg(E.AGG_COUNT, [E.Column("v")], q_sch, T.int64))]
    q_spec = [(t.data_ptr(), 0, brows) for t in (bf, bk1, bk2, bv)]
    for columnar in (False, True):
        part = PL.AggExec(PL.HashAgg, [E.GroupingExpr("k1", E.Column("k1")), E.GroupingExpr("k2", E.Column("k2"))], q_aggs, True,
                          PL.FilterExec(q_preds, PL.MemoryExec(q_sch)), columnar_state=columnar)
        w = PL.ShuffleWriterExec(part, ("hash", [E.Column("k1"), E.Column("k2")], 200), "", "")
        run_shuffle_wall("B2 q1 map side: Filter -> AggExec(Partial) -> ShuffleWriterExec 200-way, " + ("columnar partial state" if columnar else "reference format (Binary state)"),
                         w, q_spec, [bf, bk1, bk2, bv], native.default_conf(shuffle_output_on_device=1, partial_state_columnar=int(columnar), agg_initial_groups=1 << 20), brows)
    del bf, bk1, bk2, bv


# E1-E2: Filter[f < 800] -> Expand ROLLUP(k1, k2) (3 sets) -> AggExec(Partial) SUM(v), COUNT(v) -> AggExec(Final) over four device-resident
# int64 columns, k1, k2 ~ U[0, 1000).  E1 fuses the Expand into the aggregate (each row read once, one upsert per set); E2 puts a Filter that
# keeps every row between the Expand and the AggExec, which materialises the 3 projections through the standalone ExpandStage.
# Timed like B1-B2: push_device -> finish -> sync.  Algorithmic bytes: 32 B/row, the input read once.
def run_expand_wall(name, plan, spec, keep, conf, n, nsets):
    if ONLY and not any(t in name for t in ONLY.split(",")): return
    import time
    best = None
    for _ in range(REPS or 3):
        with native.NativeOp(plan.plan_bytes(), conf, 0) as op:
            torch.cuda.synchronize(); t0 = time.perf_counter()
            op.push_device(native.DeviceBatch(spec, n, 0, keepalive=keep))
            op.finish(); op.sync()
            dt = time.perf_counter() - t0
            m = op.metrics(); n_out = 0
            while True:
                o = op.pull_device()
                if o is None: break
                n_out += o.array.length; native.release_device_array(o)
        if best is None or dt < best[0]: best = (dt, m, n_out)
    dt, m, n_out = best
    print(json.dumps({"shape": name, "rows": n, "sets": nsets, "out_rows": n_out, "wall_ms_push_to_sync": dt * 1e3, "rows_per_s": n / dt,
                      "row_sets_per_s": n * nsets / dt, "alg_GBps": 32.0 * n / dt / 1e9, "frac_of_hbm_peak": 32.0 * n / dt / 1e9 / peak,
                      "launches": m["gpu_kernel_launches"], "num_groups": m["num_groups"]}), flush=True)


erows = int(os.environ.get("ROWS", 1 << 26))
if any(t in (ONLY or "E1,E2") for t in ("E1", "E2")):
    ef = torch.randint(0, 1000, (erows,), dtype=torch.int64, device=dev, generator=g)
    ek1 = torch.randint(0, 1000, (erows,), dtype=torch.int64, device=dev, generator=g)
    ek2 = torch.randint(0, 1000, (erows,), dtype=torch.int64, device=dev, generator=g)
    ev = torch.randint(-10**6, 10**6, (erows,), dtype=torch.int64, device=dev, generator=g)
    e_sch = T.Schema([T.Field(nm, T.int64, False) for nm in ("k1", "k2", "v", "f")])
    x_sch = T.Schema([T.Field("k1", T.int64, True), T.Field("k2", T.int64, True), T.Field("v", T.int64, False), T.Field("spark_grouping_id", T.int64, False)])
    null64 = E.Literal(None, T.int64)
    e_projs = [[E.Column("k1"), E.Column("k2"), E.Column("v"), E.Literal(0, T.int64)], [E.Column("k1"), null64, E.Column("v"), E.Literal(1, T.int64)],
               [null64, null64, E.Column("v"), E.Literal(3, T.int64)]]
    e_g = [E.GroupingExpr(nm, E.Column(nm)) for nm in ("k1", "k2", "spark_grouping_id")]
    e_aggs = lambda mode, ch: [E.AggExpr("s", mode, PL.create_agg(E.AGG_SUM, ch, x_sch, T.int64)), E.AggExpr("c", mode, PL.create_agg(E.AGG_COUNT, ch, x_sch, T.int64))]
    e_spec = [(t.data_ptr(), 0, erows) for t in (ek1, ek2, ev, ef)]
    for fused in (True, False):
        ex = PL.ExpandExec(x_sch, e_projs, PL.FilterExec([E.BinaryExpr(E.Column("f"), "Lt", E.Literal(800, T.int64))], PL.MemoryExec(e_sch)))
        below = ex if fused else PL.FilterExec([E.BinaryExpr(E.Column("v"), "GtEq", E.Literal(-10**6, T.int64))], ex)
        part = PL.AggExec(PL.HashAgg, e_g, e_aggs(E.PARTIAL, [E.Column("v")]), True, below)
        fin = PL.AggExec(PL.HashAgg, e_g, e_aggs(E.FINAL, [E.placeholder(T.int64)]), False, part)
        run_expand_wall("E1 Filter -> Expand ROLLUP(k1, k2) fused into AggExec(Partial) -> AggExec(Final)" if fused else
                        "E2 Filter -> Expand ROLLUP(k1, k2) -> Filter(all rows) -> AggExec(Partial) -> AggExec(Final), standalone Expand",
                        fin, e_spec, [ef, ek1, ek2, ev], native.default_conf(agg_initial_groups=1 << 20), erows, 3)
    del ef, ek1, ek2, ev


# W1: WindowExec over 2^28 pre-sorted device rows: p = row >> 8 (2^20 partitions of 256 rows), o = (row & 255) >> 2 (peer groups of 4),
# non-null int64 v; row_number, rank, dense_rank, SUM(v), COUNT(v).  Kernel time = the window kernels' events (flags + one reduce-then-scan
# per function): every key and argument is an input column (SUM's TryCast to int64 is v itself), so the window stage is the op's first stage
# and hot_kernel_ns is exactly its events.  Algorithmic bytes: 24 B read (p, o, v) + 28 B written (3 x int32 + 2 x int64) per row.  Results are checked against torch
# after the timed region.
# W2: SortExec(p, o) -> WindowExec(rank, group limit 100) over 2^26 rows, p ~ U[0, 2^16), o ~ U[0, 1000) (the q67 shape), timed as
# whole-op wall time push_device -> finish -> sync; the number of surviving rows is checked against torch.
def cuda_col(o, i, nbytes, dtype):
    return torch.as_tensor(__import__("bench").CudaView(o.array.children[i].contents.buffers[1], nbytes, o), device="cuda").view(dtype)


if any(t in (ONLY or "W1,W2") for t in ("W1", "W2")):
    import time
    w_sch = T.Schema([T.Field(nm, T.int64, False) for nm in ("p", "o", "v")])
    part, order = [E.Column("p")], [(E.Column("o"), False, True)]
    wx = lambda nm, f: E.WindowExpr.rank_like(nm, f)
    if "W1" in (ONLY or "W1"):
        idx = torch.arange(rows, dtype=torch.int64, device=dev)
        wp, wo = idx >> 8, (idx & 255) >> 2
        wv = torch.randint(-10**6, 10**6, (rows,), dtype=torch.int64, device=dev, generator=g)
        w1 = PL.WindowExec(PL.MemoryExec(w_sch), [wx("rn", E.ROW_NUMBER), wx("rk", E.RANK), wx("dr", E.DENSE_RANK),
                                                   E.WindowExpr.agg("s", E.AGG_SUM, [E.Column("v")], T.int64), E.WindowExpr.agg("c", E.AGG_COUNT, [E.Column("v")], T.int64, False)], part, order)
        best = None
        for _ in range(REPS or 3):
            with native.NativeOp(w1.plan_bytes(), native.default_conf(), 0) as op:
                op.push_device(native.DeviceBatch([(t.data_ptr(), 0, rows) for t in (wp, wo, wv)], rows, 0, keepalive=(wp, wo, wv)))
                op.finish()
                o = op.pull_device()
                m = op.metrics()
                if best is None or m["hot_kernel_ns"] < best[0]:
                    pos = idx & 255
                    cs = torch.cumsum(wv.view(-1, 256), 1).view(-1)
                    ok = bool((cuda_col(o, 3, rows * 4, torch.int32) == (pos + 1).int()).all()) and bool((cuda_col(o, 4, rows * 4, torch.int32) == ((pos >> 2) * 4 + 1).int()).all()) \
                        and bool((cuda_col(o, 5, rows * 4, torch.int32) == ((pos >> 2) + 1).int()).all()) and bool((cuda_col(o, 6, rows * 8, torch.int64) == cs).all()) \
                        and bool((cuda_col(o, 7, rows * 8, torch.int64) == pos + 1).all())
                    best = (m["hot_kernel_ns"], m, ok)
                native.release_device_array(o)
        t, m, ok = best
        gbs = 52.0 * rows / t
        print(json.dumps({"shape": "W1 WindowExec row_number, rank, dense_rank, SUM, COUNT over 2^20 partitions", "rows": rows, "verified": ok,
                          "window_kernel_ms": t / 1e6, "rows_per_s": rows / (t * 1e-9), "alg_GBps": gbs, "frac_of_hbm_peak": gbs / peak,
                          "launches": m["gpu_kernel_launches"]}), flush=True)
        del idx, wp, wo, wv, cs, pos
        torch.cuda.empty_cache()
    if "W2" in (ONLY or "W2"):
        n2 = int(os.environ.get("ROWS", 1 << 26))
        wp = torch.randint(0, 1 << 16, (n2,), dtype=torch.int64, device=dev, generator=g)
        wo = torch.randint(0, 1000, (n2,), dtype=torch.int64, device=dev, generator=g)
        wv = torch.randint(-10**6, 10**6, (n2,), dtype=torch.int64, device=dev, generator=g)
        w2 = PL.WindowExec(PL.SortExec(PL.MemoryExec(w_sch), [(E.Column("p"), False, True), (E.Column("o"), False, True)]), [wx("rk", E.RANK)], part, order, 100, False)
        best = None
        for _ in range(REPS or 3):
            with native.NativeOp(w2.plan_bytes(), native.default_conf(), 0) as op:
                torch.cuda.synchronize(); t0 = time.perf_counter()
                op.push_device(native.DeviceBatch([(t.data_ptr(), 0, n2) for t in (wp, wo, wv)], n2, 0, keepalive=(wp, wo, wv)))
                op.finish(); op.sync()
                dt = time.perf_counter() - t0
                m = op.metrics(); n_out = 0
                while True:
                    o = op.pull_device()
                    if o is None: break
                    n_out += o.array.length; native.release_device_array(o)
            if best is None or dt < best[0]: best = (dt, m, n_out)
        dt, m, n_out = best
        key, _ = torch.sort(wp * 1024 + wo)
        i2 = torch.arange(n2, device=dev)
        pstart = torch.cummax(torch.where(torch.cat([torch.ones(1, dtype=torch.bool, device=dev), (key[1:] >> 10) != (key[:-1] >> 10)]), i2, 0), 0).values
        head = torch.cummax(torch.where(torch.cat([torch.ones(1, dtype=torch.bool, device=dev), key[1:] != key[:-1]]), i2, 0), 0).values
        expect = int(((head - pstart + 1) <= 100).sum())
        print(json.dumps({"shape": "W2 SortExec(p, o) -> WindowExec(rank, group limit 100)", "rows": n2, "out_rows": n_out, "verified": n_out == expect,
                          "wall_ms_push_to_sync": dt * 1e3, "rows_per_s": n2 / dt, "launches": m["gpu_kernel_launches"]}), flush=True)
