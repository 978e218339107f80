"""The C-ABI library loads without a GPU and exports every symbol include/blaze_b200.h declares."""
import ctypes as C
import os
import re

from blaze_b200 import native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    hdr = open(os.path.join(ROOT, "include", "blaze_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(b200q_[a-z0-9_]+)\s*\(", hdr)))


def test_every_declared_symbol_is_exported():
    names = _declared()
    assert len(names) >= 18 and set(names) == set(native.SYMBOLS)
    lib = C.CDLL(native.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/blaze_b200.h but not exported"


def test_identity_calls_work_without_gpu():
    assert native.lib.b200q_version() >= 100
    assert b"sm_90a" in native.lib.b200q_build_info()
    assert native.device_count() >= 0
    c = native.default_conf()
    assert c.batch_size == 10000 and c.suggested_batch_mem_size == 8388608          # commons/src/lib.rs:74-82
    assert c.partial_agg_skipping_ratio == 0.999 and c.partial_agg_skipping_min_rows == 20000   # agg_ctx.rs:177-178
    assert c.struct_size == C.sizeof(native.Conf)


def test_struct_layouts_match_the_header():
    # sizes implied by the header's field lists (LP64)
    assert C.sizeof(native.ArrowArray) == 80 and C.sizeof(native.ArrowSchema) == 72
    assert C.sizeof(native.ArrowDeviceArray) == 80 + 8 + 8 + 8 + 24
    assert C.sizeof(native.Metrics) == 8 + 15 * 8


def test_no_cpu_fallback_without_device():
    if native.device_count() > 0:
        return
    from blaze_b200 import exprs as E, plans as PL, types as T
    s = T.Schema([T.Field("a", T.int64, False)])
    plan = PL.FilterExec([E.BinaryExpr(E.Column("a"), "Lt", E.Literal(1, T.int64))], PL.MemoryExec(s))
    try:
        native.NativeOp(plan.plan_bytes())
        assert False, "op creation must fail loudly without a CUDA device"
    except native.NativeError as e:
        assert e.code == native.ERR_NO_DEVICE
