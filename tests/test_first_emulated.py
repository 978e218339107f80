"""A subset of tests/test_gpu_first.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): the FIRST slot-lock
protocol under many threads per group, every value type bit for bit, Partial -> Final through both state formats, the dropDuplicates
and multi-DISTINCT shapes and a fused ROLLUP, checked without a GPU.  Deferred replays need more than 2^19 groups, beyond what the
emulator runs in reasonable time; they are covered on the GPU only."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_first_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_first.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "kat or (every_value_type and (i8 or f64 or dec or bool) and not two_ops) or global_first or rollup or drop_dup "
                              "or partial_final_forms and (three or columnar) or multi_distinct"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
