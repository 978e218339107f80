"""A subset of tests/test_gpu_agg_numeric_edges.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py):
the wide tile kernel and the generic kernel against the exact reference on f64 zeros and specials, decimal128 carries and
i128 wrapping, and int64 extremes, checked without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_numeric_edges_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_agg_numeric_edges.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "numeric_edges and (default or generic) and ((f64 and sum) or (f64 and min) or dec38_0 or (int and min and not narrow)) "
                              "or partial_state"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and "14 passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
