"""A subset of tests/test_gpu_window.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): the KATs as one batch
and as 1-row batches, random tables against the oracle, batch splits, the group limit and the combining rule, whole ops, the
brute-force check, numeric edges against tests/exact_agg.py and the stage structure, without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_window_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_window.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "kats or random_vs_oracle and (int32 or float64 or decimal) and p1 or batch_splits and 2048 "
                              "or group_limit and (0- or 2147483648-) or combines or one_op or brute or exact_bound or min_max or no_projection "
                              "or refuses_a_parent"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
