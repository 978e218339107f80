"""A subset of tests/test_gpu_expr_numeric_edges.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py):
integer, float and decimal expressions through the VM kernel and the default dispatch, NaN payloads, the errors, the lean
kernel and the merged filter intervals, checked without a GPU.  The H100 run has the final say on NaN bits and on the
conversion instructions, which the emulator maps to host arithmetic."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_expr_numeric_edges_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_expr_numeric_edges.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "vm_direct and (64 or decimal) or nan_payloads and vm or errors and 64 and 1 or overflow_is and 1 "
                              "or lean_kernel_at and Lt and (-1 or 9223372036854775807) or intervals and int64-float64-0"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
