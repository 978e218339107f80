"""A subset of tests/test_gpu_strings.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): the Utf8 VM
instructions, the selection vector of the filter kernel and the variable-width gather kernels, checked without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_strings_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_strings.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "kat or edge_cases or predicate and (0 or 6 or 12 or 15 or 17 or 21) or carry_utf8_columns and half or unreferenced "
                              "or sliced_host or direct_import or misaligned or staging or literal_pool or count_and_sum or fused or long_strings or identity "
                              "or schema or unsupported"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
