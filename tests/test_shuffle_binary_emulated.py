"""A subset of tests/test_gpu_shuffle_binary.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): the Binary
shuffle path (data-byte sums, ranking, 64-bit length scans, record layout, length planes and the warp-cooperative byte copy) and the
record-aligned compression blocks, checked without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_binary_shuffle_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_shuffle_binary.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "mixed_schemas and (0.2-64 or 0.0-10000-4096) or all_empty or committed or map_side and keys1 or refused and not large"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and "9 passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
