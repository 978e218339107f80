"""A subset of tests/test_gpu_tile_stream.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): the tile
kernels' row-to-lane mapping, filter-first predicated loads, next-tile filter prefetch and deferred-row indices, checked
without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_tile_stream_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_tile_stream.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "ragged_tails or selectivity and (none or one or runs) or shared_and_two or bit_offsets and 13 "
                              "or narrow_keys and int8 or count_of_a_column or wide_kernel_arguments and 0.1 and (dec or int) or hashed_fallback"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and "18 passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
