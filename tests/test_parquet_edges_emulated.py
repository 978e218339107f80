"""A subset of tests/test_gpu_parquet_edges.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): decimals at
every storage width class, dictionary index widths 0..9 (the width-0 rewrite included), widths growing page by page with a mid-chunk
fallback to PLAIN, one page per row, NULL runs next to bit-packed levels, the refusals and 25 of the seeded pruning predicates,
checked without a GPU.  The emulator runs the real host framing and the kernels' logic; the H100 run has the final say on the device."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_parquet_edges_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_parquet_edges.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "decimal and (p1- or p2- or p9- or p10- or p18- or p19- or p38-) or 1entries or 2entries or 5entries or 257entries "
                              "or grows or one_page_per_row and 4097 and runs or level_runs and 13 or refused or seed100"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
