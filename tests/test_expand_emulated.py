"""A subset of tests/test_gpu_expand.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): the standalone
ExpandStage, the grouping-set aggregate kernel (constant keys, per-set arguments, skipped accumulators) and its refusals, checked
without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_expand_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_expand.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "kats or at_the_top or filter_above or utf8 or rollup_cube_grouping_sets and one_op "
                              "or multi_distinct and with_regular or refused or zero_projections"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and "15 passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
