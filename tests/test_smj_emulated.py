"""A subset of tests/test_gpu_smj.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): reference goldens of every
join type, right-only rows settled across one-row left batches, sort options over NULL keys with one and two keys, unsorted input
on both sides and misuse of the attach call — so the CPU suite covers the merge kernels' logic without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_sort_merge_join_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_smj.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "goldens and (inner_one or left_sort_order or right_multiple or full_multiple or anti or semi or existence) "
                              "or settled or misuse or before_attach or unsorted_across or unsorted_right "
                              "or sort_options and i64 and (inner or full) and desc_nf"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
