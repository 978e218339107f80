"""tests/test_gpu_step_fixed_cost.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): the hashed-slot emit with
and without keys outside the sampled dense range, the counters of every launch coming back through the kernel-written snapshot.
Table growth under deferral needs more than 2^19 groups and the stream / event pool test needs torch on a real device: GPU only."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_step_fixed_cost_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_step_fixed_cost.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider", "-k", "hashed_emit"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and "4 passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
