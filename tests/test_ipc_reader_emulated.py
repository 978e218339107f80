"""A subset of tests/test_gpu_ipc_reader.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): round trips of
every type with and without NULLs (records at every bit offset mod 32, records above staging_rows, a record straddling two blocks),
the push rules and every malformed-push class, checked without a GPU.  The reduce plans over the map side's files, the join probe and
pull_device are covered on the GPU only."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_ipc_reader_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_ipc_reader.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "round_trip_every_type and (i32-none or bool-some or bin-flag or dec-some or utf8-some or f64-some) "
                              "or malformed or push_rules or straddling or empty_pushes"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
