"""A subset of tests/test_gpu_bloom.py on the EMULATED device (tools/emu, see tests/test_pipeline_emulated.py): XxHash64 over
the Bool / Int8 / Int16 / Int32 / Int64 / Date32 / Timestamp / Utf8 children, might_contain with negative combined hashes and
narrow ints, the NULL cases, the per-program filter limit, and the BLOOM_FILTER aggregate's None cases and Partial /
PartialMerge / Final in both state forms, checked without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_bloom_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"), os.path.join(ROOT, "tests", "test_gpu_bloom.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "reference_vectors or every_type_with_nulls and children9 or negative_combined or null_filter "
                              "or row_for_row and 64-30 and not 67108864 or more_than_four or bloom_agg_none_cases or partial_partial_merge_final"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
