"""A subset of tests/test_gpu_join_scale.py and tests/test_gpu_sort_scale.py on the EMULATED device (tools/emu, see
tests/test_pipeline_emulated.py), at their small sizes: the fused join path with payloads of every width at odd offsets,
sides of 17 columns, one duplicate among 10^6 build keys, integer keys at their extremes and of mixed widths, two keys in both orders, probe clusters that wrap,
the refusal of a 2^32-row output and the 2^21-row single-key join; sorts of the float and decimal edges, digits that never
vary and fetch around the tile size — without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++ (C++20)")
def test_join_and_sort_on_the_emulated_device(tmp_path):
    env = dict(os.environ, B200Q_EMU_DIR=str(tmp_path), B200Q_EMU_REUSE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "run_gpu_suite.py"),
                        os.path.join(ROOT, "tests", "test_gpu_join_scale.py"), os.path.join(ROOT, "tests", "test_gpu_sort_scale.py"),
                        "-m", "gpu", "-q", "-p", "no:cacheprovider",
                        "-k", "unique_build_keys and n1e3 and m50 or column_counts and 17 or extremes and mapR or two_keys or wrap "
                              "or refused and 2048 or one_probe_row or one_pair "
                              "or key_types and (f32 or f64 or dec) and asc or decimal_words or digits and (dec or f64) or fetch"],
                       capture_output=True, text=True, env=env, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
