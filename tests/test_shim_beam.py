"""CPU: the small cases of tests/test_gpu_beam.py (cts_beam_select against its restatement over several steps, cts_beam_fork_kv with
swaps, 3-cycles and tails at offsets 0, 1 and page_size - 1, the argument errors) executed from the kernel SOURCE through the "CUDA on
CPU" shim (driven by tools/shim_gpu_tests.py)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_beam_cases_pass_from_kernel_source():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", "test_gpu_beam.py")],
                       capture_output=True, text=True, timeout=2400, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= 11 and "failed" not in r.stdout, tail
