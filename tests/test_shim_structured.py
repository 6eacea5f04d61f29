"""CPU: the small cases of tests/test_gpu_structured.py (mask build at V = 1000 / 1003 for 1 and 37 states, mask apply with NaN / inf and
row strides, the advance, argument errors) and the tiny-model cases of tests/test_gpu_zz_k_structured.py executed from the kernel SOURCE
through the "CUDA on CPU" shim (driven by tools/shim_gpu_tests.py)."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,least", [("test_gpu_structured.py", 10), ("test_gpu_zz_k_structured.py", 6)])
def test_structured_cases_pass_from_kernel_source(name, least):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", name)],
                       capture_output=True, text=True, timeout=2400, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= least and "failed" not in r.stdout, tail
