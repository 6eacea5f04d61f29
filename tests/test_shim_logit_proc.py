"""CPU: the small cases of tests/test_gpu_logit_proc.py (apply against the statement at V = 1000 / 1003 with NaN / inf, strides and
optional tables, the repetition-penalty-only case, the update, argument errors) and the tiny-model cases of
tests/test_gpu_zz_m_logit_proc.py executed from the kernel SOURCE through the "CUDA on CPU" shim (driven by tools/shim_gpu_tests.py)."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,least", [("test_gpu_logit_proc.py", 20), ("test_gpu_zz_m_logit_proc.py", 7)])
def test_logit_proc_cases_pass_from_kernel_source(name, least):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", name)],
                       capture_output=True, text=True, timeout=2400, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= least and "failed" not in r.stdout, tail
