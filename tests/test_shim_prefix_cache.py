"""CPU: the small cases of tests/test_gpu_attn_prefill_paged.py (the paged prefill attention against the fp32 statement, bit for bit
against cts_attn_prefill and against a full prefill, foreign cache rows, argument errors) and of tests/test_gpu_zz_h_prefix_cache.py
(prefix caching on the tiny model) executed from the kernel SOURCE through the "CUDA on CPU" shim (driven by tools/shim_gpu_tests.py)."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,least", [("test_gpu_attn_prefill_paged.py", 30), ("test_gpu_zz_h_prefix_cache.py", 8)])
def test_prefix_cache_cases_pass_from_kernel_source(name, least):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", name)],
                       capture_output=True, text=True, timeout=2400, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= least and "failed" not in r.stdout, tail
