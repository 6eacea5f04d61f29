"""CPU: the small cases of tests/test_gpu_logprobs.py (cts_logprobs against log_softmax: small vocabularies, ties and non-finite entries,
row strides, column mode, argument errors) and the tiny-model cases of tests/test_gpu_zz_i_logprobs.py executed from the kernel SOURCE
through the "CUDA on CPU" shim (driven by tools/shim_gpu_tests.py)."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,least", [("test_gpu_logprobs.py", 50), ("test_gpu_zz_i_logprobs.py", 3)])
def test_logprobs_cases_pass_from_kernel_source(name, least):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", name)],
                       capture_output=True, text=True, timeout=2400, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= least and "failed" not in r.stdout, tail
