"""CPU: the kernel cases of tests/test_gpu_fp8.py (every e4m3 code at every fragment position, split-K partials at the small shapes, the
dequantisation bit for bit) executed from the kernel SOURCE of csrc/gemm_fp8.cu through the "CUDA on CPU" shim (tests/cuda_on_cpu/fp8.py,
driven by tools/shim_gpu_tests.py)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fp8_kernel_cases_pass_from_kernel_source():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", "test_gpu_fp8.py")],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= 20 and "failed" not in r.stdout, tail
