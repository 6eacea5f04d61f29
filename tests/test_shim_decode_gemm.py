"""CPU: the kernel cases of tests/test_gpu_decode_gemm.py at the small shapes (the streaming decode GEMM against gemm_tn_kernel, bit for
bit, in every tile height / K blocks per slot / ring depth, and its argument errors) executed from the kernel SOURCE of
csrc/gemm_tcgen05.cu through the "CUDA on CPU" shim (driven by tools/shim_gpu_tests.py)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_decode_gemm_kernel_cases_pass_from_kernel_source():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", "test_gpu_decode_gemm.py")],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= 20 and "failed" not in r.stdout, tail
