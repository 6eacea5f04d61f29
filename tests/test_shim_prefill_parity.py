"""CPU: the reduced-width cases of tests/test_gpu_zz_p_prefill_parity.py executed from the kernel SOURCE through the "CUDA on CPU" shim
(driven by tools/shim_gpu_tests.py): the prefill layer stages against their fp64 statements, the three RMSNorm kernels at h = 4096 /
5120 (the generic kernel with two and three vector slots), the RoPE chunk loop past 65535 rows, the persistent GEMM over several L2
groups with an uneven last one, and the prefill attention over ragged, NaN-padded buffers."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_prefill_parity_passes_from_kernel_source():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", "test_gpu_zz_p_prefill_parity.py")],
                       capture_output=True, text=True, timeout=2400, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= 35 and "failed" not in r.stdout, tail
