"""CPU: the tiny-model cases of tests/test_gpu_zz_g_decode_parity.py (the default decode path at batch 1 and 8 in bf16 and fp16 and the
native step at batch 8: every
step's logits and every written KV row against the oracle, no cache row outside the live slots moved; and the decode of a batch on a
NaN-filled cache bit-identical to the decode on a zeroed one) executed from the kernel SOURCE through the "CUDA on CPU" shim (driven
by tools/shim_gpu_tests.py)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_decode_parity_and_isolation_pass_from_kernel_source():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", "test_gpu_zz_g_decode_parity.py")],
                       capture_output=True, text=True, timeout=1500, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= 9 and "failed" not in r.stdout, tail
