"""CPU: a quick subset of tests/test_gpu_zz_o_sampling_rows.py executed from the kernel SOURCE through the "CUDA on CPU" shim (driven by
tools/shim_gpu_tests.py): cts_sample_advance_rows with uniform parameters against cts_sample_advance on a far-tail row, the edge rows
and an odd vocabulary; greedy and sampled rows mixed in one launch against cts_greedy_advance and the statement; and the min_tokens
and allowed-id masks chained into it.  About two minutes."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ("(far_tail and bf16-start-1.0) or (edges and bf16) or (vocab_sizes and 1003) or (mixed and 1000) "
         "or (refused and bf16 and (min_tokens or allowed_ids))")


def test_rows_sampler_cases_pass_from_kernel_source():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", "test_gpu_zz_o_sampling_rows.py"),
                        "-k", CASES], capture_output=True, text=True, timeout=1200, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= 15 and "failed" not in r.stdout, tail
