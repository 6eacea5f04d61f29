"""CPU: a quick subset of tests/test_gpu_zz_n_sampling_dist.py executed from the kernel SOURCE through the "CUDA on CPU" shim (driven by
tools/shim_gpu_tests.py): the far tail behind a dominant token (400 draws, every token with mass, the tail distribution), the
min_tokens and allowed-id masks chained into the sampler (no refused id), top-k ties, degenerate rows against greedy, and draw-for-draw
agreement at the small vocabularies.  The whole selection (``python tools/shim_gpu_tests.py tests/test_gpu_zz_n_sampling_dist.py``)
takes about ten minutes."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ("(tail_support and bf16-start-g18-t1) or (refused_ids and (min_tokens or allowed_ids) and bf16) or ties "
         "or (degenerate and (1000 or 1003)) or (draw_for_draw and not 152064 and not 8193)")


def test_sampler_cases_pass_from_kernel_source():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shim_gpu_tests.py"), os.path.join("tests", "test_gpu_zz_n_sampling_dist.py"),
                        "-k", CASES], capture_output=True, text=True, timeout=1200, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    passed = [int(n) for n in re.findall(r"(\d+) passed", r.stdout)]
    assert passed and passed[0] >= 11 and "failed" not in r.stdout, tail
