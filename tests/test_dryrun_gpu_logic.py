"""The LOGIC of the training / sampling / executor GPU tests (shapes, arguments, reference arithmetic, tolerances) is exercised on
CPU on every run: tools/dryrun_train_gpu_tests.py executes those test files with the C-ABI replaced by the torch test double, in a
subprocess (it monkeypatches torch.cuda).  A red GPU run of those files then points at a kernel, not at a test bug."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gpu_test_files_of_the_training_path_pass_through_the_double():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "dryrun_train_gpu_tests.py")], capture_output=True, text=True, timeout=900,
                       cwd=ROOT)
    tail = (r.stdout + r.stderr)[-1500:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and " failed" not in r.stdout, tail
