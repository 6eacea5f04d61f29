"""Dry-run of the training / sampling / native-step GPU test files on a machine WITHOUT a GPU: `ctx()` returns the torch test double, `.cuda()` is the
identity and `device="cuda"` is dropped, so the TEST LOGIC (shapes, arguments, reference arithmetic, tolerances) is
exercised end to end.  A failure on the GPU then points at a kernel, not at the test.  TEST INFRASTRUCTURE ONLY.

    python tools/dryrun_train_gpu_tests.py [pytest args]
"""
import sys, functools
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch, pytest
for name in ("empty", "full", "zeros", "ones", "randn", "tensor", "empty_like", "zeros_like"):
    orig = getattr(torch, name)
    def mk(orig):
        @functools.wraps(orig)
        def f(*a, **k):
            if k.get("device") in ("cuda",) or str(k.get("device", "")).startswith("cuda"):
                k.pop("device")
            return orig(*a, **k)
        return f
    setattr(torch, name, mk(orig))
torch.Tensor.cuda = lambda self, *a, **k: self
torch.cuda.synchronize = lambda *a, **k: None
torch.cuda.is_available = lambda: True
torch.cuda.current_device = lambda: 0
torch.cuda.is_current_stream_capturing = lambda: False
torch.Tensor.pin_memory = lambda self: self
from tests.cabi_double import TorchDouble
from chatts_b200 import _cabi
dbl = TorchDouble()
_cabi.get_context = lambda device=None: dbl
import tests.gpu_util as gu
gu.ctx = lambda: dbl
gu.record = lambda *a, **k: None
import chatts_b200.model as mm
_orig_init = mm.ChatTSForCausalLM.__init__
def _init(self, config, state_dict, device="cpu", **kw):
    kw["use_cuda_graph"] = False          # no CUDA streams / graphs on the CPU
    _orig_init(self, config, state_dict, device="cpu", **kw)
mm.ChatTSForCausalLM.__init__ = _init
import chatts_b200.ts_encoder as te
_orig_te = te.TimeSeriesEmbedding.__init__
def _te_init(self, config, weights, device="cpu", **kw):
    _orig_te(self, config, weights, device="cpu", **kw)
te.TimeSeriesEmbedding.__init__ = _te_init
extra = sys.argv[1:]
if "-k" not in extra:          # the ChatTS-8B-shaped case generates its weights on the device: GPU only
    extra += ["-k", "not (directional and True)"]
sys.exit(pytest.main([os.path.join(ROOT, "tests", f) for f in ("test_gpu_train_kernels.py", "test_gpu_zz_c_train.py", "test_gpu_zz_b_sampling.py", "test_gpu_zz_a_native_step.py",
                                                         "test_gpu_zz_d_attn_bwd_wgmma.py", "test_gpu_zz_e_fused_decode.py")] +
                     ["-q", "-p", "no:cacheprovider", "--runxfail", "-m", "gpu"] + extra))
