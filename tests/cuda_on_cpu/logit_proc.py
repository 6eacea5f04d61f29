"""TEST INFRASTRUCTURE ONLY -- the logits-processor kernels (chatts_b200/csrc/logit_proc.cu) compiled by g++ against the "CUDA on CPU"
shim into libchatts_shim_logit_proc.so, linked against libchatts_shim.so (build.py) so both share ONE shim runtime; attach() binds the
entry points onto a shim Context (shim.py).  The source is copied unchanged."""
import ctypes as C
import os
import shutil
import subprocess

from . import build as shim_build

SOURCE = "logit_proc.cu"
SYMBOLS = ("cts_logit_proc_apply", "cts_logit_proc_update")
OUT = os.path.join(os.path.dirname(shim_build.OUT), "libchatts_shim_logit_proc.so")


def build(force=False):
    base = shim_build.build()                                 # also places the shim headers next to the copied sources
    bdir = os.path.dirname(base)
    src = os.path.join(shim_build.CSRC, SOURCE)
    deps = [src, base, os.path.abspath(__file__), os.path.join(shim_build.ROOT, "include", "chatts_b200.h")]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    cpp = os.path.join(bdir, SOURCE.replace(".cu", ".cpp"))
    shutil.copyfile(src, cpp)
    tmp = OUT + f".{os.getpid()}.tmp"
    flags = ["-std=c++17", "-O2", "-fno-strict-aliasing", "-g", "-fPIC", "-pthread", "-w", "-I", bdir, "-I",
             os.path.join(shim_build.ROOT, "include")]
    r = subprocess.run(["g++"] + flags + ["-shared", cpp, "-o", tmp, "-L", bdir, "-l:" + os.path.basename(base), f"-Wl,-rpath,{bdir}"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("logit_proc shim build failed:\n" + r.stderr[-6000:])
    os.replace(tmp, OUT)
    return OUT


def attach(ctx):
    """Give a shim Context (shim.shim_context()) the logits-processor entry points, with the argument types of the real binding."""
    from chatts_b200 import _cabi
    lib, real = C.CDLL(build()), _cabi.load_library()
    for name in SYMBOLS:
        fn, rf = getattr(lib, name), getattr(real, name)
        fn.argtypes, fn.restype = rf.argtypes, rf.restype
        setattr(ctx.lib, name, fn)
    return ctx
