"""TEST INFRASTRUCTURE ONLY -- the FP8 kernels (chatts_b200/csrc/gemm_fp8.cu) compiled by g++ against the "CUDA on CPU" shim into
libchatts_shim_fp8.so.  It is linked against libchatts_shim.so (build.py), so both libraries share ONE shim runtime (fibers, dynamic shared
memory, mbarriers, the ctx); attach() binds its entry points onto a shim Context (shim.py).  The source is copied unchanged: it spells its
warp-level instructions for the shim itself (CTS_HOST_SHIM branches)."""
import ctypes as C
import os
import shutil
import subprocess

from . import build as shim_build

SOURCE = "gemm_fp8.cu"
SYMBOLS = ("cts_gemm_fp8", "cts_gemm_fp8_suggest_split", "cts_fp8_dequant")
OUT = os.path.join(os.path.dirname(shim_build.OUT), "libchatts_shim_fp8.so")


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
        raise RuntimeError("FP8 shim build failed:\n" + r.stderr[-6000:])
    os.replace(tmp, OUT)
    return OUT


def attach(ctx):
    """Give a shim Context (shim.shim_context()) the FP8 entry points, with the argument types of the real binding."""
    from chatts_b200 import _cabi
    lib, real = C.CDLL(build()), _cabi.load_library()
    for name in SYMBOLS:
        fn, rf = getattr(lib, name), getattr(real, name)
        fn.argtypes, fn.restype = rf.argtypes, rf.restype
        setattr(ctx.lib, name, fn)
    return ctx
