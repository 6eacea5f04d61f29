"""TEST INFRASTRUCTURE ONLY -- the beam-search kernels (chatts_b200/csrc/beam.cu) compiled by g++ against the "CUDA on CPU"
shim into libchatts_shim_beam.so, linked against libchatts_shim.so (build.py) so both share ONE shim runtime; attach() binds the
entry points onto a shim Context (shim.py).  The source is copied unchanged."""
import ctypes as C
import os
import shutil
import subprocess

from . import build as shim_build

SOURCE = "beam.cu"
SYMBOLS = ("cts_beam_select", "cts_beam_fork_kv")
OUT = os.path.join(os.path.dirname(shim_build.OUT), "libchatts_shim_beam.so")


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
        raise RuntimeError("beam shim build failed:\n" + r.stderr[-6000:])
    os.replace(tmp, OUT)
    return OUT


def attach(ctx):
    """Give a shim Context (shim.shim_context()) the beam-search entry points, with the argument types of the real binding."""
    from chatts_b200 import _cabi
    lib, real = C.CDLL(build()), _cabi.load_library()
    for name in SYMBOLS:
        fn, rf = getattr(lib, name), getattr(real, name)
        fn.argtypes, fn.restype = rf.argtypes, rf.restype
        setattr(ctx.lib, name, fn)
    return ctx
