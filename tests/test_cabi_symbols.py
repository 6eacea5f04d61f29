"""CPU: the C-ABI library loads and exports every symbol include/chatts_b200.h declares; the product path
fails loudly (no fallback) when there is no GPU."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "chatts_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(cts_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from chatts_b200 import _cabi
    if not os.path.exists(_cabi.LIB_PATH):
        from chatts_b200.build import build
        build(verbose=False)
    lib = ctypes.CDLL(_cabi.LIB_PATH)
    syms = _header_symbols()
    assert len(syms) >= 18
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/chatts_b200.h but not exported"
    assert sorted(_cabi.SYMBOLS) == syms, "chatts_b200/_cabi.py SYMBOLS out of sync with the header"
    lib.cts_arch.restype = ctypes.c_char_p
    assert lib.cts_arch() == b"sm_90a"
    assert lib.cts_version() >= 100


def test_sass_is_hopper_native():
    """wgmma / TMA must be in the shipped SASS (HGMMA, UTMALDG), next to the warp-level HMMA of the attention kernels."""
    import shutil
    import subprocess
    from chatts_b200 import _cabi
    if shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        pytest.skip("cuobjdump not available")
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([exe, "-sass", _cabi.LIB_PATH], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "HMMA"):
        assert mnemonic in sass, mnemonic
    assert "sm_90a" in subprocess.run([exe, "-lelf", _cabi.LIB_PATH], capture_output=True, text=True).stdout


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_silent_fallback_without_gpu():
    from chatts_b200 import ChatTSConfig, _cabi
    from chatts_b200.model import ChatTSForCausalLM
    from chatts_b200.weights import synthetic_state_dict
    with pytest.raises(_cabi.CtsError):
        _cabi.Context()
    cfg = ChatTSConfig.tiny()
    with pytest.raises(_cabi.CtsError):
        ChatTSForCausalLM(cfg, synthetic_state_dict(cfg, device="cpu"))


def test_product_never_imports_oracle():
    import glob
    for f in glob.glob(os.path.join(ROOT, "chatts_b200", "**", "*.py"), recursive=True):
        src = open(f).read()
        assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f


def _header_prototypes():
    """{symbol: [parameter kinds]} parsed from the header; kinds: 'p' pointer, 'i' int, 'l' long long, 'f' float, 'u' unsigned long long."""
    src = open(os.path.join(ROOT, "include", "chatts_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"typedef struct\s*\w*\s*\{.*?\}\s*\w+;", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(?:int|long long|const char\*|void|unsigned)\s+(cts_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        name, params = m.group(1), m.group(2).strip()
        kinds = []
        if params and params != "void":
            for prm in params.split(","):
                prm = " ".join(prm.split())
                if "*" in prm:
                    kinds.append("p")
                elif prm.startswith("unsigned long long"):
                    kinds.append("u")
                elif prm.startswith("long long"):
                    kinds.append("l")
                elif prm.startswith("float"):
                    kinds.append("f")
                elif prm.startswith("int") or prm.startswith("unsigned"):
                    kinds.append("i")
                else:
                    kinds.append("?" + prm)
        protos[name] = kinds
    return protos


def test_ctypes_signatures_match_the_header():
    """Every hand-written `argtypes` list in chatts_b200/_cabi.py against the prototype in include/chatts_b200.h: same number of
    parameters, same class (pointer / int / long long / float) in every position.  A mismatch here is a corrupted call on the GPU."""
    from chatts_b200 import _cabi
    if not os.path.exists(_cabi.LIB_PATH):
        from chatts_b200.build import build
        build(verbose=False)
    lib = _cabi.load_library() if hasattr(_cabi, "load_library") else _cabi._load()
    protos = _header_prototypes()
    assert set(protos) >= set(_cabi.SYMBOLS) - {"cts_arch", "cts_version"}, sorted(set(_cabi.SYMBOLS) - set(protos))
    C = ctypes
    kind_of = {C.c_void_p: "p", C.c_char_p: "p", C.c_int: "i", C.c_longlong: "l", C.c_float: "f", C.c_ulonglong: "u"}
    checked = 0
    for name, kinds in sorted(protos.items()):
        fn = getattr(lib, name)
        if fn.argtypes is None:
            continue
        got = []
        for a in fn.argtypes:
            if a in kind_of:
                got.append(kind_of[a])
            elif hasattr(a, "contents") or getattr(a, "_type_", None) is not None and not isinstance(getattr(a, "_type_", None), str):
                got.append("p")                                  # POINTER(struct) / POINTER(c_void_p)
            else:
                got.append("?" + repr(a))
        assert got == kinds, f"{name}: ctypes {''.join(got)} vs header {''.join(kinds)}"
        checked += 1
    assert checked >= 40, checked


def test_ctypes_structs_match_the_header_layout(tmp_path):
    """The argument structs of the C-ABI: field names, offsets and sizes as gcc lays them out from include/chatts_b200.h against the
    ctypes.Structure mirrors in chatts_b200/_cabi.py (a drifted struct is silent corruption on the GPU, not an error)."""
    import shutil
    import subprocess
    from chatts_b200 import _cabi
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    pairs = {"cts_gemm_args": _cabi.GemmArgs, "cts_chain_args": _cabi.ChainArgs, "cts_fused_gemm_args": _cabi.FusedGemmArgs,
             "cts_ts_encode_args": _cabi.TsEncodeArgs, "cts_layer_weights": _cabi.LayerWeights, "cts_decoder_step_args": _cabi.DecoderStepArgs}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "chatts_b200.h"', "int main(void) {"]
    for cname, st in pairs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in st._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu %zu\\n", offsetof({cname}, {fname}), sizeof((({cname}*)0)->{fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    r = subprocess.run([gcc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr          # a field name that exists only on the Python side fails here
    out = subprocess.run([str(exe)], capture_output=True, text=True).stdout.split("\n")
    got = {}
    for ln in out:
        parts = ln.split()
        if parts:
            got[parts[0]] = tuple(int(x) for x in parts[1:])
    for cname, st in pairs.items():
        assert got[cname] == (ctypes.sizeof(st),), f"sizeof({cname}) = {got[cname][0]} in C, {ctypes.sizeof(st)} in ctypes (missing trailing field?)"
        for fname, _ in st._fields_:
            f = getattr(st, fname)
            assert got[f"{cname}.{fname}"] == (f.offset, f.size), f"{cname}.{fname}: C {got[f'{cname}.{fname}']} vs ctypes {(f.offset, f.size)}"
