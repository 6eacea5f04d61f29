"""TEST INFRASTRUCTURE ONLY -- builds libchatts_shim.so: a few kernel source files of chatts_b200/csrc compiled by g++ against the
"CUDA on CPU" shim (common.cuh in this directory).  The sources are COPIED next to the shim header (so their `#include "common.cuh"`
resolves to it) into a build directory and compiled (SUBSTITUTIONS lists the only textual changes made to a copy)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "chatts_b200", "csrc")
SOURCES = ["sampling.cu", "train_elementwise.cu", "allreduce_ll.cu", "attention_bwd.cu", "attention_bwd_wgmma.cu", "gemm_decode_fused.cu", "gemm_tcgen05.cu", "lora_wgrad_mma.cu", "attention.cu", "elementwise.cu", "ts_frontend.cu", "decoder_step.cu", "allreduce.cu", "ts_encoder_fused.cu", "gemm_w4.cu", "gemm_w4_mma.cu"]
OUT = os.path.join(HERE, "_build", "libchatts_shim.so")
# Files that are GPU-validated are not edited for the shim's sake (not even a spelling): their two non-portable spellings are replaced
# in the COPY.  Everything else in the copy is the product source, byte for byte.
_CP16 = '"cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz) : "memory");'
SUBSTITUTIONS = {
    # the warp-level instructions: cp.async is a copy, ldmatrix / mma.sync go to the fragment-exact emulation of common.cuh
    "lora_wgrad_mma.cu": [
        ("asm volatile(" + _CP16, "if (valid) memcpy(smem, gmem, 16); else memset(smem, 0, 16); (void)sz;"),
        ('asm volatile("cp.async.commit_group;" ::: "memory");', ""),
        ('asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");', ""),
        ('''asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));''', "shim_ldmatrix_x4(addr, r, true);"),
        ('''asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));''',
         "shim_mma_m16n8k16(c, a, b0, b1, true);"),
        ('''asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));''',
         "shim_mma_m16n8k16(c, a, b0, b1, false);"),
    ],
    "attention.cu": [
        ("asm volatile(" + _CP16, "if (valid) memcpy(smem, gmem, 16); else memset(smem, 0, 16); (void)sz;"),
        ('asm volatile("cp.async.commit_group;" ::: "memory");', ""),
        ('asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");', ""),
        ('''asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));''', "shim_ldmatrix_x4(addr, r, false);"),
        ('''asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));''', "shim_ldmatrix_x4(addr, r, true);"),
        ('''asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));''',
         "{ const uint32_t a_[4] = {a0, a1, a2, a3}; shim_mma_m16n8k16(c, a_, b0, b1, true); }"),
        ('''asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));''',
         "{ const uint32_t a_[4] = {a0, a1, a2, a3}; shim_mma_m16n8k16(c, a_, b0, b1, false); }"),
        ("extern __shared__ __align__(128) uint8_t pf_smem[];", "uint8_t* pf_smem = g_dyn_smem;"),
        ("extern __shared__ uint8_t dec_raw[];", "uint8_t* dec_raw = g_dyn_smem;"),
        ("extern __shared__ uint8_t wg_raw[];", "uint8_t* wg_raw = g_dyn_smem;"),
    ],
    "attention_bwd_wgmma.cu": [("extern __shared__ uint8_t bq_raw[];", "uint8_t* bq_raw = g_dyn_smem;"),
                               ("extern __shared__ uint8_t bkv_raw[];", "uint8_t* bkv_raw = g_dyn_smem;")],
    "elementwise.cu": [("    ss_cta = v;\n  }\n  cluster.sync();", "    ss_cta = v;\n    shim_publish_static(&ss_cta);\n  }\n  cluster.sync();"),
                       ("*cluster.map_shared_rank(&ss_cta, r)", "*(float*)shim_static_peer((unsigned)r)")],
    "allreduce.cu": [
        ('asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");', "shim_st_release(p, v);"),
        ('asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");', "v = shim_ld_acquire(p);"),
        ('asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");',
         "{ const volatile float* s_ = reinterpret_cast<const volatile float*>(p); v.x = s_[0]; v.y = s_[1]; v.z = s_[2]; v.w = s_[3]; }"),
        ('asm volatile("st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(best), "f"(gidx) : "memory");',
         "{ volatile float* d_ = reinterpret_cast<volatile float*>(dst); d_[0] = best; d_[1] = gidx; }"),
        ('asm volatile("ld.relaxed.sys.global.v2.f32 {%0, %1}, [%2];" : "=f"(a), "=f"(c) : "l"(src) : "memory");',
         "{ const volatile float* s_ = reinterpret_cast<const volatile float*>(src); a = s_[0]; c = s_[1]; }"),
        ("    ss_cta = v;\n  }\n  cluster.sync();", "    ss_cta = v;\n    shim_publish_static(&ss_cta);\n  }\n  cluster.sync();"),
        ("*cluster.map_shared_rank(&ss_cta, r)", "*(float*)shim_static_peer((unsigned)r)"),
    ],
    "gemm_w4_mma.cu": [
        ('''asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));''', "shim_ldmatrix_x4(addr, r, false);"),
        ('''asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));''',
         "shim_mma_m16n8k16(c, a, b0, b1, true);"),
        ('''asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));''',
         "shim_mma_m16n8k16(c, a, b0, b1, false);"),
    ],
    "gemm_tcgen05.cu": [("extern __shared__ uint8_t smem_raw[];", "uint8_t* smem_raw = g_dyn_smem;"),
                        ('asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");', "tma_store_wait_read0();")],
}


def build(force=False):
    bdir = os.path.dirname(OUT)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.join(HERE, f) for f in ("common.cuh", "mma.h", "cooperative_groups.h", "tensormap.cuh", "shim_runtime.cpp", "build.py")]
    deps.append(os.path.join(ROOT, "include", "chatts_b200.h"))
    deps.append(os.path.join(CSRC, "trace.cuh"))
    deps.append(os.path.join(CSRC, "ts_rows.cuh"))
    if not force and os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    os.makedirs(bdir, exist_ok=True)
    cpps = []
    for s in SOURCES:
        dst = os.path.join(bdir, s.replace(".cu", ".cpp"))
        text = open(os.path.join(CSRC, s)).read()
        for old, new in SUBSTITUTIONS.get(s, []):
            assert old in text, (s, old)
            text = text.replace(old, new)
        open(dst, "w").write(text)
        cpps.append(dst)
    for f in ("common.cuh", "mma.h", "cooperative_groups.h", "tensormap.cuh", "shim_runtime.cpp"):
        shutil.copyfile(os.path.join(HERE, f), os.path.join(bdir, f))
    shutil.copyfile(os.path.join(CSRC, "ts_rows.cuh"), os.path.join(bdir, "ts_rows.cuh"))
    shutil.copyfile(os.path.join(CSRC, "trace.cuh"), os.path.join(bdir, "trace.cuh"))      # the real header: its CTS_HOST_SHIM branch makes every mark a no-op
    flags = ["-std=c++17", "-O2", "-fno-strict-aliasing", "-g", "-fPIC", "-pthread", "-w", "-I", bdir, "-I", os.path.join(ROOT, "include")]
    units = [os.path.join(bdir, "shim_runtime.cpp")] + cpps

    def compile_one(src):
        obj = src[:-4] + ".o"
        r = subprocess.run(["g++"] + flags + ["-c", src, "-o", obj], capture_output=True, text=True)
        return obj, r

    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        results = list(ex.map(compile_one, units))
    for obj, r in results:
        if r.returncode != 0:
            raise RuntimeError("shim build failed:\n" + r.stderr[-6000:])
    tmp = OUT + f".{os.getpid()}.tmp"
    r = subprocess.run(["g++", "-shared", "-pthread", "-o", tmp] + [o for o, _ in results] + ["-lrt"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("shim link failed:\n" + r.stderr[-6000:])
    os.replace(tmp, OUT)                                      # atomic: a concurrent reader never sees a half-written library
    return OUT


if __name__ == "__main__":
    print(build(force=True))
