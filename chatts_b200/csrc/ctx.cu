// chatts_b200 -- context, error reporting, TMA descriptor encoding.
#include <stdarg.h>
#include <stdlib.h>

#include "common.cuh"
#include "tensormap.cuh"

int cts_set_error(cts_ctx* ctx, int code, const char* fmt, ...) {
  if (ctx) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
    va_end(ap);
  }
  return code;
}

extern "C" int cts_version(void) { return 100; }

extern "C" const char* cts_arch(void) {
#if defined(CTS_BUILD_ARCH)
  return CTS_BUILD_ARCH;
#else
  return "unknown";
#endif
}

extern "C" int cts_ctx_create(int device, cts_ctx** out) {
  if (!out) return CTS_ERR_BAD_ARG;
  *out = nullptr;
  cts_ctx* ctx = (cts_ctx*)calloc(1, sizeof(cts_ctx));
  if (!ctx) return CTS_ERR_CUDA;
  ctx->device = device;
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    fprintf(stderr, "chatts_b200: cudaSetDevice(%d) failed: %s\n", device, cudaGetErrorString(e));
    free(ctx);
    return CTS_ERR_CUDA;
  }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) {
    free(ctx);
    return CTS_ERR_CUDA;
  }
  if (prop.major != 9 || prop.minor != 0) {
    fprintf(stderr, "chatts_b200: device %d is sm_%d%d; this library contains sm_90a code only\n", device, prop.major,
            prop.minor);
    free(ctx);
    return CTS_ERR_UNSUPPORTED;
  }
  ctx->sm_count = prop.multiProcessorCount;
  ctx->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  // cuTensorMapEncodeTiled comes from the driver; resolve it at run time so the library does not link
  // libcuda (the build container has no driver).
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
    fprintf(stderr, "chatts_b200: cannot resolve cuTensorMapEncodeTiled\n");
    free(ctx);
    return CTS_ERR_CUDA;
  }
  ctx->encode_tiled = (PFN_cuTensorMapEncodeTiled_v12000)fn;
  const char* e1 = getenv("CTS_L2_PREFETCH_MB");
  ctx->l2_prefetch_mb = e1 ? atoi(e1) : 0;
  const char* e4 = getenv("CTS_NO_PERSISTENT_GEMM");
  ctx->no_persistent_gemm = e4 ? atoi(e4) : 0;
  const char* e5 = getenv("CTS_NORM_CLUSTER");
  ctx->norm_cluster = e5 ? atoi(e5) : 8;
  const char* e2 = getenv("CTS_DECODE_SMEM_KB");
  ctx->decode_stages = e2 ? atoi(e2) : 75;   // shared-memory ring of a decode GEMM CTA: 3 CTAs per SM of 3-4 stages each
  // a few zero-initialised device words for kernels that synchronise through global counters (the fused TS encoder's grid barrier);
  // allocated here so that nothing is allocated inside a CUDA-graph capture
  {
    int cur = 0;
    cudaGetDevice(&cur);
    cudaSetDevice(device);
    ctx->scratch = nullptr;
    ctx->scratch_bytes = 4096;
    if (cudaMalloc(&ctx->scratch, ctx->scratch_bytes) != cudaSuccess || cudaMemset(ctx->scratch, 0, ctx->scratch_bytes) != cudaSuccess) {
      fprintf(stderr, "chatts_b200: cannot allocate the context scratch\n");
      ctx->scratch = nullptr;
    }
    cudaSetDevice(cur);
  }
  const char* e8 = getenv("CTS_TS_FUSED");
  ctx->no_ts_fused = (e8 && atoi(e8) == 0) ? 1 : 0;
  const char* e6 = getenv("CTS_NEXT_PREFETCH");
  ctx->no_next_prefetch = (e6 && atoi(e6) == 0) ? 1 : 0;
  const char* e7 = getenv("CTS_NEXT_PREFETCH_MB");
  ctx->next_prefetch_mb = e7 ? atoi(e7) : 0;     // off by default: the prefetched bytes are read twice (once into L2, once by the GEMM)
  const char* e9 = getenv("CTS_NO_STREAM_GEMM");
  ctx->no_stream_gemm = e9 ? atoi(e9) : 0;
  const char* e10 = getenv("CTS_STREAM_CTAS");
  ctx->stream_ctas = e10 ? atoi(e10) : 2;
  const char* e11 = getenv("CTS_STREAM_ROWS");
  ctx->stream_rows = e11 ? atoi(e11) : 128;
  const char* e12 = getenv("CTS_STREAM_KBLOCKS");
  ctx->stream_kblocks = e12 ? atoi(e12) : 1;
  *out = ctx;
  return CTS_OK;
}

extern "C" void cts_ctx_destroy(cts_ctx* ctx) {
  if (!ctx) return;
  if (ctx->scratch) cudaFree(ctx->scratch);
  free(ctx);
}

extern "C" const char* cts_last_error(const cts_ctx* ctx) { return ctx ? ctx->err : "null ctx"; }

// 2-D row-major [rows, cols] tensor of 2-byte elements, box = [box_rows, 64 cols] (128 bytes), 128B swizzle.
int cts_make_tmap_2d(cts_ctx* ctx, CUtensorMap* tm, const void* base, long long rows, long long cols, long long ld_elems,
                     int box_rows, int is_bf16) {
  if (((uintptr_t)base & 15) != 0) return cts_set_error(ctx, CTS_ERR_BAD_ARG, "tensor map: base not 16-byte aligned");
  if ((ld_elems * 2) % 16 != 0) return cts_set_error(ctx, CTS_ERR_BAD_ARG, "tensor map: row pitch %lld B not a multiple of 16", ld_elems * 2);
  if (box_rows < 1 || box_rows > 256) return cts_set_error(ctx, CTS_ERR_BAD_ARG, "tensor map: box rows %d", box_rows);
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)(ld_elems * 2)};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = ctx->encode_tiled(tm, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                                 const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cts_set_error(ctx, CTS_ERR_CUDA, "cuTensorMapEncodeTiled failed: CUresult %d", (int)r);
  return CTS_OK;
}

int cts_make_tmap_2d_dense(cts_ctx* ctx, CUtensorMap* tm, const void* base, long long rows, long long cols, long long ld_elems,
                           int box_rows, int box_cols, int is_bf16) {
  if (((uintptr_t)base & 15) != 0) return cts_set_error(ctx, CTS_ERR_BAD_ARG, "tensor map: base not 16-byte aligned");
  if ((ld_elems * 2) % 16 != 0) return cts_set_error(ctx, CTS_ERR_BAD_ARG, "tensor map: row pitch %lld B not a multiple of 16", ld_elems * 2);
  if (box_rows < 1 || box_rows > 256 || box_cols < 8 || box_cols > 256 || (box_cols * 2) % 16 != 0)
    return cts_set_error(ctx, CTS_ERR_BAD_ARG, "tensor map: box %d x %d", box_rows, box_cols);
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)(ld_elems * 2)};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = ctx->encode_tiled(tm, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                                 const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                 CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cts_set_error(ctx, CTS_ERR_CUDA, "cuTensorMapEncodeTiled (dense) failed: CUresult %d", (int)r);
  return CTS_OK;
}

// Optional device-side timeline (csrc/trace.cuh): installs `buf` ([0] cursor = 0, [1] capacity in records, then {tag, time} pairs;
// NULL switches tracing off) in every instrumented translation unit.  A debugging / profiling aid; never on in a measurement.
extern "C" int cts_trace_set_gemm(unsigned long long* buf);
extern "C" int cts_trace_set_elementwise(unsigned long long* buf);
extern "C" int cts_trace_set_attention(unsigned long long* buf);
extern "C" int cts_trace_set_allreduce_ll(unsigned long long* buf);
extern "C" int cts_trace_set_fused(unsigned long long* buf);
extern "C" int cts_trace_set_ts_fused(unsigned long long* buf);
extern "C" int cts_trace_set_w4(unsigned long long* buf);
extern "C" int cts_trace_enable(cts_ctx* ctx, unsigned long long* buf) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  if (cts_trace_set_gemm(buf) || cts_trace_set_elementwise(buf) || cts_trace_set_attention(buf) || cts_trace_set_allreduce_ll(buf) || cts_trace_set_fused(buf) || cts_trace_set_ts_fused(buf) || cts_trace_set_w4(buf))
    return cts_set_error(ctx, CTS_ERR_CUDA, "cts_trace_enable: cudaMemcpyToSymbol failed");
  return CTS_OK;
}
