// chatts_b200 -- shared device/host helpers (sm_90a only).
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/chatts_b200.h"

struct cts_ctx {
  int device;
  int sm_count;
  int max_smem_optin;
  char err[512];
  // lazily created scratch for kernels that need a few flags / counters
  void* scratch;
  size_t scratch_bytes;
  PFN_cuTensorMapEncodeTiled_v12000 encode_tiled;
  int l2_prefetch_mb;   // tuning knob (CTS_L2_PREFETCH_MB): weight bytes a decode GEMM prefetches into L2 while it waits
  int no_persistent_gemm;     // CTS_NO_PERSISTENT_GEMM=1: A/B switch back to the one-tile-per-CTA kernel for big T
  int norm_cluster;           // CTS_NORM_CLUSTER: max thread-block-cluster size of the decode RMSNorm kernel (default 8)
  int decode_stages;    // tuning knob (CTS_DECODE_SMEM_KB): shared-memory budget per CTA of the decode GEMM
  int no_ts_fused;      // CTS_TS_FUSED=0: the TS encoder always takes the multi-launch path (A/B testing)
  int no_next_prefetch; // CTS_NEXT_PREFETCH=0: ignore the next-GEMM weight prefetch hints (A/B testing)
  int next_prefetch_mb; // CTS_NEXT_PREFETCH_MB (default 0 = off): budget of the hint the C++ step executor passes (model.py passes its own)
};

int cts_set_error(cts_ctx* ctx, int code, const char* fmt, ...);

#define CTS_CHECK_ARG(ctx, cond, msg)                                         \
  do {                                                                        \
    if (!(cond)) return cts_set_error((ctx), CTS_ERR_BAD_ARG, "%s: %s", __func__, (msg)); \
  } while (0)

#define CTS_CUDA(ctx, expr)                                                   \
  do {                                                                        \
    cudaError_t _e = (expr);                                                  \
    if (_e != cudaSuccess)                                                    \
      return cts_set_error((ctx), CTS_ERR_CUDA, "%s: %s -> %s", __func__, #expr, cudaGetErrorString(_e)); \
  } while (0)

#define CTS_LAUNCH_CHECK(ctx)                                                 \
  do {                                                                        \
    cudaError_t _e = cudaGetLastError();                                      \
    if (_e != cudaSuccess)                                                    \
      return cts_set_error((ctx), CTS_ERR_CUDA, "%s: launch -> %s", __func__, cudaGetErrorString(_e)); \
  } while (0)

static inline long long cdiv_ll(long long a, long long b) { return (a + b - 1) / b; }

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  Every kernel of the library is launched with the
// programmatic-stream-serialization attribute, calls pdl_trigger() first thing (so its successor may be
// scheduled as soon as all of this grid's CTAs are resident) and pdl_wait() before it touches anything a
// predecessor produced.  Prologues (barrier init, tensor-map prefetch and -- in the GEMM -- the
// TMA prefetch of the WEIGHT tiles, which no kernel ever writes) thereby overlap the predecessor's tail:
// the decode step is ~480 short kernels, and this removes the launch/ramp bubble between them.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     unsigned cluster_x, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[n].val.programmaticStreamSerializationAllowed = 1;
  ++n;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ----------------------------------------------------------------------------------------------
// dtype helpers: the model dtype is bf16 or fp16 (F5 in SURVEY.md: the reference runs fp16, the
// baseline configs say bf16).  Every elementwise result is rounded to the model dtype exactly where
// the HF/torch reference rounds it.
// ----------------------------------------------------------------------------------------------
template <typename T> struct DT;
template <> struct DT<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <> struct DT<__half> {
  static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
// round-trip through the model dtype (the "nn.Linear output is bf16" rounding points)
template <typename T> __device__ __forceinline__ float rnd(float v) { return DT<T>::to_f(DT<T>::from_f(v)); }

template <typename T> __device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const T* p = reinterpret_cast<const T*>(&u);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = DT<T>::to_f(p[i]);
}
template <typename T> __device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  T* p = reinterpret_cast<T*>(&u);
#pragma unroll
  for (int i = 0; i < 8; ++i) p[i] = DT<T>::from_f(f[i]);
  return u;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// exact-erf GELU (nn.GELU() default, chatts_vllm.py:87)
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }

// ----------------------------------------------------------------------------------------------
// PTX: mbarrier, TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (CUDA error surfaced through the C-ABI) instead of a
// hung GPU box.  ~2^26 polls of a HW-sleeping try_wait is seconds, far beyond any legitimate wait.
#ifndef CTS_WAIT_LIMIT
#define CTS_WAIT_LIMIT (1u << 26)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t n = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++n > CTS_WAIT_LIMIT) {
      printf("chatts_b200: mbarrier wait timed out (block %d,%d,%d thread %d)\n", blockIdx.x, blockIdx.y, blockIdx.z,
             threadIdx.x);
      __trap();
    }
  }
}

// L2 cache-hint policies (createpolicy encodings used by CUTLASS' TMA::CacheHintSm90)
#define CTS_L2_EVICT_NORMAL 0x1000000000000000ull
#define CTS_L2_EVICT_FIRST 0x12F0000000000000ull
#define CTS_L2_EVICT_LAST 0x14F0000000000000ull

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1,
                                            uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
// TMA prefetch of a tile into L2 only (no shared-memory destination, no barrier)
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* tm, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tm), "r"(c0), "r"(c1) : "memory");
}
// TMA store shared -> global (bulk async-group completion)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(tm), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }   // full completion (writes performed), not just the smem reads
__device__ __forceinline__ void tma_load_2d_nohint(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}
// plain bulk copy global -> shared (1-D, size multiple of 16 B, 16 B aligned both sides)
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// wgmma (sm_90a): one warpgroup (four consecutive warps, the first one a multiple of 4) computes
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T with A and B K-major in 128B-swizzled shared memory and D in
// registers.  The swap-AB GEMMs keep a 128-row weight tile as two such 64-row halves (Acc128 below).
// ----------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major, 128-byte swizzle, rows of exactly 128 bytes
// (start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout [62,64) with SWIZZLE_128B = 1).  SBO = 8 rows * 128 B.
// Advancing 16 elements (32 bytes) along K inside the swizzle atom is +2 on the descriptor.
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMA
__device__ __forceinline__ void wgmma_fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

template <int N, bool BF16> __device__ __forceinline__ void wgmma_m64k16(float* d, uint64_t a, uint64_t b, int scale_d);
template <> __device__ __forceinline__ void wgmma_m64k16<16, true>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_m64k16<16, false>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_m64k16<32, true>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_m64k16<32, false>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_m64k16<64, true>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_m64k16<64, false>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_m64k16<128, true>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_m64k16<128, false>(float* d, uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d));
}

// The same descriptor with explicit strides, for MN-major operands (the N index contiguous in 128-byte rows): LBO = bytes
// between consecutive 64-element blocks along N, SBO = bytes between consecutive 8-row groups along K.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// D[64 x 128] += A[64 x 16] * B[16 x 128] with A in registers (the m64k16 fragment: a0 = (row r, k 2t..2t+1), a1 = (r + 8, 2t..),
// a2 = (r, 2t + 8..), a3 = (r + 8, 2t + 8..)) and B MN-major in shared memory (transposed operand); always accumulates.
template <bool BF16> __device__ __forceinline__ void wgmma_m64n128k16_rs_tb(float* d, const uint32_t* a, uint64_t b);
template <> __device__ __forceinline__ void wgmma_m64n128k16_rs_tb<true>(float* d, const uint32_t* a, uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, 1, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_m64n128k16_rs_tb<false>(float* d, const uint32_t* a, uint64_t b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, 1, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}

// Fragment layout of an m64nN fp32 accumulator: register i of thread (warp w, lane l) of the warpgroup holds
// row 16 w + l / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l & 3) + (i & 1).
__device__ __forceinline__ int acc_row(int i) { return ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2) + ((i >> 1) & 1) * 8; }
__device__ __forceinline__ int acc_col(int i) { return (i >> 2) * 8 + (threadIdx.x & 3) * 2 + (i & 1); }

// The 128 x BN fp32 accumulator of a swap-AB tile (rows = weight rows, columns = tokens), held by one warpgroup:
// d[h] is the m64 half with rows 64 h .. 64 h + 63.
template <int BN> struct Acc128 {
  float d[2][BN / 2];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[h][i] = 0.f;
  }
  __device__ __forceinline__ void fence_operands() {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) wgmma_fence_operand(d[h][i]);
  }
  // one 64-wide K block: A = [128 rows x 128 B] at a_addr, B = [BN rows x 128 B] at b_addr, both 128B-swizzled.
  // Issues the MMAs and commits them as one group; the caller waits (wgmma_wait) before it reuses the operands.
  template <bool BF16> __device__ __forceinline__ void mma_kblock(uint32_t a_addr, uint32_t b_addr, bool first) {
    fence_operands();
    wgmma_fence();
    const uint64_t a0 = gmma_desc_k_sw128(a_addr), a1 = gmma_desc_k_sw128(a_addr + 64 * 128), b = gmma_desc_k_sw128(b_addr);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const int sc = (first && kk == 0) ? 0 : 1;
      wgmma_m64k16<BN, BF16>(d[0], a0 + 2 * kk, b + 2 * kk, sc);
      wgmma_m64k16<BN, BF16>(d[1], a1 + 2 * kk, b + 2 * kk, sc);
    }
    wgmma_commit();
    fence_operands();
  }
  // park the accumulator in shared memory as fp32 [128 rows][ld] (ld % 32 == 8 or 24 keeps the float2 stores conflict-free)
  __device__ __forceinline__ void store(float* s, int ld) const {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2)
        *reinterpret_cast<float2*>(s + (64 * h + acc_row(i)) * ld + acc_col(i)) = make_float2(d[h][i], d[h][i + 1]);
  }
};
template <int BN> __host__ __device__ constexpr int acc_ld() { return BN + 8; }
template <int BN> __host__ __device__ constexpr int acc_smem_bytes() { return 128 * acc_ld<BN>() * 4; }
// 16 consecutive columns of one accumulator row, read back from the parked tile (thread-per-row epilogues)
__device__ __forceinline__ void acc_ld16(const float* s, int ld, int row, int col, uint32_t* v) {
  const float4* p = reinterpret_cast<const float4*>(s + row * ld + col);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 f = p[j];
    v[4 * j] = __float_as_uint(f.x); v[4 * j + 1] = __float_as_uint(f.y); v[4 * j + 2] = __float_as_uint(f.z); v[4 * j + 3] = __float_as_uint(f.w);
  }
}
