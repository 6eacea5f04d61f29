// TEST INFRASTRUCTURE ONLY -- "CUDA on CPU": stands in for chatts_b200/csrc/common.cuh when a kernel source file is compiled with g++
// (tests/cuda_on_cpu/build.py copies the .cu next to this header, so its `#include "common.cuh"` lands here).  It provides the CUDA
// vocabulary those files use -- thread / block indices, __shared__, __syncthreads, warp shuffles, atomics, bf16 / fp16 storage types,
// vector types, launch_pdl -- with the execution model
//     one OS thread per CUDA thread, the threads of ONE block at a time, blocks of a grid one after the other,
// and the library's own host helpers (cts_ctx, error macros, DT<>, rnd, pack8, warp_sum ...) restated for the host.  The KERNEL
// BODIES and the C-ABI entry points are the product's, untouched: what runs here is the same source nvcc compiles for sm_90a,
// which turns "this kernel has never executed" into "its source executes and passes its GPU test on CPU" for the kernels that need
// no tensor core, TMA or cluster (sampling, AdamW / clip / adapter packing, the elementwise backward kernels, the LL all-reduce).
// Not a performance model, not a memory-model checker (x86 is stronger than PTX), never part of the product.
#pragma once
#include <math.h>
#include <pthread.h>
#include <sched.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <functional>
#include <thread>
#include <tuple>
#include <type_traits>
#include <vector>

#include "chatts_b200.h"

#define CTS_HOST_SHIM 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __cvta_generic_to_shared(p) ((uintptr_t)(p))
#define __shared__ static thread_local          // one OS thread per CTA (its CUDA threads are fibers of that thread)
#define __grid_constant__

// ---------------------------------------------------------------------------------------------- vector types
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
struct int2 { int x, y; };
struct int4 { int x, y, z, w; };
struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
static inline uint2 make_uint2(uint32_t a, uint32_t b) { return {a, b}; }
static inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return {a, b, c, d}; }
static inline float2 make_float2(float a, float b) { return {a, b}; }
static inline float4 make_float4(float a, float b, float c, float d) { return {a, b, c, d}; }

// ---------------------------------------------------------------------------------------------- bf16 / fp16 storage types
struct __nv_bfloat16 { uint16_t bits; };
struct __half { uint16_t bits; };
struct __nv_bfloat162 { __nv_bfloat16 x, y; };
static inline float shim_u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t shim_f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float __bfloat162float(__nv_bfloat16 v) { return shim_u2f((uint32_t)v.bits << 16); }
static inline __nv_bfloat16 __float2bfloat16_rn(float f) {
  uint32_t u = shim_f2u(f);
  if ((u & 0x7FFFFFFFu) > 0x7F800000u) return {(uint16_t)0x7FFF};                     // NaN
  u += 0x7FFFu + ((u >> 16) & 1u);                                                    // round to nearest even
  return {(uint16_t)(u >> 16)};
}
static inline __nv_bfloat162 __hsub2(__nv_bfloat162 a, __nv_bfloat162 b);
static inline __nv_bfloat162 __hmul2(__nv_bfloat162 a, __nv_bfloat162 b);
static inline float __half2float(__half v) { _Float16 h; memcpy(&h, &v.bits, 2); return (float)h; }
static inline __half __float2half_rn(float f) { _Float16 h = (_Float16)f; __half r; memcpy(&r.bits, &h, 2); return r; }
// packed pairs (csrc/gemm_w4.cu): element-wise, the exact result rounded ONCE to the 16-bit type, like the hardware instructions
struct __half2 { __half x, y; };
static inline __half2 __hsub2(__half2 a, __half2 b) { return {__float2half_rn(__half2float(a.x) - __half2float(b.x)), __float2half_rn(__half2float(a.y) - __half2float(b.y))}; }
static inline __half2 __hmul2(__half2 a, __half2 b) { return {__float2half_rn(__half2float(a.x) * __half2float(b.x)), __float2half_rn(__half2float(a.y) * __half2float(b.y))}; }

// ---------------------------------------------------------------------------------------------- execution model
// The CUDA threads of a block are FIBERS of one OS thread (hand-rolled x86-64 context switch, shim_runtime.cpp), scheduled round
// robin; a fiber leaves the CPU only at a barrier, a shuffle or an explicit shim_yield().  No locks anywhere: the block state below is
// only ever touched by the fiber that is running.  Blocks of a grid run one after the other.
struct ShimBlock {
  int alive = 0, arrived = 0;
  unsigned long gen = 0;
  int named_arrived[16] = {0};                             // named barriers (bar.sync id, n)
  unsigned long named_gen[16] = {0};
  struct Warp { int alive = 0, arrived = 0; unsigned long gen = 0; uint64_t slot[32]; } warp[64];   // shuffles / __syncwarp
};
extern thread_local ShimBlock g_blk;
struct ShimIdx { unsigned x, y, z; };
extern thread_local ShimIdx g_tid, g_bid;                  // g_tid is swapped by the scheduler with every fiber switch
extern ShimIdx g_bdim, g_gdim;
#define threadIdx g_tid
#define blockIdx g_bid
#define blockDim g_bdim
#define gridDim g_gdim
void shim_yield();                                         // give the other fibers of the block a turn

static inline int shim_linear_tid() { return (int)(g_tid.x + g_bdim.x * (g_tid.y + g_bdim.y * g_tid.z)); }

static inline void __syncthreads() {
  const unsigned long my = g_blk.gen;
  if (++g_blk.arrived >= g_blk.alive) { g_blk.arrived = 0; ++g_blk.gen; return; }
  while (g_blk.gen == my) shim_yield();
}
static inline void named_bar_sync(int id, int n) {        // bar.sync id, n : the first n arrivals of a generation release each other
  const unsigned long my = g_blk.named_gen[id];
  if (++g_blk.named_arrived[id] >= n) { g_blk.named_arrived[id] = 0; ++g_blk.named_gen[id]; return; }
  while (g_blk.named_gen[id] == my) shim_yield();
}
static inline void shim_warp_rendezvous() {
  ShimBlock::Warp& w = g_blk.warp[shim_linear_tid() >> 5];
  const unsigned long my = w.gen;
  if (++w.arrived >= w.alive) { w.arrived = 0; ++w.gen; return; }
  while (w.gen == my) shim_yield();
}
static inline void __syncwarp(unsigned = 0xffffffffu) { shim_warp_rendezvous(); }
template <typename V> static inline V shim_shfl(V v, int src_lane) {
  static_assert(sizeof(V) <= 8, "shuffle of at most 64 bits");
  ShimBlock::Warp& w = g_blk.warp[shim_linear_tid() >> 5];
  const int lane = shim_linear_tid() & 31;
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(V));
  w.slot[lane] = bits;
  shim_warp_rendezvous();                                  // everybody has written
  V out = v;
  if (src_lane >= 0 && src_lane < 32) { const uint64_t b = w.slot[src_lane]; memcpy(&out, &b, sizeof(V)); }
  shim_warp_rendezvous();                                  // everybody has read: the slots may be rewritten
  return out;
}
template <typename V> static inline V __shfl_xor_sync(unsigned, V v, int m) { return shim_shfl(v, (shim_linear_tid() & 31) ^ m); }
template <typename V> static inline V __shfl_down_sync(unsigned, V v, int d) { const int l = shim_linear_tid() & 31; return shim_shfl(v, l + d < 32 ? l + d : l); }
template <typename V> static inline V __shfl_up_sync(unsigned, V v, int d) { const int l = shim_linear_tid() & 31; return shim_shfl(v, l - d >= 0 ? l - d : l); }
template <typename V> static inline V __shfl_sync(unsigned, V v, int src) { return shim_shfl(v, src & 31); }

void shim_run_block(const std::function<void()>& body, dim3 block);
extern thread_local uint8_t* g_dyn_smem;                   // dynamic shared memory of the running CTA
extern thread_local size_t g_dyn_bytes;
void shim_set_dyn_smem(size_t bytes);
#define CTS_DYN_SMEM(name) uint8_t* name = g_dyn_smem
#define __align__(x)
#define cudaFuncAttributeMaxDynamicSharedMemorySize 8
template <typename F> static inline int cudaFuncSetAttribute(F, int, int) { return 0; }

// ---- thread-block clusters: the CTAs of one cluster run concurrently (one OS thread each); distributed shared memory is the
// other CTAs' DYNAMIC shared memory (static __shared__ variables are not mappable here -- none of the shimmed kernels needs that)
struct ShimCluster {
  int size = 1;
  uint8_t* dyn_base[1024] = {nullptr};                     // 1024: a cooperative launch runs its WHOLE grid as one "cluster" (grid barriers need every CTA live)
  void* static_ptr[1024] = {nullptr};                        // a STATIC shared variable published for the peers (shim_publish_static)
  pthread_barrier_t bar;
};
extern thread_local ShimCluster* g_cluster;
extern thread_local int g_cluster_rank;
namespace cooperative_groups {
struct cluster_group {
  void sync() const {                                      // every thread of every CTA: the CTA's fibers meet first, then the CTAs
    __syncthreads();
    if (g_cluster && g_cluster->size > 1 && shim_linear_tid() == 0) pthread_barrier_wait(&g_cluster->bar);
    __syncthreads();
  }
  unsigned num_blocks() const { return g_cluster ? (unsigned)g_cluster->size : 1u; }
  unsigned block_rank() const { return (unsigned)g_cluster_rank; }
  template <typename V> V* map_shared_rank(V* p, unsigned r) const {
    if (g_cluster == nullptr || g_cluster->size == 1) return p;           // a cluster of one: rank 0 is this CTA
    uint8_t* q = (uint8_t*)p;
    if (q < g_dyn_smem || q >= g_dyn_smem + g_dyn_bytes + 1024) { fprintf(stderr, "shim: map_shared_rank of a non-dynamic shared address\n"); abort(); }
    return (V*)(g_cluster->dyn_base[r] + (q - g_dyn_smem));
  }
};
static inline cluster_group this_cluster() { return cluster_group(); }
}  // namespace cooperative_groups

// distributed shared memory on a static __shared__ variable (one per kernel is enough for the library): the owner publishes its
// address before the cluster barrier, the peers look it up after it
extern thread_local void* g_static_self;
static inline void shim_publish_static(void* p) { if (g_cluster) g_cluster->static_ptr[g_cluster_rank] = p; g_static_self = p; }
static inline void* shim_static_peer(unsigned r) { return g_cluster ? g_cluster->static_ptr[r] : g_static_self; }

void shim_launch(const std::function<void()>& body, dim3 grid, dim3 block, size_t smem, dim3 cluster);

// cudaLaunchKernelEx with the two attributes the library uses
enum { cudaLaunchAttributeProgrammaticStreamSerialization = 1, cudaLaunchAttributeClusterDimension = 2, cudaLaunchAttributeCooperative = 3 };
struct cudaLaunchAttribute {
  int id;
  union { int programmaticStreamSerializationAllowed; int cooperative; struct { unsigned x, y, z; } clusterDim; } val;
};
// a kernel that synchronises its whole grid (grid barriers through a global counter) asks for it with this flag on the host shim:
// every CTA of the grid then runs concurrently (one OS thread each), i.e. the grid is scheduled as ONE cluster whose ranks are the
// linear CTA indices -- the kernel maps its real cluster ranks to those under CTS_HOST_SHIM
extern thread_local bool g_whole_grid_next;
static inline void shim_next_launch_whole_grid() { g_whole_grid_next = true; }
struct cudaLaunchConfig_t { dim3 gridDim, blockDim; size_t dynamicSmemBytes = 0; void* stream = nullptr; cudaLaunchAttribute* attrs = nullptr; unsigned numAttrs = 0; };
template <typename... KArgs, typename... Args>
static inline int cudaLaunchKernelEx(const cudaLaunchConfig_t* cfg, void (*kern)(KArgs...), Args... args) {
  auto tup = std::make_tuple(static_cast<KArgs>(args)...);
  dim3 cl(1, 1, 1);
  for (unsigned i = 0; i < cfg->numAttrs; ++i)
    if (cfg->attrs[i].id == cudaLaunchAttributeClusterDimension) cl = dim3(cfg->attrs[i].val.clusterDim.x, cfg->attrs[i].val.clusterDim.y, cfg->attrs[i].val.clusterDim.z);
  for (unsigned i = 0; i < cfg->numAttrs; ++i)
    if (cfg->attrs[i].id == cudaLaunchAttributeCooperative && cfg->attrs[i].val.cooperative) g_whole_grid_next = true;
  if (g_whole_grid_next) { cl = cfg->gridDim; g_whole_grid_next = false; }
  shim_launch([&] { std::apply(kern, tup); }, cfg->gridDim, cfg->blockDim, cfg->dynamicSmemBytes, cl);
  return 0;
}

template <typename... KArgs, typename... Args>
static inline int launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, void*, unsigned cluster_x, Args... args) {
  auto tup = std::make_tuple(static_cast<KArgs>(args)...);
  shim_launch([&] { std::apply(kern, tup); }, grid, block, smem, dim3(cluster_x ? cluster_x : 1, 1, 1));
  return 0;
}

// ---------------------------------------------------------------------------------------------- intrinsics
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline unsigned atomicOr(unsigned* p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline float atomicAdd(float* p, float v) {
  uint32_t* u = reinterpret_cast<uint32_t*>(p);
  uint32_t old = __atomic_load_n(u, __ATOMIC_SEQ_CST);
  for (;;) {
    const uint32_t want = shim_f2u(shim_u2f(old) + v);
    if (__atomic_compare_exchange_n(u, &old, want, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) return shim_u2f(old);
  }
}
static inline int atomicMax(int* p, int v) {
  int old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}
static inline int atomicMin(int* p, int v) {
  int old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (old > v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}
static inline int atomicExch(int* p, int v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
static inline int atomicCAS(int* p, int cmp, int v) { __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST); return cmp; }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __threadfence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __trap() { fflush(stdout); abort(); }
#define __expf(x) expf(x)        // glibc declares a __expf of its own
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline float __fdividef(float a, float b) { return a / b; }
static inline float __uint_as_float(uint32_t u) { return shim_u2f(u); }
static inline uint32_t __float_as_uint(float f) { return shim_f2u(f); }
static inline float __int_as_float(int i) { return shim_u2f((uint32_t)i); }
static inline int __float_as_int(float f) { return (int)shim_f2u(f); }
template <typename V> static inline V __ldg(const V* p) { return *p; }
template <typename V> static inline V __ldcv(const V* p) { return *p; }
template <typename V> static inline V __ldcs(const V* p) { return *p; }
template <typename V> static inline V __ldcg(const V* p) { return *p; }
template <typename V> static inline void __stcg(V* p, V v) { *p = v; }
template <typename V> static inline void __stcs(V* p, V v) { *p = v; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }

// ---------------------------------------------------------------------------------------------- the library's host helpers
typedef void* cudaStream_t;
typedef int cudaError_t;
#define cudaSuccess 0
#define cudaErrorInvalidValue 1
static inline const char* cudaGetErrorString(int) { return "shim"; }

struct cts_ctx {
  int device;
  int sm_count;
  int decode_stages, l2_prefetch_mb, no_persistent_gemm, norm_cluster, max_smem_optin;
  int no_next_prefetch, next_prefetch_mb, no_ts_fused;
  void* scratch;                                           // zero-initialised counters (grid barrier of the fused TS encoder)          // next-GEMM L2 prefetch hint (a no-op on the host: tma_prefetch_l2_2d does nothing)
  char err[512];
};
int cts_set_error(cts_ctx* ctx, int code, const char* fmt, ...);

#define CTS_CHECK_ARG(ctx, cond, msg)                                         \
  do {                                                                        \
    if (!(cond)) return cts_set_error((ctx), CTS_ERR_BAD_ARG, "%s: %s", __func__, (msg)); \
  } while (0)
#define CTS_CUDA(ctx, expr)                                                   \
  do {                                                                        \
    cudaError_t _e = (expr);                                                  \
    if (_e != cudaSuccess) return cts_set_error((ctx), CTS_ERR_CUDA, "%s: %s", __func__, #expr); \
  } while (0)
#define CTS_LAUNCH_CHECK(ctx) do { } while (0)

static inline long long cdiv_ll(long long a, long long b) { return (a + b - 1) / b; }
static inline void pdl_wait() {}
static inline void pdl_trigger() {}

template <typename T> struct DT;
template <> struct DT<__nv_bfloat16> {
  static inline float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  static inline __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <> struct DT<__half> {
  static inline float to_f(__half v) { return __half2float(v); }
  static inline __half from_f(float v) { return __float2half_rn(v); }
};
template <typename T> static inline float rnd(float v) { return DT<T>::to_f(DT<T>::from_f(v)); }
template <typename T> static inline void unpack8(const uint4& u, float* f) {
  const T* p = reinterpret_cast<const T*>(&u);
  for (int i = 0; i < 8; ++i) f[i] = DT<T>::to_f(p[i]);
}
template <typename T> static inline uint4 pack8(const float* f) {
  uint4 u;
  T* p = reinterpret_cast<T*>(&u);
  for (int i = 0; i < 8; ++i) p[i] = DT<T>::from_f(f[i]);
  return u;
}
static inline float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
static inline float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
static inline float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
static inline float silu_f(float x) { return x / (1.0f + expf(-x)); }

// ================================================================================================================================
// Functional emulation of the Hopper pieces the tensor-core kernels use: mbarrier (arrive / expect_tx / complete_tx / parity wait),
// TMA tile loads and stores (128-byte swizzle or dense boxes, zero fill / clipping at the tensor edge) and the warpgroup MMA of the
// swap-AB GEMMs (Acc128: shared-memory matrix descriptors decoded, 128-byte swizzle applied on the ADDRESS bits as the hardware does,
// every thread computing its own registers of the documented m64nNk16 accumulator fragment).  The MMA completes synchronously at
// issue (CTS_SHIM_ASYNC delays TMA loads / stores only), so this checks what the kernels COMPUTE and that their barrier protocols
// are live, not MMA-completion hazards.
// ================================================================================================================================
#include <unordered_map>
// 32-bit shared-window addresses: the low half of the host pointer; the high half is remembered per CTA (all shared objects a kernel
// takes the address of this way -- its dynamic shared memory or its static arrays -- live in one region)
extern thread_local uint64_t g_smem_hi;
static inline uint32_t smem_u32(const void* p) { g_smem_hi = (uint64_t)(uintptr_t)p >> 32; return (uint32_t)(uintptr_t)p; }
static inline uint8_t* shim_smem_from_u32(uint32_t a) { return (uint8_t*)(uintptr_t)((g_smem_hi << 32) | a); }
struct CUtensorMap { const void* base; long long rows, cols, ld; int box_rows, box_cols, swizzled, is_bf16; };

// CTS_SHIM_ASYNC=1 -- adversarially LATE completion of the TMA loads and stores: they are queued at issue and performed (in issue order)
// only when some thread of the CTA is blocked in an mbarrier wait or in one of the explicit completion waits, and at the latest when the
// CTA ends.  A consumer that reads shared or global memory without having waited for the producing copy, or a producer that refills a
// slot before its consumers released it, then sees stale or clobbered data and its test fails.  The warpgroup MMAs complete at issue.
// (Off: everything completes at issue.)
#include <deque>
extern thread_local std::deque<std::function<void()>> g_async;
extern int g_async_mode;
static inline void shim_async(std::function<void()> fn) { if (g_async_mode) g_async.push_back(std::move(fn)); else fn(); }
static inline bool shim_async_one() { if (g_async.empty()) return false; auto fn = std::move(g_async.front()); g_async.pop_front(); fn(); return true; }
static inline void shim_async_all() { while (shim_async_one()) {} }

struct ShimMbar { int count = 0, pending = 0; long long tx = 0; unsigned long phases = 0; };
extern thread_local std::unordered_map<const void*, ShimMbar> g_mbar;
static inline void shim_mbar_check(ShimMbar& b) { if (b.pending == 0 && b.tx == 0) { ++b.phases; b.pending = b.count; } }
static inline void mbar_init(uint64_t* bar, uint32_t count) { ShimMbar& b = g_mbar[bar]; b = ShimMbar(); b.count = b.pending = (int)count; }
static inline void fence_mbar_init() {}
static inline void fence_proxy_async_smem() {}
static inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { ShimMbar& b = g_mbar[bar]; b.tx += bytes; --b.pending; shim_mbar_check(b); }
static inline void mbar_arrive(uint64_t* bar) { ShimMbar& b = g_mbar[bar]; --b.pending; shim_mbar_check(b); }
static inline void shim_mbar_complete_tx(uint64_t* bar, long long bytes) { ShimMbar& b = g_mbar[bar]; b.tx -= bytes; shim_mbar_check(b); }
static inline bool mbar_try_wait(uint64_t* bar, uint32_t parity) { return (g_mbar[bar].phases & 1u) != parity; }
#define CTS_WAIT_LIMIT (1u << 22)
static inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t n = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++n > CTS_WAIT_LIMIT) { printf("shim: mbarrier wait timed out (block %u,%u,%u thread %u)\n", blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x); __trap(); }
    if (!shim_async_one()) shim_yield();                   // somebody is waiting: the oldest outstanding asynchronous operation completes now
  }
}
#define CTS_L2_EVICT_NORMAL 0x1000000000000000ull
#define CTS_L2_EVICT_FIRST 0x12F0000000000000ull
#define CTS_L2_EVICT_LAST 0x14F0000000000000ull

static inline uint8_t* shim_swz128(uint8_t* p) { return (uint8_t*)((uintptr_t)p ^ ((((uintptr_t)p >> 7) & 7) << 4)); }
static inline void shim_tma_copy(uint8_t* smem, const CUtensorMap* tm, int c0, int c1, bool to_smem) {
  for (int r = 0; r < tm->box_rows; ++r)
    for (int c = 0; c < tm->box_cols; ++c) {
      const long long row = (long long)c1 + r, col = (long long)c0 + c;
      const bool in = row >= 0 && row < tm->rows && col >= 0 && col < tm->cols;
      uint8_t* sp = tm->swizzled ? shim_swz128(smem + (size_t)r * 128 + (size_t)c * 2) : smem + ((size_t)r * tm->box_cols + c) * 2;
      uint16_t* gp = (uint16_t*)tm->base + row * tm->ld + col;
      if (to_smem) *(uint16_t*)sp = in ? *gp : (uint16_t)0;
      else if (in) *gp = *(uint16_t*)sp;
    }
}
static inline void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1, uint64_t) {
  const CUtensorMap t = *tm;
  shim_async([=] { shim_tma_copy((uint8_t*)smem_dst, &t, c0, c1, true); shim_mbar_complete_tx(bar, (long long)t.box_rows * t.box_cols * 2); });
}
static inline void tma_load_2d_nohint(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) { tma_load_2d(smem_dst, tm, bar, c0, c1, 0); }
static inline void tma_prefetch_l2_2d(const CUtensorMap*, int, int) {}
static inline void tma_prefetch_desc(const CUtensorMap*) {}
static inline void tma_store_2d(const CUtensorMap* tm, const void* smem_src, int c0, int c1) {
  const CUtensorMap t = *tm;
  shim_async([=] { shim_tma_copy((uint8_t*)smem_src, &t, c0, c1, false); });
}
static inline void tma_store_commit() {}
static inline void tma_store_wait_read0() { shim_async_all(); }
static inline void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  shim_async([=] { memcpy(smem_dst, gsrc, bytes); shim_mbar_complete_tx(bar, bytes); });
}
static inline bool elect_one() { return (shim_linear_tid() & 31) == 0; }
static inline uint8_t* shim_smem_ptr(uint32_t addr18) {                           // 18-bit shared-window address -> this CTA's dynamic shared memory
  return g_dyn_smem + ((addr18 - ((uint32_t)(uintptr_t)g_dyn_smem & 0x3FFFFu)) & 0x3FFFFu);
}
static inline float shim_ld_elem(const uint8_t* p, bool bf16) {
  uint16_t v = *(const uint16_t*)shim_swz128((uint8_t*)p);
  if (bf16) return shim_u2f((uint32_t)v << 16);
  __half h; h.bits = v; return __half2float(h);
}
// operand element (r, k): r = row of A (M) or of B (N); major 0 = K-major (rows of 128 B), 1 = MN-major (the r index is contiguous)
static inline float shim_operand(uint64_t desc, int major, int r, int k, bool bf16) {
  const uint32_t start = (uint32_t)(desc & 0x3FFF) << 4, lbo = (uint32_t)((desc >> 16) & 0x3FFF) << 4, sbo = (uint32_t)((desc >> 32) & 0x3FFF) << 4;
  if (((desc >> 62) & 3) != 1) { printf("shim: only SWIZZLE_128B shared-memory descriptors are emulated\n"); __trap(); }
  const uint8_t* base = shim_smem_ptr(start);
  const size_t off = major == 0 ? (size_t)(r / 8) * sbo + (size_t)(r % 8) * 128 + (size_t)k * 2
                                : (size_t)(r / 64) * lbo + (size_t)(k / 8) * sbo + (size_t)(k % 8) * 128 + (size_t)(r % 64) * 2;
  return shim_ld_elem(base + off, bf16);
}
static inline uint64_t gmma_desc_k_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
static inline void wgmma_fence() {}
static inline void wgmma_commit() {}
template <int N> static inline void wgmma_wait() {}
static inline int acc_row(int i) { return ((shim_linear_tid() >> 5) & 3) * 16 + ((shim_linear_tid() & 31) >> 2) + ((i >> 1) & 1) * 8; }
static inline int acc_col(int i) { return (i >> 2) * 8 + (shim_linear_tid() & 3) * 2 + (i & 1); }
static inline float shim_half_of(uint32_t word, int half, bool bf16);
static inline uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) |
         ((uint64_t)1 << 62);
}
static inline void wgmma_fence_operand(float&) {}
// m64nNk16, both operands K-major in shared memory: every thread computes its own accumulator registers
template <int N, bool BF16> static inline void wgmma_m64k16(float* d, uint64_t a, uint64_t b, int scale_d) {
  for (int i = 0; i < N / 2; ++i) {
    float acc = scale_d ? d[i] : 0.f;
    for (int k = 0; k < 16; ++k) acc += shim_operand(a, 0, acc_row(i), k, BF16) * shim_operand(b, 0, acc_col(i), k, BF16);
    d[i] = acc;
  }
}
// m64n128k16 with A in registers (the warpgroup's fragments are gathered through a per-CTA table) and B MN-major
template <bool BF16> static inline void wgmma_m64n128k16_rs_tb(float* d, const uint32_t* a, uint64_t b) {
  static thread_local uint32_t ga[128][4];
  const int tl = shim_linear_tid() & 127;
  for (int e = 0; e < 4; ++e) ga[tl][e] = a[e];
  named_bar_sync(14, 128);
  auto A = [&](int row, int k) {                 // a0: (g, 2t..) a1: (g+8, 2t..) a2: (g, 2t+8..) a3: (g+8, 2t+8..) of warp row / 16
    const int owner = (row / 16) * 32 + (row % 8) * 4 + (k % 8) / 2, e = ((row % 16) >= 8 ? 1 : 0) + (k >= 8 ? 2 : 0);
    return shim_half_of(ga[owner][e], k % 2, BF16);
  };
  for (int i = 0; i < 64; ++i) {
    float acc = d[i];
    for (int k = 0; k < 16; ++k) acc += A(acc_row(i), k) * shim_operand(b, 1, acc_col(i), k, BF16);
    d[i] = acc;
  }
  named_bar_sync(14, 128);
}
template <int BN> struct Acc128 {
  float d[2][BN / 2];
  void zero() { for (int h = 0; h < 2; ++h) for (int i = 0; i < BN / 2; ++i) d[h][i] = 0.f; }
  template <bool BF16> void mma_kblock(uint32_t a_addr, uint32_t b_addr, bool first) {
    // the operand rows this thread's registers touch, decoded once per K block: 2 x 2 rows of A, BN / 4 rows of B
    float A[2][2][64], B[BN / 4][64];
    const uint64_t b = gmma_desc_k_sw128(b_addr);
    for (int j = 0; j < BN / 4; ++j)
      for (int kk = 0; kk < 4; ++kk)
        for (int k = 0; k < 16; ++k) B[j][16 * kk + k] = shim_operand(b + 2 * kk, 0, acc_col((j >> 1) * 4 + (j & 1)), k, BF16);
    for (int h = 0; h < 2; ++h) {
      const uint64_t a = gmma_desc_k_sw128(a_addr + 64 * 128 * h);
      for (int r = 0; r < 2; ++r)
        for (int kk = 0; kk < 4; ++kk)
          for (int k = 0; k < 16; ++k) A[h][r][16 * kk + k] = shim_operand(a + 2 * kk, 0, acc_row(2 * r), k, BF16);
    }
    for (int h = 0; h < 2; ++h)
      for (int i = 0; i < BN / 2; ++i) {
        const float* ar = A[h][(i >> 1) & 1];
        const float* br = B[(i >> 2) * 2 + (i & 1)];
        float acc = first ? 0.f : d[h][i];
        for (int k = 0; k < 64; ++k) acc += ar[k] * br[k];
        d[h][i] = acc;
      }
  }
  void store(float* s, int ld) const {
    for (int h = 0; h < 2; ++h)
      for (int i = 0; i < BN / 2; ++i) s[(64 * h + acc_row(i)) * ld + acc_col(i)] = d[h][i];
  }
};
template <int BN> constexpr int acc_ld() { return BN + 8; }
template <int BN> constexpr int acc_smem_bytes() { return 128 * acc_ld<BN>() * 4; }
static inline void acc_ld16(const float* s, int ld, int row, int col, uint32_t* v) {
  for (int j = 0; j < 16; ++j) v[j] = shim_f2u(s[row * ld + col + j]);
}

// ---- warp-level matrix instructions (ldmatrix, mma.sync m16n8k16), emulated over the fibers of a warp:
// every lane publishes its operands, then computes its own result registers from the documented fragment layouts
static inline void shim_warp_allgather(uint64_t v, uint64_t* out) {
  ShimBlock::Warp& w = g_blk.warp[shim_linear_tid() >> 5];
  w.slot[shim_linear_tid() & 31] = v;
  shim_warp_rendezvous();
  for (int i = 0; i < 32; ++i) out[i] = w.slot[i];
  shim_warp_rendezvous();
}
static inline void shim_ldmatrix_x4(uint32_t addr, uint32_t* r, bool trans) {
  uint64_t rows[32];
  shim_warp_allgather((uint64_t)(uintptr_t)shim_smem_from_u32(addr), rows);      // lane 8j+i supplies row i of matrix j
  const int l = shim_linear_tid() & 31;
  for (int j = 0; j < 4; ++j) {
    if (!trans) {
      memcpy(&r[j], (const uint8_t*)(uintptr_t)rows[8 * j + l / 4] + (l % 4) * 4, 4);
    } else {
      uint16_t lo, hi;
      memcpy(&lo, (const uint8_t*)(uintptr_t)rows[8 * j + 2 * (l % 4)] + (l / 4) * 2, 2);
      memcpy(&hi, (const uint8_t*)(uintptr_t)rows[8 * j + 2 * (l % 4) + 1] + (l / 4) * 2, 2);
      r[j] = (uint32_t)lo | ((uint32_t)hi << 16);
    }
  }
}
static inline float shim_half_of(uint32_t word, int half, bool bf16) {
  const uint16_t v = (uint16_t)(half ? word >> 16 : word & 0xFFFFu);
  if (bf16) return shim_u2f((uint32_t)v << 16);
  __half h; h.bits = v; return __half2float(h);
}
static inline void shim_mma_m16n8k16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1, bool bf16) {
  uint64_t a01[32], a23[32], bb[32];
  shim_warp_allgather((uint64_t)a[0] | ((uint64_t)a[1] << 32), a01);
  shim_warp_allgather((uint64_t)a[2] | ((uint64_t)a[3] << 32), a23);
  shim_warp_allgather((uint64_t)b0 | ((uint64_t)b1 << 32), bb);
  const int l = shim_linear_tid() & 31, g = l / 4, t = l % 4;
  auto A = [&](int i, int k) {               // a0: (g, 2t..) a1: (g+8, 2t..) a2: (g, 2t+8..) a3: (g+8, 2t+8..)
    const int lane = (i % 8) * 4 + (k % 8) / 2;
    const uint64_t pr = k >= 8 ? a23[lane] : a01[lane];
    return shim_half_of((uint32_t)(i >= 8 ? pr >> 32 : pr), k % 2, bf16);
  };
  auto B = [&](int k, int n) {               // b0: (k = 2t.., n = g) b1: (k = 2t+8.., n = g)
    const uint64_t pr = bb[n * 4 + (k % 8) / 2];
    return shim_half_of((uint32_t)(k >= 8 ? pr >> 32 : pr), k % 2, bf16);
  };
  for (int idx = 0; idx < 4; ++idx) {
    const int row = g + (idx >= 2 ? 8 : 0), col = 2 * t + (idx & 1);
    float acc = c[idx];
    for (int k = 0; k < 16; ++k) acc += A(row, k) * B(k, col);
    c[idx] = acc;
  }
}

// ---- device allocations that other PROCESSES map (cudaMalloc + cudaIpc*): POSIX shared memory; the 64-byte handle carries the name
struct cudaIpcMemHandle_t { char reserved[64]; };
#define cudaIpcMemLazyEnablePeerAccess 1
int cudaMalloc(void** p, size_t bytes);
int cudaFree(void* p);
static inline int cudaMemset(void* p, int v, size_t n) { memset(p, v, n); return 0; }
int cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p);
int cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned flags);
int cudaIpcCloseMemHandle(void* p);
// system-scope flag traffic of the one-shot all-reduce / vocab-parallel argmax: plain atomics; pollers give way to the other fibers and ranks
static inline void shim_st_release(int* p, int v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static inline int shim_ld_acquire(const int* p) {
  const int v = __atomic_load_n(p, __ATOMIC_ACQUIRE);
  shim_yield();
  static thread_local unsigned n = 0;
  if ((++n & 255u) == 0) sched_yield();
  return v;
}

static inline __nv_bfloat162 __hsub2(__nv_bfloat162 a, __nv_bfloat162 b) {
  return {__float2bfloat16_rn(__bfloat162float(a.x) - __bfloat162float(b.x)), __float2bfloat16_rn(__bfloat162float(a.y) - __bfloat162float(b.y))};
}
static inline __nv_bfloat162 __hmul2(__nv_bfloat162 a, __nv_bfloat162 b) {
  return {__float2bfloat16_rn(__bfloat162float(a.x) * __bfloat162float(b.x)), __float2bfloat16_rn(__bfloat162float(a.y) * __bfloat162float(b.y))};
}
