// chatts_b200 -- W4A16 decode GEMM for the GPTQ-Int4 checkpoints the reference advertises (README.md:52,262-263):
//     partial[s][t][n] = sum_{k in split s} x[t][k] * sc[n][k / g] * (q[n][k] - zp[n][k / g])        (fp32 accumulate)
// A decode step is bound by the HBM stream of the weights; 4-bit codes are a quarter of the bf16 bytes (ChatTS-14B: 7 GB per step
// instead of 28), so the kernel keeps the swap-AB wgmma structure of gemm_tn_kernel -- weight tile = the 128-row MMA operand A, the
// tokens = the MMA N dimension, accumulator in registers -- and moves the dequantisation INTO the operand path:
//   warp 4      TMA producer: packed tiles [128 rows x 32 B] (64 K codes per row) into a deep staging ring (6 x 4 KB in flight
//               per CTA -- what keeps HBM busy -- requested BEFORE the dependency wait: nobody writes weights)
//   warps 5..   work item = one 32-bit word of codes (a row's 8 K elements): int4 -> bf16/fp16 with the magic-number trick (code | 0x4300 is the bf16
//               128 + code; - (128 + zp), x scale in packed half2 arithmetic = round(scale x (code - zp)) exactly, the value
//               weights.py:dequantize_gptq_linear(scale_dtype = model dtype) stores for the prefill) -> the 128B-swizzled K-major A tile of an
//               MMA stage; warp 5 also requests the token tile of that stage
//   warps 0..3  wgmma warpgroup, then the epilogue
// Split-K partials (CTS_EPI_PARTIAL_F32 semantics): the decode step's reduce kernels finish the projections as they do for bf16
// weights, so a quantised layer changes ONE launch in the step.  T <= 32 tokens (decode); prefill uses the dequantised copy
// (HBM holds both).  Result: bit-identical to cts_gemm on the dequantised weight (same values, same MMA order).
#include <type_traits>

#include "common.cuh"
#ifndef CTS_DYN_SMEM
#define CTS_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#endif
#include "tensormap.cuh"
#include "trace.cuh"

namespace {

constexpr int kBM = 128, kBK = 64;
constexpr int kDqWarps = 8;             // dequantising warps per CTA: the int4 -> 16-bit conversion is instruction-issue bound (ncu: 39 % issue
                                        // active with 4 warps and 1.5 CTAs per SM), so it gets as many warps as the shared memory budget allows CTAs
constexpr int kDqThreads = kDqWarps * 32;
constexpr int kDq0 = 160;              // first dequantising thread: after the MMA warpgroup and the producer warp
constexpr int kThreads = kDq0 + kDqThreads;
constexpr int kStg = 8;                 // staging ring of packed tiles (4 KB each): 48 KB of weight stream in flight per CTA, two CTAs per SM
                                        // (the first runs had 5 slots = 20 KB: the 4-bit stream was latency-bound at ~1.6 TB/s)
constexpr int kMs = 3;                  // MMA stages (dequantised A tile 16 KB + token tile): the conversion of block i+2 must not wait for the MMA of block i
constexpr int kPacked = kBM * kBK / 2;  // 4096 bytes
constexpr int kMaxGroups = 44;          // groups a CTA's K range may touch (scale 2 B + zero point 1 B per row kept in shared memory: 16.5 KB;
                                        // 44 covers an unsplit K = 5120 at group size 128)

struct W4Params {
  long long n, k, t;
  int kb_total, split_k, group_size, n_groups;
  const void* sc;          // [n, n_groups] model dtype
  const uint8_t* zp;       // [n, n_groups]
  float* out;              // fp32 [split_k, t, n]
};

template <typename T> struct Magic;
template <> struct Magic<__nv_bfloat16> {
  static constexpr uint32_t kOr = 0x43004300u;                       // bf16 128.0 in both halves: 128 + code
  // packed (128 + zp): in [128, 256) a bf16 ulp is 1, so 128 + zp is the bit pattern 0x4300 + zp (zp <= 16)
  static __device__ __forceinline__ uint32_t bias(uint32_t zp) { return (0x4300u + zp) * 0x00010001u; }
  static __device__ __forceinline__ uint32_t cvt(uint32_t codes, uint32_t b2, uint32_t s2) {
    const uint32_t y = codes | kOr;
    __nv_bfloat162 d = __hsub2(*reinterpret_cast<const __nv_bfloat162*>(&y), *reinterpret_cast<const __nv_bfloat162*>(&b2));   // exact small ints
    __nv_bfloat162 w = __hmul2(d, *reinterpret_cast<const __nv_bfloat162*>(&s2));                                              // one rounding
    return *reinterpret_cast<uint32_t*>(&w);
  }
};
template <> struct Magic<__half> {
  static constexpr uint32_t kOr = 0x64006400u;                       // fp16 1024.0: 1024 + code (ulp 1 in [1024, 2048))
  static __device__ __forceinline__ uint32_t bias(uint32_t zp) { return (0x6400u + zp) * 0x00010001u; }
  static __device__ __forceinline__ uint32_t cvt(uint32_t codes, uint32_t b2, uint32_t s2) {
    const uint32_t y = codes | kOr;
    __half2 d = __hsub2(*reinterpret_cast<const __half2*>(&y), *reinterpret_cast<const __half2*>(&b2));
    __half2 w = __hmul2(d, *reinterpret_cast<const __half2*>(&s2));
    return *reinterpret_cast<uint32_t*>(&w);
  }
};

template <typename T, int BN>
__global__ void __launch_bounds__(kThreads, 2)   // two CTAs per SM: the split heuristic below sizes one wave of them
gemm_w4_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_x, const W4Params p) {
  CTS_DYN_SMEM(smem_raw);
  __shared__ uint64_t stg_full[kStg], stg_empty[kStg], mma_full[kMs], mma_empty[kMs];
  __shared__ uint16_t sc_s[kMaxGroups][kBM];       // scale bits per (group, row)
  __shared__ uint8_t zp_s[kMaxGroups][kBM];        // integer zero point per (group, row)

  constexpr int kABytes = kBM * kBK * 2;
  constexpr int kMStage = kABytes + BN * kBK * 2;
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;
  static_assert(BN == 16 || BN == 32, "decode-sized token tile");

  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* mma_s = smem;                                   // kMs x kMStage (1024-byte aligned tiles)
  uint8_t* stg_s = smem + (size_t)kMs * kMStage;           // kStg x 4 KB

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f0 = blockIdx.x * kBM;
  const int split = blockIdx.z;
  const int kb0 = (int)(((long long)p.kb_total * split) / p.split_k);
  const int kb1 = (int)(((long long)p.kb_total * (split + 1)) / p.split_k);
  const int nkb = kb1 - kb0;
  const int g0 = (kb0 * kBK) / p.group_size;               // first group of this CTA's K range

  pdl_trigger();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_x);
    for (int s = 0; s < kStg; ++s) { mbar_init(&stg_full[s], 1); mbar_init(&stg_empty[s], kDqWarps); }
    for (int s = 0; s < kMs; ++s) { mbar_init(&mma_full[s], 1 + kDqWarps); mbar_init(&mma_empty[s], 1); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ------------------------------ TMA producer: the packed weight stream (weights are static: no dependency wait) ------------------------------
    if (lane == 0) {
      CTS_TRACE(CTS_TK_GEMM, 0);
      for (int i = 0; i < nkb; ++i) {
        const int s = i % kStg;
        mbar_wait(&stg_empty[s], (((uint32_t)(i / kStg)) & 1u) ^ 1u);
        mbar_expect_tx(&stg_full[s], (uint32_t)kPacked);
        tma_load_2d(stg_s + (size_t)s * kPacked, &tm_q, &stg_full[s], (kb0 + i) * (kBK / 4), f0, CTS_L2_EVICT_FIRST);     // 16 two-byte units = 64 codes
      }
      CTS_TRACE(CTS_TK_GEMM, 2);
    }
  } else if (warp < 4) {
    // ------------------------------ MMA warpgroup ------------------------------
    Acc128<BN> acc;
    acc.zero();
    for (int i = 0; i < nkb; ++i) {
      const int s = i % kMs;
      mbar_wait(&mma_full[s], ((uint32_t)(i / kMs)) & 1u);
      const uint32_t a_addr = smem_u32(mma_s + (size_t)s * kMStage);
      acc.template mma_kblock<kIsBf16>(a_addr, a_addr + kABytes, i == 0);
      wgmma_wait<1>();
      if (i > 0 && threadIdx.x == 0) mbar_arrive(&mma_empty[(i - 1) % kMs]);
    }
    wgmma_wait<0>();
    if (nkb > 0 && threadIdx.x == 0) mbar_arrive(&mma_empty[(nkb - 1) % kMs]);
    // ------------------------------ epilogue: fp32 partial of this split ------------------------------
    float* dst = p.out + (long long)split * p.t * p.n;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) {
        const long long fo = (long long)f0 + 64 * h + acc_row(i), t = acc_col(i);
        if (t < p.t && fo < p.n) dst[t * p.n + fo] = acc.d[h][i];
      }
  } else {
    // ------------------------------ dequantisers (thread = weight row) ------------------------------
    const int r = (int)threadIdx.x - kDq0;                    // 0..kDqThreads-1; the first 128 also own a row of the (group, row) table
    const long long f = (long long)f0 + r;
    const bool f_ok = f < p.n && r < kBM;
    if (r < kBM) {
      // scale / zero point of this row for every group the CTA's K range touches (static data: before the dependency wait)
      const int g1 = nkb > 0 ? ((kb1 * kBK - 1) / p.group_size) : g0;
      const T* sc = reinterpret_cast<const T*>(p.sc);
      for (int g = g0; g <= g1 && g - g0 < kMaxGroups; ++g) {
        uint16_t su = 0;
        uint8_t zv = 0;
        if (f_ok && g < p.n_groups) {
          const T sv = sc[f * p.n_groups + g];
          su = *reinterpret_cast<const uint16_t*>(&sv);
          zv = p.zp[f * p.n_groups + g];
        }
        sc_s[g - g0][r] = su;
        zp_s[g - g0][r] = zv;
      }
    }
    named_bar_sync(1, kDqThreads);                          // the (group, row) table is read by other threads than the ones that wrote it
    pdl_wait();                                             // the token operand comes from the predecessor
    if (threadIdx.x == kDq0) CTS_TRACE(CTS_TK_GEMM, 1);
    for (int i = 0; i < nkb; ++i) {
      const int ss = i % kStg, ms = i % kMs;
      mbar_wait(&mma_empty[ms], (((uint32_t)(i / kMs)) & 1u) ^ 1u);        // the MMAs that read this stage have completed
      uint8_t* a_tile = mma_s + (size_t)ms * kMStage;
      if (threadIdx.x == kDq0) {                                          // the token tile of this stage (L2-resident, evict-last)
        mbar_expect_tx(&mma_full[ms], (uint32_t)(BN * kBK * 2));
        tma_load_2d(a_tile + kABytes, &tm_x, &mma_full[ms], (kb0 + i) * kBK, 0, CTS_L2_EVICT_LAST);
      }
      mbar_wait(&stg_full[ss], ((uint32_t)(i / kStg)) & 1u);
      // Work item = (row, 16-byte output chunk) = ONE 32-bit word of codes: the 32 lanes of a warp take 4 consecutive rows x 8 chunks,
      // so a warp reads 128 contiguous bytes of the packed tile and writes 4 complete 128-byte rows of the swizzled operand tile --
      // both conflict-free (the first version mapped a thread to a whole row: every 16-byte store of a warp hit 32 different rows,
      // 16 wavefronts each, and the kernel ran at the speed of the shared-memory store pipe).
      const uint32_t* stg32 = reinterpret_cast<const uint32_t*>(stg_s + (size_t)ss * kPacked);
      const int g = ((kb0 + i) * kBK) / p.group_size - g0;
      const int wq = warp - kDq0 / 32;                                    // 0..kDqWarps-1
      constexpr int kIts = kBM / (4 * kDqWarps);                          // 4 rows per warp and iteration
      uint32_t wv[kIts];
#pragma unroll
      for (int it = 0; it < kIts; ++it) wv[it] = stg32[(it * 4 * kDqWarps + wq * 4 + (lane >> 3)) * 8 + (lane & 7)];
#pragma unroll
      for (int it = 0; it < kIts; ++it) {
        const int rr = it * 4 * kDqWarps + wq * 4 + (lane >> 3), ch = lane & 7;
        const uint32_t s2 = (uint32_t)sc_s[g][rr] * 0x00010001u, b2 = Magic<T>::bias((uint32_t)zp_s[g][rr]);
        uint4 o;
        o.x = Magic<T>::cvt(wv[it] & 0x000F000Fu, b2, s2);
        o.y = Magic<T>::cvt((wv[it] >> 4) & 0x000F000Fu, b2, s2);
        o.z = Magic<T>::cvt((wv[it] >> 8) & 0x000F000Fu, b2, s2);
        o.w = Magic<T>::cvt((wv[it] >> 12) & 0x000F000Fu, b2, s2);
        *reinterpret_cast<uint4*>(a_tile + (uint32_t)rr * 128 + ((ch ^ (rr & 7)) << 4)) = o;
      }
      fence_proxy_async_smem();                                           // generic-proxy writes -> visible to the tensor core
      __syncwarp();
      if (lane == 0) {
        // the staging slot is released only now, after every word read from it has been USED: the TMA that refills it runs in the
        // async proxy, and a slot released right after issuing the loads (5-slot version) produced one stale block in ~1 of 50 runs
        mbar_arrive(&stg_empty[ss]);
        mbar_arrive(&mma_full[ms]);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_GEMM, 3);
}

template <typename T, int BN>
int launch_w4(cts_ctx* ctx, const cts_gemm_w4_args* a, cudaStream_t stream) {
  const bool is_bf16 = a->dtype == CTS_BF16;
  CUtensorMap tm_q, tm_x;
  // the packed codes as a dense (un-swizzled) matrix of 2-byte units: [n, k/4], box = 128 rows x 16 units (32 B = 64 codes)
  int rc = cts_make_tmap_2d_dense(ctx, &tm_q, a->qw, a->n, a->k / 4, a->k / 4, kBM, kBK / 4, 1);
  if (rc) return rc;
  rc = cts_make_tmap_2d(ctx, &tm_x, a->x, a->t, a->k, a->x_ld, BN, is_bf16);
  if (rc) return rc;
  W4Params p;
  p.n = a->n; p.k = a->k; p.t = a->t;
  p.kb_total = (int)cdiv_ll(a->k, kBK);
  p.split_k = a->split_k; p.group_size = a->group_size; p.n_groups = (int)(a->k / a->group_size);
  p.sc = a->scales; p.zp = (const uint8_t*)a->zeros; p.out = a->out;
  constexpr int kMStage = kBM * kBK * 2 + BN * kBK * 2;
  const size_t smem = (size_t)kMs * kMStage + (size_t)kStg * kPacked + 1024;
  auto kern = gemm_w4_kernel<T, BN>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
#ifndef CTS_HOST_SHIM
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
#endif
  dim3 grid((unsigned)cdiv_ll(a->n, kBM), 1, (unsigned)a->split_k);
  CTS_CUDA(ctx, launch_pdl(kern, grid, dim3(kThreads), smem, stream, 1, tm_q, tm_x, p));
  return CTS_OK;
}

}  // namespace

// split-K factor for the W4 stream: one wave of the CTAs an SM holds (~98 KB of shared memory per CTA -> 2 per SM)
extern "C" int cts_gemm_w4_suggest_split(cts_ctx* ctx, long long n, long long k) {
  if (!ctx || n <= 0 || k <= 0) return 1;
  const long long tiles = cdiv_ll(n, kBM), kb = cdiv_ll(k, kBK);
  long long s = (4LL * ctx->sm_count) / tiles;          // ~two waves of the two CTAs an SM holds (__launch_bounds__)
  if (s > kb / 2) s = kb / 2;
  if (s > 16) s = 16;
  if (s < 1) s = 1;
  return (int)s;
}

extern "C" int cts_gemm_w4(cts_ctx* ctx, const cts_gemm_w4_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr && a->qw && a->scales && a->zeros && a->x && a->out, "null pointer");
  CTS_CHECK_ARG(ctx, a->n > 0 && a->k > 0 && a->t > 0 && a->t <= 32, "n, k > 0 and 1 <= t <= 32 (decode-sized step; prefill uses the dequantised weight)");
  CTS_CHECK_ARG(ctx, a->dtype == CTS_BF16 || a->dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, a->k % 64 == 0, "k must be a multiple of 64");
  CTS_CHECK_ARG(ctx, a->group_size >= 64 && a->group_size % 64 == 0 && a->k % a->group_size == 0, "group_size must be a multiple of 64 dividing k");
  CTS_CHECK_ARG(ctx, a->split_k >= 1 && a->split_k <= cdiv_ll(a->k, kBK), "split_k");
  CTS_CHECK_ARG(ctx, a->x_ld >= a->k, "x_ld smaller than k");
  // groups one CTA may touch: its K range is at most ceil(kb_total / split) + 1 blocks
  const long long blocks = cdiv_ll(cdiv_ll(a->k, kBK), a->split_k) + 1;
  CTS_CHECK_ARG(ctx, blocks * kBK / a->group_size + 2 <= kMaxGroups, "K range per split touches more than 44 groups: raise split_k");
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dtype == CTS_BF16) return a->t <= 16 ? launch_w4<__nv_bfloat16, 16>(ctx, a, st) : launch_w4<__nv_bfloat16, 32>(ctx, a, st);
  return a->t <= 16 ? launch_w4<__half, 16>(ctx, a, st) : launch_w4<__half, 32>(ctx, a, st);
}

CTS_TRACE_SETTER(cts_trace_set_w4)
