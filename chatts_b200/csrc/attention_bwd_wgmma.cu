// chatts_b200 -- attention backward on wgmma (head_dim 128): the FlashAttention-2 recomputation of attention_bwd.cu
// (P = exp(scale S - lse), dV = P^T dO, dP = dO V^T, dS = P o (dP - delta), dQ = scale dS K, dK = scale dS^T Q) with the
// operand forms of the wgmma prefill kernel (attention.cu): TMA loads with the 128-byte swizzle, S and dP from wgmma with both
// operands K-major in shared memory, P / dS converted in registers and fed back as the register A operand of the second MMA,
// whose B operand (K, Q or dO) is read MN-major from the same shared-memory tile.
//
//   attn_bwd_dq_wgmma_kernel   grid (ceil(max_seqlen / 64), nh, batch): 64 query rows of one head; Q and dO stay in shared
//                              memory, the K / V tiles of the causal range stream through a two-stage TMA ring.
//   attn_bwd_dkv_wgmma_kernel  grid (ceil(max_seqlen / 64), nkv, batch): 64 key rows of one kv head; K and V stay, the (Q, dO)
//                              tiles of every q head of the group and every query tile at or below the diagonal stream through
//                              the ring.  dK / dV are summed over the group in registers: no atomics, a fixed summation order.
// Warps 0..3 are the MMA warpgroup, warp 4 the TMA producer.  delta comes from attn_bwd_delta_kernel (attention_bwd.cu).
#include <type_traits>

#include "common.cuh"
#include "tensormap.cuh"

namespace {

constexpr int kBt = 64, kBThreads = 160, kBStages = 2;
constexpr int kBHalf = 64 * 128;                 // one [64 rows x 128 B] swizzled half of a 64 x 128 tile (8 KiB)
constexpr int kBTile = 2 * kBHalf;               // a 64 x 128 tile
constexpr int kBStage = 2 * kBTile;              // two tiles per ring stage
constexpr int kBSmem = 2 * kBTile + kBStages * kBStage;
constexpr float kL2e = 1.4426950408889634f;

template <typename T> __device__ __forceinline__ uint32_t bpack2(float lo, float hi) {
  T v[2] = {DT<T>::from_f(lo), DT<T>::from_f(hi)};
  return *reinterpret_cast<uint32_t*>(v);
}

// acc[32] (+)= A[64 x 128] B[64 x 128]^T, both 64 x 128 tiles K-major (two swizzled halves each) at a_addr / b_addr
template <bool BF16> __device__ __forceinline__ void mma_nt_64x64(float* acc, uint32_t a_addr, uint32_t b_addr) {
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const uint32_t off = (uint32_t)(kk >> 2) * kBHalf;
    wgmma_m64k16<64, BF16>(acc, gmma_desc_k_sw128(a_addr + off) + 2 * (kk & 3), gmma_desc_k_sw128(b_addr + off) + 2 * (kk & 3), kk > 0);
  }
}
// acc[64] += A[64 x 64] (register fragments a[4][4]) * B[64 x 128], B = a 64 x 128 tile read MN-major (its rows are the K index)
template <bool BF16> __device__ __forceinline__ void mma_rs_64x128(float* acc, const uint32_t (*a)[4], uint32_t b_addr) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_m64n128k16_rs_tb<BF16>(acc, a[kk], gmma_desc_sw128(b_addr + (uint32_t)kk * 16 * 128, kBHalf, 1024));
}
template <int N> __device__ __forceinline__ void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) wgmma_fence_operand(r[i]);
}
__device__ __forceinline__ void load_tile(uint8_t* dst, const CUtensorMap* tm, uint64_t* bar, int col0, int row) {
  tma_load_2d(dst, tm, bar, col0, row, CTS_L2_EVICT_LAST);
  tma_load_2d(dst + kBHalf, tm, bar, col0 + 64, row, CTS_L2_EVICT_LAST);
}

// ------------------------------------------------------------------------------------------------ dQ
template <typename T>
__global__ void __launch_bounds__(kBThreads, 1)
attn_bwd_dq_wgmma_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                         const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_do,
                         const float* __restrict__ lse, const float* __restrict__ delta, const int* __restrict__ cu_seqlens, int nh,
                         int nkv, float scale, T* __restrict__ dq) {
  extern __shared__ uint8_t bq_raw[];
  __shared__ uint64_t fix_bar, full_bar[kBStages], empty_bar[kBStages];
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;
  const uint32_t raw = smem_u32(bq_raw);
  uint8_t* smem = bq_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* q_s = smem;                                   // Q tile, then dO tile
  uint8_t* ring = smem + 2 * kBTile;                     // [stage][K tile | V tile]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (nh / nkv);

  pdl_trigger();
  if (threadIdx.x == 0) {
    mbar_init(&fix_bar, 1);
    for (int s = 0; s < kBStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  const int seq0 = cu_seqlens[b], len = cu_seqlens[b + 1] - seq0;
  const int q0 = qt * kBt;
  if (q0 >= len) return;                                 // CTA-uniform; nothing was issued yet
  const int ntiles = (min(len, q0 + kBt) + kBt - 1) / kBt;   // causal: keys 0 .. q0 + 63

  if (warp == 4) {
    if (lane == 0) {
      mbar_expect_tx(&fix_bar, 2u * kBTile);
      load_tile(q_s, &tm_q, &fix_bar, head * 128, seq0 + q0);
      load_tile(q_s + kBTile, &tm_do, &fix_bar, head * 128, seq0 + q0);
      for (int j = 0; j < ntiles; ++j) {
        const int s = j % kBStages;
        mbar_wait(&empty_bar[s], ((uint32_t)(j / kBStages) & 1u) ^ 1u);
        mbar_expect_tx(&full_bar[s], (uint32_t)kBStage);
        uint8_t* st = ring + (size_t)s * kBStage;
        load_tile(st, &tm_k, &full_bar[s], kvh * 128, seq0 + j * kBt);
        load_tile(st + kBTile, &tm_v, &full_bar[s], kvh * 128, seq0 + j * kBt);
      }
    }
    return;
  }
  if (warp > 4) return;

  const float sl2 = scale * kL2e;
  const int rows[2] = {q0 + acc_row(0), q0 + acc_row(2)};
  float lse2[2], dlt[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool ok = rows[h] < len;
    lse2[h] = ok ? lse[(long long)(seq0 + rows[h]) * nh + head] * kL2e : 0.f;
    dlt[h] = ok ? delta[(long long)(seq0 + rows[h]) * nh + head] : 0.f;
  }
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  const uint32_t q_addr = smem_u32(q_s), do_addr = q_addr + kBTile;
  mbar_wait(&fix_bar, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int s = j % kBStages;
    mbar_wait(&full_bar[s], (uint32_t)(j / kBStages) & 1u);
    const uint32_t k_addr = smem_u32(ring + (size_t)s * kBStage), v_addr = k_addr + kBTile;
    float sc[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { sc[i] = 0.f; dp[i] = 0.f; }
    fence_regs<32>(sc);
    fence_regs<32>(dp);
    wgmma_fence();
    mma_nt_64x64<kIsBf16>(sc, q_addr, k_addr);           // S  = Q K^T
    mma_nt_64x64<kIsBf16>(dp, do_addr, v_addr);          // dP = dO V^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(sc);
    fence_regs<32>(dp);
    uint32_t a[4][4];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1, row = rows[h];
      float ds[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = j * kBt + acc_col(i + e);
        const float p = (col <= row && row < len) ? exp2f(sc[i + e] * sl2 - lse2[h]) : 0.f;
        ds[e] = p * (dp[i + e] - dlt[h]) * scale;
      }
      a[i >> 3][(i >> 1) & 3] = bpack2<T>(ds[0], ds[1]);
    }
    fence_regs<64>(acc);
    wgmma_fence();
    mma_rs_64x128<kIsBf16>(acc, a, k_addr);              // dQ += dS K
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<64>(acc);
    if (threadIdx.x == 0) mbar_arrive(&empty_bar[s]);
  }
  const long long ld = (long long)nh * 128;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (rows[h] >= len) continue;
    T* orow = dq + (long long)(seq0 + rows[h]) * ld + head * 128;
#pragma unroll
    for (int i = 2 * h; i < 64; i += 4) *reinterpret_cast<uint32_t*>(orow + acc_col(i)) = bpack2<T>(acc[i], acc[i + 1]);
  }
}

// ------------------------------------------------------------------------------------------------ dK / dV
template <typename T>
__global__ void __launch_bounds__(kBThreads, 1)
attn_bwd_dkv_wgmma_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                          const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_do,
                          const float* __restrict__ lse, const float* __restrict__ delta, const int* __restrict__ cu_seqlens, int nh,
                          int nkv, float scale, T* __restrict__ dk, T* __restrict__ dv) {
  extern __shared__ uint8_t bkv_raw[];
  __shared__ uint64_t fix_bar, full_bar[kBStages], empty_bar[kBStages];
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;
  const uint32_t raw = smem_u32(bkv_raw);
  uint8_t* smem = bkv_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* k_s = smem;                                   // K tile, then V tile
  uint8_t* ring = smem + 2 * kBTile;                     // [stage][Q tile | dO tile]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kt = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int G = nh / nkv;

  pdl_trigger();
  if (threadIdx.x == 0) {
    mbar_init(&fix_bar, 1);
    for (int s = 0; s < kBStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  const int seq0 = cu_seqlens[b], len = cu_seqlens[b + 1] - seq0;
  const int k0 = kt * kBt;
  if (k0 >= len) return;
  const int nq = (len + kBt - 1) / kBt - kt;              // query tiles kt .. (at or below the diagonal)
  const int items = G * nq;                              // (q head of the group, query tile), head-major

  if (warp == 4) {
    if (lane == 0) {
      mbar_expect_tx(&fix_bar, 2u * kBTile);
      load_tile(k_s, &tm_k, &fix_bar, kvh * 128, seq0 + k0);
      load_tile(k_s + kBTile, &tm_v, &fix_bar, kvh * 128, seq0 + k0);
      for (int it = 0; it < items; ++it) {
        const int s = it % kBStages, head = kvh * G + it / nq, qrow = seq0 + (kt + it % nq) * kBt;
        mbar_wait(&empty_bar[s], ((uint32_t)(it / kBStages) & 1u) ^ 1u);
        mbar_expect_tx(&full_bar[s], (uint32_t)kBStage);
        uint8_t* st = ring + (size_t)s * kBStage;
        load_tile(st, &tm_q, &full_bar[s], head * 128, qrow);
        load_tile(st + kBTile, &tm_do, &full_bar[s], head * 128, qrow);
      }
    }
    return;
  }
  if (warp > 4) return;

  const float sl2 = scale * kL2e;
  const int keys[2] = {k0 + acc_row(0), k0 + acc_row(2)};
  float dka[64], dva[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) { dka[i] = 0.f; dva[i] = 0.f; }
  const uint32_t k_addr = smem_u32(k_s), v_addr = k_addr + kBTile;
  mbar_wait(&fix_bar, 0);
  for (int it = 0; it < items; ++it) {
    const int s = it % kBStages, head = kvh * G + it / nq, q0 = (kt + it % nq) * kBt;
    mbar_wait(&full_bar[s], (uint32_t)(it / kBStages) & 1u);
    const uint32_t q_addr = smem_u32(ring + (size_t)s * kBStage), do_addr = q_addr + kBTile;
    float sc[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { sc[i] = 0.f; dp[i] = 0.f; }
    fence_regs<32>(sc);
    fence_regs<32>(dp);
    wgmma_fence();
    mma_nt_64x64<kIsBf16>(sc, k_addr, q_addr);           // S^T  = K Q^T   (rows = keys, columns = queries)
    mma_nt_64x64<kIsBf16>(dp, v_addr, do_addr);          // dP^T = V dO^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(sc);
    fence_regs<32>(dp);
    uint32_t ap[4][4], ads[4][4];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int key = keys[(i >> 1) & 1];
      float p[2], ds[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int qi = q0 + acc_col(i + e);
        const bool ok = key <= qi && qi < len;
        const long long sidx = (long long)(seq0 + qi) * nh + head;
        p[e] = ok ? exp2f(sc[i + e] * sl2 - __ldg(lse + sidx) * kL2e) : 0.f;
        ds[e] = ok ? p[e] * (dp[i + e] - __ldg(delta + sidx)) * scale : 0.f;
      }
      ap[i >> 3][(i >> 1) & 3] = bpack2<T>(p[0], p[1]);
      ads[i >> 3][(i >> 1) & 3] = bpack2<T>(ds[0], ds[1]);
    }
    fence_regs<64>(dva);
    fence_regs<64>(dka);
    wgmma_fence();
    mma_rs_64x128<kIsBf16>(dva, ap, do_addr);            // dV += P^T dO
    mma_rs_64x128<kIsBf16>(dka, ads, q_addr);            // dK += dS^T Q
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<64>(dva);
    fence_regs<64>(dka);
    if (threadIdx.x == 0) mbar_arrive(&empty_bar[s]);
  }
  const long long ld = (long long)nkv * 128;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (keys[h] >= len) continue;
    T* krow = dk + (long long)(seq0 + keys[h]) * ld + kvh * 128;
    T* vrow = dv + (long long)(seq0 + keys[h]) * ld + kvh * 128;
#pragma unroll
    for (int i = 2 * h; i < 64; i += 4) {
      *reinterpret_cast<uint32_t*>(krow + acc_col(i)) = bpack2<T>(dka[i], dka[i + 1]);
      *reinterpret_cast<uint32_t*>(vrow + acc_col(i)) = bpack2<T>(dva[i], dva[i + 1]);
    }
  }
}

template <typename T>
int launch(cts_ctx* ctx, const void* q, const void* k, const void* v, const void* dout, const float* lse, const float* delta,
           const int* cu_seqlens, int batch, int max_seqlen, long long total_tokens, int nh, int nkv, float scale, void* dq, void* dk,
           void* dv, cudaStream_t st) {
  const bool bf = std::is_same<T, __nv_bfloat16>::value;
  CUtensorMap tm_q, tm_k, tm_v, tm_do;
  int rc = cts_make_tmap_2d(ctx, &tm_q, q, total_tokens, (long long)nh * 128, (long long)nh * 128, kBt, bf);
  if (rc) return rc;
  rc = cts_make_tmap_2d(ctx, &tm_do, dout, total_tokens, (long long)nh * 128, (long long)nh * 128, kBt, bf);
  if (rc) return rc;
  rc = cts_make_tmap_2d(ctx, &tm_k, k, total_tokens, (long long)nkv * 128, (long long)nkv * 128, kBt, bf);
  if (rc) return rc;
  rc = cts_make_tmap_2d(ctx, &tm_v, v, total_tokens, (long long)nkv * 128, (long long)nkv * 128, kBt, bf);
  if (rc) return rc;
  const size_t smem = (size_t)kBSmem + 1024;
  const unsigned tiles = (unsigned)((max_seqlen + kBt - 1) / kBt);
  auto kq = attn_bwd_dq_wgmma_kernel<T>;
  auto kkv = attn_bwd_dkv_wgmma_kernel<T>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kq, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CTS_CUDA(ctx, cudaFuncSetAttribute(kkv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CTS_CUDA(ctx, launch_pdl(kq, dim3(tiles, (unsigned)nh, (unsigned)batch), dim3(kBThreads), smem, st, 1, tm_q, tm_k, tm_v, tm_do, lse, delta,
                           cu_seqlens, nh, nkv, scale, (T*)dq));
  CTS_CUDA(ctx, launch_pdl(kkv, dim3(tiles, (unsigned)nkv, (unsigned)batch), dim3(kBThreads), smem, st, 1, tm_q, tm_k, tm_v, tm_do, lse,
                           delta, cu_seqlens, nh, nkv, scale, (T*)dk, (T*)dv));
  return CTS_OK;
}

}  // namespace

// head_dim 128; delta = rowsum(dO o O) must already be in `delta` (attn_bwd_delta_kernel on the same stream)
int cts_attn_bwd_wgmma_launch(cts_ctx* ctx, const void* q, const void* k, const void* v, const void* dout, const float* lse,
                              const float* delta, const int* cu_seqlens, int batch, int max_seqlen, long long total_tokens, int nh,
                              int nkv, float scale, void* dq, void* dk, void* dv, int dtype, cudaStream_t st) {
  if (dtype == CTS_BF16)
    return launch<__nv_bfloat16>(ctx, q, k, v, dout, lse, delta, cu_seqlens, batch, max_seqlen, total_tokens, nh, nkv, scale, dq, dk, dv, st);
  return launch<__half>(ctx, q, k, v, dout, lse, delta, cu_seqlens, batch, max_seqlen, total_tokens, nh, nkv, scale, dq, dk, dv, st);
}
