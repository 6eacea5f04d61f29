// chatts_b200 -- causal GQA attention (the arithmetic of transformers qwen2/modeling_qwen2.py:161-184, which the
// reference reaches through vLLM's Attention layer, chatts/vllm/chatts_vllm.py:595-598).
//
//  cts_attn_prefill : variable-length causal attention over the tokens of one call (no prefix).  Tensor-core
//                     (HMMA via nvcuda::wmma) flash attention in two passes over the KV tiles: pass 1 finds the
//                     row max / row sum, pass 2 accumulates exp(s - m) V in fragments, so no accumulator rescale
//                     is needed; head_dim 64.  head_dim 128 runs attn_prefill_wgmma_kernel (wgmma, single-pass online
//                     softmax with S and O in registers).
//  cts_attn_decode  : one query token per sequence against the PAGED KV cache, flash-decoding split over pages.
//                     HBM-bound (GQA intensity = nh/nkv flop/B): K/V pages are pulled with cp.async.bulk into a
//                     double-buffered shared-memory ring (mbarrier complete_tx), all q heads of a kv head share
//                     each page; partial (m, l, o) per split are merged by a second tiny kernel.
#include <mma.h>

#include <type_traits>

#include "common.cuh"
#include "trace.cuh"
#include "tensormap.cuh"

namespace {

using namespace nvcuda;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <typename T> struct WT;
template <> struct WT<__nv_bfloat16> { using type = __nv_bfloat16; };
template <> struct WT<__half> { using type = __half; };

// ================================================================================================
// prefill
// ================================================================================================
constexpr int kPfQ = 64;        // query rows per CTA (16 per warp)
constexpr int kPfKV = 64;       // kv tokens per tile
constexpr int kPfThreads = 128;

template <int HD> struct PfSmem {
  static constexpr int LD = HD + 8;                       // padded row, elements
  static constexpr int SLD = kPfKV + 8;                   // padded score row, floats
  static constexpr size_t q_bytes = (size_t)kPfQ * LD * 2;
  static constexpr size_t kv_bytes = (size_t)kPfKV * LD * 2;
  static constexpr size_t s_bytes = (size_t)4 * 16 * SLD * 4;   // per-warp 16 x 64 fp32
  static constexpr size_t p_bytes = (size_t)4 * 16 * SLD * 2;   // per-warp 16 x 64 model dtype
  static constexpr size_t o_bytes = (size_t)4 * 16 * (HD + 8) * 4;
  // layout: Q | K0 | V0 | K1 | V1 | S | P ;  the O staging reuses the K0.. region at the end
  static constexpr size_t total = q_bytes + 4 * kv_bytes + s_bytes + p_bytes;
};

template <typename T, int HD>
__device__ __forceinline__ void pf_load_tile(T* dst, const T* __restrict__ src, long long row_stride, int rows_valid) {
  // 64 rows x HD elements, 16 B per cp.async
  constexpr int LD = PfSmem<HD>::LD;
  constexpr int CH = HD / 8;
  for (int i = threadIdx.x; i < kPfKV * CH; i += kPfThreads) {
    const int r = i / CH, c = i % CH;
    const bool ok = r < rows_valid;
    cp_async16(dst + r * LD + c * 8, src + (ok ? (long long)r * row_stride + c * 8 : 0), ok);
  }
}

// LSE = true (the training forward, cts_attn_prefill_lse) adds one store per query row: lse[token][head] = log sum_j exp(scale s_j).
template <typename T, int HD, bool LSE>
__global__ void __launch_bounds__(kPfThreads)
attn_prefill_kernel(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v,
                    const int* __restrict__ cu_seqlens, int nh, int nkv, float scale, T* __restrict__ out, float* __restrict__ lse) {
  using SM = PfSmem<HD>;
  constexpr int LD = SM::LD, SLD = SM::SLD;
  extern __shared__ __align__(128) uint8_t pf_smem[];
  T* q_s = reinterpret_cast<T*>(pf_smem);
  T* kv_s = reinterpret_cast<T*>(pf_smem + SM::q_bytes);                       // [2][K|V][64][LD]
  float* s_all = reinterpret_cast<float*>(pf_smem + SM::q_bytes + 4 * SM::kv_bytes);
  T* p_all = reinterpret_cast<T*>(pf_smem + SM::q_bytes + 4 * SM::kv_bytes + SM::s_bytes);

  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.z, head = blockIdx.y, qt = blockIdx.x;
  const int seq0 = cu_seqlens[b], len = cu_seqlens[b + 1] - seq0;
  const int q0 = qt * kPfQ;
  if (q0 >= len) return;
  const int kvh = head / (nh / nkv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long q_stride = (long long)nh * HD, kv_stride = (long long)nkv * HD;
  const T* q_g = q + ((long long)seq0 + q0) * q_stride + (long long)head * HD;
  const T* k_g = k + (long long)seq0 * kv_stride + (long long)kvh * HD;
  const T* v_g = v + (long long)seq0 * kv_stride + (long long)kvh * HD;

  const int n_tiles = (min(q0 + kPfQ, len) + kPfKV - 1) / kPfKV;   // causal: kv <= last q row of this CTA

  auto kbuf = [&](int st) { return kv_s + (size_t)st * 2 * kPfKV * LD; };
  auto vbuf = [&](int st) { return kv_s + (size_t)st * 2 * kPfKV * LD + (size_t)kPfKV * LD; };
  auto issue_tile = [&](int j, int st, bool with_v) {
    const int kv0 = j * kPfKV;
    const int valid = min(kPfKV, len - kv0);
    pf_load_tile<T, HD>(kbuf(st), k_g + (long long)kv0 * kv_stride, kv_stride, valid);
    if (with_v) pf_load_tile<T, HD>(vbuf(st), v_g + (long long)kv0 * kv_stride, kv_stride, valid);
    cp_async_commit();
  };

  // Q tile (rows beyond the sequence are zero-filled)
  pf_load_tile<T, HD>(q_s, q_g, q_stride, min(kPfQ, len - q0));
  cp_async_commit();
  issue_tile(0, 0, false);

  float* s_w = s_all + (size_t)warp * 16 * SLD;
  T* p_w = p_all + (size_t)warp * 16 * SLD;
  // row statistics: lanes (2r, 2r+1) own row r of this warp's 16 rows; each covers 32 of the 64 columns
  const int r_loc = lane >> 1, c_half = lane & 1;
  const int row_g = q0 + warp * 16 + r_loc;             // query index inside the sequence
  float m_run = -INFINITY, l_run = 0.f;
  const float sl2 = scale * 1.4426950408889634f;        // scores are used as s * scale * log2(e) inside exp2f

  wmma::fragment<wmma::matrix_a, 16, 16, 16, T, wmma::row_major> qf[HD / 16];

  // ------------------------------- pass 1: row max and row sum -------------------------------
  for (int j = 0; j < n_tiles; ++j) {
    const int st = j & 1;
    if (j + 1 < n_tiles) issue_tile(j + 1, st ^ 1, false);
    if (j + 1 < n_tiles) cp_async_wait<1>(); else cp_async_wait<0>();
    __syncthreads();
    if (j == 0) {
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) wmma::load_matrix_sync(qf[kk], q_s + (size_t)warp * 16 * LD + kk * 16, LD);
    }
    const int kv0 = j * kPfKV;
    if (kv0 <= q0 + warp * 16 + 15) {                   // warp-uniform: tile intersects this warp's causal range
#pragma unroll
      for (int nt = 0; nt < kPfKV / 16; ++nt) {
        wmma::fragment<wmma::accumulator, 16, 16, 16, float> sf;
        wmma::fill_fragment(sf, 0.f);
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
          wmma::fragment<wmma::matrix_b, 16, 16, 16, T, wmma::col_major> kf;
          wmma::load_matrix_sync(kf, kbuf(st) + (size_t)nt * 16 * LD + kk * 16, LD);
          wmma::mma_sync(sf, qf[kk], kf, sf);
        }
        wmma::store_matrix_sync(s_w + nt * 16, sf, SLD, wmma::mem_row_major);
      }
      __syncwarp();
      float mx = -INFINITY;
      for (int c = 0; c < 32; ++c) {
        const int col = c_half * 32 + c;
        const float s = (kv0 + col <= row_g) ? s_w[r_loc * SLD + col] : -INFINITY;
        mx = fmaxf(mx, s);
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      const float m_new = fmaxf(m_run, mx);
      float sum = 0.f;
      if (m_new > -INFINITY) {
        for (int c = 0; c < 32; ++c) {
          const int col = c_half * 32 + c;
          if (kv0 + col <= row_g) sum += exp2f((s_w[r_loc * SLD + col] - m_new) * sl2);
        }
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      l_run = (m_run > -INFINITY ? l_run * exp2f((m_run - m_new) * sl2) : 0.f) + sum;
      m_run = m_new;
      __syncwarp();
    }
    __syncthreads();
  }

  // ------------------------------- pass 2: O = sum exp(s - m) V -------------------------------
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> of[HD / 16];
#pragma unroll
  for (int i = 0; i < HD / 16; ++i) wmma::fill_fragment(of[i], 0.f);
  issue_tile(0, 0, true);
  for (int j = 0; j < n_tiles; ++j) {
    const int st = j & 1;
    if (j + 1 < n_tiles) issue_tile(j + 1, st ^ 1, true);
    if (j + 1 < n_tiles) cp_async_wait<1>(); else cp_async_wait<0>();
    __syncthreads();
    const int kv0 = j * kPfKV;
    if (kv0 <= q0 + warp * 16 + 15) {
#pragma unroll
      for (int nt = 0; nt < kPfKV / 16; ++nt) {
        wmma::fragment<wmma::accumulator, 16, 16, 16, float> sf;
        wmma::fill_fragment(sf, 0.f);
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
          wmma::fragment<wmma::matrix_b, 16, 16, 16, T, wmma::col_major> kf;
          wmma::load_matrix_sync(kf, kbuf(st) + (size_t)nt * 16 * LD + kk * 16, LD);
          wmma::mma_sync(sf, qf[kk], kf, sf);
        }
        wmma::store_matrix_sync(s_w + nt * 16, sf, SLD, wmma::mem_row_major);
      }
      __syncwarp();
      for (int c = 0; c < 32; ++c) {
        const int col = c_half * 32 + c;
        float p = 0.f;
        if (kv0 + col <= row_g && m_run > -INFINITY) p = exp2f((s_w[r_loc * SLD + col] - m_run) * sl2);
        p_w[r_loc * SLD + col] = DT<T>::from_f(p);
      }
      __syncwarp();
#pragma unroll
      for (int kt = 0; kt < kPfKV / 16; ++kt) {
        wmma::fragment<wmma::matrix_a, 16, 16, 16, T, wmma::row_major> pf;
        wmma::load_matrix_sync(pf, p_w + kt * 16, SLD);
#pragma unroll
        for (int dn = 0; dn < HD / 16; ++dn) {
          wmma::fragment<wmma::matrix_b, 16, 16, 16, T, wmma::row_major> vf;
          wmma::load_matrix_sync(vf, vbuf(st) + (size_t)kt * 16 * LD + dn * 16, LD);
          wmma::mma_sync(of[dn], pf, vf, of[dn]);
        }
      }
      __syncwarp();
    }
    __syncthreads();
  }

  // ------------------------------- epilogue: O / l -> out -------------------------------
  // stage this warp's 16 x HD fp32 block through shared memory (the KV ring is free now)
  float* o_w = reinterpret_cast<float*>(pf_smem + SM::q_bytes) + (size_t)warp * 16 * (HD + 8);
#pragma unroll
  for (int dn = 0; dn < HD / 16; ++dn) wmma::store_matrix_sync(o_w + dn * 16, of[dn], HD + 8, wmma::mem_row_major);
  __syncwarp();
  if (row_g < len) {
    const float inv = l_run > 0.f ? 1.0f / l_run : 0.f;
    T* o_g = out + ((long long)seq0 + row_g) * q_stride + (long long)head * HD;
    for (int c = 0; c < HD / 2; c += 8) {
      const int col = c_half * (HD / 2) + c;
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = o_w[r_loc * (HD + 8) + col + e] * inv;
      *reinterpret_cast<uint4*>(o_g + col) = pack8<T>(f);
    }
    if constexpr (LSE) {
      if (c_half == 0) lse[((long long)seq0 + row_g) * nh + head] = l_run > 0.f ? m_run * scale + logf(l_run) : -INFINITY;
    }
  }
}

// ================================================================================================
// prefill on wgmma (head_dim 128): one CTA = 64 query rows of one (sequence, head).  Warp 4 streams Q once and the K/V tiles
// of the causal range through a two-stage TMA ring (128-byte swizzle, two 64-column halves per 128-wide row); warps 0..3 are
// one warpgroup that computes S[64 x 64] = Q K^T with wgmma (both operands K-major in shared memory), runs the online softmax
// on the S registers (thread = two query rows, a quad of lanes shares a row), and accumulates O[64 x 128] += P V with P fed
// straight from registers as the A operand and V as the MN-major B operand.  S and O never leave the registers; the epilogue
// writes O / l (and the log-sum-exp for the backward).
// ================================================================================================
constexpr int kWgQ = 64, kWgKV = 64, kWgStages = 2, kWgThreads = 160;
template <typename T> __device__ __forceinline__ uint32_t pack2(float lo, float hi);   // defined with the decode kernel below
constexpr int kWgHalf = 64 * 128;                         // one [64 rows x 128 B] swizzled half of a Q, K or V tile (8 KiB)
constexpr int kWgStageBytes = 4 * kWgHalf;                // K and V tile
constexpr int kWgSmem = 2 * kWgHalf + kWgStages * kWgStageBytes;

template <typename T, bool LSE>
__global__ void __launch_bounds__(kWgThreads, 2)
attn_prefill_wgmma_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                          const __grid_constant__ CUtensorMap tm_v, const int* __restrict__ cu_seqlens, int nh, int nkv, float scale,
                          T* __restrict__ out, float* __restrict__ lse) {
  extern __shared__ uint8_t wg_raw[];
  __shared__ uint64_t q_bar, full_bar[kWgStages], empty_bar[kWgStages];
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;
  const uint32_t raw = smem_u32(wg_raw);
  uint8_t* smem = wg_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* q_s = smem;                                   // [2 halves][64 rows x 128 B]
  uint8_t* kv_s = smem + 2 * kWgHalf;                    // [stage][K half 0 | K half 1 | V half 0 | V half 1]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / (nh / nkv);

  pdl_trigger();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q); tma_prefetch_desc(&tm_k); tma_prefetch_desc(&tm_v);
    mbar_init(&q_bar, 1);
    for (int s = 0; s < kWgStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();                                            // Q / K / V / cu_seqlens come from the predecessors
  const int seq0 = cu_seqlens[b], len = cu_seqlens[b + 1] - seq0;
  const int q0 = qt * kWgQ;
  if (q0 >= len) return;                                 // CTA-uniform; nothing was issued yet
  const int kv_end = min(len, q0 + kWgQ);                // causal: keys 0 .. q0 + 63
  const int ntiles = (kv_end + kWgKV - 1) / kWgKV;

  if (warp == 4) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      mbar_expect_tx(&q_bar, 2u * kWgHalf);
      tma_load_2d(q_s, &tm_q, &q_bar, head * 128, seq0 + q0, CTS_L2_EVICT_FIRST);
      tma_load_2d(q_s + kWgHalf, &tm_q, &q_bar, head * 128 + 64, seq0 + q0, CTS_L2_EVICT_FIRST);
      for (int j = 0; j < ntiles; ++j) {
        const int s = j % kWgStages;
        mbar_wait(&empty_bar[s], ((uint32_t)(j / kWgStages) & 1u) ^ 1u);
        mbar_expect_tx(&full_bar[s], (uint32_t)kWgStageBytes);
        uint8_t* st = kv_s + (size_t)s * kWgStageBytes;
        const int row = seq0 + j * kWgKV;
        tma_load_2d(st, &tm_k, &full_bar[s], kvh * 128, row, CTS_L2_EVICT_LAST);
        tma_load_2d(st + kWgHalf, &tm_k, &full_bar[s], kvh * 128 + 64, row, CTS_L2_EVICT_LAST);
        tma_load_2d(st + 2 * kWgHalf, &tm_v, &full_bar[s], kvh * 128, row, CTS_L2_EVICT_LAST);
        tma_load_2d(st + 3 * kWgHalf, &tm_v, &full_bar[s], kvh * 128 + 64, row, CTS_L2_EVICT_LAST);
      }
    }
    return;
  }
  if (warp > 4) return;

  // ------------------------------ MMA + softmax warpgroup ------------------------------
  const float sl2 = scale * 1.4426950408889634f;         // softmax in log2 units
  const int r0 = q0 + acc_row(0), r1 = r0 + 8;           // this thread's two query rows (sequence positions)
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(q_s);
  mbar_wait(&q_bar, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int s = j % kWgStages;
    mbar_wait(&full_bar[s], (uint32_t)(j / kWgStages) & 1u);
    const uint32_t k_addr = smem_u32(kv_s + (size_t)s * kWgStageBytes), v_addr = k_addr + 2 * kWgHalf;
    float sc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) wgmma_fence_operand(sc[i]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {                     // head_dim 128 = two 64-wide halves x four k16 steps
      const uint32_t off = (uint32_t)(kk >> 2) * kWgHalf;
      wgmma_m64k16<64, kIsBf16>(sc, gmma_desc_k_sw128(q_addr + off) + 2 * (kk & 3), gmma_desc_k_sw128(k_addr + off) + 2 * (kk & 3), kk > 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 32; ++i) wgmma_fence_operand(sc[i]);
    // causal + length mask, scale, row maxima (a row lives in the 4 lanes of a quad)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int h = (i >> 1) & 1, row = h ? r1 : r0, col = j * kWgKV + acc_col(i);
      const float v = (col > row || col >= len) ? -INFINITY : sc[i] * sl2;
      sc[i] = v;
      mx[h] = fmaxf(mx[h], v);
    }
    float corr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_run[h], mx[h]);
      corr[h] = m_new == -INFINITY ? 1.f : exp2f(m_run[h] - m_new);
      m_run[h] = m_new;
    }
    float sum[2] = {0.f, 0.f};
    uint32_t a[4][4];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      const float p0 = m_run[h] == -INFINITY ? 0.f : exp2f(sc[i] - m_run[h]);
      const float p1 = m_run[h] == -INFINITY ? 0.f : exp2f(sc[i + 1] - m_run[h]);
      sum[h] += p0 + p1;
      a[i >> 3][(i >> 1) & 3] = pack2<T>(p0, p1);       // i = 8 kk + 2 e: register e of the k-step kk fragment
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
      sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
      l_run[h] = l_run[h] * corr[h] + sum[h];
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] *= corr[(i >> 1) & 1];
#pragma unroll
    for (int i = 0; i < 64; ++i) wgmma_fence_operand(o[i]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)                       // 16 keys per step: V rows kk*16.., both 64-wide halves of head_dim
      wgmma_m64n128k16_rs_tb<kIsBf16>(o, a[kk], gmma_desc_sw128(v_addr + (uint32_t)kk * 16 * 128, kWgHalf, 1024));
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 64; ++i) wgmma_fence_operand(o[i]);
    if (threadIdx.x == 0) mbar_arrive(&empty_bar[s]);   // the warpgroup's MMAs of this stage are complete
  }
  // ------------------------------ epilogue: O / l ------------------------------
  const long long ld = (long long)nh * 128;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = h ? r1 : r0;
    if (row >= len) continue;
    const float inv = l_run[h] > 0.f ? 1.f / l_run[h] : 0.f;
    T* orow = out + (long long)(seq0 + row) * ld + head * 128;
#pragma unroll
    for (int i = 2 * h; i < 64; i += 4)                  // registers of row h: i with (i >> 1) & 1 == h, in pairs of columns
      *reinterpret_cast<uint32_t*>(orow + acc_col(i)) = pack2<T>(o[i] * inv, o[i + 1] * inv);
    if constexpr (LSE) {
      if ((lane & 3) == 0)
        lse[(long long)(seq0 + row) * nh + head] = l_run[h] > 0.f ? m_run[h] * 0.6931471805599453f + logf(l_run[h]) : -INFINITY;
    }
  }
}

// ================================================================================================
// decode: tensor-core flash-decoding over TMA-staged, 128B-swizzled KV pages
// ================================================================================================
// grid (num_splits, nkv, batch); 5 warps: warps 0..3 consume (each owns 16 of the 64 tokens of a tile and runs its
// own online softmax, merged once at the end), warp 4 is the TMA producer.  A tile = 64 tokens = 64/page_size pages;
// every page of the cache is [page_size rows x head_dim] contiguous, fetched as head_dim/64 boxes of
// [page_size x 128 B] with the 128-byte swizzle so that ldmatrix reads are bank-conflict free.
//   S[16 x 16] = Q[16(heads, G valid) x d] K^T   mma.sync m16n8k16, K via ldmatrix
//   O[16 x d] += P[16 x 16] V                    V via ldmatrix.trans
// The tensor cores are used to cut instruction count, not for FLOPs: the kernel is bound by the KV stream
// (GQA intensity nh/nkv flop per byte).  The last CTA of a (sequence, kv head) to finish merges the split partials
// (self-resetting counter), so there is no separate combine launch.
constexpr int kDecConsumers = 128;
constexpr int kDecThreads = 160;
constexpr int kDecStages = 3;
constexpr int kDecTile = 64;
constexpr int kDecMaxPagesSm = 256;   // page ids a CTA keeps in shared memory (tiles x pages per tile; beyond that: global reads)
constexpr int kMaxGroup = 8;    // q heads per kv head (rows 8..15 of the MMA tile are padding)

__host__ __device__ inline long long dec_ws_stride(int hd) { return hd + 2; }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
template <typename T> __device__ __forceinline__ void mma16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                               uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void mma16816<__nv_bfloat16>(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                                     uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void mma16816<__half>(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                              uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
template <typename T> __device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  T v[2] = {DT<T>::from_f(lo), DT<T>::from_f(hi)};
  return *reinterpret_cast<uint32_t*>(v);
}

template <typename T, int HD>
__global__ void __launch_bounds__(kDecThreads)
attn_decode_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v, const T* __restrict__ q,
                   const int* __restrict__ page_table, int max_pages, const int* __restrict__ seq_lens, int nh, int nkv,
                   int page_size, float scale, int num_splits, float* __restrict__ ws, int* __restrict__ counters,
                   T* __restrict__ out) {
  constexpr int NHALF = HD / 64;                 // 128-byte column blocks per row
  constexpr int KSTEPS = HD / 16;
  constexpr int HALF_BYTES = kDecTile * 128;     // one [64 rows x 128 B] swizzled block
  constexpr int TILE_BYTES = NHALF * HALF_BYTES; // K (or V) tile
  extern __shared__ uint8_t dec_raw[];
  __shared__ uint64_t full_bar[kDecStages];
  __shared__ uint64_t empty_bar[kDecStages];
  __shared__ int is_last_s;
  const uint32_t raw = smem_u32(dec_raw);
  uint8_t* smem = dec_raw + (((raw + 1023u) & ~1023u) - raw);      // [stage][K tile | V tile]

  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int G = nh / nkv;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  pdl_trigger();
  if (tid == 0) {
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    for (int s = 0; s < kDecStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kDecConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_ATTN_DECODE, 0);

  // seq_lens / page_table are STEP STATE: written by the advance kernel at the end of the previous step (or by the host before
  // the step) and by nobody inside a step, whose first kernel (embed_gather) waits for everything before it BEFORE it lets its
  // successors start -- so they may be read ahead of the dependency wait.  So may every KV row of an earlier position: the
  // predecessor (RoPE / KV write of THIS layer) writes only row seq_len - 1.
  const int seq_len = seq_lens[b];
  const int n_tiles = (seq_len + kDecTile - 1) / kDecTile;
  const int tps = (n_tiles + num_splits - 1) / num_splits;
  const int tl0 = split * tps, tl1 = min(n_tiles, tl0 + tps);
  const int ntl = max(tl1 - tl0, 0);
  const int npp = kDecTile / page_size;          // pages per tile
  const int t_new = (seq_len - 1) / kDecTile;    // the tile that holds the row written by the predecessor
  // page ids of this CTA's tiles, fetched once by the producer warp (one L2 round trip instead of one per tile inside the ring loop)
  __shared__ int pg_s[kDecMaxPagesSm];
  int n_pre = 0;                                 // tiles whose loads were issued before the dependency wait
  if (warp == kDecConsumers / 32) {
    const int n_pg = min(ntl * npp, kDecMaxPagesSm);
    for (int i = lane; i < n_pg; i += 32) {
      int pg = tl0 * npp + i;
      pg = pg < max_pages ? pg : max_pages - 1;
      pg_s[i] = page_table[(long long)b * max_pages + pg];
    }
    __syncwarp();
    if (lane == 0) {
      for (int it = 0; it < ntl && it < kDecStages && tl0 + it < t_new; ++it) {       // stage it is free: first use of the ring
        mbar_expect_tx(&full_bar[it], (uint32_t)(2 * TILE_BYTES));
        uint8_t* ks = smem + (size_t)it * 2 * TILE_BYTES;
        uint8_t* vs = ks + TILE_BYTES;
        for (int j = 0; j < npp; ++j) {
          const int row0 = (pg_s[it * npp + j] * nkv + kvh) * page_size;
#pragma unroll
          for (int h = 0; h < NHALF; ++h) {
            tma_load_2d(ks + h * HALF_BYTES + j * page_size * 128, &tm_k, &full_bar[it], h * 64, row0, CTS_L2_EVICT_FIRST);
            tma_load_2d(vs + h * HALF_BYTES + j * page_size * 128, &tm_v, &full_bar[it], h * 64, row0, CTS_L2_EVICT_FIRST);
          }
        }
        n_pre = it + 1;
      }
    }
  }
  pdl_wait();          // q and the freshly written KV row come from the predecessor; the split workspace from the previous launch
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_ATTN_DECODE, 1);

  // accumulators of this warp (rows g = lane/4 are real heads when g < G)
  const int g = lane >> 2, tq = lane & 3;
  float oacc[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f;
  float m_run = -INFINITY, l_run = 0.f;

  if (warp == kDecConsumers / 32) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      for (int it = n_pre; it < ntl; ++it) {
        const int s = it % kDecStages;
        const uint32_t ph = (uint32_t)(it / kDecStages) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        mbar_expect_tx(&full_bar[s], (uint32_t)(2 * TILE_BYTES));
        uint8_t* ks = smem + (size_t)s * 2 * TILE_BYTES;
        uint8_t* vs = ks + TILE_BYTES;
        for (int j = 0; j < npp; ++j) {
          int page;
          if (it * npp + j < kDecMaxPagesSm) {
            page = pg_s[it * npp + j];
          } else {
            int pg = (tl0 + it) * npp + j;
            pg = pg < max_pages ? pg : max_pages - 1;        // pages past the sequence are masked; keep the read in bounds
            page = page_table[(long long)b * max_pages + pg];
          }
          const int row0 = (page * nkv + kvh) * page_size;
#pragma unroll
          for (int h = 0; h < NHALF; ++h) {
            tma_load_2d(ks + h * HALF_BYTES + j * page_size * 128, &tm_k, &full_bar[s], h * 64, row0, CTS_L2_EVICT_FIRST);
            tma_load_2d(vs + h * HALF_BYTES + j * page_size * 128, &tm_v, &full_bar[s], h * 64, row0, CTS_L2_EVICT_FIRST);
          }
        }
      }
    }
  } else {
    // ------------------------------ consumers ------------------------------
    // Q as the A operand: row g = head, the padding rows (g+8) are zero
    uint32_t qa[KSTEPS][2];
    {
      const T* qrow = q + ((long long)b * nh + (long long)kvh * G + (g < G ? g : 0)) * HD;
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        qa[kk][0] = g < G ? *reinterpret_cast<const uint32_t*>(qrow + kk * 16 + tq * 2) : 0u;
        qa[kk][1] = g < G ? *reinterpret_cast<const uint32_t*>(qrow + kk * 16 + 8 + tq * 2) : 0u;
      }
    }
    const float sl2 = scale * 1.4426950408889634f;
    const int lm = lane >> 3, lr = lane & 7;       // ldmatrix: this lane supplies row lr of matrix lm
    for (int it = 0; it < ntl; ++it) {
      const int s = it % kDecStages;
      mbar_wait(&full_bar[s], (uint32_t)(it / kDecStages) & 1u);
      const uint32_t kbase = smem_u32(smem + (size_t)s * 2 * TILE_BYTES);
      const uint32_t vbase = kbase + TILE_BYTES;
      // ---- S = Q K^T for this warp's 16 tokens (2 n-tiles of 8)
      float sacc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        const int row = warp * 16 + (lm >> 1) * 8 + lr;          // matrices: (nt0,k0-7) (nt0,k8-15) (nt1,k0-7) (nt1,k8-15)
        const int chunk = (kk & 3) * 2 + (lm & 1);
        uint32_t bf[4];
        ldsm_x4(kbase + (kk >> 2) * HALF_BYTES + row * 128 + ((chunk ^ (row & 7)) << 4), bf);
        mma16816<T>(sacc[0], qa[kk][0], 0u, qa[kk][1], 0u, bf[0], bf[1]);
        mma16816<T>(sacc[1], qa[kk][0], 0u, qa[kk][1], 0u, bf[2], bf[3]);
      }
      // ---- online softmax on row g (values of a row live in the 4 lanes of a quad)
      const int tok0 = (tl0 + it) * kDecTile + warp * 16 + tq * 2;
      float sv[2][2];
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const bool valid = tok0 + nt * 8 + j < seq_len;
          sv[nt][j] = valid ? sacc[nt][j] * sl2 : -INFINITY;
          mx = fmaxf(mx, sv[nt][j]);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run, mx);
      float alpha = 1.f, p[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
      if (m_new > -INFINITY) {
        alpha = m_run > -INFINITY ? exp2f(m_run - m_new) : 0.f;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int j = 0; j < 2; ++j) p[nt][j] = exp2f(sv[nt][j] - m_new);      // exp2(-inf) = 0 for masked tokens
      }
      float ps = p[0][0] + p[0][1] + p[1][0] + p[1][1];
      ps += __shfl_xor_sync(0xffffffffu, ps, 1);
      ps += __shfl_xor_sync(0xffffffffu, ps, 2);
      l_run = l_run * alpha + ps;
      m_run = m_new;
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) { oacc[i][0] *= alpha; oacc[i][1] *= alpha; }
      // ---- O += P V ; P (row g x 16 tokens) is the A operand straight from the S accumulator layout
      const uint32_t pa0 = pack2<T>(p[0][0], p[0][1]), pa2 = pack2<T>(p[1][0], p[1][1]);
#pragma unroll
      for (int dp = 0; dp < HD / 16; ++dp) {
        const int row = warp * 16 + (lm & 1) * 8 + lr;           // matrices: (tok0-7,dn) (tok8-15,dn) (tok0-7,dn+1) (tok8-15,dn+1)
        const int chunk = 2 * dp + (lm >> 1);
        uint32_t bf[4];
        ldsm_x4_trans(vbase + (chunk >> 3) * HALF_BYTES + row * 128 + (((chunk & 7) ^ (row & 7)) << 4), bf);
        mma16816<T>(oacc[2 * dp], pa0, 0u, pa2, 0u, bf[0], bf[1]);
        mma16816<T>(oacc[2 * dp + 1], pa0, 0u, pa2, 0u, bf[2], bf[3]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    }
  }
  __syncthreads();     // every tile consumed: the ring can be reused as merge scratch

  // ---- merge the 4 consumer warps (disjoint token subsets) -> this split's (m, l, o)
  float* m_sm = reinterpret_cast<float*>(smem);                 // [4][8]
  float* l_sm = m_sm + 32;                                      // [4][8]
  float* o_sm = l_sm + 32;                                      // [4][8][HD]
  if (warp < kDecConsumers / 32 && g < G) {
    if (tq == 0) { m_sm[warp * 8 + g] = m_run; l_sm[warp * 8 + g] = l_run; }
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      o_sm[(warp * 8 + g) * HD + i * 8 + tq * 2] = oacc[i][0];
      o_sm[(warp * 8 + g) * HD + i * 8 + tq * 2 + 1] = oacc[i][1];
    }
  }
  __syncthreads();
  const long long wstride = dec_ws_stride(HD);
  const long long head0 = (long long)b * nh + (long long)kvh * G;
  for (int i = tid; i < G * HD; i += kDecThreads) {
    const int gg = i / HD, d = i % HD;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < 4; ++w) M = fmaxf(M, m_sm[w * 8 + gg]);
    float L = 0.f, O = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float mw = m_sm[w * 8 + gg];
      const float f = mw > -INFINITY ? exp2f(mw - M) : 0.f;
      L += l_sm[w * 8 + gg] * f;
      O += o_sm[(w * 8 + gg) * HD + d] * f;
    }
    if (num_splits == 1) {
      out[(head0 + gg) * HD + d] = DT<T>::from_f(L > 0.f ? O / L : 0.f);
    } else {
      float* w = ws + ((head0 + gg) * num_splits + split) * wstride;
      w[2 + d] = O;
      if (d == 0) { w[0] = M; w[1] = L; }
    }
  }
  if (num_splits == 1) return;
  // ---- the last split of this (sequence, kv head) to arrive merges all partials
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int prev = atomicAdd(&counters[b * nkv + kvh], 1);
    is_last_s = prev == num_splits - 1;
  }
  __syncthreads();
  if (!is_last_s) return;
  __threadfence();
  for (int i = tid; i < G * HD; i += kDecThreads) {
    const int gg = i / HD, d = i % HD;
    const float* w = ws + (head0 + gg) * num_splits * wstride;
    // all loads of a batch of splits are issued before the first use: a run-time-bounded loop of dependent uses costs one L2 round
    // trip per split (16 splits at b = 1: ~20 us of pure latency, measured with csrc/trace.cuh).  Same arithmetic, same order.
    constexpr int kMB = 8;
    float M = -INFINITY;
    for (int s0 = 0; s0 < num_splits; s0 += kMB) {
      float mv[kMB];
#pragma unroll
      for (int u = 0; u < kMB; ++u) mv[u] = s0 + u < num_splits ? __ldcg(w + (s0 + u) * wstride) : -INFINITY;
#pragma unroll
      for (int u = 0; u < kMB; ++u) M = fmaxf(M, mv[u]);
    }
    float L = 0.f, O = 0.f;
    for (int s0 = 0; s0 < num_splits; s0 += kMB) {
      float mv[kMB], lv[kMB], ov[kMB];
#pragma unroll
      for (int u = 0; u < kMB; ++u) {
        const bool ok = s0 + u < num_splits;
        mv[u] = ok ? __ldcg(w + (s0 + u) * wstride) : -INFINITY;
        lv[u] = ok ? __ldcg(w + (s0 + u) * wstride + 1) : 0.f;
        ov[u] = ok ? __ldcg(w + (s0 + u) * wstride + 2 + d) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kMB; ++u)
        if (s0 + u < num_splits) {
          const float f = mv[u] > -INFINITY ? exp2f(mv[u] - M) : 0.f;
          L += lv[u] * f;
          O += ov[u] * f;
        }
    }
    out[(head0 + gg) * HD + d] = DT<T>::from_f(L > 0.f ? O / L : 0.f);
  }
  if (tid == 0) counters[b * nkv + kvh] = 0;       // self-resetting for the next launch
}

}  // namespace

static int attn_prefill_impl(cts_ctx* ctx, const void* q, const void* k, const void* v, const int* cu_seqlens, int batch,
                             int max_seqlen, long long total_tokens_hint, int nh, int nkv, int head_dim, float scale, void* out,
                             float* lse, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, q && k && v && cu_seqlens && out, "null pointer");
  CTS_CHECK_ARG(ctx, nh > 0 && nkv > 0 && nh % nkv == 0, "nh must be a positive multiple of nkv");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (head_dim != 64 && head_dim != 128) return cts_set_error(ctx, CTS_ERR_UNSUPPORTED, "cts_attn_prefill: head_dim %d (64 or 128)", head_dim);
  if (batch == 0 || max_seqlen == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, batch <= 65535 && nh <= 65535, "grid");
  cudaStream_t st = (cudaStream_t)stream;
  if (head_dim == 128) {
    // wgmma path: Q/K/V through TMA tensor maps over the packed [tokens, heads*128] activations
    const long long total_tokens = total_tokens_hint > 0 ? total_tokens_hint : (long long)batch * max_seqlen;
    CUtensorMap tm_q, tm_k, tm_v;
    int rc = cts_make_tmap_2d(ctx, &tm_q, q, total_tokens, (long long)nh * 128, (long long)nh * 128, kWgQ, dtype == CTS_BF16);
    if (rc) return rc;
    rc = cts_make_tmap_2d(ctx, &tm_k, k, total_tokens, (long long)nkv * 128, (long long)nkv * 128, kWgKV, dtype == CTS_BF16);
    if (rc) return rc;
    rc = cts_make_tmap_2d(ctx, &tm_v, v, total_tokens, (long long)nkv * 128, (long long)nkv * 128, kWgKV, dtype == CTS_BF16);
    if (rc) return rc;
    dim3 gw((unsigned)((max_seqlen + kWgQ - 1) / kWgQ), (unsigned)nh, (unsigned)batch);
    const size_t smem_w = (size_t)kWgSmem + 1024;
#define WG_LAUNCH(TT, LSEV)                                                                                  \
  {                                                                                                          \
    auto kern = attn_prefill_wgmma_kernel<TT, LSEV>;                                                         \
    CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_w));     \
    CTS_CUDA(ctx, launch_pdl(kern, gw, dim3(kWgThreads), smem_w, st, 1, tm_q, tm_k, tm_v, cu_seqlens, nh, nkv, scale, (TT*)out, lse)); \
  }
    if (dtype == CTS_BF16) {
      if (lse) WG_LAUNCH(__nv_bfloat16, true) else WG_LAUNCH(__nv_bfloat16, false)
    } else {
      if (lse) WG_LAUNCH(__half, true) else WG_LAUNCH(__half, false)
    }
#undef WG_LAUNCH
    return CTS_OK;
  }
  dim3 grid((unsigned)((max_seqlen + kPfQ - 1) / kPfQ), (unsigned)nh, (unsigned)batch);
#define PF_LAUNCH2(TT, HDV, LSEV)                                                                            \
  {                                                                                                          \
    auto kern = attn_prefill_kernel<TT, HDV, LSEV>;                                                          \
    const size_t smem = PfSmem<HDV>::total;                                                                  \
    CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));       \
    CTS_CUDA(ctx, launch_pdl(kern, grid, dim3(kPfThreads), smem, st, 1, (const TT*)q, (const TT*)k, (const TT*)v, cu_seqlens, nh, nkv, \
                             scale, (TT*)out, lse));                                                         \
  }
#define PF_LAUNCH(TT, HDV) { if (lse) PF_LAUNCH2(TT, HDV, true) else PF_LAUNCH2(TT, HDV, false) }
  if (dtype == CTS_BF16) {
    if (head_dim == 128) PF_LAUNCH(__nv_bfloat16, 128) else PF_LAUNCH(__nv_bfloat16, 64)
  } else {
    if (head_dim == 128) PF_LAUNCH(__half, 128) else PF_LAUNCH(__half, 64)
  }
#undef PF_LAUNCH
#undef PF_LAUNCH2
  CTS_LAUNCH_CHECK(ctx);
  return CTS_OK;
}

extern "C" int cts_attn_prefill(cts_ctx* ctx, const void* q, const void* k, const void* v, const int* cu_seqlens, int batch,
                                int max_seqlen, long long total_tokens_hint, int nh, int nkv, int head_dim, float scale, void* out,
                                int dtype, void* stream) {
  return attn_prefill_impl(ctx, q, k, v, cu_seqlens, batch, max_seqlen, total_tokens_hint, nh, nkv, head_dim, scale, out, nullptr,
                           dtype, stream);
}

// training forward: same kernels + the softmax statistics the backward needs (csrc/attention_bwd.cu)
extern "C" int cts_attn_prefill_lse(cts_ctx* ctx, const void* q, const void* k, const void* v, const int* cu_seqlens, int batch,
                                    int max_seqlen, long long total_tokens_hint, int nh, int nkv, int head_dim, float scale,
                                    void* out, float* lse, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, lse != nullptr, "null lse");
  return attn_prefill_impl(ctx, q, k, v, cu_seqlens, batch, max_seqlen, total_tokens_hint, nh, nkv, head_dim, scale, out, lse, dtype,
                           stream);
}

extern "C" long long cts_attn_decode_workspace_floats(int batch, int nh, int head_dim, int num_splits) {
  // fp32 partials [batch, nh, splits, head_dim + 2] followed by int32 arrival counters [batch * nh] (upper bound on
  // batch * nkv).  The caller zero-fills the buffer ONCE; the counters reset themselves after every launch.
  return (long long)batch * nh * num_splits * dec_ws_stride(head_dim) + (long long)batch * nh;
}

extern "C" int cts_attn_decode(cts_ctx* ctx, const void* q, const void* k_cache, const void* v_cache, int num_pages,
                               const int* page_table, int max_pages, const int* seq_lens, int batch, int nh, int nkv,
                               int head_dim, int page_size, float scale, int num_splits, float* workspace, void* out, int dtype,
                               void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, q && k_cache && v_cache && page_table && seq_lens && workspace && out, "null pointer");
  CTS_CHECK_ARG(ctx, nh > 0 && nkv > 0 && nh % nkv == 0 && nh / nkv <= kMaxGroup, "nh/nkv must be an integer <= 8");
  CTS_CHECK_ARG(ctx, page_size == 16 || page_size == 32 || page_size == 64, "page_size must be 16, 32 or 64");
  CTS_CHECK_ARG(ctx, num_splits >= 1 && num_splits <= 65535, "num_splits");
  CTS_CHECK_ARG(ctx, num_pages > 0 && max_pages > 0, "num_pages / max_pages");
  CTS_CHECK_ARG(ctx, (long long)num_pages * nkv * page_size < 2147483647LL, "KV cache too large for 32-bit TMA row coordinates");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (head_dim != 64 && head_dim != 128) return cts_set_error(ctx, CTS_ERR_UNSUPPORTED, "cts_attn_decode: head_dim %d (64 or 128)", head_dim);
  if (batch == 0) return CTS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = (long long)num_pages * nkv * page_size;
  CUtensorMap tm_k, tm_v;
  int rc = cts_make_tmap_2d(ctx, &tm_k, k_cache, rows, head_dim, head_dim, page_size, dtype == CTS_BF16);
  if (rc) return rc;
  rc = cts_make_tmap_2d(ctx, &tm_v, v_cache, rows, head_dim, head_dim, page_size, dtype == CTS_BF16);
  if (rc) return rc;
  int* counters = reinterpret_cast<int*>(workspace + (long long)batch * nh * num_splits * dec_ws_stride(head_dim));
  dim3 grid((unsigned)num_splits, (unsigned)nkv, (unsigned)batch);
  const size_t smem = (size_t)kDecStages * 2 * (head_dim / 64) * kDecTile * 128 + 1024;
#define DEC_LAUNCH(TT, HDV)                                                                                    \
  {                                                                                                            \
    auto kern = attn_decode_kernel<TT, HDV>;                                                                   \
    CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));         \
    CTS_CUDA(ctx, launch_pdl(kern, grid, dim3(kDecThreads), smem, st, 1, tm_k, tm_v, (const TT*)q, page_table, max_pages, seq_lens, \
                             nh, nkv, page_size, scale, num_splits, workspace, counters, (TT*)out));           \
  }
  if (dtype == CTS_BF16) {
    if (head_dim == 128) DEC_LAUNCH(__nv_bfloat16, 128) else DEC_LAUNCH(__nv_bfloat16, 64)
  } else {
    if (head_dim == 128) DEC_LAUNCH(__half, 128) else DEC_LAUNCH(__half, 64)
  }
#undef DEC_LAUNCH
  return CTS_OK;
}

CTS_TRACE_SETTER(cts_trace_set_attention)
