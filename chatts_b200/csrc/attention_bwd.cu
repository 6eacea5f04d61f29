// chatts_b200 -- backward of the causal GQA attention for the LoRA fine-tune step (SURVEY.md 8(a) row A9).
// Arithmetic: transformers qwen2/modeling_qwen2.py:161-184 (softmax(scale Q K^T) V, causal, repeat_kv) under autograd, in
// the FlashAttention-2 recomputation form -- nothing of size [S, S] is ever stored:
//     P  = exp(scale S - lse)            lse from the forward (cts_attn_prefill_lse)
//     dV = P^T dO        dP = dO V^T        delta_i = sum_d dO_id O_id
//     dS = P o (dP - delta)               dQ = scale dS K        dK = scale dS^T Q
// Three launches:  attn_bwd_delta_kernel (delta),  attn_bwd_dq_kernel (one CTA = 64 query rows of one head, loops over the
// causal KV tiles),  attn_bwd_dkv_kernel (one CTA = 64 KV rows of one kv head, loops over the q heads of the group and the
// query tiles at or below the diagonal; dK/dV of a kv head are summed over its q heads in registers -> no atomics, fixed
// summation order).  S / dP are recomputed in both kernels (2x QK^T-sized work) in exchange for determinism.
//
// HMMA through nvcuda::wmma (m16n16k16, fp32 accumulate), cp.async double buffering; no mbarrier / flag spin anywhere in this
// file.  head_dim 128 runs the wgmma kernels of attention_bwd_wgmma.cu by default; these kernels serve head_dim 64 and are the
// reference the wgmma kernels are tested against (CTS_ATTN_BWD_WGMMA=0).
#include <mma.h>
#include <stdlib.h>

#include "common.cuh"

// the kernel's dynamic shared memory as a byte array (one spelling, so that tests/cuda_on_cpu can supply its own; defined here and not
// in common.cuh so that the header the GPU-validated kernels were compiled with stays byte-identical)
#ifndef CTS_DYN_SMEM
#define CTS_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#endif

namespace {

using namespace nvcuda;

#ifdef CTS_HOST_SHIM      // tests/cuda_on_cpu: the asynchronous copy is a copy
__device__ __forceinline__ void bw_cp_async16(void* smem, const void* gmem, bool valid) {
  if (valid) memcpy(smem, gmem, 16); else memset(smem, 0, 16);
}
__device__ __forceinline__ void bw_cp_async_commit() {}
template <int N> __device__ __forceinline__ void bw_cp_async_wait() {}
#else
__device__ __forceinline__ void bw_cp_async16(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void bw_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bw_cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#endif

constexpr int kBwTile = 64;       // query rows per CTA (dq) / kv rows per CTA (dkv); also the tile of the streamed operand
constexpr int kBwThreads = 128;   // 4 warps x 16 rows
constexpr float kLog2e = 1.4426950408889634f;

template <int HD> struct BwSmem {
  static constexpr int LD = HD + 8;                                   // padded row, elements
  static constexpr int SLD = kBwTile + 8;                             // padded score row
  static constexpr size_t tile_bytes = (size_t)kBwTile * LD * 2;      // one [64 x HD] operand tile
  static constexpr size_t s_bytes = (size_t)4 * 16 * SLD * 4;         // per-warp 16 x 64 fp32
  static constexpr size_t p_bytes = (size_t)4 * 16 * SLD * 2;         // per-warp 16 x 64 model dtype
  static constexpr size_t stat_bytes = (size_t)2 * 2 * kBwTile * 4;   // [stage][lse|delta][64] fp32 (dkv kernel)
  // layout: A | B | ring[2 stages][2 tiles] | S | dP | P | stats
  static constexpr size_t off_ring = 2 * tile_bytes;
  static constexpr size_t off_s = off_ring + 4 * tile_bytes;
  static constexpr size_t off_dp = off_s + s_bytes;
  static constexpr size_t off_p = off_dp + s_bytes;
  static constexpr size_t off_stat = off_p + p_bytes;
  static constexpr size_t total = off_stat + stat_bytes;
  static constexpr size_t stage_floats = (size_t)16 * (HD + 8);       // per-warp fp32 staging of a 16 x HD block
};

// 64 rows x HD elements, 16 B per cp.async; rows >= rows_valid are zero-filled
template <typename T, int HD>
__device__ __forceinline__ void bw_load_tile(T* dst, const T* __restrict__ src, long long row_stride, int rows_valid) {
  constexpr int LD = BwSmem<HD>::LD;
  constexpr int CH = HD / 8;
  for (int i = threadIdx.x; i < kBwTile * CH; i += kBwThreads) {
    const int r = i / CH, c = i % CH;
    const bool ok = r < rows_valid;
    bw_cp_async16(dst + r * LD + c * 8, src + (ok ? (long long)r * row_stride + c * 8 : 0), ok);
  }
}

// ------------------------------------------------------------------------------------------------ delta = rowsum(dO o O)
template <typename T>
__global__ void __launch_bounds__(256)
attn_bwd_delta_kernel(const T* __restrict__ o, const T* __restrict__ d_o, float* __restrict__ delta, long long rows, int hd) {
  pdl_trigger();
  pdl_wait();
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);       // row = token * nh + head
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const T* a = o + row * hd;
  const T* b = d_o + row * hd;
  float s = 0.f;
  for (int c = lane * 2; c < hd; c += 64) s += DT<T>::to_f(a[c]) * DT<T>::to_f(b[c]) + DT<T>::to_f(a[c + 1]) * DT<T>::to_f(b[c + 1]);
  s = warp_sum(s);
  if (lane == 0) delta[row] = s;
}

// ------------------------------------------------------------------------------------------------ dQ
// grid (ceil(max_seqlen / 64), nh, batch).  Warp w owns query rows [16w, 16w + 16) of the tile.
template <typename T, int HD>
__global__ void __launch_bounds__(kBwThreads)
attn_bwd_dq_kernel(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, const T* __restrict__ d_o,
                   const float* __restrict__ lse, const float* __restrict__ delta, const int* __restrict__ cu_seqlens, int nh,
                   int nkv, float scale, T* __restrict__ dq) {
  using SM = BwSmem<HD>;
  constexpr int LD = SM::LD, SLD = SM::SLD;
  CTS_DYN_SMEM(bw_smem);
  T* q_s = reinterpret_cast<T*>(bw_smem);
  T* do_s = reinterpret_cast<T*>(bw_smem + SM::tile_bytes);
  T* ring = reinterpret_cast<T*>(bw_smem + SM::off_ring);                      // [2][K|V][64][LD]
  float* s_all = reinterpret_cast<float*>(bw_smem + SM::off_s);
  float* dp_all = reinterpret_cast<float*>(bw_smem + SM::off_dp);
  T* p_all = reinterpret_cast<T*>(bw_smem + SM::off_p);

  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.z, head = blockIdx.y, qt = blockIdx.x;
  const int seq0 = cu_seqlens[b], len = cu_seqlens[b + 1] - seq0;
  const int q0 = qt * kBwTile;
  if (q0 >= len) return;
  const int kvh = head / (nh / nkv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long q_stride = (long long)nh * HD, kv_stride = (long long)nkv * HD;
  const T* q_g = q + ((long long)seq0 + q0) * q_stride + (long long)head * HD;
  const T* do_g = d_o + ((long long)seq0 + q0) * q_stride + (long long)head * HD;
  const T* k_g = k + (long long)seq0 * kv_stride + (long long)kvh * HD;
  const T* v_g = v + (long long)seq0 * kv_stride + (long long)kvh * HD;
  const int n_tiles = (min(q0 + kBwTile, len) + kBwTile - 1) / kBwTile;       // causal: kv <= last query row of this CTA

  auto kbuf = [&](int st) { return ring + (size_t)st * 2 * kBwTile * LD; };
  auto vbuf = [&](int st) { return ring + (size_t)st * 2 * kBwTile * LD + (size_t)kBwTile * LD; };
  auto issue_tile = [&](int j, int st) {
    const int kv0 = j * kBwTile;
    const int valid = min(kBwTile, len - kv0);
    bw_load_tile<T, HD>(kbuf(st), k_g + (long long)kv0 * kv_stride, kv_stride, valid);
    bw_load_tile<T, HD>(vbuf(st), v_g + (long long)kv0 * kv_stride, kv_stride, valid);
    bw_cp_async_commit();
  };

  const int q_valid = min(kBwTile, len - q0);
  bw_load_tile<T, HD>(q_s, q_g, q_stride, q_valid);
  bw_load_tile<T, HD>(do_s, do_g, q_stride, q_valid);
  bw_cp_async_commit();
  issue_tile(0, 0);

  float* s_w = s_all + (size_t)warp * 16 * SLD;
  float* dp_w = dp_all + (size_t)warp * 16 * SLD;
  T* p_w = p_all + (size_t)warp * 16 * SLD;
  // lanes (2r, 2r+1) own row r of this warp's 16 rows; each covers 32 of the 64 columns
  const int r_loc = lane >> 1, c_half = lane & 1;
  const int row_g = q0 + warp * 16 + r_loc;
  const bool row_ok = row_g < len;
  const float lse2 = row_ok ? lse[((long long)seq0 + row_g) * nh + head] * kLog2e : 0.f;
  const float dlt = row_ok ? delta[((long long)seq0 + row_g) * nh + head] : 0.f;
  const float sl2 = scale * kLog2e;

  wmma::fragment<wmma::matrix_a, 16, 16, 16, T, wmma::row_major> qf[HD / 16], dof[HD / 16];
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc[HD / 16];
#pragma unroll
  for (int i = 0; i < HD / 16; ++i) wmma::fill_fragment(acc[i], 0.f);

  for (int j = 0; j < n_tiles; ++j) {
    const int st = j & 1;
    if (j + 1 < n_tiles) issue_tile(j + 1, st ^ 1);
    if (j + 1 < n_tiles) bw_cp_async_wait<1>(); else bw_cp_async_wait<0>();
    __syncthreads();
    if (j == 0) {
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        wmma::load_matrix_sync(qf[kk], q_s + (size_t)warp * 16 * LD + kk * 16, LD);
        wmma::load_matrix_sync(dof[kk], do_s + (size_t)warp * 16 * LD + kk * 16, LD);
      }
    }
    const int kv0 = j * kBwTile;
    if (kv0 <= q0 + warp * 16 + 15) {                      // warp-uniform: the tile intersects this warp's causal range
#pragma unroll
      for (int nt = 0; nt < kBwTile / 16; ++nt) {
        wmma::fragment<wmma::accumulator, 16, 16, 16, float> sf, df;
        wmma::fill_fragment(sf, 0.f);
        wmma::fill_fragment(df, 0.f);
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
          wmma::fragment<wmma::matrix_b, 16, 16, 16, T, wmma::col_major> bf;
          wmma::load_matrix_sync(bf, kbuf(st) + (size_t)nt * 16 * LD + kk * 16, LD);     // B[d][kv] = K[kv][d]
          wmma::mma_sync(sf, qf[kk], bf, sf);
          wmma::load_matrix_sync(bf, vbuf(st) + (size_t)nt * 16 * LD + kk * 16, LD);     // B[d][kv] = V[kv][d]
          wmma::mma_sync(df, dof[kk], bf, df);
        }
        wmma::store_matrix_sync(s_w + nt * 16, sf, SLD, wmma::mem_row_major);
        wmma::store_matrix_sync(dp_w + nt * 16, df, SLD, wmma::mem_row_major);
      }
      __syncwarp();
      for (int c = 0; c < 32; ++c) {
        const int col = c_half * 32 + c;
        float ds = 0.f;
        if (row_ok && kv0 + col <= row_g) {
          const float p = exp2f(s_w[r_loc * SLD + col] * sl2 - lse2);
          ds = p * (dp_w[r_loc * SLD + col] - dlt) * scale;
        }
        p_w[r_loc * SLD + col] = DT<T>::from_f(ds);
      }
      __syncwarp();
#pragma unroll
      for (int kt = 0; kt < kBwTile / 16; ++kt) {
        wmma::fragment<wmma::matrix_a, 16, 16, 16, T, wmma::row_major> af;
        wmma::load_matrix_sync(af, p_w + kt * 16, SLD);
#pragma unroll
        for (int dn = 0; dn < HD / 16; ++dn) {
          wmma::fragment<wmma::matrix_b, 16, 16, 16, T, wmma::row_major> bf;
          wmma::load_matrix_sync(bf, kbuf(st) + (size_t)kt * 16 * LD + dn * 16, LD);     // B[kv][d] = K[kv][d]
          wmma::mma_sync(acc[dn], af, bf, acc[dn]);
        }
      }
      __syncwarp();
    }
    __syncthreads();
  }

  // epilogue: this warp's 16 x HD fp32 block through shared memory (the KV ring is free after the last barrier)
  float* o_w = reinterpret_cast<float*>(bw_smem + SM::off_ring) + (size_t)warp * SM::stage_floats;
#pragma unroll
  for (int dn = 0; dn < HD / 16; ++dn) wmma::store_matrix_sync(o_w + dn * 16, acc[dn], HD + 8, wmma::mem_row_major);
  __syncwarp();
  if (row_ok) {
    T* o_g = dq + ((long long)seq0 + row_g) * q_stride + (long long)head * HD;
    for (int c = 0; c < HD / 2; c += 8) {
      const int col = c_half * (HD / 2) + c;
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = o_w[r_loc * (HD + 8) + col + e];
      *reinterpret_cast<uint4*>(o_g + col) = pack8<T>(f);
    }
  }
}

// ------------------------------------------------------------------------------------------------ dK, dV
// grid (ceil(max_seqlen / 64), nkv, batch).  Warp w owns kv rows [16w, 16w + 16) of the tile; the loop runs over
// (q head of the group, query tile >= the diagonal tile), Q / dO tiles double-buffered by cp.async.
template <typename T, int HD>
__global__ void __launch_bounds__(kBwThreads)
attn_bwd_dkv_kernel(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, const T* __restrict__ d_o,
                    const float* __restrict__ lse, const float* __restrict__ delta, const int* __restrict__ cu_seqlens, int nh,
                    int nkv, float scale, T* __restrict__ dk, T* __restrict__ dv) {
  using SM = BwSmem<HD>;
  constexpr int LD = SM::LD, SLD = SM::SLD;
  CTS_DYN_SMEM(bw_smem);
  T* k_s = reinterpret_cast<T*>(bw_smem);
  T* v_s = reinterpret_cast<T*>(bw_smem + SM::tile_bytes);
  T* ring = reinterpret_cast<T*>(bw_smem + SM::off_ring);                      // [2][Q|dO][64][LD]
  float* s_all = reinterpret_cast<float*>(bw_smem + SM::off_s);
  float* dp_all = reinterpret_cast<float*>(bw_smem + SM::off_dp);
  T* p_all = reinterpret_cast<T*>(bw_smem + SM::off_p);
  float* stat = reinterpret_cast<float*>(bw_smem + SM::off_stat);              // [2][lse*log2e | delta][64]

  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.z, kvh = blockIdx.y, kt0 = blockIdx.x;
  const int seq0 = cu_seqlens[b], len = cu_seqlens[b + 1] - seq0;
  const int kv0 = kt0 * kBwTile;
  if (kv0 >= len) return;
  const int G = nh / nkv;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long q_stride = (long long)nh * HD, kv_stride = (long long)nkv * HD;
  const T* k_g = k + ((long long)seq0 + kv0) * kv_stride + (long long)kvh * HD;
  const T* v_g = v + ((long long)seq0 + kv0) * kv_stride + (long long)kvh * HD;
  const int nq = (len + kBwTile - 1) / kBwTile;            // query tiles of the sequence
  const int nI = nq - kt0;                                 // tiles at or below the diagonal (query tile index >= kt0)
  const int n_iter = G * nI;

  auto qbuf = [&](int st) { return ring + (size_t)st * 2 * kBwTile * LD; };
  auto dobuf = [&](int st) { return ring + (size_t)st * 2 * kBwTile * LD + (size_t)kBwTile * LD; };
  auto issue_tile = [&](int n, int st) {
    const int head = kvh * G + n / nI;
    const int q0 = (kt0 + n % nI) * kBwTile;
    const int valid = min(kBwTile, len - q0);
    const long long off = ((long long)seq0 + q0) * q_stride + (long long)head * HD;
    bw_load_tile<T, HD>(qbuf(st), q + off, q_stride, valid);
    bw_load_tile<T, HD>(dobuf(st), d_o + off, q_stride, valid);
    bw_cp_async_commit();
    if (threadIdx.x < kBwTile) {                           // the stage was last read before the previous barrier
      const int qi = q0 + threadIdx.x;
      const bool ok = qi < len;
      const long long sidx = ((long long)seq0 + (ok ? qi : 0)) * nh + head;
      stat[(size_t)st * 2 * kBwTile + threadIdx.x] = ok ? lse[sidx] * kLog2e : 0.f;
      stat[(size_t)st * 2 * kBwTile + kBwTile + threadIdx.x] = ok ? delta[sidx] : 0.f;
    }
  };

  const int kv_valid = min(kBwTile, len - kv0);
  bw_load_tile<T, HD>(k_s, k_g, kv_stride, kv_valid);
  bw_load_tile<T, HD>(v_s, v_g, kv_stride, kv_valid);
  bw_cp_async_commit();
  issue_tile(0, 0);

  float* s_w = s_all + (size_t)warp * 16 * SLD;
  float* dp_w = dp_all + (size_t)warp * 16 * SLD;
  T* p_w = p_all + (size_t)warp * 16 * SLD;
  const int r_loc = lane >> 1, c_half = lane & 1;
  const int kv_g = kv0 + warp * 16 + r_loc;                // kv index (inside the sequence) of this lane pair's row
  const bool kv_ok = kv_g < len;
  const float sl2 = scale * kLog2e;
  const T* k_w = k_s + (size_t)warp * 16 * LD;
  const T* v_w = v_s + (size_t)warp * 16 * LD;

  wmma::fragment<wmma::accumulator, 16, 16, 16, float> dk_acc[HD / 16], dv_acc[HD / 16];
#pragma unroll
  for (int i = 0; i < HD / 16; ++i) { wmma::fill_fragment(dk_acc[i], 0.f); wmma::fill_fragment(dv_acc[i], 0.f); }

  for (int n = 0; n < n_iter; ++n) {
    const int st = n & 1;
    if (n + 1 < n_iter) issue_tile(n + 1, st ^ 1);
    if (n + 1 < n_iter) bw_cp_async_wait<1>(); else bw_cp_async_wait<0>();
    __syncthreads();
    const int q0 = (kt0 + n % nI) * kBwTile;
    const float* lse_s = stat + (size_t)st * 2 * kBwTile;
    const float* dlt_s = lse_s + kBwTile;
    // S^T = K_w Q^T and dP^T = V_w dO^T   (16 kv rows x 64 query columns)
#pragma unroll
    for (int nt = 0; nt < kBwTile / 16; ++nt) {
      wmma::fragment<wmma::accumulator, 16, 16, 16, float> sf, df;
      wmma::fill_fragment(sf, 0.f);
      wmma::fill_fragment(df, 0.f);
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        wmma::fragment<wmma::matrix_a, 16, 16, 16, T, wmma::row_major> af;
        wmma::fragment<wmma::matrix_b, 16, 16, 16, T, wmma::col_major> bf;
        wmma::load_matrix_sync(af, k_w + kk * 16, LD);
        wmma::load_matrix_sync(bf, qbuf(st) + (size_t)nt * 16 * LD + kk * 16, LD);       // B[d][q] = Q[q][d]
        wmma::mma_sync(sf, af, bf, sf);
        wmma::load_matrix_sync(af, v_w + kk * 16, LD);
        wmma::load_matrix_sync(bf, dobuf(st) + (size_t)nt * 16 * LD + kk * 16, LD);      // B[d][q] = dO[q][d]
        wmma::mma_sync(df, af, bf, df);
      }
      wmma::store_matrix_sync(s_w + nt * 16, sf, SLD, wmma::mem_row_major);
      wmma::store_matrix_sync(dp_w + nt * 16, df, SLD, wmma::mem_row_major);
    }
    __syncwarp();
    // P^T (model dtype, for dV) ; keep P in fp32 in s_w for dS^T
    for (int c = 0; c < 32; ++c) {
      const int col = c_half * 32 + c;
      const int qi = q0 + col;
      float p = 0.f;
      if (kv_ok && qi < len && kv_g <= qi) p = exp2f(s_w[r_loc * SLD + col] * sl2 - lse_s[col]);
      s_w[r_loc * SLD + col] = p;
      p_w[r_loc * SLD + col] = DT<T>::from_f(p);
    }
    __syncwarp();
#pragma unroll
    for (int kt = 0; kt < kBwTile / 16; ++kt) {
      wmma::fragment<wmma::matrix_a, 16, 16, 16, T, wmma::row_major> af;
      wmma::load_matrix_sync(af, p_w + kt * 16, SLD);
#pragma unroll
      for (int dn = 0; dn < HD / 16; ++dn) {
        wmma::fragment<wmma::matrix_b, 16, 16, 16, T, wmma::row_major> bf;
        wmma::load_matrix_sync(bf, dobuf(st) + (size_t)kt * 16 * LD + dn * 16, LD);      // B[q][d] = dO[q][d]
        wmma::mma_sync(dv_acc[dn], af, bf, dv_acc[dn]);
      }
    }
    __syncwarp();
    // dS^T = P^T o (dP^T - delta) * scale
    for (int c = 0; c < 32; ++c) {
      const int col = c_half * 32 + c;
      const float ds = s_w[r_loc * SLD + col] * (dp_w[r_loc * SLD + col] - dlt_s[col]) * scale;
      p_w[r_loc * SLD + col] = DT<T>::from_f(ds);
    }
    __syncwarp();
#pragma unroll
    for (int kt = 0; kt < kBwTile / 16; ++kt) {
      wmma::fragment<wmma::matrix_a, 16, 16, 16, T, wmma::row_major> af;
      wmma::load_matrix_sync(af, p_w + kt * 16, SLD);
#pragma unroll
      for (int dn = 0; dn < HD / 16; ++dn) {
        wmma::fragment<wmma::matrix_b, 16, 16, 16, T, wmma::row_major> bf;
        wmma::load_matrix_sync(bf, qbuf(st) + (size_t)kt * 16 * LD + dn * 16, LD);       // B[q][d] = Q[q][d]
        wmma::mma_sync(dk_acc[dn], af, bf, dk_acc[dn]);
      }
    }
    __syncwarp();
    __syncthreads();
  }

  // epilogue: dK then dV of this warp's 16 rows through its own fp32 staging block (the Q/dO ring is free)
  float* o_w = reinterpret_cast<float*>(bw_smem + SM::off_ring) + (size_t)warp * SM::stage_floats;
  for (int which = 0; which < 2; ++which) {
#pragma unroll
    for (int dn = 0; dn < HD / 16; ++dn)
      wmma::store_matrix_sync(o_w + dn * 16, which == 0 ? dk_acc[dn] : dv_acc[dn], HD + 8, wmma::mem_row_major);
    __syncwarp();
    if (kv_ok) {
      T* o_g = (which == 0 ? dk : dv) + ((long long)seq0 + kv_g) * kv_stride + (long long)kvh * HD;
      for (int c = 0; c < HD / 2; c += 8) {
        const int col = c_half * (HD / 2) + c;
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = o_w[r_loc * (HD + 8) + col + e];
        *reinterpret_cast<uint4*>(o_g + col) = pack8<T>(f);
      }
    }
    __syncwarp();
  }
}

}  // namespace

// wgmma version for head_dim 128 (attention_bwd_wgmma.cu), the default; CTS_ATTN_BWD_WGMMA=0 selects the HMMA kernels below
int cts_attn_bwd_wgmma_launch(cts_ctx* ctx, const void* q, const void* k, const void* v, const void* dout, const float* lse,
                              const float* delta, const int* cu_seqlens, int batch, int max_seqlen, long long total_tokens, int nh,
                              int nkv, float scale, void* dq, void* dk, void* dv, int dtype, cudaStream_t st);
static bool attn_bwd_use_wgmma() {        // read per call (host side, once per launch): tests flip it inside one process
  const char* e = getenv("CTS_ATTN_BWD_WGMMA");
  return !(e && e[0] == '0');
}

extern "C" int cts_attn_bwd(cts_ctx* ctx, const void* q, const void* k, const void* v, const void* out, const void* dout,
                            const float* lse, const int* cu_seqlens, int batch, int max_seqlen, long long total_tokens, int nh,
                            int nkv, int head_dim, float scale, float* delta_ws, void* dq, void* dk, void* dv, int dtype,
                            void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, q && k && v && out && dout && lse && cu_seqlens && delta_ws && dq && dk && dv, "null pointer");
  CTS_CHECK_ARG(ctx, nh > 0 && nkv > 0 && nh % nkv == 0, "nh must be a positive multiple of nkv");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, total_tokens >= 0, "total_tokens");
  if (head_dim != 64 && head_dim != 128) return cts_set_error(ctx, CTS_ERR_UNSUPPORTED, "cts_attn_bwd: head_dim %d (64 or 128)", head_dim);
  if (batch == 0 || max_seqlen == 0 || total_tokens == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, batch <= 65535 && nh <= 65535, "grid");
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = total_tokens * nh;
  const unsigned tiles = (unsigned)((max_seqlen + kBwTile - 1) / kBwTile);
  if (head_dim == 128 && attn_bwd_use_wgmma()) {
    if (dtype == CTS_BF16) {
      CTS_CUDA(ctx, launch_pdl(attn_bwd_delta_kernel<__nv_bfloat16>, dim3((unsigned)cdiv_ll(rows, 8)), dim3(256), 0, st, 1,
                               (const __nv_bfloat16*)out, (const __nv_bfloat16*)dout, delta_ws, rows, 128));
    } else {
      CTS_CUDA(ctx, launch_pdl(attn_bwd_delta_kernel<__half>, dim3((unsigned)cdiv_ll(rows, 8)), dim3(256), 0, st, 1, (const __half*)out,
                               (const __half*)dout, delta_ws, rows, 128));
    }
    return cts_attn_bwd_wgmma_launch(ctx, q, k, v, dout, lse, delta_ws, cu_seqlens, batch, max_seqlen, total_tokens, nh, nkv, scale, dq,
                                     dk, dv, dtype, st);
  }
#define BW_LAUNCH(TT, HDV)                                                                                                  \
  {                                                                                                                         \
    CTS_CUDA(ctx, launch_pdl(attn_bwd_delta_kernel<TT>, dim3((unsigned)cdiv_ll(rows, 8)), dim3(256), 0, st, 1, (const TT*)out,  \
                             (const TT*)dout, delta_ws, rows, HDV));                                                         \
    const size_t smem = BwSmem<HDV>::total;                                                                                 \
    auto kq = attn_bwd_dq_kernel<TT, HDV>;                                                                                  \
    CTS_CUDA(ctx, cudaFuncSetAttribute(kq, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                        \
    CTS_CUDA(ctx, launch_pdl(kq, dim3(tiles, (unsigned)nh, (unsigned)batch), dim3(kBwThreads), smem, st, 1, (const TT*)q,    \
                             (const TT*)k, (const TT*)v, (const TT*)dout, lse, (const float*)delta_ws, cu_seqlens, nh, nkv,  \
                             scale, (TT*)dq));                                                                               \
    auto kkv = attn_bwd_dkv_kernel<TT, HDV>;                                                                                \
    CTS_CUDA(ctx, cudaFuncSetAttribute(kkv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                       \
    CTS_CUDA(ctx, launch_pdl(kkv, dim3(tiles, (unsigned)nkv, (unsigned)batch), dim3(kBwThreads), smem, st, 1, (const TT*)q,  \
                             (const TT*)k, (const TT*)v, (const TT*)dout, lse, (const float*)delta_ws, cu_seqlens, nh, nkv,  \
                             scale, (TT*)dk, (TT*)dv));                                                                      \
  }
  if (dtype == CTS_BF16) {
    if (head_dim == 128) BW_LAUNCH(__nv_bfloat16, 128) else BW_LAUNCH(__nv_bfloat16, 64)
  } else {
    if (head_dim == 128) BW_LAUNCH(__half, 128) else BW_LAUNCH(__half, 64)
  }
#undef BW_LAUNCH
  return CTS_OK;
}
