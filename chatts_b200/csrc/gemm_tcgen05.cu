// chatts_b200 -- weight-streaming wgmma GEMM:  Y[T,N] = X[T,K] * W[N,K]^T  (+ fused epilogues)
//
// Replaces every nn.Linear on the ChatTS hot path: the TS-encoder MLP (chatts/vllm/chatts_vllm.py:83-91,188)
// and the Qwen2 projections / lm_head the reference reaches through transformers / vLLM
// (modeling_qwen2.py:44-48,217-219,245; chatts_vllm.py:595-610).
//
// "Swap-AB" design: the WEIGHT tile is the 128-row MMA operand A (K-major, streamed once from HBM by TMA with
// an evict-first hint), the TOKENS are the MMA N dimension (operand B, K-major, L2 resident, evict-last).  A
// decode batch of 1..32 tokens therefore still fills the M = 2 x 64 rows of the wgmma instructions and the
// kernel is bound by the HBM stream of W; longer prompts use N = 64 / 128 tiles of the same kernel.  The
// accumulator lives in the registers of the MMA warpgroup, which parks it in shared memory (row = output
// feature, column = token) for the thread-per-feature epilogue: bias / GELU / SwiGLU / residual / split-K
// partial stores / row scatter.
//
//   warps 0..3  : MMA warpgroup (wgmma.mma_async, both 64-row halves of the tile), then the epilogue;
//                 warp w owns output features 32*w .. +31 in the epilogue
//   warp 4      : TMA producer (one elected lane), mbarrier full/empty ring of `stages` slots
//   warp 5      : idle
//
// grid = (ceil(N/128), ceil(T/BN), split_k).
#include <type_traits>

#include "common.cuh"
#include "tensormap.cuh"
#include "trace.cuh"

namespace {

constexpr int kBM = 128;        // weight rows per tile == two wgmma M = 64 halves
constexpr int kBK = 64;         // K elements per stage == 128 bytes == one 128B-swizzle atom
constexpr int kMaxStages = 12;
constexpr int kThreads = 192;

struct GemmParams {
  long long n, k, t, out_ld;
  const void* bias;
  const void* residual;
  void* out;
  const int* row_map;
  int kb_total;
  int split_k;
  int stages;
  int epilogue;
  float* splitk_ws;  // CTS_EPI_SPLITK_F32: fp32 [split_k, t, n] scratch
  int* tile_cnt;     // CTS_EPI_SPLITK_F32: arrival counter per output tile (zero-initialised, self-resetting)
  int l2_prefetch;   // persistent kernel: feature tiles per L2 group (0: feature-fastest order)
  int staged;        // 1: epilogue goes accumulator -> shared-memory output tile -> TMA store (big tiles)
  // next-GEMM weight prefetch (cts_gemm_args.next_*): units of the next launch = next_tiles x next_split, each reads K blocks
  // [kb_total' * z / split', ...) of the 128-row tile x; this grid prefetches the first next_pf blocks of every unit into L2
  int next_tiles, next_split, next_kb_total, next_pf;
};

template <int BN, bool DUAL> __host__ __device__ constexpr int stage_bytes() { return kBM * kBK * 2 * (DUAL ? 2 : 1) + BN * kBK * 2; }
// where the parked fp32 accumulator lives: decode tiles (never staged) reuse the idle pipeline ring, bigger tiles sit behind
// it because the staged epilogue builds its output / residual tiles in the ring
template <int BN> __host__ __device__ constexpr bool acc_in_ring() { return BN <= 32; }

template <typename T, int BN, bool DUAL>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_w2,
               const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_next, const __grid_constant__ CUtensorMap tm_out,
               const __grid_constant__ CUtensorMap tm_res, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kMaxStages];
  __shared__ uint64_t empty_bar[kMaxStages];
  __shared__ uint64_t res_bar;
  __shared__ int last_flag;

  constexpr int kStage = stage_bytes<BN, DUAL>();
  constexpr int kABytes = kBM * kBK * 2;
  constexpr int kLd = acc_ld<BN>();
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;

  // 128B-swizzled tiles need a 1024-byte aligned base
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int f0 = blockIdx.x * kBM;
  const int t0 = blockIdx.y * BN;
  const int split = blockIdx.z;
  const int stages = p.stages;

  // this CTA's K range, in 64-element blocks
  const int kb0 = (int)(((long long)p.kb_total * split) / p.split_k);
  const int kb1 = (int)(((long long)p.kb_total * (split + 1)) / p.split_k);
  const int nkb = kb1 - kb0;

  pdl_trigger();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_x);
    if (DUAL) tma_prefetch_desc(&tm_w2);
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);
    }
    mbar_init(&res_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      // Phase 1 (before the dependency wait): the WEIGHT tiles of the first `stages` K blocks.  Nobody writes
      // weights, so this stream may start while the predecessor kernel is still running (PDL).
      const int npre = nkb < stages ? nkb : stages;
      CTS_TRACE(CTS_TK_GEMM, 0);
      for (int i = 0; i < npre; ++i) {
        mbar_expect_tx(&full_bar[i], (uint32_t)kStage);
        uint8_t* st = smem + (size_t)i * kStage;
        const int kc = (kb0 + i) * kBK;
        tma_load_2d(st, &tm_w, &full_bar[i], kc, f0, CTS_L2_EVICT_FIRST);
        if (DUAL) tma_load_2d(st + kABytes, &tm_w2, &full_bar[i], kc, f0, CTS_L2_EVICT_FIRST);
      }
      pdl_wait();   // activations are produced by the predecessor
      CTS_TRACE(CTS_TK_GEMM, 1);
      for (int i = 0; i < npre; ++i) {
        uint8_t* st = smem + (size_t)i * kStage;
        tma_load_2d(st + kABytes * (DUAL ? 2 : 1), &tm_x, &full_bar[i], (kb0 + i) * kBK, t0, CTS_L2_EVICT_LAST);
      }
      for (int i = npre; i < nkb; ++i) {
        const int s = i % stages;
        const uint32_t ph = (uint32_t)(i / stages) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        mbar_expect_tx(&full_bar[s], (uint32_t)kStage);
        uint8_t* st = smem + (size_t)s * kStage;
        const int kc = (kb0 + i) * kBK;
        tma_load_2d(st, &tm_w, &full_bar[s], kc, f0, CTS_L2_EVICT_FIRST);
        if (DUAL) tma_load_2d(st + kABytes, &tm_w2, &full_bar[s], kc, f0, CTS_L2_EVICT_FIRST);
        tma_load_2d(st + kABytes * (DUAL ? 2 : 1), &tm_x, &full_bar[s], kc, t0, CTS_L2_EVICT_LAST);
      }
      CTS_TRACE(CTS_TK_GEMM, 2);
      // This CTA's own stream is fully requested: keep HBM busy through the drain / kernel boundary / small dependent kernel by
      // pulling the first blocks the NEXT GEMM will read into L2 (fire-and-forget, no shared memory, no barrier).
      if (p.next_pf > 0) {
        const int units = p.next_tiles * p.next_split;
        const int n_ours = (int)(gridDim.x * gridDim.y * gridDim.z);
        const int c = (int)(blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z));
        for (int u = c; u < units; u += n_ours) {
          const int x2 = u % p.next_tiles, z2 = u / p.next_tiles;
          const int kbn0 = (int)(((long long)p.next_kb_total * z2) / p.next_split);
          const int kbn1 = (int)(((long long)p.next_kb_total * (z2 + 1)) / p.next_split);
          const int cnt = (kbn1 - kbn0) < p.next_pf ? (kbn1 - kbn0) : p.next_pf;
          for (int i = 0; i < cnt; ++i) tma_prefetch_l2_2d(&tm_next, (kbn0 + i) * kBK, x2 * kBM);
        }
      }
    }
  } else if (warp < 4) {
    // ------------------------------ MMA warpgroup ------------------------------
    Acc128<BN> acc, acc2;                 // acc2: the w2 (up) product of CTS_EPI_SWIGLU
    acc.zero();
    if (DUAL) acc2.zero();
    for (int i = 0; i < nkb; ++i) {
      const int s = i % stages;
      mbar_wait(&full_bar[s], (uint32_t)(i / stages) & 1u);
      const uint32_t a_addr = smem_u32(smem + (size_t)s * kStage);
      const uint32_t b_addr = a_addr + kABytes * (DUAL ? 2 : 1);
      acc.template mma_kblock<kIsBf16>(a_addr, b_addr, i == 0);
      if (DUAL) acc2.template mma_kblock<kIsBf16>(a_addr + kABytes, b_addr, i == 0);
      wgmma_wait<DUAL ? 2 : 1>();         // the previous K block's MMAs have read their slot
      if (i > 0 && threadIdx.x == 0) mbar_arrive(&empty_bar[(i - 1) % stages]);
    }
    wgmma_wait<0>();
    if (nkb > 0 && threadIdx.x == 0) mbar_arrive(&empty_bar[(nkb - 1) % stages]);
    // ------------------------------ epilogue ------------------------------
    named_bar_sync(1, 128);               // every warp's MMAs are done with the ring
    float* acc_s = reinterpret_cast<float*>(acc_in_ring<BN>() ? smem : smem + (size_t)stages * kStage);
    acc.store(acc_s, kLd);
    if (DUAL) acc2.store(acc_s + kBM * kLd, kLd);
    pdl_wait();   // residual / row_map / the output buffers belong to predecessors until now
    named_bar_sync(1, 128);
    const int q = warp & 3;
    const long long f = (long long)f0 + q * 32 + lane;
    const bool f_ok = f < p.n;
    const int row = q * 32 + lane;
    float bias = 0.f;
    if (p.bias != nullptr && f_ok) bias = DT<T>::to_f(reinterpret_cast<const T*>(p.bias)[f]);
    const int epi = p.epilogue;
    if (p.staged) {
      // ---- big tiles: stage the [BN tokens x 128 features] output tile in shared memory (the pipeline ring is idle
      // once the accumulator is complete) and write it with ONE TMA store (coalesced, clipped at the tensor edge);
      // the residual tile arrives the same way.  Keeps the epilogue a small fraction of the 128x256 mainloop.
      T* out_s = reinterpret_cast<T*>(smem);                          // [BN][128]
      T* res_s = reinterpret_cast<T*>(smem + (size_t)BN * kBM * 2);   // [BN][128]
      const int ft = q * 32 + lane;
      if (epi == CTS_EPI_RESIDUAL) {
        if (threadIdx.x == 64) {
          mbar_expect_tx(&res_bar, (uint32_t)(BN * kBM * 2));
          tma_load_2d_nohint(res_s, &tm_res, &res_bar, f0, t0);
        }
        mbar_wait(&res_bar, 0);
      }
#pragma unroll 1
      for (int c = 0; c < BN; c += 16) {
        if ((long long)t0 + c >= p.t) break;
        uint32_t v[16], v2[16];
        acc_ld16(acc_s, kLd, row, c, v);
        if (DUAL) acc_ld16(acc_s + kBM * kLd, kLd, row, c, v2);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float acc = __uint_as_float(v[j]);
          float r;
          if (epi == CTS_EPI_SWIGLU) {
            r = rnd<T>(silu_f(rnd<T>(acc))) * rnd<T>(__uint_as_float(v2[j]));
          } else {
            r = acc + bias;
            if (epi == CTS_EPI_GELU) r = gelu_erf(rnd<T>(r));
            else if (epi == CTS_EPI_RESIDUAL) r = rnd<T>(r) + DT<T>::to_f(res_s[(c + j) * kBM + ft]);
          }
          out_s[(c + j) * kBM + ft] = DT<T>::from_f(r);
        }
      }
      fence_proxy_async_smem();                 // generic-proxy smem writes -> visible to the TMA engine
      named_bar_sync(1, 128);                   // the four epilogue warps
      if (threadIdx.x == 64) {
        tma_store_2d(&tm_out, out_s, f0, t0);
        tma_store_commit();
        tma_store_wait_read0();
      }
    } else if (epi == CTS_EPI_SPLITK_F32) {
      // ---- split-K with in-kernel reduction: every split leaves its fp32 partial in the scratch; the LAST split of a
      // tile to arrive (arrival counter, threadfence-reduction pattern) sums the partials in split order -- a fixed
      // order, so the result is deterministic -- and writes the reduced fp32 tile.  Consumers then read ONE partial.
      float* dst = p.split_k > 1 ? p.splitk_ws + (long long)split * p.t * p.n : reinterpret_cast<float*>(p.out);
#pragma unroll 1
      for (int c = 0; c < BN; c += 16) {
        if ((long long)t0 + c >= p.t) break;
        uint32_t v[16];
        acc_ld16(acc_s, kLd, row, c, v);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const long long t = (long long)t0 + c + j;
          if (t < p.t && f_ok) dst[t * p.n + f] = __uint_as_float(v[j]);
        }
      }
      if (p.split_k > 1) {
        __threadfence();
        named_bar_sync(1, 128);
        const int tile_id = blockIdx.y * gridDim.x + blockIdx.x;
        if (threadIdx.x == 64) last_flag = (atomicAdd(&p.tile_cnt[tile_id], 1) == p.split_k - 1);
        named_bar_sync(1, 128);
        if (last_flag) {
          __threadfence();
          const long long tmax = p.t - t0 < BN ? p.t - t0 : BN;
          if (f_ok) {
            float* o = reinterpret_cast<float*>(p.out);
#pragma unroll 2
            for (long long tt = 0; tt < tmax; ++tt) {
              const long long off = (t0 + tt) * p.n + f;
              float a = 0.f;
              for (int s2 = 0; s2 < p.split_k; ++s2) a += __ldcg(p.splitk_ws + (long long)s2 * p.t * p.n + off);
              o[off] = a;
            }
          }
          if (threadIdx.x == 64) p.tile_cnt[tile_id] = 0;
        }
      }
    } else {
#pragma unroll 1
    for (int c = 0; c < BN; c += 16) {
      if ((long long)t0 + c >= p.t) break;   // warp-uniform
      uint32_t v[16], v2[16];
      acc_ld16(acc_s, kLd, row, c, v);
      if (DUAL) acc_ld16(acc_s + kBM * kLd, kLd, row, c, v2);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const long long t = (long long)t0 + c + j;
        if (t >= p.t || !f_ok) continue;
        const float acc = __uint_as_float(v[j]);
        if (epi == CTS_EPI_PARTIAL_F32) {
          reinterpret_cast<float*>(p.out)[((long long)split * p.t + t) * p.n + f] = acc;
          continue;
        }
        long long row = t;
        if (p.row_map != nullptr) {
          row = p.row_map[t];
          if (row < 0) continue;
        }
        float r;
        if (epi == CTS_EPI_SWIGLU) {
          const float g = rnd<T>(acc);
          const float u = rnd<T>(__uint_as_float(v2[j]));
          r = rnd<T>(silu_f(g)) * u;
        } else {
          r = acc + bias;
          if (epi == CTS_EPI_GELU) {
            r = gelu_erf(rnd<T>(r));
          } else if (epi == CTS_EPI_RESIDUAL) {
            r = rnd<T>(r) + DT<T>::to_f(reinterpret_cast<const T*>(p.residual)[row * p.out_ld + f]);
          }
        }
        reinterpret_cast<T*>(p.out)[row * p.out_ld + f] = DT<T>::from_f(r);
      }
    }
    }
  }

  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_GEMM, 3);
}

// =================================================================================================================
// Persistent weight-streaming kernel for decode-sized steps (t <= 32, one token tile), epilogues PARTIAL_F32 and NONE (split 1).
// The work is a list of units = (weight-row tile of 64 H rows, K split), dealt round-robin to `ctas per SM x SMs` resident CTAs.  The
// producer keeps one ring of `stages` slots full across unit boundaries; a slot holds KS consecutive 64-wide K blocks of the weight tile
// (KS x 128 contiguous bytes of every row) and of the token tile.  The weight tiles of the first `stages` slots are requested before the
// dependency wait (nobody writes weights), the token tiles and every store after it.  Each split covers the 64-wide K blocks
// [kb_total s / split, kb_total (s + 1) / split) and each output is accumulated by the same m64nBNk16 wgmma sequence in ascending K as in
// gemm_tn_kernel, so the fp32 partials are bit-identical to that kernel's at the same split factor; the ring depth, the tile height and
// KS change only which bytes travel together.  The accumulator is stored straight from the fragment registers (eight consecutive
// features per 32-byte sector), so the ring never stalls on an epilogue.
//   warps 0..3 : MMA warpgroup + epilogue;  warp 4 : TMA producer (one lane)
// =================================================================================================================
constexpr int kSMaxStages = 16;
constexpr int kSThreads = 160;

struct StreamParams {
  long long n, t, out_ld;
  const void* bias;   // CTS_EPI_NONE only (may be null)
  void* out;          // PARTIAL_F32: fp32 [split_k, t, n];  NONE: T [t, out_ld]
  int kb_total, split_k, tiles, stages, epilogue;
};

template <int BN, int H, int KS> __host__ __device__ constexpr int stream_stage_bytes() { return KS * (H * 64 + BN) * kBK * 2; }

template <typename T, int BN, int H, int KS>
__global__ void __launch_bounds__(kSThreads, 1)
gemm_stream_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x, const StreamParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kSMaxStages];
  __shared__ uint64_t empty_bar[kSMaxStages];

  constexpr int kRows = 64 * H;
  constexpr int kWBlk = kRows * kBK * 2;       // one 64-wide K block of the weight tile
  constexpr int kXBlk = BN * kBK * 2;          // ... and of the token tile
  constexpr int kStage = stream_stage_bytes<BN, H, KS>();
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;

  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* ring = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.stages;
  const int units = p.tiles * p.split_k;
  auto unit = [&](int u, int& tile, int& split, int& kb0, int& kb1) {
    tile = u % p.tiles;
    split = u / p.tiles;
    kb0 = (int)(((long long)p.kb_total * split) / p.split_k);
    kb1 = (int)(((long long)p.kb_total * (split + 1)) / p.split_k);
  };

  pdl_trigger();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_x);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      auto issue_w = [&](int s, int f0, int kb, int nb) {
        mbar_expect_tx(&full_bar[s], (uint32_t)(nb * (kWBlk + kXBlk)));
        uint8_t* st = ring + (size_t)s * kStage;
        for (int b = 0; b < nb; ++b) tma_load_2d(st + b * kWBlk, &tm_w, &full_bar[s], (kb + b) * kBK, f0, CTS_L2_EVICT_FIRST);
      };
      int pre = 0;
      for (int u = blockIdx.x; u < units && pre < S; u += gridDim.x) {
        int tile, split, kb0, kb1;
        unit(u, tile, split, kb0, kb1);
        for (int kb = kb0; kb < kb1 && pre < S; kb += KS, ++pre) issue_w(pre, tile * kRows, kb, min(KS, kb1 - kb));
      }
      pdl_wait();   // activations are produced by the predecessor
      int s = 0, n = 0;
      uint32_t ph = 1u;                           // parity of the "slot is empty" phase waited for (a fresh barrier passes)
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        int tile, split, kb0, kb1;
        unit(u, tile, split, kb0, kb1);
        for (int kb = kb0; kb < kb1; kb += KS, ++n) {
          const int nb = min(KS, kb1 - kb);
          if (n >= pre) {
            mbar_wait(&empty_bar[s], ph);
            issue_w(s, tile * kRows, kb, nb);
          }
          uint8_t* xs = ring + (size_t)s * kStage + KS * kWBlk;
          for (int b = 0; b < nb; ++b) tma_load_2d(xs + b * kXBlk, &tm_x, &full_bar[s], (kb + b) * kBK, 0, CTS_L2_EVICT_LAST);
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // ------------------------------ MMA warpgroup + epilogue ------------------------------
    pdl_wait();   // the output buffers belong to predecessors until now
    Acc128<BN> acc;                               // H == 1 uses the first m64 half only
    float (&d)[2][BN / 2] = acc.d;
    int s = 0;
    uint32_t ph = 0u;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      int tile, split, kb0, kb1;
      unit(u, tile, split, kb0, kb1);
      for (int kb = kb0; kb < kb1; kb += KS) {
        const int nb = min(KS, kb1 - kb);
        mbar_wait(&full_bar[s], ph);
        const uint32_t wa = smem_u32(ring + (size_t)s * kStage), xa = wa + KS * kWBlk;
        if constexpr (H == 2) {
#pragma unroll
          for (int b = 0; b < KS; ++b)
            if (b < nb) acc.template mma_kblock<kIsBf16>(wa + b * kWBlk, xa + b * kXBlk, kb == kb0 && b == 0);
        } else {                                  // the same sequence on one m64 half
          for (int i = 0; i < BN / 2; ++i) wgmma_fence_operand(d[0][i]);
          wgmma_fence();
#pragma unroll
          for (int b = 0; b < KS; ++b) {
            if (b < nb) {
              const uint64_t ad = gmma_desc_k_sw128(wa + b * kWBlk), bd = gmma_desc_k_sw128(xa + b * kXBlk);
#pragma unroll
              for (int kk = 0; kk < 4; ++kk)
                wgmma_m64k16<BN, kIsBf16>(d[0], ad + 2 * kk, bd + 2 * kk, (kb == kb0 && b == 0 && kk == 0) ? 0 : 1);
            }
          }
          wgmma_commit();
          for (int i = 0; i < BN / 2; ++i) wgmma_fence_operand(d[0][i]);
        }
        wgmma_wait<0>();
        if (threadIdx.x == 0) mbar_arrive(&empty_bar[s]);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
      // ------------------------------ epilogue, from the fragment registers ------------------------------
      const long long f0 = (long long)tile * kRows;
      if (p.epilogue == CTS_EPI_PARTIAL_F32) {
        float* dst = reinterpret_cast<float*>(p.out) + (long long)split * p.t * p.n;
#pragma unroll
        for (int h = 0; h < H; ++h)
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) {
            const long long f = f0 + 64 * h + acc_row(i), t = acc_col(i);
            if (t < p.t && f < p.n) dst[t * p.n + f] = d[h][i];
          }
      } else {
        T* dst = reinterpret_cast<T*>(p.out);
        const T* bias = reinterpret_cast<const T*>(p.bias);
#pragma unroll
        for (int h = 0; h < H; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const long long f = f0 + 64 * h + acc_row(2 * e);
            const float bv = (bias != nullptr && f < p.n) ? DT<T>::to_f(bias[f]) : 0.f;
#pragma unroll
            for (int i = 2 * e; i < BN / 2; i += 4)
#pragma unroll
              for (int j = 0; j < 2; ++j) {
                const long long t = acc_col(i + j);
                if (t < p.t && f < p.n) dst[t * p.out_ld + f] = DT<T>::from_f(d[h][i + j] + bv);
              }
          }
      }
    }
  }
}

// =================================================================================================================
// Persistent variant for big token counts (prefill): one CTA per SM walks the output tiles (128 features x 128 tokens) and
// the TMA ring runs continuously across tiles, so the weight / token loads of tile i+1 stream while the MMA warpgroup runs
// the epilogue of tile i (accumulator registers -> shared-memory output tile -> TMA store, residual tile by TMA load).
// Epilogues: NONE / GELU / RESIDUAL, and SWIGLU_IL for gate_up weights stored INTERLEAVED (each 128-row weight tile = 64 gate
// rows then the 64 matching up rows): gate row r and up row r + 64 sit in the same register of the two accumulator halves, so
// SwiGLU is thread-local and the tile emits 64 output features.
// =================================================================================================================
constexpr int kPBN = 128;
constexpr int kPStages = 4;
constexpr int kPStageBytes = kBM * kBK * 2 + kPBN * kBK * 2;     // 32 KiB
constexpr int kPOutBytes = kPBN * kBM * 2;                        // 32 KiB staging tile

template <typename T>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tn_persistent_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x,
                          const __grid_constant__ CUtensorMap tm_out, const __grid_constant__ CUtensorMap tm_res,
                          const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kPStages], empty_bar[kPStages], res_bar;
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* out_s = smem + kPStages * kPStageBytes;
  uint8_t* res_s = out_s + kPOutBytes;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (int)((p.n + kBM - 1) / kBM), tiles_n = (int)((p.t + kPBN - 1) / kPBN);
  const int total_tiles = tiles_m * tiles_n;
  const int nkb = p.kb_total;
  const int epi = p.epilogue;
  // L2-aware rasterisation: the feature tiles are walked in groups of `gm` whose weights (gm x 128 x K) fit in L2; inside
  // a group the token tiles advance slowly and the gm feature tiles fast, so the tiles in flight share a few token tiles
  // and the group's weights stay L2-resident across all token tiles.  DRAM then sees the weights once and the
  // activations once per group (instead of the weights once per token tile).
  const int gm = p.l2_prefetch > 0 ? p.l2_prefetch : tiles_m;
  auto tile_coords = [&](int id, int& m_blk, int& n_blk) {
    const int per_group = gm * tiles_n;
    const int g = id / per_group, r = id - g * per_group;
    const int gm_here = min(gm, tiles_m - g * gm);
    n_blk = r / gm_here;
    m_blk = g * gm + (r - n_blk * gm_here);
  };

  pdl_trigger();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_w); tma_prefetch_desc(&tm_x); tma_prefetch_desc(&tm_out);
    for (int s = 0; s < kPStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    mbar_init(&res_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      pdl_wait();
      uint32_t it = 0;                                   // global K-block counter across this CTA's tiles
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int mb, nb;
        tile_coords(tile, mb, nb);
        const int f0 = mb * kBM, t0 = nb * kPBN;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % kPStages;
          mbar_wait(&empty_bar[s], ((it / kPStages) & 1u) ^ 1u);
          mbar_expect_tx(&full_bar[s], (uint32_t)kPStageBytes);
          uint8_t* st = smem + (size_t)s * kPStageBytes;
          tma_load_2d(st, &tm_w, &full_bar[s], kb * kBK, f0, CTS_L2_EVICT_NORMAL);
          tma_load_2d(st + kBM * kBK * 2, &tm_x, &full_bar[s], kb * kBK, t0, CTS_L2_EVICT_NORMAL);
        }
      }
    }
  } else if (warp < 4) {
    // ------------------------------ MMA warpgroup + epilogue ------------------------------
    pdl_wait();
    uint32_t it = 0, res_uses = 0;
    T* outp = reinterpret_cast<T*>(out_s);
    const T* resp = reinterpret_cast<const T*>(res_s);
    const T* biasp = reinterpret_cast<const T*>(p.bias);
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int mb, nb;
      tile_coords(tile, mb, nb);
      const int f0 = mb * kBM, t0 = nb * kPBN;
      if (epi == CTS_EPI_RESIDUAL && threadIdx.x == 0) {  // the residual tile lands while the mainloop runs
        fence_proxy_async_smem();                         // the previous tile's generic-proxy reads of res_s (ordered by the named barrier) before the TMA write
        mbar_expect_tx(&res_bar, (uint32_t)kPOutBytes);
        tma_load_2d_nohint(res_s, &tm_res, &res_bar, f0, t0);
      }
      Acc128<kPBN> acc;
      acc.zero();
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = it % kPStages;
        mbar_wait(&full_bar[s], (it / kPStages) & 1u);
        const uint32_t a_addr = smem_u32(smem + (size_t)s * kPStageBytes);
        acc.template mma_kblock<kIsBf16>(a_addr, a_addr + kBM * kBK * 2, kb == 0);
        wgmma_wait<1>();
        if (kb > 0 && threadIdx.x == 0) mbar_arrive(&empty_bar[(it - 1) % kPStages]);
      }
      wgmma_wait<0>();
      if (nkb > 0 && threadIdx.x == 0) mbar_arrive(&empty_bar[(it - 1) % kPStages]);
      if (epi == CTS_EPI_RESIDUAL) {
        mbar_wait(&res_bar, res_uses & 1u);
        ++res_uses;
      }
      if (epi == CTS_EPI_SWIGLU_IL) {
#pragma unroll
        for (int i = 0; i < kPBN / 2; ++i) {
          const float g = rnd<T>(acc.d[0][i]);
          const float u = rnd<T>(acc.d[1][i]);
          outp[acc_col(i) * 64 + acc_row(i)] = DT<T>::from_f(rnd<T>(silu_f(g)) * u);
        }
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float bias[2] = {0.f, 0.f};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const long long f = (long long)f0 + 64 * h + acc_row(2 * e);
            if (biasp != nullptr && f < p.n) bias[e] = DT<T>::to_f(biasp[f]);
          }
#pragma unroll
          for (int i = 0; i < kPBN / 2; ++i) {
            const int ft = 64 * h + acc_row(i), tt = acc_col(i);
            float r = acc.d[h][i] + bias[(i >> 1) & 1];
            if (epi == CTS_EPI_GELU) r = gelu_erf(rnd<T>(r));
            else if (epi == CTS_EPI_RESIDUAL) r = rnd<T>(r) + DT<T>::to_f(resp[tt * kBM + ft]);
            outp[tt * kBM + ft] = DT<T>::from_f(r);
          }
        }
      }
      fence_proxy_async_smem();                           // generic-proxy smem writes -> visible to the TMA engine
      named_bar_sync(1, 128);
      if (threadIdx.x == 0) {
        if (epi == CTS_EPI_SWIGLU_IL) tma_store_2d(&tm_out, out_s, f0 / 2, t0);
        else tma_store_2d(&tm_out, out_s, f0, t0);
        tma_store_commit();
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");     // staging tile may be rewritten
      }
      named_bar_sync(1, 128);                             // staging and residual tiles are free again
    }
    if (threadIdx.x == 0) tma_store_wait_read0();         // all stores fully performed before the CTA retires
  }
}

template <typename T>
int launch_persistent(cts_ctx* ctx, const cts_gemm_args* a, cudaStream_t stream) {
  const bool is_bf16 = a->dtype == CTS_BF16;
  const bool il = a->epilogue == CTS_EPI_SWIGLU_IL;
  CUtensorMap tm_w, tm_x, tm_out, tm_res;
  int rc = cts_make_tmap_2d(ctx, &tm_w, a->w, a->n, a->k, a->w_ld, kBM, is_bf16);
  if (rc) return rc;
  rc = cts_make_tmap_2d(ctx, &tm_x, a->x, a->t, a->k, a->x_ld, kPBN, is_bf16);
  if (rc) return rc;
  rc = cts_make_tmap_2d_dense(ctx, &tm_out, a->out, a->t, il ? a->n / 2 : a->n, a->out_ld, kPBN, il ? 64 : kBM, is_bf16);
  if (rc) return rc;
  tm_res = tm_out;
  if (a->epilogue == CTS_EPI_RESIDUAL) {
    rc = cts_make_tmap_2d_dense(ctx, &tm_res, a->residual, a->t, a->n, a->out_ld, kPBN, kBM, is_bf16);
    if (rc) return rc;
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.n = a->n; p.k = a->k; p.t = a->t; p.out_ld = a->out_ld;
  p.bias = a->bias; p.residual = a->residual; p.out = a->out;
  p.kb_total = (int)cdiv_ll(a->k, kBK);
  p.split_k = 1; p.epilogue = a->epilogue; p.stages = kPStages;
  {
    // feature tiles per L2 group: keep the group's weights within ~20 MB (40 % of the H100's 50 MB L2), balanced over the groups
    const long long tiles_m = cdiv_ll(a->n, kBM);
    long long gmax = (20LL << 20) / ((long long)kBM * a->k * 2);
    if (gmax < 1) gmax = 1;
    const long long groups = cdiv_ll(tiles_m, gmax);
    p.l2_prefetch = (int)cdiv_ll(tiles_m, groups);       // field reused as "group_m" by the persistent kernel
    if (ctx->l2_prefetch_mb < 0) p.l2_prefetch = 0;      // CTS_L2_PREFETCH_MB=-1: plain feature-fastest order (A/B testing)
  }
  const size_t smem = (size_t)kPStages * kPStageBytes + 2 * kPOutBytes + 1024;
  auto kern = gemm_tn_persistent_kernel<T>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const long long tiles = cdiv_ll(a->n, kBM) * cdiv_ll(a->t, kPBN);
  const unsigned grid = (unsigned)(tiles < ctx->sm_count ? tiles : ctx->sm_count);
  CTS_CUDA(ctx, launch_pdl(kern, dim3(grid), dim3(kThreads), smem, stream, 1, tm_w, tm_x, tm_out, tm_res, p));
  return CTS_OK;
}

template <typename T, int BN, bool DUAL>
int launch(cts_ctx* ctx, const cts_gemm_args* a, cudaStream_t stream) {
  const bool is_bf16 = a->dtype == CTS_BF16;
  CUtensorMap tm_w, tm_w2, tm_x;
  int rc = cts_make_tmap_2d(ctx, &tm_w, a->w, a->n, a->k, a->w_ld, kBM, is_bf16);
  if (rc) return rc;
  if (DUAL) {
    rc = cts_make_tmap_2d(ctx, &tm_w2, a->w2, a->n, a->k, a->w_ld, kBM, is_bf16);
    if (rc) return rc;
  } else {
    tm_w2 = tm_w;
  }
  rc = cts_make_tmap_2d(ctx, &tm_x, a->x, a->t, a->k, a->x_ld, BN, is_bf16);
  if (rc) return rc;
  // big tiles without a row scatter: output (and residual) tiles move by TMA through shared memory (the ring is idle by then)
  const bool staged = BN >= 64 && a->row_map == nullptr && a->epilogue != CTS_EPI_PARTIAL_F32 && a->epilogue != CTS_EPI_SPLITK_F32 && (a->out_ld * 2) % 16 == 0 &&
                      ((uintptr_t)a->out & 15) == 0 && (a->epilogue != CTS_EPI_RESIDUAL || ((uintptr_t)a->residual & 15) == 0);
  CUtensorMap tm_out = tm_x, tm_res = tm_x;
  if (staged) {
    rc = cts_make_tmap_2d_dense(ctx, &tm_out, a->out, a->t, a->n, a->out_ld, BN, kBM, is_bf16);
    if (rc) return rc;
    if (a->epilogue == CTS_EPI_RESIDUAL) {
      rc = cts_make_tmap_2d_dense(ctx, &tm_res, a->residual, a->t, a->n, a->out_ld, BN, kBM, is_bf16);
      if (rc) return rc;
    }
  }

  GemmParams p;
  p.n = a->n; p.k = a->k; p.t = a->t; p.out_ld = a->out_ld;
  p.bias = a->bias; p.residual = a->residual; p.out = a->out; p.row_map = a->row_map;
  p.splitk_ws = (float*)a->splitk_ws; p.tile_cnt = a->tile_counters;
  p.kb_total = (int)cdiv_ll(a->k, kBK);
  p.split_k = a->split_k;
  p.epilogue = a->epilogue;
  // next-GEMM weight prefetch (decode-sized launches only; CTS_NEXT_PREFETCH=0 switches the hint off for A/B runs)
  CUtensorMap tm_next = tm_w;
  p.next_tiles = p.next_split = p.next_kb_total = p.next_pf = 0;
  if (BN <= 32 && a->next_w != nullptr && a->next_prefetch_bytes > 0 && a->next_n > 0 && a->next_k > 0 && a->next_split >= 1 && !ctx->no_next_prefetch) {
    rc = cts_make_tmap_2d(ctx, &tm_next, a->next_w, a->next_n, a->next_k, a->next_ld > 0 ? a->next_ld : a->next_k, kBM, is_bf16);
    if (rc) return rc;
    p.next_tiles = (int)cdiv_ll(a->next_n, kBM);
    p.next_split = a->next_split;
    p.next_kb_total = (int)cdiv_ll(a->next_k, kBK);
    const long long units = (long long)p.next_tiles * p.next_split;
    long long pf = a->next_prefetch_bytes / (units * kBM * kBK * 2);
    const long long per_unit = cdiv_ll(p.next_kb_total, p.next_split);
    if (pf > per_unit) pf = per_unit;
    p.next_pf = (int)pf;
  }
  constexpr int kStage = stage_bytes<BN, DUAL>();
  // small-N (decode / short-prompt / TS-encoder) tiles: leave room for two or three CTAs per SM so one CTA's prologue/epilogue overlaps the
  // other's stream; large-N (prefill) tiles take the whole SM.
  const int budget = (BN <= 32) ? ctx->decode_stages * 1024 : (BN <= 128 ? 100 * 1024 : 200 * 1024);
  int stages = budget / kStage;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) stages = 2;
  p.stages = stages;
  p.staged = staged ? 1 : 0;
  p.l2_prefetch = 0;
  if (staged && stages * kStage < 2 * BN * kBM * 2) stages = (2 * BN * kBM * 2 + kStage - 1) / kStage;
  p.stages = stages;
  const size_t acc_bytes = (size_t)acc_smem_bytes<BN>() * (DUAL ? 2 : 1);
  const size_t ring = (size_t)stages * kStage;
  const size_t smem = (acc_in_ring<BN>() ? (ring > acc_bytes ? ring : acc_bytes) : ring + acc_bytes) + 1024;
  auto kern = gemm_tn_kernel<T, BN, DUAL>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)cdiv_ll(a->n, kBM), (unsigned)cdiv_ll(a->t, BN), (unsigned)a->split_k);
  CTS_CUDA(ctx, launch_pdl(kern, grid, dim3(kThreads), smem, stream, 1, tm_w, tm_w2, tm_x, tm_next, tm_out, tm_res, p));
  return CTS_OK;
}

// The decode GEMM selection and shape of a context: read by ctx.cu at context creation.  The CPU shim's stand-in context has no such
// fields; there the same variables (same defaults) are read from the environment at each launch.
struct StreamCfg { int off, ctas, rows, kblocks; };
static inline StreamCfg stream_cfg(const cts_ctx* ctx) {
#ifndef CTS_HOST_SHIM
  return {ctx->no_stream_gemm, ctx->stream_ctas, ctx->stream_rows, ctx->stream_kblocks};
#else
  auto env = [](const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; };
  return {env("CTS_NO_STREAM_GEMM", 0), env("CTS_STREAM_CTAS", 2), env("CTS_STREAM_ROWS", 128), env("CTS_STREAM_KBLOCKS", 1)};
#endif
}

template <typename T, int BN, int H, int KS>
int launch_stream(cts_ctx* ctx, const StreamCfg& cfg, const cts_gemm_args* a, cudaStream_t stream) {
  const bool is_bf16 = a->dtype == CTS_BF16;
  CUtensorMap tm_w, tm_x;
  int rc = cts_make_tmap_2d(ctx, &tm_w, a->w, a->n, a->k, a->w_ld, 64 * H, is_bf16);
  if (rc) return rc;
  rc = cts_make_tmap_2d(ctx, &tm_x, a->x, a->t, a->k, a->x_ld, BN, is_bf16);
  if (rc) return rc;
  StreamParams p;
  p.n = a->n; p.t = a->t; p.out_ld = a->out_ld;
  p.bias = a->bias; p.out = a->out;
  p.kb_total = (int)cdiv_ll(a->k, kBK);
  p.split_k = a->split_k;
  p.tiles = (int)cdiv_ll(a->n, 64 * H);
  p.epilogue = a->epilogue;
  // the ring takes whatever shared memory the resident CTAs of an SM leave each other
  constexpr int kStage = stream_stage_bytes<BN, H, KS>();
  const int ctas = cfg.ctas;
  const int budget = (ctx->max_smem_optin + 1024) / ctas - 3 * 1024;
  int stages = (budget - 1024) / kStage;
  if (stages > kSMaxStages) stages = kSMaxStages;
  if (stages < 2)
    return cts_set_error(ctx, CTS_ERR_BAD_ARG, "cts_gemm: %d CTAs per SM leave room for fewer than two %d KB stages", ctas, kStage / 1024);
  p.stages = stages;
  const size_t smem = (size_t)stages * kStage + 1024;
  auto kern = gemm_stream_kernel<T, BN, H, KS>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
#ifndef CTS_HOST_SHIM
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
#endif
  const long long units = (long long)p.tiles * p.split_k;
  long long grid = (long long)ctas * ctx->sm_count;
  if (grid > units) grid = units;
  CTS_CUDA(ctx, launch_pdl(kern, dim3((unsigned)grid), dim3(kSThreads), smem, stream, 1, tm_w, tm_x, p));
  return CTS_OK;
}

template <typename T, int BN>
int dispatch_stream(cts_ctx* ctx, const StreamCfg& c, const cts_gemm_args* a, cudaStream_t st) {
  const int ks = c.kblocks;
  if (c.rows == 64)
    return ks == 1 ? launch_stream<T, BN, 1, 1>(ctx, c, a, st) : ks == 2 ? launch_stream<T, BN, 1, 2>(ctx, c, a, st) : launch_stream<T, BN, 1, 4>(ctx, c, a, st);
  return ks == 1 ? launch_stream<T, BN, 2, 1>(ctx, c, a, st) : ks == 2 ? launch_stream<T, BN, 2, 2>(ctx, c, a, st) : launch_stream<T, BN, 2, 4>(ctx, c, a, st);
}

template <typename T>
int dispatch_stream_bn(cts_ctx* ctx, const StreamCfg& c, const cts_gemm_args* a, cudaStream_t st) {
  return a->t <= 16 ? dispatch_stream<T, 16>(ctx, c, a, st) : dispatch_stream<T, 32>(ctx, c, a, st);
}

template <typename T, bool DUAL>
int dispatch_bn(cts_ctx* ctx, const cts_gemm_args* a, cudaStream_t stream) {
  const long long t = a->t;
  if (t <= 16) return launch<T, 16, DUAL>(ctx, a, stream);
  if (t <= 32) return launch<T, 32, DUAL>(ctx, a, stream);
  // one warpgroup holds the whole 128 x BN accumulator in registers: BN <= 128, and <= 64 with the second (w2) accumulator
  if (t <= 64 || DUAL) return launch<T, 64, DUAL>(ctx, a, stream);
  return launch<T, 128, false>(ctx, a, stream);
}

}  // namespace

extern "C" int cts_gemm(cts_ctx* ctx, const cts_gemm_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr, "null args");
  CTS_CHECK_ARG(ctx, a->w && a->x && a->out, "null w/x/out");
  CTS_CHECK_ARG(ctx, a->n > 0 && a->k > 0 && a->t > 0, "n, k, t must be positive");
  CTS_CHECK_ARG(ctx, a->dtype == CTS_BF16 || a->dtype == CTS_F16, "dtype must be CTS_BF16 or CTS_F16");
  CTS_CHECK_ARG(ctx, a->epilogue >= CTS_EPI_NONE && a->epilogue <= CTS_EPI_SWIGLU_IL, "unknown epilogue");
  CTS_CHECK_ARG(ctx, a->split_k >= 1, "split_k must be >= 1");
  CTS_CHECK_ARG(ctx, a->split_k == 1 || a->epilogue == CTS_EPI_PARTIAL_F32 || a->epilogue == CTS_EPI_SPLITK_F32,
                "split_k > 1 needs CTS_EPI_PARTIAL_F32 or CTS_EPI_SPLITK_F32");
  CTS_CHECK_ARG(ctx, a->epilogue != CTS_EPI_SPLITK_F32 || a->split_k == 1 || (a->splitk_ws && a->tile_counters),
                "CTS_EPI_SPLITK_F32 with split_k > 1 needs splitk_ws and tile_counters");
  CTS_CHECK_ARG(ctx, a->split_k <= cdiv_ll(a->k, kBK), "split_k exceeds the number of 64-wide K blocks");
  CTS_CHECK_ARG(ctx, a->split_k <= 65535 && cdiv_ll(a->t, 16) <= 65535 * 16LL, "grid too large");
  CTS_CHECK_ARG(ctx, (a->epilogue == CTS_EPI_SWIGLU) == (a->w2 != nullptr), "w2 is required by (and only by) CTS_EPI_SWIGLU");
  CTS_CHECK_ARG(ctx, a->epilogue != CTS_EPI_RESIDUAL || a->residual != nullptr, "CTS_EPI_RESIDUAL needs residual");
  CTS_CHECK_ARG(ctx, a->w_ld >= a->k && a->x_ld >= a->k, "leading dimension smaller than k");
  CTS_CHECK_ARG(ctx, a->epilogue == CTS_EPI_PARTIAL_F32 || a->epilogue == CTS_EPI_SPLITK_F32 ||
                         a->out_ld >= (a->epilogue == CTS_EPI_SWIGLU_IL ? a->n / 2 : a->n), "out_ld smaller than n");
  cudaStream_t st = (cudaStream_t)stream;
  // decode-sized launches that write fp32 partials (or, at split 1, the plain output) go to the persistent streaming kernel; row
  // scatters, the dual SwiGLU accumulators, the in-kernel split-K reduction and launches carrying the next-GEMM L2 hint stay on
  // gemm_tn_kernel (so does everything under CTS_NO_STREAM_GEMM=1)
  const bool next_hint = a->next_w != nullptr && a->next_prefetch_bytes > 0;
  const StreamCfg cfg = stream_cfg(ctx);
  if (a->t <= 32 && (a->epilogue == CTS_EPI_PARTIAL_F32 || (a->epilogue == CTS_EPI_NONE && a->split_k == 1)) && a->row_map == nullptr &&
      a->w2 == nullptr && !next_hint && !cfg.off) {
    CTS_CHECK_ARG(ctx, cfg.ctas >= 1 && cfg.ctas <= 4 && (cfg.rows == 64 || cfg.rows == 128) && (cfg.kblocks == 1 || cfg.kblocks == 2 || cfg.kblocks == 4),
                  "decode GEMM shape: CTS_STREAM_CTAS 1..4, CTS_STREAM_ROWS 64 or 128, CTS_STREAM_KBLOCKS 1, 2 or 4");
    return a->dtype == CTS_BF16 ? dispatch_stream_bn<__nv_bfloat16>(ctx, cfg, a, st) : dispatch_stream_bn<__half>(ctx, cfg, a, st);
  }
  CTS_CHECK_ARG(ctx, a->epilogue != CTS_EPI_SWIGLU_IL || (a->n % 128 == 0 && a->t > 128 && a->row_map == nullptr),
                "CTS_EPI_SWIGLU_IL needs n % 128 == 0, t > 128 and no row_map (small t: CTS_EPI_PARTIAL_F32 + cts_reduce_swiglu)");
  const bool pers_epi = a->epilogue == CTS_EPI_NONE || a->epilogue == CTS_EPI_GELU || a->epilogue == CTS_EPI_RESIDUAL ||
                        a->epilogue == CTS_EPI_SWIGLU_IL;
  if (a->t > 128 && pers_epi && a->row_map == nullptr && a->split_k == 1 && (a->out_ld * 2) % 16 == 0 &&
      ((uintptr_t)a->out & 15) == 0 && (a->epilogue != CTS_EPI_RESIDUAL || ((uintptr_t)a->residual & 15) == 0) &&
      !ctx->no_persistent_gemm) {
    return a->dtype == CTS_BF16 ? launch_persistent<__nv_bfloat16>(ctx, a, st) : launch_persistent<__half>(ctx, a, st);
  }
  CTS_CHECK_ARG(ctx, a->epilogue != CTS_EPI_SWIGLU_IL, "CTS_EPI_SWIGLU_IL is only implemented by the persistent kernel");
  const bool dual = a->epilogue == CTS_EPI_SWIGLU;
  if (a->dtype == CTS_BF16)
    return dual ? dispatch_bn<__nv_bfloat16, true>(ctx, a, st) : dispatch_bn<__nv_bfloat16, false>(ctx, a, st);
  return dual ? dispatch_bn<__half, true>(ctx, a, st) : dispatch_bn<__half, false>(ctx, a, st);
}

extern "C" int cts_gemm_suggest_split(cts_ctx* ctx, long long n, long long k, long long t, int dual) {
  if (!ctx || n <= 0 || k <= 0 || t <= 0) return 1;
  const int bn = t <= 16 ? 16 : t <= 32 ? 32 : t <= 64 ? 64 : 128;
  // dual = 1: the caller passes n = intermediate size of an INTERLEAVED gate/up weight, whose GEMM has 2 n / 128 tiles, counted against
  // three slots per SM instead of two (on 132 SMs: 216 tiles at the 14B shape, split 1).  The factors fix the partial planes the reduce
  // tails read and the fp32 order of their sum; gemm_stream_kernel deals the resulting (tile, split) units over its persistent CTAs, so
  // they no longer have to match a number of resident CTAs.
  const long long tiles = cdiv_ll(dual ? 2 * n : n, kBM) * cdiv_ll(t, bn);
  const long long kb = cdiv_ll(k, kBK);
  const long long slots = (long long)ctx->sm_count * (bn <= 128 ? (dual && bn <= 32 ? 3 : 2) : 1);
  if (tiles >= slots) return 1;
  long long s = slots / tiles;
  // keep >= 8 K blocks (1 KiB of each weight row) per split -- except at decode-sized t, where a short K range per CTA is exactly
  // what a latency-bound launch wants (tensor-parallel shards: o_proj at TP8 has 10 K blocks; one CTA per tile would walk them
  // serially through a 3-stage ring): there 2 blocks per split suffice
  const long long per_split_min = bn <= 32 ? 2 : 8;
  const long long max_by_k = kb / per_split_min > 0 ? kb / per_split_min : 1;
  if (s > max_by_k) s = max_by_k;
  if (s > 16) s = 16;
  if (s < 1) s = 1;
  return (int)s;
}

CTS_TRACE_SETTER(cts_trace_set_gemm)
