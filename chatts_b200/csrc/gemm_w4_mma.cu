// chatts_b200 -- W4A16 decode GEMM, register-operand version (GPTQ-Int4 checkpoints, README.md:52,262-263):
//     partial[s][t][n] = sum_{k in split s} x[t][k] * sc[n][k / g] * (q[n][k] - zp[n][k / g])        (fp32 accumulate)
// Why a second kernel: gemm_w4.cu keeps the wgmma structure and writes the dequantised 16-bit tile to shared memory for the tensor
// core to read back; per 128 x 64 block that is 16 KB written + 18 KB read by the MMA + the 4-bit tile in and out = 44 KB through a
// 128 B/clk shared-memory port, i.e. at most ~24 weights per clock and SM where HBM delivers 46 -- the kernel measured NO faster than
// the bf16 GEMM.  Here the weight operand never touches shared memory as 16-bit data:
//   * load-time layout (weights.py:repack_w4_mma): for every (256-feature tile, 64-K block) one contiguous 8 KB chunk whose 32-bit
//     words ARE the A fragments of mma.sync.m16n8k16 -- lane (g, t) of m-tile j finds, for each of the block's four k16 steps, one
//     word holding the 8 codes {rows g / g+8} x {k 2t, 2t+1, 2t+8, 2t+9} in the nibble order that `(w >> 4i) & 0x000F000F` turns
//     into fragment register a_i; next to it 1 KB of {scale, 128+zero-point} pairs of the block's group
//   * warp 8, one lane: per 128-K pipeline stage one cp.async.bulk of 16 KB of codes (evict-first) + the group's scales, issued for the
//     whole ring BEFORE the dependency wait (nobody writes weights), and -- after the wait -- the two token tiles [8 NT rows x 64 K] by
//     TMA (128B swizzle) onto the SAME barrier: one wait and one arrival per stage and warp (3-5 stages of 19-25 KB per CTA, two or
//     three CTAs per SM = 150-200 KB in flight per SM)
//   * warps 0..7: one LDS.128 per m-tile and 64-K block = the fragments of four k16 steps; int4 -> bf16/fp16 in registers with the magic-number trick
//     of gemm_w4.cu (exactly the value dequantize_w4 stores for the prefill copy); B fragments by ldmatrix from the swizzled token
//     tile; mma.sync with the fp32 accumulators of 2 m-tiles x NT n-tiles in registers
//   * persistent CTAs over (tile, K split) units, the producers run ahead across unit boundaries
// What the loop is bound by, measured: instruction issue on the ALU side plus barrier round trips -- 57-59 % issue-active with six warps
// per scheduler at 64-96 registers, ALU pipe ~50 %, FMA pipe ~25 %.  Two experiments bracket it:
//   * rejected: feeding the MMA the pairs (128 + code) themselves and applying the
//     group's scale / zero point in fp32 once per group and accumulator (no HADD2 / HMUL2 per weight, one more MMA per k16 step with an
//     all-ones A operand for sum_k x_k) removed a quarter of the loop's instructions -- all of them FMA-pipe work that was overlapping for
//     free -- and was NOT faster (gate_up at t = 1: 26.7 us against 25.8);
//   * kept: going from 64-K stages on two rings to 128-K stages on one ring halves the waits, arrivals, ring steps and scale fetches per
//     weight (all ALU / control work): 25.8 -> 19.9 us.
// Output: the fp32 split-K partials [split, t, n] of CTS_EPI_PARTIAL_F32, so the decode step's reduce tails are unchanged.  The A
// operand holds the same 16-bit values as the dense copy; the fp32 summation order differs from the wgmma GEMM (parity is a
// tolerance, tests/test_gpu_w4.py), unlike gemm_w4.cu which is bit-identical and stays as the checker for this kernel.
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"
#ifndef CTS_DYN_SMEM
#define CTS_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#endif
#include "tensormap.cuh"

namespace {

constexpr int kTileN = 256, kBK = 64, kWarps = 8;
constexpr int kKS = 2;                               // K blocks per pipeline stage: one barrier round trip, one ring step, one scale fetch per 128 K
constexpr int kWBytes = kTileN * kBK / 2;            // 8192: the codes of one (tile, K block)
constexpr int kSzBytes = kTileN * 4;                 // 1024: {scale bits | (magic + zero point) << 16} per feature of one group
constexpr int kThreads = (kWarps + 1) * 32;          // eight compute warps + one producer warp
constexpr int kMaxStages = 12;

struct W4mParams {
  long long n, k, t;
  int ks_total, split_k, kb_per_group, n_groups, tiles, stages, sz_groups;   // ks_total = K / 128; sz_groups = group entries a stage carries (2 at group size 64, else 1)
  const uint8_t* qw;       // [tiles][K / 64][8192]
  const uint8_t* szp;      // [tiles][n_groups][1024]
  float* out;              // fp32 [split_k, t, n]
};

template <typename T> struct MagicM;
template <> struct MagicM<__nv_bfloat16> {
  static constexpr uint32_t kOr = 0x43004300u;                       // bf16 128.0 in both halves: 128 + code (ulp 1 in [128, 256))
  // y = the pair 128 + code; (y - (128 + zp)) is an exact small integer, times the scale = ONE rounding = dequantize_w4's value
  static __device__ __forceinline__ uint32_t sub_mul(uint32_t y, uint32_t b2, uint32_t s2) {
    __nv_bfloat162 d = __hsub2(*reinterpret_cast<const __nv_bfloat162*>(&y), *reinterpret_cast<const __nv_bfloat162*>(&b2));
    __nv_bfloat162 w = __hmul2(d, *reinterpret_cast<const __nv_bfloat162*>(&s2));
    return *reinterpret_cast<uint32_t*>(&w);
  }
};
template <> struct MagicM<__half> {
  static constexpr uint32_t kOr = 0x64006400u;                       // fp16 1024.0: 1024 + code
  static __device__ __forceinline__ uint32_t sub_mul(uint32_t y, uint32_t b2, uint32_t s2) {
    __half2 d = __hsub2(*reinterpret_cast<const __half2*>(&y), *reinterpret_cast<const __half2*>(&b2));
    __half2 w = __hmul2(d, *reinterpret_cast<const __half2*>(&s2));
    return *reinterpret_cast<uint32_t*>(&w);
  }
};

// a constant the compiler must keep in a register (so that (w & mask) | magic is ONE lop3 with three register operands)
__device__ __forceinline__ uint32_t w4m_opaque(uint32_t v) {
#ifndef CTS_HOST_SHIM
  uint32_t r;
  asm volatile("mov.b32 %0, %1;" : "=r"(r) : "r"(v));
  return r;
#else
  return v;
#endif
}
__device__ __forceinline__ uint32_t w4m_and_or(uint32_t a, uint32_t m, uint32_t k) {
#ifndef CTS_HOST_SHIM
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(m), "r"(k));       // (a & m) | k
  return d;
#else
  return (a & m) | k;
#endif
}
__device__ __forceinline__ void w4m_ldsm_x4(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
template <typename T> __device__ __forceinline__ void w4m_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void w4m_mma<__nv_bfloat16>(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void w4m_mma<__half>(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// the weight stream is read once: evict-first, as the TMA tiles of the dense GEMM
__device__ __forceinline__ void w4m_bulk_stream(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
#ifndef CTS_HOST_SHIM
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(CTS_L2_EVICT_FIRST)
               : "memory");
#else
  bulk_load_1d(smem_dst, gsrc, bytes, bar);
#endif
}

// unit u of the persistent schedule -> (tile, split, range of 128-K stages)
__device__ __forceinline__ void w4m_unit(const W4mParams& p, int u, int& tile, int& split, int& ks0, int& ks1) {
  tile = u % p.tiles;
  split = u / p.tiles;
  ks0 = (int)(((long long)p.ks_total * split) / p.split_k);
  ks1 = (int)(((long long)p.ks_total * (split + 1)) / p.split_k);
}

// One pipeline stage in shared memory: [token tile of K block 0 | token tile of K block 1 | 16 KB of codes | sz_groups KB of scales / zero
// points], 1 KB aligned (the 128B swizzle of the token tiles repeats every 8 rows).
template <typename T, int NT>
__global__ void __launch_bounds__(kThreads, NT == 1 ? 3 : 2)
gemm_w4_mma_kernel(const __grid_constant__ CUtensorMap tm_x, const W4mParams p) {
  CTS_DYN_SMEM(smem_raw);
  __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];

  constexpr int kXBytes = NT * 8 * kBK * 2;                 // token tile of one K block: 8 NT rows of 128 bytes
  constexpr int kXStage = kKS * kXBytes;
  const int stage_bytes = kXStage + kKS * kWBytes + p.sz_groups * kSzBytes;
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* ring = smem_raw + (((raw + 1023u) & ~1023u) - raw);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.stages;
  const int units = p.tiles * p.split_k;

  pdl_trigger();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_x);
    for (int s = 0; s < S; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kWarps); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kWarps) {
    // ------------------------------ producer: codes + scales (static: requested BEFORE the dependency wait), token tiles after it ------------------------------
    if (lane == 0) {
      auto issue_static = [&](int s, int tile, int ks) {
        uint8_t* dst = ring + (size_t)s * stage_bytes + kXStage;
        mbar_expect_tx(&full_bar[s], (uint32_t)stage_bytes);
        w4m_bulk_stream(dst, p.qw + ((size_t)tile * (p.ks_total * kKS) + (size_t)ks * kKS) * kWBytes, (uint32_t)(kKS * kWBytes), &full_bar[s]);
        const int grp = (ks * kKS) / p.kb_per_group;          // first group the stage touches (sz_groups = 2: the two blocks are two groups)
        bulk_load_1d(dst + kKS * kWBytes, p.szp + ((size_t)tile * p.n_groups + grp) * kSzBytes, (uint32_t)(p.sz_groups * kSzBytes), &full_bar[s]);
      };
      auto issue_tokens = [&](int s, int ks) {
        uint8_t* dst = ring + (size_t)s * stage_bytes;
#pragma unroll
        for (int b = 0; b < kKS; ++b) tma_load_2d(dst + b * kXBytes, &tm_x, &full_bar[s], (ks * kKS + b) * kBK, 0, CTS_L2_EVICT_LAST);
      };
      // the first S stages of this CTA's schedule: static part now, token tiles once the predecessor has finished
      int pre = 0;
      {
        int s = 0;
        for (int u = blockIdx.x; u < units && s < S; u += gridDim.x) {
          int tile, split, ks0, ks1;
          w4m_unit(p, u, tile, split, ks0, ks1);
          for (int ks = ks0; ks < ks1 && s < S; ++ks, ++s) issue_static(s, tile, ks);
        }
        pre = s;
      }
      pdl_wait();
      int s = 0, n = 0;
      uint32_t ph = 1u;                                      // parity of the "slot is empty" phase being waited for (fresh barrier: passes)
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        int tile, split, ks0, ks1;
        w4m_unit(p, u, tile, split, ks0, ks1);
        for (int ks = ks0; ks < ks1; ++ks, ++n) {
          if (n >= pre) {
            mbar_wait(&empty_bar[s], ph);
            issue_static(s, tile, ks);
          }
          issue_tokens(s, ks);
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // ------------------------------ dequantise in registers + mma.sync ------------------------------
    // The loop is instruction-issue bound (ncu: 57-59 % issue-active with six warps per scheduler, `wait` the top stall), so per 64-K
    // block only what the arithmetic needs is left -- 2 LDS.128, 8 x (3 shifts + 4 lop3 + 4 HADD2 + 4 HMUL2), the ldmatrix of the token
    // fragments, the MMAs -- and everything else is paid once per 128-K stage: ONE barrier wait and ONE arrival (codes, scales and both
    // token tiles share the stage's barrier), one scale fetch, one ring step.
    const int g = lane >> 2, tq = lane & 3;
    const int lrow = lane & 7, lmat = lane >> 3;             // ldmatrix: this lane supplies row `lrow` of matrix `lmat`
    float acc[2][NT][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[mi][nt][j] = 0.f;
    uint32_t sA[2] = {0, 0}, bA[2] = {0, 0}, sB[2] = {0, 0}, bB[2] = {0, 0};   // {scale, magic + zp} of rows g / g + 8 of the two m-tiles
    const uint32_t kMask = w4m_opaque(0x000F000Fu), kMagic = w4m_opaque(MagicM<T>::kOr);
    const uint32_t w_off = (uint32_t)(kXStage + (warp * 2 * 32 + lane) * 16);   // this lane's word quadruple of m-tile 2 warp (+ 512: m-tile 2 warp + 1)
    const uint32_t sz_off = (uint32_t)(kXStage + kKS * kWBytes + (warp * 2 * 16 + g) * 4);
    // ldmatrix row addresses inside a token tile for k16 step 0; step ks: XOR with ks << 5 (the chunk index 2 ks + h enters the 128B swizzle by XOR)
    uint32_t x_off[NT == 1 ? 1 : NT / 2];
    if constexpr (NT == 1) {
      x_off[0] = (uint32_t)(lrow * 128 + (((2 * (lmat >> 1) + (lmat & 1)) ^ lrow) << 4));          // matrices (ks, half) = (0,0), (0,1), (1,0), (1,1); pair q: XOR q << 6
    } else {
#pragma unroll
      for (int pr = 0; pr < NT / 2; ++pr) x_off[pr] = (uint32_t)(((2 * pr + (lmat >> 1)) * 8 + lrow) * 128 + (((lmat & 1) ^ lrow) << 4));
    }
    const bool per_block_groups = p.sz_groups == 2;          // group size 64: each K block of a stage has its own scales
    int s = 0;
    uint32_t ph = 0u;                                        // parity of the "slot is full" phase
    const uint8_t* st = ring;                                // slot s
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      int tile, split, ks0, ks1;
      w4m_unit(p, u, tile, split, ks0, ks1);
      for (int ks = ks0; ks < ks1; ++ks) {
        mbar_wait(&full_bar[s], ph);
#pragma unroll
        for (int b = 0; b < kKS; ++b) {
          uint4 wv[2];
          wv[0] = *reinterpret_cast<const uint4*>(st + w_off + b * kWBytes);
          wv[1] = *reinterpret_cast<const uint4*>(st + w_off + b * kWBytes + 512);
          if (b == 0 || per_block_groups) {
            const uint8_t* sz = st + sz_off + (per_block_groups ? b * kSzBytes : 0);
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
              const uint32_t va = *reinterpret_cast<const uint32_t*>(sz + mi * 64), vb = *reinterpret_cast<const uint32_t*>(sz + mi * 64 + 32);
              sA[mi] = (va & 0xFFFFu) * 0x00010001u; bA[mi] = (va >> 16) * 0x00010001u;      // both halves of a packed pair
              sB[mi] = (vb & 0xFFFFu) * 0x00010001u; bB[mi] = (vb >> 16) * 0x00010001u;
            }
          }
          const uint32_t xs = smem_u32(st) + (uint32_t)(b * kXBytes);
          uint32_t rq[4] = {0u, 0u, 0u, 0u};                  // NT == 1: the fragments of a pair of k16 steps
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            uint32_t bf[NT][2];                               // B fragments of this k16 step
            if constexpr (NT == 1) {
              if ((kk & 1) == 0) w4m_ldsm_x4((xs + x_off[0]) ^ (uint32_t)((kk >> 1) << 6), rq);
              bf[0][0] = (kk & 1) ? rq[2] : rq[0]; bf[0][1] = (kk & 1) ? rq[3] : rq[1];
            } else {
              // one ldmatrix.x4 = one k16 step of two 8-token tiles: matrices (nt, half) = (2p, 0), (2p, 1), (2p + 1, 0), (2p + 1, 1)
#pragma unroll
              for (int pr = 0; pr < NT / 2; ++pr) {
                uint32_t r[4];
                w4m_ldsm_x4((xs + x_off[pr]) ^ (uint32_t)(kk << 5), r);
                bf[2 * pr][0] = r[0]; bf[2 * pr][1] = r[1]; bf[2 * pr + 1][0] = r[2]; bf[2 * pr + 1][1] = r[3];
              }
            }
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
              const uint32_t w = kk == 0 ? wv[mi].x : kk == 1 ? wv[mi].y : kk == 2 ? wv[mi].z : wv[mi].w;
              uint32_t a[4];
              a[0] = MagicM<T>::sub_mul(w4m_and_or(w, kMask, kMagic), bA[mi], sA[mi]);
              a[1] = MagicM<T>::sub_mul(w4m_and_or(w >> 4, kMask, kMagic), bB[mi], sB[mi]);
              a[2] = MagicM<T>::sub_mul(w4m_and_or(w >> 8, kMask, kMagic), bA[mi], sA[mi]);
              a[3] = MagicM<T>::sub_mul(w4m_and_or(w >> 12, kMask, kMagic), bB[mi], sB[mi]);
#pragma unroll
              for (int nt = 0; nt < NT; ++nt) w4m_mma<T>(acc[mi][nt], a, bf[nt][0], bf[nt][1]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[s]);          // every word of the slot has been consumed into registers by all lanes of this warp
        st += stage_bytes;
        if (++s == S) { s = 0; ph ^= 1u; st = ring; }
      }
      // ---- the unit's fp32 partial: c0/c1 = (row g, tokens 2t, 2t+1), c2/c3 = (row g + 8, same tokens)
      float* dst = p.out + (long long)split * p.t * p.n;
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const long long f = (long long)tile * kTileN + (warp * 2 + mi) * 16 + g;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const long long tk = nt * 8 + 2 * tq;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const long long ff = f + (j >> 1) * 8, tt = tk + (j & 1);
            if (tt < p.t && ff < p.n) dst[tt * p.n + ff] = acc[mi][nt][j];
            acc[mi][nt][j] = 0.f;
          }
        }
      }
    }
  }
}

// Resident CTAs per SM: three of the t <= 8 kernel (64 registers) when the projection has enough 256-feature tiles to give every CTA a
// long unit (gate_up: 108 tiles), else two with deeper rings
static inline int w4m_ctas_per_sm(long long tiles, long long t) {
  static const int forced = [] { const char* e = getenv("CTS_W4M_CTAS"); return e ? atoi(e) : 0; }();      // A/B knob (2 or 3)
  if (forced == 2 || (forced == 3 && t <= 8)) return forced;
  return (t <= 8 && tiles >= 64) ? 3 : 2;
}

template <typename T, int NT>
int launch_w4m(cts_ctx* ctx, const cts_gemm_w4f_args* a, cudaStream_t stream) {
  const bool is_bf16 = a->dtype == CTS_BF16;
  CUtensorMap tm_x;
  int rc = cts_make_tmap_2d(ctx, &tm_x, a->x, a->t, a->k, a->x_ld, NT * 8, is_bf16);
  if (rc) return rc;
  W4mParams p;
  p.n = a->n; p.k = a->k; p.t = a->t;
  p.ks_total = (int)(a->k / (kKS * kBK));
  p.split_k = a->split_k;
  p.kb_per_group = a->group_size / kBK;
  p.n_groups = (int)(a->k / a->group_size);
  p.sz_groups = p.kb_per_group == 1 ? kKS : 1;
  p.tiles = (int)cdiv_ll(a->n, kTileN);
  p.qw = (const uint8_t*)a->qw; p.szp = (const uint8_t*)a->szp; p.out = a->out;
  constexpr int kXBytes = NT * 8 * kBK * 2;
  const int stage_bytes = kKS * kXBytes + kKS * kWBytes + p.sz_groups * kSzBytes;
  // CTAs per SM (w4m_ctas_per_sm): the ring of each takes what its share of the shared memory leaves after the static part
  const int kCtas = w4m_ctas_per_sm(p.tiles, a->t);
  const int budget = (ctx->max_smem_optin > 0 ? ctx->max_smem_optin + 1024 : 228 * 1024) / kCtas - 3 * 1024;
  int st = (budget - 1024) / stage_bytes;
  if (st > kMaxStages) st = kMaxStages;
  if (st < 2) return cts_set_error(ctx, CTS_ERR_BAD_ARG, "cts_gemm_w4_mma: shared memory budget too small");
  p.stages = st;
  const size_t smem = (size_t)st * stage_bytes + 1024;
  auto kern = gemm_w4_mma_kernel<T, NT>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
#ifndef CTS_HOST_SHIM
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
#endif
  const long long units = (long long)p.tiles * p.split_k;
  long long grid = (long long)kCtas * ctx->sm_count;
  if (grid > units) grid = units;
  CTS_CUDA(ctx, launch_pdl(kern, dim3((unsigned)grid), dim3(kThreads), smem, stream, 1, tm_x, p));
  return CTS_OK;
}

}  // namespace

// split-K factor of the persistent schedule: units = tiles x split are dealt round-robin to the resident CTAs (w4m_ctas_per_sm); the
// cost of a choice is the longest CTA's stream in 16 KB stages plus the partial it writes per unit (t KB of fp32 = t / 16 stage equivalents)
extern "C" int cts_gemm_w4_mma_suggest_split(cts_ctx* ctx, long long n, long long k, long long t) {
  if (!ctx || n <= 0 || k <= 0) return 1;
  const long long tiles = cdiv_ll(n, kTileN), ks = k / (kKS * kBK), ctas = (long long)w4m_ctas_per_sm(tiles, t) * ctx->sm_count;
  long long best = 1;
  double best_cost = 1e30;
  for (long long s = 1; s <= 16 && s * 2 <= ks; ++s) {
    const long long waves = cdiv_ll(tiles * s, ctas);
    const double cost = (double)waves * ((double)cdiv_ll(ks, s) + (double)(t < 1 ? 1 : t) / 16.0 + 0.5);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = s; }
  }
  return (int)best;
}

extern "C" int cts_gemm_w4_mma(cts_ctx* ctx, const cts_gemm_w4f_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr && a->qw && a->szp && a->x && a->out, "null pointer");
  CTS_CHECK_ARG(ctx, a->n > 0 && a->k > 0 && a->t > 0 && a->t <= 32, "n, k > 0 and 1 <= t <= 32 (decode-sized step; prefill uses the dequantised weight)");
  CTS_CHECK_ARG(ctx, a->dtype == CTS_BF16 || a->dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, a->k % 128 == 0, "k must be a multiple of 128 (a pipeline stage is two 64-K blocks)");
  CTS_CHECK_ARG(ctx, a->group_size >= 64 && a->group_size % 64 == 0 && a->k % a->group_size == 0 && (a->group_size == 64 || a->group_size % 128 == 0),
                "group_size must be 64 or a multiple of 128, and divide k");
  CTS_CHECK_ARG(ctx, a->split_k >= 1 && a->split_k <= a->k / 128, "split_k");
  CTS_CHECK_ARG(ctx, a->x_ld >= a->k, "x_ld smaller than k");
  CTS_CHECK_ARG(ctx, (((uintptr_t)a->qw | (uintptr_t)a->szp) & 15) == 0, "qw / szp must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dtype == CTS_BF16)
    return a->t <= 8 ? launch_w4m<__nv_bfloat16, 1>(ctx, a, st) : a->t <= 16 ? launch_w4m<__nv_bfloat16, 2>(ctx, a, st) : launch_w4m<__nv_bfloat16, 4>(ctx, a, st);
  return a->t <= 8 ? launch_w4m<__half, 1>(ctx, a, st) : a->t <= 16 ? launch_w4m<__half, 2>(ctx, a, st) : launch_w4m<__half, 4>(ctx, a, st);
}
