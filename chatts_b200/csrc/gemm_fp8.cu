// chatts_b200 -- W8A16 decode GEMM for FP8 (e4m3) weights with per-output-channel scales (ChatTSForCausalLM.quantize_fp8):
//     partial[s][t][n] = s_n * sum_{k in split s} x[t][k] * e4m3(q[n][k])        (fp32 accumulate, the scale applied once in fp32)
// and cts_fp8_dequant, which writes one projection back as a row-major 16-bit matrix for the prefill-sized GEMMs.
// Structure of csrc/gemm_w4_mma.cu, one byte per weight instead of half a byte:
//   * load-time layout (weights.py:pack_fp8_mma): for every (256-feature tile, 64-K block) one contiguous 16 KB chunk whose 32-bit words
//     ARE the A fragments of mma.sync.m16n8k16 -- lane (g, t) of m-tile m finds, for k16 step ks, two words: {a0 | a1} = the codes of
//     rows g / g + 8 at k 2t, 2t + 1 and {a2 | a3} = the same rows at k 2t + 8, 2t + 9 (low byte = lower k = low half of the register);
//     the words of k16 steps {0, 1} and {2, 3} are two LDS.128 per lane, laid out lane-contiguous (no bank conflict)
//   * warp 8, one lane: per 64-K pipeline stage one cp.async.bulk of the 16 KB of codes (evict-first), issued for the whole ring
//     BEFORE the dependency wait (nobody writes weights), and -- after the wait -- the token tile [8 NT rows x 64 K] by TMA (128B
//     swizzle) onto the SAME barrier
//   * warps 0..7: e4m3 -> 16-bit in registers, B fragments by ldmatrix from the swizzled token tile, mma.sync with the fp32 accumulators
//     of 2 m-tiles x NT n-tiles in registers; the row scale multiplies the accumulator once per (unit, row), so the streamed loop carries
//     no scale traffic at all
//   * persistent CTAs over (tile, K split) units, the producers run ahead across unit boundaries
// Conversion, exact for all 254 finite codes (subnormals and -0 included):
//   * fp16: cvt.rn.f16x2.e4m3x2 -- every e4m3 value is an fp16 normal (2^-9 .. 448) or zero
//   * bf16: there is no e4m3 -> bf16 instruction.  The fp16 pattern of the same code, shifted right by 3 with its sign kept, IS a bf16
//     pattern: fp16 exponent field e becomes the bf16 exponent field e, so the value is e4m3 * 2^(15 - 127) = e4m3 * 2^-112, and since the
//     fp16 exponent field of a non-zero code is >= 6 the bf16 operand is a normal number (2^-121 .. 448 * 2^-112), never a subnormal the
//     tensor core could flush.  The accumulator is multiplied by 2^112 (exact) before the row scale.  Four instructions per register
//     (cvt, shift, two lop3) against one for fp16.
// mma.sync, not wgmma with A from registers (the m16n8k16 A fragment is also wgmma's m64k16 register-A layout, one warp per 16 rows, so
// this packing could feed either): only the mma.sync kernel was built and measured.  On an H100 (400 W power limit) it takes 52 us for
// ChatTS-14B's gate_up at t = 1 (27648 x 5120 codes, 2.7 TB/s) against 124 us for the bf16 split-K GEMM; a wgmma variant is untested.
// Output: the fp32 split-K partials [split, t, n] of CTS_EPI_PARTIAL_F32, so the decode step's reduce tails are unchanged.
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"
#ifndef CTS_DYN_SMEM
#define CTS_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#endif
#include "tensormap.cuh"

namespace {

constexpr int kTileN = 256, kBK = 64, kWarps = 8;
constexpr int kWBytes = kTileN * kBK;                // 16384: the codes of one (tile, K block)
constexpr int kThreads = (kWarps + 1) * 32;          // eight compute warps + one producer warp
constexpr int kMaxStages = 12;

struct F8Params {
  long long n, k, t;
  int kb_total, split_k, tiles, stages;              // kb_total = K / 64
  const uint8_t* qw;       // [tiles][K / 64][16384]
  const float* scales;     // fp32 [n]
  float* out;              // fp32 [split_k, t, n]
};

#ifdef CTS_HOST_SHIM
static inline uint32_t f8_shim_f16(uint32_t b) {       // one e4m3 code -> fp16 bits (exact)
  const uint32_t e = (b >> 3) & 15u, m = b & 7u;
  const float v = e ? ldexpf(1.0f + (float)m / 8.0f, (int)e - 7) : ldexpf((float)m, -9);
  return (uint32_t)__float2half_rn(v).bits | ((b & 0x80u) << 8);
}
#endif

// the four e4m3 codes of a word -> two f16x2 registers (bytes 0, 1 -> lo; bytes 2, 3 -> hi; lower byte = lower half)
__device__ __forceinline__ void f8_to_f16x2(uint32_t w, uint32_t& lo, uint32_t& hi) {
#ifndef CTS_HOST_SHIM
  asm("{ .reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.rn.f16x2.e4m3x2 %0, l;\n\tcvt.rn.f16x2.e4m3x2 %1, h; }" : "=r"(lo), "=r"(hi) : "r"(w));
#else
  lo = f8_shim_f16(w & 0xFFu) | (f8_shim_f16((w >> 8) & 0xFFu) << 16);
  hi = f8_shim_f16((w >> 16) & 0xFFu) | (f8_shim_f16(w >> 24) << 16);
#endif
}

// f16x2 of e4m3 values -> bf16x2 of the same values times 2^-112 (see the header)
__device__ __forceinline__ uint32_t f8_f16_to_bf16_scaled(uint32_t h) { return ((h >> 3) & 0x0FFF0FFFu) | (h & 0x80008000u); }

template <typename T> struct F8Conv;
template <> struct F8Conv<__half> {
  static constexpr float kUnscale = 1.0f;
  static __device__ __forceinline__ void cvt(uint32_t w, uint32_t& lo, uint32_t& hi) { f8_to_f16x2(w, lo, hi); }
};
template <> struct F8Conv<__nv_bfloat16> {
  static constexpr float kUnscale = 5192296858534827628530496329220096.0f;      // 2^112
  static __device__ __forceinline__ void cvt(uint32_t w, uint32_t& lo, uint32_t& hi) {
    f8_to_f16x2(w, lo, hi);
    lo = f8_f16_to_bf16_scaled(lo);
    hi = f8_f16_to_bf16_scaled(hi);
  }
};

__device__ __forceinline__ void f8_ldsm_x4(uint32_t addr, uint32_t* r) {
#ifndef CTS_HOST_SHIM
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
#else
  shim_ldmatrix_x4(addr, r, false);
#endif
}
template <typename T> __device__ __forceinline__ void f8_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void f8_mma<__nv_bfloat16>(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
#ifndef CTS_HOST_SHIM
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
#else
  shim_mma_m16n8k16(c, a, b0, b1, true);
#endif
}
template <> __device__ __forceinline__ void f8_mma<__half>(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
#ifndef CTS_HOST_SHIM
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
#else
  shim_mma_m16n8k16(c, a, b0, b1, false);
#endif
}
// the weight stream is read once: evict-first
__device__ __forceinline__ void f8_bulk_stream(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
#ifndef CTS_HOST_SHIM
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(CTS_L2_EVICT_FIRST)
               : "memory");
#else
  bulk_load_1d(smem_dst, gsrc, bytes, bar);
#endif
}

// unit u of the persistent schedule -> (tile, split, range of 64-K blocks)
__device__ __forceinline__ void f8_unit(const F8Params& p, int u, int& tile, int& split, int& kb0, int& kb1) {
  tile = u % p.tiles;
  split = u / p.tiles;
  kb0 = (int)(((long long)p.kb_total * split) / p.split_k);
  kb1 = (int)(((long long)p.kb_total * (split + 1)) / p.split_k);
}

// One pipeline stage in shared memory: [token tile of the K block (NT KB) | 16 KB of codes], 1 KB aligned (the 128B swizzle of the
// token tile repeats every 8 rows).
template <typename T, int NT>
__global__ void __launch_bounds__(kThreads, NT == 1 ? 3 : 2)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tm_x, const F8Params p) {
  CTS_DYN_SMEM(smem_raw);
  __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];

  constexpr int kXBytes = NT * 8 * kBK * 2;                 // token tile: 8 NT rows of 128 bytes
  constexpr int kStage = kXBytes + kWBytes;
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
    // ------------------------------ producer: codes (static: requested BEFORE the dependency wait), token tiles after it ------------------------------
    if (lane == 0) {
      auto issue_static = [&](int s, int tile, int kb) {
        mbar_expect_tx(&full_bar[s], (uint32_t)kStage);
        f8_bulk_stream(ring + (size_t)s * kStage + kXBytes, p.qw + ((size_t)tile * p.kb_total + (size_t)kb) * kWBytes, (uint32_t)kWBytes, &full_bar[s]);
      };
      int pre = 0;
      {
        int s = 0;
        for (int u = blockIdx.x; u < units && s < S; u += gridDim.x) {
          int tile, split, kb0, kb1;
          f8_unit(p, u, tile, split, kb0, kb1);
          for (int kb = kb0; kb < kb1 && s < S; ++kb, ++s) issue_static(s, tile, kb);
        }
        pre = s;
      }
      pdl_wait();
      int s = 0, n = 0;
      uint32_t ph = 1u;                                      // parity of the "slot is empty" phase being waited for (fresh barrier: passes)
      for (int u = blockIdx.x; u < units; u += gridDim.x) {
        int tile, split, kb0, kb1;
        f8_unit(p, u, tile, split, kb0, kb1);
        for (int kb = kb0; kb < kb1; ++kb, ++n) {
          if (n >= pre) {
            mbar_wait(&empty_bar[s], ph);
            issue_static(s, tile, kb);
          }
          tma_load_2d(ring + (size_t)s * kStage, &tm_x, &full_bar[s], kb * kBK, 0, CTS_L2_EVICT_LAST);
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // ------------------------------ e4m3 -> 16-bit in registers + mma.sync ------------------------------
    const int g = lane >> 2, tq = lane & 3;
    const int lrow = lane & 7, lmat = lane >> 3;             // ldmatrix: this lane supplies row `lrow` of matrix `lmat`
    float acc[2][NT][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[mi][nt][j] = 0.f;
    // this lane's first word quadruple: m-tile 2 warp, k16 steps {0, 1}; + 512: steps {2, 3}; + 1024: m-tile 2 warp + 1
    const uint32_t w_off = (uint32_t)(kXBytes + warp * 4 * 512 + lane * 16);
    // ldmatrix row addresses inside the token tile for k16 step 0; step kk: XOR (the chunk index 2 kk + h enters the 128B swizzle by XOR)
    uint32_t x_off[NT == 1 ? 1 : NT / 2];
    if constexpr (NT == 1) {
      x_off[0] = (uint32_t)(lrow * 128 + (((2 * (lmat >> 1) + (lmat & 1)) ^ lrow) << 4));          // matrices (kk, half) = (0,0), (0,1), (1,0), (1,1); pair q: XOR q << 6
    } else {
#pragma unroll
      for (int pr = 0; pr < NT / 2; ++pr) x_off[pr] = (uint32_t)(((2 * pr + (lmat >> 1)) * 8 + lrow) * 128 + (((lmat & 1) ^ lrow) << 4));
    }
    int s = 0;
    uint32_t ph = 0u;                                        // parity of the "slot is full" phase
    const uint8_t* st = ring;                                // slot s
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
      int tile, split, kb0, kb1;
      f8_unit(p, u, tile, split, kb0, kb1);
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[s], ph);
        uint4 wv[2][2];                                      // [m-tile][k16 step pair]
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
          for (int h = 0; h < 2; ++h) wv[mi][h] = *reinterpret_cast<const uint4*>(st + w_off + mi * 1024 + h * 512);
        const uint32_t xs = smem_u32(st);
        uint32_t rq[4] = {0u, 0u, 0u, 0u};                  // NT == 1: the B fragments of a pair of k16 steps
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          uint32_t bf[NT][2];
          if constexpr (NT == 1) {
            if ((kk & 1) == 0) f8_ldsm_x4((xs + x_off[0]) ^ (uint32_t)((kk >> 1) << 6), rq);
            bf[0][0] = (kk & 1) ? rq[2] : rq[0]; bf[0][1] = (kk & 1) ? rq[3] : rq[1];
          } else {
#pragma unroll
            for (int pr = 0; pr < NT / 2; ++pr) {
              uint32_t r[4];
              f8_ldsm_x4((xs + x_off[pr]) ^ (uint32_t)(kk << 5), r);
              bf[2 * pr][0] = r[0]; bf[2 * pr][1] = r[1]; bf[2 * pr + 1][0] = r[2]; bf[2 * pr + 1][1] = r[3];
            }
          }
#pragma unroll
          for (int mi = 0; mi < 2; ++mi) {
            const uint4& q = wv[mi][kk >> 1];
            const uint32_t w01 = (kk & 1) ? q.z : q.x, w23 = (kk & 1) ? q.w : q.y;
            uint32_t a[4];
            F8Conv<T>::cvt(w01, a[0], a[1]);
            F8Conv<T>::cvt(w23, a[2], a[3]);
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) f8_mma<T>(acc[mi][nt], a, bf[nt][0], bf[nt][1]);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[s]);          // codes and token tile of the slot have been consumed by all lanes of this warp
        st += kStage;
        if (++s == S) { s = 0; ph ^= 1u; st = ring; }
      }
      // ---- the unit's fp32 partial: c0/c1 = (row g, tokens 2t, 2t+1), c2/c3 = (row g + 8, same tokens), times the row scale
      float* dst = p.out + (long long)split * p.t * p.n;
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const long long f = (long long)tile * kTileN + (warp * 2 + mi) * 16 + g;
        const float s0 = f < p.n ? p.scales[f] : 0.f, s1 = f + 8 < p.n ? p.scales[f + 8] : 0.f;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const long long tk = nt * 8 + 2 * tq;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const long long ff = f + (j >> 1) * 8, tt = tk + (j & 1);
            if (tt < p.t && ff < p.n) dst[tt * p.n + ff] = (acc[mi][nt][j] * F8Conv<T>::kUnscale) * ((j >> 1) ? s1 : s0);
            acc[mi][nt][j] = 0.f;
          }
        }
      }
    }
  }
}

// Resident CTAs per SM: three of the t <= 8 kernel when the projection has enough 256-feature tiles to give every CTA a long unit,
// else two with deeper rings (the policy of gemm_w4_mma.cu)
static inline int f8_ctas_per_sm(long long tiles, long long t) { return (t <= 8 && tiles >= 64) ? 3 : 2; }

template <typename T, int NT>
int launch_f8(cts_ctx* ctx, const cts_gemm_fp8_args* a, cudaStream_t stream) {
  const bool is_bf16 = a->dtype == CTS_BF16;
  CUtensorMap tm_x;
  int rc = cts_make_tmap_2d(ctx, &tm_x, a->x, a->t, a->k, a->x_ld, NT * 8, is_bf16);
  if (rc) return rc;
  F8Params p;
  p.n = a->n; p.k = a->k; p.t = a->t;
  p.kb_total = (int)(a->k / kBK);
  p.split_k = a->split_k;
  p.tiles = (int)cdiv_ll(a->n, kTileN);
  p.qw = (const uint8_t*)a->qw; p.scales = a->scales; p.out = a->out;
  constexpr int stage_bytes = NT * 8 * kBK * 2 + kWBytes;
  const int kCtas = f8_ctas_per_sm(p.tiles, a->t);
  const int budget = (ctx->max_smem_optin > 0 ? ctx->max_smem_optin + 1024 : 228 * 1024) / kCtas - 3 * 1024;
  int st = (budget - 1024) / stage_bytes;
  if (st > kMaxStages) st = kMaxStages;
  if (st < 2) return cts_set_error(ctx, CTS_ERR_BAD_ARG, "cts_gemm_fp8: shared memory budget too small");
  p.stages = st;
  const size_t smem = (size_t)st * stage_bytes + 1024;
  auto kern = gemm_fp8_kernel<T, NT>;
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

// ---------------------------------------------------------------------------------------------- dequantisation (prefill-sized steps)
// One CTA per (256-feature tile, 64-K block): the 16 KB chunk is read with 16-byte loads, every lane decodes the fragments it would feed
// the MMA into a [256][64] 16-bit tile in shared memory (rows padded to 144 bytes: the fragment writes of a warp hit 32 distinct banks),
// and the tile leaves as 128-byte rows of 16-byte stores.  Value: dtype(fp32(code) * s_n), one rounding, as the host statement.
// The successor is a cts_gemm whose WEIGHT is this kernel's output, and cts_gemm requests its first weight tiles BEFORE its dependency
// wait (weights are otherwise never written): fp8_order_kernel, launched in between, waits for this grid to complete and never triggers,
// so that GEMM is scheduled only once the dequantised matrix is complete and visible.
constexpr int kDqRowBytes = 144;

template <typename T>
__global__ void __launch_bounds__(256) fp8_dequant_kernel(const uint8_t* __restrict__ qw, const float* __restrict__ scales, T* __restrict__ out,
                                                          long long n, long long out_ld, int kb_total) {
  __shared__ __align__(16) uint8_t tile_s[kTileN * kDqRowBytes];
  pdl_trigger();
  const int tile = blockIdx.x / kb_total, kb = blockIdx.x % kb_total;
  const uint8_t* chunk = qw + ((size_t)tile * kb_total + kb) * kWBytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  // 1024 16-byte words per chunk: word i = (m-tile m, k16 step pair h) of lane l with i = (2 m + h) * 32 + l; warp w takes i = w * 32 + l + 256 r
  for (int r = 0; r < 4; ++r) {
    const int mh = warp + 8 * r, m = mh >> 1, h = mh & 1;
    const uint4 q = *reinterpret_cast<const uint4*>(chunk + (size_t)(mh * 32 + lane) * 16);
    const long long row0 = (long long)tile * kTileN + m * 16 + g;
    const float sc0 = row0 < n ? scales[row0] : 0.f, sc1 = row0 + 8 < n ? scales[row0 + 8] : 0.f;
    const uint32_t wq[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {                            // word i: k16 step 2 h + (i >> 1); i even: k 2t, 2t+1, odd: k 2t+8, 2t+9
      uint32_t lo, hi;                                       // lo: row g, hi: row g + 8
      f8_to_f16x2(wq[i], lo, hi);
      const int col = 16 * (2 * h + (i >> 1)) + 2 * tq + 8 * (i & 1);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const uint32_t v = rr ? hi : lo;
        const float s = rr ? sc1 : sc0;
        __half h0, h1;
#ifndef CTS_HOST_SHIM
        h0 = __ushort_as_half((unsigned short)(v & 0xFFFFu)); h1 = __ushort_as_half((unsigned short)(v >> 16));
#else
        h0.bits = (uint16_t)(v & 0xFFFFu); h1.bits = (uint16_t)(v >> 16);
#endif
        const float f0 = __half2float(h0) * s, f1 = __half2float(h1) * s;
        uint32_t packed;
        if constexpr (std::is_same<T, __nv_bfloat16>::value) {
          const __nv_bfloat16 b0 = __float2bfloat16_rn(f0), b1 = __float2bfloat16_rn(f1);
          packed = (uint32_t)*reinterpret_cast<const uint16_t*>(&b0) | ((uint32_t)*reinterpret_cast<const uint16_t*>(&b1) << 16);
        } else {
          const __half b0 = __float2half_rn(f0), b1 = __float2half_rn(f1);
          packed = (uint32_t)*reinterpret_cast<const uint16_t*>(&b0) | ((uint32_t)*reinterpret_cast<const uint16_t*>(&b1) << 16);
        }
        *reinterpret_cast<uint32_t*>(tile_s + (m * 16 + g + 8 * rr) * kDqRowBytes + col * 2) = packed;
      }
    }
  }
  __syncthreads();
  pdl_wait();                                                // the previous kernel may still read the scratch matrix this one overwrites
  for (int i = threadIdx.x; i < kTileN * 8; i += 256) {
    const int row = i >> 3, c = i & 7;
    const long long f = (long long)tile * kTileN + row;
    if (f < n)
      *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(out + f * out_ld + (long long)kb * kBK) + c * 16) =
          *reinterpret_cast<const uint4*>(tile_s + row * kDqRowBytes + c * 16);
  }
}

// one CTA: completes only after the dequantisation grid has completed (and no early trigger for its own successor)
__global__ void fp8_order_kernel() { pdl_wait(); }

}  // namespace

// split-K factor of the persistent schedule: units = tiles x split are dealt round-robin to the resident CTAs; the cost of a choice is
// the longest CTA's stream in 16 KB stages plus the partial it writes per unit (t KB of fp32 = t / 16 stage equivalents)
extern "C" int cts_gemm_fp8_suggest_split(cts_ctx* ctx, long long n, long long k, long long t) {
  if (!ctx || n <= 0 || k <= 0) return 1;
  const long long tiles = cdiv_ll(n, kTileN), kb = k / kBK, ctas = (long long)f8_ctas_per_sm(tiles, t) * ctx->sm_count;
  long long best = 1;
  double best_cost = 1e30;
  for (long long s = 1; s <= 16 && s * 2 <= kb; ++s) {
    const long long waves = cdiv_ll(tiles * s, ctas);
    const double cost = (double)waves * ((double)cdiv_ll(kb, s) + (double)(t < 1 ? 1 : t) / 16.0 + 0.5);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = s; }
  }
  return (int)best;
}

extern "C" int cts_gemm_fp8(cts_ctx* ctx, const cts_gemm_fp8_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr && a->qw && a->scales && a->x && a->out, "null pointer");
  CTS_CHECK_ARG(ctx, a->n > 0 && a->k > 0 && a->t > 0 && a->t <= 32, "n, k > 0 and 1 <= t <= 32 (decode-sized step; larger steps use cts_fp8_dequant + cts_gemm)");
  CTS_CHECK_ARG(ctx, a->dtype == CTS_BF16 || a->dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, a->k % 64 == 0, "k must be a multiple of 64 (a pipeline stage is one 64-K block)");
  CTS_CHECK_ARG(ctx, a->split_k >= 1 && a->split_k <= a->k / 64, "split_k");
  CTS_CHECK_ARG(ctx, a->x_ld >= a->k, "x_ld smaller than k");
  CTS_CHECK_ARG(ctx, ((uintptr_t)a->qw & 15) == 0, "qw must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dtype == CTS_BF16)
    return a->t <= 8 ? launch_f8<__nv_bfloat16, 1>(ctx, a, st) : a->t <= 16 ? launch_f8<__nv_bfloat16, 2>(ctx, a, st) : launch_f8<__nv_bfloat16, 4>(ctx, a, st);
  return a->t <= 8 ? launch_f8<__half, 1>(ctx, a, st) : a->t <= 16 ? launch_f8<__half, 2>(ctx, a, st) : launch_f8<__half, 4>(ctx, a, st);
}

extern "C" int cts_fp8_dequant(cts_ctx* ctx, const cts_fp8_dequant_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr && a->qw && a->scales && a->out, "null pointer");
  CTS_CHECK_ARG(ctx, a->n > 0 && a->k > 0 && a->k % 64 == 0, "n > 0 and k a positive multiple of 64");
  CTS_CHECK_ARG(ctx, a->dtype == CTS_BF16 || a->dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, a->out_ld >= a->k && a->out_ld % 8 == 0 && ((uintptr_t)a->out & 15) == 0 && ((uintptr_t)a->qw & 15) == 0,
                "out must be 16-byte aligned with out_ld >= k a multiple of 8; qw 16-byte aligned");
  const int kb_total = (int)(a->k / kBK);
  const long long blocks = cdiv_ll(a->n, kTileN) * kb_total;
  CTS_CHECK_ARG(ctx, blocks < (1ll << 31), "matrix too large");
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dtype == CTS_BF16)
    CTS_CUDA(ctx, launch_pdl(fp8_dequant_kernel<__nv_bfloat16>, dim3((unsigned)blocks), dim3(256), 0, st, 1, (const uint8_t*)a->qw, a->scales,
                             (__nv_bfloat16*)a->out, a->n, a->out_ld, kb_total));
  else
    CTS_CUDA(ctx, launch_pdl(fp8_dequant_kernel<__half>, dim3((unsigned)blocks), dim3(256), 0, st, 1, (const uint8_t*)a->qw, a->scales,
                             (__half*)a->out, a->n, a->out_ld, kb_total));
  CTS_CUDA(ctx, launch_pdl(fp8_order_kernel, dim3(1), dim3(32), 0, st, 1));
  return CTS_OK;
}
