// chatts_b200 -- decode "chain" kernel: everything between two attention calls of a decode step in ONE persistent,
// cooperatively launched kernel (T <= 32 tokens):
//
//   phase 0  o_proj GEMM        (split-K partials)          A = wo            B = attention output
//   phase 1  residual + RMSNorm (post-attention)            h += sum partials ; xn = norm(h) * ln2
//   phase 2  gate_up GEMM       (split-K partials)          A = wgu (interleaved)  B = xn
//   phase 3  SwiGLU             act = silu(gate) * up
//   phase 4  down GEMM          (split-K partials)          A = wd            B = act
//   phase 5  residual + RMSNorm (next layer's input norm or the final norm)
//   phase 6  QKV GEMM of the NEXT layer (split-K partials)  A = wqkv          B = xn
//   phase 7  bias + (Qwen3 q/k norm) + RoPE + paged KV write of the next layer
//
// (modeling_qwen2.py:269-310 minus the attention itself; the per-phase arithmetic and rounding points are the ones of the
// stand-alone kernels in gemm_tcgen05.cu (the wgmma GEMMs) / elementwise.cu.)  Why: a decode step was ~440 dependent kernels whose
// boundaries cost ~3-4 us each in the captured graph; here the phases are separated by grid barriers (one atomic + an
// acquire spin, ~1 us) and -- the main point -- the TMA producer keeps streaming: as soon as a CTA has issued the last
// weight tile of a GEMM phase it pre-loads the first `stages` WEIGHT tiles of the NEXT GEMM phase into the shared-memory
// ring (weights depend on nothing), so the HBM stream does not stop at the barrier and the memory-bound elementwise
// phases run under a full ring.
//
// One CTA owns at most one (128-row tile, K-split) unit per GEMM phase (the grid is a single wave: 3 CTAs per SM); warp
// roles are those of gemm_tn_kernel (warps 0..3 the wgmma warpgroup and its epilogue, warp 4 TMA producer); the
// elementwise phases use all 192 threads of all CTAs.  Every wait is bounded (trap instead of hang).
#include <cooperative_groups.h>

#include <type_traits>

#include "common.cuh"
#include "tensormap.cuh"

namespace {

constexpr int kBM = 128, kBK = 64, kThreads = 192, kMaxStages = 8;
constexpr int kNormChunks = 8;     // CTAs per token in the RMSNorm phases

struct ChainGemm {
  int n, k, tiles_m, split, kb_total;
};

struct ChainParams {
  int T, H, I, nh, nkv, d;
  int phase_begin, phase_end;      // phases [begin, end) are executed
  int norm5_has_partial;           // phase 5 adds the down-proj partials (0 for the "head" chain: plain norm of h)
  ChainGemm g[4];                  // 0 o_proj, 1 gate_up, 2 down, 3 qkv
  float* ws;                       // split-K partials, reused by every GEMM phase
  float* ssq;                      // [T][kNormChunks] partial sums of squares
  int* sync;                       // [0] grid-barrier counter, [1] exit counter (zero-initialised, self-resetting)
  void* h; void* xn; void* act;
  const void* ln_post; const void* ln_next;
  float eps;
  const void* bqkv; const void* qn; const void* kn;
  const int* positions; const void* cos_tab; const void* sin_tab; const int* slot_map;
  void* q_out; void* k_cache; void* v_cache;
  int page_size;
  int stages;
};

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

template <typename T, int BN>
__global__ void __launch_bounds__(kThreads, 3)
decode_chain_kernel(const __grid_constant__ CUtensorMap tm_wo, const __grid_constant__ CUtensorMap tm_wgu,
                    const __grid_constant__ CUtensorMap tm_wd, const __grid_constant__ CUtensorMap tm_wqkv,
                    const __grid_constant__ CUtensorMap tm_ao, const __grid_constant__ CUtensorMap tm_xn,
                    const __grid_constant__ CUtensorMap tm_act, const ChainParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kMaxStages], empty_bar[kMaxStages];
  __shared__ float red_s[kThreads / 32];

  constexpr int kABytes = kBM * kBK * 2;
  constexpr int kStage = kABytes + BN * kBK * 2;
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;

  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int G = gridDim.x, cta = blockIdx.x;
  const int stages = p.stages;
  const int T_ = p.T;

  if (tid == 0) {
    tma_prefetch_desc(&tm_wo); tma_prefetch_desc(&tm_wgu); tma_prefetch_desc(&tm_wd); tma_prefetch_desc(&tm_wqkv);
    tma_prefetch_desc(&tm_ao); tma_prefetch_desc(&tm_xn); tma_prefetch_desc(&tm_act);
    for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    fence_mbar_init();
  }
  __syncthreads();

  // ---- running pipeline state (persists across phases)
  uint32_t it_p = 0;          // K blocks whose A tile the producer has issued (producer lane only)
  uint32_t it_b = 0;          // K blocks whose B tile the producer has issued (<= it_p)
  uint32_t it_m = 0;          // K blocks consumed by the MMA warpgroup
  int n_bar = 0;              // grid barriers passed

  auto grid_barrier = [&]() {
    __syncthreads();
    if (tid == 0) {
      fence_proxy_async_all();
      __threadfence();
      atomicAdd(&p.sync[0], 1);
      const int target = (n_bar + 1) * G;
      unsigned spins = 0;
      while (ld_acquire_gpu(&p.sync[0]) < target) {
        __nanosleep(20);
        if (++spins > (1u << 24)) {
          printf("chatts_b200: decode-chain grid barrier %d timed out (cta %d)\n", n_bar, cta);
          __trap();
        }
      }
      __threadfence();
      fence_proxy_async_all();
    }
    __syncthreads();
    ++n_bar;
  };

  auto gemm_of = [&](int gi) -> const CUtensorMap* { return gi == 0 ? &tm_wo : gi == 1 ? &tm_wgu : gi == 2 ? &tm_wd : &tm_wqkv; };
  auto act_of = [&](int gi) -> const CUtensorMap* { return gi == 0 ? &tm_ao : gi == 2 ? &tm_act : &tm_xn; };
  auto unit_of = [&](int gi, int& f0, int& kb0, int& nkb, int& split) -> bool {
    const ChainGemm& g = p.g[gi];
    if (cta >= g.tiles_m * g.split) return false;
    const int m = cta % g.tiles_m;
    split = cta / g.tiles_m;
    f0 = m * kBM;
    kb0 = (int)(((long long)g.kb_total * split) / g.split);
    nkb = (int)(((long long)g.kb_total * (split + 1)) / g.split) - kb0;
    return true;
  };
  // producer: issue the WEIGHT tiles of K blocks [done, upto) of this CTA's unit of GEMM gi (B tiles follow separately)
  auto issue_weights = [&](int gi, int f0, int kb0, int from, int upto) {
    const CUtensorMap* tw = gemm_of(gi);
    for (int i = from; i < upto; ++i, ++it_p) {
      const int s = it_p % stages;
      mbar_wait(&empty_bar[s], ((it_p / stages) & 1u) ^ 1u);
      mbar_expect_tx(&full_bar[s], (uint32_t)kStage);
      tma_load_2d(smem + (size_t)s * kStage, tw, &full_bar[s], (kb0 + i) * kBK, f0, CTS_L2_EVICT_FIRST);
    }
  };
  auto issue_acts = [&](int gi, int kb0, int from, int upto) {
    const CUtensorMap* tx = act_of(gi);
    for (int i = from; i < upto; ++i, ++it_b) {
      const int s = it_b % stages;
      tma_load_2d(smem + (size_t)s * kStage + kABytes, tx, &full_bar[s], (kb0 + i) * kBK, 0, CTS_L2_EVICT_LAST);
    }
  };

  // weights pre-issued for the upcoming GEMM phase (producer lane state)
  int pre_gi = -1, pre_n = 0;
  auto prefetch_next_gemm = [&](int gi) {          // called by the producer lane only
    int f0, kb0, nkb, split;
    pre_gi = gi;
    pre_n = 0;
    if (gi < 0 || !unit_of(gi, f0, kb0, nkb, split)) return;
    pre_n = nkb < stages ? nkb : stages;
    issue_weights(gi, f0, kb0, 0, pre_n);
  };

  // ------------------------------------------------------------------ one split-K GEMM phase
  auto gemm_phase = [&](int gi, int next_gi) {
    int f0 = 0, kb0 = 0, nkb = 0, split = 0;
    const bool active = unit_of(gi, f0, kb0, nkb, split);
    const ChainGemm& g = p.g[gi];
    if (warp == 4) {
      if (lane == 0) {
        if (active) {
          int done = 0;
          if (pre_gi == gi) done = pre_n;            // weight tiles already in flight since before the last barrier
          else { done = nkb < stages ? nkb : stages; issue_weights(gi, f0, kb0, 0, done); }
          issue_acts(gi, kb0, 0, done);
          for (int i = done; i < nkb; ++i) {
            issue_weights(gi, f0, kb0, i, i + 1);
            issue_acts(gi, kb0, i, i + 1);
          }
        }
        prefetch_next_gemm(next_gi);                 // keep the HBM stream going across the coming barrier(s)
      }
    } else if (warp < 4 && active) {
      Acc128<BN> acc;
      acc.zero();
      for (int i = 0; i < nkb; ++i, ++it_m) {
        const int s = it_m % stages;
        mbar_wait(&full_bar[s], (it_m / stages) & 1u);
        const uint32_t a_addr = smem_u32(smem + (size_t)s * kStage);
        acc.template mma_kblock<kIsBf16>(a_addr, a_addr + kABytes, i == 0);
        wgmma_wait<1>();
        if (i > 0 && tid == 0) mbar_arrive(&empty_bar[(it_m - 1) % stages]);
      }
      wgmma_wait<0>();
      if (nkb > 0 && tid == 0) mbar_arrive(&empty_bar[(it_m - 1) % stages]);
      float* dst = p.ws + (long long)split * T_ * g.n;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) {
          const long long f = (long long)f0 + 64 * h + acc_row(i);
          const int c = acc_col(i);
          if (c < T_ && f < g.n) dst[(long long)c * g.n + f] = acc.d[h][i];
        }
    }
  };

  // ------------------------------------------------------------------ residual + RMSNorm (two sub-phases, 8 CTAs per token)
  auto norm_phase = [&](int gi_partial, const T* norm_w) {
    const int token = cta / kNormChunks, chunk = cta % kNormChunks;
    const bool active = token < T_;
    const int hc = p.H / kNormChunks, nvec = hc / 8;
    const int col0 = chunk * hc;
    T* h = reinterpret_cast<T*>(p.h);
    T* xn = reinterpret_cast<T*>(p.xn);
    float r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const bool mine = active && tid < nvec;
    float ss = 0.f;
    if (mine) {
      const long long off = (long long)token * p.H + col0 + tid * 8;
      unpack8<T>(*reinterpret_cast<const uint4*>(h + off), r);
      if (gi_partial >= 0) {
        const int S = p.g[gi_partial].split;
        const long long stride = (long long)T_ * p.H;
        const float* pp = p.ws + off;
        float4 lo = __ldcg(reinterpret_cast<const float4*>(pp)), hi = __ldcg(reinterpret_cast<const float4*>(pp + 4));
        for (int s = 1; s < S; ++s) {
          const float4 l2 = __ldcg(reinterpret_cast<const float4*>(pp + s * stride));
          const float4 h2 = __ldcg(reinterpret_cast<const float4*>(pp + s * stride + 4));
          lo.x += l2.x; lo.y += l2.y; lo.z += l2.z; lo.w += l2.w; hi.x += h2.x; hi.y += h2.y; hi.z += h2.z; hi.w += h2.w;
        }
        const float a[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = rnd<T>(r[j] + rnd<T>(a[j]));
        *reinterpret_cast<uint4*>(h + off) = pack8<T>(r);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += r[j] * r[j];
    }
    ss = warp_sum(ss);
    if (lane == 0) red_s[warp] = ss;
    __syncthreads();
    if (tid == 0 && active) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kThreads / 32; ++w) v += red_s[w];
      p.ssq[token * kNormChunks + chunk] = v;
    }
    grid_barrier();
    if (mine) {
      float tot = 0.f;
#pragma unroll
      for (int c = 0; c < kNormChunks; ++c) tot += __ldcg(p.ssq + token * kNormChunks + c);
      const float inv = 1.0f / sqrtf(tot / (float)p.H + p.eps);
      float w[8], o[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(norm_w + col0 + tid * 8), w);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = w[j] * rnd<T>(r[j] * inv);
      *reinterpret_cast<uint4*>(xn + (long long)token * p.H + col0 + tid * 8) = pack8<T>(o);
    }
  };

  // ------------------------------------------------------------------ SwiGLU on the interleaved gate/up partials
  auto swiglu_phase = [&]() {
    const int S = p.g[1].split;
    const long long n = 2LL * p.I, stride = (long long)T_ * n;
    const int per_tok = p.I / 8;
    T* act = reinterpret_cast<T*>(p.act);
    for (long long item = (long long)cta * kThreads + tid; item < (long long)T_ * per_tok; item += (long long)G * kThreads) {
      const int t = (int)(item / per_tok), i0 = (int)(item % per_tok) * 8;
      const long long gcol = (long long)(i0 >> 6) * 128 + (i0 & 63);
      const float* pg = p.ws + (long long)t * n + gcol;
      float g8[8] = {0, 0, 0, 0, 0, 0, 0, 0}, u8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      for (int s = 0; s < S; ++s) {
        const float4 a = __ldcg(reinterpret_cast<const float4*>(pg + s * stride)), b = __ldcg(reinterpret_cast<const float4*>(pg + s * stride + 4));
        const float4 c = __ldcg(reinterpret_cast<const float4*>(pg + s * stride + 64)), e = __ldcg(reinterpret_cast<const float4*>(pg + s * stride + 68));
        g8[0] += a.x; g8[1] += a.y; g8[2] += a.z; g8[3] += a.w; g8[4] += b.x; g8[5] += b.y; g8[6] += b.z; g8[7] += b.w;
        u8[0] += c.x; u8[1] += c.y; u8[2] += c.z; u8[3] += c.w; u8[4] += e.x; u8[5] += e.y; u8[6] += e.z; u8[7] += e.w;
      }
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rnd<T>(silu_f(rnd<T>(g8[j]))) * rnd<T>(u8[j]);
      *reinterpret_cast<uint4*>(act + (long long)t * p.I + i0) = pack8<T>(o);
    }
  };

  // ------------------------------------------------------------------ bias + (q/k norm) + RoPE + KV write
  auto rope_phase = [&]() {
    const int S = p.g[3].split;
    const int d = p.d, half = d >> 1, cph = half >> 3;
    const int heads = p.nh + 2 * p.nkv;
    const long long width = (long long)heads * d, stride = (long long)T_ * width;
    const long long items = (long long)T_ * heads * cph;
    const long long items_pad = (items + 31) / 32 * 32;
    const T* bias = reinterpret_cast<const T*>(p.bqkv);
    const T* qn = reinterpret_cast<const T*>(p.qn);
    const T* kn = reinterpret_cast<const T*>(p.kn);
    const T* cos_tab = reinterpret_cast<const T*>(p.cos_tab);
    const T* sin_tab = reinterpret_cast<const T*>(p.sin_tab);
    for (long long item = (long long)cta * kThreads + tid; item < items_pad; item += (long long)G * kThreads) {
      const bool active = item < items;
      const long long it2 = active ? item : 0;
      const int t = (int)(it2 / (heads * cph));
      const int rem = (int)(it2 % (heads * cph));
      const int head = rem / cph, j = rem % cph;
      const long long c0 = (long long)head * d + j * 8, c1 = c0 + half;
      const float* pp = p.ws + (long long)t * width;
      float x0[8] = {0, 0, 0, 0, 0, 0, 0, 0}, x1[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      for (int s = 0; s < S; ++s) {
        const float* ps = pp + s * stride;
        const float4 a = __ldcg(reinterpret_cast<const float4*>(ps + c0)), b = __ldcg(reinterpret_cast<const float4*>(ps + c0 + 4));
        const float4 c = __ldcg(reinterpret_cast<const float4*>(ps + c1)), e = __ldcg(reinterpret_cast<const float4*>(ps + c1 + 4));
        x0[0] += a.x; x0[1] += a.y; x0[2] += a.z; x0[3] += a.w; x0[4] += b.x; x0[5] += b.y; x0[6] += b.z; x0[7] += b.w;
        x1[0] += c.x; x1[1] += c.y; x1[2] += c.z; x1[3] += c.w; x1[4] += e.x; x1[5] += e.y; x1[6] += e.z; x1[7] += e.w;
      }
      if (bias) {
        float b0[8], b1[8];
        unpack8<T>(*reinterpret_cast<const uint4*>(bias + c0), b0);
        unpack8<T>(*reinterpret_cast<const uint4*>(bias + c1), b1);
#pragma unroll
        for (int e = 0; e < 8; ++e) { x0[e] += b0[e]; x1[e] += b1[e]; }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) { x0[e] = rnd<T>(x0[e]); x1[e] = rnd<T>(x1[e]); }
      const bool is_q = head < p.nh;
      const bool is_k = !is_q && head < p.nh + p.nkv;
      if (qn != nullptr || kn != nullptr) {
        float ss = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) ss += x0[e] * x0[e] + x1[e] * x1[e];
        for (int o = cph >> 1; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        const float inv = 1.0f / sqrtf(ss / (float)d + p.eps);
        const T* nw = is_q ? qn : (is_k ? kn : nullptr);
        if (nw != nullptr) {
          float w0[8], w1[8];
          unpack8<T>(*reinterpret_cast<const uint4*>(nw + j * 8), w0);
          unpack8<T>(*reinterpret_cast<const uint4*>(nw + half + j * 8), w1);
#pragma unroll
          for (int e = 0; e < 8; ++e) { x0[e] = rnd<T>(w0[e] * rnd<T>(x0[e] * inv)); x1[e] = rnd<T>(w1[e] * rnd<T>(x1[e] * inv)); }
        }
      }
      if (!active) continue;
      if (is_q || is_k) {
        const int pos = p.positions[t];
        float cs[8], sn[8];
        unpack8<T>(*reinterpret_cast<const uint4*>(cos_tab + (long long)pos * half + j * 8), cs);
        unpack8<T>(*reinterpret_cast<const uint4*>(sin_tab + (long long)pos * half + j * 8), sn);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float r0 = rnd<T>(rnd<T>(x0[e] * cs[e]) + rnd<T>(-x1[e] * sn[e]));
          const float r1 = rnd<T>(rnd<T>(x1[e] * cs[e]) + rnd<T>(x0[e] * sn[e]));
          x0[e] = r0; x1[e] = r1;
        }
      }
      const uint4 lo = pack8<T>(x0), hi = pack8<T>(x1);
      if (is_q) {
        T* o = reinterpret_cast<T*>(p.q_out) + (long long)t * p.nh * d + (long long)head * d + j * 8;
        *reinterpret_cast<uint4*>(o) = lo;
        *reinterpret_cast<uint4*>(o + half) = hi;
        continue;
      }
      const int kvh = is_k ? head - p.nh : head - p.nh - p.nkv;
      T* cache = reinterpret_cast<T*>(is_k ? p.k_cache : p.v_cache);
      const int slot = p.slot_map[t];
      if (slot >= 0) {
        const long long page = slot / p.page_size, off = slot % p.page_size;
        T* o = cache + ((page * p.nkv + kvh) * p.page_size + off) * d + j * 8;
        *reinterpret_cast<uint4*>(o) = lo;
        *reinterpret_cast<uint4*>(o + half) = hi;
      }
    }
  };

  // ================================================================== the chain
  const int pb = p.phase_begin, pe = p.phase_end;
  auto next_gemm_after = [&](int phase) -> int {      // GEMM index of the first GEMM phase > `phase` inside [pb, pe), else -1
    for (int ph = phase + 1; ph < pe; ++ph)
      if ((ph & 1) == 0) return ph >> 1;
    return -1;
  };
  if (warp == 4 && lane == 0) {
    // weights of the first GEMM phase of this launch: in flight before anything else
    const int first = (pb & 1) == 0 ? (pb >> 1) : next_gemm_after(pb);
    prefetch_next_gemm(first);
  }
  for (int ph = pb; ph < pe; ++ph) {
    switch (ph) {
      case 0: gemm_phase(0, next_gemm_after(0)); break;
      case 1: norm_phase(0, reinterpret_cast<const T*>(p.ln_post)); break;
      case 2: gemm_phase(1, next_gemm_after(2)); break;
      case 3: swiglu_phase(); break;
      case 4: gemm_phase(2, next_gemm_after(4)); break;
      case 5: norm_phase(p.norm5_has_partial ? 2 : -1, reinterpret_cast<const T*>(p.ln_next)); break;
      case 6: gemm_phase(3, -1); break;
      case 7: rope_phase(); break;
    }
    if (ph + 1 < pe) grid_barrier();
  }

  // ---- teardown: the last CTA to leave resets the barrier counters for the next launch
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const int done = atomicAdd(&p.sync[1], 1) + 1;
    if (done == G) {
      p.sync[0] = 0;
      p.sync[1] = 0;
      __threadfence();
    }
  }
}

template <typename T, int BN>
int launch_chain(cts_ctx* ctx, const cts_chain_args* a, cudaStream_t st) {
  const bool bf = a->dtype == CTS_BF16;
  const int H = a->hidden, I = a->inter, d = a->head_dim, nh = a->nh, nkv = a->nkv, T_ = a->t;
  const int qkv_n = (nh + 2 * nkv) * d;
  ChainParams p;
  memset(&p, 0, sizeof(p));
  p.T = T_; p.H = H; p.I = I; p.nh = nh; p.nkv = nkv; p.d = d;
  p.phase_begin = a->phase_begin; p.phase_end = a->phase_end; p.norm5_has_partial = a->norm5_has_partial;
  const int ns[4] = {H, 2 * I, H, qkv_n}, ks[4] = {nh * d, H, I, H};
  int max_units = kNormChunks * T_;
  for (int i = 0; i < 4; ++i) {
    p.g[i].n = ns[i]; p.g[i].k = ks[i];
    p.g[i].tiles_m = (ns[i] + kBM - 1) / kBM;
    p.g[i].split = a->split[i] > 0 ? a->split[i] : 1;
    p.g[i].kb_total = (ks[i] + kBK - 1) / kBK;
    if (p.g[i].split > p.g[i].kb_total) return cts_set_error(ctx, CTS_ERR_BAD_ARG, "cts_decode_chain: split %d > K blocks", p.g[i].split);
    const int ph = 2 * i;
    if (ph >= a->phase_begin && ph < a->phase_end && p.g[i].tiles_m * p.g[i].split > max_units) max_units = p.g[i].tiles_m * p.g[i].split;
  }
  p.ws = a->ws; p.ssq = a->ssq; p.sync = a->sync;
  p.h = a->h; p.xn = a->xn; p.act = a->act; p.ln_post = a->ln_post; p.ln_next = a->ln_next; p.eps = a->eps;
  p.bqkv = a->bqkv; p.qn = a->q_norm_w; p.kn = a->k_norm_w; p.positions = a->positions; p.cos_tab = a->cos_tab; p.sin_tab = a->sin_tab;
  p.slot_map = a->slot_map; p.q_out = a->q_out; p.k_cache = a->k_cache; p.v_cache = a->v_cache; p.page_size = a->page_size;
  constexpr int kStage = kBM * kBK * 2 + BN * kBK * 2;
  int stages = (ctx->decode_stages * 1024) / kStage;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) stages = 2;
  p.stages = stages;
  const size_t smem = (size_t)stages * kStage + 1024;

  CUtensorMap tm_wo, tm_wgu, tm_wd, tm_wqkv, tm_ao, tm_xn, tm_act;
  int rc;
  const void* dummy_w = a->wo ? a->wo : (a->wgu ? a->wgu : (a->wd ? a->wd : a->wqkv));
#define MK(tm, ptr, rows, cols, box)                                                                 \
  rc = cts_make_tmap_2d(ctx, &tm, (ptr) ? (ptr) : dummy_w, rows, cols, cols, box, bf);              \
  if (rc) return rc;
  MK(tm_wo, a->wo, H, nh * d, kBM)
  MK(tm_wgu, a->wgu, 2 * I, H, kBM)
  MK(tm_wd, a->wd, H, I, kBM)
  MK(tm_wqkv, a->wqkv, qkv_n, H, kBM)
  MK(tm_ao, a->ao ? a->ao : a->xn, T_, nh * d, BN)
  MK(tm_xn, a->xn, T_, H, BN)
  MK(tm_act, a->act ? a->act : a->xn, T_, I, BN)
#undef MK

  auto kern = decode_chain_kernel<T, BN>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
  // co-resident capacity: the occupancy API, cross-checked against the plain resource arithmetic (227 KB of shared memory
  // and 64 K registers per SM).  All CTAs must be resident at once: the phases are separated by grid barriers.
  int per_sm_api = 0;
  CTS_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_api, kern, kThreads, smem));
  cudaFuncAttributes fa;
  CTS_CUDA(ctx, cudaFuncGetAttributes(&fa, kern));
  const int regs_per_cta = ((fa.numRegs + 7) / 8 * 8) * kThreads;
  int per_sm_res = (int)((227 * 1024) / (smem + fa.sharedSizeBytes + 1024));
  if (regs_per_cta > 0 && 65536 / regs_per_cta < per_sm_res) per_sm_res = 65536 / regs_per_cta;
  if (per_sm_res > 32) per_sm_res = 32;
  const bool cooperative = per_sm_api >= per_sm_res;            // otherwise: plain launch on the resource arithmetic
  const int per_sm = per_sm_api > per_sm_res ? per_sm_api : per_sm_res;
  const int capacity = per_sm * ctx->sm_count;
  if (max_units > capacity)
    return cts_set_error(ctx, CTS_ERR_UNSUPPORTED, "cts_decode_chain: %d work units exceed the co-resident capacity %d (api %d, resources %d per SM)",
                         max_units, capacity, per_sm_api, per_sm_res);
  const int grid = max_units;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cooperative ? 1 : 0;
  CTS_CUDA(ctx, cudaLaunchKernelEx(&cfg, kern, tm_wo, tm_wgu, tm_wd, tm_wqkv, tm_ao, tm_xn, tm_act, p));
  return CTS_OK;
}

}  // namespace

extern "C" int cts_decode_chain(cts_ctx* ctx, const cts_chain_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr, "null args");
  CTS_CHECK_ARG(ctx, a->t >= 1 && a->t <= 32, "t must be in 1..32 (decode)");
  CTS_CHECK_ARG(ctx, a->phase_begin >= 0 && a->phase_end <= 8 && a->phase_begin < a->phase_end, "phase range");
  CTS_CHECK_ARG(ctx, a->dtype == CTS_BF16 || a->dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, a->hidden % (8 * kNormChunks) == 0 && a->hidden / (8 * kNormChunks) <= kThreads, "hidden must be a multiple of 64 and <= 12288");
  CTS_CHECK_ARG(ctx, a->inter % 64 == 0, "inter must be a multiple of 64 (interleaved gate/up)");
  CTS_CHECK_ARG(ctx, a->head_dim % 16 == 0 && ((a->head_dim / 16) & (a->head_dim / 16 - 1)) == 0 && a->head_dim <= 512, "head_dim");
  CTS_CHECK_ARG(ctx, a->ws && a->ssq && a->sync && a->h && a->xn, "null workspace / activations");
  const int pb = a->phase_begin, pe = a->phase_end;
  auto has = [&](int ph) { return ph >= pb && ph < pe; };
  CTS_CHECK_ARG(ctx, !has(0) || (a->wo && a->ao), "phase 0 needs wo, ao");
  CTS_CHECK_ARG(ctx, !has(1) || a->ln_post, "phase 1 needs ln_post");
  CTS_CHECK_ARG(ctx, !has(2) || a->wgu, "phase 2 needs wgu");
  CTS_CHECK_ARG(ctx, !has(3) || a->act, "phase 3 needs act");
  CTS_CHECK_ARG(ctx, !has(4) || (a->wd && a->act), "phase 4 needs wd, act");
  CTS_CHECK_ARG(ctx, !has(5) || a->ln_next, "phase 5 needs ln_next");
  CTS_CHECK_ARG(ctx, !has(6) || a->wqkv, "phase 6 needs wqkv");
  CTS_CHECK_ARG(ctx, !has(7) || (a->positions && a->cos_tab && a->sin_tab && a->slot_map && a->q_out && a->k_cache && a->v_cache && a->page_size > 0),
                "phase 7 needs the RoPE / KV-cache arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (a->dtype == CTS_BF16)
    return a->t <= 16 ? launch_chain<__nv_bfloat16, 16>(ctx, a, st) : launch_chain<__nv_bfloat16, 32>(ctx, a, st);
  return a->t <= 16 ? launch_chain<__half, 16>(ctx, a, st) : launch_chain<__half, 32>(ctx, a, st);
}
