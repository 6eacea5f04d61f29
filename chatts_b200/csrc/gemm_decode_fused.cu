// chatts_b200 -- decode GEMM with the split-K reduction AND the projection's tail fused in, through a thread-block cluster.
//
// The decode step is nine dependent stages per layer (weight stream, attention, small kernels and their ramps).  Four of the nine exist only because the skinny decode GEMMs split K over CTAs and a
// second kernel has to add the fp32 partials before it can apply bias / RoPE / SwiGLU / the residual.  Here the K splits of
// one 128-feature tile form ONE CLUSTER (grid.z = split <= 8 = cluster.z): every CTA runs the same TMA -> wgmma -> registers
// mainloop as gemm_tn_kernel, parks its fp32 accumulator tile in its own shared memory, and after a cluster barrier the
// CTAs reduce disjoint TOKENS of the tile over distributed shared memory (split order: the same summation order as the
// stand-alone reduce kernels, so results are bit-identical to the multi-kernel path) and apply the tail in place:
//
//   CTS_FUSED_RESIDUAL  h[t][f] = dtype(h[t][f] + dtype(sum))                                o_proj / down_proj (modeling_qwen2.py:302,308)
//   CTS_FUSED_SWIGLU    act[t][i] = dtype(silu(dtype(gate_i)) * dtype(up_i))   (interleaved gate/up weight)   (:47)
//   CTS_FUSED_QKV_ROPE  dtype(sum + bias) -> Qwen3 q/k RMSNorm -> RoPE -> q_out / paged KV write                (:116-146,217-222)
//
// A 128-row tile of the QKV weight is exactly one head (head_dim 128; two heads at head_dim 64), and a tile of the
// interleaved gate_up weight holds 64 (gate, up) pairs, so every tail is tile-local.  Per layer this removes the
// RoPE/KV-write and the SwiGLU launches, turns the two reduce+residual+RMSNorm launches into plain RMSNorms and removes the
// fp32 partial round trip through L2 (9 -> 7 stages; folding the RMSNorm weight into the next projection would make it 5).
//
// OPT-IN (CTS_DECODE_FUSED=1 / use_fused_decode=True): written after the round-1 GPU budget was spent, never executed.  T <= 32
// tokens, split <= 8.  Every mbarrier wait is bounded (trap, not hang); the cluster barriers are reached by all threads of all
// CTAs unconditionally.
#include <cooperative_groups.h>

#include <type_traits>

#include "common.cuh"

// the kernel's dynamic shared memory as a byte array (one spelling, so that tests/cuda_on_cpu can supply its own; defined here and not
// in common.cuh so that the header the GPU-validated kernels were compiled with stays byte-identical)
#ifndef CTS_DYN_SMEM
#define CTS_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#endif
#include "tensormap.cuh"
#include "trace.cuh"

namespace {

namespace cg = cooperative_groups;

constexpr int kBM = 128, kBK = 64, kThreads = 192, kMaxStages = 12;

struct FusedParams {
  long long n, k, t;
  int kb_total, split, stages, mode;
  const void* bias;
  void* h;                // RESIDUAL: [t, n] residual stream, updated in place
  void* act;              // SWIGLU: [t, n/2]
  // QKV_ROPE
  const int* positions; const void* cos_tab; const void* sin_tab; const int* slot_map;
  void* q_out; void* k_cache; void* v_cache;
  const void* q_norm; const void* k_norm; float eps;
  int nh, nkv, d, page_size;
  // NORM_IN: the token operand is RMSNorm(norm_h) * norm_w, produced by the epilogue warps straight into the swizzled B tiles
  const void* norm_h; const void* norm_w; const float* ssq_in; int ssq_tiles; float norm_eps;
  float* ssq_out;         // RESIDUAL: [t][tiles of n] sum of squares of the updated h per 128-feature tile (or NULL)
  // RESIDUAL of a row-parallel projection under tensor parallelism: all-reduce over peer memory inside the kernel (see tp_tail)
  uint8_t* const* peer_region; int* peer_state; int peer_rank, peer_world, peer_max_tokens;
};

// ---- wire format of the in-kernel all-reduce (shared with allreduce_ll.cu): the epoch travels inside every 8-byte word
constexpr unsigned kPeerSpinLimit = 1u << 24;
#ifdef CTS_HOST_SHIM      // tests/cuda_on_cpu: the same wire format on the host (8-byte halves written / read separately; ranks are processes)
__device__ __forceinline__ void st_ll16(void* p, uint32_t d0, uint32_t d1, uint32_t epoch) {
  volatile uint64_t* q = reinterpret_cast<volatile uint64_t*>(p);
  q[0] = (uint64_t)d0 | ((uint64_t)epoch << 32);
  sched_yield();
  q[1] = (uint64_t)d1 | ((uint64_t)epoch << 32);
}
__device__ __forceinline__ uint4 ld_ll16(const void* p) {
  const volatile uint64_t* q = reinterpret_cast<const volatile uint64_t*>(p);
  const uint64_t a = q[0], b = q[1];
  shim_yield();
  static thread_local unsigned n = 0;
  if ((++n & 255u) == 0) sched_yield();
  return uint4{(uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32)};
}
__device__ __forceinline__ void st_ll8(void* p, uint32_t d, uint32_t epoch) {
  *reinterpret_cast<volatile uint64_t*>(p) = (uint64_t)d | ((uint64_t)epoch << 32);
}
__device__ __forceinline__ uint2 ld_ll8(const void* p) {
  const uint64_t a = *reinterpret_cast<const volatile uint64_t*>(p);
  shim_yield();
  static thread_local unsigned n = 0;
  if ((++n & 255u) == 0) sched_yield();
  return uint2{(uint32_t)a, (uint32_t)(a >> 32)};
}
#else
__device__ __forceinline__ void st_ll16(void* p, uint32_t d0, uint32_t d1, uint32_t epoch) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(d0), "r"(epoch), "r"(d1), "r"(epoch) : "memory");
}
__device__ __forceinline__ uint4 ld_ll16(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_ll8(void* p, uint32_t d, uint32_t epoch) {
  asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(d), "r"(epoch) : "memory");
}
__device__ __forceinline__ uint2 ld_ll8(const void* p) {
  uint2 v;
  asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
#endif
__device__ void peer_timeout(const char* what, int rank) {
  printf("chatts_b200: fused GEMM + all-reduce timed out in %s on rank %d (block %d,%d thread %d)\n", what, rank, blockIdx.x, blockIdx.z,
         threadIdx.x);
  __trap();
}
template <typename T> __device__ __forceinline__ uint32_t pack_pair(float a, float b) {
  T v[2] = {DT<T>::from_f(a), DT<T>::from_f(b)};
  return *reinterpret_cast<uint32_t*>(v);
}

template <typename T, int BN, bool NORM_IN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_decode_fused_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x, const FusedParams p) {
  CTS_DYN_SMEM(smem_raw);
  __shared__ uint64_t full_bar[kMaxStages];
  __shared__ uint64_t empty_bar[kMaxStages];
  __shared__ float xch[kBM];            // tile-local exchange (SwiGLU up values / RoPE partners)
  __shared__ float red[4];              // per-warp partial sums of the q/k RMSNorm statistic
  __shared__ float rstd_s[32];          // NORM_IN: rsqrt(mean(h^2) + eps) of every token

  constexpr int kABytes = kBM * kBK * 2;
  constexpr int kStage = kABytes + BN * kBK * 2;
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;
  static_assert(BN <= 32, "decode-sized token tile");

  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  float* part_s = reinterpret_cast<float*>(smem);          // [BN][128] fp32, reuses the pipeline ring once the accumulator is complete

  cg::cluster_group cluster = cg::this_cluster();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f0 = blockIdx.x * kBM;
  const int split = blockIdx.z;                            // == rank inside the (1, 1, split) cluster
  const int S = p.split;
  const int stages = p.stages;
  const int kb0 = (int)(((long long)p.kb_total * split) / S);
  const int kb1 = (int)(((long long)p.kb_total * (split + 1)) / S);
  const int nkb = kb1 - kb0;
  const int T_ = (int)p.t;

  pdl_trigger();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_x);
    // NORM_IN: the full barrier covers the weight tile only; the MMA warpgroup writes B itself right before its MMAs
    for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ------------------------------ TMA producer (as gemm_tn_kernel: weights before the dependency wait) ------------------------------
    if (lane == 0) {
      const int npre = nkb < stages ? nkb : stages;
      constexpr uint32_t kTx = NORM_IN ? (uint32_t)kABytes : (uint32_t)kStage;
      CTS_TRACE(CTS_TK_FUSED, 0);
      for (int i = 0; i < npre; ++i) {
        mbar_expect_tx(&full_bar[i], kTx);
        tma_load_2d(smem + (size_t)i * kStage, &tm_w, &full_bar[i], (kb0 + i) * kBK, f0, CTS_L2_EVICT_FIRST);
      }
      pdl_wait();
      CTS_TRACE(CTS_TK_FUSED, 1);
      if (!NORM_IN)
        for (int i = 0; i < npre; ++i)
          tma_load_2d(smem + (size_t)i * kStage + kABytes, &tm_x, &full_bar[i], (kb0 + i) * kBK, 0, CTS_L2_EVICT_LAST);
      for (int i = npre; i < nkb; ++i) {
        const int s = i % stages;
        mbar_wait(&empty_bar[s], (((uint32_t)(i / stages)) & 1u) ^ 1u);
        mbar_expect_tx(&full_bar[s], kTx);
        uint8_t* st = smem + (size_t)s * kStage;
        tma_load_2d(st, &tm_w, &full_bar[s], (kb0 + i) * kBK, f0, CTS_L2_EVICT_FIRST);
        if (!NORM_IN) tma_load_2d(st + kABytes, &tm_x, &full_bar[s], (kb0 + i) * kBK, 0, CTS_L2_EVICT_LAST);
      }
      CTS_TRACE(CTS_TK_FUSED, 2);
    }
  } else if (warp < 4) {
    // ------------------------------ MMA warpgroup ------------------------------
    pdl_wait();
    const int et = (int)threadIdx.x;                          // 0..127
    if (NORM_IN) {
      // B operand: xn = norm_w * dtype(h * rstd) written as the swizzled K-major token tile of each stage
      // (modeling_qwen2.py:258-263 -- the same values the stand-alone RMSNorm kernel stores, without the launch and the round trip;
      //  the row statistic comes from the per-tile sums of squares the previous fused RESIDUAL projection left in ssq_in)
      if (et < BN) {
        float tot = 0.f;
        if (et < T_)
          for (int j = 0; j < p.ssq_tiles; ++j) tot += p.ssq_in[(long long)et * p.ssq_tiles + j];       // fixed order
        rstd_s[et] = 1.0f / sqrtf(tot / (float)p.k + p.norm_eps);
      }
      named_bar_sync(1, 128);
    }
    const T* hsrc = reinterpret_cast<const T*>(p.norm_h);
    const T* nw = reinterpret_cast<const T*>(p.norm_w);
    Acc128<BN> acc;
    acc.zero();
    for (int i = 0; i < nkb; ++i) {
      const int s = i % stages;
      if (NORM_IN) {                                          // slot s was last read by the MMAs of block i - stages: complete
        uint8_t* bt = smem + (size_t)s * kStage + kABytes;    // [BN rows x 128 B], 128B swizzle
        for (int it = et; it < BN * 8; it += 128) {
          const int t = it >> 3, ch = it & 7;
          const long long k0 = (long long)(kb0 + i) * kBK + ch * 8;
          uint4 o = make_uint4(0u, 0u, 0u, 0u);
          if (t < T_ && k0 < p.k) {                           // k is a multiple of 8 (16-byte rows)
            float hv[8], wv[8], xv[8];
            unpack8<T>(*reinterpret_cast<const uint4*>(hsrc + (long long)t * p.k + k0), hv);
            unpack8<T>(*reinterpret_cast<const uint4*>(nw + k0), wv);
            const float r = rstd_s[t];
#pragma unroll
            for (int e = 0; e < 8; ++e) xv[e] = wv[e] * rnd<T>(hv[e] * r);
            o = pack8<T>(xv);
          }
          *reinterpret_cast<uint4*>(bt + (uint32_t)t * 128 + ((ch ^ (t & 7)) << 4)) = o;
        }
        fence_proxy_async_smem();                             // generic-proxy writes -> visible to the tensor core
        named_bar_sync(1, 128);
      }
      mbar_wait(&full_bar[s], ((uint32_t)(i / stages)) & 1u);
      const uint32_t a_addr = smem_u32(smem + (size_t)s * kStage);
      acc.template mma_kblock<kIsBf16>(a_addr, a_addr + kABytes, i == 0);
      wgmma_wait<1>();
      if (i > 0 && threadIdx.x == 0) mbar_arrive(&empty_bar[(i - 1) % stages]);
    }
    wgmma_wait<0>();
    if (nkb > 0 && threadIdx.x == 0) mbar_arrive(&empty_bar[(nkb - 1) % stages]);
    // ------------------------------ epilogue, part A: park this split's fp32 tile in shared memory ------------------------------
    named_bar_sync(1, 128);                                   // every warp's MMAs are done with the ring
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) part_s[acc_col(i) * kBM + 64 * h + acc_row(i)] = acc.d[h][i];
  }
  __syncthreads();
  cluster.sync();                                            // every split's tile is in its CTA's shared memory

  if (warp >= 2) {
    // ------------------------------ epilogue, part B: this CTA reduces tokens t = split, split + S, ... and applies the tail ------------------------------
    const int ft = (warp & 3) * 32 + lane;                   // feature inside the tile (note: warp & 3 is a permutation of 0..3)
    const long long f = (long long)f0 + ft;
    const bool f_ok = f < p.n;
    const int mode = p.mode;
    // tokens in groups of 4: the 4 x S distributed-shared-memory loads of a group are independent and issued back to back, so
    // the DSMEM latency is paid once per group instead of once per token; the sum of a token still runs in split order
    constexpr int kGroup = 4;
    float accs[kGroup];
    if (mode == CTS_FUSED_RESIDUAL && p.peer_region != nullptr) {
      // ------------------------------ tensor-parallel tail: GEMM + all-reduce + residual in this launch ------------------------------
      // Two-shot all-reduce at (tile, token) granularity, flags inside the data (the protocol of allreduce_ll.cu, model-checked in
      // tests/test_peer_ll_protocol.py).  The three passes run over ALL of this CTA's tokens each, so the two NVLink hops are paid
      // once per CTA, not once per token.  h is identical on every rank before and after (the owner alone reads its residual).
      const int W = p.peer_world, me = p.peer_rank, Tmax = p.peer_max_tokens;
      const int hw = (int)(p.n / W);                          // columns per owner; hw % 128 == 0 (host-checked): a tile has ONE owner
      const int owner = f0 / hw;
      const int col = f0 - owner * hw + ft;                   // column inside the owner's chunk
      const uint32_t epoch = (uint32_t)(p.peer_state[0] + 1); // advanced by the last CTA of every call (end of this kernel)
      const long long ag_off = (long long)Tmax * p.n * 8, sq_off = (long long)Tmax * p.n * 12;
      uint8_t* mine = p.peer_region[me];
      uint8_t* own_reg = p.peer_region[owner];
      const bool even = (ft & 1) == 0;                        // one lane per PAIR of features does the wire work
      T* hrow = reinterpret_cast<T*>(p.h);
      // pass A: this rank's full-K partial of (tile, token) -> the owner's region, slot [me]
      for (int tb = split; tb < T_; tb += kGroup * S) {
#pragma unroll
        for (int u2 = 0; u2 < kGroup; ++u2) {
          const int t2 = tb + u2 * S;
          float a2 = 0.f;
          if (t2 < T_)
            for (int s2 = 0; s2 < S; ++s2) a2 += *cluster.map_shared_rank(&part_s[t2 * kBM + ft], s2);      // split order, DSMEM
          accs[u2] = a2;
        }
#pragma unroll
        for (int u = 0; u < kGroup; ++u) {
          const int t = tb + u * S;
          const float nb = __shfl_down_sync(0xffffffffu, accs[u], 1);
          if (t < T_ && even)
            st_ll16(own_reg + ((((long long)me * Tmax + t) * hw + col) >> 1) * 16, __float_as_uint(accs[u]), __float_as_uint(nb), epoch);
        }
      }
      // pass B (owner of this tile's columns): contributions in RANK ORDER + residual, rounded; broadcast h and the tile's sum of squares
      if (owner == me) {
        for (int t = split; t < T_; t += S) {
          float h0 = 0.f, h1 = 0.f;
          if (even) {
            uint4 uu[8];
            unsigned spins = 0;
            for (;;) {
              bool ok = true;
#pragma unroll
              for (int r = 0; r < 8; ++r)
                if (r < W) {
                  uu[r] = ld_ll16(mine + ((((long long)r * Tmax + t) * hw + col) >> 1) * 16);
                  ok = ok && uu[r].y == epoch && uu[r].w == epoch;
                }
              if (ok) break;
              if (++spins > kPeerSpinLimit) peer_timeout("reduce-scatter", me);
            }
            float a0 = 0.f, a1 = 0.f;
#pragma unroll
            for (int r = 0; r < 8; ++r)
              if (r < W) {
                a0 += __uint_as_float(uu[r].x);
                a1 += __uint_as_float(uu[r].z);
              }
            const uint32_t rv = *reinterpret_cast<const uint32_t*>(hrow + (long long)t * p.n + f);
            const T* rp = reinterpret_cast<const T*>(&rv);
            h0 = rnd<T>(DT<T>::to_f(rp[0]) + rnd<T>(a0));
            h1 = rnd<T>(DT<T>::to_f(rp[1]) + rnd<T>(a1));
            const uint32_t wv = pack_pair<T>(h0, h1);
            const long long unit = ((long long)me * Tmax + t) * hw + col;
            const long long addr = ag_off + (unit >> 2) * 16 + ((unit >> 1) & 1) * 8;
#pragma unroll
            for (int r = 0; r < 8; ++r)
              if (r < W) st_ll8(p.peer_region[r] + addr, wv, epoch);
          }
          if (p.ssq_out != nullptr) {                         // kernel-uniform
            const float ss = warp_sum(h0 * h0 + h1 * h1);
            if (lane == 0) red[ft >> 5] = ss;
            named_bar_sync(1, 128);
            if (ft < W)
              st_ll8(p.peer_region[ft] + sq_off + ((long long)t * gridDim.x + blockIdx.x) * 8, __float_as_uint(red[0] + red[1] + red[2] + red[3]),
                     epoch);
            named_bar_sync(1, 128);                          // red is rewritten by the next token
          }
        }
      }
      // pass C (every rank, the owner included): h and the statistic from the broadcast -- the same numbers everywhere
      for (int t = split; t < T_; t += S) {
        if (even) {
          const long long unit = ((long long)owner * Tmax + t) * hw + col;
          const uint8_t* src = mine + ag_off + (unit >> 2) * 16 + ((unit >> 1) & 1) * 8;
          uint2 v;
          unsigned spins = 0;
          while ((v = ld_ll8(src)).y != epoch)
            if (++spins > kPeerSpinLimit) peer_timeout("all-gather", me);
          *reinterpret_cast<uint32_t*>(hrow + (long long)t * p.n + f) = v.x;
        } else if (ft == 1 && p.ssq_out != nullptr) {
          const uint8_t* src = mine + sq_off + ((long long)t * gridDim.x + blockIdx.x) * 8;
          uint2 v;
          unsigned spins = 0;
          while ((v = ld_ll8(src)).y != epoch)
            if (++spins > kPeerSpinLimit) peer_timeout("statistics gather", me);
          p.ssq_out[(long long)t * gridDim.x + blockIdx.x] = __uint_as_float(v.x);
        }
      }
    } else
    for (int tb = split; tb < T_; tb += kGroup * S)
    for (int u = 0; u < kGroup; ++u) {
      if (u == 0) {
#pragma unroll
        for (int u2 = 0; u2 < kGroup; ++u2) {
          const int t2 = tb + u2 * S;
          float a2 = 0.f;
          if (t2 < T_)
            for (int s2 = 0; s2 < S; ++s2) a2 += *cluster.map_shared_rank(&part_s[t2 * kBM + ft], s2);      // split order, DSMEM
          accs[u2] = a2;
        }
      }
      const int t = tb + u * S;
      if (t >= T_) break;                                    // CTA-uniform
      const float acc = accs[u];
      if (mode == CTS_FUSED_RESIDUAL) {
        float r = 0.f;
        if (f_ok) {
          T* hp = reinterpret_cast<T*>(p.h) + (long long)t * p.n + f;
          r = rnd<T>(DT<T>::to_f(*hp) + rnd<T>(acc));
          *hp = DT<T>::from_f(r);
        }
        if (p.ssq_out != nullptr) {                           // kernel-uniform: this tile's share of sum(h^2) for the next RMSNorm
          const float ss = warp_sum(r * r);
          if (lane == 0) red[ft >> 5] = ss;
          named_bar_sync(1, 128);
          if (ft == 0) p.ssq_out[(long long)t * gridDim.x + blockIdx.x] = red[0] + red[1] + red[2] + red[3];
          named_bar_sync(1, 128);
        }
      } else if (mode == CTS_FUSED_SWIGLU) {
        // tile = 64 gate rows then the 64 matching up rows: the up half publishes dtype(u), the gate half finishes
        if (ft >= 64) xch[ft - 64] = rnd<T>(acc);
        named_bar_sync(1, 128);
        if (ft < 64 && f_ok) {
          const long long i = (long long)(f0 >> 1) + ft;     // output feature: tile * 64 + ft
          reinterpret_cast<T*>(p.act)[(long long)t * (p.n >> 1) + i] = DT<T>::from_f(rnd<T>(silu_f(rnd<T>(acc))) * xch[ft]);
        }
        named_bar_sync(1, 128);                              // xch is rewritten by the next token
      } else {
        // QKV: bias, per-head RMSNorm (Qwen3), RoPE, q_out / paged KV write -- head = f / d, all inside this tile
        const int d = p.d, half = d >> 1;
        const int head = (int)(f / d), i = (int)(f % d);
        const bool is_q = head < p.nh, is_k = !is_q && head < p.nh + p.nkv;
        float x = acc;
        if (p.bias != nullptr && f_ok) x += DT<T>::to_f(reinterpret_cast<const T*>(p.bias)[f]);
        x = rnd<T>(x);
        if (p.q_norm != nullptr || p.k_norm != nullptr) {    // kernel-uniform
          // statistic over the d features of the head: d = 128 -> the four warps, d = 64 -> warps {0,1} and {2,3} of the tile
          float ss = warp_sum(f_ok ? x * x : 0.f);
          if (lane == 0) red[ft >> 5] = ss;
          named_bar_sync(1, 128);
          float tot;
          if (d == 128) tot = red[0] + red[1] + red[2] + red[3];
          else tot = (ft < 64) ? red[0] + red[1] : red[2] + red[3];
          named_bar_sync(1, 128);
          const T* nw = reinterpret_cast<const T*>(is_q ? p.q_norm : (is_k ? p.k_norm : nullptr));
          if (nw != nullptr && f_ok) {
            const float inv = 1.0f / sqrtf(tot / (float)d + p.eps);
            x = rnd<T>(DT<T>::to_f(nw[i]) * rnd<T>(x * inv));
          }
        }
        xch[ft] = x;
        named_bar_sync(1, 128);
        if (f_ok) {
          if (is_q || is_k) {
            const int pos = p.positions[t];
            const int ii = i < half ? i : i - half;
            const float c = DT<T>::to_f(reinterpret_cast<const T*>(p.cos_tab)[(long long)pos * half + ii]);
            const float sn = DT<T>::to_f(reinterpret_cast<const T*>(p.sin_tab)[(long long)pos * half + ii]);
            const float xp = xch[i < half ? ft + half : ft - half];                      // rotate_half partner
            x = i < half ? rnd<T>(rnd<T>(x * c) + rnd<T>(-xp * sn)) : rnd<T>(rnd<T>(x * c) + rnd<T>(xp * sn));
          }
          if (is_q) {
            reinterpret_cast<T*>(p.q_out)[(long long)t * p.nh * d + (long long)head * d + i] = DT<T>::from_f(x);
          } else {
            const int kvh = is_k ? head - p.nh : head - p.nh - p.nkv;
            T* cache = reinterpret_cast<T*>(is_k ? p.k_cache : p.v_cache);
            const int slot = p.slot_map ? p.slot_map[t] : -1;
            if (cache != nullptr && slot >= 0) {
              const long long page = slot / p.page_size, off = slot % p.page_size;
              cache[((page * p.nkv + kvh) * p.page_size + off) * d + i] = DT<T>::from_f(x);
            }
          }
        }
        named_bar_sync(1, 128);                              // xch / red are rewritten by the next token
      }
    }
  }
  cluster.sync();                                            // nobody leaves while a peer still reads its tile
  __syncthreads();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_FUSED, 3);
  if (p.peer_region != nullptr && threadIdx.x == 0) {        // the last CTA of the grid to finish publishes the next epoch
    __threadfence();
    const int done = atomicAdd(&p.peer_state[1], 1) + 1;
    if (done == (int)(gridDim.x * gridDim.z)) {
      p.peer_state[1] = 0;
      p.peer_state[0] = p.peer_state[0] + 1;
      __threadfence();
    }
  }
}

template <typename T, int BN, bool NORM_IN>
int launch_fused(cts_ctx* ctx, const cts_fused_gemm_args* a, cudaStream_t stream) {
  const bool is_bf16 = a->dtype == CTS_BF16;
  CUtensorMap tm_w, tm_x;
  int rc = cts_make_tmap_2d(ctx, &tm_w, a->w, a->n, a->k, a->k, kBM, is_bf16);
  if (rc) return rc;
  if (NORM_IN) {
    tm_x = tm_w;                                            // unused: the token operand is produced in the kernel
  } else {
    rc = cts_make_tmap_2d(ctx, &tm_x, a->x, a->t, a->k, a->k, BN, is_bf16);
    if (rc) return rc;
  }
  FusedParams p;
  memset(&p, 0, sizeof(p));
  p.n = a->n; p.k = a->k; p.t = a->t;
  p.kb_total = (int)cdiv_ll(a->k, kBK);
  p.split = a->split_k; p.mode = a->mode;
  p.bias = a->bias; p.h = a->h; p.act = a->act;
  p.positions = a->positions; p.cos_tab = a->cos_tab; p.sin_tab = a->sin_tab; p.slot_map = a->slot_map;
  p.q_out = a->q_out; p.k_cache = a->k_cache; p.v_cache = a->v_cache; p.q_norm = a->q_norm; p.k_norm = a->k_norm; p.eps = a->eps;
  p.nh = a->nh; p.nkv = a->nkv; p.d = a->head_dim; p.page_size = a->page_size;
  p.norm_h = a->norm_h; p.norm_w = a->norm_w; p.ssq_in = a->ssq_in; p.ssq_tiles = a->ssq_tiles; p.norm_eps = a->norm_eps;
  p.ssq_out = a->ssq_out;
  p.peer_region = (uint8_t* const*)a->peer_regions; p.peer_state = a->peer_state;
  p.peer_rank = a->peer_rank; p.peer_world = a->peer_world; p.peer_max_tokens = a->peer_max_tokens;
  constexpr int kStage = kBM * kBK * 2 + BN * kBK * 2;
  int stages = ctx->decode_stages * 1024 / kStage;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) stages = 2;
  while ((size_t)stages * kStage < (size_t)BN * kBM * 4) ++stages;       // the parked fp32 tile reuses the ring
  p.stages = stages;
  const size_t smem = (size_t)stages * kStage + 1024;
  auto kern = gemm_decode_fused_kernel<T, BN, NORM_IN>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)cdiv_ll(a->n, kBM), 1, (unsigned)a->split_k);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = 1;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = (unsigned)a->split_k;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  CTS_CUDA(ctx, cudaLaunchKernelEx(&cfg, kern, tm_w, tm_x, p));
  return CTS_OK;
}

}  // namespace

extern "C" int cts_gemm_decode_fused(cts_ctx* ctx, const cts_fused_gemm_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr && a->w, "null args / w");
  CTS_CHECK_ARG(ctx, a->n > 0 && a->k > 0 && a->t > 0 && a->t <= 32, "n, k > 0 and 1 <= t <= 32 (decode-sized step)");
  CTS_CHECK_ARG(ctx, a->dtype == CTS_BF16 || a->dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, a->split_k >= 1 && a->split_k <= 8, "1 <= split_k <= 8 (portable cluster size)");
  CTS_CHECK_ARG(ctx, a->split_k <= cdiv_ll(a->k, kBK), "split_k exceeds the number of 64-wide K blocks");
  CTS_CHECK_ARG(ctx, a->mode >= CTS_FUSED_RESIDUAL && a->mode <= CTS_FUSED_QKV_ROPE, "mode");
  if (a->mode == CTS_FUSED_RESIDUAL) CTS_CHECK_ARG(ctx, a->h != nullptr, "CTS_FUSED_RESIDUAL needs h");
  if (a->mode == CTS_FUSED_SWIGLU) CTS_CHECK_ARG(ctx, a->act != nullptr && a->n % 128 == 0, "CTS_FUSED_SWIGLU needs act and n % 128 == 0");
  if (a->mode == CTS_FUSED_QKV_ROPE) {
    CTS_CHECK_ARG(ctx, a->positions && a->cos_tab && a->sin_tab && a->q_out, "CTS_FUSED_QKV_ROPE needs positions, cos/sin tables, q_out");
    CTS_CHECK_ARG(ctx, (a->head_dim == 64 || a->head_dim == 128) && a->nh > 0 && a->nkv > 0 &&
                           a->n == (long long)(a->nh + 2 * a->nkv) * a->head_dim, "head_dim 64 or 128, n = (nh + 2 nkv) * head_dim");
    CTS_CHECK_ARG(ctx, a->page_size > 0 || a->k_cache == nullptr, "page_size");
  }
  if (a->peer_regions != nullptr) {
    CTS_CHECK_ARG(ctx, a->mode == CTS_FUSED_RESIDUAL && a->peer_state != nullptr, "the in-kernel all-reduce belongs to CTS_FUSED_RESIDUAL and needs peer_state");
    CTS_CHECK_ARG(ctx, a->peer_world >= 2 && a->peer_world <= 8 && a->peer_rank >= 0 && a->peer_rank < a->peer_world, "peer_world in 2..8, peer_rank");
    CTS_CHECK_ARG(ctx, a->n % (128LL * a->peer_world) == 0, "n must be a multiple of 128 * peer_world (a tile has one owner)");
    CTS_CHECK_ARG(ctx, a->t <= a->peer_max_tokens, "t exceeds peer_max_tokens");
    CTS_CHECK_ARG(ctx, a->peer_region_bytes >= (long long)a->peer_max_tokens * a->n * 12 + (long long)a->peer_max_tokens * (a->n / 128) * 8,
                  "symmetric region too small");
  }
  const bool norm_in = a->norm_h != nullptr;
  if (norm_in) {
    CTS_CHECK_ARG(ctx, a->norm_w && a->ssq_in && a->ssq_tiles > 0 && a->k % 8 == 0, "NORM_IN needs norm_w, ssq_in, ssq_tiles > 0 and k % 8 == 0");
  } else {
    CTS_CHECK_ARG(ctx, a->x != nullptr, "x is required unless norm_h is given");
  }
  cudaStream_t st = (cudaStream_t)stream;
#define FUSED_GO(TT)                                                                                              \
  if (norm_in) return a->t <= 16 ? launch_fused<TT, 16, true>(ctx, a, st) : launch_fused<TT, 32, true>(ctx, a, st); \
  return a->t <= 16 ? launch_fused<TT, 16, false>(ctx, a, st) : launch_fused<TT, 32, false>(ctx, a, st);
  if (a->dtype == CTS_BF16) { FUSED_GO(__nv_bfloat16) }
  FUSED_GO(__half)
#undef FUSED_GO
}

CTS_TRACE_SETTER(cts_trace_set_fused)
