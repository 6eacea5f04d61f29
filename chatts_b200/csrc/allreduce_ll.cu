// chatts_b200 -- tensor-parallel row-parallel tail, LOW-LATENCY variant: a two-shot all-reduce whose flags travel INSIDE the
// data (the "LL" idea of collective libraries: every 8-byte word on the wire is {4 bytes of payload, 4 bytes of epoch}), so the
// kernel contains no system-scope fence, no separate flag store and no second round trip per hop:
//
//     h = resid + dtype( sum over ranks of partial_r ) ;  norm_out = RMSNorm(h) * w          (vllm qwen2.py:100-116,168-174)
//
// The one-shot kernel of allreduce.cu pushes every rank's full fp32 partial to every rank ((W-1) x T x H x 4 bytes of NVLink
// egress per call, ordered by fence + release flag + acquire poll); at TP8 those calls dominate the decode step.  Here, per call and token:
//   phase A  each rank sums its split-K partials and SCATTERS: columns of owner j go to rank j          (reduce-scatter, fp32)
//   phase B  the owner waits for the W contributions of its columns (polling the epoch words of the data itself), adds them in
//            RANK ORDER, adds the residual, rounds -> its H/W columns of h, plus the sum of squares of those columns; it
//            BROADCASTS both                                                                         (all-gather, model dtype)
//   phase C  every rank waits for the W chunks of h and the W x C partial sums of squares, adds those in a fixed order (so every
//            rank computes the same statistic from the same numbers: h and norm_out are bit-identical on all ranks without a
//            broadcast of the result), writes resid_out and norm_out.
// Egress per call: T x H x (8 + 4) bytes instead of (W-1) x T x H x 4; two one-way NVLink hops instead of two round trips.
//
// Wire format: 16-byte units {d0, epoch, d1, epoch}.  A unit is valid when BOTH epoch words equal the call's epoch (an 8-byte
// aligned half of a vector store is delivered atomically; the two halves may arrive separately).  Epochs only grow (state[0] is
// advanced by the last CTA of every call) and the region starts zeroed, so a stale unit never looks valid.  The two buffer sets
// alternate between o_proj and down_proj exactly as in allreduce.cu: a rank that completes call n+1 has received data from every
// peer's call n+1, which those peers launched after their call n had completed -- that is what licenses overwriting the units of
// call n in call n+2 (tests/test_peer_ll_protocol.py runs this protocol under random schedules, torn stores included).
//
// Region layout (one per buffer set and rank, `region_bytes` >= max_tokens*h*12 + world*max_tokens*128):
//   RS  [src rank][max_tokens][h/W] fp32 as units of 2 columns      at 0                  (max_tokens*h*8 bytes)
//   AG  [owner  ][max_tokens][h/W] dtype as units of 4 columns      at max_tokens*h*8     (max_tokens*h*4 bytes)
//   SQ  [owner  ][max_tokens][8]   one float per unit               at max_tokens*h*12
// grid (C, T): CTA (c, t) handles, of token t, sub-slice c (h/(W*C) columns) of EVERY owner's chunk.
#include "common.cuh"
#include "trace.cuh"

namespace {

constexpr int kLLThreads = 256;
constexpr int kLLMaxRanks = 8;
constexpr int kLLMaxC = 8;
constexpr unsigned kLLSpinLimit = 1u << 24;

#ifdef CTS_HOST_SHIM
// tests/cuda_on_cpu: the same wire format on the host -- two 8-byte halves written and read separately (a scheduling point in
// between, so that a torn unit is actually observable), ranks are processes sharing the regions
__device__ __forceinline__ void st_ll(void* p, uint32_t d0, uint32_t d1, uint32_t epoch) {
  volatile uint64_t* q = reinterpret_cast<volatile uint64_t*>(p);
  q[0] = (uint64_t)d0 | ((uint64_t)epoch << 32);
  sched_yield();
  q[1] = (uint64_t)d1 | ((uint64_t)epoch << 32);
}
__device__ __forceinline__ uint4 ld_ll(const void* p) {
  const volatile uint64_t* q = reinterpret_cast<const volatile uint64_t*>(p);
  const uint64_t a = q[0], b = q[1];
  uint4 v = {(uint32_t)a, (uint32_t)(a >> 32), (uint32_t)b, (uint32_t)(b >> 32)};
  shim_yield();                                            // pollers must let the other threads of the block (and the peers) run
  static unsigned n = 0;
  if ((++n & 1023u) == 0) sched_yield();
  return v;
}
#else
__device__ __forceinline__ void st_ll(void* p, uint32_t d0, uint32_t d1, uint32_t epoch) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(d0), "r"(epoch), "r"(d1), "r"(epoch) : "memory");
}
__device__ __forceinline__ uint4 ld_ll(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
#endif
__device__ __forceinline__ bool ll_ok(const uint4& v, uint32_t epoch) { return v.y == epoch && v.w == epoch; }

__device__ void ll_timeout(const char* what, int rank) {
  printf("chatts_b200: peer all-reduce (LL) timed out in %s on rank %d (block %d,%d thread %d)\n", what, rank, blockIdx.x, blockIdx.y,
         threadIdx.x);
  __trap();
}

template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b) {
  T v[2] = {DT<T>::from_f(a), DT<T>::from_f(b)};
  return *reinterpret_cast<uint32_t*>(v);
}
template <typename T> __device__ __forceinline__ void unpack2(uint32_t u, float& a, float& b) {
  const T* v = reinterpret_cast<const T*>(&u);
  a = DT<T>::to_f(v[0]);
  b = DT<T>::to_f(v[1]);
}

template <typename T, int W>
__global__ void __launch_bounds__(kLLThreads)
peer_allreduce_ll_kernel(const float* __restrict__ local_part, int S, long long t_total, uint8_t* const* __restrict__ peer_region,
                         int* __restrict__ state, int rank, int max_tokens, const T* __restrict__ resid_in, T* __restrict__ resid_out,
                         const T* __restrict__ norm_w, float eps, T* __restrict__ norm_out, int h) {
  pdl_trigger();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_OTHER, 0);
  pdl_wait();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_OTHER, 1);
  const int C = (int)gridDim.x, c = (int)blockIdx.x;
  const long long t = blockIdx.y;
  const int hw = h / W, wc = hw / C;                     // owner chunk, sub-slice of this CTA (wc % 4 == 0, host-checked)
  const uint32_t epoch = (uint32_t)(state[0] + 1);      // state[0] is only advanced by the last CTA of this kernel to finish
  const long long ag_off = (long long)max_tokens * h * 8, sq_off = (long long)max_tokens * h * 12;
  __shared__ uint8_t* reg[kLLMaxRanks];
  __shared__ float red[kLLThreads / 32];
  __shared__ float sq_s[kLLMaxRanks * kLLMaxC];
  __shared__ float rstd_s;
  if (threadIdx.x < W) reg[threadIdx.x] = peer_region[threadIdx.x];
  __syncthreads();

  // ---- phase A: sum my split-K partials, scatter the columns of owner j to rank j (my own chunk goes through my own region: one
  // code path, and the local store costs nothing next to the NVLink ones)
  {
    const long long stride = t_total * (long long)h;
    const int upo = wc / 2;                              // units per owner in this CTA
    for (int u = threadIdx.x; u < W * upo; u += kLLThreads) {
      const int j = u / upo, k = (u - j * upo) * 2;
      const float* p = local_part + t * h + (long long)j * hw + c * wc + k;
      // all partial loads of a batch in flight before the first add (a run-time-bounded loop of dependent adds pays one L2 round
      // trip per split); the sum still runs in split order
      float2 a = *reinterpret_cast<const float2*>(p);
      constexpr int kB = 8;
      for (int s0 = 1; s0 < S; s0 += kB) {
        float2 b[kB];
#pragma unroll
        for (int u = 0; u < kB; ++u)
          if (s0 + u < S) b[u] = *reinterpret_cast<const float2*>(p + (long long)(s0 + u) * stride);
#pragma unroll
        for (int u = 0; u < kB; ++u)
          if (s0 + u < S) {
            a.x += b[u].x;
            a.y += b[u].y;
          }
      }
      uint8_t* dst = reg[j] + ((((long long)rank * max_tokens + t) * hw + c * wc + k) >> 1) * 16;
      st_ll(dst, __float_as_uint(a.x), __float_as_uint(a.y), epoch);
    }
  }

  // ---- phase B (owner of chunk `rank`, sub-slice c): wait for the W contributions, add in rank order, residual, round, broadcast
  float ss = 0.f;
  {
    const int q = threadIdx.x;                           // 4 columns = 2 RS units = 1 AG unit per thread
    if (q < wc / 4) {
      const int k = q * 4;
      uint4 u0[W], u1[W];
      unsigned spins = 0;
      for (;;) {
        bool ok = true;
#pragma unroll
        for (int r = 0; r < W; ++r) {
          const uint8_t* src = reg[rank] + ((((long long)r * max_tokens + t) * hw + c * wc + k) >> 1) * 16;
          u0[r] = ld_ll(src);
          u1[r] = ld_ll(src + 16);
        }
#pragma unroll
        for (int r = 0; r < W; ++r) ok = ok && ll_ok(u0[r], epoch) && ll_ok(u1[r], epoch);
        if (ok) break;
        if (++spins > kLLSpinLimit) ll_timeout("reduce-scatter", rank);
      }
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
      for (int r = 0; r < W; ++r) {                      // rank order: the same sum the one-shot kernel and the NCCL-free oracle form
        a0 += __uint_as_float(u0[r].x);
        a1 += __uint_as_float(u0[r].z);
        a2 += __uint_as_float(u1[r].x);
        a3 += __uint_as_float(u1[r].z);
      }
      const long long col = (long long)rank * hw + c * wc + k;
      const uint2 rv = *reinterpret_cast<const uint2*>(resid_in + t * h + col);
      float r0, r1, r2, r3;
      unpack2<T>(rv.x, r0, r1);
      unpack2<T>(rv.y, r2, r3);
      const float h0 = rnd<T>(r0 + rnd<T>(a0)), h1 = rnd<T>(r1 + rnd<T>(a1)), h2 = rnd<T>(r2 + rnd<T>(a2)), h3 = rnd<T>(r3 + rnd<T>(a3));
      ss = h0 * h0 + h1 * h1 + h2 * h2 + h3 * h3;
      const uint32_t w0 = pack2<T>(h0, h1), w1 = pack2<T>(h2, h3);
      const long long unit = (((long long)rank * max_tokens + t) * hw + c * wc + k) >> 2;
#pragma unroll
      for (int j = 0; j < W; ++j) st_ll(reg[j] + ag_off + unit * 16, w0, w1, epoch);
    }
    // sum of squares of this sub-slice: fixed reduction tree (identical on every launch)
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x < W) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kLLThreads / 32; ++w) v += red[w];
      st_ll(reg[threadIdx.x] + sq_off + (((long long)rank * max_tokens + t) * kLLMaxC + c) * 16, __float_as_uint(v), 0u, epoch);
    }
  }

  // ---- phase C: gather h (sub-slice c of every owner's chunk) and the W x C partial statistics
  {
    if (threadIdx.x < W * C) {
      const int o = threadIdx.x / C, cc = threadIdx.x - o * C;
      const uint8_t* src = reg[rank] + sq_off + (((long long)o * max_tokens + t) * kLLMaxC + cc) * 16;
      uint4 v;
      unsigned spins = 0;
      while (!ll_ok(v = ld_ll(src), epoch))
        if (++spins > kLLSpinLimit) ll_timeout("statistics gather", rank);
      sq_s[threadIdx.x] = __uint_as_float(v.x);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int i = 0; i < W * C; ++i) tot += sq_s[i];    // owner-major, fixed order: the same number on every rank
      rstd_s = 1.0f / sqrtf(tot / (float)h + eps);
    }
    __syncthreads();
    const float inv = rstd_s;
    const int upo = wc / 4;
    for (int u = threadIdx.x; u < W * upo; u += kLLThreads) {
      const int o = u / upo, k = (u - o * upo) * 4;
      const uint8_t* src = reg[rank] + ag_off + ((((long long)o * max_tokens + t) * hw + c * wc + k) >> 2) * 16;
      uint4 v;
      unsigned spins = 0;
      while (!ll_ok(v = ld_ll(src), epoch))
        if (++spins > kLLSpinLimit) ll_timeout("all-gather", rank);
      const long long off = t * h + (long long)o * hw + c * wc + k;
      *reinterpret_cast<uint2*>(resid_out + off) = make_uint2(v.x, v.z);
      if (norm_out != nullptr) {
        float x0, x1, x2, x3, w0, w1, w2, w3;
        unpack2<T>(v.x, x0, x1);
        unpack2<T>(v.z, x2, x3);
        const uint2 wv = *reinterpret_cast<const uint2*>(norm_w + (long long)o * hw + c * wc + k);
        unpack2<T>(wv.x, w0, w1);
        unpack2<T>(wv.y, w2, w3);
        *reinterpret_cast<uint2*>(norm_out + off) =
            make_uint2(pack2<T>(w0 * rnd<T>(x0 * inv), w1 * rnd<T>(x1 * inv)), pack2<T>(w2 * rnd<T>(x2 * inv), w3 * rnd<T>(x3 * inv)));
      }
    }
  }

  // ---- the last CTA of the grid to finish publishes the new epoch for the next call
  __syncthreads();
  if (threadIdx.x == 0) {
    CTS_TRACE(CTS_TK_OTHER, 3);
    __threadfence();
    const int done = atomicAdd(&state[1], 1) + 1;
    if (done == (int)(gridDim.x * gridDim.y)) {
      state[1] = 0;
      state[0] = (int)epoch;
      __threadfence();
    }
  }
}

template <typename T, int W>
cudaError_t launch_ll(unsigned C, const float* local_partial, int split_k, long long t, const void* peer_regions, int* state, int rank,
                      int max_tokens, const void* resid_in, void* resid_out, const void* norm_w, float eps, void* norm_out, int h,
                      cudaStream_t st) {
  return launch_pdl(peer_allreduce_ll_kernel<T, W>, dim3(C, (unsigned)t), dim3(kLLThreads), 0, st, 1, local_partial, split_k, t,
                    (uint8_t* const*)peer_regions, state, rank, max_tokens, (const T*)resid_in, (T*)resid_out, (const T*)norm_w, eps,
                    (T*)norm_out, h);
}

template <typename T>
cudaError_t launch_ll_w(int world, unsigned C, const float* lp, int sk, long long t, const void* pr, int* state, int rank, int mt,
                        const void* ri, void* ro, const void* nw, float eps, void* no, int h, cudaStream_t st) {
  switch (world) {
    case 2: return launch_ll<T, 2>(C, lp, sk, t, pr, state, rank, mt, ri, ro, nw, eps, no, h, st);
    case 4: return launch_ll<T, 4>(C, lp, sk, t, pr, state, rank, mt, ri, ro, nw, eps, no, h, st);
    case 8: return launch_ll<T, 8>(C, lp, sk, t, pr, state, rank, mt, ri, ro, nw, eps, no, h, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

extern "C" long long cts_peer_ll_region_bytes(int world, int max_tokens, long long h) {
  return (long long)max_tokens * h * 12 + (long long)world * max_tokens * kLLMaxC * 16;
}

extern "C" int cts_peer_allreduce_ll(cts_ctx* ctx, const float* local_partial, int split_k, const void* peer_regions,
                                     long long region_bytes, int* state, int rank, int world, int max_tokens, const void* resid_in,
                                     void* resid_out, const void* norm_w, float eps, void* norm_out, long long t, long long h, int dtype,
                                     void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, local_partial && split_k >= 1 && peer_regions && state && resid_in && resid_out, "null pointer");
  CTS_CHECK_ARG(ctx, (world == 2 || world == 4 || world == 8) && rank >= 0 && rank < world, "the LL all-reduce is built for 2, 4 or 8 ranks");
  CTS_CHECK_ARG(ctx, (norm_w == nullptr) == (norm_out == nullptr), "norm_w / norm_out mismatch");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, t > 0 && t <= max_tokens && t <= 65535, "t must be in 1..max_tokens");
  CTS_CHECK_ARG(ctx, h > 0 && h % (4LL * world) == 0, "h must be a multiple of 4 * world");
  CTS_CHECK_ARG(ctx, region_bytes >= cts_peer_ll_region_bytes(world, max_tokens, h), "symmetric region too small for the LL layout");
  // C sub-slices per owner chunk: the largest C that keeps >= 32 four-column groups per CTA (and <= 256: one per thread in phase B);
  // a chunk too small for that is not split at all
  const long long hw = h / world;
  unsigned C = 0;
  for (unsigned cand : {8u, 4u, 2u, 1u}) {
    if (hw % (4LL * cand) != 0) continue;
    const long long groups = hw / (4LL * cand);
    if (groups >= 32 && groups <= kLLThreads) { C = cand; break; }
  }
  if (C == 0 && hw / 4 <= kLLThreads) C = 1;
  CTS_CHECK_ARG(ctx, C != 0, "h / world too large for one CTA row (needs h / (world * 8 * 4) <= 256)");
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = dtype == CTS_BF16
                      ? launch_ll_w<__nv_bfloat16>(world, C, local_partial, split_k, t, peer_regions, state, rank, max_tokens, resid_in,
                                                   resid_out, norm_w, eps, norm_out, (int)h, st)
                      : launch_ll_w<__half>(world, C, local_partial, split_k, t, peer_regions, state, rank, max_tokens, resid_in, resid_out,
                                            norm_w, eps, norm_out, (int)h, st);
  CTS_CUDA(ctx, e);
  return CTS_OK;
}

CTS_TRACE_SETTER(cts_trace_set_allreduce_ll)
