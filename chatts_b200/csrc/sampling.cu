// chatts_b200 -- stochastic sampling + device-side advance of the decode loop (K13, sampled variant).
// Replaces, for temperature / top-k / top-p decoding (chatts/utils/inference_tsmllm_deepspeed.py:95-100 calls
// generate(temperature=0.2); chatts/utils/llm_utils.py:166-170 builds vLLM SamplingParams(temperature, top_p)):
// transformers' TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> softmax -> multinomial, and the same
// host bookkeeping as cts_greedy_advance, so that a SAMPLED decode step is also one graph-replayable launch sequence
// with no host round trip.
//
// One CTA per sequence, no sort: the kept set {i : z_i >= tau} is found by bisection over the 16-bit ordered key of the
// (bf16 / fp16) logit -- at most 16 counting passes per filter over a row that stays in L2 (304 KB at V = 152k):
//   top-k : the largest tau with  count(z_i >= tau) >= k
//   top-p : the largest tau (>= tau_k) with  sum_{z_i >= tau} p_i >= top_p * mass(top-k set)     (ties at tau are all kept)
// then one inverse-CDF pass in INDEX order over the kept set with a counter-based uniform u(seed, step, sequence)
// (splitmix64), so a (seed, step) pair always gives the same token -- restated on the CPU in tests/cabi_double.py.
// Each thread owns a contiguous chunk with an fp32 sum; the prefix over chunks and the target u * total are fp64, so a tail token
// behind a dominant one (below ulp(1) of an fp32 prefix) keeps its share.  One block max names the single chunk that holds the
// target, and that chunk is walked from 0 against the target's offset into it.  Only tokens with mass are ever returned: a -inf
// logit (a structured-output or allowed-id refusal, a min_tokens stop id) never is.  A row without usable mass (no finite logit)
// gives cts_greedy_advance's token, found by a block-wide argmax.
// cts_sample_advance_rows runs the same kernel with every parameter read per row (the continuous engine's slots): a row with
// temperature <= 0 is greedy, and its draw is keyed on the row's own (seed, draw_step, draw_key) rather than (step, CTA index), so a
// request's tokens do not depend on the slot it occupies or on the round its steps fall in.
#include "common.cuh"

namespace {

constexpr int kSaThreads = 1024;

__host__ __device__ inline unsigned long long splitmix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// monotone map of a 16-bit float pattern to an unsigned key (larger value <=> larger key); NaN patterns sort above +inf
__device__ __forceinline__ unsigned key16(unsigned short b) { return (b & 0x8000u) ? (unsigned)(unsigned short)~b : (unsigned)(b | 0x8000u); }

template <typename T> __device__ __forceinline__ unsigned short bits16(T v) { return *reinterpret_cast<unsigned short*>(&v); }

__device__ __forceinline__ float block_sum_f(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = threadIdx.x < 32 ? red[threadIdx.x] : 0.f;      // 32 warps
  if (threadIdx.x < 32) t = warp_sum(t);
  if (threadIdx.x == 0) red[0] = t;
  __syncthreads();
  return red[0];
}
__device__ __forceinline__ float block_max_f(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = threadIdx.x < 32 ? red[threadIdx.x] : -INFINITY;
  if (threadIdx.x < 32) t = warp_max(t);
  if (threadIdx.x == 0) red[0] = t;
  __syncthreads();
  return red[0];
}

// cts_greedy_advance's token of one row for thread 0 (the first maximum, NaN never wins, 0 when no value exceeds -inf): a greedy row,
// or a sampled one without usable mass.  Kept out of line so that it does not weigh on the sampler's register allocation.
template <typename T>
__device__ __attribute__((noinline)) int block_argmax(const T* __restrict__ row, long long vocab, unsigned long long* red) {
  float best = -INFINITY;
  long long best_i = vocab;
  for (long long i = threadIdx.x; i < vocab; i += kSaThreads) {
    const float x = DT<T>::to_f(row[i]);
    if (x > best) { best = x; best_i = i; }                                  // strided: the first maximum of this thread's indices
  }
  // key = ordered value bits above the complemented index: the block max is the first maximum (-0 and +0 tie)
  unsigned u = __float_as_uint(best);
  if ((u << 1) == 0u) u = 0u;
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  unsigned long long key = best_i < vocab ? ((unsigned long long)u << 32) | (unsigned)~(unsigned)best_i : 0ull;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, key, o);
    key = w > key ? w : key;
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = key;
  __syncthreads();
  if (threadIdx.x < 32) {
    key = red[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long w = __shfl_xor_sync(0xffffffffu, key, o);
      key = w > key ? w : key;
    }
  }
  return key ? (int)~(unsigned)key : 0;
}

// Per-row sampling parameters (cts_sample_advance_rows): each non-null array replaces the launch's scalar for row b, and the draw is
// u(seed, draw_step[b], draw_key[b]) instead of u(seed, step_ptr[0], b).  All null: cts_sample_advance.
struct RowParams {
  const float* temperature;
  const int* top_k;
  const float* top_p;
  const unsigned long long* seed;
  const int* draw_key;
  int* draw_step;
};

template <typename T>
__global__ void __launch_bounds__(kSaThreads)
sample_advance_kernel(const T* __restrict__ logits, long long vocab, float inv_temp, int top_k, float top_p, unsigned long long seed,
                      RowParams rp, int* __restrict__ out_tokens, int out_ld, int* __restrict__ step_ptr, int* __restrict__ cur_ids,
                      int* __restrict__ positions, int* __restrict__ seq_lens, int* __restrict__ slot_map,
                      const int* __restrict__ page_table, int max_pages, int page_size) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  __shared__ double scan_s[32];
  __shared__ double total_s;
  __shared__ int winner_s;
  __shared__ unsigned long long argmax_s[32];
  const int b = blockIdx.x;
  // a row with temperature <= 0 (or NaN) is greedy
  bool greedy = false;
  if (rp.temperature) {
    const float t = rp.temperature[b];
    greedy = !(t > 0.f);
    inv_temp = greedy ? 1.f : 1.0f / t;                                      // IEEE division (no fast math): the host's 1.0f / temperature
  }
  if (rp.top_k) top_k = rp.top_k[b];
  if (rp.top_p) top_p = rp.top_p[b];
  if (rp.seed) seed = rp.seed[b];
  const T* row = logits + (long long)b * vocab;
  // contiguous chunk of indices per thread (multiple of 8 so the vector path stays aligned)
  const long long per = ((vocab + kSaThreads - 1) / kSaThreads + 7) / 8 * 8;
  const long long i0 = (long long)threadIdx.x * per;
  const long long i1 = i0 + per < vocab ? i0 + per : vocab;
  const bool vec = (vocab & 7) == 0 && (reinterpret_cast<uintptr_t>(row) & 15) == 0;

  // visit(fn): fn(index, value as float, 16-bit pattern) over this thread's chunk
  auto visit = [&](auto&& fn) {
    if (vec) {
      for (long long i = i0; i < i1; i += 8) {
        const uint4 u = *reinterpret_cast<const uint4*>(row + i);
        const T* p = reinterpret_cast<const T*>(&u);
#pragma unroll
        for (int j = 0; j < 8; ++j) fn(i + j, DT<T>::to_f(p[j]), bits16<T>(p[j]));
      }
    } else {
      for (long long i = i0; i < i1; ++i) fn(i, DT<T>::to_f(row[i]), bits16<T>(row[i]));
    }
  };

  if (threadIdx.x == 0) winner_s = -1;
  const int col = step_ptr ? step_ptr[0] : 0;                                // the output column; the draw's step when not per row
  if (!greedy) {
    // ---- max and partition function of z = logit / temperature
    float m = -INFINITY;
    visit([&](long long, float x, unsigned short) { if (x > m) m = x; });      // NaN never wins
    m = block_max_f(m, red);
    auto prob = [&](float x) { return x == x ? __expf((x - m) * inv_temp) : 0.f; };   // unnormalised; NaN logits get mass 0
    unsigned kmax = 0;
    visit([&](long long, float x, unsigned short bb) { if (x == x) { const unsigned k = key16(bb); if (k > kmax) kmax = k; } });
    kmax = (unsigned)block_max_f((float)kmax, red);                            // keys < 2^16 are exact in fp32
    auto mass_ge = [&](unsigned tau) {
      float s = 0.f;
      visit([&](long long, float x, unsigned short bb) { if (x == x && key16(bb) >= tau) s += prob(x); });
      return block_sum_f(s, red);
    };
    auto count_ge = [&](unsigned tau) {
      float c = 0.f;
      visit([&](long long, float x, unsigned short bb) { if (x == x && key16(bb) >= tau) c += 1.f; });
      return block_sum_f(c, red);                                              // counts <= 2^24 are exact in fp32
    };
    unsigned tau = 0;
    if (top_k > 0 && (long long)top_k < vocab) {
      unsigned lo = 0, hi = kmax + 1;                                          // count(>= lo) >= k holds, count(>= hi) = 0 does not
      while (hi - lo > 1) {
        const unsigned mid = lo + ((hi - lo) >> 1);
        if (count_ge(mid) >= (float)top_k) lo = mid; else hi = mid;
      }
      tau = lo;
    }
    float mass = mass_ge(tau);
    if (top_p > 0.f && top_p < 1.f) {
      const float target = top_p * mass;
      unsigned lo = tau, hi = kmax + 1;
      while (hi - lo > 1) {
        const unsigned mid = lo + ((hi - lo) >> 1);
        if (mass_ge(mid) >= target) lo = mid; else hi = mid;
      }
      if (lo != tau) { tau = lo; mass = mass_ge(tau); }
    }
    // ---- inverse CDF in index order over the kept set
    const int dstep = rp.draw_step ? rp.draw_step[b] : col;
    const int dkey = rp.draw_key ? rp.draw_key[b] : b;
    const unsigned long long h = splitmix64(seed ^ splitmix64(((unsigned long long)(unsigned)dstep << 32) | (unsigned)dkey));
    const double u = (double)(h >> 40) * (1.0 / 16777216.0);                  // 24 random bits -> [0, 1)
    float loc = 0.f;
    visit([&](long long, float x, unsigned short bb) { if (x == x && key16(bb) >= tau) loc += prob(x); });
    // block exclusive scan of the per-thread sums (threads own increasing index ranges), in fp64: in fp32 a prefix near the total
    // only resolves ulp(1) ~ 1.2e-7, more than a tail token behind a dominant one holds, and its rounding would both leave gaps
    // between neighbouring chunks and line every chunk start up with the grid of fp32 targets (over-weighting each chunk's first
    // token)
    double incl = loc;
  #pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double n = __shfl_up_sync(0xffffffffu, incl, o);
      if ((threadIdx.x & 31) >= o) incl += n;
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 31) scan_s[threadIdx.x >> 5] = incl;
    __syncthreads();
    if (threadIdx.x < 32) {
      double w = scan_s[threadIdx.x], wi = w;
  #pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double n = __shfl_up_sync(0xffffffffu, wi, o);
        if (threadIdx.x >= o) wi += n;
      }
      scan_s[threadIdx.x] = wi - w;                                            // exclusive prefix of the warp totals
      if (threadIdx.x == 31) total_s = wi;                                     // grand total (same summation tree every launch)
    }
    __syncthreads();
    const double rel = u * total_s - (scan_s[threadIdx.x >> 5] + (incl - loc));   // where the draw lies from this chunk's start
    // the owner of the draw: the last thread with mass that starts at or before it -- exactly one thread, however the prefixes
    // of neighbouring chunks are rounded (NaN mass: none)
    const float owner = block_max_f(loc > 0.f && rel >= 0.0 ? (float)threadIdx.x : -1.f, red);
    if ((float)threadIdx.x == owner) {
      // walk the chunk from 0: an fp32 sum started at the prefix (~ total) would not move for a tail token
      const float t_loc = (float)rel;
      float acc = 0.f;
      int pick = -1, last = -1;
      visit([&](long long i, float x, unsigned short bb) {
        if (pick < 0 && x == x && key16(bb) >= tau) {
          const float p = prob(x);
          if (p > 0.f) {
            acc += p;
            last = (int)i;
            if (t_loc < acc) pick = (int)i;
          }
        }
      });
      winner_s = pick >= 0 ? pick : last;                                      // rounding left the walk short: the last token WITH mass
    }
  }
  __syncthreads();
  int tok = winner_s;
  if (tok < 0) tok = block_argmax(row, vocab, argmax_s);
  if (threadIdx.x == 0) {
    if (rp.draw_step) rp.draw_step[b] += 1;                                  // tokens the row has produced, greedy ones included
    if (out_tokens) out_tokens[(long long)b * out_ld + col] = tok;
    if (cur_ids) cur_ids[b] = tok;
    if (positions) {
      const int np = positions[b] + 1;
      positions[b] = np;
      if (seq_lens) seq_lens[b] = seq_lens[b] + 1;
      if (slot_map && page_table) {
        const int pg = np / page_size;
        slot_map[b] = pg < max_pages ? page_table[(long long)b * max_pages + pg] * page_size + np % page_size : -1;
      }
    }
    if (step_ptr) {
      __threadfence();
      const int done = atomicAdd(&step_ptr[1], 1) + 1;                       // step_ptr = {step, done-counter}
      if (done == (int)gridDim.x) {
        step_ptr[1] = 0;
        step_ptr[0] = col + 1;
      }
    }
  }
}

}  // namespace

namespace {
int launch_sample_advance(cts_ctx* ctx, const void* logits, long long vocab, int batch, float inv_temp, int top_k, float top_p,
                          unsigned long long seed, const RowParams& rp, int* out_tokens, int out_ld, int* step_ptr, int* cur_ids,
                          int* positions, int* seq_lens, int* slot_map, const int* page_table, int max_pages, int page_size, int dtype,
                          void* stream) {
  if (dtype == CTS_BF16) {
    CTS_CUDA(ctx, launch_pdl(sample_advance_kernel<__nv_bfloat16>, dim3((unsigned)batch), dim3(kSaThreads), 0, (cudaStream_t)stream, 1,
                             (const __nv_bfloat16*)logits, vocab, inv_temp, top_k, top_p, seed, rp, out_tokens, out_ld, step_ptr, cur_ids,
                             positions, seq_lens, slot_map, page_table, max_pages, page_size));
  } else {
    CTS_CUDA(ctx, launch_pdl(sample_advance_kernel<__half>, dim3((unsigned)batch), dim3(kSaThreads), 0, (cudaStream_t)stream, 1,
                             (const __half*)logits, vocab, inv_temp, top_k, top_p, seed, rp, out_tokens, out_ld, step_ptr, cur_ids, positions,
                             seq_lens, slot_map, page_table, max_pages, page_size));
  }
  return CTS_OK;
}
}  // namespace

extern "C" int cts_sample_advance(cts_ctx* ctx, const void* logits, long long vocab, int batch, float temperature, int top_k,
                                  float top_p, unsigned long long seed, int* out_tokens, int out_ld, int* step_ptr, int* cur_ids,
                                  int* positions, int* seq_lens, int* slot_map, const int* page_table, int max_pages, int page_size,
                                  int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, logits != nullptr && vocab > 0 && vocab <= (1LL << 24) && batch >= 0, "logits / vocab (<= 2^24) / batch");
  CTS_CHECK_ARG(ctx, temperature > 0.f, "temperature must be > 0 (greedy decoding is cts_greedy_advance)");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, page_size > 0 || slot_map == nullptr, "page_size");
  if (batch == 0) return CTS_OK;
  return launch_sample_advance(ctx, logits, vocab, batch, 1.0f / temperature, top_k, top_p, seed, RowParams{}, out_tokens, out_ld, step_ptr,
                               cur_ids, positions, seq_lens, slot_map, page_table, max_pages, page_size, dtype, stream);
}

extern "C" int cts_sample_advance_rows(cts_ctx* ctx, const void* logits, long long vocab, int batch, const float* temperature,
                                       const int* top_k, const float* top_p, const unsigned long long* seed, const int* draw_key,
                                       int* draw_step, int* out_tokens, int out_ld, int* step_ptr, int* cur_ids, int* positions,
                                       int* seq_lens, int* slot_map, const int* page_table, int max_pages, int page_size, int dtype,
                                       void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, logits != nullptr && vocab > 0 && vocab <= (1LL << 24) && batch >= 0, "logits / vocab (<= 2^24) / batch");
  CTS_CHECK_ARG(ctx, temperature != nullptr && top_k != nullptr && top_p != nullptr && seed != nullptr && draw_key != nullptr &&
                     draw_step != nullptr, "null per-row temperature / top_k / top_p / seed / draw_key / draw_step");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, page_size > 0 || slot_map == nullptr, "page_size");
  if (batch == 0) return CTS_OK;
  const RowParams rp{temperature, top_k, top_p, seed, draw_key, draw_step};
  return launch_sample_advance(ctx, logits, vocab, batch, 1.f, 0, 1.f, 0ull, rp, out_tokens, out_ld, step_ptr, cur_ids, positions, seq_lens,
                               slot_map, page_table, max_pages, page_size, dtype, stream);
}

// ------------------------------------------------------------------------------------------------
// Log probabilities (vLLM's raw logprobs): per row, log_softmax of the 16-bit logits at the chosen id, the chosen id's rank, and the
// k largest entries.  A row is cut into slices of kLpSlice logits, one CTA each; every CTA reduces its slice to (max, sum of exp,
// count above the chosen logit, its k best (value, id) keys) in the workspace, and the last CTA of the row to arrive merges the
// slices in slice order (so the result does not depend on arrival order) and resets the row's arrival counter.
// ------------------------------------------------------------------------------------------------
namespace {
constexpr int kLpThreads = 256;
constexpr int kLpPer = 8;                            // logits per thread: one 16-byte load
constexpr int kLpSlice = kLpThreads * kLpPer;        // logits per CTA
constexpr int kLpMaxK = 20;

// a top-k key: the value's ordered bits above the complemented id, so the larger key is the larger value and, among equal values,
// the smaller id; -0 is folded onto +0 (equal values tie).  0 is never a key (the smallest, -inf, has high word 0x007fffff).
__device__ __forceinline__ unsigned long long lp_key(float x, int id) {
  unsigned u = __float_as_uint(x);
  if ((u << 1) == 0u) u = 0u;
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (unsigned)~(unsigned)id;
}
__device__ __forceinline__ float lp_key_value(unsigned long long key) {
  const unsigned u = (unsigned)(key >> 32);
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
__device__ __forceinline__ int lp_key_id(unsigned long long key) { return (int)~(unsigned)key; }

// (max, sum of exp(x - max)) of two parts; NaN never enters, -inf contributes nothing
__device__ __forceinline__ void lp_merge(float& m, float& s, float m2, float s2) {
  const float mm = fmaxf(m, m2);
  if (mm == -INFINITY) { m = mm; s = 0.f; return; }
  s = (m == mm ? s : s * expf(m - mm)) + (m2 == mm ? s2 : s2 * expf(m2 - mm));
  m = mm;
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}
__device__ __forceinline__ unsigned long long block_max_u64(unsigned long long v, unsigned long long* red) {
  v = warp_max_u64(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = threadIdx.x < kLpThreads / 32 ? red[threadIdx.x] : 0ull;
  if (threadIdx.x < 32) v = warp_max_u64(v);
  if (threadIdx.x == 0) red[0] = v;
  __syncthreads();
  return red[0];
}
// block-wide (max, sum, count), combined in a fixed tree
__device__ __forceinline__ void block_lp_stats(float& m, float& s, int& c, float* fred, int* cred) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
    lp_merge(m, s, m2, s2);
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { fred[threadIdx.x >> 5] = m; fred[32 + (threadIdx.x >> 5)] = s; cred[threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kLpThreads / 32; ++w) { lp_merge(m, s, fred[w], fred[32 + w]); c += cred[w]; }
    fred[0] = m; fred[32] = s; cred[0] = c;
  }
  __syncthreads();
  m = fred[0]; s = fred[32]; c = cred[0];
}

// one slice record in the workspace: {max, sum} {count, -} then k keys (8-byte words)
template <typename T>
__global__ void __launch_bounds__(kLpThreads)
logprobs_kernel(const T* __restrict__ logits, long long vocab, long long ld, const int* __restrict__ chosen, int chosen_ld,
                const int* __restrict__ step_ptr, int k, float* __restrict__ out_logprob, int* __restrict__ out_rank,
                int* __restrict__ out_topk_ids, float* __restrict__ out_topk_logprobs, int out_ld, int* __restrict__ counters,
                unsigned long long* __restrict__ records) {
  pdl_trigger();
  pdl_wait();
  __shared__ float fred[64];
  __shared__ int cred[32];
  __shared__ unsigned long long kred[32];
  __shared__ int last_s;
  const int slice = blockIdx.x, nslice = gridDim.x, r = blockIdx.y;
  const T* row = logits + (long long)r * ld;
  const int col = step_ptr ? step_ptr[0] - 1 : 0;
  const int cid = chosen ? chosen[(long long)r * chosen_ld + col] : -1;
  const float xc = (cid >= 0 && cid < vocab) ? DT<T>::to_f(row[cid]) : NAN;

  // ---- this CTA's slice: 8 logits per thread
  const long long i0 = (long long)slice * kLpSlice + (long long)threadIdx.x * kLpPer;
  float x[kLpPer];
  if (i0 + kLpPer <= vocab && (ld & 7) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + i0);
    const T* p = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int j = 0; j < kLpPer; ++j) x[j] = DT<T>::to_f(p[j]);
  } else {
#pragma unroll
    for (int j = 0; j < kLpPer; ++j) x[j] = i0 + j < vocab ? DT<T>::to_f(row[i0 + j]) : NAN;
  }
  float m = -INFINITY, s = 0.f;
  int c = 0;
#pragma unroll
  for (int j = 0; j < kLpPer; ++j) {
    const float v = x[j];
    if (v != v) continue;                                                    // NaN: no mass, no rank, not a candidate
    c += v > xc;
    if (v > m) { s = s * expf(m - v) + 1.f; m = v; }
    else if (v != -INFINITY) s += expf(v - m);
  }
  block_lp_stats(m, s, c, fred, cred);
  unsigned long long* rec = records + ((long long)r * nslice + slice) * (2 + k);
  if (threadIdx.x == 0) {
    rec[0] = ((unsigned long long)__float_as_uint(s) << 32) | __float_as_uint(m);
    rec[1] = (unsigned)c;
  }
  // k best of the slice: k rounds of a block max over each thread's best key below the previous winner
  auto best_below = [&](unsigned long long lim) {
    unsigned long long b = 0ull;
#pragma unroll
    for (int j = 0; j < kLpPer; ++j) {
      if (x[j] == x[j]) {
        const unsigned long long kk = lp_key(x[j], (int)(i0 + j));
        if (kk < lim && kk > b) b = kk;
      }
    }
    return b;
  };
  unsigned long long mine = k > 0 ? best_below(~0ull) : 0ull;
  for (int j = 0; j < k; ++j) {
    const unsigned long long w = block_max_u64(mine, kred);
    if (threadIdx.x == 0) rec[2 + j] = w;
    if (w != 0ull && mine == w) mine = best_below(w);                        // keys are unique: one thread moves on
  }

  // ---- the last CTA of the row merges the slices
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last_s = atomicAdd(&counters[r], 1) == nslice - 1;
  }
  __syncthreads();
  if (!last_s) return;
  __threadfence();
  const unsigned long long* recs = records + (long long)r * nslice * (2 + k);
  m = -INFINITY; s = 0.f; c = 0;
  for (int q = threadIdx.x; q < nslice; q += kLpThreads) {
    const unsigned long long a = __ldcg(recs + (long long)q * (2 + k));
    lp_merge(m, s, __uint_as_float((unsigned)a), __uint_as_float((unsigned)(a >> 32)));
    c += (int)(unsigned)__ldcg(recs + (long long)q * (2 + k) + 1);
  }
  block_lp_stats(m, s, c, fred, cred);
  const float log_s = logf(s);
  const long long o = (long long)r * out_ld + col;
  if (threadIdx.x == 0) {
    if (out_logprob) out_logprob[o] = (xc - m) - log_s;
    if (out_rank) out_rank[o] = xc == xc ? 1 + c : 0;
    counters[r] = 0;                                                         // ready for the next launch (graph replays included)
  }
  const long long ncand = (long long)nslice * k;
  auto cand_below = [&](unsigned long long lim) {
    unsigned long long b = 0ull;
    for (long long q = threadIdx.x; q < ncand; q += kLpThreads) {
      const unsigned long long kk = __ldcg(recs + (q / k) * (2 + k) + 2 + q % k);
      if (kk < lim && kk > b) b = kk;
    }
    return b;
  };
  mine = k > 0 ? cand_below(~0ull) : 0ull;
  for (int j = 0; j < k; ++j) {
    const unsigned long long w = block_max_u64(mine, kred);
    if (threadIdx.x == 0) {
      out_topk_ids[o * k + j] = w ? lp_key_id(w) : -1;
      out_topk_logprobs[o * k + j] = w ? (lp_key_value(w) - m) - log_s : NAN;
    }
    if (w != 0ull && mine == w) mine = cand_below(w);
  }
}
}  // namespace

extern "C" long long cts_logprobs_workspace_floats(int rows, long long vocab, int k) {
  if (rows <= 0 || vocab <= 0 || k < 0) return 0;
  const long long nslice = (vocab + kLpSlice - 1) / kLpSlice;
  return (long long)rows * nslice * (2 + k) * 2;
}

extern "C" int cts_logprobs(cts_ctx* ctx, const void* logits, long long vocab, long long ld, int rows, const int* chosen, int chosen_ld,
                            const int* step_ptr, int k, float* out_logprob, int* out_rank, int* out_topk_ids, float* out_topk_logprobs,
                            int out_ld, float* workspace, int* counters, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, vocab > 0 && vocab <= (1LL << 24) && ld >= vocab && rows >= 0 && rows <= 65535, "vocab (<= 2^24) / ld (>= vocab) / rows (<= 65535)");
  CTS_CHECK_ARG(ctx, k >= 0 && k <= kLpMaxK, "k must be in [0, 20]");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (rows == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, logits != nullptr && workspace != nullptr && counters != nullptr, "null logits / workspace / counters");
  CTS_CHECK_ARG(ctx, (reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "workspace must be 8-byte aligned");
  CTS_CHECK_ARG(ctx, (out_logprob == nullptr && out_rank == nullptr) || (chosen != nullptr && chosen_ld >= 1), "chosen ids for the chosen logprob / rank");
  CTS_CHECK_ARG(ctx, k == 0 || (out_topk_ids != nullptr && out_topk_logprobs != nullptr), "null top-k outputs");
  CTS_CHECK_ARG(ctx, out_ld >= 1, "out_ld");
  const long long nslice = (vocab + kLpSlice - 1) / kLpSlice;
  auto* records = reinterpret_cast<unsigned long long*>(workspace);
  const dim3 grid((unsigned)nslice, (unsigned)rows);
  if (dtype == CTS_BF16)
    CTS_CUDA(ctx, launch_pdl(logprobs_kernel<__nv_bfloat16>, grid, dim3(kLpThreads), 0, (cudaStream_t)stream, 1, (const __nv_bfloat16*)logits,
                             vocab, ld, chosen, chosen_ld, step_ptr, k, out_logprob, out_rank, out_topk_ids, out_topk_logprobs, out_ld, counters,
                             records));
  else
    CTS_CUDA(ctx, launch_pdl(logprobs_kernel<__half>, grid, dim3(kLpThreads), 0, (cudaStream_t)stream, 1, (const __half*)logits, vocab, ld,
                             chosen, chosen_ld, step_ptr, k, out_logprob, out_rank, out_topk_ids, out_topk_logprobs, out_ld, counters, records));
  return CTS_OK;
}

// ------------------------------------------------------------------------------------------------
// Repetition penalty (transformers RepetitionPenaltyLogitsProcessor; the checkpoint's generation_config.json may set it): for every
// token id that already occurs in the row's sequence -- prompt and generated part -- logit = logit / penalty if logit > 0 else
// logit * penalty, applied ONCE however often the token occurred.  The occurrence set is a bit mask [batch, ceil(vocab / 32)]:
//   cts_rep_penalty_mark  sets the bits of (row, token) pairs (the prompt once, then the new token of every step)
//   cts_rep_penalty_apply rewrites the logits of the marked tokens in place, before the argmax / sampling kernel reads them.
// ------------------------------------------------------------------------------------------------
namespace {
__global__ void rep_mark_kernel(const int* __restrict__ tokens, const int* __restrict__ rows, int n, unsigned* __restrict__ seen,
                                int words_per_row, long long vocab) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = tokens[i];
  const int r = rows != nullptr ? rows[i] : i;
  if (t < 0 || t >= vocab || r < 0) return;
  atomicOr(&seen[(long long)r * words_per_row + (t >> 5)], 1u << (t & 31));
}

template <typename T>
__global__ void rep_apply_kernel(T* __restrict__ logits, long long vocab, long long ld, const unsigned* __restrict__ seen,
                                 int words_per_row, float penalty) {
  pdl_trigger();
  pdl_wait();
  const long long b = blockIdx.y;
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= words_per_row) return;
  unsigned bits = seen[b * words_per_row + w];
  while (bits) {
    const int j = __ffs(bits) - 1;
    bits &= bits - 1;
    const long long t = (long long)w * 32 + j;
    if (t < vocab) {
      const float v = DT<T>::to_f(logits[b * ld + t]);
      logits[b * ld + t] = DT<T>::from_f(v > 0.f ? v / penalty : v * penalty);      // the processor works in the logits' dtype
    }
  }
}
}  // namespace

extern "C" int cts_rep_penalty_mark(cts_ctx* ctx, const int* tokens, const int* rows, int n, unsigned* seen, int words_per_row,
                                    long long vocab, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, n >= 0 && words_per_row > 0 && vocab > 0 && vocab <= 32LL * words_per_row, "n / words_per_row / vocab");
  if (n == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, tokens != nullptr && seen != nullptr, "null tokens / seen");
  CTS_CUDA(ctx, launch_pdl(rep_mark_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, 1, tokens, rows, n, seen,
                           words_per_row, vocab));
  return CTS_OK;
}

extern "C" int cts_rep_penalty_apply(cts_ctx* ctx, void* logits, long long vocab, long long ld, int batch, const unsigned* seen,
                                     int words_per_row, float penalty, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, batch >= 0 && batch <= 65535 && vocab > 0 && ld >= vocab && words_per_row > 0 && vocab <= 32LL * words_per_row, "shape");
  CTS_CHECK_ARG(ctx, penalty > 0.f, "penalty must be > 0");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (batch == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, logits != nullptr && seen != nullptr, "null logits / seen");
  dim3 grid((unsigned)((words_per_row + 255) / 256), (unsigned)batch);
  if (dtype == CTS_BF16)
    CTS_CUDA(ctx, launch_pdl(rep_apply_kernel<__nv_bfloat16>, grid, dim3(256), 0, (cudaStream_t)stream, 1, (__nv_bfloat16*)logits, vocab, ld, seen,
                             words_per_row, penalty));
  else
    CTS_CUDA(ctx, launch_pdl(rep_apply_kernel<__half>, grid, dim3(256), 0, (cudaStream_t)stream, 1, (__half*)logits, vocab, ld, seen, words_per_row,
                             penalty));
  return CTS_OK;
}
