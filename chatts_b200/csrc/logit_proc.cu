// chatts_b200 -- logits processors of vLLM / OpenAI sampling: allowed_token_ids, logit_bias, min_tokens, repetition, presence and
// frequency penalties, one pass over the 16-bit logits between the decode step and the advance (chatts_b200/logit_proc.py drives it).
//   cts_logit_proc_apply   per row b and token t, in fp32, rounded once to the logits' dtype:
//                            1. bias[bias_row[b], t] == -inf (an id outside allowed_token_ids)  ->  x = -inf
//                            2. otherwise x += bias[bias_row[b], t]                             (logit_bias; 0 adds nothing)
//                            3. n_generated[b] < min_tokens[b] and t is one of the row's stop ids  ->  x = -inf
//                            4. seen bit of t set: x = x > 0 ? x / rep[b] : x * rep[b]         (cts_rep_penalty_apply's rule)
//                            5. counts[b, t] = c > 0: x = (x - frequency[b] * c) - presence[b]  (two roundings, as vLLM's apply_penalties)
//                          An entry no step touched keeps its 16-bit pattern; a row whose parameters are all neutral returns at once.
//   cts_logit_proc_update  after the advance: counts[b, cur_ids[b]] += 1, the seen bit of cur_ids[b] set, n_generated[b] += 1.
// Counts are uint16: a row generates fewer tokens than the model has positions, and logit_proc.py asserts that bound (< 65 536) where
// it allocates the table.  Half the bytes of int32 in the one [batch, vocab] table the apply kernel reads in full.
#include "common.cuh"

namespace {

constexpr int kLpThreads = 256;
constexpr int kLpVec = 8;                                    // 16 bytes of 16-bit logits per thread
constexpr int kLpSlice = kLpThreads * kLpVec;                // logits per CTA
constexpr int kLpMaxStop = 64;

// a product rounded on its own, never contracted into an FMA with the subtraction that follows it: torch and vLLM round both
__device__ __forceinline__ float mul_rn(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}

template <typename T>
__global__ void __launch_bounds__(kLpThreads)
logit_proc_apply_kernel(T* __restrict__ logits, long long vocab, long long ld, const float* __restrict__ rep,
                        const float* __restrict__ presence, const float* __restrict__ frequency, const unsigned* __restrict__ seen,
                        int words, const unsigned short* __restrict__ counts, const float* __restrict__ bias, int n_bias,
                        const int* __restrict__ bias_row, const int* __restrict__ n_generated, const int* __restrict__ min_tokens,
                        const int* __restrict__ stop_ids, int max_stop) {
  pdl_trigger();
  pdl_wait();
  __shared__ int stop_s[kLpMaxStop];
  __shared__ int n_stop_s;
  const long long b = blockIdx.y;
  const float p = rep[b], pres = presence[b], freq = frequency[b];
  const int br = bias_row[b];
  const bool use_bias = bias != nullptr && br >= 0 && br < n_bias;
  const bool use_min = max_stop > 0 && n_generated[b] < min_tokens[b];
  const bool use_rep = p != 1.f;
  const bool use_cnt = counts != nullptr && (pres != 0.f || freq != 0.f);
  if (!(use_bias || use_min || use_rep || use_cnt)) return;  // uniform per CTA: before any barrier
  if (use_min) {
    if (threadIdx.x == 0) {
      int n = 0;
      while (n < max_stop && stop_ids[b * max_stop + n] >= 0) ++n;   // padded with -1
      n_stop_s = n;
    }
    for (int k = threadIdx.x; k < max_stop; k += kLpThreads) stop_s[k] = stop_ids[b * max_stop + k];
    __syncthreads();
  }
  const long long i0 = (long long)blockIdx.x * kLpSlice + (long long)threadIdx.x * kLpVec;
  if (i0 >= vocab) return;
  const int n = vocab - i0 < kLpVec ? (int)(vocab - i0) : kLpVec;
  T* row = logits + b * ld + i0;
  T x[kLpVec];
  const bool vec = n == kLpVec && (reinterpret_cast<uintptr_t>(row) & 15) == 0;
  if (vec) {
    *reinterpret_cast<uint4*>(x) = *reinterpret_cast<const uint4*>(row);
  } else {
#pragma unroll
    for (int j = 0; j < kLpVec; ++j) if (j < n) x[j] = row[j];
  }
  float bv[kLpVec];
  if (use_bias) {
    const float* brow = bias + (long long)br * vocab + i0;
    if (n == kLpVec && (reinterpret_cast<uintptr_t>(brow) & 15) == 0) {
      *reinterpret_cast<float4*>(bv) = __ldg(reinterpret_cast<const float4*>(brow));
      *reinterpret_cast<float4*>(bv + 4) = __ldg(reinterpret_cast<const float4*>(brow + 4));
    } else {
#pragma unroll
      for (int j = 0; j < kLpVec; ++j) if (j < n) bv[j] = __ldg(brow + j);
    }
  }
  unsigned short cv[kLpVec];
  if (use_cnt) {
    const unsigned short* crow = counts + b * vocab + i0;
    if (n == kLpVec && (reinterpret_cast<uintptr_t>(crow) & 15) == 0) {
      *reinterpret_cast<uint4*>(cv) = *reinterpret_cast<const uint4*>(crow);
    } else {
#pragma unroll
      for (int j = 0; j < kLpVec; ++j) if (j < n) cv[j] = crow[j];
    }
  }
  // i0 is a multiple of 8: the slice's seen bits lie in one word
  const unsigned sbits = use_rep ? (seen[b * words + (i0 >> 5)] >> (i0 & 31)) : 0u;
  bool any = false;
#pragma unroll
  for (int j = 0; j < kLpVec; ++j) {
    if (j >= n) continue;
    float v = DT<T>::to_f(x[j]);
    bool touched = false;
    if (use_bias) {
      const float bj = bv[j];
      if (bj == -INFINITY) { v = -INFINITY; touched = true; }
      else if (bj != 0.f) { v = v + bj; touched = true; }
    }
    if (use_min) {
      const long long t = i0 + j;
      for (int k = 0; k < n_stop_s; ++k)
        if (stop_s[k] == t) { v = -INFINITY; touched = true; }
    }
    if (use_rep && ((sbits >> j) & 1u)) { v = v > 0.f ? v / p : mul_rn(v, p); touched = true; }
    if (use_cnt && cv[j] != 0) {
      v = (v - mul_rn(freq, (float)cv[j])) - pres;
      touched = true;
    }
    if (touched) { x[j] = DT<T>::from_f(v); any = true; }
  }
  if (!any) return;
  if (vec) {
    *reinterpret_cast<uint4*>(row) = *reinterpret_cast<const uint4*>(x);
  } else {
#pragma unroll
    for (int j = 0; j < kLpVec; ++j) if (j < n) row[j] = x[j];
  }
}

__global__ void logit_proc_update_kernel(const int* __restrict__ cur_ids, int batch, long long vocab, unsigned* __restrict__ seen,
                                         int words, unsigned short* __restrict__ counts, int* __restrict__ n_generated) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const int t = cur_ids[b];
  if (t < 0 || t >= vocab) return;
  if (counts != nullptr) counts[(long long)b * vocab + t] += 1;
  seen[(long long)b * words + (t >> 5)] |= 1u << (t & 31);  // one thread per row: no other writer of the word
  n_generated[b] += 1;
}
}  // namespace

extern "C" int cts_logit_proc_apply(cts_ctx* ctx, void* logits, long long vocab, long long ld, int batch, const float* rep,
                                    const float* presence, const float* frequency, const unsigned* seen, int words_per_row,
                                    const unsigned short* counts, const float* bias, int n_bias, const int* bias_row,
                                    const int* n_generated, const int* min_tokens, const int* stop_ids, int max_stop, int dtype,
                                    void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, batch >= 0 && batch <= 65535 && vocab > 0 && vocab < (1LL << 31) && ld >= vocab, "shape");
  CTS_CHECK_ARG(ctx, words_per_row >= (vocab + 31) / 32, "words_per_row must be >= ceil(vocab / 32)");
  CTS_CHECK_ARG(ctx, max_stop >= 0 && max_stop <= kLpMaxStop, "max_stop must be 0..64");
  CTS_CHECK_ARG(ctx, n_bias >= 0, "n_bias");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (batch == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, logits && rep && presence && frequency && seen && bias_row && n_generated && min_tokens, "null pointer");
  CTS_CHECK_ARG(ctx, (n_bias == 0 || bias) && (max_stop == 0 || stop_ids), "null bias / stop_ids");
  const dim3 grid((unsigned)((vocab + kLpSlice - 1) / kLpSlice), (unsigned)batch);
  if (dtype == CTS_BF16)
    CTS_CUDA(ctx, launch_pdl(logit_proc_apply_kernel<__nv_bfloat16>, grid, dim3(kLpThreads), 0, (cudaStream_t)stream, 1,
                             (__nv_bfloat16*)logits, vocab, ld, rep, presence, frequency, seen, words_per_row, counts, n_bias ? bias : nullptr,
                             n_bias, bias_row, n_generated, min_tokens, stop_ids, max_stop));
  else
    CTS_CUDA(ctx, launch_pdl(logit_proc_apply_kernel<__half>, grid, dim3(kLpThreads), 0, (cudaStream_t)stream, 1, (__half*)logits, vocab,
                             ld, rep, presence, frequency, seen, words_per_row, counts, n_bias ? bias : nullptr, n_bias, bias_row, n_generated,
                             min_tokens, stop_ids, max_stop));
  return CTS_OK;
}

extern "C" int cts_logit_proc_update(cts_ctx* ctx, const int* cur_ids, int batch, long long vocab, unsigned* seen, int words_per_row,
                                     unsigned short* counts, int* n_generated, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, batch >= 0 && batch <= 65535 && vocab > 0 && vocab < (1LL << 31), "batch / vocab");
  CTS_CHECK_ARG(ctx, words_per_row >= (vocab + 31) / 32, "words_per_row must be >= ceil(vocab / 32)");
  if (batch == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, cur_ids && seen && n_generated, "null pointer");
  CTS_CUDA(ctx, launch_pdl(logit_proc_update_kernel, dim3((unsigned)((batch + 127) / 128)), dim3(128), 0, (cudaStream_t)stream, 1, cur_ids,
                           batch, vocab, seen, words_per_row, counts, n_generated));
  return CTS_OK;
}
