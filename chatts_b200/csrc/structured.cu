// chatts_b200 -- structured outputs: a byte automaton (DFA) over the token vocabulary, kept on the device, constrains decoding
// without a host round trip per step (chatts_b200/structured.py compiles a choice list or a regex to the DFA).
//   cts_struct_mask_build  once per (automaton, tokenizer, stop ids): allowed bits [S, ceil(V / 32)] -- token t is allowed in state s
//                          iff walking its bytes from s stays defined; a stop id iff s is accepting
//   cts_struct_mask_apply  every step, before the advance: logits[b, i] = -inf where bit i of allowed[state[b]] is clear
//   cts_struct_advance     every step, after the advance: state[b] = the state reached by walking the bytes of cur_ids[b]
// A row whose state is negative is unconstrained: both per-step kernels leave it alone.
#include "common.cuh"

namespace {

constexpr int kMaxStop = 64;

// walks the bytes [b0, b1) of one token from state s; -1 once a byte has no transition
__device__ __forceinline__ int walk(const int* __restrict__ trans, int s, const unsigned char* __restrict__ bytes, long long b0,
                                    long long b1) {
  for (long long i = b0; i < b1 && s >= 0; ++i) s = __ldg(&trans[(long long)s * 256 + bytes[i]]);
  return s;
}

// one thread per (state, 32-token word): 32 walks -> one word of the mask, written once (no atomics, same bits every launch)
__global__ void struct_mask_build_kernel(const int* __restrict__ trans, const unsigned char* __restrict__ accept, int num_states,
                                         const long long* __restrict__ offsets, const unsigned char* __restrict__ bytes, long long vocab,
                                         const int* __restrict__ stop_ids, int n_stop, unsigned* __restrict__ allowed, int words) {
  pdl_trigger();
  pdl_wait();
  __shared__ int stop_s[kMaxStop];
  for (int i = threadIdx.x; i < n_stop; i += blockDim.x) stop_s[i] = stop_ids[i];
  __syncthreads();
  const int s = blockIdx.y;
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= words || s >= num_states) return;
  const bool acc = accept[s] != 0;
  unsigned bits = 0;
  const long long t0 = (long long)w * 32;
  for (int j = 0; j < 32; ++j) {
    const long long t = t0 + j;
    if (t >= vocab) break;
    const long long b0 = offsets[t], b1 = offsets[t + 1];
    if (b1 > b0 && walk(trans, s, bytes, b0, b1) >= 0) bits |= 1u << j;
  }
  for (int k = 0; k < n_stop; ++k) {                         // a stop id ends the output: allowed exactly in accepting states
    const long long d = (long long)stop_s[k] - t0;
    if (d >= 0 && d < 32) bits = acc ? (bits | (1u << d)) : (bits & ~(1u << d));
  }
  allowed[(long long)s * words + w] = bits;
}

// one thread per logit; a clear bit writes -inf, a set bit (and every row with state < 0) is not touched
template <typename T>
__global__ void struct_mask_apply_kernel(T* __restrict__ logits, long long vocab, long long ld, const int* __restrict__ state,
                                         const unsigned* __restrict__ allowed, int words) {
  pdl_trigger();
  pdl_wait();
  const long long b = blockIdx.y;
  const int s = state[b];
  if (s < 0) return;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= vocab) return;
  const unsigned word = __ldg(&allowed[(long long)s * words + (i >> 5)]);
  if (!((word >> (i & 31)) & 1u)) logits[b * ld + i] = DT<T>::from_f(-INFINITY);
}

// one thread per row: the new token's walk is a handful of bytes
__global__ void struct_advance_kernel(const int* __restrict__ cur_ids, int batch, int* __restrict__ state, const int* __restrict__ trans,
                                      const long long* __restrict__ offsets, const unsigned char* __restrict__ bytes, long long vocab,
                                      const int* __restrict__ stop_ids, int n_stop) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const int s = state[b];
  if (s < 0) return;
  const int t = cur_ids[b];
  if (t < 0 || t >= vocab) return;
  for (int k = 0; k < n_stop; ++k)
    if (stop_ids[k] == t) return;                            // a stop id leaves the state as it is
  const int n = walk(trans, s, bytes, offsets[t], offsets[t + 1]);
  if (n >= 0) state[b] = n;                                  // a token the mask refused (possible only if no allowed logit was finite)
}                                                            // leaves the state as it is
}  // namespace

extern "C" int cts_struct_mask_build(cts_ctx* ctx, const int* trans, const unsigned char* accept, int num_states, const long long* offsets,
                                     const unsigned char* bytes, long long vocab, const int* stop_ids, int n_stop, unsigned* allowed,
                                     int words_per_state, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, num_states > 0 && num_states <= 65535 && vocab > 0 && vocab < (1LL << 31), "num_states / vocab");
  CTS_CHECK_ARG(ctx, words_per_state == (vocab + 31) / 32, "words_per_state must be ceil(vocab / 32)");
  CTS_CHECK_ARG(ctx, n_stop >= 0 && n_stop <= kMaxStop, "n_stop must be 0..64");
  CTS_CHECK_ARG(ctx, trans && accept && offsets && bytes && allowed && (n_stop == 0 || stop_ids), "null pointer");
  dim3 grid((unsigned)((words_per_state + 127) / 128), (unsigned)num_states);
  CTS_CUDA(ctx, launch_pdl(struct_mask_build_kernel, grid, dim3(128), 0, (cudaStream_t)stream, 1, trans, accept, num_states, offsets, bytes,
                           vocab, stop_ids, n_stop, allowed, words_per_state));
  return CTS_OK;
}

extern "C" int cts_struct_mask_apply(cts_ctx* ctx, void* logits, long long vocab, long long ld, int batch, const int* state,
                                     const unsigned* allowed, int words_per_state, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, batch >= 0 && batch <= 65535 && vocab > 0 && ld >= vocab && words_per_state >= (vocab + 31) / 32, "shape");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (batch == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, logits && state && allowed, "null pointer");
  dim3 grid((unsigned)((vocab + 255) / 256), (unsigned)batch);
  if (dtype == CTS_BF16)
    CTS_CUDA(ctx, launch_pdl(struct_mask_apply_kernel<__nv_bfloat16>, grid, dim3(256), 0, (cudaStream_t)stream, 1, (__nv_bfloat16*)logits,
                             vocab, ld, state, allowed, words_per_state));
  else
    CTS_CUDA(ctx, launch_pdl(struct_mask_apply_kernel<__half>, grid, dim3(256), 0, (cudaStream_t)stream, 1, (__half*)logits, vocab, ld,
                             state, allowed, words_per_state));
  return CTS_OK;
}

extern "C" int cts_struct_advance(cts_ctx* ctx, const int* cur_ids, int batch, int* state, const int* trans, const long long* offsets,
                                  const unsigned char* bytes, long long vocab, const int* stop_ids, int n_stop, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, batch >= 0 && vocab > 0 && vocab < (1LL << 31) && n_stop >= 0 && n_stop <= kMaxStop, "batch / vocab / n_stop");
  if (batch == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, cur_ids && state && trans && offsets && bytes && (n_stop == 0 || stop_ids), "null pointer");
  CTS_CUDA(ctx, launch_pdl(struct_advance_kernel, dim3((unsigned)((batch + 127) / 128)), dim3(128), 0, (cudaStream_t)stream, 1, cur_ids, batch,
                           state, trans, offsets, bytes, vocab, stop_ids, n_stop));
  return CTS_OK;
}
