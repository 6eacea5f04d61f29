// chatts_b200 -- tensor-parallel row-parallel tail as ONE kernel over NVLink peer memory:
//     h = resid + dtype( sum over ranks of partial_r ) ;  norm_out = RMSNorm(h) * w
// replaces "RowParallelLinear -> NCCL all-reduce -> residual add -> RMSNorm" (vllm qwen2.py:100-116,168-174,
// 299-311; SURVEY.md §2.2 K9/K11, §5) for the decode-sized messages (b*5120 fp32 = 20..640 KiB) where the
// collective is latency-bound: every rank's o_proj / down_proj GEMM leaves its fp32 partial in a symmetric
// (cudaIpc-mapped) buffer; this kernel (1) reduces the rank's split-K partials and PUSHES its chunk into slot [rank] of
// every peer's buffer (posted NVLink writes), (2) signals "my chunk has landed" into every peer's flag array with a
// system-scope release store and waits with acquire loads until all peers have signalled this epoch, (3) sums the
// local slots in rank order -- the same order on every rank, so all ranks hold bit-identical h without a broadcast --
// fused with the residual add and the next RMSNorm.  No NCCL call, no extra launch, no copy.  (allreduce_ll.cu is the
// two-shot variant with the flags inside the data.)  The two partial buffers (o_proj / down_proj) alternate, so
// the barrier of call n+1 is what licenses overwriting the buffer of call n.
#include <cooperative_groups.h>

#include "common.cuh"

namespace {

__device__ __forceinline__ void st_release_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

constexpr int kThreads = 128;
constexpr int kMaxVec = 4;       // h / C <= 8 * 4 * 128 columns per CTA
constexpr int kMaxRanks = 16;
constexpr int kMaxCluster = 8;   // CTAs (one cluster) per token

// grid (C, T), cluster (C,1,1): CTA (c, t) owns columns [c*h/C, (c+1)*h/C) of token t.
template <typename T>
__global__ void __launch_bounds__(kThreads)
peer_allreduce_residual_rmsnorm_kernel(const float* __restrict__ local_part, int S, long long t_total,
                                       float* const* __restrict__ peer_rows, int* const* __restrict__ peer_flags,
                                       int* __restrict__ state, int rank, int world, int max_tokens,
                                       const T* __restrict__ resid_in, T* __restrict__ resid_out, const T* __restrict__ norm_w,
                                       float eps, T* __restrict__ norm_out, int h) {
  pdl_trigger();
  pdl_wait();
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int C = (int)cluster.num_blocks();
  const int crank = (int)cluster.block_rank();
  const long long t = blockIdx.y;
  const int hc = h / C, col0 = crank * hc, nvec = hc / 8;
  __shared__ float* src[kMaxRanks];
  __shared__ float red[kThreads / 32];
  __shared__ float ss_cta;
  const int epoch = state[0] + 1;      // state[0] is only advanced by the last CTA of this kernel to finish
  if (threadIdx.x < world) src[threadIdx.x] = peer_rows[threadIdx.x];
  __syncthreads();
  // ---- phase A: reduce this rank's split-K partials of my column chunk (fixed split order) and PUSH the result into
  // slot [rank] of EVERY rank's row buffer (posted NVLink writes; the release store below orders them before the flag)
  {
    const long long stride = t_total * (long long)h;
    const long long slot_off = ((long long)rank * max_tokens + t) * h + col0;
#pragma unroll
    for (int it = 0; it < kMaxVec; ++it) {
      const int v = it * kThreads + threadIdx.x;
      if (v < nvec) {
        const float* p = local_part + t * h + col0 + (long long)v * 8;
        float4 lo = *reinterpret_cast<const float4*>(p), hi = *reinterpret_cast<const float4*>(p + 4);
        for (int s = 1; s < S; ++s) {
          const float4 l2 = *reinterpret_cast<const float4*>(p + s * stride), h2 = *reinterpret_cast<const float4*>(p + s * stride + 4);
          lo.x += l2.x; lo.y += l2.y; lo.z += l2.z; lo.w += l2.w; hi.x += h2.x; hi.y += h2.y; hi.z += h2.z; hi.w += h2.w;
        }
        for (int r = 0; r < world; ++r) {
          float* dst = src[r] + slot_off + (long long)v * 8;
          *reinterpret_cast<float4*>(dst) = lo;
          *reinterpret_cast<float4*>(dst + 4) = hi;
        }
      }
    }
  }
  __syncthreads();
  // ---- barrier for (token t, chunk crank): tell every peer my chunk is ready, wait for theirs
  const long long slot = (t * kMaxCluster + crank);
  if (threadIdx.x < world) {
    __threadfence_system();      // cumulative: the CTA's pushes (ordered before this thread by the barrier) precede the flag
    st_release_sys(peer_flags[threadIdx.x] + (long long)rank * max_tokens * kMaxCluster + slot, epoch);
    const int* mine = peer_flags[rank] + (long long)threadIdx.x * max_tokens * kMaxCluster + slot;
    unsigned spins = 0;
    while (ld_acquire_sys(mine) < epoch) {
      if (++spins > (1u << 26)) {
        printf("chatts_b200: peer all-reduce timed out waiting for rank %d (epoch %d)\n", threadIdx.x, epoch);
        __trap();
      }
    }
  }
  __syncthreads();
  // ---- phase B: every rank's chunk is now in MY buffer (slot r = rank r): sum in rank order (bit-identical on all ranks)
  float vals[kMaxVec][8];
  float ss = 0.f;
#pragma unroll
  for (int it = 0; it < kMaxVec; ++it) {
    const int v = it * kThreads + threadIdx.x;
    if (v < nvec) {
      float4 lo[kMaxRanks / 2], hi[kMaxRanks / 2];
      float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int r0 = 0; r0 < world; r0 += kMaxRanks / 2) {
#pragma unroll
        for (int j = 0; j < kMaxRanks / 2; ++j) {
          if (r0 + j < world) {
            const float* p = src[rank] + ((long long)(r0 + j) * max_tokens + t) * h + col0 + (long long)v * 8;   // local slot of rank r
            lo[j] = __ldcv(reinterpret_cast<const float4*>(p));
            hi[j] = __ldcv(reinterpret_cast<const float4*>(p + 4));
          }
        }
#pragma unroll
        for (int j = 0; j < kMaxRanks / 2; ++j) {
          if (r0 + j < world) {
            a[0] += lo[j].x; a[1] += lo[j].y; a[2] += lo[j].z; a[3] += lo[j].w;
            a[4] += hi[j].x; a[5] += hi[j].y; a[6] += hi[j].z; a[7] += hi[j].w;
          }
        }
      }
      const long long off = t * h + col0 + (long long)v * 8;
      float rr[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(resid_in + off), rr);
#pragma unroll
      for (int j = 0; j < 8; ++j) rr[j] = rnd<T>(rr[j] + rnd<T>(a[j]));
      *reinterpret_cast<uint4*>(resid_out + off) = pack8<T>(rr);
#pragma unroll
      for (int j = 0; j < 8; ++j) { vals[it][j] = rr[j]; ss += rr[j] * rr[j]; }
    }
  }
  // ---- RMSNorm statistic across the cluster (DSMEM)
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) v += red[w];
    ss_cta = v;
  }
  cluster.sync();
  float tot = 0.f;
  for (int r = 0; r < C; ++r) tot += *cluster.map_shared_rank(&ss_cta, r);
  cluster.sync();
  if (norm_out != nullptr) {
    const float inv = 1.0f / sqrtf(tot / (float)h + eps);
#pragma unroll
    for (int it = 0; it < kMaxVec; ++it) {
      const int v = it * kThreads + threadIdx.x;
      if (v < nvec) {
        float w[8], o[8];
        unpack8<T>(*reinterpret_cast<const uint4*>(norm_w + col0 + (long long)v * 8), w);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = w[j] * rnd<T>(vals[it][j] * inv);
        *reinterpret_cast<uint4*>(norm_out + t * h + col0 + (long long)v * 8) = pack8<T>(o);
      }
    }
  }
  // last CTA of the grid to finish publishes the new epoch for the next call
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int done = atomicAdd(&state[1], 1) + 1;
    if (done == (int)(gridDim.x * gridDim.y)) {
      state[1] = 0;
      state[0] = epoch;
      __threadfence();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Vocab-parallel greedy sampling without a collective library call: every rank takes the argmax of ITS logits
// shard, PUSHES (value, global index) into every peer's candidate table over NVLink (release store), waits until
// all peers' candidates for this sequence have landed (acquire loads on its own flags), picks the global winner
// (largest value, lowest index on ties -- identical on every rank) and advances the device-side decode state.
// Replaces "ParallelLMHead logits all-gather + sampler" (chatts_vllm.py:607-610) for greedy decoding, which lets a
// tensor-parallel decode step be captured in one CUDA graph.  One CTA per sequence.
template <typename T>
__global__ void __launch_bounds__(1024)
peer_greedy_advance_kernel(const T* __restrict__ logits, long long vshard, int rank, int world, float2* const* __restrict__ peer_cand,
                           int* const* __restrict__ peer_flags, int* __restrict__ state, int max_b, int* __restrict__ out_tokens,
                           int out_ld, int* __restrict__ step_ptr, int* __restrict__ cur_ids, int* __restrict__ positions,
                           int* __restrict__ seq_lens, int* __restrict__ slot_map, const int* __restrict__ page_table, int max_pages,
                           int page_size) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x;
  const int epoch = state[0] + 1;
  const T* row = logits + (long long)b * vshard;
  float best = -INFINITY;
  long long best_i = vshard;
  for (long long i = threadIdx.x; i < vshard; i += blockDim.x) {
    const float f = DT<T>::to_f(row[i]);
    if (f > best) { best = f; best_i = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; }
  }
  __shared__ float sb[32];
  __shared__ long long si[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { sb[warp] = best; si[warp] = best_i; }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    best = lane < nw ? sb[lane] : -INFINITY;
    best_i = lane < nw ? si[lane] : vshard;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const long long oi = __shfl_xor_sync(0xffffffffu, best_i, o);
      if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; }
    }
    // push my candidate to every rank (slot [rank][b]) and then the flag
    const float gidx = __int_as_float((int)(best_i + (long long)rank * vshard));
    if (lane < world) {
      float2* dst = peer_cand[lane] + (long long)rank * max_b + b;
      asm volatile("st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(best), "f"(gidx) : "memory");
      st_release_sys(peer_flags[lane] + rank * max_b + b, epoch);
    }
    // wait for every rank's candidate of this sequence
    if (lane < world) {
      const int* mine = peer_flags[rank] + lane * max_b + b;
      unsigned spins = 0;
      while (ld_acquire_sys(mine) < epoch) {
        if (++spins > (1u << 26)) { printf("chatts_b200: peer argmax timed out (rank %d waits for %d)\n", rank, lane); __trap(); }
      }
    }
    __syncwarp();
    float v = -INFINITY;
    int idx = 0x7fffffff;
    if (lane < world) {
      const float2* src = peer_cand[rank] + (long long)lane * max_b + b;
      float a, c;
      asm volatile("ld.relaxed.sys.global.v2.f32 {%0, %1}, [%2];" : "=f"(a), "=f"(c) : "l"(src) : "memory");
      v = a;
      idx = __float_as_int(c);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
      if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
    }
    if (lane == 0) {
      const int tok = idx == 0x7fffffff ? 0 : idx;
      const int step = step_ptr[0];
      out_tokens[(long long)b * out_ld + step] = tok;
      cur_ids[b] = tok;
      const int np = positions[b] + 1;
      positions[b] = np;
      seq_lens[b] = seq_lens[b] + 1;
      const int pg = np / page_size;
      slot_map[b] = pg < max_pages ? page_table[(long long)b * max_pages + pg] * page_size + np % page_size : -1;
      __threadfence();
      const int done = atomicAdd(&state[1], 1) + 1;
      if (done == (int)gridDim.x) {
        state[1] = 0;
        state[0] = epoch;
        step_ptr[0] = step + 1;
      }
    }
  }
}

}  // namespace

extern "C" int cts_ipc_alloc(cts_ctx* ctx, long long bytes, void** dptr, unsigned char* handle64) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, bytes > 0 && dptr && handle64, "args");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  CTS_CUDA(ctx, cudaMalloc(dptr, (size_t)bytes));
  CTS_CUDA(ctx, cudaMemset(*dptr, 0, (size_t)bytes));
  cudaIpcMemHandle_t hnd;
  CTS_CUDA(ctx, cudaIpcGetMemHandle(&hnd, *dptr));
  memcpy(handle64, &hnd, 64);
  return CTS_OK;
}

extern "C" int cts_ipc_open(cts_ctx* ctx, const unsigned char* handle64, void** dptr) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, handle64 && dptr, "args");
  cudaIpcMemHandle_t hnd;
  memcpy(&hnd, handle64, 64);
  CTS_CUDA(ctx, cudaIpcOpenMemHandle(dptr, hnd, cudaIpcMemLazyEnablePeerAccess));
  return CTS_OK;
}

extern "C" int cts_ipc_close(cts_ctx* ctx, void* dptr) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CUDA(ctx, cudaIpcCloseMemHandle(dptr));
  return CTS_OK;
}

extern "C" int cts_ipc_free(cts_ctx* ctx, void* dptr) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CUDA(ctx, cudaFree(dptr));
  return CTS_OK;
}

extern "C" int cts_peer_allreduce_residual_rmsnorm(cts_ctx* ctx, const float* local_partial, int split_k, const void* peer_rows,
                                                   const void* peer_flags, int* state, int rank, int world, int max_tokens,
                                                   const void* resid_in, void* resid_out, const void* norm_w, float eps,
                                                   void* norm_out, long long t, long long h, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, local_partial && split_k >= 1 && peer_rows && peer_flags && state && resid_in && resid_out, "null pointer");
  CTS_CHECK_ARG(ctx, world >= 1 && world <= kMaxRanks && rank >= 0 && rank < world, "rank / world");
  CTS_CHECK_ARG(ctx, (norm_w == nullptr) == (norm_out == nullptr), "norm_w / norm_out mismatch");
  CTS_CHECK_ARG(ctx, h > 0 && h % 8 == 0, "h must be a multiple of 8");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, t > 0 && t <= max_tokens && t <= 65535, "t must be in 1..max_tokens");
  unsigned C = 1;
  for (unsigned c : {8u, 4u, 2u}) {
    if (h % (8 * c) == 0 && h / (8 * c) >= 32) { C = c; break; }
  }
  CTS_CHECK_ARG(ctx, h / C <= 8LL * kMaxVec * kThreads, "h too large");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == CTS_BF16)
    CTS_CUDA(ctx, launch_pdl(peer_allreduce_residual_rmsnorm_kernel<__nv_bfloat16>, dim3(C, (unsigned)t), dim3(kThreads), 0, st, C,
                             local_partial, split_k, t, (float* const*)peer_rows, (int* const*)peer_flags, state, rank, world,
                             max_tokens, (const __nv_bfloat16*)resid_in, (__nv_bfloat16*)resid_out, (const __nv_bfloat16*)norm_w, eps,
                             (__nv_bfloat16*)norm_out, (int)h));
  else
    CTS_CUDA(ctx, launch_pdl(peer_allreduce_residual_rmsnorm_kernel<__half>, dim3(C, (unsigned)t), dim3(kThreads), 0, st, C,
                             local_partial, split_k, t, (float* const*)peer_rows, (int* const*)peer_flags, state, rank, world,
                             max_tokens, (const __half*)resid_in, (__half*)resid_out, (const __half*)norm_w, eps, (__half*)norm_out,
                             (int)h));
  return CTS_OK;
}

extern "C" int cts_peer_greedy_advance(cts_ctx* ctx, const void* logits, long long vocab_shard, int batch, int rank, int world,
                                       const void* peer_cand, const void* peer_flags, int* state, int max_batch, int* out_tokens,
                                       int out_ld, int* step_ptr, int* cur_ids, int* positions, int* seq_lens, int* slot_map,
                                       const int* page_table, int max_pages, int page_size, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, logits && peer_cand && peer_flags && state && out_tokens && step_ptr && cur_ids && positions && seq_lens &&
                         slot_map && page_table, "null pointer");
  CTS_CHECK_ARG(ctx, world >= 1 && world <= 32 && rank >= 0 && rank < world, "rank / world");
  CTS_CHECK_ARG(ctx, batch >= 0 && batch <= max_batch && vocab_shard > 0 && vocab_shard * world < 2147483647LL, "sizes");
  CTS_CHECK_ARG(ctx, page_size > 0 && max_pages > 0, "paging");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (batch == 0) return CTS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == CTS_BF16)
    CTS_CUDA(ctx, launch_pdl(peer_greedy_advance_kernel<__nv_bfloat16>, dim3(batch), dim3(1024), 0, st, 1, (const __nv_bfloat16*)logits,
                             vocab_shard, rank, world, (float2* const*)peer_cand, (int* const*)peer_flags, state, max_batch, out_tokens,
                             out_ld, step_ptr, cur_ids, positions, seq_lens, slot_map, page_table, max_pages, page_size));
  else
    CTS_CUDA(ctx, launch_pdl(peer_greedy_advance_kernel<__half>, dim3(batch), dim3(1024), 0, st, 1, (const __half*)logits, vocab_shard,
                             rank, world, (float2* const*)peer_cand, (int* const*)peer_flags, state, max_batch, out_tokens, out_ld,
                             step_ptr, cur_ids, positions, seq_lens, slot_map, page_table, max_pages, page_size));
  return CTS_OK;
}
