// chatts_b200 -- the memory-bound glue of the decoder, each fused with the split-K reduction of the GEMM
// that precedes it so that no projection result makes an extra HBM round trip:
//   cts_reduce_bias_act          TS-MLP layer tail: sum partials + bias (+ exact-erf GELU), optional row scatter
//   cts_reduce_residual_rmsnorm  o_proj / down_proj tail: sum partials + residual add + next RMSNorm
//   cts_reduce_swiglu            gate_up tail (when gate_up ran split-K)
//   cts_qkv_rope_cache           QKV tail: sum partials + bias + RoPE + paged KV-cache write
//   cts_embed_gather             token embedding lookup (rows of <ts> patches are skipped: the encoder scatters them)
//   cts_greedy_advance           argmax + device-side decode bookkeeping (graph-replayable decode loop)
// Rounding points follow transformers' Qwen2 in the model dtype (modeling_qwen2.py line numbers in the header).
#include <cooperative_groups.h>

#include "common.cuh"
#include "trace.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void reduce_bias_act_kernel(const float* __restrict__ part, int S, long long t_total, long long n,
                                       const T* __restrict__ bias, int act, T* __restrict__ out, long long out_ld,
                                       const int* __restrict__ row_map) {
  pdl_trigger();
  pdl_wait();
  const long long t = blockIdx.y;
  long long row = t;
  if (row_map) {
    row = row_map[t];
    if (row < 0) return;
  }
  const long long col4 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (col4 >= n) return;
  const long long stride = t_total * n;
  const float* p = part + t * n + col4;
  if (col4 + 3 < n && (n & 3) == 0) {
    float4 a = *reinterpret_cast<const float4*>(p);
    for (int s = 1; s < S; ++s) {
      float4 b = *reinterpret_cast<const float4*>(p + s * stride);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    float v[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float r = v[j] + (bias ? DT<T>::to_f(bias[col4 + j]) : 0.f);
      if (act == CTS_EPI_GELU) r = gelu_erf(rnd<T>(r));
      out[row * out_ld + col4 + j] = DT<T>::from_f(r);
    }
  } else {
    for (int j = 0; j < 4 && col4 + j < n; ++j) {
      float a = p[j];
      for (int s = 1; s < S; ++s) a += p[j + s * stride];
      float r = a + (bias ? DT<T>::to_f(bias[col4 + j]) : 0.f);
      if (act == CTS_EPI_GELU) r = gelu_erf(rnd<T>(r));
      out[row * out_ld + col4 + j] = DT<T>::from_f(r);
    }
  }
}


// Split-K partials are read S at a time with ALL loads of a batch issued before the first add: a `for (s < S)` loop with a run-time
// bound issues one load, waits a full L2 round trip (~0.7 us) for the add, and only then issues the next -- 7 partials cost ~5 us of
// pure latency in a kernel that moves a few megabytes (measured with csrc/trace.cuh: 5.5 us per RMSNorm launch).  The additions still
// run in split order (s = 0, 1, ..., S-1), so results are bit-identical to the sequential loop.
constexpr int kPartBatch = 8;
__device__ __forceinline__ void sum_partials8(const float* __restrict__ p, long long stride, int S, float* a) {
  float4 lo[kPartBatch], hi[kPartBatch];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = 0.f;
  for (int s0 = 0; s0 < S; s0 += kPartBatch) {
#pragma unroll
    for (int u = 0; u < kPartBatch; ++u)
      if (s0 + u < S) {
        lo[u] = *reinterpret_cast<const float4*>(p + (long long)(s0 + u) * stride);
        hi[u] = *reinterpret_cast<const float4*>(p + (long long)(s0 + u) * stride + 4);
      }
#pragma unroll
    for (int u = 0; u < kPartBatch; ++u)
      if (s0 + u < S) {
        if (s0 + u == 0) {            // the first partial initialises the sum (x + 0.f would turn -0.f into +0.f)
          a[0] = lo[u].x; a[1] = lo[u].y; a[2] = lo[u].z; a[3] = lo[u].w; a[4] = hi[u].x; a[5] = hi[u].y; a[6] = hi[u].z; a[7] = hi[u].w;
        } else {
          a[0] += lo[u].x; a[1] += lo[u].y; a[2] += lo[u].z; a[3] += lo[u].w; a[4] += hi[u].x; a[5] += hi[u].y; a[6] += hi[u].z; a[7] += hi[u].w;
        }
      }
  }
}
__device__ __forceinline__ void sum_partials2(const float* __restrict__ p0, const float* __restrict__ p1, long long stride, int S,
                                              float& a0, float& a1) {
  float v0[kPartBatch], v1[kPartBatch];
  a0 = a1 = 0.f;
  for (int s0 = 0; s0 < S; s0 += kPartBatch) {
#pragma unroll
    for (int u = 0; u < kPartBatch; ++u)
      if (s0 + u < S) {
        v0[u] = p0[(long long)(s0 + u) * stride];
        v1[u] = p1[(long long)(s0 + u) * stride];
      }
#pragma unroll
    for (int u = 0; u < kPartBatch; ++u)
      if (s0 + u < S) {
        a0 = (s0 + u == 0) ? v0[u] : a0 + v0[u];
        a1 = (s0 + u == 0) ? v1[u] : a1 + v1[u];
      }
  }
}

// ------------------------------------------------------------------------------------------------
// one CTA per token; H elements kept in registers between the two passes (H <= 8 * 8 * blockDim)
constexpr int kNormThreads = 256;
constexpr int kNormMaxVec = 8;   // up to 8 x 8 elements per thread -> H <= 16384

template <typename T, int NV>
__global__ void __launch_bounds__(kNormThreads)
reduce_residual_rmsnorm_kernel(const float* __restrict__ part, int S, const T* __restrict__ resid_in,
                               T* __restrict__ resid_out, const T* __restrict__ norm_w, float eps,
                               T* __restrict__ norm_out, long long t_total, int h) {
  pdl_trigger();
  pdl_wait();
  const long long t = blockIdx.x;
  const int nvec = h / 8;
  float vals[NV][8];
  float ss = 0.f;
  const long long stride = t_total * (long long)h;
#pragma unroll
  for (int it = 0; it < NV; ++it) {
    const int v = it * kNormThreads + threadIdx.x;
    if (v < nvec) {
      float r[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(resid_in + t * h + (long long)v * 8), r);
      if (S > 0) {
        float a[8];
        sum_partials8(part + t * h + (long long)v * 8, stride, S, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = rnd<T>(r[j] + rnd<T>(a[j]));   // residual + dtype(proj)  (:302,:308)
        if (resid_out) *reinterpret_cast<uint4*>(resid_out + t * h + (long long)v * 8) = pack8<T>(r);
      } else if (resid_out && resid_out != resid_in) {
        *reinterpret_cast<uint4*>(resid_out + t * h + (long long)v * 8) = pack8<T>(r);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { vals[it][j] = r[j]; ss += r[j] * r[j]; }
    }
  }
  if (norm_out == nullptr) return;
  __shared__ float red[kNormThreads / 32];
  __shared__ float inv_s;
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < kNormThreads / 32 ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) inv_s = 1.0f / sqrtf(v / (float)h + eps);   // rsqrt(mean(x^2)+eps)  (:261-262)
  }
  __syncthreads();
  const float inv = inv_s;
#pragma unroll
  for (int it = 0; it < NV; ++it) {
    const int v = it * kNormThreads + threadIdx.x;
    if (v < nvec) {
      float w[8], o[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(norm_w + (long long)v * 8), w);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = w[j] * rnd<T>(vals[it][j] * inv);   // weight * x.to(dtype)  (:263)
      *reinterpret_cast<uint4*>(norm_out + t * h + (long long)v * 8) = pack8<T>(o);
    }
  }
}

// Plain RMSNorm of many rows (prefill-sized T, no partials to reduce: the GEMM before it applied the residual in its epilogue): ONE WARP
// per row, the row held in registers as packed 16-byte vectors between the two passes, warp shuffles only -- no block barrier.  The
// one-CTA-per-token kernel above spends two __syncthreads and a shared-memory round trip per 10 KB row.
constexpr int kRowWarps = 8;

template <typename T, int NVW>
__global__ void __launch_bounds__(kRowWarps * 32)
rmsnorm_rows_kernel(const T* __restrict__ x, const T* __restrict__ norm_w, float eps, T* __restrict__ norm_out, long long t_total, int h) {
  pdl_trigger();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long t = (long long)blockIdx.x * kRowWarps + warp;
  if (t >= t_total) return;
  const int nvec = h / 8;
  uint4 row[NVW];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NVW; ++i) {
    const int v = i * 32 + lane;
    if (v < nvec) {
      row[i] = *reinterpret_cast<const uint4*>(x + t * h + (long long)v * 8);
      float r[8];
      unpack8<T>(row[i], r);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += r[j] * r[j];
    }
  }
  ss = warp_sum(ss);
  const float inv = 1.0f / sqrtf(ss / (float)h + eps);                     // rsqrt(mean(x^2)+eps)  (modeling_qwen2.py:261-262)
#pragma unroll
  for (int i = 0; i < NVW; ++i) {
    const int v = i * 32 + lane;
    if (v < nvec) {
      float r[8], w[8], o[8];
      unpack8<T>(row[i], r);
      unpack8<T>(*reinterpret_cast<const uint4*>(norm_w + (long long)v * 8), w);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = w[j] * rnd<T>(r[j] * inv);         // weight * x.to(dtype)  (:263)
      *reinterpret_cast<uint4*>(norm_out + t * h + (long long)v * 8) = pack8<T>(o);
    }
  }
}

// Cluster version: C CTAs (one thread-block cluster) share a token; each owns h/C columns, the sum of squares is
// exchanged through distributed shared memory.  At decode (T <= 32 tokens) this turns a 32-CTA kernel into a
// 256-CTA one, so the split-K partials are pulled from L2 by every SM instead of by 32 of them.
constexpr int kClThreads = 128;
constexpr int kClMaxVec = 4;     // h / C <= 8 * 4 * 128 = 4096 columns per CTA

template <typename T>
__global__ void __launch_bounds__(kClThreads)
reduce_residual_rmsnorm_cluster_kernel(const float* __restrict__ part, int S, const T* __restrict__ resid_in,
                                       T* __restrict__ resid_out, const T* __restrict__ norm_w, float eps,
                                       T* __restrict__ norm_out, long long t_total, int h) {
  pdl_trigger();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_NORM, 0);
  pdl_wait();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_NORM, 1);
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int C = (int)cluster.num_blocks();
  const int crank = (int)cluster.block_rank();
  const long long t = blockIdx.y;
  const int hc = h / C, col0 = crank * hc, nvec = hc / 8;
  float vals[kClMaxVec][8];
  float ss = 0.f;
  const long long stride = t_total * (long long)h;
#pragma unroll
  for (int it = 0; it < kClMaxVec; ++it) {
    const int v = it * kClThreads + threadIdx.x;
    if (v < nvec) {
      const long long off = t * h + col0 + (long long)v * 8;
      float r[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(resid_in + off), r);
      if (S > 0) {
        float a[8];
        sum_partials8(part + off, stride, S, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = rnd<T>(r[j] + rnd<T>(a[j]));
        if (resid_out) *reinterpret_cast<uint4*>(resid_out + off) = pack8<T>(r);
      } else if (resid_out && resid_out != resid_in) {
        *reinterpret_cast<uint4*>(resid_out + off) = pack8<T>(r);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { vals[it][j] = r[j]; ss += r[j] * r[j]; }
    }
  }
  __shared__ float red[kClThreads / 32];
  __shared__ float ss_cta;
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kClThreads / 32; ++w) v += red[w];
    ss_cta = v;
  }
  cluster.sync();
  float tot = 0.f;
  for (int r = 0; r < C; ++r) tot += *cluster.map_shared_rank(&ss_cta, r);     // fixed order: same value in all CTAs
  cluster.sync();                                                              // nobody exits while peers still read
  if (norm_out == nullptr) return;
  const float inv = 1.0f / sqrtf(tot / (float)h + eps);
#pragma unroll
  for (int it = 0; it < kClMaxVec; ++it) {
    const int v = it * kClThreads + threadIdx.x;
    if (v < nvec) {
      float w[8], o[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(norm_w + col0 + (long long)v * 8), w);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = w[j] * rnd<T>(vals[it][j] * inv);
      *reinterpret_cast<uint4*>(norm_out + t * h + col0 + (long long)v * 8) = pack8<T>(o);
    }
  }
}

// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void reduce_swiglu_kernel(const float* __restrict__ part, int S, long long t_total, long long inter,
                                     T* __restrict__ out, int interleaved) {
  pdl_trigger();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_SWIGLU, 0);
  pdl_wait();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_SWIGLU, 1);
  const long long t = blockIdx.y;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= inter) return;
  const long long n = 2 * inter;
  // column of gate_i / up_i in the projection output: stacked [gate | up], or interleaved per 128-wide tile
  // (64 gate columns then the 64 matching up columns -- the layout CTS_EPI_SWIGLU_IL uses)
  const long long gi = interleaved ? (i >> 6) * 128 + (i & 63) : i;
  const long long ui = interleaved ? gi + 64 : inter + i;
  float g = 0.f, u = 0.f;
  for (int s = 0; s < S; ++s) {
    const float* p = part + ((long long)s * t_total + t) * n;
    g += p[gi];
    u += p[ui];
  }
  const float r = rnd<T>(silu_f(rnd<T>(g))) * rnd<T>(u);
  out[t * inter + i] = DT<T>::from_f(r);
}

// Vector variant (inter % 8 == 0): a thread owns 8 consecutive outputs -- 8 gate and the 8 matching up columns are contiguous in both
// layouts (the interleaved one keeps 64-column runs) -- so a split costs four 16-byte loads, all splits' loads are in flight together
// (sum_partials8) and the store is one 16-byte vector.  448 CTAs of 128 threads at the 14B shape instead of 1728 of 256: the
// scalar kernel's CTAs filled every thread slot of the SMs and kept the next GEMM's CTAs (and their weight prefetch) out for ~10 us.
constexpr int kSwiThreads = 128;
template <typename T>
__global__ void __launch_bounds__(kSwiThreads)
reduce_swiglu_vec_kernel(const float* __restrict__ part, int S, long long t_total, long long inter, T* __restrict__ out,
                         int interleaved) {
  pdl_trigger();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_SWIGLU, 0);
  pdl_wait();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_SWIGLU, 1);
  const long long t = blockIdx.y;
  const long long i = ((long long)blockIdx.x * kSwiThreads + threadIdx.x) * 8;
  if (i >= inter) return;
  const long long n = 2 * inter;
  const long long gi = interleaved ? (i >> 6) * 128 + (i & 63) : i;
  const long long ui = interleaved ? gi + 64 : inter + i;
  const float* p = part + t * n;
  const long long stride = t_total * n;
  float g[8], u[8], r[8];
  sum_partials8(p + gi, stride, S, g);
  sum_partials8(p + ui, stride, S, u);
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = rnd<T>(silu_f(rnd<T>(g[j]))) * rnd<T>(u[j]);
  *reinterpret_cast<uint4*>(out + t * inter + i) = pack8<T>(r);
}

// ------------------------------------------------------------------------------------------------
constexpr int kRopeHeadsPerBlock = 4;
// Scalar variant, used for split-K partial input (decode): many small CTAs pull the fp32 partials from L2 in parallel.
// grid (ceil((nh + 2*nkv) / 4), T); block = 4 x head_dim/2 threads: thread i of a head owns dims i and i + d/2 (the
// rotate_half pair, modeling_qwen2.py:116-120,141-145).
template <typename T>
__global__ void qkv_rope_cache_scalar_kernel(const void* __restrict__ src, int src_is_partial, int S, const T* __restrict__ bias,
                                      const int* __restrict__ positions, const T* __restrict__ cos_tab,
                                      const T* __restrict__ sin_tab, const int* __restrict__ slot_map,
                                      T* __restrict__ q_out, T* __restrict__ k_cache, T* __restrict__ v_cache,
                                      T* __restrict__ k_out, T* __restrict__ v_out, long long t_total, int nh, int nkv,
                                      int d, int page_size, const T* __restrict__ q_norm_w, const T* __restrict__ k_norm_w,
                                      float norm_eps) {
  pdl_trigger();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_ROPE, 0);
  pdl_wait();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_ROPE, 1);
  const int half = d >> 1;
  const int hl = threadIdx.x / half;                    // head slot inside the block (kRopeHeadsPerBlock heads per CTA)
  const int head = blockIdx.x * kRopeHeadsPerBlock + hl;
  const long long t = blockIdx.y;
  const int i = threadIdx.x % half;
  const bool active = head < nh + 2 * nkv;
  const long long width = (long long)(nh + 2 * nkv) * d;
  const long long c0 = (long long)(active ? head : 0) * d + i, c1 = c0 + half;
  float x0, x1;
  if (src_is_partial) {
    const float* p = reinterpret_cast<const float*>(src) + t * width;
    const long long stride = t_total * width;
    sum_partials2(p + c0, p + c1, stride, S, x0, x1);
    if (bias) { x0 += DT<T>::to_f(bias[c0]); x1 += DT<T>::to_f(bias[c1]); }
    x0 = rnd<T>(x0); x1 = rnd<T>(x1);                 // nn.Linear output in the model dtype
  } else {
    const T* p = reinterpret_cast<const T*>(src) + t * width;
    x0 = DT<T>::to_f(p[c0]); x1 = DT<T>::to_f(p[c1]);
  }
  const bool is_q = head < nh;
  const bool is_k = !is_q && head < nh + nkv;
  if (q_norm_w != nullptr || k_norm_w != nullptr) {          // block-uniform (a CTA may hold q, k and v heads)
    // Qwen3 per-head RMSNorm of q / k over head_dim before RoPE (transformers qwen3/modeling_qwen3.py q_norm/k_norm;
    // vllm qwen3.py) -- same fp32-statistic / dtype rounding points as Qwen2RMSNorm
    __shared__ float red[32];
    float ss = active ? x0 * x0 + x1 * x1 : 0.f;
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    const int wph = half >= 32 ? half / 32 : 1;        // warps per head (head_dim/2 is a multiple of 32 here)
    for (int w = 0; w < wph; ++w) tot += red[hl * wph + w];
    const float inv = 1.0f / sqrtf(tot / (float)d + norm_eps);
    const T* nw = is_q ? q_norm_w : (is_k ? k_norm_w : nullptr);
    if (active && nw != nullptr) {
      x0 = rnd<T>(DT<T>::to_f(nw[i]) * rnd<T>(x0 * inv));
      x1 = rnd<T>(DT<T>::to_f(nw[i + half]) * rnd<T>(x1 * inv));
    }
  }
  if (!active) return;
  if (is_q || is_k) {
    const int pos = positions[t];
    // cos/sin are [max_pos, d/2]: emb = cat(freqs, freqs) (:110) makes both halves share the same angle
    const float c = DT<T>::to_f(cos_tab[(long long)pos * half + i]);
    const float s = DT<T>::to_f(sin_tab[(long long)pos * half + i]);
    // q_embed = (q * cos) + (rotate_half(q) * sin), every product and the sum rounded to dtype (:144)
    const float r0 = rnd<T>(rnd<T>(x0 * c) + rnd<T>(-x1 * s));
    const float r1 = rnd<T>(rnd<T>(x1 * c) + rnd<T>(x0 * s));
    x0 = r0; x1 = r1;
  }
  if (is_q) {
    T* o = q_out + t * (long long)nh * d + (long long)head * d;
    o[i] = DT<T>::from_f(x0);
    o[i + half] = DT<T>::from_f(x1);
    return;
  }
  const int kvh = is_k ? head - nh : head - nh - nkv;
  T* lin = is_k ? k_out : v_out;
  if (lin) {
    T* o = lin + t * (long long)nkv * d + (long long)kvh * d;
    o[i] = DT<T>::from_f(x0);
    o[i + half] = DT<T>::from_f(x1);
  }
  T* cache = is_k ? k_cache : v_cache;
  if (cache && slot_map) {
    const int slot = slot_map[t];
    if (slot >= 0) {
      const long long page = slot / page_size, off = slot % page_size;
      T* o = cache + ((page * nkv + kvh) * page_size + off) * d;     // [num_pages, nkv, page_size, d]
      o[i] = DT<T>::from_f(x0);
      o[i + half] = DT<T>::from_f(x1);
    }
  }
}

// grid (ceil(heads * (d/16) / 256), T); thread = (head, chunk of 8 rotary pairs): it owns dims [8j, 8j+8) and the
// matching dims of the upper half (the rotate_half pair, modeling_qwen2.py:116-120,141-145) -> every global access is a
// 16-byte vector.  The d/16 threads of a head sit in one warp, so the Qwen3 per-head RMSNorm is a sub-warp shuffle.
constexpr int kRopeThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kRopeThreads)
qkv_rope_cache_kernel(const void* __restrict__ src, int src_is_partial, int S, const T* __restrict__ bias,
                      const int* __restrict__ positions, const T* __restrict__ cos_tab, const T* __restrict__ sin_tab,
                      const int* __restrict__ slot_map, T* __restrict__ q_out, T* __restrict__ k_cache, T* __restrict__ v_cache,
                      T* __restrict__ k_out, T* __restrict__ v_out, long long t_total, int nh, int nkv, int d, int page_size,
                      const T* __restrict__ q_norm_w, const T* __restrict__ k_norm_w, float norm_eps) {
  pdl_trigger();
  pdl_wait();
  const int half = d >> 1;
  const int cph = half >> 3;                          // 8-pair chunks per head (8 for d = 128): power of two <= 32
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  const int head = item / cph, j = item % cph;
  const long long t = blockIdx.y;
  const int heads = nh + 2 * nkv;
  const bool active = head < heads;
  const long long width = (long long)heads * d;
  const long long c0 = (long long)(active ? head : 0) * d + j * 8, c1 = c0 + half;
  float x0[8], x1[8];
  if (src_is_partial) {
    const float* p = reinterpret_cast<const float*>(src) + t * width;
    const long long stride = t_total * width;
    float4 a = *reinterpret_cast<const float4*>(p + c0), b = *reinterpret_cast<const float4*>(p + c0 + 4);
    float4 c = *reinterpret_cast<const float4*>(p + c1), e = *reinterpret_cast<const float4*>(p + c1 + 4);
    for (int s = 1; s < S; ++s) {
      const float* ps = p + s * stride;
      const float4 a2 = *reinterpret_cast<const float4*>(ps + c0), b2 = *reinterpret_cast<const float4*>(ps + c0 + 4);
      const float4 c2 = *reinterpret_cast<const float4*>(ps + c1), e2 = *reinterpret_cast<const float4*>(ps + c1 + 4);
      a.x += a2.x; a.y += a2.y; a.z += a2.z; a.w += a2.w; b.x += b2.x; b.y += b2.y; b.z += b2.z; b.w += b2.w;
      c.x += c2.x; c.y += c2.y; c.z += c2.z; c.w += c2.w; e.x += e2.x; e.y += e2.y; e.z += e2.z; e.w += e2.w;
    }
    x0[0] = a.x; x0[1] = a.y; x0[2] = a.z; x0[3] = a.w; x0[4] = b.x; x0[5] = b.y; x0[6] = b.z; x0[7] = b.w;
    x1[0] = c.x; x1[1] = c.y; x1[2] = c.z; x1[3] = c.w; x1[4] = e.x; x1[5] = e.y; x1[6] = e.z; x1[7] = e.w;
    if (bias) {
      float b0[8], b1[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(bias + c0), b0);
      unpack8<T>(*reinterpret_cast<const uint4*>(bias + c1), b1);
#pragma unroll
      for (int e2 = 0; e2 < 8; ++e2) { x0[e2] += b0[e2]; x1[e2] += b1[e2]; }
    }
#pragma unroll
    for (int e2 = 0; e2 < 8; ++e2) { x0[e2] = rnd<T>(x0[e2]); x1[e2] = rnd<T>(x1[e2]); }   // nn.Linear output in the model dtype
  } else {
    const T* p = reinterpret_cast<const T*>(src) + t * width;
    unpack8<T>(*reinterpret_cast<const uint4*>(p + c0), x0);
    unpack8<T>(*reinterpret_cast<const uint4*>(p + c1), x1);
  }
  const bool is_q = head < nh;
  const bool is_k = !is_q && head < nh + nkv;
  if (q_norm_w != nullptr || k_norm_w != nullptr) {
    // Qwen3 per-head RMSNorm of q / k over head_dim before RoPE (transformers qwen3/modeling_qwen3.py q_norm/k_norm)
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) ss += x0[e] * x0[e] + x1[e] * x1[e];
    for (int o = cph >> 1; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);     // the cph lanes of this head
    const float inv = 1.0f / sqrtf(ss / (float)d + norm_eps);
    const T* nw = is_q ? q_norm_w : (is_k ? k_norm_w : nullptr);
    if (active && nw != nullptr) {
      float w0[8], w1[8];
      unpack8<T>(*reinterpret_cast<const uint4*>(nw + j * 8), w0);
      unpack8<T>(*reinterpret_cast<const uint4*>(nw + half + j * 8), w1);
#pragma unroll
      for (int e = 0; e < 8; ++e) { x0[e] = rnd<T>(w0[e] * rnd<T>(x0[e] * inv)); x1[e] = rnd<T>(w1[e] * rnd<T>(x1[e] * inv)); }
    }
  }
  if (!active) return;
  if (is_q || is_k) {
    const int pos = positions[t];
    // cos/sin are [max_pos, d/2]: emb = cat(freqs, freqs) (:110) makes both halves share the same angle
    float cs[8], sn[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(cos_tab + (long long)pos * half + j * 8), cs);
    unpack8<T>(*reinterpret_cast<const uint4*>(sin_tab + (long long)pos * half + j * 8), sn);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      // q_embed = (q * cos) + (rotate_half(q) * sin), every product and the sum rounded to dtype (:144)
      const float r0 = rnd<T>(rnd<T>(x0[e] * cs[e]) + rnd<T>(-x1[e] * sn[e]));
      const float r1 = rnd<T>(rnd<T>(x1[e] * cs[e]) + rnd<T>(x0[e] * sn[e]));
      x0[e] = r0; x1[e] = r1;
    }
  }
  const uint4 lo = pack8<T>(x0), hi = pack8<T>(x1);
  if (is_q) {
    T* o = q_out + t * (long long)nh * d + (long long)head * d + j * 8;
    *reinterpret_cast<uint4*>(o) = lo;
    *reinterpret_cast<uint4*>(o + half) = hi;
    return;
  }
  const int kvh = is_k ? head - nh : head - nh - nkv;
  T* lin = is_k ? k_out : v_out;
  if (lin) {
    T* o = lin + t * (long long)nkv * d + (long long)kvh * d + j * 8;
    *reinterpret_cast<uint4*>(o) = lo;
    *reinterpret_cast<uint4*>(o + half) = hi;
  }
  T* cache = is_k ? k_cache : v_cache;
  if (cache && slot_map) {
    const int slot = slot_map[t];
    if (slot >= 0) {
      const long long page = slot / page_size, off = slot % page_size;
      T* o = cache + ((page * nkv + kvh) * page_size + off) * d + j * 8;     // [num_pages, nkv, page_size, d]
      *reinterpret_cast<uint4*>(o) = lo;
      *reinterpret_cast<uint4*>(o + half) = hi;
    }
  }
}

// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void embed_gather_kernel(const T* __restrict__ table, const int* __restrict__ ids, T* __restrict__ out,
                                    long long h, long long vocab) {
  // STEP BARRIER: the first kernel of a decode step (and of a prefill) waits for everything before it -- the previous step's advance
  // kernel, host-side state updates -- BEFORE it lets its successors start.  Every later kernel of the step may therefore read the
  // step state (seq_lens, page table, positions, slots) and the KV rows of earlier positions ahead of its own dependency wait
  // (attn_decode_kernel prefetches its KV tiles that way).
  pdl_wait();
  pdl_trigger();
  const long long t = blockIdx.x;
  const int id = ids[t];
  if (id < 0 || id >= vocab) return;
  const uint4* src = reinterpret_cast<const uint4*>(table + (long long)id * h);
  uint4* dst = reinterpret_cast<uint4*>(out + t * h);
  for (int v = threadIdx.x; v < h / 8; v += blockDim.x) dst[v] = __ldg(src + v);
}

// ------------------------------------------------------------------------------------------------
// one CTA per sequence: argmax over the vocabulary (first maximum wins, like torch.argmax), then advance
template <typename T>
__global__ void __launch_bounds__(1024)
greedy_advance_kernel(const T* __restrict__ logits, long long vocab, int* __restrict__ out_tokens, int out_ld,
                      int* __restrict__ step_ptr, int* __restrict__ cur_ids, int* __restrict__ positions,
                      int* __restrict__ seq_lens, int* __restrict__ slot_map, const int* __restrict__ page_table,
                      int max_pages, int page_size) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x;
  const T* row = logits + (long long)b * vocab;
  float best = -INFINITY;
  long long best_i = vocab;
  if ((vocab & 7) == 0 && (reinterpret_cast<uintptr_t>(row) & 15) == 0) {
    const uint4* v = reinterpret_cast<const uint4*>(row);
    for (long long i = threadIdx.x; i < vocab / 8; i += blockDim.x) {
      float f[8];
      unpack8<T>(__ldg(v + i), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        // NaN never wins; ties keep the smaller index
        if (f[j] > best) { best = f[j]; best_i = i * 8 + j; }
      }
    }
  } else {
    for (long long i = threadIdx.x; i < vocab; i += blockDim.x) {
      const float f = DT<T>::to_f(row[i]);
      if (f > best) { best = f; best_i = i; }
    }
  }
  // warp then block argmax (value desc, index asc)
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
    best_i = lane < nw ? si[lane] : vocab;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const long long oi = __shfl_xor_sync(0xffffffffu, best_i, o);
      if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; }
    }
    if (lane == 0) {
      const int tok = best_i < vocab ? (int)best_i : 0;
      const int step = step_ptr ? step_ptr[0] : 0;      // step_ptr[0] only changes after every CTA has passed here
      if (out_tokens) out_tokens[(long long)b * out_ld + step] = tok;
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
        const int done = atomicAdd(&step_ptr[1], 1) + 1;     // step_ptr = {step, done-counter}
        if (done == (int)gridDim.x) {
          step_ptr[1] = 0;
          step_ptr[0] = step + 1;
        }
      }
    }
  }
}

}  // namespace

#define DISPATCH_T(dtype, ...)                      \
  if ((dtype) == CTS_BF16) {                        \
    using T = __nv_bfloat16;                        \
    __VA_ARGS__;                                    \
  } else {                                          \
    using T = __half;                               \
    __VA_ARGS__;                                    \
  }

extern "C" int cts_reduce_bias_act(cts_ctx* ctx, const float* partial, int split_k, long long t, long long n,
                                   const void* bias, int act, void* out, long long out_ld, const int* row_map, int dtype,
                                   void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, partial && out, "null partial / out");
  CTS_CHECK_ARG(ctx, split_k >= 1 && t >= 0 && n > 0, "sizes");
  CTS_CHECK_ARG(ctx, act == CTS_EPI_NONE || act == CTS_EPI_GELU, "act must be CTS_EPI_NONE or CTS_EPI_GELU");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, t <= 65535, "t > 65535 (use the fused GEMM epilogue for large t)");
  if (t == 0) return CTS_OK;
  const int threads = 128;
  dim3 grid((unsigned)cdiv_ll(cdiv_ll(n, 4), threads), (unsigned)t);
  DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(reduce_bias_act_kernel<T>, grid, dim3(threads), 0, (cudaStream_t)stream, 1, partial, split_k, t,
                                              n, (const T*)bias, act, (T*)out, out_ld, row_map)));
  return CTS_OK;
}

extern "C" int cts_reduce_residual_rmsnorm(cts_ctx* ctx, const float* partial, int split_k, const void* resid_in,
                                           void* resid_out, const void* norm_w, float eps, void* norm_out, long long t,
                                           long long h, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, resid_in != nullptr, "null resid_in");
  CTS_CHECK_ARG(ctx, (partial == nullptr) == (split_k == 0), "partial / split_k mismatch");
  CTS_CHECK_ARG(ctx, (norm_w == nullptr) == (norm_out == nullptr), "norm_w / norm_out mismatch");
  CTS_CHECK_ARG(ctx, h > 0 && h % 8 == 0 && h <= 8LL * kNormMaxVec * kNormThreads, "h must be a multiple of 8 and <= 16384");
  CTS_CHECK_ARG(ctx, split_k == 0 || resid_out != nullptr, "resid_out required when reducing partials");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (t == 0) return CTS_OK;
  // thread-block cluster over the hidden dimension when the row is wide enough (DSMEM exchange of the sum of squares)
  unsigned C = 1;
  for (unsigned c : {8u, 4u, 2u}) {
    if (c > (unsigned)ctx->norm_cluster) continue;
    if (h % (8 * c) == 0 && h / (8 * c) >= 32 && h / c <= 8LL * kClMaxVec * kClThreads) { C = c; break; }
  }
  if (C > 1 && t <= 256) {      // decode-sized T: spread each token over a cluster; big T already fills the GPU
    DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(reduce_residual_rmsnorm_cluster_kernel<T>, dim3(C, (unsigned)t), dim3(kClThreads), 0,
                                                (cudaStream_t)stream, C, partial, split_k, (const T*)resid_in, (T*)resid_out,
                                                (const T*)norm_w, eps, (T*)norm_out, t, (int)h)));
  } else if (split_k == 0 && norm_out != nullptr && (resid_out == nullptr || resid_out == resid_in) && t > 256 && h / 8 <= 32 * 24) {
    // many rows, nothing to reduce: one warp per row
    const int nvw = (int)cdiv_ll(h / 8, 32);
    const dim3 rgrid((unsigned)cdiv_ll(t, kRowWarps));
#define ROWS_LAUNCH(NVV)                                                                                                      \
    DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(rmsnorm_rows_kernel<T, NVV>, rgrid, dim3(kRowWarps * 32), 0, (cudaStream_t)stream, 1, \
                                                (const T*)resid_in, (const T*)norm_w, eps, (T*)norm_out, t, (int)h)))
    if (nvw <= 4) { ROWS_LAUNCH(4); } else if (nvw <= 8) { ROWS_LAUNCH(8); } else if (nvw <= 16) { ROWS_LAUNCH(16); }
    else if (nvw <= 20) { ROWS_LAUNCH(20); } else { ROWS_LAUNCH(24); }
#undef ROWS_LAUNCH
  } else {
    const int nv = (int)cdiv_ll(h / 8, kNormThreads);
#define NORM_LAUNCH(NVV)                                                                                                      \
    DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(reduce_residual_rmsnorm_kernel<T, NVV>, dim3((unsigned)t), dim3(kNormThreads), 0, \
                                                (cudaStream_t)stream, 1, partial, split_k, (const T*)resid_in, (T*)resid_out,  \
                                                (const T*)norm_w, eps, (T*)norm_out, t, (int)h)))
    if (nv <= 1) { NORM_LAUNCH(1); } else if (nv <= 2) { NORM_LAUNCH(2); } else if (nv <= 3) { NORM_LAUNCH(3); }
    else if (nv <= 4) { NORM_LAUNCH(4); } else { NORM_LAUNCH(8); }
#undef NORM_LAUNCH
  }
  return CTS_OK;
}

extern "C" int cts_reduce_swiglu(cts_ctx* ctx, const float* partial, int split_k, long long t, long long inter, void* out,
                                 int interleaved, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, partial && out && split_k >= 1 && inter > 0, "args");
  CTS_CHECK_ARG(ctx, !interleaved || inter % 64 == 0, "interleaved gate/up layout needs inter % 64 == 0");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, t <= 65535, "t > 65535");
  if (t == 0) return CTS_OK;
  if (inter % 8 == 0 && ((uintptr_t)partial & 15) == 0 && ((uintptr_t)out & 15) == 0) {
    dim3 vgrid((unsigned)cdiv_ll(inter / 8, kSwiThreads), (unsigned)t);
    DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(reduce_swiglu_vec_kernel<T>, vgrid, dim3(kSwiThreads), 0, (cudaStream_t)stream, 1, partial,
                                                split_k, t, inter, (T*)out, interleaved)));
    return CTS_OK;
  }
  dim3 grid((unsigned)cdiv_ll(inter, 256), (unsigned)t);
  DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(reduce_swiglu_kernel<T>, grid, dim3(256), 0, (cudaStream_t)stream, 1, partial, split_k, t,
                                              inter, (T*)out, interleaved)));
  return CTS_OK;
}

extern "C" int cts_qkv_rope_cache(cts_ctx* ctx, const void* src, int src_is_partial, int split_k, const void* bias,
                                  const int* positions, const void* cos_tab, const void* sin_tab, const int* slot_map,
                                  void* q_out, void* k_cache, void* v_cache, void* k_out, void* v_out, long long t, int nh,
                                  int nkv, int head_dim, int page_size, const void* q_norm_w, const void* k_norm_w, float norm_eps,
                                  int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, src && positions && cos_tab && sin_tab && q_out, "null pointer");
  CTS_CHECK_ARG(ctx, nh > 0 && nkv > 0 && head_dim > 0 && head_dim % 2 == 0 && head_dim <= 512, "head config");
  CTS_CHECK_ARG(ctx, !src_is_partial || split_k >= 1, "split_k");
  CTS_CHECK_ARG(ctx, page_size > 0, "page_size");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, t <= 65535 * 1024LL, "t too large");
  if (t == 0) return CTS_OK;
  // t can exceed 65535 in a big prefill: fold into chunks of the y grid dimension
  const long long width = (long long)(nh + 2 * nkv) * head_dim;
  CTS_CHECK_ARG(ctx, head_dim % 16 == 0 && ((head_dim / 16) & (head_dim / 16 - 1)) == 0 && head_dim / 16 <= 32,
                "head_dim must be 16 * 2^n (<= 512)");
  const int threads = t <= 64 ? 64 : kRopeThreads;      // decode: more, smaller CTAs pull the split-K partials from L2
  for (long long tb = 0; tb < t; tb += 65535) {
    const long long tc = (t - tb) < 65535 ? (t - tb) : 65535;
    dim3 grid((unsigned)cdiv_ll((long long)(nh + 2 * nkv) * (head_dim / 16), threads), (unsigned)tc);
    if (src_is_partial) {
      CTS_CHECK_ARG(ctx, t <= 65535, "partial input with t > 65535");
    }
    const void* src_c = src_is_partial ? src : (const void*)((const char*)src + tb * width * 2);
    if (src_is_partial && (head_dim / 2) % 32 == 0) {
      dim3 sgrid((unsigned)((nh + 2 * nkv + kRopeHeadsPerBlock - 1) / kRopeHeadsPerBlock), (unsigned)tc);
      DISPATCH_T(dtype,
                 CTS_CUDA(ctx, launch_pdl(qkv_rope_cache_scalar_kernel<T>, sgrid, dim3(kRopeHeadsPerBlock * (head_dim / 2)), 0,
                                          (cudaStream_t)stream, 1, src_c, src_is_partial, split_k, (const T*)bias, positions + tb,
                                          (const T*)cos_tab, (const T*)sin_tab, slot_map ? slot_map + tb : (const int*)nullptr,
                                          (T*)q_out + tb * (long long)nh * head_dim, (T*)k_cache, (T*)v_cache,
                                          k_out ? (T*)k_out + tb * (long long)nkv * head_dim : (T*)nullptr,
                                          v_out ? (T*)v_out + tb * (long long)nkv * head_dim : (T*)nullptr, t, nh, nkv, head_dim,
                                          page_size, (const T*)q_norm_w, (const T*)k_norm_w, norm_eps)));
      continue;
    }
    DISPATCH_T(dtype,
               CTS_CUDA(ctx, launch_pdl(qkv_rope_cache_kernel<T>, grid, dim3(threads), 0, (cudaStream_t)stream, 1, src_c, src_is_partial,
                                        split_k, (const T*)bias, positions + tb, (const T*)cos_tab, (const T*)sin_tab,
                                        slot_map ? slot_map + tb : (const int*)nullptr, (T*)q_out + tb * (long long)nh * head_dim,
                                        (T*)k_cache, (T*)v_cache, k_out ? (T*)k_out + tb * (long long)nkv * head_dim : (T*)nullptr,
                                        v_out ? (T*)v_out + tb * (long long)nkv * head_dim : (T*)nullptr,
                                        src_is_partial ? t : tc, nh, nkv, head_dim, page_size, (const T*)q_norm_w, (const T*)k_norm_w,
                                        norm_eps)));
  }
  return CTS_OK;
}

extern "C" int cts_embed_gather(cts_ctx* ctx, const void* table, const int* ids, void* out, long long t, long long h,
                                long long vocab, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, table && ids && out, "null pointer");
  CTS_CHECK_ARG(ctx, h > 0 && h % 8 == 0, "h must be a multiple of 8");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  if (t == 0) return CTS_OK;
  DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(embed_gather_kernel<T>, dim3((unsigned)t), dim3(128), 0, (cudaStream_t)stream, 1,
                                              (const T*)table, ids, (T*)out, h, vocab)));
  return CTS_OK;
}

extern "C" int cts_greedy_advance(cts_ctx* ctx, const void* logits, long long vocab, int batch, int* out_tokens, int out_ld,
                                  int* step_ptr, int* cur_ids, int* positions, int* seq_lens, int* slot_map,
                                  const int* page_table, int max_pages, int page_size, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, logits && vocab > 0 && batch >= 0, "args");
  CTS_CHECK_ARG(ctx, dtype == CTS_BF16 || dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, page_size > 0 || slot_map == nullptr, "page_size");
  if (batch == 0) return CTS_OK;
  DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(greedy_advance_kernel<T>, dim3(batch), dim3(1024), 0, (cudaStream_t)stream, 1,
                                              (const T*)logits, vocab, out_tokens, out_ld, step_ptr, cur_ids, positions, seq_lens,
                                              slot_map, page_table, max_pages, page_size > 0 ? page_size : 1)));
  return CTS_OK;
}

CTS_TRACE_SETTER(cts_trace_set_elementwise)
