// chatts_b200 -- memory-bound kernels of the LoRA fine-tune step (SURVEY.md 8(a) row A9; include/chatts_b200.h, "A9").
// The reference repo has no training code (README.md:216-218); the arithmetic restated here is peft's lora.Linear,
// transformers' ForCausalLMLoss / Qwen2RMSNorm / rotate_half RoPE / SiLU-gated MLP under autograd, torch.optim.AdamW and
// clip_grad_norm_ -- see oracle/lora.py for the CPU statement these are checked against.
//
//   cts_swiglu / cts_swiglu_bwd    SiLU-gated product from a model-dtype gate_up tensor, and its backward
//   cts_rmsnorm_bwd                RMSNorm backward (frozen weight) fused with the residual-stream gradient add
//   cts_qkv_rope_bwd               RoPE^T (+ Qwen3 per-head q/k RMSNorm backward), dv pass-through -> dqkv
//   cts_ce_loss_grad               cross entropy forward + in-place backward over the label rows
//   cts_gather_rows                row select / zero-filling scatter
//   cts_lora_wgrad                 skinny weight gradients dB = s dY^T U, dA = dU^T X (HBM-bound)
//   cts_adamw, cts_grad_norm_clip  optimiser on flat fp32 arenas
//   cts_lora_pack                  fp32 master adapters -> model-dtype fused GEMM operands (+ transposed copies)
//
// Every kernel follows the library's PDL protocol (pdl_trigger, then pdl_wait before touching memory).  None of them
// spins on a flag or a barrier other than __syncthreads(), so a bug here can produce a wrong number but not a hang.
#include "common.cuh"

namespace {

__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// column of feature i in a gate_up row: stacked = (i, inter + i); interleaved = 64 gate columns then the 64 matching up
// columns per 128-column tile (CTS_EPI_SWIGLU_IL)
__device__ __forceinline__ long long gate_col(long long i, long long inter, int interleaved) {
  return interleaved ? (i >> 6) * 128 + (i & 63) : i;
}
__device__ __forceinline__ long long up_col(long long i, long long inter, int interleaved) {
  return interleaved ? (i >> 6) * 128 + (i & 63) + 64 : inter + i;
}

// ------------------------------------------------------------------------------------------------ SwiGLU
// grid (ceil(inter / 8 / 256), t); thread = 8 consecutive features (never straddles a 64-feature group)
template <typename T>
__global__ void __launch_bounds__(256)
swiglu_fwd_kernel(const T* __restrict__ gu, long long inter, int interleaved, T* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const long long t = blockIdx.y;
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= inter) return;
  const T* row = gu + t * 2 * inter;
  float g[8], u[8], o[8];
  unpack8<T>(*reinterpret_cast<const uint4*>(row + gate_col(i, inter, interleaved)), g);
  unpack8<T>(*reinterpret_cast<const uint4*>(row + up_col(i, inter, interleaved)), u);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = rnd<T>(silu_f(g[j])) * u[j];       // act_fn(gate) is a dtype tensor, then * up (:47)
  *reinterpret_cast<uint4*>(out + t * inter + i) = pack8<T>(o);
}

template <typename T>
__global__ void __launch_bounds__(256)
swiglu_bwd_kernel(const T* __restrict__ gu, const T* __restrict__ dact, long long inter, int interleaved, T* __restrict__ dgu) {
  pdl_trigger();
  pdl_wait();
  const long long t = blockIdx.y;
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i >= inter) return;
  const long long gc = gate_col(i, inter, interleaved), uc = up_col(i, inter, interleaved);
  const T* row = gu + t * 2 * inter;
  float g[8], u[8], d[8], dg[8], du[8];
  unpack8<T>(*reinterpret_cast<const uint4*>(row + gc), g);
  unpack8<T>(*reinterpret_cast<const uint4*>(row + uc), u);
  unpack8<T>(*reinterpret_cast<const uint4*>(dact + t * inter + i), d);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float sg = sigmoid_f(g[j]);
    du[j] = d[j] * rnd<T>(g[j] * sg);                                   // d/du = silu(g) (the dtype tensor the forward used)
    dg[j] = d[j] * u[j] * sg * (1.0f + g[j] * (1.0f - sg));             // d/dg = u * silu'(g)
  }
  T* orow = dgu + t * 2 * inter;
  *reinterpret_cast<uint4*>(orow + gc) = pack8<T>(dg);
  *reinterpret_cast<uint4*>(orow + uc) = pack8<T>(du);
}

// ------------------------------------------------------------------------------------------------ RMSNorm backward
// one CTA per token.  y = w * dtype(x * rstd):  g = dy * w,  dx = rstd * g - x * rstd^3 * (sum_j g_j x_j) / h
constexpr int kNbThreads = 256;

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();                                   // red may still be read from a previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < kNbThreads / 32; ++w) tot += red[w];
  return tot;
}

template <typename T>
__global__ void __launch_bounds__(kNbThreads)
rmsnorm_bwd_kernel(const T* dy, const T* __restrict__ x, const T* __restrict__ w, float eps, const T* dres_in, T* dx_out,
                   int h) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[kNbThreads / 32];
  const long long t = blockIdx.x;
  const int nvec = h / 8;
  const T* xr = x + t * h;
  const T* dyr = dy + t * h;
  float ss = 0.f, gx = 0.f;
  for (int v = threadIdx.x; v < nvec; v += kNbThreads) {
    float xv[8], dv[8], wv[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(xr + v * 8), xv);
    unpack8<T>(*reinterpret_cast<const uint4*>(dyr + v * 8), dv);
    unpack8<T>(*reinterpret_cast<const uint4*>(w + v * 8), wv);
#pragma unroll
    for (int j = 0; j < 8; ++j) { ss += xv[j] * xv[j]; gx += dv[j] * wv[j] * xv[j]; }
  }
  ss = block_sum_256(ss, red);
  gx = block_sum_256(gx, red);
  const float rstd = 1.0f / sqrtf(ss / (float)h + eps);
  const float c = rstd * rstd * rstd * gx / (float)h;
  // second pass re-reads the row (L1/L2 resident); dx_out may alias dy or dres_in: every thread reads its own 8 elements
  // of all three inputs before it writes them
  for (int v = threadIdx.x; v < nvec; v += kNbThreads) {
    float xv[8], dv[8], wv[8], rv[8], o[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(xr + v * 8), xv);
    unpack8<T>(*reinterpret_cast<const uint4*>(dyr + v * 8), dv);
    unpack8<T>(*reinterpret_cast<const uint4*>(w + v * 8), wv);
    if (dres_in) {
      unpack8<T>(*reinterpret_cast<const uint4*>(dres_in + t * h + v * 8), rv);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) rv[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = rv[j] + rstd * dv[j] * wv[j] - xv[j] * c;
    *reinterpret_cast<uint4*>(dx_out + t * h + v * 8) = pack8<T>(o);
  }
}

// ------------------------------------------------------------------------------------------------ RoPE (+ q/k norm) backward
// same thread mapping as qkv_rope_cache_kernel: thread = (head, chunk of 8 rotary pairs); the d/16 threads of a head sit in
// one warp (d/16 is a power of two <= 32), so the per-head RMSNorm statistics are sub-warp shuffles.
constexpr int kRbThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kRbThreads)
qkv_rope_bwd_kernel(const T* __restrict__ dq, const T* __restrict__ dk, const T* __restrict__ dv, const T* __restrict__ qkv,
                    const int* __restrict__ positions, const T* __restrict__ cos_tab, const T* __restrict__ sin_tab,
                    const T* __restrict__ q_norm_w, const T* __restrict__ k_norm_w, float norm_eps, T* __restrict__ dqkv,
                    int nh, int nkv, int d) {
  pdl_trigger();
  pdl_wait();
  const int half = d >> 1;
  const int cph = half >> 3;
  const int item = blockIdx.x * blockDim.x + threadIdx.x;
  const int head = item / cph, j = item % cph;
  const long long t = blockIdx.y;
  const int heads = nh + 2 * nkv;
  const bool active = head < heads;
  const int hd = active ? head : 0;
  const bool is_q = hd < nh;
  const bool is_k = !is_q && hd < nh + nkv;
  const long long width = (long long)heads * d;
  const long long c0 = (long long)hd * d + j * 8, c1 = c0 + half;
  // incoming gradient of this head (post-RoPE q / k, or v)
  const T* src;
  if (is_q) src = dq + t * (long long)nh * d + (long long)hd * d;
  else if (is_k) src = dk + t * (long long)nkv * d + (long long)(hd - nh) * d;
  else src = dv + t * (long long)nkv * d + (long long)(hd - nh - nkv) * d;
  float g0[8], g1[8];
  unpack8<T>(*reinterpret_cast<const uint4*>(src + j * 8), g0);
  unpack8<T>(*reinterpret_cast<const uint4*>(src + half + j * 8), g1);
  if (is_q || is_k) {
    // y0 = x0 c - x1 s, y1 = x1 c + x0 s  =>  dx0 = dy0 c + dy1 s, dx1 = dy1 c - dy0 s
    const int pos = positions[t];
    float cs[8], sn[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(cos_tab + (long long)pos * half + j * 8), cs);
    unpack8<T>(*reinterpret_cast<const uint4*>(sin_tab + (long long)pos * half + j * 8), sn);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float a = g0[e] * cs[e] + g1[e] * sn[e];
      const float b = g1[e] * cs[e] - g0[e] * sn[e];
      g0[e] = a; g1[e] = b;
    }
  }
  if (q_norm_w != nullptr || k_norm_w != nullptr) {          // kernel-uniform: every lane takes part in the shuffles
    const T* nw = is_q ? q_norm_w : (is_k ? k_norm_w : nullptr);
    float x0[8], x1[8], w0[8], w1[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(qkv + t * width + c0), x0);
    unpack8<T>(*reinterpret_cast<const uint4*>(qkv + t * width + c1), x1);
    float ss = 0.f, gx = 0.f;
    if (nw != nullptr) {
      unpack8<T>(*reinterpret_cast<const uint4*>(nw + j * 8), w0);
      unpack8<T>(*reinterpret_cast<const uint4*>(nw + half + j * 8), w1);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        g0[e] *= w0[e]; g1[e] *= w1[e];                      // g = dy * w
        ss += x0[e] * x0[e] + x1[e] * x1[e];
        gx += g0[e] * x0[e] + g1[e] * x1[e];
      }
    }
    for (int o = cph >> 1; o > 0; o >>= 1) {
      ss += __shfl_xor_sync(0xffffffffu, ss, o);
      gx += __shfl_xor_sync(0xffffffffu, gx, o);
    }
    if (nw != nullptr) {
      const float rstd = 1.0f / sqrtf(ss / (float)d + norm_eps);
      const float c = rstd * rstd * rstd * gx / (float)d;
#pragma unroll
      for (int e = 0; e < 8; ++e) { g0[e] = rstd * g0[e] - x0[e] * c; g1[e] = rstd * g1[e] - x1[e] * c; }
    }
  }
  if (!active) return;
  *reinterpret_cast<uint4*>(dqkv + t * width + c0) = pack8<T>(g0);
  *reinterpret_cast<uint4*>(dqkv + t * width + c1) = pack8<T>(g1);
}

// ------------------------------------------------------------------------------------------------ cross entropy
// one CTA per label row: online (max, sum) over the vocabulary, then the in-place gradient
constexpr int kCeThreads = 1024;

template <typename T>
__global__ void __launch_bounds__(kCeThreads)
ce_loss_grad_kernel(T* __restrict__ logits, long long ld, const int* __restrict__ targets, long long vocab, float grad_scale,
                    float* __restrict__ row_loss) {
  pdl_trigger();
  pdl_wait();
  __shared__ float sm[32], sl[32];
  __shared__ float lse_s;
  const long long r = blockIdx.x;
  T* row = logits + r * ld;
  const int tgt = targets[r];
  const long long nvec = vocab / 8;
  float m = -INFINITY, l = 0.f;
  for (long long v = threadIdx.x; v < nvec; v += kCeThreads) {
    float f[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(row + v * 8), f);
    float mx = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) mx = fmaxf(mx, f[j]);
    const float mn = fmaxf(m, mx);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += expf(f[j] - mn);
    l = (m > -INFINITY ? l * expf(m - mn) : 0.f) + s;
    m = mn;
  }
  // warp, then block merge of (m, l)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o), ol = __shfl_xor_sync(0xffffffffu, l, o);
    const float mn = fmaxf(m, om);
    l = (m > -INFINITY ? l * expf(m - mn) : 0.f) + (om > -INFINITY ? ol * expf(om - mn) : 0.f);
    m = mn;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { sm[warp] = m; sl[warp] = l; }
  __syncthreads();
  if (warp == 0) {
    m = sm[lane]; l = sl[lane];                      // 32 warps exactly
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o), ol = __shfl_xor_sync(0xffffffffu, l, o);
      const float mn = fmaxf(m, om);
      l = (m > -INFINITY ? l * expf(m - mn) : 0.f) + (om > -INFINITY ? ol * expf(om - mn) : 0.f);
      m = mn;
    }
    if (lane == 0) {
      const float lse = m + logf(l);
      lse_s = lse;
      const bool counted = tgt >= 0 && tgt < vocab;
      row_loss[r] = counted ? lse - DT<T>::to_f(row[tgt]) : 0.f;      // read before any thread overwrites the row
    }
  }
  __syncthreads();
  const float lse = lse_s;
  const bool counted = tgt >= 0 && tgt < vocab;
  for (long long v = threadIdx.x; v < nvec; v += kCeThreads) {
    float f[8];
    unpack8<T>(*reinterpret_cast<const uint4*>(row + v * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p = counted ? expf(f[j] - lse) : 0.f;
      if (counted && v * 8 + j == (long long)tgt) p -= 1.0f;
      f[j] = p * grad_scale;
    }
    *reinterpret_cast<uint4*>(row + v * 8) = pack8<T>(f);
  }
}

// loss_out[0] = (accumulate ? loss_out[0] : 0) + scale * sum(row_loss)   -- one CTA, fixed order
__global__ void __launch_bounds__(1024) ce_loss_reduce_kernel(const float* __restrict__ row_loss, long long n, float scale,
                                                               float* __restrict__ loss_out, int accumulate) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  float s = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) s += row_loss[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) loss_out[0] = (accumulate ? loss_out[0] : 0.f) + scale * v;
  }
}

// ------------------------------------------------------------------------------------------------ row gather
template <typename T>
__global__ void gather_rows_kernel(const T* __restrict__ src, const int* __restrict__ idx, long long h, T* __restrict__ dst) {
  pdl_trigger();
  pdl_wait();
  const long long i = blockIdx.x;
  const int s = idx[i];
  uint4* d = reinterpret_cast<uint4*>(dst + i * h);
  if (s < 0) {
    for (int v = threadIdx.x; v < h / 8; v += blockDim.x) d[v] = make_uint4(0u, 0u, 0u, 0u);
    return;
  }
  const uint4* p = reinterpret_cast<const uint4*>(src + (long long)s * h);
  for (int v = threadIdx.x; v < h / 8; v += blockDim.x) d[v] = p[v];
}

// ------------------------------------------------------------------------------------------------ LoRA weight gradient
// out[m][j] += scale * sum_t P[t][col(m)] * Q[t][q_col0 + j].  CTA = 64 features (lane -> 2 adjacent ones) x 16 rank
// columns; the 8 warps stride the CTA's token range; P is streamed once (128 B per warp and token), Q (<= 32 B per
// token) is a warp-uniform broadcast load that stays in L1/L2.  grid (ceil(M/64), ceil(r/16), token splits).
constexpr int kWgThreads = 256, kWgM = 64, kWgR = 16;

template <typename T>
__global__ void __launch_bounds__(kWgThreads)
lora_wgrad_kernel(const T* __restrict__ P, long long p_ld, long long p_col0, int p_il, long long M, const T* __restrict__ Q,
                  long long q_ld, long long q_col0, int r, long long t_total, float scale, float* __restrict__ out, long long so_m,
                  long long so_r) {
  pdl_trigger();
  pdl_wait();
  __shared__ float acc_s[kWgThreads / 32][kWgM][kWgR + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long m = (long long)blockIdx.x * kWgM + lane * 2;       // M is even: m and m + 1 are valid together
  const int j0 = blockIdx.y * kWgR;
  const int rc = min(kWgR, r - j0);
  const bool m_ok = m < M;
  long long col;
  if (p_il == 0) col = p_col0 + m;
  else col = (m >> 6) * 128 + (m & 63) + (p_il == 2 ? 64 : 0);        // m even: m + 1 stays inside the 64-feature group
  const long long per = (t_total + gridDim.z - 1) / gridDim.z;
  const long long t0 = (long long)blockIdx.z * per;
  const long long t1 = t0 + per < t_total ? t0 + per : t_total;
  float a0[kWgR], a1[kWgR];
#pragma unroll
  for (int j = 0; j < kWgR; ++j) { a0[j] = 0.f; a1[j] = 0.f; }
  // 16 rank columns of a token = 32 bytes: two 16-byte loads when the slice is aligned, scalar loads otherwise
  const bool q_vec = rc == kWgR && (q_ld % 8) == 0 && ((q_col0 + j0) % 8) == 0 && ((uintptr_t)Q & 15) == 0;
  for (long long t = t0 + warp; t < t1; t += kWgThreads / 32) {
    float p0 = 0.f, p1 = 0.f;
    if (m_ok) {
      // col is even and p_ld is even: one aligned 4-byte load brings both features
      const uint32_t raw = *reinterpret_cast<const uint32_t*>(P + t * p_ld + col);
      const T* pp = reinterpret_cast<const T*>(&raw);
      p0 = DT<T>::to_f(pp[0]);
      p1 = DT<T>::to_f(pp[1]);
    }
    const T* qq = Q + t * q_ld + q_col0 + j0;
    float qv[kWgR];
    if (q_vec) {
      unpack8<T>(*reinterpret_cast<const uint4*>(qq), qv);
      unpack8<T>(*reinterpret_cast<const uint4*>(qq + 8), qv + 8);
    } else {
#pragma unroll
      for (int j = 0; j < kWgR; ++j) qv[j] = j < rc ? DT<T>::to_f(qq[j]) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < kWgR; ++j) {
      a0[j] = fmaf(p0, qv[j], a0[j]);
      a1[j] = fmaf(p1, qv[j], a1[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < kWgR; ++j) { acc_s[warp][lane * 2][j] = a0[j]; acc_s[warp][lane * 2 + 1][j] = a1[j]; }
  __syncthreads();
  for (int e = threadIdx.x; e < kWgM * kWgR; e += kWgThreads) {
    const int mm = e / kWgR, j = e % kWgR;
    const long long mg = (long long)blockIdx.x * kWgM + mm;
    if (mg >= M || j >= rc) continue;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kWgThreads / 32; ++w) s += acc_s[w][mm][j];
    float* o = out + mg * so_m + (long long)(j0 + j) * so_r;
    if (gridDim.z == 1) *o += scale * s;                               // sole writer of this element in this launch
    else atomicAdd(o, scale * s);
  }
}

// ------------------------------------------------------------------------------------------------ optimiser
__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                     float* __restrict__ v, long long n, float lr, float b1, float b2, float eps,
                                                     float wd, float bc1, float bc2_sqrt, const float* __restrict__ grad_scale) {
  pdl_trigger();
  pdl_wait();
  const float gs = grad_scale ? grad_scale[0] : 1.0f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i] * gs;
    float pi = p[i] * (1.0f - lr * wd);                                // decoupled decay
    const float mi = b1 * m[i] + (1.0f - b1) * gi;
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    pi -= (lr / bc1) * mi / denom;
    p[i] = pi;
  }
}

constexpr int kGnBlocks = 1024, kGnThreads = 256;

__global__ void __launch_bounds__(kGnThreads) sumsq_partial_kernel(const float* __restrict__ g, long long n, float* __restrict__ ws) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[kGnThreads / 32];
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) s += g[i] * g[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int w = 0; w < kGnThreads / 32; ++w) tot += red[w];
    ws[blockIdx.x] = tot;
  }
}

__global__ void __launch_bounds__(kGnBlocks) grad_norm_final_kernel(const float* __restrict__ ws, int n_part, float max_norm,
                                                                     float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  float s = threadIdx.x < n_part ? ws[threadIdx.x] : 0.f;
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) {
      const float nrm = sqrtf(v);
      out[0] = nrm;
      out[1] = max_norm > 0.f ? fminf(1.0f, max_norm / (nrm + 1e-6f)) : 1.0f;
    }
  }
}

// ------------------------------------------------------------------------------------------------ adapter packing
template <typename T>
__global__ void __launch_bounds__(256) lora_pack_kernel(const float* __restrict__ master, const long long* __restrict__ desc,
                                                         T* __restrict__ work) {
  pdl_trigger();
  pdl_wait();
  const long long* d = desc + (long long)blockIdx.y * CTS_PACK_DESC_LONGS;
  const long long src_off = d[0], rows = d[1], cols = d[2], dst_off = d[3], dst_ld = d[4], row0 = d[5], il = d[6], col0 = d[7],
                  dstT_off = d[8], dstT_ld = d[9];
  const float scale = __int_as_float((int)d[10]);
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < rows * cols; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / cols, j = e % cols;
    const long long rm = il == 0 ? row0 + i : (i >> 6) * 128 + (i & 63) + (il == 2 ? 64 : 0);
    const T val = DT<T>::from_f(master[src_off + e] * scale);
    work[dst_off + rm * dst_ld + col0 + j] = val;
    work[dstT_off + (col0 + j) * dstT_ld + rm] = val;
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

#define CTS_CHECK_DTYPE(ctx, dtype) CTS_CHECK_ARG(ctx, (dtype) == CTS_BF16 || (dtype) == CTS_F16, "dtype must be CTS_BF16 or CTS_F16")

extern "C" int cts_swiglu(cts_ctx* ctx, const void* gu, long long t, long long inter, int interleaved, void* out, int dtype,
                          void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, gu && out && inter > 0 && t >= 0, "args");
  CTS_CHECK_ARG(ctx, inter % 8 == 0 && (!interleaved || inter % 64 == 0), "inter must be a multiple of 8 (64 when interleaved)");
  CTS_CHECK_DTYPE(ctx, dtype);
  CTS_CHECK_ARG(ctx, t <= 65535LL * 65535LL, "t too large");
  for (long long tb = 0; tb < t; tb += 65535) {
    const long long tc = t - tb < 65535 ? t - tb : 65535;
    dim3 grid((unsigned)cdiv_ll(inter / 8, 256), (unsigned)tc);
    DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(swiglu_fwd_kernel<T>, grid, dim3(256), 0, (cudaStream_t)stream, 1,
                                                (const T*)gu + tb * 2 * inter, inter, interleaved, (T*)out + tb * inter)));
  }
  return CTS_OK;
}

extern "C" int cts_swiglu_bwd(cts_ctx* ctx, const void* gu, const void* dact, long long t, long long inter, int interleaved,
                              void* dgu, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, gu && dact && dgu && inter > 0 && t >= 0, "args");
  CTS_CHECK_ARG(ctx, inter % 8 == 0 && (!interleaved || inter % 64 == 0), "inter must be a multiple of 8 (64 when interleaved)");
  CTS_CHECK_DTYPE(ctx, dtype);
  for (long long tb = 0; tb < t; tb += 65535) {
    const long long tc = t - tb < 65535 ? t - tb : 65535;
    dim3 grid((unsigned)cdiv_ll(inter / 8, 256), (unsigned)tc);
    DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(swiglu_bwd_kernel<T>, grid, dim3(256), 0, (cudaStream_t)stream, 1,
                                                (const T*)gu + tb * 2 * inter, (const T*)dact + tb * inter, inter, interleaved,
                                                (T*)dgu + tb * 2 * inter)));
  }
  return CTS_OK;
}

extern "C" int cts_rmsnorm_bwd(cts_ctx* ctx, const void* dy, const void* x, const void* w, float eps, const void* dres_in,
                               void* dx_out, long long t, long long h, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, dy && x && w && dx_out, "null pointer");
  CTS_CHECK_ARG(ctx, h > 0 && h % 8 == 0 && h <= (1 << 20), "h must be a positive multiple of 8");
  CTS_CHECK_ARG(ctx, t >= 0 && t <= 0x7fffffffLL, "t");
  CTS_CHECK_DTYPE(ctx, dtype);
  if (t == 0) return CTS_OK;
  DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(rmsnorm_bwd_kernel<T>, dim3((unsigned)t), dim3(kNbThreads), 0, (cudaStream_t)stream, 1,
                                              (const T*)dy, (const T*)x, (const T*)w, eps, (const T*)dres_in, (T*)dx_out, (int)h)));
  return CTS_OK;
}

extern "C" int cts_qkv_rope_bwd(cts_ctx* ctx, const void* dq, const void* dk, const void* dv, const void* qkv, const int* positions,
                                const void* cos_tab, const void* sin_tab, const void* q_norm_w, const void* k_norm_w, float norm_eps,
                                void* dqkv, long long t, int nh, int nkv, int head_dim, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, dq && dk && dv && positions && cos_tab && sin_tab && dqkv, "null pointer");
  CTS_CHECK_ARG(ctx, (q_norm_w == nullptr && k_norm_w == nullptr) || qkv != nullptr, "q/k norm backward needs the saved qkv");
  CTS_CHECK_ARG(ctx, nh > 0 && nkv > 0, "head config");
  CTS_CHECK_ARG(ctx, head_dim % 16 == 0 && ((head_dim / 16) & (head_dim / 16 - 1)) == 0 && head_dim / 16 <= 32 && head_dim >= 16,
                "head_dim must be 16 * 2^n (<= 512)");
  CTS_CHECK_DTYPE(ctx, dtype);
  const long long width = (long long)(nh + 2 * nkv) * head_dim;
  for (long long tb = 0; tb < t; tb += 65535) {
    const long long tc = t - tb < 65535 ? t - tb : 65535;
    dim3 grid((unsigned)cdiv_ll((long long)(nh + 2 * nkv) * (head_dim / 16), kRbThreads), (unsigned)tc);
    DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(qkv_rope_bwd_kernel<T>, grid, dim3(kRbThreads), 0, (cudaStream_t)stream, 1,
                                                (const T*)dq + tb * (long long)nh * head_dim, (const T*)dk + tb * (long long)nkv * head_dim,
                                                (const T*)dv + tb * (long long)nkv * head_dim,
                                                qkv ? (const T*)qkv + tb * width : (const T*)nullptr, positions + tb, (const T*)cos_tab,
                                                (const T*)sin_tab, (const T*)q_norm_w, (const T*)k_norm_w, norm_eps,
                                                (T*)dqkv + tb * width, nh, nkv, head_dim)));
  }
  return CTS_OK;
}

extern "C" int cts_ce_loss_grad(cts_ctx* ctx, void* logits, long long ld, const int* targets, long long n_rows, long long vocab,
                                float grad_scale, float* row_loss, float* loss_out, int accumulate, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, logits && targets && row_loss && loss_out, "null pointer");
  CTS_CHECK_ARG(ctx, vocab > 0 && vocab % 8 == 0 && ld >= vocab && ld % 8 == 0, "vocab and ld must be multiples of 8, ld >= vocab");
  CTS_CHECK_ARG(ctx, n_rows >= 0 && n_rows <= 0x7fffffffLL, "n_rows");
  CTS_CHECK_ARG(ctx, ((uintptr_t)logits & 15) == 0, "logits must be 16-byte aligned");
  CTS_CHECK_DTYPE(ctx, dtype);
  if (n_rows > 0) {
    DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(ce_loss_grad_kernel<T>, dim3((unsigned)n_rows), dim3(kCeThreads), 0, (cudaStream_t)stream, 1,
                                                (T*)logits, ld, targets, vocab, grad_scale, row_loss)));
  }
  CTS_CUDA(ctx, launch_pdl(ce_loss_reduce_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream, 1, (const float*)row_loss, n_rows,
                           grad_scale, loss_out, accumulate));
  return CTS_OK;
}

extern "C" int cts_gather_rows(cts_ctx* ctx, const void* src, const int* idx, long long n_out, long long h, void* dst, int dtype,
                               void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, src && idx && dst, "null pointer");
  CTS_CHECK_ARG(ctx, h > 0 && h % 8 == 0, "h must be a multiple of 8");
  CTS_CHECK_ARG(ctx, n_out >= 0 && n_out <= 0x7fffffffLL, "n_out");
  CTS_CHECK_DTYPE(ctx, dtype);
  if (n_out == 0) return CTS_OK;
  DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(gather_rows_kernel<T>, dim3((unsigned)n_out), dim3(128), 0, (cudaStream_t)stream, 1,
                                              (const T*)src, idx, h, (T*)dst)));
  return CTS_OK;
}

// tensor-core variant (lora_wgrad_mma.cu), the default; CTS_WGRAD_MMA=0 selects the FMA kernel
bool cts_lora_wgrad_mma_enabled();
bool cts_lora_wgrad_mma_ok(const void* p, long long p_ld, long long p_col0, int p_il, long long m, const void* q, long long q_ld,
                           long long q_col0, int r);
int cts_lora_wgrad_mma_launch(cts_ctx* ctx, const void* p, long long p_ld, long long p_col0, int p_il, long long m, const void* q,
                              long long q_ld, long long q_col0, int r, long long t, float scale, float* out, long long so_m,
                              long long so_r, int dtype, cudaStream_t st);

extern "C" int cts_lora_wgrad(cts_ctx* ctx, const void* p, long long p_ld, long long p_col0, int p_il, long long m, const void* q,
                              long long q_ld, long long q_col0, int r, long long t, float scale, float* out, long long so_m,
                              long long so_r, int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, p && q && out, "null pointer");
  CTS_CHECK_ARG(ctx, m > 0 && m % 2 == 0 && p_ld % 2 == 0 && p_col0 % 2 == 0 && ((uintptr_t)p & 3) == 0,
                "m, p_ld and p_col0 must be even (paired feature loads)");
  CTS_CHECK_ARG(ctx, p_il >= 0 && p_il <= 2 && (p_il == 0 || m % 64 == 0), "p_il in {0,1,2}; interleaved layout needs m % 64 == 0");
  CTS_CHECK_ARG(ctx, r > 0 && r <= 64 && t >= 0, "1 <= r <= 64");
  CTS_CHECK_DTYPE(ctx, dtype);
  if (t == 0) return CTS_OK;
  if (cts_lora_wgrad_mma_enabled() && cts_lora_wgrad_mma_ok(p, p_ld, p_col0, p_il, m, q, q_ld, q_col0, r))
    return cts_lora_wgrad_mma_launch(ctx, p, p_ld, p_col0, p_il, m, q, q_ld, q_col0, r, t, scale, out, so_m, so_r, dtype,
                                     (cudaStream_t)stream);
  const long long tiles = cdiv_ll(m, kWgM) * cdiv_ll(r, kWgR);
  long long splits = (4LL * ctx->sm_count) / tiles;                  // ~4 CTAs per SM over the whole grid
  const long long max_splits = cdiv_ll(t, 256);                      // at least 256 tokens (32 per warp) per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits > 1024) splits = 1024;
  if (splits < 1) splits = 1;
  dim3 grid((unsigned)cdiv_ll(m, kWgM), (unsigned)cdiv_ll(r, kWgR), (unsigned)splits);
  DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(lora_wgrad_kernel<T>, grid, dim3(kWgThreads), 0, (cudaStream_t)stream, 1, (const T*)p, p_ld,
                                              p_col0, p_il, m, (const T*)q, q_ld, q_col0, r, t, scale, out, so_m, so_r)));
  return CTS_OK;
}

extern "C" int cts_adamw(cts_ctx* ctx, float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                         float eps, float weight_decay, int step, const float* grad_scale, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, p && g && m && v && n >= 0, "null pointer");
  CTS_CHECK_ARG(ctx, step >= 1, "step counts from 1");
  if (n == 0) return CTS_OK;
  const float bc1 = 1.0f - powf(beta1, (float)step);
  const float bc2_sqrt = sqrtf(1.0f - powf(beta2, (float)step));
  long long blocks = cdiv_ll(n, 256 * 4);
  if (blocks > 8LL * ctx->sm_count) blocks = 8LL * ctx->sm_count;
  if (blocks < 1) blocks = 1;
  CTS_CUDA(ctx, launch_pdl(adamw_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, 1, p, g, m, v, n, lr, beta1, beta2,
                           eps, weight_decay, bc1, bc2_sqrt, grad_scale));
  return CTS_OK;
}

extern "C" long long cts_grad_norm_ws_floats(void) { return kGnBlocks; }

extern "C" int cts_grad_norm_clip(cts_ctx* ctx, const float* g, long long n, float max_norm, float* ws, float* out, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, g && ws && out && n >= 0, "null pointer");
  long long blocks = cdiv_ll(n > 0 ? n : 1, kGnThreads * 8);
  if (blocks > kGnBlocks) blocks = kGnBlocks;
  CTS_CUDA(ctx, launch_pdl(sumsq_partial_kernel, dim3((unsigned)blocks), dim3(kGnThreads), 0, (cudaStream_t)stream, 1, g, n, ws));
  CTS_CUDA(ctx, launch_pdl(grad_norm_final_kernel, dim3(1), dim3(kGnBlocks), 0, (cudaStream_t)stream, 1, (const float*)ws, (int)blocks,
                           max_norm, out));
  return CTS_OK;
}

extern "C" int cts_lora_pack(cts_ctx* ctx, const float* master, const long long* desc, int n_desc, long long max_elems, void* work,
                             int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, master && desc && work, "null pointer");
  CTS_CHECK_ARG(ctx, n_desc >= 0 && n_desc <= 65535 && max_elems >= 0, "n_desc");
  CTS_CHECK_DTYPE(ctx, dtype);
  if (n_desc == 0 || max_elems == 0) return CTS_OK;
  long long bx = cdiv_ll(max_elems, 256 * 4);
  if (bx > 64) bx = 64;
  if (bx < 1) bx = 1;
  dim3 grid((unsigned)bx, (unsigned)n_desc);
  DISPATCH_T(dtype, CTS_CUDA(ctx, launch_pdl(lora_pack_kernel<T>, grid, dim3(256), 0, (cudaStream_t)stream, 1, master, desc, (T*)work)));
  return CTS_OK;
}
