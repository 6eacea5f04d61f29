// chatts_b200 -- tensor-core variant of the skinny LoRA weight gradient (cts_lora_wgrad, include/chatts_b200.h):
//     out[m][j] += scale * sum_t P[t][col(m)] * Q[t][q_col0 + j]
// The FMA kernel of train_elementwise.cu issues ~58 instructions per 64 features x 16 ranks x 1 token; here the same tile costs
// two ldmatrix + two mma.sync per SIXTEEN tokens, so the kernel is left with streaming P (HBM-bound: 2r flop per 2-byte element).
// The reduction index (tokens) is the slow axis of both operands, so both go through shared memory and ldmatrix.trans
// (tokens x features / tokens x ranks tiles, staged by cp.async, double-buffered):
//     A[m = feature][k = token] = Ps[token][feature]^T      B[k = token][n = rank] = Qs[token][rank]
// CTA = 64 features (4 warps x 16) x 16 ranks; grid (ceil(M/64), ceil(r/16), token splits), fp32 atomics across the splits
// exactly like the FMA kernel.  cts_lora_wgrad falls back to the
// (validated) FMA kernel whenever a 16-byte alignment precondition does not hold.  No flag / barrier spin.
#include <stdlib.h>

#include "common.cuh"

namespace {

constexpr int kTok = 64;                     // tokens per staged chunk
constexpr int kFeat = 64, kRank = 16, kThreads = 128;
constexpr int kPRow = kFeat * 2 + 16;        // padded shared row of the P tile (144 B: conflict-free ldmatrix)
constexpr int kQRow = kRank * 2 + 16;        // padded shared row of the Q tile (48 B)

__device__ __forceinline__ void wg_cp16(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void wg_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void wg_ldsm_x4_trans(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
template <typename T> __device__ __forceinline__ void wg_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void wg_mma<__nv_bfloat16>(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void wg_mma<__half>(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
lora_wgrad_mma_kernel(const T* __restrict__ P, long long p_ld, long long p_col0, int p_il, long long M, const T* __restrict__ Q,
                      long long q_ld, long long q_col0, int r, long long t_total, float scale, float* __restrict__ out, long long so_m,
                      long long so_r) {
  pdl_trigger();
  pdl_wait();
  __shared__ __align__(16) uint8_t ps[2][kTok * kPRow];
  __shared__ __align__(16) uint8_t qs[2][kTok * kQRow];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long m0 = (long long)blockIdx.x * kFeat;
  const int j0 = blockIdx.y * kRank;
  const int rc = min(kRank, r - j0);                 // multiple of 8 (checked by the host)
  // first column of this CTA's 64 features (one 64-feature group of the interleaved layout, or a plain range)
  const long long col0 = p_il == 0 ? p_col0 + m0 : (m0 >> 6) * 128 + (p_il == 2 ? 64 : 0);
  const int feat_valid = (int)min((long long)kFeat, M - m0);     // multiple of 8
  const long long per = (t_total + gridDim.z - 1) / gridDim.z;
  const long long t0 = (long long)blockIdx.z * per;
  const long long t1 = t0 + per < t_total ? t0 + per : t_total;
  const int n_chunks = t1 > t0 ? (int)((t1 - t0 + kTok - 1) / kTok) : 0;

  auto issue = [&](int c, int st) {
    const long long tb = t0 + (long long)c * kTok;
    // P tile: 64 tokens x 8 chunks of 16 B;  Q tile: 64 tokens x 2 chunks
    for (int i = threadIdx.x; i < kTok * 8; i += kThreads) {
      const int row = i >> 3, ch = i & 7;
      const bool ok = tb + row < t1 && ch * 8 < feat_valid;
      wg_cp16(ps[st] + row * kPRow + ch * 16, P + (ok ? (tb + row) * p_ld + col0 + ch * 8 : 0), ok);
    }
    for (int i = threadIdx.x; i < kTok * 2; i += kThreads) {
      const int row = i >> 1, ch = i & 1;
      const bool ok = tb + row < t1 && ch * 8 < rc;
      wg_cp16(qs[st] + row * kQRow + ch * 16, Q + (ok ? (tb + row) * q_ld + q_col0 + j0 + ch * 8 : 0), ok);
    }
    wg_commit();
  };

  float acc[2][4];
#pragma unroll
  for (int nb = 0; nb < 2; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[nb][e] = 0.f;

  if (n_chunks > 0) issue(0, 0);
  for (int c = 0; c < n_chunks; ++c) {
    const int st = c & 1;
    if (c + 1 < n_chunks) issue(c + 1, st ^ 1);
    if (c + 1 < n_chunks) wg_wait<1>(); else wg_wait<0>();
    __syncthreads();
    const uint32_t pbase = smem_u32(ps[st]), qbase = smem_u32(qs[st]);
#pragma unroll
    for (int ks = 0; ks < kTok / 16; ++ks) {
      // A = Ps[16 tokens][this warp's 16 features]^T : matrices (tok 0:8, feat 0:8), (tok 0:8, feat 8:16), (tok 8:16, feat 0:8),
      // (tok 8:16, feat 8:16) -> a0..a3 of the m16n8k16 A fragment (rows = features, cols = tokens)
      uint32_t a[4], b[4];
      const int arow = ks * 16 + (lane & 7) + 8 * (lane >> 4);
      const int acol = warp * 16 + 8 * ((lane >> 3) & 1);
      wg_ldsm_x4_trans(pbase + (uint32_t)arow * kPRow + (uint32_t)acol * 2, a);
      // B = Qs[16 tokens][16 ranks]: matrices (tok 0:8, r 0:8), (tok 8:16, r 0:8), (tok 0:8, r 8:16), (tok 8:16, r 8:16)
      const int brow = ks * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
      const int bcol = 8 * (lane >> 4);
      wg_ldsm_x4_trans(qbase + (uint32_t)brow * kQRow + (uint32_t)bcol * 2, b);
      wg_mma<T>(acc[0], a, b[0], b[1]);
      wg_mma<T>(acc[1], a, b[2], b[3]);
    }
    __syncthreads();                                  // the stage is refilled by the next iteration's issue
  }
  // D fragment: c0,c1 = (row g, cols 2t, 2t+1), c2,c3 = (row g + 8, same cols); rows = features, cols = ranks
  const int g = lane >> 2, tq = lane & 3;
#pragma unroll
  for (int nb = 0; nb < 2; ++nb)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const long long mg = m0 + warp * 16 + g + (e >= 2 ? 8 : 0);
      const int j = nb * 8 + tq * 2 + (e & 1);
      if (mg >= M || j >= rc) continue;
      float* o = out + mg * so_m + (long long)(j0 + j) * so_r;
      if (gridDim.z == 1) *o += scale * acc[nb][e];
      else atomicAdd(o, scale * acc[nb][e]);
    }
}

}  // namespace

// The default (the GPU tests check it against the FMA kernel's result);
// CTS_WGRAD_MMA=0 selects the FMA kernel.
bool cts_lora_wgrad_mma_enabled() {
  const char* e = getenv("CTS_WGRAD_MMA");
  return !(e && e[0] == '0');
}

// preconditions of the vector / ldmatrix path; false -> the caller uses the FMA kernel
bool cts_lora_wgrad_mma_ok(const void* p, long long p_ld, long long p_col0, int p_il, long long m, const void* q, long long q_ld,
                           long long q_col0, int r) {
  if ((((uintptr_t)p) & 15) || (((uintptr_t)q) & 15)) return false;
  if (p_ld % 8 || q_ld % 8 || q_col0 % 8 || r % 8 || m % 8) return false;
  if (p_il == 0 ? (p_col0 % 8 != 0) : (m % 64 != 0)) return false;
  return true;
}

int cts_lora_wgrad_mma_launch(cts_ctx* ctx, const void* p, long long p_ld, long long p_col0, int p_il, long long m, const void* q,
                              long long q_ld, long long q_col0, int r, long long t, float scale, float* out, long long so_m,
                              long long so_r, int dtype, cudaStream_t st) {
  const long long tiles = cdiv_ll(m, kFeat) * cdiv_ll(r, kRank);
  long long splits = (4LL * ctx->sm_count) / tiles;
  const long long max_splits = cdiv_ll(t, 4 * kTok);               // at least 256 tokens per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits > 1024) splits = 1024;
  if (splits < 1) splits = 1;
  dim3 grid((unsigned)cdiv_ll(m, kFeat), (unsigned)cdiv_ll(r, kRank), (unsigned)splits);
  if (dtype == CTS_BF16) {
    CTS_CUDA(ctx, launch_pdl(lora_wgrad_mma_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, st, 1, (const __nv_bfloat16*)p, p_ld, p_col0,
                             p_il, m, (const __nv_bfloat16*)q, q_ld, q_col0, r, t, scale, out, so_m, so_r));
  } else {
    CTS_CUDA(ctx, launch_pdl(lora_wgrad_mma_kernel<__half>, grid, dim3(kThreads), 0, st, 1, (const __half*)p, p_ld, p_col0, p_il, m,
                             (const __half*)q, q_ld, q_col0, r, t, scale, out, so_m, so_r));
  }
  return CTS_OK;
}
