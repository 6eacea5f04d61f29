// chatts_b200 -- the Value-Preserved Time-Series Encoder as ONE launch for the metric-sized prompt (north_star: "the TS encoder is a
// single fused kernel"): patchify + last-value pad + position-embedding gather (chatts_vllm.py:107-183) -> num_layers x
// [Linear (+ exact-erf GELU)] (chatts_vllm.py:83-91,186-188) -> rows scattered into the merged embedding sequence at the <ts>
// positions (chatts_vllm.py:569-573).  Up to 256 patch rows (8 series x 256 points = 128 rows at the BASELINE.json metric prompt).
//
// At that size the encoder is bound by the HBM stream of its 212 MB of weights (5 layers x 5120^2 bf16), and the multi-launch path
// (3 front-end + 5 GEMM + 5 split-K tail launches, 126 us = 0.27 of the HBM roof) pays a kernel boundary per stage.  Here:
//   * one persistent grid, (hidden/128 feature tiles) x (S K-splits), the S splits of a tile forming one thread-block CLUSTER;
//   * phase 0: the CTAs assemble the patch rows ([values | position embeddings], 16-byte vector stores) into rows_ws;
//   * per layer: swap-AB wgmma GEMM exactly as gemm_decode_fused.cu (weight tile = the 128-row MMA operand A streamed by TMA with
//     an evict-first hint, the patch rows = the MMA N dimension, accumulator [128 features x rows] fp32 in registers), the split's tile
//     parked in shared memory, reduced over DISTRIBUTED SHARED MEMORY in split order, bias + GELU applied, rows written as the next
//     layer's K-major operand (last layer: scattered through row_map into inputs_embeds);
//   * between layers a grid barrier (bounded spin -> trap, never a hang) -- and while a CTA waits there its TMA producer already
//     streams the first weight tiles of the NEXT layer into the idle ring (weights depend on nothing), so HBM does not idle.
// Rounding points are those of the multi-launch path (Linear output -> dtype, GELU on that, -> dtype); the K partition differs (S
// instead of the GEMM's own split factor), so results agree to fp32 summation order, not bit for bit.
#include <cooperative_groups.h>

#include <type_traits>

#include "common.cuh"
#ifndef CTS_DYN_SMEM
#define CTS_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#endif
#include "tensormap.cuh"
#include "trace.cuh"
#include "ts_rows.cuh"

namespace {

namespace cg = cooperative_groups;

// warps 0..7: two MMA warpgroups (the second one only for 256-row tiles: each holds 128 rows of the token tile), warp 8: TMA producer
constexpr int kBM = 128, kBK = 64, kThreads = 288, kMaxStages = 8;
constexpr int kTsMaxLayers = 6;

struct alignas(64) TsMaps {
  CUtensorMap w[kTsMaxLayers];     // W_l [hidden, K_l], box [64, 128]
  CUtensorMap x[3];                // 0: rows_ws [rows, in0]; 1, 2: activation ping-pong [rows, hidden]; box [64, BN]
};

struct TsFusedParams {
  // front end (chatts_vllm.py:107-183)
  const void* x; int row_len, nf, patch, mode, emb_dim, max_seq_len, in0, n_series;
  const void* pos_table; const int* valid_len; const int* row_offset; const int* max_valid;
  void* rows_ws;
  // MLP
  int num_layers, hidden, rows, split, stages;
  const void* bias[kTsMaxLayers];
  void* act[2];
  void* out; long long out_ld; const int* row_map;
  int* sync;                       // [0] grid-barrier arrivals (monotonic inside a launch), [1] exits (the last CTA resets both)
};

__device__ __forceinline__ int ld_acquire_gpu_i(const int* p) {
#ifdef CTS_HOST_SHIM
  shim_yield();
  return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#else
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ void fence_proxy_async_all_ts() {
#ifndef CTS_HOST_SHIM
  asm volatile("fence.proxy.async;" ::: "memory");
#endif
}

template <typename T, int BN>
__global__ void __launch_bounds__(kThreads, 1)
ts_encoder_fused_kernel(const __grid_constant__ TsMaps maps, const TsFusedParams p) {
  CTS_DYN_SMEM(smem_raw);
  __shared__ uint64_t full_bar[kMaxStages];
  __shared__ uint64_t empty_bar[kMaxStages];
  __shared__ int row_series_s;

  constexpr int kABytes = kBM * kBK * 2;
  constexpr int kStage = kABytes + BN * kBK * 2;
  constexpr bool kIsBf16 = std::is_same<T, __nv_bfloat16>::value;
  static_assert(BN == 64 || BN == 128 || BN == 256, "row tile");
  constexpr int kWN = BN > 128 ? 128 : BN;                  // token rows per MMA warpgroup
  constexpr int kWGs = BN / kWN;                           // MMA warpgroups

  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  float* part_s = reinterpret_cast<float*>(smem);          // [BN][128] fp32: reuses the (idle) pipeline ring once the accumulator is complete

  cg::cluster_group cluster = cg::this_cluster();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f0 = blockIdx.x * kBM;
  const int split = blockIdx.z, S = p.split, stages = p.stages, R = p.rows;
  const int G = (int)(gridDim.x * gridDim.z);
  const int cta = (int)(blockIdx.x + gridDim.x * blockIdx.z);
#ifdef CTS_HOST_SHIM      // tests/cuda_on_cpu runs a grid-barrier kernel as ONE big cluster (every CTA an OS thread): the K splits of this tile
  auto peer = [&](int s2) { return (unsigned)(blockIdx.x + gridDim.x * s2); };
#else
  auto peer = [&](int s2) { return (unsigned)s2; };           // cluster = (1, 1, S): rank = split index
#endif

  if (threadIdx.x == 0) {
    for (int l = 0; l < p.num_layers; ++l) tma_prefetch_desc(&maps.w[l]);
    for (int i = 0; i < 3; ++i) tma_prefetch_desc(&maps.x[i]);
    for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kWGs); }
    fence_mbar_init();
  }
  __syncthreads();

  // K range of this CTA's unit in layer l
  auto unit = [&](int l, int& kb0, int& nkb) {
    const int K = l == 0 ? p.in0 : p.hidden;
    const int kb_total = (K + kBK - 1) / kBK;
    kb0 = (int)(((long long)kb_total * split) / S);
    nkb = (int)(((long long)kb_total * (split + 1)) / S) - kb0;
  };
  // producer state (lane 0 of warp 8): global iteration counter over every K block of every layer; `pre` = weight tiles of the
  // current layer already requested before the grid barrier
  int it_p = 0, pre = 0;
  auto issue_weights = [&](int l, int kb0, int from, int upto) {
    for (int i = from; i < upto; ++i) {
      const int it = it_p + i;
      const int s = it % stages;
      mbar_wait(&empty_bar[s], (((uint32_t)(it / stages)) & 1u) ^ 1u);
      mbar_expect_tx(&full_bar[s], (uint32_t)kStage);
      tma_load_2d(smem + (size_t)s * kStage, &maps.w[l], &full_bar[s], (kb0 + i) * kBK, f0, CTS_L2_EVICT_FIRST);
    }
  };
  int n_bar = 0;
  auto grid_barrier = [&]() {
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_proxy_async_all_ts();
      __threadfence();
      atomicAdd(&p.sync[0], 1);
      const int target = G * (n_bar + 1);
      unsigned spins = 0;
      while (ld_acquire_gpu_i(&p.sync[0]) < target) {
#ifndef CTS_HOST_SHIM
        __nanosleep(20);
#endif
        if (++spins > (1u << 24)) {
          printf("chatts_b200: TS-encoder grid barrier %d timed out (cta %d of %d)\n", n_bar, cta, G);
          __trap();
        }
      }
      __threadfence();
      fence_proxy_async_all_ts();
    }
    __syncthreads();
    ++n_bar;
  };

  // No pdl_trigger() up front: a successor launched early would compete for the SMs this grid needs to be fully resident on.
  // The producer may still request layer 0's weight tiles before the dependency wait (nobody writes weights).
  int kb0, nkb;
  unit(0, kb0, nkb);
  if (warp == 8 && lane == 0) {
    CTS_TRACE(CTS_TK_OTHER, 0);
    pre = nkb < stages ? nkb : stages;
    issue_weights(0, kb0, 0, pre);
  }
  pdl_wait();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_OTHER, 1);

  // ------------------------------ phase 0: patch rows -> rows_ws [R, in0] ------------------------------
  {
    const T* xin = reinterpret_cast<const T*>(p.x);
    const T* ptab = reinterpret_cast<const T*>(p.pos_table);
    const float denom = (float)max(1, p.max_valid[0] - 1);
    const int chunks = p.in0 >> 3;
    for (int r = cta; r < R; r += G) {
      if (threadIdx.x == 0) {                               // series of row r: the last s with row_offset[s] <= r (binary search)
        int lo = 0, hi = p.n_series - 1;
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (p.row_offset[mid] <= r) lo = mid; else hi = mid - 1;
        }
        row_series_s = lo;
      }
      __syncthreads();
      const int s = row_series_s;
      const int vl = p.valid_len[s];
      const int p0 = (r - p.row_offset[s]) * p.patch;
      T* dst = reinterpret_cast<T*>(p.rows_ws) + (size_t)r * p.in0;
      for (int j = threadIdx.x; j < chunks; j += kThreads)
        *reinterpret_cast<uint4*>(dst + j * 8) =
            ts_row_chunk<T>(xin + (size_t)s * p.row_len, p.nf, p.patch, p.mode, ptab, p.emb_dim, p.max_seq_len, vl, p0, j * 8, denom);
      __syncthreads();                                      // row_series_s is rewritten by the next row
    }
  }
  grid_barrier();
  if (threadIdx.x == 0) CTS_TRACE(CTS_TK_OTHER, 4);       // rows assembled, layer 0 may start

  int it_c = 0;                                             // consumer (MMA) iteration counter, mirrors it_p
  for (int l = 0; l < p.num_layers; ++l) {
    unit(l, kb0, nkb);
    const CUtensorMap* tx = &maps.x[l == 0 ? 0 : 1 + ((l - 1) & 1)];
    if (warp == 8) {
      // ------------------------------ TMA producer ------------------------------
      if (lane == 0) {
        for (int i = 0; i < pre; ++i) {                     // token tiles of the stages whose weight tile is already on its way
          const int s = (it_p + i) % stages;
          tma_load_2d(smem + (size_t)s * kStage + kABytes, tx, &full_bar[s], (kb0 + i) * kBK, 0, CTS_L2_EVICT_LAST);
        }
        for (int i = pre; i < nkb; ++i) {
          const int it = it_p + i;
          const int s = it % stages;
          mbar_wait(&empty_bar[s], (((uint32_t)(it / stages)) & 1u) ^ 1u);
          mbar_expect_tx(&full_bar[s], (uint32_t)kStage);
          uint8_t* st = smem + (size_t)s * kStage;
          tma_load_2d(st, &maps.w[l], &full_bar[s], (kb0 + i) * kBK, f0, CTS_L2_EVICT_FIRST);
          tma_load_2d(st + kABytes, tx, &full_bar[s], (kb0 + i) * kBK, 0, CTS_L2_EVICT_LAST);
        }
        it_p += nkb;
        pre = 0;
        CTS_TRACE(CTS_TK_OTHER, 5);                         // this layer's last load requested
        // This CTA's stream of layer l is fully requested: pull ITS unit of layer l + 1 into L2 now (fire-and-forget), so HBM keeps
        // streaming through the drain, the cluster barrier, the DSMEM tail and the grid barrier; the prefetched lines are the ones
        // this CTA itself reads next, and nothing else streams meanwhile.
        if (l + 1 < p.num_layers) {
          int kb0n, nkbn;
          unit(l + 1, kb0n, nkbn);
          for (int i = 0; i < nkbn; ++i) tma_prefetch_l2_2d(&maps.w[l + 1], (kb0n + i) * kBK, f0);
        }
      }
    } else if (warp < 4 * kWGs) {
      // ------------------------------ MMA warpgroup(s) ------------------------------
      const int wg = warp >> 2;
      const bool wg_lead = (threadIdx.x & 127) == 0;
      Acc128<kWN> acc;
      acc.zero();
      for (int i = 0; i < nkb; ++i) {
        const int it = it_c + i;
        const int s = it % stages;
        mbar_wait(&full_bar[s], ((uint32_t)(it / stages)) & 1u);
        const uint32_t a_addr = smem_u32(smem + (size_t)s * kStage);
        acc.template mma_kblock<kIsBf16>(a_addr, a_addr + kABytes + wg * kWN * 128, i == 0);
        wgmma_wait<1>();
        if (i > 0 && wg_lead) mbar_arrive(&empty_bar[(it - 1) % stages]);
      }
      wgmma_wait<0>();
      if (nkb > 0 && wg_lead) mbar_arrive(&empty_bar[(it_c + nkb - 1) % stages]);
      it_c += nkb;
      if (threadIdx.x == 64) CTS_TRACE(CTS_TK_OTHER, 6);    // accumulator complete
      // ------------------------------ epilogue, part A: park this split's fp32 tile in shared memory ------------------------------
      named_bar_sync(1, 128 * kWGs);                        // every warp's MMAs are done with the ring
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < kWN / 2; ++i) {
          const int c = wg * kWN + acc_col(i);
          if (c < R) part_s[c * kBM + 64 * h + acc_row(i)] = acc.d[h][i];
        }
    } else {
      it_c += nkb;                                          // idle warps keep the (unused) counter in step
    }
    __syncthreads();
    cluster.sync();                                         // every split's tile is in its CTA's shared memory
    if (threadIdx.x == 64) CTS_TRACE(CTS_TK_OTHER, 7);

    if (warp >= 2 && warp < 6) {                          // the 128 threads part B is written for (et = 0..127)
      // ------------------------------ epilogue, part B: rows r = split, split + S, ...: reduce over DSMEM in split order, apply the tail ------------------------------
      // Work item = (one of this CTA's rows, 4 consecutive features): S 16-byte loads from the peers' parked tiles, issued for TWO items
      // before the first add (a scalar, one-row-at-a-time tail pays a DSMEM round trip per row), then bias + GELU on four values and
      // ONE 8-byte store.
      const int et = (int)threadIdx.x - 64;                  // 0..127
      const bool last = l + 1 == p.num_layers;
      const T* bias_p = reinterpret_cast<const T*>(p.bias[l]);
      T* dst_act = reinterpret_cast<T*>(p.act[l & 1]);
      const int n_my = R > split ? (R - split + S - 1) / S : 0;
      const int n_items = n_my * 32;
      constexpr int kBatch = 2;
      for (int it0 = et; it0 < n_items; it0 += 128 * kBatch) {
        float4 acc[kBatch];
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
          const int it = it0 + u * 128;
          acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (it < n_items) {
            const int r = split + S * (it >> 5), c4 = it & 31;
            float4 v[8];
#pragma unroll
            for (int s2 = 0; s2 < 8; ++s2)
              if (s2 < S) v[s2] = *reinterpret_cast<const float4*>(cluster.map_shared_rank(&part_s[r * kBM + c4 * 4], peer(s2)));
#pragma unroll
            for (int s2 = 0; s2 < 8; ++s2)                    // split order
              if (s2 < S) { acc[u].x += v[s2].x; acc[u].y += v[s2].y; acc[u].z += v[s2].z; acc[u].w += v[s2].w; }
          }
        }
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
          const int it = it0 + u * 128;
          if (it >= n_items) continue;
          const int r = split + S * (it >> 5), c4 = it & 31;
          const long long f = (long long)f0 + c4 * 4;
          if (f >= p.hidden) continue;                       // hidden % 8 == 0: a 4-feature chunk is entirely inside or outside
          float o[4] = {acc[u].x, acc[u].y, acc[u].z, acc[u].w};
          if (bias_p != nullptr) {
            const uint2 bv = *reinterpret_cast<const uint2*>(bias_p + f);
            const T* bp = reinterpret_cast<const T*>(&bv);
#pragma unroll
            for (int e = 0; e < 4; ++e) o[e] += DT<T>::to_f(bp[e]);
          }
          T ov[4];
          if (!last) {
#pragma unroll
            for (int e = 0; e < 4; ++e) ov[e] = DT<T>::from_f(gelu_erf(rnd<T>(o[e])));      // Linear output in the model dtype, exact-erf GELU on it (:87)
            *reinterpret_cast<uint2*>(dst_act + (long long)r * p.hidden + f) = *reinterpret_cast<const uint2*>(ov);
          } else {
            const int dr = p.row_map != nullptr ? p.row_map[r] : r;                        // the sp-mask scatter into the embedding sequence (:569-573)
#pragma unroll
            for (int e = 0; e < 4; ++e) ov[e] = DT<T>::from_f(o[e]);
            if (dr >= 0) *reinterpret_cast<uint2*>(reinterpret_cast<T*>(p.out) + (long long)dr * p.out_ld + f) = *reinterpret_cast<const uint2*>(ov);
          }
        }
      }
    }
    if (threadIdx.x == 64) CTS_TRACE(CTS_TK_OTHER, 8);      // tail done
    if (l + 1 < p.num_layers) {
      // The grid barrier doubles as the second cluster barrier: when it opens, every CTA has finished reading its peers' parked
      // tiles (so the rings may be refilled) and every row of this layer's output is written and visible to TMA.
      grid_barrier();
      if (threadIdx.x == 0) CTS_TRACE(CTS_TK_OTHER, 4);
    } else {
      __syncthreads();
      cluster.sync();                                       // nobody leaves while a peer still reads its parked tile
      if (threadIdx.x == 64) CTS_TRACE(CTS_TK_OTHER, 9);
    }
  }

  __syncthreads();
  pdl_trigger();
  if (threadIdx.x == 0) {
    CTS_TRACE(CTS_TK_OTHER, 3);
    __threadfence();
    if (atomicAdd(&p.sync[1], 1) == G - 1) {                // the last CTA to leave re-arms the counters for the next launch
      p.sync[0] = 0;
      p.sync[1] = 0;
      __threadfence();
    }
  }
}

template <typename T, int BN>
int launch_ts_fused(cts_ctx* ctx, const cts_ts_encode_args* a, int* sync, cudaStream_t stream) {
  const bool is_bf16 = a->dtype == CTS_BF16;
  TsMaps maps;
  memset(&maps, 0, sizeof(maps));
  int rc;
  for (int l = 0; l < a->num_layers; ++l) {
    const long long K = l == 0 ? a->in0 : a->hidden;
    rc = cts_make_tmap_2d(ctx, &maps.w[l], a->weights[l], a->hidden, K, K, kBM, is_bf16);
    if (rc) return rc;
  }
  for (int l = a->num_layers; l < kTsMaxLayers; ++l) maps.w[l] = maps.w[0];
  rc = cts_make_tmap_2d(ctx, &maps.x[0], a->rows_ws, a->total_rows, a->in0, a->in0, BN, is_bf16);
  if (rc) return rc;
  for (int i = 0; i < 2; ++i) {
    rc = cts_make_tmap_2d(ctx, &maps.x[1 + i], a->act_ws[i], a->total_rows, a->hidden, a->hidden, BN, is_bf16);
    if (rc) return rc;
  }
  TsFusedParams p;
  memset(&p, 0, sizeof(p));
  p.x = a->x; p.row_len = a->row_len; p.nf = a->num_features; p.patch = a->patch_size; p.mode = a->mode; p.emb_dim = a->emb_dim;
  p.max_seq_len = a->max_seq_len; p.in0 = a->in0; p.n_series = a->n_series;
  p.pos_table = a->pos_table; p.valid_len = a->valid_len; p.row_offset = a->row_offset; p.max_valid = a->max_valid;
  p.rows_ws = a->rows_ws;
  p.num_layers = a->num_layers; p.hidden = a->hidden; p.rows = (int)a->total_rows;
  for (int l = 0; l < a->num_layers; ++l) p.bias[l] = a->biases[l];
  p.act[0] = a->act_ws[0]; p.act[1] = a->act_ws[1];
  p.out = a->out; p.out_ld = a->out_ld; p.row_map = a->row_map;
  p.sync = sync;
  constexpr int kStage = kBM * kBK * 2 + BN * kBK * 2;
  constexpr int kPart = BN * kBM * 4;
  // two CTAs per SM when the parked tile allows it (BN <= 128: 3 x 32 KB ring >= the 64 KB tile), else one
  int stages = BN <= 128 ? 3 : 3;
  while (stages * kStage < kPart) ++stages;
  if (stages > kMaxStages) stages = kMaxStages;
  p.stages = stages;
  const size_t smem = (size_t)stages * kStage + 1024;
  auto kern = ts_encoder_fused_kernel<T, BN>;
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
#ifndef CTS_HOST_SHIM
  // without the maximum carve-out the driver may place only ONE CTA per SM
  CTS_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
#endif
  const int tiles = (int)cdiv_ll(a->hidden, kBM);
  // K splits per tile = cluster size: the largest S <= 8 for which ALL tiles' clusters are resident at once (the kernel synchronises
  // with grid barriers) -- asked of the driver for the real launch configuration (clusters must fit a GPC), not estimated
  const int kb_max = (int)cdiv_ll(a->hidden, kBK);
  int S = 0;
#ifdef CTS_HOST_SHIM
  S = kb_max < 4 ? kb_max : 4;
#else
  // The driver's cluster-occupancy query may count ONE CTA of this kernel per SM although two fit by every resource.  Sound bound from what the query does answer: the SMs that hold a cluster of c CTAs
  // at one CTA per SM hold a cluster of 2c at two per SM, so  clusters(2c at 2/SM) >= clusters(c at 1/SM).
  auto api_clusters = [&](int c) {
    cudaLaunchConfig_t q = {};
    q.gridDim = dim3((unsigned)tiles, 1, (unsigned)c);
    q.blockDim = dim3(kThreads);
    q.dynamicSmemBytes = smem;
    cudaLaunchAttribute qa[1];
    qa[0].id = cudaLaunchAttributeClusterDimension;
    qa[0].val.clusterDim.x = 1;
    qa[0].val.clusterDim.y = 1;
    qa[0].val.clusterDim.z = (unsigned)c;
    q.attrs = qa;
    q.numAttrs = 1;
    int n = 0;
    return cudaOccupancyMaxActiveClusters(&n, kern, &q) == cudaSuccess ? n : 0;
  };
  int per_sm_api = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_api, kern, kThreads, smem);
  cudaFuncAttributes fattr;
  CTS_CUDA(ctx, cudaFuncGetAttributes(&fattr, kern));
  const long long smem_cta = (long long)smem + (long long)fattr.sharedSizeBytes + 1024;
  const long long regs_cta = (long long)((fattr.numRegs + 7) / 8 * 8) * kThreads;
  const bool two_fit = per_sm_api >= 2 || (2 * smem_cta <= 227LL * 1024 && 2 * regs_cta <= 65536 && 2 * kThreads <= 2048);
  for (int cand = 8; cand >= 1 && S == 0; --cand) {
    if (cand > kb_max) continue;
    if (api_clusters(cand) >= tiles) { S = cand; break; }
    if (per_sm_api < 2 && two_fit && cand % 2 == 0 && api_clusters(cand / 2) >= tiles) S = cand;
  }
  (void)cudaGetLastError();
  if (const char* dbg = getenv("CTS_TS_FUSED_DEBUG")) {
    if (atoi(dbg) == 1) {
      int per_sm = -1;
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem);
      cudaFuncAttributes fa;
      cudaFuncGetAttributes(&fa, kern);
      fprintf(stderr, "[ts_fused] BN=%d smem dyn %zu static %zu regs %d: blocks/SM (api) %d, chosen split %d, tiles %d\n", BN, smem,
              (size_t)fa.sharedSizeBytes, fa.numRegs, per_sm, S, tiles);
      for (int cand = 8; cand >= 1; --cand) {
        cudaLaunchConfig_t q = {};
        q.gridDim = dim3((unsigned)tiles, 1, (unsigned)cand);
        q.blockDim = dim3(kThreads);
        q.dynamicSmemBytes = smem;
        cudaLaunchAttribute qa[1];
        qa[0].id = cudaLaunchAttributeClusterDimension;
        qa[0].val.clusterDim.x = 1; qa[0].val.clusterDim.y = 1; qa[0].val.clusterDim.z = (unsigned)cand;
        q.attrs = qa; q.numAttrs = 1;
        int n_clusters = -1;
        cudaError_t e = cudaOccupancyMaxActiveClusters(&n_clusters, kern, &q);
        fprintf(stderr, "[ts_fused]   cluster %d: max active clusters %d (%s)\n", cand, n_clusters, cudaGetErrorString(e));
      }
      (void)cudaGetLastError();
    }
  }
  if (const char* fs = getenv("CTS_TS_FUSED_SPLIT")) {          // experiment switch: a split the grid cannot hold traps at the first barrier
    const int f = atoi(fs);
    if (f >= 1 && f <= 8 && f <= kb_max) S = f;
  }
#endif
  if (S < 1) return cts_set_error(ctx, CTS_ERR_UNSUPPORTED, "cts_ts_encode_fused: %d feature tiles cannot all be resident", tiles);
  p.split = S;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)tiles, 1, (unsigned)S);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  // Co-residency of the whole grid (it synchronises with grid barriers): the driver was asked above how many clusters of this
  // configuration are resident at once and S was chosen so that ALL of them are; the kernel triggers its programmatic successor
  // only when it is done, so nothing launched later can take its SMs, and a predecessor that still holds some drains on its own.
  // CTS_TS_FUSED_COOP=1 adds the cooperative-launch attribute (the same guarantee enforced by the driver) instead of the
  // programmatic one -- kept as an A/B switch because the two attributes are not documented to combine.
#ifdef CTS_HOST_SHIM
  shim_next_launch_whole_grid();                           // tests/cuda_on_cpu: every CTA of this grid must be live at once (grid barriers)
#endif
  cudaLaunchAttribute attr[2];
  const char* coop = getenv("CTS_TS_FUSED_COOP");
  if (coop && atoi(coop) == 1) {
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
  } else {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
  }
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = 1;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = (unsigned)S;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  CTS_CUDA(ctx, cudaLaunchKernelEx(&cfg, kern, maps, p));
  return CTS_OK;
}

}  // namespace

// 1 when cts_ts_encode_fused can take this problem (else the caller uses the multi-launch path)
extern "C" int cts_ts_encode_fused_ok(const cts_ts_encode_args* a) {
  if (!a) return 0;
  return a->total_rows >= 1 && a->total_rows <= 256 && a->num_layers >= 1 && a->num_layers <= kTsMaxLayers && a->hidden % 8 == 0 &&
         a->hidden >= 64 && a->in0 % 8 == 0 && a->in0 >= 8 && (a->mode != 1 || a->pos_table != nullptr) && a->n_series >= 1;
}

// The fused encoder: ONE launch for patchify + MLP + row scatter.  Inputs as cts_ts_encode, but the count stage must have run
// (valid_len, row_offset, max_valid are INPUTS here: the host needs the counts before it can size the merged sequence anyway).
extern "C" int cts_ts_encode_fused(cts_ctx* ctx, const cts_ts_encode_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr && a->weights && a->biases && a->x, "null args / weight tables / x");
  CTS_CHECK_ARG(ctx, cts_ts_encode_fused_ok(a), "shape outside the fused kernel's range (1..256 rows, <= 6 layers, hidden % 8 == 0, in0 % 8 == 0)");
  CTS_CHECK_ARG(ctx, a->valid_len && a->row_offset && a->max_valid, "the count stage's outputs are inputs here");
  CTS_CHECK_ARG(ctx, a->rows_ws && a->act_ws[0] && a->act_ws[1] && a->out, "null workspace / out");
  CTS_CHECK_ARG(ctx, a->dtype == CTS_BF16 || a->dtype == CTS_F16, "dtype");
  CTS_CHECK_ARG(ctx, ctx->scratch != nullptr, "context scratch missing");
  int* sync = reinterpret_cast<int*>(ctx->scratch);
  cudaStream_t st = (cudaStream_t)stream;
#define TS_GO(TT)                                                                  \
  if (a->total_rows <= 64) return launch_ts_fused<TT, 64>(ctx, a, sync, st);       \
  if (a->total_rows <= 128) return launch_ts_fused<TT, 128>(ctx, a, sync, st);     \
  return launch_ts_fused<TT, 256>(ctx, a, sync, st);
  if (a->dtype == CTS_BF16) { TS_GO(__nv_bfloat16) }
  TS_GO(__half)
#undef TS_GO
}

CTS_TRACE_SETTER(cts_trace_set_ts_fused)
