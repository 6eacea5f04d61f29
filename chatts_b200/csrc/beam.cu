// chatts_b200 -- beam search on the device: the selection step of transformers' GenerationMixin._beam_search and copy-on-write forks
// of the paged KV cache, so a beam-search step makes no host round trip.
//   cts_beam_select   one CTA per prompt: top `keep` continuations over the prompt's num_beams rows of per-row candidates (cts_logprobs
//                     top-k), the next running beams, the finished hypotheses, the early-stop heuristic, then the advance of every beam
//                     row (back-pointers, cur_ids / positions / seq_lens / slot_map, page-table row, fork descriptor)
//   cts_beam_fork_kv  copies the filled rows of a parent's old tail page into a child's new tail page, every layer, K and V
// Page rule: a page is written only while it is the tail of exactly one beam row.  Full pages are shared by reference; a child whose
// parent is another row gets a copy of the parent's partial tail in its spare page, and its old tail becomes its spare.
// Every score is plain IEEE fp32 (+ and / round to nearest; nothing to contract into an FMA), the arithmetic of transformers on the CPU.
#include "common.cuh"

namespace {

constexpr int kBsThreads = 256;
constexpr int kBsMaxKeep = 20;                       // the top-k limit of cts_logprobs
constexpr int kBsMaxBeams = kBsMaxKeep / 2;          // keep >= 2 * num_beams
constexpr int kBsMaxCand = kBsMaxBeams * kBsMaxKeep;
constexpr int kBsMaxEos = 16;
constexpr float kBsBig = -1.0e9f;                    // transformers' "very large negative" score

__global__ void __launch_bounds__(kBsThreads)
beam_select_kernel(int nb, int keep, long long vocab, const int* __restrict__ cand_ids, const float* __restrict__ cand_lp,
                   const int* __restrict__ eos_ids, int n_eos, const float* __restrict__ len_den, int max_new, int early_stopping,
                   float length_penalty, float* __restrict__ run_scores, float* __restrict__ fin_scores, int* __restrict__ fin_info,
                   int* __restrict__ prompt_flags, int* __restrict__ step_ptr, int* __restrict__ bp_tokens, int* __restrict__ bp_parents,
                   int* __restrict__ cur_ids, int* __restrict__ positions, int* __restrict__ seq_lens, int* __restrict__ slot_map,
                   int* __restrict__ page_table, int* __restrict__ page_table_old, const int* __restrict__ own_pages,
                   int* __restrict__ spare_pages, int max_pages, int page_size, int* __restrict__ fork) {
  pdl_trigger();
  pdl_wait();
  __shared__ float c_score[kBsMaxCand];
  __shared__ long long c_flat[kBsMaxCand];
  __shared__ float t_score[kBsMaxKeep], r_val[kBsMaxKeep];
  __shared__ int t_tok[kBsMaxKeep], t_beam[kBsMaxKeep], t_hit[kBsMaxKeep];
  __shared__ float m_val[kBsMaxBeams + kBsMaxKeep];
  __shared__ int m_info[kBsMaxBeams + kBsMaxKeep][4];
  __shared__ float old_run[kBsMaxBeams];
  __shared__ int sel[kBsMaxBeams], new_pos[kBsMaxBeams], eos_s[kBsMaxEos];
  const int b = blockIdx.x, tid = threadIdx.x, rows = gridDim.x * nb, row0 = b * nb;
  const int n = nb * keep;
  const int s = step_ptr[0];
  if (tid < nb) {
    old_run[tid] = run_scores[row0 + tid];
    new_pos[tid] = positions[row0 + tid] + 1;
  }
  if (tid < n_eos) eos_s[tid] = eos_ids[tid];
  __syncthreads();
  // ---- candidates: running score + the row's log-prob; ties go to the smaller flattened index beam * vocab + id
  if (tid < n) {
    const int j = tid / keep;
    const int id = cand_ids[(long long)(row0 + j) * keep + tid % keep];
    const float lp = cand_lp[(long long)(row0 + j) * keep + tid % keep];
    const bool valid = id >= 0 && id < vocab && lp == lp;
    c_score[tid] = valid ? old_run[j] + lp : -INFINITY;
    c_flat[tid] = valid ? (long long)j * vocab + id : (long long)nb * vocab + tid;
  }
  __syncthreads();
  if (tid < n) {
    const float v = c_score[tid];
    const long long f = c_flat[tid];
    int rank = 0;
    for (int u = 0; u < n; ++u) rank += c_score[u] > v || (c_score[u] == v && c_flat[u] < f);
    if (rank < keep) {
      t_score[rank] = v;
      t_tok[rank] = f < (long long)nb * vocab ? (int)(f % vocab) : -1;
      t_beam[rank] = (int)(f / vocab) < nb ? (int)(f / vocab) : 0;
    }
  }
  __syncthreads();
  // ---- stopping criteria of each kept candidate (EOS, max length); the running beams are the best num_beams that hit none
  if (tid < keep) {
    bool hit = s + 1 >= max_new;
    for (int e = 0; e < n_eos; ++e) hit |= t_tok[tid] == eos_s[e];
    t_hit[tid] = hit;
    r_val[tid] = hit ? t_score[tid] + kBsBig : t_score[tid];
  }
  __syncthreads();
  if (tid < keep) {
    const float v = r_val[tid];
    int rank = 0;
    for (int u = 0; u < keep; ++u) rank += r_val[u] > v || (r_val[u] == v && u < tid);
    if (rank < nb) sel[rank] = tid;
  }
  const bool done_before = prompt_flags[2 * b + 1] != 0;
  // ---- finished hypotheses: the top num_beams candidates that hit a criterion, length-penalised, merged into the num_beams best
  if (!done_before) {
    const bool unsat = prompt_flags[2 * b] != 0;
    bool full = early_stopping == 1;
    for (int i = 0; i < nb; ++i) full = full && fin_info[(long long)(row0 + i) * 4 + 3] != 0;
    if (tid < nb) {
      m_val[tid] = fin_scores[row0 + tid];
      for (int q = 0; q < 4; ++q) m_info[tid][q] = fin_info[(long long)(row0 + tid) * 4 + q];
    } else if (tid < nb + keep) {
      const int c = tid - nb;
      float q = t_score[c] / len_den[min(s + 1, max_new)];            // len_den has max_new + 1 entries
      if (full) q = q + kBsBig;
      if (!unsat) q = q + kBsBig;
      const bool did = t_hit[c] && c < nb;
      if (!did) q = q + kBsBig;
      m_val[tid] = q;
      m_info[tid][0] = s;
      m_info[tid][1] = row0 + t_beam[c];
      m_info[tid][2] = t_tok[c];
      m_info[tid][3] = did;
    }
    __syncthreads();
    if (tid < nb + keep) {
      const float v = m_val[tid];
      int rank = 0;
      for (int u = 0; u < nb + keep; ++u) rank += m_val[u] > v || (m_val[u] == v && u < tid);
      if (rank < nb) {
        fin_scores[row0 + rank] = v;
        for (int q = 0; q < 4; ++q) fin_info[(long long)(row0 + rank) * 4 + q] = m_info[tid][q];
      }
    }
    __syncthreads();
    if (tid == 0) {
      // _check_early_stop_heuristic and _beam_search_has_unfinished_sequences for this prompt
      const int best_len = (early_stopping == 2 && length_penalty > 0.f) ? max_new : s + 1;
      const float best = r_val[sel[0]] / len_den[best_len];
      float worst = INFINITY;
      bool all_fin = true, any_better = false, all_hit = true;
      for (int i = 0; i < nb; ++i) {
        worst = fminf(worst, fin_scores[row0 + i]);
        all_fin = all_fin && fin_info[(long long)(row0 + i) * 4 + 3] != 0;
      }
      for (int i = 0; i < nb; ++i) any_better |= best > (fin_info[(long long)(row0 + i) * 4 + 3] != 0 ? worst : kBsBig);
      for (int c = 0; c < keep; ++c) all_hit = all_hit && t_hit[c];
      const bool unsat_new = unsat && any_better;
      prompt_flags[2 * b] = unsat_new;
      prompt_flags[2 * b + 1] = !unsat_new || (early_stopping == 1 && all_fin) || all_hit;
    }
  }
  __syncthreads();
  // ---- page tables: the prompt's rows up to the tail column are read in full before any is rewritten
  int pmax = 0;
  for (int i = 0; i < nb; ++i) pmax = max(pmax, min(new_pos[i] / page_size, max_pages - 1));
  for (int e = tid; e < nb * (pmax + 1); e += kBsThreads) {
    const long long o = (long long)(row0 + e / (pmax + 1)) * max_pages + e % (pmax + 1);
    page_table_old[o] = page_table[o];
  }
  __syncthreads();
  for (int e = tid; e < nb * (pmax + 1); e += kBsThreads) {
    const int i = e / (pmax + 1), col = e % (pmax + 1);
    const int parent = row0 + t_beam[sel[i]];
    if (col < new_pos[i] / page_size) page_table[(long long)(row0 + i) * max_pages + col] = page_table_old[(long long)parent * max_pages + col];
  }
  if (tid < nb) {
    const int r = row0 + tid, c = sel[tid], parent = row0 + t_beam[c], pos = new_pos[tid];
    const int pg = pos / page_size, off = pos % page_size;
    int f_src = 0, f_dst = 0, f_n = 0, slot = -1;
    if (pg < max_pages) {
      int tail;
      if (off == 0) {
        tail = own_pages[(long long)r * max_pages + pg];                      // the new position opens a page: the row's own
      } else if (parent != r) {
        tail = spare_pages[r];                                                // copy-on-write into the spare; the old tail is the new spare
        spare_pages[r] = page_table_old[(long long)r * max_pages + pg];
        f_src = page_table_old[(long long)parent * max_pages + pg];
        f_dst = tail;
        f_n = off;
      } else {
        tail = page_table_old[(long long)r * max_pages + pg];
      }
      page_table[(long long)r * max_pages + pg] = tail;
      slot = tail * page_size + off;
    }
    fork[3 * r] = f_src;
    fork[3 * r + 1] = f_dst;
    fork[3 * r + 2] = f_n;
    if (s < max_new) {
      bp_tokens[(long long)s * rows + r] = t_tok[c];
      bp_parents[(long long)s * rows + r] = parent;
    }
    run_scores[r] = r_val[c];
    cur_ids[r] = t_tok[c] >= 0 ? t_tok[c] : 0;
    positions[r] = pos;
    seq_lens[r] = seq_lens[r] + 1;
    slot_map[r] = slot;
  }
  if (tid == 0) {
    __threadfence();
    const int arrived = atomicAdd(&step_ptr[1], 1) + 1;                       // step_ptr = {step, arrival counter}
    if (arrived == (int)gridDim.x) {
      step_ptr[1] = 0;
      step_ptr[0] = s + 1;
    }
  }
}

// grid (layers * 2 * nkv, rows): one (layer, K or V, kv head) slab of one forked row per CTA
__global__ void __launch_bounds__(128)
beam_fork_kv_kernel(unsigned short* __restrict__ kv, long long num_pages, int nkv, int page_size, int head_dim, const int* __restrict__ fork) {
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.y;
  const int n = fork[3 * r + 2];
  if (n <= 0) return;
  const long long lk = blockIdx.x / nkv, h = blockIdx.x % nkv;
  const long long page_elems = (long long)nkv * page_size * head_dim;
  unsigned short* base = kv + lk * num_pages * page_elems + h * page_size * head_dim;
  const unsigned short* src = base + (long long)fork[3 * r] * page_elems;
  unsigned short* dst = base + (long long)fork[3 * r + 1] * page_elems;
  const long long count = (long long)n * head_dim;
  if ((head_dim & 7) == 0) {
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    const long long c4 = count / 8;
    long long i = threadIdx.x;
    for (; i + 3 * 128 < c4; i += 4 * 128) {
      const uint4 a = __ldcs(s4 + i), bb = __ldcs(s4 + i + 128), c = __ldcs(s4 + i + 256), d = __ldcs(s4 + i + 384);
      d4[i] = a; d4[i + 128] = bb; d4[i + 256] = c; d4[i + 384] = d;
    }
    for (; i < c4; i += 128) d4[i] = __ldcs(s4 + i);
  } else {
    for (long long i = threadIdx.x; i < count; i += 128) dst[i] = src[i];
  }
}

}  // namespace

extern "C" int cts_beam_select(cts_ctx* ctx, int batch, int num_beams, int keep, long long vocab, const int* cand_ids,
                               const float* cand_logprobs, const int* eos_ids, int n_eos, const float* len_den, int max_new,
                               int early_stopping, float length_penalty, float* run_scores, float* fin_scores, int* fin_info,
                               int* prompt_flags, int* step_ptr, int* bp_tokens, int* bp_parents, int* cur_ids, int* positions,
                               int* seq_lens, int* slot_map, int* page_table, int* page_table_old, const int* own_pages, int* spare_pages,
                               int max_pages, int page_size, int* fork, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, batch >= 0 && batch <= 65535 && num_beams >= 1 && num_beams <= kBsMaxBeams, "batch / num_beams (1..10)");
  CTS_CHECK_ARG(ctx, keep >= 2 * num_beams && keep <= kBsMaxKeep, "keep must be in [2 * num_beams, 20]");
  CTS_CHECK_ARG(ctx, vocab >= keep && vocab <= (1LL << 24), "vocab must be in [keep, 2^24]");
  CTS_CHECK_ARG(ctx, n_eos >= 0 && n_eos <= kBsMaxEos && (n_eos == 0 || eos_ids != nullptr), "n_eos (0..16) / eos_ids");
  CTS_CHECK_ARG(ctx, max_new >= 1 && early_stopping >= 0 && early_stopping <= 2, "max_new / early_stopping (0 False, 1 True, 2 never)");
  CTS_CHECK_ARG(ctx, max_pages >= 1 && page_size >= 1, "max_pages / page_size");
  if (batch == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, cand_ids && cand_logprobs && len_den && run_scores && fin_scores && fin_info && prompt_flags && step_ptr &&
                         bp_tokens && bp_parents && cur_ids && positions && seq_lens && slot_map && page_table && page_table_old &&
                         own_pages && spare_pages && fork, "null pointer");
  CTS_CUDA(ctx, launch_pdl(beam_select_kernel, dim3((unsigned)batch), dim3(kBsThreads), 0, (cudaStream_t)stream, 1, num_beams, keep,
                           vocab, cand_ids, cand_logprobs, eos_ids, n_eos, len_den, max_new, early_stopping, length_penalty, run_scores,
                           fin_scores, fin_info, prompt_flags, step_ptr, bp_tokens, bp_parents, cur_ids, positions, seq_lens, slot_map,
                           page_table, page_table_old, own_pages, spare_pages, max_pages, page_size, fork));
  return CTS_OK;
}

extern "C" int cts_beam_fork_kv(cts_ctx* ctx, void* kv, int layers, long long num_pages, int nkv, int page_size, int head_dim,
                                const int* fork, int rows, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, layers >= 1 && num_pages >= 1 && nkv >= 1 && page_size >= 1 && head_dim >= 1, "cache shape");
  CTS_CHECK_ARG(ctx, (long long)layers * 2 * nkv <= 0x7fffffffLL && rows >= 0 && rows <= 65535, "layers * 2 * nkv / rows (<= 65535)");
  if (rows == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, kv != nullptr && fork != nullptr, "null kv / fork");
  CTS_CHECK_ARG(ctx, (reinterpret_cast<uintptr_t>(kv) & 15) == 0, "kv must be 16-byte aligned");
  CTS_CUDA(ctx, launch_pdl(beam_fork_kv_kernel, dim3((unsigned)(layers * 2 * nkv), (unsigned)rows), dim3(128), 0, (cudaStream_t)stream, 1,
                           (unsigned short*)kv, num_pages, nkv, page_size, head_dim, fork));
  return CTS_OK;
}
