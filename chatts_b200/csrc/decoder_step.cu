// chatts_b200 -- host-side executors of the C-ABI (no device code here): the whole decode step and two thin aliases
// that SURVEY.md 8(b) lists among the symbols the boundary must export.
//
//   cts_decoder_step : embed gather -> n_layers x [QKV GEMM -> bias/RoPE/KV write -> paged flash-decode -> o_proj GEMM ->
//                      +residual/RMSNorm -> gate_up GEMM -> SwiGLU -> down GEMM -> +residual/RMSNorm] -> lm_head -> greedy
//                      advance, enqueued on one stream by ONE C call (transformers qwen2/modeling_qwen2.py:269-310 per layer,
//                      chatts/vllm/chatts_vllm.py:595-610 for the call site and the logits) -- the same launches, in the same
//                      order, with the same split-K factors as chatts_b200/model.py:_decode_body makes through ~440 ctypes
//                      calls; capturable into a CUDA graph like them.  Every projection takes the split-K partial path (also
//                      when the factor is 1), whose reduce kernels round exactly where the fused epilogues do.
//   cts_rmsnorm      : Qwen2RMSNorm alone (modeling_qwen2.py:258-263)  = cts_reduce_residual_rmsnorm without partials
//   cts_lm_head      : logits = hidden @ lm_head^T (chatts_vllm.py:607-610) = cts_gemm, CTS_EPI_NONE
#include "common.cuh"

extern "C" int cts_rmsnorm(cts_ctx* ctx, const void* x, const void* w, float eps, void* out, long long t, long long h, int dtype,
                           void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, x && w && out, "null pointer");
  return cts_reduce_residual_rmsnorm(ctx, nullptr, 0, x, nullptr, w, eps, out, t, h, dtype, stream);
}

extern "C" int cts_lm_head(cts_ctx* ctx, const void* hidden, const void* w, void* logits, long long t, long long h, long long vocab,
                           int dtype, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  cts_gemm_args a;
  memset(&a, 0, sizeof(a));
  a.w = w; a.x = hidden; a.out = logits;
  a.n = vocab; a.k = h; a.t = t;
  a.w_ld = h; a.x_ld = h; a.out_ld = vocab;
  a.dtype = dtype; a.epilogue = CTS_EPI_NONE; a.split_k = 1;
  return cts_gemm(ctx, &a, stream);
}

// the weight the NEXT GEMM of the chain streams (L2 prefetch hint of cts_gemm_args, as chatts_b200/model.py passes it)
struct NextW { const void* w; long long n, k; int split; };

static int step_gemm_partial(cts_ctx* ctx, const void* x, const void* w, long long n, long long k, long long t, int split, float* ws,
                             int dtype, void* stream, NextW nx = NextW{nullptr, 0, 0, 0}) {
  cts_gemm_args a;
  memset(&a, 0, sizeof(a));
  a.w = w; a.x = x; a.out = ws;
  a.n = n; a.k = k; a.t = t;
  a.w_ld = k; a.x_ld = k; a.out_ld = n;
  a.dtype = dtype; a.epilogue = CTS_EPI_PARTIAL_F32; a.split_k = split;
  if (nx.w != nullptr && t <= 32 && ctx->next_prefetch_mb > 0) {
    a.next_w = nx.w; a.next_n = nx.n; a.next_k = nx.k; a.next_ld = nx.k; a.next_split = nx.split;
    a.next_prefetch_bytes = (long long)ctx->next_prefetch_mb << 20;
  }
  return cts_gemm(ctx, &a, stream);
}

extern "C" long long cts_decoder_step_ws_floats(const cts_decoder_step_args* a) {
  if (!a) return 0;
  const long long t = a->batch, H = a->hidden, I = a->inter, QKV = (long long)(a->nh + 2 * a->nkv) * a->head_dim;
  long long m = 1;
  const long long c[4] = {a->split_qkv * t * QKV, a->split_o * t * H, a->split_gu * t * 2 * I, a->split_d * t * H};
  for (int i = 0; i < 4; ++i) if (c[i] > m) m = c[i];
  return m;
}

extern "C" int cts_decoder_step(cts_ctx* ctx, const cts_decoder_step_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr && a->layers != nullptr, "null args / layers");
  CTS_CHECK_ARG(ctx, a->n_layers > 0 && a->batch > 0 && a->batch <= 128, "1 <= batch <= 128 (decode-sized step), n_layers > 0");
  CTS_CHECK_ARG(ctx, a->hidden > 0 && a->inter > 0 && a->inter % 64 == 0 && a->nh > 0 && a->nkv > 0 && a->head_dim > 0 && a->vocab > 0,
                "model shape");
  CTS_CHECK_ARG(ctx, a->split_qkv >= 1 && a->split_o >= 1 && a->split_gu >= 1 && a->split_d >= 1, "split factors must be >= 1");
  CTS_CHECK_ARG(ctx, a->embed && a->final_norm && a->lm_head && a->cos_tab && a->sin_tab, "null model tensor");
  CTS_CHECK_ARG(ctx, a->cur_ids && a->positions && a->seq_lens && a->slot_map && a->page_table, "null decode state");
  CTS_CHECK_ARG(ctx, a->h && a->xn && a->q && a->ao && a->act && a->logits && a->ws && a->attn_ws, "null activation buffer");
  CTS_CHECK_ARG(ctx, a->ws_floats >= cts_decoder_step_ws_floats(a), "split-K workspace too small (cts_decoder_step_ws_floats)");
  const long long T = a->batch, H = a->hidden, I = a->inter;
  const int nh = a->nh, nkv = a->nkv, d = a->head_dim, dt = a->dtype;
  const long long QKV = (long long)(nh + 2 * nkv) * d;
  const float scale = 1.0f / sqrtf((float)d);
  int rc;
#define STEP(call) do { rc = (call); if (rc != CTS_OK) return rc; } while (0)
  STEP(cts_embed_gather(ctx, a->embed, a->cur_ids, a->h, T, H, a->vocab_rows > 0 ? a->vocab_rows : a->vocab, dt, stream));
  STEP(cts_reduce_residual_rmsnorm(ctx, nullptr, 0, a->h, nullptr, a->layers[0].ln1, a->eps, a->xn, T, H, dt, stream));
  for (int l = 0; l < a->n_layers; ++l) {
    const cts_layer_weights* w = &a->layers[l];
    CTS_CHECK_ARG(ctx, w->wqkv && w->wo && w->wgu && w->wd && w->ln1 && w->ln2 && w->k_cache && w->v_cache, "null layer tensor");
    // QKV projection (+bias, +Qwen3 q/k norm) + RoPE + paged KV write
    STEP(step_gemm_partial(ctx, a->xn, w->wqkv, QKV, H, T, a->split_qkv, a->ws, dt, stream, NextW{w->wo, H, (long long)nh * d, a->split_o}));
    STEP(cts_qkv_rope_cache(ctx, a->ws, 1, a->split_qkv, w->bqkv, a->positions, a->cos_tab, a->sin_tab, a->slot_map, a->q, w->k_cache,
                            w->v_cache, nullptr, nullptr, T, nh, nkv, d, a->page_size, w->q_norm, w->k_norm, a->eps, dt, stream));
    STEP(cts_attn_decode(ctx, a->q, w->k_cache, w->v_cache, a->num_pages, a->page_table, a->max_pages, a->seq_lens, (int)T, nh, nkv, d,
                         a->page_size, scale, a->attn_splits, a->attn_ws, a->ao, dt, stream));
    // o_proj + residual + post-attention RMSNorm
    STEP(step_gemm_partial(ctx, a->ao, w->wo, H, (long long)nh * d, T, a->split_o, a->ws, dt, stream, NextW{w->wgu, 2 * I, H, a->split_gu}));
    STEP(cts_reduce_residual_rmsnorm(ctx, a->ws, a->split_o, a->h, a->h, w->ln2, a->eps, a->xn, T, H, dt, stream));
    // gate/up (interleaved weight) + SwiGLU
    STEP(step_gemm_partial(ctx, a->xn, w->wgu, 2 * I, H, T, a->split_gu, a->ws, dt, stream, NextW{w->wd, H, I, a->split_d}));
    STEP(cts_reduce_swiglu(ctx, a->ws, a->split_gu, T, I, a->act, 1, dt, stream));
    // down_proj + residual + the next layer's input RMSNorm (or the final norm)
    const void* nw = l + 1 < a->n_layers ? a->layers[l + 1].ln1 : a->final_norm;
    STEP(step_gemm_partial(ctx, a->act, w->wd, H, I, T, a->split_d, a->ws, dt, stream,
                           l + 1 < a->n_layers ? NextW{a->layers[l + 1].wqkv, QKV, H, a->split_qkv} : NextW{a->lm_head, a->vocab, H, 1}));
    STEP(cts_reduce_residual_rmsnorm(ctx, a->ws, a->split_d, a->h, a->h, nw, a->eps, a->xn, T, H, dt, stream));
  }
  STEP(cts_lm_head(ctx, a->xn, a->lm_head, a->logits, T, H, a->vocab, dt, stream));
  if (a->sample)
    STEP(cts_greedy_advance(ctx, a->logits, a->vocab, (int)T, a->out_tokens, a->out_ld, a->step_ptr, a->cur_ids, a->positions,
                            a->seq_lens, a->slot_map, a->page_table, a->max_pages, a->page_size, dt, stream));
#undef STEP
  return CTS_OK;
}

// cts_ts_encode: A3..A7 of the TS encoder from one C call (chatts_vllm.py:93-193 + the row scatter of :569-573): patch counts ->
// patchify -> num_layers x [wgmma GEMM (+ split-K tail) with bias / exact-erf GELU], the last layer scattering its rows
// through row_map into the embedding sequence.  `total_rows` (= sum of patch counts) is a HOST number: the caller sizes the
// merged sequence with it anyway (it comes from its own mask arithmetic or from a copy of cts_ts_patch_count's output).
// Same launches as chatts_b200/ts_encoder.py:TimeSeriesEmbedding.encode.
extern "C" int cts_ts_encode(cts_ctx* ctx, const cts_ts_encode_args* a, void* stream) {
  if (!ctx) return CTS_ERR_BAD_ARG;
  CTS_CHECK_ARG(ctx, a != nullptr && a->weights && a->biases, "null args / weight tables");
  CTS_CHECK_ARG(ctx, a->num_layers >= 1 && a->hidden > 0 && a->in0 > 0 && a->n_series >= 0 && a->total_rows >= 0, "shape");
  CTS_CHECK_ARG(ctx, a->valid_len && a->patch_cnt && a->row_offset && a->max_valid, "null metadata buffers");
  int rc;
#define STEP(call) do { rc = (call); if (rc != CTS_OK) return rc; } while (0)
  STEP(cts_ts_patch_count(ctx, a->x, a->dtype, a->n_series, a->row_len, a->num_features, a->patch_size, a->valid_len, a->patch_cnt,
                          a->row_offset, a->max_valid, stream));
  if (a->total_rows == 0 || a->n_series == 0) return CTS_OK;
  CTS_CHECK_ARG(ctx, a->rows_ws && a->act_ws[0] && a->act_ws[1] && a->out, "null workspace / out");
  if (cts_ts_encode_fused_ok(a) && !ctx->no_ts_fused) return cts_ts_encode_fused(ctx, a, stream);      // metric-sized prompts: ONE launch
  const int max_patches = (a->row_len / a->num_features + a->patch_size - 1) / a->patch_size;
  STEP(cts_ts_patchify(ctx, a->x, a->dtype, a->n_series, a->row_len, a->num_features, a->patch_size, a->mode, a->pos_table, a->emb_dim,
                       a->max_seq_len, a->valid_len, a->row_offset, a->max_valid, max_patches, a->rows_ws, a->in0, stream));
  const void* hcur = a->rows_ws;
  long long k = a->in0;
  for (int li = 0; li < a->num_layers; ++li) {
    const bool last = li == a->num_layers - 1;
    void* dst = last ? a->out : a->act_ws[li & 1];
    const long long dst_ld = last ? a->out_ld : a->hidden;
    const int* rmap = last ? a->row_map : nullptr;
    const int act = last ? CTS_EPI_NONE : CTS_EPI_GELU;
    const int split = cts_gemm_suggest_split(ctx, a->hidden, k, a->total_rows, 0);
    cts_gemm_args g;
    memset(&g, 0, sizeof(g));
    g.w = a->weights[li]; g.x = hcur;
    g.n = a->hidden; g.k = k; g.t = a->total_rows;
    g.w_ld = k; g.x_ld = k; g.dtype = a->dtype;
    if (split > 1) {
      CTS_CHECK_ARG(ctx, a->splitk_ws && a->splitk_floats >= (long long)split * a->total_rows * a->hidden, "split-K workspace too small");
      g.out = a->splitk_ws; g.out_ld = a->hidden; g.epilogue = CTS_EPI_PARTIAL_F32; g.split_k = split;
      STEP(cts_gemm(ctx, &g, stream));
      STEP(cts_reduce_bias_act(ctx, a->splitk_ws, split, a->total_rows, a->hidden, a->biases[li], act, dst, dst_ld, rmap, a->dtype, stream));
    } else {
      g.bias = a->biases[li]; g.out = dst; g.out_ld = dst_ld; g.row_map = rmap; g.epilogue = act; g.split_k = 1;
      STEP(cts_gemm(ctx, &g, stream));
    }
    hcur = dst;
    k = a->hidden;
  }
#undef STEP
  return CTS_OK;
}
