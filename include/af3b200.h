/* libaf3b200.so -- C ABI of the H100-native (sm_90a) Audio Flamingo 3 audio->text hot path.
 *
 * Boundary (SURVEY.md 8-b): the reference path sits behind PyTorch nn.Module call conventions, not an FFI
 * registry, so there is no pre-existing binding to copy.  Each entry point below names the reference interface
 * it replaces ([O] = transformers 5.5.0, the executable statement of the AF3 path; see SURVEY.md section 0):
 *   AF3M = models/audioflamingo3/modeling_audioflamingo3.py   WFE = models/whisper/feature_extraction_whisper.py
 *   Q2M  = models/qwen2/modeling_qwen2.py                      GEN = generation/utils.py
 *   CACHE = cache_utils.py   SDPA = integrations/sdpa_attention.py   FP8 = integrations/finegrained_fp8.py
 *
 * Conventions: plain pointers and sizes only (no torch types); every pointer is a DEVICE pointer unless the
 * parameter name starts with h_; `stream` is a cudaStream_t passed as void*; all calls are asynchronous on
 * `stream`; return 0 on success, non-zero on error with a message available from af3_last_error() (thread
 * local).  No ownership transfer: outputs are written into caller-allocated buffers.  bf16 tensors are row-major with
 * the stated pitch.
 * State and threading (there is NO engine handle): every call launches on the CALLER'S CURRENT CUDA device, which must
 * be the device that owns all pointers of the call (cudaSetDevice first; per-device kernel attributes and SM counts
 * are cached per device ordinal, so several GPUs in one process work).  The process-wide switches af3_set_pdl and
 * af3_trace_begin/end are plain globals: drive the library from one launching thread per process (the reference's
 * host is single-threaded too, SURVEY.md 8-b).  Workspaces are caller-owned and must not be shared by concurrent
 * streams.
 */
#ifndef AF3B200_H
#define AF3B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* af3_last_error(void);
int af3_abi_version(void);

/* Programmatic dependent launch for subsequent launches of the decode-step kernels (GEMM, RMSNorm, RoPE, decode
 * attention, embedding gather, argmax): the next kernel's prologue and weight prefetch overlap the previous kernel's
 * tail; results are identical.  Process-wide switch, off by default. */
void af3_set_pdl(int enable);

/* In-graph timeline of the decode-step kernel chain (measurement aid; no reference counterpart).  Between
 * af3_trace_begin(buf, bytes) and af3_trace_end() every launch of a decode-step kernel (few-token GEMM, RMSNorm, rope
 * table, decode attention, embedding gather, argmax) is given the next slot of af3_trace_slot_bytes() bytes in `buf`
 * (device memory, zero-initialised by the caller) and its first 160 CTAs store %globaltimer there at 4 marks: entry,
 * after griddepcontrol.wait, main loop done, exit.  The slot address is a launch parameter, so a CUDA graph captured
 * while the trace is open keeps recording on every replay (the buffer holds the last replay).  af3_trace_seq() = slots
 * handed out so far; af3_trace_end() returns that count and stops handing out slots.  Process-wide, not thread-safe. */
size_t af3_trace_slot_bytes(void);
int af3_trace_begin(void* buf, size_t bytes);
int af3_trace_end(void);
int af3_trace_seq(void);

/* ---- epilogue flags for af3_gemm_bf16 ---- */
#define AF3_EPI_BIAS 1
#define AF3_EPI_GELU 2
#define AF3_EPI_RESID 4
#define AF3_EPI_SWIGLU 8
#define AF3_EPI_F32OUT 16
#define AF3_EPI_SWIGLU_CONCAT 64 /* with AF3_EPI_SWIGLU: w is [gate (n_feat rows); up (n_feat rows)], n_feat % 128 == 0 */

/* out[tok, feat] = epi( x[tok,:] . w[feat,:] ), wgmma tensor cores.  Replaces F.linear at
 * [O] AF3M:111-114,141,153-154,204-205,398-402; Q2M:41-48,199-202,474-475 and F.conv1d (as im2col GEMM) at
 * AF3M:343-344.  With AF3_EPI_SWIGLU, w holds gate/up rows interleaved in blocks of 128 (see af3_pack_gate_up) -- or, with
 * AF3_EPI_SWIGLU_CONCAT, simply concatenated [gate; up] (so the two nn.Linear weights can be views of one matrix) --
 * and out = silu(gate)*up with n_feat = intermediate size.  res_period > 0 adds resid[tok % res_period]. */
int af3_gemm_bf16(void* stream, const void* x, int ldx, const void* w, int ldw, void* out, int ldo, int n_tok,
                  int n_feat, int K, int flags, const void* bias, const void* resid, int ld_res, int res_period);

/* Same, with a caller-provided ZERO-INITIALISED device workspace of af3_gemm_workspace_bytes() bytes (reusable across
 * calls on one stream; the kernel leaves it zeroed where it matters).  With it, few-token GEMMs whose weight matrix
 * has too few 128-row tiles to fill the GPU (decode-step q/k/v, o and down projections) are split along K across
 * CTAs and reduced deterministically by the last-arriving CTA of each tile. */
size_t af3_gemm_workspace_bytes(void);
int af3_gemm_bf16_ws(void* stream, const void* x, int ldx, const void* w, int ldw, void* out, int ldo, int n_tok,
                     int n_feat, int K, int flags, const void* bias, const void* resid, int ld_res, int res_period,
                     void* workspace, size_t workspace_bytes);

/* gate [F,K], up [F,K] -> packed [2*ceil(F/128)*128, K]: per 128 features, 128 gate rows then 128 up rows. */
int af3_pack_gate_up(void* stream, const void* gate, const void* up, void* packed, int F, int K);

/* ---- FP8 decoder projections (block-scaled e4m3, the FineGrainedFP8 format of [O] FP8:793-865 with 128 x 128 weight
 * blocks).  ABI v4 gained these three entry points additively; nothing else changed.  Together they replace the
 * FP8Linear.forward calls ([O] FP8:248-284): activation quantization, block-scaled matmul, bias.
 *
 * Activation quantization rule (per token row and 128-column group): amax = max |x| in fp32 from the bf16 values,
 * s = amax / 448 (IEEE division, round to nearest), or s = 1 when amax == 0; q = e4m3(x / s) rounded to nearest even with
 * saturation -- what torch's (x.float() / s).to(torch.float8_e4m3fn) gives.
 * Scale layouts: activation scales are [K/128][rows] fp32 (group g of row t at scales[g * rows + t]); weight scales are
 * weight_scale_inv as stored by FineGrainedFP8, [w_rows/128][K/128] fp32 row-major.
 *
 * x bf16 [rows, K] (pitch ldx elements, 16-byte aligned) -> q e4m3 [rows, K] (pitch K bytes), scales [K/128][rows].
 * K % 128 == 0. */
int af3_quant_fp8(void* stream, const void* x, int ldx, void* q, float* scales, int rows, int K);

/* out[t, n] = epi( bf16( sum_kb (sum_{k in kb} x[t,k] w[n,k]) * x_scales[kb][t] * w_scale_inv[n/128][kb] ) ): each 128-wide
 * k-block's partial sum leaves the tensor-core accumulator and is scaled in fp32.  x e4m3 [n_tok, K] (pitch ldx bytes) with
 * x_scales from af3_quant_fp8 (n_tok rows); w e4m3 [n_feat, K] (pitch ldw bytes), or with AF3_EPI_SWIGLU |
 * AF3_EPI_SWIGLU_CONCAT the [gate (n_feat rows); up (n_feat rows)] concatenation.  flags: 0, AF3_EPI_BIAS (bias added to
 * the bf16 matmul result, then rounded again, as FP8Linear does), AF3_EPI_RESID (out = bf16(result + resid); out may alias
 * resid) or AF3_EPI_SWIGLU | AF3_EPI_SWIGLU_CONCAT.  K and n_feat % 128 == 0; out / resid 16-byte aligned with pitches that
 * are multiples of 8.  The workspace is that of af3_gemm_bf16_ws (split-K for few-token calls). */
int af3_gemm_fp8(void* stream, const void* x, int ldx, const float* x_scales, const void* w, int ldw, const float* w_scale_inv,
                 void* out, int ldo, int n_tok, int n_feat, int K, int flags, const void* bias, const void* resid, int ld_res,
                 void* workspace, size_t workspace_bytes);

/* FP8 counterpart of af3_gemm_qkv_rope: same outputs and cache writes, from the quantized x and the FP8 [q; k; v] weight. */
int af3_gemm_qkv_rope_fp8(void* stream, const void* x, int ldx, const float* x_scales, const void* w, int ldw,
                          const float* w_scale_inv, const void* bias, void* q_out, int ldo, int n_tok, int K, int H, int Hkv, int D,
                          const float* rope_cs, void* k_cache, void* v_cache, int Tmax, const int* pos_dev, void* workspace,
                          size_t workspace_bytes);

/* ---- Teacher-forced loss: the LM head with the cross-entropy of [O] loss/loss_utils.py ForCausalLMLoss ->
 * fixed_cross_entropy fused into its epilogue, without materialising the [n_tok, V] logits.  Additive (ABI v4).
 *
 * logits[t, v] = fp32(bf16( x[t,:] . w[v,:] )), the values af3_gemm_bf16 with AF3_EPI_F32OUT returns for n_tok > 64 (one
 * 128 x 128 token-major tile kernel whatever n_tok, so for n_tok <= 64 they may differ from the few-token kernel's by the
 * rounding of a different k order).  x bf16 [n_tok, K] (pitch ldx), w = lm_head.weight bf16 [V, K] (pitch ldw).
 * labels int64 [n_tok]: the label of every position, ALREADY SHIFTED as ForCausalLMLoss shifts them (labels padded with
 * ignore_index on the right and shifted left by one, or the caller's shift_labels).  A label is counted when it lies in
 * [0, V) and differs from ignore_index; a label outside [0, V) that is not ignore_index is never used as an index: it is
 * counted as ignored and reported (where the reference trips a device-side assert).
 * Outputs: token_nll fp32 [n_tok] = logsumexp(logits[t]) - logits[t, labels[t]] at counted positions, 0 elsewhere;
 * totals fp64 [3] = {sum of token_nll, counted positions, invalid labels}.  fixed_cross_entropy's loss is
 * totals[0] / totals[1] (reduction "mean"; NaN with no counted position) or totals[0] / num_items_in_batch ("sum").
 * logits_out (optional, fp32 [n_tok, V], pitch ldo >= V): the logits, stored by the same launch.
 * Run to run bit-identical, and independent of whether logits_out is given.  Three launches: the GEMM (per token and 128-column
 * tile: bf16-rounded values -> (max, sum exp(v - max)) in fp32; the tile holding the label column writes its logit), one warp
 * per token merging its partials in column-tile order (fp32 lse), and a one-CTA fixed-order fp64 reduction into totals.
 * scratch: af3_lm_head_xent_scratch_bytes(n_tok, V) = n_tok * (8 ceil(V / 128) + 4) bytes -- 237 MB at 24 960 tokens and
 * V = 152 064, against 15.2 GB of fp32 logits. */
size_t af3_lm_head_xent_scratch_bytes(int n_tok, int V);
int af3_lm_head_xent(void* stream, const void* x, int ldx, const void* w, int ldw, int n_tok, int V, int K, const int64_t* labels,
                     int64_t ignore_index, float* logits_out, int ldo, float* token_nll, double* totals, void* scratch);

/* Log-mel front end; replaces WhisperFeatureExtractor._torch_extract_fbank_features ([O] WFE:135-164).
 * wave fp32 [n_win, n_samples] (zero padded to 30 s by the caller as WFE:296 does), mel_filters fp32 [201,128]
 * (from audio_utils.mel_filter_bank, WFE:95-103) with the first/last non-zero bin of each filter in mel_klo/khi,
 * hann = torch.hann_window(400) (WFE:141), dft_table[n][k] = (cos, sin)(2 pi k n / 400) for n <= 200, k < 128.
 * out fp32 [n_win, 128, n_samples/160]. */
int af3_logmel(void* stream, const float* wave, int n_win, int n_samples, const float* hann /*[400]*/,
               const float* dft_table /*[201][128] (cos,sin) pairs*/, const float* mel_filters /*[201][128]*/,
               const int* mel_klo /*[128]*/, const int* mel_khi /*[128]*/, float* out, int* scratch_max /*[n_win]*/);

/* conv stem helpers (AF3M:343-344 as GEMMs): im2col with k=3, pad=1.
 * conv1: in [n_win, C, T] (fp32 or bf16 per in_is_f32) channel-major -> cols bf16 [n_win*T, 3*C], k index = kk*C+c
 * conv2: in bf16 [n_win*T, C] channel-last, stride 2 -> cols bf16 [n_win*(T/2), 3*C] */
int af3_im2col_conv1(void* stream, const void* in, int in_is_f32, void* cols, int n_win, int C, int T);
int af3_im2col_conv2(void* stream, const void* in, void* cols, int n_win, int C, int T);

/* LayerNorm over the last dim (AF3M:224,232 nn.LayerNorm eps 1e-5), bf16 in/out, fp32 statistics. */
int af3_layernorm(void* stream, const void* x, void* y, const void* gamma, const void* beta, int rows, int dim,
                  float eps);
/* AvgPool1d(2,2) over time then LayerNorm (AF3M:364-366): x [n_win*T, dim] -> y [n_win*(T/2), dim]. */
int af3_avgpool_layernorm(void* stream, const void* x, void* y, const void* gamma, const void* beta, int n_win, int T,
                          int dim, float eps);
/* Qwen2RMSNorm (Q2M:258-263): y = w * bf16(x * rsqrt(mean(x^2)+eps)); rows selected by optional row_idx. */
int af3_rmsnorm(void* stream, const void* x, void* y, const void* weight, int rows, int dim, float eps,
                const int* row_idx);

/* Bidirectional / causal softmax attention on wgmma (replaces SDPA:40-104 as called from AF3M:170-181 and
 * Q2M:227-238).  q rows come from a packed projection buffer: q[b, t, h*D + d] at q + (b*Tq + t)*ldq.
 * k, v: element (b, hk, t, d) at k + ((b*Hkv + hk)*Tk_pitch + t)*ldk + d  when kv_layout = 1 (cache layout), or
 * (b, t, hk*D + d) at k + (b*Tk + t)*ldk when kv_layout = 0 (packed projection buffer).
 * kv_len[b] (may be NULL = Tk): keys >= kv_len[b] are masked (AF3M:337-351 key padding).
 * kv_start[b] (may be NULL = 0): keys < kv_start[b] are masked (left padding, MASK:882).
 * causal: key j visible to query i iff j <= i + (Tk - Tq).   out[b, t, h*D + d] at out + (b*Tq + t)*ldo.
 * A query row with no visible key gets 0.  Rows at or past Tk are never read.  Masked keys inside a loaded 128-key tile
 * (before kv_start[b], at or past kv_len[b]) are read: K may hold anything there, but V must be finite, because the
 * tensor core multiplies it by P = 0 and 0 * NaN = NaN. */
int af3_attention(void* stream, const void* q, int ldq, const void* k, const void* v, int ldk, int kv_layout,
                  int Tk_pitch, void* out, int ldo, int B, int H, int Hkv, int D, int Tq, int Tk, float scale,
                  int causal, const int* kv_len, const int* kv_start);

/* Rotary embedding + KV-cache append (Q2M:100-146, CACHE:119-120).  qkv bf16 [n_tok, (H+2*Hkv)*D] in place on q;
 * k (rotated) and v are written to the cache [B, Hkv, Tmax, D] at position pos0 + t.  position id of token
 * (b, t) = pos0 + t - kv_start[b]  (GEN:719-721 cumsum(attention_mask)-1; padded slots get position 1 as
 * masked_fill_(mask == 0, 1) does).  pos0_dev (optional device int) overrides pos0 so a decode step can be replayed
 * from a CUDA graph.  inv_freq fp32 [D/2] = Qwen2RotaryEmbedding.inv_freq (Q2M:86-89). */
int af3_rope_kv_append(void* stream, void* qkv, void* k_cache, void* v_cache, int B, int T, int H, int Hkv, int D,
                       int Tmax, int pos0, const int* pos0_dev, const int* kv_start, const float* inv_freq);

/* Music Flamingo rotary time embedding (SURVEY 8-f.3; [O] musicflamingo/modular_musicflamingo.py:167-227) applied in place
 * to the AF-Whisper output x [W*T, dim] bf16: first 4*n_freq features rotated (window axis then time axis, interleaved
 * pairs) by angles built from timestamps [W, T] (seconds, fp32) and inv_freq [n_freq]; fp64 rotation, bf16 result. */
int af3_rotary_time_emb(void* stream, void* x, const float* timestamps, const float* inv_freq, int W, int T, int dim,
                        int n_freq, float window_duration, float max_len);

/* Flamingo-style gated residual, the element-wise half of a gated cross-attention / gated dense block (SURVEY 8-f.4; executable
 * analogue [O] transformers/models/idefics/modeling_idefics.py:796-806): out = resid + tanh(alpha) * y with the reference's bf16
 * rounding points.  alpha: bf16 [dim], or a single value when alpha_is_scalar.  row_gate (optional int32 [rows]): rows with gate 0
 * take y = 0 (tokens that attend to no media).  out may alias resid. */
int af3_gated_residual(void* stream, const void* resid, const void* y, const void* alpha, int alpha_is_scalar, const int* row_gate,
                       void* out, int rows, int dim);

/* Decode-step fusion of the q/k/v projection with RoPE and the KV append (Q2M:199-215 + CACHE:119-120 in one kernel):
 * out rows get the ROTATED query heads (columns [0, H*D)); rotated keys and the values go straight into the caches at
 * slot *pos_dev.  rope_cs [n_tok][D/2][2] fp32 from af3_rope_table (once per step, shared by all layers).
 * n_tok <= 64, D = 128, bias required (Qwen2 q/k/v have biases).  (ABI v4: RMSNorm fusion removed) */
int af3_gemm_qkv_rope(void* stream, const void* x, int ldx, const void* w, int ldw, const void* bias, void* q_out, int ldo,
                      int n_tok, int K, int H, int Hkv, int D, const float* rope_cs, void* k_cache, void* v_cache, int Tmax,
                      const int* pos_dev, void* workspace, size_t workspace_bytes);
int af3_rope_table(void* stream, float* rope_cs, int B, int D, const int* pos_dev, const int* kv_start,
                   const float* inv_freq);

/* Single-token attention over the KV cache (decode step; SDPA:40-104 with q_len = 1).  ctx_len is read from device
 * memory so the launch can live in a CUDA graph.  q at qkv (packed [B, (H+2Hkv)*D]); out [B, H*D].
 * scratch: af3_decode_attention_scratch_bytes() bytes, ZERO on first use (it holds the split arrival counters, which the
 * kernel leaves at zero).  Cache rows at or beyond ctx_len are read and multiplied by P = 0: they must hold finite values
 * (allocate the cache zero-initialised).  Requires ctx_len > kv_start[b] for every sequence. */
int af3_decode_attention(void* stream, const void* qkv, const void* k_cache, const void* v_cache, void* out,
                         float* scratch, int B, int H, int Hkv, int D, int Tmax, const int* ctx_len,
                         const int* kv_start, float scale);
size_t af3_decode_attention_scratch_bytes(int B, int H, int D, int Tmax);

/* Token embedding gather + audio-row scatter (AF3M:557, 563-566 masked_scatter).
 * ids int64 [n_tok]; audio rows taken in order from audio_embeds [n_win*frames, dim] keeping the first
 * post_len[w] frames of each window (AF3M:469-473).  out bf16 [n_tok, dim].  counts[0] = #audio tokens,
 * counts[1] = #valid audio rows (the caller raises if they differ, as masked_scatter would). */
int af3_embed_scatter(void* stream, const int64_t* ids, int n_tok, const void* embed_table, int dim,
                      int64_t audio_token_id, const void* audio_embeds, int n_win, int frames, const int* post_len,
                      void* out, int* scratch_rows /*[n_tok]*/, int* counts /*[2]*/);

/* Greedy step (GEN:2762-2800): argmax over fp32 logits [B, V] -> the first index of the row maximum.  Unlike torch.argmax,
 * which returns the index of a NaN, NaN entries are skipped; an all-NaN row yields 0.
 * scratch: af3_argmax_scratch_bytes(B) bytes of device memory (two-stage reduction). */
size_t af3_argmax_scratch_bytes(int B);
int af3_argmax(void* stream, const float* logits, int B, int V, int64_t* out_ids, void* scratch);

/* Greedy logits processors + selection in one pass over the logits: the chain [O] generation/utils.py:1037-1192
 * _get_logits_processor builds for greedy decoding, restated from [O] generation/logits_process.py -- SequenceBiasLogitsProcessor,
 * NoRepeatNGramLogitsProcessor, NoBadWordsLogitsProcessor, MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor,
 * ForcedEOSTokenLogitsProcessor, SuppressTokensLogitsProcessor, SuppressTokensAtBeginLogitsProcessor, in that order -- followed
 * by the selection of af3_argmax (first index of the processed row's maximum, NaNs skipped, an all -inf row yields 0).
 * The history the rules see is prompt_ids[b][0, S) followed by generated_ids[b][0, *gen_idx) (row pitch ld_ids for both), S
 * taken from the tables; every per-call quantity lives in device memory, so the call can be captured in a CUDA graph.
 * tables: int32 option tables written by audio_flamingo_b200.logits_process.compile_processors (header of 32 ints: S, n-gram
 * size, min_length, min_new_tokens, begin index, forced-EOS length, static flag, then counts and offsets of the EOS, begin-suppress,
 * forced-EOS, bad-word and sequence-bias records).  static_add fp32 [V]: every rule that depends on the token alone
 * (single-token bias, or -inf for single-token bad words and suppress_tokens); read only when the static flag is set.
 * cap: entries per row of the rule list (bounds the history-dependent hits).  scores (optional) fp32 [B, V] receives the
 * processed rows.  scratch: af3_logits_process_scratch_bytes(B, cap) bytes. */
size_t af3_logits_process_scratch_bytes(int B, int cap);
int af3_logits_process_argmax(void* stream, const float* logits, int B, int V, const int64_t* prompt_ids, const int64_t* generated_ids,
                              int ld_ids, const int* gen_idx, const int* tables, const float* static_add, int cap, float* scores,
                              int64_t* out_ids, void* scratch);

/* [O] generation/utils.py:2797-2805 (_sample, greedy): per generated token -- rows that have finished emit pad_token_id, the
 * token is appended, the unfinished mask is updated with the EOS set (EosTokenCriteria) and "every row finished" is published.
 * Device-side, so the whole token fits in the captured decode step.  raw_ids [B] (the argmax of the previous logits),
 * unfinished [B] (1 = running; updated), eos_ids [ctl[0]] ids, ctl = {number of EOS ids (0: no EOS handling), pad id},
 * tok_buf [B][cap] receives column *gen_idx, *gen_idx is advanced, ids_out [B] = the tokens fed to the next step,
 * done_flags[*gen_idx] = 1 iff EOS handling is on and no row is unfinished.  (ABI v3) */
int af3_token_step(void* stream, const int64_t* raw_ids, int B, int* unfinished, const int64_t* eos_ids, const int64_t* ctl, int64_t* tok_buf,
                   int cap, int* gen_idx, int64_t* ids_out, int* done_flags);

#ifdef __cplusplus
}
#endif
#endif
