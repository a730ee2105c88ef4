// extern "C" surface of libaf3b200.so (declared in include/af3b200.h).  Plain pointers and sizes only.
#include "../../include/af3b200.h"

#include "common.h"
#include "gemm_epi.h"

namespace af3 {
const char* last_error_cstr();
int rotary_time(cudaStream_t stream, bf16* x, const float* ts, const float* inv_freq, int W, int T, int dim, int n_freq,
                float window_duration, float max_len);
int gated_residual(cudaStream_t stream, const bf16* resid, const bf16* y, const bf16* alpha, int alpha_scalar, const int* row_gate,
                   bf16* out, int rows, int dim);
int token_step(cudaStream_t stream, const int64_t* raw_ids, int B, int* unfinished, const int64_t* eos, const int64_t* ctl,
               int64_t* tok_buf, int cap, int* gen_idx, int64_t* ids_out, int* done_flags);
int rope_table(cudaStream_t stream, float* cs, int B, int D, const int* pos_dev, const int* kv_start, const float* inv_freq);
int trace_begin(void* buf, size_t bytes);
int trace_end();
int trace_seq();
int logmel(cudaStream_t stream, const float* wave, int n_win, int n_samples, const float* hann, const float* table,
           const float* filt, const int* klo, const int* khi, float* out, int* win_max);
int layernorm(cudaStream_t, const bf16*, bf16*, const bf16*, const bf16*, int, int, float);
int avgpool_layernorm(cudaStream_t, const bf16*, bf16*, const bf16*, const bf16*, int, int, int, float);
int rmsnorm(cudaStream_t, const bf16*, bf16*, const bf16*, int, int, float, const int*);
int im2col_conv1(cudaStream_t, const void*, int, bf16*, int, int, int);
int im2col_conv2(cudaStream_t, const bf16*, bf16*, int, int, int);
int pack_gate_up(cudaStream_t, const bf16*, const bf16*, bf16*, int, int);
int rope_kv_append(cudaStream_t, bf16*, bf16*, bf16*, int, int, int, int, int, int, int, const int*, const int*,
                   const float*);
int embed_scatter(cudaStream_t, const int64_t*, int, const bf16*, int, int64_t, const bf16*, int, int, const int*, bf16*,
                  int*, int*);
int argmax(cudaStream_t, const float*, int, int, int64_t*, void*);
size_t argmax_scratch_bytes(int B);
size_t logits_process_scratch_bytes(int B, int cap);
int logits_process_argmax(cudaStream_t, const float*, int, int, const int64_t*, const int64_t*, int, const int*, const int*, const float*, int,
                          float*, int64_t*, void*);
int attention(cudaStream_t stream, const bf16* q, int ldq, const bf16* k, const bf16* v, int ldk, int kv_layout,
              int Tk_pitch, bf16* out, int ldo, int B, int H, int Hkv, int D, int Tq, int Tk, float scale, int causal,
              const int* kv_len, const int* kv_start);
size_t decode_attention_scratch_bytes(int B, int H, int D, int Tmax);
int decode_attention(cudaStream_t stream, const bf16* qkv, const bf16* k_cache, const bf16* v_cache, bf16* out,
                     float* scratch, int B, int H, int Hkv, int D, int Tmax, const int* ctx_len, const int* kv_start,
                     float scale);
}  // namespace af3

using af3::bf16;
#define S(stream) reinterpret_cast<cudaStream_t>(stream)
#define B16(p) reinterpret_cast<const bf16*>(p)
#define B16M(p) reinterpret_cast<bf16*>(p)
#define AF3_EPI_ROPE_INTERNAL 32  // af3::EPI_ROPE: set only by the fused q/k/v entry points

extern "C" {

const char* af3_last_error(void) { return af3::last_error_cstr(); }
int af3_abi_version(void) { return 4; }
void af3_set_pdl(int enable) { af3::set_pdl(enable != 0); }
size_t af3_trace_slot_bytes(void) { return sizeof(unsigned long long) * af3::TRACE_CTAS * af3::TRACE_MARKS; }
int af3_trace_begin(void* buf, size_t bytes) { return af3::trace_begin(buf, bytes); }
int af3_trace_end(void) { return af3::trace_end(); }
int af3_trace_seq(void) { return af3::trace_seq(); }

int af3_gemm_bf16(void* stream, const void* x, int ldx, const void* w, int ldw, void* out, int ldo, int n_tok, int n_feat,
                  int K, int flags, const void* bias, const void* resid, int ld_res, int res_period) {
    return af3::gemm_bf16(S(stream), B16(x), ldx, B16(w), ldw, out, ldo, n_tok, n_feat, K, flags, B16(bias), B16(resid),
                          ld_res, res_period, nullptr, 0, nullptr);
}

size_t af3_gemm_workspace_bytes(void) { return af3::gemm_workspace_bytes(); }

int af3_gemm_bf16_ws(void* stream, const void* x, int ldx, const void* w, int ldw, void* out, int ldo, int n_tok,
                     int n_feat, int K, int flags, const void* bias, const void* resid, int ld_res, int res_period,
                     void* workspace, size_t workspace_bytes) {
    return af3::gemm_bf16(S(stream), B16(x), ldx, B16(w), ldw, out, ldo, n_tok, n_feat, K, flags, B16(bias), B16(resid),
                          ld_res, res_period, workspace, workspace_bytes, nullptr);
}

int af3_rotary_time_emb(void* stream, void* x, const float* timestamps, const float* inv_freq, int W, int T, int dim, int n_freq,
                        float window_duration, float max_len) {
    return af3::rotary_time(S(stream), B16M(x), timestamps, inv_freq, W, T, dim, n_freq, window_duration, max_len);
}

int af3_gated_residual(void* stream, const void* resid, const void* y, const void* alpha, int alpha_is_scalar, const int* row_gate,
                       void* out, int rows, int dim) {
    return af3::gated_residual(S(stream), B16(resid), B16(y), B16(alpha), alpha_is_scalar, row_gate, B16M(out), rows, dim);
}

int af3_rope_table(void* stream, float* cs, int B, int D, const int* pos_dev, const int* kv_start, const float* inv_freq) {
    return af3::rope_table(S(stream), cs, B, D, pos_dev, kv_start, inv_freq);
}

int af3_gemm_qkv_rope(void* stream, const void* x, int ldx, const void* w, int ldw, const void* bias, void* q_out, int ldo,
                      int n_tok, int K, int H, int Hkv, int D, const float* rope_cs, void* k_cache, void* v_cache, int Tmax,
                      const int* pos_dev, void* workspace, size_t workspace_bytes) {
    if (D != 128) return af3::fail("af3_gemm_qkv_rope: head_dim must be 128");
    af3::RopeEpilogue r{rope_cs, B16M(k_cache), B16M(v_cache), pos_dev, H, Hkv, Tmax};
    return af3::gemm_bf16(S(stream), B16(x), ldx, B16(w), ldw, q_out, ldo, n_tok, (H + 2 * Hkv) * D, K,
                          AF3_EPI_BIAS | 32, B16(bias), nullptr, 0, 0, workspace, workspace_bytes, &r);
}

int af3_quant_fp8(void* stream, const void* x, int ldx, void* q, float* scales, int rows, int K) {
    return af3::quant_fp8(S(stream), B16(x), ldx, reinterpret_cast<uint8_t*>(q), scales, rows, K);
}

int af3_gemm_fp8(void* stream, const void* x, int ldx, const float* x_scales, const void* w, int ldw, const float* w_scale_inv,
                 void* out, int ldo, int n_tok, int n_feat, int K, int flags, const void* bias, const void* resid, int ld_res,
                 void* workspace, size_t workspace_bytes) {
    if (flags & AF3_EPI_ROPE_INTERNAL) return af3::fail("af3_gemm_fp8: use af3_gemm_qkv_rope_fp8 for the RoPE epilogue");
    return af3::gemm_fp8(S(stream), reinterpret_cast<const uint8_t*>(x), ldx, x_scales, reinterpret_cast<const uint8_t*>(w), ldw,
                         w_scale_inv, out, ldo, n_tok, n_feat, K, flags, B16(bias), B16(resid), ld_res, workspace, workspace_bytes,
                         nullptr);
}

int af3_gemm_qkv_rope_fp8(void* stream, const void* x, int ldx, const float* x_scales, const void* w, int ldw,
                          const float* w_scale_inv, const void* bias, void* q_out, int ldo, int n_tok, int K, int H, int Hkv, int D,
                          const float* rope_cs, void* k_cache, void* v_cache, int Tmax, const int* pos_dev, void* workspace,
                          size_t workspace_bytes) {
    if (D != 128) return af3::fail("af3_gemm_qkv_rope_fp8: head_dim must be 128");
    af3::RopeEpilogue r{rope_cs, B16M(k_cache), B16M(v_cache), pos_dev, H, Hkv, Tmax};
    return af3::gemm_fp8(S(stream), reinterpret_cast<const uint8_t*>(x), ldx, x_scales, reinterpret_cast<const uint8_t*>(w), ldw,
                         w_scale_inv, q_out, ldo, n_tok, (H + 2 * Hkv) * D, K, AF3_EPI_BIAS | AF3_EPI_ROPE_INTERNAL, B16(bias), nullptr,
                         0, workspace, workspace_bytes, &r);
}

size_t af3_lm_head_xent_scratch_bytes(int n_tok, int V) { return af3::lm_head_xent_scratch_bytes(n_tok, V); }
int af3_lm_head_xent(void* stream, const void* x, int ldx, const void* w, int ldw, int n_tok, int V, int K, const int64_t* labels,
                     int64_t ignore_index, float* logits_out, int ldo, float* token_nll, double* totals, void* scratch) {
    return af3::lm_head_xent(S(stream), B16(x), ldx, B16(w), ldw, n_tok, V, K, labels, ignore_index, logits_out, ldo, token_nll, totals,
                             scratch);
}

int af3_pack_gate_up(void* stream, const void* gate, const void* up, void* packed, int F, int K) {
    return af3::pack_gate_up(S(stream), B16(gate), B16(up), B16M(packed), F, K);
}

int af3_logmel(void* stream, const float* wave, int n_win, int n_samples, const float* hann, const float* dft_table,
               const float* mel_filters, const int* mel_klo, const int* mel_khi, float* out, int* scratch_max) {
    return af3::logmel(S(stream), wave, n_win, n_samples, hann, dft_table, mel_filters, mel_klo, mel_khi, out,
                       scratch_max);
}

int af3_im2col_conv1(void* stream, const void* in, int in_is_f32, void* cols, int n_win, int C, int T) {
    return af3::im2col_conv1(S(stream), in, in_is_f32, B16M(cols), n_win, C, T);
}
int af3_im2col_conv2(void* stream, const void* in, void* cols, int n_win, int C, int T) {
    return af3::im2col_conv2(S(stream), B16(in), B16M(cols), n_win, C, T);
}

int af3_layernorm(void* stream, const void* x, void* y, const void* gamma, const void* beta, int rows, int dim, float eps) {
    return af3::layernorm(S(stream), B16(x), B16M(y), B16(gamma), B16(beta), rows, dim, eps);
}
int af3_avgpool_layernorm(void* stream, const void* x, void* y, const void* gamma, const void* beta, int n_win, int T,
                          int dim, float eps) {
    return af3::avgpool_layernorm(S(stream), B16(x), B16M(y), B16(gamma), B16(beta), n_win, T, dim, eps);
}
int af3_rmsnorm(void* stream, const void* x, void* y, const void* weight, int rows, int dim, float eps,
                const int* row_idx) {
    return af3::rmsnorm(S(stream), B16(x), B16M(y), B16(weight), rows, dim, eps, row_idx);
}

int af3_attention(void* stream, const void* q, int ldq, const void* k, const void* v, int ldk, int kv_layout, int Tk_pitch,
                  void* out, int ldo, int B, int H, int Hkv, int D, int Tq, int Tk, float scale, int causal,
                  const int* kv_len, const int* kv_start) {
    return af3::attention(S(stream), B16(q), ldq, B16(k), B16(v), ldk, kv_layout, Tk_pitch, B16M(out), ldo, B, H, Hkv, D,
                          Tq, Tk, scale, causal, kv_len, kv_start);
}

int af3_rope_kv_append(void* stream, void* qkv, void* k_cache, void* v_cache, int B, int T, int H, int Hkv, int D,
                       int Tmax, int pos0, const int* pos0_dev, const int* kv_start, const float* inv_freq) {
    return af3::rope_kv_append(S(stream), B16M(qkv), B16M(k_cache), B16M(v_cache), B, T, H, Hkv, D, Tmax, pos0, pos0_dev,
                               kv_start, inv_freq);
}

size_t af3_decode_attention_scratch_bytes(int B, int H, int D, int Tmax) {
    return af3::decode_attention_scratch_bytes(B, H, D, Tmax);
}
int af3_decode_attention(void* stream, const void* qkv, const void* k_cache, const void* v_cache, void* out,
                         float* scratch, int B, int H, int Hkv, int D, int Tmax, const int* ctx_len,
                         const int* kv_start, float scale) {
    return af3::decode_attention(S(stream), B16(qkv), B16(k_cache), B16(v_cache), B16M(out), scratch, B, H, Hkv, D, Tmax,
                                 ctx_len, kv_start, scale);
}

int af3_embed_scatter(void* stream, const int64_t* ids, int n_tok, const void* embed_table, int dim,
                      int64_t audio_token_id, const void* audio_embeds, int n_win, int frames, const int* post_len,
                      void* out, int* scratch_rows, int* counts) {
    return af3::embed_scatter(S(stream), ids, n_tok, B16(embed_table), dim, audio_token_id, B16(audio_embeds), n_win,
                              frames, post_len, B16M(out), scratch_rows, counts);
}

int af3_token_step(void* stream, const int64_t* raw_ids, int B, int* unfinished, const int64_t* eos_ids, const int64_t* ctl, int64_t* tok_buf,
                   int cap, int* gen_idx, int64_t* ids_out, int* done_flags) {
    return af3::token_step(S(stream), raw_ids, B, unfinished, eos_ids, ctl, tok_buf, cap, gen_idx, ids_out, done_flags);
}
size_t af3_argmax_scratch_bytes(int B) { return af3::argmax_scratch_bytes(B); }
int af3_argmax(void* stream, const float* logits, int B, int V, int64_t* out_ids, void* scratch) {
    return af3::argmax(S(stream), logits, B, V, out_ids, scratch);
}
size_t af3_logits_process_scratch_bytes(int B, int cap) { return af3::logits_process_scratch_bytes(B, cap); }
int af3_logits_process_argmax(void* stream, const float* logits, int B, int V, const int64_t* prompt_ids, const int64_t* generated_ids,
                              int ld_ids, const int* gen_idx, const int* tables, const float* static_add, int cap, float* scores,
                              int64_t* out_ids, void* scratch) {
    return af3::logits_process_argmax(S(stream), logits, B, V, prompt_ids, generated_ids, ld_ids, gen_idx, tables, static_add, cap, scores,
                                      out_ids, scratch);
}

}  // extern "C"
