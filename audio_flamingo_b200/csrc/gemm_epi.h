// Epilogue flags and side-argument structs shared by the GEMM translation units (gemm_wgmma.cu) and
// the C ABI (af3_abi.cu); the flag values are the AF3_EPI_* constants of include/af3b200.h.
#pragma once
#include "common.h"

namespace af3 {

enum : int { EPI_BIAS = 1, EPI_GELU = 2, EPI_RESID = 4, EPI_SWIGLU = 8, EPI_F32OUT = 16, EPI_ROPE = 32,
              EPI_SWIGLU_CONCAT = 64 /* host-side only: weight rows are [gate; up], not interleaved (stripped before dispatch) */,
              EPI_XENT = 128 /* lm_head_xent only: softmax partials per (token, column tile), no output unless out != nullptr */ };

// rotary embedding + KV-cache append in the epilogue of the few-token fused q/k/v projection
struct RopeEpilogue {
    const float* cs;   // [n_tok][64] (cos, sin) pairs, bf16-rounded
    bf16* k_cache;
    bf16* v_cache;
    const int* pos;    // device int: cache slot of this step
    int H, Hkv, Tmax;
};

int gemm_bf16(cudaStream_t stream, const bf16* x, int ldx, const bf16* w, int ldw, void* out, int ldo, int n_tok,
              int n_feat, int K, int flags, const bf16* bias, const bf16* resid, int ld_res, int res_period,
              void* workspace, size_t workspace_bytes, const RopeEpilogue* rope);
size_t gemm_workspace_bytes();
// Block-scaled FP8 GEMM (include/af3b200.h af3_gemm_fp8): x e4m3 [n_tok, K] (pitch ldx bytes) with group scales
// sx [K/128][n_tok], w e4m3 [rows, K] (pitch ldw bytes) with weight_scale_inv sw [rows/128][K/128]
int gemm_fp8(cudaStream_t stream, const uint8_t* x, int ldx, const float* sx, const uint8_t* w, int ldw, const float* sw,
             void* out, int ldo, int n_tok, int n_feat, int K, int flags, const bf16* bias, const bf16* resid, int ld_res,
             void* workspace, size_t workspace_bytes, const RopeEpilogue* rope);
int quant_fp8(cudaStream_t stream, const bf16* x, int ldx, uint8_t* q, float* scales, int rows, int K);
// Group-wise int4 weights, bf16 activations (include/af3b200.h af3_gemm_w4a16 / af3_dequant_w4a16): w packed [rows, K/8]
// int32 (pitch ldw words), w_scale bf16 [rows, K/128] (pitch ld_scale); few-token GEMM only (n_tok <= 64)
int gemm_w4a16(cudaStream_t stream, const bf16* x, int ldx, const uint32_t* w, int ldw, const bf16* w_scale, int ld_scale, void* out,
               int ldo, int n_tok, int n_feat, int K, int flags, const bf16* bias, const bf16* resid, int ld_res, void* workspace,
               size_t workspace_bytes, const RopeEpilogue* rope);
int dequant_w4a16(cudaStream_t stream, const uint32_t* w, int ldw, const bf16* w_scale, int ld_scale, bf16* out, int rows, int K);
// LM head with the cross-entropy statistics in its epilogue (include/af3b200.h af3_lm_head_xent)
size_t lm_head_xent_scratch_bytes(int n_tok, int V);
int lm_head_xent(cudaStream_t stream, const bf16* x, int ldx, const bf16* w, int ldw, int n_tok, int V, int K, const int64_t* labels,
                 int64_t ignore_index, float* logits_out, int ldo, float* token_nll, double* totals, void* scratch);

}  // namespace af3
