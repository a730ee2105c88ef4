"""H100-native Audio Flamingo 3 forward path behind the reference's PyTorch module surface.

Mirrors (class roles, forward/generate/get_audio_features signatures, state_dict key names) the executable
reference of this path, transformers 5.5.0 ([O], SURVEY.md 2.3):
    AudioFlamingo3Encoder                     [O] AF3M:265-379
    AudioFlamingo3MultiModalProjector         [O] AF3M:382-402
    Qwen2ForCausalLM / Qwen2Model             [O] Q2M:332-487
    AudioFlamingo3ForConditionalGeneration    [O] AF3M:410-592 (+ greedy loop GEN:2658-2812)
The nn.Module tree below only *holds* parameters under the reference's names (so `load_state_dict` of a reference
checkpoint works unchanged); no nn.Module.forward of torch is ever executed.  All arithmetic runs in the hand-written
sm_90a kernels of libaf3b200.so through audio_flamingo_b200.ops; this file is launch orchestration, buffer
management (torch caching allocator, current CUDA stream) and CUDA-graph capture of the decode step.
Compute dtype: bf16 parameters/activations, fp32 accumulation/statistics, fp32 logits -- same as running the
reference with model.to(torch.bfloat16).
"""
from __future__ import annotations

import functools
import math
import os
import time
from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn

from . import _lib, logits_process, ops
from ._lib import AF3Error

bf16 = torch.bfloat16

try:  # return types identical to the reference's when transformers is importable
    from transformers.modeling_outputs import BaseModelOutputWithPooling, CausalLMOutputWithPast
except Exception:  # pragma: no cover - minimal stand-ins with the same field names

    @dataclass
    class BaseModelOutputWithPooling:  # type: ignore
        last_hidden_state: torch.Tensor = None
        pooler_output: torch.Tensor = None

    @dataclass
    class CausalLMOutputWithPast:  # type: ignore
        loss: Optional[torch.Tensor] = None
        logits: torch.Tensor = None
        past_key_values: object = None

try:
    from transformers.generation.utils import GenerateDecoderOnlyOutput
except Exception:  # pragma: no cover

    @dataclass
    class GenerateDecoderOnlyOutput:  # type: ignore
        sequences: torch.Tensor = None
        scores: Optional[tuple] = None
        logits: Optional[tuple] = None
        attentions: Optional[tuple] = None
        hidden_states: Optional[tuple] = None
        past_key_values: object = None


@dataclass
class CausalLMOutputWithTokenLosses(CausalLMOutputWithPast):
    """CausalLMOutputWithPast plus `token_losses`, fp32 [B, S]: the per-position negative log-likelihood whose mean is `loss`
    (0 at ignored positions), so that candidates scored in one batch can be ranked by their row sums.  It is the last field:
    .loss / .logits / .past_key_values and the leading tuple entries are the reference's."""

    token_losses: Optional[torch.Tensor] = None


def prepare_loss_labels(labels, shift_labels, ignore_index, B, S, V):
    """The labels ForCausalLMLoss ([O] loss/loss_utils.py) compares the logits with: `labels` [B, S] padded with ignore_index
    on the right and shifted left by one, or the caller's `shift_labels` [B, S] as they are.  -> int64 [B * S] on the labels'
    device.  Integer [B, S] tensors only; host labels outside [0, V) other than ignore_index raise ValueError here (device
    labels are checked by the kernel, which ignores them, and reported at the end of the call)."""
    src = shift_labels if shift_labels is not None else labels
    name = "shift_labels" if shift_labels is not None else "labels"
    if not torch.is_tensor(src) or src.dtype.is_floating_point or src.dtype.is_complex or src.dtype == torch.bool:
        raise ValueError(f"{name} must be an integer tensor")
    if tuple(src.shape) != (B, S):
        raise ValueError(f"{name} must have shape {(B, S)}, got {tuple(src.shape)}")
    if isinstance(ignore_index, bool) or not isinstance(ignore_index, int):
        raise ValueError(f"ignore_index must be an int, got {ignore_index!r}")
    src = src.to(torch.int64)
    if shift_labels is None:
        src = torch.nn.functional.pad(src, (0, 1), value=ignore_index)[:, 1:]
    if not src.is_cuda:
        bad = (src != ignore_index) & ((src < 0) | (src >= V))
        if bool(bad.any()):
            raise ValueError(f"{name} must lie in [0, {V}) or equal ignore_index ({ignore_index}); got {src[bad][:4].tolist()}")
    return src.reshape(-1).contiguous()


def _on_model_device(fn):
    """Runs a public entry point with the model's GPU as the current CUDA device: the C ABI launches on the current device
    (include/af3b200.h), so a model living on cuda:1 must not launch on cuda:0 (ADVICE r01)."""

    @functools.wraps(fn)
    def wrapped(self, *args, **kwargs):
        dev = self.language_model.lm_head.weight.device
        if dev.type != "cuda":
            return fn(self, *args, **kwargs)  # _check_ready() raises the "no CPU fallback" error
        with torch.cuda.device(dev):
            return fn(self, *args, **kwargs)

    return wrapped


def _cfg_get(cfg, name, default=None):
    return getattr(cfg, name, default) if not isinstance(cfg, dict) else cfg.get(name, default)


# =====================================================================================================
# FP8 weights (FineGrainedFP8 layout, [O] integrations/finegrained_fp8.py:793-905, weight_block_size = (128, 128))
# =====================================================================================================
FP8_MAX = 448.0
DECODER_PROJECTIONS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj",
                       "mlp.up_proj", "mlp.down_proj")


def quantize_fp8_blocks(w):
    """Fp8Quantize.convert with 128 x 128 blocks: per-block amax, scale = 448 / amax in fp32 (1 for an all-zero block),
    q = e4m3(clamp(w * scale)), weight_scale_inv = 1 / scale.  w [rows, cols], both multiples of 128 -> (q, weight_scale_inv
    fp32 [rows / 128, cols / 128]).  Load-time only; runs wherever w lives."""
    rows, cols = w.shape
    blocks = w.to(torch.float32).reshape(rows // 128, 128, cols // 128, 128)
    amax = blocks.abs().amax(dim=(1, 3))
    scale = torch.where(amax > 0, FP8_MAX / torch.where(amax > 0, amax, torch.ones_like(amax)), torch.ones_like(amax))
    q = torch.clamp(blocks * scale[:, None, :, None], min=-FP8_MAX, max=FP8_MAX).to(torch.float8_e4m3fn)
    return q.reshape(rows, cols), (1.0 / scale).to(torch.float32)


def dequantize_fp8_blocks(q, scale_inv):
    """Fp8Dequantize: q [rows, cols] e4m3 times its block's weight_scale_inv, in fp32."""
    rows, cols = q.shape
    return (q.to(torch.float32).reshape(rows // 128, 128, cols // 128, 128) * scale_inv[:, None, :, None]).reshape(rows, cols)


# W4A16 weights (include/af3b200.h af3_gemm_w4a16): symmetric int4, one bf16 scale per row and 128 columns, 8 values per int32
W4_GROUP = 128


def quantize_w4a16(w):
    """w [rows, cols] (cols % 128 == 0) -> (weight_packed int32 [rows, cols / 8], weight_scale bf16 [rows, cols / 128]).
    s = bf16(amax / 7.5) per group (1 for an all-zero group), q = clamp(round_half_even(w / s), -8, 7) in fp32; bits 4j .. 4j+3
    of word i hold q[8i + j] + 8.  Load-time only; runs wherever w lives."""
    rows, cols = w.shape
    g = w.to(torch.float32).reshape(rows, cols // W4_GROUP, W4_GROUP)
    amax = g.abs().amax(-1)
    s = torch.where(amax > 0, amax / torch.full_like(amax, 7.5), torch.ones_like(amax)).to(bf16)
    q = torch.clamp(torch.round(g / s.to(torch.float32)[..., None]), -8, 7).to(torch.int32) + 8
    nib = q.to(torch.int64).reshape(rows, cols // 8, 8) << (4 * torch.arange(8, device=w.device, dtype=torch.int64))
    v = nib.sum(-1)  # the word as an unsigned 32-bit value; stored as the int32 with the same bits
    return torch.where(v >= (1 << 31), v - (1 << 32), v).to(torch.int32), s


def dequantize_w4a16(packed, scale):
    """Wd = bf16(q * s) [rows, cols] from weight_packed int32 [rows, cols / 8] and weight_scale bf16 [rows, cols / 128]."""
    rows, words = packed.shape
    q = (packed.to(torch.int64)[..., None] >> (4 * torch.arange(8, device=packed.device, dtype=torch.int64))) & 15
    q = (q - 8).reshape(rows, words * 8)
    return q.to(bf16) * scale.repeat_interleave(W4_GROUP, dim=1)


def _is_decoder_projection(key):
    """'language_model.model.layers.<i>.<proj>' for the seven FP8 projections of a decoder layer"""
    return key.startswith("language_model.model.layers.") and any(key.endswith("." + p) for p in DECODER_PROJECTIONS)


# =====================================================================================================
# parameter holders (names == reference state_dict keys)
# =====================================================================================================
class _EncAttn(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.k_proj = nn.Linear(d, d, bias=False)  # AF3M:111
        self.v_proj = nn.Linear(d, d)
        self.q_proj = nn.Linear(d, d)
        self.out_proj = nn.Linear(d, d)


class _EncLayer(nn.Module):
    def __init__(self, d, ffn):
        super().__init__()
        self.self_attn = _EncAttn(d)
        self.self_attn_layer_norm = nn.LayerNorm(d)
        self.fc1 = nn.Linear(d, ffn)
        self.fc2 = nn.Linear(ffn, d)
        self.final_layer_norm = nn.LayerNorm(d)


class AudioFlamingo3Encoder(nn.Module):
    """AF-Whisper tower: conv stem -> +positions -> N pre-LN layers -> AvgPool(2) -> LayerNorm ([O] AF3M:265-379)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        d = config.hidden_size
        self.d_model, self.n_heads, self.ffn = d, config.num_attention_heads, config.intermediate_size
        self.head_dim = d // self.n_heads
        if self.head_dim not in (64, 128):
            raise AF3Error("encoder head_dim must be 64 or 128 for the wgmma attention kernel")
        self.num_mel_bins = config.num_mel_bins
        self.max_source_positions = config.max_source_positions
        if _cfg_get(config, "activation_function", "gelu") != "gelu" or _cfg_get(config, "scale_embedding", False):
            raise AF3Error("only activation_function='gelu', scale_embedding=False (the AF3 configuration) is implemented")
        self.conv1 = nn.Conv1d(self.num_mel_bins, d, kernel_size=3, padding=1)
        self.conv2 = nn.Conv1d(d, d, kernel_size=3, stride=2, padding=1)
        self.embed_positions = nn.Embedding(self.max_source_positions, d)
        self.layers = nn.ModuleList([_EncLayer(d, self.ffn) for _ in range(config.num_hidden_layers)])
        self.layer_norm = nn.LayerNorm(d)
        self._packed = None

    # ---- weight packing (once per load): conv weights to im2col order, fused QKV with the 1/sqrt(d) query scale folded
    def pack_weights(self):
        s = self.head_dim ** -0.5  # power of two for 64/128: folding it into W_q, b_q is exact in bf16 (AF3M:142)
        P = {}
        P["w1"] = self.conv1.weight.detach().permute(0, 2, 1).reshape(self.d_model, -1).contiguous()
        P["w2"] = self.conv2.weight.detach().permute(0, 2, 1).reshape(self.d_model, -1).contiguous()
        P["layers"] = []
        for l in self.layers:
            a = l.self_attn
            wqkv = torch.cat([a.q_proj.weight.detach() * s, a.k_proj.weight.detach(), a.v_proj.weight.detach()], 0).contiguous()
            bqkv = torch.cat([a.q_proj.bias.detach() * s, torch.zeros_like(a.q_proj.bias), a.v_proj.bias.detach()], 0).contiguous()
            P["layers"].append((wqkv, bqkv))
        self._packed = P

    def _check_ready(self):
        p = self.conv1.weight
        if not p.is_cuda or p.dtype != bf16:
            raise AF3Error("model must be on a CUDA device in bfloat16 (model.to('cuda', torch.bfloat16)); no CPU fallback")
        if self._packed is None:
            self.pack_weights()

    def _get_feat_extract_output_lengths(self, input_lengths):
        input_lengths = (input_lengths - 1) // 2 + 1
        output_lengths = (input_lengths - 2) // 2 + 1
        return input_lengths, output_lengths

    @torch.no_grad()
    def _encode(self, input_features, input_features_mask):
        """-> ([W*T/2... pooled rows, d] bf16, W, pooled T)."""
        self._check_ready()
        P = self._packed
        W, C, T = input_features.shape
        if C != self.num_mel_bins:
            raise ValueError(f"expected {self.num_mel_bins} mel bins, got {C}")
        T2 = (T - 1) // 2 + 1
        if T2 != self.max_source_positions:
            raise ValueError(f"input_features must have {2 * self.max_source_positions} frames (got {T}); "
                             "positions are added over the full window as in the reference (AF3M:348)")
        d, H, hd = self.d_model, self.n_heads, self.head_dim
        kv_len = None
        if input_features_mask is not None:
            lens = (input_features_mask.sum(-1).to(torch.int32) - 1) // 2 + 1        # AF3M:338-339
            kv_len = lens.contiguous()
        x_in = input_features.contiguous()
        h1 = ops.linear(ops.im2col_conv1(x_in), P["w1"], self.conv1.bias, gelu=True)                    # AF3M:343
        x = ops.linear(ops.im2col_conv2(h1, W, T), P["w2"], self.conv2.bias, gelu=True,
                       resid=self.embed_positions.weight, res_period=T2)                               # AF3M:344-348
        del h1
        for l, (wqkv, bqkv) in zip(self.layers, P["layers"]):
            y = ops.layernorm(x, l.self_attn_layer_norm.weight, l.self_attn_layer_norm.bias)
            qkv = ops.linear(y, wqkv, bqkv)
            a = torch.empty((W, T2, d), device=x.device, dtype=bf16)
            ops.attention(qkv, qkv[:, d:], qkv[:, 2 * d:], a, B=W, H=H, Hkv=H, D=hd, Tq=T2, Tk=T2, scale=1.0, causal=False,
                          kv_layout=0, ldq=3 * d, ldk=3 * d, kv_len=kv_len)                             # AF3M:170-181
            ops.linear(a.view(W * T2, d), l.self_attn.out_proj.weight, l.self_attn.out_proj.bias, resid=x, out=x)
            y = ops.layernorm(x, l.final_layer_norm.weight, l.final_layer_norm.bias, out=y)
            f = ops.linear(y, l.fc1.weight, l.fc1.bias, gelu=True)
            ops.linear(f, l.fc2.weight, l.fc2.bias, resid=x, out=x)
        out = ops.avgpool_layernorm(x, W, T2, self.layer_norm.weight, self.layer_norm.bias)             # AF3M:364-366
        return out, W, T2 // 2

    def forward(self, input_features, input_features_mask=None, **kwargs):
        out, W, Tp = self._encode(input_features, input_features_mask)
        return BaseModelOutputWithPooling(last_hidden_state=out.view(W, Tp, self.d_model))


class AudioFlamingo3MultiModalProjector(nn.Module):
    """Linear -> GELU -> Linear ([O] AF3M:382-402)."""

    def __init__(self, audio_hidden, text_hidden, bias=True):
        super().__init__()
        if not bias:
            raise AF3Error("projector_bias=False is not implemented (AF3 uses bias, AF3C:102)")
        self.linear_1 = nn.Linear(audio_hidden, text_hidden)
        self.linear_2 = nn.Linear(text_hidden, text_hidden)

    @torch.no_grad()
    def forward(self, audio_features):
        shp = audio_features.shape
        x = audio_features.reshape(-1, shp[-1])
        h = ops.linear(x, self.linear_1.weight, self.linear_1.bias, gelu=True)
        y = ops.linear(h, self.linear_2.weight, self.linear_2.bias)
        return y.view(*shp[:-1], y.shape[-1])


class _DecAttn(nn.Module):
    def __init__(self, hid, H, Hkv, D):
        super().__init__()
        self.q_proj = nn.Linear(hid, H * D, bias=True)
        self.k_proj = nn.Linear(hid, Hkv * D, bias=True)
        self.v_proj = nn.Linear(hid, Hkv * D, bias=True)
        self.o_proj = nn.Linear(H * D, hid, bias=False)


class _DecMLP(nn.Module):
    def __init__(self, hid, inter):
        super().__init__()
        self.gate_proj = nn.Linear(hid, inter, bias=False)
        self.up_proj = nn.Linear(hid, inter, bias=False)
        self.down_proj = nn.Linear(inter, hid, bias=False)


class _RMSNormW(nn.Module):
    def __init__(self, hid):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hid))


class _DecLayer(nn.Module):
    def __init__(self, hid, inter, H, Hkv, D):
        super().__init__()
        self.self_attn = _DecAttn(hid, H, Hkv, D)
        self.mlp = _DecMLP(hid, inter)
        self.input_layernorm = _RMSNormW(hid)
        self.post_attention_layernorm = _RMSNormW(hid)


class _Qwen2Model(nn.Module):
    def __init__(self, tc):
        super().__init__()
        hid, H, Hkv = tc.hidden_size, tc.num_attention_heads, tc.num_key_value_heads
        D = _cfg_get(tc, "head_dim", None) or hid // H
        self.embed_tokens = nn.Embedding(tc.vocab_size, hid)
        self.layers = nn.ModuleList([_DecLayer(hid, tc.intermediate_size, H, Hkv, D) for _ in range(tc.num_hidden_layers)])
        self.norm = _RMSNormW(hid)


class AF3KVCache:
    """Pre-allocated KV cache [layers][B, Hkv, Tmax, D] (replaces DynamicCache's grow-by-cat, [O] CACHE:88-121).
    `length` = number of filled slots (host int); `pos_dev`/`ctx_dev` mirror it on the device for graph replay."""

    def __init__(self, n_layers, B, Hkv, Tmax, D, device):
        # zero-initialised: the decode attention kernel multiplies not-yet-written rows by P = 0 on the tensor cores
        self.k = torch.zeros((n_layers, B, Hkv, Tmax, D), device=device, dtype=bf16)
        self.v = torch.zeros_like(self.k)
        self.B, self.Tmax = B, Tmax
        self.length = 0
        # int32 [B]: left-padding length per sequence.  A persistent buffer (prefill copies into it) so that a captured decode
        # graph, which holds its address, stays valid when the cache is reused for the next prompt.
        self.kv_start = torch.zeros((B,), device=device, dtype=torch.int32)
        self.pos_dev = torch.zeros((1,), device=device, dtype=torch.int32)
        self.ctx_dev = torch.ones((1,), device=device, dtype=torch.int32)

    def reset(self):
        """Back to the state of a fresh cache (same buffers): rows are re-zeroed so that the kernels' invariant -- rows beyond the
        live context are finite -- never depends on what an earlier prompt left behind (two async memsets, ~0.5 ms at config 2)."""
        self.k.zero_()
        self.v.zero_()
        self.length = 0
        self.kv_start.zero_()
        self.pos_dev.zero_()
        self.ctx_dev.fill_(1)

    def get_seq_length(self, layer_idx=0):
        return self.length

    @staticmethod
    def bucket(n_rows: int) -> int:
        """Capacity is kept at multiples of 256 rows (one decode graph per bucket, see generate())."""
        return -(-max(int(n_rows), 1) // 256) * 256

    def ensure_capacity(self, n_rows: int):
        """Grow (re-allocate + copy the live rows) so that `n_rows` slots exist: what DynamicCache's grow-by-cat gives the
        reference's callers for free ([O] CACHE:119-120).  Only the eager forward() path grows a cache; generate() sizes it
        up front because a captured decode graph holds the buffers' addresses."""
        if n_rows <= self.Tmax:
            return
        new_T = self.bucket(n_rows)
        k = torch.zeros(self.k.shape[:3] + (new_T, self.k.shape[4]), device=self.k.device, dtype=bf16)
        v = torch.zeros_like(k)
        if self.length > 0:
            k[:, :, :, : self.length].copy_(self.k[:, :, :, : self.length])
            v[:, :, :, : self.length].copy_(self.v[:, :, :, : self.length])
        self.k, self.v, self.Tmax = k, v, new_T


class _Bf16Projections:
    """The four GEMMs of one decoder layer on bf16 weights (chosen once, at pack time)."""

    def __init__(self, lm, wqkv, bqkv, wo, wgu, wdown):
        self.lm, self.wqkv, self.bqkv, self.wo, self.wgu, self.wdown = lm, wqkv, bqkv, wo, wgu, wdown

    def qkv(self, y):
        return ops.linear(y, self.wqkv, self.bqkv)

    def qkv_rope(self, y, kc, vc, rope_cs, pos_dev):
        lm = self.lm
        return ops.qkv_rope_linear(y, self.wqkv, self.bqkv, kc, vc, H=lm.H, Hkv=lm.Hkv, D=lm.D, rope_cs=rope_cs, pos_dev=pos_dev)

    def o(self, a, h):
        ops.linear(a, self.wo, resid=h, out=h)

    def gate_up(self, y):
        return ops.swiglu_linear(y, self.wgu, self.lm.inter, concat=self.lm._swiglu_concat)

    def down(self, g, h):
        ops.linear(g, self.wdown, resid=h, out=h)


class _Fp8Projections:
    """The same four GEMMs on block-scaled e4m3 weights: every input is quantized (af3_quant_fp8) right before its GEMM.
    Each weight is a (e4m3 matrix, weight_scale_inv) pair."""

    def __init__(self, lm, wqkv, bqkv, wo, wgu, wdown):
        self.lm, self.wqkv, self.bqkv, self.wo, self.wgu, self.wdown = lm, wqkv, bqkv, wo, wgu, wdown

    def qkv(self, y):
        return ops.linear_fp8(ops.quant_fp8(y), *self.wqkv, self.bqkv)

    def qkv_rope(self, y, kc, vc, rope_cs, pos_dev):
        lm = self.lm
        return ops.qkv_rope_linear_fp8(ops.quant_fp8(y), *self.wqkv, self.bqkv, kc, vc, H=lm.H, Hkv=lm.Hkv, D=lm.D, rope_cs=rope_cs,
                                       pos_dev=pos_dev)

    def o(self, a, h):
        ops.linear_fp8(ops.quant_fp8(a), *self.wo, resid=h, out=h)

    def gate_up(self, y):
        return ops.swiglu_linear_fp8(ops.quant_fp8(y), *self.wgu, self.lm.inter)

    def down(self, g, h):
        ops.linear_fp8(ops.quant_fp8(g), *self.wdown, resid=h, out=h)


class _W4A16Projections:
    """The same four GEMMs on group-wise int4 weights, each a (weight_packed, weight_scale) pair.  Up to 64 tokens the
    W4A16 few-token GEMMs run; above that (prefill, decode with more than 64 sequences) af3_dequant_w4a16 writes the
    projection's Wd into the layer stack's one bf16 scratch and the bf16 GEMM runs on it, so those results are the bf16
    model's on Wd bit for bit."""

    def __init__(self, lm, wqkv, bqkv, wo, wgu, wdown):
        self.lm, self.wqkv, self.bqkv, self.wo, self.wgu, self.wdown = lm, wqkv, bqkv, wo, wgu, wdown

    def _wd(self, w):
        return ops.dequant_w4a16(*w, out=self.lm._w4_scratch)

    def qkv(self, y):
        if y.shape[0] <= 64:
            return ops.linear_w4a16(y, *self.wqkv, self.bqkv)
        return ops.linear(y, self._wd(self.wqkv), self.bqkv)

    def qkv_rope(self, y, kc, vc, rope_cs, pos_dev):
        lm = self.lm
        return ops.qkv_rope_linear_w4a16(y, *self.wqkv, self.bqkv, kc, vc, H=lm.H, Hkv=lm.Hkv, D=lm.D, rope_cs=rope_cs, pos_dev=pos_dev)

    def o(self, a, h):
        if a.shape[0] <= 64:
            ops.linear_w4a16(a, *self.wo, resid=h, out=h)
        else:
            ops.linear(a, self._wd(self.wo), resid=h, out=h)

    def gate_up(self, y):
        if y.shape[0] <= 64:
            return ops.swiglu_linear_w4a16(y, *self.wgu, self.lm.inter)
        return ops.swiglu_linear(y, self._wd(self.wgu), self.lm.inter, concat=True)

    def down(self, g, h):
        if g.shape[0] <= 64:
            ops.linear_w4a16(g, *self.wdown, resid=h, out=h)
        else:
            ops.linear(g, self._wd(self.wdown), resid=h, out=h)


class Qwen2ForCausalLM(nn.Module):
    """Decoder ([O] Q2M:332-487) on sm_90a kernels: RMSNorm, fused QKV GEMM (+bias), RoPE + in-place KV append,
    wgmma causal GQA attention (prefill) / split-KV decode attention, o GEMM (+residual), fused SwiGLU GEMM,
    down GEMM (+residual), final norm, LM head to fp32 logits."""

    def __init__(self, tc):
        super().__init__()
        self.config = tc
        self.hid, self.H, self.Hkv = tc.hidden_size, tc.num_attention_heads, tc.num_key_value_heads
        self.D = _cfg_get(tc, "head_dim", None) or self.hid // self.H
        if self.D != 128:
            raise AF3Error("decoder head_dim must be 128 (Qwen2.5-7B geometry) for the attention kernels")
        if _cfg_get(tc, "hidden_act", "silu") != "silu":
            raise AF3Error("only hidden_act='silu' is implemented")
        self.inter, self.vocab, self.eps = tc.intermediate_size, tc.vocab_size, tc.rms_norm_eps
        rp = _cfg_get(tc, "rope_parameters", None) or {}
        self.rope_theta = rp.get("rope_theta", _cfg_get(tc, "rope_theta", 10000.0))
        if rp.get("rope_type", "default") != "default":
            raise AF3Error("only default RoPE is implemented")
        self.model = _Qwen2Model(tc)
        self.lm_head = nn.Linear(self.hid, self.vocab, bias=False)
        self.quantization = None  # "fp8": the decoder projections hold e4m3 weights + weight_scale_inv (load_reference_state_dict);
        # "w4a16": they hold weight_packed + weight_scale instead of weight
        self._w4_scratch = None
        self._packed = None
        self._proj = None
        self._inv_freq = None

    def pack_weights(self):
        """Fused q/k/v and gate/up matrices for the kernels.  The nn.Linear parameters of the reference's module tree are then
        re-pointed at VIEWS of the fused matrices (same values, same state_dict): the decoder's projection weights exist once in HBM
        (round 1 kept the originals next to the packed copies, +8.5 GB), and an in-place update of a parameter updates what the
        kernels read.  gate/up need intermediate_size % 128 == 0 for the view trick ([gate; up] layout, AF3_EPI_SWIGLU_CONCAT);
        otherwise the 128-row interleaved copy of round 1 is used."""
        P = []
        HD, KD = self.H * self.D, self.Hkv * self.D
        self._swiglu_concat = self.inter % 128 == 0
        if self.quantization == "fp8":
            return self._pack_fp8()
        if self.quantization == "w4a16":
            return self._pack_w4a16()
        for l in self.model.layers:
            a, m = l.self_attn, l.mlp
            wqkv = torch.cat([a.q_proj.weight.detach(), a.k_proj.weight.detach(), a.v_proj.weight.detach()], 0).contiguous()
            bqkv = torch.cat([a.q_proj.bias.detach(), a.k_proj.bias.detach(), a.v_proj.bias.detach()], 0).contiguous()
            a.q_proj.weight.data, a.k_proj.weight.data, a.v_proj.weight.data = wqkv[:HD], wqkv[HD:HD + KD], wqkv[HD + KD:]
            a.q_proj.bias.data, a.k_proj.bias.data, a.v_proj.bias.data = bqkv[:HD], bqkv[HD:HD + KD], bqkv[HD + KD:]
            if self._swiglu_concat:
                wgu = torch.cat([m.gate_proj.weight.detach(), m.up_proj.weight.detach()], 0).contiguous()
                m.gate_proj.weight.data, m.up_proj.weight.data = wgu[: self.inter], wgu[self.inter:]
            else:
                wgu = ops.pack_gate_up(m.gate_proj.weight.detach().contiguous(), m.up_proj.weight.detach().contiguous())
            P.append((wqkv, bqkv, wgu))
        self._packed = P
        self._proj = [_Bf16Projections(self, wqkv, bqkv, l.self_attn.o_proj.weight, wgu, l.mlp.down_proj.weight)
                      for l, (wqkv, bqkv, wgu) in zip(self.model.layers, P)]
        self._set_inv_freq()

    def _pack_fp8(self):
        """FP8 counterpart of pack_weights: one fused [q; k; v] and one [gate; up] e4m3 matrix per layer, each with its fused
        weight_scale_inv grid; the projections' weight / weight_scale_inv are re-pointed at row views of them."""
        P, proj = [], []
        HD, KD = self.H * self.D, self.Hkv * self.D
        for l in self.model.layers:
            a, m = l.self_attn, l.mlp
            wqkv = torch.cat([a.q_proj.weight.detach(), a.k_proj.weight.detach(), a.v_proj.weight.detach()], 0).contiguous()
            sqkv = torch.cat([a.q_proj.weight_scale_inv, a.k_proj.weight_scale_inv, a.v_proj.weight_scale_inv], 0).contiguous()
            bqkv = torch.cat([a.q_proj.bias.detach(), a.k_proj.bias.detach(), a.v_proj.bias.detach()], 0).contiguous()
            wgu = torch.cat([m.gate_proj.weight.detach(), m.up_proj.weight.detach()], 0).contiguous()
            sgu = torch.cat([m.gate_proj.weight_scale_inv, m.up_proj.weight_scale_inv], 0).contiguous()
            for mod, w, sc, r0, r1 in ((a.q_proj, wqkv, sqkv, 0, HD), (a.k_proj, wqkv, sqkv, HD, HD + KD), (a.v_proj, wqkv, sqkv, HD + KD, HD + 2 * KD),
                                       (m.gate_proj, wgu, sgu, 0, self.inter), (m.up_proj, wgu, sgu, self.inter, 2 * self.inter)):
                mod.weight.data = w[r0:r1]
                mod.weight_scale_inv = sc[r0 // 128:r1 // 128]
            a.q_proj.bias.data, a.k_proj.bias.data, a.v_proj.bias.data = bqkv[:HD], bqkv[HD:HD + KD], bqkv[HD + KD:]
            P.append((wqkv, bqkv, wgu))
            proj.append(_Fp8Projections(self, (wqkv, sqkv), bqkv, (a.o_proj.weight, a.o_proj.weight_scale_inv), (wgu, sgu),
                                        (m.down_proj.weight, m.down_proj.weight_scale_inv)))
        self._packed, self._proj = P, proj
        self._set_inv_freq()

    def _pack_w4a16(self):
        """W4A16 counterpart of pack_weights: one fused [q; k; v] and one [gate; up] packed matrix per layer with their scale
        grids (packing is per row, so stacking rows is exact); the projections' weight_packed / weight_scale become row views
        of them.  Also allocates the bf16 scratch that the GEMMs of more than 64 tokens dequantize into, sized for the largest
        projection ([gate; up]: 272 MB at 7B)."""
        P, proj = [], []
        HD, KD = self.H * self.D, self.Hkv * self.D
        for l in self.model.layers:
            a, m = l.self_attn, l.mlp
            wqkv = torch.cat([a.q_proj.weight_packed, a.k_proj.weight_packed, a.v_proj.weight_packed], 0).contiguous()
            sqkv = torch.cat([a.q_proj.weight_scale, a.k_proj.weight_scale, a.v_proj.weight_scale], 0).contiguous()
            bqkv = torch.cat([a.q_proj.bias.detach(), a.k_proj.bias.detach(), a.v_proj.bias.detach()], 0).contiguous()
            wgu = torch.cat([m.gate_proj.weight_packed, m.up_proj.weight_packed], 0).contiguous()
            sgu = torch.cat([m.gate_proj.weight_scale, m.up_proj.weight_scale], 0).contiguous()
            for mod, w, sc, r0, r1 in ((a.q_proj, wqkv, sqkv, 0, HD), (a.k_proj, wqkv, sqkv, HD, HD + KD), (a.v_proj, wqkv, sqkv, HD + KD, HD + 2 * KD),
                                       (m.gate_proj, wgu, sgu, 0, self.inter), (m.up_proj, wgu, sgu, self.inter, 2 * self.inter)):
                mod.weight_packed, mod.weight_scale = w[r0:r1], sc[r0:r1]
            a.q_proj.bias.data, a.k_proj.bias.data, a.v_proj.bias.data = bqkv[:HD], bqkv[HD:HD + KD], bqkv[HD + KD:]
            P.append((wqkv, bqkv, wgu))
            proj.append(_W4A16Projections(self, (wqkv, sqkv), bqkv, (a.o_proj.weight_packed, a.o_proj.weight_scale), (wgu, sgu),
                                          (m.down_proj.weight_packed, m.down_proj.weight_scale)))
        n = max(w.shape[0] * w.shape[1] * 8 for pj in proj for w, _ in (pj.wqkv, pj.wo, pj.wgu, pj.wdown))
        self._w4_scratch = torch.empty((n,), device=self.lm_head.weight.device, dtype=bf16)
        self._packed, self._proj = P, proj
        self._set_inv_freq()

    def _set_inv_freq(self):
        # Qwen2RotaryEmbedding.compute_default_rope_parameters, evaluated on the CPU like the reference (Q2M:86-89)
        inv = 1.0 / (self.rope_theta ** (torch.arange(0, self.D, 2, dtype=torch.int64).to(dtype=torch.float) / self.D))
        self._inv_freq = inv.to(self.lm_head.weight.device)

    def _check_ready(self):
        p = self.lm_head.weight
        if not p.is_cuda or p.dtype != bf16:
            raise AF3Error("model must be on a CUDA device in bfloat16 (model.to('cuda', torch.bfloat16)); no CPU fallback")
        if self._packed is None:
            self.pack_weights()

    def new_cache(self, B, Tmax):
        dev = self.lm_head.weight.device
        return AF3KVCache(len(self.model.layers), B, self.Hkv, Tmax, self.D, dev)

    # ------------------------------------------------------------------ core stacks
    def _layers(self, h, B, T, cache: AF3KVCache, decode: bool, scratch=None):
        """h [B*T, hid] residual stream, updated in place and returned."""
        H, Hkv, D = self.H, self.Hkv, self.D
        pos0 = cache.length
        rope_cs = None
        fused_qkv = decode and B <= 64  # few-token ("swapped") GEMM with RoPE + KV append in its epilogue
        if fused_qkv:
            rope_cs = ops.rope_table(B, D, cache.pos_dev, cache.kv_start, self._inv_freq)
        y = None
        for li, (l, pj) in enumerate(zip(self.model.layers, self._proj)):
            kc, vc = cache.k[li], cache.v[li]
            a = torch.empty((B * T, H * D), device=h.device, dtype=bf16)
            if decode:
                if fused_qkv:
                    # q/k/v projection with RoPE + KV append in the GEMM epilogue (rope table: once per step, above)
                    y = ops.rmsnorm(h, l.input_layernorm.weight, self.eps, out=y)
                    qkv = pj.qkv_rope(y, kc, vc, rope_cs, cache.pos_dev)
                else:
                    # more than 64 sequences per GPU: token-major tensor-core GEMM + the stand-alone RoPE / append kernel reading
                    # the slot from device memory (graph replay)
                    y = ops.rmsnorm(h, l.input_layernorm.weight, self.eps, out=y)
                    qkv = pj.qkv(y)
                    ops.rope_kv_append(qkv, kc, vc, B=B, T=1, H=H, Hkv=Hkv, D=D, pos0=0, inv_freq=self._inv_freq,
                                       kv_start=cache.kv_start, pos0_dev=cache.pos_dev)
                ops.decode_attention(qkv, kc, vc, a, scratch, B=B, H=H, Hkv=Hkv, D=D, ctx_len=cache.ctx_dev,
                                     kv_start=cache.kv_start, scale=D ** -0.5)
            else:
                y = ops.rmsnorm(h, l.input_layernorm.weight, self.eps, out=y)
                qkv = pj.qkv(y)
                ops.rope_kv_append(qkv, kc, vc, B=B, T=T, H=H, Hkv=Hkv, D=D, pos0=pos0, inv_freq=self._inv_freq,
                                   kv_start=cache.kv_start)
                ops.attention(qkv, kc, vc, a.view(B, T, H * D), B=B, H=H, Hkv=Hkv, D=D, Tq=T, Tk=pos0 + T, scale=D ** -0.5,
                              causal=True, kv_layout=1, Tk_pitch=cache.Tmax, ldq=(H + 2 * Hkv) * D, ldk=D,
                              kv_start=cache.kv_start)
            pj.o(a, h)
            y = ops.rmsnorm(h, l.post_attention_layernorm.weight, self.eps, out=y)
            pj.down(pj.gate_up(y), h)
        return h

    def _head(self, h, row_idx=None):
        y = ops.rmsnorm(h, self.model.norm.weight, self.eps, row_idx=row_idx)
        return ops.linear(y, self.lm_head.weight, out_f32=True)

    def loss_head(self, y, labels, ignore_index=-100, num_items_in_batch=None, store_logits=False):
        """LM head + ForCausalLMLoss on the post-norm hidden states y [n_tok, hid], with labels int64 [n_tok] already shifted
        (prepare_loss_labels), without materialising the logits unless store_logits.  -> (fp32 logits [n_tok, V] or None,
        token_losses fp32 [n_tok], loss 0-dim fp32, invalid-label count 0-dim).  loss = sum / counted positions, or sum /
        num_items_in_batch when given, as fixed_cross_entropy; NaN when nothing is counted."""
        logits, nll, totals = ops.lm_head_xent(y, self.lm_head.weight, labels, ignore_index, store_logits=store_logits)
        n = totals[1] if num_items_in_batch is None else torch.as_tensor(num_items_in_batch, device=y.device).to(torch.float64)
        return logits, nll, (totals[0] / n).to(torch.float32), totals[2]

    @torch.no_grad()
    def prefill(self, inputs_embeds, kv_start, cache: AF3KVCache, logits_to_keep=1, labels=None, ignore_index=-100,
                num_items_in_batch=None):
        """inputs_embeds [B,S,hid] bf16 (consumed in place), kv_start int32 [B]. -> fp32 logits [B, keep|S, V].
        The chunk is appended at cache.length (0 for a fresh prompt; > 0 for the next slice of a chunked prefill or a later chat turn:
        RoPE positions, the causal offset and the left padding of the first chunk carry over).
        With labels (int64 [B * S] on the device, already shifted): -> (logits or None, token_losses [B, S], loss, invalid-label
        count), the loss over every position of the chunk whatever logits_to_keep.  With logits_to_keep = 0 the same launch
        stores the logits; otherwise no [B, S, V] buffer exists."""
        self._check_ready()
        B, S, _ = inputs_embeds.shape
        if B != cache.B:
            raise AF3Error(f"KV cache was allocated for {cache.B} sequences, got {B}")
        if cache.length + S > cache.Tmax:
            raise AF3Error(f"KV cache too small for this prompt ({cache.length} + {S} > capacity {cache.Tmax})")
        if cache.length == 0:  # a continuation chunk (chunked prefill, next turn) keeps the left padding of the first chunk
            if kv_start is None:
                cache.kv_start.zero_()
            else:
                cache.kv_start.copy_(kv_start)
        h = self._layers(inputs_embeds.view(B * S, self.hid), B, S, cache, decode=False)
        cache.length += S
        cache.pos_dev.fill_(cache.length)
        cache.ctx_dev.fill_(cache.length + 1)
        if labels is not None:
            if logits_to_keep not in (0, 1):
                raise AF3Error("logits_to_keep must be 0 (all positions) or 1 (last position)")
            y = ops.rmsnorm(h, self.model.norm.weight, self.eps)
            logits, nll, loss, invalid = self.loss_head(y, labels, ignore_index, num_items_in_batch, store_logits=logits_to_keep == 0)
            if logits_to_keep == 0:
                logits = logits.view(B, S, self.vocab)
            else:
                last = torch.arange(B, device=h.device, dtype=torch.int32) * S + (S - 1)
                logits = self._head(h, last).view(B, 1, self.vocab)
            return logits, nll.view(B, S), loss, invalid
        if logits_to_keep == -1:  # an inner slice of a chunked prefill: only the cache is wanted
            return None
        if logits_to_keep == 0:
            return self._head(h).view(B, S, self.vocab)
        if logits_to_keep != 1:
            raise AF3Error("logits_to_keep must be 0 (all positions) or 1 (last position)")
        last = torch.arange(B, device=h.device, dtype=torch.int32) * S + (S - 1)
        return self._head(h, last).view(B, 1, self.vocab)

    @torch.no_grad()
    def decode_step(self, token_embeds, cache: AF3KVCache, scratch):
        """One q_len = 1 step: token_embeds [B, hid] (in place) -> fp32 logits [B, V]; appends at cache.pos_dev.
        Graph-capturable: positions / context length are read from device memory and advanced on the device."""
        B = token_embeds.shape[0]
        if cache.length + 1 > cache.Tmax:  # the fused q/k/v epilogue appends at slot `length`: never past the allocation
            raise AF3Error(f"KV cache full ({cache.length} of {cache.Tmax} slots): cache.ensure_capacity() or a larger reserve is needed")
        h = self._layers(token_embeds, B, 1, cache, decode=True, scratch=scratch)
        logits = self._head(h)
        cache.pos_dev.add_(1)
        cache.ctx_dev.add_(1)
        return logits


# =====================================================================================================
# the drop-in top-level model
# =====================================================================================================
class AudioFlamingo3ForConditionalGeneration(nn.Module):
    """Drop-in for the reference class of the same name ([O] AF3M:410-592) on its audio->text inference path."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.vocab_size = config.text_config.vocab_size
        with torch.device("meta"):
            self.audio_tower = AudioFlamingo3Encoder(config.audio_config)
            self.language_model = Qwen2ForCausalLM(config.text_config)
            self.multi_modal_projector = AudioFlamingo3MultiModalProjector(
                config.audio_config.hidden_size, config.text_config.hidden_size, _cfg_get(config, "projector_bias", True))
        if _cfg_get(config, "projector_hidden_act", "gelu") != "gelu":
            raise AF3Error("only projector_hidden_act='gelu' is implemented")
        self._graph = None
        # KV cache + captured decode graph of the last generate() (batch, capacity bucket), kept between calls: capturing and instantiating the
        # ~230-node step graph costs the launching thread 0.05-0.3 s during which the GPU idles (r01 bench host-gap logs), and a
        # serving loop issues the same (batch, max length) shape over and over.  release_decode_state() frees it.
        self._decode_state = None
        self._deferred = []       # input-validation verdicts still on the device (see _defer_check)
        self.generation_config = None  # the reference model's GenerationConfig when built by from_reference(); generate() defaults
        self.stage_events = None  # bench instrumentation: when a list, (name, cuda event) is appended at stage boundaries
        self.stage_host_t = None  # ... and, when a list, (name, host perf_counter at enqueue time): GPU-bound vs launch-bound

    def _mark(self, name):
        if self.stage_events is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.stage_events.append((name, ev))
            if self.stage_host_t is not None:
                self.stage_host_t.append((name, time.perf_counter()))

    # ---- construction from the reference model / a reference state_dict
    @classmethod
    def from_reference(cls, ref_model, device="cuda", quantization=None):
        """Build from an instantiated reference model (weights are copied, cast to bf16).  quantization="fp8" or "w4a16": see
        load_reference_state_dict."""
        m = cls(ref_model.config)
        m.load_reference_state_dict(ref_model.state_dict(), device=device, quantization=quantization)
        m.generation_config = getattr(ref_model, "generation_config", None)
        return m

    @property
    def quantization(self):
        return self.language_model.quantization

    def load_reference_state_dict(self, sd, device="cuda", quantization=None):
        """Load a reference state_dict.  Weights are cast to bf16.

        quantization="fp8" stores the seven projections of every decoder layer (q, k, v, o, gate, up, down) as block-scaled
        e4m3 -- the FineGrainedFP8 format of transformers with 128 x 128 blocks: e4m3 weights plus one fp32 weight_scale_inv
        per block, quantized from the bf16 values exactly as Fp8Quantize does -- and runs them on the FP8 GEMMs with
        activations quantized per token and 128 columns.  The embedding, lm_head, audio tower and projector stay bf16.  The
        hidden, q/k/v/o and intermediate sizes must be multiples of 128.

        The state_dict may already be in that layout (`<name>.weight` float8_e4m3fn plus `<name>.weight_scale_inv`, what
        state_dict() of an FP8 model returns).  Its decoder projections are then used as they are, and the model is FP8
        whatever `quantization` says.  Any other Linear stored that way is dequantized once to bf16.

        quantization="w4a16" stores the same seven projections as group-wise int4 (include/af3b200.h af3_gemm_w4a16): one
        bf16 scale per row and 128 input columns, round to nearest, packed 8 values per int32.  The projection modules then
        carry `weight_packed` and `weight_scale` instead of `weight`, and state_dict() returns those keys; a state_dict that
        carries them for the decoder projections loads as W4A16 whatever `quantization` says (weights from another quantizer
        in this layout load as they are).  Decode with up to 64 sequences runs the int4 GEMMs; larger token counts run the
        bf16 GEMMs on the dequantized projection."""
        if quantization not in (None, "fp8", "w4a16"):
            raise AF3Error(f"quantization must be None, 'fp8' or 'w4a16', got {quantization!r}")
        scaled = {k[: -len(".weight_scale_inv")] for k in sd if k.endswith(".weight_scale_inv")}
        packed = {k[: -len(".weight_packed")] for k in sd if k.endswith(".weight_packed")}
        for base in sorted(packed):
            if base + ".weight_scale" not in sd:
                raise AF3Error(f"{base}.weight_packed without {base}.weight_scale")
        if any(_is_decoder_projection(k) for k in scaled):
            quantization = "fp8"
        if any(_is_decoder_projection(k) for k in packed):
            quantization = "w4a16"
        lm = self.language_model
        if quantization is not None:
            sizes = {"hidden_size": lm.hid, "q size": lm.H * lm.D, "k/v size": lm.Hkv * lm.D, "intermediate_size": lm.inter}
            bad = {k: v for k, v in sizes.items() if v % 128}
            if bad:
                what = "the 128 x 128 scale blocks" if quantization == "fp8" else "the 128-column scale groups"
                raise AF3Error(f"{quantization} quantization needs multiples of 128 ({what}); got {bad}")
        for name in DECODER_PROJECTIONS:  # the module tree of this load: a previous FP8 / W4A16 load changed the projections
            for l in lm.model.layers:
                mod = l.get_submodule(name)
                mod._buffers.pop("weight_scale_inv", None)
                N, K = mod.out_features, mod.in_features
                if quantization == "w4a16":
                    mod._parameters.pop("weight", None)
                    mod.register_buffer("weight_packed", torch.empty((N, K // 8), dtype=torch.int32, device="meta"))
                    mod.register_buffer("weight_scale", torch.empty((N, K // W4_GROUP), dtype=bf16, device="meta"))
                elif "weight_packed" in mod._buffers:
                    del mod._buffers["weight_packed"], mod._buffers["weight_scale"]
                    mod.weight = nn.Parameter(torch.empty((N, K), device="meta"))
        self.to_empty(device=device)
        self.to(bf16)
        own = self.state_dict()
        w4_own = {k[: -len(".weight_packed")] for k in own if k.endswith(".weight_packed")}

        def present(k):  # a W4A16 projection may come as weight_packed + weight_scale or as a plain weight
            for sfx in (".weight_packed", ".weight_scale"):
                if k.endswith(sfx) and k[: -len(sfx)] in w4_own:
                    return k[: -len(sfx)] in packed or k[: -len(sfx)] + ".weight" in sd
            return k in sd

        def expected(k):
            if k in own or (k.endswith(".weight_scale_inv") and k[: -len("_scale_inv")] in own):
                return True
            return k.endswith(".weight") and k[: -len(".weight")] in w4_own
        missing = [k for k in own if not present(k)]
        unexpected = [k for k in sd if not expected(k)]
        if missing or unexpected:
            raise AF3Error(f"state_dict mismatch: missing {missing[:4]}..., unexpected {unexpected[:4]}...")

        def bf16_value(k):
            v = sd[k]
            if v.dtype == torch.float8_e4m3fn:
                base = k[: -len(".weight")]
                if base not in scaled:
                    raise AF3Error(f"{k} is float8_e4m3fn without {base}.weight_scale_inv")
                dev = torch.device(device)
                return dequantize_fp8_blocks(v.to(dev), sd[base + ".weight_scale_inv"].to(dev, torch.float32)).to(bf16)
            return v

        fp8_params = {}
        with torch.no_grad():
            for k, v in own.items():
                base = k[: -len(".weight")] if k.endswith(".weight") else None
                if quantization == "fp8" and base is not None and _is_decoder_projection(base):
                    if sd[k].dtype == torch.float8_e4m3fn and base not in scaled:
                        raise AF3Error(f"{k} is float8_e4m3fn without {base}.weight_scale_inv")
                    if base in scaled and sd[k].dtype == torch.float8_e4m3fn:
                        q, s = sd[k].to(v.device), sd[base + ".weight_scale_inv"].to(v.device, torch.float32)
                    else:
                        q, s = quantize_fp8_blocks(sd[k].to(device=v.device, dtype=bf16))
                    fp8_params[base] = (q.contiguous(), s.contiguous())
                    continue
                if k.endswith(".weight_packed") and k[: -len(".weight_packed")] in w4_own:
                    base = k[: -len(".weight_packed")]
                    if base in packed:
                        q, s = sd[k], sd[base + ".weight_scale"]
                    else:
                        q, s = quantize_w4a16(sd[base + ".weight"].to(device=v.device, dtype=bf16))
                    v.copy_(q.to(device=v.device, dtype=torch.int32))
                    own[base + ".weight_scale"].copy_(s.to(device=v.device, dtype=bf16))
                    continue
                if k.endswith(".weight_scale") and k[: -len(".weight_scale")] in w4_own:
                    continue  # with its weight_packed
                v.copy_(bf16_value(k).to(device=v.device, dtype=bf16))
            for base, (q, s) in fp8_params.items():
                mod = self.get_submodule(base)
                mod.weight = nn.Parameter(q, requires_grad=False)
                mod.register_buffer("weight_scale_inv", s)
        lm.quantization = quantization
        self.audio_tower._packed = None
        self.language_model._packed = None
        self._graph = None
        self._decode_state = None  # its graph holds the addresses of the packed weights just dropped
        return self

    def get_input_embeddings(self):
        return self.language_model.model.embed_tokens

    def get_output_embeddings(self):
        return self.language_model.lm_head

    # ---- audio branch
    @_on_model_device
    @torch.no_grad()
    def get_audio_features(self, input_features, input_features_mask, input_ids=None, **kwargs):
        """[O] AF3M:447-475: tower -> projector -> keep the first post_len frames of every window."""
        enc, W, Tp = self.audio_tower._encode(input_features, input_features_mask)
        enc = self._post_encoder(enc, W, Tp, input_features_mask, input_ids)
        emb = self.multi_modal_projector(enc)                                   # [W*Tp, text_hidden]
        lens = input_features_mask.sum(-1).to(torch.long)
        _, post = self.audio_tower._get_feat_extract_output_lengths(lens)
        valid = torch.arange(Tp, device=emb.device)[None, :] < post[:, None]
        out = BaseModelOutputWithPooling(last_hidden_state=enc.view(W, Tp, -1))
        out.pooler_output = emb.view(W, Tp, -1)[valid]
        return out

    def _post_encoder(self, enc, W, Tp, input_features_mask, input_ids):
        """Hook between the audio tower and the projector (identity for AF3; Music Flamingo rotates here)."""
        return enc

    def _audio_embeds_raw(self, input_features, input_features_mask, input_ids=None):
        enc, W, Tp = self.audio_tower._encode(input_features, input_features_mask)
        enc = self._post_encoder(enc, W, Tp, input_features_mask, input_ids)
        emb = self.multi_modal_projector(enc)
        lens = input_features_mask.sum(-1).to(torch.int32)
        post = (((lens - 1) // 2 + 1) - 2) // 2 + 1
        return emb, W, Tp, post.to(torch.int32).contiguous()

    # ---- input validation without host<->device round trips on the hot path
    def _defer_check(self, flag, exc, message):
        """`flag`: 0-dim device tensor, non-zero = invalid input.  Raised by _raise_deferred() at the end of the public call (one
        sync after everything has been enqueued) instead of stalling the launch thread between encoder and prefill."""
        self._deferred.append((flag, exc, message))

    def _raise_deferred(self):
        pending, self._deferred = self._deferred, []
        for flag, exc, message in pending:
            if bool(flag.item()):
                raise exc(message() if callable(message) else message)

    def _left_pad_starts(self, attention_mask, B, S, device):
        """int32 [B] number of left-padding slots per row.  The kernels implement the reference processor's left padding
        ([O] AF3P:44-47): every mask row must be 0...01...1.  A host mask (what the processor returns) is validated on the host;
        a device mask is validated on the device and the verdict is read at the end of the call (_raise_deferred)."""
        msg = "attention_mask must be left padded (zeros then ones), as the AF3 processor produces"
        if attention_mask is None:
            return torch.zeros((B,), device=device, dtype=torch.int32)
        if tuple(attention_mask.shape) != (B, S):
            raise AF3Error(f"attention_mask must have shape {(B, S)}, got {tuple(attention_mask.shape)}")
        am = attention_mask
        n_valid = am.sum(-1)
        expect = torch.arange(S, device=am.device)[None, :] >= (S - n_valid)[:, None]
        bad = (am.bool() != expect).any()
        if am.is_cuda:
            self._defer_check(bad, AF3Error, msg)
        elif bool(bad):
            raise AF3Error(msg)
        return (S - n_valid).to(device=device, dtype=torch.int32).contiguous()

    @torch.no_grad()
    def _prompt_embeds(self, input_ids, input_features, input_features_mask):
        B, S = input_ids.shape
        dev = self.language_model.lm_head.weight.device
        ids = input_ids.to(dev).reshape(-1).contiguous()
        table = self.language_model.model.embed_tokens.weight
        if input_features is not None:
            emb, W, Tp, post = self._audio_embeds_raw(input_features.to(dev), input_features_mask.to(dev), input_ids.to(dev))
            x, counts = ops.embed_scatter(ids, table, self.config.audio_token_id, emb, W, Tp, post)
            # masked_scatter would fail the same way (AF3M:564); a mismatch is memory-safe here (surplus placeholders keep their
            # token embedding, surplus features are dropped), so the verdict is read at the end of the call
            self._defer_check(counts[0] != counts[1], ValueError,
                              lambda c=counts: "Audio features and audio tokens do not match: tokens {}, features {}".format(*c.tolist()))
        else:
            x, _ = ops.embed_scatter(ids, table, -1, None, 0, 1, None)
        return x.view(B, S, -1)

    # ---- forward ([O] AF3M:479-578)
    @_on_model_device
    @torch.no_grad()
    def forward(self, input_ids=None, input_features=None, input_features_mask=None, attention_mask=None,
                position_ids=None, past_key_values=None, inputs_embeds=None, labels=None, use_cache=None,
                logits_to_keep=0, reserve_tokens=None, **kwargs):
        """Same call surface as the reference.  Three cases:
          * no cache, or an empty one: prompt prefill (audio rows scattered into the prompt, AF3M:556-566);
          * live cache + exactly one new token per sequence: one cached decode step (AF3M:580-592: no audio after the first pass);
          * live cache + a longer chunk (next chat turn, optionally with new audio; one slice of a chunked prefill, GEN:3770-3806):
            the chunk is appended at the cache's current length.  Its attention_mask -- [B, chunk] or the reference's
            full-length [B, past + chunk] -- must be all ones over the chunk (the kernels keep one contiguous live range per row).
        With use_cache the returned AF3KVCache has room for `reserve_tokens` more slots (default: up to the next multiple of 256)
        and grows on demand in later calls, like DynamicCache.

        Teacher-forced loss (inference only, no backward): with `labels` [B, S] (or `shift_labels`, used as they are) the output
        carries `loss` as ForCausalLMLoss computes it -- keywords ignore_index (default -100) and num_items_in_batch as in the
        reference -- and `token_losses` fp32 [B, S].  Both the prompt prefill and a continuation chunk take labels (covering
        the chunk); the one-token cached step does not.  The loss covers every position whatever `logits_to_keep`, and is
        computed in the LM head's epilogue without the [B, S, V] logits: with logits_to_keep=1 they are never allocated (the
        memory-lean way to score), with logits_to_keep=0 the same launch also stores them."""
        if position_ids is not None:
            raise AF3Error("explicit position_ids are not supported; they are derived from the left-padded attention_mask")
        if (input_ids is None) == (inputs_embeds is None):
            raise ValueError("You must specify exactly one of input_ids or inputs_embeds")      # AF3M:548
        self.language_model._check_ready()
        lm = self.language_model
        dev = lm.lm_head.weight.device
        cache = past_key_values
        shift_labels = kwargs.get("shift_labels")
        loss_kw = None
        if labels is not None or shift_labels is not None:
            B, S = (input_ids if input_ids is not None else inputs_embeds).shape[:2]
            ignore_index = kwargs.get("ignore_index", -100)
            if cache is not None and cache.length > 0 and inputs_embeds is None and input_features is None and S == 1:
                raise AF3Error("labels on the one-token cached decode step are not implemented; pass them with the prompt or a longer chunk")
            loss_kw = dict(labels=prepare_loss_labels(labels, shift_labels, ignore_index, B, S, lm.vocab).to(dev),
                           ignore_index=ignore_index, num_items_in_batch=kwargs.get("num_items_in_batch"))

        def output(res, cache_out):
            if loss_kw is None:
                return CausalLMOutputWithPast(logits=res, past_key_values=cache_out)
            logits, token_losses, loss, invalid = res
            self._defer_check(invalid != 0, ValueError,
                              f"labels must lie in [0, {lm.vocab}) or equal ignore_index ({loss_kw['ignore_index']}): the invalid ones were ignored")
            return CausalLMOutputWithTokenLosses(loss=loss, logits=logits, past_key_values=cache_out, token_losses=token_losses)

        try:
            if cache is not None and cache.length > 0:
                single = inputs_embeds is None and input_features is None and input_ids.shape[1] == 1
                if single:
                    B = input_ids.shape[0]
                    if B != cache.B:
                        raise AF3Error(f"KV cache was allocated for {cache.B} sequences, got {B}")
                    cache.ensure_capacity(cache.length + 1)
                    x, _ = ops.embed_scatter(input_ids.to(dev).reshape(-1).contiguous(), lm.model.embed_tokens.weight, -1, None, 0, 1, None)
                    scratch = ops.decode_attention_scratch(B, lm.H, lm.D, cache.Tmax, dev)
                    logits = lm.decode_step(x, cache, scratch)
                    cache.length += 1
                    return CausalLMOutputWithPast(logits=logits.view(B, 1, -1), past_key_values=cache)
                # continuation chunk
                if inputs_embeds is None:
                    inputs_embeds = self._prompt_embeds(input_ids, input_features, input_features_mask)
                else:
                    inputs_embeds = inputs_embeds.to(dev, bf16).clone()
                B, S, _ = inputs_embeds.shape
                if attention_mask is not None:
                    am = attention_mask[:, -S:] if attention_mask.shape[1] == cache.length + S else attention_mask
                    if tuple(am.shape) != (B, S):
                        raise AF3Error(f"attention_mask must cover the new chunk [B, {S}] or the full sequence [B, {cache.length + S}]")
                    bad = (am == 0).any()
                    msg = "a continuation chunk on a live cache must be unpadded (attention_mask all ones over the chunk)"
                    if am.is_cuda:
                        self._defer_check(bad, AF3Error, msg)
                    elif bool(bad):
                        raise AF3Error(msg)
                cache.ensure_capacity(cache.length + S + (reserve_tokens or 0))
                return output(lm.prefill(inputs_embeds, None, cache, logits_to_keep=logits_to_keep, **(loss_kw or {})), cache)
            if inputs_embeds is None:
                inputs_embeds = self._prompt_embeds(input_ids, input_features, input_features_mask)
            else:
                inputs_embeds = inputs_embeds.to(dev, bf16).clone()
            B, S, _ = inputs_embeds.shape
            kv_start = self._left_pad_starts(attention_mask, B, S, dev)
            keep = bool(use_cache) or cache is not None
            if cache is None:
                # without use_cache the cache only lives for this call: exactly the prompt.  With it, room for a cached
                # continuation is reserved (ADVICE r01: a zero reserve made the first decode step write past the allocation)
                rows = S + (reserve_tokens if reserve_tokens is not None else 1) if keep else S
                cache = lm.new_cache(B, AF3KVCache.bucket(rows) if keep else max(S, 1))
            else:
                cache.ensure_capacity(S + (reserve_tokens or 0))
            return output(lm.prefill(inputs_embeds, kv_start, cache, logits_to_keep=logits_to_keep, **(loss_kw or {})),
                          cache if keep else None)
        finally:
            self._raise_deferred()

    __call__ = forward  # nn.Module.__call__ hooks are not needed on the inference path

    # ---- greedy generation ([O] GEN:2131 generate -> GEN:2658 _sample with do_sample=False)
    _IGNORED_WHEN_GREEDY = ("temperature", "top_p", "top_k", "min_p", "typical_p")        # unused by the reference too when do_sample=False
    _ACCEPTED_DEFAULTS = {"num_beams": 1, "num_return_sequences": 1, "repetition_penalty": 1.0,
                          "length_penalty": 1.0, "use_cache": True, "num_beam_groups": 1, "penalty_alpha": None,
                          "assistant_model": None, "streamer": None, "logits_processor": None,
                          "stopping_criteria": None, "synced_gpus": None}
    _OUTPUT_OPTIONS = ("return_dict_in_generate", "output_scores", "output_logits")

    def _generation_default(self, name):
        gc = getattr(self, "generation_config", None)
        return getattr(gc, name, None) if gc is not None else None

    @_on_model_device
    @torch.no_grad()
    def generate(self, input_ids=None, attention_mask=None, input_features=None, input_features_mask=None,
                 max_new_tokens=None, max_length=None, do_sample=None, eos_token_id=None, pad_token_id=None, use_cuda_graph=True,
                 return_logits=False, prefill_chunk_size=None, generation_config=None, **kwargs):
        """Greedy decoding with the reference's `generate` call surface (prompt included in the returned ids, AF3M:547-551).
        Defaults follow the reference: eos_token_id / pad_token_id / max_new_tokens / do_sample come from `generation_config`
        (argument, else `self.generation_config`) when not passed; finished rows are padded and the loop stops once every row
        has produced EOS (GEN:2797-2805).  Options of the reference this path does not implement raise instead of being ignored.
        Greedy logits processors (sequence_bias, no_repeat_ngram_size, bad_words_ids, min_length, min_new_tokens,
        forced_eos_token_id, suppress_tokens, begin_suppress_tokens; argument, else `generation_config`) run on the device inside
        the decode step (include/af3b200.h af3_logits_process_argmax) and apply to every selected token, the first one included.
        return_dict_in_generate=True returns a GenerateDecoderOnlyOutput: `scores` (output_scores) holds the processed rows and
        `logits` (output_logits) the raw ones, one [B, V] tensor per generated token; past_key_values is None (the decode cache is
        kept internally, see release_decode_state)."""
        if generation_config is not None:
            saved, self.generation_config = getattr(self, "generation_config", None), generation_config
            try:
                return self.generate(input_ids=input_ids, attention_mask=attention_mask, input_features=input_features,
                                     input_features_mask=input_features_mask, max_new_tokens=max_new_tokens, max_length=max_length,
                                     do_sample=do_sample, eos_token_id=eos_token_id, pad_token_id=pad_token_id,
                                     use_cuda_graph=use_cuda_graph, return_logits=return_logits, prefill_chunk_size=prefill_chunk_size, **kwargs)
            finally:
                self.generation_config = saved
        proc_kw = {k: kwargs.pop(k) for k in list(kwargs) if k in logits_process.OPTIONS}
        out_kw = {k: kwargs.pop(k) for k in list(kwargs) if k in self._OUTPUT_OPTIONS}
        for k, v in kwargs.items():
            if k in self._IGNORED_WHEN_GREEDY:
                continue
            if k in self._ACCEPTED_DEFAULTS and (v == self._ACCEPTED_DEFAULTS[k] or v is None):
                continue
            raise AF3Error(f"generate(): option {k}={v!r} is not implemented on the greedy GPU path "
                           "(greedy decoding, one sequence per prompt, no logits processors)")
        if do_sample is None:
            do_sample = bool(self._generation_default("do_sample"))
        if do_sample:
            raise AF3Error("only greedy decoding (do_sample=False) is implemented")
        if input_ids is None:
            raise AF3Error("generate() needs input_ids")
        lm = self.language_model
        lm._check_ready()
        dev = lm.lm_head.weight.device
        B, S = input_ids.shape
        if max_new_tokens is None:
            max_new_tokens = self._generation_default("max_new_tokens")
        if max_new_tokens is None:
            ml = max_length if max_length is not None else (self._generation_default("max_length") or 20)
            max_new_tokens = ml - S                                                      # GEN: max_length counts the prompt
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be >= 1 (prompt length {S})")
        if eos_token_id is None:
            eos_token_id = self._generation_default("eos_token_id")
        if pad_token_id is None:
            pad_token_id = self._generation_default("pad_token_id")
        if prefill_chunk_size is None:
            prefill_chunk_size = self._generation_default("prefill_chunk_size")
        eos_list = None
        if eos_token_id is not None:
            eos_list = [int(eos_token_id)] if isinstance(eos_token_id, int) else [int(e) for e in eos_token_id]
            if pad_token_id is None:
                pad_token_id = eos_list[0]                                                    # GEN: "Setting pad_token_id to eos_token_id"
        outs = {k: bool(out_kw[k] if out_kw.get(k) is not None else self._generation_default(k)) for k in self._OUTPUT_OPTIONS}
        want_scores = outs["return_dict_in_generate"] and outs["output_scores"]
        want_logits = return_logits or (outs["return_dict_in_generate"] and outs["output_logits"])
        Tmax = AF3KVCache.bucket(S + max_new_tokens)
        # processor options are validated and compiled here, on the host, before anything is enqueued
        procs = logits_process.compile_processors(logits_process.resolve_options(proc_kw, self._generation_default), eos_list, S,
                                                  S + max_new_tokens, lm.vocab, Tmax)
        try:
            self._mark("start")
            x = self._prompt_embeds(input_ids, input_features, input_features_mask)
            self._mark("audio_done")
            kv_start = self._left_pad_starts(attention_mask, B, S, dev)
            use_graph = bool(use_cuda_graph and max_new_tokens > 2)
            # Cache capacity is rounded up to a multiple of 256 rows: the captured graph depends on the capacity (cache pitch in the
            # tensor maps, scratch sizes) but not on the prompt length, so prompts of different lengths that fall into the same
            # bucket reuse one cache + graph.  The kernels only ever touch the live rows, the extra capacity costs memory only.
            # the captured graph holds raw addresses: key it on the weight storages too, so a re-pack (load_reference_state_dict) or
            # a move (.to()) can never leave a stale graph replaying against freed memory.  With processors on, the step launches
            # the processor kernels instead of the plain argmax, on buffers whose sizes are bucketed capacities: those are keyed too
            proc_spec = None
            if procs is not None:
                proc_spec = (logits_process.bucket(procs.cap), logits_process.bucket(procs.tables.size), want_scores)
            key = (B, Tmax, use_graph, os.environ.get("AF3_PDL", "1") != "0", str(dev), lm.lm_head.weight.data_ptr(),
                   lm._packed[0][0].data_ptr(), lm._packed[-1][2].data_ptr(), proc_spec)
            st = self._decode_state
            if st is not None and st["key"] == key:
                cache, step_fn = st["cache"], st["step"]       # same buffers -> the captured graph is valid as it stands
                cache.reset()
            else:
                self._decode_state = st = None                 # free the previous shape's cache and graph first
                cache = lm.new_cache(B, Tmax)
                step_fn = self._decode_runner(B, cache, use_graph, proc_spec)
                self._decode_state = {"key": key, "cache": cache, "step": step_fn}
            if prefill_chunk_size is not None and 0 < prefill_chunk_size < S:
                # chunked prefill (GEN:3770-3806): the prompt embeddings (audio rows already scattered in) go through the decoder in
                # slices of prefill_chunk_size positions appended to the live cache; peak activation memory scales with the chunk
                logits = None
                for c0 in range(0, S, prefill_chunk_size):
                    c1 = min(S, c0 + prefill_chunk_size)
                    logits = lm.prefill(x[:, c0:c1].contiguous(), kv_start, cache, logits_to_keep=1 if c1 == S else -1)
                logits = logits.view(B, -1)
            else:
                logits = lm.prefill(x, kv_start, cache, logits_to_keep=1).view(B, -1)           # GEN:3724 _prefill
            self._mark("prefill_done")
            kept_logits = [logits.clone()] if want_logits else None
            kept_scores = None
            if procs is None:
                first = ops.argmax(logits)                                                    # GEN:2793
                if want_scores:
                    kept_scores = [logits.clone()]                                            # no processor: scores are the logits
            else:
                step_fn.load_processors(input_ids, procs)
                first = step_fn.process(logits)
                if want_scores:
                    kept_scores = [step_fn.scores.clone()]
            step_fn.begin(first, eos_list, pad_token_id)
            n_done = self._token_loop(step_fn, cache, kept_logits, eos_list is not None, max_new_tokens, kept_scores)
            out = torch.empty((B, S + n_done), device=dev, dtype=torch.int64)
            out[:, :S] = input_ids.to(dev)
            out[:, S:] = step_fn.tok_buf[:, :n_done]
            result = out
            self._mark("decode_done")
            if outs["return_dict_in_generate"]:
                return GenerateDecoderOnlyOutput(sequences=result, scores=tuple(kept_scores) if want_scores else None,
                                                 logits=tuple(kept_logits) if outs["output_logits"] else None, past_key_values=None)
            if return_logits:
                return result, torch.stack(kept_logits, 1)
            return result
        finally:
            self._raise_deferred()

    def release_decode_state(self):
        """Frees the KV cache and decode graph kept from the last generate() call."""
        self._decode_state = None

    MAX_EOS_IDS = 8      # size of the device-side EOS set (af3_token_step)
    EOS_CHECK_EVERY = 8  # tokens between host reads of the "every row finished" flag (the reference syncs every token)

    def _token_loop(self, step_fn, cache, kept_logits, has_eos, max_new_tokens, kept_scores=None):
        """Greedy loop ([O] GEN:2743-2809).  The per-token bookkeeping (pad finished rows, append, EOS mask, "all finished") runs on
        the device inside the decode step (af3_token_step), so one iteration is one graph replay and nothing else; the host reads the
        "all finished" flags every EOS_CHECK_EVERY tokens (the reference syncs every token).  Returns the number of tokens generated.
        (Several steps per graph replay were measured too -- 8 per replay: 459.8 vs 456.6 ms for 127 steps, no gain -- and removed.)"""
        n_done = max_new_tokens
        for i in range(max_new_tokens):
            if i + 1 == max_new_tokens:
                step_fn.finish()                       # bookkeeping of the last token; no further model step
            else:
                logits = step_fn()                     # token i's bookkeeping + one cached step incl. the greedy argmax (GEN:2793)
                cache.length += 1
                if self.stage_host_t is not None:      # bench instrumentation: host time after enqueueing token i + 1
                    self.stage_host_t.append(("tok", time.perf_counter()))
                if kept_logits is not None:
                    kept_logits.append(logits.clone())
                if kept_scores is not None:
                    kept_scores.append(step_fn.scores.clone() if step_fn.scores is not None else logits.clone())
            if has_eos and ((i + 1) % self.EOS_CHECK_EVERY == 0 or i + 1 == max_new_tokens):
                flags = step_fn.done_flags[: i + 1].cpu()                                   # GEN:2805, one sync per EOS_CHECK_EVERY tokens
                if bool(flags.any()):
                    # tokens enqueued after the stopping step are pads of rows that had all finished: cut them off, the result
                    # equals the reference's, which stops at exactly that step
                    n_done = int(flags.nonzero()[0]) + 1
                    break
        if kept_logits is not None:
            del kept_logits[n_done:]
        if kept_scores is not None:
            del kept_scores[n_done:]
        return n_done

    def _decode_runner(self, B, cache, use_graph, proc_spec=None):
        """Returns the step object of the greedy loop: begin(first_ids, eos_list, pad) arms the device-side state, step() enqueues one
        token (bookkeeping, embedding gather, 28 layers, head, argmax) and returns the fp32 logits [B, V] buffer of the next token,
        finish() enqueues the bookkeeping of the last token; tok_buf [B, cap] / done_flags [cap] receive the tokens and the "every
        row finished" flags.  With use_graph the step is captured once in a CUDA graph and replayed; positions advance on the device.
        proc_spec = (rule-list entries per row, table capacity, scores wanted) switches the argmax to the logits processors:
        load_processors(input_ids, compiled) fills their device tables for one call, process(logits) selects the first token,
        and `scores` [B, V] receives each step's processed row when scores are wanted."""
        lm = self.language_model
        dev = lm.lm_head.weight.device
        table = lm.model.embed_tokens.weight
        scratch = ops.decode_attention_scratch(B, lm.H, lm.D, cache.Tmax, dev)
        # device-side state of the greedy loop (addresses baked into the captured graph; contents set per generate() call)
        cap = cache.Tmax
        raw_ids = torch.zeros((B,), device=dev, dtype=torch.int64)      # argmax of the previous logits
        ids_buf = torch.zeros((B,), device=dev, dtype=torch.int64)      # token fed to the next step
        unfinished = torch.ones((B,), device=dev, dtype=torch.int32)
        eos_dev = torch.zeros((self.MAX_EOS_IDS,), device=dev, dtype=torch.int64)
        ctl = torch.zeros((2,), device=dev, dtype=torch.int64)          # {number of EOS ids, pad id}
        tok_buf = torch.zeros((B, cap), device=dev, dtype=torch.int64)
        gen_idx = torch.zeros((1,), device=dev, dtype=torch.int32)
        done_flags = torch.zeros((cap,), device=dev, dtype=torch.int32)
        am_out = raw_ids
        if proc_spec is not None:
            list_cap, tab_cap, want_scores = proc_spec
            hist = torch.zeros((B, cap), device=dev, dtype=torch.int64)           # prompt ids; generated ids are read from tok_buf
            tables = torch.zeros((tab_cap,), device=dev, dtype=torch.int32)
            static_add = torch.zeros((lm.vocab,), device=dev, dtype=torch.float32)
            scores = torch.empty((B, lm.vocab), device=dev, dtype=torch.float32) if want_scores else None

        def select(logits, out):
            if proc_spec is None:
                return ops.argmax(logits, out=out)
            return ops.logits_process_argmax(logits, hist, tok_buf, gen_idx, tables, static_add, list_cap, out=out, scores=scores)

        use_pdl = os.environ.get("AF3_PDL", "1") != "0"

        def bookkeeping():
            ops.token_step(raw_ids, unfinished, eos_dev, ctl, tok_buf, gen_idx, ids_buf, done_flags)

        def eager():
            # programmatic dependent launch along the whole step: each kernel's prologue and the GEMMs' weight
            # prefetch overlap the tail of the kernel before it (the kernels order their dependent accesses themselves)
            _lib.load().af3_set_pdl(1 if use_pdl else 0)
            phase, ops.PHASE = ops.PHASE, "decode"
            try:
                bookkeeping()
                x, _ = ops.embed_scatter(ids_buf, table, -1, None, 0, 1, None)
                logits = lm.decode_step(x, cache, scratch)
                select(logits, am_out)
                return logits
            finally:
                ops.PHASE = phase
                _lib.load().af3_set_pdl(0)

        state = {"graph": None, "out": None, "warm": 0}

        class Step:
            """step() -> fp32 logits [B, V] of the next token: device-side bookkeeping of the current token, embedding gather, 28
            layers, head, argmax -- captured once in a CUDA graph when use_graph and replayed; positions advance on the device."""

            def begin(self_, first_ids, eos_list, pad_token_id):
                if eos_list is not None and len(eos_list) > self.MAX_EOS_IDS:
                    raise AF3Error(f"at most {self.MAX_EOS_IDS} eos_token_id values are supported")
                raw_ids.copy_(first_ids)
                unfinished.fill_(1)
                gen_idx.zero_()
                done_flags.zero_()
                n_eos = len(eos_list) if eos_list is not None else 0
                # scalar fills, not host-to-device copies: a copy from pageable memory would block the host until the queued
                # encoder + prefill work has drained (measured: 340 ms of lost run-ahead per generate() call)
                ctl[0:1].fill_(n_eos)
                ctl[1:2].fill_(int(pad_token_id) if pad_token_id is not None else 0)
                for j in range(n_eos):
                    eos_dev[j:j + 1].fill_(int(eos_list[j]))

            def load_processors(self_, input_ids, compiled):
                # staged through pinned memory: a pageable copy would block the host until the queued work drains (see begin)
                S = input_ids.shape[1]
                src = input_ids if input_ids.is_cuda else input_ids.pin_memory()
                hist[:, :S].copy_(src, non_blocking=True)
                tables[: compiled.tables.size].copy_(torch.from_numpy(compiled.tables).pin_memory(), non_blocking=True)
                static_add.copy_(torch.from_numpy(compiled.static_add).pin_memory(), non_blocking=True)

            def process(self_, logits):
                """Processed greedy selection of the first token (history = the prompt alone)."""
                gen_idx.zero_()
                return select(logits, None)

            def finish(self_):
                phase, ops.PHASE = ops.PHASE, "decode"
                try:
                    bookkeeping()
                finally:
                    ops.PHASE = phase

            def __call__(self_):
                if not use_graph:
                    return eager()
                if state["graph"] is None:
                    if state["warm"] < 1:  # first step eagerly (configures kernels, warms the allocator)
                        state["warm"] += 1
                        return eager()
                    g = torch.cuda.CUDAGraph()
                    torch.cuda.synchronize()
                    prof, ops.PROFILE = ops.PROFILE, None  # timing events cannot be recorded inside a capture
                    n0 = ops.LAUNCHES
                    t0 = len(ops.TRACE_LOG) if ops.TRACE_LOG is not None else 0
                    with torch.cuda.graph(g):
                        state["out"] = eager()
                    if ops.TRACE_LOG is not None:  # timeline tool: which trace-log entries are the captured step's launches
                        ops.TRACE_LOG.append(("graph_capture", t0, len(ops.TRACE_LOG)))
                    state["launches"] = ops.LAUNCHES - n0
                    ops.LAUNCHES = n0  # capture launched nothing; replays are counted below
                    ops.PROFILE = prof
                    state["graph"] = g
                state["graph"].replay()  # (capture does not execute: the first replay runs this token's step)
                ops._count(state["launches"])
                return state["out"]

        st = Step()
        st.tok_buf, st.done_flags = tok_buf, done_flags
        st.scores = scores if proc_spec is not None else None
        return st


class MusicFlamingoForConditionalGeneration(AudioFlamingo3ForConditionalGeneration):
    """Music Flamingo = the AF3 path + a rotary TIME embedding on the audio-tower output (SURVEY 8-f.3).
    Mirrors [O] transformers/models/musicflamingo/modular_musicflamingo.py:245-322 (same parameters / state_dict keys
    as AF3; the rotary buffers are non-persistent there and are recomputed here)."""

    def __init__(self, config):
        super().__init__(config)
        rp = config.rope_parameters
        if rp.get("rope_type", "default") != "default":
            raise AF3Error("only default rope parameters are implemented for the rotary time embedding")
        base = rp["rope_theta"]
        head_dim = _cfg_get(config, "head_dim", None) or config.audio_config.hidden_size
        dim = int(head_dim * rp.get("partial_rotary_factor", 1.0))
        # MoonshineRotaryEmbedding.compute_default_rope_parameters, evaluated on the CPU like the reference
        self._mf_inv_freq_cpu = 1.0 / (base ** (torch.arange(0, dim, 2, dtype=torch.int64).to(dtype=torch.float) / dim))
        self._mf_inv_freq = None
        self._mf_max_len = float(config.max_position_embeddings)
        self._mf_frame_step = config.audio_frame_step

    def _build_audio_timestamps(self, input_ids, post_lengths, max_post_length):
        """Start time (in seconds) of every pooled encoder frame, fp32 [W, max_post_length]: what the reference derives in
        [O] modular_musicflamingo.py:250-285.  A clip longer than 30 s is several consecutive windows feeding ONE run of <sound>
        placeholders; frame t of the k-th window of its clip starts at (k * max_post_length + t) * 4 * frame_step.
        Own formulation, sync-free (no torch.where / boolean indexing): every placeholder gets (its ordinal among all placeholders,
        the index of the run it belongs to); a window's run is looked up at the ordinal of its first frame, and k is the window
        index minus the first window index of that run."""
        dev = post_lengths.device
        is_audio = (input_ids == self.config.audio_token_id)                                  # [B, S]
        left_is_audio = torch.zeros_like(is_audio)
        left_is_audio[:, 1:] = is_audio[:, :-1]                                               # runs never continue across rows
        flat = is_audio.reshape(-1)
        n_pos = flat.numel()
        run_of_pos = torch.cumsum((is_audio & ~left_is_audio).reshape(-1).to(torch.long), 0) - 1
        ordinal_of_pos = torch.cumsum(flat.to(torch.long), 0) - 1
        # run index by placeholder ordinal; non-placeholder positions write into the spare last slot
        run_of_ordinal = torch.zeros((n_pos + 1,), device=dev, dtype=torch.long)
        run_of_ordinal.scatter_(0, torch.where(flat, ordinal_of_pos, torch.full_like(ordinal_of_pos, n_pos)), run_of_pos)
        W = post_lengths.shape[0]
        first_ordinal = torch.cumsum(post_lengths.to(torch.long), 0) - post_lengths.to(torch.long)
        run_of_window = run_of_ordinal[first_ordinal.clamp(max=n_pos - 1)]
        widx = torch.arange(W, device=dev, dtype=torch.long)
        first_window_of_run = torch.full((n_pos + 1,), W, device=dev, dtype=torch.long)
        first_window_of_run.scatter_reduce_(0, run_of_window, widx, reduce="amin", include_self=True)
        k = (widx - first_window_of_run[run_of_window]).to(torch.float32)
        step = self._mf_frame_step * 4
        frame_t = torch.arange(max_post_length, device=dev, dtype=torch.float32) * step
        return k.unsqueeze(1) * max_post_length * step + frame_t

    def _post_encoder(self, enc, W, Tp, input_features_mask, input_ids):
        if input_ids is None:
            raise AF3Error("Music Flamingo needs input_ids to place the audio windows in time (get_audio_features(..., input_ids=))")
        if self._mf_inv_freq is None or self._mf_inv_freq.device != enc.device:
            self._mf_inv_freq = self._mf_inv_freq_cpu.to(enc.device)
        lens = input_features_mask.sum(-1).to(torch.long)
        _, post = self.audio_tower._get_feat_extract_output_lengths(lens)
        ts = self._build_audio_timestamps(input_ids.to(enc.device), post, Tp).to(torch.float32).contiguous()
        window_duration = self._mf_frame_step * 4 * Tp
        return ops.rotary_time_emb(enc, ts, self._mf_inv_freq, W, Tp, window_duration, self._mf_max_len)
