"""ORACLE -- TEST INFRASTRUCTURE ONLY (like af3_oracle): a torch restatement of the FP8 decoder projections.

What it restates
----------------
FP8 = transformers/integrations/finegrained_fp8.py (transformers 5.5.0), the FineGrainedFP8 format with
weight_block_size = (128, 128):
  * weight quantization, Fp8Quantize.convert (FP8:801-865): per-block amax, scale = 448 / amax (1 for an all-zero block),
    q = e4m3(clamp(w * scale)), weight_scale_inv = 1 / scale;
  * dequantization, Fp8Dequantize.convert (FP8:873-905): q * weight_scale_inv of its block;
  * FP8Linear.forward (FP8:248-284): activations quantized per token and 128 columns, block-scaled matmul rounded to the
    input dtype (bf16), then the bias added and rounded again.
The activation rule is the project's (include/af3b200.h): s = amax / 448 (1 when amax == 0), q = e4m3(x / s).  The matmul is
evaluated as the promoted sum  sum_kb (sum_{k in kb} qx qw) * sx * sw  in fp64, where every 128-term partial sum of e4m3
products is exact.

FP8Linear.forward itself is never called: it fetches its matmul kernel from the Hugging Face hub.
"""
from __future__ import annotations

import copy

import torch
from torch import nn

FP8_MAX = 448.0
DECODER_PROJECTIONS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def quantize_weight(w: torch.Tensor):
    """Fp8Quantize.convert with 128 x 128 blocks -> (q e4m3 [rows, cols], weight_scale_inv fp32 [rows/128, cols/128])."""
    rows, cols = w.shape
    blocks = w.to(torch.float32).reshape(rows // 128, 128, cols // 128, 128)
    amax = blocks.abs().amax(dim=(1, 3))
    safe = torch.where(amax > 0, amax, torch.ones_like(amax))
    scale = torch.where(amax > 0, FP8_MAX / safe, torch.ones_like(amax))
    q = torch.clamp(blocks * scale[:, None, :, None], min=-FP8_MAX, max=FP8_MAX).to(torch.float8_e4m3fn)
    return q.reshape(rows, cols), (1.0 / scale).to(torch.float32)


def dequantize_weight(q: torch.Tensor, scale_inv: torch.Tensor) -> torch.Tensor:
    """Fp8Dequantize.convert: fp32 [rows, cols]."""
    rows, cols = q.shape
    return (q.to(torch.float32).reshape(rows // 128, 128, cols // 128, 128) * scale_inv[:, None, :, None]).reshape(rows, cols)


def quantize_activation(x: torch.Tensor):
    """The activation rule on bf16 values x [rows, K] -> (q e4m3 [rows, K], s fp32 [rows, K/128])."""
    rows, K = x.shape
    g = x.to(torch.bfloat16).to(torch.float32).reshape(rows, K // 128, 128)
    amax = g.abs().amax(-1)
    # tensor / tensor: torch divides by a Python scalar as a multiplication by its reciprocal, which is not the rule
    s = torch.where(amax > 0, amax / torch.full_like(amax, FP8_MAX), torch.ones_like(amax))
    q = (g / s[..., None]).to(torch.float8_e4m3fn)
    return q.reshape(rows, K), s


def promoted_matmul(qx, sx, qw, sw, absolute: bool = False) -> torch.Tensor:
    """sum_kb (sum_{k in kb} qx[t,k] qw[n,k]) * sx[t,kb] * sw[n/128,kb] in fp64 -> [rows, n].  absolute: the same sum over
    |qx| |qw| (the magnitude that bounds accumulation error)."""
    X = qx.to(torch.float64)
    W = qw.to(torch.float64)
    if absolute:
        X, W = X.abs(), W.abs()
    swr = sw.to(torch.float64).repeat_interleave(128, 0)  # [n, K/128]
    out = torch.zeros((X.shape[0], W.shape[0]), dtype=torch.float64, device=X.device)
    for b in range(X.shape[1] // 128):
        part = X[:, 128 * b:128 * (b + 1)] @ W[:, 128 * b:128 * (b + 1)].T
        out += part * sx[:, b, None].to(torch.float64) * swr[None, :, b]
    return out


def linear(x, qw, sw, bias=None) -> torch.Tensor:
    """FP8Linear.forward restated: bf16 result of the promoted matmul, plus bias rounded again.  -> bf16 [rows, n]."""
    qx, sx = quantize_activation(x)
    y = promoted_matmul(qx, sx, qw, sw).to(torch.float32).to(torch.bfloat16)
    if bias is not None:
        y = (y.float() + bias.to(torch.bfloat16).float()).to(torch.bfloat16)
    return y


class RefFP8Linear(nn.Module):
    """Drop-in for an nn.Linear of the reference model: bf16 inputs (the model's activations rounded to bf16), FP8 weights."""

    def __init__(self, lin: nn.Linear, q=None, s=None):
        super().__init__()
        if q is None:
            q, s = quantize_weight(lin.weight.detach().to(torch.bfloat16))
        self.q, self.s = q, s
        self.bias = None if lin.bias is None else lin.bias.detach().to(torch.bfloat16)

    def forward(self, x):
        shp = x.shape
        y = linear(x.reshape(-1, shp[-1]), self.q.to(x.device), self.s.to(x.device),
                   None if self.bias is None else self.bias.to(x.device))
        return y.to(x.dtype).reshape(*shp[:-1], y.shape[-1])


def fp8_reference_model(hf_model):
    """A copy of the HF model whose decoder projections are RefFP8Linear (weights quantized from their bf16 values, as a
    bf16 checkpoint is quantized at load)."""
    m = copy.deepcopy(hf_model)
    for layer in m.language_model.model.layers:
        for parent in (layer.self_attn, layer.mlp):
            for name in DECODER_PROJECTIONS:
                if hasattr(parent, name):
                    setattr(parent, name, RefFP8Linear(getattr(parent, name)))
    return m
