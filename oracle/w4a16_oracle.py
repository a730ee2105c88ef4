"""Restatement of the W4A16 weight format (include/af3b200.h af3_gemm_w4a16), written from the format's definition and
independently of audio_flamingo_b200.modeling:

  * group g of row n is W[n, 128g : 128g + 128]; amax = max |W| over it in fp32;
  * scale s[n, g] = bf16(amax / 7.5) (IEEE fp32 division, round to nearest even), 1 when amax == 0;
  * q[n, k] = clamp(round_half_even(fp32(W[n, k]) / fp32(s[n, k // 128])), -8, 7);
  * weight_packed int32 [N, K / 8]: bits 4j .. 4j + 3 of word i in row n hold q[n, 8i + j] + 8; weight_scale bf16 [N, K / 128];
  * Wd[n, k] = bf16(q[n, k] * s[n, k // 128]), one multiply rounded to nearest even.

w4a16_reference_model(hf_model) is the HF model with every decoder projection holding Wd: what a W4A16 model computes with.
"""
import copy

import numpy as np
import torch

PROJECTIONS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj", "mlp.up_proj",
               "mlp.down_proj")


def quantize(w):
    """w [N, K] -> (weight_packed int32 [N, K / 8], weight_scale bf16 [N, K / 128]), on the CPU."""
    w = w.detach().to("cpu", torch.float32)
    N, K = w.shape
    scales = np.empty((N, K // 128), dtype=np.float32)
    q = np.empty((N, K), dtype=np.int64)
    wn = w.numpy()
    for g in range(K // 128):
        blk = wn[:, 128 * g:128 * g + 128]
        amax = np.abs(blk).max(axis=1)
        s = np.where(amax == 0, np.float32(1.0), amax / np.float32(7.5)).astype(np.float32)
        s = torch.from_numpy(s).to(torch.bfloat16).to(torch.float32).numpy()   # round to bf16, nearest even
        scales[:, g] = s
        q[:, 128 * g:128 * g + 128] = np.clip(np.rint(blk / s[:, None]), -8, 7).astype(np.int64)  # rint: half to even
    u = (q + 8).reshape(N, K // 8, 8)
    words = np.zeros((N, K // 8), dtype=np.uint32)
    for j in range(8):
        words |= (u[:, :, j].astype(np.uint32) << np.uint32(4 * j))
    return torch.from_numpy(words.view(np.int32).copy()), torch.from_numpy(scales).to(torch.bfloat16)


def unpack(packed):
    """weight_packed int32 [N, K / 8] -> q int64 [N, K] in [-8, 7]."""
    words = packed.detach().cpu().numpy().view(np.uint32)
    N, W = words.shape
    q = np.empty((N, W, 8), dtype=np.int64)
    for j in range(8):
        q[:, :, j] = ((words >> np.uint32(4 * j)) & np.uint32(15)).astype(np.int64) - 8
    return torch.from_numpy(q.reshape(N, W * 8))


def dequantize(packed, scale):
    """-> Wd bf16 [N, K] = bf16(q * s) (the product of a 4-bit integer and a bf16 scale is exact in fp32: one rounding)."""
    q = unpack(packed).to(torch.float32)
    s = scale.detach().cpu().to(torch.float32)
    return (q * torch.repeat_interleave(s, 128, dim=1)).to(torch.bfloat16)


def w4a16_reference_model(hf_model):
    """A copy of the HF model whose decoder projections hold Wd of their bf16 weights (the model's own dtype otherwise)."""
    m = copy.deepcopy(hf_model)
    for layer in m.language_model.model.layers:
        for name in PROJECTIONS:
            lin = layer.get_submodule(name)
            wd = dequantize(*quantize(lin.weight.detach().to(torch.bfloat16)))
            with torch.no_grad():
                lin.weight.copy_(wd.to(lin.weight.dtype))
    return m
