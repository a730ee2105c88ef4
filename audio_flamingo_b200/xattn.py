"""Flamingo-style gated cross-attention + gated dense block on the sm_90a kernels (SURVEY.md 8-f.4, BASELINE config 4).

Audio Flamingo 2 conditions a frozen decoder on sliding-window audio features through such blocks placed before the decoder
layers (arXiv 2503.03983, after Flamingo, arXiv 2204.14198).  The `audio_flamingo_2` branch is NOT in the mounted reference and
no AF2 code exists in the container, so AF2 itself cannot be pinned.  What IS executable here is the same operator in the
installed transformers package -- `IdeficsGatedCrossAttentionLayer` ([O] models/idefics/modeling_idefics.py:684-806), the
structural analogue SURVEY.md names -- and this module mirrors exactly that layer: same parameter names / state_dict, same
forward arguments, parity-tested against it (tests/test_xattn_gpu.py).  Status of row f4 therefore: the LM-side operator is built
and pinned against an executable implementation of the operator family; the AF-CLAP sliding-window encoder and AF2's own wiring
are not built (no reference to pin against).

    x  = x + tanh(alpha_cross_attn) * CrossAttn(RMSNorm(x), media)      media rows beyond media_len are masked keys
    x  = x + tanh(alpha_dense)      * W_down(silu(W_gate RMSNorm(x)) * W_up RMSNorm(x))

All arithmetic runs in libaf3b200.so: af3_rmsnorm, af3_gemm_bf16 (q / fused k,v / o / fused SwiGLU / down), af3_attention
(non-causal, Tq != Tk, key-padding mask) and af3_gated_residual.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from ._lib import AF3Error

bf16 = torch.bfloat16


class _XAttn(nn.Module):
    def __init__(self, hidden, heads, media_dim):
        super().__init__()
        d = hidden // heads
        self.q_proj = nn.Linear(hidden, heads * d, bias=False)
        self.k_proj = nn.Linear(media_dim, heads * d, bias=False)
        self.v_proj = nn.Linear(media_dim, heads * d, bias=False)
        self.o_proj = nn.Linear(heads * d, hidden, bias=False)


class _MLP(nn.Module):
    def __init__(self, hidden, inter):
        super().__init__()
        self.gate_proj = nn.Linear(hidden, inter, bias=False)
        self.down_proj = nn.Linear(inter, hidden, bias=False)
        self.up_proj = nn.Linear(hidden, inter, bias=False)


class _Norm(nn.Module):
    def __init__(self, hidden):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden))


class GatedCrossAttentionLayer(nn.Module):
    """Drop-in for the reference analogue's layer ([O] idefics/modeling_idefics.py:684-806) on its inference path."""

    def __init__(self, hidden_size, num_attention_heads, intermediate_size, media_dim, rms_norm_eps=1e-6, alpha_type="vector"):
        super().__init__()
        self.hidden, self.heads, self.inter, self.media_dim, self.eps = hidden_size, num_attention_heads, intermediate_size, media_dim, rms_norm_eps
        self.head_dim = hidden_size // num_attention_heads
        if self.head_dim not in (64, 128):
            raise AF3Error("head_dim must be 64 or 128 for the wgmma attention kernel")
        if alpha_type not in ("vector", "float"):
            raise AF3Error("alpha_type must be 'vector' or 'float'")
        self.cross_attn = _XAttn(hidden_size, num_attention_heads, media_dim)
        self.mlp = _MLP(hidden_size, intermediate_size)
        self.input_layernorm = _Norm(hidden_size)
        self.post_attention_layernorm = _Norm(hidden_size)
        shape = (1, 1, hidden_size) if alpha_type == "vector" else (1,)
        self.alpha_cross_attn = nn.Parameter(torch.zeros(shape))
        self.alpha_dense = nn.Parameter(torch.zeros(shape))
        self._packed = None

    @classmethod
    def from_reference(cls, ref_layer, device="cuda"):
        """Build from an instantiated reference-analogue layer (weights copied, cast to bf16)."""
        ca = ref_layer.cross_attn
        if getattr(ca, "qk_layer_norms", False):
            raise AF3Error("qk_layer_norms=True is not implemented")
        m = cls(ref_layer.hidden_size, ca.num_heads, ref_layer.mlp.gate_proj.out_features, ca.k_proj.in_features,
                ref_layer.input_layernorm.variance_epsilon, "vector" if ref_layer.alpha_dense.numel() > 1 else "float")
        m.to(device=device, dtype=bf16)
        sd = ref_layer.state_dict()
        own = m.state_dict()
        if set(sd) != set(own):
            raise AF3Error(f"state_dict mismatch: {sorted(set(sd) ^ set(own))[:4]}")
        with torch.no_grad():
            for k, v in own.items():
                v.copy_(sd[k].to(device=v.device, dtype=bf16))
        return m

    def pack_weights(self):
        ca, m = self.cross_attn, self.mlp
        wkv = torch.cat([ca.k_proj.weight.detach(), ca.v_proj.weight.detach()], 0).contiguous()
        ca.k_proj.weight.data, ca.v_proj.weight.data = wkv[: self.hidden], wkv[self.hidden:]          # views: one copy in HBM
        self._concat = self.inter % 128 == 0
        if self._concat:
            wgu = torch.cat([m.gate_proj.weight.detach(), m.up_proj.weight.detach()], 0).contiguous()
            m.gate_proj.weight.data, m.up_proj.weight.data = wgu[: self.inter], wgu[self.inter:]
        else:
            wgu = ops.pack_gate_up(m.gate_proj.weight.detach().contiguous(), m.up_proj.weight.detach().contiguous())
        self._packed = (wkv, wgu)

    @torch.no_grad()
    def forward(self, hidden_states, image_hidden_states=None, image_attention_mask=None, cross_attention_gate=None, media_len=None, **kw):
        """hidden_states [B, T, hidden] bf16; image_hidden_states (the media / audio-window features) [B, Tm, media_dim] bf16.
        Masking: `media_len` int [B] = valid media rows per sequence (keys beyond are masked for every query).  The reference's
        general additive `image_attention_mask` [B, 1, T, Tm] is accepted only when it is exactly such a key-padding mask.
        cross_attention_gate [B, T]: 0 -> the token attends to no media and its cross-attention output is zeroed (idefics:797)."""
        p = self.cross_attn.q_proj.weight
        if not p.is_cuda or p.dtype != bf16:
            raise AF3Error("layer must be on a CUDA device in bfloat16; no CPU fallback")
        if image_hidden_states is None:
            raise ValueError("`image_hidden_states` (the media features to condition on) is required")     # idefics:776
        if self._packed is None:
            self.pack_weights()
        with torch.cuda.device(p.device):
            B, T, hid = hidden_states.shape
            Tm = image_hidden_states.shape[1]
            H, D = self.heads, self.head_dim
            if image_attention_mask is not None:
                am = image_attention_mask
                visible = (am[:, 0] == 0) if am.dtype.is_floating_point else am[:, 0].bool()          # [B, T, Tm]
                n_vis = visible[:, 0].sum(-1)
                prefix = torch.arange(Tm, device=am.device)[None, :] < n_vis[:, None]
                if not bool((visible == prefix[:, None, :]).all()):
                    raise AF3Error("only key-padding media masks (a prefix of valid media rows, the same for every query) are implemented")
                media_len = n_vis
            kv_len = None if media_len is None else torch.as_tensor(media_len, device=p.device).to(torch.int32).contiguous()
            x = hidden_states.to(p.device, bf16).reshape(B * T, hid).contiguous()
            media = image_hidden_states.to(p.device, bf16).reshape(B * Tm, self.media_dim).contiguous()
            gate_rows = None
            if cross_attention_gate is not None:
                gate_rows = (cross_attention_gate.to(p.device).reshape(-1) != 0).to(torch.int32).contiguous()
            wkv, wgu = self._packed
            y = ops.rmsnorm(x, self.input_layernorm.weight, self.eps)                                          # idefics:789
            q = ops.linear(y, self.cross_attn.q_proj.weight)
            kv = ops.linear(media, wkv)                                                                        # [B*Tm, 2*H*D]
            a = torch.empty((B, T, H * D), device=p.device, dtype=bf16)
            ops.attention(q, kv, kv[:, H * D:], a, B=B, H=H, Hkv=H, D=D, Tq=T, Tk=Tm, scale=D ** -0.5, causal=False, kv_layout=0,
                          ldq=H * D, ldk=2 * H * D, kv_len=kv_len)                                             # idefics:792-795
            o = ops.linear(a.view(B * T, H * D), self.cross_attn.o_proj.weight)
            x = ops.gated_residual(x, o, self.alpha_cross_attn.reshape(-1), row_gate=gate_rows)               # idefics:797-798
            y = ops.rmsnorm(x, self.post_attention_layernorm.weight, self.eps, out=y)
            g = ops.swiglu_linear(y, wgu, self.inter, concat=self._concat)                                     # idefics:803
            d = ops.linear(g, self.mlp.down_proj.weight)
            x = ops.gated_residual(x, d, self.alpha_dense.reshape(-1), out=x)                                  # idefics:805
            return x.view(B, T, hid)

    __call__ = forward
