"""The attention restatements of oracle/attention_oracle.py checked on the CPU: without rounding both reduce to the fp64
softmax, with rounding they stay inside the bound the GPU tests assert, split counts agree with each other, and the masks
are the ones transformers builds from the same attention_mask."""
import math

import pytest
import torch

from oracle import attention_oracle as A

bf16 = torch.bfloat16


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(bf16)


# (B, Tq, Tk, H, Hkv, D, scale, causal, kv_len, kv_start, profile): reduced versions of the GPU cases
PREFILL = [
    (2, 300, 300, 2, 2, 64, 1.0, False, [300, 129], None, "random"),          # encoder: scale folded into q
    (2, 260, 260, 2, 2, 64, 1.0, False, [128, 127], None, "edges"),
    (2, 200, 200, 7, 1, 128, 128 ** -0.5, True, None, [0, 129], "random"),    # decoder prefill, GQA 7
    (1, 300, 300, 2, 1, 128, 128 ** -0.5, True, None, [127], "edges"),
    (1, 260, 260, 2, 2, 128, 128 ** -0.5, True, None, None, "diagonal"),
    (2, 129, 400, 8, 1, 128, 128 ** -0.5, True, None, [0, 255], "random"),    # continuation chunk, GQA 8
    (1, 300, 300, 2, 1, 128, 128 ** -0.5, True, None, [5], "rising"),
    (1, 300, 300, 2, 1, 128, 128 ** -0.5, True, None, [5], "two_peaks"),
    (2, 5, 129, 2, 2, 128, 128 ** -0.5, False, [129, 40], None, "random"),     # cross-attention
]


def _prefill_inputs(B, Tq, Tk, H, Hkv, D, scale, causal, kv_len, kv_start, profile, seed=0):
    q = _rand((B, Tq, H, D), seed, 0.125 if scale == 1.0 else 1.0)
    k, v = _rand((B, Hkv, Tk, D), seed + 1), _rand((B, Hkv, Tk, D), seed + 2)
    for b in range(B):
        kb = k[b].transpose(0, 1)                                   # [Tk, Hkv, D] view
        if profile == "edges":
            n = kv_len[b] if kv_len else Tk
            s0 = kv_start[b] if kv_start else 0
            for hk in range(Hkv):
                A.edge_probe(q[b], k[b, hk], v[b, hk], scale, masked=[n] + ([s0 - 1] if kv_start else []),
                             visible=[n - 1] + ([s0] if kv_start else []))
        elif profile == "diagonal":
            A.diagonal_probe(q[b], kb, scale, Tk - Tq)
        elif profile != "random":
            s0 = kv_start[b] if kv_start else 0
            j = torch.arange(Tk, dtype=torch.float32)
            A.peak_scores(q[b], kb, profile, scale, s0 + Tk // 4, Tk - 1 if profile == "rising" else 3 * Tk // 4, j[:, None])
    return q, k, v


@pytest.mark.parametrize("case", PREFILL)
def test_prefill_restatement(case):
    B, Tq, Tk, H, Hkv, D, scale, causal, kv_len, kv_start, profile = case
    q, k, v = _prefill_inputs(*case)
    ref, bnd, smag, _ = A.softmax_attention_fp64(q, k, v, scale, causal, kv_len, kv_start)
    exact = A.prefill_tile_restatement(q, k, v, scale, causal, kv_len, kv_start, rounding=False)
    assert (exact - ref).abs().max().item() <= 1e-12 * max(1.0, bnd.max().item())
    got = A.prefill_tile_restatement(q, k, v, scale, causal, kv_len, kv_start).double()
    tol = A.attention_tolerance(ref, bnd, smag, D, Tk)
    assert ((got - ref).abs() <= tol).all(), ((got - ref).abs() / tol).max()


# (B, H, Hkv, Tmax, ctx, starts, profile)
DECODE = [
    (2, 28, 4, 512, 385, [0, 129], "random"),
    (2, 8, 1, 512, 257, [1, 128], "edges"),
    (1, 13, 1, 640, 600, [127], "rising"),
    (1, 16, 2, 640, 600, [5], "two_peaks"),
    (2, 9, 9, 256, 1, [0, 0], "random"),
]


def _decode_inputs(B, H, Hkv, Tmax, ctx, starts, profile, seed=10):
    scale = 128 ** -0.5
    q, k, v = _rand((B, H, 128), seed), _rand((B, Hkv, Tmax, 128), seed + 1), _rand((B, Hkv, Tmax, 128), seed + 2)
    for b in range(B):
        for hk in range(Hkv):
            if profile == "edges":
                A.edge_probe(q[b], k[b, hk], v[b, hk], scale, masked=[starts[b] - 1, ctx], visible=[starts[b], ctx - 1])
            elif profile != "random":
                A.peak_scores(q[b], k[b, hk], profile, scale, starts[b] + 3, ctx - 4, torch.arange(Tmax, dtype=torch.float32))
    return q, k, v, scale


@pytest.mark.parametrize("case", DECODE)
def test_decode_restatement(case):
    B, H, Hkv, Tmax, ctx, starts, profile = case
    q, k, v, scale = _decode_inputs(*case)
    ref, bnd, smag, _ = A.softmax_attention_fp64(q[:, None], k[:, :, :ctx], v[:, :, :ctx], scale, kv_start=starts)
    ref, bnd, smag = ref[:, 0], bnd[:, 0], smag[:, 0]
    outs = {}
    for nz in (1, 3, 4, 7):
        exact = A.decode_split_restatement(q, k, v, scale, ctx, starts, nz, rounding=False)
        assert (exact - ref).abs().max().item() <= 1e-12 * max(1.0, bnd.max().item()), nz
        got = A.decode_split_restatement(q, k, v, scale, ctx, starts, nz).double()
        assert ((got - ref).abs() <= A.attention_tolerance(ref, bnd, smag, 128, ctx)).all(), nz
        outs[nz] = got
    # one split against four: both within the bound of the fp64 softmax, so within twice of each other
    assert ((outs[1] - outs[4]).abs() <= 2 * A.attention_tolerance(ref, bnd, smag, 128, ctx)).all()


def test_probes_are_decisive():
    """A one-key leak or drop at a probed edge moves the fp64 output by far more than the bound."""
    q, k, v = _prefill_inputs(*PREFILL[1])
    ref, bnd, smag, _ = A.softmax_attention_fp64(q, k, v, 1.0, False, [128, 127])
    tol = A.attention_tolerance(ref, bnd, smag, 64, 260)
    for lens in ([129, 127], [127, 127], [128, 128], [128, 126]):
        moved = A.softmax_attention_fp64(q, k, v, 1.0, False, lens)[0]
        b = 0 if lens[0] != 128 else 1
        assert ((moved[b] - ref[b]).abs() > 16 * tol[b]).float().mean() > 0.9, lens
    q, k, v = _prefill_inputs(*PREFILL[4])
    scale = 128 ** -0.5
    ref, bnd, smag, _ = A.softmax_attention_fp64(q, k, v, scale, True)
    tol = A.attention_tolerance(ref, bnd, smag, 128, 260)
    vis = A.visible_mask(1, 260, 260, True)
    s = torch.einsum("bihd,bjhd->bhij", q.double(), k.transpose(1, 2).double()) * scale
    for moved_vis in (vis | torch.diag_embed(torch.ones(259, dtype=torch.bool), 1)[None],   # causal rule one key too wide
                      vis & ~torch.eye(260, dtype=torch.bool)[None]):                      # ... one key too narrow
        p = torch.softmax(s.masked_fill(~moved_vis[:, None], -math.inf), -1)
        moved = torch.nan_to_num(p).to(torch.float64) @ v.double()                       # [1, H, T, D]
        moved = moved.transpose(1, 2)
        rows = slice(1, 259)
        assert ((moved[0, rows] - ref[0, rows]).abs() > 16 * tol[0, rows]).float().mean() > 0.9


def _hf_mask(kind, attention_mask, T):
    """The boolean mask transformers builds (sdpa path) for this attention_mask: create_bidirectional_mask for the encoder's
    key padding (AF3M:337-351 -> MASK:1001-1087), create_causal_mask for the decoder's left padding (MASK:882)."""
    from transformers import Qwen2Config
    from transformers.masking_utils import create_bidirectional_mask, create_causal_mask

    cfg = Qwen2Config(hidden_size=64, num_attention_heads=2, num_key_value_heads=1, num_hidden_layers=1)
    cfg._attn_implementation = "sdpa"
    emb = torch.zeros((attention_mask.shape[0], T, 64))
    if kind == "encoder":
        m = create_bidirectional_mask(config=cfg, inputs_embeds=emb, attention_mask=attention_mask)
    else:
        m = create_causal_mask(config=cfg, inputs_embeds=emb, attention_mask=attention_mask, past_key_values=None,
                               position_ids=torch.arange(T)[None].expand(attention_mask.shape[0], T))
    return m


def test_masks_match_transformers():
    T = 300
    lens, starts = [300, 129, 1], [0, 127, 299]
    am = torch.stack([torch.arange(T) < n for n in lens]).long()
    m = _hf_mask("encoder", am, T)
    assert m is not None and m.dtype == torch.bool
    assert torch.equal(m[:, 0], A.visible_mask(3, T, T, False, kv_len=lens))
    am = torch.stack([torch.arange(T) >= s for s in starts]).long()
    m = _hf_mask("decoder", am, T)
    ours = A.visible_mask(3, T, T, True, kv_start=starts)
    assert torch.equal(m[:, 0], ours)
