"""SURVEY 8-f.4 (AF2's LM-side conditioning): the gated cross-attention + gated dense block on the H100 kernels vs the executable
analogue of that operator, transformers' IdeficsGatedCrossAttentionLayer ([O] idefics/modeling_idefics.py:684-806), run in bf16 on
the same GPU and in fp32 on the CPU (same seeded weights).  AF2 itself stays unpinned: see oracle/af2_oracle.py.
Tolerance: bf16 outputs of O(1..5); ours must not be further from fp32 than 1.5x the analogue's own bf16 run (floor 2 % of max |ref|)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


@pytest.mark.parametrize("alpha_type,dims,B,T,Tm,media_len", [
    ("vector", dict(), 3, 200, 300, [300, 129, 5]),                                   # head_dim 128
    ("float", dict(hidden_size=256, num_attention_heads=4, intermediate_size=384, media_dim=128), 2, 77, 40, [40, 17]),   # head_dim 64
    ("vector", dict(hidden_size=1024, num_attention_heads=8, intermediate_size=2816, media_dim=2048), 2, 512, 1500, [1500, 900]),
])
def test_gated_cross_attention_layer_matches_the_analogue(alpha_type, dims, B, T, Tm, media_len):
    from oracle import af2_oracle as A

    from audio_flamingo_b200.xattn import GatedCrossAttentionLayer

    ref32 = A.hf_gated_layer(seed=3, alpha_type=alpha_type, **dims)
    hid, md = ref32.hidden_size, ref32.cross_attn.k_proj.in_features
    g = torch.Generator().manual_seed(4)
    h = torch.randn(B, T, hid, generator=g).to(bf16)
    m = torch.randn(B, Tm, md, generator=g).to(bf16)
    gate = torch.ones(B, T)
    gate[0, 1] = 0
    gate[-1, T // 2:] = 0
    mask = A.key_padding_mask(B, T, media_len, Tm)
    ours = GatedCrossAttentionLayer.from_reference(ref32, device="cuda")
    assert set(ours.state_dict()) == set(ref32.state_dict())
    with torch.no_grad():
        r32 = ref32(h.float(), image_hidden_states=m.float(), image_attention_mask=mask, cross_attention_gate=gate)
        ref16 = A.hf_gated_layer(seed=3, alpha_type=alpha_type, **dims).to("cuda", bf16)
        r16 = ref16(h.cuda(), image_hidden_states=m.cuda(), image_attention_mask=mask.cuda().to(bf16), cross_attention_gate=gate.cuda()).float().cpu()
    o_len = ours(h.cuda(), image_hidden_states=m.cuda(), media_len=media_len, cross_attention_gate=gate.cuda()).float().cpu()
    o_mask = ours(h.cuda(), image_hidden_states=m.cuda(), image_attention_mask=mask.cuda(), cross_attention_gate=gate.cuda()).float().cpu()
    assert torch.equal(o_len, o_mask)
    e_ours, e_ref = (o_len - r32).abs().max().item(), (r16 - r32).abs().max().item()
    print(f"gated xattn [{alpha_type}, hid {hid}]: ours-vs-fp32 {e_ours:.4f}, analogue-bf16-vs-fp32 {e_ref:.4f}, max |ref| {r32.abs().max().item():.2f}")
    assert e_ours <= max(1.5 * e_ref, 0.02 * r32.abs().max().item())
    # a mask that is not a key-padding prefix is refused, not silently mis-applied
    from audio_flamingo_b200 import AF3Error

    bad = mask.clone()
    bad[0, 0, 3, 0] = torch.finfo(torch.float32).min
    with pytest.raises(AF3Error):
        ours(h.cuda(), image_hidden_states=m.cuda(), image_attention_mask=bad.cuda())


def test_gated_residual_kernel_rounding_points():
    from audio_flamingo_b200 import ops

    torch.manual_seed(0)
    r, y, a = torch.randn(37, 256).to(bf16).cuda(), torch.randn(37, 256).to(bf16).cuda(), (torch.randn(256) * 0.7).to(bf16).cuda()
    gate = (torch.arange(37) % 3 != 0).to(torch.int32).cuda()
    out = ops.gated_residual(r, y, a, row_gate=gate)
    ref = r + torch.tanh(a) * (y * gate[:, None].to(bf16))          # torch's own bf16 ops: one rounding per op
    assert torch.equal(out, ref)
    out_s = ops.gated_residual(r, y, a[:1].contiguous())
    assert torch.equal(out_s, r + torch.tanh(a[:1]) * y)
