"""Per-kernel parity on the GPU: each C-ABI kernel against a plain torch fp32 restatement of the same op with the
reference's bf16 rounding points (tolerances stated per test)."""

import numpy as np
import pytest
import torch
from test_cuda_core_kernels_gpu import logmel_reference, rope_reference
from test_attention_kernels_gpu import (BIDIRECTIONAL, CAUSAL, CONTINUATION, DECODE_PORTED, bidirectional_case, causal_case,
                                        check_decode, check_prefill, ported_decode_case)

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from audio_flamingo_b200 import ops as _ops

    return _ops


def _rand(shape, scale=1.0, seed=0, dtype=bf16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _close(got, ref, rtol, atol, what=""):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} out of tolerance, max err {err.max().item():.4g}, ref absmax {ref.abs().max().item():.4g}"


# bf16 output: 1 ulp = 2^-8 relative; accumulation-order differences in fp32 are far below that, so results may
# differ from the torch restatement only where the fp32 value sits next to a bf16 rounding boundary (<= 1 ulp).
BF16_RTOL = 2 ** -7


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (300, 512, 192), (1024, 1280, 1280), (257, 96, 320), (4000, 3840, 384)])
def test_gemm_plain(ops, M, N, K):
    x, w = _rand((M, K), 1.0, 1), _rand((N, K), 0.05, 2)
    out = ops.linear(x, w)
    ref = (x.float() @ w.float().T).to(bf16)
    _close(out, ref, BF16_RTOL, 1e-3, f"gemm {M}x{N}x{K}")


def test_gemm_unaligned_output_fallback(ops):
    """Output pitch not a multiple of 8 elements: the smem/TMA-store epilogue is not applicable, the generic direct-store
    epilogue (run-time flags) must still be exact."""
    M, N, K = 130, 100, 64
    x, w, b = _rand((M, K), 1.0, 17), _rand((N, K), 0.1, 18), _rand((N,), 0.5, 19)
    out = ops.linear(x, w, b, gelu=True)
    ref = torch.nn.functional.gelu((x.float() @ w.float().T + b.float()).to(bf16).float()).to(bf16)
    _close(out, ref, BF16_RTOL, 2e-3, "unaligned N")
    out32 = ops.linear(x[:20], w, b)  # few-token path with an odd feature count
    ref32 = (x[:20].float() @ w.float().T + b.float()).to(bf16)
    _close(out32, ref32, BF16_RTOL, 2e-3, "unaligned N (few tokens)")


@pytest.mark.parametrize("M", [1, 7, 32, 33, 64])
@pytest.mark.parametrize("N,K", [(256, 128), (3584, 512), (200, 64), (3584, 3584), (512, 4096), (96, 64), (4608, 1280)])
def test_gemm_swap_small_m(ops, M, N, K):
    x, w, b = _rand((M, K), 1.0, 3), _rand((N, K), 0.05, 4), _rand((N,), 0.5, 5)
    out = ops.linear(x, w, b)
    ref = (x.float() @ w.float().T + b.float()).to(bf16)
    _close(out, ref, BF16_RTOL, 1e-3, f"swap gemm {M}x{N}x{K}")


def test_gemm_splitk_deterministic_and_epilogue(ops):
    """Decode-shaped GEMM (32 tokens, 3584 x 18944 down projection + residual): split-K partials are reduced in a fixed
    order by the last CTA, so repeated launches are bit-identical; result matches the fp32 restatement."""
    M, N, K = 32, 3584, 18944
    x, w, res = _rand((M, K), 1.0, 14), _rand((N, K), 0.02, 15), _rand((M, N), 1.0, 16)
    outs = [ops.linear(x, w, resid=res) for _ in range(5)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    lin = (x.float() @ w.float().T).to(bf16).float()
    ref = (lin + res.float()).to(bf16)
    # one bf16 ulp of the (larger) linear output may survive the residual add even where lin + res cancels
    err = (outs[0].float() - ref.float()).abs()
    tol = 4e-3 + BF16_RTOL * (lin.abs() + res.float().abs())
    # Where the fp32 accumulator sits on a bf16 rounding tie of lin, another summation order rounds lin one ulp the other way and
    # the second rounding (after the residual add) can turn that into two ulps of the output.  Such elements must be rare and
    # exactly the reference's two roundings applied to this kernel's own linear output, itself within one ulp of lin.
    off = err > tol
    assert int(off.sum()) <= 8, f"{int(off.sum())} elements out of tolerance, max err {err.max().item()}"
    if off.any():
        lin_k = ops.linear(x, w).float()
        assert torch.equal(outs[0][off], (lin_k[off] + res.float()[off]).to(bf16)), "fused residual epilogue != its unfused chain"
        assert ((lin_k - lin).abs()[off] <= BF16_RTOL * lin.abs()[off]).all(), f"max err {err.max().item()}"


@pytest.mark.parametrize("M", [16, 640])
def test_gemm_epilogues(ops, M):
    N, K = 512, 256
    x, w, b = _rand((M, K), 1.0, 6), _rand((N, K), 0.06, 7), _rand((N,), 0.5, 8)
    res = _rand((M, N), 1.0, 9)
    acc = x.float() @ w.float().T
    lin = (acc + b.float()).to(bf16)
    # bias + GELU(erf)
    out = ops.linear(x, w, b, gelu=True)
    ref = torch.nn.functional.gelu(lin.float()).to(bf16)
    _close(out, ref, BF16_RTOL, 2e-3, "bias+gelu")
    # bias + residual
    out = ops.linear(x, w, b, resid=res)
    ref = (lin.float() + res.float()).to(bf16)
    _close(out, ref, BF16_RTOL, 4e-3, "bias+resid")
    # gelu + periodic residual (positional embedding add)
    period = 8
    pos = _rand((period, N), 1.0, 10)
    out = ops.linear(x, w, b, gelu=True, resid=pos, res_period=period)
    ref = (torch.nn.functional.gelu(lin.float()).to(bf16).float() + pos.float().repeat(M // period, 1)).to(bf16)
    _close(out, ref, 2 * BF16_RTOL, 4e-3, "gelu+pos")  # two chained bf16 roundings: up to 2 ulp
    # fp32 out of bf16-rounded values (lm_head)
    out = ops.linear(x, w, out_f32=True)
    ref = acc.to(bf16).float()
    _close(out, ref, BF16_RTOL, 1e-3, "f32out")
    assert out.dtype == torch.float32


@pytest.mark.parametrize("M", [1, 20, 32, 50, 64])
def test_gemm_few_token_epilogues(ops, M):
    """bias / GELU / residual epilogues of the few-token (split-K) kernel at the o-projection's shape class, against the fp32 restatement;
    repeated launches are bit-identical (no atomics, fixed reduction order)."""
    N, K = 3584, 3584
    x, w, b = _rand((M, K), 1.0, 80), _rand((N, K), 0.02, 81), _rand((N,), 0.5, 82)
    res = _rand((M, N), 1.0, 83)
    lin = (x.float() @ w.float().T + b.float()).to(bf16)
    out = ops.linear(x, w, b, resid=res)
    assert torch.equal(out, ops.linear(x, w, b, resid=res))
    err = (out.float() - (lin.float() + res.float()).to(bf16).float()).abs()
    assert (err <= 4e-3 + BF16_RTOL * (lin.float().abs() + res.float().abs())).all(), f"bias+resid max err {err.max().item()}"
    _close(ops.linear(x, w, b, gelu=True), torch.nn.functional.gelu(lin.float()).to(bf16), BF16_RTOL, 2e-3, "bias+gelu")
    _close(ops.linear(x, w), (x.float() @ w.float().T).to(bf16), BF16_RTOL, 1e-3, "plain")


@pytest.mark.parametrize("M", [8, 500])
@pytest.mark.parametrize("F", [128, 384, 200])
def test_gemm_swiglu(ops, M, F):
    K = 256
    x, g, u = _rand((M, K), 1.0, 11), _rand((F, K), 0.08, 12), _rand((F, K), 0.08, 13)
    packed = ops.pack_gate_up(g, u)
    out = ops.swiglu_linear(x, packed, F)
    gate = (x.float() @ g.float().T).to(bf16)
    up = (x.float() @ u.float().T).to(bf16)
    ref = (torch.nn.functional.silu(gate.float()).to(bf16).float() * up.float()).to(bf16)
    _close(out, ref, 2 * BF16_RTOL, 2e-3, f"swiglu M={M} F={F}")
    if F % 128 == 0:
        # [gate; up] layout (the two nn.Linear weights as views of one matrix): same tiles, same arithmetic -> bit-identical
        out_c = ops.swiglu_linear(x, torch.cat([g, u], 0).contiguous(), F, concat=True)
        assert torch.equal(out_c, out)


def test_layernorm_and_pool(ops):
    rows, dim = 333, 1280
    x, g, b = _rand((rows, dim), 2.0, 20), _rand((dim,), 1.0, 21), _rand((dim,), 0.3, 22)
    out = ops.layernorm(x, g, b)
    ref = torch.nn.functional.layer_norm(x.float(), (dim,), g.float(), b.float(), 1e-5).to(bf16)
    _close(out, ref, BF16_RTOL, 4e-3, "layernorm")
    n_win, T = 3, 50
    x = _rand((n_win * T, dim), 2.0, 23)
    out = ops.avgpool_layernorm(x, n_win, T, g, b)
    pooled = torch.nn.functional.avg_pool1d(x.view(n_win, T, dim).permute(0, 2, 1).float(), 2, 2).to(bf16).permute(0, 2, 1)
    ref = torch.nn.functional.layer_norm(pooled.float(), (dim,), g.float(), b.float(), 1e-5).to(bf16).reshape(-1, dim)
    _close(out, ref, BF16_RTOL, 4e-3, "avgpool+layernorm")


def test_rmsnorm(ops):
    rows, dim = 77, 3584
    x, w = _rand((rows, dim), 3.0, 24), _rand((dim,), 1.0, 25)
    out = ops.rmsnorm(x, w, 1e-6)
    h = x.float()
    h = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + 1e-6)
    ref = w * h.to(bf16)
    _close(out, ref, BF16_RTOL, 1e-3, "rmsnorm")
    idx = torch.tensor([5, 0, 76], dtype=torch.int32, device="cuda")
    out2 = ops.rmsnorm(x, w, 1e-6, row_idx=idx)
    assert torch.equal(out2, out[idx.long()])


def test_im2col(ops):
    n_win, C, T = 2, 128, 300
    x = _rand((n_win, C, T), 1.0, 26, torch.float32)
    cols = ops.im2col_conv1(x)
    xp = torch.nn.functional.pad(x.to(bf16), (1, 1))
    ref = torch.stack([xp[:, :, kk:kk + T] for kk in range(3)], dim=1)  # [w, kk, c, t]
    ref = ref.permute(0, 3, 1, 2).reshape(n_win * T, 3 * C)
    assert torch.equal(cols, ref)
    h = _rand((n_win * T, 64), 1.0, 27)
    cols2 = ops.im2col_conv2(h, n_win, T)
    hp = torch.nn.functional.pad(h.view(n_win, T, 64), (0, 0, 1, 1))
    T_out = (T - 1) // 2 + 1
    ref2 = torch.stack([hp[:, kk:kk + 2 * T_out:2, :] for kk in range(3)], dim=2).reshape(n_win * T_out, 3 * 64)
    assert torch.equal(cols2, ref2)


def test_conv_stem_as_gemm(ops):
    """conv1d(k3,p1)+GELU and conv1d(k3,s2,p1)+GELU through im2col + wgmma GEMM vs F.conv1d."""
    n_win, C, T, Dm = 2, 128, 200, 256
    x = _rand((n_win, C, T), 1.0, 28, torch.float32)
    w1, b1 = _rand((Dm, C, 3), 0.05, 29), _rand((Dm,), 0.1, 30)
    w2, b2 = _rand((Dm, Dm, 3), 0.03, 31), _rand((Dm,), 0.1, 32)
    w1p = w1.permute(0, 2, 1).reshape(Dm, 3 * C).contiguous()
    w2p = w2.permute(0, 2, 1).reshape(Dm, 3 * Dm).contiguous()
    h1 = ops.linear(ops.im2col_conv1(x), w1p, b1, gelu=True)
    ref1 = torch.nn.functional.gelu(torch.nn.functional.conv1d(x.to(bf16).float(), w1.float(), b1.float(), padding=1).to(bf16).float()).to(bf16)
    _close(h1.view(n_win, T, Dm).permute(0, 2, 1), ref1, BF16_RTOL, 2e-3, "conv1")
    h2 = ops.linear(ops.im2col_conv2(h1, n_win, T), w2p, b2, gelu=True)
    ref2 = torch.nn.functional.gelu(torch.nn.functional.conv1d(h1.view(n_win, T, Dm).permute(0, 2, 1).float(), w2.float(), b2.float(), stride=2, padding=1).to(bf16).float()).to(bf16)
    _close(h2.view(n_win, T // 2, Dm).permute(0, 2, 1), ref2, BF16_RTOL, 2e-3, "conv2")


@pytest.fixture(params=["v2", "v1"])
def attn_impl(request, monkeypatch):
    """Both row tilings of the prefill / encoder attention kernel go through the same parity cases: v2 (two consumer warpgroups,
    128 query rows per CTA = the default) and v1 (one warpgroup, 64 rows per CTA: AF3_ATTN_V1=1, kept as cross-check).
    check_prefill runs both and requires identical bits; the parameter keeps the two halves of the case list apart."""
    monkeypatch.setenv("AF3_ATTN_V1", "1" if request.param == "v1" else "0")
    return request.param


# The attention tests below run their cases through the checks of test_attention_kernels_gpu.py: the fp64 softmax bound, one
# bf16 ulp from the tile / split restatement, a bit-identical floor, identical bits for both row tilings, poisoned memory the
# kernel must mask, and output margins.
@pytest.mark.parametrize("D,H,T,lens", BIDIRECTIONAL)
def test_attention_bidirectional(ops, attn_impl, monkeypatch, D, H, T, lens):
    check_prefill(ops, monkeypatch, bidirectional_case(D, H, T, lens))


@pytest.mark.parametrize("T,starts,scores", CAUSAL)
def test_attention_causal_gqa_cache(ops, attn_impl, monkeypatch, T, starts, scores):
    check_prefill(ops, monkeypatch, causal_case(T, starts, scores))


def test_rope_kv_append(ops):
    B, T, H, Hkv, D, Tmax = 2, 50, 4, 2, 128, 128
    theta = 1e6
    qkv = _rand((B * T, (H + 2 * Hkv) * D), 1.0, 42)
    orig = qkv.clone()
    k_cache = torch.zeros((B, Hkv, Tmax, D), device="cuda", dtype=bf16)
    v_cache = torch.zeros_like(k_cache)
    inv_freq = (1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()
    starts = torch.tensor([0, 9], dtype=torch.int32, device="cuda")
    ops.rope_kv_append(qkv, k_cache, v_cache, B=B, T=T, H=H, Hkv=Hkv, D=D, pos0=0, inv_freq=inv_freq, kv_start=starts)
    q_ref, k_ref, v_ref = rope_reference(orig, B, T, H, Hkv, D, 0, inv_freq, starts)
    got = qkv.view(B, T, H + 2 * Hkv, D)
    assert (got[:, :, :H].float() - q_ref.float()).abs().max().item() <= 2 ** -6 * q_ref.float().abs().max().item()
    frac_exact = (got[:, :, :H] == q_ref).float().mean().item()
    assert frac_exact > 0.999, frac_exact  # bit-exact except where fp32 sin/cos differ in the last ulp
    assert (k_cache[:, :, :T].transpose(1, 2) == k_ref).float().mean().item() > 0.999
    assert torch.equal(v_cache[:, :, :T].transpose(1, 2), v_ref)


@pytest.mark.parametrize("B,H,Hkv,Tmax,ctx,starts,splits,scores", DECODE_PORTED)
def test_decode_attention(ops, monkeypatch, B, H, Hkv, Tmax, ctx, starts, splits, scores):
    check_decode(ops, monkeypatch, ported_decode_case(B, H, Hkv, Tmax, ctx, starts, splits, scores))


def test_embed_scatter_and_argmax(ops):
    V, dim, n_win, frames = 1000, 256, 3, 20
    table = _rand((V, dim), 1.0, 46)
    audio = _rand((n_win * frames, dim), 1.0, 47)
    post = torch.tensor([20, 7, 13], dtype=torch.int32, device="cuda")
    aid = 999
    g = torch.Generator().manual_seed(48)
    ids = torch.randint(0, 900, (2, 60), generator=g)
    ids[0, 5:25] = aid          # 20 audio tokens
    ids[1, 30:50] = aid         # 7 + 13
    ids = ids.cuda()
    out, counts = ops.embed_scatter(ids.reshape(-1), table, aid, audio, n_win, frames, post)
    ref = table[ids.reshape(-1)].clone()
    valid = (torch.arange(frames, device="cuda")[None, :] < post[:, None]).reshape(-1)
    ref[(ids.reshape(-1) == aid)] = audio[valid]
    assert torch.equal(out, ref)
    assert counts.tolist() == [40, 40]
    logits = torch.randn((5, 152064), device="cuda")
    logits[2, 777] = logits[2, 90000] = 50.0  # tie -> first index
    got = ops.argmax(logits)
    assert torch.equal(got, logits.argmax(-1))
    assert got[2].item() == 777


def test_logmel_vs_fp64(ops):
    """Log-mel kernel vs an fp64 numpy restatement of WFE:135-164 (exact DFT); tolerance 1e-4 abs on the
    (x+4)/4 scale at fp32 (the reference quotes 1e-5 between its own torch and numpy paths on speech)."""
    from transformers.audio_utils import mel_filter_bank

    filt = mel_filter_bank(num_frequency_bins=201, num_mel_filters=128, min_frequency=0.0, max_frequency=8000.0,
                           sampling_rate=16000, norm="slaney", mel_scale="slaney")
    tables = ops.LogMelTables(filt, "cuda")
    n = 480000
    rs = np.random.RandomState(0)
    wave = (rs.randn(2, n) * 0.1).astype(np.float32)
    wave[1, 160000:] = 0.0  # zero-padded short clip
    got = ops.logmel(torch.from_numpy(wave).cuda(), tables).cpu().numpy()
    ref = logmel_reference(wave, filt)
    err = np.abs(got - ref)
    assert got.shape == (2, 128, 3000)
    assert err.max() < 1e-4, err.max()


@pytest.mark.parametrize("K", [512, 3584])
@pytest.mark.parametrize("B", [32, 5, 48, 64, 1])
def test_qkv_rope_fused_gemm_matches_unfused(ops, B, K):
    """Decode-step fusion: q/k/v projection + RoPE + KV append in the GEMM epilogue == GEMM then af3_rope_kv_append
    (up to 64 sequences).  The unfused chain runs through the same kernel, so the comparison is bit-exact: same accumulation
    order, same rounding points."""
    H, Hkv, D, Tmax, slot = 28, 4, 128, 64, 37
    x, w, b = _rand((B, K), 1.0, 60), _rand(((H + 2 * Hkv) * D, K), 0.05, 61), _rand(((H + 2 * Hkv) * D,), 0.3, 62)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()
    starts = torch.randint(0, 30, (B,), dtype=torch.int32).cuda()
    pos = torch.tensor([slot], dtype=torch.int32, device="cuda")
    kc1, vc1 = torch.zeros((B, Hkv, Tmax, D), device="cuda", dtype=bf16), torch.zeros((B, Hkv, Tmax, D), device="cuda", dtype=bf16)
    kc2, vc2 = torch.zeros_like(kc1), torch.zeros_like(vc1)
    qkv1 = ops.linear(x, w, b)
    ops.rope_kv_append(qkv1, kc1, vc1, B=B, T=1, H=H, Hkv=Hkv, D=D, pos0=0, inv_freq=inv_freq, kv_start=starts, pos0_dev=pos)
    cs = ops.rope_table(B, D, pos, starts, inv_freq)
    qkv2 = ops.qkv_rope_linear(x, w, b, kc2, vc2, H=H, Hkv=Hkv, D=D, rope_cs=cs, pos_dev=pos)
    assert torch.equal(qkv2[:, :H * D], qkv1[:, :H * D])
    assert torch.equal(kc2, kc1) and torch.equal(vc2, vc1)


def test_qkv_rope_fused_gemm_never_writes_past_the_cache(ops):
    """ADVICE r01: with the cache full (slot == Tmax) the fused epilogue must drop the append instead of writing into the next
    (sequence, head) / past the allocation; the query heads are still produced."""
    B, H, Hkv, D, K, Tmax = 4, 28, 4, 128, 256, 16
    x, w, b = _rand((B, K), 1.0, 70), _rand(((H + 2 * Hkv) * D, K), 0.05, 71), _rand(((H + 2 * Hkv) * D,), 0.3, 72)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()
    guard = torch.full((2, B, Hkv, Tmax + 8, D), 7.0, device="cuda", dtype=bf16)   # 8 guard rows behind every (seq, head) block
    kc, vc = guard[0, :, :, :Tmax], guard[1, :, :, :Tmax]
    kc_c, vc_c = kc.contiguous(), vc.contiguous()                                  # the kernel takes dense [B, Hkv, Tmax, D] caches
    pos = torch.tensor([Tmax], dtype=torch.int32, device="cuda")
    cs = ops.rope_table(B, D, pos, None, inv_freq)
    before_k, before_v = kc_c.clone(), vc_c.clone()
    q = ops.qkv_rope_linear(x, w, b, kc_c, vc_c, H=H, Hkv=Hkv, D=D, rope_cs=cs, pos_dev=pos)
    torch.cuda.synchronize()
    assert torch.equal(kc_c, before_k) and torch.equal(vc_c, before_v)
    assert torch.isfinite(q[:, : H * D].float()).all()
    # the stand-alone append kernel with a device-side position has the same guard
    qkv = ops.linear(x, w, b)
    ops.rope_kv_append(qkv, kc_c, vc_c, B=B, T=1, H=H, Hkv=Hkv, D=D, pos0=0, inv_freq=inv_freq, pos0_dev=pos)
    torch.cuda.synchronize()
    assert torch.equal(kc_c, before_k) and torch.equal(vc_c, before_v)


def test_attention_v2_matches_v1_on_a_live_cache_offset(ops, monkeypatch):
    """Continuation chunk (chunked prefill / next chat turn): Tq = 200 new rows against Tk = 650 cached + new keys, causal with the
    (Tk - Tq) offset, GQA 28:4, left padding on one row.  The two row tilings give identical bits, and both meet the checks of
    check_prefill."""
    check_prefill(ops, monkeypatch, CONTINUATION)


def test_token_step_is_the_references_per_token_rule(ops):
    """af3_token_step against the reference's lines restated with torch ops ([O] GEN:2797-2805): finished rows emit pad, the token is
    appended, the unfinished mask is updated with the EOS set, "every row finished" is published -- over several consecutive tokens,
    with and without EOS handling, B above one thread block's width."""
    for B, n_eos in ((5, 1), (300, 2), (64, 0)):
        g = torch.Generator(device="cpu").manual_seed(B)
        cap, steps, pad = 16, 6, 7
        eos = torch.tensor([3, 11][:max(n_eos, 1)], dtype=torch.int64).cuda()
        eos_dev = torch.zeros((8,), dtype=torch.int64, device="cuda")
        eos_dev[: eos.numel()] = eos
        ctl = torch.tensor([n_eos, pad], dtype=torch.int64).cuda()
        unfinished = torch.ones((B,), dtype=torch.int32, device="cuda")
        tok_buf = torch.full((B, cap), -1, dtype=torch.int64, device="cuda")
        gen_idx = torch.zeros((1,), dtype=torch.int32, device="cuda")
        ids_out = torch.zeros((B,), dtype=torch.int64, device="cuda")
        flags = torch.full((cap,), -1, dtype=torch.int32, device="cuda")
        ref_unf = torch.ones((B,), dtype=torch.int64)
        for i in range(steps):
            raw = torch.randint(0, 14 if i < steps - 1 else 4, (B,), generator=g, dtype=torch.int64)
            if i == steps - 1 and n_eos:
                raw[:] = 3   # everybody finishes on the last token at the latest
            ops.token_step(raw.cuda(), unfinished, eos_dev, ctl, tok_buf, gen_idx, ids_out, flags)
            nxt = raw.clone()
            if n_eos:
                nxt = nxt * ref_unf + pad * (1 - ref_unf)                                # GEN:2797
                ref_unf = ref_unf & ~torch.isin(nxt, eos.cpu())                          # GEN:2803
            assert torch.equal(tok_buf[:, i].cpu(), nxt) and torch.equal(ids_out.cpu(), nxt)
            assert int(flags[i]) == (1 if (n_eos and int(ref_unf.max()) == 0) else 0)    # GEN:2805
            if n_eos:
                assert torch.equal(unfinished.cpu().long(), ref_unf)
        assert int(gen_idx) == steps and (tok_buf[:, steps:] == -1).all() and (flags[steps:] == -1).all()
