"""FP8 decoder projections on the GPU: the quantization kernel bit for bit against the activation rule, both GEMM modes
against the fp64 restatement of the promoted sum, the fused q/k/v + RoPE epilogue against the unfused chain, and the FP8
model end to end against the reference model with FP8 projections (oracle/fp8_oracle.py)."""
import os

os.environ.setdefault("HF_HUB_OFFLINE", "1")  # FP8Linear's matmul kernel would come from the hub: nothing here may fetch it

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

# The four decoder projection shapes of Qwen2.5-7B: (name, rows of w, K, epilogue)
SHAPES = [("qkv", 4608, 3584, "bias"), ("o", 3584, 3584, "resid"), ("gate_up", 18944, 3584, "swiglu"), ("down", 3584, 18944, "resid")]


@pytest.fixture(scope="module")
def ops():
    from audio_flamingo_b200 import ops as _ops

    return _ops


@pytest.fixture(scope="module")
def F():
    from oracle import fp8_oracle

    return fp8_oracle


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(bf16).cuda()


def _u8(t):
    return t.view(torch.uint8)


@pytest.mark.parametrize("rows", [1, 7, 64, 1000, 24960])
@pytest.mark.parametrize("K", [3584, 18944])
def test_quant_kernel_is_the_activation_rule(ops, F, rows, K):
    x = _rand((rows, K + 128), 1.0, rows + K)[:, :K]          # a pitch of K + 128 elements: not contiguous
    x[:, 128:256] = 0                                          # an all-zero group in every row
    x[rows // 2, 512:640] = 3e4                                # a large-magnitude group
    x[0, 1024:1152] *= 1e-6                                    # a tiny one
    q, s = ops.quant_fp8(x)
    qr, sr = F.quantize_activation(x)
    assert torch.equal(s, sr.T.contiguous())
    assert torch.equal(_u8(q), _u8(qr))


def _flags_ref(F, xq, sx, wq, sw, epi, bias=None, resid=None, n_feat=None):
    """-> (reference bf16 output, tolerance) from the fp64 promoted sum.

    Tolerance: the kernel's result may differ from the exact promoted sum by (a) its accumulation -- the tensor cores
    accumulate the 128 products of a k-block with fewer bits than fp32, and the fp32 promotion adds one rounding per k-block;
    both are bounded by 2^-12 of the sum of magnitudes (absum) -- and (b) one bf16 rounding flip of each rounded result
    (2^-7 of its magnitude).  Bias / residual add a second rounding; SwiGLU propagates the gate and up errors through
    silu(g) * u (|silu'| <= 1.1)."""
    mm = F.promoted_matmul(xq, sx, wq, sw)
    ab = F.promoted_matmul(xq, sx, wq, sw, absolute=True)
    acc_tol = 2.0 ** -12 * ab + 2.0 ** -7 * mm.abs()
    y = mm.float().to(bf16).float()
    if epi == "swiglu":
        g, u = y[:, :n_feat], y[:, n_feat:]
        tg, tu = acc_tol[:, :n_feat], acc_tol[:, n_feat:]
        silu = (g / (1 + torch.exp(-g))).to(bf16).float()
        ref = (silu * u).to(bf16).float()
        tol = 1.1 * u.abs() * tg + silu.abs() * tu + 2.0 ** -7 * ref.abs() + 1e-30
        return ref, tol.float()
    if epi == "bias":
        y = (y + bias.float()).to(bf16).float()
    if epi == "resid":
        y = (y + resid.float()).to(bf16).float()
    return y, (acc_tol + 2.0 ** -7 * y.abs()).float()


def _run(ops, epi, xq, wq, sw, bias, resid, n_feat):
    if epi == "swiglu":
        return ops.swiglu_linear_fp8(xq, wq, sw, n_feat)
    if epi == "bias":
        return ops.linear_fp8(xq, wq, sw, bias)
    out = resid.clone()
    return ops.linear_fp8(xq, wq, sw, resid=out, out=out)


def _problem(F, name, rows, K, epi, n_tok, seed):
    w = _rand((rows * (2 if epi == "swiglu" else 1), K), 0.02, seed)
    wq, sw = F.quantize_weight(w)
    x = _rand((n_tok, K), 1.0, seed + 1)
    n_feat = rows
    bias = _rand((rows,), 0.5, seed + 2) if epi == "bias" else None
    resid = _rand((n_tok, rows), 1.0, seed + 3) if epi == "resid" else None
    return x, wq.contiguous(), sw.contiguous(), bias, resid, n_feat


def test_quant_fp8_rejects_mis_shaped_buffers(ops):
    from audio_flamingo_b200 import AF3Error

    x = _rand((8, 256), 1.0, 3)
    with pytest.raises(AF3Error, match="scales"):
        ops.quant_fp8(x, scales=torch.empty((8, 2), device="cuda", dtype=torch.float32))
    with pytest.raises(AF3Error, match="out"):
        ops.quant_fp8(x, out=torch.empty((8, 256), device="cuda", dtype=torch.uint8))


# up to 64 tokens: the few-token kernel; from 65 on: gemm_fp8_tok_kernel (token tails at 65, 200, 1000)
@pytest.mark.parametrize("n_tok", [1, 7, 32, 33, 64, 65, 200, 1000])
@pytest.mark.parametrize("name,rows,K,epi", SHAPES)
def test_fp8_gemm_against_the_promoted_sum(ops, F, name, rows, K, epi, n_tok):
    x, wq, sw, bias, resid, n_feat = _problem(F, name, rows, K, epi, n_tok, 10 * n_tok + rows)
    xq = ops.quant_fp8(x)
    got = _run(ops, epi, xq, wq, sw, bias, resid, n_feat).float()
    qx, sx = xq[0], xq[1].T  # the GEMM is checked on the kernel's own quantized input
    ref, tol = _flags_ref(F, qx, sx, wq, sw, epi, bias, resid, n_feat)
    err = (got - ref).abs()
    bad = int((err > tol).sum())
    print(f"{name} n_tok={n_tok}: max err {err.max().item():.4g}, max err / tol {(err / tol).max().item():.3f}")
    assert bad == 0, f"{bad}/{err.numel()} out of tolerance, max err {err.max().item():.4g}"


@pytest.mark.parametrize("name,rows,K,epi", SHAPES)
def test_fp8_gemm_large_prefill_shape(ops, F, name, rows, K, epi):
    x, wq, sw, bias, resid, n_feat = _problem(F, name, rows, K, epi, 4000, 5)
    xq = ops.quant_fp8(x)
    got = _run(ops, epi, xq, wq, sw, bias, resid, n_feat).float()
    qx, sx = xq[0], xq[1].T  # the GEMM is checked on the kernel's own quantized input
    ref, tol = _flags_ref(F, qx, sx, wq, sw, epi, bias, resid, n_feat)
    assert int(((got - ref).abs() > tol).sum()) == 0


@pytest.mark.parametrize("name,rows,K,epi", [SHAPES[0], SHAPES[1], SHAPES[3]])
def test_fp8_split_k_is_deterministic_and_forced_splits_agree(ops, F, monkeypatch, name, rows, K, epi):
    from audio_flamingo_b200 import _lib

    x, wq, sw, bias, resid, n_feat = _problem(F, name, rows, K, epi, 32, 7)
    xq = ops.quant_fp8(x)
    a = _run(ops, epi, xq, wq, sw, bias, resid, n_feat)
    b = _run(ops, epi, xq, wq, sw, bias, resid, n_feat)
    assert torch.equal(a, b), "split-K output must be run-to-run identical"
    for _ in range(3):  # repeated launches (the split-K counters are left at zero)
        assert torch.equal(_run(ops, epi, xq, wq, sw, bias, resid, n_feat), a)
    _lib.load().af3_set_pdl(1)
    try:
        assert torch.equal(_run(ops, epi, xq, wq, sw, bias, resid, n_feat), a), "PDL on must give the same bits"
    finally:
        _lib.load().af3_set_pdl(0)
    qx, sx = xq[0], xq[1].T  # the GEMM is checked on the kernel's own quantized input
    ref, tol = _flags_ref(F, qx, sx, wq, sw, epi, bias, resid, n_feat)
    for s in ("1", "2", "5", "16"):
        monkeypatch.setenv("AF3_KSPLIT", s)
        got = _run(ops, epi, xq, wq, sw, bias, resid, n_feat).float()
        assert int(((got - ref).abs() > tol).sum()) == 0, f"AF3_KSPLIT={s}"


@pytest.mark.parametrize("K", [512, 3584])
@pytest.mark.parametrize("B", [32, 5, 64, 1])
def test_fp8_qkv_rope_fused_gemm_matches_unfused(ops, F, B, K):
    """The fused FP8 q/k/v + RoPE + KV append equals the FP8 GEMM then af3_rope_kv_append bit for bit (same kernel, same
    accumulation order and rounding points)."""
    H, Hkv, D, Tmax, slot = 28, 4, 128, 64, 37
    wq, sw = F.quantize_weight(_rand(((H + 2 * Hkv) * D, K), 0.05, 61))
    x, b = _rand((B, K), 1.0, 60), _rand(((H + 2 * Hkv) * D,), 0.3, 62)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()
    starts = torch.randint(0, 30, (B,), dtype=torch.int32).cuda()
    pos = torch.tensor([slot], dtype=torch.int32, device="cuda")
    kc1, vc1 = torch.zeros((B, Hkv, Tmax, D), device="cuda", dtype=bf16), torch.zeros((B, Hkv, Tmax, D), device="cuda", dtype=bf16)
    kc2, vc2 = torch.zeros_like(kc1), torch.zeros_like(vc1)
    xq = ops.quant_fp8(x)
    qkv1 = ops.linear_fp8(xq, wq, sw, b)
    ops.rope_kv_append(qkv1, kc1, vc1, B=B, T=1, H=H, Hkv=Hkv, D=D, pos0=0, inv_freq=inv_freq, kv_start=starts, pos0_dev=pos)
    cs = ops.rope_table(B, D, pos, starts, inv_freq)
    qkv2 = ops.qkv_rope_linear_fp8(xq, wq, sw, b, kc2, vc2, H=H, Hkv=Hkv, D=D, rope_cs=cs, pos_dev=pos)
    assert torch.equal(qkv2[:, :H * D], qkv1[:, :H * D])
    assert torch.equal(kc2, kc1) and torch.equal(vc2, vc1)


def test_fp8_qkv_rope_fused_gemm_never_writes_past_the_cache(ops, F):
    B, H, Hkv, D, K, Tmax = 4, 28, 4, 128, 256, 16
    wq, sw = F.quantize_weight(_rand(((H + 2 * Hkv) * D, K), 0.05, 71))
    x, b = _rand((B, K), 1.0, 70), _rand(((H + 2 * Hkv) * D,), 0.3, 72)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()
    kc, vc = torch.full((B, Hkv, Tmax, D), 7.0, device="cuda", dtype=bf16), torch.full((B, Hkv, Tmax, D), 7.0, device="cuda", dtype=bf16)
    pos = torch.tensor([Tmax], dtype=torch.int32, device="cuda")
    cs = ops.rope_table(B, D, pos, None, inv_freq)
    before_k, before_v = kc.clone(), vc.clone()
    q = ops.qkv_rope_linear_fp8(ops.quant_fp8(x), wq, sw, b, kc, vc, H=H, Hkv=Hkv, D=D, rope_cs=cs, pos_dev=pos)
    torch.cuda.synchronize()
    assert torch.equal(kc, before_k) and torch.equal(vc, before_v)
    assert torch.isfinite(q[:, : H * D].float()).all()


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("preset", ["tiny", "mid"])
@pytest.mark.parametrize("n_tok", [5, 300])
def test_fp8_model_projections_are_wired_to_their_weights(O, F, preset, n_tok):
    """Each layer's four GEMMs, as the packed FP8 model runs them (fused [q; k; v] / [gate; up] matrices, fused scale grids,
    biases), against the restatement of the same HF projections on the same bf16 input: the per-GEMM tolerance of the
    promoted sum, so a misordered fused row block or scale row, or a swapped projection, fails at once."""
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model(preset, seed=3, sharpen=8.0)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda", quantization="fp8")
    lm = ours.language_model
    lm._check_ready()
    rq = F.fp8_reference_model(ref32)
    hid, HD, KD, inter = lm.hid, lm.H * lm.D, lm.Hkv * lm.D, lm.inter

    def check(got, parts, x, epi, resid=None):
        qx, sx = F.quantize_activation(x)
        wq = torch.cat([p.q for p in parts]).cuda()
        sw = torch.cat([p.s for p in parts]).cuda()
        bias = torch.cat([p.bias for p in parts]).cuda() if parts[0].bias is not None else None
        ref, tol = _flags_ref(F, qx, sx, wq, sw, epi, bias, resid, inter if epi == "swiglu" else None)
        err = (got.float() - ref).abs()
        assert int((err > tol).sum()) == 0, f"{epi}: max err {err.max().item():.4g}"

    with torch.no_grad(), torch.cuda.device(0):
        for li, (pj, layer) in enumerate(zip(lm._proj, rq.language_model.model.layers)):
            at, mlp = layer.self_attn, layer.mlp
            y = _rand((n_tok, hid), 1.0, 100 + li)
            check(ours_qkv := pj.qkv(y), [at.q_proj, at.k_proj, at.v_proj], y, "bias")
            assert ours_qkv.shape == (n_tok, HD + 2 * KD)
            a = _rand((n_tok, HD), 1.0, 200 + li)
            h = _rand((n_tok, hid), 1.0, 300 + li)
            h0 = h.clone()
            pj.o(a, h)
            check(h, [at.o_proj], a, "resid", h0)
            check(pj.gate_up(y), [mlp.gate_proj, mlp.up_proj], y, "swiglu")
            g = _rand((n_tok, inter), 1.0, 400 + li)
            h = h0.clone()
            pj.down(g, h)
            check(h, [mlp.down_proj], g, "resid", h0)

@pytest.fixture(scope="module")
def O():
    from oracle import af3_oracle

    return af3_oracle


def _inputs(O, cfg, secs, seed=1):
    waves = O.synth_waveforms(len(secs), secs, seed=seed)
    feats, fmask = O.hf_features(waves)
    toks = [O.post_pool_len(int(n)) for n in fmask.sum(-1)]
    ids, am = O.synth_prompt(toks, cfg.text_config.vocab_size, cfg.audio_token_id, seed=seed + 1)
    return feats, fmask, ids, am


def _fwd(m, feats, fmask, ids, am):
    return m(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda()).logits.float().cpu()


@pytest.mark.parametrize("preset,secs,new", [("tiny", [10.0, 4.3, 30.0], 16), ("mid", [30.0, 12.0], 10)])
def test_fp8_model_end_to_end(O, F, monkeypatch, preset, secs, new):
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model(preset, seed=3, sharpen=8.0)
    cfg = ref32.config
    feats, fmask, ids, am = _inputs(O, cfg, secs, seed=5)
    plain = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    l_plain = _fwd(plain, feats, fmask, ids, am)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda", quantization="fp8")
    assert ours.quantization == "fp8" and plain.quantization is None
    assert ours.language_model.model.layers[0].mlp.down_proj.weight.dtype == torch.float8_e4m3fn
    lo = _fwd(ours, feats, fmask, ids, am)
    assert torch.equal(_fwd(plain, feats, fmask, ids, am), l_plain), "a bf16 model next to an FP8 one is unaffected"

    # the restatement in fp32, and in bf16 on the same GPU (the reference's own error in our compute dtype)
    rq = F.fp8_reference_model(ref32).to("cuda")
    rq16 = O.hf_restore_fp32_rotary(F.fp8_reference_model(ref32).to("cuda", bf16))
    fkw = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda())
    with torch.no_grad():
        lr = rq(**fkw).logits.float().cpu()
        lr16 = rq16(**dict(fkw, input_features=feats.cuda().to(bf16))).logits.float().cpu()
    valid = am.bool()
    std = lr[valid].std().item()
    err = (lo - lr)[valid].abs().max().item()
    err16 = (lr16 - lr)[valid].abs().max().item()
    print(f"[{preset}] fp8 logits vs fp8 restatement (fp32): ours {err:.4f}, restatement in bf16 {err16:.4f}, std {std:.3f}; "
          f"bf16 model vs it: {(l_plain - lr)[valid].abs().max().item():.4f}")
    # as tests/test_model_gpu.py bounds the bf16 path: 6 % of the logit std, or 1.5 x the reference's own error in bf16.  A
    # bf16-sized change of an activation moves some of its e4m3 codes by one step (~6 %), so FP8 chains are noisier than bf16 ones.
    assert err <= max(1.5 * err16, 0.06 * std)
    top2 = lr[:, -1].topk(2).values
    safe = (top2[:, 0] - top2[:, 1]) > 2 * err
    assert torch.equal(lo[:, -1].argmax(-1)[safe], lr[:, -1].argmax(-1)[safe])

    # greedy ids: graph == eager == PDL off; against the restatement in bf16 wherever the step is decisive (top-2 margin of our
    # logits above twice the logit error measured above)
    kw = dict(fkw, max_new_tokens=new)
    g_graph, lg = ours.generate(**kw, return_logits=True)
    assert torch.equal(ours.generate(**kw, use_cuda_graph=False), g_graph)
    monkeypatch.setenv("AF3_PDL", "0")
    assert torch.equal(ours.generate(**kw), g_graph)
    monkeypatch.delenv("AF3_PDL")
    with torch.no_grad():
        g_ref = rq16.generate(**dict(kw, input_features=feats.cuda().to(bf16)), do_sample=False)
    S = ids.shape[1]
    same = g_graph[:, S:].cpu() == g_ref[:, S:].cpu()
    for b in range(len(secs)):
        if bool(same[b].all()):
            continue
        t = int((~same[b]).nonzero()[0])
        top2 = lg[b, t].topk(2).values
        margin = (top2[0] - top2[1]).item()
        print(f"[{preset}] row {b} diverges at step {t}, margin {margin:.4f}")
        assert margin < 2 * err, "divergence at a decisive step"
    print(f"[{preset}] greedy ids identical to the fp8 restatement on {int(same.all(1).sum())}/{len(secs)} rows")

    # a FineGrainedFP8-layout state dict (quantized by transformers' Fp8Quantize) loads to the same model, and state_dict()
    # of an FP8 model round-trips
    from transformers.integrations.finegrained_fp8 import Fp8Quantize

    class _Q:
        class quantization_config:
            weight_block_size = (128, 128)

    sd = {}
    for k, v in ref32.state_dict().items():
        base = k[: -len(".weight")]
        if k.startswith("language_model.model.layers.") and k.endswith("proj.weight"):
            sd.update(Fp8Quantize(_Q()).convert({k: [v.to(bf16)]}))
        else:
            sd[k] = v
    assert any(v.dtype == torch.float8_e4m3fn for v in sd.values())
    loaded = AudioFlamingo3ForConditionalGeneration(cfg)
    loaded.load_reference_state_dict(sd, device="cuda")
    assert loaded.quantization == "fp8"
    assert torch.equal(_fwd(loaded, feats, fmask, ids, am), lo)
    sd2 = ours.state_dict()
    assert sorted(sd2) == sorted(sd)
    for k, v in sd.items():
        if v.dtype == torch.float8_e4m3fn or k.endswith("weight_scale_inv"):
            assert sd2[k].dtype == v.dtype and torch.equal(sd2[k].cpu().view(torch.uint8), v.view(torch.uint8)), k
    again = AudioFlamingo3ForConditionalGeneration(cfg)
    again.load_reference_state_dict({k: v.clone() for k, v in sd2.items()}, device="cuda")
    assert torch.equal(_fwd(again, feats, fmask, ids, am), lo)
