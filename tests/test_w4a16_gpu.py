"""W4A16 decoder projections on the GPU: the few-token GEMM against fp32 x @ Wd.T and bit for bit against the bf16 GEMM on
Wd, split-K determinism, the fused q/k/v + RoPE epilogue, the dequantization kernel, and the W4A16 model end to end
against the bf16 model and the HF model holding Wd (oracle/w4a16_oracle.py)."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

# decode-step projections of Qwen2.5-7B and a tiny geometry: (rows of w, K, epilogue)
SHAPES_7B = [(4608, 3584, "bias"), (3584, 3584, "resid"), (18944, 3584, "swiglu"), (3584, 18944, "resid")]
SHAPES_TINY = [(384, 256, "bias"), (256, 384, "resid"), (512, 256, "swiglu"), (256, 512, "none")]


@pytest.fixture(scope="module")
def ops():
    from audio_flamingo_b200 import ops as _ops

    return _ops


@pytest.fixture(scope="module")
def W():
    from oracle import w4a16_oracle

    return w4a16_oracle


@pytest.fixture(scope="module")
def O():
    from oracle import af3_oracle

    return af3_oracle


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(bf16).cuda()


def _problem(W, rows, K, epi, n_tok, seed):
    w = _rand((rows * (2 if epi == "swiglu" else 1), K), 0.02, seed)
    p, s = W.quantize(w)
    x = _rand((n_tok, K), 1.0, seed + 1)
    bias = _rand((rows,), 0.5, seed + 2) if epi == "bias" else None
    resid = _rand((n_tok, rows), 1.0, seed + 3) if epi == "resid" else None
    return x, p.cuda(), s.cuda(), W.dequantize(p, s).cuda(), bias, resid


def _run(ops, epi, x, p, s, bias, resid, rows):
    if epi == "swiglu":
        return ops.swiglu_linear_w4a16(x, p, s, rows)
    if epi == "resid":
        out = resid.clone()
        return ops.linear_w4a16(x, p, s, resid=out, out=out)
    return ops.linear_w4a16(x, p, s, bias)


def _ref(epi, x, wd, bias, resid, rows):
    """fp32 x @ Wd.T with the epilogue's bf16 rounding points, and a tolerance: the fp32 accumulation (2^-12 of the sum of
    magnitudes, as the FP8 tests bound the tensor-core sums) plus one bf16 rounding flip of each rounded value (2^-7)."""
    mm = x.float() @ wd.float().T
    acc = 2.0 ** -12 * (x.float().abs() @ wd.float().abs().T) + 2.0 ** -7 * mm.abs()
    y = mm.to(bf16).float()
    if epi == "swiglu":
        g, u, tg, tu = y[:, :rows], y[:, rows:], acc[:, :rows], acc[:, rows:]
        silu = (g / (1 + torch.exp(-g))).to(bf16).float()
        ref = (silu * u).to(bf16).float()
        return ref, 1.1 * u.abs() * tg + silu.abs() * tu + 2.0 ** -7 * ref.abs() + 1e-30
    if epi == "bias":
        y = (y + bias.float()).to(bf16).float()
    if epi == "resid":
        y = (y + resid.float()).to(bf16).float()
    return y, acc + 2.0 ** -7 * y.abs()


@pytest.mark.parametrize("n_tok", [1, 7, 32, 33, 64])
@pytest.mark.parametrize("rows,K,epi", SHAPES_TINY + SHAPES_7B)
def test_w4a16_gemm_against_the_restatement(ops, W, rows, K, epi, n_tok):
    x, p, s, wd, bias, resid = _problem(W, rows, K, epi, n_tok, 10 * n_tok + rows + K)
    got = _run(ops, epi, x, p, s, bias, resid, rows).float()
    ref, tol = _ref(epi, x, wd, bias, resid, rows)
    err = (got - ref).abs()
    assert int((err > tol).sum()) == 0, f"max err {err.max().item():.4g}, max err / tol {(err / tol).max().item():.3f}"


def _raw(lib_fn, *args):
    from audio_flamingo_b200 import _lib

    _lib.check(lib_fn(*args), lib_fn.__name__)


@pytest.mark.parametrize("n_tok", [1, 7, 32, 33, 64])
@pytest.mark.parametrize("rows,K,epi", SHAPES_TINY + SHAPES_7B)
def test_unsplit_w4a16_gemm_equals_the_bf16_gemm_on_wd(ops, W, rows, K, epi, n_tok):
    """Without a workspace both kernels run one accumulator chain in the same k order over the same products: same bits."""
    from audio_flamingo_b200 import _lib
    from audio_flamingo_b200._lib import EPI_BIAS, EPI_RESID, EPI_SWIGLU, EPI_SWIGLU_CONCAT, ptr, stream_ptr

    lib = _lib.load()
    x, p, s, wd, bias, resid = _problem(W, rows, K, epi, n_tok, 3 * n_tok + rows)
    flags = {"bias": EPI_BIAS, "resid": EPI_RESID, "swiglu": EPI_SWIGLU | EPI_SWIGLU_CONCAT, "none": 0}[epi]
    outs = []
    for w4 in (True, False):
        out = resid.clone() if epi == "resid" else torch.empty((n_tok, rows), device="cuda", dtype=bf16)
        r = out if epi == "resid" else None
        if w4:
            _raw(lib.af3_gemm_w4a16, stream_ptr(), ptr(x), x.stride(0), ptr(p), p.stride(0), ptr(s), s.stride(0), ptr(out), out.stride(0),
                 n_tok, rows, K, flags, ptr(bias), ptr(r), rows if r is not None else 0, None, 0)
        else:
            _raw(lib.af3_gemm_bf16, stream_ptr(), ptr(x), x.stride(0), ptr(wd), wd.stride(0), ptr(out), out.stride(0), n_tok, rows, K,
                 flags, ptr(bias), ptr(r), rows if r is not None else 0, 0)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("rows,K,epi", [SHAPES_7B[0], SHAPES_7B[1], SHAPES_7B[3]])
def test_w4a16_split_k_is_deterministic_and_forced_splits_agree(ops, W, monkeypatch, rows, K, epi):
    from audio_flamingo_b200 import _lib

    x, p, s, wd, bias, resid = _problem(W, rows, K, epi, 32, 7)
    a = _run(ops, epi, x, p, s, bias, resid, rows)
    for _ in range(3):
        assert torch.equal(_run(ops, epi, x, p, s, bias, resid, rows), a), "split-K output must be run-to-run identical"
    _lib.load().af3_set_pdl(1)
    try:
        assert torch.equal(_run(ops, epi, x, p, s, bias, resid, rows), a), "PDL on must give the same bits"
    finally:
        _lib.load().af3_set_pdl(0)
    ref, tol = _ref(epi, x, wd, bias, resid, rows)
    for k in ("1", "2", "5", "16"):
        monkeypatch.setenv("AF3_KSPLIT", k)
        got = _run(ops, epi, x, p, s, bias, resid, rows).float()
        assert int(((got - ref).abs() > tol).sum()) == 0, f"AF3_KSPLIT={k}"


@pytest.mark.parametrize("rows,K", [(256, 384), (4608, 3584), (37888, 3584), (3584, 18944)])
def test_dequant_kernel_is_torch_dequantization(ops, W, rows, K):
    from audio_flamingo_b200.modeling import dequantize_w4a16

    w = _rand((rows, K), 0.02, rows + K)
    w[0, :128] = 0
    w[1, :128] *= 1e-20
    p, s = W.quantize(w)
    p, s = p.cuda(), s.cuda()
    got = ops.dequant_w4a16(p, s)
    assert torch.equal(got, dequantize_w4a16(p, s))
    if rows * K < 50_000_000:
        assert torch.equal(got.cpu(), W.dequantize(p, s))


def test_w4a16_gemm_rejects_more_than_64_tokens(ops, W):
    from audio_flamingo_b200 import AF3Error

    x, p, s, wd, bias, resid = _problem(W, 256, 384, "bias", 65, 1)
    with pytest.raises(AF3Error, match="64"):
        ops.linear_w4a16(x, p, s, bias)


@pytest.mark.parametrize("K", [512, 3584])
@pytest.mark.parametrize("B", [32, 5, 64, 1])
def test_w4a16_qkv_rope_fused_gemm_matches_unfused(ops, W, B, K):
    H, Hkv, D, Tmax, slot = 28, 4, 128, 64, 37
    p, s = W.quantize(_rand(((H + 2 * Hkv) * D, K), 0.05, 61))
    p, s = p.cuda(), s.cuda()
    x, b = _rand((B, K), 1.0, 60), _rand(((H + 2 * Hkv) * D,), 0.3, 62)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()
    starts = torch.randint(0, 30, (B,), dtype=torch.int32).cuda()
    pos = torch.tensor([slot], dtype=torch.int32, device="cuda")
    kc1, vc1 = torch.zeros((B, Hkv, Tmax, D), device="cuda", dtype=bf16), torch.zeros((B, Hkv, Tmax, D), device="cuda", dtype=bf16)
    kc2, vc2 = torch.zeros_like(kc1), torch.zeros_like(vc1)
    qkv1 = ops.linear_w4a16(x, p, s, b)
    ops.rope_kv_append(qkv1, kc1, vc1, B=B, T=1, H=H, Hkv=Hkv, D=D, pos0=0, inv_freq=inv_freq, kv_start=starts, pos0_dev=pos)
    cs = ops.rope_table(B, D, pos, starts, inv_freq)
    qkv2 = ops.qkv_rope_linear_w4a16(x, p, s, b, kc2, vc2, H=H, Hkv=Hkv, D=D, rope_cs=cs, pos_dev=pos)
    assert torch.equal(qkv2[:, :H * D], qkv1[:, :H * D])
    assert torch.equal(kc2, kc1) and torch.equal(vc2, vc1)


def test_w4a16_qkv_rope_fused_gemm_never_writes_past_the_cache(ops, W):
    B, H, Hkv, D, K, Tmax = 4, 28, 4, 128, 256, 16
    p, s = W.quantize(_rand(((H + 2 * Hkv) * D, K), 0.05, 71))
    x, b = _rand((B, K), 1.0, 70), _rand(((H + 2 * Hkv) * D,), 0.3, 72)
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))).cuda()
    kc, vc = torch.full((B, Hkv, Tmax, D), 7.0, device="cuda", dtype=bf16), torch.full((B, Hkv, Tmax, D), 7.0, device="cuda", dtype=bf16)
    pos = torch.tensor([Tmax], dtype=torch.int32, device="cuda")
    cs = ops.rope_table(B, D, pos, None, inv_freq)
    before_k, before_v = kc.clone(), vc.clone()
    q = ops.qkv_rope_linear_w4a16(x, p.cuda(), s.cuda(), b, kc, vc, H=H, Hkv=Hkv, D=D, rope_cs=cs, pos_dev=pos)
    torch.cuda.synchronize()
    assert torch.equal(kc, before_k) and torch.equal(vc, before_v)
    assert torch.isfinite(q[:, : H * D].float()).all()


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("preset", ["tiny", "mid"])
@pytest.mark.parametrize("n_tok", [5, 300])
def test_w4a16_model_projections_are_wired_to_their_weights(O, W, preset, n_tok):
    """Each layer's four GEMMs as the packed W4A16 model runs them, against fp32 x @ Wd.T of the same HF projections."""
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model(preset, seed=3, sharpen=8.0)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda", quantization="w4a16")
    lm = ours.language_model
    lm._check_ready()
    hid, HD, inter = lm.hid, lm.H * lm.D, lm.inter

    def wd(*mods):
        return torch.cat([W.dequantize(*W.quantize(m.weight.detach().to(bf16))) for m in mods]).cuda()

    def check(got, w, x, epi, bias=None, resid=None):
        ref, tol = _ref(epi, x, w, bias, resid, inter)
        err = (got.float() - ref).abs()
        assert int((err > tol).sum()) == 0, f"{epi}: max err {err.max().item():.4g}"

    with torch.no_grad(), torch.cuda.device(0):
        for li, (pj, layer) in enumerate(zip(lm._proj, ref32.language_model.model.layers)):
            at, mlp = layer.self_attn, layer.mlp
            y = _rand((n_tok, hid), 1.0, 100 + li)
            bias = torch.cat([at.q_proj.bias, at.k_proj.bias, at.v_proj.bias]).to(bf16).cuda()
            check(pj.qkv(y), wd(at.q_proj, at.k_proj, at.v_proj), y, "bias", bias)
            a, h = _rand((n_tok, HD), 1.0, 200 + li), _rand((n_tok, hid), 1.0, 300 + li)
            h0 = h.clone()
            pj.o(a, h)
            check(h, wd(at.o_proj), a, "resid", resid=h0)
            check(pj.gate_up(y), wd(mlp.gate_proj, mlp.up_proj), y, "swiglu")
            g = _rand((n_tok, inter), 1.0, 400 + li)
            h = h0.clone()
            pj.down(g, h)
            check(h, wd(mlp.down_proj), g, "resid", resid=h0)


def _inputs(O, cfg, secs, seed=1):
    waves = O.synth_waveforms(len(secs), secs, seed=seed)
    feats, fmask = O.hf_features(waves)
    toks = [O.post_pool_len(int(n)) for n in fmask.sum(-1)]
    ids, am = O.synth_prompt(toks, cfg.text_config.vocab_size, cfg.audio_token_id, seed=seed + 1)
    return feats, fmask, ids, am


def _fwd(m, feats, fmask, ids, am):
    return m(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda()).logits.float().cpu()


@pytest.mark.parametrize("preset,secs,new", [("tiny", [10.0, 4.3, 30.0], 16), ("mid", [30.0, 12.0], 10)])
def test_w4a16_model_end_to_end(O, W, monkeypatch, preset, secs, new):
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model(preset, seed=3, sharpen=8.0)
    cfg = ref32.config
    feats, fmask, ids, am = _inputs(O, cfg, secs, seed=5)
    assert ids.numel() > 64
    rw = W.w4a16_reference_model(ref32)
    plain_wd = AudioFlamingo3ForConditionalGeneration.from_reference(rw, device="cuda")
    l_wd = _fwd(plain_wd, feats, fmask, ids, am)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda", quantization="w4a16")
    assert ours.quantization == "w4a16" and plain_wd.quantization is None
    d = ours.language_model.model.layers[0].mlp.down_proj
    assert d.weight_packed.dtype == torch.int32 and d.weight_scale.dtype == bf16 and "weight" not in d._parameters
    lo = _fwd(ours, feats, fmask, ids, am)
    # prefill (more than 64 tokens): dequantized projections through the bf16 GEMMs -- the bf16 model on Wd, bit for bit
    assert torch.equal(lo, l_wd)
    assert torch.equal(_fwd(plain_wd, feats, fmask, ids, am), l_wd), "a bf16 model next to a W4A16 one is unaffected"

    # against the HF model holding Wd, in fp32 and in bf16 on the same GPU: the bound tests/test_model_gpu.py puts on bf16
    rq16 = O.hf_restore_fp32_rotary(copy.deepcopy(rw).to("cuda", bf16))
    rq = rw.to("cuda")
    fkw = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda())
    with torch.no_grad():
        lr = rq(**fkw).logits.float().cpu()
        lr16 = rq16(**dict(fkw, input_features=feats.cuda().to(bf16))).logits.float().cpu()
    valid = am.bool()
    std = lr[valid].std().item()
    err = (lo - lr)[valid].abs().max().item()
    err16 = (lr16 - lr)[valid].abs().max().item()
    print(f"[{preset}] w4a16 logits vs Wd model (fp32): ours {err:.4f}, HF in bf16 {err16:.4f}, std {std:.3f}")
    assert err <= max(1.5 * err16, 0.06 * std)

    # greedy ids: graph == eager == PDL off; against the HF Wd model in bf16 wherever the step is decisive
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

    # state_dict() round-trips, and a state dict quantized by the restatement loads to the same model
    sd2 = ours.state_dict()
    again = AudioFlamingo3ForConditionalGeneration(cfg)
    again.load_reference_state_dict({k: v.clone() for k, v in sd2.items()}, device="cuda")
    assert again.quantization == "w4a16"
    assert torch.equal(_fwd(again, feats, fmask, ids, am), lo)
    sd = {}
    for k, v in ref32.state_dict().items():
        base = k[: -len(".weight")]
        if k.startswith("language_model.model.layers.") and k.endswith("proj.weight"):
            sd[base + ".weight_packed"], sd[base + ".weight_scale"] = W.quantize(v.to(bf16))
        else:
            sd[k] = v
    assert sorted(sd) == sorted(sd2)
    loaded = AudioFlamingo3ForConditionalGeneration(cfg)
    loaded.load_reference_state_dict(sd, device="cuda")
    assert loaded.quantization == "w4a16"
    assert torch.equal(_fwd(loaded, feats, fmask, ids, am), lo)
