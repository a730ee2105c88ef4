"""Teacher-forced loss on the GPU (include/af3b200.h af3_lm_head_xent and forward(labels=...)).
  * kernel level: token counts on both sides of every tile edge, V with and without a tail tile, K = 512 / 3584; labels at
    0, V - 1, in the tail tile, -100, a custom ignore_index, all ignored.  Stored logits equal ops.linear(out_f32=True) bit for
    bit (same kernel, same k order) whenever that call is token-major (n_tok > 64); token_nll is within
    1e-5 (1 + |lse|) of an fp64 logsumexp over those logits; loss-only, logits-also and repeated launches are bit-identical;
    device labels outside [0, V) are ignored (= the same labels at -100) and counted.
  * model level on the tiny preset: loss and token_losses equal F.cross_entropy over our own returned logits; loss against
    the unmodified HF model in bf16 on the same GPU; prompts with one / several windows and clips, left padding, inputs_embeds,
    a continuation chunk, shift_labels / num_items_in_batch / ignore_index, the FP8 model; logits_to_keep=1 gives the same
    loss bits as 0 and never allocates the [B, S, V] logits; malformed labels raise before any launch."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from audio_flamingo_b200 import ops

    return ops


@pytest.fixture(scope="module")
def O():
    from oracle import af3_oracle

    return af3_oracle


def _lse64(logits, chunk=512):
    return torch.cat([torch.logsumexp(logits[i:i + chunk].double(), -1) for i in range(0, logits.shape[0], chunk)])


def _labels(T, V, seed, ignore_index=-100):
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, V, (T,), generator=g)
    special = [0, V - 1, V - 1 - (V % 128) // 2 if V % 128 else V - 64, ignore_index]
    lab[:min(T, 4)] = torch.tensor(special[:min(T, 4)])
    lab[6::9] = ignore_index
    return lab.cuda()


def _check_nll(logits, lab, nll, totals, ignore_index=-100):
    V = logits.shape[1]
    counted = (lab != ignore_index) & (lab >= 0) & (lab < V)
    lse = _lse64(logits)
    tgt = logits.gather(1, torch.where(counted, lab, 0)[:, None])[:, 0].double()
    ref = torch.where(counted, lse - tgt, torch.zeros_like(lse))
    err = (nll.double() - ref).abs()
    assert bool((err <= 1e-5 * (1 + lse.abs())).all()), f"max nll error {err.max().item()}"
    assert bool((nll[~counted] == 0).all())
    assert totals[1].item() == counted.sum().item()
    assert abs(totals[0].item() - nll.double().sum().item()) <= 1e-9 * (1 + abs(totals[0].item()))


@pytest.mark.parametrize("V,K", [(152064, 3584), (2048, 512), (2051, 512), (2051, 3584)])
@pytest.mark.parametrize("T", [1, 37, 64, 65, 128, 129, 1000, 4096])
def test_kernel(ops, T, V, K):
    g = torch.Generator(device="cuda").manual_seed(T * 7 + K)
    x = (torch.randn(T, K, device="cuda", generator=g) * 0.5).to(bf16)
    w = (torch.randn(V, K, device="cuda", generator=g) * (2.0 / K ** 0.5)).to(bf16)
    lab = _labels(T, V, T + V)
    logits, nll, totals = ops.lm_head_xent(x, w, lab, store_logits=True)
    if T > 64:   # ops.linear takes the same token-major kernel
        assert torch.equal(logits, ops.linear(x, w, out_f32=True))
    else:        # bf16 values of an fp32 product: within a bf16 rounding of the fp32 matmul
        ref = x.float() @ w.float().T
        assert bool(((logits - ref).abs() <= 2 ** -8 * ref.abs() + 1e-4).all())
        assert torch.equal(logits, logits.to(bf16).float())
    _check_nll(logits, lab, nll, totals)
    _, nll2, totals2 = ops.lm_head_xent(x, w, lab)
    _, nll3, totals3 = ops.lm_head_xent(x, w, lab)
    assert torch.equal(nll2, nll) and torch.equal(totals2, totals), "loss-only launch differs from the logits-also launch"
    assert torch.equal(nll3, nll2) and torch.equal(totals3, totals2), "repeated launches differ"
    if T in (129, 1000):
        # custom ignore_index (a valid column), everything ignored, and device labels outside [0, V)
        lab5 = lab.clone()
        lab5[lab5 == -100] = 5
        lab5[10::11] = 5
        lg, n5, t5 = ops.lm_head_xent(x, w, lab5, ignore_index=5, store_logits=True)
        _check_nll(lg, lab5, n5, t5, ignore_index=5)
        _, n0, t0 = ops.lm_head_xent(x, w, torch.full_like(lab, -100))
        assert bool((n0 == 0).all()) and t0.tolist() == [0.0, 0.0, 0.0]
        bad = lab.clone()
        bad[7::13] = V
        bad[8::13] = -3
        bad[9::13] = 1 << 40
        n_bad = int(((bad != -100) & ((bad < 0) | (bad >= V))).sum())
        _, nb, tb = ops.lm_head_xent(x, w, bad)
        clean = torch.where((bad < 0) | (bad >= V), torch.full_like(bad, -100), bad)
        _, nc, tc = ops.lm_head_xent(x, w, clean)
        assert torch.equal(nb, nc) and torch.equal(tb[:2], tc[:2]) and tb[2].item() == n_bad and tc[2].item() == 0


# ------------------------------------------------------------------------------------------------ model level
def _inputs(O, cfg, secs, seed=1):
    waves = O.synth_waveforms(len(secs), secs, seed=seed)
    feats, fmask = O.hf_features(waves)
    toks = [O.post_pool_len(int(n)) for n in fmask.sum(-1)]
    ids, am = O.synth_prompt(toks, cfg.text_config.vocab_size, cfg.audio_token_id, seed=seed + 1)
    return feats, fmask, ids, am


def _text_labels(ids, am, audio_token_id):
    """-100 at padding, at audio placeholders and at each row's first real token (whose prediction sits on a pad position)."""
    lab = ids.clone()
    lab[am == 0] = -100
    lab[ids == audio_token_id] = -100
    first = (am == 0).sum(-1)
    lab[torch.arange(ids.shape[0]), first] = -100
    return lab


def _check_against_own_logits(out, shifted, ignore_index=-100, num_items=None):
    """loss / token_losses == F.cross_entropy over the logits the same call returned (fp64), within 1e-5 (1 + |lse|)."""
    V = out.logits.shape[-1]
    lg = out.logits.reshape(-1, V).double()
    lse = torch.logsumexp(lg, -1)
    ref = F.cross_entropy(lg, shifted.reshape(-1), ignore_index=ignore_index, reduction="none")
    tl = out.token_losses.reshape(-1).double()
    assert bool(((tl - ref).abs() <= 1e-5 * (1 + lse.abs())).all()), (tl - ref).abs().max().item()
    n = (shifted != ignore_index).sum().item() if num_items is None else float(num_items)
    ref_loss = ref.sum().item() / n
    assert abs(out.loss.item() - ref_loss) <= 1e-5 * (1 + lse.abs().max().item()), (out.loss.item(), ref_loss)
    assert out.loss.dtype == torch.float32 and out.loss.dim() == 0 and out.loss.is_cuda
    assert out.token_losses.shape == shifted.shape and out.token_losses.dtype == torch.float32


def _shift(lab, ignore_index=-100):
    return F.pad(lab, (0, 1), value=ignore_index)[:, 1:]


@pytest.fixture(scope="module")
def tiny(O):
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model("tiny", seed=0, sharpen=8.0)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    ref16 = O.hf_restore_fp32_rotary(O.hf_model("tiny", seed=0, sharpen=8.0).to("cuda", bf16))
    return ref32, ours, ref16


@pytest.mark.parametrize("secs", [[10.0], [30.0, 4.3, 12.0]])
def test_loss_against_reference_and_own_logits(O, tiny, secs):
    """Single audio and a left-padded batch.  Tolerance against the HF model in bf16: |lse(a) -
    lse(b)| and |a_y - b_y| are both at most max |a - b|, so two models whose logits differ by at most e give losses at most 2 e
    apart.  e is measured here and must itself satisfy the logit bound of tests/test_model_gpu.py (6 % of the logit std
    against fp32, so at most 12 % between the two bf16 paths)."""
    ref32, ours, ref16 = tiny
    cfg = ref32.config
    feats, fmask, ids, am = _inputs(O, cfg, secs)
    lab = _text_labels(ids, am, cfg.audio_token_id)
    kw = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda())
    out = ours(**kw, labels=lab.cuda())
    _check_against_own_logits(out, _shift(lab).cuda())
    lean = ours(**kw, labels=lab.cuda(), logits_to_keep=1)
    assert torch.equal(lean.loss, out.loss) and torch.equal(lean.token_losses, out.token_losses)
    assert torch.equal(lean.logits, ours(**kw, logits_to_keep=1).logits)
    if ids.numel() > 64:
        assert torch.equal(out.logits, ours(**kw).logits), "logits with labels differ from logits without"
    with torch.no_grad():
        r = ref16(**dict(kw, input_features=feats.cuda().to(bf16)), labels=lab.cuda())
        l32 = ref32(input_ids=ids, attention_mask=am, input_features=feats, input_features_mask=fmask).logits
    valid = am.bool().cuda()
    e = (out.logits - r.logits.float())[valid].abs().max().item()
    std = l32[am.bool()].std().item()
    d = abs(out.loss.item() - r.loss.float().item())
    print(f"{secs}: loss ours {out.loss.item():.5f} hf-bf16 {r.loss.float().item():.5f} |diff| {d:.5f}; max logit diff {e:.4f} "
          f"({e / std:.3f} std)")
    assert e <= 0.12 * std
    assert d <= 2 * e + 1e-4


def test_multi_window_multi_audio_prompt_and_inputs_embeds(O, tiny):
    """A 45 s clip (two windows) in one row, two clips in separate spans of another, as tests/test_model_gpu.py builds them."""
    from audio_flamingo_b200 import AF3FeatureExtractor
    from audio_flamingo_b200.processing import audio_token_length, expand_audio_spans, left_pad, split_windows, tokens_per_sample

    ref32, ours, _ = tiny
    cfg = ref32.config
    aid, V = cfg.audio_token_id, cfg.text_config.vocab_size
    clips = O.synth_waveforms(3, [45.0, 6.0, 2.5], seed=21)
    chunks, per = split_windows(clips)
    fo = AF3FeatureExtractor("cuda")(chunks, sampling_rate=16000)
    frames = fo["attention_mask"].sum(-1).cpu().tolist()
    rs = np.random.RandomState(3)
    n0 = tokens_per_sample(frames[:2], [2])[0]
    n1a, n1b = int(audio_token_length(frames[2])), int(audio_token_length(frames[3]))
    t = lambda k: rs.randint(1, V - 2, size=k).tolist()
    row0 = expand_audio_spans(t(4) + [aid] + t(9), aid, [n0])
    row1 = expand_audio_spans(t(3) + [aid] + t(5) + [aid] + t(7), aid, [n1a, n1b])
    ids, am = left_pad([row0, row1])
    kw = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=fo["input_features"], input_features_mask=fo["input_features_mask"])
    lab = _text_labels(ids, am, aid)
    _check_against_own_logits(ours(**kw, labels=lab.cuda()), _shift(lab).cuda())
    row1 = t(40)
    # inputs_embeds: the text-only row from the embedding table
    emb = ours.get_input_embeddings().weight[torch.tensor(row1).cuda()][None]
    lab1 = torch.tensor(row1)[None]
    out = ours(inputs_embeds=emb, labels=lab1.cuda())
    _check_against_own_logits(out, _shift(lab1).cuda())
    out2 = ours(input_ids=lab1.cuda(), labels=lab1)   # host labels, same prompt
    assert torch.equal(out2.loss, out.loss) and torch.equal(out2.token_losses, out.token_losses)


def test_reference_keywords(O, tiny):
    ref32, ours, ref16 = tiny
    cfg = ref32.config
    feats, fmask, ids, am = _inputs(O, cfg, [8.0, 3.0], seed=7)
    lab = _text_labels(ids, am, cfg.audio_token_id)
    kw = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda())
    rkw = dict(kw, input_features=feats.cuda().to(bf16))
    base = ours(**kw, labels=lab.cuda())
    # num_items_in_batch: reduction "sum" divided by it
    for nib in (17, torch.tensor(23)):
        o = ours(**kw, labels=lab.cuda(), num_items_in_batch=nib)
        _check_against_own_logits(o, _shift(lab).cuda(), num_items=int(nib))
        with torch.no_grad():
            r = ref16(**rkw, labels=lab.cuda(), num_items_in_batch=nib).loss.float().item()
        assert abs(o.loss.item() - r) <= abs(r) * 0.05
    # shift_labels as they are
    sl = torch.roll(_shift(lab), 1, dims=1)
    o = ours(**kw, labels=lab.cuda(), shift_labels=sl.cuda())
    _check_against_own_logits(o, sl.cuda())
    o2 = ours(**kw, shift_labels=sl)
    assert torch.equal(o2.loss, o.loss)
    # ignore_index
    lab7 = lab.clone()
    lab7[lab7 == -100] = 7
    o = ours(**kw, labels=lab7.cuda(), ignore_index=7)
    _check_against_own_logits(o, _shift(lab7, 7).cuda(), ignore_index=7)
    # nothing counted: NaN, as the reference
    o = ours(**kw, labels=torch.full_like(lab, -100))
    assert torch.isnan(o.loss) and bool((o.token_losses == 0).all())
    # tuple access as the reference's: (loss, logits, ...)
    assert base.to_tuple()[0] is base.loss and base.to_tuple()[1] is base.logits


def test_continuation_chunk_and_decode_step(O, tiny):
    from audio_flamingo_b200 import AF3Error

    ref32, ours, _ = tiny
    cfg = ref32.config
    feats, fmask, ids, am = _inputs(O, cfg, [5.0], seed=9)
    kw = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda())
    chunk = torch.randint(1, cfg.text_config.vocab_size - 2, (1, 48), generator=torch.Generator().manual_seed(4))
    res = []
    for keep in (0, 1):
        cache = ours(**kw, use_cache=True).past_key_values
        res.append(ours(input_ids=chunk.cuda(), past_key_values=cache, labels=chunk.cuda(), logits_to_keep=keep))
    _check_against_own_logits(res[0], _shift(chunk).cuda())
    assert torch.equal(res[0].loss, res[1].loss) and torch.equal(res[0].token_losses, res[1].token_losses)
    assert res[1].logits.shape[1] == 1
    # the chunk's positions equal those of the whole sequence scored at once (same cache contents, same head)
    full = ours(**dict(kw, input_ids=torch.cat([ids, chunk], 1).cuda(), attention_mask=torch.cat([am, torch.ones_like(chunk)], 1).cuda()),
                labels=torch.cat([torch.full_like(ids, -100), chunk], 1).cuda())
    S = ids.shape[1]
    assert torch.allclose(full.token_losses[:, S:], res[0].token_losses, rtol=0, atol=0.05)
    # the one-token cached step does not take labels
    cache = ours(**kw, use_cache=True).past_key_values
    with pytest.raises(AF3Error):
        ours(input_ids=chunk[:, :1].cuda(), past_key_values=cache, labels=chunk[:, :1].cuda())


def test_fp8_model(O):
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model("tiny", seed=3, sharpen=8.0)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda", quantization="fp8")
    feats, fmask, ids, am = _inputs(O, ref32.config, [10.0, 4.0], seed=5)
    lab = _text_labels(ids, am, ref32.config.audio_token_id)
    kw = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda())
    out = ours(**kw, labels=lab.cuda())
    _check_against_own_logits(out, _shift(lab).cuda())
    assert torch.equal(out.logits, ours(**kw).logits)
    assert torch.equal(ours(**kw, labels=lab.cuda(), logits_to_keep=1).loss, out.loss)


def test_few_token_logits_and_peak_memory(tiny):
    ref32, ours, _ = tiny
    V = ref32.config.text_config.vocab_size
    g = torch.Generator().manual_seed(11)
    # B * S <= 64: logits with labels come from the token-major kernel, without from the few-token one -- one bf16 rounding apart
    ids = torch.randint(1, V - 2, (2, 20), generator=g)
    a = ours(input_ids=ids.cuda(), labels=ids.cuda()).logits
    b = ours(input_ids=ids.cuda()).logits
    assert bool(((a - b).abs() <= 2 ** -6 * b.abs() + 1e-6).all())
    # a shape where B * S * V * 4 bytes dominates: logits_to_keep=1 must not allocate them
    B, S = 8, 2048
    ids = torch.randint(1, V - 2, (B, S), generator=g).cuda()
    peaks = []
    for keep in (1, 0):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = ours(input_ids=ids, labels=ids, logits_to_keep=keep)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del out
    print(f"peak growth: logits_to_keep=1 {peaks[0] / 2**20:.1f} MiB, 0 {peaks[1] / 2**20:.1f} MiB, B*S*V*4 = {B * S * V * 4 / 2**20:.1f} MiB")
    assert peaks[0] < B * S * V * 4 <= peaks[1]


def test_malformed_labels_raise_before_any_launch(tiny):
    from audio_flamingo_b200 import AF3Error, ops

    ref32, ours, _ = tiny
    V = ref32.config.text_config.vocab_size
    ids = torch.randint(1, V - 2, (2, 30), generator=torch.Generator().manual_seed(2))
    ours(input_ids=ids.cuda())   # weights packed
    bads = {"out of range": ids.clone().index_fill_(1, torch.tensor([3]), V), "negative": ids.clone().index_fill_(1, torch.tensor([4]), -2),
            "float": ids.float(), "shape": ids[:, :29], "1-d": ids[0]}
    for name, lab in bads.items():
        n0 = ops.LAUNCHES
        with pytest.raises(ValueError):
            ours(input_ids=ids.cuda(), labels=lab)
        assert ops.LAUNCHES == n0, f"{name}: kernels were launched before the error"
    # device labels out of range: ignored by the kernel, reported at the end of the call
    dev_bad = ids.clone()
    dev_bad[0, 5] = V + 3
    with pytest.raises(ValueError):
        ours(input_ids=ids.cuda(), labels=dev_bad.cuda())
    with pytest.raises(AF3Error):
        ours.generate(input_ids=ids.cuda(), max_new_tokens=2, do_sample=True)
