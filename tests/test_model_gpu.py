"""End-to-end parity on the GPU: the H100 path vs the unmodified HF reference (same seeded synthetic weights) run
(a) in bf16 on the same GPU -- the reference's own PyTorch path in the same dtype -- and (b) in fp32 (oracle
restatement / HF fp32).  Tolerances: logits are bf16-rounded values with |logit| up to ~10 at sharpen=8; bf16 GEMM
chains of 2..32 layers give ~1e-2 relative noise, so we require max|diff| <= 6% of the logit std and compare our
error against the reference-bf16's own error vs fp32 (ours must not be worse than 1.5x)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


@pytest.fixture(scope="module")
def O():
    from oracle import af3_oracle

    return af3_oracle


def _inputs(O, cfg, secs, seed=1):
    waves = O.synth_waveforms(len(secs), secs, seed=seed)
    feats, fmask = O.hf_features(waves)
    toks = [O.post_pool_len(int(n)) for n in fmask.sum(-1)]
    ids, am = O.synth_prompt(toks, cfg.text_config.vocab_size, cfg.audio_token_id, seed=seed + 1)
    return waves, feats, fmask, ids, am


@pytest.mark.parametrize("preset,secs", [("tiny", [10.0, 4.3]), ("tiny", [30.0, 30.0]), ("mid", [30.0, 7.7])])
def test_forward_logits_and_audio_features(O, preset, secs):
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model(preset, seed=0, sharpen=8.0)
    cfg = ref32.config
    waves, feats, fmask, ids, am = _inputs(O, cfg, secs)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    ref16 = O.hf_restore_fp32_rotary(O.hf_model(preset, seed=0, sharpen=8.0).to("cuda", bf16))
    with torch.no_grad():
        l32 = ref32(input_ids=ids, attention_mask=am, input_features=feats, input_features_mask=fmask).logits
        l16 = ref16(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda().to(bf16),
                    input_features_mask=fmask.cuda()).logits.float().cpu()
        a16 = ref16.get_audio_features(feats.cuda().to(bf16), fmask.cuda()).pooler_output.float().cpu()
        a32 = ref32.get_audio_features(feats, fmask).pooler_output
    out = ours(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda())
    lo = out.logits.float().cpu()
    ao = ours.get_audio_features(feats.cuda(), fmask.cuda()).pooler_output.float().cpu()
    assert lo.shape == l32.shape and ao.shape == a32.shape
    valid = am.bool()
    std = l32[valid].std().item()
    e_ours = (lo - l32)[valid].abs().max().item()
    e_ref = (l16 - l32)[valid].abs().max().item()
    ea_ours = (ao - a32).abs().max().item()
    ea_ref = (a16 - a32).abs().max().item()
    print(f"[{preset}] logits: ours-vs-fp32 {e_ours:.4f}, hf-bf16-vs-fp32 {e_ref:.4f}, std {std:.3f}; "
          f"audio: ours {ea_ours:.4f}, hf-bf16 {ea_ref:.4f}, absmax {a32.abs().max().item():.3f}")
    assert e_ours <= max(1.5 * e_ref, 0.06 * std)
    assert ea_ours <= max(1.5 * ea_ref, 0.03 * a32.abs().max().item())
    # last-position argmax agrees with fp32 wherever the fp32 top-2 margin exceeds the observed error
    top2 = l32[:, -1].topk(2).values
    safe = (top2[:, 0] - top2[:, 1]) > 2 * e_ours
    assert torch.equal(lo[:, -1].argmax(-1)[safe], l32[:, -1].argmax(-1)[safe])


@pytest.mark.parametrize("preset,secs,new", [("tiny", [10.0, 4.3, 30.0], 24), ("mid", [30.0, 12.0], 12)])
def test_generate_greedy_ids(O, preset, secs, new):
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model(preset, seed=3, sharpen=8.0)
    cfg = ref32.config
    waves, feats, fmask, ids, am = _inputs(O, cfg, secs, seed=5)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    ref16 = O.hf_restore_fp32_rotary(ref32.to("cuda", bf16))
    with torch.no_grad():
        g_ref = ref16.generate(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda().to(bf16),
                               input_features_mask=fmask.cuda(), max_new_tokens=new, do_sample=False)
    g_graph, lg = ours.generate(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(),
                                input_features_mask=fmask.cuda(), max_new_tokens=new, return_logits=True)
    g_eager = ours.generate(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(),
                            input_features_mask=fmask.cuda(), max_new_tokens=new, use_cuda_graph=False)
    assert g_graph.shape == g_ref.shape == (len(secs), ids.shape[1] + new)
    assert torch.equal(g_graph, g_eager), "CUDA-graph replay must reproduce the eager decode bit for bit"
    S = ids.shape[1]
    same = (g_graph[:, S:] == g_ref[:, S:])
    # greedy ids must be identical to the reference run in the same dtype on the same GPU, except where the
    # reference's own top-2 margin at the first divergent step is within bf16 noise (reported, then asserted small)
    for b in range(len(secs)):
        if bool(same[b].all()):
            continue
        t = int((~same[b]).nonzero()[0])
        top2 = lg[b, t].topk(2).values
        margin = (top2[0] - top2[1]).item()
        print(f"[{preset}] row {b} diverges at step {t}: ours {g_graph[b, S + t].item()} ref {g_ref[b, S + t].item()} margin {margin:.4f}")
        assert margin < 0.05 * lg[b, t].std().item(), "divergence with a decisive margin"
    print(f"[{preset}] greedy ids identical on {int(same.all(1).sum())}/{len(secs)} rows")


def test_feature_extractor_matches_reference(O):
    from audio_flamingo_b200 import AF3FeatureExtractor

    waves = O.synth_waveforms(3, [30.0, 10.0, 0.5], seed=9)
    feats, fmask = O.hf_features(waves)
    fe = AF3FeatureExtractor("cuda")
    out = fe(waves, sampling_rate=16000)
    assert torch.equal(out["attention_mask"].cpu().long(), fmask.long())
    err = (out["input_features"].cpu() - feats).abs().max().item()
    print("logmel vs WhisperFeatureExtractor max abs err", err)
    assert err < 1e-4


def test_multi_window_and_multi_audio_prompts(O):
    """SURVEY 8-f rows 1-2: a 45 s clip (2 windows) and a prompt with two separate <sound> spans; logits vs the HF
    reference in bf16 on the same GPU and vs fp32 (the model side of the reference accepts any placeholder layout)."""
    from audio_flamingo_b200 import AF3FeatureExtractor, AudioFlamingo3ForConditionalGeneration
    from audio_flamingo_b200.processing import audio_token_length, expand_audio_spans, left_pad, split_windows, tokens_per_sample

    ref32 = O.hf_model("tiny", seed=0, sharpen=8.0)
    cfg = ref32.config
    aid, V = cfg.audio_token_id, cfg.text_config.vocab_size
    clips = O.synth_waveforms(3, [45.0, 6.0, 2.5], seed=21)
    chunks, per = split_windows(clips)                      # [30 s, 15 s], [6 s], [2.5 s]
    assert per == [2, 1, 1]
    fe = AF3FeatureExtractor("cuda")
    fo = fe(chunks, sampling_rate=16000)
    frames = fo["attention_mask"].sum(-1).cpu().tolist()
    rs = np.random.RandomState(3)
    # sample 0: one <sound> for its two windows (processor semantics: summed frames); sample 1: two clips, two spans
    n0 = tokens_per_sample(frames[:2], [2])[0]
    n1a, n1b = int(audio_token_length(frames[2])), int(audio_token_length(frames[3]))
    t = lambda n: rs.randint(1, V - 2, size=n).tolist()
    row0 = expand_audio_spans(t(4) + [aid] + t(9), aid, [n0])
    row1 = expand_audio_spans(t(3) + [aid] + t(5) + [aid] + t(7), aid, [n1a, n1b])
    ids, am = left_pad([row0, row1])
    feats_ref, fmask_ref = O.hf_features(chunks)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    with torch.no_grad():
        l32 = ref32(input_ids=ids, attention_mask=am, input_features=feats_ref, input_features_mask=fmask_ref).logits
    lo = ours(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=fo["input_features"],
              input_features_mask=fo["input_features_mask"]).logits.float().cpu()
    v = am.bool()
    assert (lo - l32)[v].abs().max().item() < 0.06 * l32[v].std().item()
    # a prompt whose placeholder count does not match the features must raise like the reference's masked_scatter
    bad = ids.clone()
    bad[0, -1] = aid
    with pytest.raises(ValueError):
        ours(input_ids=bad.cuda(), attention_mask=am.cuda(), input_features=fo["input_features"], input_features_mask=fo["input_features_mask"])


def test_pdl_decode_is_bit_identical(O, monkeypatch):
    """Programmatic dependent launch only reorders prologues / weight prefetch: ids and logits must not change."""
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model("mid", seed=4, sharpen=8.0)
    cfg = ref32.config
    waves, feats, fmask, ids, am = _inputs(O, cfg, [30.0, 9.0], seed=7)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    kw = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda(),
              max_new_tokens=10, return_logits=True)
    monkeypatch.setenv("AF3_PDL", "1")
    g1, l1 = ours.generate(**kw)
    g1e, l1e = ours.generate(use_cuda_graph=False, **kw)
    monkeypatch.setenv("AF3_PDL", "0")
    g0, l0 = ours.generate(**kw)
    assert torch.equal(g1, g0) and torch.equal(l1, l0)
    assert torch.equal(g1e, g0) and torch.equal(l1e, l0)


def test_music_flamingo_rotary_time_embedding(O):
    """SURVEY 8-f.3: Music Flamingo = AF3 + rotary time embedding on the audio-tower output.  Audio features and logits
    vs the HF MusicFlamingoForConditionalGeneration (same seeded weights) in fp32 and in bf16 on the same GPU; a 45 s
    clip exercises the window axis (window index 1 -> non-zero window rotation)."""
    from transformers import MusicFlamingoConfig, MusicFlamingoForConditionalGeneration as HFMusic

    from audio_flamingo_b200 import AF3FeatureExtractor, MusicFlamingoForConditionalGeneration
    from audio_flamingo_b200.processing import expand_audio_spans, left_pad, split_windows, tokens_per_sample

    p = O.TINY
    text = dict(p["text"])
    theta = text.pop("rope_theta")
    cfg = MusicFlamingoConfig(audio_config=dict(p["audio"], model_type="musicflamingo_encoder"),
                              text_config=dict(text, rope_parameters={"rope_type": "default", "rope_theta": theta}),
                              audio_token_id=p["audio_token_id"], audio_bos_token_id=2045, audio_eos_token_id=2046,
                              rope_parameters={"rope_type": "default", "rope_theta": 1200, "partial_rotary_factor": 0.2})
    assert cfg.max_position_embeddings == 1200
    torch.manual_seed(11)
    ref32 = HFMusic(cfg).eval()
    with torch.no_grad():
        ref32.language_model.lm_head.weight.mul_(8.0)
    clips = O.synth_waveforms(2, [45.0, 8.0], seed=31)
    chunks, per = split_windows(clips)
    fe = AF3FeatureExtractor("cuda")
    fo = fe(chunks, sampling_rate=16000)
    frames = fo["attention_mask"].sum(-1).cpu().tolist()
    n0, n1 = tokens_per_sample(frames, per)
    rs = np.random.RandomState(5)
    aid, V = cfg.audio_token_id, cfg.text_config.vocab_size
    t = lambda n: rs.randint(1, 2000, size=n).tolist()
    ids, am = left_pad([expand_audio_spans(t(4) + [aid] + t(6), aid, [n0]), expand_audio_spans(t(3) + [aid] + t(9), aid, [n1])])
    feats_ref, fmask_ref = O.hf_features(chunks)
    ours = MusicFlamingoForConditionalGeneration.from_reference(ref32, device="cuda")
    with torch.no_grad():
        a32 = ref32.get_audio_features(feats_ref, fmask_ref, input_ids=ids)
        l32 = ref32(input_ids=ids, attention_mask=am, input_features=feats_ref, input_features_mask=fmask_ref).logits
    ao = ours.get_audio_features(fo["input_features"], fo["input_features_mask"], input_ids=ids.cuda())
    lo = ours(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=fo["input_features"],
              input_features_mask=fo["input_features_mask"]).logits.float().cpu()
    ea = (ao.pooler_output.float().cpu() - a32.pooler_output).abs().max().item()
    assert ea < 0.03 * a32.pooler_output.abs().max().item(), ea
    v = am.bool()
    assert (lo - l32)[v].abs().max().item() < 0.06 * l32[v].std().item()
    # the rotation must actually matter: AF3 (no rotation) on the same weights differs visibly
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    plain = AudioFlamingo3ForConditionalGeneration(cfg)
    plain.load_reference_state_dict(ref32.state_dict(), device="cuda")
    ap = plain.get_audio_features(fo["input_features"], fo["input_features_mask"]).pooler_output.float().cpu()
    assert (ap - a32.pooler_output).abs().max().item() > 5 * ea


def test_long_audio_five_windows(O):
    """SURVEY 8-f.2: long audio = more 30 s windows per sample (here 140 s -> 5 windows -> 3 502 audio tokens in one prompt);
    prefill attention runs 28 query tiles x up to 28 key tiles per head with left padding on the shorter row."""
    from audio_flamingo_b200 import AF3FeatureExtractor, AudioFlamingo3ForConditionalGeneration
    from audio_flamingo_b200.processing import expand_audio_spans, left_pad, split_windows, tokens_per_sample

    ref32 = O.hf_model("tiny", seed=0, sharpen=8.0)
    cfg = ref32.config
    aid, V = cfg.audio_token_id, cfg.text_config.vocab_size
    clips = O.synth_waveforms(2, [140.0, 33.0], seed=41)
    chunks, per = split_windows(clips)
    assert per == [5, 2]
    fe = AF3FeatureExtractor("cuda")
    fo = fe(chunks, sampling_rate=16000)
    n0, n1 = tokens_per_sample(fo["attention_mask"].sum(-1).cpu().tolist(), per)
    assert n0 == 3500 and n1 == 825
    rs = np.random.RandomState(7)
    t = lambda n: rs.randint(1, V - 2, size=n).tolist()
    ids, am = left_pad([expand_audio_spans(t(5) + [aid] + t(20), aid, [n0]), expand_audio_spans(t(5) + [aid] + t(20), aid, [n1])])
    feats_ref, fmask_ref = O.hf_features(chunks)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    with torch.no_grad():
        l32 = ref32(input_ids=ids, attention_mask=am, input_features=feats_ref, input_features_mask=fmask_ref, logits_to_keep=1).logits
        g_ref = ref32.generate(input_ids=ids, attention_mask=am, input_features=feats_ref, input_features_mask=fmask_ref,
                               max_new_tokens=4, do_sample=False)
    out = ours(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=fo["input_features"],
               input_features_mask=fo["input_features_mask"], logits_to_keep=1)
    lo = out.logits.float().cpu()
    assert lo.shape == l32.shape
    assert (lo - l32).abs().max().item() < 0.08 * l32.std().item()
    g = ours.generate(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=fo["input_features"],
                      input_features_mask=fo["input_features_mask"], max_new_tokens=4).cpu()
    top2 = l32[:, -1].topk(2).values
    if bool(((top2[:, 0] - top2[:, 1]) > 0.2).all()):
        assert torch.equal(g[:, :ids.shape[1] + 1], g_ref[:, :ids.shape[1] + 1])


def test_generate_reuses_decode_graph_across_calls(O):
    """generate() keeps the KV cache + captured decode graph of the last (batch, max length) shape.  A second prompt of the same
    shape must replay that graph (no re-capture) and give exactly what a fresh model instance gives; the first prompt run again
    must reproduce itself bit for bit (nothing of prompt B survives in the reused cache); another shape rebuilds the state."""
    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    ref32 = O.hf_model("mid", seed=6, sharpen=8.0)
    cfg = ref32.config
    _, fa, ma, ids_a, am_a = _inputs(O, cfg, [30.0, 9.0], seed=11)
    _, fb, mb, ids_b, am_b = _inputs(O, cfg, [30.0, 9.0], seed=12)   # same clip lengths -> same prompt shape, other content
    assert ids_a.shape == ids_b.shape and not torch.equal(ids_a, ids_b)
    kw = lambda f, m, i, a, n=10: dict(input_ids=i.cuda(), attention_mask=a.cuda(), input_features=f.cuda(),  # noqa: E731
                                        input_features_mask=m.cuda(), max_new_tokens=n, return_logits=True)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    fresh = AudioFlamingo3ForConditionalGeneration.from_reference(ref32, device="cuda")
    ga1, la1 = ours.generate(**kw(fa, ma, ids_a, am_a))
    st = ours._decode_state
    cap = lambda n: -(-n // 256) * 256  # noqa: E731  (cache capacity bucket)
    assert st is not None and st["key"][:2] == (2, cap(ids_a.shape[1] + 10))
    gb, lb = ours.generate(**kw(fb, mb, ids_b, am_b))
    assert ours._decode_state is st, "same shape: cache and graph must be reused, not rebuilt"
    gb_fresh, lb_fresh = fresh.generate(**kw(fb, mb, ids_b, am_b))
    assert torch.equal(gb, gb_fresh) and torch.equal(lb, lb_fresh)
    ga2, la2 = ours.generate(**kw(fa, ma, ids_a, am_a))
    assert torch.equal(ga1, ga2) and torch.equal(la1, la2)
    # another prompt length / token budget inside the same capacity bucket: still the same graph
    gc_, _ = ours.generate(**kw(fa, ma, ids_a, am_a, n=6))
    assert cap(ids_a.shape[1] + 6) == cap(ids_a.shape[1] + 10) and ours._decode_state is st
    assert torch.equal(gc_, ga1[:, : ids_a.shape[1] + 6])
    _, fs, ms, ids_s, am_s = _inputs(O, cfg, [30.0, 9.5], seed=11)      # 9.5 s instead of 9 s: a longer left-padded row
    if cap(ids_s.shape[1] + 10) == cap(ids_a.shape[1] + 10) and ids_s.shape != ids_a.shape:
        gs, ls = ours.generate(**kw(fs, ms, ids_s, am_s))
        assert ours._decode_state is st
        gs_fresh, ls_fresh = fresh.generate(**kw(fs, ms, ids_s, am_s))
        assert torch.equal(gs, gs_fresh) and torch.equal(ls, ls_fresh)
    # a different capacity bucket rebuilds the state
    gd, _ = ours.generate(**kw(fa, ma, ids_a, am_a, n=10 + 256))
    assert ours._decode_state is not st and ours._decode_state["key"][1] == cap(ids_a.shape[1] + 266)
    assert torch.equal(gd[:, : ids_a.shape[1] + 10], ga1)
    # new weights into the same instance: the kept graph points at the old packed weights and must not be replayed
    ref_w = O.hf_model("mid", seed=7, sharpen=8.0)
    gw_fresh, lw_fresh = AudioFlamingo3ForConditionalGeneration.from_reference(ref_w, device="cuda").generate(**kw(fa, ma, ids_a, am_a))
    ours.generate(**kw(fa, ma, ids_a, am_a))                      # leaves a live state for this shape
    ours.load_reference_state_dict({k: v for k, v in ref_w.state_dict().items()})
    assert ours._decode_state is None
    gw, lw = ours.generate(**kw(fa, ma, ids_a, am_a))
    assert torch.equal(gw, gw_fresh) and torch.equal(lw, lw_fresh)
    assert not torch.equal(lw, la1)
    ours.release_decode_state()
    assert ours._decode_state is None
