"""Parity at BASELINE geometry (VERDICT r01 "Next round" item 1a): the full AF3-7B stack -- 32 AF-Whisper layers + 28 Qwen2.5-7B
layers at full width, the configuration bench.py times -- against the unmodified HF reference running in bf16 ON THE SAME GPU
(and in fp32 on a subset), on a ragged batch of 8 clips (3.1 ... 30 s), 32 greedy tokens.

Weights: the reference's default-init family (N(0, 0.02) matrices / embeddings, zero biases, unit norm gains) drawn directly on the
GPU from a seeded generator, lm_head sharpened x8 (documented in oracle/af3_oracle.py: with N(0, 0.02) logits the top-1 / top-2
margins are comparable to bf16 noise and greedy parity would test nothing).  No checkpoint exists offline.

What is asserted
  * teacher-forced: at every one of the 32 steps of every row (ours fed the reference's own tokens through forward(past_key_values=)),
    our argmax equals the reference's token wherever the REFERENCE's top-2 margin exceeds 2x the observed logit error of that step;
  * free-running generate(): rows identical to the reference's ids up to their first divergence, and every first divergence sits on
    a step whose reference margin is within 2x the observed error (a bf16 near-tie), never on a decisive one;
  * our logits are not further from HF-fp32 than 1.5x what HF-bf16 itself is (subset of 2 rows, prefill logits).
What is recorded: {rows, identical, first_divergence, margin, ...}, printed as one JSON line (visible with pytest -s).
"""
import gc
import json
import os
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
ROOT = Path(__file__).resolve().parent.parent
LOUD = (64, 4.0)   # (number of token ids, row scale) of the peaked LM head; None = flat head (the round-2 first run, see below)


def _hf_model_on_gpu(O, cfg, seed, sharpen, loud=None):
    """Unmodified HF AudioFlamingo3ForConditionalGeneration, bf16, weights drawn on the GPU (a CPU init of 8.3 B parameters takes
    minutes and 33 GB)."""
    from transformers import AudioFlamingo3ForConditionalGeneration

    with torch.device("meta"):
        m = AudioFlamingo3ForConditionalGeneration(cfg)
    m = m.to_empty(device="cuda").to(bf16).eval()
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith("bias"):
                p.zero_()
            elif "norm" in name and name.endswith("weight"):
                p.fill_(1.0)
            else:
                p.normal_(0.0, 0.02, generator=g)
        m.language_model.lm_head.weight.mul_(sharpen)
        # a PEAKED output distribution, as a trained LM has: the rows of `loud[0]` token ids are scaled by loud[1].  With all
        # 152 064 rows alike the logits are i.i.d. Gaussians whose typical top-2 gap (1.25 at sharpen 8) is BELOW the bf16 noise of the
        # 60-layer stack (the max |logit diff| between two bf16 implementations, or between HF-bf16 and HF-fp32, is larger than that),
        # so greedy ids of two correct bf16 implementations -- or of HF with itself in fp32 -- differ within 32 steps on every
        # row and token parity tests nothing.  The gap among K candidates relative to the noise on them scales like
        # 1 / (eps * 2 ln K): K = 64 loud ids make most steps decisive without touching the geometry.
        if loud is not None:
            m.language_model.lm_head.weight[: loud[0]].mul_(loud[1])
    # rotary inv_freq is a non-persistent buffer: recompute after to_empty -- on the CPU, in fp32, as the reference's normal
    # loading path leaves it (from_pretrained(dtype=bf16) casts parameters, not this buffer; a blanket model.to(bf16) would round it)
    O.hf_restore_fp32_rotary(m)
    m.generation_config.pad_token_id = 0
    m.generation_config.eos_token_id = None
    return m


def test_af3_7b_full_depth_parity_vs_hf_bf16_on_the_same_gpu():
    from oracle import af3_oracle as O

    from audio_flamingo_b200 import AudioFlamingo3ForConditionalGeneration

    # peak: two bf16 copies of AF3-7B (HF's and ours, 2 x 16.6 GB) plus caches and logits; ours is freed before HF's copy is
    # converted to fp32 in place (33 GB)
    free_gb = torch.cuda.mem_get_info()[0] / 2 ** 30
    if free_gb < 45:
        pytest.skip(f"needs ~45 GB of HBM (two bf16 copies of AF3-7B, later one fp32 copy), {free_gb:.0f} GB free")
    cfg = O.hf_config("af3-7b")
    ref16 = _hf_model_on_gpu(O, cfg, seed=0, sharpen=8.0, loud=LOUD)
    ours = AudioFlamingo3ForConditionalGeneration.from_reference(ref16, device="cuda")
    secs = [30.0, 30.0, 22.5, 17.3, 12.0, 9.1, 5.5, 3.1]
    B, NEW = len(secs), 32
    waves = O.synth_waveforms(B, secs, seed=101)
    feats, fmask = O.hf_features(waves)
    toks = [O.post_pool_len(int(n)) for n in fmask.sum(-1)]
    ids, am = O.synth_prompt(toks, cfg.text_config.vocab_size, cfg.audio_token_id, seed=102)
    S = ids.shape[1]
    kw_ref = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda().to(bf16), input_features_mask=fmask.cuda())
    kw_our = dict(input_ids=ids.cuda(), attention_mask=am.cuda(), input_features=feats.cuda(), input_features_mask=fmask.cuda())

    # ---- reference: free-running greedy ids + the logits it decided on at every step
    with torch.no_grad():
        gen = ref16.generate(**kw_ref, max_new_tokens=NEW, do_sample=False, return_dict_in_generate=True, output_logits=True)
    g_ref = gen.sequences
    l_ref = torch.stack([x.float() for x in gen.logits], 1)            # [B, NEW, V] raw (pre-processor) logits
    assert g_ref.shape == (B, S + NEW)

    # ---- ours, free running (CUDA graph path, the one bench.py times)
    g_our, l_our = ours.generate(**kw_our, max_new_tokens=NEW, return_logits=True)
    assert g_our.shape == g_ref.shape

    # ---- ours, teacher forced with the reference's tokens (prefill, then cached single-token forward() steps)
    o = ours(**kw_our, use_cache=True, logits_to_keep=1, reserve_tokens=NEW)
    tf = [o.logits[:, -1].float()]
    cache = o.past_key_values
    for t in range(NEW - 1):
        o = ours(input_ids=g_ref[:, S + t: S + t + 1], past_key_values=cache)
        tf.append(o.logits[:, -1].float())
    l_tf = torch.stack(tf, 1)                                            # [B, NEW, V], same history as the reference at every step

    top2 = l_ref.topk(2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1])                               # reference's own top-2 margin, [B, NEW]
    err_tf = (l_tf - l_ref).abs().amax(-1)                               # observed logit error per (row, step)
    agree_tf = l_tf.argmax(-1) == g_ref[:, S:]
    decisive = margin > 2 * err_tf
    n_decisive = int(decisive.sum())
    wrong_decisive = int((decisive & ~agree_tf).sum())

    rows = []
    same = g_our[:, S:] == g_ref[:, S:]
    for b in range(B):
        rec = {"row": b, "clip_seconds": secs[b], "audio_tokens": toks[b], "identical": bool(same[b].all()),
               "teacher_forced_agree": int(agree_tf[b].sum()), "teacher_forced_steps": NEW,
               "min_margin": float(margin[b].min()), "max_logit_err_teacher_forced": float(err_tf[b].max())}
        if not rec["identical"]:
            t = int((~same[b]).nonzero()[0])
            e = float((l_our[b, t] - l_ref[b, t]).abs().max())          # same history up to t on both sides
            rec.update({"first_divergence": t, "margin_at_divergence": float(margin[b, t]), "logit_err_at_divergence": e,
                        "ours": int(g_our[b, S + t]), "reference": int(g_ref[b, S + t]),
                        "decisive": bool(margin[b, t] > 2 * e)})
        rows.append(rec)

    # ---- fp32 subset: is our bf16 path as close to fp32 as the reference's own bf16 path is?  (rows 0 and 7: 30 s and 3.1 s)
    #      our model, its cache and decode graph are released first: the fp32 copy of the reference needs the room
    del ours, o, cache
    gc.collect()
    torch.cuda.empty_cache()
    sub = [0, B - 1]
    ref32 = ref16.float()   # in place: bf16 values exactly representable, same weights
    O.hf_restore_fp32_rotary(ref32)
    with torch.no_grad():
        l32 = ref32(input_ids=ids[sub].cuda(), attention_mask=am[sub].cuda(), input_features=feats[sub].cuda(),
                    input_features_mask=fmask[sub].cuda(), logits_to_keep=1).logits[:, -1].float()
    e_ours32 = float((l_tf[sub, 0] - l32).abs().max())
    e_ref32 = float((l_ref[sub, 0] - l32).abs().max())
    std = float(l32.std())

    report = {
        "what": "AF3-7B full depth (32 encoder + 28 decoder layers, full width), ours vs HF transformers bf16 on the same GPU",
        "weights": "seeded N(0,0.02) default-init family drawn on the GPU, lm_head x8 (sharpen), zero biases, unit norm gains; "
                   + (f"LM-head rows of the first {LOUD[0]} ids x{LOUD[1]} (peaked output distribution)" if LOUD else "flat LM head"),
        "batch": B, "clip_seconds": secs, "prompt_len": S, "new_tokens": NEW,
        "rows_identical_free_running": int(same.all(1).sum()), "rows": rows,
        "teacher_forced": {"steps": B * NEW, "argmax_agree": int(agree_tf.sum()), "decisive_steps": n_decisive,
                           "decisive_steps_wrong": wrong_decisive, "rule": "decisive = reference top-2 margin > 2 x observed max |logit diff| of that step",
                           "median_margin": float(margin.median()), "median_logit_err": float(err_tf.median()),
                           "max_logit_err": float(err_tf.max()), "logit_std": float(l_ref.std())},
        "fp32_subset": {"rows": sub, "ours_vs_fp32_max_abs": e_ours32, "hf_bf16_vs_fp32_max_abs": e_ref32, "fp32_logit_std": std},
        "versions": {"torch": torch.__version__, "transformers": __import__("transformers").__version__,
                     "gpu": torch.cuda.get_device_name(0)},
    }
    print(json.dumps(report))

    assert wrong_decisive == 0, f"{wrong_decisive} of {n_decisive} decisive steps disagree with the reference"
    # Gaussian logits over 152 064 ids put the typical top-2 gap at ~0.2 logit std, bf16 noise over 60 layers at ~0.1: a sizeable
    # share of steps is NOT decisive under the 2x rule and says nothing either way; the count is recorded, a floor keeps the test honest
    assert n_decisive >= B * NEW // 4, f"only {n_decisive} of {B * NEW} steps are decisive: the comparison is close to vacuous"
    for r in rows:
        assert r["identical"] or not r["decisive"], f"free-running divergence on a decisive step: {r}"
    assert e_ours32 <= max(1.5 * e_ref32, 0.06 * std), (e_ours32, e_ref32, std)
